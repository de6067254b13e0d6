"""ctypes binding of the C ABI in include/ldm_b200.h.  There is NO CPU fallback: importing works anywhere, but
`load()` raises if the in-tree CUDA library has not been built (`python -c "import __graft_entry__ as g; g.build()"`)."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libldm_b200.so")

LDM_OK, LDM_ERR_INVALID, LDM_ERR_CUDA, LDM_ERR_UNSUPPORTED = 0, -1, -2, -3
PROFILE_CATEGORIES = ("embed_adaln", "qkv_gemm", "attention", "outproj_gemm", "ff1_gemm", "ff2_gemm", "head_gemm", "posterior_sample", "misc")
SAMPLING_MODES = {"deterministic": 0, "random": 1, "top_k": 2, "top_p": 3, "gumbel": 4}
# LdmModelDesc.operand_dtype: tensor-core operands fp16, bf16, or bf16 (hi, lo) pairs ("bf16x3": three MMAs per product,
# fp32-class operand precision)
OPERAND_DTYPES = {"fp16": 0, "bf16": 1, "bf16x3": 2}


# LdmModelDesc.bbox_vocab / var_order: the tokenizer's shared_bbox_vocab and var_order (helpers/layout_tokenizer.py:16-20)
BBOX_VOCABS = {"x-y-w-h": 0, "xywh": 1}
VAR_ORDERS = {"c-x-y-w-h": 0, "c-w-h-x-y": 1}
# LdmModelDesc.norm1_kind / activation: the denoiser block's timestep_type and activation (transformer_utils.py:17-31,103-170).
# The keys are every timestep_type the reference can sample with; it cannot with the *_mlp types (their MLP gets long timesteps)
NORM1_KINDS = {None: 0, "adalayernorm": 0, "adalayernorm_abs": 0, "adainnorm": 1, "adainnorm_abs": 1}
ACTIVATIONS = {"relu": 0, "gelu": 1, "gelu2": 2}


class LdmModelDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_cat", "n_bins", "n_elem", "n_attr", "d_model", "n_heads", "d_ff", "n_layers",
                                         "num_timesteps", "q_type", "operand_dtype", "device")] + \
               [(n, C.c_double) for n in ("att_1", "att_T", "ctt_1", "ctt_T")] + \
               [(n, C.c_int32) for n in ("norm1_kind", "activation", "bbox_vocab", "var_order")]


_W_FIELDS = ("cat_emb", "pos_table", "in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "linear1_w", "linear1_b",
             "linear2_w", "linear2_b", "norm1_emb", "norm1_w", "norm1_b", "norm2_w", "norm2_b", "head_ln_w", "head_ln_b", "head_w")


class LdmWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _W_FIELDS]


class LdmCond(C.Structure):
    _fields_ = [("seq", C.c_void_p), ("mask", C.c_void_p), ("seq_orig", C.c_void_p), ("refine_table", C.c_void_p),
                ("pad_disable", C.c_int32),
                ("rel_adj", C.c_void_p), ("rel_centers", C.c_void_p), ("rel_lambda", C.c_float), ("rel_num_update", C.c_int32),
                ("rel_batch_total", C.c_int32)]


class LdmSampling(C.Structure):
    _fields_ = [("mode", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float), ("top_k", C.c_int32)]


# LdmNoise.kind: the project's Philox contract, or the numbers torch's CUDA generator would give the reference's draw
NOISE_KINDS = {"contract": 0, "torch": 1}


class LdmNoise(C.Structure):
    _fields_ = [("kind", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64), ("total_layouts", C.c_int64)]


# every symbol include/ldm_b200.h declares: (restype, argtypes)
SIGNATURES = {
    "ldm_create": (C.c_int, [C.POINTER(LdmModelDesc), C.POINTER(LdmWeights), C.POINTER(C.c_void_p)]),
    "ldm_destroy": (C.c_int, [C.c_void_p]),
    "ldm_load_weights": (C.c_int, [C.c_void_p, C.POINTER(LdmWeights), C.c_void_p]),
    "ldm_step": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(LdmCond), C.POINTER(LdmSampling),
                           C.c_uint64, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_sample_loop": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(LdmCond),
                                  C.POINTER(LdmSampling), C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_step_noise": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(LdmCond), C.POINTER(LdmSampling),
                                 C.POINTER(LdmNoise), C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "ldm_sample_loop_noise": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(LdmCond),
                                        C.POINTER(LdmSampling), C.POINTER(LdmNoise), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "ldm_noise_advance": (C.c_int64, [C.c_void_p, C.c_int64, C.POINTER(LdmSampling), C.c_int32]),
    "ldm_sample_host": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(LdmSampling), C.c_uint64, C.c_int64, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "ldm_q_sample": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p]),
    "ldm_decode": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_make_cond": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p]),
    "ldm_predict_start": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_q_posterior": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_q_pred": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_q_pred_one_timestep": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_gumbel_argmax": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p]),
    "ldm_vb_terms": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ldm_launch_count": (C.c_int64, [C.c_void_p]),
    "ldm_num_classes": (C.c_int32, [C.c_void_p]),
    "ldm_seq_len": (C.c_int32, [C.c_void_p]),
    "ldm_get_schedule": (C.c_int64, [C.c_void_p, C.c_void_p, C.c_int64]),
    "ldm_get_adaln_table": (C.c_int64, [C.c_void_p, C.c_void_p, C.c_int64]),
    "ldm_profile_begin": (C.c_int, [C.c_void_p]),
    "ldm_profile_end": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.c_int32]),
    "ldm_debug_set_stop_after": (C.c_int, [C.c_void_p, C.c_int32]),
    "ldm_debug_torch_noise": (C.c_int, [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p]),
    "ldm_debug_read": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_int32]),
    "ldm_last_error": (C.c_char_p, []),
    "ldm_version": (C.c_char_p, []),
}

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built (run __graft_entry__.build()). "
                "layoutdm_b200 has no CPU or PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the library does not export a declared symbol
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


class LdmError(RuntimeError):
    pass


def check(rc: int):
    """status code -> the exception type the reference raises for the same mistake (SURVEY.md 8b)"""
    if rc == LDM_OK:
        return
    msg = load().ldm_last_error().decode()
    if rc == LDM_ERR_INVALID:
        if "NotImplementedError" in msg:
            raise NotImplementedError(msg)
        raise AssertionError(msg)
    raise LdmError(f"ldm_b200 error {rc}: {msg}")
