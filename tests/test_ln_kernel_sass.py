"""CPU: the LN GEMMs reach their tile buffer and row statistics with shared-memory instructions.

gemm_ln_kernel's epilogue passes read and write the 116 KB tile buffer in shared memory.  When the kernel's view of the
dynamic shared memory loses its state space (aligning the pointer through an integer does that), every one of those accesses
compiles to a generic LD / ST, which is slower and orders later loads behind each store.  Reads the built library's SASS;
skips when the library or cuobjdump is not there."""
import os
import re
import shutil
import subprocess

import pytest

from layoutdm_b200 import _lib


def _cuobjdump():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    for c in (os.path.join(os.path.dirname(nvcc), "cuobjdump"), shutil.which("cuobjdump")):
        if c and os.path.isfile(c) and os.access(c, os.X_OK):
            return c
    return None


def _sass_by_function(lib):
    out = subprocess.run([_cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


# the opcode of a SASS line "/*0a30*/  @!P0 LD.E.64 R4, desc[UR4][R2.64] ;"
_OPCODE = re.compile(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)(?:\.[A-Z0-9_.]+)?\s")


def test_gemm_ln_kernel_has_no_generic_loads_or_stores():
    if not os.path.isfile(_lib.LIB_PATH):
        pytest.skip("the library is not built")
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    funcs = {n: body for n, body in _sass_by_function(_lib.LIB_PATH).items() if "gemm_ln_kernel" in n}
    assert funcs, "no gemm_ln_kernel instantiation in the library"
    generic = {}
    for name, body in funcs.items():
        ops = [m.group(1) for m in map(_OPCODE.match, body) if m]
        assert "EXIT" in ops, f"{name}: no instruction parsed; did the SASS format change?"
        n = sum(op in ("LD", "ST") for op in ops)
        if n:
            generic[name] = n
    assert not generic, f"generic LD / ST (instruction count per kernel): {generic}"
