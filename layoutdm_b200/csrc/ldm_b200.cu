// C-ABI implementation (include/ldm_b200.h): handle, weight repacking, TMA descriptors and the per-step launch
// sequence of the LayoutDM denoising loop.  CUDA runtime only (the driver's cuTensorMapEncodeTiled is fetched
// through cudaGetDriverEntryPoint, so there is no link-time libcuda dependency) and no torch types.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../include/ldm_b200.h"
#include "attention.cuh"
#include "common.cuh"
#include "embed.cuh"
#include "gemm_tc.cuh"
#include "posterior_sample.cuh"
#include "relation.cuh"

using namespace ldm;

namespace {

thread_local char g_err[512] = "";
int fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
  return code;
}
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess) return fail(LDM_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

constexpr int kMaxLayers = 16;
constexpr int kHeadPad = 64;        // per-head width after padding 58 -> 64
constexpr int kQkvN = 3 * 8 * kHeadPad;   // 1536
constexpr int kAttN = 8 * kHeadPad;        // 512: attention output, heads padded like Q/K/V
constexpr int kMaxLayouts = 32767;  // layouts per call
constexpr int kLogitLd = 160;       // padded logits row (C <= 160)
constexpr int kDModel = 464;        // the kernels are laid out for the paper's backbone: d = 464 (LN tiles 224 + 240), ff = 4 d
// GEMM instantiations: <warpgroup tile width, row warpgroups, ring stages, epilogue, operand mode>
// QKV / FF1: fp16 / bf16: gemm_rowblock_kernel (resident A rows, 128-column tiles); the split mode: 128 x 256 tiles of
// gemm_tc_kernel, 4 ring stages
constexpr int kPlainBN = 256, kPlainStages = 4;
constexpr int kRbCols = RbSmem::kCols;
static_assert(kDModel <= RbSmem::kAKb * RbSmem::kKB && kAttN % kRbCols == 0 && kQkvN % 64 == 0 && 4 * kDModel % 64 == 0,
              "row-block GEMM shapes: K fits the resident A, Q tiles are whole tiles, N is whole 64-column store blocks");
constexpr int kHeadBN = 160, kHeadStages = 4;     // vocabulary head: 128 x 160 (the padded logits row)
// out-projection / FF2 (LayerNorm in the epilogue).  fp16 / bf16: gemm_ln_kernel (persistent CTA pairs, each pair one 128-row
// block, each CTA 232 of its 464 columns; epilogue warps, 32-element k-blocks: K = 512 and 1856 have no tail); the split mode:
// the fragment-epilogue kernel below, 64 x 464 tiles
constexpr int kLnBN = 232, kLnStages = 3;
constexpr int kLnSplitRows = 64;   // A box rows of the split mode's LN GEMMs (the one-plane kernel's: LnSmem<>::kRows)
// ring stages of gemm_ln_kernel: FF2 (K = 1856) waits on its operand feed and takes the most that fit; the out-projection
// (K = 512) waits on its epilogue, which measured faster beside the smaller shared-memory footprint of 3 stages (DESIGN §4)
constexpr int kLnOutStages = 3, kLnFf2Stages = 4;
using LnOut = LnSmem<kLnOutStages>;
using LnFf2 = LnSmem<kLnFf2Stages>;
// k-block of the LN GEMMs' operands (the TMA box columns) in every mode: the persistent kernel's, which is the split mode's
constexpr int kLnKB = LnFf2::R::kKB;
static_assert(LnOut::R::kKB == kLnKB && LnFf2::kCols == kLnBN && LnFf2::kPairCols == kDModel && kAttN % kLnKB == 0 &&
              4 * kDModel % kLnKB == 0 && gemm_kb(true) == kLnKB, "LN GEMM shapes");
template <int EPI, int MODE> constexpr auto kGemmPlainSplit = gemm_tc_kernel<kPlainBN, 2, kPlainStages, EPI, MODE>;
template <int MODE> constexpr auto kGemmHead = gemm_tc_kernel<kHeadBN, 2, kHeadStages, EPI_F32, MODE>;
template <int MODE> constexpr auto kGemmLn = gemm_tc_kernel<kLnBN, 1, kLnStages, EPI_LN, MODE>;
constexpr int kPlainSmem = GemmSmem<kPlainBN, 2, kPlainStages, true>::kBytes;
constexpr int kHeadSmem = GemmSmem<kHeadBN, 2, kHeadStages>::kBytes;
constexpr int kLnSmem = GemmSmem<kLnBN, 1, kLnStages>::kBytes;
// the split mode's stage (two planes of a 32-element k-block) has the bytes of the one-plane 64-element stage, so the head and
// LN GEMMs keep their stage counts in every mode
static_assert(GemmSmem<kHeadBN, 2, kHeadStages, true>::kBytes == kHeadSmem && GemmSmem<kLnBN, 1, kLnStages, true>::kBytes == kLnSmem,
              "split-mode ring stages must keep the one-plane sizes");

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int load_encode() {
  if (g_encode) return LDM_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || fn == nullptr) return fail(LDM_ERR_CUDA, "cuTensorMapEncodeTiled not available");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return LDM_OK;
}

// 2-D row-major [rows][cols] 16-bit tensor, box = box_rows x kb columns with the (2 kb)-byte swizzle (kb = 64 or 32: one box row
// is one swizzle row, the layout of a ring k-block), zero OOB fill
int make_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, int kb, bool bf16) {
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kb), box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, kb == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(LDM_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu box_rows=%u", (int)r,
                                     (unsigned long long)rows, (unsigned long long)cols, box_rows);
  return LDM_OK;
}

// 2-D row-major [rows][cols] fp32 tensor, box = box_rows x box_cols, no swizzle: a box lands as dense [box_rows][box_cols] rows
int make_map_f32(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols) {
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 4};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(LDM_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) fp32 rows=%llu cols=%llu box %u x %u", (int)r,
                                     (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
  return LDM_OK;
}

// (B,S,C) contiguous <-> padded internal logits [B*128][160]
__global__ void logits_scatter_kernel(const float* __restrict__ src, float* __restrict__ dst, int n_layouts, int S, int C) {
  const size_t n = static_cast<size_t>(n_layouts) * S * C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C); const size_t tok = i / C; const int s = static_cast<int>(tok % S); const size_t b = tok / S;
    dst[(b * 128 + s) * kLogitLd + c] = src[i];
  }
}
__global__ void logits_gather_kernel(const float* __restrict__ src, float* __restrict__ dst, int n_layouts, int S, int C) {
  const size_t n = static_cast<size_t>(n_layouts) * S * C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C); const size_t tok = i / C; const int s = static_cast<int>(tok % S); const size_t b = tok / S;
    dst[i] = src[(b * 128 + s) * kLogitLd + c];
  }
}
__global__ void fill_ids_kernel(long long* dst, long long v, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) dst[i] = v;
}

}  // namespace

struct LdmHandle {
  LdmModelDesc desc;
  int C = 0, S = 0, L = 0, T = 0, G = 0;
  int mode = OP_F16;          // operand mode (LdmModelDesc::operand_dtype)
  bool bf16 = false;          // bf16 operand data (OP_BF16, OP_BF16X3)
  bool split = false;         // OP_BF16X3: every 16-bit weight and activation buffer has a lo plane (the *_lo members)
  int64_t launches = 0;
  int pdl = 1;                // env LDM_PDL=0: no programmatic dependent launch
  int debug_stop_after = 0;   // test tap: stop the denoiser after this many launches (0 = run everything)
  bool prof = false;          // per-kernel CUDA-event timing (ldm_profile_begin/end)
  struct ProfRec { int cat; cudaEvent_t a, b; };
  std::vector<ProfRec> prof_recs;
  // parameters (device)
  float *cat_emb = nullptr, *pos = nullptr, *adaln = nullptr, *sched = nullptr, *lae = nullptr;
  void *wqkv[kMaxLayers] = {}, *wo[kMaxLayers] = {}, *w1[kMaxLayers] = {}, *w2[kMaxLayers] = {}, *whead = nullptr;
  float *bqkv[kMaxLayers] = {}, *bo[kMaxLayers] = {}, *b1[kMaxLayers] = {}, *b2[kMaxLayers] = {}, *ln2w[kMaxLayers] = {}, *ln2b[kMaxLayers] = {};
  float *hlnw = nullptr, *hlnb = nullptr;
  CUtensorMap m_wqkv[kMaxLayers], m_wo[kMaxLayers], m_w1[kMaxLayers], m_w2[kMaxLayers], m_whead;
  void *wqkv_lo[kMaxLayers] = {}, *wo_lo[kMaxLayers] = {}, *w1_lo[kMaxLayers] = {}, *w2_lo[kMaxLayers] = {}, *whead_lo = nullptr;
  CUtensorMap m_wqkv_lo[kMaxLayers], m_wo_lo[kMaxLayers], m_w1_lo[kMaxLayers], m_w2_lo[kMaxLayers], m_whead_lo;
  int *qmap = nullptr, *amap = nullptr, *hmap = nullptr;   // source row / column maps of the padded QKV, out-projection and head weights
  // workspace (device), sized for cap layouts
  int cap = 0;
  void *x16 = nullptr, *qkv16 = nullptr, *att16 = nullptr, *z16 = nullptr, *hid16 = nullptr;
  float *x32 = nullptr, *y32 = nullptr, *logits = nullptr;
  float* rel_lp = nullptr;      // [cap][S][C] log-probabilities between the posterior and the draw (cond = relation)
  long long* ids[2] = {nullptr, nullptr};
  long long* ids_final = nullptr;
  long long *c_seq = nullptr, *c_seq_orig = nullptr; unsigned char* c_mask = nullptr; float* c_tbl = nullptr;  // staging for ldm_sample_host
  CUtensorMap m_x16, m_z16, m_qkv16;                                         // 128-row boxes: QKV / FF1 / head A operands, attention's head tiles
  CUtensorMap m_att16, m_hid16;                                              // A operands of the LN GEMMs: 128-row boxes (split mode: 64)
  CUtensorMap m_qkv16_st, m_hid16_st;                                        // 128-row boxes: the row-block GEMMs' TMA stores (one-plane modes)
  CUtensorMap m_x32, m_y32;                                                  // 64 x 232 fp32 boxes: the LN GEMMs' row halves (one-plane modes)
  void *x16_lo = nullptr, *qkv16_lo = nullptr, *att16_lo = nullptr, *z16_lo = nullptr, *hid16_lo = nullptr;   // split mode only
  CUtensorMap m_x16_lo, m_z16_lo, m_qkv16_lo, m_att16_lo, m_hid16_lo;
  std::vector<void*> owned;
  // CUDA graph of the whole T-step loop (ldm_sample_loop): captured once per (batch, plan, sampling, conditioning kind) and
  // replayed; everything that changes from call to call lives in device memory (noise key block, staged cond / start ids)
  int use_graph = 1;           // env LDM_GRAPH=0: plain stream launches
  int sweep = 1;               // env LDM_SWEEP=0: every kernel walks its row blocks in ascending order (no alternating directions)
  int num_sms = 0;             // the persistent GEMMs run at most one CTA per SM
  int max_threads_sm = 0;      // with num_sms: the launch policy of torch's distribution kernels (LDM_NOISE_TORCH)
  int gemm_ctas = 0;           // env LDM_GEMM_CTAS=n (n >= 1): at most n CTAs in a persistent GEMM launch (the LN GEMMs: max(1, n / 2)
                               // CTA pairs); 0: no cap
  int ln_clusters = 0;         // one-plane modes: the CTA pairs of gemm_ln_kernel that can be resident at once
  int gemm_split = 0;          // env LDM_GEMM_SPLIT=g (g >= 1): column ranges per row block of the row-block GEMMs; 0: automatic
  int fuse_embed = 1;          // env LDM_FUSE_EMBED=0: the loop launches the embedding kernel in every step instead of fusing it into the previous draw.
                               // The split mode always launches it: the draw kernels write one 16-bit plane only
  cudaStream_t cap_stream = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  uint64_t graph_key = 0;
  unsigned long long* call_block = nullptr;   // device {seed, b_global0, torch offset, tthr, delta, total_layouts} (StepParams::call)
  uint64_t ws_generation = 0;  // bumped when the workspace is reallocated (captured pointers die)
  int64_t graph_launches = 0;  // kernel launches inside the captured graph
  std::vector<void*> staging;  // ldm_create: fp32 uploads that only feed the packing kernels, released once those have run
};

namespace {

template <typename T>
int dev_alloc(LdmHandle* h, T** p, size_t n) {
  CK(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  h->owned.push_back(*p);
  return LDM_OK;
}
template <typename T>
int dev_upload(LdmHandle* h, T** p, const T* src, size_t n) {
  int rc = dev_alloc(h, p, n);
  if (rc) return rc;
  CK(cudaMemcpy(*p, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return LDM_OK;
}

// upload that only feeds a packing / table kernel of ldm_create: freed right after those kernels have run
template <typename T>
int dev_upload_tmp(LdmHandle* h, T** p, const T* src, size_t n) {
  CK(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  h->staging.push_back(*p);
  CK(cudaMemcpy(*p, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return LDM_OK;
}
void free_staging(LdmHandle* h) {
  for (void* p : h->staging) cudaFree(p);
  h->staging.clear();
}

// 16-bit weight buffer of rows x cols (split mode: the hi plane in dst, the lo plane in dst_lo)
int alloc16(LdmHandle* h, void** dst, void** dst_lo, int rows, int cols) {
  const size_t bytes = static_cast<size_t>(rows) * cols * 2;
  CK(cudaMalloc(dst, bytes));
  h->owned.push_back(*dst);
  if (h->split) { CK(cudaMalloc(dst_lo, bytes)); h->owned.push_back(*dst_lo); }
  return LDM_OK;
}

// fp32 weight -> the 16-bit operand in dst (split mode: both planes), on stream st
int pack16(const LdmHandle* h, void* dst, void* dst_lo, const float* src_dev, const int* row_map_dev, int dst_rows, int dst_cols, int src_cols,
           cudaStream_t st, const int* col_map_dev = nullptr) {
  const int blocks = 512;
  if (h->mode == OP_BF16X3) pack_weight_kernel<OP_BF16X3><<<blocks, 256, 0, st>>>(src_dev, dst, row_map_dev, col_map_dev, dst_rows, dst_cols, src_cols, dst_lo);
  else if (h->mode == OP_BF16) pack_weight_kernel<OP_BF16><<<blocks, 256, 0, st>>>(src_dev, dst, row_map_dev, col_map_dev, dst_rows, dst_cols, src_cols, nullptr);
  else pack_weight_kernel<OP_F16><<<blocks, 256, 0, st>>>(src_dev, dst, row_map_dev, col_map_dev, dst_rows, dst_cols, src_cols, nullptr);
  CK(cudaGetLastError());
  return LDM_OK;
}

// the fields of LdmWeights with their element counts for the handle's shapes
struct WeightField { const float* LdmWeights::*member; const char* name; size_t n; };
std::vector<WeightField> weight_fields(const LdmHandle* h) {
  const size_t d = h->desc.d_model, ff = h->desc.d_ff, L = h->L, T = h->T, C = h->C, S = h->S;
  return {{&LdmWeights::cat_emb, "cat_emb", C * d},         {&LdmWeights::pos_table, "pos_table", S * d},
          {&LdmWeights::in_proj_w, "in_proj_w", L * 3 * d * d}, {&LdmWeights::in_proj_b, "in_proj_b", L * 3 * d},
          {&LdmWeights::out_proj_w, "out_proj_w", L * d * d},   {&LdmWeights::out_proj_b, "out_proj_b", L * d},
          {&LdmWeights::linear1_w, "linear1_w", L * ff * d},    {&LdmWeights::linear1_b, "linear1_b", L * ff},
          {&LdmWeights::linear2_w, "linear2_w", L * d * ff},    {&LdmWeights::linear2_b, "linear2_b", L * d},
          {&LdmWeights::norm1_emb, "norm1_emb", L * T * d},     {&LdmWeights::norm1_w, "norm1_w", L * 2 * d * d},
          {&LdmWeights::norm1_b, "norm1_b", L * 2 * d},         {&LdmWeights::norm2_w, "norm2_w", L * d},
          {&LdmWeights::norm2_b, "norm2_b", L * d},             {&LdmWeights::head_ln_w, "head_ln_w", d},
          {&LdmWeights::head_ln_b, "head_ln_b", d},             {&LdmWeights::head_w, "head_w", C * d}};
}

// Repacks fp32 DEVICE weights in the LdmWeights layout into the handle's parameter buffers, on stream st: ldm_create runs it on
// its staged host arrays, ldm_load_weights on the caller's.  The kernels are plain launches (no programmatic dependent launch),
// so each starts only once all earlier work of st has completed; every step kernel reads a weight only after its pdl_sync()
// (common.cuh), so a step queued after this routine reads the new weights (DESIGN.md, "Weights").
int pack_weights(LdmHandle* h, const LdmWeights& w, cudaStream_t st) {
  const int d = h->desc.d_model, ff = h->desc.d_ff, L = h->L, T = h->T;
  const auto copy = [&](float* dst, const float* src, size_t n) { return cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st); };
  CK(copy(h->cat_emb, w.cat_emb, static_cast<size_t>(h->C) * d));
  CK(copy(h->pos, w.pos_table, static_cast<size_t>(h->S) * d));
  CK(copy(h->hlnw, w.head_ln_w, d));
  CK(copy(h->hlnb, w.head_ln_b, d));
  // AdaLN (scale, shift) for every (layer, t)
  adaln_table_kernel<<<dim3(T, L), 256, d * sizeof(float), st>>>(w.norm1_emb, w.norm1_w, w.norm1_b, h->adaln, T, d);
  CK(cudaGetLastError());
  int rc;
  for (int l = 0; l < L; ++l) {
    const size_t dd = static_cast<size_t>(d) * d;
    if ((rc = pack16(h, h->wqkv[l], h->wqkv_lo[l], w.in_proj_w + l * 3 * dd, h->qmap, kQkvN, d, d, st))) return rc;
    qkv_bias_kernel<<<(kQkvN + 255) / 256, 256, 0, st>>>(w.in_proj_b + static_cast<size_t>(l) * 3 * d, h->qmap, h->bqkv[l], kQkvN,
                                                        2 * 8 * kHeadPad, kHeadPad, d / h->desc.n_heads);
    CK(cudaGetLastError());
    if ((rc = pack16(h, h->wo[l], h->wo_lo[l], w.out_proj_w + l * dd, nullptr, d, kAttN, d, st, h->amap))) return rc;   // K = 512: head h occupies columns h*64 .. h*64+57
    CK(copy(h->bo[l], w.out_proj_b + static_cast<size_t>(l) * d, d));
    if ((rc = pack16(h, h->w1[l], h->w1_lo[l], w.linear1_w + l * ff * static_cast<size_t>(d), nullptr, ff, d, d, st))) return rc;
    CK(copy(h->b1[l], w.linear1_b + static_cast<size_t>(l) * ff, ff));
    if ((rc = pack16(h, h->w2[l], h->w2_lo[l], w.linear2_w + l * ff * static_cast<size_t>(d), nullptr, d, ff, ff, st))) return rc;
    CK(copy(h->b2[l], w.linear2_b + static_cast<size_t>(l) * d, d));
    CK(copy(h->ln2w[l], w.norm2_w + static_cast<size_t>(l) * d, d));
    CK(copy(h->ln2b[l], w.norm2_b + static_cast<size_t>(l) * d, d));
  }
  return pack16(h, h->whead, h->whead_lo, w.head_w, h->hmap, kLogitLd, d, d, st);
}

// TMA descriptor(s) of one 16-bit operand (split mode: both planes), boxes of box_rows x kb elements
int make_op_maps(const LdmHandle* h, CUtensorMap* m, CUtensorMap* m_lo, const void* base, const void* base_lo, uint64_t rows, uint64_t cols,
                 uint32_t box_rows, int kb) {
  int rc = make_map(m, base, rows, cols, box_rows, kb, h->bf16);
  if (rc || !h->split) return rc;
  return make_map(m_lo, base_lo, rows, cols, box_rows, kb, h->bf16);
}

template <int MODE>
OpMaps<MODE> op_maps(const CUtensorMap& hi, const CUtensorMap& lo) {
  OpMaps<MODE> m;
  m.hi = hi;
  if constexpr (kOpSplit<MODE>) m.lo = lo;
  else (void)lo;
  return m;
}

// util.py:47-70 + constrained.py:64-90: float64 schedule, fp32 log tables, 8 rows of length T+1 per group
void build_schedule(const LdmModelDesc& d, int N, float* out /*[8][T+1]*/) {
  const int T = d.num_timesteps, TT = T + 1;
  std::vector<double> att(T + 1), ctt(T + 1);
  att[0] = 1.0; ctt[0] = 0.0;
  for (int i = 0; i < T; ++i) {
    att[i + 1] = static_cast<double>(i) / (T - 1) * (d.att_T - d.att_1) + d.att_1;
    ctt[i + 1] = static_cast<double>(i) / (T - 1) * (d.ctt_T - d.ctt_1) + d.ctt_1;
  }
  auto l1m = [](double la) { return std::log(1.0 - std::exp(la) + 1e-40); };
  for (int i = 0; i < TT; ++i) for (int r = 0; r < 8; ++r) out[r * TT + i] = 0.0f;
  for (int i = 0; i < T; ++i) {
    const double at = att[i + 1] / att[i];
    const double ct = 1.0 - (1.0 - ctt[i + 1]) / (1.0 - ctt[i]);
    const double bt = (1.0 - at - ct) / N;
    out[0 * TT + i] = static_cast<float>(std::log(at));
    out[1 * TT + i] = static_cast<float>(std::log(bt));
    out[2 * TT + i] = static_cast<float>(std::log(ct));
    out[6 * TT + i] = static_cast<float>(l1m(std::log(ct)));
  }
  for (int i = 0; i < TT; ++i) {
    const double a = (i < T) ? att[i + 1] : 1.0, c = (i < T) ? ctt[i + 1] : 0.0;
    const double b = (1.0 - a - c) / N;
    out[3 * TT + i] = static_cast<float>(std::log(a));
    out[4 * TT + i] = static_cast<float>(std::log(b));
    out[5 * TT + i] = static_cast<float>(std::log(c));
    out[7 * TT + i] = static_cast<float>(l1m(std::log(c)));
  }
}

enum : int { CAT_EMBED = 0, CAT_QKV, CAT_ATTN, CAT_OUTPROJ, CAT_FF1, CAT_FF2, CAT_HEAD, CAT_EPILOGUE, CAT_MISC, CAT_COUNT };

struct ProfScope {   // counts the launch; when profiling is on, brackets it with a CUDA-event pair on the launching stream
  LdmHandle* h; cudaStream_t st; cudaEvent_t b = nullptr;
  ProfScope(LdmHandle* h_, int cat, cudaStream_t st_) : h(h_), st(st_) {
    h->launches++;
    if (h->prof) {
      cudaEvent_t a; cudaEventCreate(&a); cudaEventCreate(&b);
      cudaEventRecord(a, st);
      h->prof_recs.push_back({cat, a, b});
    }
  }
  ~ProfScope() { if (b) cudaEventRecord(b, st); }
};

// Launch of one kernel of the step.  Default: programmatic dependent launch (cudaLaunchAttributeProgrammaticStreamSerialization):
// the kernel's CTAs may start while the previous kernel of the stream drains; every kernel calls pdl_sync() (griddepcontrol.wait
// + launch_dependents) after its prologue and before its first dependent global access, so barrier init / descriptor prefetch /
// parameter loads overlap the predecessor's tail and the launch latency disappears.
// cluster > 1: clusters of that many consecutive CTAs along x (cudaLaunchAttributeClusterDimension).
template <typename... KArgs, typename... Args>
cudaError_t launch_cluster(const LdmHandle* h, int cluster, void (*kernel)(KArgs...), dim3 grid, int block, int smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  cfg.attrs = at; cfg.numAttrs = 0;
  if (h->pdl) { at[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[cfg.numAttrs++].val.programmaticStreamSerializationAllowed = 1; }
  if (cluster > 1) { at[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension; at[cfg.numAttrs++].val.clusterDim = {static_cast<unsigned>(cluster), 1, 1}; }
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
cudaError_t launch_step(const LdmHandle* h, void (*kernel)(KArgs...), dim3 grid, int block, int smem, cudaStream_t st, Args&&... args) {
  return launch_cluster(h, 1, kernel, grid, block, smem, st, std::forward<Args>(args)...);
}

// the dynamic shared memory of the kernels of MODE that use more than the default 48 KB; one-plane modes: how many CTA pairs of
// gemm_ln_kernel can be resident at once (h->ln_clusters)
template <int MODE>
int set_smem(LdmHandle* h) {
  constexpr auto attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
  if constexpr (kOpSplit<MODE>) {
    CK(cudaFuncSetAttribute(kGemmPlainSplit<EPI_QKV, MODE>, attr, kPlainSmem));
    CK(cudaFuncSetAttribute(kGemmPlainSplit<EPI_RELU, MODE>, attr, kPlainSmem));
  } else {
    CK(cudaFuncSetAttribute(gemm_rowblock_kernel<EPI_QKV, MODE>, attr, RbSmem::kBytes));
    CK(cudaFuncSetAttribute(gemm_rowblock_kernel<EPI_RELU, MODE>, attr, RbSmem::kBytes));
  }
  CK(cudaFuncSetAttribute(kGemmHead<MODE>, attr, kHeadSmem));
  if constexpr (kOpSplit<MODE>) CK(cudaFuncSetAttribute(kGemmLn<MODE>, attr, kLnSmem));
  else {
    CK(cudaFuncSetAttribute(gemm_ln_kernel<MODE, kLnOutStages>, attr, LnOut::kBytes));
    CK(cudaFuncSetAttribute(gemm_ln_kernel<MODE, kLnFf2Stages>, attr, LnFf2::kBytes));
  }
  CK(cudaFuncSetAttribute(attention_kernel<MODE>, attr, kOpSplit<MODE> ? kAttSmemBytesSplit : kAttSmemBytes));
  if constexpr (!kOpSplit<MODE>) {
    // the larger of the two: the out-projection's pairs fit wherever FF2's do (the same threads and registers, less shared memory)
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2); cfg.blockDim = dim3(kLnThreads); cfg.dynamicSmemBytes = LnFf2::kBytes;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim = {2, 1, 1};
    cfg.attrs = at; cfg.numAttrs = 1;
    CK(cudaOccupancyMaxActiveClusters(&h->ln_clusters, gemm_ln_kernel<MODE, kLnFf2Stages>, &cfg));
    if (h->ln_clusters < 1) return fail(LDM_ERR_UNSUPPORTED, "gemm_ln_kernel: no CTA pair of %d bytes of shared memory fits the device", LnFf2::kBytes);
  }
  return LDM_OK;
}

void free_workspace(LdmHandle* h) {
  void** ws[] = {&h->x16, &h->qkv16, &h->att16, &h->z16, &h->hid16, &h->x16_lo, &h->qkv16_lo, &h->att16_lo, &h->z16_lo, &h->hid16_lo,
                 reinterpret_cast<void**>(&h->x32), reinterpret_cast<void**>(&h->y32),
                 reinterpret_cast<void**>(&h->logits), reinterpret_cast<void**>(&h->ids[0]), reinterpret_cast<void**>(&h->ids[1]),
                 reinterpret_cast<void**>(&h->ids_final), reinterpret_cast<void**>(&h->c_seq), reinterpret_cast<void**>(&h->c_seq_orig),
                 reinterpret_cast<void**>(&h->c_mask), reinterpret_cast<void**>(&h->rel_lp)};
  for (void** p : ws) { if (*p) cudaFree(*p); *p = nullptr; }
  h->cap = 0;
}

int ensure_workspace(LdmHandle* h, int n_layouts) {
  if (n_layouts > kMaxLayouts) return fail(LDM_ERR_UNSUPPORTED, "batch of %d layouts exceeds the %d a call supports", n_layouts, kMaxLayouts);
  if (n_layouts <= h->cap) return LDM_OK;
  // free the old workspace: nothing may still be running on it, and a failed reallocation must not leave stale pointers behind
  CK(cudaDeviceSynchronize());
  free_workspace(h);
  const size_t M = static_cast<size_t>(n_layouts) * kBM;
  const int d = h->desc.d_model, ff = h->desc.d_ff;
  if (h->split) {
    // the lo planes: ~1.24 MB per layout.  An allocation that does not fit is reported (not left as the runtime's last error)
    // and releases what this call allocated
    void** lo[] = {&h->x16_lo, &h->qkv16_lo, &h->att16_lo, &h->z16_lo, &h->hid16_lo};
    const size_t cols[] = {static_cast<size_t>(d), static_cast<size_t>(kQkvN), static_cast<size_t>(kAttN), static_cast<size_t>(d), static_cast<size_t>(ff)};
    for (int i = 0; i < 5; ++i) {
      const cudaError_t e = cudaMalloc(lo[i], M * cols[i] * 2);
      if (e != cudaSuccess) {
        cudaGetLastError();
        free_workspace(h);
        return fail(LDM_ERR_CUDA, "split-operand workspace for %d layouts does not fit: %s", n_layouts, cudaGetErrorString(e));
      }
      CK(cudaMemset(*lo[i], 0, M * cols[i] * 2));
    }
  }
  CK(cudaMalloc(&h->x16, M * d * 2));
  CK(cudaMalloc(&h->qkv16, M * kQkvN * 2));
  CK(cudaMalloc(&h->att16, M * kAttN * 2));
  CK(cudaMalloc(&h->z16, M * d * 2));
  CK(cudaMalloc(&h->hid16, M * ff * 2));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->x32), M * d * 4));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->y32), M * d * 4));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->logits), M * kLogitLd * 4));
  const size_t nid = static_cast<size_t>(n_layouts) * h->S;
  CK(cudaMalloc(reinterpret_cast<void**>(&h->ids[0]), nid * 8));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->ids[1]), nid * 8));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->ids_final), nid * 8));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->c_seq), nid * 8));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->c_seq_orig), nid * 8));
  CK(cudaMalloc(reinterpret_cast<void**>(&h->c_mask), nid));
  // zero once: the 3 padding rows of every layout tile must stay finite
  CK(cudaMemset(h->x16, 0, M * d * 2)); CK(cudaMemset(h->qkv16, 0, M * kQkvN * 2)); CK(cudaMemset(h->att16, 0, M * kAttN * 2));
  CK(cudaMemset(h->z16, 0, M * d * 2)); CK(cudaMemset(h->hid16, 0, M * ff * 2)); CK(cudaMemset(h->x32, 0, M * d * 4));
  CK(cudaMemset(h->y32, 0, M * d * 4));
  CK(cudaMemset(h->logits, 0, M * kLogitLd * 4));
  h->cap = n_layouts;
  h->ws_generation++;
  int rc;
  // the row-block GEMM's resident A k-blocks are the one-plane ring's (64 elements): QKV, FF1 and the head share these maps
  static_assert(gemm_kb(false) == RbSmem::kKB, "one A geometry for QKV / FF1 / head");
  const int kb = gemm_kb(h->split);
  if ((rc = make_op_maps(h, &h->m_x16, &h->m_x16_lo, h->x16, h->x16_lo, M, d, kBM, kb))) return rc;
  if ((rc = make_op_maps(h, &h->m_z16, &h->m_z16_lo, h->z16, h->z16_lo, M, d, kBM, kb))) return rc;
  const int ln_rows = h->split ? kLnSplitRows : LnFf2::kRows;
  if ((rc = make_op_maps(h, &h->m_att16, &h->m_att16_lo, h->att16, h->att16_lo, M, kAttN, ln_rows, kLnKB))) return rc;
  if ((rc = make_op_maps(h, &h->m_hid16, &h->m_hid16_lo, h->hid16, h->hid16_lo, M, ff, ln_rows, kLnKB))) return rc;
  // attention's Q / K / V head tiles: 128 rows x one padded head, in every mode
  if ((rc = make_op_maps(h, &h->m_qkv16, &h->m_qkv16_lo, h->qkv16, h->qkv16_lo, M, kQkvN, kBM, kHeadPad))) return rc;
  // the row-block GEMMs' stores: 64-column x 128-row boxes of the staging tile (128-byte swizzle)
  if (!h->split && (rc = make_map(&h->m_qkv16_st, h->qkv16, M, kQkvN, kBM, 64, h->bf16))) return rc;
  if (!h->split && (rc = make_map(&h->m_hid16_st, h->hid16, M, ff, kBM, 64, h->bf16))) return rc;
  // the persistent LN GEMMs' residual loads and fp32 stores: one row half of the CTA's columns per box
  if (!h->split && (rc = make_map_f32(&h->m_x32, h->x32, M, d, LnFf2::kHalf, kLnBN))) return rc;
  if (!h->split && (rc = make_map_f32(&h->m_y32, h->y32, M, d, LnFf2::kHalf, kLnBN))) return rc;
  return LDM_OK;
}

template <int MODE>
int launch_denoiser(LdmHandle* h, int n, const long long* ids_in, int t_model, cudaStream_t st, const int* t_layout = nullptr, bool skip_embed = false) {
  const auto maps = [](const CUtensorMap& hi, const CUtensorMap& lo) { return op_maps<MODE>(hi, lo); };
  const int d = h->desc.d_model, ff = h->desc.d_ff, L = h->L, T = h->T;
  const int M = n * kBM;
  // Grids: the fp16 / bf16 row-block GEMMs (QKV, FF1) and LN GEMMs (epilogue warps) are persistent (one CTA per SM): their
  // epilogues run under the next tile's MMAs.  gemm_tc_kernel stores from the fragment, so a CTA has nothing to overlap its
  // epilogue with; one tile per CTA lets the hardware hand each SM its next tile the moment it is free, which measured faster
  // for it than a static persistent split (LDM_GEMM_CTAS caps the persistent grids only)
  const auto grid = [&](int tiles, bool persistent) {
    if (!persistent) return dim3(tiles);
    return dim3(std::min({tiles, h->num_sms, h->gemm_ctas > 0 ? h->gemm_ctas : tiles}));
  };
  // QKV / FF1 (bias, q-scale | ReLU): the row-block kernel in fp16 / bf16, 128-row x 256-column tiles in the split mode.  The
  // row-block kernel cuts each row block into n_ranges column ranges, each loading the row block's A once: one range when the
  // row blocks alone fill the SMs, otherwise enough for the items to fill them (at most one per tile); LDM_GEMM_SPLIT=g forces g
  const auto plain_gemm = [&](auto epi, const OpMaps<MODE>& a, const OpMaps<MODE>& w, const CUtensorMap& out, GemmParams p) {
    constexpr int EPI = decltype(epi)::value;
    if constexpr (kOpSplit<MODE>) {
      p.n_tiles = (p.N + kPlainBN - 1) / kPlainBN;
      return launch_step(h, kGemmPlainSplit<EPI, MODE>, grid(p.n_tiles * n, false), kGemmThreads, kPlainSmem, st, a, w, p);
    } else {
      p.n_tiles = (p.N + kRbCols - 1) / kRbCols;
      const int g = h->gemm_split > 0 ? h->gemm_split : n >= h->num_sms ? 1 : (h->num_sms + n - 1) / n;
      p.n_ranges = std::min(g, p.n_tiles);
      return launch_step(h, gemm_rowblock_kernel<EPI, MODE>, grid(n * p.n_ranges, true), kRbThreads, RbSmem::kBytes, st, a, w, out, p);
    }
  };
  // the LN GEMMs (out-projection, FF2): the fragment-epilogue kernel in the split mode, 64 whole rows per tile; otherwise the
  // persistent LN kernel, min(row blocks, resident pairs, LDM_GEMM_CTAS / 2) CTA pairs, each pair one row block at a time
  // res / st: the fp32 maps of p.resid and of p.y_out or p.out32 (the one that is set; at most one is)
  const auto ln_gemm = [&](const OpMaps<MODE>& a, const OpMaps<MODE>& w, const CUtensorMap& res, const CUtensorMap& st32, const GemmParams& p) {
    if constexpr (kOpSplit<MODE>) {
      return launch_step(h, kGemmLn<MODE>, grid(M / kLnSplitRows, false), kGemmThreads, kLnSmem, st, a, w, p);
    } else {
      const int pairs = std::min({n, h->ln_clusters, h->gemm_ctas > 0 ? std::max(1, h->gemm_ctas / 2) : n});
      if (p.K == kAttN) return launch_cluster(h, 2, gemm_ln_kernel<MODE, kLnOutStages>, dim3(2 * pairs), kLnThreads, LnOut::kBytes, st, a, w, res, st32, p);
      return launch_cluster(h, 2, gemm_ln_kernel<MODE, kLnFf2Stages>, dim3(2 * pairs), kLnThreads, LnFf2::kBytes, st, a, w, res, st32, p);
    }
  };
  int done = 0;
  // alternating sweep direction: every kernel walks the row blocks opposite to its predecessor (GemmParams::rev); the embedding /
  // draw kernels run their blocks in ascending order, so the first GEMM starts from the end.  LDM_SWEEP=0: always ascending
  int dir = 0;
  auto next_rev = [&]() { dir ^= 1; return h->sweep ? dir : 0; };
  // test tap: stop after `debug_stop_after` launches
#define LDM_STAGE_DONE() do { if (h->debug_stop_after && ++done >= h->debug_stop_after) { CK(cudaGetLastError()); return LDM_OK; } } while (0)
  if (!skip_embed) {     // skipped inside the loop: the previous step's draw kernel has already written this step's x32 / x16 rows
    const int warps = n * 128, blocks = (warps * 32 + 255) / 256;
    ProfScope ps(h, CAT_EMBED, st);
    CK(launch_step(h, embed_adaln_kernel<MODE>, dim3(blocks), 256, 0, st, ids_in, (const float*)h->cat_emb, (const float*)h->pos,
                   (const float*)h->adaln, t_model, t_layout, h->x32, h->x16, n, n, h->S, d, h->x16_lo));
  }
  if (!skip_embed) LDM_STAGE_DONE();
  for (int l = 0; l < L; ++l) {
    {  // QKV projection (+bias, q * 1/sqrt(head_dim))
      GemmParams p{M, kQkvN, d, 0, h->bqkv[l], h->qkv16, kQkvN, 1.0f / sqrtf(static_cast<float>(d / h->desc.n_heads)), 8 * kHeadPad};
      p.rev = next_rev(); p.out_lo = h->qkv16_lo;
      ProfScope ps(h, CAT_QKV, st);
      CK(plain_gemm(std::integral_constant<int, EPI_QKV>{}, maps(h->m_x16, h->m_x16_lo), maps(h->m_wqkv[l], h->m_wqkv_lo[l]), h->m_qkv16_st, p));
    }
    LDM_STAGE_DONE();
    {
      ProfScope ps(h, CAT_ATTN, st);
      CK(launch_step(h, attention_kernel<MODE>, dim3(n * h->desc.n_heads), kAttThreads, kOpSplit<MODE> ? kAttSmemBytesSplit : kAttSmemBytes, st,
                     maps(h->m_qkv16, h->m_qkv16_lo), h->att16, h->S, h->desc.n_heads, n, next_rev(), h->att16_lo));
    }
    LDM_STAGE_DONE();
    {  // out-projection + bias + residual (from the NORMALISED x) -> y32 ; z16 = LayerNorm2(y)   [fused epilogue]
      GemmParams p{M, d, kAttN, 1, h->bo[l], h->z16, d, 1.0f, 0, h->x32, h->y32, h->ln2w[l], h->ln2b[l], 0, nullptr};
      p.rev = next_rev(); p.out_lo = h->z16_lo;
      ProfScope ps(h, CAT_OUTPROJ, st);
      CK(ln_gemm(maps(h->m_att16, h->m_att16_lo), maps(h->m_wo[l], h->m_wo_lo[l]), h->m_x32, h->m_y32, p));
    }
    LDM_STAGE_DONE();
    {  // FF1 + ReLU
      GemmParams p{M, ff, d, 0, h->b1[l], h->hid16, ff, 1.0f, 0};   // 14 tiles of 128 columns + one of 64 (split mode: 7 of 256 + one of 64)
      p.rev = next_rev(); p.out_lo = h->hid16_lo;
      ProfScope ps(h, CAT_FF1, st);
      CK(plain_gemm(std::integral_constant<int, EPI_RELU>{}, maps(h->m_z16, h->m_z16_lo), maps(h->m_w1[l], h->m_w1_lo[l]), h->m_hid16_st, p));
    }
    LDM_STAGE_DONE();
    {  // FF2 + bias + residual ; next block's AdaLN(h, t) (fp32 residual + 16-bit operand) or the head LayerNorm   [fused epilogue]
      GemmParams p{M, d, ff, 1, h->b2[l], nullptr, d, 1.0f, 0, h->y32, nullptr, nullptr, nullptr, 0, nullptr};
      if (l + 1 < L) {
        const float* tab = h->adaln + (static_cast<size_t>(l + 1) * T + t_model) * 2 * d;
        p.ln_scale = tab; p.ln_shift = tab + d; p.adaln = 1; p.out32 = h->x32; p.out = h->x16; p.out_lo = h->x16_lo;
        if (t_layout) { p.ln_scale = h->adaln + static_cast<size_t>(l + 1) * T * 2 * d; p.t_layout = t_layout; p.n_layouts = n; }   // per-layout rows
      } else {
        p.ln_scale = h->hlnw; p.ln_shift = h->hlnb; p.adaln = 0; p.out32 = nullptr; p.out = h->z16; p.out_lo = h->z16_lo;
      }
      p.rev = next_rev();
      ProfScope ps(h, CAT_FF2, st);
      CK(ln_gemm(maps(h->m_hid16, h->m_hid16_lo), maps(h->m_w2[l], h->m_w2_lo[l]), h->m_y32, h->m_x32, p));
    }
    LDM_STAGE_DONE();
  }
  {  // vocabulary head -> fp32 logits
    GemmParams p{M, kLogitLd, d, 1, nullptr, h->logits, kLogitLd, 1.0f, 0};
    p.rev = next_rev();
    ProfScope ps(h, CAT_HEAD, st);
    CK(launch_step(h, kGemmHead<MODE>, grid(n, false), kGemmThreads, kHeadSmem, st, maps(h->m_z16, h->m_z16_lo), maps(h->m_whead, h->m_whead_lo), p));
  }
#undef LDM_STAGE_DONE
  CK(cudaGetLastError());
  return LDM_OK;
}

// the denoiser in the handle's operand mode
int run_denoiser(LdmHandle* h, int n, const long long* ids_in, int t_model, cudaStream_t st, const int* t_layout = nullptr, bool skip_embed = false) {
  switch (h->mode) {
    case OP_BF16X3: return launch_denoiser<OP_BF16X3>(h, n, ids_in, t_model, st, t_layout, skip_embed);
    case OP_BF16: return launch_denoiser<OP_BF16>(h, n, ids_in, t_model, st, t_layout, skip_embed);
    default: return launch_denoiser<OP_F16>(h, n, ids_in, t_model, st, t_layout, skip_embed);
  }
}

int validate_common(LdmHandle* h, int B, const LdmSampling* s) {
  if (!h) return fail(LDM_ERR_INVALID, "null handle");
  if (B <= 0) return fail(LDM_ERR_INVALID, "batch size must be positive (got %d)", B);
  if (!s) return fail(LDM_ERR_INVALID, "null sampling config");
  if (s->mode < 0 || s->mode > LDM_SAMPLING_GUMBEL) return fail(LDM_ERR_INVALID, "unknown sampling mode %d (sampling.py:118 raises NotImplementedError)", s->mode);
  if (s->mode != LDM_SAMPLING_DETERMINISTIC && !(s->temperature > 0.0f)) return fail(LDM_ERR_INVALID, "temperature must be > 0");
  if (s->mode == LDM_SAMPLING_TOP_P && !(s->top_p > 0.0f && s->top_p <= 1.0f)) return fail(LDM_ERR_INVALID, "top_p must be in (0, 1] (sampling.py:96)");
  if (s->mode == LDM_SAMPLING_TOP_K && !(s->top_k >= 1 && s->top_k <= h->C)) return fail(LDM_ERR_INVALID, "top_k out of range");
  return LDM_OK;
}

// torch's launch policy for a draw of numel < 2^31 elements (calc_execution_policy, ATen/native/cuda/DistributionTemplates.h):
// 256-thread blocks, at most as many as the device holds at once; tthr threads in all, each running curand_uniform4 until the
// elements are covered, and the generator's offset advances by 4 per such call (delta)
struct TorchPolicy { uint32_t tthr, delta; };
TorchPolicy torch_policy(const LdmHandle* h, int64_t numel) {
  const int64_t grid = std::min<int64_t>(static_cast<int64_t>(h->num_sms) * (h->max_threads_sm / 256), (numel + 255) / 256);
  const int64_t tthr = 256 * grid;
  return {static_cast<uint32_t>(tthr), static_cast<uint32_t>(((numel - 1) / (tthr * 4) + 1) * 4)};
}
int64_t torch_numel(const LdmHandle* h, int64_t total_layouts) { return total_layouts * h->S * h->C; }
// total_layouts * S * C < 2^31, checked without forming the product
bool torch_batch_fits(const LdmHandle* h, int64_t total_layouts) {
  return total_layouts <= ((int64_t(1) << 31) - 1) / (static_cast<int64_t>(h->S) * h->C);
}

int validate_noise(const LdmHandle* h, int B, int64_t b_global0, const LdmNoise* nz) {
  if (!nz) return fail(LDM_ERR_INVALID, "null noise description");
  if (nz->kind != LDM_NOISE_CONTRACT && nz->kind != LDM_NOISE_TORCH) return fail(LDM_ERR_INVALID, "unknown noise kind %d", nz->kind);
  if (nz->kind == LDM_NOISE_TORCH) {
    if (b_global0 < 0 || nz->total_layouts < b_global0 + B)
      return fail(LDM_ERR_INVALID, "total_layouts=%lld must cover layouts [%lld, %lld)", (long long)nz->total_layouts, (long long)b_global0, (long long)(b_global0 + B));
    if (!torch_batch_fits(h, nz->total_layouts))
      return fail(LDM_ERR_UNSUPPORTED, "torch-generator noise needs total_layouts * S * C < 2^31 (torch splits larger draws)");
    if (nz->offset % 4) return fail(LDM_ERR_INVALID, "a torch generator offset is a multiple of 4 (got %llu)", (unsigned long long)nz->offset);
  }
  return LDM_OK;
}

StepParams base_step_params(const LdmHandle* h, int B) {
  StepParams p{};
  p.n_layouts = B; p.S = h->S; p.C = h->C; p.n_attr = h->desc.n_attr;
  p.pad_id = h->C - 2; p.mask_id = h->C - 1;
  p.constrained = h->desc.q_type == 0;
  for (int g = 0; g < h->desc.n_attr && g < kMaxAttr; ++g) {
    p.grp_start[g] = g == 0 ? 0 : h->desc.n_cat + (g - 1) * h->desc.n_bins;
    p.grp_n[g] = g == 0 ? h->desc.n_cat : h->desc.n_bins;
  }
  p.T = h->T; p.sched = h->sched; p.lae = h->lae;
  p.logits = h->logits; p.ld_logits = kLogitLd;
  p.mode = SAMP_DETERMINISTIC; p.temperature = 1.0f;
  return p;
}

// noise: its kind selects the draw kernels' contract; step t_step of a call draws at the torch offset advanced by t_step steps
int step_impl(LdmHandle* h, int B, const long long* ids_in, int t_model, int t_post, const LdmCond* cond, const LdmSampling* samp,
              const LdmNoise& noise, uint32_t step_ctr, int t_step, int64_t b_global0, long long* ids_out, float* logits_out, float* logprob_out,
              const float* logits_in, const float* logprob_in, cudaStream_t st, const unsigned long long* call = nullptr,
              bool skip_embed = false, int t_next = -1) {
  if (t_model < 0 || t_model >= h->T || t_post < 0 || t_post >= h->T)
    return fail(LDM_ERR_INVALID, "timestep out of range: t_model=%d t_post=%d T=%d (constrained.py:139)", t_model, t_post, h->T);
  int rc = ensure_workspace(h, B);
  if (rc) return rc;
  if (logprob_in == nullptr) {
    if (logits_in != nullptr) {
      ProfScope ps(h, CAT_MISC, st);
      logits_scatter_kernel<<<1024, 256, 0, st>>>(logits_in, h->logits, B, h->S, h->C);
    } else {
      rc = run_denoiser(h, B, ids_in, t_model, st, nullptr, skip_embed);
      if (rc) return rc;
    }
    if (logits_out != nullptr) {
      ProfScope ps(h, CAT_MISC, st);
      logits_gather_kernel<<<1024, 256, 0, st>>>(h->logits, logits_out, B, h->S, h->C);
    }
  }
  StepParams p = base_step_params(h, B);
  p.t_post = t_post; p.logprob_in = logprob_in; p.ids_in = ids_in;
  if (cond && cond->seq) {
    p.cond_seq = reinterpret_cast<const long long*>(cond->seq); p.cond_mask = cond->mask;
    p.cond_seq_orig = reinterpret_cast<const long long*>(cond->seq_orig); p.refine_tbl = cond->refine_table;
    p.cond_flags = (cond->mask ? COND_HAS_MASK : 0) | (cond->pad_disable ? COND_PAD_DISABLE : 0) |
                   ((cond->seq_orig && cond->refine_table) ? COND_REFINE : 0);
  }
  p.mode = samp->mode; p.temperature = samp->temperature; p.top_p = samp->top_p; p.top_k = samp->top_k;
  p.seed = noise.seed; p.step_ctr = step_ctr; p.b_global0 = b_global0; p.call = call;
  const bool torch_noise = noise.kind == LDM_NOISE_TORCH;
  if (torch_noise) {
    const TorchPolicy tp = torch_policy(h, torch_numel(h, noise.total_layouts));
    p.t_offset = noise.offset; p.t_tthr = tp.tthr; p.t_delta = tp.delta; p.t_step = t_step; p.t_total = noise.total_layouts;
  }
  const auto generic = torch_noise ? posterior_sample_kernel<TorchNoise> : posterior_sample_kernel<TokenNoise>;
  const auto group = torch_noise ? posterior_sample_group_kernel<TorchNoise> : posterior_sample_group_kernel<TokenNoise>;
  p.ids_out = ids_out; p.logprob_out = logprob_out;
  if (t_next >= 0) {     // the loop: this draw also writes the next step's embedding + AdaLN_0(t_next) rows
    p.emb_cat = h->cat_emb; p.emb_pos = h->pos; p.emb_adaln = h->adaln + static_cast<size_t>(t_next) * 2 * h->desc.d_model;
    p.emb_x32 = h->x32; p.emb_x16 = h->x16; p.emb_d = h->desc.d_model; p.emb_bf16 = h->bf16 ? 1 : 0;
  }
  const int warps = B * h->S, blocks = (warps * 32 + 255) / 256;
  // cond = relation on the device (base.py:243-284 order: strong mask [+ refinement prior] -> update() -> PAD-disable -> draw):
  //   1. posterior kernel -> log-probs with PAD-disable OFF into rel_lp   2. relation_update_kernel in place
  //   3. draw kernel from rel_lp with PAD-disable.  `update` does nothing for t < 10 (logit_adjustment.py:105): plain path then.
  const bool relation = cond && cond->seq && cond->rel_adj && logprob_in == nullptr && cond->rel_num_update > 0 && t_model >= 10;
  if (relation) {
    if (h->desc.n_attr != 5 || h->desc.n_elem + 1 > kRelMaxNodes || h->desc.n_bins > 32)
      return fail(LDM_ERR_UNSUPPORTED, "relation update needs the c-x-y-w-h layout with <= 31 elements and <= 32 bins");
    if (!h->rel_lp) CK(cudaMalloc(reinterpret_cast<void**>(&h->rel_lp), static_cast<size_t>(h->cap) * h->S * h->C * sizeof(float)));
    StepParams p1 = p;
    p1.cond_flags &= ~COND_PAD_DISABLE; p1.logprob_out = h->rel_lp; p1.emb_adaln = nullptr;    // its draw is discarded: no embedding
    {
      ProfScope ps(h, CAT_EPILOGUE, st);
      CK(launch_step(h, generic, blocks, 256, 0, st, p1));
    }
    RelationParams r{};
    r.n_layouts = B; r.S = h->S; r.C = h->C; r.n_attr = h->desc.n_attr; r.n_elem = h->desc.n_elem; r.n_cat = h->desc.n_cat;
    r.n_bins = h->desc.n_bins; r.pad_id = h->C - 2; r.lp = h->rel_lp; r.cond_seq = p.cond_seq; r.adj = cond->rel_adj; r.centers = cond->rel_centers;
    const int btot = cond->rel_batch_total > 0 ? cond->rel_batch_total : B;
    r.step = cond->rel_lambda / static_cast<float>(btot * 14);            // len(const.relation) = 14 cost functions (const.py:226-241)
    r.n_update = cond->rel_num_update;
    {
      ProfScope ps(h, CAT_EPILOGUE, st);
      CK(launch_step(h, relation_update_kernel, B, kRelThreads, 0, st, r));
    }
    StepParams p2 = p;
    p2.logprob_in = h->rel_lp;
    p2.logprob_out = logprob_out;            // tap: the adjusted log-probs after PAD-disable (what sample() sees, base.py:287)
    {
      ProfScope ps(h, CAT_EPILOGUE, st);
      CK(launch_step(h, generic, blocks, 256, 0, st, p2));
    }
    CK(cudaGetLastError());
    return LDM_OK;
  }
  {
    ProfScope ps(h, CAT_EPILOGUE, st);
    if (group_kernel_applies(p)) CK(launch_step(h, group, blocks, 256, 0, st, p));
    else CK(launch_step(h, generic, blocks, 256, 0, st, p));
  }
  CK(cudaGetLastError());
  return LDM_OK;
}

}  // namespace

extern "C" {

const char* ldm_last_error(void) { return g_err; }
const char* ldm_version(void) { return "ldm_b200 0.2 (sm_90a, wgmma)"; }

int ldm_create(const LdmModelDesc* desc, const LdmWeights* w, LdmHandle** out) {
  if (!desc || !w || !out) return fail(LDM_ERR_INVALID, "null argument");
  const int d = desc->d_model, ff = desc->d_ff, L = desc->n_layers, T = desc->num_timesteps;
  const int C = desc->n_cat + 4 * desc->n_bins + 2, S = desc->n_elem * desc->n_attr;
  if (d != kDModel || desc->n_heads != 8 || ff != 4 * kDModel)
    return fail(LDM_ERR_UNSUPPORTED, "kernels are built for d_model=464, 8 heads, d_ff=1856 (got %d, %d, %d)", d, desc->n_heads, ff);
  if (L < 1 || L > kMaxLayers || T < 2) return fail(LDM_ERR_UNSUPPORTED, "n_layers must be in [1,%d], T >= 2", kMaxLayers);
  if (C < 129 || C > kLogitLd || S > 125 || S < 1 || desc->n_attr > kMaxAttr || desc->n_attr < 1)
    return fail(LDM_ERR_UNSUPPORTED, "vocabulary C=%d must be in [129,160] and S=%d <= 125", C, S);
  if (desc->q_type != 0 && desc->q_type != 1) return fail(LDM_ERR_INVALID, "q_type must be 0 (constrained) or 1 (vanilla)");
  if (desc->q_type == 0 && desc->n_attr != 5) return fail(LDM_ERR_UNSUPPORTED, "constrained q_type needs the c-x-y-w-h layout (5 attributes)");
  if (desc->operand_dtype < OP_F16 || desc->operand_dtype > OP_BF16X3)
    return fail(LDM_ERR_INVALID, "operand_dtype must be 0 (fp16), 1 (bf16) or 2 (bf16x3), got %d", desc->operand_dtype);
  CK(cudaSetDevice(desc->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, desc->device));
  if (prop.major != 9 || prop.minor != 0) return fail(LDM_ERR_UNSUPPORTED, "sm_90a kernels need a Hopper (CC 9.0) device, found CC %d.%d", prop.major, prop.minor);
  int rc = load_encode();
  if (rc) return rc;

  LdmHandle* h = new LdmHandle();
  h->desc = *desc; h->C = C; h->S = S; h->L = L; h->T = T;
  h->mode = desc->operand_dtype; h->bf16 = h->mode != OP_F16; h->split = h->mode == OP_BF16X3;
  h->G = desc->q_type == 0 ? desc->n_attr : 1;
  if (const char* e = getenv("LDM_PDL")) h->pdl = atoi(e);
  if (const char* e = getenv("LDM_GRAPH")) h->use_graph = atoi(e);
  if (const char* e = getenv("LDM_FUSE_EMBED")) h->fuse_embed = atoi(e);
  if (h->split) h->fuse_embed = 0;
  if (const char* e = getenv("LDM_SWEEP")) h->sweep = atoi(e);
  h->num_sms = prop.multiProcessorCount;
  h->max_threads_sm = prop.maxThreadsPerMultiProcessor;
  if (const char* e = getenv("LDM_GEMM_CTAS")) h->gemm_ctas = std::max(1, atoi(e));
  if (const char* e = getenv("LDM_GEMM_SPLIT")) h->gemm_split = std::max(1, atoi(e));
#define TRY(x) do { rc = (x); if (rc) { ldm_destroy(h); return rc; } } while (0)

  // parameter buffers and the TMA descriptors of the 16-bit weights
  TRY(dev_alloc(h, &h->cat_emb, static_cast<size_t>(C) * d));
  TRY(dev_alloc(h, &h->pos, static_cast<size_t>(S) * d));
  TRY(dev_alloc(h, &h->hlnw, static_cast<size_t>(d)));
  TRY(dev_alloc(h, &h->hlnb, static_cast<size_t>(d)));
  TRY(dev_alloc(h, &h->adaln, static_cast<size_t>(L) * T * 2 * d));
  const int plain_w_rows = h->split ? kPlainBN : kRbCols;
  for (int l = 0; l < L; ++l) {
    TRY(alloc16(h, &h->wqkv[l], &h->wqkv_lo[l], kQkvN, d));
    TRY(alloc16(h, &h->wo[l], &h->wo_lo[l], d, kAttN));
    TRY(alloc16(h, &h->w1[l], &h->w1_lo[l], ff, d));
    TRY(alloc16(h, &h->w2[l], &h->w2_lo[l], d, ff));
    TRY(dev_alloc(h, &h->bqkv[l], static_cast<size_t>(kQkvN)));
    TRY(dev_alloc(h, &h->bo[l], static_cast<size_t>(d)));
    TRY(dev_alloc(h, &h->b1[l], static_cast<size_t>(ff)));
    TRY(dev_alloc(h, &h->b2[l], static_cast<size_t>(d)));
    TRY(dev_alloc(h, &h->ln2w[l], static_cast<size_t>(d)));
    TRY(dev_alloc(h, &h->ln2b[l], static_cast<size_t>(d)));
    // QKV / FF1 weights: one tile's weight rows per box (row-block kernel: 128, split mode: 256)
    TRY(make_op_maps(h, &h->m_wqkv[l], &h->m_wqkv_lo[l], h->wqkv[l], h->wqkv_lo[l], kQkvN, d, plain_w_rows, gemm_kb(h->split)));
    TRY(make_op_maps(h, &h->m_wo[l], &h->m_wo_lo[l], h->wo[l], h->wo_lo[l], d, kAttN, kLnBN, kLnKB));
    TRY(make_op_maps(h, &h->m_w1[l], &h->m_w1_lo[l], h->w1[l], h->w1_lo[l], ff, d, plain_w_rows, gemm_kb(h->split)));
    TRY(make_op_maps(h, &h->m_w2[l], &h->m_w2_lo[l], h->w2[l], h->w2_lo[l], d, ff, kLnBN, kLnKB));
  }
  TRY(alloc16(h, &h->whead, &h->whead_lo, kLogitLd, d));
  TRY(make_op_maps(h, &h->m_whead, &h->m_whead_lo, h->whead, h->whead_lo, kLogitLd, d, kHeadBN, gemm_kb(h->split)));

  // per-head padded QKV row map: dst row = which*512 + head*64 + j  <-  src row which*d + head*58 + j (j < 58)
  const int dh = d / desc->n_heads;
  std::vector<int> qmap(kQkvN);
  for (int r = 0; r < kQkvN; ++r) {
    const int which = r / (8 * kHeadPad), hh = (r % (8 * kHeadPad)) / kHeadPad, j = r % kHeadPad;
    qmap[r] = j < dh ? which * d + hh * dh + j : -1;
  }
  TRY(dev_upload(h, &h->qmap, qmap.data(), qmap.size()));
  std::vector<int> amap(kAttN);
  for (int c = 0; c < kAttN; ++c) amap[c] = (c % kHeadPad) < dh ? (c / kHeadPad) * dh + (c % kHeadPad) : -1;
  TRY(dev_upload(h, &h->amap, amap.data(), amap.size()));
  std::vector<int> hmap(kLogitLd);
  for (int r = 0; r < kLogitLd; ++r) hmap[r] = r < C ? r : -1;
  TRY(dev_upload(h, &h->hmap, hmap.data(), hmap.size()));

  // the host arrays, staged on the device, then packed as ldm_load_weights packs device arrays
  LdmWeights staged{};
  for (const WeightField& f : weight_fields(h)) {
    float* p = nullptr;
    TRY(dev_upload_tmp(h, &p, w->*f.member, f.n));
    staged.*f.member = p;
  }
  TRY(pack_weights(h, staged, nullptr));
  {
    std::vector<float> sch(static_cast<size_t>(h->G) * 8 * (T + 1));
    for (int g = 0; g < h->G; ++g) {
      const int N = desc->q_type == 0 ? (g == 0 ? desc->n_cat : desc->n_bins) + 1 : C - 1;
      build_schedule(*desc, N, sch.data() + static_cast<size_t>(g) * 8 * (T + 1));
    }
    TRY(dev_upload(h, &h->sched, sch.data(), sch.size()));
    TRY(dev_alloc(h, &h->lae, static_cast<size_t>(h->G) * (T + 1) * 4));
    TRY(dev_alloc(h, &h->call_block, static_cast<size_t>(6)));
    lae_table_kernel<<<(h->G * (T + 1) + 127) / 128, 128>>>(h->sched, h->lae, h->G, T + 1);
    if (cudaGetLastError() != cudaSuccess) { ldm_destroy(h); return fail(LDM_ERR_CUDA, "lae_table_kernel launch failed"); }
  }
  if (cudaDeviceSynchronize() != cudaSuccess) { ldm_destroy(h); return fail(LDM_ERR_CUDA, "weight packing failed: %s", cudaGetErrorString(cudaGetLastError())); }
  free_staging(h);

  TRY(h->mode == OP_BF16X3 ? set_smem<OP_BF16X3>(h) : h->mode == OP_BF16 ? set_smem<OP_BF16>(h) : set_smem<OP_F16>(h));
#undef TRY
  *out = h;
  return LDM_OK;
}

int ldm_destroy(LdmHandle* h) {
  if (!h) return LDM_OK;
  cudaSetDevice(h->desc.device);
  cudaDeviceSynchronize();
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  for (void* p : h->owned) cudaFree(p);
  free_staging(h);
  free_workspace(h);
  if (h->c_tbl) cudaFree(h->c_tbl);
  delete h;
  return LDM_OK;
}

int ldm_load_weights(LdmHandle* h, const LdmWeights* w, void* stream) {
  if (!h || !w) return fail(LDM_ERR_INVALID, "null argument");
  CK(cudaSetDevice(h->desc.device));
  for (const WeightField& f : weight_fields(h)) {
    const float* p = w->*f.member;
    if (!p) return fail(LDM_ERR_INVALID, "LdmWeights.%s is null", f.name);
    // a host or other-device pointer would fault in the packing kernels: reject it here
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) ||
        a.device != h->desc.device) {
      cudaGetLastError();
      return fail(LDM_ERR_INVALID, "LdmWeights.%s is not device memory of device %d", f.name, h->desc.device);
    }
  }
  return pack_weights(h, *w, static_cast<cudaStream_t>(stream));
}

int ldm_step_noise(LdmHandle* h, int32_t B, const int64_t* ids_in, int32_t t_model, int32_t t_post, const LdmCond* cond,
                   const LdmSampling* sampling, const LdmNoise* noise, uint32_t step_ctr, int64_t b_global0, int64_t* ids_out,
                   float* logits_out, float* logprob_out, const float* logits_in, const float* logprob_in, void* stream) {
  int rc = validate_common(h, B, sampling);
  if (rc) return rc;
  if ((rc = validate_noise(h, B, b_global0, noise))) return rc;
  if (!ids_in || !ids_out) return fail(LDM_ERR_INVALID, "ids_in / ids_out must not be null");
  CK(cudaSetDevice(h->desc.device));
  return step_impl(h, B, reinterpret_cast<const long long*>(ids_in), t_model, t_post, cond, sampling, *noise, step_ctr, 0, b_global0,
                   reinterpret_cast<long long*>(ids_out), logits_out, logprob_out, logits_in, logprob_in, static_cast<cudaStream_t>(stream));
}

int ldm_step(LdmHandle* h, int32_t B, const int64_t* ids_in, int32_t t_model, int32_t t_post, const LdmCond* cond,
             const LdmSampling* sampling, uint64_t seed, uint32_t step_ctr, int64_t b_global0, int64_t* ids_out,
             float* logits_out, float* logprob_out, const float* logits_in, const float* logprob_in, void* stream) {
  const LdmNoise noise{LDM_NOISE_CONTRACT, seed, 0, 0};
  return ldm_step_noise(h, B, ids_in, t_model, t_post, cond, sampling, &noise, step_ctr, b_global0, ids_out, logits_out, logprob_out,
                        logits_in, logprob_in, stream);
}

int64_t ldm_noise_advance(const LdmHandle* h, int64_t total_layouts, const LdmSampling* sampling, int32_t n_steps) {
  if (!h || !sampling || total_layouts <= 0 || n_steps < 0) return fail(LDM_ERR_INVALID, "bad ldm_noise_advance arguments");
  if (!torch_batch_fits(h, total_layouts))
    return fail(LDM_ERR_UNSUPPORTED, "torch-generator noise needs total_layouts * S * C < 2^31 (torch splits larger draws)");
  if (sampling->mode == LDM_SAMPLING_DETERMINISTIC) return 0;
  const int64_t per_step = static_cast<int64_t>(torch_policy(h, torch_numel(h, total_layouts)).delta) * (sampling->mode == LDM_SAMPLING_GUMBEL ? 2 : 1);
  return per_step * n_steps;
}

int ldm_debug_torch_noise(const LdmHandle* h, int64_t numel, uint64_t seed, uint64_t offset, int32_t which, float* out, void* stream) {
  if (!h || !out || numel <= 0 || numel >= (int64_t(1) << 31) || offset % 4 || (which != 0 && which != 1))
    return fail(LDM_ERR_INVALID, "bad ldm_debug_torch_noise arguments");
  CK(cudaSetDevice(h->desc.device));
  const TorchPolicy tp = torch_policy(h, numel);
  torch_noise_tap_kernel<<<1024, 256, 0, static_cast<cudaStream_t>(stream)>>>(TorchNoise(seed, offset, tp.tthr), static_cast<uint32_t>(numel), which, out);
  CK(cudaGetLastError());
  return LDM_OK;
}

namespace {

// the plain loop: fill / pick the start state, then n_steps x step_impl on stream st
int run_loop(LdmHandle* h, int B, int n_steps, const int32_t* t_model, const int32_t* t_post, const LdmCond* cond, const LdmSampling* sampling,
             const LdmNoise& noise, int64_t b_global0, const long long* ids_init, long long* ids_out, long long* ids_trace, cudaStream_t st,
             const unsigned long long* call) {
  const size_t nid = static_cast<size_t>(B) * h->S;
  const long long* cur = nullptr;
  if (ids_init) cur = ids_init;
  else if (cond && cond->seq) cur = reinterpret_cast<const long long*>(cond->seq);
  else {
    ProfScope ps(h, CAT_MISC, st);
    fill_ids_kernel<<<256, 256, 0, st>>>(h->ids[0], static_cast<long long>(h->C - 1), nid);
    cur = h->ids[0];
  }
  for (int i = 0; i < n_steps; ++i) {
    long long* dst;
    if (ids_trace) dst = ids_trace + static_cast<size_t>(i) * nid;
    else if (i == n_steps - 1) dst = ids_out;
    else dst = (cur == h->ids[0]) ? h->ids[1] : h->ids[0];
    const bool fuse = h->fuse_embed != 0;
    int rc = step_impl(h, B, cur, t_model[i], t_post[i], cond, sampling, noise, static_cast<uint32_t>(i), i, b_global0, dst, nullptr, nullptr, nullptr, nullptr, st, call,
                       fuse && i > 0, (fuse && i + 1 < n_steps) ? t_model[i + 1] : -1);
    if (rc) return rc;
    cur = dst;
  }
  if (ids_trace) CK(cudaMemcpyAsync(ids_out, cur, nid * 8, cudaMemcpyDeviceToDevice, st));
  return LDM_OK;
}

uint64_t fnv1a(uint64_t hsh, const void* data, size_t n) {
  const unsigned char* b = static_cast<const unsigned char*>(data);
  for (size_t i = 0; i < n; ++i) { hsh ^= b[i]; hsh *= 1099511628211ull; }
  return hsh;
}

}  // namespace

int ldm_sample_loop_noise(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model, const int32_t* t_post, const LdmCond* cond,
                          const LdmSampling* sampling, const LdmNoise* noise, int64_t b_global0, const int64_t* ids_init, int64_t* ids_out,
                          int64_t* ids_trace, void* stream) {
  int rc = validate_common(h, B, sampling);
  if (rc) return rc;
  if ((rc = validate_noise(h, B, b_global0, noise))) return rc;
  if (n_steps < 1 || !t_model || !t_post || !ids_out) return fail(LDM_ERR_INVALID, "bad loop arguments");
  for (int i = 0; i < n_steps; ++i) {
    if (t_model[i] < 0 || t_model[i] >= h->T || t_post[i] < 0 || t_post[i] >= h->T)
      return fail(LDM_ERR_INVALID, "timestep out of range: t_model=%d t_post=%d T=%d (constrained.py:139)", t_model[i], t_post[i], h->T);
    if (i > 0 && t_model[i] >= t_model[i - 1]) return fail(LDM_ERR_INVALID, "timesteps must be strictly decreasing (base.py:361-362 raises NotImplementedError)");
  }
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = ensure_workspace(h, B);
  if (rc) return rc;
  const size_t nid = static_cast<size_t>(B) * h->S;
  const bool has_cond = cond && cond->seq;
  if (!h->use_graph || h->prof || ids_trace || h->debug_stop_after || (has_cond && cond->rel_adj))
    return run_loop(h, B, n_steps, t_model, t_post, has_cond ? cond : nullptr, sampling, *noise, b_global0, reinterpret_cast<const long long*>(ids_init),
                    reinterpret_cast<long long*>(ids_out), reinterpret_cast<long long*>(ids_trace), st, nullptr);

  // ---- CUDA-graph replay: the static T-step plan (n_steps x 23 launches with programmatic edges) is captured once; what changes
  // from call to call is staged into handle-owned device buffers the captured kernels read ----
  LdmCond gc{};
  if (has_cond) {
    if (reinterpret_cast<const long long*>(cond->seq) != h->c_seq) CK(cudaMemcpyAsync(h->c_seq, cond->seq, nid * 8, cudaMemcpyDeviceToDevice, st));
    gc.seq = reinterpret_cast<const int64_t*>(h->c_seq);
    if (cond->mask) {
      if (cond->mask != h->c_mask) CK(cudaMemcpyAsync(h->c_mask, cond->mask, nid, cudaMemcpyDeviceToDevice, st));
      gc.mask = h->c_mask;
    }
    if (cond->seq_orig && cond->refine_table) {
      if (reinterpret_cast<const long long*>(cond->seq_orig) != h->c_seq_orig) CK(cudaMemcpyAsync(h->c_seq_orig, cond->seq_orig, nid * 8, cudaMemcpyDeviceToDevice, st));
      const size_t tb = static_cast<size_t>(h->C) * h->C * 4;
      if (!h->c_tbl) CK(cudaMalloc(reinterpret_cast<void**>(&h->c_tbl), tb));
      if (cond->refine_table != h->c_tbl) CK(cudaMemcpyAsync(h->c_tbl, cond->refine_table, tb, cudaMemcpyDeviceToDevice, st));
      gc.seq_orig = reinterpret_cast<const int64_t*>(h->c_seq_orig); gc.refine_table = h->c_tbl;
    }
    gc.pad_disable = cond->pad_disable;
  }
  if (ids_init && reinterpret_cast<const long long*>(ids_init) != h->ids[1]) CK(cudaMemcpyAsync(h->ids[1], ids_init, nid * 8, cudaMemcpyDeviceToDevice, st));
  // the noise words the captured kernels read (StepParams::call); the contract reads the first two
  const TorchPolicy tp = noise->kind == LDM_NOISE_TORCH ? torch_policy(h, torch_numel(h, noise->total_layouts)) : TorchPolicy{0, 0};
  const unsigned long long blk[6] = {noise->seed, static_cast<unsigned long long>(b_global0), noise->offset, tp.tthr, tp.delta,
                                     static_cast<unsigned long long>(noise->total_layouts)};
  CK(cudaMemcpyAsync(h->call_block, blk, sizeof(blk), cudaMemcpyHostToDevice, st));   // pageable source: staged by the driver before the call returns

  uint64_t key = 1469598103934665603ull;
  const int32_t head[7] = {B, n_steps, has_cond ? 1 + (gc.mask ? 2 : 0) + (gc.seq_orig ? 4 : 0) + (gc.pad_disable ? 8 : 0) : 0, ids_init ? 1 : 0, h->pdl, h->fuse_embed,
                           noise->kind};
  key = fnv1a(key, head, sizeof(head));
  key = fnv1a(key, t_model, sizeof(int32_t) * n_steps);
  key = fnv1a(key, t_post, sizeof(int32_t) * n_steps);
  key = fnv1a(key, sampling, sizeof(LdmSampling));
  key = fnv1a(key, &h->ws_generation, sizeof(h->ws_generation));
  if (!h->graph_exec || key != h->graph_key) {
    if (h->graph_exec) { CK(cudaStreamSynchronize(st)); cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }   // no replay of the old plan may still be running
    if (!h->cap_stream) CK(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    const int64_t l0 = h->launches;
    // any failure to record or instantiate the plan (e.g. a capture conflict in the host application) permanently falls back to plain
    // stream launches for this handle instead of failing the call
    bool ok = cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    cudaGraph_t g = nullptr;
    if (ok) {
      const LdmNoise staged{noise->kind, 0, 0, noise->total_layouts};     // every noise word the kernels read comes from call_block
      rc = run_loop(h, B, n_steps, t_model, t_post, has_cond ? &gc : nullptr, sampling, staged, 0, ids_init ? h->ids[1] : nullptr, h->ids_final, nullptr,
                    h->cap_stream, h->call_block);
      ok = cudaStreamEndCapture(h->cap_stream, &g) == cudaSuccess && g != nullptr && rc == LDM_OK;
      h->graph_launches = h->launches - l0;
      h->launches = l0;                                  // counted per replay below
    }
    if (ok) ok = cudaGraphInstantiate(&h->graph_exec, g, 0) == cudaSuccess;
    if (g) cudaGraphDestroy(g);
    if (!ok) {
      cudaGetLastError();
      h->graph_exec = nullptr; h->use_graph = 0;
      return run_loop(h, B, n_steps, t_model, t_post, has_cond ? &gc : nullptr, sampling, *noise, b_global0, ids_init ? h->ids[1] : nullptr,
                      reinterpret_cast<long long*>(ids_out), nullptr, st, nullptr);
    }
    h->graph_key = key;
  }
  CK(cudaGraphLaunch(h->graph_exec, st));
  h->launches += h->graph_launches;
  if (reinterpret_cast<long long*>(ids_out) != h->ids_final) CK(cudaMemcpyAsync(ids_out, h->ids_final, nid * 8, cudaMemcpyDeviceToDevice, st));
  return LDM_OK;
}

int ldm_sample_loop(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model, const int32_t* t_post, const LdmCond* cond,
                    const LdmSampling* sampling, uint64_t seed, int64_t b_global0, const int64_t* ids_init, int64_t* ids_out,
                    int64_t* ids_trace, void* stream) {
  const LdmNoise noise{LDM_NOISE_CONTRACT, seed, 0, 0};
  return ldm_sample_loop_noise(h, B, n_steps, t_model, t_post, cond, sampling, &noise, b_global0, ids_init, ids_out, ids_trace, stream);
}

int ldm_sample_host(LdmHandle* h, int32_t B, int32_t n_steps, const int32_t* t_model, const int32_t* t_post,
                    const int64_t* cond_seq, const uint8_t* cond_mask, const int64_t* cond_seq_orig, const float* refine_table,
                    int32_t pad_disable, const LdmSampling* sampling, uint64_t seed, int64_t b_global0, const int64_t* ids_init,
                    int64_t* ids_out, void* stream, int64_t* h2d_bytes, int64_t* d2h_bytes) {
  int rc = validate_common(h, B, sampling);
  if (rc) return rc;
  if (!ids_out) return fail(LDM_ERR_INVALID, "ids_out_host must not be null");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = ensure_workspace(h, B);
  if (rc) return rc;
  const size_t nid = static_cast<size_t>(B) * h->S;
  int64_t up = 0;
  LdmCond cond{};
  if (cond_seq) {
    CK(cudaMemcpyAsync(h->c_seq, cond_seq, nid * 8, cudaMemcpyHostToDevice, st)); up += nid * 8;
    cond.seq = reinterpret_cast<const int64_t*>(h->c_seq);
    if (cond_mask) { CK(cudaMemcpyAsync(h->c_mask, cond_mask, nid, cudaMemcpyHostToDevice, st)); up += nid; cond.mask = h->c_mask; }
    if (cond_seq_orig && refine_table) {
      CK(cudaMemcpyAsync(h->c_seq_orig, cond_seq_orig, nid * 8, cudaMemcpyHostToDevice, st)); up += nid * 8;
      cond.seq_orig = reinterpret_cast<const int64_t*>(h->c_seq_orig);
      const size_t tb = static_cast<size_t>(h->C) * h->C * 4;
      if (!h->c_tbl) CK(cudaMalloc(reinterpret_cast<void**>(&h->c_tbl), tb));
      CK(cudaMemcpyAsync(h->c_tbl, refine_table, tb, cudaMemcpyHostToDevice, st)); up += tb;
      cond.refine_table = h->c_tbl;
    }
    cond.pad_disable = pad_disable;
  }
  const int64_t* init_dev = nullptr;
  if (ids_init) {
    // the start state travels from the host like any other input (x_T); it lands in the second ping-pong buffer
    CK(cudaMemcpyAsync(h->ids[1], ids_init, nid * 8, cudaMemcpyHostToDevice, st)); up += nid * 8;
    init_dev = reinterpret_cast<const int64_t*>(h->ids[1]);
  }
  rc = ldm_sample_loop(h, B, n_steps, t_model, t_post, cond_seq ? &cond : nullptr, sampling, seed, b_global0, init_dev,
                       reinterpret_cast<int64_t*>(h->ids_final), nullptr, stream);
  if (rc) return rc;
  CK(cudaMemcpyAsync(ids_out, h->ids_final, nid * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (h2d_bytes) *h2d_bytes = up;
  if (d2h_bytes) *d2h_bytes = static_cast<int64_t>(nid * 8);
  return LDM_OK;
}

int ldm_q_sample(LdmHandle* h, int32_t B, const int64_t* x0, const int32_t* t, uint64_t seed, int64_t b_global0, int64_t* xt, void* stream) {
  if (!h || !x0 || !t || !xt || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_q_sample arguments");
  CK(cudaSetDevice(h->desc.device));
  StepParams p = base_step_params(h, B);
  p.seed = seed; p.b_global0 = b_global0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int warps = B * h->S, blocks = (warps * 32 + 255) / 256;
  {
    ProfScope ps(h, CAT_MISC, st);
    q_sample_kernel<<<blocks, 256, 0, st>>>(p, reinterpret_cast<const long long*>(x0), t, reinterpret_cast<long long*>(xt));
  }
  CK(cudaGetLastError());
  return LDM_OK;
}

int ldm_decode(LdmHandle* h, int32_t B, const int64_t* ids, const float* centers, float* bbox, int64_t* label, uint8_t* mask, void* stream) {
  if (!h || !ids || !bbox || !label || !mask || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_decode arguments");
  if (h->desc.n_attr != 5) return fail(LDM_ERR_UNSUPPORTED, "decode needs the c-x-y-w-h token layout");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = B * h->desc.n_elem;
  {
    ProfScope ps(h, CAT_MISC, st);
    decode_kernel<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const long long*>(ids), centers, bbox, reinterpret_cast<long long*>(label), mask,
                                                  B, h->desc.n_elem, h->desc.n_attr, h->desc.n_cat, h->desc.n_bins);
  }
  CK(cudaGetLastError());
  return LDM_OK;
}

int ldm_make_cond(LdmHandle* h, int32_t B, int32_t cond_type, const int64_t* label, const float* bbox, const uint8_t* elem_mask,
                  const float* centers, int64_t* seq, uint8_t* mask, int64_t* seq_orig, void* stream) {
  if (!h || !label || !bbox || !elem_mask || !seq || !mask || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_make_cond arguments");
  if (h->desc.n_attr != 5) return fail(LDM_ERR_UNSUPPORTED, "make_cond needs the c-x-y-w-h token layout");
  if (cond_type < COND_TYPE_C || cond_type > COND_TYPE_GT)
    return fail(LDM_ERR_UNSUPPORTED, "cond_type %d: only c / cwh / refinement / gt are built on the device (task.py:27-151 raises NotImplementedError for unknown types)", cond_type);
  if (cond_type == COND_TYPE_REFINEMENT && !seq_orig) return fail(LDM_ERR_INVALID, "refinement needs seq_orig_out");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = B * h->desc.n_elem;
  const double dd = 1.0 / h->desc.n_bins;
  {
    ProfScope ps(h, CAT_MISC, st);
    make_cond_kernel<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const long long*>(label), bbox, elem_mask, centers,
                                                     reinterpret_cast<long long*>(seq), mask,
                                                     cond_type == COND_TYPE_REFINEMENT ? reinterpret_cast<long long*>(seq_orig) : nullptr, B,
                                                     h->desc.n_elem, h->desc.n_cat, h->desc.n_bins, h->C - 2, h->C - 1, cond_type,
                                                     static_cast<float>(dd), static_cast<float>(1.0 - dd));
  }
  CK(cudaGetLastError());
  return LDM_OK;
}

namespace {

int run_denoiser_per_layout_t(LdmHandle* h, int B, const long long* ids, const int32_t* t_dev, cudaStream_t st) {
  int rc = ensure_workspace(h, B);
  if (rc) return rc;
  return run_denoiser(h, B, ids, 0, st, t_dev);
}

}  // namespace

int ldm_predict_start(LdmHandle* h, int32_t B, const int64_t* xt_ids, const int32_t* t_dev, float* log_x0_out, float* logits_out, void* stream) {
  if (!h || !xt_ids || !t_dev || !log_x0_out || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_predict_start arguments");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = run_denoiser_per_layout_t(h, B, reinterpret_cast<const long long*>(xt_ids), t_dev, st);
  if (rc) return rc;
  if (logits_out) { ProfScope ps(h, CAT_MISC, st); logits_gather_kernel<<<1024, 256, 0, st>>>(h->logits, logits_out, B, h->S, h->C); }
  StepParams p = base_step_params(h, B);
  p.ids_in = reinterpret_cast<const long long*>(xt_ids); p.t_layout = t_dev; p.lx0_out = log_x0_out;   // ids_out == nullptr: no draw
  const int blocks = (B * h->S * 32 + 255) / 256;
  { ProfScope ps(h, CAT_EPILOGUE, st); CK(launch_step(h, posterior_sample_kernel<>, blocks, 256, 0, st, p)); }
  CK(cudaGetLastError());
  return LDM_OK;
}

int ldm_q_posterior(LdmHandle* h, int32_t B, const float* log_x_start, const int64_t* xt_ids, const int32_t* t_dev, float* out, void* stream) {
  if (!h || !log_x_start || !xt_ids || !t_dev || !out || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_q_posterior arguments");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  StepParams p = base_step_params(h, B);
  p.ids_in = reinterpret_cast<const long long*>(xt_ids); p.t_layout = t_dev; p.lx0_in = log_x_start; p.logprob_out = out;
  const int blocks = (B * h->S * 32 + 255) / 256;
  { ProfScope ps(h, CAT_EPILOGUE, st); CK(launch_step(h, posterior_sample_kernel<>, blocks, 256, 0, st, p)); }
  CK(cudaGetLastError());
  return LDM_OK;
}

namespace {
int q_pred_impl(LdmHandle* h, int32_t B, const float* log_x, const int32_t* t_dev, float* out, void* stream, int one_step) {
  if (!h || !log_x || !t_dev || !out || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_q_pred arguments");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  StepParams p = base_step_params(h, B);
  p.t_layout = t_dev;
  { ProfScope ps(h, CAT_MISC, st); q_pred_kernel<<<1024, 256, 0, st>>>(p, log_x, out, one_step); }
  CK(cudaGetLastError());
  return LDM_OK;
}
}  // namespace

int ldm_q_pred(LdmHandle* h, int32_t B, const float* log_x_start, const int32_t* t_dev, float* out, void* stream) {
  return q_pred_impl(h, B, log_x_start, t_dev, out, stream, 0);
}
int ldm_q_pred_one_timestep(LdmHandle* h, int32_t B, const float* log_x_t, const int32_t* t_dev, float* out, void* stream) {
  return q_pred_impl(h, B, log_x_t, t_dev, out, stream, 1);
}

int ldm_gumbel_argmax(LdmHandle* h, int32_t B, const float* logits, uint64_t seed, int64_t b_global0, int64_t* ids_out, void* stream) {
  if (!h || !logits || !ids_out || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_gumbel_argmax arguments");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = (B * h->S * 32 + 255) / 256;
  { ProfScope ps(h, CAT_MISC, st); gumbel_argmax_kernel<<<blocks, 256, 0, st>>>(logits, reinterpret_cast<long long*>(ids_out), B, h->S, h->C, seed, b_global0); }
  CK(cudaGetLastError());
  return LDM_OK;
}

int ldm_vb_terms(LdmHandle* h, int32_t B, const int64_t* x0_ids, const int64_t* xt_ids, const int32_t* t_dev, float mask_weight_mask,
                 float mask_weight_other, float* kl_out, float* nll_out, float* kl_aux_out, float* log_model_prob_out,
                 int64_t* x0_recon_out, int64_t* xtm1_recon_out, void* stream) {
  if (!h || !x0_ids || !xt_ids || !t_dev || !kl_out || !nll_out || B <= 0) return fail(LDM_ERR_INVALID, "bad ldm_vb_terms arguments");
  CK(cudaSetDevice(h->desc.device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = run_denoiser_per_layout_t(h, B, reinterpret_cast<const long long*>(xt_ids), t_dev, st);
  if (rc) return rc;
  // per-token terms live in the (free at this point) fp32 residual buffer of the workspace: 3 x [B][S] floats
  float* tok = h->y32;
  const size_t nt = static_cast<size_t>(B) * h->S;
  VbParams v{};
  v.sp = base_step_params(h, B);
  v.sp.ids_in = reinterpret_cast<const long long*>(xt_ids); v.sp.t_layout = t_dev; v.sp.logprob_out = log_model_prob_out;
  v.x0 = reinterpret_cast<const long long*>(x0_ids); v.w_mask = mask_weight_mask; v.w_other = mask_weight_other;
  v.kl_tok = tok; v.nll_tok = tok + nt; v.aux_tok = kl_aux_out ? tok + 2 * nt : nullptr;
  v.x0_recon = reinterpret_cast<long long*>(x0_recon_out); v.xtm1_recon = reinterpret_cast<long long*>(xtm1_recon_out);
  const int blocks = (B * h->S * 32 + 255) / 256, rblocks = (B * 32 + 255) / 256;
  { ProfScope ps(h, CAT_EPILOGUE, st); CK(launch_step(h, vb_terms_kernel, blocks, 256, 0, st, v)); }
  { ProfScope ps(h, CAT_MISC, st); CK(launch_step(h, row_mean_kernel, rblocks, 256, 0, st, (const float*)v.kl_tok, kl_out, B, h->S)); }
  { ProfScope ps(h, CAT_MISC, st); CK(launch_step(h, row_mean_kernel, rblocks, 256, 0, st, (const float*)v.nll_tok, nll_out, B, h->S)); }
  if (kl_aux_out) { ProfScope ps(h, CAT_MISC, st); CK(launch_step(h, row_mean_kernel, rblocks, 256, 0, st, (const float*)v.aux_tok, kl_aux_out, B, h->S)); }
  CK(cudaGetLastError());
  return LDM_OK;
}

int64_t ldm_launch_count(const LdmHandle* h) { return h ? h->launches : 0; }

int ldm_profile_begin(LdmHandle* h) {
  if (!h) return fail(LDM_ERR_INVALID, "null handle");
  h->prof = true;
  return LDM_OK;
}

int ldm_profile_end(LdmHandle* h, float* ms_per_category, int64_t* launches_per_category, int32_t n_categories) {
  if (!h) return fail(LDM_ERR_INVALID, "null handle");
  h->prof = false;
  CK(cudaDeviceSynchronize());
  for (int i = 0; i < n_categories; ++i) { if (ms_per_category) ms_per_category[i] = 0.0f; if (launches_per_category) launches_per_category[i] = 0; }
  for (auto& r : h->prof_recs) {
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, r.a, r.b);
    if (r.cat < n_categories) { if (ms_per_category) ms_per_category[r.cat] += ms; if (launches_per_category) launches_per_category[r.cat]++; }
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  h->prof_recs.clear();
  return LDM_OK;
}

#ifdef LDM_LN_PROBE
// the LN GEMMs' phase stamps (gemm_tc.cuh, ln_probe) since the last call, then cleared; returns the bytes copied, or -1
int64_t ldm_probe_ln_read(void* dst, int64_t capacity_bytes) {
  const int64_t bytes = sizeof(g_ln_probe);
  if (!dst || capacity_bytes < bytes) return -1;
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(dst, g_ln_probe, bytes) != cudaSuccess) return -1;
  static const unsigned char zeros[sizeof(g_ln_probe)] = {};
  return cudaMemcpyToSymbol(g_ln_probe, zeros, bytes) == cudaSuccess ? bytes : -1;
}
#endif

int ldm_debug_set_stop_after(LdmHandle* h, int32_t n_launches) {
  if (!h) return fail(LDM_ERR_INVALID, "null handle");
  h->debug_stop_after = n_launches;
  return LDM_OK;
}

int64_t ldm_debug_read(const LdmHandle* h, const char* name, void* dst, int64_t capacity_bytes, int32_t n_layouts) {
  if (!h || !name || n_layouts > h->cap) return -1;
  const size_t M = static_cast<size_t>(n_layouts) * kBM;
  const int d = h->desc.d_model, ff = h->desc.d_ff;
  const void* src = nullptr; size_t bytes = 0;
  if (!strcmp(name, "x32")) { src = h->x32; bytes = M * d * 4; }
  else if (!strcmp(name, "y32")) { src = h->y32; bytes = M * d * 4; }
  else if (!strcmp(name, "x16")) { src = h->x16; bytes = M * d * 2; }
  else if (!strcmp(name, "z16")) { src = h->z16; bytes = M * d * 2; }
  else if (!strcmp(name, "att16")) { src = h->att16; bytes = M * kAttN * 2; }
  else if (!strcmp(name, "qkv16")) { src = h->qkv16; bytes = M * kQkvN * 2; }
  else if (!strcmp(name, "hid16")) { src = h->hid16; bytes = M * ff * 2; }
  else if (!strcmp(name, "logits")) { src = h->logits; bytes = M * kLogitLd * 4; }
  else if (!strcmp(name, "x16_lo")) { src = h->x16_lo; bytes = M * d * 2; }
  else if (!strcmp(name, "z16_lo")) { src = h->z16_lo; bytes = M * d * 2; }
  else if (!strcmp(name, "att16_lo")) { src = h->att16_lo; bytes = M * kAttN * 2; }
  else if (!strcmp(name, "qkv16_lo")) { src = h->qkv16_lo; bytes = M * kQkvN * 2; }
  else if (!strcmp(name, "hid16_lo")) { src = h->hid16_lo; bytes = M * ff * 2; }
  else return -1;
  if (!h->split && strstr(name, "_lo") != nullptr) return -1;   // lo planes exist in the split mode only
  if (dst && capacity_bytes >= static_cast<int64_t>(bytes)) {
    if (cudaDeviceSynchronize() != cudaSuccess) return -2;
    if (cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
  }
  return static_cast<int64_t>(bytes);
}
int32_t ldm_num_classes(const LdmHandle* h) { return h ? h->C : 0; }
int32_t ldm_seq_len(const LdmHandle* h) { return h ? h->S : 0; }

int64_t ldm_get_schedule(const LdmHandle* h, float* dst, int64_t capacity) {
  if (!h) return 0;
  const int64_t n = static_cast<int64_t>(h->G) * 8 * (h->T + 1);
  if (dst && capacity >= n) cudaMemcpy(dst, h->sched, n * 4, cudaMemcpyDeviceToHost);
  return n;
}
int64_t ldm_get_adaln_table(const LdmHandle* h, float* dst, int64_t capacity) {
  if (!h) return 0;
  const int64_t n = static_cast<int64_t>(h->L) * h->T * 2 * h->desc.d_model;
  if (dst && capacity >= n) cudaMemcpy(dst, h->adaln, n * 4, cudaMemcpyDeviceToHost);
  return n;
}

}  // extern "C"
