// Shared device helpers for the LayoutDM sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers, Philox, misc.
// Everything here is plain inline PTX for sm_90a (H100); no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ldm {

#define LDM_DEVINL __device__ __forceinline__

constexpr float kLogEps = -69.07755278982137f;  // log(1e-30), T/models/categorical_diffusion/util.py:7-8

// ------------------------------------------------------------------------------------------------------------
// shared-memory addressing
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
LDM_DEVINL void st_shared_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
// the dynamic shared memory `raw` (an extern __shared__ array) rounded up to 1024 bytes, the 128-byte swizzle's atom.  The
// offset comes from the shared address, so the result is still `raw` plus an offset and keeps the shared state space: aligned
// through a generic integer, every access through it compiled to a generic LD / ST
LDM_DEVINL uint8_t* smem_align1024(uint8_t* raw) { return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u); }

// ------------------------------------------------------------------------------------------------------------
// programmatic dependent launch (every kernel of the step is launched with programmatic stream serialization): the
// prologue (barrier init, descriptor prefetch, parameter loads from constant tables) runs while the
// previous kernel drains; pdl_wait() returns once the previous grid has completed and its writes are visible.  No global
// access that depends on (or could overwrite the inputs of) the previous kernel may precede it.
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
LDM_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
LDM_DEVINL void pdl_sync() { pdl_wait(); pdl_launch_dependents(); }

// ------------------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
LDM_DEVINL void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

LDM_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LDM_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
LDM_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug traps instead of hanging the GPU.  ~2^28 polls >> any legal wait.
LDM_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) { asm volatile("trap;"); }
  }
}

// ------------------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) 2-D tile load, completion on an mbarrier
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
LDM_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// TMA 2-D tile store from shared memory, completion tracked per thread in bulk groups
LDM_DEVINL void tma_store_2d(const CUtensorMap* map, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
LDM_DEVINL void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still reading their shared-memory source
template <int N>
LDM_DEVINL void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every bulk group of this thread complete (its global writes done)
LDM_DEVINL void bulk_wait_group_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// orders this thread's generic-proxy shared-memory writes before later async-proxy (TMA) reads of them
LDM_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// warp-specialised register split: every warp of a warpgroup executes it; the new per-thread count is a multiple of 8
template <int R>
LDM_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
LDM_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ------------------------------------------------------------------------------------------------------------
// thread-block clusters (1-D): the CTA's rank, the cluster's index and count, the cluster barrier, stores into a peer's
// shared memory
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
LDM_DEVINL uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
LDM_DEVINL uint32_t cluster_count_x() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return r; }
// every thread of every CTA of the cluster arrives (release) and waits (acquire); also a barrier of the CTA's own threads
LDM_DEVINL void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// the shared::cluster address of this CTA's shared-memory location p in cluster CTA `rank`
LDM_DEVINL uint32_t map_peer(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
// 4-byte store into another CTA's shared memory (addresses from map_peer) that counts its bytes on that CTA's mbarrier bar
LDM_DEVINL void st_async_f32(uint32_t addr, float v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.f32 [%0], %1, [%2];" ::"r"(addr), "f"(v), "r"(bar) : "memory");
}

// named barrier among a subset of the CTA's warps (id 1..15; id 0 is __syncthreads)
LDM_DEVINL void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
// counts the calling warp's threads toward the barrier without waiting for it
LDM_DEVINL void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ------------------------------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): D[64 x N] (+)= A[64 x 16] * B[16 x N], fp32 accumulators in registers.
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): n8 block j holds
//   d[4j + 0], d[4j + 1] = row 16w + l/4,     columns 8j + 2(l%4) + {0, 1}
//   d[4j + 2], d[4j + 3] = row 16w + l/4 + 8, same columns
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
LDM_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
LDM_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int N>
LDM_DEVINL void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of an operand tile with the SW-byte swizzle (what TMA SWIZZLE_<SW>B writes; tile base
// aligned to the 8-row swizzle atom, 8 SW bytes).  K-major: rows of SW / 2 16-bit elements (SW bytes), 8-row groups 8 SW bytes
// apart (SBO); a k-step of 16 advances the start address by 32 B.  MN-major (SW = 128: 64 contiguous N elements per 128-B
// row, one row per K index): 8-K-row groups 1024 B apart.
// Bit layout (PTX ISA "matrix descriptor" for wgmma): [0,14) addr>>4, [16,30) LBO>>4 (unused here), [32,46) SBO>>4,
// [62,64) swizzle mode (1 = 128B, 2 = 64B).
template <int SW>
LDM_DEVINL uint64_t make_smem_desc(uint32_t smem_addr) {
  static_assert(SW == 128 || SW == 64, "the kernels use the 128- and 64-byte swizzles");
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(8 * SW >> 4) << 32;
  d |= static_cast<uint64_t>(SW == 128 ? 1 : 2) << 62;
  return d;
}

// both operands from shared memory, both K-major
// operand lists of the wrappers below: LDM_ACCn = "{%0, ..., %(n-1)}", LDM_OUTn = the matching "+f" constraints
#define LDM_F(i) "+f"(d[i])
#define LDM_ACC128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define LDM_OUT128 LDM_F(0), LDM_F(1), LDM_F(2), LDM_F(3), LDM_F(4), LDM_F(5), LDM_F(6), LDM_F(7), LDM_F(8), LDM_F(9), LDM_F(10), LDM_F(11), LDM_F(12), LDM_F(13), LDM_F(14), LDM_F(15), LDM_F(16), LDM_F(17), LDM_F(18), LDM_F(19), LDM_F(20), LDM_F(21), LDM_F(22), LDM_F(23), LDM_F(24), LDM_F(25), LDM_F(26), LDM_F(27), LDM_F(28), LDM_F(29), LDM_F(30), LDM_F(31), LDM_F(32), LDM_F(33), LDM_F(34), LDM_F(35), LDM_F(36), LDM_F(37), LDM_F(38), LDM_F(39), LDM_F(40), LDM_F(41), LDM_F(42), LDM_F(43), LDM_F(44), LDM_F(45), LDM_F(46), LDM_F(47), LDM_F(48), LDM_F(49), LDM_F(50), LDM_F(51), LDM_F(52), LDM_F(53), LDM_F(54), LDM_F(55), LDM_F(56), LDM_F(57), LDM_F(58), LDM_F(59), LDM_F(60), LDM_F(61), LDM_F(62), LDM_F(63), LDM_F(64), LDM_F(65), LDM_F(66), LDM_F(67), LDM_F(68), LDM_F(69), LDM_F(70), LDM_F(71), LDM_F(72), LDM_F(73), LDM_F(74), LDM_F(75), LDM_F(76), LDM_F(77), LDM_F(78), LDM_F(79), LDM_F(80), LDM_F(81), LDM_F(82), LDM_F(83), LDM_F(84), LDM_F(85), LDM_F(86), LDM_F(87), LDM_F(88), LDM_F(89), LDM_F(90), LDM_F(91), LDM_F(92), LDM_F(93), LDM_F(94), LDM_F(95), LDM_F(96), LDM_F(97), LDM_F(98), LDM_F(99), LDM_F(100), LDM_F(101), LDM_F(102), LDM_F(103), LDM_F(104), LDM_F(105), LDM_F(106), LDM_F(107), LDM_F(108), LDM_F(109), LDM_F(110), LDM_F(111), LDM_F(112), LDM_F(113), LDM_F(114), LDM_F(115), LDM_F(116), LDM_F(117), LDM_F(118), LDM_F(119), LDM_F(120), LDM_F(121), LDM_F(122), LDM_F(123), LDM_F(124), LDM_F(125), LDM_F(126), LDM_F(127)
#define LDM_ACC116 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115}"
#define LDM_OUT116 LDM_F(0), LDM_F(1), LDM_F(2), LDM_F(3), LDM_F(4), LDM_F(5), LDM_F(6), LDM_F(7), LDM_F(8), LDM_F(9), LDM_F(10), LDM_F(11), LDM_F(12), LDM_F(13), LDM_F(14), LDM_F(15), LDM_F(16), LDM_F(17), LDM_F(18), LDM_F(19), LDM_F(20), LDM_F(21), LDM_F(22), LDM_F(23), LDM_F(24), LDM_F(25), LDM_F(26), LDM_F(27), LDM_F(28), LDM_F(29), LDM_F(30), LDM_F(31), LDM_F(32), LDM_F(33), LDM_F(34), LDM_F(35), LDM_F(36), LDM_F(37), LDM_F(38), LDM_F(39), LDM_F(40), LDM_F(41), LDM_F(42), LDM_F(43), LDM_F(44), LDM_F(45), LDM_F(46), LDM_F(47), LDM_F(48), LDM_F(49), LDM_F(50), LDM_F(51), LDM_F(52), LDM_F(53), LDM_F(54), LDM_F(55), LDM_F(56), LDM_F(57), LDM_F(58), LDM_F(59), LDM_F(60), LDM_F(61), LDM_F(62), LDM_F(63), LDM_F(64), LDM_F(65), LDM_F(66), LDM_F(67), LDM_F(68), LDM_F(69), LDM_F(70), LDM_F(71), LDM_F(72), LDM_F(73), LDM_F(74), LDM_F(75), LDM_F(76), LDM_F(77), LDM_F(78), LDM_F(79), LDM_F(80), LDM_F(81), LDM_F(82), LDM_F(83), LDM_F(84), LDM_F(85), LDM_F(86), LDM_F(87), LDM_F(88), LDM_F(89), LDM_F(90), LDM_F(91), LDM_F(92), LDM_F(93), LDM_F(94), LDM_F(95), LDM_F(96), LDM_F(97), LDM_F(98), LDM_F(99), LDM_F(100), LDM_F(101), LDM_F(102), LDM_F(103), LDM_F(104), LDM_F(105), LDM_F(106), LDM_F(107), LDM_F(108), LDM_F(109), LDM_F(110), LDM_F(111), LDM_F(112), LDM_F(113), LDM_F(114), LDM_F(115)
#define LDM_ACC80 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}"
#define LDM_OUT80 LDM_F(0), LDM_F(1), LDM_F(2), LDM_F(3), LDM_F(4), LDM_F(5), LDM_F(6), LDM_F(7), LDM_F(8), LDM_F(9), LDM_F(10), LDM_F(11), LDM_F(12), LDM_F(13), LDM_F(14), LDM_F(15), LDM_F(16), LDM_F(17), LDM_F(18), LDM_F(19), LDM_F(20), LDM_F(21), LDM_F(22), LDM_F(23), LDM_F(24), LDM_F(25), LDM_F(26), LDM_F(27), LDM_F(28), LDM_F(29), LDM_F(30), LDM_F(31), LDM_F(32), LDM_F(33), LDM_F(34), LDM_F(35), LDM_F(36), LDM_F(37), LDM_F(38), LDM_F(39), LDM_F(40), LDM_F(41), LDM_F(42), LDM_F(43), LDM_F(44), LDM_F(45), LDM_F(46), LDM_F(47), LDM_F(48), LDM_F(49), LDM_F(50), LDM_F(51), LDM_F(52), LDM_F(53), LDM_F(54), LDM_F(55), LDM_F(56), LDM_F(57), LDM_F(58), LDM_F(59), LDM_F(60), LDM_F(61), LDM_F(62), LDM_F(63), LDM_F(64), LDM_F(65), LDM_F(66), LDM_F(67), LDM_F(68), LDM_F(69), LDM_F(70), LDM_F(71), LDM_F(72), LDM_F(73), LDM_F(74), LDM_F(75), LDM_F(76), LDM_F(77), LDM_F(78), LDM_F(79)
#define LDM_ACC64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define LDM_OUT64 LDM_F(0), LDM_F(1), LDM_F(2), LDM_F(3), LDM_F(4), LDM_F(5), LDM_F(6), LDM_F(7), LDM_F(8), LDM_F(9), LDM_F(10), LDM_F(11), LDM_F(12), LDM_F(13), LDM_F(14), LDM_F(15), LDM_F(16), LDM_F(17), LDM_F(18), LDM_F(19), LDM_F(20), LDM_F(21), LDM_F(22), LDM_F(23), LDM_F(24), LDM_F(25), LDM_F(26), LDM_F(27), LDM_F(28), LDM_F(29), LDM_F(30), LDM_F(31), LDM_F(32), LDM_F(33), LDM_F(34), LDM_F(35), LDM_F(36), LDM_F(37), LDM_F(38), LDM_F(39), LDM_F(40), LDM_F(41), LDM_F(42), LDM_F(43), LDM_F(44), LDM_F(45), LDM_F(46), LDM_F(47), LDM_F(48), LDM_F(49), LDM_F(50), LDM_F(51), LDM_F(52), LDM_F(53), LDM_F(54), LDM_F(55), LDM_F(56), LDM_F(57), LDM_F(58), LDM_F(59), LDM_F(60), LDM_F(61), LDM_F(62), LDM_F(63)
#define LDM_ACC32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define LDM_OUT32 LDM_F(0), LDM_F(1), LDM_F(2), LDM_F(3), LDM_F(4), LDM_F(5), LDM_F(6), LDM_F(7), LDM_F(8), LDM_F(9), LDM_F(10), LDM_F(11), LDM_F(12), LDM_F(13), LDM_F(14), LDM_F(15), LDM_F(16), LDM_F(17), LDM_F(18), LDM_F(19), LDM_F(20), LDM_F(21), LDM_F(22), LDM_F(23), LDM_F(24), LDM_F(25), LDM_F(26), LDM_F(27), LDM_F(28), LDM_F(29), LDM_F(30), LDM_F(31)
template <bool BF16>
LDM_DEVINL void wgmma_ss_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " LDM_ACC128 ", %128, %129, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT128 : "l"(da), "l"(db), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " LDM_ACC128 ", %128, %129, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT128 : "l"(da), "l"(db), "r"(accumulate));
}
template <bool BF16>
LDM_DEVINL void wgmma_ss_n232(float (&d)[116], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %118, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n232k16.f32.bf16.bf16 " LDM_ACC116 ", %116, %117, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT116 : "l"(da), "l"(db), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %118, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n232k16.f32.f16.f16 " LDM_ACC116 ", %116, %117, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT116 : "l"(da), "l"(db), "r"(accumulate));
}
template <bool BF16>
LDM_DEVINL void wgmma_ss_n160(float (&d)[80], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 " LDM_ACC80 ", %80, %81, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT80 : "l"(da), "l"(db), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 " LDM_ACC80 ", %80, %81, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT80 : "l"(da), "l"(db), "r"(accumulate));
}
template <bool BF16>
LDM_DEVINL void wgmma_ss_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " LDM_ACC64 ", %64, %65, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT64 : "l"(da), "l"(db), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " LDM_ACC64 ", %64, %65, p, 1, 1, 0, 0;\n\t}\n"
                 : LDM_OUT64 : "l"(da), "l"(db), "r"(accumulate));
}
// A from registers (four 16-bit pairs per thread, accumulator fragment order), B MN-major (transposed) from shared memory
template <bool BF16>
LDM_DEVINL void wgmma_rs_n64_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " LDM_ACC32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
                 : LDM_OUT32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " LDM_ACC32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
                 : LDM_OUT32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
#undef LDM_ACC128
#undef LDM_OUT128
#undef LDM_ACC116
#undef LDM_OUT116
#undef LDM_ACC80
#undef LDM_OUT80
#undef LDM_ACC64
#undef LDM_OUT64
#undef LDM_ACC32
#undef LDM_OUT32
#undef LDM_F

// ------------------------------------------------------------------------------------------------------------
// operand modes (LdmModelDesc::operand_dtype; accumulation is always fp32):
//   OP_F16, OP_BF16 : one 16-bit operand per value
//   OP_BF16X3       : every 16-bit operand is a pair of bf16 planes, hi = bf16(x), lo = bf16(x - hi), and a product is
//                     a_hi w_hi + a_hi w_lo + a_lo w_hi (three wgmmas into one accumulator).  The dropped a_lo w_lo is at most
//                     2^-16 |a w|, and hi + lo is within 2^-16 |x| of x: fp32-class operands on bf16 tensor cores.
// ------------------------------------------------------------------------------------------------------------
enum : int { OP_F16 = 0, OP_BF16 = 1, OP_BF16X3 = 2 };
template <int MODE> struct OpT;
template <> struct OpT<OP_F16> {
  using T = __half; using T2 = __half2;
  static LDM_DEVINL uint32_t pack(float a, float b) { __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }
  static LDM_DEVINL T from(float a) { return __float2half_rn(a); }
};
template <> struct OpT<OP_BF16> {
  using T = __nv_bfloat16; using T2 = __nv_bfloat162;
  static LDM_DEVINL uint32_t pack(float a, float b) { __nv_bfloat162 h = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }
  static LDM_DEVINL T from(float a) { return __float2bfloat16_rn(a); }
};
template <> struct OpT<OP_BF16X3> : OpT<OP_BF16> {
  // the pair of (a, b): hi = (bf16(a), bf16(b)), lo = (bf16(a - hi_a), bf16(b - hi_b)); x - hi is exact in fp32
  static LDM_DEVINL void pack_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h); lo = *reinterpret_cast<const uint32_t*>(&l);
  }
  static LDM_DEVINL void from_pair(float a, T& hi, T& lo) { hi = __float2bfloat16_rn(a); lo = __float2bfloat16_rn(a - __bfloat162float(hi)); }
};
// the wgmma input type of a mode
template <int MODE> constexpr bool kOpBf16 = MODE != OP_F16;
template <int MODE> constexpr bool kOpSplit = MODE == OP_BF16X3;

// TMA descriptors of one operand: the 16-bit plane, plus the lo plane in the split mode (kernel parameters; a one-plane struct
// has the layout of a bare CUtensorMap)
template <int MODE> struct OpMaps { CUtensorMap hi; };
template <> struct OpMaps<OP_BF16X3> { CUtensorMap hi, lo; };

// ------------------------------------------------------------------------------------------------------------
// Philox4x32-10 (the noise contract shared with oracle/layoutdm_oracle.py::uniforms)
// ------------------------------------------------------------------------------------------------------------
LDM_DEVINL uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0; k.y += W1;
  }
  return c;
}

// u in (0,1): ((word >> 9) + 0.5) * 2^-23  (exact in fp32)
LDM_DEVINL float u01_from_bits(uint32_t w) { return (static_cast<float>(w >> 9) + 0.5f) * 1.1920928955078125e-07f; }

// Gumbel noise of a uniform (sampling.py:112-116)
LDM_DEVINL float gumbel_of(float u) { return -logf(-logf(u + 1e-30f) + 1e-30f); }

// Counter word 1 of the noise contract: the step in bits 0..23, the stream in bits 24+ (0 = draw, 1 = Gumbel of
// name="gumbel", 2 = q_sample / gumbel_argmax).
LDM_DEVINL uint32_t noise_ctr(uint32_t step, uint32_t stream) { return (step & 0xFFFFFFu) | (stream << 24); }

// The noise of one token: key = seed, tok = (b_global0 + b) * S + s.  Class c draws word c & 3 of Philox block c >> 2.
struct TokenNoise {
  uint2 key; uint32_t tok_lo, tok_hi;
  LDM_DEVINL TokenNoise(unsigned long long seed, unsigned long long b_global0, int b, int S, int s) {
    const unsigned long long tok = (b_global0 + b) * static_cast<unsigned long long>(S) + s;
    key = make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
    tok_lo = static_cast<uint32_t>(tok); tok_hi = static_cast<uint32_t>(tok >> 32);
  }
  LDM_DEVINL uint4 block(int blk, uint32_t ctr) const { return philox4x32_10(make_uint4(static_cast<uint32_t>(blk), ctr, tok_lo, tok_hi), key); }
  static LDM_DEVINL int block_of(int c) { return c >> 2; }
  static LDM_DEVINL uint32_t word_of(const uint4& r, int c) { const int k = c & 3; return k == 0 ? r.x : k == 1 ? r.y : k == 2 ? r.z : r.w; }
  // the words of lane l's classes 4l..4l+3 and 128+l (the class ownership of the one-warp-per-token kernels)
  LDM_DEVINL void lane_words(int lane, uint32_t ctr, uint32_t (&w)[5]) const {
    const uint4 a = block(block_of(4 * lane), ctr), b = block(block_of(128 + lane), ctr);
    w[0] = word_of(a, 4 * lane); w[1] = word_of(a, 4 * lane + 1); w[2] = word_of(a, 4 * lane + 2); w[3] = word_of(a, 4 * lane + 3);
    w[4] = word_of(b, 128 + lane);
  }
  // what draw_class needs of the contract: the lane's classes must be able to win by at least this much (in units of the
  // temperature) for the classes outside a vocabulary group to be unreachable; see posterior_sample_group_kernel
  static constexpr float kGroupMargin = 40.0f;
};

// The draw's view of TokenNoise: words(stream, w) fills the lane's N words of a stream; Gumbel noise (added to the lane's
// log-probabilities) from stream 1, Exp(1) variates from stream 0.  Every slot is drawn whatever `on` says: the words come in Philox blocks of four classes.
template <int N, class Words>
struct ContractDraw {
  Words words;
  LDM_DEVINL void add_gumbel(const bool (&)[N], float (&lg)[N]) const {
    uint32_t w[N];
    words(1u, w);
#pragma unroll
    for (int j = 0; j < N; ++j) lg[j] += gumbel_of(u01_from_bits(w[j]));
  }
  LDM_DEVINL void exponential(const bool (&)[N], float (&e)[N]) const {
    uint32_t w[N];
    words(0u, w);
#pragma unroll
    for (int j = 0; j < N; ++j) e[j] = -logf(u01_from_bits(w[j]));
  }
};
template <int N, class Words>
LDM_DEVINL ContractDraw<N, Words> contract_draw(Words w) { return ContractDraw<N, Words>{w}; }

// ------------------------------------------------------------------------------------------------------------
// The second noise contract: the numbers torch's CUDA generator gives `exponential_` / `uniform_` on a contiguous tensor of
// numel < 2^31 elements (ATen/native/cuda/DistributionTemplates.h, distribution_elementwise_grid_stride_kernel with
// curand_uniform4; tthr = 256 * grid threads of calc_execution_policy).  Element i is word (i / tthr) & 3 of the
// Philox4x32-10 block with counter offset / 4 + i / (4 tthr) in words 0-1 and subsequence i % tthr in words 2-3,
// key = seed (curand_init(seed, i % tthr, offset)).
// ------------------------------------------------------------------------------------------------------------
struct TorchNoise {
  uint2 key; unsigned long long ctr0; uint32_t tthr;
  __host__ __device__ __forceinline__ TorchNoise(unsigned long long seed, unsigned long long offset, uint32_t tthr_) : ctr0(offset >> 2), tthr(tthr_) {
    key = make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  }
  LDM_DEVINL uint32_t word(uint32_t i) const {
    const uint32_t q = i / tthr, sub = i - q * tthr;
    const unsigned long long ctr = ctr0 + (q >> 2);
    return TokenNoise::word_of(philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), sub, 0u), key), q & 3);
  }
  // curand_uniform: w 2^-32 + 2^-33, in (0, 1]
  static LDM_DEVINL float uniform(uint32_t w) { return __fmaf_rn(__uint2float_rn(w), 0x1p-32f, 0x1p-33f); }
  // uniform_ on [0, 1) (uniform_kernel: 1 -> 0)
  static LDM_DEVINL float rand(uint32_t w) { const float u = uniform(w); return u == 1.0f ? 0.0f : u; }
  // exponential_(1) (ATen/core/TransformationHelper.h, transformation::exponential): -log(u), -log -> eps / 2 near 1; at::log
  // of a float is the fast __logf on the device (ATen/NumericUtils.h)
  static LDM_DEVINL float exponential(uint32_t w) { const float u = uniform(w); return u >= 1.0f - 0x1p-24f ? 0x1p-24f : -__logf(u); }
  // a class outside a group has p ~ 1e-30 / temperature: it cannot win unless exp(margin) < e_max / e_min * Gumbel spread
  // = (22.9 / 2^-24) * exp(16.7 + 4.3), exp(40.7); the margin of the contract would not do
  static constexpr float kGroupMargin = 48.0f;
};

// The draw's view of TorchNoise for one token (b, s) of an (n_total, S, C) batch, b global: multinomial over the (B S, C)
// probabilities draws exponential_ at `exp`'s offset into empty_like(probs), in memory order: element (b S + s) C + c of the
// contiguous copy the rearrange makes for n_total > 1, element c S + s for n_total == 1, where the rearrange is a view with
// strides (1, S) that empty_like keeps (i_exp + exp_cs * c).  name="gumbel" first draws element (b C + c) S + s of rand_like on
// the contiguous (B, C, S) log-probabilities at `gum`'s offset.  One Philox block per class, and only for the slots with `on`
// (classes that can win).
template <int N>
struct TorchDraw {
  TorchNoise exp, gum; uint32_t i_exp, exp_cs, i_gum, S; const int (&cls)[N];
  LDM_DEVINL void add_gumbel(const bool (&on)[N], float (&lg)[N]) const {
#pragma unroll
    for (int j = 0; j < N; ++j) if (on[j]) lg[j] += gumbel_of(TorchNoise::rand(gum.word(i_gum + static_cast<uint32_t>(cls[j]) * S)));
  }
  LDM_DEVINL void exponential(const bool (&on)[N], float (&e)[N]) const {
#pragma unroll
    for (int j = 0; j < N; ++j) e[j] = on[j] ? TorchNoise::exponential(exp.word(i_exp + exp_cs * static_cast<uint32_t>(cls[j]))) : 1.0f;
  }
};

LDM_DEVINL float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

LDM_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
LDM_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
LDM_DEVINL double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace ldm
