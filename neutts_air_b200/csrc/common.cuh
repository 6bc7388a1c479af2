// Shared device helpers for the sm_90a kernels: mbarrier, bulk/TMA copies, wgmma (warpgroup MMA),
// programmatic dependent launch, small math utilities.
// Everything is inline PTX; no CUTLASS/CuTe headers are included.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

#define NT_DEVINL __device__ __forceinline__

#include "wgmma.cuh"

// Spin bound for every mbarrier wait: a protocol bug becomes a trap (the launch fails with
// an error the host reports) instead of a hung GPU box.  try_wait itself suspends the thread for
// a hardware-defined slice per call, so 2^22 tries is seconds — far beyond any legitimate wait
// in these kernels (the longest is one decode step, ~1 ms).
#ifndef NT_SPIN_LIMIT
#define NT_SPIN_LIMIT (1u << 22)
#endif

namespace nt {

constexpr int kWarp = 32;

NT_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
NT_DEVINL int lane_id() { return threadIdx.x & 31; }
// One lane of a fully converged warp (the same lane on every call).  Code issuing uniform-datapath instructions
// (TMA) must sit under THIS predicate inside warp-uniform control flow: behind a plain `if (lane == 0)` the compiler
// cannot prove that a single thread is active and wraps every such instruction in an ELECT / BRA.U.ANY loop with
// R2UR moves.
// Call it AT the use site, after any data-dependent wait loop: elect.sync (full mask) is also the reconvergence point,
// and the compiler emits the guarded UTMALDG unpredicated (only the operand moves carry the predicate), so
// a diverged lane group without the leader would execute it with stale uniform registers (memcheck: out-of-range
// shared address; found with a cached `leader` flag behind an mbarrier spin).
NT_DEVINL bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// value of lane 0, which the compiler then knows to be warp-uniform
NT_DEVINL int uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }
NT_DEVINL int warp_id() { return threadIdx.x >> 5; }

// ---------------------------------------------------------------- PDL (griddepcontrol)
// launch_dependents: lets the next kernel in the stream start its prologue (weight
// prefetch) early; wait: blocks until the previous kernel has fully completed and its
// writes are visible.  Rule used throughout: before pdl_wait() a kernel may only touch
// immutable weight memory and its own shared memory.
NT_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
NT_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
NT_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
NT_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
NT_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
NT_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
NT_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
NT_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
#ifdef NT_WGMMA_KERNELS
// Translation units with wgmma kernels: a function call anywhere in such a kernel makes ptxas serialize its wgmma
// pipeline, so a timeout traps in line without the report.
NT_DEVINL void nt_timeout(const char*) { __trap(); }
#else
// out of line on purpose: the report is cold code, inlined it would sit (printf argument set-up and all) in the
// instruction stream of every wait loop of kernels that already fight for the instruction cache
__device__ __noinline__ inline void nt_timeout(const char* what) {
  printf("neutts_b200: timed out waiting for %s (block %d,%d thread %d)\n", what, blockIdx.x, blockIdx.y, threadIdx.x);
  __trap();
}
#endif
NT_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > NT_SPIN_LIMIT) nt_timeout("an mbarrier");
  }
}

// ---------------------------------------------------------------- 1-D bulk copy (TMA engine, no tensor map)
// global -> shared, completion counted on an mbarrier.  dst/src 16-byte aligned, bytes % 16 == 0.
NT_DEVINL void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
NT_DEVINL void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------- 2-D tiled TMA load
NT_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
NT_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// Same with an L2 eviction-priority hint (createpolicy): weights that stream through once per decode step are loaded
// evict_first so that they do not push the small hot set (KV pages, hand-off buffers, logits) out of the 50 MB L2.
NT_DEVINL uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
NT_DEVINL void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
// K-major operand tile in shared memory written by TMA with CU_TENSOR_MAP_SWIZZLE_128B:
// rows of 128 bytes, 8-row groups 1024 bytes apart (SBO), layout type 1 (SWIZZLE_128B).
// Field layout of the sm_90 wgmma matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base offset [49,52) (0: tiles are 1024-byte aligned), layout [62,64).  Adding 2 to the descriptor advances the
// start by 32 bytes = one K step of a bf16 (16) or tf32 (8) instruction; adding 512 advances by 64 rows.
NT_DEVINL uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (ignored for swizzled K-major), canonical value 1
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO = 1024 B between 8-row core groups
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}
// Register fence before the first wgmma that reads accumulators this thread wrote (or a new batch of MMAs).
NT_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
NT_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// Wait until at most N committed groups of this warp are pending: their shared-memory operands may then be reused.
template <int N>
NT_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keep the compiler from moving accumulator reads / writes across an asynchronous wgmma.
template <int R>
NT_DEVINL void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i]) : : "memory");
}
// Accumulator fragments of one warp (rows [16 w, 16 w + 16) of a 64-row wgmma tile, see wgmma.cuh) -> fp32 rows in
// shared memory: dst[row * ld + col], rows offset by row0.
template <int N>
NT_DEVINL void wgmma_store_rows(const float (&d)[N / 2], float* dst, int ld, int row0) {
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int r = row0 + 16 * w + (l >> 2), c = 2 * (l & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(dst + static_cast<long long>(r) * ld + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(dst + static_cast<long long>(r + 8) * ld + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// ---------------------------------------------------------------- math / conversion
NT_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
NT_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// 8 bf16 packed in a uint4 -> 8 floats (bf16 -> fp32 is a 16-bit shift)
NT_DEVINL void bf16x8_to_f32(const uint4& p, float (&f)[8]) {
  f[0] = __uint_as_float(p.x << 16);
  f[1] = __uint_as_float(p.x & 0xffff0000u);
  f[2] = __uint_as_float(p.y << 16);
  f[3] = __uint_as_float(p.y & 0xffff0000u);
  f[4] = __uint_as_float(p.z << 16);
  f[5] = __uint_as_float(p.z & 0xffff0000u);
  f[6] = __uint_as_float(p.w << 16);
  f[7] = __uint_as_float(p.w & 0xffff0000u);
}
NT_DEVINL float silu(float x) { return x / (1.0f + __expf(-x)); }
NT_DEVINL uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace nt
