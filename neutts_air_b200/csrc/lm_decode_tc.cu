// Persistent wgmma decode kernel: ALL layers, the lm_head, the sampler and the whole multi-step decode loop in
// ONE cooperative launch of one CTA per SM, for every batch size 1..64.
//
//   GEMM phases (qkv | o_proj | gate/up | down | lm_head) run on the tensor cores (warpgroup MMA):
//     * A operand = WEIGHTS, exactly as they lie in HBM (K-major): 128 rows x 64 k tiles (16 KB) fetched by 2-D TMA
//       (SWIZZLE_128B) through per-matrix tensor maps built once at nt_lm_create; one warp streams this CTA's tiles
//       of the WHOLE step into a deep mbarrier ring and runs ahead across phase boundaries (weights are immutable);
//     * B operand = ACTIVATIONS, K-major [tokens x 64 k] chunks in shared memory: tokens sit on the MMA N axis
//       (N = 16 | 32 | 64).  Batch <= 8 feeds every activation as a bf16 hi + lo pair on two N columns (~16 mantissa
//       bits, the decode path keeps fp32-grade activations); larger batches use plain bf16 like the prefill path;
//     * one MMA warpgroup issues wgmma (two M = 64 halves of the 128-row tile) with the accumulators in registers,
//       then hands each finished tile [128 weight rows x N] to the four epilogue warps through shared memory (one
//       fp32 row per epilogue lane) while it already accumulates the next item.
//   Work split: every weight matrix is cut into (128-row tile, K slice) items spread over the CTAs so that each
//   SM streams the same number of bytes per layer; matrices with few row tiles (qkv 9, o 7, down 7) split K and
//   write raw partial sums, folded IN SLICE ORDER by their consumer (bit-reproducible, no atomics).  gate/up keeps
//   K whole (SwiGLU is not linear) on its own set of CTAs.
//   Phases of a layer (grid barrier between them):
//       [fold+RMSNorm] qkv -> RoPE/KV-append + split-KV attention -> merge + o_proj -> [fold+RMSNorm] gate/up+SwiGLU
//       -> down
//     batch <= 4: the consumers fold the split-K slices and normalise while staging their B operand (5 barriers per
//     layer); larger batches: token-owner CTAs fold + normalise into bf16 rows that the consumers fetch by TMA
//     (7 barriers per layer, no per-CTA re-reading of the whole batch).
//   lm_head epilogue: logits -> HBM once, plus the processed maximum of every 128-row tile; the sampler then needs
//   only the top_k tiles with the largest maxima (provably a superset of the top-k logits), so selection costs
//   ~10 us on one CTA per sequence instead of a pass over the vocabulary.
//
// Replaces transformers generation/utils.py:2743-2805 + modeling_qwen2.py:280-309,353-413 for the decode loop
// (SURVEY.md §8a rows A1, A3-A12); up to batch 16 it takes the place of the 196-launch per-op chain.
#define NT_WGMMA_KERNELS
#include "lm_device.cuh"
#include "lm_decode_tc.cuh"

#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace nt {

// ------------------------------------------------------------------------------------------ small device helpers
NT_DEVINL unsigned tc_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
NT_DEVINL long long tc_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// (value, stamp) pairs: relaxed gpu-scope loads (served by L2, never by a stale L1 line)
NT_DEVINL float4 ldp2(const float2* p) {
  float4 v;
  asm volatile("ld.relaxed.gpu.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
NT_DEVINL float2 ldp1(const float2* p) {
  float2 v;
  asm volatile("ld.relaxed.gpu.global.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}
NT_DEVINL uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}
NT_DEVINL void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
NT_DEVINL void bar_epi() { asm volatile("bar.sync 2, 128;" ::: "memory"); }  // the four epilogue warps

struct TcProf {   // timeline of one CTA: buf[n] = %globaltimer, buf[512 + n] = mark id
  long long* buf;
  int n;
  bool fine;     // fine-grained marks on (one chosen layer)
  NT_DEVINL void mark(int id = 0) {
    if (buf && n < 512) buf[n] = tc_ns(), buf[512 + n] = id, ++n;
  }
};

// bf16 hi/lo split of an fp32 value: hi = rn(x), lo = rn(x - hi); hi + lo carries ~16 mantissa bits
NT_DEVINL void split_hilo(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16(x);
  lo = __float2bfloat16(x - __bfloat162float(hi));
}
// element (row n, k) of a K-major SWIZZLE_128B chunk [rows][64 bf16]: 16-byte group g = k / 8 sits at g ^ (n & 7)
NT_DEVINL __nv_bfloat16* chunk_elem(uint8_t* chunk, int n, int k) {
  return reinterpret_cast<__nv_bfloat16*>(chunk + n * 128 + ((((k >> 3) ^ (n & 7)) << 4) | ((k & 7) << 1)));
}


NT_DEVINL void tc_spin_check(uint32_t& spins, const char* what) {
  if (++spins > (1u << 22)) nt_timeout(what);
}

// 4 consecutive elements of row b: residual pairs (or nothing) + the split-K slices in slice order; polls the stamps
NT_DEVINL void tc_fold4(const float2* hsrc, int hstamp, const float2* parts, int nparts, int pstamp, int rows, int B, int H, int b,
                        int i4, float (&acc)[4]) {
  acc[0] = acc[1] = acc[2] = acc[3] = 0.f;
  if (hsrc) {
    uint32_t spins = 0;
    for (;;) {
      const float4 a0 = ldp2(hsrc + static_cast<long long>(b) * H + i4), a1 = ldp2(hsrc + static_cast<long long>(b) * H + i4 + 2);
      if (__float_as_int(a0.y) == hstamp && __float_as_int(a0.w) == hstamp && __float_as_int(a1.y) == hstamp &&
          __float_as_int(a1.w) == hstamp) {
        acc[0] = a0.x, acc[1] = a0.z, acc[2] = a1.x, acc[3] = a1.z;
        break;
      }
      tc_spin_check(spins, "the residual stream");
    }
  }
  for (int s0 = 0; s0 < nparts; s0 += 8) {
    float4 t0[8], t1[8];
    uint32_t spins = 0;
    for (;;) {
      bool ok = true;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (s0 + j < nparts) {
          const float2* p = parts + (static_cast<long long>(s0 + j) * B + b) * rows + i4;
          t0[j] = ldp2(p), t1[j] = ldp2(p + 2);
        } else {
          t0[j] = t1[j] = make_float4(0.f, __int_as_float(pstamp), 0.f, __int_as_float(pstamp));
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        ok = ok && __float_as_int(t0[j].y) == pstamp && __float_as_int(t0[j].w) == pstamp && __float_as_int(t1[j].y) == pstamp &&
             __float_as_int(t1[j].w) == pstamp;
      if (ok) break;
      tc_spin_check(spins, "split-K slices");
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[0] += t0[j].x, acc[1] += t0[j].z, acc[2] += t1[j].x, acc[3] += t1[j].z;
  }
}

constexpr int kPhQ = 0, kPhO = 1, kPhG = 2, kPhD = 3;
constexpr int kAttWarpsMax = 4;   // most warps that walk KV pages in the attention phase


// shared-memory misc block (after the ring and the union region)
struct TcMisc {
  uint64_t full_bar[16];
  uint64_t empty_bar[16];
  uint64_t bop_bar;
  uint64_t acc_full;      // the accumulator tile in shared memory is written (MMA warpgroup -> epilogue warps)
  uint64_t acc_empty;     // ... and has been read
  uint64_t att_bar[kAttWarpsMax];
  uint64_t go_bar;        // step gate of the stream / MMA warps: one completion per released decode step
  int stop;               // set before the last completion: leave instead of running the step
  int pos[kTcMaxBatch];   // this step's seq_lens snapshot
  int apage[32];          // physical pages of this CTA's attention split (this step)
  int mask_eos[kTcMaxBatch];
  float inv_t[kTcMaxBatch];   // 1 / temperature per sequence (the launch's sampling controls)
  float red[64];
  float tile_max[2][4][kTcMaxBatch];
  float rstd[8];
  int sel[8];
  int nchunks[4];         // B-operand chunks of this CTA's items per split phase
  int ckb[4][16];         // k-block staged in chunk c (qkv / down: k-block of the input; o_proj: head)
  TcPlan plan;
};

// Attention staging (AW = 2 or 4 page-walking warps, TcParams::att_warps): every warp owns a K page + V page buffer
// (SWIZZLE_128B, filled by TMA; 8 KB each => 1024-byte aligned) and walks the pages of this CTA's split independently;
// per-warp partial outputs merge through shared memory.  Layout behind att_off:
//   K[AW][8 KB] | V[AW][8 KB] | o[AW][8][64] f32 | ml[AW][8][2] f32 | q[8][64] f32 | knew[64] | vnew[64]
__host__ __device__ constexpr size_t tc_attn_layout_bytes(int aw) {
  return size_t(2) * aw * 8192 + (size_t(aw) * 8 * 64 + size_t(aw) * 8 * 2 + 8 * 64 + 128) * 4;
}

// ------------------------------------------------------------------------------------------ the kernel
template <int NT, bool HILO, bool FOLD>
__global__ void __launch_bounds__(kTcThreads, 1) decode_tc_kernel(const __grid_constant__ TcParams P) {
  constexpr int CHUNK = NT * 128;            // bytes of one B-operand k-block
  constexpr int NTOK = HILO ? 8 : NT;        // token slots on the N axis
  constexpr int ACC_LD = NT + 4;             // fp32 row stride of the accumulator tile in shared memory
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  uint8_t* ring = smem;
  uint8_t* uni = smem + P.uni_off;
  TcMisc* ms = reinterpret_cast<TcMisc*>(smem + P.misc_off);
  float* accs = reinterpret_cast<float*>(smem + P.acc_off);   // [128][ACC_LD]
  const int tid = threadIdx.x, warp = uniform(tid >> 5), lane = tid & 31;
  const int NS = P.nstages;
  const int L = P.n_layers;
  const int B = P.B;
  const int H = P.hidden;
  const int KBH = H >> 6;                    // k-blocks of a hidden-sized K
  const CUtensorMap* wmaps = reinterpret_cast<const CUtensorMap*>(P.wmaps);
  const CUtensorMap* xmap = reinterpret_cast<const CUtensorMap*>(P.xmap);
  const CUtensorMap* amap = reinterpret_cast<const CUtensorMap*>(P.amap);

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&ms->full_bar[s], 1);
      mbar_init(&ms->empty_bar[s], 4);   // one arrival per MMA warp
    }
    mbar_init(&ms->bop_bar, 1);
    mbar_init(&ms->acc_full, 4);         // the four MMA warps
    mbar_init(&ms->acc_empty, 4);        // the four epilogue warps
    for (int i = 0; i < kAttWarpsMax; ++i) mbar_init(&ms->att_bar[i], 1);
    mbar_init(&ms->go_bar, 1);
    fence_barrier_init();
    ms->stop = 0;
    mbar_arrive(&ms->go_bar);   // step 0 is released from the start
  }
  for (int i = tid; i < static_cast<int>(sizeof(TcPlan) / 4); i += kTcThreads)
    reinterpret_cast<int*>(&ms->plan)[i] = reinterpret_cast<const int*>(P.plan + blockIdx.x)[i];
  if (tid < B) ms->inv_t[tid] = row_sampling(P.samp, tid).inv_t;
  __syncthreads();
  const TcPlan& plan = ms->plan;
  if (tid < 4) {  // chunk tables of the split phases (items in plan order, k-blocks ascending)
    int c = 0;
    for (int i = 0; i < plan.n[tid]; ++i)
      for (int kb = 0; kb < plan.it[tid][i].nkb && c < 16; ++kb, ++c) ms->ckb[tid][c] = plan.it[tid][i].kb0 + kb;
    ms->nchunks[tid] = c;
  } else if (tid == 4) {   // this CTA's positions in the lm_head tile list
    ms->plan.head_t0 = static_cast<int>((static_cast<long long>(P.head_n) * blockIdx.x) / gridDim.x);
    ms->plan.head_t1 = static_cast<int>((static_cast<long long>(P.head_n) * (blockIdx.x + 1)) / gridDim.x);
  }
  __syncthreads();
  const int n_head_tiles = plan.head_t1 - plan.head_t0;
  // position in the lm_head tile list -> row tile (the identity while the vocabulary range is off)
  auto head_tile = [&](int v) -> int {
    return v == P.head_eos_at ? P.head_eos : P.head_lo + v - (P.head_eos_at >= 0 && v > P.head_eos_at ? 1 : 0);
  };

  // stream / MMA warps (whole warp): released one decode step at a time, so that an early exit (every sequence done)
  // never leaves bulk copies in flight.  An mbarrier phase per step; `stop` is written before the releasing arrive.
  auto wait_go = [&](int step) -> bool {
    mbar_wait(&ms->go_bar, static_cast<uint32_t>(step) & 1u);
    return *reinterpret_cast<volatile int*>(&ms->stop) == 0;
  };
  if (warp == kTcStreamWarp) {
    // ================================================================== weight stream
    // The whole warp walks the plan (warp-uniform control flow); one elected lane issues the copies.  elect.sync is
    // re-executed at every use: it is also the point where the lanes RECONVERGE after a data-dependent wait loop --
    // the compiler emits the TMA / MMA instruction itself unpredicated (only its operand moves are predicated), so a
    // lane group that reached it without the leader would issue it with stale operands.
    // weights pass through L2 once per step: evict_first keeps KV pages, hand-off buffers and logits resident
    const uint64_t wpolicy = P.weights_evict_first ? l2_policy_evict_first() : 0ull;
    int slot = 0;
    uint32_t par = 0;       // parity of the slot's NEXT completion of empty_bar that we must have seen
    bool wrapped = false;   // ring used at least once
    auto push = [&](const CUtensorMap* m, int kcol, int row) {
      if (wrapped) mbar_wait(&ms->empty_bar[slot], par ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&ms->full_bar[slot], 16384);
        if (wpolicy) tma_load_2d_hint(ring + static_cast<size_t>(slot) * 16384, m, kcol, row, &ms->full_bar[slot], wpolicy);
        else tma_load_2d(ring + static_cast<size_t>(slot) * 16384, m, kcol, row, &ms->full_bar[slot]);
      }
      if (++slot == NS) slot = 0, par ^= 1, wrapped = true;
    };
    for (int step = 0; step < P.n_steps; ++step) {
      if (!wait_go(step)) break;
      for (int l = 0; l < L; ++l)
        for (int ph = 0; ph < 4; ++ph) {
          const CUtensorMap* m = wmaps + 4 * l + ph;
          const int n_it = uniform(plan.n[ph]);
          for (int i = 0; i < n_it; ++i) {
            const int tile = uniform(plan.it[ph][i].tile), kb0 = uniform(plan.it[ph][i].kb0), nkb = uniform(plan.it[ph][i].nkb);
            for (int kb = 0; kb < nkb; ++kb) push(m, (kb0 + kb) * 64, tile * 128);
          }
        }
      const CUtensorMap* hm = wmaps + 4 * P.total_layers;
      const int t0 = uniform(plan.head_t0), t1 = uniform(plan.head_t1);
      for (int t = t0; t < t1; ++t) {
        const int row0 = uniform(head_tile(t)) * 128;
        for (int kb = 0; kb < KBH; ++kb) push(hm, kb * 64, row0);
      }
    }
  } else if (warp >= kTcMmaWarp0) {
    // ================================================================== MMA warpgroup (warps kTcMmaWarp0 .. + 3)
    // acc0 = weight rows [0, 64) of the tile, acc1 = rows [64, 128).  One k-block's MMAs form a commit group; a ring
    // slot is released (one arrival per warp) once the next group has been issued and the older one retired.
    int slot = 0;
    uint32_t par = 0;
    uint32_t bop_n = 0, acc_n = 0;
    const uint32_t bop_addr = smem_u32(uni);
    const uint32_t ring_addr = smem_u32(ring);
    // one item: nkb ring tiles against B chunks chunk0, chunk0 + 1, ...
    auto run_item = [&](int nkb, int chunk0) {
      float acc0[NT / 2], acc1[NT / 2];
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc0[i] = acc1[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&ms->full_bar[slot], par);
        const uint64_t adesc = wgmma_desc_sw128(ring_addr + static_cast<uint32_t>(slot) * 16384u);
        const uint64_t bdesc = wgmma_desc_sw128(bop_addr + static_cast<uint32_t>(chunk0 + kb) * CHUNK);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_bf16<NT>(acc0, adesc + 2 * k, bdesc + 2 * k, 1u);
          wgmma_bf16<NT>(acc1, adesc + 512 + 2 * k, bdesc + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&ms->empty_bar[prev]);
        }
        prev = slot;
        if (++slot == NS) slot = 0, par ^= 1;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      __syncwarp();
      if (prev >= 0 && lane == 0) mbar_arrive(&ms->empty_bar[prev]);
      mbar_wait(&ms->acc_empty, (acc_n & 1) ^ 1);
      wgmma_store_rows<NT>(acc0, accs, ACC_LD, 0);
      wgmma_store_rows<NT>(acc1, accs, ACC_LD, 64);
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->acc_full);
      ++acc_n;
    };
    const int gu_split = uniform(plan.gu_split);
    const int n_head = uniform(n_head_tiles);
    for (int step = 0; step < P.n_steps; ++step) {
      if (!wait_go(step)) break;
      for (int l = 0; l < L; ++l)
        for (int ph = 0; ph < 4; ++ph) {
          const int n_it = uniform(plan.n[ph]);
          if (n_it == 0) continue;
          mbar_wait(&ms->bop_bar, bop_n & 1);
          ++bop_n;
          int chunk = 0;
          for (int i = 0; i < n_it; ++i) {
            const int nkb = uniform(plan.it[ph][i].nkb);
            if (ph == kPhG && !gu_split) {
              run_item(nkb, 0);   // whole K, all items share the staged input
            } else {
              run_item(nkb, chunk);
              chunk += nkb;
            }
          }
        }
      if (n_head > 0) {
        mbar_wait(&ms->bop_bar, bop_n & 1);
        ++bop_n;
        for (int t = 0; t < n_head; ++t) run_item(KBH, 0);
      }
    }
  } else {
    // ================================================================== worker warps 0..7
    const SyncConsumers csync;
    const unsigned G = gridDim.x;
    unsigned target = 0;
    uint32_t acc_n = 0;
    TcProf prof{nullptr, 0, false};
    auto pm = [&](int id) { if (tid == 0 && prof.fine) prof.mark(id); };
    const int n_rep = P.n_heads / P.n_kv;
    const int split_cap = P.split_cap;
    constexpr bool fold_cta = FOLD;   // batch <= 4: consumers fold the split-K slices themselves (no fold phases, no barriers)
    const int I = P.inter;
    float* xf = reinterpret_cast<float*>(uni + 14 * CHUNK);   // fold_in_cta: fp32 folded rows [B][H] behind the B chunks
    float* xw = xf + 4096;                                      // ... and the RMSNorm weight row [H] (H <= 1024)
    const int AW = P.att_warps;
    uint8_t* att = smem + P.att_off;
    auto att_k = [&](int w) { return reinterpret_cast<__nv_bfloat16*>(att + static_cast<size_t>(w) * 8192); };
    auto att_v = [&](int w) { return reinterpret_cast<__nv_bfloat16*>(att + static_cast<size_t>(AW + w) * 8192); };
    float* att_o = reinterpret_cast<float*>(att + static_cast<size_t>(2 * AW) * 8192);   // [AW][8][64]
    float* att_ml = att_o + AW * 8 * 64;                                                  // [AW][8][2]
    float* att_q = att_ml + AW * 8 * 2;                                                   // [8][64]
    float* att_knew = att_q + 8 * 64;
    float* att_vnew = att_knew + 64;
    const bool att_separate = P.att_off != P.uni_off;   // dedicated staging: KV pages are fetched ahead of the phase
    int fold_no = 0;   // fold_in_cta: folds done in this launch (ping-pong parity + stamp of the residual stream)

    // ---- grid barrier; `post` runs on thread 0 between the release and the trailing CTA barrier
    auto grid_sync = [&](auto post) {   // post runs on the whole of warp 0 (it issues TMA under elect_one())
      csync();
      if (warp == 0) {
        target += G;
        if (lane == 0) {
          __threadfence();
          atomicAdd(P.gbar, 1u);
          uint32_t spins = 0;
          while (tc_ld_acquire(P.gbar) < target) {
            if (++spins > (1u << 24)) nt_timeout("the grid barrier");
          }
          prof.mark(200);
        }
        __syncwarp();
        post();
      }
      csync();
    };
    auto no_post = [] {};
    auto stamp_of = [&](int step, int l) { return P.stamp_base + step * (L + 1) + l + 1; };

    // ---- B operand by TMA from global bf16 rows (thread 0, after the barrier that published them)
    //      (whole warp 0, converged: one elected lane issues)
    auto load_bop_split = [&](const CUtensorMap* m, int ph) {   // chunks of the items' own k ranges, item after item
      const int n = uniform(plan.n[ph]);
      if (n == 0) return;
      const int nch = uniform(ms->nchunks[ph]);
      if (elect_one()) {   // no wait inside: one election covers the whole batch of copies
        fence_proxy_async_all();
        mbar_arrive_expect_tx(&ms->bop_bar, static_cast<uint32_t>(nch) * CHUNK);
        for (int c = 0; c < nch; ++c) tma_load_2d(uni + c * CHUNK, m, ms->ckb[ph][c] * 64, 0, &ms->bop_bar);
      }
    };
    auto load_bop_full = [&](const CUtensorMap* m, bool need) {  // all KBH chunks of the hidden-sized K
      if (!uniform(need ? 1 : 0)) return;
      if (elect_one()) {
        fence_proxy_async_all();
        mbar_arrive_expect_tx(&ms->bop_bar, static_cast<uint32_t>(KBH) * CHUNK);
        for (int kb = 0; kb < KBH; ++kb) tma_load_2d(uni + kb * CHUNK, m, kb * 64, 0, &ms->bop_bar);
      }
    };
    // thread-staged B operand is complete: every writer fenced its writes towards the async proxy
    auto bop_ready = [&] {
      fence_proxy_async();
      csync();
      if (tid == 0) mbar_arrive(&ms->bop_bar);
    };

    // ---- accumulator of the next item -> registers (epilogue warps 0..3; lane = weight row of the tile)
    auto acc_take = [&](float (&v)[NT]) {
      mbar_wait(&ms->acc_full, acc_n & 1);
      const float4* src = reinterpret_cast<const float4*>(accs + (warp * 32 + lane) * ACC_LD);
#pragma unroll
      for (int j = 0; j < NT / 4; ++j) {
        const float4 t = src[j];
        v[4 * j] = t.x, v[4 * j + 1] = t.y, v[4 * j + 2] = t.z, v[4 * j + 3] = t.w;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->acc_empty);
      ++acc_n;
      if constexpr (HILO) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += v[j + 8];
      }
    };

    // ---- epilogue of the split-K phases: raw partial sums as (value, stamp) pairs, one row per lane
    auto epi_partials = [&](int ph, float2* part, int rows, int stamp) {
      if (warp >= 4) return;
      const float sf = __int_as_float(stamp);
      for (int i = 0; i < plan.n[ph]; ++i) {
        const TcItem it = plan.it[ph][i];
        float v[NT];
        acc_take(v);
        pm(10);
        const int row = it.tile * 128 + warp * 32 + lane;
        if (row < rows) {
          float2* dst = part + (static_cast<long long>(it.slice) * B) * rows + row;
#pragma unroll
          for (int n = 0; n < NTOK; ++n)
            if (n < B) dst[static_cast<long long>(n) * rows] = make_float2(v[n], sf);
        }
      }
    };

    // ---- batch > 4: fold + RMSNorm of ONE token row by its owner CTA -> residual stream (fp32) + normalised bf16 rows
    auto fold_phase = [&](const float2* parts, int nparts, int pstamp, int rows, const float* norm_w) {
      const int b = blockIdx.x;
      if (b >= B) return;
      float* hb = P.h + static_cast<long long>(b) * H;
      float ss = 0.f;
      for (int i4 = tid * 4; i4 < H; i4 += 4 * kConsumerThreads) {
        float acc[4];
        tc_fold4(nullptr, 0, parts, nparts, pstamp, rows, B, H, b, i4, acc);
        const float4 hv = __ldcg(reinterpret_cast<const float4*>(hb + i4));
        acc[0] += hv.x, acc[1] += hv.y, acc[2] += hv.z, acc[3] += hv.w;
        *reinterpret_cast<float4*>(hb + i4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        ss += acc[0] * acc[0] + acc[1] * acc[1] + acc[2] * acc[2] + acc[3] * acc[3];
      }
      ss = warp_sum(ss);
      if (lane == 0) ms->red[warp] = ss;
      csync();
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kConsumerWarps; ++w) t += ms->red[w];
      const float sc = rsqrtf(t / static_cast<float>(H) + P.eps);
      for (int i4 = tid * 4; i4 < H; i4 += 4 * kConsumerThreads) {
        const float4 hv = *reinterpret_cast<const float4*>(hb + i4);   // this thread's own stores above
        const float4 g = __ldg(reinterpret_cast<const float4*>(norm_w + i4));
        const float xn[4] = {g.x * (hv.x * sc), g.y * (hv.y * sc), g.z * (hv.z * sc), g.w * (hv.w * sc)};
        if constexpr (HILO) {
          __nv_bfloat16 hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) split_hilo(xn[j], hi[j], lo[j]);
          *reinterpret_cast<uint2*>(P.xa + static_cast<long long>(b) * H + i4) =
              make_uint2(pack2(hi[0], hi[1]), pack2(hi[2], hi[3]));
          *reinterpret_cast<uint2*>(P.xa + static_cast<long long>(8 + b) * H + i4) =
              make_uint2(pack2(lo[0], lo[1]), pack2(lo[2], lo[3]));
        } else {
          *reinterpret_cast<uint2*>(P.xa + static_cast<long long>(b) * H + i4) =
              make_uint2(pack_bf16x2(xn[0], xn[1]), pack_bf16x2(xn[2], xn[3]));
        }
      }
    };

    // ---- batch <= 4: fold ALL rows in this CTA (residual pairs + slices, slice order), normalise, stage the B chunks
    //      of phase `ph` (-1: every k-block).  The designated CTA publishes the folded stream for the next fold.
    auto fold_stage = [&](const float2* parts, int nparts, int pstamp, int rows, const float* norm_w, int ph, bool writer) {
      const float2* hsrc = P.h2 + static_cast<long long>(fold_no & 1) * B * H;
      const int hstamp = P.hstamp_base + fold_no;
      const int nq = H >> 2;
      pm(1);
      float ssb[4] = {0.f, 0.f, 0.f, 0.f};   // this thread's share of every row's sum of squares
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < B) {
          for (int q = tid; q < nq; q += kConsumerThreads) {
            const int i4 = q * 4;
            float acc[4];
            const float4 nw = __ldg(reinterpret_cast<const float4*>(norm_w + i4));   // in flight together with the slices
            tc_fold4(hsrc, hstamp, parts, nparts, pstamp, rows, B, H, b, i4, acc);
            *reinterpret_cast<float4*>(xf + b * H + i4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
            if (b == 0) *reinterpret_cast<float4*>(xw + i4) = nw;
            ssb[b] += (acc[0] * acc[0] + acc[1] * acc[1]) + (acc[2] * acc[2] + acc[3] * acc[3]);
          }
        }
      }
      pm(2);
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < B) {
          const float t = warp_sum(ssb[b]);
          if (lane == 0) ms->red[b * kConsumerWarps + warp] = t;
        }
      }
      csync();
      float rs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < B) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < kConsumerWarps; ++w) t += ms->red[b * kConsumerWarps + w];   // fixed order: every CTA gets the same bits
          rs[b] = rsqrtf(t / static_cast<float>(H) + P.eps);
        }
      }
      const int nch = ph < 0 ? KBH : ms->nchunks[ph];
      const int per = B * 64;
      for (int e = tid; e < nch * per; e += kConsumerThreads) {
        const int c = e / per, r = e - c * per, b = r >> 6, k = r & 63;
        const int i = (ph < 0 ? c : ms->ckb[ph][c]) * 64 + k;
        const float rstd = b == 0 ? rs[0] : (b == 1 ? rs[1] : (b == 2 ? rs[2] : rs[3]));
        const float xn = xw[i] * (xf[b * H + i] * rstd);
        __nv_bfloat16 hi, lo;
        split_hilo(xn, hi, lo);
        uint8_t* cb = uni + c * CHUNK;
        *chunk_elem(cb, b, k) = hi;
        *chunk_elem(cb, 8 + b, k) = lo;
      }
      pm(4);
      bop_ready();
      pm(5);
      if (writer) {
        float2* hdst = P.h2 + static_cast<long long>((fold_no + 1) & 1) * B * H;
        const float sf = __int_as_float(hstamp + 1);
        for (int q = tid; q < B * nq; q += kConsumerThreads) {
          const float4 v = *reinterpret_cast<const float4*>(xf + q * 4);
          float4* d = reinterpret_cast<float4*>(hdst + q * 4);
          d[0] = make_float4(v.x, sf, v.y, sf);
          d[1] = make_float4(v.z, sf, v.w, sf);
        }
      }
      ++fold_no;
    };

    // ---- attention item of this CTA: (sequence, kv head, split)
    const int per_b = P.n_kv * split_cap;
    const int my_b = blockIdx.x / per_b, my_kvh = (blockIdx.x % per_b) / split_cap, my_split = blockIdx.x % split_cap;

    uint32_t att_par = 0;   // parity of this warp's page barrier (warps 0..3)
    const CUtensorMap* kvmap = &P.kvmap;
    // physical page of logical page pg of this CTA's split (cached at step start)
    auto page_of = [&](int pg, int p0) -> int {
      return (pg - p0 < 32) ? ms->apage[pg - p0] : __ldcg(P.kv.page_table + my_b * P.kv.max_pages_per_seq + pg);
    };
    auto cache_pages = [&] {   // after ms->pos is set (and a barrier); followed by a barrier
      if (my_b >= B || tid >= 32) return;
      const SplitGeom geo = split_geom(ms->pos[my_b], P.kv.max_ctx, split_cap);
      if (my_split >= geo.nsplit) return;
      const int p0 = my_split * geo.pps, p1 = min(p0 + geo.pps, geo.npages);
      if (p0 + tid < p1) ms->apage[tid] = __ldcg(P.kv.page_table + my_b * P.kv.max_pages_per_seq + p0 + tid);
    };
    // lane 0 of an attention warp: K and V page of (sequence, kv head) -> this warp's buffers
    //   (whole attention warp, converged; fence: see the proxy fence after the sampler's grid barrier)
    auto issue_page = [&](int l, int pg, int p0, bool fence) {
      const int krow0 = l * 2 * P.kv.num_pages * P.kv.n_kv_heads * 64;
      const int vrow0 = krow0 + P.kv.num_pages * P.kv.n_kv_heads * 64;
      const int page = uniform(page_of(pg, p0));
      if (elect_one()) {
        if (fence) fence_proxy_async_all();
        mbar_arrive_expect_tx(&ms->att_bar[warp], 2 * 8192);
        tma_load_2d(att_k(warp), kvmap, 0, krow0 + (page * P.kv.n_kv_heads + my_kvh) * 64, &ms->att_bar[warp]);
        tma_load_2d(att_v(warp), kvmap, 0, vrow0 + (page * P.kv.n_kv_heads + my_kvh) * 64, &ms->att_bar[warp]);
      }
    };
    // dedicated staging: the first round of pages of layer l is fetched before the layer's projections run (they do
    // not depend on them: the new token's row is patched into the staged page)
    auto attn_prefetch = [&](int l) {
      if (!att_separate || my_b >= B || warp >= AW) return;
      const SplitGeom geo = split_geom(uniform(ms->pos[my_b]), P.kv.max_ctx, split_cap);
      if (my_split >= geo.nsplit) return;
      const int p0 = my_split * geo.pps, p1 = min(p0 + geo.pps, geo.npages);
      // no proxy fence here: the rows these pages hold were written in EARLIER steps (this step's row is patched in
      // shared memory) and every step starts behind a grid barrier + proxy fence
      if (p0 + warp < p1) issue_page(l, p0 + warp, p0, false);
    };
    auto attention_phase = [&](int l, int stamp) {
      if (my_b >= B) return;
      const int pos = uniform(ms->pos[my_b]);
      const SplitGeom geo = split_geom(pos, P.kv.max_ctx, split_cap);
      if (my_split >= geo.nsplit) return;
      const int b = my_b, kvh = my_kvh;
      const int p0 = my_split * geo.pps, p1 = min(p0 + geo.pps, geo.npages);
      const bool appends = pos < P.kv.max_ctx && (pos >> 6) >= p0 && (pos >> 6) < p1;
      if (!att_separate) {
        // the pages do not depend on this layer's projections (the new row is patched in below): fetch the first round now
        csync();   // the union region is ours (previous phase of this CTA is through with it)
        if (warp < AW && p0 + warp < p1) issue_page(l, p0 + warp, p0, true);
      }
      pm(21);
      // prologue: fold the qkv slices (slice order) + bias, RoPE; q of the group -> shared; new K/V row
      const float* bias = P.bqkv[l];
      const int QN = P.qkv_n;
      const float2* pq = P.pq2 + static_cast<long long>(b) * QN;
      const long long sstride = static_cast<long long>(B) * QN;
      for (int idx = tid; idx < n_rep * 32 + 64; idx += kConsumerThreads) {
        int row0;
        const int which = idx < n_rep * 32 ? 0 : (idx < n_rep * 32 + 32 ? 1 : 2);
        const int i = idx & 31;
        if (which == 0) row0 = (kvh * n_rep + (idx >> 5)) * 64 + 2 * i;
        else if (which == 1) row0 = (P.n_heads + kvh) * 64 + 2 * i;
        else row0 = (P.n_heads + P.n_kv + kvh) * 64 + 2 * i;
        if (which != 0 && !appends) continue;
        const float2 bia = __ldg(reinterpret_cast<const float2*>(bias + row0));
        float sn = 0.f, cs = 1.f;
        if (which != 2) sincosf(static_cast<float>(pos) * __ldg(P.inv_freq + i), &sn, &cs);
        float2 a = make_float2(0.f, 0.f);
        for (int s0 = 0; s0 < P.sq; s0 += 8) {
          float4 t[8];
          uint32_t spins = 0;
          for (;;) {
            bool ok = true;
#pragma unroll
            for (int j = 0; j < 8; ++j)
              t[j] = (s0 + j < P.sq) ? ldp2(pq + (s0 + j) * sstride + row0) : make_float4(0.f, __int_as_float(stamp), 0.f, __int_as_float(stamp));
#pragma unroll
            for (int j = 0; j < 8; ++j) ok = ok && __float_as_int(t[j].y) == stamp && __float_as_int(t[j].w) == stamp;
            if (ok) break;
            tc_spin_check(spins, "qkv slices");
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) a.x += t[j].x, a.y += t[j].z;
        }
        a.x += bia.x, a.y += bia.y;
        if (which == 2) {
          att_vnew[2 * i] = a.x, att_vnew[2 * i + 1] = a.y;
        } else {
          const float lo = a.x * cs - a.y * sn, hi = a.y * cs + a.x * sn;   // rows (2i, 2i+1) = dims (i, i + 32)
          if (which == 0) att_q[(idx >> 5) * 64 + i] = lo, att_q[(idx >> 5) * 64 + i + 32] = hi;
          else att_knew[i] = lo, att_knew[i + 32] = hi;
        }
      }
      pm(22);
      csync();
      if (appends && tid >= 128 && tid < 192) {  // the new token's K/V row joins the cache (bf16) for the steps to come
        const int d = tid - 128;
        const int page = page_of(pos >> 6, p0);
        P.kv.page_ptr(l, 0, page, kvh)[(pos & 63) * 64 + d] = __float2bfloat16(att_knew[d]);
        P.kv.page_ptr(l, 1, page, kvh)[(pos & 63) * 64 + d] = __float2bfloat16(att_vnew[d]);
      }
      if (warp < AW) {
        const int g = lane >> 2, t = lane & 3, lrow = lane & 7, lmat = lane >> 3;
        // query fragments: row g = head g of the group (rows >= n_rep and rows 8..15 are zero); scale * log2(e) folded in
        uint32_t qa[4][4];
        {
          const float* qp = att_q + min(g, n_rep - 1) * 64;
          const float sc = (g < n_rep) ? P.scale_log2 : 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 a0 = *reinterpret_cast<const float2*>(qp + 16 * j + 2 * t);
            const float2 a2 = *reinterpret_cast<const float2*>(qp + 16 * j + 8 + 2 * t);
            qa[j][0] = pack_bf16x2(a0.x * sc, a0.y * sc);
            qa[j][1] = 0u;
            qa[j][2] = pack_bf16x2(a2.x * sc, a2.y * sc);
            qa[j][3] = 0u;
          }
        }
        float o[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
        float m0 = -INFINITY, l0 = 0.f;
        const uint32_t kbase = smem_u32(att_k(warp)), vbase = smem_u32(att_v(warp));
        for (int pg = p0 + warp; pg < p1; pg += AW) {
          mbar_wait(&ms->att_bar[warp], att_par);
          att_par ^= 1;
          if (warp == 0) pm(23);
          if (appends && pg == (pos >> 6)) {  // patch the staged page with the new row (the copy may predate our store)
            const int r = pos & 63;
            uint8_t* kb8 = reinterpret_cast<uint8_t*>(att_k(warp));
            uint8_t* vb8 = reinterpret_cast<uint8_t*>(att_v(warp));
            *reinterpret_cast<uint32_t*>(chunk_elem(kb8, r, 2 * lane)) = pack_bf16x2(att_knew[2 * lane], att_knew[2 * lane + 1]);
            *reinterpret_cast<uint32_t*>(chunk_elem(vb8, r, 2 * lane)) = pack_bf16x2(att_vnew[2 * lane], att_vnew[2 * lane + 1]);
            __syncwarp();
          }
          float sc[8][4];
#pragma unroll
          for (int n = 0; n < 8; ++n) {
            sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
            const int row = 8 * n + lrow;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              uint32_t kb[4];
              ldmatrix_x4(kb, kbase + row * 128 + (((4 * half + lmat) ^ lrow) << 4));
              mma_bf16_16816(sc[n], qa[2 * half], kb[0], kb[1]);
              mma_bf16_16816(sc[n], qa[2 * half + 1], kb[2], kb[3]);
            }
          }
          const int k0 = pg * 64;
          if (k0 + 64 > geo.n_ctx) {
#pragma unroll
            for (int n = 0; n < 8; ++n) {
              const int kv0 = k0 + 8 * n + 2 * t;
              if (kv0 >= geo.n_ctx) sc[n][0] = -INFINITY;
              if (kv0 + 1 >= geo.n_ctx) sc[n][1] = -INFINITY;
            }
          }
          float mx = -INFINITY;
#pragma unroll
          for (int n = 0; n < 8; ++n) mx = fmaxf(mx, fmaxf(sc[n][0], sc[n][1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1)), mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float mn = fmaxf(m0, mx);  // the first token of every page walked is valid -> finite
          const float c = exp2f(m0 - mn);
          m0 = mn;
          l0 *= c;
#pragma unroll
          for (int n = 0; n < 8; ++n) o[n][0] *= c, o[n][1] *= c;
          uint32_t pa[4][4];
#pragma unroll
          for (int n = 0; n < 8; ++n) {
            const float p0v = exp2f(sc[n][0] - mn), p1v = exp2f(sc[n][1] - mn);
            l0 += p0v + p1v;
            pa[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p0v, p1v);
            pa[n >> 1][(n & 1) * 2 + 1] = 0u;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int row = 16 * j + 8 * (lmat & 1) + lrow;
#pragma unroll
            for (int nd = 0; nd < 8; nd += 2) {
              uint32_t vb[4];
              ldmatrix_x4_trans(vb, vbase + row * 128 + (((nd + (lmat >> 1)) ^ lrow) << 4));
              mma_bf16_16816(o[nd], pa[j], vb[0], vb[1]);
              mma_bf16_16816(o[nd + 1], pa[j], vb[2], vb[3]);
            }
          }
          __syncwarp();  // all lanes are done with the buffers before they are refilled
          if (pg + AW < p1) issue_page(l, pg + AW, p0, !att_separate);
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1), l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        if (g < n_rep) {
#pragma unroll
          for (int n = 0; n < 8; ++n) *reinterpret_cast<float2*>(att_o + (warp * 8 + g) * 64 + 8 * n + 2 * t) = make_float2(o[n][0], o[n][1]);
          if (t == 0) att_ml[(warp * 8 + g) * 2] = m0, att_ml[(warp * 8 + g) * 2 + 1] = l0;
        }
      }
      csync();
      const float sf = __int_as_float(stamp);
      for (int i = tid; i < n_rep * 64; i += kConsumerThreads) {
        const int h = i >> 6, d = i & 63;
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < kAttWarpsMax; ++w)
          if (w < AW) M = fmaxf(M, att_ml[(w * 8 + h) * 2]);
        float Ls = 0.f, O = 0.f;
#pragma unroll
        for (int w = 0; w < kAttWarpsMax; ++w) {
          if (w < AW) {
            const float wgt = exp2f(att_ml[(w * 8 + h) * 2] - M);   // 0 for a warp that walked no page (m = -inf, l = 0)
            Ls += wgt * att_ml[(w * 8 + h) * 2 + 1];
            O += wgt * att_o[(w * 8 + h) * 64 + d];
          }
        }
        const long long hh = static_cast<long long>(b) * P.n_heads + kvh * n_rep + h;
        P.ao2[(hh * P.max_splits + my_split) * 64 + d] = make_float2(O, sf);
        if (d == 0) *reinterpret_cast<float4*>(P.aml2 + (hh * P.max_splits + my_split) * 2) = make_float4(M, sf, Ls, sf);
      }
      pm(25);
      csync();   // the union region is free again
    };

    // ---- o_proj input: merge the split-KV partials of the heads this CTA's items need, straight into B chunks
    // The B chunks of the previous GEMM phase are free once the epilogue warps have taken its last accumulator: the MMA
    // warpgroup has then retired every wgmma that reads them.  Warps 4..7 skip the epilogue (and a CTA without an
    // attention split skips the attention barriers), so the staging below starts with a consumer barrier.
    auto stage_attn = [&](int stamp) {
      csync();
      const int nch = ms->nchunks[kPhO];
      const int per = B * 64;
      for (int e = tid; e < nch * per; e += kConsumerThreads) {
        const int c = e / per, r = e - c * per, b = r >> 6, d = r & 63;
        const int head = ms->ckb[kPhO][c];
        const SplitGeom g = split_geom(ms->pos[b], P.kv.max_ctx, split_cap);
        const long long hh = static_cast<long long>(b) * P.n_heads + head;
        const float2* ml = P.aml2 + hh * P.max_splits * 2;
        const float2* po = P.ao2 + hh * P.max_splits * 64 + d;
        float4 mv[8];
        float2 ov[8];
        uint32_t spins = 0;
        for (;;) {   // split_cap <= 8: one batch of loads
          bool ok = true;
#pragma unroll
          for (int s = 0; s < 8; ++s)
            if (s < g.nsplit) mv[s] = ldp2(ml + 2 * s), ov[s] = ldp1(po + s * 64);
#pragma unroll
          for (int s = 0; s < 8; ++s)
            if (s < g.nsplit)
              ok = ok && __float_as_int(mv[s].y) == stamp && __float_as_int(mv[s].w) == stamp && __float_as_int(ov[s].y) == stamp;
          if (ok) break;
          tc_spin_check(spins, "attention partials");
        }
        float M = -INFINITY;
#pragma unroll
        for (int s = 0; s < 8; ++s)
          if (s < g.nsplit) M = fmaxf(M, mv[s].x);
        float Ls = 0.f, O = 0.f;
#pragma unroll
        for (int s = 0; s < 8; ++s)
          if (s < g.nsplit) {
            const float wgt = exp2f(mv[s].x - M);
            Ls += wgt * mv[s].z;
            O += wgt * ov[s].x;
          }
        const float val = O / Ls;
        uint8_t* cb = uni + c * CHUNK;
        if constexpr (HILO) {
          __nv_bfloat16 hi, lo;
          split_hilo(val, hi, lo);
          *chunk_elem(cb, b, d) = hi;
          *chunk_elem(cb, 8 + b, d) = lo;
        } else {
          *chunk_elem(cb, b, d) = __float2bfloat16(val);
        }
      }
      pm(31);
      bop_ready();
      pm(32);
    };

    // ---- batch <= 4: down_proj input from the (value, stamp) SwiGLU outputs, two elements per thread
    auto stage_act = [&](int stamp) {
      csync();   // the B chunks of the gate/up phase are free (see stage_attn)
      const int nch = ms->nchunks[kPhD];
      const int per = B * 32;
      for (int e = tid; e < nch * per; e += kConsumerThreads) {
        const int c = e / per, r = e - c * per, b = r >> 5, k = (r & 31) * 2;
        const int kbd = ms->ckb[kPhD][c];
        float4 t;
        if (plan.gu_split) {
          // flat plan: activations j, j + 1 = gate/up rows 2j .. 2j + 3 of tile kbd; fold its K slices (slice order), then SwiGLU
          const int nsl = __ldg(P.gu_nsl + kbd);
          const float2* p = P.pg2 + static_cast<long long>(b) * 2 * I + 2 * (kbd * 64 + k);
          const long long sstride = static_cast<long long>(B) * 2 * I;
          float4 u0[kTcMaxGuSlices], u1[kTcMaxGuSlices];
          uint32_t spins = 0;
          for (;;) {
            bool ok = true;
#pragma unroll
            for (int sl = 0; sl < kTcMaxGuSlices; ++sl)
              if (sl < nsl) u0[sl] = ldp2(p + sl * sstride), u1[sl] = ldp2(p + sl * sstride + 2);
#pragma unroll
            for (int sl = 0; sl < kTcMaxGuSlices; ++sl)
              if (sl < nsl)
                ok = ok && __float_as_int(u0[sl].y) == stamp && __float_as_int(u0[sl].w) == stamp && __float_as_int(u1[sl].y) == stamp &&
                     __float_as_int(u1[sl].w) == stamp;
            if (ok) break;
            tc_spin_check(spins, "gate/up slices");
          }
          float g0 = 0.f, up0 = 0.f, g1 = 0.f, up1 = 0.f;
#pragma unroll
          for (int sl = 0; sl < kTcMaxGuSlices; ++sl)
            if (sl < nsl) g0 += u0[sl].x, up0 += u0[sl].z, g1 += u1[sl].x, up1 += u1[sl].z;
          t.x = silu(g0) * up0, t.z = silu(g1) * up1;
        } else {
          const float2* p = P.act2 + static_cast<long long>(b) * I + kbd * 64 + k;
          uint32_t spins = 0;
          for (;;) {
            t = ldp2(p);
            if (__float_as_int(t.y) == stamp && __float_as_int(t.w) == stamp) break;
            tc_spin_check(spins, "SwiGLU outputs");
          }
        }
        __nv_bfloat16 h0, l0, h1, l1;
        split_hilo(t.x, h0, l0);
        split_hilo(t.z, h1, l1);
        uint8_t* cb = uni + c * CHUNK;
        *reinterpret_cast<uint32_t*>(chunk_elem(cb, b, k)) = pack2(h0, h1);
        *reinterpret_cast<uint32_t*>(chunk_elem(cb, 8 + b, k)) = pack2(l0, l1);
      }
      pm(41);
      bop_ready();
      pm(42);
    };

    // ---- gate/up epilogue: rows (2j, 2j+1) = (gate_j, up_j) on adjacent lanes -> act[b][j] = silu(gate) * up
    auto epi_swiglu = [&](int stamp) {
      if (warp >= 4) return;
      const float sf = __int_as_float(stamp);
      for (int i = 0; i < plan.n[kPhG]; ++i) {
        const TcItem it = plan.it[kPhG][i];
        float v[NT];
        acc_take(v);
        pm(50);
        const int row = it.tile * 128 + warp * 32 + lane;
        const int j = row >> 1;
#pragma unroll
        for (int n = 0; n < NTOK; ++n) {
          const float up = __shfl_down_sync(0xffffffffu, v[n], 1);
          if (n < B && !(lane & 1) && j < I) {
            const float a = silu(v[n]) * up;
            if (fold_cta) {
              P.act2[static_cast<long long>(n) * I + j] = make_float2(a, sf);
            } else if constexpr (HILO) {
              __nv_bfloat16 hi, lo;
              split_hilo(a, hi, lo);
              P.act[static_cast<long long>(n) * I + j] = hi;
              P.act[static_cast<long long>(8 + n) * I + j] = lo;
            } else {
              P.act[static_cast<long long>(n) * I + j] = __float2bfloat16(a);
            }
          }
        }
      }
    };

    // ---- lm_head epilogue: logits -> HBM, processed maximum of the 128-row tile per sequence
    auto epi_head = [&] {
      if (warp >= 4) return;
      const int V = P.vocab;
      const int eos = P.samp.sp.eos_id;
      for (int t = 0; t < n_head_tiles; ++t) {
        const int tile = head_tile(plan.head_t0 + t);
        float v[NT];
        acc_take(v);
        const int row = tile * 128 + warp * 32 + lane;
        const bool ok = row < V;
        const bool allowed = tile != P.head_eos || row == eos;   // the EOS tile outside the vocabulary range: EOS only
        float (*tm)[kTcMaxBatch] = ms->tile_max[t & 1];
        float pv[NTOK];
#pragma unroll
        for (int n = 0; n < NTOK; ++n) {
          pv[n] = -INFINITY;
          if (n < B) {
            if (ok) P.logits[static_cast<long long>(n) * V + row] = allowed ? v[n] : -INFINITY;
            if (ok && allowed && !(ms->mask_eos[n] && row == eos)) pv[n] = v[n] * ms->inv_t[n];
          }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {   // all columns advance together: independent shuffles pipeline
#pragma unroll
          for (int n = 0; n < NTOK; ++n) pv[n] = fmaxf(pv[n], __shfl_xor_sync(0xffffffffu, pv[n], off));
        }
        if (lane == 0) {
#pragma unroll
          for (int n = 0; n < NTOK; ++n)
            if (n < B) tm[warp][n] = pv[n];
        }
        bar_epi();
        if (tid < B) P.tmax[static_cast<long long>(tid) * P.ntiles + tile] = fmaxf(fmaxf(tm[0][tid], tm[1][tid]), fmaxf(tm[2][tid], tm[3][tid]));
        // tile_max is double-buffered by tile parity: the barrier of tile t+1 orders these reads before tile t+2's writes
      }
    };

    // ---- sampler for sequence b = blockIdx.x: top-k tiles by maximum -> their logits >= threshold -> exact top-k
    auto sample_phase = [&] {
      const int b = blockIdx.x;
      if (b >= B) return;
      float2* h2dst = fold_cta ? P.h2 + (static_cast<long long>(fold_no & 1) * B + b) * H : nullptr;
      const float h2stamp = __int_as_float(P.hstamp_base + fold_no);
      // the epilogue stored PROCESSED maxima (temperature, EOS mask): no scale, no tile to fix up
      sample_tiles_seq(P.samp, b, P.tmax, P.ntiles, 1.0f, -1, 0.f, P.logits, P.vocab, ms->mask_eos[b] != 0, uni, P.uni_bytes, ms->sel,
                       csync, pm, h2dst, h2stamp);
    };

    // =============================================================== the decode loop
    if (fold_cta) {  // hand the prefill's residual rows to the stamped ping-pong buffer (stamp of "fold -1")
      if (static_cast<int>(blockIdx.x) < B) {
        const int b = blockIdx.x;
        const float sf = __int_as_float(P.hstamp_base);
        for (int i = tid; i < H; i += kConsumerThreads)
          P.h2[static_cast<long long>(b) * H + i] = make_float2(__ldcg(P.h + static_cast<long long>(b) * H + i), sf);
      }
      grid_sync(no_post);
    }
    for (int step = 0; step < P.n_steps; ++step) {
      if (P.prof && tid == 0 && step == P.prof_step && blockIdx.x < 2) {   // CTA 0 (split phases + attention), CTA 1 (gate/up)
        prof.buf = P.prof + 1024 * blockIdx.x;
        prof.n = 0;
        prof.mark();
      } else {
        prof.buf = nullptr;
      }
      if (tid < B) {
        ms->pos[tid] = __ldcg(P.kv.seq_lens + tid);
        ms->mask_eos[tid] = __ldcg(P.samp.n_generated + tid) < P.samp.sp.min_new_tokens ? 1 : 0;
      }
      csync();
      cache_pages();
      fence_proxy_async_all();   // KV rows appended in earlier steps (generic proxy, behind grid barriers) -> this step's TMA reads
      csync();
      // Both layer loops are written as ONE loop over half-layers / segments with a single call site per building block:
      // the blocks are big inlined lambdas, and a kernel whose layer body does not fit the instruction cache pays for it
      // in every phase (the first version of this loop compiled to 510 KB of SASS).
      if constexpr (FOLD) {
        // ---------------- batch <= 4: no grid barrier inside the layers, every hand-off is polled
        for (int hl = 0; hl <= 2 * L; ++hl) {
          const int l = hl >> 1;
          const bool second = (hl & 1) != 0, head = hl == 2 * L;
          const int st = stamp_of(step, l);
          prof.fine = prof.buf != nullptr && l == 2;
          // fold (residual + split-K slices of the previous GEMM) + RMSNorm + B-operand staging
          const float2* parts = second ? P.po2 : P.pd2;
          const int nparts = second ? P.so : (l > 0 ? P.sd : 0);
          const int pstamp = second ? st : stamp_of(step, l - 1);
          const float* norm_w = head ? P.final_norm : (second ? P.ln2[l] : P.ln1[l]);
          const int sph = head ? -1 : (second ? (plan.gu_split ? kPhG : -1) : kPhQ);
          const bool writer = !head && (second ? plan.fold_g != 0 : plan.fold_q != 0);
          const bool need = head ? n_head_tiles > 0 : plan.n[second ? kPhG : kPhQ] > 0;
          if (!second && !head) attn_prefetch(l);
          if (need) fold_stage(parts, nparts, pstamp, H, norm_w, sph, writer);
          else ++fold_no;
          if (head) break;
          if (second && !plan.gu_split) {
            epi_swiglu(st);
            if (tid == 0) prof.mark(103);
            if (plan.n[kPhD] > 0) stage_act(st);
            epi_partials(kPhD, P.pd2, H, st);
            if (tid == 0) prof.mark(104);
            continue;
          }
          for (int e = 0; e < 2; ++e) {   // the two GEMMs of the half-layer: qkv | o_proj, or gate/up | down
            if (e == 1) {
              if (!second) {
                attention_phase(l, st);
                if (tid == 0) prof.mark(101);
                if (plan.n[kPhO] > 0) stage_attn(st);
              } else if (plan.n[kPhD] > 0) {
                stage_act(st);
              }
            }
            const int ph = (second ? kPhG : kPhQ) + e;   // kPhQ, kPhO | kPhG, kPhD
            float2* part = ph == kPhQ ? P.pq2 : (ph == kPhO ? P.po2 : (ph == kPhG ? P.pg2 : P.pd2));
            const int rows = ph == kPhQ ? P.qkv_n : (ph == kPhG ? 2 * I : H);
            epi_partials(ph, part, rows, st);
            if (tid == 0) prof.mark(100 + ph + (ph > 0 ? 1 : 0));   // 100 qkv, 102 o_proj, 103 gate/up, 104 down
          }
        }
      } else {
        // ---------------- batch > 4: token-owner fold phases feed the consumers by TMA (3 barriers per layer).
        // Segments of a layer, each entered through a grid barrier whose post step fetches the B operand:
        //   0: qkv epilogue, attention, merge + o_proj, fold -> 1: gate/up + SwiGLU -> 2: down_proj, fold
        fold_phase(nullptr, 0, 0, H, L > 0 ? P.ln1[0] : P.final_norm);
        for (int q = 0;; ++q) {
          const int l = q / 3, seg = q - 3 * l;
          const int st = stamp_of(step, l);
          const bool head = l == L;
          {
            const bool full = head || seg == 1;
            const CUtensorMap* m = seg == 2 ? amap : xmap;
            const int lph = seg == 0 ? kPhQ : kPhD;
            const bool need = head ? n_head_tiles > 0 : plan.n[kPhG] > 0;
            grid_sync([&] {
              if (full) load_bop_full(m, need);
              else load_bop_split(m, lph);
            });
          }
          if (head) break;
          prof.fine = prof.buf != nullptr && l == 2;
          if (seg == 1) {
            epi_swiglu(st);
            if (tid == 0) prof.mark(103);
            continue;
          }
          for (int e = (seg == 0 ? 0 : 1); e < 2; ++e) {   // segment 0: qkv then o_proj; segment 2: down_proj
            const int ph = seg == 0 ? (e == 0 ? kPhQ : kPhO) : kPhD;
            if (ph == kPhO) {
              attention_phase(l, st);
              if (tid == 0) prof.mark(101);
              if (plan.n[kPhO] > 0) stage_attn(st);
            }
            float2* part = ph == kPhQ ? P.pq2 : (ph == kPhO ? P.po2 : P.pd2);
            epi_partials(ph, part, ph == kPhQ ? P.qkv_n : H, st);
            if (tid == 0) prof.mark(100 + ph + (ph > 0 ? 1 : 0));   // 100 qkv, 102 o_proj, 103 gate/up, 104 down
          }
          const bool last = l + 1 == L;
          if (seg == 0) fold_phase(P.po2, P.so, st, H, P.ln2[l]);
          else fold_phase(P.pd2, P.sd, st, H, last ? P.final_norm : P.ln1[l + 1]);
          if (tid == 0) prof.mark(seg == 0 ? 105 : 106);
        }
      }
      // ---- lm_head
      epi_head();
      if (tid == 0) prof.mark(110);
      grid_sync(no_post);
      // ---- sampler (+ tests: keep every step's logits)
      if (P.logits_out) {
        const long long n = static_cast<long long>(B) * P.vocab;
        float* dst = P.logits_out + static_cast<long long>(step) * P.logits_step_stride;
        for (long long i = static_cast<long long>(blockIdx.x) * kConsumerThreads + tid; i < n; i += static_cast<long long>(G) * kConsumerThreads)
          dst[i] = __ldcg(P.logits + i);
      }
      prof.fine = prof.buf != nullptr;
      sample_phase();
      if (tid == 0) prof.mark(111);
      grid_sync(no_post);
      bool all_done = true;
      for (int b = 0; b < B; ++b) all_done = all_done && (__ldcg(P.samp.done + b) != 0);
      if (all_done || step + 1 == P.n_steps) break;
      if (tid == 0) mbar_arrive(&ms->go_bar);   // releases step + 1
    }
    csync();
    if (tid == 0) {   // wake a warp that waits for a step that will not run
      *reinterpret_cast<volatile int*>(&ms->stop) = 1;
      mbar_arrive(&ms->go_bar);
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------ host side
static size_t tc_chunk_bytes(int nt) {   // B chunks (+ fold_in_cta: fp32 rows and the norm weights), 1024-aligned
  const size_t u = size_t(14) * nt * 128 + (nt == 16 ? 20 * 1024 : 0);
  return (u + 1023) & ~size_t(1023);
}
static size_t tc_attn_bytes(int aw) { return (tc_attn_layout_bytes(aw) + 1023) & ~size_t(1023); }

bool tc_fold_in_cta(int B, int hidden) {
  // Every consumer re-folds ALL rows in the in-CTA fold, so its cost grows with the batch while the fold phases' is
  // flat: the in-CTA fold runs at batch 1 only.
  return B == 1 && size_t(hidden) * 4 <= 16 * 1024 && hidden <= 1024;
}

int tc_build_plan(const TcShape& s, int G, bool flat, TcPlan* plan, unsigned char* gu_nsl, TcPlanInfo* info) {
  if (G < 8 || G > 256) return set_error(NT_ERR_INVALID, "decode_tc: %d SMs unsupported", G);
  if (s.hidden % 64 || s.inter % 64) return set_error(NT_ERR_INVALID, "decode_tc: hidden / inter must be multiples of 64");
  const int Tq = (s.qkv_n + 127) / 128, To = (s.hidden + 127) / 128, Tg = (2 * s.inter + 127) / 128;
  const int KBh = s.hidden / 64, KBo = s.n_heads, KBi = s.inter / 64;
  if (KBh > 14) return set_error(NT_ERR_INVALID, "decode_tc: hidden %d > 896 does not fit the shared-memory plan", s.hidden);
  for (int c = 0; c < G; ++c) plan[c] = TcPlan{};
  auto add = [&](int cta, int ph, TcItem it) -> bool {
    TcPlan& p = plan[cta];
    if (p.n[ph] >= kTcMaxItems) return false;
    p.it[ph][p.n[ph]++] = it;
    return true;
  };
  std::vector<int> rest;
  int sg = 1;
  if (flat) {
    // gate/up as (tile, k-block) units in tile-major order: CTA c owns units [U c / G, U (c + 1) / G)
    const int U = Tg * KBh;
    std::vector<int> nsl(Tg, 0);
    for (int c = 0; c < G; ++c) {
      int u0 = int((static_cast<long long>(U) * c) / G);
      const int u1 = int((static_cast<long long>(U) * (c + 1)) / G);
      while (u0 < u1) {
        const int t = u0 / KBh, kb0 = u0 % KBh;
        const int n = (u1 - u0 < KBh - kb0) ? (u1 - u0) : (KBh - kb0);
        if (nsl[t] >= kTcMaxGuSlices || !add(c, kPhG, TcItem{short(t), short(kb0), short(n), short(nsl[t])}))
          return set_error(NT_ERR_INVALID, "decode_tc: flat gate/up plan does not fit");
        ++nsl[t];
        u0 += n;
      }
      plan[c].gu_split = 1;
    }
    for (int t = 0; t < Tg; ++t) {
      if (gu_nsl) gu_nsl[t] = static_cast<unsigned char>(nsl[t]);
      if (nsl[t] > sg) sg = nsl[t];
    }
    for (int c = 0; c < G; ++c) rest.push_back(c);
  } else {
    // gate/up keeps K whole (its SwiGLU epilogue is not linear): its row tiles go to a dedicated, evenly spread subset
    int ngu = Tg < G ? Tg : G;
    std::vector<int> gu;
    if (G - ngu < 16) {  // too few CTAs would be left for the split phases: everybody does everything
      for (int c = 0; c < G; ++c) gu.push_back(c), rest.push_back(c);
    } else {
      for (int c = 0; c < G; ++c) {
        const bool is_gu = ((c + 1) * ngu) / G > (c * ngu) / G;
        (is_gu ? gu : rest).push_back(c);
      }
    }
    for (int t = 0; t < Tg; ++t)
      if (!add(gu[t % gu.size()], kPhG, TcItem{short(t), 0, short(KBh), 0})) return set_error(NT_ERR_INVALID, "decode_tc: too many gate/up tiles per CTA");
  }
  const int nr = int(rest.size());
  int rot = 0;
  auto split_phase = [&](int ph, int T, int KB, int* slices) -> bool {
    int S = nr / T;
    if (flat && ph != kPhD && S > (KB + 1) / 2) S = (KB + 1) / 2;   // measured at batch 1: 7 slices 702 us / step, 14 slices 759
    if (S < 1) S = 1;
    if (S > KB) S = KB;
    if (S > kTcMaxSlices) S = kTcMaxSlices;
    while ((KB + S - 1) / S > 14) ++S;   // an item's k-blocks must fit the staging area
    *slices = S;
    for (int t = 0; t < T; ++t)
      for (int z = 0; z < S; ++z) {
        const int k0 = (KB * z) / S, k1 = (KB * (z + 1)) / S;
        if (!add(rest[rot % nr], ph, TcItem{short(t), short(k0), short(k1 - k0), short(z)})) return false;
        ++rot;
      }
    return true;
  };
  if (!split_phase(kPhQ, Tq, KBh, &info->sq) || !split_phase(kPhO, To, KBo, &info->so) || !split_phase(kPhD, To, KBi, &info->sd))
    return set_error(NT_ERR_INVALID, "decode_tc: too many split-K items per CTA");
  int worst = 0;
  bool fq = false, fg = false;
  for (int c = 0; c < G; ++c) {
    for (int ph = 0; ph < 4; ++ph) {
      if (ph == kPhG && !flat) continue;
      int chunks = 0;
      for (int i = 0; i < plan[c].n[ph]; ++i) chunks += plan[c].it[ph][i].nkb;
      if (chunks > worst) worst = chunks;
    }
    if (!fq && plan[c].n[kPhQ] > 0) plan[c].fold_q = 1, fq = true;
    if (!fg && plan[c].n[kPhG] > 0) plan[c].fold_g = 1, fg = true;
  }
  if (worst > 14) return set_error(NT_ERR_INVALID, "decode_tc: %d k-blocks per CTA exceed the staging area", worst);
  info->max_chunks = worst;
  info->sg = sg;
  info->gu_split = flat ? 1 : 0;
  const int nt = (s.vocab + 127) / 128;
  info->ntiles = nt;
  return NT_OK;
}

template <int NT, bool HILO, bool FOLD>
static int launch_tc(TcParams& P, int num_sms, cudaStream_t stream) {
  auto kern = decode_tc_kernel<NT, HILO, FOLD>;
  const size_t budget = 227 * 1024;
  const size_t misc = (sizeof(TcMisc) + 127) & ~size_t(127);
  const size_t acc = (size_t(128) * (NT + 4) * 4 + 127) & ~size_t(127);   // accumulator tile [128][NT + 4] fp32
  // batch <= 4: the attention staging sits BEHIND the B chunks, so a layer's KV pages are fetched while the qkv
  // projection still runs; otherwise the two alias (a phase uses one or the other)
  const bool separate = P.fold_in_cta != 0;
  // dedicated staging: two page-walking warps (a split is 1..4 pages at batch <= 4), which leaves the weight ring 8 stages
  P.att_warps = separate ? 2 : 4;
  const size_t chunks = tc_chunk_bytes(NT), att = tc_attn_bytes(P.att_warps);
  const size_t uni = separate ? chunks + att : (chunks > att ? chunks : att);
  int ns = int((budget - uni - misc - acc - 1024) / 16384);
  if (ns > 16) ns = 16;
  if (ns < 3) return set_error(NT_ERR_INVALID, "decode_tc: shared memory plan leaves %d ring stages", ns);
  const size_t smem = size_t(ns) * 16384 + uni + misc + acc + 1024;
  P.nstages = ns;
  P.uni_off = unsigned(size_t(ns) * 16384);
  P.uni_bytes = unsigned(uni);
  P.att_off = P.uni_off + (separate ? unsigned(chunks) : 0u);
  P.misc_off = P.uni_off + P.uni_bytes;
  P.acc_off = P.misc_off + unsigned(misc);
  NT_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  int per_sm = 0;
  NT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kTcThreads, smem));
  if (per_sm < 1) return set_error(NT_ERR_CUDA, "decode_tc: a CTA does not fit on an SM (%zu B shared memory)", smem);
  NT_CUDA_CHECK(cudaMemsetAsync(P.gbar, 0, sizeof(unsigned) * 64, stream));
  void* args[] = {&P};
  cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kern), dim3(num_sms), dim3(kTcThreads), args, smem, stream);
  if (e != cudaSuccess) return set_error(NT_ERR_CUDA, "decode_tc launch failed: %s", cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return NT_OK;
}

int launch_decode_tc(TcParams& P, int B, int num_sms, const TcPlanInfo& info, cudaStream_t stream) {
  if (B < 1 || B > kTcMaxBatch) return set_error(NT_ERR_INVALID, "decode_tc: batch %d not in 1..%d", B, kTcMaxBatch);
  if (P.n_heads % P.n_kv || P.n_heads / P.n_kv > 8) return set_error(NT_ERR_INVALID, "decode_tc: unsupported GQA ratio");
  P.B = B;
  // attention items: (sequence, kv head, split) -> one CTA each
  int cap = num_sms / (B * P.n_kv);
  if (cap < 1) return set_error(NT_ERR_INVALID, "decode_tc: %d sequences x %d kv heads exceed %d SMs", B, P.n_kv, num_sms);
  if (cap > 8) cap = 8;   // the merge fetches all (m, l, o) partials of an element in one batch of loads
  if (cap > P.max_splits) cap = P.max_splits;
  P.split_cap = cap;
  const int nt = B <= 16 ? 16 : (B <= 32 ? 32 : 64);
  if (info.max_chunks > 14) return set_error(NT_ERR_INVALID, "decode_tc: %d k-blocks per CTA exceed the staging area", info.max_chunks);
  P.fold_in_cta = tc_fold_in_cta(B, P.hidden) ? 1 : 0;
  P.weights_evict_first = 1;
  if (info.gu_split && !P.fold_in_cta) return set_error(NT_ERR_INVALID, "decode_tc: the flat plan needs the in-CTA fold (batch <= 4)");
  const bool hilo = B <= 8;
  if (hilo) return P.fold_in_cta ? launch_tc<16, true, true>(P, num_sms, stream) : launch_tc<16, true, false>(P, num_sms, stream);
  if (nt == 16) return launch_tc<16, false, false>(P, num_sms, stream);
  if (nt == 32) return launch_tc<32, false, false>(P, num_sms, stream);
  return launch_tc<64, false, false>(P, num_sms, stream);
}

}  // namespace nt
