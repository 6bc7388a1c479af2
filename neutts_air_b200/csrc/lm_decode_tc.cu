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
//     batch 1: no grid barrier inside a layer; the last producer of each o_proj / down_proj row tile folds it into the
//     residual stream, and the consumers normalise that row while staging their B operand; the last producer of each
//     qkv / gate/up row tile hands attention (bias + RoPE applied) and down_proj (SwiGLU applied) finished rows; larger batches:
//     token-owner CTAs fold + normalise into bf16 rows that the consumers fetch by TMA (3 barriers per layer, no
//     per-CTA re-reading of the whole batch).
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
// arrival at a self-resetting counter: returns the old value, stores old + 1, or 0 when old == last.  Relaxed: it
// only elects a CTA, the data it then reads carry their own stamps.
NT_DEVINL unsigned tc_arrive_inc(unsigned* p, unsigned last) {
  unsigned old;
  asm volatile("atom.relaxed.gpu.global.inc.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(last) : "memory");
  return old;
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
// register budget of the calling warpgroup (every thread of it executes the same instruction)
template <int R> NT_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> NT_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
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


NT_DEVINL void tc_spin_check(uint32_t& spins, const char* what) {
  if (++spins > (1u << 22)) nt_timeout(what);
}

// RoPE of the adjacent qkv rows (2i, 2i + 1) = dims (i, i + 32) of a head, sc = rope_sincos(pos, inv_freq[i]):
// rope_pair's rotation, but dim i + 32 fuses x sin and rounds y cos where rope_pair does the opposite -- the rounding
// this kernel has always had, which keeps its decode output bit-identical
NT_DEVINL float2 tc_rope(float2 a, float2 sc) {
  return make_float2(__fmaf_rn(a.x, sc.y, -__fmul_rn(a.y, sc.x)), __fmaf_rn(a.x, sc.x, __fmul_rn(a.y, sc.y)));
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
  float rep_pen[kTcMaxBatch]; // repetition penalty per sequence (1: none, or the slot is unrecorded)
  float len_c[kTcMaxBatch];   // this step's EOS decay constant per sequence (0: none; length control)
  float red[64];
  float tile_max[2][4][kTcMaxBatch];
  float rstd[8];
  int sel[8];
  int tile_last[2];       // batch 1: this CTA arrived last at the split-K tile it just stored (epilogue warps)
  int bchunks[4];         // B-operand chunks of this CTA's items per split phase
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
// RAS: repetition-aware sampling compiled in (launches with the table on); without it the table-off sampler carries
// none of its code
template <int NT, bool HILO, bool FOLD, bool RAS>
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
  if (tid < B) {
    ms->inv_t[tid] = row_sampling(P.samp, tid).inv_t;
    ms->rep_pen[tid] = (P.rep_tab && P.rep_rec[tid]) ? P.rep_tab[tid].penalty : 1.f;
  }
  __syncthreads();
  const TcPlan& plan = ms->plan;
  if (tid < 4) {  // chunk tables of the split phases (items in plan order, k-blocks ascending)
    int c = 0;
    for (int i = 0; i < plan.n[tid]; ++i)
      for (int kb = 0; kb < plan.it[tid][i].nkb && c < 16; ++kb, ++c) ms->ckb[tid][c] = plan.it[tid][i].kb0 + kb;
    ms->bchunks[tid] = c;
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
  // Register budgets per warpgroup (__launch_bounds__(512, 1) starts every thread at 128): WG3 keeps what the weight
  // stream needs, WG2 the accumulators of two m64 x NT halves, and the worker warpgroups take the rest.
  // 128 * (kRegStream + kRegMma) + 256 * kRegWork = 64 K registers.
  constexpr int kRegStream = 24, kRegMma = NT == 64 ? 104 : (NT == 32 ? 72 : 56), kRegWork = (65536 / 128 - kRegStream - kRegMma) / 2;
  static_assert(kRegWork % 8 == 0 && kRegWork <= 256, "setmaxnreg takes a multiple of 8 up to 256");
  // Each setmaxnreg opens the branch of its role, so that ptxas allocates the role's code under that budget.  The
  // worker branch comes first: laid out behind the other two, ptxas kept it at the entry budget of 128.
  if (warp < kTcMmaWarp0) {
    setmaxnreg_inc<kRegWork>();
    // ================================================================== worker warps 0..7
    const SyncConsumers csync;
    const unsigned G = gridDim.x;
    unsigned target = 0;
    uint32_t acc_n = 0;
    TcProf prof{nullptr, 0, false};
    auto pm = [&](int id) { if (tid == 0 && prof.fine) prof.mark(id); };
    const int n_rep = P.n_heads / P.n_kv;
    const int split_cap = P.split_cap;
    constexpr bool fold_cta = FOLD;   // batch 1: split-K tiles folded by their last producer (no fold phases, no barriers)
    const int I = P.inter;
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
    // fold_in_cta: folds done in this launch.  Residual version n (stamp hstamp_base + n, buffer n & 1 of the h2
    // ping-pong) is what fold n normalises: the sampler's row (or the prefill's, n = 0; copy 0 only, read behind a grid
    // barrier) for the first fold of a step, else the previous one plus the o_proj or down_proj slices, written tile by
    // tile by their last producers into all kTcH2Copies copies.
    // Why two buffers suffice: writing version n over version n - 2 (rows of one tile t) needs every reader of
    // version n - 2 to be done with it.  They are
    //   * the last producer of tile t for version n - 1: it read those rows into the value it wrote for n - 1, and the
    //     writer of n polls version n - 1 of tile t before it writes;
    //   * the consumers of fold n - 2, which read the whole row.  A consumer has items in the GEMM that follows its
    //     fold and runs them after the read.  Version n - 1 of tile t needs the slices of every item of that GEMM:
    //     every slice of a gate/up or qkv tile is read by the tile's last producer, which publishes the tile only
    //     after that read.  Gate/up tiles feed down_proj k-blocks, and every down tile's slices cover all of them; qkv
    //     tiles feed the attention of every split (q rows) or of the appending split (k/v rows; split 0 reads them
    //     when no split appends), and every o_proj tile's slices cover all heads and merge all their splits.  The
    //     writer of n polls version n - 1 of tile t, so it comes after every such read.
    //   After the final norm the sampler writes the next version behind a grid barrier.
    // qkv2 and act2 (the finished qkv and SwiGLU rows, stamp of the layer) hold one version.  The next layer's writer
    // of a qkv2 tile is elected by qkv items that read the residual version behind this layer's down_proj, and the
    // writer of an act2 tile by gate/up items behind the next layer's o_proj: by the chains above, those versions need
    // every attention split's partials (which come after its qkv2 read) and every down item's slice (which comes
    // after its act2 read).  The stamps reject whatever an earlier layer or launch left.
    int fold_no = 0;

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
      const int nch = uniform(ms->bchunks[ph]);
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

    // ---- batch 1: the CTA that stores the last of a row tile's S split-K slices folds the tile (epilogue warps; lane =
    //      row of the tile) and publishes finished rows, which the consumers poll as one pair per element:
    //        o_proj, down_proj: residual version fold_no - 1 plus the slices -> residual version fold_no (h2), read by
    //          the consumers of fold fold_no (tc_fold4 with no slices);
    //        qkv: the slices plus the bias, RoPE on q and k rows -> qkv2, read by the attention prologue;
    //        gate/up (flat plan): the slices, then SwiGLU of the (gate, up) row pairs -> act2, read by stage_act.
    //      The additions are the ones every consumer used to do, in the same order: acc = residual (or 0), then slice
    //      0 .. S - 1, plus the zero padding of the readers' batches of eight (none for gate/up), then the bias -- the
    //      same fp32 additions, so the same bits.  The residual is stored kTcH2Copies times: with one copy every CTA of
    //      the grid polled the same 7 KB, and on H100 that hot spot cost more than the L2 traffic the fold saves
    //      (bench.py measured 885-895 us per step with one copy, 825-836 us with four).  qkv2 and act2 have at most 8
    //      and 7 readers per line and are stored once.
    //      The counter only elects the last arriver (S arrivals per tile and layer; it wraps to 0 on the last one, and
    //      the next layer's arrivals all depend on this fold).  Every value read is a (value, stamp) pair polled until
    //      its stamp matches, so the arrival needs no release/acquire: a slice whose store is not yet visible to the
    //      elected CTA is simply polled again.  Each lane issues its loads before the election returns, so the
    //      arrival's round trip and the reads overlap; the other S - 1 producers drop what they loaded.
    uint32_t tf_n = 0;   // tile_fold calls (parity of ms->tile_last)
    auto tile_fold = [&](int ph, const float2* part, int rows, int S, int stamp, int tile, int l) {
      const bool resid = ph == kPhO || ph == kPhD;
      unsigned* cnt = P.tile_cnt + (ph == kPhQ ? kTcQkvCnt : (ph == kPhG ? kTcGuCnt : (ph == kPhD ? kTcMaxTiles : 0))) + tile;
      int* last = &ms->tile_last[tf_n++ & 1];   // two slots: a lane still reading one never sees the next election
      if (tid == 0) *last = tc_arrive_inc(cnt, static_cast<unsigned>(S - 1)) == static_cast<unsigned>(S - 1);
      const int row = tile * 128 + warp * 32 + lane;
      const bool in = row < rows;
      const int hstamp = P.hstamp_base + fold_no;
      const float2* hsrc = P.h2 + static_cast<long long>((fold_no - 1) & 1) * kTcH2Copies * H + row;
      const float2* psrc = part + row;
      const float pad = __int_as_float(stamp);
      float2 r = in && resid ? ldp1(hsrc) : make_float2(0.f, __int_as_float(hstamp - 1));
      const float bias = in && ph == kPhQ ? __ldg(P.bqkv[l] + row) : 0.f;
      float2 t[kTcMaxSlices];
#pragma unroll
      for (int j = 0; j < kTcMaxSlices; ++j) t[j] = in && j < S ? ldp1(psrc + static_cast<long long>(j) * rows) : make_float2(0.f, pad);
      bar_epi();
      if (!*last) return;
      pm(11);
      uint32_t spins = 0;
      while (__float_as_int(r.y) != hstamp - 1) {
        tc_spin_check(spins, "the residual stream");
        r = ldp1(hsrc);
      }
      spins = 0;
      for (;;) {
        bool ok = true;
#pragma unroll
        for (int j = 0; j < kTcMaxSlices; ++j) ok = ok && __float_as_int(t[j].y) == stamp;
        if (ok) break;
        tc_spin_check(spins, "split-K slices");
#pragma unroll
        for (int j = 0; j < kTcMaxSlices; ++j)
          if (in && j < S && __float_as_int(t[j].y) != stamp) t[j] = ldp1(psrc + static_cast<long long>(j) * rows);
      }
      // the readers' order: slices in batches of eight, the last batch padded with zeros (gate/up: no padding)
      const int nadd = ph == kPhG ? S : (S + 7) & ~7;
      float acc = r.x;
#pragma unroll
      for (int j = 0; j < kTcMaxSlices; ++j)
        if (j < nadd) acc += t[j].x;
      if (resid) {
        if (in) {
          float2* dst = P.h2 + static_cast<long long>(fold_no & 1) * kTcH2Copies * H + row;
#pragma unroll
          for (int c = 0; c < kTcH2Copies; ++c) dst[static_cast<long long>(c) * H] = make_float2(acc, __int_as_float(hstamp));
        }
      } else {
        // rows (2j, 2j + 1) pair up on adjacent lanes: q/k dims (j, j + 32) of a head, v dims, or (gate_j, up_j)
        if (ph == kPhQ) acc += bias;
        const float odd = __shfl_down_sync(0xffffffffu, acc, 1);
        if (in && !(lane & 1)) {
          if (ph == kPhG) {
            P.act2[row >> 1] = make_float2(silu(acc) * odd, pad);
          } else {
            float2 v = make_float2(acc, odd);
            if (row < (P.n_heads + P.n_kv) * 64) v = tc_rope(v, rope_sincos(ms->pos[0], __ldg(P.inv_freq + ((row & 63) >> 1))));
            *reinterpret_cast<float4*>(P.qkv2 + row) = make_float4(v.x, pad, v.y, pad);
          }
        }
      }
      pm(12);
    };

    // ---- epilogue of the split-K phases: raw partial sums as (value, stamp) pairs, one row per lane
    auto epi_partials = [&](int ph, float2* part, int rows, int stamp, int l) {
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
        if constexpr (FOLD) {
          const int S = ph == kPhQ ? P.sq : (ph == kPhO ? P.so : (ph == kPhG ? __ldg(P.gu_nsl + it.tile) : P.sd));
          tile_fold(ph, part, rows, S, stamp, it.tile, l);
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

    // ---- batch 1: read residual version fold_no (folded by the last producers of its row tiles, see tile_fold),
    //      normalise, stage the B chunks of phase `ph` (-1: every k-block).  Thread q < H / 4 keeps elements
    //      4q .. 4q + 3 in registers from the read to the staging, so no fp32 copy of the row takes shared memory away
    //      from the weight ring.
    auto fold_stage = [&](const float* norm_w, int ph, bool copies) {
      // copy blockIdx % kTcH2Copies of a tile-folded version: the grid's polls spread over four times the L2 lines
      const float2* hsrc = P.h2 + (static_cast<long long>(fold_no & 1) * kTcH2Copies + (copies ? blockIdx.x % kTcH2Copies : 0)) * H;
      const int hstamp = P.hstamp_base + fold_no;
      const int i4 = tid * 4;
      const bool mine = i4 < H;   // H <= 4 * kConsumerThreads (tc_fold_in_cta)
      pm(1);
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      float4 nw = make_float4(0.f, 0.f, 0.f, 0.f);
      if (mine) {
        nw = __ldg(reinterpret_cast<const float4*>(norm_w + i4));   // in flight together with the slices
        tc_fold4(hsrc, hstamp, nullptr, 0, 0, H, B, H, 0, i4, acc);
      }
      pm(2);
      const float ss = warp_sum((acc[0] * acc[0] + acc[1] * acc[1]) + (acc[2] * acc[2] + acc[3] * acc[3]));
      if (lane == 0) ms->red[warp] = ss;
      csync();   // also: the B chunks of the previous phase are free (see stage_attn)
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kConsumerWarps; ++w) t += ms->red[w];   // fixed order: every CTA gets the same bits
      const float rstd = rsqrtf(t / static_cast<float>(H) + P.eps);
      if (mine) {
        const float xn[4] = {nw.x * (acc[0] * rstd), nw.y * (acc[1] * rstd), nw.z * (acc[2] * rstd), nw.w * (acc[3] * rstd)};
        __nv_bfloat16 hi[4], lo[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split_hilo(xn[j], hi[j], lo[j]);
        const uint2 vhi = make_uint2(pack2(hi[0], hi[1]), pack2(hi[2], hi[3])), vlo = make_uint2(pack2(lo[0], lo[1]), pack2(lo[2], lo[3]));
        const int kb = i4 >> 6, k4 = i4 & 63;   // 4 consecutive k of one row: one 8-byte run of a 16-byte swizzle group
        auto put = [&](int c) {
          uint8_t* cb = uni + c * CHUNK;
          *reinterpret_cast<uint2*>(chunk_elem(cb, 0, k4)) = vhi;
          *reinterpret_cast<uint2*>(chunk_elem(cb, 8, k4)) = vlo;
        };
        if (ph < 0) {
          put(kb);
        } else {   // every chunk that holds k-block kb (two items of one K slice stage it twice)
          const int nch = ms->bchunks[ph];
          for (int c = 0; c < nch; ++c)
            if (ms->ckb[ph][c] == kb) put(c);
        }
      }
      pm(4);
      bop_ready();
      pm(5);
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
      const int page = uniform(page_of(pg, p0));
      if (elect_one()) {
        if (fence) fence_proxy_async_all();
        mbar_arrive_expect_tx(&ms->att_bar[warp], 2 * 8192);
        tma_load_2d(att_k(warp), kvmap, 0, P.kv.tmap_row(l, 0, page, my_kvh), &ms->att_bar[warp]);
        tma_load_2d(att_v(warp), kvmap, 0, P.kv.tmap_row(l, 1, page, my_kvh), &ms->att_bar[warp]);
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
      // batch 1: every finished qkv row tile must be read by some split, or the h2 ping-pong and the single qkv2 version
      // lose their ordering (see fold_no)
      const bool kv_rows = appends || (FOLD && pos >= P.kv.max_ctx && my_split == 0);
      if (!att_separate) {
        // the pages do not depend on this layer's projections (the new row is patched in below): fetch the first round now
        csync();   // the union region is ours (previous phase of this CTA is through with it)
        if (warp < AW && p0 + warp < p1) issue_page(l, p0 + warp, p0, true);
      }
      pm(21);
      // prologue: q of the group -> shared; new K/V row.  Batch 1 reads the rows the last producer of each qkv tile
      // finished (tile_fold); larger batches fold the qkv slices (slice order) + bias and apply RoPE here.
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
        if (which != 0 && !kv_rows) continue;
        float2 r;
        if constexpr (FOLD) {
          uint32_t spins = 0;
          for (;;) {
            const float4 t = ldp2(P.qkv2 + row0);
            if (__float_as_int(t.y) == stamp && __float_as_int(t.w) == stamp) {
              r = make_float2(t.x, t.z);
              break;
            }
            tc_spin_check(spins, "qkv rows");
          }
        } else {
          const float2 bia = __ldg(reinterpret_cast<const float2*>(bias + row0));
          // ahead of the wait for the slices, which hides its latency
          const float2 sc = which != 2 ? rope_sincos(pos, __ldg(P.inv_freq + i)) : make_float2(0.f, 1.f);
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
          r = which == 2 ? a : tc_rope(a, sc);
        }
        if (which == 2) att_vnew[2 * i] = r.x, att_vnew[2 * i + 1] = r.y;
        else if (which == 0) att_q[(idx >> 5) * 64 + i] = r.x, att_q[(idx >> 5) * 64 + i + 32] = r.y;
        else att_knew[i] = r.x, att_knew[i + 32] = r.y;
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
        uint32_t qa[4][4];
        decode_query_frags(att_q, n_rep, P.scale_log2, qa);
        float o[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
        float m[1] = {-INFINITY}, lsum[1] = {0.f};
        const uint32_t kbase = smem_u32(att_k(warp)), vbase = smem_u32(att_v(warp));
        for (int pg = p0 + warp; pg < p1; pg += AW) {
          mbar_wait(&ms->att_bar[warp], att_par);
          att_par ^= 1;
          if (warp == 0) pm(23);
          if (appends && pg == (pos >> 6)) patch_staged_row(att_k(warp), att_v(warp), pos & 63, att_knew, att_vnew);
          const int k0 = pg * 64;
          attn_page_step<1>(kbase, vbase, qa, o, m, lsum, k0 + 64 > geo.n_ctx, [&](int, int key) { return k0 + key >= geo.n_ctx; });
          __syncwarp();  // all lanes are done with the buffers before they are refilled
          if (pg + AW < p1) issue_page(l, pg + AW, p0, !att_separate);
        }
        decode_store_partial(o, m[0], lsum[0], n_rep, att_o + warp * 8 * 64, att_ml + warp * 8 * 2);
      }
      csync();
      const float sf = __int_as_float(stamp);
      for (int i = tid; i < n_rep * 64; i += kConsumerThreads) {
        const int h = i >> 6, d = i & 63;
        const SoftmaxPart r = merge_parts<kAttWarpsMax>(AW, [&](int w) {
          return SoftmaxPart{att_ml[(w * 8 + h) * 2], att_ml[(w * 8 + h) * 2 + 1], att_o[(w * 8 + h) * 64 + d]};
        });
        const long long hh = static_cast<long long>(b) * P.n_heads + kvh * n_rep + h;
        P.ao2[(hh * P.max_splits + my_split) * 64 + d] = make_float2(r.o, sf);
        if (d == 0) *reinterpret_cast<float4*>(P.aml2 + (hh * P.max_splits + my_split) * 2) = make_float4(r.m, sf, r.l, sf);
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
      const int nch = ms->bchunks[kPhO];
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
        const SoftmaxPart mp = merge_parts<8>(g.nsplit, [&](int s) { return SoftmaxPart{mv[s].x, mv[s].z, ov[s].x}; });
        const float val = mp.o / mp.l;
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

    // ---- batch 1: down_proj input from the (value, stamp) SwiGLU outputs, two elements per thread.  They come from
    //      epi_swiglu (whole-K gate/up) or, in the flat plan, from the last producer of each gate/up tile (tile_fold).
    auto stage_act = [&](int stamp) {
      csync();   // the B chunks of the gate/up phase are free (see stage_attn)
      const int nch = ms->bchunks[kPhD];
      const int per = B * 32;
      for (int e = tid; e < nch * per; e += kConsumerThreads) {
        const int c = e / per, r = e - c * per, b = r >> 5, k = (r & 31) * 2;
        const int kbd = ms->ckb[kPhD][c];
        float4 t;
        const float2* p = P.act2 + static_cast<long long>(b) * I + kbd * 64 + k;
        uint32_t spins = 0;
        for (;;) {
          t = ldp2(p);
          if (__float_as_int(t.y) == stamp && __float_as_int(t.w) == stamp) break;
          tc_spin_check(spins, "SwiGLU outputs");
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
        // repetition penalty, before the store and the processed maximum: this warp's 32 rows are one bitmap word per
        // column (a broadcast load); the bits were set by the sampler of the previous step, behind a grid barrier
        const int wi = tile * 4 + warp;
        if (P.rep_tab && wi < P.samp.rep_words) {   // warp-uniform
#pragma unroll
          for (int n = 0; n < NTOK; ++n) {
            if (n < B && ms->rep_pen[n] != 1.f) {
              const uint32_t word = __ldcg(P.samp.rep_hist + static_cast<long long>(n) * P.samp.rep_words + wi);
              if ((word >> lane) & 1u) v[n] = rep_penalize(v[n], ms->rep_pen[n]);
            }
          }
        }
        // length control: the EOS decay after the penalty, before the store, the mask and 1 / T (one lane of one warp)
        if (P.samp.len_tab && row == eos) {
#pragma unroll
          for (int n = 0; n < NTOK; ++n)
            if (n < B && ms->len_c[n] != 0.f) v[n] = len_decay(v[n], ms->len_c[n]);
        }
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
      float2* h2dst = fold_cta ? P.h2 + static_cast<long long>(fold_no & 1) * kTcH2Copies * H : nullptr;   // copy 0 (B = 1)
      const float h2stamp = __int_as_float(P.hstamp_base + fold_no);
      // the epilogue stored PROCESSED maxima (temperature, EOS mask): no scale, no tile to fix up
      sample_tiles_seq<RAS>(P.samp, b, P.tmax, P.ntiles, 1.0f, -1, 0.f, P.logits, P.vocab, ms->mask_eos[b] != 0, uni, P.uni_bytes, ms->sel,
                       csync, pm, h2dst, h2stamp, false);
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
        // n_generated was written by the previous step's sampler, before the grid barrier that follows it
        const int ngen = __ldcg(P.samp.n_generated + tid);
        ms->mask_eos[tid] = ngen < row_min_new(P.samp, tid) ? 1 : 0;
        ms->len_c[tid] = len_decay_c(P.samp, tid, ngen);
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
          // RMSNorm of the residual stream (already folded by the previous GEMM's last producers) + B-operand staging
          const float* norm_w = head ? P.final_norm : (second ? P.ln2[l] : P.ln1[l]);
          const int sph = head ? -1 : (second ? (plan.gu_split ? kPhG : -1) : kPhQ);
          const bool need = head ? n_head_tiles > 0 : plan.n[second ? kPhG : kPhQ] > 0;
          if (!second && !head) attn_prefetch(l);
          if (need) fold_stage(norm_w, sph, hl > 0);
          else ++fold_no;
          if (head) break;
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
            // one call site each: the down epilogue (with its tile fold) is inlined once
            if (ph == kPhG && !plan.gu_split) epi_swiglu(st);   // whole-K gate/up: SwiGLU in the epilogue
            else epi_partials(ph, part, rows, st, l);
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
            epi_partials(ph, part, ph == kPhQ ? P.qkv_n : H, st, l);
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
    } else if (warp < kTcStreamWarp) {
    setmaxnreg_dec<kRegMma>();
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
    setmaxnreg_dec<kRegStream>();
    // the parked warps 13..15 (they make WG3 a whole warpgroup) run no step and go on to the closing block barrier
    const int n_steps = warp == kTcStreamWarp ? P.n_steps : 0;
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
    for (int step = 0; step < n_steps; ++step) {
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
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------ host side
static size_t tc_chunk_bytes(int nt) { return size_t(14) * nt * 128; }   // the B chunks (a multiple of 1024 bytes)
static size_t tc_attn_bytes(int aw) { return (tc_attn_layout_bytes(aw) + 1023) & ~size_t(1023); }

bool tc_fold_in_cta(int B, int hidden) {
  // The in-CTA fold (tile_fold, fold_stage) handles one token row: every consumer reads the whole row, a cost that
  // would grow with the batch while the fold phases' is flat.  It runs at batch 1 only.
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
  for (int c = 0; c < G; ++c) {
    for (int ph = 0; ph < 4; ++ph) {
      if (ph == kPhG && !flat) continue;
      int chunks = 0;
      for (int i = 0; i < plan[c].n[ph]; ++i) chunks += plan[c].it[ph][i].nkb;
      if (chunks > worst) worst = chunks;
    }
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
  auto kern = P.samp.ras_tab ? decode_tc_kernel<NT, HILO, FOLD, true> : decode_tc_kernel<NT, HILO, FOLD, false>;
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
  NT_CUDA_CHECK(cudaMemsetAsync(P.gbar, 0, sizeof(unsigned) * kTcBarWords, stream));
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
  if (P.fold_in_cta && (P.qkv_n + 127) / 128 > kTcMaxQkvTiles) return set_error(NT_ERR_INVALID, "decode_tc: qkv width %d has too many row tiles", P.qkv_n);
  P.weights_evict_first = 1;
  if (info.gu_split && !P.fold_in_cta) return set_error(NT_ERR_INVALID, "decode_tc: the flat plan needs the in-CTA fold (batch <= 4)");
  const bool hilo = B <= 8;
  if (hilo) return P.fold_in_cta ? launch_tc<16, true, true>(P, num_sms, stream) : launch_tc<16, true, false>(P, num_sms, stream);
  if (nt == 16) return launch_tc<16, false, false>(P, num_sms, stream);
  if (nt == 32) return launch_tc<32, false, false>(P, num_sms, stream);
  return launch_tc<64, false, false>(P, num_sms, stream);
}

}  // namespace nt
