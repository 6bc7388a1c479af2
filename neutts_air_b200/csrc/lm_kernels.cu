// Speech-LM kernels for sm_90a (SURVEY.md §8a, rows A1-A12).
//
// Decode (memory-bound, batch <= 4 on CUDA cores):
//   gemv_kernel        weight rows stream HBM -> shared memory through a cp.async.bulk (TMA
//                      engine) ring guarded by mbarriers; 8 consumer warps + 1 producer warp.
//                      Fused prologue: RMSNorm of the input vector (modeling_qwen2.py:258-263).
//                      Fused epilogues: bias + RoPE + KV-page append (:217-225), residual add
//                      (:302,:308), SiLU(gate)*up (:46-48).  The weight prefetch is issued
//                      BEFORE griddepcontrol.wait so it overlaps the previous kernel (PDL).
//   attn_decode_kernel GQA attention over 64-token pages (one CTA per sequence and KV head, warp pairs
//                      walk the pages); fp32 online softmax (:161-183).
//   topk kernels       min-new-tokens EOS mask, temperature, top-k, softmax, multinomial
//                      (logits_process.py:224-233,296-299,580-586; utils.py:2789-2791).
// Prefill helpers (the GEMMs go through gemm_tc.cu): embedding gather, RMSNorm rows,
// RoPE + KV append, causal GQA attention.
#include "lm_device.cuh"

#include <cuda.h>

#include <cfloat>
#include <mutex>

namespace nt {

// =================================================================================== GEMV
constexpr int kGemvThreads = (kConsumerWarps + 1) * 32;

// x planes: element k = 8c + j of batch row b lives in xs[(2b + j/4) * nch + c] component j%4, so
// the two float4 reads that pair with one 16-byte bf16 weight chunk are conflict-free.
template <int NB, typename Sync>
NT_DEVINL void load_x_planes(const float* x, long long ldx, int K, const float* norm_w /*global or shared*/, float eps, float4* xs,
                             float* s_part /*[8][4]*/, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nch = K >> 3, nvec = K >> 2;
  float ssq[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) ssq[b] = 0.f;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    const float4* src = reinterpret_cast<const float4*>(x + b * ldx);
    for (int m0 = 0; m0 < nvec; m0 += 4 * kConsumerThreads) {  // 4 independent loads in flight per thread
      float4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = m0 + j * kConsumerThreads + tid;
        v[j] = (m < nvec) ? __ldcg(src + m) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int m = m0 + j * kConsumerThreads + tid;
        if (m < nvec) {
          xs[(2 * b + (m & 1)) * nch + (m >> 1)] = v[j];
          ssq[b] += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
        }
      }
    }
  }
  if (norm_w) {
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float t = warp_sum(ssq[b]);
      if (lane == 0) s_part[warp * 4 + b] = t;
    }
    sync();
    // every thread rebuilds the row scale from the 8 warp partials and rescales the elements it wrote itself
    const float4* nw = reinterpret_cast<const float4*>(norm_w);
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kConsumerWarps; ++w) t += s_part[w * 4 + b];
      const float sc = rsqrtf(t / static_cast<float>(K) + eps);
      for (int m = tid; m < nvec; m += kConsumerThreads) {
        float4& v = xs[(2 * b + (m & 1)) * nch + (m >> 1)];
        const float4 g = nw[m];
        v.x = v.x * sc * g.x, v.y = v.y * sc * g.y, v.z = v.z * sc * g.z, v.w = v.w * sc * g.w;
      }
    }
  }
  sync();
}

// dot products of one unit (two adjacent bf16 rows in shared memory) with the NB x-vectors over
// 16-byte chunks [c_lo, c_hi), strided by lane.  Partial sums stay per lane.
template <int NB>
NT_DEVINL void unit_dot(const uint4* r0, const uint4* r1, const float4* xs, int nch, int c_lo, int c_hi, int lane,
                        float (&d0)[NB], float (&d1)[NB]) {
  for (int c = c_lo + lane; c < c_hi; c += 32) {
    float f0[8], f1[8];
    bf16x8_to_f32(r0[c], f0);
    bf16x8_to_f32(r1[c], f1);
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float4 xa = xs[(2 * b) * nch + c];
      const float4 xb = xs[(2 * b + 1) * nch + c];
      d0[b] += f0[0] * xa.x + f0[1] * xa.y + f0[2] * xa.z + f0[3] * xa.w + f0[4] * xb.x + f0[5] * xb.y + f0[6] * xb.z +
               f0[7] * xb.w;
      d1[b] += f1[0] * xa.x + f1[1] * xa.y + f1[2] * xa.z + f1[3] * xa.w + f1[4] * xb.x + f1[5] * xb.y + f1[6] * xb.z +
               f1[7] * xb.w;
    }
  }
}

// Batch-1 fast path for warp slices of <= 128 chunks (K <= 1024 per unit, or K <= 8192 split over the 8 warps):
// the lane's slice of the input vector (chunks c_lo + lane + 32 k, k < 4) stays in registers for the whole phase, so a unit costs two 16-byte shared loads per chunk instead of four, and
// the fully unrolled loop puts all weight loads of the unit in flight at once.
struct XRegs {
  float4 a[4], b[4];
};
NT_DEVINL void load_xregs(const float4* xs, int nch, int c_lo, int c_hi, int lane, XRegs& xr) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c_lo + lane + 32 * k;
    const bool ok = c < c_hi;
    xr.a[k] = ok ? xs[c] : make_float4(0.f, 0.f, 0.f, 0.f);
    xr.b[k] = ok ? xs[nch + c] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
NT_DEVINL void unit_dot_x1(const uint4* r0, const uint4* r1, int c_lo, int c_hi, int lane, const XRegs& xr, float& d0,
                            float& d1) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c_lo + lane + 32 * k;
    if (c < c_hi) {
      float f0[8], f1[8];
      bf16x8_to_f32(r0[c], f0);
      bf16x8_to_f32(r1[c], f1);
      const float4 xa = xr.a[k], xb = xr.b[k];
      d0 += f0[0] * xa.x + f0[1] * xa.y + f0[2] * xa.z + f0[3] * xa.w + f0[4] * xb.x + f0[5] * xb.y + f0[6] * xb.z + f0[7] * xb.w;
      d1 += f1[0] * xa.x + f1[1] * xa.y + f1[2] * xa.z + f1[3] * xa.w + f1[4] * xb.x + f1[5] * xb.y + f1[6] * xb.z + f1[7] * xb.w;
    }
  }
}

// Epilogue of one unit (rows 2u, 2u+1).  All lanes hold the full sums; lane b finishes batch row b.
template <int NB>
NT_DEVINL void gemv_epilogue(const GemvParams& p, int u, float (&d0)[NB], float (&d1)[NB], int lane) {
  if (lane >= NB) return;
  const int b = lane;
  float a0 = d0[0], a1 = d1[0];
#pragma unroll
  for (int i = 1; i < NB; ++i)
    if (b == i) a0 = d0[i], a1 = d1[i];
  const int r0 = 2 * u;
  if (p.bias) {
    a0 += __ldg(p.bias + r0);
    a1 += __ldg(p.bias + r0 + 1);
  }
  if (p.epi == GEMV_STORE) {
    if (p.residual) {
      const float2 r = __ldcg(reinterpret_cast<const float2*>(p.residual + b * p.ldr + r0));
      a0 += r.x;
      a1 += r.y;
    }
    *reinterpret_cast<float2*>(p.out + b * p.ldo + r0) = make_float2(a0, a1);
  } else if (p.epi == GEMV_SWIGLU) {
    p.out[b * p.ldo + u] = silu(a0) * a1;
  } else {  // GEMV_QKV_ROPE
    const int head = u >> 5;  // 32 units per 64-row head
    const int i = u & 31;
    const int pos = __ldcg(p.kv.seq_lens + b);
    const int n_kv = p.kv.n_kv_heads;
    if (head < p.n_heads + n_kv) {
      const float2 r = rope_pair(a0, a1, pos, __ldg(p.inv_freq + i));
      if (head < p.n_heads) {
        float* q = p.q_out + (static_cast<long long>(b) * p.n_heads + head) * 64;
        q[i] = r.x;
        q[i + 32] = r.y;
      } else if (pos < p.kv.max_ctx) {
        const int page = __ldcg(p.kv.page_table + b * p.kv.max_pages_per_seq + (pos >> 6));
        __nv_bfloat16* kp = p.kv.page_ptr(p.layer, 0, page, head - p.n_heads) + (pos & 63) * 64;
        kp[i] = __float2bfloat16(r.x);
        kp[i + 32] = __float2bfloat16(r.y);
      }
    } else if (pos < p.kv.max_ctx) {
      const int page = __ldcg(p.kv.page_table + b * p.kv.max_pages_per_seq + (pos >> 6));
      __nv_bfloat16* vp = p.kv.page_ptr(p.layer, 1, page, head - p.n_heads - n_kv) + (pos & 63) * 64;
      *reinterpret_cast<__nv_bfloat162*>(vp + 2 * i) = __floats2bfloat162_rn(a0, a1);
    }
  }
}

// One ring stage of a GEMV phase, executed by the 8 consumer warps.
//   wpu == 1: the stage holds up to 8 units, warp w owns unit w;
//   wpu == 8: the stage holds one unit, the warps split K and reduce through `red` (double-buffered
//             by `parity`), warp 0 finishes.
// `release` is called once per warp as soon as the warp has finished reading the stage.
template <int NB, typename Release>
NT_DEVINL void gemv_consume_stage(const GemvParams& p, const uint8_t* st, const float4* xs, float* red, int wpu,
                                  int first_unit_local, int units_in_stage, int u_begin, int parity, Release release,
                                  const XRegs& xr, bool use_xr) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nch = p.K >> 3;
  const int unit_bytes = 4 * p.K;
  float d0[NB], d1[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) d0[b] = d1[b] = 0.f;
  if (wpu == 1) {
    const bool has = warp < units_in_stage;
    if (has) {
      const uint4* r0 = reinterpret_cast<const uint4*>(st + static_cast<size_t>(warp) * unit_bytes);
      if (NB == 1 && use_xr)
        unit_dot_x1(r0, r0 + nch, 0, nch, lane, xr, d0[0], d1[0]);
      else
        unit_dot<NB>(r0, r0 + nch, xs, nch, 0, nch, lane, d0, d1);
    }
    __syncwarp();
    release();
    if (has) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        d0[b] = warp_sum(d0[b]);
        d1[b] = warp_sum(d1[b]);
      }
      gemv_epilogue<NB>(p, u_begin + first_unit_local + warp, d0, d1, lane);
    }
  } else {
    const int c_lo = (nch * warp) / kConsumerWarps, c_hi = (nch * (warp + 1)) / kConsumerWarps;
    const uint4* r0 = reinterpret_cast<const uint4*>(st);
    if (NB == 1 && use_xr)
      unit_dot_x1(r0, r0 + nch, c_lo, c_hi, lane, xr, d0[0], d1[0]);
    else
      unit_dot<NB>(r0, r0 + nch, xs, nch, c_lo, c_hi, lane, d0, d1);
    __syncwarp();
    release();
    float* rbuf = red + parity * (kConsumerWarps * 2 * 4);
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      d0[b] = warp_sum(d0[b]);
      d1[b] = warp_sum(d1[b]);
    }
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        rbuf[(warp * 2 + 0) * 4 + b] = d0[b];
        rbuf[(warp * 2 + 1) * 4 + b] = d1[b];
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");  // the 8 consumer warps (also the whole CTA minus the producer)
    if (warp == 0) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float t0 = 0.f, t1 = 0.f;
        for (int w = 0; w < kConsumerWarps; ++w) {
          t0 += rbuf[(w * 2 + 0) * 4 + b];
          t1 += rbuf[(w * 2 + 1) * 4 + b];
        }
        d0[b] = t0, d1[b] = t1;
      }
      gemv_epilogue<NB>(p, u_begin + first_unit_local, d0, d1, lane);
    }
  }
}

struct GemvSmemPlan {
  int stage_bytes, nstages, units_per_stage, wpu;
  size_t ring_off, x_off, bar_off, red_off, total;
};

static GemvSmemPlan gemv_plan(int K, int nb) {
  GemvSmemPlan p;
  const int unit_bytes = 4 * K;  // two bf16 rows
  p.wpu = (K >= 2048) ? kConsumerWarps : 1;
  p.units_per_stage = (p.wpu == 1) ? kConsumerWarps : 1;
  p.stage_bytes = unit_bytes * p.units_per_stage;
  p.nstages = (p.wpu == 1) ? 3 : 4;
  size_t off = 0;
  p.ring_off = off;
  off += size_t(p.stage_bytes) * p.nstages;
  p.x_off = off;
  off += size_t(nb) * K * 4;
  p.red_off = off;
  off += 2 * kConsumerWarps * 2 * 4 * sizeof(float);  // [parity][warp][row][nb<=4]
  p.bar_off = off;
  off += 2 * 8 * sizeof(uint64_t) + 64;
  p.total = off + 128;  // alignment slack
  return p;
}

template <int NB>
__global__ void __launch_bounds__(kGemvThreads, 1) gemv_kernel(const GemvParams p, const GemvSmemPlan plan) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  uint8_t* ring = smem + plan.ring_off;
  float4* xs = reinterpret_cast<float4*>(smem + plan.x_off);
  float* red = reinterpret_cast<float*>(smem + plan.red_off);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + plan.bar_off);
  uint64_t* empty_bar = full_bar + 8;
  __shared__ float s_part[kConsumerWarps * 4];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.K;
  const int nunits = p.rows >> 1;
  const int u_begin = static_cast<int>((static_cast<long long>(nunits) * blockIdx.x) / gridDim.x);
  const int u_end = static_cast<int>((static_cast<long long>(nunits) * (blockIdx.x + 1)) / gridDim.x);
  const int my_units = u_end - u_begin;
  const int ups = plan.units_per_stage;
  const int total_stages = (my_units + ups - 1) / ups;
  const int unit_bytes = 4 * K;
  const int NS = plan.nstages;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.W) + static_cast<long long>(u_begin) * unit_bytes;
  auto issue_stage = [&](int it) {
    const int s = it % NS;
    const int u0 = it * ups;
    const int n = min(ups, my_units - u0);
    const uint32_t bytes = static_cast<uint32_t>(n) * unit_bytes;
    mbar_arrive_expect_tx(&full_bar[s], bytes);
    bulk_g2s(ring + static_cast<size_t>(s) * plan.stage_bytes, wbase + static_cast<long long>(u0) * unit_bytes, bytes,
             &full_bar[s]);
  };

  // weight prefetch: independent of the previous kernel, so it goes before the dependency wait
  if (warp == kConsumerWarps && lane == 0) {
    const int pre = min(NS, total_stages);
    for (int it = 0; it < pre; ++it) issue_stage(it);
  }

  pdl_wait();

  if (warp == kConsumerWarps) {
    // ---- producer: refill slots as the consumers release them
    if (lane == 0) {
      for (int it = NS; it < total_stages; ++it) {
        const int s = it % NS;
        const uint32_t ph = ((it / NS) - 1) & 1;  // completion of the slot's previous use
        mbar_wait(&empty_bar[s], ph);
        issue_stage(it);
      }
    }
    return;
  }

  // ---- consumers: input vector(s) -> shared memory planes (+ fused RMSNorm), then the stages
  load_x_planes<NB>(p.x, p.ldx, K, p.norm_w, p.eps, xs, s_part, SyncConsumers());
  XRegs xr = {};
  const int nch_p = K >> 3;
  const int xc_lo = plan.wpu == 1 ? 0 : (nch_p * warp) / kConsumerWarps;
  const int xc_hi = plan.wpu == 1 ? nch_p : (nch_p * (warp + 1)) / kConsumerWarps;
  const bool use_xr = (NB == 1) && (xc_hi - xc_lo) <= 128;
  if (use_xr) load_xregs(xs, nch_p, xc_lo, xc_hi, lane, xr);
  int s = 0;
  uint32_t ph = 0;
  for (int it = 0; it < total_stages; ++it) {
    mbar_wait(&full_bar[s], ph);
    const int first = it * ups;
    const int cur = s;
    gemv_consume_stage<NB>(p, ring + static_cast<size_t>(cur) * plan.stage_bytes, xs, red, plan.wpu, first,
                           min(ups, my_units - first), u_begin, it & 1, [&]() {
                             if (lane == 0) mbar_arrive(&empty_bar[cur]);
                           }, xr, use_xr);
    if (++s == NS) s = 0, ph ^= 1;
  }
}

int launch_gemv(const GemvParams& p, int nb, int num_sms, cudaStream_t stream) {
  if (nb < 1 || nb > 4) return set_error(NT_ERR_INVALID, "gemv: batch %d not in 1..4", nb);
  if (p.rows & 1) return set_error(NT_ERR_INVALID, "gemv: odd row count %d", p.rows);
  if (p.K % 64) return set_error(NT_ERR_INVALID, "gemv: K=%d must be a multiple of 64", p.K);
  GemvSmemPlan plan = gemv_plan(p.K, nb);
  if (plan.total > 227 * 1024) return set_error(NT_ERR_INVALID, "gemv: K=%d needs %zu B of shared memory", p.K, plan.total);
  const int grid = min(num_sms, p.rows / 2);
  void (*kern)(const GemvParams, const GemvSmemPlan) = nullptr;
  switch (nb) {
    case 1: kern = gemv_kernel<1>; break;
    case 2: kern = gemv_kernel<2>; break;
    case 3: kern = gemv_kernel<3>; break;
    default: kern = gemv_kernel<4>; break;
  }
  return launch_kernel(kern, dim3(grid), dim3(kGemvThreads), plan.total, stream, true, p, plan);
}

// One TMA descriptor over the whole paged KV pool viewed as rows of 64 bf16 (a K or V page of one head = 64 rows,
// box = 64 rows x 128 bytes, SWIZZLE_128B).  Row of (layer, k|v, page, head, token):
//   ((layer * 2 + is_v) * num_pages + page) * n_kv_heads + head) * 64 + token
int kv_pool_tmap(const KVLayout& kv, int n_layers, CUtensorMap* out) {
  static std::mutex mu;
  static CUtensorMap cached;
  static const void* c_base = nullptr;
  static long long c_rows = 0;
  const long long rows = static_cast<long long>(n_layers) * 2 * kv.num_pages * kv.n_kv_heads * 64;
  if (rows >= (1ll << 31)) return set_error(NT_ERR_INVALID, "attention: KV pool too large for one TMA descriptor");
  std::lock_guard<std::mutex> lock(mu);
  if (c_base != kv.pages || c_rows != rows) {
    if (int rc = make_tmap(&cached, NT_BF16, kv.pages, static_cast<uint64_t>(rows), 64, 64, 64)) return rc;
    c_base = kv.pages, c_rows = rows;
  }
  *out = cached;
  return NT_OK;
}

// =================================================================================== decode attention
// grid (n_kv_heads, B), 512 threads: one CTA per (sequence, kv head), no cross-CTA partials.  The 16 warps form
// 8 pairs; each pair owns a 16 KB K/V staging buffer and walks pages pair, pair+8, ... on its own (TMA -> the
// pair's mbarrier -> fp32 scores -> online softmax -> P.V; each warp takes 32 of the page's 64 tokens), so the
// page loads of different pairs overlap and only the final merge needs a CTA-wide barrier.  The 16 warp partials
// merge through shared memory in warp order.
//
// Shared-memory bandwidth is what bounds this kernel (ncu: 18.8 k wavefronts per CTA, 5-way "conflicts"), so the
// layout is chosen to make every query read a whole-warp broadcast: lane = token, all lanes walk the same 16-byte
// chunk c of their K rows at the same time, and the K page lands in shared memory through a SWIZZLE_128B tensor
// map (chunk c of row r sits at chunk c ^ (r & 7)), which keeps those row-strided reads conflict-free.
// (History: split-KV grid + last-arriver merge 29 us; 8 warps x whole pages 17 us; per-lane rotated chunk order
// with non-broadcast query reads 21 us.)
constexpr int kAttnPairs = 8;
constexpr int kAttnWarps = 2 * kAttnPairs;
struct AttnWarpSmem {
  __nv_bfloat16 k[kAttnPairs][64 * 64];   // swizzled (TMA); each buffer 8 KB => 1024-byte aligned
  __nv_bfloat16 v[kAttnPairs][64 * 64];   // linear (bulk copy)
  float q[8][64];               // pre-scaled by softmax scale * log2(e)
  float p[kAttnWarps][32][8];   // probabilities [token][head]
  float o[kAttnWarps][8][64];   // per-warp unnormalised outputs
  float ml[kAttnWarps][8][2];
  uint64_t bar[kAttnPairs];
};
__global__ void __launch_bounds__(32 * kAttnWarps) attn_decode_kernel(const AttnDecParams p, const __grid_constant__ CUtensorMap kmap) {
  extern __shared__ uint8_t attn_raw[];
  // array + offset keeps the shared address space visible to the compiler (LDS, not generic loads)
  AttnWarpSmem* sm = reinterpret_cast<AttnWarpSmem*>(attn_raw + ((1024u - (smem_u32(attn_raw) & 1023u)) & 1023u));
  pdl_launch_dependents();
  const int kvh = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int pair = warp >> 1, sub = warp & 1;
  const int n_rep = p.n_rep;
  if (sub == 0 && lane == 0) {
    if (pair == 0) tma_prefetch_desc(&kmap);
    mbar_init(&sm->bar[pair], 1);
    fence_barrier_init();
  }
  pdl_wait();
  const int n_ctx = min(__ldcg(p.kv.seq_lens + b) + 1, p.kv.max_ctx);
  const int npages = (n_ctx + 63) >> 6;
  for (int i = tid; i < n_rep * 64; i += 32 * kAttnWarps)
    sm->q[i >> 6][i & 63] = p.scale_log2 * __ldcg(p.q + (static_cast<long long>(b) * p.n_heads + kvh * n_rep + (i >> 6)) * 64 + (i & 63));
  __syncthreads();

  float m[8], l[8], acc[8][2];
#pragma unroll
  for (int h = 0; h < 8; ++h) m[h] = -INFINITY, l[h] = 0.f, acc[h][0] = 0.f, acc[h][1] = 0.f;
  uint32_t parity = 0;
  const __nv_bfloat16* kb = sm->k[pair] + (sub * 32 + lane) * 64;  // this lane's token row of the page
  const __nv_bfloat16* vb = sm->v[pair] + sub * 32 * 64;           // this warp's 32 token rows
  for (int pg = pair; pg < npages; pg += kAttnPairs) {
    if (sub == 0 && lane == 0) {
      const int page = __ldcg(p.kv.page_table + b * p.kv.max_pages_per_seq + pg);
      asm volatile("fence.proxy.async;" ::: "memory");
      mbar_arrive_expect_tx(&sm->bar[pair], 2 * 8192);
      tma_load_2d(sm->k[pair], &kmap, 0, p.kv.tmap_row(p.layer, 0, page, kvh), &sm->bar[pair]);
      bulk_g2s(sm->v[pair], p.kv.page_ptr(p.layer, 1, page, kvh), 8192, &sm->bar[pair]);
    }
    mbar_wait(&sm->bar[pair], parity);
    parity ^= 1;
    const int tok0 = pg * 64 + sub * 32;
    if (tok0 < n_ctx) {  // warp-uniform: the second half of the last page may be entirely beyond the context
      float d[8];
#pragma unroll
      for (int h = 0; h < 8; ++h) d[h] = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        float f[8];
        bf16x8_to_f32(*reinterpret_cast<const uint4*>(kb + ((c ^ (lane & 7)) << 3)), f);  // logical chunk c, swizzled
#pragma unroll
        for (int h = 0; h < 8; ++h) {
          if (h < n_rep) {
            const float4 qa = *reinterpret_cast<const float4*>(&sm->q[h][c * 8]);      // same address in all lanes
            const float4 qb = *reinterpret_cast<const float4*>(&sm->q[h][c * 8 + 4]);
            d[h] += f[0] * qa.x + f[1] * qa.y + f[2] * qa.z + f[3] * qa.w + f[4] * qb.x + f[5] * qb.y + f[6] * qb.z + f[7] * qb.w;
          }
        }
      }
      // online softmax (fp32, base-2); running (m, l) replicated in every lane
      const bool valid = (tok0 + lane) < n_ctx;
#pragma unroll
      for (int h = 0; h < 8; ++h) {
        if (h < n_rep) {
          const float sc = valid ? d[h] : -INFINITY;
          const float mn = fmaxf(m[h], warp_max(sc));   // token tok0 is valid -> finite
          d[h] = exp2f(sc - mn);
          const float c = exp2f(m[h] - mn);             // 0 on the warp's first page
          l[h] = l[h] * c + warp_sum(d[h]);
          m[h] = mn;
          acc[h][0] *= c, acc[h][1] *= c;
        }
      }
      *reinterpret_cast<float4*>(&sm->p[warp][lane][0]) = make_float4(d[0], d[1], d[2], d[3]);
      *reinterpret_cast<float4*>(&sm->p[warp][lane][4]) = make_float4(d[4], d[5], d[6], d[7]);
      __syncwarp();
      // P.V: lane = dims (2 lane, 2 lane + 1); probabilities are whole-warp broadcasts
#pragma unroll 8
      for (int t = 0; t < 32; ++t) {
        const float2 vv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vb + t * 64 + 2 * lane));
        const float4 pa = *reinterpret_cast<const float4*>(&sm->p[warp][t][0]);
        const float4 pb = *reinterpret_cast<const float4*>(&sm->p[warp][t][4]);
        const float pr[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
#pragma unroll
        for (int h = 0; h < 8; ++h)
          if (h < n_rep) acc[h][0] += pr[h] * vv.x, acc[h][1] += pr[h] * vv.y;
      }
    }
    // both warps of the pair are done with the buffers before the next copies overwrite them
    asm volatile("bar.sync %0, 64;" ::"r"(1 + pair) : "memory");
  }
#pragma unroll
  for (int h = 0; h < 8; ++h) {
    if (h < n_rep) {
      *reinterpret_cast<float2*>(&sm->o[warp][h][2 * lane]) = make_float2(acc[h][0], acc[h][1]);
      if (lane == 0) sm->ml[warp][h][0] = m[h], sm->ml[warp][h][1] = l[h];
    }
  }
  __syncthreads();
  for (int i = tid; i < n_rep * 64; i += 32 * kAttnWarps) {
    const int h = i >> 6, d = i & 63;
    // captured by value: by reference, ptxas gives this kernel 2 more registers (CUDA 12.9)
    const SoftmaxPart r = merge_parts<kAttnWarps>(kAttnWarps, [=](int w) { return SoftmaxPart{sm->ml[w][h][0], sm->ml[w][h][1], sm->o[w][h][d]}; });
    const long long hh = static_cast<long long>(b) * p.n_heads + kvh * n_rep + h;
    if (p.out) p.out[hh * 64 + d] = r.o / r.l;
    if (p.out_bf16) p.out_bf16[hh * 64 + d] = __float2bfloat16(r.o / r.l);
  }
}


// Batched-decode variant on tensor cores (batch > 4, where GEMM inputs are bf16 anyway): same CTA shape -- one CTA
// per (sequence, kv head), warps walk pages warp, warp+8, ... through private 16 KB K/V buffers (both pages by
// swizzled TMA) -- but a page is one attn_page_step: S[16 x 64] = Q K^T with the n_rep query heads in rows
// 0..n_rep-1 of the A tile (rows 8..15 are zero), online softmax on the accumulator fragments, O += P V with P
// rounded to bf16.  ~150 instructions per page instead of ~2 200 on the fp32 path.
struct AttnMmaSmem {
  __nv_bfloat16 k[8][64 * 64];
  __nv_bfloat16 v[8][64 * 64];
  float o[8][8][64];   // per-warp unnormalised outputs [head][dim]
  float ml[8][8][2];
  uint64_t bar[8];
  float q[8][64];      // prologue: this group's rotated queries, the new token's K / V row
  float knew[64], vnew[64];
};
__global__ void __launch_bounds__(256) attn_decode_mma_kernel(const AttnDecParams p, const __grid_constant__ CUtensorMap kvmap) {
  extern __shared__ uint8_t attn_raw[];
  AttnMmaSmem* sm = reinterpret_cast<AttnMmaSmem*>(attn_raw + ((1024u - (smem_u32(attn_raw) & 1023u)) & 1023u));
  pdl_launch_dependents();
  const int kvh = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_rep = p.n_rep;
  if (lane == 0) {
    if (warp == 0) tma_prefetch_desc(&kvmap);
    mbar_init(&sm->bar[warp], 1);
    fence_barrier_init();
  }
  pdl_wait();
  const int pos = __ldcg(p.kv.seq_lens + b);   // position of the new token
  const int n_ctx = min(pos + 1, p.kv.max_ctx);
  const int npages = (n_ctx + 63) >> 6;
  const bool appends = pos < p.kv.max_ctx;
  // RoPE + KV append of this (sequence, kv head) -- what rope_append_kernel did in a launch of its own: pair u of a
  // head holds dims (i, i + 32) (rows are pair-interleaved at pack time), V is plain.  Slices summed in slice order.
  const float* row = p.qkv + static_cast<long long>(b) * p.qkv_n;
  const int n_kv = p.kv.n_kv_heads;
  for (int idx = tid; idx < (n_rep + 2) * 32; idx += 256) {
    const int which = idx < n_rep * 32 ? 0 : (idx < n_rep * 32 + 32 ? 1 : 2);
    const int i = idx & 31;
    const int col = (which == 0 ? (kvh * n_rep + (idx >> 5)) : (which == 1 ? p.n_heads + kvh : p.n_heads + n_kv + kvh)) * 64 + 2 * i;
    float2 v = __ldcg(reinterpret_cast<const float2*>(row + col));
    for (int z = 1; z < p.qkv_parts; ++z) {
      const float2 w = __ldcg(reinterpret_cast<const float2*>(row + z * p.qkv_pstride + col));
      v.x += w.x, v.y += w.y;
    }
    if (which == 2) {
      sm->vnew[2 * i] = v.x, sm->vnew[2 * i + 1] = v.y;
    } else {
      const float2 r = rope_pair(v.x, v.y, pos, __ldg(p.inv_freq + i));
      if (which == 0) sm->q[idx >> 5][i] = r.x, sm->q[idx >> 5][i + 32] = r.y;
      else sm->knew[i] = r.x, sm->knew[i + 32] = r.y;
    }
  }
  __syncthreads();
  if (appends && tid < 64) {   // the row joins the cache for the steps to come; this step patches it into the staged page
    const int page = __ldcg(p.kv.page_table + b * p.kv.max_pages_per_seq + (pos >> 6));
    p.kv.page_ptr(p.layer, 0, page, kvh)[(pos & 63) * 64 + tid] = __float2bfloat16(sm->knew[tid]);
    p.kv.page_ptr(p.layer, 1, page, kvh)[(pos & 63) * 64 + tid] = __float2bfloat16(sm->vnew[tid]);
  }
  uint32_t qa[4][4];
  decode_query_frags(&sm->q[0][0], n_rep, p.scale_log2, qa);
  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m[1] = {-INFINITY}, l[1] = {0.f};
  const uint32_t kbase = smem_u32(sm->k[warp]), vbase = smem_u32(sm->v[warp]);
  uint32_t parity = 0;
  for (int pg = warp; pg < npages; pg += 8) {
    if (lane == 0) {
      const int page = __ldcg(p.kv.page_table + b * p.kv.max_pages_per_seq + pg);
      asm volatile("fence.proxy.async;" ::: "memory");
      mbar_arrive_expect_tx(&sm->bar[warp], 2 * 8192);
      tma_load_2d(sm->k[warp], &kvmap, 0, p.kv.tmap_row(p.layer, 0, page, kvh), &sm->bar[warp]);
      tma_load_2d(sm->v[warp], &kvmap, 0, p.kv.tmap_row(p.layer, 1, page, kvh), &sm->bar[warp]);
    }
    mbar_wait(&sm->bar[warp], parity);
    parity ^= 1;
    if (appends && pg == (pos >> 6)) patch_staged_row(sm->k[warp], sm->v[warp], pos & 63, sm->knew, sm->vnew);
    const int k0 = pg * 64;
    attn_page_step<1>(kbase, vbase, qa, o, m, l, k0 + 64 > n_ctx, [&](int, int key) { return k0 + key >= n_ctx; });
    __syncwarp();  // all lanes are done with the buffers before lane 0 refills them
  }
  decode_store_partial(o, m[0], l[0], n_rep, &sm->o[warp][0][0], &sm->ml[warp][0][0]);
  __syncthreads();
  for (int i = tid; i < n_rep * 64; i += 256) {
    const int h = i >> 6, d = i & 63;
    const SoftmaxPart r = merge_parts<8>(8, [=](int w) { return SoftmaxPart{sm->ml[w][h][0], sm->ml[w][h][1], sm->o[w][h][d]}; });
    const long long hh = static_cast<long long>(b) * p.n_heads + kvh * n_rep + h;
    if (p.out) p.out[hh * 64 + d] = r.o / r.l;
    if (p.out_bf16) p.out_bf16[hh * 64 + d] = __float2bfloat16(r.o / r.l);
  }
}

int launch_attn_decode(const AttnDecParams& p, int B, int n_layers, cudaStream_t stream) {
  if (p.n_rep < 1 || p.n_rep > 8) return set_error(NT_ERR_INVALID, "attention: %d query heads per KV head unsupported (1..8)", p.n_rep);
  const int smem = int(sizeof(AttnWarpSmem)) + 1024;
  CUtensorMap kmap;
  if (int rc = kv_pool_tmap(p.kv, n_layers, &kmap)) return rc;
  if (B > 4) {  // tensor-core variant: bf16 query / probabilities, like every other GEMM input of the batched path
    if (!p.qkv) return set_error(NT_ERR_INVALID, "attention: batch %d > 4 needs the fused RoPE + KV append (qkv)", B);
    const int msmem = int(sizeof(AttnMmaSmem)) + 1024;
    return launch_kernel(attn_decode_mma_kernel, dim3(p.kv.n_kv_heads, B), dim3(256), msmem, stream, true, p, kmap);
  }
  return launch_kernel(attn_decode_kernel, dim3(p.kv.n_kv_heads, B), dim3(32 * kAttnWarps), smem, stream, true, p, kmap);
}

// =================================================================================== sampler
// candidate arrays: [sequence][kCandPitch], the general path of sample_tiles_seq writes up to 256 * kTopKeep
// candidates per sequence
size_t sampler_scratch_floats(int B) { return size_t(B) * kCandPitch; }

// The general path of sample_tiles_seq stages one key per 128-id tile in shared memory: at most kMaxTiles tiles
// (50 KB of keys), i.e. V <= 1 638 400.
constexpr int kMaxTiles = 12800;

int launch_sampler_check(const SamplerParams& p) {
  if (p.sp.top_k < 1 || p.sp.top_k > kTopKeep) return set_error(NT_ERR_INVALID, "sampler: top_k=%d not in 1..64", p.sp.top_k);
  if (!(p.sp.temperature > 0.f)) return set_error(NT_ERR_INVALID, "sampler: temperature must be > 0");
  if ((p.V + 127) / 128 > kMaxTiles) return set_error(NT_ERR_INVALID, "sampler: vocabulary too large (%d)", p.V);
  return NT_OK;
}

// Raw maximum of every 128-id tile of logits rows [0, B) -> tmax [B][nt] (the last tile may be partial): the maxima
// the lm_head GEMM epilogue writes when it tiles the vocabulary by 128, for every other lm_head and for
// nt_op_topk_sample.  grid (ceil(nt / 8), B), 256 threads: one warp per tile, one float4 per lane.
__global__ void __launch_bounds__(256) tile_max_kernel(const float* logits, int V, float* tmax, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int tile = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (tile >= nt) return;
  const float* lg = logits + static_cast<long long>(blockIdx.y) * V;
  const int r0 = tile * 128 + lane * 4;
  float m = -INFINITY;
  // row b starts b * V floats in: with V % 4 != 0 only some rows are 16-byte aligned for the float4 load
  if ((reinterpret_cast<uintptr_t>(lg) & 15) == 0 && r0 + 3 < V) {
    const float4 x = __ldcg(reinterpret_cast<const float4*>(lg + r0));
    m = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
  } else {
    for (int q = 0; q < 4; ++q)
      if (r0 + q < V) m = fmaxf(m, __ldcg(lg + r0 + q));
  }
  m = warp_max(m);
  if (lane == 0) tmax[static_cast<long long>(blockIdx.y) * nt + tile] = m;
}
int launch_tile_max(const float* logits, int B, int V, float* tmax, cudaStream_t s) {
  const int nt = (V + 127) / 128;
  return launch_kernel(tile_max_kernel, dim3((nt + 7) / 8, B), dim3(256), 0, s, true, logits, V, tmax, nt);
}

// Tile-max sampler outside the persistent decode kernel: tmax holds the RAW maximum of every 128-column tile per
// sequence (the lm_head GEMM epilogue's, or launch_tile_max's); one CTA per sequence picks the candidate tiles from
// those maxima and ranks the few dozen candidate logits (sample_tiles_seq, the scheme of the persistent decode kernel).
struct NoMarkI {
  NT_DEVINL void operator()(int) const {}
};
constexpr unsigned kTilesScratch = 96 * 1024;
__global__ void __launch_bounds__(kConsumerThreads) topk_tiles_kernel(const __grid_constant__ SamplerParams p, const float* tmax, const int nt,
                                                                      const int32_t* skip) {
  extern __shared__ uint8_t tiles_raw[];
  uint8_t* uni = tiles_raw + ((1024u - (smem_u32(tiles_raw) & 1023u)) & 1023u);
  __shared__ int sel[8];
  __shared__ float fix;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = p.row_slot ? __ldg(p.row_slot + b) : b;
  if (skip && __ldg(skip + slot) >= 0) return;   // CTA-uniform: an unconditional slot of a guided pair
  const int src = p.row_src ? __ldg(p.row_src + b) : -1;   // logits / tile-maxima row (-1: row b)
  const bool stateless = p.n_generated_override != nullptr;
  const int ngen = stateless ? __ldcg(p.n_generated_override + b) : __ldcg(p.n_generated + slot);
  const bool mask_eos = ngen < row_min_new(p, slot);
  const float inv_t = row_sampling(p, slot).inv_t;
  int fix_tile = -1;
  float fix_val = 0.f;
  if (mask_eos) {   // the raw maximum of the tile that holds EOS may be the (masked) EOS logit itself: redo that tile without it
    fix_tile = p.sp.eos_id >> 7;
    if (warp == 0) {
      float m = -INFINITY;
      for (int q = 0; q < 4; ++q) {
        const int r = fix_tile * 128 + lane * 4 + q;
        if (r < p.V && r != p.sp.eos_id) m = fmaxf(m, __ldcg(p.logits + static_cast<long long>(src >= 0 ? src : b) * p.V + r));
      }
      m = warp_max(m);
      if (lane == 0) fix = m * inv_t;
    }
    __syncthreads();
    fix_val = fix;
  }
  sample_tiles_seq(p, b, tmax, nt, inv_t, fix_tile, fix_val, p.logits, p.V, mask_eos, uni, kTilesScratch, sel, SyncAll(), NoMarkI(),
                   static_cast<float2*>(nullptr), 0.f, stateless, slot, src);
}

int launch_sampler_tiles(const SamplerParams& p, int B, const float* tmax, int nt, cudaStream_t stream, const int32_t* skip) {
  if (int rc0 = launch_sampler_check(p)) return rc0;
  const int smem = int(kTilesScratch) + 1024;
  return launch_kernel(topk_tiles_kernel, dim3(B), dim3(kConsumerThreads), smem, stream, true, p, tmax, nt, skip);
}

// =================================================================================== vocabulary range
__global__ void fill_neg_inf_kernel(float* p, long long n) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
    p[i] = -INFINITY;
}
int launch_fill_neg_inf(float* p, long long n, cudaStream_t s) {
  if (n <= 0) return NT_OK;
  const long long blocks = (n + 255) / 256;
  return launch_kernel(fill_neg_inf_kernel, dim3(static_cast<unsigned>(blocks < 1024 ? blocks : 1024)), dim3(256), 0, s, true, p, n);
}

// grid B, 128 threads: thread r owns row tile * 128 + r of logits row blockIdx.x
__global__ void vocab_eos_tile_kernel(float* logits, int V, int eos, float* tmax, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int tile = eos >> 7, row = tile * 128 + threadIdx.x;
  float* lg = logits + static_cast<long long>(blockIdx.x) * V;
  if (row < V && row != eos) lg[row] = -INFINITY;
  if (tmax && threadIdx.x == 0) tmax[static_cast<long long>(blockIdx.x) * nt + tile] = lg[eos];
}
int launch_vocab_eos_tile(float* logits, int B, int V, int eos, float* tmax, int nt, cudaStream_t s) {
  return launch_kernel(vocab_eos_tile_kernel, dim3(B), dim3(128), 0, s, true, logits, V, eos, tmax, nt);
}

// =================================================================================== repetition penalty
// grid B, 256 threads: the history row of one slot is built in shared memory (ceil(V / 32) words) and written once
__global__ void __launch_bounds__(256) rep_history_kernel(uint32_t* hist, int words, const nt_slot_penalty* tab, int32_t* recorded,
                                                          const int32_t* row_slot, const int32_t* ids, const int32_t* cu, int V) {
  extern __shared__ uint32_t rep_row[];
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, s = row_slot ? row_slot[i] : i;
  for (int w = threadIdx.x; w < words; w += blockDim.x) rep_row[w] = 0u;
  __syncthreads();
  if (tab[s].include_prompt) {
    for (int t = cu[i] + threadIdx.x; t < cu[i + 1]; t += blockDim.x) {
      const int id = ids[t];
      if (id >= 0 && id < V) atomicOr(&rep_row[id >> 5], 1u << (id & 31));
    }
  }
  __syncthreads();
  uint32_t* dst = hist + static_cast<long long>(s) * words;
  for (int w = threadIdx.x; w < words; w += blockDim.x) dst[w] = rep_row[w];
  if (threadIdx.x == 0) recorded[s] = 1;
}
int launch_rep_history(uint32_t* hist, int words, const nt_slot_penalty* tab, int32_t* recorded, const int32_t* row_slot,
                       const int32_t* ids, const int32_t* cu, int B, int V, cudaStream_t s) {
  return launch_kernel(rep_history_kernel, dim3(B), dim3(256), size_t(words) * sizeof(uint32_t), s, true, hist, words, tab, recorded,
                       row_slot, ids, cu, V);
}

// grid (B, kRepSplit), 256 threads: the kRepSplit CTAs of row i share its tiles.  A warp takes 8 tiles (32 bitmap
// words, one per lane) at a time and skips the tiles with no id in the history (a 500-token prompt touches ~40 % of
// the Air vocabulary's tiles, and one warp walking them in series is latency-bound); lane l owns rows tile * 128 + 4 l .. + 3, i.e. bits 4 (l % 8) .. + 3 of the tile's word l / 8.  The
// history ids are distinct, so every logit is rewritten once and each tile belongs to one warp (no race).
__global__ void __launch_bounds__(256) rep_penalty_kernel(float* logits, int V, const uint32_t* hist, int words, const nt_slot_penalty* tab,
                                                          const int32_t* recorded, const int32_t* row_slot, float* tmax, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, s = row_slot ? row_slot[i] : i;
  const float pen = tab[s].penalty;
  if (!recorded[s] || pen == 1.f) return;
  const uint32_t* hrow = hist + static_cast<long long>(s) * words;
  float* lg = logits + static_cast<long long>(i) * V;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nw = (blockDim.x >> 5) * gridDim.y;
  for (int g = blockIdx.y * (blockDim.x >> 5) + warp; g * 8 < nt; g += nw) {
    const int w = g * 32 + lane;
    const uint32_t word = w < words ? __ldcg(hrow + w) : 0u;
    const uint32_t any = __ballot_sync(0xffffffffu, word != 0u);
    for (int j = 0; j < 8; ++j) {
      if (!((any >> (4 * j)) & 0xfu)) continue;   // warp-uniform
      const int tile = g * 8 + j;
      const uint32_t bits = (__shfl_sync(0xffffffffu, word, 4 * j + (lane >> 3)) >> (4 * (lane & 7))) & 0xfu;
      float m = -INFINITY;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = tile * 128 + 4 * lane + q;
        if (r < V) {
          float v = lg[r];
          if ((bits >> q) & 1u) {
            v = rep_penalize(v, pen);
            lg[r] = v;
          }
          m = fmaxf(m, v);
        }
      }
      m = warp_max(m);
      if (tmax && lane == 0) tmax[static_cast<long long>(i) * nt + tile] = m;
    }
  }
}
int launch_rep_penalty(float* logits, int B, int V, const uint32_t* hist, int words, const nt_slot_penalty* tab,
                       const int32_t* recorded, const int32_t* row_slot, float* tmax, int nt, cudaStream_t s) {
  constexpr int kRepSplit = 16;
  return launch_kernel(rep_penalty_kernel, dim3(B, kRepSplit), dim3(256), 0, s, true, logits, V, hist, words, tab, recorded, row_slot,
                       tmax, nt);
}

// =================================================================================== length control
// grid B, 128 threads: thread r owns row (eos tile) * 128 + r of logits row b, which holds slot b.  The decay is read
// from n_generated before this step's sampler advances it, so it is the n the sampler draws at.
__global__ void len_decay_kernel(const SamplerParams p, float* logits, float* tmax, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, eos = p.sp.eos_id, tile = eos >> 7, row = tile * 128 + threadIdx.x;
  const float c = len_decay_c(p, b, __ldcg(p.n_generated + b));
  if (c == 0.f) return;   // CTA-uniform: no decay for this slot at this step
  float* lg = logits + static_cast<long long>(b) * p.V;
  float v = row < p.V ? lg[row] : -INFINITY;
  if (row == eos) lg[row] = v = len_decay(v, c);
  if (!tmax) return;
  __shared__ float red[4];
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) tmax[static_cast<long long>(b) * nt + tile] = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
}
int launch_len_decay(const SamplerParams& p, int B, float* logits, float* tmax, int nt, cudaStream_t s) {
  return launch_kernel(len_decay_kernel, dim3(B), dim3(128), 0, s, true, p, logits, tmax, nt);
}

// =================================================================================== classifier-free guidance
// Online log-sum-exp in fp32 with the accurate expf: a (max, sum exp(x - max)) pair per thread, merged in a fixed order.
NT_DEVINL void lse_add(float& m, float& s, float x) {
  if (x > m) {
    s = s * expf(m - x) + 1.f;
    m = x;
  } else if (x > -INFINITY) {
    s += expf(x - m);
  }
}
NT_DEVINL void lse_merge(float& m, float& s, float m1, float s1) {
  const float mm = fmaxf(m, m1);
  s = mm == -INFINITY ? 0.f : s * expf(m - mm) + s1 * expf(m1 - mm);
  m = mm;
}
// the 4 ids r0 .. r0 + 3 of one row (a float4 where the row is 16-byte aligned there; ids >= V read -inf)
NT_DEVINL float4 load4(const float* lg, int r0, int V) {
  if ((reinterpret_cast<uintptr_t>(lg + r0) & 15) == 0 && r0 + 3 < V) return __ldcg(reinterpret_cast<const float4*>(lg + r0));
  float v[4];
  for (int q = 0; q < 4; ++q) v[q] = r0 + q < V ? __ldcg(lg + r0 + q) : -INFINITY;
  return make_float4(v[0], v[1], v[2], v[3]);
}
// the tiles [t0, t1) of CTA x when nt tiles are shared by kGuideSplit CTAs
NT_DEVINL void guide_chunk(int nt, int x, int& t0, int& t1) {
  const int per = (nt + kGuideSplit - 1) / kGuideSplit;
  t0 = min(nt, x * per), t1 = min(nt, t0 + per);
}

// grid (kGuideSplit, B, 2), 256 threads: CTA (x, r, z) folds its share of the tiles of row r (z = 0) or of r's partner
// (z = 1) into part[r][z][x]; a warp takes one 128-id tile at a time, a lane 4 ids.
__global__ void __launch_bounds__(256) guidance_lse_kernel(const float* logits, int V, const nt_slot_guidance* tab, float2* part, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.y, u = __ldg(&tab[r].partner);
  if (u < 0) return;
  const float* lg = logits + static_cast<long long>(blockIdx.z ? u : r) * V;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t0, t1;
  guide_chunk(nt, blockIdx.x, t0, t1);
  float m = -INFINITY, s = 0.f;
  for (int t = t0 + warp; t < t1; t += 8) {
    const float4 v = load4(lg, t * 128 + 4 * lane, V);
    lse_add(m, s, v.x), lse_add(m, s, v.y), lse_add(m, s, v.z), lse_add(m, s, v.w);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, off), __shfl_xor_sync(0xffffffffu, s, off));
  __shared__ float2 red[8];
  if (lane == 0) red[warp] = make_float2(m, s);
  __syncthreads();
  if (threadIdx.x == 0) {
    m = -INFINITY, s = 0.f;
    for (int w = 0; w < 8; ++w) lse_merge(m, s, red[w].x, red[w].y);
    part[(static_cast<long long>(r) * 2 + blockIdx.z) * kGuideSplit + blockIdx.x] = make_float2(m, s);
  }
}

// grid (kGuideSplit, B), 256 threads: CTA (x, r) folds both rows' partials in index order (every CTA of the row gets
// the same log-sum-exps), then rewrites its share of c row r and the tile maxima.
__global__ void __launch_bounds__(256) guidance_mix_kernel(float* logits, int V, const nt_slot_guidance* tab, const float2* part,
                                                           float* tmax, int nt) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.y, u = __ldg(&tab[r].partner);
  if (u < 0) return;
  __shared__ float lse[2];
  if (threadIdx.x < 2) {
    const float2* pr = part + (static_cast<long long>(r) * 2 + threadIdx.x) * kGuideSplit;
    float m = -INFINITY, s = 0.f;
    for (int x = 0; x < kGuideSplit; ++x) {
      const float2 v = __ldcg(pr + x);
      lse_merge(m, s, v.x, v.y);
    }
    lse[threadIdx.x] = m + logf(s);
  }
  __syncthreads();
  const float lse_c = lse[0], lse_u = lse[1], g = __ldg(&tab[r].scale);
  float* lc = logits + static_cast<long long>(r) * V;
  const float* lu = logits + static_cast<long long>(u) * V;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int t0, t1;
  guide_chunk(nt, blockIdx.x, t0, t1);
  for (int t = t0 + warp; t < t1; t += 8) {
    const int r0 = t * 128 + 4 * lane;
    const float4 c4 = load4(lc, r0, V), u4 = load4(lu, r0, V);
    const float xc[4] = {c4.x, c4.y, c4.z, c4.w}, xu[4] = {u4.x, u4.y, u4.z, u4.w};
    float y[4], mx = -INFINITY;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      // transformers' `g * (scores - uncond) + uncond` on the log-softmaxes, unfused; a suppressed id stays -inf
      // (g * (-inf - -inf) would be NaN)
      const float ls_u = __fsub_rn(xu[q], lse_u);
      y[q] = (xc[q] == -INFINITY || xu[q] == -INFINITY) ? -INFINITY
                                                        : __fadd_rn(__fmul_rn(g, __fsub_rn(__fsub_rn(xc[q], lse_c), ls_u)), ls_u);
      mx = fmaxf(mx, y[q]);
    }
    if ((reinterpret_cast<uintptr_t>(lc + r0) & 15) == 0 && r0 + 3 < V) {
      *reinterpret_cast<float4*>(lc + r0) = make_float4(y[0], y[1], y[2], y[3]);
    } else {
      for (int q = 0; q < 4; ++q)
        if (r0 + q < V) lc[r0 + q] = y[q];
    }
    mx = warp_max(mx);
    if (tmax && lane == 0) tmax[static_cast<long long>(r) * nt + t] = mx;
  }
}

int launch_guidance_combine(float* logits, int B, int V, const nt_slot_guidance* tab, float2* part, float* tmax, int nt,
                            cudaStream_t s) {
  int rc = launch_kernel(guidance_lse_kernel, dim3(kGuideSplit, B, 2), dim3(256), 0, s, true, static_cast<const float*>(logits), V, tab,
                         part, nt);
  return rc ? rc : launch_kernel(guidance_mix_kernel, dim3(kGuideSplit, B), dim3(256), 0, s, true, logits, V, tab,
                                 static_cast<const float2*>(part), tmax, nt);
}

// grid B, 256 threads: CTA i mirrors the sampler's state update of row i's slot onto its partner
__global__ void __launch_bounds__(256) guidance_follow_kernel(const SamplerParams p, const nt_slot_guidance* tab) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = p.row_slot ? __ldg(p.row_slot + blockIdx.x) : static_cast<int>(blockIdx.x);
  const int u = __ldg(&tab[c].partner);
  if (u < 0) return;
  __shared__ int s_tok;
  if (threadIdx.x == 0) {
    s_tok = -1;
    if (!__ldcg(p.done + u)) {
      const int n = __ldcg(p.n_generated + c), tok = __ldcg(p.cur_token + c);
      p.out_tokens[static_cast<long long>(u) * p.max_new + n - 1] = tok;
      p.n_generated[u] = n;
      p.cur_token[u] = tok;
      const int cached = __ldcg(p.seq_lens + u) + p.advance;
      p.seq_lens[u] = cached;
      int d = __ldcg(p.done + c);
      if (cached + 1 >= p.max_ctx) p.done[c] = d = 1;
      p.done[u] = d;
      s_tok = tok;
    }
  }
  __syncthreads();
  if (s_tok < 0 || !p.h) return;
  const __nv_bfloat16* e = p.embed + static_cast<long long>(s_tok) * p.hidden;
  for (int i = threadIdx.x; i < p.hidden; i += blockDim.x) p.h[static_cast<long long>(u) * p.hidden + i] = __bfloat162float(e[i]);
}
int launch_guidance_follow(const SamplerParams& p, int B, const nt_slot_guidance* tab, cudaStream_t s) {
  return launch_kernel(guidance_follow_kernel, dim3(B), dim3(256), 0, s, true, p, tab);
}

// =================================================================================== prefill helpers
__global__ void embed_rows_kernel(const __nv_bfloat16* embed, const int32_t* ids, int hidden, float* h) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const __nv_bfloat16* e = embed + static_cast<long long>(ids[t]) * hidden;
  for (int i = threadIdx.x; i < hidden; i += blockDim.x) h[static_cast<long long>(t) * hidden + i] = __bfloat162float(e[i]);
}
int launch_embed_rows(const __nv_bfloat16* embed, const int32_t* ids, int T, int hidden, float* h, cudaStream_t s) {
  return launch_kernel(embed_rows_kernel, dim3(T), dim3(256), 0, s, true, embed, ids, hidden, h);
}

// one warp per row; fp32 statistics; out = w * (x * rsqrt(mean(x^2)+eps))  (modeling_qwen2.py:258-263)
// 16-byte loads, eight of them in flight per lane (the scalar version spent 16 us per launch on load latency).
// With `parts`: first folds the split-K slices of the preceding in-place GEMM into the residual stream,
// x[row] += parts[0][row] + parts[1][row] + ... in slice order (so the sum is reproducible), and writes x back.
__global__ void __launch_bounds__(256) rmsnorm_rows_kernel(float* x, const float* w, float eps, int rows, int cols,
                                                           float* out_f32, __nv_bfloat16* out_bf16, const float* parts,
                                                           int nparts, long long pstride) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4* xr = reinterpret_cast<float4*>(x + static_cast<long long>(row) * cols);
  const float4* wr = reinterpret_cast<const float4*>(w);
  const int nvec = cols >> 2;  // cols % 4 == 0 (checked by the launcher)
  float ss = 0.f;
  for (int i0 = lane; i0 < nvec; i0 += 32 * 8) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (i0 + 32 * j < nvec) ? xr[i0 + 32 * j] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (nparts > 0) {
      for (int z = 0; z < nparts; ++z) {
        const float4* pr = reinterpret_cast<const float4*>(parts + z * pstride + static_cast<long long>(row) * cols);
        float4 t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t[j] = (i0 + 32 * j < nvec) ? __ldcg(pr + i0 + 32 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j].x += t[j].x, v[j].y += t[j].y, v[j].z += t[j].z, v[j].w += t[j].w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (i0 + 32 * j < nvec) xr[i0 + 32 * j] = v[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
  }
  ss = warp_sum(ss);
  const float sc = rsqrtf(ss / static_cast<float>(cols) + eps);
  for (int i0 = lane; i0 < nvec; i0 += 32 * 8) {
    float4 v[8], g[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i0 + 32 * j < nvec) v[j] = xr[i0 + 32 * j], g[j] = wr[i0 + 32 * j];   // x: this lane's own writes above
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int i = i0 + 32 * j;
      if (i < nvec) {
        const float4 o = make_float4(g[j].x * (v[j].x * sc), g[j].y * (v[j].y * sc), g[j].z * (v[j].z * sc), g[j].w * (v[j].w * sc));
        if (out_f32) reinterpret_cast<float4*>(out_f32 + static_cast<long long>(row) * cols)[i] = o;
        if (out_bf16)
          reinterpret_cast<uint2*>(out_bf16 + static_cast<long long>(row) * cols)[i] = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      }
    }
  }
}
// Few rows (batched decode): one CTA per row, one float4 per thread, the residual + every split-K slice + the norm
// weight loaded in ONE round trip (the warp-per-row kernel above walks the slices one dependent round trip at a time:
// 6 us per launch at 5 slices, 49 launches per decode step).  Slices are added in slice order, the sum of squares is
// reduced in a fixed order: bit-reproducible.  cols <= 1024, nparts <= 8.
__global__ void __launch_bounds__(256) rmsnorm_rows_wide_kernel(float* x, const float* w, float eps, int cols, float* out_f32,
                                                                __nv_bfloat16* out_bf16, const float* parts, int nparts,
                                                                long long pstride) {
  __shared__ float red[8];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x, i = threadIdx.x, nvec = cols >> 2;
  float4* xr = reinterpret_cast<float4*>(x + static_cast<long long>(row) * cols);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f), g = v;
  if (i < nvec) {
    v = xr[i];
    g = __ldg(reinterpret_cast<const float4*>(w) + i);
    float4 t[8];
#pragma unroll
    for (int z = 0; z < 8; ++z)
      if (z < nparts) t[z] = __ldcg(reinterpret_cast<const float4*>(parts + z * pstride + static_cast<long long>(row) * cols) + i);
#pragma unroll
    for (int z = 0; z < 8; ++z)
      if (z < nparts) v.x += t[z].x, v.y += t[z].y, v.z += t[z].z, v.w += t[z].w;
    if (nparts > 0) xr[i] = v;
  }
  const float ss = warp_sum(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w);
  if ((i & 31) == 0) red[i >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) tot += red[k];
  const float sc = rsqrtf(tot / static_cast<float>(cols) + eps);
  if (i < nvec) {
    const float4 o = make_float4(g.x * (v.x * sc), g.y * (v.y * sc), g.z * (v.z * sc), g.w * (v.w * sc));
    if (out_f32) reinterpret_cast<float4*>(out_f32 + static_cast<long long>(row) * cols)[i] = o;
    if (out_bf16) reinterpret_cast<uint2*>(out_bf16 + static_cast<long long>(row) * cols)[i] = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
  }
}

int launch_rmsnorm_rows(const float* x, const float* w, float eps, int rows, int cols, float* out_f32,
                        __nv_bfloat16* out_bf16, cudaStream_t s, const float* parts, int nparts, long long pstride,
                        bool per_warp) {
  if (cols % 4) return set_error(NT_ERR_INVALID, "rmsnorm: cols must be a multiple of 4");
  if (!per_warp && rows <= 256 && cols <= 1024 && nparts <= 8)
    return launch_kernel(rmsnorm_rows_wide_kernel, dim3(rows), dim3(256), 0, s, true, const_cast<float*>(x), w, eps, cols, out_f32,
                         out_bf16, parts, nparts, pstride);
  // few rows (batched decode): one warp per CTA so the rows spread over the SMs; many rows (prefill): 8 per CTA
  const int wpc = rows >= 2048 ? 8 : (rows >= 512 ? 2 : 1);
  return launch_kernel(rmsnorm_rows_kernel, dim3((rows + wpc - 1) / wpc), dim3(32 * wpc), 0, s, true, const_cast<float*>(x), w, eps,
                       rows, cols, out_f32, out_bf16, parts, nparts, pstride);
}

// thread = one unit (pair of packed columns) of one token
__global__ void __launch_bounds__(256) rope_append_kernel(const float* qkv, int qkv_n, const int32_t* tok_seq,
                                                          const int32_t* tok_pos, int n_heads, const float* inv_freq,
                                                          float* q_out, const KVLayout kv, int layer, int nparts,
                                                          long long pstride) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const int u = blockIdx.y * 256 + threadIdx.x;
  if (u >= (qkv_n >> 1)) return;
  float2 v = *reinterpret_cast<const float2*>(qkv + static_cast<long long>(t) * qkv_n + 2 * u);
  for (int z = 1; z < nparts; ++z) {  // split-K slices of the projection, summed in slice order (qkv = slice 0)
    const float2 w = __ldcg(reinterpret_cast<const float2*>(qkv + z * pstride + static_cast<long long>(t) * qkv_n + 2 * u));
    v.x += w.x, v.y += w.y;
  }
  const int head = u >> 5, i = u & 31;
  const int b = tok_seq[t], pos = tok_pos[t];
  const int n_kv = kv.n_kv_heads;
  if (head < n_heads + n_kv) {
    const float2 r = rope_pair(v.x, v.y, pos, inv_freq[i]);
    if (head < n_heads) {
      float* q = q_out + (static_cast<long long>(t) * n_heads + head) * 64;
      q[i] = r.x, q[i + 32] = r.y;
    } else {
      const int page = kv.page_table[b * kv.max_pages_per_seq + (pos >> 6)];
      __nv_bfloat16* kp = kv.page_ptr(layer, 0, page, head - n_heads) + (pos & 63) * 64;
      kp[i] = __float2bfloat16(r.x), kp[i + 32] = __float2bfloat16(r.y);
    }
  } else {
    const int page = kv.page_table[b * kv.max_pages_per_seq + (pos >> 6)];
    __nv_bfloat16* vp = kv.page_ptr(layer, 1, page, head - n_heads - n_kv) + (pos & 63) * 64;
    *reinterpret_cast<__nv_bfloat162*>(vp + 2 * i) = __floats2bfloat162_rn(v.x, v.y);
  }
}
int launch_rope_append(const float* qkv, int T, int qkv_n, const int32_t* tok_seq, const int32_t* tok_pos, int n_heads,
                       const float* inv_freq, float* q_out, const KVLayout& kv, int layer, cudaStream_t s, int nparts,
                       long long pstride) {
  return launch_kernel(rope_append_kernel, dim3(T, ((qkv_n >> 1) + 255) / 256), dim3(256), 0, s, true, qkv, qkv_n, tok_seq,
                       tok_pos, n_heads, inv_freq, q_out, kv, layer, nparts, pstride);
}

// Causal GQA flash attention for prefill on tensor cores (mma.sync m16n8k16 bf16, fp32 accumulate).
// grid (ceil(max_len/16), n_kv_heads, B), n_rep warps: a CTA owns 16 query tokens of one sequence and one KV head;
// warp h holds the 16 x 64 query tile of head kvh*n_rep + h as A fragments (bf16, softmax scale * log2e folded in)
// and all warps share the K/V tiles.  A KV tile is one 64-token page: K and V land in shared memory through the
// SWIZZLE_128B pool descriptor (double-buffered, one mbarrier per buffer); each warp runs attn_page_step on it with
// both 8-row halves of its query tile live (log2-domain online softmax, P rounded to bf16 for the P.V MMA as in
// FlashAttention-2).  Replaces a CUDA-core kernel that took 81 % of the prefill (451 us per layer at batch 1).
constexpr int kPfQ = 16;
__global__ void __launch_bounds__(256) attn_prefill_kernel(const AttnPrefillParams p, const __grid_constant__ CUtensorMap kvmap) {
  __shared__ __align__(1024) __nv_bfloat16 sK[2][64 * 64];
  __shared__ __align__(1024) __nv_bfloat16 sV[2][64 * 64];
  __shared__ __align__(8) uint64_t full_bar[2];
  pdl_launch_dependents();
  const int qb = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    tma_prefetch_desc(&kvmap);
    mbar_init(&full_bar[0], 1);
    mbar_init(&full_bar[1], 1);
    fence_barrier_init();
  }
  pdl_wait();
  const int t0 = __ldg(p.cu_seqlens + b), len = __ldg(p.cu_seqlens + b + 1) - t0;
  const int q0 = qb * kPfQ;
  if (q0 >= len) return;  // CTA-uniform
  __syncthreads();
  const int kend = min(len, q0 + kPfQ);      // keys [0, kend) are visible to some query of this block
  const int ntiles = (kend + 63) >> 6;
  auto issue = [&](int tile) {
    const int page = __ldg(p.kv.page_table + b * p.kv.max_pages_per_seq + tile);
    const int buf = tile & 1;
    asm volatile("fence.proxy.async;" ::: "memory");
    mbar_arrive_expect_tx(&full_bar[buf], 2 * 8192);
    tma_load_2d(sK[buf], &kvmap, 0, p.kv.tmap_row(p.layer, 0, page, kvh), &full_bar[buf]);
    tma_load_2d(sV[buf], &kvmap, 0, p.kv.tmap_row(p.layer, 1, page, kvh), &full_bar[buf]);
  };
  if (tid == 0) issue(0);

  // query fragments of head `warp`: rows g and g + 8 of the block, 4 k-steps of 16 dims
  const int g = lane >> 2, t = lane & 3;
  const int head = kvh * p.n_rep + warp;
  const int r0 = min(q0 + g, len - 1), r1 = min(q0 + g + 8, len - 1);  // clamp the ragged tail (stores are masked)
  uint32_t qa[4][4];
  {
    const float* q0p = p.q + (static_cast<long long>(t0 + r0) * p.n_heads + head) * 64;
    const float* q1p = p.q + (static_cast<long long>(t0 + r1) * p.n_heads + head) * 64;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a0 = *reinterpret_cast<const float2*>(q0p + 16 * j + 2 * t);
      const float2 a1 = *reinterpret_cast<const float2*>(q1p + 16 * j + 2 * t);
      const float2 a2 = *reinterpret_cast<const float2*>(q0p + 16 * j + 8 + 2 * t);
      const float2 a3 = *reinterpret_cast<const float2*>(q1p + 16 * j + 8 + 2 * t);
      qa[j][0] = pack_bf16x2(a0.x * p.scale_log2, a0.y * p.scale_log2);
      qa[j][1] = pack_bf16x2(a1.x * p.scale_log2, a1.y * p.scale_log2);
      qa[j][2] = pack_bf16x2(a2.x * p.scale_log2, a2.y * p.scale_log2);
      qa[j][3] = pack_bf16x2(a3.x * p.scale_log2, a3.y * p.scale_log2);
    }
  }
  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // rows g / g + 8 (l: this lane's partial sum)
  const int qi0 = q0 + g, qi1 = q0 + g + 8;

  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    __syncthreads();  // every warp is done with the buffer the next copy overwrites
    if (tid == 0 && tile + 1 < ntiles) issue(tile + 1);
    mbar_wait(&full_bar[buf], (tile >> 1) & 1);
    // causal / length mask (only tiles that reach past the first query of the block need it)
    const int k0 = tile * 64;
    attn_page_step<2>(smem_u32(sK[buf]), smem_u32(sV[buf]), qa, o, m, l, k0 + 63 > q0 || k0 + 64 > len, [&](int half, int key) {
      const int kv = k0 + key;
      return kv > (half ? qi1 : qi0) || kv >= len;
    });
  }
  const float i0 = 1.0f / quad_sum(l[0]), i1 = 1.0f / quad_sum(l[1]);
  __nv_bfloat16* o0p = p.out + (static_cast<long long>(t0 + qi0) * p.n_heads + head) * 64 + 2 * t;
  __nv_bfloat16* o1p = p.out + (static_cast<long long>(t0 + qi1) * p.n_heads + head) * 64 + 2 * t;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    if (qi0 < len) *reinterpret_cast<uint32_t*>(o0p + 8 * n) = pack_bf16x2(o[n][0] * i0, o[n][1] * i0);
    if (qi1 < len) *reinterpret_cast<uint32_t*>(o1p + 8 * n) = pack_bf16x2(o[n][2] * i1, o[n][3] * i1);
  }
}
int launch_attn_prefill(const AttnPrefillParams& p, int B, int n_layers, cudaStream_t s) {
  if (p.n_rep < 1 || p.n_rep > 8) return set_error(NT_ERR_INVALID, "prefill attention: %d query heads per KV head unsupported", p.n_rep);
  CUtensorMap kvmap;
  if (int rc = kv_pool_tmap(p.kv, n_layers, &kvmap)) return rc;
  return launch_kernel(attn_prefill_kernel, dim3((p.max_len + kPfQ - 1) / kPfQ, p.kv.n_kv_heads, B), dim3(32 * p.n_rep), 0, s, true, p,
                       kvmap);
}

__global__ void gather_rows_kernel(const float* src, const int32_t* rows, int cols, float* dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x;
  const float* s = src + static_cast<long long>(rows[r]) * cols;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) dst[static_cast<long long>(r) * cols + i] = s[i];
}
int launch_gather_rows(const float* src, const int32_t* rows, int n, int cols, float* dst, cudaStream_t s) {
  return launch_kernel(gather_rows_kernel, dim3(n), dim3(256), 0, s, true, src, rows, cols, dst);
}

// =================================================================================== teacher-forced scoring
// One warp per scored row i: the final RMSNorm of h[src[i]] as rmsnorm_rows_kernel computes it (the same per-lane
// float4 sums and warp reduction), rounded to bf16 into xn[i] (the lm_head's A operand); tgt[i] = ids[src[i] + 1], the
// token the row predicts.
__global__ void __launch_bounds__(256) score_rows_kernel(const float* h, const int32_t* src, const int32_t* ids, int n, int cols,
                                                         const float* w, float eps, __nv_bfloat16* xn, int32_t* tgt) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const int r = src[i];
  if (lane == 0) tgt[i] = ids[r + 1];
  const float4* xr = reinterpret_cast<const float4*>(h + static_cast<long long>(r) * cols);
  const float4* wr = reinterpret_cast<const float4*>(w);
  const int nvec = cols >> 2;
  float ss = 0.f;
  for (int i0 = lane; i0 < nvec; i0 += 32 * 8) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (i0 + 32 * j < nvec) ? xr[i0 + 32 * j] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
  }
  ss = warp_sum(ss);
  const float sc = rsqrtf(ss / static_cast<float>(cols) + eps);
  uint2* out = reinterpret_cast<uint2*>(xn + static_cast<long long>(i) * cols);
  for (int k = lane; k < nvec; k += 32) {
    const float4 v = xr[k], g = wr[k];
    out[k] = make_uint2(pack_bf16x2(g.x * (v.x * sc), g.y * (v.y * sc)), pack_bf16x2(g.z * (v.z * sc), g.w * (v.w * sc)));
  }
}
int launch_score_rows(const float* h, const int32_t* src, const int32_t* ids, int n, int cols, const float* w, float eps,
                      __nv_bfloat16* xn, int32_t* tgt, cudaStream_t s) {
  if (cols % 4) return set_error(NT_ERR_INVALID, "score rows: cols must be a multiple of 4");
  return launch_kernel(score_rows_kernel, dim3((n + 7) / 8), dim3(256), 0, s, true, h, src, ids, n, cols, w, eps, xn, tgt);
}

// One warp per row: M = max of the tile maxima, S = sum s_t exp(m_t - M), each lane over tiles lane, lane + 32, ...
// in order and the lanes combined by a fixed butterfly, so a row's result depends on its pairs alone.
__global__ void __launch_bounds__(256) score_combine_kernel(const float2* lse, long long ld, int nt, const float* zt, int n,
                                                            float* out) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  const float2* p = lse + static_cast<long long>(r) * ld;
  float m = -INFINITY;
  for (int t = lane; t < nt; t += 32) m = fmaxf(m, p[t].x);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int t = lane; t < nt; t += 32) {
    const float2 q = p[t];
    s += q.y * expf(q.x - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[r] = zt[r] - (m + logf(s));
}
int launch_score_combine(const float2* lse, long long ld, int nt, const float* zt, int n, float* out, cudaStream_t s) {
  return launch_kernel(score_combine_kernel, dim3((n + 7) / 8), dim3(256), 0, s, true, lse, ld, nt, zt, n, out);
}

// one CTA per listed slot: compact page-table row + the slot's fresh length, counters and Philox key
__global__ void slots_setup_kernel(const int32_t* args, int B, const int32_t* page_table, int max_pages, int32_t* table,
                                   int32_t* seq_lens, int32_t* n_generated, int32_t* done, int32_t* slot_key, int32_t* ras_redraws) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, s = args[i];
  for (int j = threadIdx.x; j < max_pages; j += blockDim.x)
    table[static_cast<long long>(i) * max_pages + j] = page_table[static_cast<long long>(s) * max_pages + j];
  if (threadIdx.x == 0) {
    slot_key[s] = args[B + i];
    seq_lens[s] = args[2 * B + i];
    n_generated[s] = 0;
    done[s] = 0;
    if (ras_redraws) ras_redraws[s] = 0;
  }
}
int launch_slots_setup(const int32_t* args, int B, const int32_t* page_table, int max_pages, int32_t* table, int32_t* seq_lens,
                       int32_t* n_generated, int32_t* done, int32_t* slot_key, int32_t* ras_redraws, cudaStream_t s) {
  return launch_kernel(slots_setup_kernel, dim3(B), dim3(128), 0, s, true, args, B, page_table, max_pages, table, seq_lens, n_generated,
                       done, slot_key, ras_redraws);
}

// grid (children, n_layers * 2 * n_kv [+ 1 with hist]), 128 threads.  CTA (c, y < n_layers * 2 * n_kv) copies the first
// P % 64 rows (128 B each, 8 x 16 B) of one (layer, K|V, kv head) block of child c's last prompt page; CTA (c, last y)
// copies the history row and the recorded flag.
__global__ void __launch_bounds__(128) fork_tails_kernel(const int32_t* args, int nc, const KVLayout kv, int n_units, uint32_t* hist,
                                                         int words, int32_t* recorded) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x, y = blockIdx.y;
  const int parent = args[c], child = args[nc + c], P = args[2 * nc + c];
  if (y < n_units) {
    const int rows = P & 63;
    if (rows == 0) return;   // the prompt ends on a page boundary: every prompt page is full and shared
    const int pg = P >> 6;
    const int src = kv.page_table[static_cast<long long>(parent) * kv.max_pages_per_seq + pg];
    const int dst = kv.page_table[static_cast<long long>(child) * kv.max_pages_per_seq + pg];
    const int kvh = y % kv.n_kv_heads, is_v = (y / kv.n_kv_heads) & 1, layer = y / (2 * kv.n_kv_heads);
    const uint4* s = reinterpret_cast<const uint4*>(kv.page_ptr(layer, is_v, src, kvh));
    uint4* d = reinterpret_cast<uint4*>(kv.page_ptr(layer, is_v, dst, kvh));
    for (int i = threadIdx.x; i < rows * 8; i += blockDim.x) d[i] = s[i];
    return;
  }
  const uint32_t* hs = hist + static_cast<long long>(parent) * words;
  uint32_t* hd = hist + static_cast<long long>(child) * words;
  for (int w = threadIdx.x; w < words; w += blockDim.x) hd[w] = hs[w];
  if (threadIdx.x == 0) recorded[child] = recorded[parent];
}
int launch_fork_tails(const int32_t* args, int nc, const KVLayout& kv, int n_layers, uint32_t* hist, int words, int32_t* recorded,
                      cudaStream_t s) {
  if (nc <= 0) return NT_OK;
  const int n_units = n_layers * 2 * kv.n_kv_heads;
  return launch_kernel(fork_tails_kernel, dim3(nc, n_units + (hist ? 1 : 0)), dim3(128), 0, s, true, args, nc, kv, n_units, hist, words,
                       recorded);
}

}  // namespace nt
