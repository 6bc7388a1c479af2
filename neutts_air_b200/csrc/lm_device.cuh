// Device-side building blocks shared by the per-op kernels (lm_kernels.cu) and the persistent wgmma decode kernel
// (lm_decode_tc.cu): sync functors, ld_cg, the mma.sync helpers, RoPE, the tensor-core attention page step and the
// merge of its partials, the split-KV geometry and the sampler pieces.
// Every block-cooperative function takes a `Sync` functor: SyncAll (= __syncthreads, per-op kernels) or
// SyncConsumers (named barrier over 256 consumer threads, for kernels whose other warps never join).
// All functions assume the cooperating threads are threadIdx.x in [0, 256).
#pragma once
#include "lm_kernels.cuh"

namespace nt {

constexpr int kConsumerWarps = 8;
constexpr int kConsumerThreads = kConsumerWarps * 32;

struct SyncAll {
  NT_DEVINL void operator()() const { __syncthreads(); }
};
struct SyncConsumers {
  NT_DEVINL void operator()() const { asm volatile("bar.sync 1, 256;" ::: "memory"); }
};

// mutable cross-CTA state is always read through L2 (L1 is not coherent across SMs)
template <typename T>
NT_DEVINL T ld_cg(const T* p) {
  return __ldcg(p);
}

// ---- legacy tensor-core path used by the attention kernels (wgmma needs 64 rows of M; these tiles have 7-16)
NT_DEVINL void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
NT_DEVINL void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
NT_DEVINL void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// element (row n, k) of a K-major SWIZZLE_128B chunk [rows][64 bf16]: 16-byte group g = k / 8 sits at g ^ (n & 7)
NT_DEVINL __nv_bfloat16* chunk_elem(uint8_t* chunk, int n, int k) {
  return reinterpret_cast<__nv_bfloat16*>(chunk + n * 128 + ((((k >> 3) ^ (n & 7)) << 4) | ((k & 7) << 1)));
}

// (sin, cos) of the RoPE angle pos * inv_freq_i (modeling_qwen2.py:116-146)
NT_DEVINL float2 rope_sincos(int pos, float inv_freq_i) {
  float s, c;
  sincosf(static_cast<float>(pos) * inv_freq_i, &s, &c);
  return make_float2(s, c);
}
// RoPE of one packed pair: projection rows (2i, 2i+1) hold dims (i, i + 32) of a q / k head (pair-interleaved at pack
// time), rotated by half-split RoPE at position pos; returns dims (i, i + 32).  The fma and the rounded product are
// spelled out so that the result does not depend on how ptxas contracts the expression at a call site.
NT_DEVINL float2 rope_pair(float x, float y, int pos, float inv_freq_i) {
  const float2 sc = rope_sincos(pos, inv_freq_i);
  return make_float2(__fmaf_rn(x, sc.y, -__fmul_rn(y, sc.x)), __fmaf_rn(y, sc.y, __fmul_rn(x, sc.x)));
}

// ---- tensor-core attention over 64-token KV pages (attn_prefill_kernel, attn_decode_mma_kernel, decode_tc_kernel).
// Fragment coordinates of m16n8k16: lane = 4 g + t; accumulator entry e of key group n is query row g + 8 (e >> 1),
// key 8 n + 2 t + (e & 1) of the page.
NT_DEVINL float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
NT_DEVINL float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// One page step of one warp: S = Q K^T from the staged K page (SWIZZLE_128B, ldmatrix), masking, base-2 online softmax
// on the accumulator fragments, P rounded to bf16, O += P V from the staged V page (ldmatrix .trans).  qa: A fragments
// of the 16-row query tile, scale * log2(e) folded in.  H: live 8-row halves of the tile (1: rows 8..15 are zero and
// their statistics are not kept; 2: both).  m / l: running maximum and this lane's partial sum of each live half.
// masked: dead(half, key) is true for every (query row half, key of the page) the query must not see.  The first key
// of every page must be visible to every live row (m stays finite).
template <int H, typename Dead>
NT_DEVINL void attn_page_step(uint32_t kbase, uint32_t vbase, const uint32_t (&qa)[4][4], float (&o)[8][4], float (&m)[H],
                              float (&l)[H], bool masked, Dead dead) {
  const int lane = threadIdx.x & 31, t = lane & 3, lrow = lane & 7, lmat = lane >> 3;
  // S = Q K^T: 8 key groups of 8 tokens; ldmatrix: lane supplies row (lane & 7) of matrix (lane >> 3)
  float sc[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
    const int row = 8 * n + lrow;  // key token within the page; row & 7 == lrow
#pragma unroll
    for (int half = 0; half < 2; ++half) {  // dims 0..31 / 32..63: 4 chunks of 8 dims each
      uint32_t kb[4];
      ldmatrix_x4(kb, kbase + row * 128 + (((4 * half + lmat) ^ lrow) << 4));
      mma_bf16_16816(sc[n], qa[2 * half], kb[0], kb[1]);
      mma_bf16_16816(sc[n], qa[2 * half + 1], kb[2], kb[3]);
    }
  }
  if (masked) {
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 2 * H; ++e)
        if (dead(e >> 1, 8 * n + 2 * t + (e & 1))) sc[n][e] = -INFINITY;
  }
#pragma unroll
  for (int h = 0; h < H; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) mx = fmaxf(mx, fmaxf(sc[n][2 * h], sc[n][2 * h + 1]));
    const float mn = fmaxf(m[h], quad_max(mx));
    const float c = exp2f(m[h] - mn);   // 0 on the first page
    m[h] = mn;
    l[h] *= c;
#pragma unroll
    for (int n = 0; n < 8; ++n) o[n][2 * h] *= c, o[n][2 * h + 1] *= c;
  }
  uint32_t pa[4][4];  // P as A fragments: k-step j covers key groups 2j, 2j+1
#pragma unroll
  for (int n = 0; n < 8; ++n) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t pk = 0u;
      if (h < H) {
        const float p0 = exp2f(sc[n][2 * h] - m[h]), p1 = exp2f(sc[n][2 * h + 1] - m[h]);
        l[h] += p0 + p1;
        pk = pack_bf16x2(p0, p1);
      }
      pa[n >> 1][(n & 1) * 2 + h] = pk;
    }
  }
  // O += P V: k-steps of 16 keys, output dim groups of 8 (two per ldmatrix)
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int row = 16 * j + 8 * (lmat & 1) + lrow;  // key token; row & 7 == lrow
#pragma unroll
    for (int nd = 0; nd < 8; nd += 2) {
      uint32_t vb[4];
      ldmatrix_x4_trans(vb, vbase + row * 128 + (((nd + (lmat >> 1)) ^ lrow) << 4));
      mma_bf16_16816(o[nd], pa[j], vb[0], vb[1]);
      mma_bf16_16816(o[nd + 1], pa[j], vb[2], vb[3]);
    }
  }
}

// Decode query tile: row g = query head g of the KV head's group, from q [n_rep][64] fp32 (shared memory), times
// scale_log2, as bf16 A fragments; rows >= n_rep and rows 8..15 are zero.
NT_DEVINL void decode_query_frags(const float* q, int n_rep, float scale_log2, uint32_t (&qa)[4][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* qp = q + min(g, n_rep - 1) * 64;
  const float sc = (g < n_rep) ? scale_log2 : 0.f;
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

// The new token's K and V rows (fp32 [64] each) -> row r of the staged K and V pages (bf16, SWIZZLE_128B), two dims per
// lane: the page copy may predate the row's store to the cache.  Whole warp, before its ldmatrix reads of the page.
NT_DEVINL void patch_staged_row(void* kstage, void* vstage, int r, const float* knew, const float* vnew) {
  const int lane = threadIdx.x & 31;
  *reinterpret_cast<uint32_t*>(chunk_elem(static_cast<uint8_t*>(kstage), r, 2 * lane)) = pack_bf16x2(knew[2 * lane], knew[2 * lane + 1]);
  *reinterpret_cast<uint32_t*>(chunk_elem(static_cast<uint8_t*>(vstage), r, 2 * lane)) = pack_bf16x2(vnew[2 * lane], vnew[2 * lane + 1]);
  __syncwarp();
}

// A decode warp's partial for the merge: rows g < n_rep store their unnormalised output to o_w [8][64] and (m, l) to
// ml_w [8][2], l summed over the quad first.
NT_DEVINL void decode_store_partial(const float (&o)[8][4], float m, float l, int n_rep, float* o_w, float* ml_w) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  l = quad_sum(l);
  if (g < n_rep) {
#pragma unroll
    for (int n = 0; n < 8; ++n) *reinterpret_cast<float2*>(o_w + g * 64 + 8 * n + 2 * t) = make_float2(o[n][0], o[n][1]);
    if (t == 0) ml_w[2 * g] = m, ml_w[2 * g + 1] = l;
  }
}

// One base-2 online-softmax partial of one (head, dim): running maximum, sum of exponentials, unnormalised output.
struct SoftmaxPart {
  float m, l, o;
};
// Merge of the partials part(0) .. part(n - 1), n <= kMax, summed in index order (warp or split 0 first).
template <int kMax, typename Part>
NT_DEVINL SoftmaxPart merge_parts(int n, Part part) {
  SoftmaxPart r{-INFINITY, 0.f, 0.f};
#pragma unroll
  for (int w = 0; w < kMax; ++w)
    if (w < n) r.m = fmaxf(r.m, part(w).m);
#pragma unroll
  for (int w = 0; w < kMax; ++w) {
    if (w < n) {
      const SoftmaxPart e = part(w);
      const float wgt = exp2f(e.m - r.m);  // 0 for a partial that saw no token (m = -inf, l = 0)
      r.l += wgt * e.l;
      r.o += wgt * e.o;
    }
  }
  return r;
}

// split geometry shared by the producer of the partials and their consumer
struct SplitGeom {
  int n_ctx, npages, pps, nsplit;
};
NT_DEVINL SplitGeom split_geom(int seq_len, int max_ctx, int max_splits) {
  SplitGeom g;
  g.n_ctx = min(seq_len + 1, max_ctx);
  g.npages = (g.n_ctx + 63) >> 6;
  g.pps = (g.npages + max_splits - 1) / max_splits;
  g.nsplit = (g.npages + g.pps - 1) / g.pps;
  return g;
}

// =================================================================================== sampler pieces
struct Cand {
  float v;
  int i;
};
NT_DEVINL bool cand_before(const Cand& a, const Cand& b) { return a.v > b.v || (a.v == b.v && a.i < b.i); }

NT_DEVINL void philox4x32_10(uint32_t (&ctr)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n1 = lo1, n2 = hi0 ^ ctr[3] ^ k1, n3 = lo0;
    ctr[0] = n0, ctr[1] = n1, ctr[2] = n2, ctr[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

constexpr int kTopKeep = 64;
constexpr int kCandPitch = 256 * kTopKeep;          // row pitch of the candidate arrays (sampler_scratch_floats)
constexpr int kSelList = 512;                       // radix select switches to a compacted list below this size
constexpr int kSelScratch = 264 + kSelList;         // uint32 words of scratch the selector needs

// order-preserving float <-> uint key (larger float <=> larger key; -inf is the smallest finite key)
NT_DEVINL uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
NT_DEVINL float key2f(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Block-wide radix select (4 passes of 8 bits, MSB first) over n keys in shared memory: finds the key
// of the k-th largest element and how many elements equal to it belong to the top-k.
//   pass 0 aggregates equal bins inside a warp with match.any (logits crowd into a few top-byte bins);
//   later passes use plain shared atomics (bins are spread) and, once at most kSelList keys still match
//   the prefix, run on a compacted list instead of rescanning all n keys.
template <typename Sync>
NT_DEVINL void radix_select_kth(const uint32_t* keys, int n, int k, uint32_t* scratch, uint32_t& thr, int& take_eq, Sync sync) {
  uint32_t* hist = scratch;        // [256]
  uint32_t* sel = scratch + 256;   // [0] bin, [1] remaining, [2] count in bin, [3] list length
  uint32_t* list = scratch + 264;  // [kSelList]
  const int tid = threadIdx.x, lane = tid & 31;
  uint32_t prefix = 0, mask = 0;
  int remaining = k;
  const uint32_t* src = keys;
  int ns = n;
#pragma unroll 1
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = tid; i < 256; i += kConsumerThreads) hist[i] = 0;
    if (tid == 0) sel[3] = 0;
    sync();
    if (pass == 0) {
      const int n_pad = (ns + 31) & ~31;
      for (int i = tid; i < n_pad; i += kConsumerThreads) {
        const uint32_t bin = (i < ns) ? (src[i] >> 24) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        if (bin != 0xffffffffu && lane == (__ffs(peers) - 1)) atomicAdd(&hist[bin], __popc(peers));
      }
    } else {
      for (int i = tid; i < ns; i += kConsumerThreads) {
        const uint32_t key = src[i];
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
    }
    sync();
    if (tid < 32) {
      uint32_t c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[8 * lane + j];
        sum += c[j];
      }
      uint32_t suf = sum;  // elements in bins >= 8*lane
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t t = __shfl_down_sync(0xffffffffu, suf, off);
        if (lane + off < 32) suf += t;
      }
      const uint32_t above = suf - sum;
      if (above < static_cast<uint32_t>(remaining) && static_cast<uint32_t>(remaining) <= suf) {
        uint32_t acc = above;
#pragma unroll
        for (int j = 7; j >= 0; --j) {
          if (acc + c[j] >= static_cast<uint32_t>(remaining)) {
            sel[0] = 8 * lane + j;
            sel[1] = remaining - acc;
            sel[2] = c[j];
            break;
          }
          acc += c[j];
        }
      }
    }
    sync();
    prefix |= sel[0] << shift;
    mask |= 0xffu << shift;
    remaining = static_cast<int>(sel[1]);
    const int in_bin = static_cast<int>(sel[2]);
    if (pass < 3 && src == keys && in_bin <= kSelList) {
      // compact the keys that still match the prefix; the remaining passes scan only those
      const int ns_pad = (ns + 31) & ~31;
      for (int i = tid; i < ns_pad; i += kConsumerThreads) {  // warp-aggregated append: one shared atomic per warp and round
        const uint32_t key = (i < ns) ? src[i] : 0u;
        const bool hit = (i < ns) && ((key & mask) == prefix);
        const uint32_t m = __ballot_sync(0xffffffffu, hit);
        if (m) {
          uint32_t base = 0;
          if (lane == 0) base = atomicAdd(&sel[3], static_cast<uint32_t>(__popc(m)));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (hit) list[base + __popc(m & ((1u << lane) - 1u))] = key;
        }
      }
      sync();
      src = list;
      ns = in_bin;
    } else {
      sync();
    }
  }
  thr = prefix;
  take_eq = remaining;
}

// Deterministic compaction of the top-k winners (keys > thr, plus the first take_eq keys == thr in
// index order) into slots [0, k).  scratch: >= 16 uint32.
template <typename Sync, typename Emit>
NT_DEVINL void compact_topk(const uint32_t* keys, int n, uint32_t thr, int take_eq, uint32_t* scratch, Sync sync, Emit emit) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (n + kConsumerThreads - 1) / kConsumerThreads;
  const int lo = min(n, tid * per), hi = min(n, lo + per);
  int ngt = 0, neq = 0;
  for (int i = lo; i < hi; ++i) {
    const uint32_t key = keys[i];
    ngt += key > thr;
    neq += key == thr;
  }
  int sgt = ngt, seq = neq;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, sgt, off), b = __shfl_up_sync(0xffffffffu, seq, off);
    if (lane >= off) sgt += a, seq += b;
  }
  uint32_t* wg = scratch;      // [8] per-warp totals (greater)
  uint32_t* we = scratch + 8;  // [8] per-warp totals (equal)
  sync();
  if (lane == 31) wg[warp] = sgt, we[warp] = seq;
  sync();
  int bg = 0, be = 0, total_gt = 0;
  for (int w = 0; w < kConsumerWarps; ++w) {
    if (w < warp) bg += wg[w], be += we[w];
    total_gt += wg[w];
  }
  int pos_gt = bg + sgt - ngt;
  int idx_eq = be + seq - neq;
  for (int i = lo; i < hi; ++i) {
    const uint32_t key = keys[i];
    if (key > thr) {
      emit(pos_gt++, i);
    } else if (key == thr) {
      if (idx_eq < take_eq) emit(total_gt + idx_eq, i);
      ++idx_eq;
    }
  }
}

// Sampling controls of the row whose state lives in `slot`: its entry of the per-slot table when that is on, else the
// launch scalars with top-p and min-p off.  Every sampler path reads temperature and top_k here, so all of them form
// the same fp32 1 / T.
struct RowSampling {
  float inv_t;
  int top_k;
  float top_p, min_p;
};
NT_DEVINL RowSampling row_sampling(const SamplerParams& p, int slot) {
  RowSampling r;
  if (p.slot_sp) {
    const nt_slot_sampling e = p.slot_sp[slot];
    r.inv_t = 1.0f / e.temperature, r.top_k = e.top_k, r.top_p = e.top_p, r.min_p = e.min_p;
  } else {
    r.inv_t = 1.0f / p.sp.temperature, r.top_k = p.sp.top_k, r.top_p = 1.f, r.min_p = 0.f;
  }
  return r;
}

// RepetitionPenaltyLogitsProcessor on one score of an id in the history: a true IEEE division (not a product with the
// reciprocal), so the result is bit-identical to torch's fp32 `score / penalty`; -inf stays -inf
NT_DEVINL float rep_penalize(float s, float penalty) { return s < 0.f ? __fmul_rn(s, penalty) : __fdiv_rn(s, penalty); }

// MinNewTokensLengthLogitsProcessor: EOS stays masked while the slot's n_generated is below this floor
NT_DEVINL int row_min_new(const SamplerParams& p, int slot) { return p.len_tab ? p.len_tab[slot].min_new_tokens : p.sp.min_new_tokens; }

// ExponentialDecayLengthPenalty: the constant c_k of the slot with n tokens generated (k = n - decay_start) while
// n > decay_start, else 0 (the table holds 0 for every k of an entry without decay)
NT_DEVINL float len_decay_c(const SamplerParams& p, int slot, int n) {
  if (!p.len_tab) return 0.f;
  const int k = n - p.len_tab[slot].decay_start;
  return k > 0 && k <= p.len_pitch ? __ldg(p.len_c + static_cast<long long>(slot) * p.len_pitch + k - 1) : 0.f;
}
// transformers' `scores + |scores| * c` on the EOS score: the fp32 product, then the fp32 sum (no fused multiply-add)
NT_DEVINL float len_decay(float s, float c) { return __fadd_rn(s, __fmul_rn(fabsf(s), c)); }

// logits processors (MinNewTokensLength -> Temperature), then the order-preserving key
NT_DEVINL uint32_t processed_key(float logit, int idx, bool mask_eos, int eos_id, float inv_t) {
  if (mask_eos && idx == eos_id) logit = -INFINITY;
  return f2key(logit * inv_t);
}

// log(sum_v exp(lg[v])) over one logits row of V scores on the 256 consumer threads, id `eos` left out while mask_eos
// (ids the vocabulary range suppresses hold -inf and add nothing).  Each thread keeps an online (max, sum) in fp32 over
// its float4 columns; the warps' pairs meet in red (8 float2 of shared memory, free until the caller's next barrier).
// Every thread returns the result.
template <typename Sync>
NT_DEVINL float row_logsumexp(const float* lg, int V, int eos, bool mask_eos, float2* red, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int skip = mask_eos ? eos : -1;
  float m = -INFINITY, s = 0.f;
  auto add = [&](float x, float y, float z, float w) {
    const float c = fmaxf(fmaxf(x, y), fmaxf(z, w));
    if (c > m) s *= __expf(m - c), m = c;
    if (m > -INFINITY) s += (__expf(x - m) + __expf(y - m)) + (__expf(z - m) + __expf(w - m));
  };
  auto combine = [](float& m0, float& s0, float m1, float s1) {
    const float mm = fmaxf(m0, m1);
    s0 = mm == -INFINITY ? 0.f : s0 * __expf(m0 - mm) + s1 * __expf(m1 - mm);
    m0 = mm;
  };
  // ids [0, head) and [head + 4 n4, V) one by one (the row need not start 16-byte aligned), the rest as float4
  const int head = min(V, static_cast<int>(((16u - (reinterpret_cast<uintptr_t>(lg) & 15u)) & 15u) >> 2));
  const int n4 = (V - head) >> 2;
  if (tid < 8) {
    const int i = tid < 4 ? (tid < head ? tid : V) : head + 4 * n4 + tid - 4;
    add((i < V && i != skip) ? __ldcg(lg + i) : -INFINITY, -INFINITY, -INFINITY, -INFINITY);
  }
  const float4* body = reinterpret_cast<const float4*>(lg + head);
  constexpr int kU = 8;   // independent 16-byte loads in flight per thread: the pass is bound by L2 latency
  for (int i = tid; i < n4; i += kU * kConsumerThreads) {
    float4 x[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int j = i + u * kConsumerThreads;
      x[u] = j < n4 ? __ldcg(body + j) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int q = skip - (head + 4 * (i + u * kConsumerThreads));
      if (q == 0) x[u].x = -INFINITY;
      if (q == 1) x[u].y = -INFINITY;
      if (q == 2) x[u].z = -INFINITY;
      if (q == 3) x[u].w = -INFINITY;
      add(x[u].x, x[u].y, x[u].z, x[u].w);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) combine(m, s, __shfl_xor_sync(0xffffffffu, m, off), __shfl_xor_sync(0xffffffffu, s, off));
  if (lane == 0) red[warp] = make_float2(m, s);
  sync();
  m = -INFINITY, s = 0.f;
#pragma unroll
  for (int w = 0; w < kConsumerWarps; ++w) combine(m, s, red[w].x, red[w].y);
  return m + logf(s);
}

// Repetition-aware redraw on the 256 consumer threads: one draw from the softmax of the whole processed row lg[0, V)
// times inv_t (id `eos` left out while mask_eos; ids the vocabulary range suppresses hold -inf and add nothing), by
// inverse CDF in ascending id order with uniform u2.  Thread t sums exp(s * inv_t - m) over its chunk of consecutive
// ids (ceil(V / 256) rounded up to a multiple of 4, read as float4 when the row is 16-byte aligned); a block scan of
// the chunk sums in thread order bounds every chunk, and warp 0 walks the one chunk that holds u2 * total, 32 ids per
// scan, 256 ids per round trip to L2.  Fixed order, no float atomics: a rerun is bit-identical.  m: the row's processed
// maximum (so every term is <= 1 and the top id's is exactly 1).  sh: sample_finish's ras_sh (24 words).  Every thread
// returns the token; thread 0 also leaves its log-probability s * inv_t - logsumexp(s * inv_t) in sh[4].
template <typename Sync>
NT_DEVINL int ras_full_row_draw(const SamplerParams& p, const float* lg, bool mask_eos, float inv_t, float m, float u2, int* sh,
                                Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int V = p.V, skip = mask_eos ? p.sp.eos_id : -1;
  const int per = ((V + kConsumerThreads - 1) / kConsumerThreads + 3) & ~3;
  const int lo = min(V, tid * per), hi = min(V, lo + per);
  auto term = [&](int i, float x) { return i == skip ? 0.f : __expf(__fmul_rn(x, inv_t) - m); };
  float part = 0.f;
  if ((reinterpret_cast<uintptr_t>(lg) & 15) == 0) {   // CTA-uniform; chunks start at multiples of 4
    for (int i0 = lo; i0 < hi; i0 += 32) {               // 8 float4 loads in flight per thread
      float4 x[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + 4 * u;
        if (i + 3 < hi) {
          x[u] = __ldcg(reinterpret_cast<const float4*>(lg + i));
        } else {
          x[u].x = i < hi ? __ldcg(lg + i) : -INFINITY;
          x[u].y = i + 1 < hi ? __ldcg(lg + i + 1) : -INFINITY;
          x[u].z = i + 2 < hi ? __ldcg(lg + i + 2) : -INFINITY;
          x[u].w = -INFINITY;   // i + 3 >= hi
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + 4 * u;
        part += term(i, x[u].x);
        part += term(i + 1, x[u].y);
        part += term(i + 2, x[u].z);
        part += term(i + 3, x[u].w);
      }
    }
  } else {
    for (int i0 = lo; i0 < hi; i0 += 8) {
      float x[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) x[u] = i0 + u < hi ? __ldcg(lg + i0 + u) : -INFINITY;
#pragma unroll
      for (int u = 0; u < 8; ++u) part += term(i0 + u, x[u]);
    }
  }
  float incl = part;   // inclusive scan over the warp's chunks
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 0.f;
  const unsigned mass = __ballot_sync(0xffffffffu, part > 0.f);
  float* wsum = reinterpret_cast<float*>(sh + 8);
  unsigned* wmass = reinterpret_cast<unsigned*>(sh + 16);
  if (lane == 31) wsum[warp] = incl;
  if (lane == 0) wmass[warp] = mass;
  sync();
  float base = 0.f, total = 0.f;   // the same sequential sum for every thread: chunk bounds meet exactly
  int last_t = -1;                 // the last thread whose chunk has mass
#pragma unroll
  for (int w = 0; w < kConsumerWarps; ++w) {
    if (w == warp) base = total;
    total += wsum[w];
    if (wmass[w]) last_t = 32 * w + 31 - __clz(static_cast<int>(wmass[w]));
  }
  const float target = u2 * total, lo_cdf = base + excl, hi_cdf = base + incl;
  // the chunk holding the target; when rounding puts the target at the total, the last chunk with mass
  if (part > 0.f && lo_cdf <= target && (target < hi_cdf || tid == last_t)) sh[5] = tid, sh[6] = __float_as_int(lo_cdf);
  sync();
  if (warp == 0) {
    const int t = sh[5], wlo = min(V, t * per), whi = min(V, wlo + per);
    float cum = __int_as_float(sh[6]);
    int tok = -1, last = -1;   // warp-uniform
    for (int i0 = wlo; i0 < whi && tok < 0; i0 += 8 * 32) {
      float x[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + 32 * u + lane;
        x[u] = i < whi ? __ldcg(lg + i) : -INFINITY;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + 32 * u + lane;
        const float e = i < whi ? term(i, x[u]) : 0.f;
        float c = e;   // inclusive scan of the 32 ids
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const float a = __shfl_up_sync(0xffffffffu, c, off);
          if (lane >= off) c += a;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, e > 0.f && cum + c > target);
        const unsigned pos = __ballot_sync(0xffffffffu, e > 0.f);
        if (tok < 0) {
          if (hit) {
            tok = i0 + 32 * u + __ffs(hit) - 1;
          } else {
            if (pos) last = i0 + 32 * u + 31 - __clz(static_cast<int>(pos));
            cum += __shfl_sync(0xffffffffu, c, 31);
          }
        }
      }
    }
    if (lane == 0) sh[3] = tok >= 0 ? tok : last;
  }
  sync();
  const int tok = sh[3];
  if (tid == 0) sh[4] = __float_as_int((__fmul_rn(__ldcg(lg + tok), inv_t) - m) - logf(total));
  return tok;
}

// Whether token tok occurs at least min_count times among slot s's generated tokens [max(0, ngen - window), ngen) (its
// repetition-aware entry; window 0 = off), read from the slot's ring 16 entries per round trip to L2 (one thread).
NT_DEVINL bool ras_window_hit(const SamplerParams& p, int s, int ngen, int tok) {
  const nt_slot_ras re = p.ras_tab[s];
  const int lo = max(0, ngen - re.window);
  const int32_t* ring = p.ras_ring + static_cast<long long>(s) * kRasRing;
  int c = 0;
  for (int j0 = ngen - 1; j0 >= lo; j0 -= 16) {
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int j = j0 - u;
      c += (j >= lo && __ldcg(ring + (j & (kRasRing - 1))) == tok) ? 1 : 0;
    }
  }
  return re.window > 0 && c >= re.min_count;
}

// model log-probability of token tok: log-softmax over the processed logits row lg (penalty, EOS mask, range; no
// temperature or warpers), lse = row_logsumexp of that row
NT_DEVINL float model_logprob(const SamplerParams& p, const float* lg, int tok, bool mask_eos, float lse) {
  const float st = (tok < 0 || tok >= p.V || (mask_eos && tok == p.sp.eos_id)) ? -INFINITY : __ldcg(lg + tok);
  return st - lse;
}

// Thread 0 of the sampler: the drawn token of sample row b into slot s, at n_generated ngen -- the capture, its
// log-probabilities (when on), and unless the row is stateless or finished, out_tokens and the state that goes with it.
// redrawn: a repetition-aware redraw (counted per slot).
NT_DEVINL void sample_commit(const SamplerParams& p, int b, int s, int ngen, int tok, bool logprobs, float sampled, float model,
                             bool write_state, bool redrawn, int* s_tok) {
  *s_tok = tok;
  if (p.dbg_token) p.dbg_token[b] = tok;
  if (logprobs) reinterpret_cast<float2*>(p.logprob_out)[static_cast<long long>(s) * p.max_new + ngen] = make_float2(sampled, model);
  if (write_state) {
    p.out_tokens[static_cast<long long>(s) * p.max_new + ngen] = tok;
    // the history bit of this token: the persistent kernel's epi_head reads it at the next step, behind the grid
    // barrier this thread arrives at after the sampler (see DESIGN.md §4, repetition penalty)
    if (p.rep_hist) atomicOr(p.rep_hist + static_cast<long long>(s) * p.rep_words + (tok >> 5), 1u << (tok & 31));
    // the repetition-aware window's entry, read by later steps behind the same barrier
    if (p.ras_ring) p.ras_ring[static_cast<long long>(s) * kRasRing + (ngen & (kRasRing - 1))] = tok;
    if (redrawn) p.ras_redraws[s] = __ldcg(p.ras_redraws + s) + 1;
    p.n_generated[s] = ngen + 1;
    p.cur_token[s] = tok;
    const int cached = __ldcg(p.seq_lens + s) + p.advance;  // decode: this step's input token is now in the KV cache
    if (p.advance) p.seq_lens[s] = cached;
    const int total = cached + 1;  // tokens in context once `tok` is appended
    const int lim = p.sp.limits ? min(p.sp.max_new_tokens, __ldg(p.sp.limits + s)) : p.sp.max_new_tokens;
    if (tok == p.sp.eos_id || ngen + 1 >= lim || ngen + 1 >= p.max_new || total >= p.max_ctx) p.done[s] = 1;
  }
}

// The repetition-aware redraw of a live, sampled row (all 256 consumer threads; sample_finish's ras_sh holds u2 and the
// row's processed maximum): the full-row draw, then thread 0 commits the new token with its log-probability in the
// full distribution.  Out of line, so that the kernels' register allocation of the common path does not carry it.  p is
// taken by reference: every kernel that samples declares its parameters __grid_constant__, so the reference points at
// the kernel's parameter space (otherwise each thread would copy the parameters to local memory at entry).
template <typename Sync>
__device__ __noinline__ void ras_redraw(const SamplerParams& p, int b, int s, int ngen, const float* lg, bool mask_eos, float lse,
                                        bool logprobs, int* s_tok, int* sh, Sync sync) {
  const int tok = ras_full_row_draw(p, lg, mask_eos, row_sampling(p, s).inv_t, __int_as_float(sh[2]), __int_as_float(sh[1]), sh, sync);
  if (threadIdx.x == 0)
    sample_commit(p, b, s, ngen, tok, logprobs, __int_as_float(sh[4]), logprobs ? model_logprob(p, lg, tok, mask_eos, lse) : 0.f,
                  true, true, s_tok);
  sync();
}

// Tail of the sampler for sequence b, given the k kept candidates sorted (score desc, index asc) in win[0..k):
// softmax over them (TopK processor + softmax, utils.py:2789), the slot's top-p and min-p cuts (which keep a prefix
// k' <= k of the window, renormalised), Philox draw over the prefix, state update, stop flags, and the next
// token's embedding -> residual stream row (fp32; optionally also as (value, stamp) pairs for the polled hand-off).
// With p.logprob_out, the written token's (sampled, model) log-probabilities go next to it (DESIGN.md §4, per-token
// log-probabilities); the model one takes one extra pass over logits row b.
// kRas = false compiles repetition-aware sampling out (the persistent kernel's instantiations for a launch with the
// table off); the ring entry is written either way.
// Clobbers win[kTopKeep .. 2 kTopKeep) (exponentials).  b: sample row; slot >= 0: the slot whose state row b updates
// (prefill into chosen slots), else slot b; src >= 0: the logits row sample row b reads (several takes of one
// prompt), else row b.
template <bool kRas = true, typename Sync>
NT_DEVINL void sample_finish(const SamplerParams& p, int b, int k, Cand* win, int* s_tok, bool stateless, int ngen, bool is_done, Sync sync,
                             float2* h2dst = nullptr, float h2stamp = 0.f, int slot = -1, int src = -1) {
  const int tid = threadIdx.x;
  const int s = slot >= 0 ? slot : b;
  float* ev = reinterpret_cast<float*>(win + kTopKeep);   // [kTopKeep] exp(score - max)
  const bool logprobs = p.logprob_out && !stateless && !is_done;   // CTA-uniform
  const bool mask_eos = ngen < row_min_new(p, s);
  const float* lg = p.logits + static_cast<long long>(src >= 0 ? src : b) * p.V;
  float lse = 0.f;
  if (logprobs) lse = row_logsumexp(lg, p.V, p.sp.eos_id, mask_eos, reinterpret_cast<float2*>(ev + kTopKeep), sync);
  // repetition-aware sampling's shared words, behind row_logsumexp's pairs: [0] redraw flag (CTA-uniform after the
  // barrier), [1] u2, [2] the row's processed maximum, [3] redrawn token, [4] its log-probability, [5, 6] the chunk
  // holding the target and its lower bound, [8, 16) warp sums, [16, 24) warp masks of chunks with mass
  int* ras_sh = reinterpret_cast<int*>(ev + kTopKeep + 2 * kConsumerWarps);
  if (tid < 32) {
    const float m = win[0].v;
    float e0 = (tid < k) ? __expf(win[tid].v - m) : 0.f;
    float e1 = (tid + 32 < k) ? __expf(win[tid + 32].v - m) : 0.f;
    float sum = warp_sum(e0 + e1);
    const RowSampling rs = row_sampling(p, s);
    if (rs.top_p < 1.f || rs.min_p > 0.f) {   // warp-uniform; top_p == 1 and min_p == 0 leave the window as it is
      // lane l holds window entries l and 32 + l.  top-p (TopPLogitsWarper): entry j stays iff the probability mass
      // before it, an exclusive prefix sum of q = e / sum in window order, is < top_p, so entry 0 always stays.
      // min-p (MinPLogitsWarper): q_j >= min_p * q_0, i.e. e_j >= min_p since e_0 = exp(0) = 1.  Both keep a prefix.
      const float q0 = e0 / sum, q1 = e1 / sum;
      float c0 = q0, c1 = q1;   // inclusive scans of each half
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const float a = __shfl_up_sync(0xffffffffu, c0, off), bb = __shfl_up_sync(0xffffffffu, c1, off);
        if (tid >= off) c0 += a, c1 += bb;
      }
      const float tot0 = __shfl_sync(0xffffffffu, c0, 31);
      const float u0 = __shfl_up_sync(0xffffffffu, c0, 1), u1 = __shfl_up_sync(0xffffffffu, c1, 1);
      const float x0 = tid == 0 ? 0.f : u0, x1 = tid == 0 ? tot0 : tot0 + u1;   // exclusive prefixes
      const bool keep0 = tid < k && (rs.top_p >= 1.f || x0 < rs.top_p) && e0 >= rs.min_p;
      const bool keep1 = tid + 32 < k && (rs.top_p >= 1.f || x1 < rs.top_p) && e1 >= rs.min_p;
      const uint32_t f0 = __ballot_sync(0xffffffffu, !keep0), f1 = __ballot_sync(0xffffffffu, !keep1);
      k = max(1, f0 ? __ffs(f0) - 1 : (f1 ? 31 + __ffs(f1) : 64));   // first entry cut
      e0 = tid < k ? e0 : 0.f;
      e1 = tid + 32 < k ? e1 : 0.f;
      sum = warp_sum(e0 + e1);
    }
    if (p.dbg_topk_val) {
      p.dbg_topk_val[b * kTopKeep + tid] = (tid < k) ? e0 / sum : 0.f;
      p.dbg_topk_val[b * kTopKeep + tid + 32] = (tid + 32 < k) ? e1 / sum : 0.f;
      p.dbg_topk_idx[b * kTopKeep + tid] = (tid < k) ? win[tid].i : -1;
      p.dbg_topk_idx[b * kTopKeep + tid + 32] = (tid + 32 < k) ? win[tid + 32].i : -1;
    }
    ev[tid] = e0, ev[tid + 32] = e1;
    __syncwarp();
    if (tid == 0) {
      int tok;
      uint32_t word1 = 0;   // Philox word 1 of the draw's block: the repetition-aware redraw's uniform
      if (p.sp.forced && !stateless) {
        tok = p.sp.forced[static_cast<long long>(s) * p.max_new + ngen];
      } else if (p.sp.greedy) {
        tok = win[0].i;
      } else {
        // stream key: the slot's own key once a refill set one (-1 otherwise), so a refilled slot does not replay
        // its previous occupant's draws
        const int key = p.slot_key ? __ldg(p.slot_key + s) : -1;
        uint32_t ctr[4] = {static_cast<uint32_t>(stateless ? p.step_override : ngen), static_cast<uint32_t>(key >= 0 ? key : s + p.slot_base),
                           0u, 0u};
        philox4x32_10(ctr, static_cast<uint32_t>(p.sp.seed), static_cast<uint32_t>(p.sp.seed >> 32));
        const float u = (ctr[0] >> 8) * (1.0f / 16777216.0f);  // [0,1)
        const float target = u * sum;
        float cum = 0.f;
        tok = win[k - 1].i;
        for (int j = 0; j < k; ++j) {   // sequential inverse CDF over the sorted candidates (multinomial semantics)
          cum += ev[j];
          if (cum > target) {
            tok = win[j].i;
            break;
          }
        }
        word1 = ctr[1];
      }
      // Repetition-aware sampling: the drawn token's count among the slot's last `window` generated tokens (ring
      // entries written by earlier steps' samplers, behind the grid barrier or launch boundary that followed them).
      // Thread 0 counts on its own, so that nothing stands between its draw and its state update.
      bool redraw = false;
      if (kRas && p.ras_tab) {
        if (!stateless && !is_done && !p.sp.forced && !p.sp.greedy) redraw = ras_window_hit(p, s, ngen, tok);
        ras_sh[0] = redraw ? 1 : 0;
      }
      if (redraw) {
        ras_sh[1] = __float_as_int((word1 >> 8) * (1.0f / 16777216.0f));
        ras_sh[2] = __float_as_int(win[0].v);   // the processed maximum of the row: the full pass's shift
      } else {
        float model = 0.f, sampled = 0.f;
        if (logprobs) {
          model = model_logprob(p, lg, tok, mask_eos, lse);
          // sampled: the token's log-probability in the kept window the draw used (greedy: transformers applies no
          // warpers, so it is the model value); -inf for a forced id outside the window
          sampled = model;
          if (p.sp.forced || !p.sp.greedy) {
            int j = 0;
            while (j < k && win[j].i != tok) ++j;
            sampled = j < k ? (win[j].v - win[0].v) - logf(sum) : -INFINITY;
          }
        }
        sample_commit(p, b, s, ngen, tok, logprobs, sampled, model, !stateless && !is_done, false, s_tok);
      }
    }
  }
  sync();
  if (kRas && p.ras_tab && ras_sh[0]) ras_redraw(p, b, s, ngen, lg, mask_eos, lse, logprobs, s_tok, ras_sh, sync);   // CTA-uniform
  if (!stateless && !is_done && p.h) {
    const int tok = *s_tok;
    const __nv_bfloat16* e = p.embed + static_cast<long long>(tok) * p.hidden;
    for (int i = tid; i < p.hidden; i += kConsumerThreads) {
      const float f = __bfloat162float(e[i]);
      p.h[static_cast<long long>(b) * p.hidden + i] = f;
      if (h2dst) h2dst[i] = make_float2(f, h2stamp);
    }
  } else if (h2dst) {   // finished sequence: the row keeps its value, but the next fold still waits for the stamp
    for (int i = tid; i < p.hidden; i += kConsumerThreads) h2dst[i] = make_float2(p.h[static_cast<long long>(b) * p.hidden + i], h2stamp);
  }
}

// General path of sample_tiles_seq, second half, for sequence b: top-k of the ncand candidate scores (already
// processed) in row b of the candidate arrays, softmax, draw, state update, next embedding.  keys: [ncand] uint32
// shared; scratch: [kSelScratch]; win: [2*kTopKeep].  Stateless (see sample_tiles_seq) when p.n_generated_override is
// set: a run-time test here, where a caller's compile-time flag shifts ptxas's spills in the persistent kernel.
template <bool kRas = true, typename Sync>
NT_DEVINL void sample_stage2_seq(const SamplerParams& p, int b, int ncand, uint32_t* keys, uint32_t* scratch, Cand* win, int* s_tok,
                                 Sync sync, int slot = -1, int src = -1) {
  const int tid = threadIdx.x;
  const bool stateless = p.n_generated_override != nullptr;
  const int s = slot >= 0 ? slot : b;
  const int ngen = stateless ? __ldcg(p.n_generated_override + b) : __ldcg(p.n_generated + s);
  const bool is_done = stateless ? false : (__ldcg(p.done + s) != 0);
  const float* cv = p.cand_val + static_cast<long long>(b) * kCandPitch;
  const int32_t* ci = p.cand_idx + static_cast<long long>(b) * kCandPitch;
  Cand* raw = win + kTopKeep;  // unsorted winners
  sync();
  for (int e0 = 0; e0 < ncand; e0 += 8 * kConsumerThreads) {  // 8 independent loads in flight per thread
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = e0 + j * kConsumerThreads + tid;
      v[j] = (e < ncand) ? __ldcg(cv + e) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = e0 + j * kConsumerThreads + tid;
      if (e < ncand) keys[e] = f2key(v[j]);
    }
  }
  if (tid < kTopKeep) raw[tid].v = -INFINITY, raw[tid].i = 0x7fffffff;
  sync();
  const int k = min(min(row_sampling(p, s).top_k, kTopKeep), ncand);
  uint32_t thr;
  int take_eq;
  radix_select_kth(keys, ncand, k, scratch, thr, take_eq, sync);
  compact_topk(keys, ncand, thr, take_eq, scratch, sync, [&](int slot, int i) {
    raw[slot].v = key2f(keys[i]);
    raw[slot].i = __ldcg(ci + i);
  });
  sync();
  if (tid < kTopKeep) {  // rank sort of the 64 winners: (score desc, index asc), ties of padding by slot
    const Cand me = raw[tid];
    int rank = 0;
    for (int j = 0; j < kTopKeep; ++j) {
      const Cand o = raw[j];
      rank += (cand_before(o, me) || (o.v == me.v && o.i == me.i && j < tid)) ? 1 : 0;
    }
    win[rank] = me;
  }
  sync();
  sample_finish<kRas>(p, b, k, win, s_tok, stateless, ngen, is_done, sync, nullptr, 0.f, slot, src);
}

// Sampler of the tile-max schemes, for sequence b, on 256 threads (0..255) of one CTA.  The lm_head epilogue left the
// logits in HBM plus the maximum of every 128-row tile; only tiles whose maximum reaches the top_k-th best can hold a
// top-k logit.  Direct path: every thread takes the largest of its <= 8 tile maxima; the top_k-th largest of those
// 256 values, L, is a valid candidate threshold (at least top_k distinct tiles reach it, so the top_k logits all do);
// tiles reaching L are scanned, logits >= L are ranked in shared memory by (score desc, index asc).  Two round trips
// to L2, six barriers, no radix passes.  Fallbacks for small vocabularies / mass ties: radix select over the tile
// maxima with shared-memory candidates, then the general two-pass path through the global candidate arrays.
//   tmax: [*, nt] tile maxima (times tmax_scale = processed maxima); fix_tile >= 0: that tile's processed maximum is
//   fix_val instead (the tile holding a masked EOS, when the maxima were taken on raw logits).
//   uni / uni_bytes: >= 16 KB of shared scratch (1024-byte aligned); sel: >= 4 ints of shared memory.
//   stateless (nt_op_topk_sample): n_generated_override[b] is the row's count, the row is live and no state is written.
//   src >= 0: the logits and tile-maxima row sample row b reads (see sample_finish), else row b.
template <bool kRas = true, typename Sync, typename Mark>
NT_DEVINL void sample_tiles_seq(const SamplerParams& p, int b, const float* tmax, int nt, float tmax_scale, int fix_tile, float fix_val,
                                const float* logits, int V, bool mask_eos, uint8_t* uni, unsigned uni_bytes, int* sel, Sync sync, Mark pm,
                                float2* h2dst, float h2stamp, bool stateless, int slot = -1, int src = -1) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.hidden;
  uint32_t* scratch = reinterpret_cast<uint32_t*>(uni);
  int* tiles = reinterpret_cast<int*>(scratch + kSelScratch);   // [64] chosen tiles
  int* counts = tiles + 64;                                      // [64] candidates per chosen tile, then offsets
  Cand* win = reinterpret_cast<Cand*>(counts + 64);              // [2 * kTopKeep]
  int* s_tok = reinterpret_cast<int*>(win + 2 * kTopKeep);
  uint32_t* keys = reinterpret_cast<uint32_t*>(s_tok + 4);       // the rest of the scratch region
  const int key_cap = static_cast<int>((uni_bytes - (kSelScratch + 128 + 4) * 4 - 2 * kTopKeep * sizeof(Cand)) / 4);
  const RowSampling rs = row_sampling(p, slot >= 0 ? slot : b);
  const float inv_t = rs.inv_t;
  const int top_k = rs.top_k;
  const int eos = p.sp.eos_id;
  const int ngen = stateless ? __ldcg(p.n_generated_override + b) : __ldcg(p.n_generated + (slot >= 0 ? slot : b));
  const bool is_done = stateless ? false : __ldcg(p.done + (slot >= 0 ? slot : b)) != 0;
  const int src_row = src >= 0 ? src : b;
  const float* lg = logits + static_cast<long long>(src_row) * V;
  // the row starts src_row * V floats in: with V % 4 != 0 only some rows are 16-byte aligned for the float4 loads (CTA-uniform)
  const bool vec4 = (reinterpret_cast<uintptr_t>(lg) & 15) == 0;
  auto tile_max = [&](int i) -> float {
    const float v = __ldcg(tmax + static_cast<long long>(src_row) * nt + i) * tmax_scale;
    return i == fix_tile ? fix_val : v;
  };
  pm(120);
  // ---- direct path (large vocabularies).  Every thread takes the largest of its <= 8 tile maxima; the top_k-th
  //      largest of those 256 values, L, is a valid candidate threshold: at least top_k distinct tiles reach it,
  //      so the top_k logits all do (it sits a hair below the exact top_k-th tile maximum, since two of the best
  //      tiles rarely share a thread).  Tiles whose maximum reaches L are scanned, logits >= L are ranked in
  //      shared memory by (score desc, index asc).  Two round trips to L2, six CTA barriers, no radix passes.
  {
    constexpr int kPer = 8, kTileCap = 256, kCandCap = 512;
    const int ktop = min(top_k, kTopKeep);
    float* gmax = reinterpret_cast<float*>(keys);                         // [256]
    int* tl = reinterpret_cast<int*>(keys + kConsumerThreads);            // [kTileCap]
    Cand* fc = reinterpret_cast<Cand*>(keys + kConsumerThreads + kTileCap);  // [kCandCap]
    int* cnt = sel;                                                   // [0] tiles, [1] candidates, [2] L
    if (nt <= kPer * kConsumerThreads && key_cap >= kConsumerThreads + kTileCap + 2 * kCandCap) {
      float tm[kPer];
      float best = -INFINITY;
#pragma unroll
      for (int u = 0; u < kPer; ++u) {
        const int i = tid + u * kConsumerThreads;
        tm[u] = (i < nt) ? tile_max(i) : -INFINITY;
      }
#pragma unroll
      for (int u = 0; u < kPer; ++u) best = fmaxf(best, tm[u]);
      pm(126);
      gmax[tid] = best;
      if (tid < 3) cnt[tid] = (tid == 2) ? __float_as_int(-INFINITY) : 0;
      sync();
      pm(127);
      int rank = 0;   // (value desc, thread asc) is a total order: the ranks are a permutation of 0..255
      for (int j4 = 0; j4 < kConsumerThreads; j4 += 4) {
        const float4 g = *reinterpret_cast<const float4*>(gmax + j4);
        rank += (g.x > best || (g.x == best && j4 < tid)) ? 1 : 0;
        rank += (g.y > best || (g.y == best && j4 + 1 < tid)) ? 1 : 0;
        rank += (g.z > best || (g.z == best && j4 + 2 < tid)) ? 1 : 0;
        rank += (g.w > best || (g.w == best && j4 + 3 < tid)) ? 1 : 0;
      }
      pm(128);
      if (rank == ktop - 1) cnt[2] = __float_as_int(best);
      sync();
      const float L = __int_as_float(cnt[2]);
      pm(121);
      if (L > -INFINITY) {   // CTA-uniform
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
          const bool hit = tm[u] >= L;   // padding slots hold -inf
          const uint32_t m = __ballot_sync(0xffffffffu, hit);
          if (m) {
            int base = 0;
            if (lane == 0) base = atomicAdd(&cnt[0], __popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            const int o = base + __popc(m & ((1u << lane) - 1u));
            if (hit && o < kTileCap) tl[o] = tid + u * kConsumerThreads;
          }
        }
        sync();
        const int ntl = cnt[0];
        pm(122);
        if (ntl <= kTileCap) {   // CTA-uniform
          for (int j0 = warp; j0 < ntl; j0 += 4 * kConsumerWarps) {   // 4 tiles per warp in flight
            float4 x[4];
            int tile[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int j = j0 + u * kConsumerWarps;
              tile[u] = (j < ntl) ? tl[j] : -1;
              x[u] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
              if (tile[u] >= 0) {
                const int r0 = tile[u] * 128 + lane * 4;
                if (vec4 && r0 + 3 < V) {
                  x[u] = __ldcg(reinterpret_cast<const float4*>(lg + r0));
                } else {
                  if (r0 < V) x[u].x = __ldcg(lg + r0);
                  if (r0 + 1 < V) x[u].y = __ldcg(lg + r0 + 1);
                  if (r0 + 2 < V) x[u].z = __ldcg(lg + r0 + 2);
                  if (r0 + 3 < V) x[u].w = __ldcg(lg + r0 + 3);
                }
              }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              if (tile[u] < 0) continue;   // warp-uniform
              const int r0 = tile[u] * 128 + lane * 4;
              const float xv[4] = {x[u].x, x[u].y, x[u].z, x[u].w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float val = (mask_eos && r0 + q == eos) ? -INFINITY : xv[q] * inv_t;   // rows >= V stayed -inf
                const bool hit = val >= L;
                const uint32_t m = __ballot_sync(0xffffffffu, hit);
                if (m) {
                  int base = 0;
                  if (lane == 0) base = atomicAdd(&cnt[1], __popc(m));
                  base = __shfl_sync(0xffffffffu, base, 0);
                  const int o = base + __popc(m & ((1u << lane) - 1u));
                  if (hit && o < kCandCap) fc[o].v = val, fc[o].i = r0 + q;
                }
              }
            }
          }
          sync();
          const int nc = cnt[1];
          pm(123);
          if (nc <= kCandCap) {   // CTA-uniform
            const int k2 = min(ktop, nc);
            for (int i = tid; i < nc; i += kConsumerThreads) {
              const Cand me = fc[i];
              int r = 0;
              for (int j = 0; j < nc; ++j) r += cand_before(fc[j], me) ? 1 : 0;
              if (r < k2) win[r] = me;
            }
            sync();
            pm(124);
            sample_finish<kRas>(p, b, k2, win, s_tok, stateless, ngen, is_done, sync, h2dst, h2stamp, slot, src);
            pm(125);
            return;
          }
        }
      }
      sync();   // leave the direct path together (its scratch aliases the general path's keys)
    }
  }
  for (int i = tid; i < nt; i += kConsumerThreads) keys[i] = f2key(tile_max(i));
  if (tid < 64) tiles[tid] = -1, counts[tid] = 0;
  sync();
  const int k = min(min(top_k, kTopKeep), nt);
  uint32_t thr;
  int take_eq;
  radix_select_kth(keys, nt, k, scratch, thr, take_eq, sync);
  // fewer tiles than top_k: the tile maxima bound nothing, every logit of every tile is a candidate
  const uint32_t cthr = nt < top_k ? 1u : thr;
  // the k tiles: maxima above the threshold, then the first take_eq tiles (index order) that equal it
  compact_topk(keys, nt, thr, take_eq, scratch, sync, [&](int slot, int i) { tiles[slot] = i; });
  sync();
  auto tile_keys = [&](int tile, uint32_t (&kk)[4]) {   // this lane's 4 logits of the tile -> processed keys
    const int r0 = tile * 128 + lane * 4;
    float4 x = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (vec4 && r0 + 3 < V) {
      x = __ldcg(reinterpret_cast<const float4*>(lg + r0));
    } else {
      if (r0 < V) x.x = __ldcg(lg + r0);
      if (r0 + 1 < V) x.y = __ldcg(lg + r0 + 1);
      if (r0 + 2 < V) x.z = __ldcg(lg + r0 + 2);
      if (r0 + 3 < V) x.w = __ldcg(lg + r0 + 3);
    }
    kk[0] = (r0 < V) ? processed_key(x.x, r0, mask_eos, eos, inv_t) : 0u;
    kk[1] = (r0 + 1 < V) ? processed_key(x.y, r0 + 1, mask_eos, eos, inv_t) : 0u;
    kk[2] = (r0 + 2 < V) ? processed_key(x.z, r0 + 2, mask_eos, eos, inv_t) : 0u;
    kk[3] = (r0 + 3 < V) ? processed_key(x.w, r0 + 3, mask_eos, eos, inv_t) : 0u;
  };
  // ---- fast path: the candidates (key >= threshold) of the chosen tiles go straight into shared memory; all loads
  //      of a warp's tiles are in flight together (one round trip to L2), the exact top-k is a rank sort.
  constexpr int kFastCap = 512;
  Cand* fc = reinterpret_cast<Cand*>(keys + ((nt + 3) & ~3));
  int* fcnt = &sel[1];
  const bool fast_fits = key_cap >= ((nt + 3) & ~3) + 2 * kFastCap;
  if (tid == 0) *fcnt = 0;
  sync();
  if (fast_fits) {
    constexpr int kPerWarp = (kTopKeep + kConsumerWarps - 1) / kConsumerWarps;
    uint32_t kk[kPerWarp][4];
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
      const int j = warp + u * kConsumerWarps;
      if (j < k) tile_keys(tiles[j], kk[u]);
    }
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
      const int j = warp + u * kConsumerWarps;
      if (j < k) {
        const int tile = tiles[j];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const bool hit = kk[u][q] >= cthr && kk[u][q] != 0u;
          const uint32_t m = __ballot_sync(0xffffffffu, hit);
          if (m) {
            int base = 0;
            if (lane == 0) base = atomicAdd(fcnt, __popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            const int o = base + __popc(m & ((1u << lane) - 1u));
            if (hit && o < kFastCap) fc[o].v = key2f(kk[u][q]), fc[o].i = tile * 128 + lane * 4 + q;
          }
        }
      }
    }
  }
  sync();
  const int nc = fast_fits ? *fcnt : kFastCap + 1;
  if (nc <= kFastCap) {
    const int k2 = min(min(top_k, kTopKeep), nc);
    for (int i = tid; i < nc; i += kConsumerThreads) {   // rank among the candidates: (score desc, index asc) is a total order
      const Cand me = fc[i];
      int rank = 0;
      for (int j = 0; j < nc; ++j) rank += cand_before(fc[j], me) ? 1 : 0;
      if (rank < k2) win[rank] = me;
    }
    sync();
    sample_finish<kRas>(p, b, k2, win, s_tok, stateless, ngen, is_done, sync, h2dst, h2stamp, slot, src);
    return;
  }
  // ---- general path (thousands of candidates: tiny vocabularies, or exact ties at the threshold)
  // Stage 2 keeps the first of the candidates tied at its threshold by position, so the candidate arrays list them in
  // id order (smaller id wins, as on every other path): chosen tiles by index, each tile's candidates in id order.
  {
    int me = -1, r = 0;
    if (tid < k) {
      me = tiles[tid];
      for (int j = 0; j < k; ++j) r += tiles[j] < me ? 1 : 0;
    }
    sync();
    if (tid < k) tiles[r] = me;
    sync();
  }
  // pass 1: candidates (key >= threshold) per chosen tile
  for (int j = warp; j < k; j += kConsumerWarps) {
    uint32_t kk[4];
    tile_keys(tiles[j], kk);
    int c = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) c += __popc(__ballot_sync(0xffffffffu, kk[q] >= cthr && kk[q] != 0u));
    if (lane == 0) counts[j] = c;
  }
  sync();
  if (warp == 0) {  // exclusive prefix over <= 64 tiles
    const int c0 = counts[lane], c1 = counts[lane + 32];
    int s0 = c0, s1 = c1;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, s0, off), bb = __shfl_up_sync(0xffffffffu, s1, off);
      if (lane >= off) s0 += a, s1 += bb;
    }
    const int tot0 = __shfl_sync(0xffffffffu, s0, 31);
    const int tot = tot0 + __shfl_sync(0xffffffffu, s1, 31);
    counts[lane] = s0 - c0;
    counts[lane + 32] = tot0 + s1 - c1;
    if (lane == 0) sel[0] = tot;
  }
  sync();
  const int ncand = min(min(sel[0], key_cap), 256 * kTopKeep);   // beyond: thousands of exact ties at the threshold
  // pass 2: write the candidates at their deterministic offsets
  float* cv = p.cand_val + static_cast<long long>(b) * kCandPitch;
  int32_t* ci = p.cand_idx + static_cast<long long>(b) * kCandPitch;
  for (int j = warp; j < k; j += kConsumerWarps) {
    uint32_t kk[4];
    const int tile = tiles[j];
    tile_keys(tile, kk);
    bool hit[4];
    int c = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      hit[q] = kk[q] >= cthr && kk[q] != 0u;
      c += hit[q] ? 1 : 0;
    }
    int incl = c;   // lane prefix: lane l's candidates follow those of lanes < l (ids tile * 128 + 4 l + q)
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    int o = counts[j] + incl - c;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (hit[q]) {
        if (o < ncand) {
          cv[o] = key2f(kk[q]);
          ci[o] = tile * 128 + lane * 4 + q;
        }
        ++o;
      }
    }
  }
  sync();
  sample_stage2_seq<kRas>(p, b, ncand, keys, scratch, win, s_tok, sync, slot, src);
  if (h2dst) {  // the next token's embedding becomes the residual stream of the next step's first fold
    sync();
    for (int i = tid; i < H; i += kConsumerThreads) h2dst[i] = make_float2(p.h[static_cast<long long>(b) * H + i], h2stamp);
  }
}

}  // namespace nt
