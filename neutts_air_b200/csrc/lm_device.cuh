// Device-side building blocks shared by the per-op kernels (lm_kernels.cu) and the persistent wgmma decode kernel
// (lm_decode_tc.cu): sync functors, ld_cg, the mma.sync helpers, the split-KV geometry and the sampler pieces.
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

// ---- legacy tensor-core path used by both attention kernels (wgmma needs 64 rows of M; these tiles have 7-16)
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

constexpr int kTopChunk = 2048;
constexpr int kTopKeep = 64;
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

// Top-kTopKeep of n processed scores already held as keys in shared memory -> candidate slots
// [o, o + kTopKeep) of the global candidate arrays (processed score, global index = idx_base + i).
template <typename Sync>
NT_DEVINL void emit_local_topk(const SamplerParams& p, const uint32_t* keys, int n, int idx_base, long long o, uint32_t* scratch,
                               Sync sync) {
  const int tid = threadIdx.x;
  const int k = min(kTopKeep, n);
  if (k > 0) {
    uint32_t thr;
    int take_eq;
    radix_select_kth(keys, n, k, scratch, thr, take_eq, sync);
    compact_topk(keys, n, thr, take_eq, scratch, sync, [&](int slot, int i) {
      p.cand_val[o + slot] = key2f(keys[i]);
      p.cand_idx[o + slot] = idx_base + i;
    });
  }
  for (int s = k + tid; s < kTopKeep; s += kConsumerThreads) {
    p.cand_val[o + s] = -INFINITY;
    p.cand_idx[o + s] = 0x7fffffff;
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

// logits processors (MinNewTokensLength -> Temperature), then the order-preserving key
NT_DEVINL uint32_t processed_key(float logit, int idx, bool mask_eos, int eos_id, float inv_t) {
  if (mask_eos && idx == eos_id) logit = -INFINITY;
  return f2key(logit * inv_t);
}

// Sampler stage 1 for one (sequence b, chunk): processors + exact top-64 of a 2048-logit chunk read
// from global memory.  keys: [kTopChunk] uint32 shared; scratch: [kSelScratch] uint32 shared.
template <typename Sync>
NT_DEVINL void sample_stage1_chunk(const SamplerParams& p, int b, int chunk, uint32_t* keys, uint32_t* scratch, Sync sync, int slot = -1) {
  const int tid = threadIdx.x;
  const int ngen = p.n_generated_override ? __ldcg(p.n_generated_override + b) : __ldcg(p.n_generated + (slot >= 0 ? slot : b));
  const bool mask_eos = ngen < p.sp.min_new_tokens;
  const float inv_t = row_sampling(p, slot >= 0 ? slot : b).inv_t;
  const float* lg = p.logits + static_cast<long long>(b) * p.V;
  const int base = chunk * kTopChunk;
  const int n = min(kTopChunk, p.V - base);
  sync();  // keys/scratch may still be in use by the previous call of this CTA
  {
    float v[kTopChunk / kConsumerThreads];
#pragma unroll
    for (int j = 0; j < kTopChunk / kConsumerThreads; ++j) {
      const int e = j * kConsumerThreads + tid;
      v[j] = (e < n) ? __ldcg(lg + base + e) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kTopChunk / kConsumerThreads; ++j) {
      const int e = j * kConsumerThreads + tid;
      if (e < n) keys[e] = processed_key(v[j], base + e, mask_eos, p.sp.eos_id, inv_t);
    }
  }
  sync();
  emit_local_topk(p, keys, n, base, (static_cast<long long>(b) * p.nchunks + chunk) * kTopKeep, scratch, sync);
}

// Tail of the sampler for sequence b, given the k kept candidates sorted (score desc, index asc) in win[0..k):
// softmax over them (TopK processor + softmax, utils.py:2789), the slot's top-p and min-p cuts (which keep a prefix
// k' <= k of the window, renormalised), Philox draw over the prefix, state update, stop flags, and the next
// token's embedding -> residual stream row (fp32; optionally also as (value, stamp) pairs for the polled hand-off).
// Clobbers win[kTopKeep .. 2 kTopKeep) (exponentials).  b: logits row; slot >= 0: the slot whose state row b updates
// (prefill into chosen slots), else slot b.
template <typename Sync>
NT_DEVINL void sample_finish(const SamplerParams& p, int b, int k, Cand* win, int* s_tok, bool stateless, int ngen, bool is_done, Sync sync,
                             float2* h2dst = nullptr, float h2stamp = 0.f, int slot = -1) {
  const int tid = threadIdx.x;
  const int s = slot >= 0 ? slot : b;
  float* ev = reinterpret_cast<float*>(win + kTopKeep);   // [kTopKeep] exp(score - max)
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
      }
      *s_tok = tok;
      if (p.dbg_token) p.dbg_token[b] = tok;
      if (!stateless && !is_done) {
        p.out_tokens[static_cast<long long>(s) * p.max_new + ngen] = tok;
        p.n_generated[s] = ngen + 1;
        p.cur_token[s] = tok;
        const int cached = __ldcg(p.seq_lens + s) + p.advance;  // decode: this step's input token is now in the KV cache
        if (p.advance) p.seq_lens[s] = cached;
        const int total = cached + 1;  // tokens in context once `tok` is appended
        const int lim = p.sp.limits ? min(p.sp.max_new_tokens, __ldg(p.sp.limits + s)) : p.sp.max_new_tokens;
        if (tok == p.sp.eos_id || ngen + 1 >= lim || ngen + 1 >= p.max_new || total >= p.max_ctx) p.done[s] = 1;
      }
    }
  }
  sync();
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

// Sampler stage 2 for sequence b: top-k of the candidate scores (already processed), softmax, draw,
// state update, next embedding.  keys: [ncand] uint32 shared; scratch: [kSelScratch]; win: [2*kTopKeep].
struct NoMark {
  NT_DEVINL void operator()() const {}
};
template <typename Sync, typename Mark = NoMark>
NT_DEVINL void sample_stage2_seq(const SamplerParams& p, int b, int ncand, uint32_t* keys, uint32_t* scratch, Cand* win, int* s_tok,
                                 Sync sync, Mark mark = Mark(), long long cand_stride = -1, int slot = -1) {
  const int tid = threadIdx.x;
  const bool stateless = p.n_generated_override != nullptr;
  const int s = slot >= 0 ? slot : b;
  const int ngen = stateless ? __ldcg(p.n_generated_override + b) : __ldcg(p.n_generated + s);
  const bool is_done = stateless ? false : (__ldcg(p.done + s) != 0);
  // candidate rows: [b * stride, b * stride + ncand); stride = ncand unless the caller's rows have their own pitch
  const long long cstride = cand_stride >= 0 ? cand_stride : static_cast<long long>(ncand);
  const float* cv = p.cand_val + static_cast<long long>(b) * cstride;
  const int32_t* ci = p.cand_idx + static_cast<long long>(b) * cstride;
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
  mark();  // keys staged
  const int k = min(min(row_sampling(p, s).top_k, kTopKeep), ncand);
  uint32_t thr;
  int take_eq;
  radix_select_kth(keys, ncand, k, scratch, thr, take_eq, sync);
  mark();  // threshold found
  compact_topk(keys, ncand, thr, take_eq, scratch, sync, [&](int slot, int i) {
    raw[slot].v = key2f(keys[i]);
    raw[slot].i = __ldcg(ci + i);
  });
  sync();
  mark();  // winners gathered
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
  mark();  // winners sorted

  sample_finish(p, b, k, win, s_tok, stateless, ngen, is_done, sync, nullptr, 0.f, slot);
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
template <typename Sync, typename Mark>
NT_DEVINL void sample_tiles_seq(const SamplerParams& p, int b, const float* tmax, int nt, float tmax_scale, int fix_tile, float fix_val,
                                const float* logits, int V, bool mask_eos, uint8_t* uni, unsigned uni_bytes, int* sel, Sync sync, Mark pm,
                                float2* h2dst, float h2stamp, int slot = -1) {
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
  const bool stateless = false;
  const int ngen = __ldcg(p.n_generated + (slot >= 0 ? slot : b));
  const bool is_done = __ldcg(p.done + (slot >= 0 ? slot : b)) != 0;
  const float* lg = logits + static_cast<long long>(b) * V;
  // row b starts b * V floats in: with V % 4 != 0 only some rows are 16-byte aligned for the float4 loads (CTA-uniform)
  const bool vec4 = (reinterpret_cast<uintptr_t>(lg) & 15) == 0;
  auto tile_max = [&](int i) -> float {
    const float v = __ldcg(tmax + static_cast<long long>(b) * nt + i) * tmax_scale;
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
            sample_finish(p, b, k2, win, s_tok, stateless, ngen, is_done, sync, h2dst, h2stamp, slot);
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
    sample_finish(p, b, k2, win, s_tok, stateless, ngen, is_done, sync, h2dst, h2stamp, slot);
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
  constexpr long long kCandPitch = 256 * kTopKeep;   // row pitch of the candidate arrays (sampler_scratch_floats)
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
  sample_stage2_seq(p, b, ncand, keys, scratch, win, s_tok, sync, NoMark(), kCandPitch, slot);
  if (h2dst) {  // the next token's embedding becomes the residual stream of the next step's first fold
    sync();
    for (int i = tid; i < H; i += kConsumerThreads) h2dst[i] = make_float2(p.h[static_cast<long long>(b) * H + i], h2stamp);
  }
}

}  // namespace nt
