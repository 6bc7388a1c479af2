// Persistent decode megakernel (batch <= 4): ALL layers, the lm_head, the sampler and the whole
// multi-step decode loop run in one cooperative launch of one CTA per SM.
//
//   * one producer warp per CTA streams this CTA's slice of every weight matrix, in phase order,
//     HBM -> shared memory with cp.async.bulk into a deep mbarrier ring (~170 KB in flight per SM);
//     weights are immutable, so the stream runs ahead across phase boundaries and hides the grid
//     barriers;
//   * eight consumer warps execute the phases (fused RMSNorm + QKV GEMV + bias + RoPE + KV-page
//     append | split-KV GQA attention | o_proj + residual | RMSNorm + gate/up + SiLU*up | down +
//     residual | lm_head | radix-select top-k + multinomial draw + next embedding) and meet at a
//     grid-wide barrier (one L2 atomic + acquire spin) between dependent phases;
//   * no host involvement between tokens: stop flags, KV lengths and sampled ids live on the device.
//
// Replaces the per-token loop of transformers generation/utils.py:2743-2805 (one host sync per
// step there) and the ~25 ATen launches per layer listed in SURVEY.md §2.1.
#include "lm_device.cuh"
#include "lm_mega.cuh"

#include <cstdlib>

namespace nt {

NT_DEVINL unsigned ld_relaxed_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
NT_DEVINL unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

NT_DEVINL long long global_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// optional in-kernel timeline (thread 0 of the first and the last CTA, one chosen step)
struct Prof {
  long long* buf;
  int n;
  NT_DEVINL void mark() {
    if (buf && n < kProfMarks) buf[n++] = global_ns();
  }
};

// Grid-wide barrier over the consumer warps of all CTAs: one relaxed L2 atomic per CTA on a
// monotonically growing counter (release fence before it), then thread 0 spins with acquire loads
// until the counter reaches this barrier's target.  A flag-array variant (one word per CTA, coalesced
// polling, no atomics) was slower: one poller per SM hammering the flag lines delays the flag stores themselves.
NT_DEVINL void grid_sync(unsigned* gbar, unsigned& target, unsigned nblocks, Prof& prof) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (threadIdx.x == 0) {
    prof.mark();  // all consumer warps of this CTA are done
    target += nblocks;
    __threadfence();
    atomicAdd(gbar, 1u);
    prof.mark();  // arrival published
    uint32_t spins = 0;
    while (ld_acquire_gpu(gbar) < target) {
      if (++spins > (1u << 23)) {
        printf("neutts_b200: grid barrier timed out (block %d, target %u, seen %u)\n", blockIdx.x, target, *gbar);
        __trap();
      }
    }
    prof.mark();  // barrier released
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

struct PhaseSlice {
  int u_begin, my_units, ups, stages, unit_bytes;
};
NT_DEVINL PhaseSlice phase_slice(const MegaPhase& ph) {
  PhaseSlice s;
  const int nunits = ph.rows >> 1;
  s.u_begin = static_cast<int>((static_cast<long long>(nunits) * blockIdx.x) / gridDim.x);
  const int u_end = static_cast<int>((static_cast<long long>(nunits) * (blockIdx.x + 1)) / gridDim.x);
  s.my_units = u_end - s.u_begin;
  s.ups = (ph.K >= 2048) ? 1 : kConsumerWarps;
  s.stages = (s.my_units + s.ups - 1) / s.ups;
  s.unit_bytes = 4 * ph.K;
  return s;
}

NT_DEVINL void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
NT_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
NT_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

template <int NB>
__global__ void __launch_bounds__((kConsumerWarps + 1) * 32, 1) decode_mega_kernel(const MegaParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  uint8_t* ring = smem + P.ring_off;
  float4* xs = reinterpret_cast<float4*>(smem + P.x_off);
  uint8_t* uni = smem + P.union_off;  // AttnSmem | head-phase logits + selector scratch ; x+uni together: final selection
  float* red = reinterpret_cast<float*>(smem + P.misc_off);
  float* s_part = red + 2 * kConsumerWarps * 2 * 4;
  int* pos_cache = reinterpret_cast<int*>(s_part + kConsumerWarps * 4);
  int* page_cache = pos_cache + 4;
  float* norm_buf = reinterpret_cast<float*>(page_cache + 4);
  float* bias_buf = norm_buf + P.hidden;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + P.bar_off);
  uint64_t* empty_bar = full_bar + 8;
  AttnSync* async_ = reinterpret_cast<AttnSync*>(empty_bar + 8);
  volatile int* s_go = reinterpret_cast<volatile int*>(async_ + 1);  // producer gate: steps released so far, -1 = stop

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int NS = P.nstages;
  const int L = P.n_layers;
  const int n_phases = 4 * L + 1;
  AttnSmem* asmem = reinterpret_cast<AttnSmem*>(uni);

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps);
    }
    mbar_init(&async_->bar, 1);
    async_->uses = 0;
    fence_barrier_init();
    *s_go = 1;
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ============================================================ producer warp
    if (lane == 0) {
      uint32_t g = 0;  // global stage counter (ring position)
      for (int step = 0; step < P.n_steps; ++step) {
        uint32_t spins = 0;
        int go;
        while ((go = *s_go) >= 0 && go <= step) {  // released one step at a time (early exit safety)
          __nanosleep(64);
          if (++spins > (1u << 25)) {
            printf("neutts_b200: producer gate timed out (block %d)\n", blockIdx.x);
            __trap();
          }
        }
        if (go < 0) break;
        for (int ph = 0; ph < n_phases; ++ph) {
          const int pidx = (ph == n_phases - 1) ? (4 * P.total_layers) : ph;  // lm_head is the last table entry
          if (P.l2_prefetch && (ph & 3) == 0 && ph < 4 * L) {
            // entering layer l: pull this CTA's slices of layer l+1 (or the head of the lm_head slice) into L2
            const int l = ph >> 2;
            if (l + 1 < L) {
              for (int q = 0; q < 4; ++q) {
                const MegaPhase np = P.phases[4 * (l + 1) + q];
                const PhaseSlice ns = phase_slice(np);
                if (ns.my_units > 0)
                  bulk_prefetch_l2(reinterpret_cast<const uint8_t*>(np.W) + static_cast<long long>(ns.u_begin) * ns.unit_bytes,
                                   static_cast<uint32_t>(ns.my_units) * ns.unit_bytes);
              }
            }
            if (l + 2 >= L) {
              const MegaPhase hp = P.phases[4 * P.total_layers];
              const PhaseSlice hs = phase_slice(hp);
              const long long total = static_cast<long long>(hs.my_units) * hs.unit_bytes;
              const long long chunk = P.l2_head_bytes / 2;
              const long long off = (l + 2 == L) ? 0 : chunk;
              if (off < total)
                bulk_prefetch_l2(reinterpret_cast<const uint8_t*>(hp.W) + static_cast<long long>(hs.u_begin) * hs.unit_bytes + off,
                                 static_cast<uint32_t>(min(chunk, total - off)) & ~15u);
            }
          }
          const MegaPhase mp = P.phases[pidx];
          const PhaseSlice sl = phase_slice(mp);
          const uint8_t* wbase = reinterpret_cast<const uint8_t*>(mp.W) + static_cast<long long>(sl.u_begin) * sl.unit_bytes;
          for (int it = 0; it < sl.stages; ++it, ++g) {
            const int slot = g % NS;
            if (g >= static_cast<uint32_t>(NS)) mbar_wait(&empty_bar[slot], ((g / NS) - 1) & 1);
            const int u0 = it * sl.ups;
            const uint32_t bytes = static_cast<uint32_t>(min(sl.ups, sl.my_units - u0)) * sl.unit_bytes;
            mbar_arrive_expect_tx(&full_bar[slot], bytes);
            bulk_g2s(ring + static_cast<size_t>(slot) * P.stage_bytes, wbase + static_cast<long long>(u0) * sl.unit_bytes, bytes,
                     &full_bar[slot]);
          }
        }
      }
    }
    return;
  }

  // ============================================================== consumer warps
  uint32_t g = 0;
  unsigned target = 0;
  const unsigned G = gridDim.x;
  Prof prof{nullptr, 0};
  const SyncConsumers csync;
  const int H = P.hidden, I = P.inter, HD = P.n_heads * 64;
  const int n_rep = P.n_heads / P.kv.n_kv_heads;
  const int split_cap = P.split_cap;

  // this CTA's slice of every layer's QKV bias (immutable) -> shared memory, once
  const PhaseSlice qkv_sl = phase_slice(P.phases[0]);
  const int bias_rows = 2 * qkv_sl.my_units;
  const bool bias_cached = bias_rows <= P.bias_cap;
  if (bias_cached)
    for (int i = tid; i < L * bias_rows; i += kConsumerThreads) {
      const int l = i / bias_rows, r = i - l * bias_rows;
      bias_buf[l * P.bias_cap + r] = __ldg(P.bqkv[l] + 2 * qkv_sl.u_begin + r);
    }

  auto prefetch_norm = [&](const float* w) {  // asynchronous global -> shared copy of one RMSNorm weight vector
    if (tid < (H >> 2)) cp_async16(norm_buf + 4 * tid, w + 4 * tid);
    cp_async_commit();
  };

  // ring position of the next stage to consume: slot = g % NS, parity = (g / NS) & 1, kept incrementally (no
  // integer division in the stage loop)
  int slot = 0;
  uint32_t slot_par = 0;
  auto run_stages = [&](const GemvParams& gp, const PhaseSlice& sl, int it0 = 0, int it1 = -1) {
    if (it1 < 0) it1 = sl.stages;
    if (tid == 0 && it0 == 0) prof.mark();  // input vector staged
    XRegs xr = {};
    // the slice of the input this warp multiplies in every stage of the phase: the whole vector when a warp owns
    // whole units, its eighth of K when the 8 warps share one unit
    const int nch_p = gp.K >> 3;
    const int xc_lo = sl.ups == 1 ? (nch_p * warp) / kConsumerWarps : 0;
    const int xc_hi = sl.ups == 1 ? (nch_p * (warp + 1)) / kConsumerWarps : nch_p;
    const bool use_xr = (NB == 1) && (xc_hi - xc_lo) <= 128;
    if (use_xr) load_xregs(xs, nch_p, xc_lo, xc_hi, lane, xr);
    for (int it = it0; it < it1; ++it, ++g) {
      mbar_wait(&full_bar[slot], slot_par);
      if (tid == 0 && (it == 0 || it == sl.stages - 1)) prof.mark();  // first / last stage of the phase has landed
      const int first = it * sl.ups;
      const int cur = slot;
      gemv_consume_stage<NB>(gp, ring + static_cast<size_t>(cur) * P.stage_bytes, xs, red, sl.ups == 1 ? kConsumerWarps : 1, first,
                             min(sl.ups, sl.my_units - first), sl.u_begin, it & 1, [&]() {
                               if (lane == 0) mbar_arrive(&empty_bar[cur]);
                             }, xr, use_xr);
      if (++slot == NS) slot = 0, slot_par ^= 1;
    }
  };

  AttnDecParams ap;
  memset(&ap, 0, sizeof(ap));
  ap.q = P.q, ap.kv = P.kv, ap.n_heads = P.n_heads, ap.n_rep = n_rep, ap.scale_log2 = P.scale_log2;
  ap.part_o = P.part_o, ap.part_ml = P.part_ml, ap.counters = P.counters, ap.out = P.attn, ap.out_bf16 = nullptr;
  ap.max_splits = P.max_splits, ap.layer = 0;
  // the attention item of this CTA (at most one): (sequence, kv head, split)
  const int per_b = P.kv.n_kv_heads * split_cap;
  const int my_b = blockIdx.x / per_b, my_kvh = (blockIdx.x % per_b) / split_cap, my_split = blockIdx.x % split_cap;

  for (int step = 0; step < P.n_steps; ++step) {
    if (P.prof && tid == 0 && step == P.prof_step && (blockIdx.x == 0 || blockIdx.x == G - 1)) {
      prof.buf = P.prof + (blockIdx.x == 0 ? 0 : kProfMarks);
      prof.n = 0;
      prof.mark();
    } else {
      prof.buf = nullptr;
    }
    // per-step snapshot of the sequence lengths and of the page that receives the new token
    if (tid < NB) {
      const int pos = __ldcg(P.kv.seq_lens + tid);
      pos_cache[tid] = pos;
      page_cache[tid] = (pos < P.kv.max_ctx) ? __ldcg(P.kv.page_table + tid * P.kv.max_pages_per_seq + (pos >> 6)) : 0;
    }
    prefetch_norm(P.ln1[0]);
    csync();
    SplitGeom geo{0, 0, 1, 0};
    const bool has_item = my_b < NB;
    if (has_item) geo = split_geom(pos_cache[my_b], P.kv.max_ctx, split_cap);
    const bool item_live = has_item && my_split < geo.nsplit;
    const bool can_prefetch_kv = item_live && (my_split * geo.pps < geo.npages - 1);  // first page is not the one being appended to

    for (int l = 0; l < L; ++l) {
      GemvParams gp;
      // ---- QKV: fused RMSNorm + bias + RoPE + KV-page append
      gp = GemvParams{};
      gp.rows = P.qkv_n, gp.K = H, gp.eps = P.eps, gp.bias = P.bqkv[l];
      gp.epi = GEMV_QKV_ROPE, gp.q_out = P.q, gp.kv = P.kv, gp.layer = l, gp.n_heads = P.n_heads, gp.inv_freq = P.inv_freq;
      gp.pos_cache = pos_cache, gp.page_cache = page_cache;
      if (bias_cached) gp.bias_smem = bias_buf + l * P.bias_cap, gp.row0 = 2 * qkv_sl.u_begin;
      cp_async_wait_all();
      load_x_planes<NB>(P.h, H, H, norm_buf, P.eps, xs, s_part, csync);
      run_stages(gp, qkv_sl);
      ap.layer = l;
      if (can_prefetch_kv && tid == 0) attn_issue_page(ap, my_b, my_kvh, my_split * geo.pps, asmem, async_);
      grid_sync(P.gbar, target, G, prof);
      // ---- split-KV attention: partial (m, l, o) per split, merged by the consumers of the output
      prefetch_norm(P.ln2[l]);  // lands long before the barrier's release fence
      if (item_live) attn_split_item(ap, my_b, my_kvh, my_split, geo.pps, geo.npages, geo.n_ctx, asmem, async_, can_prefetch_kv, csync);
      grid_sync(P.gbar, target, G, prof);
      // ---- o_proj + residual (input = merged attention output)
      gp = GemvParams{};
      gp.rows = H, gp.K = HD, gp.epi = GEMV_STORE, gp.out = P.h, gp.ldo = H, gp.residual = P.h, gp.ldr = H;
      load_attn_merged<NB>(ap, pos_cache, split_cap, xs, reinterpret_cast<float*>(uni), csync);
      run_stages(gp, phase_slice(P.phases[4 * l + 1]));
      grid_sync(P.gbar, target, G, prof);
      // ---- RMSNorm + gate/up + SiLU*up
      gp = GemvParams{};
      gp.rows = 2 * I, gp.K = H, gp.eps = P.eps, gp.epi = GEMV_SWIGLU, gp.out = P.act, gp.ldo = I;
      cp_async_wait_all();
      load_x_planes<NB>(P.h, H, H, norm_buf, P.eps, xs, s_part, csync);
      prefetch_norm(l + 1 < L ? P.ln1[l + 1] : P.final_norm);  // norm_buf is free again: every thread passed the staging barrier
      run_stages(gp, phase_slice(P.phases[4 * l + 2]));
      grid_sync(P.gbar, target, G, prof);
      // ---- down + residual
      gp = GemvParams{};
      gp.rows = H, gp.K = I, gp.epi = GEMV_STORE, gp.out = P.h, gp.ldo = H, gp.residual = P.h, gp.ldr = H;
      load_x_planes<NB>(P.act, I, I, nullptr, 0.f, xs, s_part, csync);
      run_stages(gp, phase_slice(P.phases[4 * l + 3]));
      grid_sync(P.gbar, target, G, prof);
    }
    // ---- lm_head (fused final RMSNorm); the CTA keeps its own logits in shared memory and selects a local
    //      top-64 per sequence right away (no second pass over the logits, no extra barrier).  With a small
    //      grid (concurrent instances) the CTA's rows are processed in segments of head_ld rows.
    {
      const PhaseSlice hs = phase_slice(P.phases[4 * P.total_layers]);
      float* lsm = reinterpret_cast<float*>(uni);
      GemvParams gp{};
      gp.rows = P.vocab, gp.K = H, gp.eps = P.eps, gp.epi = GEMV_STORE, gp.out = P.logits, gp.ldo = P.vocab;
      gp.smem_out = lsm, gp.smem_ld = P.head_ld;
      cp_async_wait_all();
      load_x_planes<NB>(P.h, H, H, norm_buf, P.eps, xs, s_part, csync);
      uint32_t* scratch = reinterpret_cast<uint32_t*>(lsm + NB * P.head_ld);
      const float inv_t = 1.0f / P.samp.sp.temperature;
      const int seg_stages = P.head_ld / (2 * hs.ups);  // stages per segment (ups units = 2*ups rows per stage)
      for (int seg = 0; seg < P.head_segs; ++seg) {
        const int it0 = seg * seg_stages, it1 = min(hs.stages, it0 + seg_stages);
        const int first_row = 2 * (hs.u_begin + it0 * hs.ups);
        const int n_local = max(0, min(2 * hs.my_units - 2 * it0 * hs.ups, 2 * (it1 - it0) * hs.ups));
        gp.row0 = first_row;
        if (it0 < it1) run_stages(gp, hs, it0, it1);
        csync();
#pragma unroll 1
        for (int b = 0; b < NB; ++b) {
          const bool mask_eos = __ldcg(P.samp.n_generated + b) < P.samp.sp.min_new_tokens;
          uint32_t* keys = reinterpret_cast<uint32_t*>(lsm + b * P.head_ld);
          for (int e = tid; e < n_local; e += kConsumerThreads)
            keys[e] = processed_key(lsm[b * P.head_ld + e], first_row + e, mask_eos, P.samp.sp.eos_id, inv_t);
          csync();
          emit_local_topk(P.samp, keys, n_local, first_row,
                          ((static_cast<long long>(b) * G + blockIdx.x) * P.head_segs + seg) * kTopKeep, scratch, csync);
        }
        csync();
      }
    }
    grid_sync(P.gbar, target, G, prof);
    if (P.logits_out) {  // tests: keep every step's logits
      const long long n = static_cast<long long>(NB) * P.vocab;
      float* dst = P.logits_out + static_cast<long long>(step) * P.logits_step_stride;
      for (long long i = static_cast<long long>(blockIdx.x) * kConsumerThreads + tid; i < n; i += static_cast<long long>(G) * kConsumerThreads)
        dst[i] = __ldcg(P.logits + i);
    }
    // ---- final selection: CTA b finishes sequence b (top-k over G*64 candidates, softmax, draw, state, next embedding)
    if (static_cast<int>(blockIdx.x) < NB) {
      const int ncand = static_cast<int>(G) * P.head_segs * kTopKeep;
      uint32_t* keys = reinterpret_cast<uint32_t*>(xs);  // x planes + union region are contiguous and idle here
      uint32_t* scratch = keys + ncand;
      Cand* win = reinterpret_cast<Cand*>(scratch + kSelScratch);
      int* s_tok = reinterpret_cast<int*>(win + 2 * kTopKeep);
      sample_stage2_seq(P.samp, blockIdx.x, ncand, keys, scratch, win, s_tok, csync, [&]() {
        if (tid == 0) prof.mark();
      });
    }
    grid_sync(P.gbar, target, G, prof);
    // ---- stop when every sequence is finished (same decision in every CTA: flags were published before the barrier)
    bool all_done = true;
    for (int b = 0; b < NB; ++b) all_done = all_done && (__ldcg(P.samp.done + b) != 0);
    if (all_done || step + 1 == P.n_steps) break;
    if (tid == 0) *s_go = step + 2;  // release the producer into the next step
  }
  cp_async_wait_all();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (tid == 0) *s_go = -1;
}

int launch_decode_mega(MegaParams& P, int nb, int num_sms, cudaStream_t stream) {
  if (nb < 1 || nb > 4) return set_error(NT_ERR_INVALID, "megakernel: batch %d not in 1..4", nb);
  if (num_sms > 256) num_sms = 256;
  // ---- shared-memory plan
  const int HD = P.n_heads * 64;
  const int k_small = P.hidden, k_big = P.inter > HD ? P.inter : HD;
  auto unit_stage = [](int K) { return (K >= 2048 ? 1 : kConsumerWarps) * 4 * K; };
  int stage = unit_stage(P.hidden);
  if (unit_stage(P.inter) > stage) stage = unit_stage(P.inter);
  if (unit_stage(HD) > stage) stage = unit_stage(HD);
  stage = (stage + 127) & ~127;
  const size_t x_bytes = (size_t(nb) * (k_big > k_small ? k_big : k_small) * 4 + 127) & ~size_t(127);
  // union region: attention staging | head-phase logits (nb rows) + selector scratch
  const int head_rows = 2 * ((P.vocab / 2 + num_sms - 1) / num_sms);  // rows of the lm_head per CTA (max)
  P.head_ld = head_rows < 1536 ? ((head_rows + 15) & ~15) : 1536;         // rows kept in shared memory per segment
  P.head_segs = (head_rows + P.head_ld - 1) / P.head_ld;
  if (num_sms * P.head_segs > 256) return set_error(NT_ERR_INVALID, "megakernel: vocabulary too large for the candidate arrays");
  size_t uni = size_t(nb) * P.head_ld * 4 + kSelScratch * 4 + 64;
  if (sizeof(AttnSmem) > uni) uni = sizeof(AttnSmem);
  uni = (uni + 127) & ~size_t(127);
  // the final selection needs G*64 keys + scratch + winners inside x + union
  const size_t final_need = size_t(num_sms) * P.head_segs * kTopKeep * 4 + kSelScratch * 4 + 2 * kTopKeep * sizeof(Cand) + 64;
  if (x_bytes + uni < final_need) uni = ((final_need - x_bytes) + 127) & ~size_t(127);
  const int qkv_units = P.qkv_n / 2;
  P.bias_cap = 2 * ((qkv_units + num_sms - 1) / num_sms) + 2;
  if (P.bias_cap > 64) P.bias_cap = 0;  // huge slices: read the bias from global memory instead
  const size_t misc = ((2 * kConsumerWarps * 2 * 4 + kConsumerWarps * 4) * sizeof(float) + 8 * sizeof(int) + size_t(P.hidden) * 4 +
                       size_t(P.total_layers) * P.bias_cap * 4 + 127) & ~size_t(127);
  const size_t bars = (16 * sizeof(uint64_t) + sizeof(AttnSync) + 16 + 127) & ~size_t(127);
  const size_t fixed = x_bytes + uni + misc + bars + 128;
  const size_t budget = 227 * 1024;
  if (fixed + 2 * size_t(stage) > budget) return set_error(NT_ERR_INVALID, "megakernel: model does not fit the shared-memory plan");
  int ns = int((budget - fixed) / stage);
  if (ns > 8) ns = 8;
  P.nstages = ns;
  P.stage_bytes = stage;
  P.split_cap = 16 / nb > 0 ? 16 / nb : 1;
  if (P.split_cap > P.max_splits) P.split_cap = P.max_splits;
  if (nb * P.kv.n_kv_heads * P.split_cap > num_sms) return set_error(NT_ERR_INVALID, "megakernel: too few SMs for the attention items");
  P.l2_prefetch = getenv("NT_NO_L2_PREFETCH") ? 0 : 1;
  P.l2_head_bytes = 256 * 1024;
  size_t off = 0;
  P.ring_off = off, off += size_t(ns) * stage;
  P.x_off = off, off += x_bytes;
  P.union_off = off, off += uni;
  P.misc_off = off, off += misc;
  P.bar_off = off, off += bars;
  const size_t smem = off + 128;
  P.samp.nchunks = num_sms;  // candidate arrays are indexed [sequence][CTA][64] in this path

  void (*kern)(const MegaParams) = nullptr;
  switch (nb) {
    case 1: kern = decode_mega_kernel<1>; break;
    case 2: kern = decode_mega_kernel<2>; break;
    case 3: kern = decode_mega_kernel<3>; break;
    default: kern = decode_mega_kernel<4>; break;
  }
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem)) return rc;   // per (kernel, device)
  int per_sm = 0;
  NT_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, (kConsumerWarps + 1) * 32, smem));
  if (per_sm < 1) return set_error(NT_ERR_CUDA, "megakernel: a CTA does not fit on an SM (%zu B shared memory)", smem);
  NT_CUDA_CHECK(cudaMemsetAsync(P.gbar, 0, sizeof(unsigned) * 64, stream));  // one counter per instance, 256 B apart
  void* args[] = {&P};
  cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kern), dim3(num_sms), dim3((kConsumerWarps + 1) * 32), args, smem, stream);
  if (e != cudaSuccess) return set_error(NT_ERR_CUDA, "megakernel launch failed: %s", cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return NT_OK;
}

}  // namespace nt
