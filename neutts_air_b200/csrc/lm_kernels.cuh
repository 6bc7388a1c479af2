// Kernel parameter blocks + launch prototypes for the speech-LM path (SURVEY.md §8a rows A1-A12).
#pragma once
#include "common.cuh"
#include "internal.h"

namespace nt {

// Static description of the KV page pool (see nt_lm_state.kv_pages in the public header).
struct KVLayout {
  __nv_bfloat16* pages;
  const int32_t* page_table;
  const int32_t* seq_lens;
  int n_kv_heads, num_pages, max_pages_per_seq, max_ctx;
  long long layer_stride;  // elements between layers  = 2 * kv_stride
  long long kv_stride;     // elements between K and V = num_pages * n_kv_heads * 64 * 64
  NT_DEVINL __nv_bfloat16* page_ptr(int layer, int is_v, int page, int kvh) const {
    return pages + layer * layer_stride + is_v * kv_stride + (static_cast<long long>(page) * n_kv_heads + kvh) * 4096;
  }
  // first row of the same page in the pool map of kv_pool_tmap (rows of 64 bf16; fits in int, kv_pool_tmap checks).
  // The page-independent part stands apart: in this shape ptxas spills no more in decode_tc_kernel than with the row
  // of the layer computed ahead of the page lookup.
  NT_DEVINL int tmap_row(int layer, int is_v, int page, int kvh) const {
    return (layer * 2 * num_pages * n_kv_heads + kvh) * 64 + (is_v * num_pages + page) * (n_kv_heads * 64);
  }
};

enum GemvEpi { GEMV_STORE = 0, GEMV_SWIGLU = 1, GEMV_QKV_ROPE = 2 };

struct GemvParams {
  const __nv_bfloat16* W;  // [rows, K], rows even ("units" are adjacent row pairs)
  int rows, K;
  const float* x;          // [nb, ldx] fp32 activations
  long long ldx;
  const float* norm_w;     // fused RMSNorm weight or nullptr
  float eps;
  const float* bias;       // [rows] or nullptr
  int epi;
  // GEMV_STORE / GEMV_SWIGLU
  float* out;              // STORE: [nb, ldo] indexed by row; SWIGLU: indexed by unit
  long long ldo;
  const float* residual;   // [nb, ldr] or nullptr (may alias out)
  long long ldr;
  // GEMV_QKV_ROPE
  float* q_out;            // [nb, n_heads*64]
  KVLayout kv;
  int layer, n_heads;
  const float* inv_freq;   // [32]
};

constexpr int kGemvMaxBatch = 4;  // gemv_kernel has one instance per batch size 1..4
int launch_gemv(const GemvParams& p, int nb, int num_sms, cudaStream_t stream);

struct AttnDecParams {
  const float* q;   // [B, n_heads*64]
  KVLayout kv;
  int layer, n_heads, n_rep;
  float* out;        // [B, n_heads*64]
  __nv_bfloat16* out_bf16;  // optional copy for the tensor-core o_proj
  // Placed after the outputs: with scale_log2 right behind n_rep, ptxas gives both attention kernels
  // 5 / 12 more registers (sm_90a, CUDA 12.9).
  float scale_log2;  // head_dim^-0.5 * log2(e)
  // Fused RoPE + KV append, required by the tensor-core variant (batch > 4), which ignores `q`: the kernel reads the
  // projection output itself ([B, qkv_n] fp32, bias already added, `qkv_parts` split-K slices `qkv_pstride` floats
  // apart, summed in slice order), rotates q / k at position seq_lens[b] and appends the new K/V row to the cache.
  const float* qkv;
  int qkv_n, qkv_parts;
  long long qkv_pstride;
  const float* inv_freq;
};
int launch_attn_decode(const AttnDecParams& p, int B, int n_layers, cudaStream_t stream);  // n_layers: extent of the KV pool

struct SamplerParams {
  const float* logits;  // [B, V]
  int V;
  nt_sampling sp;
  // state
  int32_t* seq_lens;
  int32_t* cur_token;
  int32_t* out_tokens;
  int32_t* n_generated;
  int32_t* done;
  int max_new, max_ctx;
  int advance;  // 1 in a decode step (seq_lens += 1 for live slots), 0 after prefill
  // candidates scratch: [B][kCandPitch] (val, idx), the general path of sample_tiles_seq
  float* cand_val;
  int32_t* cand_idx;
  // next-step embedding
  const __nv_bfloat16* embed;
  float* h;  // [B, hidden]
  int hidden;
  // optional debug outputs (unit tests)
  float* dbg_topk_val;     // [B, 64]
  int32_t* dbg_topk_idx;   // [B, 64]
  int32_t* dbg_token;      // [B]
  const int32_t* n_generated_override;  // nt_op_topk_sample: read-only counters, no state update
  int32_t step_override;
  int32_t slot_base;  // global slot index of local sequence 0 (keys the Philox counter)
  // Prefill into chosen slots: logits row i updates the state of slot row_slot[i] (nullptr: row i is slot i).  Read
  // by the stand-alone sampler kernels only; the persistent decode kernel samples row b into slot b.
  const int32_t* row_slot;
  // Several takes of one prompt (nt_lm_prefill_fork): sample row i reads logits row and tile-maxima row row_src[i]
  // (nullptr: row i).  The capture, the residual row and the candidate scratch stay indexed by sample row i.  Read by
  // the stand-alone sampler kernels only.
  const int32_t* row_src;
  const int32_t* slot_key;  // optional [max_batch] Philox stream key per slot; -1: slot + slot_base
  // optional [max_batch] temperature / top_k / top_p / min_p per slot (nt_lm_set_slot_sampling), read through
  // row_sampling() with the row's slot; nullptr: sp.temperature and sp.top_k for every row, no top-p / min-p cut
  const nt_slot_sampling* slot_sp;
  // repetition penalty (nt_lm_set_repetition_penalty): [max_batch][rep_words] history bitmap of every slot, nullptr =
  // off.  sample_finish sets the bit of every token it writes to out_tokens.
  uint32_t* rep_hist;
  int rep_words;
  // length control (nt_lm_set_length_control): per-slot entries, nullptr = off (sp.min_new_tokens for every slot), and
  // [max_batch][len_pitch] decay constants, entry k - 1 = c_k (all zero for an entry without decay)
  const nt_slot_length* len_tab;
  const float* len_c;
  int len_pitch;
  // per-token log-probabilities (nt_lm_set_logprobs): [max_batch][max_new][2] (sampled, model), nullptr = off.
  // sample_finish writes the pair of every token it writes to out_tokens.
  float* logprob_out;
  // repetition-aware sampling (nt_lm_set_repetition_aware_sampling): per-slot (window, min_count) table, nullptr = off.
  // ras_ring [max_batch][kRasRing]: sample_finish writes entry n % kRasRing of every token n it writes to out_tokens,
  // table on or off; ras_redraws [max_batch]: redraws of the slot since the prefill that filled it.
  const nt_slot_ras* ras_tab;
  int32_t* ras_ring;
  int32_t* ras_redraws;
};
constexpr int kRasRing = 64;   // generated tokens each slot keeps for the repetition window (the largest window)
int launch_sampler_check(const SamplerParams& p);
// tmax: [B][nt] RAW maxima of the 128-column tiles of p.logits (GEMM epilogue, gemm_dispatch(..., tile_max), or
// launch_tile_max).  p.n_generated_override set: stateless (nt_op_topk_sample).  skip (optional, [max_batch]): rows
// whose slot s has skip[s] >= 0 are not sampled (the unconditional slots of guided pairs; launch_guidance_follow
// writes their state).
int launch_sampler_tiles(const SamplerParams& p, int B, const float* tmax, int nt, cudaStream_t stream,
                         const int32_t* skip = nullptr);
// tmax [B][ceil(V / 128)] = the raw maximum of every 128-column tile of logits rows [0, B)
int launch_tile_max(const float* logits, int B, int V, float* tmax, cudaStream_t s);
size_t sampler_scratch_floats(int B);  // per-array element count for cand_val / cand_idx
// Vocabulary range (nt_lm_set_vocab_range).  launch_fill_neg_inf: p[0, n) = -inf (the logits rows and tile maxima of a
// launch, before its lm_head writes the tiles it computes).  launch_vocab_eos_tile: after an lm_head that computed the
// whole 128-row tile holding `eos` although only `eos` is allowed there, rows [0, B) of that tile read -inf except eos,
// and tmax (optional, [B][nt] raw maxima) holds the eos logit as the tile's maximum.
int launch_fill_neg_inf(float* p, long long n, cudaStream_t s);
int launch_vocab_eos_tile(float* logits, int B, int V, int eos, float* tmax, int nt, cudaStream_t s);
// Repetition penalty.  launch_rep_history: one CTA per prefill row i builds the history row of slot row_slot[i] (row i
// when row_slot is nullptr): cleared, then the ids ids[cu[i] .. cu[i + 1]) when the slot's entry includes the prompt;
// the slot becomes recorded.  launch_rep_penalty: the CTAs of logits row i of `logits` [B][V] rewrite the logit of
// every id in slot row_slot[i]'s history (recorded slots with a penalty != 1 only) and recompute the raw maximum of
// every 128-row tile it touched in tmax [B][nt] (optional).
int launch_rep_history(uint32_t* hist, int words, const nt_slot_penalty* tab, int32_t* recorded, const int32_t* row_slot,
                       const int32_t* ids, const int32_t* cu, int B, int V, cudaStream_t s);
int launch_rep_penalty(float* logits, int B, int V, const uint32_t* hist, int words, const nt_slot_penalty* tab,
                       const int32_t* recorded, const int32_t* row_slot, float* tmax, int nt, cudaStream_t s);
// Length control, decode steps only: logits row b [B][V] holds slot b; where the slot's decay is active at its
// n_generated, the EOS logit becomes s + |s| c_k and the raw maximum of the EOS tile in tmax [B][nt] (optional) is
// recomputed.  p supplies V, eos_id, n_generated and the length-control pointers.
int launch_len_decay(const SamplerParams& p, int B, float* logits, float* tmax, int nt, cudaStream_t s);
// Classifier-free guidance (nt_lm_set_guidance).  launch_guidance_combine: tab holds one entry per logits row r < B of
// `logits` [B][V]; where tab[r].partner = u >= 0 (row r is a guided c row, row u its unconditional partner), row r
// becomes g * (ls_c - ls_u) + ls_u in fp32, in that order (g = tab[r].scale, ls = x - log-sum-exp of the row), and -inf
// where either logit is -inf; tmax (optional, [B][nt]) receives the raw maximum of every tile of the new row.  Two
// launches: kGuideSplit CTAs per row fold (max, sum exp) partials into part [B][2][kGuideSplit], then kGuideSplit CTAs
// per c row fold those in index order and rewrite their share of the tiles.  No float atomics: reruns are
// bit-identical.
constexpr int kGuideSplit = 32;
int launch_guidance_combine(float* logits, int B, int V, const nt_slot_guidance* tab, float2* part, float* tmax, int nt,
                            cudaStream_t s);
// launch_guidance_follow, after the sampler: for each sample row i < B whose slot c (p.row_slot[i], or i) has a partner
// slot u in the slot table tab, u takes c's new token unless it is finished already: out_tokens, cur_token and
// n_generated mirror c's, seq_lens[u] += p.advance, done[u] = done[c], and (p.h set) residual row u = embed[token].  If
// u's context would reach max_ctx, both slots finish, the rule the sampler applies to c's own context.
int launch_guidance_follow(const SamplerParams& p, int B, const nt_slot_guidance* tab, cudaStream_t s);

int launch_embed_rows(const __nv_bfloat16* embed, const int32_t* ids, int T, int hidden, float* h, cudaStream_t s);
// parts != nullptr: x is updated in place first (x += sum of nparts split-K slices, slice order) -- see SplitK.
// per_warp: always the one-warp-per-row kernel, whose per-row arithmetic does not depend on `rows`.
int launch_rmsnorm_rows(const float* x, const float* w, float eps, int rows, int cols, float* out_f32,
                        __nv_bfloat16* out_bf16, cudaStream_t s, const float* parts = nullptr, int nparts = 0,
                        long long pstride = 0, bool per_warp = false);
// Teacher-forced scoring (nt_lm_score).  launch_score_rows: for each of n scored rows, xn[i] = bf16(final RMSNorm of
// h[src[i]]) and tgt[i] = ids[src[i] + 1].  launch_score_combine: out[r] = zt[r] - log-sum-exp of row r's nt tile pairs
// (lse, row pitch ld; see gemm_logsoftmax), folded in a fixed order.
int launch_score_rows(const float* h, const int32_t* src, const int32_t* ids, int n, int cols, const float* w, float eps,
                      __nv_bfloat16* xn, int32_t* tgt, cudaStream_t s);
int launch_score_combine(const float2* lse, long long ld, int nt, const float* zt, int n, float* out, cudaStream_t s);
// qkv: [T, qkv_n] fp32 in packed (pair-interleaved) column order -> q natural order + K/V pages
int launch_rope_append(const float* qkv, int T, int qkv_n, const int32_t* tok_seq, const int32_t* tok_pos, int n_heads,
                       const float* inv_freq, float* q_out, const KVLayout& kv, int layer, cudaStream_t s, int nparts = 1,
                       long long pstride = 0);  // nparts > 1: qkv points at split-K slices [nparts][T][qkv_n] to be summed
struct AttnPrefillParams {
  const float* q;  // [T, n_heads*64]
  KVLayout kv;
  int layer, n_heads, n_rep;
  float scale_log2;
  const int32_t* cu_seqlens;  // device [B+1]
  __nv_bfloat16* out;         // [T, n_heads*64]
  int max_len;
};
int launch_attn_prefill(const AttnPrefillParams& p, int B, int n_layers, cudaStream_t s);
// one TMA descriptor (box 64 rows x 128 B, SWIZZLE_128B) over the whole paged KV pool viewed as rows of 64 bf16
int kv_pool_tmap(const KVLayout& kv, int n_layers, ::CUtensorMap_st* out);
int launch_gather_rows(const float* src, const int32_t* rows, int n, int cols, float* dst, cudaStream_t s);
// Prefill into chosen slots.  args: device [3][B] = slots, Philox stream keys, prompt lengths.  Gathers the listed
// slots' page-table rows into table [B][max_pages] and resets those slots' seq_lens / n_generated / done / slot_key, and
// their repetition-aware redraw counters when ras_redraws is given.
int launch_slots_setup(const int32_t* args, int B, const int32_t* page_table, int max_pages, int32_t* table, int32_t* seq_lens,
                       int32_t* n_generated, int32_t* done, int32_t* slot_key, int32_t* ras_redraws, cudaStream_t s);
// Several takes of one prompt.  args: device [3][nc] = parent slot, child slot, prompt length P of each child.  For
// every child with P % 64 != 0, rows [0, P % 64) of the parent's page P / 64 (its partly filled last prompt page) are
// copied into the child's page P / 64, in every layer, K and V, every KV head; full prompt pages are shared through
// the page table and never copied.  hist != nullptr: the child's repetition-penalty history row and recorded flag
// become copies of the parent's, in the same launch.
int launch_fork_tails(const int32_t* args, int nc, const KVLayout& kv, int n_layers, uint32_t* hist, int words, int32_t* recorded,
                      cudaStream_t s);

}  // namespace nt
