/* neutts_b200 — C-ABI of the H100 (sm_90a) implementation of NeuTTS-Air's two inference
 * hot paths.  Plain pointers and sizes only; no torch / C++ types cross this boundary.
 *
 * The reference has no FFI of its own (it is 465 lines of Python over `transformers` and
 * `neucodec`); the two inner seams this library replaces are
 *
 *   seam 1 (speech LM)  neutts/neutts.py:334-352  NeuTTS._infer_torch ->
 *                       self.backbone.generate(prompt, max_length=2048, eos_token_id=...,
 *                       do_sample=True, temperature=1.0, top_k=50, use_cache=True,
 *                       min_new_tokens=50)                     -> nt_lm_prefill + nt_lm_decode
 *   seam 2 (codec)      neutts/neutts.py:273-295  NeuTTS._decode ->
 *                       self.codec.decode_code(codes[B,1,N]) -> float[B,1,480N]
 *                                                              -> nt_codec_decode
 *
 * Conventions
 *   - every function returns 0 on success, a negative nt_status otherwise; nt_last_error()
 *     returns a human-readable message for the calling thread's last failure;
 *   - all device memory (weights, KV pages, workspaces, inputs, outputs) is allocated and
 *     owned by the caller (the Python shim uses torch tensors); the library never frees it;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on that stream
 *     unless stated otherwise;
 *   - matrices are row-major [out_features, in_features] exactly as torch.nn.Linear stores
 *     them; "bf16" means __nv_bfloat16, "f32" float.
 */
#ifndef NEUTTS_B200_H_
#define NEUTTS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  NT_OK = 0,
  NT_ERR_INVALID = -1,   /* bad argument / unsupported shape  -> ValueError in the shim  */
  NT_ERR_CUDA = -2,      /* CUDA runtime / driver failure     -> RuntimeError            */
  NT_ERR_NOMEM = -3,     /* caller-provided workspace too small                          */
  NT_ERR_STATE = -4      /* call order violated (e.g. decode before prefill)             */
} nt_status;

const char* nt_last_error(void);
/* library/ABI version, bumped on any signature change */
int nt_abi_version(void);   /* 2: nt_sampling gained limits + slot_base; 3: nt_codec_config.precision */
/* number of kernels launched by this library since load (all streams); bench.py reports the delta */
uint64_t nt_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Generic tensor-core GEMM (wgmma + TMA):  C[M,N] = epilogue(A[M,K] . W[N,K]^T)
 * Used by prefill, batched decode and the codec.  Replaces torch addmm/mm as reached from
 * transformers modeling_qwen2.py:46-48,217-219,244,475 and the codec's Linear/Conv1d layers.
 * ------------------------------------------------------------------------------------------ */
typedef enum { NT_BF16 = 0, NT_TF32 = 1 } nt_dtype;          /* A/W element type: bf16, or f32 fed as tf32 */
typedef enum { NT_ACT_NONE = 0, NT_ACT_SILU = 1, NT_ACT_SWIGLU = 2 } nt_act;

typedef struct {
  nt_dtype dtype;
  int M, N, K;
  const void* A;      /* [M, K] elements, row stride lda (elements).  lda < K is allowed: rows
                         then overlap, which is how Conv1d is expressed (im2col as a view)   */
  int64_t lda;
  const void* W;      /* [N, K], row stride ldw */
  int64_t ldw;
  const float* bias;      /* [N] or NULL */
  const float* residual;  /* [M, ldr] f32 or NULL; may alias out_f32 */
  int64_t ldr;
  nt_act act;             /* SWIGLU: columns (2j, 2j+1) = (gate_j, up_j) -> one output column j */
  float* out_f32;         /* [M, ldc] or NULL */
  void* out_bf16;         /* [M, ldc] or NULL */
  int64_t ldc;
  /* row mask for padded-batch layouts: if valid_period > 0 only rows with
     (row % valid_period) < valid_len are written */
  int valid_period, valid_len;
} nt_gemm_args;

int nt_gemm(const nt_gemm_args* args, void* stream);

/* GEMM conformance hook (tests): nt_gemm with the dispatcher's internal choices exposed.
 * bn: 0 = dispatcher's choice, else 32 | 64 | 128.  ring: -1 = dispatcher's choice, 0 = deep, 1 = shallow (half-depth).
 * w_const: W may be fetched before the PDL wait.  split_ws / split_floats: lend a split-K workspace; split_info int64[2]
 * receives (used, slice_stride).  a_lo_rows / w_lo_rows > 0: 3xTF32 (tf32 only, lo halves that many rows below).
 * tile_max / tile_ld: per-row maxima of every column tile (plain fp32 epilogue). */
int nt_debug_gemm(const nt_gemm_args* a, int bn, int ring, int w_const, float* split_ws, int64_t split_floats,
                  int64_t* split_info, int a_lo_rows, int w_lo_rows, float* tile_max, int64_t tile_ld, void* stream);
/* Teacher-forced scoring's lm_head epilogue alone (tests): bf16 A [M][K], W [N][K] (row stride K, K % 64 == 0);
 * per row r and 128-column tile t, lse float2 [r * lse_ld + t] = (max, sum exp(v - max)); zt[r] = logit tgt[r]. */
int nt_debug_gemm_logsoftmax(const void* A, int M, int K, const void* W, int N, const int32_t* tgt, void* lse,
                             int64_t lse_ld, float* zt, void* stream);

/* ------------------------------------------------------------------------------------------
 * Speech LM (seam 1)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int vocab_size, hidden, inter, n_layers, n_heads, n_kv_heads, head_dim; /* head_dim must be 64 */
  float rms_eps, rope_theta;
  int max_batch;      /* sequences resident at once */
  int max_ctx;        /* context limit (prompt + generated), reference: 2048 (neutts.py:85) */
  int page_size;      /* KV page, tokens; must be 64 */
  int num_pages;      /* pages in the pool (shared by all layers: one page id addresses every layer) */
  int max_prefill_tokens; /* sum of prompt lengths per nt_lm_prefill call */
} nt_lm_config;

/* Device pointers.  Packed layouts (built by neutts_air_b200/lm.py:pack_weights):
 *   wqkv  [ (n_heads+2*n_kv_heads)*64, hidden ] bf16, rows ordered q heads, k heads, v heads;
 *         inside every q/k head the 64 rows are interleaved (0,32,1,33,...,31,63) so RoPE
 *         partners are adjacent; v heads keep natural order.  bqkv follows the same order.
 *   wgu   [ 2*inter, hidden ] bf16, rows interleaved (gate_0, up_0, gate_1, up_1, ...).
 *   wo    [ hidden, n_heads*64 ],  wd [ hidden, inter ],  embed / lm_head [ vocab, hidden ].
 * The per-layer arrays are host arrays of n_layers device pointers. */
typedef struct {
  const void* embed;
  const void* lm_head;
  const float* final_norm;
  const float* const* ln1;
  const void* const* wqkv;
  const float* const* bqkv;
  const void* const* wo;
  const float* const* ln2;
  const void* const* wgu;
  const void* const* wd;
} nt_lm_weights;

/* Caller-owned device state for a batch of sequences (slots 0..B-1). */
typedef struct {
  void* kv_pages;        /* bf16 [n_layers][2 (k,v)][num_pages][n_kv_heads][page_size][64] */
  int32_t* page_table;   /* [max_batch][max_ctx/page_size] page ids */
  int32_t* seq_lens;     /* [max_batch] tokens already in the KV cache */
  int32_t* cur_token;    /* [max_batch] last sampled token (input of the next decode step) */
  int32_t* out_tokens;   /* [max_batch][max_new] generated ids (includes the EOS if hit) */
  int32_t* n_generated;  /* [max_batch] */
  int32_t* done;         /* [max_batch] 1 once EOS sampled or max_ctx reached */
  int32_t max_new;       /* row length of out_tokens */
} nt_lm_state;

/* Sampling semantics of transformers generation (logits_process.py:224-233,296-299,580-586;
 * utils.py:2789-2791): EOS masked while n_generated < min_new_tokens, logits / temperature,
 * keep the top_k largest, softmax, one multinomial draw (Philox4x32-10 keyed by seed, slot, step). */
typedef struct {
  int32_t eos_id;
  int32_t min_new_tokens;
  int32_t max_new_tokens;   /* stop after this many generated tokens (<= state.max_new) */
  int32_t top_k;            /* 1..64 */
  float temperature;
  uint64_t seed;
  int32_t greedy;           /* 1: argmax instead of sampling (tests) */
  const int32_t* forced;    /* optional [max_batch][max_new] teacher-forced tokens (tests), else NULL */
  const int32_t* limits;    /* optional device [max_batch]: per-sequence cap on generated tokens (transformers'
                               max_length is prompt + generated PER SEQUENCE, stopping_criteria.py:73-84), else NULL */
  int32_t slot_base;        /* global index of slot 0: keys the Philox stream, so chunks / ranks draw independently */
} nt_sampling;

typedef struct nt_lm nt_lm;

size_t nt_lm_workspace_bytes(const nt_lm_config* cfg);
int nt_lm_create(const nt_lm_config* cfg, const nt_lm_weights* w, void* workspace, size_t workspace_bytes, nt_lm** out);
int nt_lm_destroy(nt_lm* lm);

/* Prefill B prompts packed back to back: ids [total] (device), cu_seqlens [B+1] (host).
 * Fills the KV cache, samples the first token of every sequence (A2 + A10-A12 of SURVEY §8a).
 * logits_out: optional device f32 [B][vocab] receiving the last-position logits.
 * This is nt_lm_prefill_fork with n = 1: prompt b in slot b, every slot reset. */
int nt_lm_prefill(nt_lm* lm, const nt_lm_state* st, const int32_t* ids, const int32_t* cu_seqlens_host, int B,
                  const nt_sampling* sp, float* logits_out, void* stream);

/* Prefill B prompts into the listed slots (distinct, < max_batch) while every other slot keeps its KV pages,
 * tokens and counters.  ids / cu_seqlens_host as in nt_lm_prefill; slots_host, stream_ids_host: host [B].
 * Samples the first token of each listed slot.  Philox is keyed by stream_ids[i] (>= 0) instead of slot + slot_base
 * for that slot until the next nt_lm_prefill (which restores slot + slot_base for all slots).  Afterwards
 * nt_lm_decode(B_decode) continues every live slot < B_decode.  logits_out: optional [B][vocab] in call order.
 * The caller writes the listed slots' page-table rows (and limits entries) before the call, on the same stream.
 * Needs an earlier nt_lm_prefill; cur_token must hold a valid token id in every slot (a zeroed state does). */
int nt_lm_prefill_slots(nt_lm* lm, const nt_lm_state* st, const int32_t* slots_host, const int32_t* stream_ids_host,
                        const int32_t* ids, const int32_t* cu_seqlens_host, int B, const nt_sampling* sp,
                        float* logits_out, void* stream);

/* n takes of each of B prompts from one prefill (transformers' num_return_sequences).  A full prefill: it resets
 * every slot.  Take j of prompt i lives in slot i*n + j (repeat_interleave order);
 * 1 <= B*n <= max_batch.  The prompts are prefilled once, into the page-table rows of the parent slots i*n, so
 * logits_out (optional, [B][vocab]) is bit-identical for every n on the same B prompts.  Page sharing: the
 * caller writes every take's page-table row before the call, naming the parent's pages for the P_i / 64 full prompt
 * pages and the take's own pages from page P_i / 64 on; the call copies rows [0, P_i % 64) of the parent's page
 * P_i / 64 into each other take's page P_i / 64 (every layer, K and V).  Afterwards every take has seq_lens = P_i,
 * n_generated = done = 0, Philox stream i*n + j + slot_base, and a copy of its parent's repetition-penalty history;
 * its first token is drawn from the parent's logits row.  Decoding never writes a shared page: every decode path
 * writes K/V only at position seq_lens[s] of slot s, which lies in the take's own pages. */
int nt_lm_prefill_fork(nt_lm* lm, const nt_lm_state* st, const int32_t* ids, const int32_t* cu_seqlens_host, int B, int n,
                       const nt_sampling* sp, float* logits_out, void* stream);

/* Teacher-forced scoring: per-token log-probabilities of given sequences under the model alone, from one prefill pass.
 * For sequence b with tokens x_0 .. x_{L-1} (L = L_b) and start s = start_host[b], the score of token t (s <= t < L) is
 *   log_softmax(lm_head(final_norm(h_{t-1})))[x_t]
 * under causal attention over x_0 .. x_{t-1}: transformers' -cross_entropy(logits[s-1:L-1], ids[s:L]).  No repetition
 * penalty, EOS mask, vocabulary range, temperature or warper applies; the per-slot tables and the range are ignored
 * and left as they are.
 *   ids: device [total], the B sequences back to back; cu_seqlens_host: host [B+1]; start_host: host [B].
 *   out: device fp32 [sum_b (L_b - s_b)], the scores of sequence 0, then sequence 1, ...
 *   scratch: caller-owned device memory, 256-byte aligned, of at least nt_lm_score_scratch_bytes(cfg) bytes.
 * Rules: 1 <= B <= max_batch, sum L_b <= max_prefill_tokens, 1 <= s_b < L_b <= max_ctx; a violation returns
 * NT_ERR_INVALID.  The caller writes page-table rows 0..B-1 as for nt_lm_prefill; the prefill chain fills those pages.
 * Afterwards slot b < B has seq_lens = L_b, every slot has n_generated = 0 and done = 1, and nt_lm_decode /
 * nt_lm_prefill_slots return NT_ERR_STATE until the next nt_lm_prefill or nt_lm_prefill_fork.  Nothing is sampled:
 * out_tokens, cur_token, the log-probability buffer, the repetition-penalty histories, the Philox keys and the
 * settings tables are not written.
 * The lm_head runs over the scored rows in blocks of R = min(1024, max_prefill_tokens) rows with the log-softmax fused
 * into its epilogue: per row and 128-column vocabulary tile only the pair (max, sum exp) and the target logit leave
 * the GEMM, and a combine kernel folds the pairs in a fixed order.  Every token row's arithmetic is independent of the
 * other sequences in the call, so a sequence's scores are bit-identical however it is batched. */
/* scratch bytes of nt_lm_score (0 for an invalid config; needs no GPU):
 *   a(8 * R * ceil(vocab_size / 128)) + a(4 * R) + 2 * a(4 * max_prefill_tokens),  a(x) = x rounded up to 256 */
size_t nt_lm_score_scratch_bytes(const nt_lm_config* cfg);
int nt_lm_score(nt_lm* lm, const nt_lm_state* st, const int32_t* ids, const int32_t* cu_seqlens_host, const int32_t* start_host,
                int B, float* out, void* scratch, size_t scratch_bytes, void* stream);

/* Run n_steps decode steps for slots 0..B-1 with no host synchronisation in between
 * (finished slots keep their state; their work is skipped on device).
 * logits_out: optional device f32 [n_steps][B][vocab] (tests only; forces logits to HBM). */
int nt_lm_decode(nt_lm* lm, const nt_lm_state* st, int B, int n_steps, const nt_sampling* sp, float* logits_out,
                 void* stream);

/* Per-slot sampling controls, applied in transformers' processor order (generation/utils.py, logits_process.py):
 * EOS mask -> logit * (1.0f / temperature) -> top_k (exactly k, the smaller id wins ties) -> top_p -> min_p ->
 * softmax over what is left -> one multinomial draw with the same Philox counter as without the controls.
 * top_p and min_p act on the window sorted by (score desc, id asc) with its fp32 softmax q: entry j stays iff
 * sum_{i<j} q_i < top_p (entry 0 always stays) and q_j >= min_p * q_0.  top_p = 1 and min_p = 0 cut nothing. */
typedef struct {
  float temperature;  /* finite, > 0 */
  int32_t top_k;      /* 1..64 */
  float top_p;        /* (0, 1] */
  float min_p;        /* [0, 1) */
} nt_slot_sampling;

/* host_table: host array of max_batch entries, row s for slot s; NULL switches the table off, and then
 * nt_sampling.temperature / top_k govern every slot with top-p and min-p off.  While the table is on, its
 * temperature and top_k replace nt_sampling's for every sampler launch of nt_lm_prefill, nt_lm_prefill_slots and
 * nt_lm_decode (nt_sampling's own values are still validated); greedy and teacher-forced runs ignore it.  The copy
 * is enqueued on `stream`, so it is ordered before the next prefill or decode on that stream.  Every entry is
 * validated first; a bad one returns NT_ERR_INVALID and leaves the previous table in force.
 * nt_op_topk_sample does not read the table: it takes nt_sampling's scalars only. */
int nt_lm_set_slot_sampling(nt_lm* lm, const nt_slot_sampling* host_table, void* stream);

/* Vocabulary range (speech-token-only decoding; transformers' suppress_tokens with every id outside the allowed set).
 * Every later sampler launch of nt_lm_prefill, nt_lm_prefill_slots and nt_lm_decode may only draw an id in
 * [lo, hi) or the launch's nt_sampling.eos_id (EOS stays masked while n_generated < min_new_tokens).  The lm_head
 * then computes only the 128-row tiles of [lo, hi) and the tile that holds EOS; in every logits output each
 * suppressed id reads -inf and each allowed id is bit-identical to the same call with the range off.  The range holds
 * for every slot.  lo = 0, hi = vocab_size switches it off (the default).  Rules: 0 <= lo < hi <= vocab_size,
 * hi - lo >= 64, lo % 128 == 0, and hi % 128 == 0 or hi == vocab_size; a bad range returns NT_ERR_INVALID and leaves
 * the previous one in force.  Host state only: it applies to the launches enqueued on `stream` after the call, and
 * each launch carries it in its kernel parameters (nothing is copied to the device), so a graph a caller captures
 * keeps the range that was in force at capture.
 * nt_op_topk_sample and nt_lm_head_gemv ignore the range. */
int nt_lm_set_vocab_range(nt_lm* lm, int32_t lo, int32_t hi, void* stream);

/* Per-slot repetition penalty (transformers' RepetitionPenaltyLogitsProcessor).  Each slot's history is the set of
 * distinct ids of the prompt its last nt_lm_prefill / nt_lm_prefill_slots filled it with (include_prompt = 1), plus
 * every token written to out_tokens for it since (teacher-forced runs: the forced token).  Every id in the history
 * has its logit s replaced once by s < 0 ? s * penalty : s / penalty (IEEE fp32), before the EOS mask, the vocabulary
 * range and the temperature; it applies to greedy and teacher-forced runs too.  Every logits output and tile maximum
 * holds the penalised scores; every id outside the history is bit-identical to the table off.
 * The history lives on the device: a bitmap of the vocabulary per slot, built by each prefill and updated by the
 * sampler itself, so the token drawn at step t is penalised at step t + 1 inside one multi-step launch. */
typedef struct {
  float penalty;          /* finite, > 0; 1 = no penalty for this slot */
  int32_t include_prompt; /* 1: prompt ids count (transformers' default), 0: only generated ids */
} nt_slot_penalty;

/* host_table: max_batch entries (row s = slot s), or NULL = off (the default: nothing recorded, nothing penalised).
 * Every entry is validated first; a bad one returns NT_ERR_INVALID and leaves the previous table in force.  The copy is
 * enqueued on `stream`.  Switching the table on marks every slot unrecorded: an unrecorded slot is not penalised until
 * a prefill fills it again (tokens drawn while the table was off were never recorded).  New values in a table that
 * stays on take effect at the next launch, and the histories are kept.
 * nt_op_topk_sample and nt_lm_head_gemv ignore the penalty. */
int nt_lm_set_repetition_penalty(nt_lm* lm, const nt_slot_penalty* host_table, void* stream);

/* Per-slot length control: transformers' MinNewTokensLengthLogitsProcessor and ExponentialDecayLengthPenalty, applied
 * after the repetition penalty and before the vocabulary range, the temperature and the warpers.  With n the slot's
 * n_generated when its next token is drawn (tokens generated since its prompt):
 *   - EOS is masked (-inf) while n < min_new_tokens; the entry replaces nt_sampling.min_new_tokens for the slot;
 *   - while n > decay_start, with k = n - decay_start, the EOS score s becomes s + |s| * c_k (fp32 product, then fp32
 *     sum), where c_k = (float)(pow(decay_factor, k) - 1) is computed in double on the host, as transformers does.
 * Both act on the EOS logit alone and apply to greedy and teacher-forced runs too: every logits output and tile maximum
 * holds the decayed EOS score, and every other id is bit-identical to the table off.  An entry with decay_factor == 1
 * never touches the score.  A prefill draws token 0 of the slots it fills, where only the mask can apply. */
typedef struct {
  int32_t min_new_tokens;  /* >= 0 */
  int32_t decay_start;     /* >= 0 and >= min_new_tokens - 1 (the decay never meets the -inf of the mask) */
  double decay_factor;     /* finite, > 0; 1 = no decay */
} nt_slot_length;

/* host_table: max_batch entries (row s = slot s), or NULL = off (the default: nt_sampling.min_new_tokens for every slot,
 * no decay).  Every entry is validated first; a bad one returns NT_ERR_INVALID and leaves the previous table in force.
 * The table and each slot's c_k for k = 1 .. max_ctx are copied on `stream`; new values take effect at the next launch.
 * A c_k that is not finite in fp32 is refused by the launch that could reach it: nt_lm_prefill_slots,
 * nt_lm_prefill_fork and nt_lm_decode return NT_ERR_INVALID while some slot the call samples (the listed slots, the
 * B * n takes, or slots 0 .. B - 1) has a non-finite c_k with k <= nt_sampling.max_new_tokens - decay_start.  Other
 * slots may keep entries of an earlier call with a shorter cap.
 * nt_op_topk_sample, nt_lm_head_gemv and nt_lm_score ignore the table. */
int nt_lm_set_length_control(nt_lm* lm, const nt_slot_length* host_table, void* stream);

/* Per-slot Repetition Aware Sampling (VALL-E 2; CosyVoice 2's ras_sampling).  At every sampled draw of a slot whose
 * entry is on, with n the slot's n_generated: the sampler draws token t as usual (u1 = Philox word 0 of counter
 * {n, stream key, 0, 0}); if t occurs at least min_count times among the slot's generated tokens [max(0, n - window), n)
 * (its prompt never counts), t is replaced by one draw from the full distribution, the softmax of the processed scores
 * times 1 / T over the whole vocabulary row (no top-k / top-p / min-p cut), by inverse CDF in ascending id order with
 * u2 = (Philox word 1 of the same block >> 8) * 2^-24.  Suppressed ids (vocabulary range, EOS while masked) stay out.
 * The redrawn token is kept even if it repeats too.  Greedy and teacher-forced runs never redraw, nor does token 0
 * (its window is empty).  With nt_lm_set_logprobs on, a redrawn token's `sampled` value is its log-probability in the
 * full distribution.  Every draw that does not trigger is bit-identical to the table off. */
typedef struct {
  int32_t window;     /* 0 = off for this slot, else 1..64 */
  int32_t min_count;  /* 1..window */
} nt_slot_ras;

/* host_table: max_batch entries (row s = slot s), or NULL = off (the default).  Every entry is validated first; a bad
 * one returns NT_ERR_INVALID and leaves the previous table in force.  The table is copied on `stream`; new values take
 * effect at the next launch.  nt_lm_debug_ptr(lm, "ras_redraws") is a device int32 [max_batch] count of each slot's
 * redraws since the prefill that filled it.  nt_op_topk_sample, nt_lm_head_gemv and nt_lm_score ignore the table. */
int nt_lm_set_repetition_aware_sampling(nt_lm* lm, const nt_slot_ras* host_table, void* stream);

/* Per-token log-probabilities.  out: caller-owned device fp32 [max_batch][max_new][2] (8-byte aligned); entry [s][n]
 * belongs to out_tokens[s][n] and is written wherever that token is (every sampler launch of nt_lm_prefill,
 * nt_lm_prefill_slots and nt_lm_decode); nothing else is written.  NULL switches it off (the default).
 *   [0] sampled: log-probability of the token in the distribution the sampler drew from, the kept window after
 *       penalty -> EOS mask -> vocabulary range -> 1 / T -> top_k -> top_p -> min_p, renormalised (transformers'
 *       compute_transition_scores(normalize_logits=True) on output_scores).  Greedy runs: equal to [1], since
 *       transformers applies no warpers there.  Teacher-forced runs: -inf when the forced id lies outside the window.
 *   [1] model: log-softmax of the token over the whole vocabulary, on the scores after the repetition penalty, the
 *       min-new-tokens EOS mask (EOS left out of the sum while masked) and the vocabulary range (suppressed ids add
 *       nothing), before temperature and the warpers.
 * Host state only, like nt_lm_set_vocab_range.  nt_op_topk_sample and nt_lm_head_gemv ignore it. */
int nt_lm_set_logprobs(nt_lm* lm, float* out, void* stream);

/* Classifier-free guidance (transformers' guidance_scale with negative_prompt_ids,
 * UnbatchedClassifierFreeGuidanceLogitsProcessor).  A guided pair is two slots: c (conditional: its prompt, its tokens
 * are the ones returned) and u = table[c].partner (unconditional: the negative prompt, then every token c draws).  At
 * every sampler launch, right after the lm_head (and the vocabulary range's EOS tile), c's logits row becomes
 *   g * (ls_c - ls_u) + ls_u      (fp32, in that order; g = table[c].scale)
 * with ls the log-softmax of the row over the ids the lm_head computes; an id that reads -inf in either row stays -inf.
 * The repetition penalty, EOS mask, length decay, temperature, warpers, Philox draw and log-probabilities then act on
 * that row as usual, with c's settings.  u is never sampled: after each sampler launch its out_tokens, cur_token and
 * n_generated mirror c's, its seq_lens advances, its done is c's, and its next input is c's token.  If u's context
 * would reach max_ctx, both slots finish (cap c through nt_sampling.limits so that u fits).  The combine reads u's raw
 * logits; u's own table entries only shape u's logits outputs.  Slots outside a pair are bit-identical to the table off.
 * Rules (NT_ERR_INVALID, previous table kept): partner in -1 .. max_batch - 1 and not the slot itself; a partner serves
 * one c and has no partner of its own; scale finite, > 0 and != 1 wherever partner >= 0 (ignored elsewhere).
 * While the table is on: nt_lm_decode runs the per-op chain at every batch (NT_DECODE_IMPL=tc returns NT_ERR_INVALID),
 * and every pair with a slot below the call's batch must lie wholly below it; nt_lm_prefill and nt_lm_prefill_slots
 * need both slots of every pair they touch in the same call; nt_lm_prefill_fork returns NT_ERR_INVALID.  Switching the
 * table on or off rebuilds the cached decode graph; new contents of a table that stays on reach it at replay.
 * nt_op_topk_sample, nt_lm_head_gemv and nt_lm_score ignore the table. */
typedef struct {
  int32_t partner;   /* u slot of this c slot, or -1 */
  float scale;       /* guidance scale g */
} nt_slot_guidance;

/* table: host array of max_batch entries (row s = slot s), or NULL = off (the default).  Copied on `stream`. */
int nt_lm_set_guidance(nt_lm* lm, const nt_slot_guidance* table, void* stream);

/* Timed single-kernel entry for the roofline measurement: the lm_head GEMV (+ final RMSNorm)
 * exactly as the decode step launches it.  h: f32 [B][hidden] -> logits f32 [B][vocab]. */
int nt_lm_head_gemv(nt_lm* lm, const float* h, int B, float* logits, void* stream);

/* Per-stage parity hooks (tests): run only the first n_layers layers (-1 = all), and look up an
 * internal activation buffer by name ("h", "q", "qkv", "attn", "act", "logits", "xn", "attn_bf16",
 * "act_bf16", "h_last", "tmax"); the pointer lies inside the caller's workspace. */
int nt_lm_debug_set_layers(nt_lm* lm, int n_layers);
/* Decode on n_ctas CTAs as if the device had that many SMs (tests): the persistent kernel's grid and work plans, its
 * "batch x kv heads <= CTAs" gate and the GEMV grids all take n_ctas, and both plans are rebuilt for it (a whole-K
 * plan the planner rejects there sends every decode to the per-op chain).  0 restores the default, the device's SM
 * count capped at 256; otherwise 8 <= n_ctas <= min(device SMs, 256), else NT_ERR_INVALID.  Synchronises the device
 * and drops the cached decode graph when the count changes.  The wgmma GEMMs keep sizing from the device. */
int nt_lm_debug_set_sms(nt_lm* lm, int n_ctas);
/* launch-latency probe: n dependent trivial kernels (grid x block) each incrementing *counter */
int nt_debug_launch_chain(int n, int grid, int block, int* counter, void* stream);
void* nt_lm_debug_ptr(nt_lm* lm, const char* name);
/* persistent decode kernel timeline: buf = device int64 [2][1024] receiving %globaltimer marks of decode
 * step `step` from CTAs 0 and 1 (NULL disables) */
int nt_lm_debug_set_profile(nt_lm* lm, long long* buf, int step);
/* sampler window capture (tests): caller-owned device buffers topk_val fp32 [max_batch][64], topk_idx int32
 * [max_batch][64] and token int32 [max_batch] receive, per logits row, the kept probabilities, the kept ids (-1
 * padded) and the selected token of every sampler launch (prefill, prefill into slots, decode chain, persistent
 * decode kernel).  Row b is logits row b: call order in nt_lm_prefill_slots.  Each launch overwrites them, so a
 * multi-step persistent decode launch leaves its last step.  NULL pointers switch the capture off.  Debug "tmax"
 * (nt_lm_debug_ptr) holds the per-128-column tile maxima of the last tile-max sampler input. */
int nt_lm_debug_capture_sampler(nt_lm* lm, float* topk_val, int32_t* topk_idx, int32_t* token);
/* work plan of the persistent decode kernel (tests): runs the host planner for a model shape on n_sms CTAs with
 * whole-K (flat = 0) or flat (flat = 1) gate/up, and makes no CUDA call.  Outputs (each may be NULL):
 * items int16 [n_sms][4][4][4]: per CTA, phase (0 qkv, 1 o_proj, 2 gate/up, 3 down_proj) and item (tile, first k-block,
 * k-blocks, slice), a k-block being 64 elements of K; counts int32 [n_sms][4]: items per phase; flags int32 [n_sms][3]:
 * fold_q, fold_g (1 on the first CTA that consumes the ln1 / ln2 fold, i.e. has qkv / gate-up items), gu_split;
 * gu_nsl uint8 [gu_cap]: K slices of every gate/up tile (flat plan); info int32 [7]: K slices
 * of the qkv, o_proj and down_proj phases, most slices of a gate/up tile, lm_head tiles, most k-blocks a CTA stages in
 * one phase, gu_split.  NT_ERR_INVALID with a message when the plan does not fit the kernel. */
int nt_debug_decode_plan(int hidden, int inter, int n_heads, int n_kv, int vocab, int n_sms, int flat, int16_t* items,
                         int32_t* counts, int32_t* flags, uint8_t* gu_nsl, int gu_cap, int32_t* info);

/* ------------------------------------------------------------------------------------------
 * NeuCodec decoder (seam 2)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int hidden, depth, heads, head_dim;   /* 1024, 12, 16, 64 */
  int mlp_hidden;                       /* 4096 */
  int groups;                           /* GroupNorm groups (32) */
  int embed_kernel;                     /* 7 */
  int n_fft, hop;                       /* 1920, 480 */
  int fsq_levels, fsq_dims;             /* 4, 8 */
  float norm_eps, rope_base, mag_clip;
  int rope_time_axis;                   /* 1: rotary over frames; 0: upstream quirk (no-op, skipped) */
  int max_batch, max_frames;
  int precision;                        /* arithmetic of the tensor-core GEMMs (fp32 storage, fp32 accumulate):
                                           0 = TF32, with 3xTF32 (hi/lo operand split, fp32-grade products) for the ISTFT
                                               head and the inverse-DFT GEMMs only ("mixed")
                                           1 = TF32 everywhere (fastest; 3.4e-4 abs RMS on speech-level weights)
                                           2 = 3xTF32 everywhere (fp32-grade; what the Python host passes by default:
                                               the only mode within 1e-3 RMS of the fp32 path on adversarial heads) */
} nt_codec_config;

/* All f32, device.  Conv weights are pre-flattened tap-major: [C_out, k*C_in] with
 * W2[co, tap*C_in + ci] = W[co, ci, tap].  fsq_w/fsq_b are the collapsed
 * fc_post_a(project_out(.)) affine: [hidden, fsq_dims], [hidden]. */
typedef struct {
  const float* fsq_w; const float* fsq_b;
  const float* embed_w; const float* embed_b;
  /* 4 resnet blocks (2 prior, 2 post): arrays of 4 device pointers each */
  const float* const* rn_n1w; const float* const* rn_n1b; const float* const* rn_c1w; const float* const* rn_c1b;
  const float* const* rn_n2w; const float* const* rn_n2b; const float* const* rn_c2w; const float* const* rn_c2b;
  /* depth transformer blocks */
  const float* const* att_norm; const float* const* wqkv; const float* const* wproj;
  const float* const* ffn_norm; const float* const* fc1; const float* const* fc2;
  const float* final_ln_w; const float* final_ln_b;
  const float* head_w;   /* [n_fft+2, hidden] */
  const float* head_b;
  const float* idft_basis; /* [n_fft, Kpad] f32: windowed inverse-rDFT basis, Kpad = roundup(n_fft+2, 32) */
} nt_codec_weights;

typedef struct nt_codec nt_codec;

size_t nt_codec_workspace_bytes(const nt_codec_config* cfg);
int nt_codec_create(const nt_codec_config* cfg, const nt_codec_weights* w, void* workspace, size_t workspace_bytes,
                    nt_codec** out);
int nt_codec_destroy(nt_codec* c);
/* codes: device int32 [B][N] (all items the same length N); pcm: device f32 [B][hop*N].  Every int32 id decodes as
 * id mod fsq_levels**fsq_dims (floor modulo: -1 is the last code). */
int nt_codec_decode(nt_codec* c, const int32_t* codes, int B, int N, float* pcm, void* stream);
/* Per-stage parity hooks (tests).  Later nt_codec_decode calls run only stages first..last (last = -1: through the
 * last stage; (0, -1), the default, runs them all).  Stages in launch order:
 *   0 fsq (codes -> x0, after the memsets of x0, x1, x2)   1 embed (conv k7, x0 -> x1)
 *   per resnet block (2 before the transformer blocks, 2 after), 4 each:
 *     gn1 (x1 -> x2) | conv1 (x2 -> x3) | gn2 (x3 -> x2) | conv2 (x2 + x1 -> x1)
 *   per transformer block, 8 each (7 when rope_time_axis = 0, which has no rope stage):
 *     norm1 (x1 -> xn) | qkv (xn -> qkv) | rope (qkv in place) | attn (qkv -> att) | proj (att + x1 -> x1) |
 *     norm2 (x1 -> xn) | fc1 + SiLU (xn -> hbuf) | fc2 (hbuf + x1 -> x1)
 *   final LN (x1 -> xn) | head (xn -> sp) | spec (sp in place) | idft (sp -> fr) | ola (fr -> pcm)
 * A 3xTF32 GEMM's operand split belongs to its stage.  A call that starts past stage 0 reads the buffers as the
 * previous call (or the caller) left them.  A range outside 0..n_stages-1 returns NT_ERR_INVALID.  nt_codec_debug_ptr
 * looks up a workspace buffer by name ("x0", "x1", "x2", "x3", "xn", "qkv", "hbuf", "att", "sp", "fr"; NULL for any
 * other name).  Activations are channels-last fp32 rows; item b, frame t sits at row b*(N+6) + 3 + t. */
int nt_codec_debug_set_stages(nt_codec* c, int first, int last);
void* nt_codec_debug_ptr(nt_codec* c, const char* name);

/* ------------------------------------------------------------------------------------------
 * Output resampler: 24 kHz PCM -> sample_rate, optionally as 16-bit PCM, for whole rows and for streams
 * ------------------------------------------------------------------------------------------
 * Semantics of torchaudio.functional.resample(x, 24000, sample_rate) with its defaults (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99).  With g = gcd(24000, sample_rate), orig = 24000 / g, target = sample_rate / g:
 * width = ceil(6 * orig / (0.99 * min(orig, target))), taps = 2 * width + orig, and output sample k * target + p is
 * the dot product of phase p of the filter table with x_pad[k * orig .. k * orig + taps), x_pad being x with `width`
 * zeros in front and width + orig zeros behind; a row of L samples gives ceil(target * L / orig) samples.  At 24000 there
 * is no filter (width 0, one tap of 1.0).  The table is computed in float64 and rounded once to fp32; outputs accumulate
 * in fp32 over the taps in ascending order.  Rates whose fp32 table (target x taps) exceeds 227 KB, the shared memory
 * an sm_90 block can opt into, are rejected.
 * Streams: after L samples of a row have arrived, output frame k (samples k * target .. k * target + target - 1) is final
 * once k * orig + width + orig <= L.  A push emits exactly the frames that became final and keeps the samples the first
 * frame not yet final reads (fewer than taps); a final push pads with zeros, emits the rest, so a row's total is
 * ceil(target * L / orig), and leaves the row reset.  Every output is bit-identical however its row was split into pushes.
 * 16-bit PCM (NT_PCM_S16): each output y becomes __float2int_rn(fminf(fmaxf(y, -1), 1) * 32767) in fp32: clipped to
 * [-32767, 32767], rounded half to even. */
typedef enum { NT_PCM_F32 = 0, NT_PCM_S16 = 1 } nt_pcm_format;

typedef struct {
  int32_t orig, target;     /* 24000 / g, sample_rate / g */
  int32_t width, taps;
  size_t table_bytes;       /* device bytes of the filter table (16-byte aligned) */
  size_t row_bytes;         /* device bytes of one row's stream state (16-byte aligned) */
} nt_resampler_info;

typedef struct nt_resampler nt_resampler;

/* Geometry and sizes for a rate (needs no GPU); NT_ERR_INVALID, with the limit in the message, for a rejected rate. */
int nt_resampler_query(int sample_rate, nt_resampler_info* info);
/* table: caller-owned device memory of info.table_bytes, filled here (synchronously); state: device memory of
 * max_rows * info.row_bytes (NULL when max_rows is 0), read and written by nt_resampler_push on the rows it names.
 * Every row starts reset.  Needs an sm_90 device. */
int nt_resampler_create(int sample_rate, int pcm_format, int max_rows, void* table, void* state, nt_resampler** out);
int nt_resampler_destroy(nt_resampler* rs);
/* Rows [n] (host) start a new stream: their held samples are dropped.  Host state only. */
int nt_resampler_reset(nt_resampler* rs, const int32_t* rows, int n);
/* Resample n items in one launch per 128 items.  in: device fp32, item i at in[in_offsets[i] .. in_offsets[i + 1]);
 * out: device fp32 or int16 (the pcm_format of create), item i at out[out_offsets[i] .. out_offsets[i + 1]).  Offsets
 * are host arrays of n + 1 non-decreasing entries.  rows: host [n] distinct rows < max_rows, whose streams continue;
 * final_flags: host [n] (NULL: none final), nonzero ends that row's stream.  rows = NULL resamples each item whole as
 * a one-shot row (no state is read or written; final_flags is ignored).  Each item's output span must be exactly the
 * number of samples the contract above makes final, else NT_ERR_INVALID and nothing is launched. */
int nt_resampler_push(nt_resampler* rs, int n, const int32_t* rows, const int32_t* final_flags, const float* in,
                      const int64_t* in_offsets, void* out, const int64_t* out_offsets, void* stream);

/* ------------------------------------------------------------------------------------------
 * Speaking rate: a phase-vocoder time stretch of 24 kHz PCM, for whole rows and for streams
 * ------------------------------------------------------------------------------------------
 * Semantics of librosa.effects.time_stretch(x, rate=r), 0.5 <= r <= 2.0 (r > 1 is faster speech; pitch is kept), as
 * torch / torchaudio compute it in float64 for a row x of L samples:
 *   S  = stft(x, n_fft 1024, hop 256, periodic Hann window, center, zero padding)       T = 1 + L / 256 frames
 *   S2 = torchaudio.functional.phase_vocoder(S, r, linspace(0, pi * 256, 513))         K = ceil(T / r) frames
 *   y  = istft(S2, same window, center, length = round(L / r))
 * Output frame j sits at tau_j = j * r (fp64 product, never accumulated) and reads analysis frames a0_j = floor(tau_j)
 * and a1_j = floor(tau_j + 1) (the fp64 sum, as torchaudio's (time_steps + 1).long()), frames at or past T being zero;
 * K is torch.arange's count, ceil(T / r) in fp64; round is half to even.  (torch.arange's own values can differ from
 * j * r by an ulp, depending on the CPU's vector width; where that crosses an integer torchaudio interpolates another
 * frame pair.  The product is the contract here, the same on every machine.)
 * The analysis and synthesis DFTs are wgmma GEMMs in 3xTF32 against windowed bases computed in float64; the vocoder
 * runs in fp64 on the fp32 spectra with an fp64 phase accumulator wrapped to [-pi, pi] at every frame; the overlap-add
 * sums frames in ascending order in fp32 and divides by the fp32 window-square envelope.
 * Streams: with n input samples of a row received,
 *   - analysis frame a is complete once n >= 256 a + 512 (its last input sample is x[256 a + 511]);
 *   - output frame j is ready once frames a0_j and a1_j are complete: J(n) = the number of j with 256 a1_j + 512 <= n
 *     (a prefix, since a1_j grows with j);
 *   - output sample e reads output frames floor((e + 512 - 1023) / 256) .. floor((e + 512) / 256), so it is final once
 *     e < 256 J(n) - 512.  That bound is always below round(n / r) - 511 <= round(L / r) - 511 for r <= 2, so a later
 *     length = round(L / r) can never trim a sample a push has emitted.
 * A push emits exactly the samples that became final: max(0, 256 J(n) - 512) in total after a non-final push.  A final
 * push pads with zeros, emits the rest, so a row's total is round(L / r), and leaves the row reset.  Every output is
 * bit-identical however its row was split into pushes and whichever other rows share a push. */
typedef struct {
  int32_t n_fft, hop;          /* 1024, 256 */
  int32_t max_items;           /* rows per round of launches */
  int32_t chunk;               /* input samples per row per round: a push walks longer inputs in rounds */
  int32_t spec_ld;             /* debug "spec": fp32 rows of spec_ld floats, Re of bins 0..512 then Im of bins 0..512 */
  int32_t stretch_ld;          /* debug "stretch": 3xTF32 hi rows of stretch_ld floats (Re | Im as above), the lo
                                  halves stretch_lo_rows rows further down; a value is hi + lo */
  int32_t stretch_lo_rows;
  size_t table_bytes;          /* device bytes of the bases (filled by create) */
  size_t row_bytes;            /* device bytes of one row's stream state */
  size_t scratch_bytes;        /* device bytes of the scratch one push uses (independent of the input length) */
} nt_stretch_info;

typedef struct nt_stretch nt_stretch;

/* Sizes (needs no GPU). */
int nt_stretch_query(nt_stretch_info* info);
/* table, state (max_rows * row_bytes; NULL when max_rows is 0) and scratch: caller-owned device memory, 256-byte aligned.
 * The table is filled here (synchronously).  Every row starts reset.  Needs an sm_90 device. */
int nt_stretch_create(int max_rows, void* table, void* state, void* scratch, nt_stretch** out);
int nt_stretch_destroy(nt_stretch* st);
/* Rows [n] (host) start a new stream: their held samples, phases and speed are dropped.  Host state only. */
int nt_stretch_reset(nt_stretch* st, const int32_t* rows, int n);
/* Stretch n items.  in: device fp32, item i at in[in_offsets[i] .. in_offsets[i + 1]); out: device fp32, item i at
 * out[out_offsets[i] .. out_offsets[i + 1]); offsets are host arrays of n + 1 non-decreasing entries.  speeds: host [n]
 * fp64, each in [0.5, 2.0].  rows: host [n] distinct rows < max_rows, whose streams continue; final_flags: host [n]
 * (NULL: none final), nonzero ends that row's stream.  A row keeps the speed of its first push after a reset until its
 * stream ends; a push that names another speed for it returns NT_ERR_INVALID.  rows = NULL stretches each item whole
 * (one final push per item through the same path, on state rows inside the scratch; final_flags is ignored).  Each
 * item's output span must be exactly the number of samples the contract above makes final, else NT_ERR_INVALID and
 * nothing is launched.  Inputs longer than info.chunk are walked in rounds of that many samples per row, at most
 * info.max_items rows per round; each round is five launches on `stream` (pack, analysis GEMM, vocoder, synthesis
 * GEMM, overlap-add), the GEMMs skipped when no frame is due. */
int nt_stretch_push(nt_stretch* st, int n, const int32_t* rows, const int32_t* final_flags, const double* speeds,
                    const float* in, const int64_t* in_offsets, float* out, const int64_t* out_offsets, void* stream);
/* Stage hooks (tests): the scratch buffers of the last round, by name: "spec" (analysis spectra: row rb + a - a0 is
 * frame a of the round's row whose A rows start at rb; a lone row's first round starts at row 0 with frame 0),
 * "stretch" (stretched spectra, hi / lo halves; a lone one-shot row of at most info.chunk samples holds its frames
 * 0 .. K-1 at rows 0 .. K-1), "frames" (windowed time frames, 1024 floats per stretched row); NULL for other names. */
void* nt_stretch_debug_ptr(nt_stretch* st, const char* name);

/* ------------------------------------------------------------------------------------------
 * Loudness: ITU-R BS.1770-4 integrated loudness of mono rows, and normalisation to a target
 * ------------------------------------------------------------------------------------------
 * Input: mono fp32 PCM at rate r, r a multiple of 10 Hz in [8000, 192000] (so a gating block is exactly four steps;
 * any other rate is NT_ERR_INVALID).  Everything below is computed in fp64.
 *   K-weighting: two biquads in cascade, zero initial state, no clamping; coefficients as torchaudio's formulas,
 *     normalised by a0: treble_biquad(gain 4.0, central_freq 1500, Q 1/sqrt(2)), then highpass_biquad(38, Q 0.5).
 *   Blocks: gate = round(0.4 r), step = gate / 4; nb = floor((n - gate) / step) + 1 full blocks (none when n < gate);
 *     block j is y[j step, j step + gate) and z_j the mean of y^2 over it.
 *   Gating: l_j = -0.691 + 10 log10(z_j); absolute gate l_j > -70; G_r = -0.691 + 10 log10(mean z over the blocks
 *     above the absolute gate) - 10; relative gate l_j > G_r and l_j > -70;
 *     L = -0.691 + 10 log10(mean z over the blocks that pass both).  L is NaN when no block passes (silence, n < gate).
 * L equals torchaudio.functional.loudness(x[None], r) in float64 whenever both K-weighting stages stay inside [-1, 1].
 * Two differences are deliberate: torchaudio's lfilter clamps every stage's output to [-1, 1] (BS.1770 does not, and
 * neither does this meter), and torchaudio raises for n < gate where this meter returns NaN.
 * Normalisation to a target T: g = 10^((T - L) / 20) in fp64 and each output sample is float32(g * (double)x), rounded
 * once.  A row whose L or T is NaN comes back bit for bit unchanged.  There is no limiter: outputs may exceed +-1.
 * The recursion runs in chunks of info.chunk samples (chunk divides step): pass 1 runs every chunk from zero state,
 * the true start states follow exactly by linearity (per step, then along the row), and pass 2 re-runs every chunk from
 * its true state.  No float atomics: two runs give the same bits. */
typedef struct {
  int32_t gate, step;          /* samples per gating block and per 100 ms step */
  int32_t chunk;               /* samples one thread filters */
  int32_t chunks_per_step;     /* step / chunk */
} nt_loudness_info;

/* Geometry for a rate (needs no GPU); NT_ERR_INVALID, with the reason, for a rejected rate. */
int nt_loudness_query(int sample_rate, nt_loudness_info* info);
/* Device workspace bytes nt_loudness_run needs for these rows (host offsets, n + 1 non-decreasing entries); 0 for
 * n == 0 or invalid arguments (the reason in nt_last_error). */
size_t nt_loudness_workspace_bytes(int sample_rate, int n, const int64_t* in_offsets);
/* Measure n rows and optionally normalise them, stateless, on `stream`.  in: device fp32, row i at
 * in[in_offsets[i] .. in_offsets[i + 1]) (host offsets).  lufs: device fp64 [n], L of every row.  targets: host fp64
 * [n] in LUFS, or NULL to measure only; a NaN target leaves its row unchanged, an infinite one is NT_ERR_INVALID.  out:
 * device fp32 at the same offsets (may equal in), written only when targets is not NULL.  workspace: device memory,
 * 16-byte aligned, of at least nt_loudness_workspace_bytes (NT_ERR_NOMEM otherwise).  Rows go in groups of 128; each
 * group is one host-to-device copy of the chunk transition powers followed by up to six launches.  Nothing
 * synchronises the host. */
int nt_loudness_run(int sample_rate, int n, const float* in, const int64_t* in_offsets, const double* targets,
                    double* lufs, float* out, void* workspace, size_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Single-op entry points (unit tests; each mirrors one row of SURVEY.md §8a)
 * ------------------------------------------------------------------------------------------ */
int nt_op_rmsnorm(const float* x, const float* w, float eps, int rows, int cols, float* out_f32, void* out_bf16,
                  void* stream);
/* scalar controls only (nt_sampling's temperature and top_k for every row; no per-slot table, no top-p / min-p) */
int nt_op_topk_sample(const float* logits, int B, int V, const nt_sampling* sp, const int32_t* n_generated,
                      int32_t step, int32_t* out_token, float* out_topk_val, int32_t* out_topk_idx, void* workspace,
                      size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEUTTS_B200_H_ */
