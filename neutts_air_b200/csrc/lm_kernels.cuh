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
  // Fused RoPE + KV append (tensor-core variant, batch > 4): when qkv != nullptr the kernel reads the projection output
  // itself ([B, qkv_n] fp32, bias already added, `qkv_parts` split-K slices `qkv_pstride` floats apart, summed in slice
  // order), rotates q / k at position seq_lens[b], appends the new K/V row to the cache and ignores `q`.
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
  // candidates scratch: [B, nchunks, 64] (val, idx)
  float* cand_val;
  int32_t* cand_idx;
  int nchunks;
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
  const int32_t* slot_key;  // optional [max_batch] Philox stream key per slot; -1: slot + slot_base
  // optional [max_batch] temperature / top_k / top_p / min_p per slot (nt_lm_set_slot_sampling), read through
  // row_sampling() with the row's slot; nullptr: sp.temperature and sp.top_k for every row, no top-p / min-p cut
  const nt_slot_sampling* slot_sp;
};
int launch_sampler(const SamplerParams& p, int B, cudaStream_t stream);
int launch_sampler_check(const SamplerParams& p);
// tmax: [B][nt] RAW maxima of the 128-column tiles of p.logits (GEMM epilogue, gemm_dispatch(..., tile_max))
int launch_sampler_tiles(const SamplerParams& p, int B, const float* tmax, int nt, cudaStream_t stream);
size_t sampler_scratch_floats(int B, int V);  // per-array element count for cand_val / cand_idx
// Vocabulary range (nt_lm_set_vocab_range).  launch_fill_neg_inf: p[0, n) = -inf (the logits rows and tile maxima of a
// launch, before its lm_head writes the tiles it computes).  launch_vocab_eos_tile: after an lm_head that computed the
// whole 128-row tile holding `eos` although only `eos` is allowed there, rows [0, B) of that tile read -inf except eos,
// and tmax (optional, [B][nt] raw maxima) holds the eos logit as the tile's maximum.
int launch_fill_neg_inf(float* p, long long n, cudaStream_t s);
int launch_vocab_eos_tile(float* logits, int B, int V, int eos, float* tmax, int nt, cudaStream_t s);
int sampler_nchunks(int V);

int launch_embed_rows(const __nv_bfloat16* embed, const int32_t* ids, int T, int hidden, float* h, cudaStream_t s);
// parts != nullptr: x is updated in place first (x += sum of nparts split-K slices, slice order) -- see SplitK
int launch_rmsnorm_rows(const float* x, const float* w, float eps, int rows, int cols, float* out_f32,
                        __nv_bfloat16* out_bf16, cudaStream_t s, const float* parts = nullptr, int nparts = 0,
                        long long pstride = 0);
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
// slots' page-table rows into table [B][max_pages] and resets those slots' seq_lens / n_generated / done / slot_key.
int launch_slots_setup(const int32_t* args, int B, const int32_t* page_table, int max_pages, int32_t* table, int32_t* seq_lens,
                       int32_t* n_generated, int32_t* done, int32_t* slot_key, cudaStream_t s);

}  // namespace nt
