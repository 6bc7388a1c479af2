// Parameter block of the persistent decode megakernel (lm_mega.cu).
#pragma once
#include "lm_kernels.cuh"

namespace nt {

struct MegaPhase {  // one weight matrix streamed by the producer warps
  const __nv_bfloat16* W;
  int rows, K;
};

struct MegaParams {
  // model
  int n_layers;      // layers to run (== total_layers unless a debug limit is set)
  int total_layers;  // the lm_head entry sits at phases[4 * total_layers]
  int hidden, inter, n_heads, qkv_n, vocab;
  float eps, scale_log2;
  const MegaPhase* phases;        // device [4 * total_layers + 1]: (qkv, o, gate/up, down) per layer, lm_head
  const float* const* ln1;        // device arrays of per-layer pointers
  const float* const* bqkv;
  const float* const* ln2;
  const float* final_norm;
  const float* inv_freq;
  // activations (global memory, fp32)
  float *h, *q, *attn, *act, *logits;
  KVLayout kv;
  float *part_o, *part_ml;
  int* counters;
  int max_splits;
  SamplerParams samp;
  unsigned* gbar;     // grid barrier counter, zeroed before every launch
  int n_steps;
  float* logits_out;  // optional: this group's first row of [n_steps][batch][vocab]
  long long logits_step_stride;  // elements between consecutive steps in logits_out (batch * vocab)
  long long* prof;    // optional timeline buffer [2 CTAs][kProfMarks] of %globaltimer ns
  int prof_step;
  // shared-memory plan and tuning (filled by launch_decode_mega)
  int nstages, stage_bytes;
  int head_ld;        // rows of the per-CTA logits copy kept in shared memory per lm_head segment
  int head_segs;      // segments the CTA's lm_head rows are processed in (1 on a full-chip grid)
  int bias_cap;       // per-layer slots of the cached QKV bias slice (0 = not cached)
  int split_cap;      // attention splits per (sequence, kv head): 16 / batch
  int l2_prefetch;    // producer prefetches the next layer's slices into L2
  long long l2_head_bytes;
  size_t ring_off, x_off, union_off, misc_off, bar_off;
};

constexpr int kProfMarks = 1024;
int launch_decode_mega(MegaParams& P, int nb, int num_sms, cudaStream_t stream);

}  // namespace nt
