// Parameter block + work plan of the persistent wgmma decode kernel (lm_decode_tc.cu): ONE cooperative launch
// runs every layer, the lm_head, the sampler and the whole multi-step decode loop for batch 1..64.
#pragma once
#include <cuda.h>

#include "lm_kernels.cuh"

namespace nt {

constexpr int kTcMaxItems = 4;      // work items of one GEMM phase a CTA may own
constexpr int kTcMmaWarp0 = 8;      // warps 8..11: the MMA warpgroup (warpgroup-aligned)
constexpr int kTcStreamWarp = 12;   // the weight-stream warp
constexpr int kTcThreads = 416;     // 8 worker warps + 1 MMA warpgroup + 1 weight-stream warp
constexpr int kTcMaxBatch = 64;
constexpr int kTcDefaultMaxBatch = 16;  // nt_lm_decode's default: larger batches take the per-op chain
constexpr int kTcMaxSlices = 16;
constexpr int kTcMaxGuSlices = 4;   // K slices of one gate/up tile in the flat plan (batch <= 4)

// One GEMM work item: rows [tile*128, tile*128+128) of a weight matrix times k-blocks [kb0, kb0+nkb) of the
// activations (a k-block = 64 elements = one 128-byte swizzle row).  Items of the split-K phases (qkv, o, down)
// write raw partial sums into slice `slice`; gate/up items cover the whole K (their epilogue is not linear).
struct TcItem {
  short tile, kb0, nkb, slice;
};

// Per-CTA plan, identical for every layer (the four weight matrices of a layer have the same shape in every
// layer).  Built on the host (tc_build_plan), read once.  The lm_head split is not built on the host: the kernel
// fills head_t0 / head_t1 in its shared copy, CTA c taking positions [n c / G, n (c + 1) / G) of TcParams' lm_head
// tile list (n = head_n), so a launch's vocabulary range lives in the kernel parameters alone.
struct TcPlan {
  int n[4];                       // items per phase: 0 = qkv, 1 = o_proj, 2 = gate/up, 3 = down
  TcItem it[4][kTcMaxItems];
  int head_t0, head_t1;           // positions [t0, t1) of the lm_head tile list (filled by the kernel)
  int fold_q, fold_g;             // batch <= 4: this CTA writes the folded residual stream back (one CTA per fold point)
  int gu_split;                   // 1: gate/up items carry their own K range and write raw partial sums (flat plan)
};

struct TcPlanInfo {               // what the host needs to know about a plan
  int sq, so, sd, sg;             // K slices per phase (sg: most slices any gate/up tile has; 1 = whole K)
  int ntiles;                     // lm_head row tiles
  int max_chunks;                 // most B-operand k-blocks a CTA stages in one phase
  int gu_split;
};

struct TcParams {
  alignas(64) CUtensorMap kvmap;  // the paged KV pool as rows of 64 bf16 (box 64 x 64, SWIZZLE_128B); re-encoded when the pool moves
  // model
  int n_layers, total_layers, hidden, inter, n_heads, n_kv, qkv_n, vocab, B;
  float eps, scale_log2;
  const CUtensorMap_st* wmaps;    // device [4 * total_layers + 1]: (qkv, o, gate/up, down) per layer, lm_head; box 128 x 64
  const CUtensorMap_st* xmap;     // xa  [64 rows][hidden] bf16, box NT x 64
  const CUtensorMap_st* amap;     // act [64 rows][inter]  bf16, box NT x 64
  const TcPlan* plan;             // device [gridDim.x]
  const float* const* ln1;
  const float* const* bqkv;
  const float* const* ln2;
  const float* final_norm;
  const float* inv_freq;
  // activations
  float* h;                       // [B][hidden] residual stream (fp32): prefill hand-off, sampler output, fold phases
  __nv_bfloat16* xa;              // normalised GEMM input rows: batch <= 8: rows b = hi, 8 + b = lo (bf16 split)
  __nv_bfloat16* act;             // SwiGLU output rows, same row convention (batch > 4)
  // Hand-off buffers hold (value, stamp) pairs written with one 8-byte store: the consumer polls the data itself
  // until every pair carries the stamp of the (step, layer) it waits for -- no fence, no flag, no grid barrier.
  float2 *pq2, *po2, *pd2;        // split-K partial sums [slice][B][rows]
  int sq, so, sd;                 // slices per phase
  float2 *ao2, *aml2;             // split-KV attention partials [B][n_heads][max_splits][64] / [..][2] = ((m, .), (l, .))
  float2* act2;                   // batch <= 4, whole-K gate/up: SwiGLU output [B][inter] (fp32 value, stamp)
  float2* pg2;                    // batch <= 4, flat plan: gate/up partial sums [slice][B][2 * inter]
  const unsigned char* gu_nsl;    // flat plan: K slices of every gate/up tile (device, [tiles])
  float2* h2;                     // batch <= 4: residual stream, ping-pong [2][B][hidden]
  int stamp_base, hstamp_base;    // stamps of this launch lie above these (host counters)
  int max_splits, split_cap;
  KVLayout kv;
  float* logits;                  // [B][vocab]
  float* tmax;                    // [B][ntiles] processed maximum of every 128-row lm_head tile
  int ntiles;
  // lm_head tile list, head_n tiles spread evenly over the CTAs: tile head_eos at position head_eos_at, the others
  // head_lo, head_lo + 1, ... in order.  Vocabulary range off: head_n = ntiles, head_lo = 0, head_eos_at = -1 (every
  // tile).  Range on: the range's tiles, plus the EOS tile when it lies outside them (only EOS is allowed there).
  int head_n, head_lo, head_eos, head_eos_at;
  SamplerParams samp;
  unsigned* gbar;
  int n_steps;
  float* logits_out;
  long long logits_step_stride;
  long long* prof;
  int prof_step;
  // shared-memory plan
  int nstages;
  unsigned uni_off, uni_bytes, misc_off, acc_off;
  int att_warps;                  // page-walking warps of the attention phase (2 | 4)
  unsigned att_off;               // attention staging: inside the union region (aliased) or behind it (batch <= 4: pages prefetched)
  int fold_in_cta;                // 1: batch <= 4, consumers fold the split-K slices themselves (no fold phases)
  int weights_evict_first;        // 1: weight tiles are fetched with the L2 evict_first policy
};

struct TcShape {  // everything the planner needs
  int hidden, inter, n_heads, n_kv, qkv_n, vocab;
};
// Returns NT_OK and fills plan[G] (+ gu_nsl[tiles of gate/up] for the flat plan) and info; NT_ERR_INVALID when the
// shape does not fit the kernel.  flat: gate/up is cut into equal (tile, k-block) ranges over ALL CTAs and its
// SwiGLU moves into the down_proj staging (batch <= 4 only: larger batches hand the activations over by TMA).
int tc_build_plan(const TcShape& s, int G, bool flat, TcPlan* plan, unsigned char* gu_nsl, TcPlanInfo* info);
bool tc_fold_in_cta(int B, int hidden);
int launch_decode_tc(TcParams& P, int B, int num_sms, const TcPlanInfo& info, cudaStream_t stream);

}  // namespace nt
