// C-ABI orchestration of the speech-LM path: prefill (tensor-core GEMMs), decode steps
// (PDL-chained streaming kernels replayed from a CUDA graph), fused sampler.
// Replaces the loop at transformers generation/utils.py:2743-2805 as reached from
// neutts/neutts.py:338-347; nothing here synchronises with the host between steps
// (the reference syncs every step at utils.py:2805).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include <cuda.h>

#include "lm_decode_tc.cuh"
#include "lm_kernels.cuh"

namespace nt {

std::atomic<uint64_t> g_launches{0};
static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// Function attributes are per device context: a process that runs engines on two GPUs (backbone on cuda:0, codec on
// cuda:1) must set them on both.  One table keyed by (kernel, device ordinal) serves the carve-out preference and the
// dynamic shared-memory limit of every launch that goes through launch_kernel().
struct KernelAttrState {
  bool carveout = false;
  size_t dyn_smem = 0;
};
static KernelAttrState& kernel_attr_state(const void* kernel, std::unique_lock<std::mutex>& lock) {
  static std::mutex mu;
  static std::vector<std::pair<std::pair<const void*, int>, KernelAttrState>> table;
  lock = std::unique_lock<std::mutex>(mu);
  int dev = 0;
  cudaGetDevice(&dev);
  for (auto& e : table)
    if (e.first.first == kernel && e.first.second == dev) return e.second;
  table.push_back({{kernel, dev}, KernelAttrState()});
  return table.back().second;
}
void prefer_max_smem_carveout(const void* kernel) {
  std::unique_lock<std::mutex> lock;
  KernelAttrState& st = kernel_attr_state(kernel, lock);
  if (st.carveout) return;
  st.carveout = true;
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
int ensure_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return NT_OK;
  std::unique_lock<std::mutex> lock;
  KernelAttrState& st = kernel_attr_state(kernel, lock);
  if (st.dyn_smem >= bytes) return NT_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
  if (e != cudaSuccess) return set_error(NT_ERR_CUDA, "cudaFuncSetAttribute(%zu B of dynamic shared memory) failed: %s", bytes, cudaGetErrorString(e));
  st.dyn_smem = bytes;
  return NT_OK;
}

// launch-latency probe: a chain of dependent trivial kernels
__global__ void noop_chain_kernel(int* p) {
  pdl_launch_dependents();
  pdl_wait();
  if (p && threadIdx.x == 0 && blockIdx.x == 0) p[0] += 1;
}

}  // namespace nt

using namespace nt;

struct nt_lm {
  nt_lm_config cfg;
  int qkv_n, num_sms, max_splits, nchunks, max_rows;
  const __nv_bfloat16* embed;
  const __nv_bfloat16* lm_head;
  const float* final_norm;
  std::vector<const float*> ln1, bqkv, ln2;
  std::vector<const __nv_bfloat16*> wqkv, wo, wgu, wd;
  // workspace
  float *h, *q, *attn, *act, *logits, *cand_val, *inv_freq, *qkv, *h_last, *splitk_ws;
  size_t splitk_floats;
  int *cand_idx, *tok_seq, *tok_pos, *cu_dev, *last_rows, *iota;
  __nv_bfloat16 *xn, *attn_bf16, *act_bf16;
  // persistent decode kernel tables (device)
  const float** ptr_tab;   // [3][n_layers]: ln1, bqkv, ln2
  unsigned* gbar;          // grid barrier counters
  // cached decode-step graph
  cudaGraphExec_t graph = nullptr;
  std::vector<uint8_t> graph_key;
  cudaStream_t cap_stream = nullptr;  // capture happens here (torch's default stream is the legacy
                                      // stream, which cannot be captured); replay on the caller's stream
  uint64_t graph_kernels = 0;         // kernel nodes in the captured step (for nt_launch_count)
  bool prefilled = false;
  int debug_layers = -1;              // >= 0: run only this many layers (per-stage parity tests)
  long long* prof = nullptr;          // persistent decode kernel timeline buffer
  int prof_step = 0;
  // sampler window capture (nt_lm_debug_capture_sampler): copied into every SamplerParams, nullptr = off
  float* dbg_topk_val = nullptr;
  int32_t *dbg_topk_idx = nullptr, *dbg_token = nullptr;
  // persistent wgmma decode kernel (lm_decode_tc.cu): plan, tensor maps and buffers live in the workspace
  bool tc_ok = false, tc_flat_ok = false;
  TcPlanInfo tc_info[2] = {};         // [0]: whole-K gate/up plan (any batch), [1]: flat plan (batch <= 4)
  int tc_rows = 0;
  unsigned char* tc_gu_nsl = nullptr; // flat plan: K slices per gate/up tile
  uint8_t* tc_maps = nullptr;         // CUtensorMap[4 * n_layers + 1] weights, then xa x {16,32,64}, act x {16,32,64}
  TcPlan* tc_plan = nullptr;
  __nv_bfloat16 *tc_xa = nullptr, *tc_act = nullptr;
  float *tc_tmax = nullptr;
  float2 *tc_pq2 = nullptr, *tc_po2 = nullptr, *tc_pd2 = nullptr, *tc_ao2 = nullptr, *tc_aml2 = nullptr, *tc_act2 = nullptr, *tc_pg2 = nullptr,
         *tc_h2 = nullptr;
  size_t tc_pair_bytes = 0;           // extent of the stamped buffers (contiguous, starting at tc_pq2)
  int tc_stamp = 0, tc_hstamp = 0;    // stamps handed out so far (see TcParams::stamp_base)
  // prefill into chosen slots (nt_lm_prefill_slots)
  int* slot_key = nullptr;            // [max_batch] Philox stream key per slot, -1: slot + slot_base
  int* slot_args = nullptr;           // [3][max_batch] slots, stream keys, prompt lengths of the last call
  int* slot_table = nullptr;          // [max_batch][max_pages] the listed slots' page-table rows, in call order
  // per-slot sampling controls (nt_lm_set_slot_sampling): copied into every SamplerParams while on
  nt_slot_sampling* slot_sp = nullptr;  // [max_batch]
  bool slot_sp_on = false;
  // vocabulary range (nt_lm_set_vocab_range): allowed ids [vr_lo, vr_hi) + EOS while vr_on
  bool vr_on = false;
  int vr_lo = 0, vr_hi = 0;
};

// The lm_head tiles a launch computes under the vocabulary range: [t_lo, t_hi), plus eos_tile when EOS lies outside
// them (eos_tile = -1 otherwise).  off: every tile.
struct VocabTiles {
  bool on;
  int t_lo, t_hi, eos_tile;
  int count() const { return t_hi - t_lo + (eos_tile >= 0 ? 1 : 0); }
};
static VocabTiles vocab_tiles(const nt_lm* lm, int eos) {
  VocabTiles v;
  v.on = lm->vr_on;
  v.t_lo = lm->vr_on ? lm->vr_lo / 128 : 0;
  v.t_hi = ((lm->vr_on ? lm->vr_hi : lm->cfg.vocab_size) + 127) / 128;
  const int et = eos / 128;
  v.eos_tile = (lm->vr_on && (et < v.t_lo || et >= v.t_hi)) ? et : -1;
  return v;
}

// Every launch under the range first sets its logits rows [0, B) and their tile maxima to -inf; the lm_head then
// writes only the tiles it computes, so each suppressed id reads -inf on every sampler path.
static int vocab_fill(nt_lm* lm, int B, cudaStream_t stream) {
  if (!lm->vr_on) return NT_OK;
  const int V = lm->cfg.vocab_size, nt = (V + 127) / 128;
  int rc = launch_fill_neg_inf(lm->logits, static_cast<long long>(B) * V, stream);
  if (!rc && lm->tc_tmax) rc = launch_fill_neg_inf(lm->tc_tmax, static_cast<long long>(B < lm->tc_rows ? B : lm->tc_rows) * nt, stream);
  return rc;
}

template <typename F>
static size_t lm_carve(const nt_lm_config& c, void* ws, size_t bytes, F&& assign) {
  Arena a(ws, bytes);
  const int H = c.hidden, I = c.inter, V = c.vocab_size;
  const int qkv_n = (c.n_heads + 2 * c.n_kv_heads) * 64;
  const int rows = c.max_prefill_tokens > c.max_batch ? c.max_prefill_tokens : c.max_batch;
  const int max_splits = c.max_ctx / c.page_size;
  assign(a, H, I, V, qkv_n, rows, max_splits);
  return a.off;
}

#define LM_CARVE_BODY(L)                                                                       \
  [&](Arena& a, int H, int I, int V, int qkv_n, int rows, int max_splits) {                    \
    (L)->h = a.take<float>(size_t(rows) * H);                                                  \
    (L)->q = a.take<float>(size_t(rows) * c.n_heads * 64);                                     \
    (L)->attn = a.take<float>(size_t(c.max_batch) * c.n_heads * 64);                           \
    (L)->act = a.take<float>(size_t(c.max_batch) * I);                                         \
    (L)->logits = a.take<float>(size_t(c.max_batch) * V);                                      \
    (L)->cand_val = a.take<float>(sampler_scratch_floats(c.max_batch, V));                     \
    (L)->cand_idx = a.take<int>(sampler_scratch_floats(c.max_batch, V));                       \
    (L)->inv_freq = a.take<float>(64);                                                         \
    (L)->qkv = a.take<float>(size_t(rows) * qkv_n);                                            \
    (L)->h_last = a.take<float>(size_t(c.max_batch) * H);                                      \
    (L)->tok_seq = a.take<int>(rows);                                                          \
    (L)->tok_pos = a.take<int>(rows);                                                          \
    (L)->cu_dev = a.take<int>(c.max_batch + 1);                                                \
    (L)->last_rows = a.take<int>(c.max_batch);                                                 \
    (L)->iota = a.take<int>(c.max_batch);                                                      \
    (L)->xn = a.take<__nv_bfloat16>(size_t(rows) * H);                                         \
    (L)->attn_bf16 = a.take<__nv_bfloat16>(size_t(rows) * c.n_heads * 64);                     \
    (L)->act_bf16 = a.take<__nv_bfloat16>(size_t(rows) * I);                                   \
    (L)->ptr_tab = a.take<const float*>(size_t(3) * c.n_layers);                               \
    (L)->gbar = a.take<unsigned>(64);                                                          \
    (L)->splitk_floats = size_t(8) * 128 * (qkv_n > H ? qkv_n : H);                            \
    (L)->splitk_ws = a.take<float>(size_t(8) * 128 * (qkv_n > H ? qkv_n : H));                 \
    (L)->tc_rows = c.max_batch < kTcMaxBatch ? c.max_batch : kTcMaxBatch;                      \
    (L)->tc_maps = a.take<uint8_t>(size_t(128) * (size_t(4) * c.n_layers + 1 + 6));            \
    (L)->tc_plan = a.take<TcPlan>(512);                                                        \
    (L)->tc_gu_nsl = a.take<unsigned char>(4096);                                              \
    (L)->tc_xa = a.take<__nv_bfloat16>(size_t(kTcMaxBatch) * H);                               \
    (L)->tc_act = a.take<__nv_bfloat16>(size_t(kTcMaxBatch) * I);                              \
    (L)->tc_tmax = a.take<float>(size_t((L)->tc_rows) * ((V + 127) / 128));                    \
    (L)->tc_pq2 = a.take<float2>(size_t(kTcMaxSlices) * (L)->tc_rows * qkv_n);                 \
    (L)->tc_po2 = a.take<float2>(size_t(kTcMaxSlices) * (L)->tc_rows * H);                     \
    (L)->tc_pd2 = a.take<float2>(size_t(kTcMaxSlices) * (L)->tc_rows * H);                     \
    (L)->tc_ao2 = a.take<float2>(size_t((L)->tc_rows) * c.n_heads * max_splits * 64);          \
    (L)->tc_aml2 = a.take<float2>(size_t((L)->tc_rows) * c.n_heads * max_splits * 2);          \
    (L)->tc_act2 = a.take<float2>(size_t(4) * I);                                              \
    (L)->tc_pg2 = a.take<float2>(size_t(kTcMaxGuSlices) * 4 * 2 * I);                          \
    (L)->tc_h2 = a.take<float2>(size_t(2) * 4 * H);                                            \
    (L)->tc_pair_bytes = size_t(reinterpret_cast<uint8_t*>((L)->tc_h2 + size_t(2) * 4 * H) - reinterpret_cast<uint8_t*>((L)->tc_pq2)); \
    (L)->slot_key = a.take<int>(c.max_batch);                                                  \
    (L)->slot_args = a.take<int>(size_t(3) * c.max_batch);                                     \
    (L)->slot_table = a.take<int>(size_t(c.max_batch) * max_splits);                           \
    (L)->slot_sp = a.take<nt_slot_sampling>(c.max_batch);                                     \
  }

static int lm_check_config(const nt_lm_config* c) {
  if (!c) return set_error(NT_ERR_INVALID, "null config");
  if (c->head_dim != 64) return set_error(NT_ERR_INVALID, "head_dim %d unsupported (64 only)", c->head_dim);
  if (c->page_size != 64) return set_error(NT_ERR_INVALID, "page_size %d unsupported (64 only)", c->page_size);
  if (c->hidden % 64 || c->inter % 64) return set_error(NT_ERR_INVALID, "hidden/inter must be multiples of 64");
  if (c->n_heads % c->n_kv_heads || c->n_heads / c->n_kv_heads > 8)
    return set_error(NT_ERR_INVALID, "unsupported GQA ratio %d/%d", c->n_heads, c->n_kv_heads);
  if (c->vocab_size & 1) return set_error(NT_ERR_INVALID, "vocab_size must be even");
  if (c->max_ctx % 64 || c->max_ctx <= 0) return set_error(NT_ERR_INVALID, "max_ctx must be a positive multiple of 64");
  if (c->max_batch < 1 || c->max_prefill_tokens < 1 || c->num_pages < 1) return set_error(NT_ERR_INVALID, "bad sizes");
  return NT_OK;
}

extern "C" const char* nt_last_error(void) { return g_err; }
extern "C" int nt_abi_version(void) { return 3; }
extern "C" uint64_t nt_launch_count(void) { return g_launches.load(); }

extern "C" size_t nt_lm_workspace_bytes(const nt_lm_config* cfg) {
  if (lm_check_config(cfg)) return 0;
  const nt_lm_config& c = *cfg;
  nt_lm dummy;
  return lm_carve(c, nullptr, 0, LM_CARVE_BODY(&dummy)) + 256;
}

extern "C" int nt_lm_create(const nt_lm_config* cfg, const nt_lm_weights* w, void* workspace, size_t workspace_bytes,
                            nt_lm** out) {
  int rc = lm_check_config(cfg);
  if (rc) return rc;
  if (!w || !workspace || !out) return set_error(NT_ERR_INVALID, "nt_lm_create: null argument");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return set_error(NT_ERR_INVALID, "workspace must be 256-byte aligned");
  const nt_lm_config& c = *cfg;
  nt_lm* lm = new nt_lm();
  lm->cfg = c;
  const size_t need = lm_carve(c, workspace, workspace_bytes, LM_CARVE_BODY(lm));
  if (need > workspace_bytes) {
    delete lm;
    return set_error(NT_ERR_NOMEM, "workspace too small: need %zu, got %zu", need, workspace_bytes);
  }
  lm->qkv_n = (c.n_heads + 2 * c.n_kv_heads) * 64;
  lm->max_splits = c.max_ctx / c.page_size;
  lm->nchunks = sampler_nchunks(c.vocab_size);
  lm->max_rows = c.max_prefill_tokens > c.max_batch ? c.max_prefill_tokens : c.max_batch;
  lm->embed = static_cast<const __nv_bfloat16*>(w->embed);
  lm->lm_head = static_cast<const __nv_bfloat16*>(w->lm_head);
  lm->final_norm = w->final_norm;
  for (int l = 0; l < c.n_layers; ++l) {
    lm->ln1.push_back(w->ln1[l]);
    lm->bqkv.push_back(w->bqkv[l]);
    lm->ln2.push_back(w->ln2[l]);
    lm->wqkv.push_back(static_cast<const __nv_bfloat16*>(w->wqkv[l]));
    lm->wo.push_back(static_cast<const __nv_bfloat16*>(w->wo[l]));
    lm->wgu.push_back(static_cast<const __nv_bfloat16*>(w->wgu[l]));
    lm->wd.push_back(static_cast<const __nv_bfloat16*>(w->wd[l]));
  }
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    delete lm;
    return set_error(NT_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  }
  if (prop.major != 9 || prop.minor != 0) {
    delete lm;
    return set_error(NT_ERR_CUDA, "device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
  }
  lm->num_sms = prop.multiProcessorCount;
  // rotary inverse frequencies (modeling_qwen2.py:95-100), iota, per-layer norm / bias pointers
  float invf[64] = {0};
  for (int i = 0; i < 32; ++i) invf[i] = static_cast<float>(1.0 / std::pow(static_cast<double>(c.rope_theta), (2.0 * i) / 64.0));
  std::vector<int> iota(c.max_batch);
  for (int i = 0; i < c.max_batch; ++i) iota[i] = i;
  std::vector<const float*> pt(size_t(3) * c.n_layers);
  for (int l = 0; l < c.n_layers; ++l) {
    pt[l] = lm->ln1[l];
    pt[c.n_layers + l] = lm->bqkv[l];
    pt[2 * c.n_layers + l] = lm->ln2[l];
  }
  if (cudaMemcpy(lm->inv_freq, invf, sizeof(invf), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(lm->iota, iota.data(), iota.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(lm->ptr_tab, pt.data(), pt.size() * sizeof(const float*), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(lm->slot_key, 0xff, size_t(c.max_batch) * sizeof(int)) != cudaSuccess) {
    delete lm;
    return set_error(NT_ERR_CUDA, "workspace initialisation failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  {
    // persistent wgmma decode kernel: work plan + every tensor map, built once (re-encoding the maps on every GEMM
    // call costs host time on each step).  A shape the plan cannot take leaves tc_ok false -> the per-op chain.
    std::vector<TcPlan> plan(512);
    std::vector<unsigned char> nsl(4096, 0);
    TcShape ts{c.hidden, c.inter, c.n_heads, c.n_kv_heads, lm->qkv_n, c.vocab_size};
    const int G = lm->num_sms > 256 ? 256 : lm->num_sms;
    lm->tc_flat_ok = (2 * c.inter + 127) / 128 <= 4096 &&
                     tc_build_plan(ts, G, true, plan.data() + 256, nsl.data(), &lm->tc_info[1]) == NT_OK;
    if (tc_build_plan(ts, G, false, plan.data(), nullptr, &lm->tc_info[0]) == NT_OK) {
      const size_t nmaps = size_t(4) * c.n_layers + 1 + 6;
      std::vector<CUtensorMap> maps(nmaps);
      const int HD = c.n_heads * 64;
      int mrc = NT_OK;
      for (int l = 0; l < c.n_layers && !mrc; ++l) {
        mrc = make_tmap(&maps[4 * l + 0], NT_BF16, lm->wqkv[l], lm->qkv_n, c.hidden, c.hidden, 128);
        if (!mrc) mrc = make_tmap(&maps[4 * l + 1], NT_BF16, lm->wo[l], c.hidden, HD, HD, 128);
        if (!mrc) mrc = make_tmap(&maps[4 * l + 2], NT_BF16, lm->wgu[l], 2 * c.inter, c.hidden, c.hidden, 128);
        if (!mrc) mrc = make_tmap(&maps[4 * l + 3], NT_BF16, lm->wd[l], c.hidden, c.inter, c.inter, 128);
      }
      if (!mrc) mrc = make_tmap(&maps[4 * c.n_layers], NT_BF16, lm->lm_head, c.vocab_size, c.hidden, c.hidden, 128);
      const int nts[3] = {16, 32, 64};
      for (int i = 0; i < 3 && !mrc; ++i) {
        mrc = make_tmap(&maps[4 * c.n_layers + 1 + i], NT_BF16, lm->tc_xa, kTcMaxBatch, c.hidden, c.hidden, nts[i]);
        if (!mrc) mrc = make_tmap(&maps[4 * c.n_layers + 4 + i], NT_BF16, lm->tc_act, kTcMaxBatch, c.inter, c.inter, nts[i]);
      }
      static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap size");
      if (!mrc && cudaMemcpy(lm->tc_maps, maps.data(), nmaps * sizeof(CUtensorMap), cudaMemcpyHostToDevice) == cudaSuccess &&
          cudaMemcpy(lm->tc_plan, plan.data(), 512 * sizeof(TcPlan), cudaMemcpyHostToDevice) == cudaSuccess &&
          cudaMemcpy(lm->tc_gu_nsl, nsl.data(), nsl.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
          cudaMemset(lm->tc_xa, 0, size_t(kTcMaxBatch) * c.hidden * 2) == cudaSuccess &&
          cudaMemset(lm->tc_act, 0, size_t(kTcMaxBatch) * c.inter * 2) == cudaSuccess &&
          cudaMemset(lm->tc_pq2, 0, lm->tc_pair_bytes) == cudaSuccess)   // stamp 0 = "never written"
        lm->tc_ok = true;
    }
  }
  if (cudaStreamCreateWithFlags(&lm->cap_stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete lm;
    return set_error(NT_ERR_CUDA, "stream creation failed");
  }
  *out = lm;
  return NT_OK;
}

extern "C" int nt_lm_destroy(nt_lm* lm) {
  if (!lm) return NT_OK;
  if (lm->graph) cudaGraphExecDestroy(lm->graph);
  if (lm->cap_stream) cudaStreamDestroy(lm->cap_stream);
  delete lm;
  return NT_OK;
}

static KVLayout make_kv(const nt_lm* lm, const nt_lm_state* st) {
  const nt_lm_config& c = lm->cfg;
  KVLayout kv;
  kv.pages = static_cast<__nv_bfloat16*>(st->kv_pages);
  kv.page_table = st->page_table;
  kv.seq_lens = st->seq_lens;
  kv.n_kv_heads = c.n_kv_heads;
  kv.num_pages = c.num_pages;
  kv.max_pages_per_seq = c.max_ctx / c.page_size;
  kv.max_ctx = c.max_ctx;
  kv.kv_stride = static_cast<long long>(c.num_pages) * c.n_kv_heads * 64 * 64;
  kv.layer_stride = 2 * kv.kv_stride;
  return kv;
}

static SamplerParams make_sampler(const nt_lm* lm, const nt_lm_state* st, const nt_sampling* sp) {
  SamplerParams s;
  memset(&s, 0, sizeof(s));
  s.logits = lm->logits;
  s.V = lm->cfg.vocab_size;
  s.sp = *sp;
  s.seq_lens = st->seq_lens;
  s.cur_token = st->cur_token;
  s.out_tokens = st->out_tokens;
  s.n_generated = st->n_generated;
  s.done = st->done;
  s.max_new = st->max_new;
  s.max_ctx = lm->cfg.max_ctx;
  s.cand_val = lm->cand_val;
  s.cand_idx = lm->cand_idx;
  s.nchunks = lm->nchunks;
  s.embed = lm->embed;
  s.h = lm->h;
  s.hidden = lm->cfg.hidden;
  s.slot_base = sp->slot_base;
  s.slot_key = lm->slot_key;
  s.slot_sp = lm->slot_sp_on ? lm->slot_sp : nullptr;
  s.dbg_topk_val = lm->dbg_topk_val, s.dbg_topk_idx = lm->dbg_topk_idx, s.dbg_token = lm->dbg_token;
  return s;
}

static int check_sampling(const nt_lm* lm, const nt_lm_state* st, const nt_sampling* sp) {
  if (!sp) return set_error(NT_ERR_INVALID, "null sampling params");
  if (sp->eos_id < 0 || sp->eos_id >= lm->cfg.vocab_size) return set_error(NT_ERR_INVALID, "eos_id out of range");
  if (sp->max_new_tokens < 1 || sp->max_new_tokens > st->max_new)
    return set_error(NT_ERR_INVALID, "max_new_tokens %d not in 1..%d", sp->max_new_tokens, st->max_new);
  return NT_OK;
}

// lm_head on B hidden rows (fp32, un-normalised) -> lm->logits / `logits`
// tile-max sampler after the tensor-core lm_head (batch > 4): the GEMM must tile the vocabulary by 128 columns
static bool use_tile_sampler(const nt_lm* lm, int B) {
  return B > kGemvMaxBatch && B <= lm->tc_rows && lm->tc_tmax && gemm_tile_n(B, lm->cfg.vocab_size, false) == 128;
}
static int run_sampler(nt_lm* lm, const SamplerParams& s, int B, cudaStream_t stream) {
  if (use_tile_sampler(lm, B)) return launch_sampler_tiles(s, B, lm->tc_tmax, (lm->cfg.vocab_size + 127) / 128, stream);
  return launch_sampler(s, B, stream);
}

// eos >= 0: apply the vocabulary range with this EOS id (every sampler launch); -1: every row (nt_lm_head_gemv).  Under
// the range the lm_head runs once over the range's rows and once over the EOS tile (when EOS lies outside them), each
// a row slice of the full-vocabulary launch with the same per-row arithmetic, so every computed logit is bit-identical
// to the range off; the rows it does not compute keep the -inf of vocab_fill.
static int lm_head_rows(nt_lm* lm, const float* hrows, int B, float* logits, cudaStream_t stream, const SplitK* pend = nullptr,
                        int eos = -1) {
  const nt_lm_config& c = lm->cfg;
  const int V = c.vocab_size, nt = (V + 127) / 128;
  const VocabTiles vt = eos >= 0 ? vocab_tiles(lm, eos) : VocabTiles{false, 0, nt, -1};
  // row slices [r0, r1): the range (or everything), then the EOS tile
  const int r0[2] = {vt.t_lo * 128, vt.eos_tile * 128};
  const int r1[2] = {vt.t_hi * 128 < V ? vt.t_hi * 128 : V, (vt.eos_tile + 1) * 128 < V ? (vt.eos_tile + 1) * 128 : V};
  const int nslices = vt.eos_tile >= 0 ? 2 : 1;
  int rc;
  if (B <= kGemvMaxBatch) {
    for (int i = 0; i < nslices; ++i) {
      GemvParams g;
      memset(&g, 0, sizeof(g));
      g.W = lm->lm_head + static_cast<long long>(r0[i]) * c.hidden, g.rows = r1[i] - r0[i], g.K = c.hidden;
      g.x = hrows, g.ldx = c.hidden;
      g.norm_w = lm->final_norm, g.eps = c.rms_eps;
      g.epi = GEMV_STORE, g.out = logits + r0[i], g.ldo = V;
      if ((rc = launch_gemv(g, B, lm->num_sms, stream))) return rc;
    }
    return vt.eos_tile >= 0 ? launch_vocab_eos_tile(logits, B, V, eos, nullptr, nt, stream) : NT_OK;
  }
  // pend: the last down_proj left split-K slices that still have to be folded into hrows (batched decode only)
  const bool fold = pend && pend->used > 1;
  rc = launch_rmsnorm_rows(hrows, lm->final_norm, c.rms_eps, B, c.hidden, nullptr, lm->xn, stream, fold ? pend->ws : nullptr,
                               fold ? pend->used : 0, fold ? pend->slice_stride : 0);
  if (rc) return rc;
  float* tmax = (use_tile_sampler(lm, B) && logits == lm->logits) ? lm->tc_tmax : nullptr;
  if (!vt.on) {
    nt_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = B, a.N = V, a.K = c.hidden;
    a.A = lm->xn, a.lda = c.hidden, a.W = lm->lm_head, a.ldw = c.hidden;
    a.out_f32 = logits, a.ldc = V;
    return gemm_dispatch(a, stream, nullptr, true, nullptr, tmax);
  }
  // slices run at the full-vocabulary tile width; their tile maxima land at absolute tile indices (128-column tiles)
  const int bn = gemm_tile_n(B, V, false);
  for (int i = 0; i < nslices; ++i) {
    nt_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = B, a.N = r1[i] - r0[i], a.K = c.hidden;
    a.A = lm->xn, a.lda = c.hidden, a.W = lm->lm_head + static_cast<long long>(r0[i]) * c.hidden, a.ldw = c.hidden;
    a.out_f32 = logits + r0[i], a.ldc = V;
    if ((rc = gemm_dispatch(a, stream, nullptr, true, nullptr, tmax ? tmax + r0[i] / 128 : nullptr, bn, nt))) return rc;
  }
  return vt.eos_tile >= 0 ? launch_vocab_eos_tile(logits, B, V, eos, tmax, nt, stream) : NT_OK;
}

// Transformer layers over `rows` token rows held in lm->h, via tensor-core GEMMs.
// mode 0: prefill (causal attention over the prompt);  mode 1: one new token per sequence.
// table: page table to address the KV cache with, row b for sequence b of the call (default: the state's).
static int layers_gemm(nt_lm* lm, const nt_lm_state* st, int rows, int B, int mode, int max_len, cudaStream_t stream,
                       SplitK* tail = nullptr, const int32_t* table = nullptr) {
  const nt_lm_config& c = lm->cfg;
  KVLayout kv = make_kv(lm, st);
  if (table) kv.page_table = table;
  const int H = c.hidden, I = c.inter, QN = lm->qkv_n, HD = c.n_heads * 64;
  const float scale_log2 = (1.0f / 8.0f) * 1.4426950408889634f;
  int rc;
  const int n_layers = lm->debug_layers >= 0 ? lm->debug_layers : c.n_layers;
  // o_proj / down_proj accumulate into the residual stream; with few row tiles (batched decode, short prompts)
  // they split K over grid.z into lm->splitk_ws and the RMSNorm that follows folds the slices into lm->h.
  // The last layer's down_proj splits only when the caller takes over the fold (`tail`: decode, where the final
  // norm of lm_head_rows reads lm->h next); in prefill a row gather comes first, so it stays whole.
  SplitK pend;
  pend.ws = lm->splitk_ws, pend.ws_floats = lm->splitk_floats, pend.used = 1, pend.slice_stride = 0;
  for (int l = 0; l < n_layers; ++l) {
    if ((rc = launch_rmsnorm_rows(lm->h, lm->ln1[l], c.rms_eps, rows, H, nullptr, lm->xn, stream,
                                  pend.used > 1 ? pend.ws : nullptr, pend.used > 1 ? pend.used : 0, pend.slice_stride)))
      return rc;
    pend.used = 1;
    nt_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = rows, a.N = QN, a.K = H, a.A = lm->xn, a.lda = H, a.W = lm->wqkv[l], a.ldw = H;
    a.bias = lm->bqkv[l], a.out_f32 = lm->qkv, a.ldc = QN;
    // few row tiles: the projection splits K into slices that rope_append sums (the bias rides on slice 0)
    SplitK qsplit;
    qsplit.ws = lm->splitk_ws, qsplit.ws_floats = lm->splitk_floats, qsplit.used = 1, qsplit.slice_stride = 0;
    if ((rc = gemm_dispatch(a, stream, &qsplit, true))) return rc;
    const int32_t* tseq = mode == 0 ? lm->tok_seq : lm->iota;
    const int32_t* tpos = mode == 0 ? lm->tok_pos : st->seq_lens;
    // decode on the tensor-core attention kernel (batch > 4): RoPE + KV append run in that kernel's prologue
    const bool fuse_rope = mode == 1 && B > 4;
    if (!fuse_rope &&
        (rc = launch_rope_append(qsplit.used > 1 ? qsplit.ws : lm->qkv, rows, QN, tseq, tpos, c.n_heads, lm->inv_freq, lm->q, kv, l, stream,
                                 qsplit.used, qsplit.slice_stride)))
      return rc;
    if (mode == 0) {
      AttnPrefillParams ap;
      ap.q = lm->q, ap.kv = kv, ap.layer = l, ap.n_heads = c.n_heads, ap.n_rep = c.n_heads / c.n_kv_heads;
      ap.scale_log2 = scale_log2, ap.cu_seqlens = lm->cu_dev, ap.out = lm->attn_bf16, ap.max_len = max_len;
      if ((rc = launch_attn_prefill(ap, B, c.n_layers, stream))) return rc;
    } else {
      AttnDecParams ad;
      memset(&ad, 0, sizeof(ad));
      ad.q = lm->q, ad.kv = kv, ad.layer = l, ad.n_heads = c.n_heads, ad.n_rep = c.n_heads / c.n_kv_heads;
      ad.scale_log2 = scale_log2, ad.out = lm->attn, ad.out_bf16 = lm->attn_bf16;
      if (fuse_rope) {
        ad.qkv = qsplit.used > 1 ? qsplit.ws : lm->qkv, ad.qkv_n = QN, ad.qkv_parts = qsplit.used;
        ad.qkv_pstride = qsplit.slice_stride, ad.inv_freq = lm->inv_freq;
      }
      if ((rc = launch_attn_decode(ad, B, c.n_layers, stream))) return rc;
    }
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = rows, a.N = H, a.K = HD, a.A = lm->attn_bf16, a.lda = HD, a.W = lm->wo[l], a.ldw = HD;
    a.residual = lm->h, a.ldr = H, a.out_f32 = lm->h, a.ldc = H;
    if ((rc = gemm_dispatch(a, stream, &pend, true))) return rc;
    if ((rc = launch_rmsnorm_rows(lm->h, lm->ln2[l], c.rms_eps, rows, H, nullptr, lm->xn, stream,
                                  pend.used > 1 ? pend.ws : nullptr, pend.used > 1 ? pend.used : 0, pend.slice_stride)))
      return rc;
    pend.used = 1;
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = rows, a.N = 2 * I, a.K = H, a.A = lm->xn, a.lda = H, a.W = lm->wgu[l], a.ldw = H;
    a.act = NT_ACT_SWIGLU, a.out_bf16 = lm->act_bf16, a.ldc = I;
    if ((rc = gemm_dispatch(a, stream, nullptr, true))) return rc;
    memset(&a, 0, sizeof(a));
    a.dtype = NT_BF16, a.M = rows, a.N = H, a.K = I, a.A = lm->act_bf16, a.lda = I, a.W = lm->wd[l], a.ldw = I;
    a.residual = lm->h, a.ldr = H, a.out_f32 = lm->h, a.ldc = H;
    if ((rc = gemm_dispatch(a, stream, (l + 1 < n_layers || tail) ? &pend : nullptr, true))) return rc;
  }
  if (tail) *tail = pend;
  return NT_OK;
}

// Checks cu_seqlens [B+1] and stages the per-token tables of a prefill: the sequence and position of every token row,
// the last row of every sequence.  lens / max_len: the prompt lengths.
static int prefill_stage(nt_lm* lm, const int32_t* cu, int B, std::vector<int>& lens, int& max_len, cudaStream_t stream) {
  const nt_lm_config& c = lm->cfg;
  const int T = cu[B];
  if (cu[0] != 0 || T < B || T > c.max_prefill_tokens)
    return set_error(NT_ERR_INVALID, "prefill tokens %d not in %d..%d", T, B, c.max_prefill_tokens);
  std::vector<int> tseq(T), tpos(T), last(B);
  lens.assign(B, 0);
  max_len = 0;
  for (int b = 0; b < B; ++b) {
    const int len = cu[b + 1] - cu[b];
    if (len < 1 || len >= c.max_ctx) return set_error(NT_ERR_INVALID, "prompt %d has length %d (must be 1..%d)", b, len, c.max_ctx - 1);
    for (int t = 0; t < len; ++t) tseq[cu[b] + t] = b, tpos[cu[b] + t] = t;
    last[b] = cu[b + 1] - 1;
    lens[b] = len;
    if (len > max_len) max_len = len;
  }
  NT_CUDA_CHECK(cudaMemcpyAsync(lm->tok_seq, tseq.data(), T * sizeof(int), cudaMemcpyHostToDevice, stream));
  NT_CUDA_CHECK(cudaMemcpyAsync(lm->tok_pos, tpos.data(), T * sizeof(int), cudaMemcpyHostToDevice, stream));
  NT_CUDA_CHECK(cudaMemcpyAsync(lm->cu_dev, cu, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
  NT_CUDA_CHECK(cudaMemcpyAsync(lm->last_rows, last.data(), B * sizeof(int), cudaMemcpyHostToDevice, stream));
  // host vectors above are pageable: the runtime stages them before returning, so they may go out of scope
  return NT_OK;
}

// Prompt rows -> KV cache + last-position logits in lm->logits (and logits_out).  table: see layers_gemm.
static int prefill_forward(nt_lm* lm, const nt_lm_state* st, const int32_t* ids, const int32_t* cu, int B, int max_len,
                           const int32_t* table, float* logits_out, int eos, cudaStream_t stream) {
  const nt_lm_config& c = lm->cfg;
  int rc;
  if ((rc = vocab_fill(lm, B, stream))) return rc;
  if ((rc = launch_embed_rows(lm->embed, ids, cu[B], c.hidden, lm->h, stream))) return rc;
  if ((rc = layers_gemm(lm, st, cu[B], B, 0, max_len, stream, nullptr, table))) return rc;
  if ((rc = launch_gather_rows(lm->h, lm->last_rows, B, c.hidden, lm->h_last, stream))) return rc;
  if ((rc = lm_head_rows(lm, lm->h_last, B, lm->logits, stream, nullptr, eos))) return rc;
  if (logits_out)
    NT_CUDA_CHECK(cudaMemcpyAsync(logits_out, lm->logits, size_t(B) * c.vocab_size * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  return NT_OK;
}

extern "C" int nt_lm_prefill(nt_lm* lm, const nt_lm_state* st, const int32_t* ids, const int32_t* cu, int B,
                             const nt_sampling* sp, float* logits_out, void* stream_) {
  if (!lm || !st || !ids || !cu) return set_error(NT_ERR_INVALID, "nt_lm_prefill: null argument");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const nt_lm_config& c = lm->cfg;
  if (B < 1 || B > c.max_batch) return set_error(NT_ERR_INVALID, "batch %d not in 1..%d", B, c.max_batch);
  int rc = check_sampling(lm, st, sp);
  if (rc) return rc;
  std::vector<int> lens;
  int max_len = 0;
  if ((rc = prefill_stage(lm, cu, B, lens, max_len, stream))) return rc;
  if ((rc = prefill_forward(lm, st, ids, cu, B, max_len, nullptr, logits_out, sp->eos_id, stream))) return rc;
  NT_CUDA_CHECK(cudaMemcpyAsync(st->seq_lens, lens.data(), B * sizeof(int), cudaMemcpyHostToDevice, stream));
  NT_CUDA_CHECK(cudaMemsetAsync(lm->slot_key, 0xff, size_t(c.max_batch) * sizeof(int), stream));  // every slot: slot + slot_base
  SamplerParams s = make_sampler(lm, st, sp);
  if ((rc = run_sampler(lm, s, B, stream))) return rc;
  lm->prefilled = true;
  return NT_OK;
}

// Prefill into the listed slots while every other slot keeps its KV pages, tokens and counters.  The prefill chain
// addresses KV by the sequence index of the call, so a small kernel first gathers the listed slots' page-table rows
// into a compact table in call order (and resets those slots' length, counters and Philox key); the chain then runs
// unchanged on that table.  The sampler maps logits row i to slot slots[i].  lm->h served as the prefill's token-row
// scratch and row s of it is slot s's next decode input, so afterwards every slot's row is re-embedded from
// cur_token: the survivors get back exactly what their last sampler step wrote there.
extern "C" int nt_lm_prefill_slots(nt_lm* lm, const nt_lm_state* st, const int32_t* slots, const int32_t* stream_ids,
                                   const int32_t* ids, const int32_t* cu, int B, const nt_sampling* sp, float* logits_out,
                                   void* stream_) {
  if (!lm || !st || !slots || !stream_ids || !ids || !cu) return set_error(NT_ERR_INVALID, "nt_lm_prefill_slots: null argument");
  if (!lm->prefilled) return set_error(NT_ERR_STATE, "nt_lm_prefill_slots called before nt_lm_prefill");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const nt_lm_config& c = lm->cfg;
  if (B < 1 || B > c.max_batch) return set_error(NT_ERR_INVALID, "batch %d not in 1..%d", B, c.max_batch);
  int rc = check_sampling(lm, st, sp);
  if (rc) return rc;
  std::vector<int> args(size_t(3) * B);
  std::vector<char> seen(c.max_batch, 0);
  for (int i = 0; i < B; ++i) {
    if (slots[i] < 0 || slots[i] >= c.max_batch || seen[slots[i]])
      return set_error(NT_ERR_INVALID, "slot %d: slots must be distinct and in 0..%d", slots[i], c.max_batch - 1);
    if (stream_ids[i] < 0) return set_error(NT_ERR_INVALID, "stream id %d must be >= 0", stream_ids[i]);
    seen[slots[i]] = 1;
    args[i] = slots[i], args[B + i] = stream_ids[i];
  }
  std::vector<int> lens;
  int max_len = 0;
  if ((rc = prefill_stage(lm, cu, B, lens, max_len, stream))) return rc;
  for (int i = 0; i < B; ++i) args[2 * B + i] = lens[i];
  NT_CUDA_CHECK(cudaMemcpyAsync(lm->slot_args, args.data(), args.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  const int max_pages = c.max_ctx / c.page_size;
  if ((rc = launch_slots_setup(lm->slot_args, B, st->page_table, max_pages, lm->slot_table, st->seq_lens, st->n_generated, st->done,
                               lm->slot_key, stream)))
    return rc;
  if ((rc = prefill_forward(lm, st, ids, cu, B, max_len, lm->slot_table, logits_out, sp->eos_id, stream))) return rc;
  SamplerParams s = make_sampler(lm, st, sp);
  s.row_slot = lm->slot_args;
  s.h = nullptr;  // the residual rows are rebuilt below, for every slot
  if ((rc = run_sampler(lm, s, B, stream))) return rc;
  return launch_embed_rows(lm->embed, st->cur_token, c.max_batch, c.hidden, lm->h, stream);
}

// one decode step for slots 0..B-1 (all launches asynchronous, PDL-chained)
static int decode_step(nt_lm* lm, const nt_lm_state* st, int B, const nt_sampling* sp, cudaStream_t stream) {
  const nt_lm_config& c = lm->cfg;
  int rc;
  SplitK tail;
  tail.ws = nullptr, tail.ws_floats = 0, tail.used = 1, tail.slice_stride = 0;
  if (B <= kGemvMaxBatch) {
    const KVLayout kv = make_kv(lm, st);
    const int H = c.hidden, I = c.inter, HD = c.n_heads * 64;
    const float scale_log2 = (1.0f / 8.0f) * 1.4426950408889634f;
    const int n_layers = lm->debug_layers >= 0 ? lm->debug_layers : c.n_layers;
    for (int l = 0; l < n_layers; ++l) {
      GemvParams g;
      memset(&g, 0, sizeof(g));
      g.W = lm->wqkv[l], g.rows = lm->qkv_n, g.K = H, g.x = lm->h, g.ldx = H;
      g.norm_w = lm->ln1[l], g.eps = c.rms_eps, g.bias = lm->bqkv[l];
      g.epi = GEMV_QKV_ROPE, g.q_out = lm->q, g.kv = kv, g.layer = l, g.n_heads = c.n_heads, g.inv_freq = lm->inv_freq;
      if ((rc = launch_gemv(g, B, lm->num_sms, stream))) return rc;

      AttnDecParams ad;
      memset(&ad, 0, sizeof(ad));
      ad.q = lm->q, ad.kv = kv, ad.layer = l, ad.n_heads = c.n_heads, ad.n_rep = c.n_heads / c.n_kv_heads;
      ad.scale_log2 = scale_log2, ad.out = lm->attn, ad.out_bf16 = nullptr;
      if ((rc = launch_attn_decode(ad, B, c.n_layers, stream))) return rc;

      memset(&g, 0, sizeof(g));
      g.W = lm->wo[l], g.rows = H, g.K = HD, g.x = lm->attn, g.ldx = HD;
      g.epi = GEMV_STORE, g.out = lm->h, g.ldo = H, g.residual = lm->h, g.ldr = H;
      if ((rc = launch_gemv(g, B, lm->num_sms, stream))) return rc;

      memset(&g, 0, sizeof(g));
      g.W = lm->wgu[l], g.rows = 2 * I, g.K = H, g.x = lm->h, g.ldx = H;
      g.norm_w = lm->ln2[l], g.eps = c.rms_eps;
      g.epi = GEMV_SWIGLU, g.out = lm->act, g.ldo = I;
      if ((rc = launch_gemv(g, B, lm->num_sms, stream))) return rc;

      memset(&g, 0, sizeof(g));
      g.W = lm->wd[l], g.rows = H, g.K = I, g.x = lm->act, g.ldx = I;
      g.epi = GEMV_STORE, g.out = lm->h, g.ldo = H, g.residual = lm->h, g.ldr = H;
      if ((rc = launch_gemv(g, B, lm->num_sms, stream))) return rc;
    }
  } else {
    if ((rc = layers_gemm(lm, st, B, B, 1, 0, stream, &tail))) return rc;
  }
  if ((rc = lm_head_rows(lm, lm->h, B, lm->logits, stream, &tail, sp->eos_id))) return rc;
  SamplerParams s = make_sampler(lm, st, sp);
  s.advance = 1;
  return run_sampler(lm, s, B, stream);
}

extern "C" int nt_lm_decode(nt_lm* lm, const nt_lm_state* st, int B, int n_steps, const nt_sampling* sp,
                            float* logits_out, void* stream_) {
  if (!lm || !st) return set_error(NT_ERR_INVALID, "nt_lm_decode: null argument");
  if (!lm->prefilled) return set_error(NT_ERR_STATE, "nt_lm_decode called before nt_lm_prefill");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const nt_lm_config& c = lm->cfg;
  if (B < 1 || B > c.max_batch) return set_error(NT_ERR_INVALID, "batch %d not in 1..%d", B, c.max_batch);
  int rc = check_sampling(lm, st, sp);
  if (rc) return rc;
  if (n_steps < 0) return set_error(NT_ERR_INVALID, "negative step count");

  // NT_DECODE_IMPL = tc (persistent wgmma kernel) | perop (per-op kernel chain).  Unset: the persistent kernel up to
  // kTcDefaultMaxBatch sequences; its step time grows with the batch while the chain's is nearly flat, so the chain
  // takes the larger batches.  The chain also serves every shape the persistent kernel's plan does not take.
  const char* impl = getenv("NT_DECODE_IMPL");
  bool want_tc = B <= kTcDefaultMaxBatch;
  if (impl && impl[0]) {
    if (strcmp(impl, "tc") && strcmp(impl, "perop"))
      return set_error(NT_ERR_INVALID, "NT_DECODE_IMPL=%s: valid values are tc and perop", impl);
    want_tc = impl[0] == 't';
  }
  if (n_steps == 0) return NT_OK;
  if ((rc = vocab_fill(lm, B, stream))) return rc;   // once per launch: no step writes a suppressed row or tile maximum
  const int tc_layers = lm->debug_layers >= 0 ? lm->debug_layers : c.n_layers;
  if (want_tc && lm->tc_ok && B <= lm->tc_rows && B * c.n_kv_heads <= lm->num_sms) {
    TcParams P;
    memset(&P, 0, sizeof(P));
    P.n_layers = tc_layers, P.total_layers = c.n_layers;
    P.hidden = c.hidden, P.inter = c.inter, P.n_heads = c.n_heads, P.n_kv = c.n_kv_heads, P.qkv_n = lm->qkv_n, P.vocab = c.vocab_size;
    P.eps = c.rms_eps, P.scale_log2 = (1.0f / 8.0f) * 1.4426950408889634f;
    const CUtensorMap* maps = reinterpret_cast<const CUtensorMap*>(lm->tc_maps);
    const int nti = B <= 16 ? 0 : (B <= 32 ? 1 : 2);
    P.wmaps = maps, P.xmap = maps + 4 * c.n_layers + 1 + nti, P.amap = maps + 4 * c.n_layers + 4 + nti;
    const int pi = (lm->tc_flat_ok && tc_fold_in_cta(B, c.hidden)) ? 1 : 0;
    const TcPlanInfo& info = lm->tc_info[pi];
    P.plan = lm->tc_plan + 256 * pi;
    P.pg2 = lm->tc_pg2, P.gu_nsl = lm->tc_gu_nsl;
    P.ln1 = lm->ptr_tab, P.bqkv = lm->ptr_tab + c.n_layers, P.ln2 = lm->ptr_tab + 2 * c.n_layers;
    P.final_norm = lm->final_norm, P.inv_freq = lm->inv_freq;
    P.h = lm->h, P.xa = lm->tc_xa, P.act = lm->tc_act;
    P.pq2 = lm->tc_pq2, P.po2 = lm->tc_po2, P.pd2 = lm->tc_pd2;
    P.sq = info.sq, P.so = info.so, P.sd = info.sd;
    P.ao2 = lm->tc_ao2, P.aml2 = lm->tc_aml2, P.act2 = lm->tc_act2, P.h2 = lm->tc_h2, P.max_splits = lm->max_splits;
    // (value, stamp) hand-offs: every launch takes a fresh range of stamps, so nothing left in the buffers by an
    // earlier launch (or by another batch size) can ever match
    const int need_s = n_steps * (tc_layers + 1) + 2, need_h = n_steps * (2 * tc_layers + 1) + 4;
    if (lm->tc_stamp > 0x7fff0000 - need_s || lm->tc_hstamp > 0x7fff0000 - need_h) {
      NT_CUDA_CHECK(cudaMemsetAsync(lm->tc_pq2, 0, lm->tc_pair_bytes, stream));
      lm->tc_stamp = lm->tc_hstamp = 0;
    }
    P.stamp_base = lm->tc_stamp, P.hstamp_base = lm->tc_hstamp;
    lm->tc_stamp += need_s, lm->tc_hstamp += need_h;
    P.kv = make_kv(lm, st);
    if ((rc = kv_pool_tmap(P.kv, c.n_layers, &P.kvmap))) return rc;
    P.logits = lm->logits, P.tmax = lm->tc_tmax, P.ntiles = info.ntiles;
    // lm_head tile list under the vocabulary range: the EOS tile sits before or after the range's tiles, in tile order
    const VocabTiles vt = vocab_tiles(lm, sp->eos_id);
    P.head_n = vt.count(), P.head_lo = vt.t_lo, P.head_eos = vt.eos_tile;
    P.head_eos_at = vt.eos_tile < 0 ? -1 : (vt.eos_tile < vt.t_lo ? 0 : vt.t_hi - vt.t_lo);
    P.samp = make_sampler(lm, st, sp);
    P.samp.advance = 1;
    P.gbar = lm->gbar;
    P.n_steps = n_steps;
    P.logits_out = logits_out;
    P.logits_step_stride = static_cast<long long>(B) * c.vocab_size;
    P.prof = lm->prof, P.prof_step = lm->prof_step;
    if ((rc = launch_sampler_check(P.samp))) return rc;
    return launch_decode_tc(P, B, lm->num_sms > 256 ? 256 : lm->num_sms, info, stream);
  }

  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  NT_CUDA_CHECK(cudaStreamIsCapturing(stream, &cap));
  const bool use_graph = !logits_out && cap == cudaStreamCaptureStatusNone && n_steps > 1;
  if (!use_graph) {
    for (int i = 0; i < n_steps; ++i) {
      if ((rc = decode_step(lm, st, B, sp, stream))) return rc;
      if (logits_out)
        NT_CUDA_CHECK(cudaMemcpyAsync(logits_out + size_t(i) * B * c.vocab_size, lm->logits,
                                      size_t(B) * c.vocab_size * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
    return NT_OK;
  }
  // graph keyed by everything baked into the kernel parameters
  std::vector<uint8_t> key(sizeof(int) + sizeof(nt_lm_state) + sizeof(nt_sampling));
  memcpy(key.data(), &B, sizeof(int));
  memcpy(key.data() + sizeof(int), st, sizeof(nt_lm_state));
  memcpy(key.data() + sizeof(int) + sizeof(nt_lm_state), sp, sizeof(nt_sampling));
  if (!lm->graph || key != lm->graph_key) {
    if (lm->graph) {
      cudaGraphExecDestroy(lm->graph);
      lm->graph = nullptr;
    }
    cudaGraph_t g = nullptr;
    const uint64_t before = g_launches.load();
    NT_CUDA_CHECK(cudaStreamBeginCapture(lm->cap_stream, cudaStreamCaptureModeThreadLocal));
    rc = decode_step(lm, st, B, sp, lm->cap_stream);
    cudaError_t e = cudaStreamEndCapture(lm->cap_stream, &g);
    lm->graph_kernels = g_launches.load() - before;  // recorded, not executed: counted per replay instead
    g_launches.store(before);
    if (rc) {
      if (g) cudaGraphDestroy(g);
      return rc;
    }
    if (e != cudaSuccess) return set_error(NT_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    e = cudaGraphInstantiate(&lm->graph, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) {
      lm->graph = nullptr;
      return set_error(NT_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    }
    lm->graph_key = key;
  }
  for (int i = 0; i < n_steps; ++i) {
    NT_CUDA_CHECK(cudaGraphLaunch(lm->graph, stream));
    g_launches.fetch_add(lm->graph_kernels, std::memory_order_relaxed);
  }
  return NT_OK;
}

extern "C" int nt_lm_set_slot_sampling(nt_lm* lm, const nt_slot_sampling* table, void* stream_) {
  if (!lm) return set_error(NT_ERR_INVALID, "nt_lm_set_slot_sampling: null handle");
  const bool on = table != nullptr;
  if (on) {
    for (int s = 0; s < lm->cfg.max_batch; ++s) {
      const nt_slot_sampling& e = table[s];
      if (!(std::isfinite(e.temperature) && e.temperature > 0.f))
        return set_error(NT_ERR_INVALID, "slot %d: temperature %g must be finite and > 0", s, e.temperature);
      if (e.top_k < 1 || e.top_k > 64) return set_error(NT_ERR_INVALID, "slot %d: top_k=%d not in 1..64", s, e.top_k);
      if (!(e.top_p > 0.f && e.top_p <= 1.f)) return set_error(NT_ERR_INVALID, "slot %d: top_p %g not in (0, 1]", s, e.top_p);
      if (!(e.min_p >= 0.f && e.min_p < 1.f)) return set_error(NT_ERR_INVALID, "slot %d: min_p %g not in [0, 1)", s, e.min_p);
    }
    // pageable source: the runtime has staged it by the time the call returns
    NT_CUDA_CHECK(cudaMemcpyAsync(lm->slot_sp, table, size_t(lm->cfg.max_batch) * sizeof(nt_slot_sampling), cudaMemcpyHostToDevice,
                                  reinterpret_cast<cudaStream_t>(stream_)));
  }
  // the cached decode graph baked the table pointer (or its absence) into its sampler node; new values in a table
  // that stays on are read at the next replay
  if (on != lm->slot_sp_on && lm->graph) {
    cudaGraphExecDestroy(lm->graph);
    lm->graph = nullptr;
  }
  lm->slot_sp_on = on;
  return NT_OK;
}

extern "C" int nt_lm_set_vocab_range(nt_lm* lm, int32_t lo, int32_t hi, void* stream) {
  (void)stream;   // host state only: read by the launches enqueued after this call
  if (!lm) return set_error(NT_ERR_INVALID, "nt_lm_set_vocab_range: null handle");
  const int V = lm->cfg.vocab_size;
  if (!(0 <= lo && lo < hi && hi <= V)) return set_error(NT_ERR_INVALID, "vocab range [%d, %d) not inside [0, %d)", lo, hi, V);
  if (hi - lo < 64) return set_error(NT_ERR_INVALID, "vocab range [%d, %d) holds fewer than 64 ids", lo, hi);
  if (lo % 128 || (hi % 128 && hi != V))
    return set_error(NT_ERR_INVALID, "vocab range [%d, %d): lo must be a multiple of 128, hi too unless it is %d", lo, hi, V);
  const bool on = !(lo == 0 && hi == V);
  // the cached decode graph baked the lm_head launches of the previous range
  if ((on != lm->vr_on || lo != lm->vr_lo || hi != lm->vr_hi) && lm->graph) {
    cudaGraphExecDestroy(lm->graph);
    lm->graph = nullptr;
  }
  lm->vr_on = on;
  lm->vr_lo = on ? lo : 0;
  lm->vr_hi = on ? hi : 0;
  return NT_OK;
}

// Debug / per-stage parity hooks: limit the number of layers run (-1 = all) and expose the
// internal activation buffers (device pointers into the caller's workspace).
extern "C" int nt_lm_debug_set_layers(nt_lm* lm, int n_layers) {
  if (!lm || n_layers > lm->cfg.n_layers) return set_error(NT_ERR_INVALID, "nt_lm_debug_set_layers: bad argument");
  lm->debug_layers = n_layers;
  if (lm->graph) {
    cudaGraphExecDestroy(lm->graph);
    lm->graph = nullptr;
  }
  return NT_OK;
}
extern "C" int nt_lm_debug_set_profile(nt_lm* lm, long long* buf, int step) {
  if (!lm) return set_error(NT_ERR_INVALID, "nt_lm_debug_set_profile: null handle");
  lm->prof = buf;
  lm->prof_step = step;
  return NT_OK;
}
extern "C" int nt_lm_debug_capture_sampler(nt_lm* lm, float* topk_val, int32_t* topk_idx, int32_t* token) {
  if (!lm) return set_error(NT_ERR_INVALID, "nt_lm_debug_capture_sampler: null handle");
  if (!topk_val != !topk_idx || !topk_val != !token)
    return set_error(NT_ERR_INVALID, "nt_lm_debug_capture_sampler: pass all three buffers or none");
  lm->dbg_topk_val = topk_val, lm->dbg_topk_idx = topk_idx, lm->dbg_token = token;
  // the cached decode graph baked the previous pointers into its sampler node (the graph key does not see them)
  if (lm->graph) {
    cudaGraphExecDestroy(lm->graph);
    lm->graph = nullptr;
  }
  return NT_OK;
}
extern "C" int nt_debug_decode_plan(int hidden, int inter, int n_heads, int n_kv, int vocab, int n_sms, int flat,
                                    int16_t* items, int32_t* counts, int32_t* flags, uint8_t* gu_nsl, int gu_cap,
                                    int32_t* info) {
  if (hidden < 64 || inter < 64 || n_heads < 1 || n_kv < 1 || vocab < 1)
    return set_error(NT_ERR_INVALID, "nt_debug_decode_plan: bad shape");
  if (n_sms < 8 || n_sms > 256) return set_error(NT_ERR_INVALID, "decode_tc: %d SMs unsupported", n_sms);
  const TcShape ts{hidden, inter, n_heads, n_kv, (n_heads + 2 * n_kv) * 64, vocab};
  const int tg = (2 * inter + 127) / 128;
  if (flat && gu_nsl && gu_cap < tg) return set_error(NT_ERR_INVALID, "nt_debug_decode_plan: gu_nsl holds %d < %d tiles", gu_cap, tg);
  std::vector<TcPlan> plan(n_sms);
  std::vector<unsigned char> nsl(flat ? tg : 0, 0);
  TcPlanInfo pi = {};
  const int rc = tc_build_plan(ts, n_sms, flat != 0, plan.data(), flat ? nsl.data() : nullptr, &pi);
  if (rc) return rc;
  for (int c = 0; c < n_sms; ++c) {
    for (int ph = 0; ph < 4; ++ph) {
      if (counts) counts[4 * c + ph] = plan[c].n[ph];
      for (int i = 0; i < kTcMaxItems && items; ++i) {
        const TcItem& it = plan[c].it[ph][i];
        int16_t* o = items + ((size_t(c) * 4 + ph) * kTcMaxItems + i) * 4;
        o[0] = it.tile, o[1] = it.kb0, o[2] = it.nkb, o[3] = it.slice;
      }
    }
    if (flags) flags[3 * c] = plan[c].fold_q, flags[3 * c + 1] = plan[c].fold_g, flags[3 * c + 2] = plan[c].gu_split;
  }
  if (flat && gu_nsl) memcpy(gu_nsl, nsl.data(), nsl.size());
  if (info) {
    const int v[7] = {pi.sq, pi.so, pi.sd, pi.sg, pi.ntiles, pi.max_chunks, pi.gu_split};
    memcpy(info, v, sizeof(v));
  }
  return NT_OK;
}

extern "C" void* nt_lm_debug_ptr(nt_lm* lm, const char* name) {
  if (!lm || !name) return nullptr;
  const struct { const char* n; void* p; } tab[] = {
      {"h", lm->h}, {"q", lm->q}, {"qkv", lm->qkv}, {"attn", lm->attn}, {"act", lm->act}, {"logits", lm->logits},
      {"xn", lm->xn}, {"attn_bf16", lm->attn_bf16}, {"act_bf16", lm->act_bf16}, {"h_last", lm->h_last},
      {"tmax", lm->tc_tmax}};
  for (const auto& e : tab)
    if (!strcmp(e.n, name)) return e.p;
  return nullptr;
}

extern "C" int nt_debug_launch_chain(int n, int grid, int block, int* counter, void* stream) {
  for (int i = 0; i < n; ++i) {
    int rc = launch_kernel(noop_chain_kernel, dim3(grid), dim3(block), 0, reinterpret_cast<cudaStream_t>(stream), true, counter);
    if (rc) return rc;
  }
  return NT_OK;
}

extern "C" int nt_lm_head_gemv(nt_lm* lm, const float* h, int B, float* logits, void* stream) {
  if (!lm || !h || !logits) return set_error(NT_ERR_INVALID, "nt_lm_head_gemv: null argument");
  if (B < 1 || B > 4) return set_error(NT_ERR_INVALID, "nt_lm_head_gemv: batch %d not in 1..4", B);
  return lm_head_rows(lm, h, B, logits, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int nt_op_rmsnorm(const float* x, const float* w, float eps, int rows, int cols, float* out_f32, void* out_bf16,
                             void* stream) {
  if (!x || !w || (!out_f32 && !out_bf16)) return set_error(NT_ERR_INVALID, "nt_op_rmsnorm: null argument");
  return launch_rmsnorm_rows(x, w, eps, rows, cols, out_f32, static_cast<__nv_bfloat16*>(out_bf16),
                             reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int nt_op_topk_sample(const float* logits, int B, int V, const nt_sampling* sp, const int32_t* n_generated,
                                 int32_t step, int32_t* out_token, float* out_topk_val, int32_t* out_topk_idx,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  if (!logits || !sp || !n_generated || !workspace) return set_error(NT_ERR_INVALID, "nt_op_topk_sample: null argument");
  Arena a(workspace, workspace_bytes);
  SamplerParams s;
  memset(&s, 0, sizeof(s));
  s.logits = logits, s.V = V, s.sp = *sp;
  s.nchunks = sampler_nchunks(V);
  s.cand_val = a.take<float>(sampler_scratch_floats(B, V));
  s.cand_idx = a.take<int>(sampler_scratch_floats(B, V));
  if (!a.ok()) return set_error(NT_ERR_NOMEM, "nt_op_topk_sample: workspace too small (need %zu)", a.off);
  s.n_generated_override = n_generated;
  s.step_override = step;
  s.dbg_token = out_token, s.dbg_topk_val = out_topk_val, s.dbg_topk_idx = out_topk_idx;
  s.max_new = 1 << 30, s.max_ctx = 1 << 30;
  return launch_sampler(s, B, reinterpret_cast<cudaStream_t>(stream));
}
