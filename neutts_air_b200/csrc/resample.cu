// Polyphase resampler for the synthesised 24 kHz PCM: torchaudio.functional.resample(x, 24000, sample_rate) with its
// defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), optionally fused with the 16-bit PCM conversion.
// One kernel serves one-shot rows and streams: every row of a launch reads its carried history and its new input,
// writes the outputs that are final, and (streams) writes the history the next push needs.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include "common.cuh"
#include "internal.h"

namespace nt {
namespace {

constexpr int kSrcRate = 24000;
constexpr int kWidth = 6;                          // lowpass_filter_width
constexpr double kRolloff = 0.99;
constexpr size_t kSmemOptIn = 227 * 1024;          // sm_90 per-block dynamic shared-memory opt-in
constexpr int kMaxItems = 128;                     // rows per launch (kernel parameter space)
constexpr int kThreads = 512;

struct Geometry {
  int orig, nnew, width, taps, pitch;
  size_t table_bytes, row_bytes;
  int hist_cap;                                    // floats per history buffer (two per row)
};

int geometry(int sample_rate, Geometry* g) {
  if (sample_rate <= 0) return set_error(NT_ERR_INVALID, "sample_rate %d must be a positive integer", sample_rate);
  const int gcd = std::gcd(kSrcRate, sample_rate);
  g->orig = kSrcRate / gcd;
  g->nnew = sample_rate / gcd;
  if (sample_rate == kSrcRate) {                   // torchaudio applies no filter at equal rates: a one-tap identity
    g->width = 0;
    g->taps = 1;
  } else {
    const double base = std::min(g->orig, g->nnew) * kRolloff;
    g->width = static_cast<int>(std::ceil(kWidth * static_cast<double>(g->orig) / base));
    g->taps = 2 * g->width + g->orig;
  }
  const double bytes = 4.0 * g->nnew * static_cast<double>(g->taps);
  if (bytes > static_cast<double>(kSmemOptIn))
    return set_error(NT_ERR_INVALID,
                     "sample_rate %d needs a %.0f-byte filter table (%d phases x %d taps); the limit is %zu bytes, the "
                     "shared memory one sm_90 block can hold",
                     sample_rate, bytes, g->nnew, g->taps, kSmemOptIn);
  // odd row pitch: lanes on different phases then read different banks; only when the padded table still fits
  g->pitch = g->taps;
  if (g->nnew > 1 && g->taps % 2 == 0 && 4ull * g->nnew * (g->taps + 1) <= kSmemOptIn) g->pitch = g->taps + 1;
  g->table_bytes = (4ull * g->nnew * g->pitch + 15) & ~size_t(15);
  g->hist_cap = (g->taps + 63) & ~63;
  g->row_bytes = 2ull * 4 * g->hist_cap;
  return NT_OK;
}

// The filter of torchaudio's _get_sinc_resample_kernel in float64, rounded once to fp32: phase p, tap i reads input
// (k * orig - width + i) for output frame k.
std::vector<float> make_table(const Geometry& g) {
  std::vector<float> tab(g.table_bytes / 4, 0.f);
  if (g.width == 0) {
    tab[0] = 1.f;
    return tab;
  }
  const double base = std::min(g.orig, g.nnew) * kRolloff;
  const double scale = base / g.orig;
  for (int p = 0; p < g.nnew; ++p)
    for (int i = 0; i < g.taps; ++i) {
      double t = (-static_cast<double>(p) / g.nnew + static_cast<double>(i - g.width) / g.orig) * base;
      t = std::min(std::max(t, -static_cast<double>(kWidth)), static_cast<double>(kWidth));
      const double c = std::cos(t * M_PI / kWidth / 2);
      const double window = c * c;
      t *= M_PI;
      const double k = t == 0 ? 1.0 : std::sin(t) / t;
      tab[static_cast<size_t>(p) * g.pitch + i] = static_cast<float>(k * (window * scale));
    }
  return tab;
}

// Per launch: the rows and their spans.  flags: bit 0 final, bit 1 fresh (history = `width` zeros, nothing stored),
// bit 2 the parity of the history buffer to read.
struct Items {
  int32_t row[kMaxItems];          // -1: one-shot item without state
  int32_t held[kMaxItems];         // history samples before this push
  uint8_t flags[kMaxItems];
  long long in_off[kMaxItems + 1];
  long long out_off[kMaxItems + 1];
};

// Grid (blocks per row, rows).  Output j of a row is frame k = j / new, phase p = j % new: the dot product of table row
// p with taps 0 .. taps-1 of comb[k * orig ..], where comb = history ++ new input ++ zeros.  Every output sums its taps
// in ascending order and skips only zero-valued taps (the leading zeros of a fresh row and the trailing zeros of a
// final push), so it does not depend on how the input was split into pushes.
__global__ void __launch_bounds__(kThreads) resample_kernel(const __grid_constant__ Items it, const float4* __restrict__ table,
                                                            int table4, float* state, const float* __restrict__ in,
                                                            void* out, int s16, int orig, int nnew, int taps, int pitch,
                                                            int hist_cap) {
  const int i = blockIdx.y;
  const int row = it.row[i], h = it.held[i], fl = it.flags[i];
  const bool fin = fl & 1, fresh = fl & 2;
  const int par = (fl >> 2) & 1;
  const long long n = it.in_off[i + 1] - it.in_off[i];
  const long long span = it.out_off[i + 1] - it.out_off[i];
  const float* x = in + it.in_off[i];
  float* rs = row >= 0 ? state + 2ll * hist_cap * row : nullptr;
  const float* hist = rs && !fresh ? rs + par * hist_cap : nullptr;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;

  if (rs && !fin) {   // the next push's history: comb[D, h + n), D = frames emitted * orig, into the other buffer
    const long long D = span / nnew * orig, keep = h + n - D;
    float* dst = rs + (par ^ 1) * hist_cap;
    for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < keep; t += stride) {
      const long long c = D + t;
      dst[t] = c < h ? (hist ? hist[c] : 0.f) : x[c - h];
    }
  }
  if (static_cast<long long>(blockIdx.x) * blockDim.x >= span) return;

  extern __shared__ float4 s_tab4[];
  for (int q = threadIdx.x; q < table4; q += blockDim.x) s_tab4[q] = table[q];
  __syncthreads();
  const float* s_tab = reinterpret_cast<const float*>(s_tab4);
  const long long hn = h + n;
  for (long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; j < span; j += stride) {
    const long long k = j / nnew;
    const int p = static_cast<int>(j - k * nnew);
    const long long base = k * orig;
    const float* tp = s_tab + p * pitch;
    const int t0 = static_cast<int>(std::max(0ll, std::min<long long>(taps, h - base)));
    const int t1 = static_cast<int>(std::max<long long>(t0, std::min<long long>(taps, hn - base)));
    float acc = 0.f;
    if (hist)
      for (int t = 0; t < t0; ++t) acc = fmaf(tp[t], __ldg(hist + base + t), acc);
    const float* xs = x + (base - h);
#pragma unroll 4
    for (int t = t0; t < t1; ++t) acc = fmaf(tp[t], __ldg(xs + t), acc);
    const long long o = it.out_off[i] + j;
    if (s16)
      static_cast<int16_t*>(out)[o] = static_cast<int16_t>(__float2int_rn(fminf(fmaxf(acc, -1.f), 1.f) * 32767.f));
    else
      static_cast<float*>(out)[o] = acc;
  }
}

}  // namespace
}  // namespace nt

using namespace nt;

struct nt_resampler {
  Geometry g;
  int sample_rate, pcm_format, max_rows, n_sms;
  float* table;
  float* state;
  // host mirror of every row: held samples, history parity, fresh
  std::vector<int32_t> held;
  std::vector<uint8_t> par, fresh;
};

extern "C" int nt_resampler_query(int sample_rate, nt_resampler_info* info) {
  Geometry g;
  if (int rc = geometry(sample_rate, &g)) return rc;
  if (info) {
    info->orig = g.orig;
    info->target = g.nnew;
    info->width = g.width;
    info->taps = g.taps;
    info->table_bytes = g.table_bytes;
    info->row_bytes = g.row_bytes;
  }
  return NT_OK;
}

extern "C" int nt_resampler_create(int sample_rate, int pcm_format, int max_rows, void* table, void* state,
                                   nt_resampler** out) {
  Geometry g;
  if (int rc = geometry(sample_rate, &g)) return rc;
  if (pcm_format != NT_PCM_F32 && pcm_format != NT_PCM_S16)
    return set_error(NT_ERR_INVALID, "pcm_format %d is neither NT_PCM_F32 nor NT_PCM_S16", pcm_format);
  if (max_rows < 0) return set_error(NT_ERR_INVALID, "max_rows %d is negative", max_rows);
  if (!table || !out || (max_rows > 0 && !state)) return set_error(NT_ERR_INVALID, "nt_resampler_create: null argument");
  if ((reinterpret_cast<uintptr_t>(table) & 15) || (reinterpret_cast<uintptr_t>(state) & 15))
    return set_error(NT_ERR_INVALID, "table and state must be 16-byte aligned");
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess || prop.major != 9 ||
      prop.minor != 0)
    return set_error(NT_ERR_CUDA, "no sm_90 CUDA device: this library has no CPU fallback");
  const std::vector<float> tab = make_table(g);
  NT_CUDA_CHECK(cudaMemcpy(table, tab.data(), g.table_bytes, cudaMemcpyHostToDevice));
  nt_resampler* r = new nt_resampler();
  r->g = g;
  r->sample_rate = sample_rate;
  r->pcm_format = pcm_format;
  r->max_rows = max_rows;
  r->n_sms = prop.multiProcessorCount;
  r->table = static_cast<float*>(table);
  r->state = static_cast<float*>(state);
  r->held.assign(max_rows, g.width);
  r->par.assign(max_rows, 0);
  r->fresh.assign(max_rows, 1);
  *out = r;
  return NT_OK;
}

extern "C" int nt_resampler_destroy(nt_resampler* r) {
  delete r;
  return NT_OK;
}

extern "C" int nt_resampler_reset(nt_resampler* r, const int32_t* rows, int n) {
  if (!r || (n > 0 && !rows) || n < 0) return set_error(NT_ERR_INVALID, "nt_resampler_reset: bad argument");
  for (int i = 0; i < n; ++i)
    if (rows[i] < 0 || rows[i] >= r->max_rows)
      return set_error(NT_ERR_INVALID, "row %d not in 0..%d", rows[i], r->max_rows - 1);
  for (int i = 0; i < n; ++i) r->held[rows[i]] = r->g.width, r->par[rows[i]] = 0, r->fresh[rows[i]] = 1;
  return NT_OK;
}

extern "C" int nt_resampler_push(nt_resampler* r, int n, const int32_t* rows, const int32_t* final_flags,
                                 const float* in, const int64_t* in_offsets, void* out, const int64_t* out_offsets,
                                 void* stream) {
  if (!r || n < 0 || (n > 0 && (!in_offsets || !out_offsets)))
    return set_error(NT_ERR_INVALID, "nt_resampler_push: bad argument");
  if (n == 0) return NT_OK;
  const Geometry& g = r->g;
  std::vector<uint8_t> seen(rows ? r->max_rows : 0, 0);
  if (in_offsets[0] < 0 || out_offsets[0] < 0) return set_error(NT_ERR_INVALID, "negative offset");
  for (int i = 0; i < n; ++i) {
    const long long ni = in_offsets[i + 1] - in_offsets[i], span = out_offsets[i + 1] - out_offsets[i];
    if (ni < 0 || span < 0) return set_error(NT_ERR_INVALID, "item %d: offsets must not decrease", i);
    if (ni > (1ll << 30)) return set_error(NT_ERR_INVALID, "item %d: %lld input samples in one push (limit 2^30)", i, ni);
    long long held = g.width, want;
    const bool fin = !rows || (final_flags && final_flags[i]);
    if (rows) {
      const int row = rows[i];
      if (row < 0 || row >= r->max_rows) return set_error(NT_ERR_INVALID, "row %d not in 0..%d", row, r->max_rows - 1);
      if (seen[row]) return set_error(NT_ERR_INVALID, "row %d appears twice in one push", row);
      seen[row] = 1;
      held = r->held[row];
    }
    if (fin)
      want = (static_cast<long long>(g.nnew) * (held + ni - g.width) + g.orig - 1) / g.orig;
    else
      want = held + ni >= g.taps ? ((held + ni - g.taps) / g.orig + 1) * g.nnew : 0;
    if (span != want)
      return set_error(NT_ERR_INVALID, "item %d: output span %lld, but %lld samples are final after this push", i, span, want);
  }
  if (in_offsets[n] > in_offsets[0] && !in) return set_error(NT_ERR_INVALID, "nt_resampler_push: null input");
  if (out_offsets[n] > out_offsets[0] && !out) return set_error(NT_ERR_INVALID, "nt_resampler_push: null output");

  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t smem = g.table_bytes;
  for (int c0 = 0; c0 < n; c0 += kMaxItems) {
    const int m = std::min(kMaxItems, n - c0);
    Items it;
    std::memset(&it, 0, sizeof(it));
    long long max_span = 0;
    for (int i = 0; i < m; ++i) {
      const int k = c0 + i;
      const int row = rows ? rows[k] : -1;
      const bool fin = !rows || (final_flags && final_flags[k]);
      it.row[i] = row;
      it.held[i] = row >= 0 ? r->held[row] : g.width;
      it.flags[i] = static_cast<uint8_t>((fin ? 1 : 0) | ((row < 0 || r->fresh[row]) ? 2 : 0) | (row >= 0 ? r->par[row] << 2 : 0));
      it.in_off[i] = in_offsets[k];
      it.out_off[i] = out_offsets[k];
      max_span = std::max<long long>(max_span, out_offsets[k + 1] - out_offsets[k]);
    }
    it.in_off[m] = in_offsets[c0 + m];
    it.out_off[m] = out_offsets[c0 + m];
    // about two waves of blocks over the launch, at least one block per row (it writes the row's history)
    const long long tiles = (max_span + kThreads - 1) / kThreads;
    const long long per_row = std::max(1ll, (2ll * r->n_sms + m - 1) / m);
    const int gx = static_cast<int>(std::max(1ll, std::min(tiles, per_row)));
    if (int rc = launch_kernel(resample_kernel, dim3(gx, m), dim3(kThreads), smem, s, false, it,
                               reinterpret_cast<const float4*>(r->table), static_cast<int>(g.table_bytes / 16), r->state,
                               in, out, r->pcm_format == NT_PCM_S16 ? 1 : 0, g.orig, g.nnew, g.taps, g.pitch, g.hist_cap))
      return rc;
    for (int i = 0; i < m && rows; ++i) {
      const int row = rows[c0 + i];
      const long long ni = in_offsets[c0 + i + 1] - in_offsets[c0 + i];
      if (final_flags && final_flags[c0 + i]) {
        r->held[row] = g.width, r->par[row] = 0, r->fresh[row] = 1;
      } else {
        const long long span = out_offsets[c0 + i + 1] - out_offsets[c0 + i];
        r->held[row] = static_cast<int32_t>(r->held[row] + ni - span / g.nnew * g.orig);
        r->par[row] ^= 1;
        r->fresh[row] = 0;
      }
    }
  }
  return NT_OK;
}
