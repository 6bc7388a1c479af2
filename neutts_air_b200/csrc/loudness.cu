// Integrated loudness (ITU-R BS.1770-4, torchaudio.functional.loudness's semantics without its clamp) of ragged mono
// rows, and normalisation of each row to a target.  Everything runs in fp64; every sum has a fixed order.
//
// The K-weighting is two DF2T biquads in cascade: a 4-state linear system s' = A s + B x.  Each row is cut into chunks
// of c samples, c dividing the 100 ms step, so a segment [j * step, (j + 1) * step) holds m = step / c chunks and every
// 400 ms gating block is four whole segments.  Only whole segments up to the last full block are filtered: the tail
// after it reaches no block.
//   chunk_zero_kernel      one thread per chunk runs it from zero state: its end state e_k
//   segment_fold_kernel    one thread per segment: P_q = state at chunk q's start from a zero segment start
//                          (P_0 = 0, P_{q+1} = A^c P_q + e_q) in place of e_q, and E_j = P_m
//   row_scan_kernel        one thread per row: the true segment start states S_0 = 0, S_{j+1} = A^step S_j + E_j
//   chunk_energy_kernel    one thread per chunk: true start state A^(c q) S_j + P_q, re-run, sum of y^2 in order
//   gate_kernel            one block per row: block energies, both gates, L, and the gain 10^((T - L) / 20)
//   apply_gain_kernel      out = float(g * (double)x); a row whose gain is NaN is copied unchanged
// By linearity the chunk start states equal the serial recursion's in exact arithmetic: no transient is truncated.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "internal.h"

namespace nt {
namespace {

constexpr int kMinRate = 8000, kMaxRate = 192000;
constexpr int kMaxChunk = 256;        // samples one thread filters serially
constexpr int kMaxItems = 128;        // rows per group of launches (kernel parameter space)
constexpr int kChunkThreads = 64;
constexpr int kGateThreads = 256;
constexpr double kBias = -0.691, kAbsGate = -70.0;

struct Geometry {
  int gate, step, chunk, m;
};

int geometry(int r, Geometry* g) {
  if (r < kMinRate || r > kMaxRate || r % 10 != 0)
    return set_error(NT_ERR_INVALID, "sample_rate %d must be a multiple of 10 Hz in [%d, %d]", r, kMinRate, kMaxRate);
  g->gate = static_cast<int>(std::lround(0.4 * r));
  g->step = g->gate / 4;
  g->chunk = 1;
  for (int c = std::min(kMaxChunk, g->step); c >= 1; --c)
    if (g->step % c == 0) {
      g->chunk = c;
      break;
    }
  g->m = g->step / g->chunk;
  return NT_OK;
}

// Whole segments a row of n samples filters: floor(n / step) when it holds at least one block, else 0.
long long segments(const Geometry& g, long long n) { return n >= g.gate ? n / g.step : 0; }

// b0, b1, b2, a1, a2 of each stage, normalised by a0 (torchaudio's treble_biquad and highpass_biquad formulas).
struct KWeight {
  double b[2][3], a[2][2];
};

KWeight k_weighting(int r) {
  KWeight k;
  double w0 = 2 * M_PI * 1500.0 / r;
  double alpha = std::sin(w0) / 2 / (1 / std::sqrt(2.0));
  const double A = std::exp(4.0 / 40 * std::log(10.0));
  const double t1 = 2 * std::sqrt(A) * alpha, t2 = (A - 1) * std::cos(w0), t3 = (A + 1) * std::cos(w0);
  double a0 = (A + 1) - t2 + t1;
  k.b[0][0] = A * ((A + 1) + t2 + t1) / a0;
  k.b[0][1] = -2 * A * ((A - 1) + t3) / a0;
  k.b[0][2] = A * ((A + 1) + t2 - t1) / a0;
  k.a[0][0] = 2 * ((A - 1) - t3) / a0;
  k.a[0][1] = ((A + 1) - t2 - t1) / a0;
  w0 = 2 * M_PI * 38.0 / r;
  alpha = std::sin(w0) / 2.0 / 0.5;
  a0 = 1 + alpha;
  k.b[1][0] = (1 + std::cos(w0)) / 2 / a0;
  k.b[1][1] = (-1 - std::cos(w0)) / a0;
  k.b[1][2] = k.b[1][0];
  k.a[1][0] = -2 * std::cos(w0) / a0;
  k.a[1][1] = (1 - alpha) / a0;
  return k;
}

// One sample through the cascade (DF2T, as scipy's lfilter): s[0..1] the shelf's state, s[2..3] the high-pass's.
__host__ __device__ __forceinline__ double kstep(const KWeight& k, double x, double s[4]) {
  const double y1 = k.b[0][0] * x + s[0];
  s[0] = k.b[0][1] * x - k.a[0][0] * y1 + s[1];
  s[1] = k.b[0][2] * x - k.a[0][1] * y1;
  const double y2 = k.b[1][0] * y1 + s[2];
  s[2] = k.b[1][1] * y1 - k.a[1][0] * y2 + s[3];
  s[3] = k.b[1][2] * y1 - k.a[1][1] * y2;
  return y2;
}

struct Mat4 {
  double v[16];   // row-major
};

Mat4 mul(const Mat4& x, const Mat4& y) {
  Mat4 o;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double acc = 0;
      for (int t = 0; t < 4; ++t) acc += x.v[i * 4 + t] * y.v[t * 4 + j];
      o.v[i * 4 + j] = acc;
    }
  return o;
}

Mat4 identity() {
  Mat4 o{};
  for (int i = 0; i < 4; ++i) o.v[i * 5] = 1;
  return o;
}

// A^(c q) for q = 0 .. m: the zero-input transition over q chunks.  A's column t is one step from unit state t.
std::vector<Mat4> chunk_powers(const KWeight& k, const Geometry& g) {
  Mat4 A{};
  for (int t = 0; t < 4; ++t) {
    double s[4] = {0, 0, 0, 0};
    s[t] = 1;
    kstep(k, 0.0, s);
    for (int i = 0; i < 4; ++i) A.v[i * 4 + t] = s[i];
  }
  Mat4 Ac = identity();
  for (int i = 0; i < g.chunk; ++i) Ac = mul(A, Ac);
  std::vector<Mat4> pw(g.m + 1);
  pw[0] = identity();
  for (int q = 0; q < g.m; ++q) pw[q + 1] = mul(Ac, pw[q]);
  return pw;
}

// o = M s + e; o may alias s or e.
__device__ __forceinline__ void matvec_add(const double* __restrict__ M, const double s[4], const double e[4],
                                           double o[4]) {
  double r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double acc = e[i];
#pragma unroll
    for (int t = 0; t < 4; ++t) acc = fma(M[i * 4 + t], s[t], acc);
    r[i] = acc;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = r[i];
}

__device__ __forceinline__ void load4(const double* p, double s[4]) {
  const double2 a = reinterpret_cast<const double2*>(p)[0], b = reinterpret_cast<const double2*>(p)[1];
  s[0] = a.x, s[1] = a.y, s[2] = b.x, s[3] = b.y;
}

__device__ __forceinline__ void store4(double* p, const double s[4]) {
  reinterpret_cast<double2*>(p)[0] = make_double2(s[0], s[1]);
  reinterpret_cast<double2*>(p)[1] = make_double2(s[2], s[3]);
}

// Per group of launches: item i is a row at in[in_off[i] .. in_off[i + 1]) whose whole segments are the global
// segments seg_base[i] .. seg_base[i + 1] - 1 (chunks m times that); target NaN: measure only.
struct Items {
  long long in_off[kMaxItems + 1];
  long long seg_base[kMaxItems + 1];
  double target[kMaxItems];
  int row0;                           // global index of item 0 (lufs and gain are indexed by row)
};

struct Plan {
  KWeight k;
  int chunk, m;
};

__global__ void __launch_bounds__(kChunkThreads) chunk_zero_kernel(const __grid_constant__ Items it,
                                                                   const __grid_constant__ Plan p,
                                                                   const float* __restrict__ in, double* state) {
  const int i = blockIdx.y;
  const long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k >= (it.seg_base[i + 1] - it.seg_base[i]) * p.m) return;
  const float* x = in + it.in_off[i] + k * p.chunk;
  double s[4] = {0, 0, 0, 0};
  for (int t = 0; t < p.chunk; ++t) kstep(p.k, static_cast<double>(__ldg(x + t)), s);
  store4(state + (it.seg_base[i] * p.m + k) * 4, s);
}

__global__ void __launch_bounds__(kChunkThreads) segment_fold_kernel(const __grid_constant__ Items it, int m,
                                                                     const double* __restrict__ pw, double* state,
                                                                     double* seg) {
  const int i = blockIdx.y;
  const long long j = it.seg_base[i] + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= it.seg_base[i + 1]) return;
  const double* Ac = pw + 16;
  double t[4] = {0, 0, 0, 0}, e[4];
  for (int q = 0; q < m; ++q) {
    double* sp = state + (j * m + q) * 4;
    load4(sp, e);
    store4(sp, t);
    matvec_add(Ac, t, e, t);
  }
  store4(seg + j * 4, t);
}

__global__ void __launch_bounds__(kMaxItems) row_scan_kernel(const __grid_constant__ Items it, int n_items, int m,
                                                            const double* __restrict__ pw, double* seg) {
  const int i = threadIdx.x;
  if (i >= n_items) return;
  const double* Astep = pw + 16 * m;
  double s[4] = {0, 0, 0, 0}, e[4];
  for (long long j = it.seg_base[i]; j < it.seg_base[i + 1]; ++j) {
    load4(seg + j * 4, e);
    store4(seg + j * 4, s);
    matvec_add(Astep, s, e, s);
  }
}

__global__ void __launch_bounds__(kChunkThreads) chunk_energy_kernel(const __grid_constant__ Items it,
                                                                     const __grid_constant__ Plan p,
                                                                     const float* __restrict__ in,
                                                                     const double* __restrict__ pw,
                                                                     const double* __restrict__ state,
                                                                     const double* __restrict__ seg, double* energy) {
  const int i = blockIdx.y;
  const long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k >= (it.seg_base[i + 1] - it.seg_base[i]) * p.m) return;
  const long long kg = it.seg_base[i] * p.m + k;
  const int q = static_cast<int>(k % p.m);
  double S[4], P[4], s[4];
  load4(seg + (kg / p.m) * 4, S);
  load4(state + kg * 4, P);
  matvec_add(pw + 16 * q, S, P, s);
  const float* x = in + it.in_off[i] + k * p.chunk;
  double acc = 0;
  for (int t = 0; t < p.chunk; ++t) {
    const double y = kstep(p.k, static_cast<double>(__ldg(x + t)), s);
    acc = fma(y, y, acc);
  }
  energy[kg] = acc;
}

// Sum of (count, energy) over the blocks of one row whose loudness passes `gate`, in a fixed order: each thread walks
// its blocks in ascending order, then a tree over the threads.
__device__ void gated_sum(const double* __restrict__ energy, long long c0, int m, long long nb, double inv_gate,
                          double gate, double* s_sum, long long* s_cnt, double* sum, long long* cnt) {
  double acc = 0;
  long long c = 0;
  for (long long j = threadIdx.x; j < nb; j += blockDim.x) {
    double q = 0;
    for (long long t = c0 + j * m; t < c0 + (j + 4) * m; ++t) q += energy[t];
    const double z = q * inv_gate;
    if (kBias + 10 * log10(z) > gate) acc += z, ++c;
  }
  s_sum[threadIdx.x] = acc;
  s_cnt[threadIdx.x] = c;
  __syncthreads();
  for (int w = blockDim.x / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s_sum[threadIdx.x] += s_sum[threadIdx.x + w], s_cnt[threadIdx.x] += s_cnt[threadIdx.x + w];
    __syncthreads();
  }
  *sum = s_sum[0];
  *cnt = s_cnt[0];
  __syncthreads();
}

__global__ void __launch_bounds__(kGateThreads) gate_kernel(const __grid_constant__ Items it, int m, int gate_len,
                                                            const double* __restrict__ energy, double* lufs,
                                                            double* gain) {
  __shared__ double s_sum[kGateThreads];
  __shared__ long long s_cnt[kGateThreads];
  const int i = blockIdx.x;
  const long long ns = it.seg_base[i + 1] - it.seg_base[i];
  const long long nb = ns > 0 ? ns - 3 : 0;
  const long long c0 = it.seg_base[i] * m;
  const double inv_gate = 1.0 / gate_len;
  double sum, rel;
  long long cnt;
  gated_sum(energy, c0, m, nb, inv_gate, kAbsGate, s_sum, s_cnt, &sum, &cnt);
  double L = NAN;
  if (cnt > 0) {
    rel = kBias + 10 * log10(sum / cnt) - 10;
    gated_sum(energy, c0, m, nb, inv_gate, fmax(rel, kAbsGate), s_sum, s_cnt, &sum, &cnt);
    L = kBias + 10 * log10(sum / cnt);
  }
  if (threadIdx.x == 0) {
    lufs[it.row0 + i] = L;
    gain[it.row0 + i] = pow(10.0, (it.target[i] - L) / 20.0);   // NaN when L or the target is NaN
  }
}

__global__ void apply_gain_kernel(const __grid_constant__ Items it, const double* __restrict__ gain, const float* in,
                                  float* out) {
  const int i = blockIdx.y;
  const double g = gain[it.row0 + i];
  const bool keep = isnan(g);
  if (keep && in == out) return;
  const long long n = it.in_off[i + 1] - it.in_off[i];
  const float* x = in + it.in_off[i];
  float* y = out + it.in_off[i];
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < n;
       t += static_cast<long long>(gridDim.x) * blockDim.x)
    y[t] = keep ? x[t] : __double2float_rn(g * static_cast<double>(x[t]));
}

struct Layout {
  size_t bytes;
  double *pw, *state, *energy, *seg, *gain;
};

// Workspace carve-up for n rows: the chunk powers, per chunk a state and an energy, per segment a state, per row a gain.
Layout layout(const Geometry& g, int n, const int64_t* off, void* base) {
  long long segs = 0;
  for (int i = 0; i < n; ++i) segs += segments(g, off[i + 1] - off[i]);
  Arena a(base, ~size_t(0));
  Layout l;
  l.pw = a.take<double>(16ull * (g.m + 1));
  l.state = a.take<double>(4ull * segs * g.m);
  l.energy = a.take<double>(static_cast<size_t>(segs) * g.m);
  l.seg = a.take<double>(4ull * segs);
  l.gain = a.take<double>(n);
  l.bytes = a.off;
  return l;
}

int check_offsets(int n, const int64_t* off) {
  if (n < 0) return set_error(NT_ERR_INVALID, "n %d is negative", n);
  if (n > 0 && !off) return set_error(NT_ERR_INVALID, "in_offsets is NULL");
  if (n > 0 && off[0] < 0) return set_error(NT_ERR_INVALID, "negative offset");
  for (int i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return set_error(NT_ERR_INVALID, "row %d: offsets must not decrease", i);
  return NT_OK;
}

}  // namespace
}  // namespace nt

using namespace nt;

extern "C" int nt_loudness_query(int sample_rate, nt_loudness_info* info) {
  Geometry g{};
  if (int rc = geometry(sample_rate, &g)) return rc;
  if (info) {
    info->gate = g.gate;
    info->step = g.step;
    info->chunk = g.chunk;
    info->chunks_per_step = g.m;
  }
  return NT_OK;
}

extern "C" size_t nt_loudness_workspace_bytes(int sample_rate, int n, const int64_t* in_offsets) {
  Geometry g{};
  if (geometry(sample_rate, &g) || check_offsets(n, in_offsets) || n == 0) return 0;
  return layout(g, n, in_offsets, nullptr).bytes;
}

extern "C" int nt_loudness_run(int sample_rate, int n, const float* in, const int64_t* in_offsets,
                               const double* targets, double* lufs, float* out, void* workspace, size_t bytes,
                               void* stream) {
  Geometry g{};
  if (int rc = geometry(sample_rate, &g)) return rc;
  if (int rc = check_offsets(n, in_offsets)) return rc;
  if (n == 0) return NT_OK;
  if (in_offsets[n] > in_offsets[0] && !in) return set_error(NT_ERR_INVALID, "nt_loudness_run: null input");
  if (!lufs) return set_error(NT_ERR_INVALID, "nt_loudness_run: null lufs");
  if (targets) {
    if (in_offsets[n] > in_offsets[0] && !out) return set_error(NT_ERR_INVALID, "nt_loudness_run: null output");
    for (int i = 0; i < n; ++i)
      if (std::isinf(targets[i])) return set_error(NT_ERR_INVALID, "row %d: target %f is not finite", i, targets[i]);
  }
  const Layout need = layout(g, n, in_offsets, nullptr);
  if (!workspace || bytes < need.bytes)
    return set_error(NT_ERR_NOMEM, "workspace of %zu bytes, %zu needed", workspace ? bytes : 0, need.bytes);
  if (reinterpret_cast<uintptr_t>(workspace) & 15) return set_error(NT_ERR_INVALID, "workspace must be 16-byte aligned");
  const Layout l = layout(g, n, in_offsets, workspace);

  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Plan p;
  p.k = k_weighting(sample_rate);
  p.chunk = g.chunk;
  p.m = g.m;
  const std::vector<Mat4> pw = chunk_powers(p.k, g);
  NT_CUDA_CHECK(cudaMemcpyAsync(l.pw, pw.data(), pw.size() * sizeof(Mat4), cudaMemcpyHostToDevice, s));

  long long seg0 = 0;
  for (int c0 = 0; c0 < n; c0 += kMaxItems) {
    const int mi = std::min(kMaxItems, n - c0);
    Items it;
    std::memset(&it, 0, sizeof(it));
    it.row0 = c0;
    long long max_segs = 0, max_len = 0;
    for (int i = 0; i <= mi; ++i) {
      it.in_off[i] = in_offsets[c0 + i];
      it.seg_base[i] = seg0;
      if (i == mi) break;
      const long long len = in_offsets[c0 + i + 1] - in_offsets[c0 + i], ns = segments(g, len);
      it.target[i] = targets ? targets[c0 + i] : NAN;
      seg0 += ns;
      max_segs = std::max(max_segs, ns);
      max_len = std::max(max_len, len);
    }
    if (max_segs > 0) {
      const long long chunks = max_segs * g.m;
      const dim3 gc(static_cast<unsigned>((chunks + kChunkThreads - 1) / kChunkThreads), mi);
      const dim3 gs(static_cast<unsigned>((max_segs + kChunkThreads - 1) / kChunkThreads), mi);
      if (int rc = launch_kernel(chunk_zero_kernel, gc, dim3(kChunkThreads), 0, s, false, it, p, in, l.state)) return rc;
      if (int rc = launch_kernel(segment_fold_kernel, gs, dim3(kChunkThreads), 0, s, false, it, g.m,
                                 static_cast<const double*>(l.pw), l.state, l.seg))
        return rc;
      if (int rc = launch_kernel(row_scan_kernel, dim3(1), dim3(kMaxItems), 0, s, false, it, mi, g.m,
                                 static_cast<const double*>(l.pw), l.seg))
        return rc;
      if (int rc = launch_kernel(chunk_energy_kernel, gc, dim3(kChunkThreads), 0, s, false, it, p, in,
                                 static_cast<const double*>(l.pw), static_cast<const double*>(l.state),
                                 static_cast<const double*>(l.seg), l.energy))
        return rc;
    }
    if (int rc = launch_kernel(gate_kernel, dim3(mi), dim3(kGateThreads), 0, s, false, it, g.m, g.gate,
                               static_cast<const double*>(l.energy), lufs, l.gain))
      return rc;
    if (targets && max_len > 0) {
      const int gx = static_cast<int>(std::min<long long>(64, (max_len + 1023) / 1024));
      if (int rc = launch_kernel(apply_gain_kernel, dim3(gx, mi), dim3(256), 0, s, false, it,
                                 static_cast<const double*>(l.gain), in, out))
        return rc;
    }
  }
  return NT_OK;
}
