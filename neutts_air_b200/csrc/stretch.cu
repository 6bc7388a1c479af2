// Speaking rate for the synthesised 24 kHz PCM: a phase-vocoder time stretch with the semantics of
// librosa.effects.time_stretch as torch / torchaudio compute it (include/neutts_b200.h states them exactly):
//   stft (n_fft 1024, hop 256, periodic Hann, center, zero padding) -> torchaudio.functional.phase_vocoder(rate r)
//   -> istft (same window, center, length round(L / r)).
// One push runs five launches per round of at most kChunk input samples per row:
//   pack      history ++ input -> 3xTF32 hi / lo rows of 256 samples (frame t reads rows t .. t+3: the wgmma GEMM's
//             overlapped-row A operand, as the codec's k=7 convolutions use it) and the next push's history;
//   analysis  wgmma GEMM, 3xTF32, against the windowed DFT basis -> Re | Im of every complete analysis frame;
//   vocoder   one thread per (row, bin) walks the output frames in order; the phase accumulator is fp64, wrapped to
//             [-pi, pi] after every step, so its error does not grow with the row's length;
//   synthesis wgmma GEMM, 3xTF32, against the windowed inverse-rDFT basis -> time frames;
//   ola       overlap-add in ascending frame order, divided by the window-square envelope, istft's trim.
// Neither GEMM splits K and both run one pinned variant (3xTF32, 64-column tiles), so every element's reduction order
// is independent of how many rows a launch holds; with the carried state (input history, phase accumulators, the
// last three stretched frames) a row's output is bit-identical however it was split into pushes, and a one-shot row
// is the same stream path with one final push.  Scratch is bounded by kMaxItems rows of kChunk samples per round.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "internal.h"

namespace nt {
namespace {

constexpr int kNfft = 1024, kHop = 256, kBins = kNfft / 2 + 1;   // 513 bins
constexpr int kSpecN = 2 * kBins;                                // analysis GEMM columns: Re 0..512 | Im 0..512
constexpr int kSpecLd = 1028;                                    // analysis output row pitch (floats)
constexpr int kS2Ld = 1056;                                      // stretched spectrum row: Re | Im | 30 zeros (K % 32 == 0)
constexpr int kMaxItems = 32;                                    // rows per round
constexpr int kChunk = 8192;                                     // input samples per row per round
// per row and round: analysis frames < chunk/hop + 5, output frames < 2 (chunk/hop) + 11 (r >= 0.5), plus the three
// carried ones; both caps keep a margin and push() checks them
constexpr int kMaxA = kChunk / kHop + 8;
constexpr int kMaxS = 2 * (kChunk / kHop) + 16;
constexpr int kHistCap = 1280;                                   // held input samples < 1280 between pushes
constexpr int kCarry = 3;                                        // stretched frames a later output sample still reads
constexpr double kMinRate = 0.5, kMaxRate = 2.0;

// device row state: two history buffers (ping-pong), fp64 phase accumulators, the last three stretched frames
constexpr size_t kHistBytes = 2ull * kHistCap * 4;
constexpr size_t kAccOff = kHistBytes;
constexpr size_t kCarryOff = kAccOff + 520 * 8;
constexpr size_t kRowBytes = (kCarryOff + 4ull * kCarry * kSpecLd + 255) & ~size_t(255);

// table: analysis basis hi | lo [2][kSpecN][kNfft], synthesis basis hi | lo [2][kNfft][kS2Ld], window squares [kNfft]
constexpr size_t kWaFloats = 2ull * kSpecN * kNfft;
constexpr size_t kWsFloats = 2ull * kNfft * kS2Ld;
constexpr size_t kTableBytes = 4 * (kWaFloats + kWsFloats + kNfft);

// scratch (256-byte aligned blocks)
constexpr size_t a256(size_t b) { return (b + 255) & ~size_t(255); }
constexpr int kCapA = kMaxItems * (kMaxA + 3);                   // A rows (256 samples) per half
constexpr int kCapS = kMaxItems * kMaxS;                         // stretched rows per half
constexpr size_t kOffA = 0;
constexpr size_t kOffSpec = kOffA + a256(2ull * kCapA * kHop * 4);
constexpr size_t kOffS2 = kOffSpec + a256(4ull * kCapA * kSpecLd);
constexpr size_t kOffFr = kOffS2 + a256(2ull * kCapS * kS2Ld * 4);
constexpr size_t kOffStates = kOffFr + a256(4ull * kCapS * kNfft);
constexpr size_t kScratchBytes = kOffStates + kMaxItems * kRowBytes;

// one round's rows, structure of arrays (kernel parameter space)
struct Items {
  char* st[kMaxItems];             // row state
  long long in_off[kMaxItems];     // first input sample of this round (floats from `in`)
  long long out_off[kMaxItems];    // where output sample e0 goes
  long long e0[kMaxItems], e1[kMaxItems];   // output samples [e0, e1) become final this round
  double r[kMaxItems];
  int n[kMaxItems];                // input samples this round
  int held[kMaxItems];             // history samples (x_pad from 256 * a0)
  int keep[kMaxItems], drop[kMaxItems];     // next history: x_pad[256 * a0 + drop, + keep)
  int flags[kMaxItems];            // bit 0 final, bit 1 fresh (history = zeros), bit 2 history parity
  int rb[kMaxItems], nfa[kMaxItems], a0[kMaxItems];   // A / spectrum row base, analysis frames, first frame index
  int sb[kMaxItems], jb[kMaxItems], j0[kMaxItems], j1[kMaxItems];   // stretched row base of frame jb; frames [j0, j1)
  int T[kMaxItems];                // analysis frames of the row (final round; INT_MAX otherwise)
};
static_assert(sizeof(Items) <= 4000, "kernel parameters");

NT_DEVINL void split_store(float v, float* hi, float* lo) {   // 3xTF32 halves, as codec.cu's split_tf32_kernel
  const float h = __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u);
  *hi = h;
  *lo = v - h;
}

// grid (blocks, rows): the round's analysis rows and the next push's history
__global__ void __launch_bounds__(256) pack_kernel(const __grid_constant__ Items it, const float* __restrict__ in, float* A) {
  const int i = blockIdx.y;
  const int fl = it.flags[i];
  const int held = it.held[i], n = it.n[i];
  const int par = (fl >> 2) & 1;
  const float* hist = (fl & 2) ? nullptr : reinterpret_cast<const float*>(it.st[i]) + par * kHistCap;
  const float* x = in + it.in_off[i];
  auto src = [&](int c) -> float { return c < held ? (hist ? hist[c] : 0.f) : (c - held < n ? x[c - held] : 0.f); };
  const int stride = gridDim.x * blockDim.x;
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (!(fl & 1)) {
    float* dst = reinterpret_cast<float*>(it.st[i]) + (par ^ 1) * kHistCap;
    for (int t = t0; t < it.keep[i]; t += stride) dst[t] = src(it.drop[i] + t);
  }
  if (!it.nfa[i]) return;
  const int len = (it.nfa[i] + 3) * kHop;
  float* hi = A + static_cast<long long>(it.rb[i]) * kHop;
  float* lo = hi + static_cast<long long>(kCapA) * kHop;
  for (int t = t0; t < len; t += stride) split_store(src(t), hi + t, lo + t);
}

// torch.linspace(0, pi * hop, 513, dtype=float64)[k]
NT_DEVINL double phase_advance(int k) {
  const double end = M_PI * kHop, step = end / (kBins - 1);
  return k < kBins / 2 ? step * k : end - step * (kBins - 1 - k);
}

NT_DEVINL double wrap_pi(double p) { return p - 2.0 * M_PI * rint(p / (2.0 * M_PI)); }

// grid (ceil(513 / 128), rows), 128 threads: one thread per (row, bin), output frames in order (torchaudio's
// phase_vocoder in fp64 on the fp32 analysis spectra; output Re | Im in fp32, stored as 3xTF32 halves)
__global__ void __launch_bounds__(128) vocoder_kernel(const __grid_constant__ Items it, const float* __restrict__ spec, float* S2) {
  const int i = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int j0 = it.j0[i], j1 = it.j1[i], jb = it.jb[i];
  const int nrows = (j1 > j0 || it.e1[i] > it.e0[i]) ? j1 - jb : 0;
  if (nrows == 0 || k >= kBins) return;
  float* hi = S2 + static_cast<long long>(it.sb[i]) * kS2Ld;
  float* lo = hi + static_cast<long long>(kCapS) * kS2Ld;
  if (k < kS2Ld - kSpecN)
    for (int r = 0; r < nrows; ++r) hi[r * kS2Ld + kSpecN + k] = lo[r * kS2Ld + kSpecN + k] = 0.f;
  double* accp = reinterpret_cast<double*>(it.st[i] + kAccOff) + k;
  float* carry = reinterpret_cast<float*>(it.st[i] + kCarryOff);
  for (int j = jb; j < j0; ++j) {
    const long long o = static_cast<long long>(j - jb) * kS2Ld;
    split_store(carry[(j % kCarry) * kSpecLd + k], hi + o + k, lo + o + k);
    split_store(carry[(j % kCarry) * kSpecLd + kBins + k], hi + o + kBins + k, lo + o + kBins + k);
  }
  if (j1 == j0) return;
  const int a0 = it.a0[i], T = it.T[i];
  const float* sp = spec + static_cast<long long>(it.rb[i]) * kSpecLd;
  int ca = -1;             // frame held in (cn, cp): consecutive output frames mostly share their analysis frames
  double cn = 0.0, cp = 0.0;
  auto frame = [&](int a, double* nrm, double* ang) {
    if (a == ca) {
      *nrm = cn, *ang = cp;
      return;
    }
    double re = 0.0, im = 0.0;
    if (a < T) {
      const float* f = sp + static_cast<long long>(a - a0) * kSpecLd;
      re = f[k], im = f[kBins + k];
    }
    *nrm = hypot(re, im), *ang = atan2(im, re);
    ca = a, cn = *nrm, cp = *ang;
  };
  double acc;
  if (j0 == 0) {
    double nrm;
    frame(0, &nrm, &acc);
  } else {
    acc = *accp;
  }
  const double r = it.r[i], adv = phase_advance(k);
  for (int j = j0; j < j1; ++j) {
    // torchaudio: frames time_steps.long() and (time_steps + 1).long(); the second is floor(tau) + 2 when tau + 1
    // rounds up to an integer
    const double tau = static_cast<double>(j) * r, f = floor(tau), alpha = tau - f;
    double n0, p0, n1, p1;
    frame(static_cast<int>(f), &n0, &p0);
    frame(static_cast<int>(tau + 1.0), &n1, &p1);
    const double mag = alpha * n1 + (1.0 - alpha) * n0;
    double s, c;
    sincos(acc, &s, &c);
    const float re = static_cast<float>(mag * c), im = static_cast<float>(mag * s);
    const long long o = static_cast<long long>(j - jb) * kS2Ld;
    split_store(re, hi + o + k, lo + o + k);
    split_store(im, hi + o + kBins + k, lo + o + kBins + k);
    if (j >= j1 - kCarry) carry[(j % kCarry) * kSpecLd + k] = re, carry[(j % kCarry) * kSpecLd + kBins + k] = im;
    acc = wrap_pi(acc + (wrap_pi(p1 - p0 - adv) + adv));
  }
  *accp = acc;
}

// grid (blocks, rows): output sample e of a row is x_ola[e + 512] / envelope, frames summed in ascending order
__global__ void __launch_bounds__(256) ola_kernel(const __grid_constant__ Items it, const float* __restrict__ frames,
                                                  const float* __restrict__ win2, float* out) {
  const int i = blockIdx.y;
  const long long e0 = it.e0[i], span = it.e1[i] - e0;
  const int jb = it.jb[i], j1 = it.j1[i];
  const float* fr = frames + static_cast<long long>(it.sb[i]) * kNfft;
  float* o = out + it.out_off[i];
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < span;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = e0 + t + kNfft / 2;
    const long long jhi = std::min<long long>(p / kHop, j1 - 1);
    const long long jlo = std::max<long long>(0, (p - (kNfft - 1) + kHop - 1) / kHop);
    float acc = 0.f, env = 0.f;
    for (long long j = jlo; j <= jhi; ++j) {
      const int m = static_cast<int>(p - j * kHop);
      acc += fr[(j - jb) * kNfft + m];
      env += __ldg(win2 + m);
    }
    o[t] = env > 0.f ? acc / env : 0.f;
  }
}

// windowed bases in float64, split once into 3xTF32 halves: lo = the float64 value minus hi, rounded to fp32
void make_table(std::vector<float>& tab) {
  tab.assign(kTableBytes / 4, 0.f);
  auto hi_of = [](double v) {
    const float f = static_cast<float>(v);
    uint32_t u;
    std::memcpy(&u, &f, 4);
    u = (u + 0x1000u) & 0xffffe000u;
    float h;
    std::memcpy(&h, &u, 4);
    return h;
  };
  auto put = [&](float* hi, float* lo, double v) {
    *hi = hi_of(v);
    *lo = static_cast<float>(v - *hi);
  };
  std::vector<double> win(kNfft);
  for (int m = 0; m < kNfft; ++m) win[m] = 0.5 - 0.5 * std::cos(2.0 * M_PI * m / kNfft);   // periodic Hann
  float* wa = tab.data();
  float* ws = wa + kWaFloats;
  float* w2 = ws + kWsFloats;
  const size_t wa_lo = size_t(kSpecN) * kNfft, ws_lo = size_t(kNfft) * kS2Ld;
  for (int k = 0; k < kBins; ++k)
    for (int m = 0; m < kNfft; ++m) {
      const double ang = 2.0 * M_PI * static_cast<double>((static_cast<long long>(k) * m) % kNfft) / kNfft;
      const size_t re = size_t(k) * kNfft + m, im = size_t(kBins + k) * kNfft + m;
      put(wa + re, wa + wa_lo + re, win[m] * std::cos(ang));     // X_k = sum_m x_m w_m e^{-i ang}
      put(wa + im, wa + wa_lo + im, -win[m] * std::sin(ang));
      // irfft (Im of bins 0 and 512 ignored) times the window: y_m = w_m / N (sum_k c_k (Re_k cos - Im_k sin))
      const double ck = (k == 0 || k == kBins - 1) ? 1.0 : 2.0;
      const size_t sre = size_t(m) * kS2Ld + k, sim = size_t(m) * kS2Ld + kBins + k;
      put(ws + sre, ws + ws_lo + sre, win[m] * ck * std::cos(ang) / kNfft);
      put(ws + sim, ws + ws_lo + sim, (k == 0 || k == kBins - 1) ? 0.0 : -win[m] * ck * std::sin(ang) / kNfft);
    }
  for (int m = 0; m < kNfft; ++m) w2[m] = static_cast<float>(win[m] * win[m]);
}

bool rate_ok(double r) { return std::isfinite(r) && r >= kMinRate && r <= kMaxRate; }

}  // namespace
}  // namespace nt

using namespace nt;

// host mirror of one row's stream (the device state is the history, the accumulators and the carried frames)
struct StretchRow {
  long long recv = 0;   // input samples received since the reset
  long long emitted = 0;
  int J = 0;            // output frames computed
  int par = 0;          // history buffer holding the held samples
  bool bound = false;   // speed fixed by the first push
  double r = 1.0;
};

struct nt_stretch {
  int max_rows = 0, n_sms = 0;
  float* table = nullptr;
  char* state = nullptr;
  char* scratch = nullptr;
  std::vector<StretchRow> rows;
};

namespace {

long long floor_tau(long long j, double r) { return static_cast<long long>(static_cast<double>(j) * r); }
long long next_frame(long long j, double r) { return static_cast<long long>(static_cast<double>(j) * r + 1.0); }

// output frames ready once n samples arrived: j with 256 next_frame(j) + 512 <= n (a prefix: next_frame grows with j)
long long frames_ready(long long n, double r) {
  if (n < kNfft - kHop) return 0;
  const long long G = (n - kNfft / 2) / kHop;
  long long j = static_cast<long long>(std::ceil(static_cast<double>(G) / r));
  while (j > 0 && next_frame(j - 1, r) > G) --j;
  while (next_frame(j, r) <= G) ++j;
  return j;
}

long long frames_total(long long L, double r) { return static_cast<long long>(std::ceil(static_cast<double>(1 + L / kHop) / r)); }
long long out_total(long long L, double r) { return static_cast<long long>(std::nearbyint(static_cast<double>(L) / r)); }
long long emitted_after(long long n, bool fin, double r) {
  return fin ? out_total(n, r) : std::max(0ll, kHop * frames_ready(n, r) - kNfft / 2);
}

struct Work {
  StretchRow* m;
  char* st;
  const float* in;      // device pointer to this item's input
  long long n, done;    // input samples, consumed so far
  bool fin;
  long long out;        // device offset of the next output sample
};

int run_round(nt_stretch* S, std::vector<Work*>& ws, const float* in, float* out, cudaStream_t s) {
  Items it;
  std::memset(&it, 0, sizeof(it));
  int ra = 0, rs = 0;
  long long max_len = 0, max_span = 0;
  const int m = static_cast<int>(ws.size());
  for (int i = 0; i < m; ++i) {
    Work& w = *ws[i];
    StretchRow& row = *w.m;
    const double r = row.r;
    const int n = static_cast<int>(std::min<long long>(kChunk, w.n - w.done));
    const bool fin = w.fin && w.done + n == w.n;
    const long long recv = row.recv + n;
    const long long a0 = floor_tau(row.J, r);
    const long long held = row.recv + kNfft / 2 - kHop * a0;
    const long long j1 = fin ? frames_total(recv, r) : frames_ready(recv, r);
    const long long T = 1 + recv / kHop;
    const long long e1 = emitted_after(recv, fin, r);
    long long nfa = 0;
    if (j1 > row.J) {
      long long a1 = next_frame(j1 - 1, r);
      if (fin) a1 = std::min(a1, T - 1);
      nfa = std::max(0ll, a1 - a0 + 1);
    }
    const long long jb = std::max(0, row.J - kCarry);
    const long long nfs = (j1 > row.J || e1 > row.emitted) ? j1 - jb : 0;
    long long drop = 0, keep = 0;
    if (!fin) {
      drop = kHop * (floor_tau(j1, r) - a0);
      keep = held + n - drop;
    }
    if (nfa > kMaxA || nfs > kMaxS || held > kHistCap || keep < 0 || keep > kHistCap || drop < 0 || j1 > INT_MAX / 2 ||
        e1 < row.emitted)
      return set_error(NT_ERR_STATE, "nt_stretch_push: round plan out of bounds (frames %lld / %lld, history %lld)", nfa, nfs, keep);
    it.st[i] = w.st;
    it.in_off[i] = (w.in - in) + w.done;
    it.out_off[i] = w.out;
    it.e0[i] = row.emitted, it.e1[i] = e1;
    it.r[i] = r;
    it.n[i] = n;
    it.held[i] = static_cast<int>(held);
    it.keep[i] = static_cast<int>(keep), it.drop[i] = static_cast<int>(drop);
    it.flags[i] = (fin ? 1 : 0) | (row.recv == 0 ? 2 : 0) | (row.par << 2);
    it.rb[i] = ra, it.nfa[i] = static_cast<int>(nfa), it.a0[i] = static_cast<int>(a0);
    it.sb[i] = rs, it.jb[i] = static_cast<int>(jb), it.j0[i] = row.J, it.j1[i] = static_cast<int>(j1);
    it.T[i] = fin ? static_cast<int>(T) : INT_MAX;
    ra += nfa ? static_cast<int>(nfa) + 3 : 0;
    rs += static_cast<int>(nfs);
    max_len = std::max(max_len, std::max(keep, nfa ? (nfa + 3) * kHop : 0));
    max_span = std::max(max_span, e1 - row.emitted);
    w.out += e1 - row.emitted;
    w.done += n;
    if (fin) {
      *w.m = StretchRow();
    } else {
      row.recv = recv, row.J = static_cast<int>(j1), row.emitted = e1, row.par ^= 1, row.bound = true;
    }
  }
  float* A = reinterpret_cast<float*>(S->scratch + kOffA);
  float* spec = reinterpret_cast<float*>(S->scratch + kOffSpec);
  float* S2 = reinterpret_cast<float*>(S->scratch + kOffS2);
  float* fr = reinterpret_cast<float*>(S->scratch + kOffFr);
  const float* wa = S->table;
  const float* wsyn = S->table + kWaFloats;
  const float* win2 = wsyn + kWsFloats;
  const int per_row = std::max(1, (2 * S->n_sms + m - 1) / m);
  if (max_len > 0) {
    const int gx = static_cast<int>(std::min<long long>(per_row, (max_len + 255) / 256));
    if (int rc = launch_kernel(pack_kernel, dim3(gx, m), dim3(256), 0, s, false, it, in, A)) return rc;
  }
  if (ra > 3) {
    nt_gemm_args a;
    std::memset(&a, 0, sizeof(a));
    a.dtype = NT_TF32;
    a.M = ra - 3, a.N = kSpecN, a.K = kNfft;
    a.A = A, a.lda = kHop, a.W = wa, a.ldw = kNfft;
    a.out_f32 = spec, a.ldc = kSpecLd;
    const Split3 s3{kCapA, kSpecN};
    if (int rc = gemm_dispatch(a, s, nullptr, true, &s3, nullptr, 64)) return rc;
  }
  if (rs > 0) {
    if (int rc = launch_kernel(vocoder_kernel, dim3((kBins + 127) / 128, m), dim3(128), 0, s, false, it, (const float*)spec, S2))
      return rc;
    nt_gemm_args a;
    std::memset(&a, 0, sizeof(a));
    a.dtype = NT_TF32;
    a.M = rs, a.N = kNfft, a.K = kS2Ld;
    a.A = S2, a.lda = kS2Ld, a.W = wsyn, a.ldw = kS2Ld;
    a.out_f32 = fr, a.ldc = kNfft;
    const Split3 s3{kCapS, kNfft};
    if (int rc = gemm_dispatch(a, s, nullptr, true, &s3, nullptr, 64)) return rc;
  }
  if (max_span > 0) {
    const int gx = static_cast<int>(std::min<long long>(per_row, (max_span + 255) / 256));
    if (int rc = launch_kernel(ola_kernel, dim3(gx, m), dim3(256), 0, s, false, it, (const float*)fr, win2, out)) return rc;
  }
  return NT_OK;
}

}  // namespace

extern "C" int nt_stretch_query(nt_stretch_info* info) {
  if (!info) return set_error(NT_ERR_INVALID, "nt_stretch_query: null info");
  info->n_fft = kNfft;
  info->hop = kHop;
  info->max_items = kMaxItems;
  info->chunk = kChunk;
  info->spec_ld = kSpecLd;
  info->stretch_ld = kS2Ld;
  info->stretch_lo_rows = kCapS;
  info->table_bytes = kTableBytes;
  info->row_bytes = kRowBytes;
  info->scratch_bytes = kScratchBytes;
  return NT_OK;
}

extern "C" int nt_stretch_create(int max_rows, void* table, void* state, void* scratch, nt_stretch** out) {
  if (max_rows < 0) return set_error(NT_ERR_INVALID, "max_rows %d is negative", max_rows);
  if (!table || !scratch || !out || (max_rows > 0 && !state)) return set_error(NT_ERR_INVALID, "nt_stretch_create: null argument");
  if ((reinterpret_cast<uintptr_t>(table) | reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(scratch)) & 255)
    return set_error(NT_ERR_INVALID, "table, state and scratch must be 256-byte aligned");
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess || prop.major != 9 ||
      prop.minor != 0)
    return set_error(NT_ERR_CUDA, "no sm_90 CUDA device: this library has no CPU fallback");
  std::vector<float> tab;
  make_table(tab);
  NT_CUDA_CHECK(cudaMemcpy(table, tab.data(), kTableBytes, cudaMemcpyHostToDevice));
  nt_stretch* S = new nt_stretch();
  S->max_rows = max_rows;
  S->n_sms = prop.multiProcessorCount;
  S->table = static_cast<float*>(table);
  S->state = static_cast<char*>(state);
  S->scratch = static_cast<char*>(scratch);
  S->rows.assign(max_rows, StretchRow());
  *out = S;
  return NT_OK;
}

extern "C" int nt_stretch_destroy(nt_stretch* S) {
  delete S;
  return NT_OK;
}

extern "C" int nt_stretch_reset(nt_stretch* S, const int32_t* rows, int n) {
  if (!S || (n > 0 && !rows) || n < 0) return set_error(NT_ERR_INVALID, "nt_stretch_reset: bad argument");
  for (int i = 0; i < n; ++i)
    if (rows[i] < 0 || rows[i] >= S->max_rows) return set_error(NT_ERR_INVALID, "row %d not in 0..%d", rows[i], S->max_rows - 1);
  for (int i = 0; i < n; ++i) S->rows[rows[i]] = StretchRow();
  return NT_OK;
}

extern "C" int nt_stretch_push(nt_stretch* S, int n, const int32_t* rows, const int32_t* final_flags, const double* speeds,
                               const float* in, const int64_t* in_offsets, float* out, const int64_t* out_offsets,
                               void* stream) {
  if (!S || n < 0 || (n > 0 && (!in_offsets || !out_offsets || !speeds)))
    return set_error(NT_ERR_INVALID, "nt_stretch_push: bad argument");
  if (n == 0) return NT_OK;
  if (in_offsets[0] < 0 || out_offsets[0] < 0) return set_error(NT_ERR_INVALID, "negative offset");
  std::vector<uint8_t> seen(rows ? S->max_rows : 0, 0);
  for (int i = 0; i < n; ++i) {
    const long long ni = in_offsets[i + 1] - in_offsets[i], span = out_offsets[i + 1] - out_offsets[i];
    if (ni < 0 || span < 0) return set_error(NT_ERR_INVALID, "item %d: offsets must not decrease", i);
    if (ni > (1ll << 32)) return set_error(NT_ERR_INVALID, "item %d: %lld input samples in one push (limit 2^32)", i, ni);
    const double r = speeds[i];
    if (!rate_ok(r)) return set_error(NT_ERR_INVALID, "item %d: speed %g is not in [0.5, 2.0]", i, r);
    StretchRow row;
    bool fin = true;
    if (rows) {
      const int rw = rows[i];
      if (rw < 0 || rw >= S->max_rows) return set_error(NT_ERR_INVALID, "row %d not in 0..%d", rw, S->max_rows - 1);
      if (seen[rw]) return set_error(NT_ERR_INVALID, "row %d appears twice in one push", rw);
      seen[rw] = 1;
      row = S->rows[rw];
      if (row.bound && row.r != r)
        return set_error(NT_ERR_INVALID, "row %d: speed %g differs from its stream's %g (reset the row to change it)", rw, r, row.r);
      fin = final_flags && final_flags[i];
    }
    const long long recv = row.recv + ni;
    if (recv > (1ll << 32)) return set_error(NT_ERR_INVALID, "row stream of %lld samples (limit 2^32)", recv);
    const long long want = emitted_after(recv, fin, r) - row.emitted;
    if (span != want)
      return set_error(NT_ERR_INVALID, "item %d: output span %lld, but %lld samples are final after this push", i, span, want);
  }
  if (in_offsets[n] > in_offsets[0] && !in) return set_error(NT_ERR_INVALID, "nt_stretch_push: null input");
  if (out_offsets[n] > out_offsets[0] && !out) return set_error(NT_ERR_INVALID, "nt_stretch_push: null output");

  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::vector<StretchRow> oneshot(rows ? 0 : std::min(n, kMaxItems));
  for (int g0 = 0; g0 < n; g0 += kMaxItems) {
    const int gm = std::min(kMaxItems, n - g0);
    std::vector<Work> work(gm);
    for (int i = 0; i < gm; ++i) {
      const int k = g0 + i;
      Work& w = work[i];
      if (rows) {
        w.m = &S->rows[rows[k]];
        w.st = S->state + static_cast<size_t>(rows[k]) * kRowBytes;
        w.fin = final_flags && final_flags[k];
      } else {
        oneshot[i] = StretchRow();
        w.m = &oneshot[i];
        w.st = S->scratch + kOffStates + static_cast<size_t>(i) * kRowBytes;
        w.fin = true;
      }
      w.m->r = speeds[k];
      w.m->bound = true;
      w.in = in + in_offsets[k];
      w.n = in_offsets[k + 1] - in_offsets[k];
      w.done = 0;
      w.out = out_offsets[k];
    }
    // rounds: every row with input left (or a final push not yet made) takes up to kChunk samples
    std::vector<bool> closed(gm, false);
    for (;;) {
      std::vector<Work*> ws;
      for (int i = 0; i < gm; ++i) {
        Work& w = work[i];
        if (w.done < w.n || (w.fin && !closed[i])) {
          ws.push_back(&w);
          if (w.fin && w.n - w.done <= kChunk) closed[i] = true;
        }
      }
      if (ws.empty()) break;
      if (int rc = run_round(S, ws, in, out, s)) return rc;
    }
  }
  return NT_OK;
}

extern "C" void* nt_stretch_debug_ptr(nt_stretch* S, const char* name) {
  if (!S || !name) return nullptr;
  if (!std::strcmp(name, "spec")) return S->scratch + kOffSpec;
  if (!std::strcmp(name, "stretch")) return S->scratch + kOffS2;
  if (!std::strcmp(name, "frames")) return S->scratch + kOffFr;
  return nullptr;
}
