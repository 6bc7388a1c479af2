// Host-side internals shared by the translation units of libneutts_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <utility>

#include "../../include/neutts_b200.h"

struct CUtensorMap_st;  // <cuda.h>

namespace nt {

int set_error(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
// Every kernel of the library asks for the maximum shared-memory carveout, so consecutive kernels never force the
// SM to switch its L1 / shared-memory split (the big-tile kernels need ~180 KB; the small ones do not use L1 much).
void prefer_max_smem_carveout(const void* kernel);
// opt-in to > 48 KB of dynamic shared memory, once per (kernel, device)
int ensure_dynamic_smem(const void* kernel, size_t bytes);

#define NT_CUDA_CHECK(expr)                                                                          \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return ::nt::set_error(NT_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Launch with optional programmatic-dependent-launch attribute (the kernel must call
// pdl_wait() before touching anything a predecessor writes).
template <typename... KArgs, typename... Args>
int launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                  Args&&... args) {
  prefer_max_smem_carveout(reinterpret_cast<const void*>(kernel));
  if (int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kernel), smem)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
  if (e != cudaSuccess) return set_error(NT_ERR_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return NT_OK;
}

// Optional split-K lease: when the GEMM accumulates in place (residual == out_f32) or has no residual, and has too
// few tiles to fill the GPU, it writes `used` raw partial slices [used][M][ldc] into ws instead of touching out_f32
// (bias rides on slice 0); the consumer must fold them in slice order (x += s0 + s1 + ... / y = s0 + s1 + ...)
// -- rmsnorm_rows and rope_append do.
struct SplitK {
  float* ws;
  size_t ws_floats;
  int used;                // out: 1 = no split happened (normal epilogue ran)
  long long slice_stride;  // out: floats between slices
};
// w_const: W holds model weights that no kernel writes, so the kernel may fetch them ahead of the PDL dependency
// 3xTF32 in one pass (gemm_tc.cu): a.A / a.W point at the hi halves, the lo halves lie a_lo_rows / w_lo_rows rows
// further down in the same matrices (same row strides)
struct Split3 {
  int a_lo_rows, w_lo_rows;
};
// tile_max (optional, plain fp32 epilogue): [M][ceil(N / gemm_tile_n)] maximum of every row inside every column tile
// (row pitch tile_ld when > 0).  bn > 0 forces the tile width (32 | 64 | 128): a GEMM over a column range of a wider
// matrix then runs the instruction shape, and so the arithmetic, of the GEMM over the whole matrix.
// ring >= 0 forces the shared-memory ring (0 deep, 1 shallow) instead of the choice by grid size (tests); the ring
// depth changes the pipelining only, never the arithmetic.  3xTF32 always runs the deep ring.
int gemm_dispatch(const nt_gemm_args& a, cudaStream_t stream, SplitK* split = nullptr, bool w_const = false,
                  const Split3* s3 = nullptr, float* tile_max = nullptr, int bn = 0, long long tile_ld = 0,
                  int ring = -1);
int gemm_tile_n(int M, int N, bool swiglu);
// Teacher-forced scoring: logits = A[M,K] . W[N,K]^T (bf16, K-major, row stride K) at a fixed 128-column tile, never
// stored.  Per row r and column tile t: lse[r * lse_ld + t] = (max, sum exp(v - max)) over the tile's columns < N; the
// tile holding tgt[r] also writes that logit to zt[r].  Each row's arithmetic is independent of M.
int gemm_logsoftmax(const void* A, int M, int K, const void* W, int N, const int32_t* tgt, float2* lse, long long lse_ld,
                    float* zt, cudaStream_t stream);

// 2-D TMA descriptor over a row-major matrix (rows x cols elements, row stride ld elements); box = box_rows x 128
// bytes, SWIZZLE_128B (gemm_tc.cu)
int make_tmap(::CUtensorMap_st* out, nt_dtype dt, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);

// workspace carving helper (256-byte aligned sub-allocations from a caller-owned buffer)
struct Arena {
  uint8_t* base;
  size_t size, off;
  Arena(void* p, size_t n) : base(static_cast<uint8_t*>(p)), size(n), off(0) {}
  template <typename T>
  T* take(size_t count) {
    size_t bytes = (count * sizeof(T) + 255) & ~size_t(255);
    T* r = reinterpret_cast<T*>(base ? base + off : nullptr);
    off += bytes;
    return r;
  }
  bool ok() const { return off <= size; }
};

}  // namespace nt
