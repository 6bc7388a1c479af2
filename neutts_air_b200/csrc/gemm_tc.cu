// wgmma GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] . W[N,K]^T), fp32 accumulation in registers.
//
//   - operands K-major in global memory, tiles of 128 bytes along K (64 bf16 / 32 tf32)
//     staged by TMA (SWIZZLE_128B) into a multi-stage shared-memory ring;
//   - one warpgroup (warps 4..7) issues wgmma.mma_async (two M=64 halves of the 128-row tile, N=BN,
//     K=16|8 per instruction) and keeps the accumulator tile in registers;
//   - once the K loop has drained the ring, the accumulators go through shared memory (the ring) so that each
//     thread owns one output row, and the same four warps apply bias / residual / SiLU / SwiGLU before writing
//     fp32 and/or bf16 rows;
//   - Conv1d is the same kernel: the K loop walks (tap, channel-block) and shifts the A row
//     coordinate by `tap`, so no im2col buffer exists anywhere.
//
// Replaces, for the hot path: torch addmm/mm behind transformers modeling_qwen2.py:46-48
// (MLP), :217-219 (q/k/v), :244 (o_proj), :475 (lm_head) and the codec's Linear / Conv1d
// layers (SURVEY.md §8a rows A2, A4, A8-A10, B2-B6).
#include <cstdlib>

#define NT_WGMMA_KERNELS
#include "common.cuh"
#include "internal.h"

namespace nt {

struct GemmEpilogue {
  const float* bias;
  const float* residual;
  long long ldr;
  int act;  // nt_act
  float* out_f32;
  __nv_bfloat16* out_bf16;
  long long ldc;
  int valid_period, valid_len;
  int split_k;             // > 1: grid.z K-slices; slice z stores its raw partial sums at out_f32 + z * split_stride
  long long split_stride;  // (no residual / activation; bias rides on slice 0) -- the consumer adds them in z order
  int w_const;             // W is never written on the device: its first ring of tiles may load before the PDL wait
  int w_stream;            // W is read exactly once by this launch (one row tile): fetch it with the L2 evict_first policy
  float* tile_max;         // optional [M][tile_ld]: maximum of the row's stored values inside this CTA's BN columns (lm_head ->
                           //   tile-max sampler); plain fp32 epilogue only
  long long tile_ld;
};

// kShallow: half-depth ring (<= 113 KB of shared memory) for grids of more than one wave of CTAs.
// kS3 (tf32 only): 3xTF32 in ONE pass.  Both operands arrive as hi/lo halves (hi = the value rounded to TF32, lo = the
// exact remainder), the lo half stored `*_lo_rows` rows below the hi half in the same matrix, so one tensor map per
// operand serves both; a stage holds A_hi | A_lo | W_hi | W_lo and every k-block issues A_lo.W_hi, A_hi.W_lo, A_hi.W_hi
// into the same accumulators: fp32-grade products on the TF32 pipe without intermediate round trips to HBM.
template <int BN, bool kShallow = false, bool kS3 = false>
struct GemmCfg {
  static constexpr int BM = 128;
  static constexpr int A_BYTES = BM * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = (kS3 ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr int STAGES = kS3 ? (BN == 128 ? 3 : (BN == 64 ? 4 : 5))
                                    : (kShallow ? (BN <= 64 ? 4 : 3) : ((BN <= 64) ? 8 : (BN == 128 ? 6 : 4)));
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int OUT_LD = BN + 4;   // fp32 row stride of the accumulator tile staged in the drained ring
  static_assert(BM * OUT_LD * 4 <= STAGES * STAGE_BYTES, "accumulator staging must fit the ring");
};

template <int kFmt, int BN, bool kShallow, bool kS3 = false>
__global__ void __launch_bounds__(256, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmEpilogue ep, int M,
               int N, int num_kb, int kb_per_tap, int a_lo_rows, int w_lo_rows) {
  using Cfg = GemmCfg<BN, kShallow, kS3>;
  constexpr int W_OFF = (kS3 ? 2 : 1) * Cfg::A_BYTES;   // byte offset of the W tile(s) inside a stage
  constexpr int STAGES = Cfg::STAGES;
  constexpr int BK_ELEMS = (kFmt == 2) ? 32 : 64;  // 128 bytes along K

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  uint8_t* tiles = smem_raw + pad;  // 1024-byte aligned (SWIZZLE_128B atoms)
  uint64_t* bars = reinterpret_cast<uint64_t*>(tiles + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  const int warp = uniform(warp_id());   // provably warp-uniform: role branches below stay convergent (elect_one())
  const int lane = lane_id();
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * Cfg::BM;
  // split-K: this CTA owns k-blocks [kb_lo, kb_hi)
  const int kb_lo = ep.split_k > 1 ? static_cast<int>((static_cast<long long>(num_kb) * blockIdx.z) / ep.split_k) : 0;
  const int kb_hi = ep.split_k > 1 ? static_cast<int>((static_cast<long long>(num_kb) * (blockIdx.z + 1)) / ep.split_k) : num_kb;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);   // one arrival per MMA warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  // Programmatic dependent launch: let the next kernel's CTAs start their prologue now (they block in their own
  // griddepcontrol.wait until this grid has completed), and start streaming this kernel's weights -- which no
  // kernel ever writes -- while the previous kernel is still finishing.
  pdl_launch_dependents();
  const int early = ep.w_const ? min(STAGES, kb_hi - kb_lo) : 0;
  const uint64_t wpol = ep.w_stream ? l2_policy_evict_first() : 0ull;
  auto load_w = [&](void* dst, int c0, int c1, uint64_t* bar) {
    if (wpol) tma_load_2d_hint(dst, &tmB, c0, c1, bar, wpol);
    else tma_load_2d(dst, &tmB, c0, c1, bar);
  };
  if (warp == 0) {
    if (elect_one()) {
      for (int i = 0; i < early; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], Cfg::STAGE_BYTES);
        load_w(tiles + i * Cfg::STAGE_BYTES + W_OFF, (kb_lo + i) * BK_ELEMS, n0, &full_bar[i]);
        if (kS3) load_w(tiles + i * Cfg::STAGE_BYTES + W_OFF + Cfg::B_BYTES, (kb_lo + i) * BK_ELEMS, n0 + w_lo_rows, &full_bar[i]);
      }
    }
  }
  pdl_wait();  // inputs (A, residual) may come from the previous kernel in the stream

  // Producer warp: warp-uniform loop, the TMA instructions under the elect.sync predicate (see elect_one() in
  // common.cuh).
  if (warp == 0) {
    // ------------------------------------------------------------ TMA producer
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      const int s = (kb - kb_lo) % STAGES;
      const uint32_t ph = ((kb - kb_lo) / STAGES) & 1;
      const bool b_in_flight = (kb - kb_lo) < early;
      if (!b_in_flight) mbar_wait(&empty_bar[s], ph ^ 1);
      if (elect_one()) {   // re-elected after every wait: elect.sync is also where the lanes reconverge
        if (!b_in_flight) mbar_arrive_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
        uint8_t* sa = tiles + s * Cfg::STAGE_BYTES;
        uint8_t* sb = sa + W_OFF;
        const int tap = kb / kb_per_tap;
        const int acol = (kb - tap * kb_per_tap) * BK_ELEMS;
        tma_load_2d(sa, &tmA, acol, m0 + tap, &full_bar[s]);
        if (kS3) tma_load_2d(sa + Cfg::A_BYTES, &tmA, acol, m0 + tap + a_lo_rows, &full_bar[s]);
        if (!b_in_flight) {
          load_w(sb, kb * BK_ELEMS, n0, &full_bar[s]);
          if (kS3) load_w(sb + Cfg::B_BYTES, kb * BK_ELEMS, n0 + w_lo_rows, &full_bar[s]);
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------ MMA warpgroup + epilogue
    // acc0 = rows [0, 64) of the tile, acc1 = rows [64, 128); one k-block's MMAs form a commit group, and the ring
    // slot of a k-block is released once the next group has been issued and the older one retired.
    float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
    const uint32_t tiles_addr = smem_u32(tiles);
    auto mma = [&](uint64_t ad, uint64_t bd) {
      if constexpr (kFmt == 2) {
        wgmma_tf32<BN>(acc0, ad, bd, 1u);
        wgmma_tf32<BN>(acc1, ad + 512, bd, 1u);
      } else {
        wgmma_bf16<BN>(acc0, ad, bd, 1u);
        wgmma_bf16<BN>(acc1, ad + 512, bd, 1u);
      }
    };
    int prev = -1;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      const int s = (kb - kb_lo) % STAGES;
      const uint32_t ph = ((kb - kb_lo) / STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint32_t sa = tiles_addr + static_cast<uint32_t>(s) * Cfg::STAGE_BYTES;
      const uint32_t sb = sa + W_OFF;
      const uint64_t adesc = wgmma_desc_sw128(sa);
      const uint64_t bdesc = wgmma_desc_sw128(sb);
      wgmma_fence();
      if (kS3) {   // small terms first: A_lo.W_hi, A_hi.W_lo, then A_hi.W_hi
        const uint64_t alo = wgmma_desc_sw128(sa + Cfg::A_BYTES), blo = wgmma_desc_sw128(sb + Cfg::B_BYTES);
#pragma unroll
        for (int k = 0; k < 4; ++k) mma(alo + 2 * k, bdesc + 2 * k);
#pragma unroll
        for (int k = 0; k < 4; ++k) mma(adesc + 2 * k, blo + 2 * k);
#pragma unroll
        for (int k = 0; k < 4; ++k) mma(adesc + 2 * k, bdesc + 2 * k);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) mma(adesc + 2 * k, bdesc + 2 * k);  // 4 x 32 bytes of K per stage
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);   // frees the smem slot of the previous k-block
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    // every TMA load of this CTA has been consumed: the ring is free to hold the fp32 tile [128][OUT_LD]
    asm volatile("bar.sync 1, 128;" ::: "memory");
    float* stage = reinterpret_cast<float*>(tiles);
    wgmma_store_rows<BN>(acc0, stage, Cfg::OUT_LD, 0);
    wgmma_store_rows<BN>(acc1, stage, Cfg::OUT_LD, 64);
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int q = warp - 4;  // rows [32 q, 32 q + 32) of the tile, one per lane
    const float* srow = stage + (q * 32 + lane) * Cfg::OUT_LD;
    const int row = m0 + q * 32 + lane;
    bool row_ok = row < M;
    if (ep.valid_period > 0 && (row % ep.valid_period) >= ep.valid_len) row_ok = false;
    float tmx = -INFINITY;
#pragma unroll 1
    for (int c = 0; c < BN / 32; ++c) {
      const int col0 = n0 + c * 32;
      if (!row_ok || col0 >= N) continue;
      float v[32];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 t = reinterpret_cast<const float4*>(srow + c * 32)[j];
        v[4 * j] = t.x, v[4 * j + 1] = t.y, v[4 * j + 2] = t.z, v[4 * j + 3] = t.w;
      }
      const bool full = (col0 + 32 <= N);
      if (ep.split_k > 1) {
        float* dst = ep.out_f32 + blockIdx.z * ep.split_stride + row * ep.ldc + col0;
        if (ep.bias && blockIdx.z == 0) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (full || col0 + j < N) v[j] += __ldg(ep.bias + col0 + j);
        }
        if (full && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
          for (int j = 0; j < 8; ++j) reinterpret_cast<float4*>(dst)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        } else {
          for (int j = 0; j < 32; ++j)
            if (col0 + j < N) dst[j] = v[j];
        }
        continue;
      }
      if (ep.bias) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (full || col0 + j < N) v[j] += __ldg(ep.bias + col0 + j);
      }
      if (ep.act == NT_ACT_SWIGLU) {
        // (gate, up) interleaved on the N axis -> 16 outputs
        const long long ocol0 = col0 >> 1;
        float o[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) o[j] = silu(v[2 * j]) * v[2 * j + 1];
        const int nvalid = full ? 16 : ((N - col0) >> 1);
        if (ep.out_bf16) {
          __nv_bfloat16* dst = ep.out_bf16 + row * ep.ldc + ocol0;
          if (nvalid == 16 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
            uint4 p0 = make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                                  pack_bf16x2(o[6], o[7]));
            uint4 p1 = make_uint4(pack_bf16x2(o[8], o[9]), pack_bf16x2(o[10], o[11]), pack_bf16x2(o[12], o[13]),
                                  pack_bf16x2(o[14], o[15]));
            reinterpret_cast<uint4*>(dst)[0] = p0;
            reinterpret_cast<uint4*>(dst)[1] = p1;
          } else {
            for (int j = 0; j < nvalid; ++j) dst[j] = __float2bfloat16(o[j]);
          }
        }
        if (ep.out_f32) {
          float* dst = ep.out_f32 + row * ep.ldc + ocol0;
          for (int j = 0; j < nvalid; ++j) dst[j] = o[j];
        }
        continue;
      }
      if (ep.residual) {
        const float* r = ep.residual + row * ep.ldr + col0;
        if (full && ((reinterpret_cast<uintptr_t>(r) & 15) == 0)) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 t = reinterpret_cast<const float4*>(r)[j];
            v[4 * j] += t.x, v[4 * j + 1] += t.y, v[4 * j + 2] += t.z, v[4 * j + 3] += t.w;
          }
        } else {
          for (int j = 0; j < 32; ++j)
            if (col0 + j < N) v[j] += r[j];
        }
      }
      if (ep.act == NT_ACT_SILU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = silu(v[j]);
      }
      if (ep.tile_max) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (full || col0 + j < N) tmx = fmaxf(tmx, v[j]);
      }
      if (ep.out_f32) {
        float* dst = ep.out_f32 + row * ep.ldc + col0;
        if (full && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            reinterpret_cast<float4*>(dst)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        } else {
          for (int j = 0; j < 32; ++j)
            if (col0 + j < N) dst[j] = v[j];
        }
      }
      if (ep.out_bf16) {
        __nv_bfloat16* dst = ep.out_bf16 + row * ep.ldc + col0;
        if (full && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            reinterpret_cast<uint4*>(dst)[j] =
                make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                           pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
        } else {
          for (int j = 0; j < 32; ++j)
            if (col0 + j < N) dst[j] = __float2bfloat16(v[j]);
        }
      }
    }
    if (ep.tile_max && row_ok) ep.tile_max[static_cast<long long>(row) * ep.tile_ld + blockIdx.x] = tmx;
  }
}

// ------------------------------------------------------------------------------------------ host side

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

// rows x cols (elements) matrix with row stride ld (elements); box = box_rows x 128 bytes.
int make_tmap(CUtensorMap* out, nt_dtype dt, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                     uint32_t box_rows) {
  PFN_tmapEncodeTiled fn = get_encode_fn();
  if (!fn) return set_error(NT_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  const uint32_t esz = (dt == NT_BF16) ? 2 : 4;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {ld * esz};
  cuuint32_t box[2] = {128 / esz, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dt == NT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(NT_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", int(r));
  return NT_OK;
}

template <int kFmt, int BN, bool kShallow, bool kS3 = false>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int M, int N, int num_kb,
                       int kb_per_tap, cudaStream_t stream, int a_lo_rows = 0, int w_lo_rows = 0) {
  const int splits = ep.split_k > 1 ? ep.split_k : 1;
  using Cfg = GemmCfg<BN, kShallow, kS3>;
  auto kern = gemm_tc_kernel<kFmt, BN, kShallow, kS3>;   // launch_kernel opts in to the dynamic shared memory per device
  dim3 grid((N + BN - 1) / BN, (M + Cfg::BM - 1) / Cfg::BM, splits);
  return launch_kernel(kern, grid, dim3(256), Cfg::SMEM_BYTES, stream, /*pdl=*/true, ta, tb, ep, M, N, num_kb,
                       kb_per_tap, a_lo_rows, w_lo_rows);
}

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// tile width the dispatcher picks for an M x N problem (callers that consume per-tile results need to know)
int gemm_tile_n(int M, int N, bool swiglu) {
  const int mt = (M + 127) / 128;
  int bn = 128;
  if (mt * ((N + 127) / 128) < num_sms() * 13 / 16) bn = 64;
  if (mt * ((N + 63) / 64) < num_sms() * 11 / 16) bn = 32;
  if (swiglu && bn < 64) bn = 64;
  return bn;
}

int gemm_dispatch(const nt_gemm_args& a, cudaStream_t stream, SplitK* split, bool w_const, const Split3* s3, float* tile_max, int bn_req,
                  long long tile_ld) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return set_error(NT_ERR_INVALID, "gemm: empty problem");
  const int esz = a.dtype == NT_BF16 ? 2 : 4;
  const int bk = 128 / esz;
  if ((a.lda * esz) % 16 || (a.ldw * esz) % 16) return set_error(NT_ERR_INVALID, "gemm: row strides must be 16-byte multiples");
  if ((reinterpret_cast<uintptr_t>(a.A) | reinterpret_cast<uintptr_t>(a.W)) & 15)
    return set_error(NT_ERR_INVALID, "gemm: operands must be 16-byte aligned");
  if (a.act == NT_ACT_SWIGLU && (a.N & 1)) return set_error(NT_ERR_INVALID, "gemm: SwiGLU needs even N");
  if (a.act == NT_ACT_SWIGLU && a.residual) return set_error(NT_ERR_INVALID, "gemm: SwiGLU + residual unsupported");
  if (!a.out_f32 && !a.out_bf16) return set_error(NT_ERR_INVALID, "gemm: no output");

  // Conv1d-as-GEMM: A rows overlap (lda < K) -> K loop walks taps, shifting the A row.
  int taps = 1;
  uint64_t a_cols = a.K;
  if (a.lda < a.K) {
    if (a.K % a.lda || a.lda % bk) return set_error(NT_ERR_INVALID, "gemm: overlapped A needs K %% lda == 0 and lda %% %d == 0", bk);
    taps = int(a.K / a.lda);
    a_cols = a.lda;
  }
  const int num_kb = (a.K + bk - 1) / bk;
  const int kb_per_tap = (taps > 1) ? int(a.lda / bk) : num_kb;
  // rows reachable through the tap shift must stay addressable: caller guarantees
  // A has M + taps - 1 rows.
  const uint64_t a_rows = uint64_t(a.M) + taps - 1;

  // tile-N choice: keep >= ~1 wave of CTAs when the problem allows it
  const int mt = (a.M + 127) / 128;
  const int bn = bn_req > 0 ? bn_req : gemm_tile_n(a.M, a.N, a.act == NT_ACT_SWIGLU);
  if (bn != 32 && bn != 64 && bn != 128) return set_error(NT_ERR_INVALID, "gemm: tile width %d not in {32, 64, 128}", bn);
  if (tile_max && (split || a.act != NT_ACT_NONE || a.out_bf16)) return set_error(NT_ERR_INVALID, "gemm: tile maxima need the plain fp32 epilogue");

  if (s3 && (a.dtype != NT_TF32 || split)) return set_error(NT_ERR_INVALID, "gemm: 3xTF32 needs tf32 operands and no split-K");
  CUtensorMap ta, tb;
  // 3xTF32: the lo halves lie a_lo_rows / w_lo_rows rows below the hi halves in the same matrices
  int rc = make_tmap(&ta, a.dtype, a.A, s3 ? uint64_t(s3->a_lo_rows) + a_rows : a_rows, a_cols, a.lda, 128);
  if (rc) return rc;
  rc = make_tmap(&tb, a.dtype, a.W, s3 ? uint64_t(s3->w_lo_rows) + a.N : a.N, a.K, a.ldw, bn);
  if (rc) return rc;

  GemmEpilogue ep;
  ep.bias = a.bias;
  ep.residual = a.residual;
  ep.ldr = a.ldr;
  ep.act = a.act;
  ep.out_f32 = a.out_f32;
  ep.out_bf16 = reinterpret_cast<__nv_bfloat16*>(a.out_bf16);
  ep.ldc = a.ldc;
  ep.valid_period = a.valid_period;
  ep.valid_len = a.valid_len;
  // split-K (only when the caller lends a workspace and will fold the slices itself): few tiles would leave most
  // SMs idle, so grid.z slices of the K loop store raw partial sums; the summation order stays fixed (z order)
  ep.split_k = 1;
  ep.split_stride = 0;
  ep.w_const = w_const ? 1 : 0;
  ep.tile_max = tile_max;
  ep.tile_ld = tile_ld > 0 ? tile_ld : (a.N + bn - 1) / bn;
  ep.w_stream = (w_const && mt == 1) ? 1 : 0;
  if (split) {
    split->used = 1;
    const int tiles = mt * ((a.N + bn - 1) / bn);
    const bool in_place = a.residual == a.out_f32 && a.ldr == a.ldc;
    if (tiles <= 48 && taps == 1 && a.act == NT_ACT_NONE && !a.out_bf16 && a.out_f32 && (in_place || !a.residual) &&
        a.valid_period == 0 && num_kb >= 8) {
      int sk = (num_sms() - 4) / tiles;
      if (sk > num_kb / 4) sk = num_kb / 4;
      if (sk > 8) sk = 8;
      const size_t slice = size_t(a.M) * size_t(a.ldc);
      if (sk > 1 && slice * sk <= split->ws_floats) {
        ep.split_k = sk, ep.split_stride = static_cast<long long>(slice);
        ep.out_f32 = split->ws, ep.residual = nullptr;
        split->used = sk, split->slice_stride = static_cast<long long>(slice);
      }
    }
  }

  const int ctas = mt * ((a.N + bn - 1) / bn) * (ep.split_k > 1 ? ep.split_k : 1);
  // Two CTAs per SM (half-depth ring) for every grid of more than one wave: one CTA's prologue / epilogue overlaps
  // the other's main loop, and grids just over a multiple of the SM count lose their short last wave.
  const bool shallow = ctas > num_sms();
#define NT_GEMM_CASE(FMT, BNV)                                                                           \
  return shallow ? launch_gemm<FMT, BNV, true>(ta, tb, ep, a.M, a.N, num_kb, kb_per_tap, stream)         \
                 : launch_gemm<FMT, BNV, false>(ta, tb, ep, a.M, a.N, num_kb, kb_per_tap, stream)
  if (s3) {
    if (bn == 128) return launch_gemm<2, 128, false, true>(ta, tb, ep, a.M, a.N, num_kb, kb_per_tap, stream, s3->a_lo_rows, s3->w_lo_rows);
    if (bn == 64) return launch_gemm<2, 64, false, true>(ta, tb, ep, a.M, a.N, num_kb, kb_per_tap, stream, s3->a_lo_rows, s3->w_lo_rows);
    return launch_gemm<2, 32, false, true>(ta, tb, ep, a.M, a.N, num_kb, kb_per_tap, stream, s3->a_lo_rows, s3->w_lo_rows);
  }
  if (a.dtype == NT_BF16) {
    if (bn == 128) NT_GEMM_CASE(1, 128);
    if (bn == 64) NT_GEMM_CASE(1, 64);
    NT_GEMM_CASE(1, 32);
  } else {
    if (bn == 128) NT_GEMM_CASE(2, 128);
    if (bn == 64) NT_GEMM_CASE(2, 64);
    NT_GEMM_CASE(2, 32);
  }
#undef NT_GEMM_CASE
}

}  // namespace nt

extern "C" int nt_gemm(const nt_gemm_args* args, void* stream) {
  if (!args) return nt::set_error(NT_ERR_INVALID, "nt_gemm: null args");
  return nt::gemm_dispatch(*args, reinterpret_cast<cudaStream_t>(stream), nullptr, /*w_const=*/false);
}
