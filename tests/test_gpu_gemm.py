"""Every wgmma GEMM instantiation of gemm_tc.cu against float64, at the edges of its tiles.

``nt_debug_gemm`` is nt_gemm with the dispatcher's internal choices exposed (tile width BN, ring depth, split-K
workspace, the 3xTF32 hi / lo layout, tile maxima); ``nt_debug_gemm_logsoftmax`` is the log-softmax epilogue of
teacher-forced scoring.  The 17 instantiations -- {bf16, tf32} x BN {32, 64, 128} x {deep, shallow ring}, 3xTF32 x BN
and log-softmax x ring -- are test parameters, so each runs here whatever BN and ring this GPU's SM count would make
the dispatcher pick for the model.  A few cases go through the public nt_gemm, so the dispatcher's own choice stays
covered too.

Arithmetic each mode is held to:
    bf16     float64 on the same operands.  bf16 x bf16 products are exact in fp32, so the only error is accumulation.
    tf32     float64 on the operands truncated to TF32 (the tensor core reads the top 19 bits of an fp32 operand);
             separately, against the product of the untruncated operands.
    3xtf32   float64 on the fp32 operands that the hi / lo halves add up to; plain TF32 on the same operands must
             show TF32_APART times 3xTF32's whole-matrix error.
Error measure: relative RMS per (row, 32-column chunk) -- the unit one epilogue lane writes -- over the RMS of the
row's product (for SwiGLU, times the sensitivity of its output to the product), so that one wrong chunk cannot be
averaged away and a bias or residual cannot dilute it.

Guards, data only: A and W hold NaN in their stride padding [K, ld) and in the rows past M / N; every output has
ldc > N and rows past M, and those cells and the rows a row mask skips hold a sentinel bit pattern that must survive
bit for bit.

Exact checks, the contracts of internal.h: the bf16 output is RNE of the same call's fp32 output; split-K slice z is
the product over k-blocks [num_kb z / used, num_kb (z + 1) / used) with the bias on slice 0 only, and out_f32 is not
touched; tile maxima are the maxima of the stored row values per column tile; a column range at a forced BN computes
what the whole matrix computes; log-softmax rows do not depend on M and share the max and the target logit with the
plain BN = 128 GEMM.  Deep and shallow rings give the same bits, and rows do not depend on M.

``test_fault_models_exceed_the_bars`` (CPU) shows that the faults these checks exist for land at least 10x past the
bars or break an exact check.
"""
from __future__ import annotations

import ctypes as C
import math
import subprocess

import pytest
import torch

from tests.helpers import tf32_truncate

# Worst errors measured on one H100 80GB HBM3 (132 SMs, 700 W power limit) over the whole case matrix -- every
# instantiation, shape and epilogue -- per mode and K, relative RMS per (row, 32-column chunk):
#   bf16          K = 16: 2.0e-7, 64: 3.2e-7, 72: 6.9e-7, 896: 8.0e-6, 4864: 2.2e-5
#   tf32          K = 8: 3.0e-7, 32: 7.6e-7, 40: 6.0e-7, 1024: 1.6e-5, 1922: 1.7e-5, 7168: 5.6e-5
#   tf32-exact    K = 8: 3.1e-3, 32: 3.2e-3, 40: 3.6e-3, 1024: 4.8e-3, 1922: 2.5e-3, 7168: 2.7e-3
#   3xtf32        K = 8: 4.4e-7, 32: 6.0e-7, 40: 9.1e-7, 1024: 2.7e-5, 1922: 5.0e-5, 7168: 1.6e-4
#   log-softmax   |lse - lse64| per (row, tile) 3.0e-6 (K = 896)
# The worst chunks are the narrow ones at the N edge (N = 33 leaves one column).  The error grows with K in every mode,
# 3xTF32 included: the tensor core's fp32 accumulation does not round to nearest, so at K >= 1024 the accumulation,
# not the operands, sets the bar.  The bars sit ~4x above:
BARS = {
    "bf16": {16: 8e-7, 64: 1.3e-6, 72: 2.8e-6, 896: 3.2e-5, 4864: 9e-5},
    "tf32": {8: 1.2e-6, 32: 3e-6, 40: 3e-6, 1024: 6.4e-5, 1922: 7e-5, 7168: 2.3e-4},
    "tf32-exact": {8: 1.3e-2, 32: 1.3e-2, 40: 1.4e-2, 1024: 2e-2, 1922: 1e-2, 7168: 1.1e-2},
    "3xtf32": {8: 1.8e-6, 32: 2.4e-6, 40: 3.7e-6, 1024: 1.1e-4, 1922: 2e-4, 7168: 6.4e-4},
    "lse": {896: 1.2e-5},
}
# plain TF32's whole-matrix error over 3xTF32's, on the same operands at the same BN; measured at least 15.2x (K = 7168),
# 54x (K = 1922), 105x (K = 1024), over 3000x (K <= 40)
TF32_APART = 4.0          # plain TF32 over 3xTF32, whole-matrix errors of the two kernels on the same operands
WORST: dict = {}
APART: dict = {}          # K -> smallest ratio of plain TF32's whole-matrix error to 3xTF32's, and where

STORE = [(m, bn, r) for m in ("bf16", "tf32") for bn in (32, 64, 128) for r in ("deep", "shallow")] + \
        [("3xtf32", bn, "deep") for bn in (32, 64, 128)]
STORE_IDS = [f"{m}-bn{bn}-{r}" for m, bn, r in STORE]
RING = {"deep": 0, "shallow": 1}
MS = (1, 7, 127, 128, 129, 1031)
NS = (17, 33, 130, 1922, 256)
KS = {"bf16": (16, 64, 72, 896, 4864), "tf32": (8, 32, 40, 1024, 1922, 7168)}
KS["3xtf32"] = KS["tf32"]
PAD_ROWS = 3
SENT32 = -0x21524111           # 0xDEADBEEF
SENT16 = -0x4111               # 0xBEEF
NAN = float("nan")


def bar_of(mode: str, K: int):
    """(key, bar) of ``mode`` at K: the bar of the smallest listed K >= K (the error grows with K)."""
    ks = sorted(BARS[mode])
    k = next((k for k in ks if k >= K), ks[-1])
    return k, BARS[mode][k]


def record(inst: str, mode: str, K: int, err: float, tag: str) -> None:
    k, b = bar_of(mode, K)
    if not err < WORST.get((inst, mode, k), (-1.0, ""))[0]:
        WORST[(inst, mode, k)] = (err, tag)
    assert err < b, (inst, mode, K, tag, err, b)


def _card() -> str:
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "power limit unknown"
    return f"{name}, {_sms()} SMs, {pl}"


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print(f"\nGEMM worst error per (instantiation, mode, K) on {_card()} (bar):")
        for (inst, mode, k), (v, tag) in sorted(WORST.items()):
            print(f"  {inst:18s} {mode:10s} K<={k:<5d} {v:.3e}  ({BARS[mode][k]:.1e})  at {tag}")
        worst = {}
        for (_, mode, k), (v, _) in WORST.items():
            worst[(mode, k)] = max(worst.get((mode, k), 0.0), v)
        print("GEMM worst per (mode, K): " + ", ".join(f"{m} {k}: {v:.2e}" for (m, k), v in sorted(worst.items())))
    for k, (v, tag) in sorted(APART.items()):
        print(f"  plain TF32 on 3xTF32's operands, K={k}: error at least {v:.1f}x 3xTF32's, at {tag}")


# ====================================================================================== float64 side
def chunk_errors(got, ref, scale):
    """Relative RMS per (row, 32-column chunk) of ``got`` against ``ref`` [M, N], over the RMS of ``scale``'s row; inf
    wherever a chunk holds a value that is not finite."""
    got, ref, scale = got.double(), ref.double(), scale.double()
    M, N = ref.shape
    pad = (-N) % 32
    d = torch.nn.functional.pad(got - ref, (0, pad)).view(M, -1, 32)
    width = torch.full((d.shape[1],), 32.0, dtype=torch.float64, device=d.device)
    width[-1] = 32 - pad
    e = (d.pow(2).sum(-1) / width).sqrt() / scale.pow(2).mean(-1, keepdim=True).sqrt().clamp_min(1e-300)
    fin = torch.nn.functional.pad(torch.isfinite(got), (0, pad), value=True).view(M, -1, 32).all(-1)
    return torch.where(fin, e, torch.full_like(e, math.inf))


def worst(got, ref, scale=None) -> float:
    return float(chunk_errors(got, ref, ref if scale is None else scale).max())


def swiglu_scale(p):
    """Scale of SwiGLU's output error for product errors of the size of p's row RMS: that RMS times
    |silu'(g) u| + |silu(g)| per output, with (g, u) = the interleaved columns of p."""
    g, u = p[:, 0::2], p[:, 1::2]
    sg = torch.sigmoid(g)
    sens = (sg * (1 + g * (1 - sg)) * u).abs() + (g * sg).abs()
    return sens * p.pow(2).mean(-1, keepdim=True).sqrt()


def tf32_split(x):
    """3xTF32 halves as the codec forms them: hi = x rounded to the 10-bit TF32 mantissa, lo = x - hi (exact)."""
    i = x.float().contiguous().view(torch.int32)
    hi = ((i + 0x1000) & ~0x1FFF).view(torch.float32)
    return hi, x.float() - hi


def tf32_round(x):
    """fp32 -> TF32 by round to nearest even (the fault model of a tensor core that rounded its operands)."""
    i = x.float().contiguous().view(torch.int32)
    return ((i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF).view(torch.float32)


def slice_cols(K: int, bk: int, used: int, z: int, shift: int = 0):
    """Columns of K that split-K slice z of ``used`` reduces (k-blocks of bk elements); ``shift`` moves its k-block
    range (fault model)."""
    num_kb = (K + bk - 1) // bk
    lo, hi = num_kb * z // used + shift, num_kb * (z + 1) // used + shift
    return slice(min(lo * bk, K), min(hi * bk, K))


# ====================================================================================== device side
def _rup(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class Ops:
    """One problem's operands in the layout the kernel reads, and their float64 meaning.

    A is [a_rows, a_cols] (a_rows = M + taps - 1; a_cols = K, or lda for a Conv1d whose K walks ``taps`` shifted rows),
    W is [N, K].  The device buffers hold NaN in the stride padding and in PAD_ROWS rows past the operand; in 3xTF32 the
    lo halves follow the hi halves directly (a_lo_rows = a_rows, w_lo_rows = N).  ``ref`` is the float64 product the
    mode is held to, ``exact`` the product of the fp32 (or bf16) values themselves."""

    def __init__(self, mode: str, M: int, N: int, K: int, seed: int, taps: int = 1):
        dev = torch.device("cuda:0")
        bf = mode == "bf16"
        step = 8 if bf else 4                          # 16 bytes
        self.mode, self.M, self.N, self.K = mode, M, N, K
        if taps == 1:
            a_cols, a_rows, self.lda = K, M, _rup(K, step) + step
        else:
            a_cols, a_rows, self.lda = K // taps, M + taps - 1, K // taps
        self.ldw = _rup(K, step) + step
        g = torch.Generator(device=dev).manual_seed(seed)
        A = torch.randn(a_rows, a_cols, device=dev, generator=g)
        W = torch.randn(N, K, device=dev, generator=g) / math.sqrt(K)
        if bf:
            A, W = A.bfloat16().float(), W.bfloat16().float()
        self.A32, self.W32 = A, W
        dt = torch.bfloat16 if bf else torch.float32
        halves = 2 if mode == "3xtf32" else 1
        self.A = torch.full((halves * a_rows + PAD_ROWS, self.lda), NAN, dtype=dt, device=dev)
        self.W = torch.full((halves * N + PAD_ROWS, self.ldw), NAN, dtype=dt, device=dev)
        if mode == "3xtf32":
            (ah, al), (wh, wl) = tf32_split(A), tf32_split(W)
            self.A[:a_rows, :a_cols], self.A[a_rows:2 * a_rows, :a_cols] = ah, al
            self.W[:N, :K], self.W[N:2 * N, :K] = wh, wl
            self.lo_rows = (a_rows, N)
        else:
            self.A[:a_rows, :a_cols], self.W[:N, :K] = A.to(dt), W.to(dt)
            self.lo_rows = (0, 0)
        Ae = A if taps == 1 else torch.cat([A[t:t + M] for t in range(taps)], dim=1)          # [M, K]
        self.exact = Ae.double() @ W.double().T
        self.ref = tf32_truncate(Ae).double() @ tf32_truncate(W).double().T if mode == "tf32" else self.exact

    def plain_tf32(self):
        """The same fp32 operands laid out for a plain TF32 GEMM (3xTF32's comparison)."""
        A = torch.full((self.A32.shape[0] + PAD_ROWS, self.lda), NAN, device=self.A.device)
        W = torch.full((self.N + PAD_ROWS, self.ldw), NAN, device=self.W.device)
        A[:self.A32.shape[0], :self.A32.shape[1]], W[:self.N, :self.K] = self.A32, self.W32
        return A, W


def gemm(mode: str, o: Ops, *, bn: int = 0, ring: int = -1, out_f32=None, out_bf16=None, ldc: int = 0, bias=None,
         residual=None, ldr: int = 0, act: int = 0, valid=(0, 0), w_const: int = 0, split_ws=None, tile_max=None,
         tile_ld: int = 0, public: bool = False, A=None, W=None, plain: bool = False):
    """One GEMM through nt_debug_gemm (or the public nt_gemm), no synchronisation.  Returns (used, slice_stride)."""
    from neutts_air_b200 import _lib

    L = _lib.lib()
    a = _lib.GemmArgs()
    a.dtype = _lib.NT_BF16 if mode == "bf16" else _lib.NT_TF32
    a.M, a.N, a.K = o.M, o.N, o.K
    a.A, a.lda = (A if A is not None else o.A).data_ptr(), o.lda
    a.W, a.ldw = (W if W is not None else o.W).data_ptr(), o.ldw
    p = lambda t: t.data_ptr() if t is not None else None
    a.bias, a.residual, a.ldr, a.act = p(bias), p(residual), ldr, act
    a.out_f32, a.out_bf16, a.ldc = p(out_f32), p(out_bf16), ldc
    a.valid_period, a.valid_len = valid
    stream = _lib.current_stream_ptr()
    if public:
        _lib.check(L.nt_gemm(C.byref(a), stream))
        return 1, 0
    info = (C.c_int64 * 2)(-1, -1)
    lo = (0, 0) if plain else o.lo_rows
    _lib.check(L.nt_debug_gemm(C.byref(a), bn, ring, w_const, p(split_ws), split_ws.numel() if split_ws is not None else 0,
                               info, lo[0], lo[1], p(tile_max), tile_ld, stream))
    return int(info[0]), int(info[1])


def sentinel(rows: int, cols: int, dtype=torch.float32):
    it = torch.int32 if dtype == torch.float32 else torch.int16
    return torch.full((rows, cols), SENT32 if dtype == torch.float32 else SENT16, dtype=it, device="cuda:0").view(dtype)


def assert_untouched(buf, before, rows_ok, ncols: int, tag: str) -> None:
    """Every cell outside rows_ok x [0, ncols) is bit-identical to ``before``."""
    written = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    written[:rows_ok.numel()][rows_ok, :ncols] = True
    it = torch.int32 if buf.dtype == torch.float32 else torch.int16
    same = buf.view(it) == before.view(it)
    assert bool(same[~written].all()), (tag, "a cell outside the result changed", int((~same & ~written).sum()))


def assert_bf16_is_rne(ob, of, rows_ok, ncols: int, tag: str) -> None:
    """bf16 output == round-to-nearest-even of the fp32 output, bit for bit."""
    want = of[:rows_ok.numel()][rows_ok, :ncols].bfloat16().view(torch.int16)
    got = ob[:rows_ok.numel()][rows_ok, :ncols].view(torch.int16)
    assert torch.equal(got, want), (tag, "bf16 output is not RNE of the fp32 output", int((got != want).sum()))


def check_product(inst: str, mode: str, o: Ops, got, exp, scale, tag: str, exact_exp=None) -> None:
    """Record the mode's error of ``got`` against ``exp`` (and, for plain TF32, against ``exact_exp``)."""
    record(inst, mode, o.K, worst(got, exp, scale), tag)
    if mode == "tf32" and exact_exp is not None:
        record(inst, "tf32-exact", o.K, worst(got, exact_exp, scale), tag)


def all_rows(M: int):
    return torch.ones(M, dtype=torch.bool, device="cuda:0")


# ====================================================================================== the instantiation matrix
@pytest.mark.gpu
@pytest.mark.parametrize("mode,bn,ring", STORE, ids=STORE_IDS)
def test_gemm_shapes(cuda, mode, bn, ring):
    """Every (M, N, K) of the tile-edge grid, plain fp32 epilogue, guards on every side."""
    inst = f"{mode}-bn{bn}-{ring}"
    for K in KS[mode]:
        for M in MS:
            for N in NS:
                tag = f"M={M} N={N} K={K}"
                o = Ops(mode, M, N, K, seed=M * 131 + N * 7 + K)
                ldc = _rup(N, 4) + 4
                out = sentinel(M + PAD_ROWS, ldc)
                before = out.clone()
                gemm(mode, o, bn=bn, ring=RING[ring], out_f32=out, ldc=ldc)
                torch.cuda.synchronize()
                assert_untouched(out, before, all_rows(M), N, tag)
                check_product(inst, mode, o, out[:M, :N], o.ref, o.ref, tag, o.exact)
                if mode == "3xtf32" and M >= 7:
                    A, W = o.plain_tf32()
                    pl = torch.empty(M, ldc, device=cuda)
                    gemm("tf32", o, bn=bn, ring=0, out_f32=pl, ldc=ldc, A=A, W=W, plain=True)
                    torch.cuda.synchronize()
                    whole = lambda t: float((t[:M, :N].double() - o.exact).norm() / o.exact.norm())
                    ratio = whole(pl) / max(whole(out), 1e-300)
                    if ratio < APART.get(K, (math.inf, ""))[0]:
                        APART[K] = (ratio, f"{inst} {tag}")
                    assert ratio > TF32_APART, (inst, tag, whole(pl), whole(out))


def _epi_shapes(mode: str):
    return ((129, 130, 72), (300, 1922, 896)) if mode == "bf16" else ((129, 130, 40), (300, 1922, 1024))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,bn,ring", STORE, ids=STORE_IDS)
def test_gemm_epilogues(cuda, mode, bn, ring):
    """bias; residual with ldr != ldc; bias + residual aliasing out_f32 under a row mask; SiLU and SwiGLU with fp32 and
    bf16 outputs from one call; bf16 alone on unaligned rows; Conv1d taps under the codec's row mask."""
    inst = f"{mode}-bn{bn}-{ring}"
    r = RING[ring]
    g = torch.Generator(device=cuda).manual_seed(bn + r)
    for M, N, K in _epi_shapes(mode):
        o = Ops(mode, M, N, K, seed=M + N + K + 1)
        prod = o.ref
        bias = torch.randn(N, device=cuda, generator=g)
        b64 = bias.double()
        ldc = _rup(N, 4) + 4
        # bias + residual, ldr != ldc
        res = torch.randn(M, ldc + 8, device=cuda, generator=g)
        out = sentinel(M + PAD_ROWS, ldc)
        before = out.clone()
        gemm(mode, o, bn=bn, ring=r, out_f32=out, ldc=ldc, bias=bias, residual=res, ldr=ldc + 8)
        torch.cuda.synchronize()
        tag = f"bias+residual M={M} N={N} K={K}"
        assert_untouched(out, before, all_rows(M), N, tag)
        check_product(inst, mode, o, out[:M, :N], prod + b64 + res[:, :N].double(), prod, tag,
                      o.exact + b64 + res[:, :N].double())
        # bias + residual aliasing out_f32, rows masked by (row % 50) < 37: the masked rows keep the residual
        out = sentinel(M + PAD_ROWS, ldc)
        out[:M, :N] = torch.randn(M, N, device=cuda, generator=g)
        before = out.clone()
        rows_ok = torch.arange(M, device=cuda) % 50 < 37
        gemm(mode, o, bn=bn, ring=r, out_f32=out, ldc=ldc, bias=bias, residual=out, ldr=ldc, valid=(50, 37))
        torch.cuda.synchronize()
        tag = f"bias+residual in place, row mask M={M} N={N} K={K}"
        assert_untouched(out, before, rows_ok, N, tag)
        want = before[:M, :N].double() + prod + b64
        check_product(inst, mode, o, out[:M, :N][rows_ok], want[rows_ok], prod[rows_ok], tag,
                      (before[:M, :N].double() + o.exact + b64)[rows_ok])
        # SiLU, fp32 and bf16 rows from the same call
        of, ob = sentinel(M + PAD_ROWS, ldc + 4), sentinel(M + PAD_ROWS, ldc + 4, torch.bfloat16)
        bf, bb = of.clone(), ob.clone()
        gemm(mode, o, bn=bn, ring=r, out_f32=of, out_bf16=ob, ldc=ldc + 4, bias=bias, act=1)
        torch.cuda.synchronize()
        tag = f"SiLU fp32+bf16 M={M} N={N} K={K}"
        assert_untouched(of, bf, all_rows(M), N, tag)
        assert_untouched(ob, bb, all_rows(M), N, tag)
        assert_bf16_is_rne(ob, of, all_rows(M), N, tag)
        silu = torch.nn.functional.silu
        check_product(inst, mode, o, of[:M, :N], silu(prod + b64), prod, tag, silu(o.exact + b64))
        # SwiGLU over interleaved (gate, up) columns: N / 2 outputs, the last 16-column group partial
        Nh = N // 2
        assert Nh % 16
        ldh = _rup(Nh, 8) + 8
        of, ob = sentinel(M + PAD_ROWS, ldh), sentinel(M + PAD_ROWS, ldh, torch.bfloat16)
        bf, bb = of.clone(), ob.clone()
        gemm(mode, o, bn=bn, ring=r, out_f32=of, out_bf16=ob, ldc=ldh, bias=bias, act=2)
        torch.cuda.synchronize()
        tag = f"SwiGLU fp32+bf16 M={M} N={N} K={K}"
        assert_untouched(of, bf, all_rows(M), Nh, tag)
        assert_untouched(ob, bb, all_rows(M), Nh, tag)
        assert_bf16_is_rne(ob, of, all_rows(M), Nh, tag)
        sw = lambda p: silu(p[:, 0::2] + b64[0::2]) * (p[:, 1::2] + b64[1::2])
        check_product(inst, mode, o, of[:M, :Nh], sw(prod), swiglu_scale(prod + b64), tag, sw(o.exact))
        # fp32 alone, then bf16 alone, both on rows that are not 16-byte aligned (odd ldc): the bf16 rows are RNE of the
        # fp32 rows of the other call, since both run the same instruction stream
        ldo = N + 3
        of, ob = sentinel(M + PAD_ROWS, ldo), sentinel(M + PAD_ROWS, ldo, torch.bfloat16)
        bf, bb = of.clone(), ob.clone()
        gemm(mode, o, bn=bn, ring=r, out_f32=of, ldc=ldo)
        gemm(mode, o, bn=bn, ring=r, out_bf16=ob, ldc=ldo)
        torch.cuda.synchronize()
        tag = f"unaligned rows M={M} N={N} K={K}"
        assert_untouched(of, bf, all_rows(M), N, tag)
        assert_untouched(ob, bb, all_rows(M), N, tag)
        assert_bf16_is_rne(ob, of, all_rows(M), N, tag)
        check_product(inst, mode, o, of[:M, :N], prod, prod, tag, o.exact)
    # Conv1d (k = 3) over a padded-batch layout: items of 56 rows, 50 valid, as the codec lays them out; A rows overlap
    # (lda = channels < K), with and without a residual accumulated in place
    Cc = 128
    for Co, with_res in ((96, False), (130, True)):
        M = 3 * 56 - 6
        o = Ops(mode, M, Co, 3 * Cc, seed=Co, taps=3)
        bias = torch.randn(Co, device=cuda, generator=g)
        ldc = Co + 4
        out = sentinel(M + PAD_ROWS, ldc)
        rows_ok = torch.arange(M, device=cuda) % 56 < 50
        if with_res:
            out[:M, :Co] = torch.randn(M, Co, device=cuda, generator=g)
        before = out.clone()
        gemm(mode, o, bn=bn, ring=r, out_f32=out, ldc=ldc, bias=bias, residual=out if with_res else None,
             ldr=ldc if with_res else 0, valid=(56, 50))
        torch.cuda.synchronize()
        tag = f"conv taps=3 Cin={Cc} Cout={Co}{' +residual' if with_res else ''}"
        assert_untouched(out, before, rows_ok, Co, tag)
        base = before[:M, :Co].double() if with_res else 0.0
        want = (base + o.ref + bias.double())[rows_ok]
        check_product(inst, mode, o, out[:M, :Co][rows_ok], want, o.ref[rows_ok], tag,
                      (base + o.exact + bias.double())[rows_ok])


# ====================================================================================== split-K
SPLIT_CASES = [
    # mode, M, N, K, residual in place
    ("bf16", 7, 896, 4864, False), ("bf16", 129, 130, 896, True), ("bf16", 1, 1922, 4864, True),
    ("tf32", 7, 1922, 7168, False), ("tf32", 64, 130, 1922, True), ("tf32", 1, 33, 1024, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("bn", (32, 64, 128))
@pytest.mark.parametrize("mode,M,N,K,in_place", SPLIT_CASES, ids=[f"{c[0]}-M{c[1]}-N{c[2]}-K{c[3]}" for c in SPLIT_CASES])
def test_gemm_split_k(cuda, mode, M, N, K, in_place, bn):
    """Slices the dispatcher agrees to cut (<= 48 tiles, >= 8 k-blocks, residual in place or none): slice z against
    float64 over its own k-blocks, the bias on slice 0 only, the slices summed in z order against the whole product,
    and out_f32 untouched."""
    inst = f"{mode}-bn{bn}-split"
    g = torch.Generator(device=cuda).manual_seed(M + N + bn)
    o = Ops(mode, M, N, K, seed=K + bn)
    bias = torch.randn(N, device=cuda, generator=g)
    ldc = _rup(N, 4) + 4
    out = sentinel(M + PAD_ROWS, ldc)
    if in_place:
        out[:M, :N] = torch.randn(M, N, device=cuda, generator=g)
    before = out.clone()
    ws = torch.full((8 * M * ldc + 64,), NAN, device=cuda)
    used, stride = gemm(mode, o, bn=bn, out_f32=out, ldc=ldc, bias=bias, residual=out if in_place else None,
                        ldr=ldc if in_place else 0, split_ws=ws)
    torch.cuda.synchronize()
    tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
    bk = 64 if mode == "bf16" else 32
    num_kb = (K + bk - 1) // bk
    sk = min((_sms() - 4) // tiles, num_kb // 4, 8) if tiles <= 48 and num_kb >= 8 else 1
    assert used == max(sk, 1) and stride == (M * ldc if used > 1 else 0), (used, stride, tiles)
    base = before[:M, :N].double() if in_place else 0.0
    if used == 1:                                                     # too many tiles: the normal epilogue ran
        assert bool(torch.isnan(ws).all()), "split-K workspace written although the GEMM did not split"
        assert_untouched(out, before, all_rows(M), N, "no split")
        record(inst, mode, K, worst(out[:M, :N], o.ref + bias.double() + base, o.ref), f"no split, {tiles} tiles")
        return
    assert torch.equal(out.view(torch.int32), before.view(torch.int32)), "out_f32 written although the GEMM split"
    A = o.A[:M, :K].double() if mode == "bf16" else tf32_truncate(o.A[:M, :K]).double()
    W = o.W[:N, :K].double() if mode == "bf16" else tf32_truncate(o.W[:N, :K]).double()
    total = torch.zeros(M, N, device=cuda)
    for z in range(used):
        cols = slice_cols(K, bk, used, z)
        sl = ws[z * stride:z * stride + M * ldc].view(M, ldc)
        exp = A[:, cols] @ W[:, cols].T
        tag = f"slice {z}/{used} k[{cols.start}:{cols.stop}) M={M} N={N} K={K}"
        got = sl[:, :N]
        if z == 0:
            exp = exp + bias.double()
        record(inst, mode, K, worst(got, exp, A[:, cols] @ W[:, cols].T), tag)
        total += got                                                 # fp32, z order: the consumers' fold
        assert bool(torch.isnan(sl[:, N:]).all()), (tag, "split slice written past N")
    assert bool(torch.isnan(ws[used * stride:]).all()), "split-K wrote past its last slice"
    record(inst, mode, K, worst(total.double() + base, o.ref + bias.double() + base, o.ref), f"sum of {used} slices")


# ====================================================================================== tile maxima
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ("bf16", "tf32"))
@pytest.mark.parametrize("bn", (32, 64, 128))
def test_gemm_tile_max(cuda, mode, bn):
    """tile_max[r, t] is the maximum of the fp32 values the same call stored in row r inside column tile t, bit for
    bit, for a last tile that ends past N; and a column range of a wider matrix at the forced BN, with its maxima at
    tile_max + r0 / BN and the whole matrix's tile count as pitch (the lm_head's vocabulary range), reproduces the
    whole-matrix GEMM's logits and maxima bit for bit."""
    K = 896 if mode == "bf16" else 1024
    g = torch.Generator(device=cuda).manual_seed(bn)
    for M, N in ((7, 1922), (129, 4001)):
        o = Ops(mode, M, N, K, seed=M + bn)
        nt = (N + bn - 1) // bn
        ldc = N
        out = sentinel(M + PAD_ROWS, ldc)
        tmx = sentinel(M + PAD_ROWS, nt)
        before = tmx.clone()
        bias = torch.randn(N, device=cuda, generator=g)
        gemm(mode, o, bn=bn, out_f32=out, ldc=ldc, bias=bias, tile_max=tmx)
        torch.cuda.synchronize()
        tag = f"tile max M={M} N={N}"
        assert_untouched(tmx, before, all_rows(M), nt, tag)
        padded = torch.nn.functional.pad(out[:M, :N], (0, nt * bn - N), value=-math.inf)
        want = padded.view(M, nt, bn).amax(-1)
        assert torch.equal(tmx[:M].view(torch.int32), want.view(torch.int32)), (tag, "tile maxima")
        record(f"{mode}-bn{bn}-tilemax", mode, K, worst(out[:M, :N], o.ref + bias.double(), o.ref), tag)
        # column ranges [r0, r1) at the forced BN, written into a matrix of the whole width
        cuts = [0, bn * (nt // 3), bn * (2 * nt // 3), N]
        part = sentinel(M + PAD_ROWS, ldc)
        ptm = sentinel(M + PAD_ROWS, nt)
        for r0, r1 in zip(cuts, cuts[1:]):
            a = Ops.__new__(Ops)
            a.__dict__.update(o.__dict__)
            a.N = r1 - r0
            gemm(mode, a, bn=bn, out_f32=part[:, r0:], ldc=ldc, bias=bias[r0:], tile_max=ptm[:, r0 // bn:], tile_ld=nt,
                 W=o.W[r0:])
        torch.cuda.synchronize()
        assert torch.equal(part.view(torch.int32), out.view(torch.int32)), (tag, "column ranges differ from the whole")
        assert torch.equal(ptm.view(torch.int32), tmx.view(torch.int32)), (tag, "range maxima differ from the whole")


# ====================================================================================== log-softmax
def _logsoftmax(A, M: int, K: int, W, N: int, tgt):
    from neutts_air_b200 import _lib

    nt = (N + 127) // 128
    lse = torch.full((M + PAD_ROWS, nt + 1, 2), NAN, device=A.device)
    zt = torch.full((M + PAD_ROWS,), NAN, device=A.device)
    _lib.check(_lib.lib().nt_debug_gemm_logsoftmax(A.data_ptr(), M, K, W.data_ptr(), N, tgt.data_ptr(), lse.data_ptr(),
                                                   nt + 1, zt.data_ptr(), _lib.current_stream_ptr()))
    torch.cuda.synchronize()
    return lse, zt


@pytest.mark.gpu
@pytest.mark.parametrize("ring", ("deep", "shallow"), ids=("logsoftmax-deep", "logsoftmax-shallow"))
def test_gemm_logsoftmax(cuda, ring):
    """(max, sum exp) per (row, 128-column tile) and the target logit against float64; the max and the target logit
    bit-identical to the plain bf16 BN = 128 GEMM of the same operands; rows bit-identical between an M = 1 call and
    the same row of an M = 300 call.  The ring is reached through the number of CTAs."""
    K = 896
    N = 1922 if ring == "deep" else _sms() * 128 + 100
    nt = (N + 127) // 128
    inst = f"logsoftmax-{ring}"
    g = torch.Generator(device=cuda).manual_seed(N)
    M = 300
    assert ((3 * nt > _sms()) if ring == "shallow" else (3 * nt <= _sms()))
    assert (nt > _sms()) == (ring == "shallow")        # the M = 1 calls run the same ring
    A = torch.randn(M, K, device=cuda, generator=g).bfloat16()
    W = (torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K)).bfloat16()
    tgt = torch.randint(0, N, (M,), device=cuda, generator=g, dtype=torch.int32)
    tgt[:4] = torch.tensor([0, N - 1, (nt - 1) * 128, 127], dtype=torch.int32)
    lse, zt = _logsoftmax(A, M, K, W, N, tgt)
    assert bool(torch.isnan(lse[:M, nt:]).all()) and bool(torch.isnan(lse[M:]).all()) and bool(torch.isnan(zt[M:]).all())
    ref = A.double() @ W.double().T                                              # [M, N]
    padded = torch.nn.functional.pad(ref, (0, nt * 128 - N), value=-math.inf).view(M, nt, 128)
    m64 = padded.amax(-1)
    lse64 = m64 + (padded - m64[..., None]).exp().sum(-1).log()
    m, s = lse[:M, :nt, 0].double(), lse[:M, :nt, 1].double()
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    record(inst, "bf16", K, float(((m - m64).abs() / rms).max()), f"tile max M={M} N={N}")
    record(inst, "lse", K, float((m + s.log() - lse64).abs().max()) if bool(torch.isfinite(s).all()) else math.inf,
           f"lse M={M} N={N}")
    zt64 = ref.gather(1, tgt.long()[:, None])[:, 0]
    record(inst, "bf16", K, float(((zt[:M].double() - zt64).abs() / rms[:, 0]).max()), f"target logit M={M} N={N}")
    # the plain bf16 BN = 128 GEMM of the same operands, at the same ring
    o = Ops.__new__(Ops)
    o.mode, o.M, o.N, o.K, o.lda, o.ldw, o.A, o.W, o.lo_rows = "bf16", M, N, K, K, K, A, W, (0, 0)
    out = torch.empty(M, N, device=cuda)
    tmx = torch.empty(M, nt, device=cuda)
    gemm("bf16", o, bn=128, ring=1 if 3 * nt > _sms() else 0, out_f32=out, ldc=N, tile_max=tmx)
    torch.cuda.synchronize()
    assert torch.equal(lse[:M, :nt, 0].contiguous().view(torch.int32), tmx.view(torch.int32)), "max != plain GEMM tile max"
    assert torch.equal(zt[:M].view(torch.int32), out.gather(1, tgt.long()[:, None])[:, 0].view(torch.int32)), \
        "target logit != plain GEMM logit"
    for r in (0, 1, 127, 128, 299):
        l1, z1 = _logsoftmax(A[r:r + 1], 1, K, W, N, tgt[r:r + 1])
        assert torch.equal(l1[0, :nt].view(torch.int32), lse[r, :nt].view(torch.int32)), ("row depends on M", r)
        assert torch.equal(z1[0].view(torch.int32), zt[r].view(torch.int32)), ("target logit depends on M", r)


# ====================================================================================== invariances
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ("bf16", "tf32"))
@pytest.mark.parametrize("bn", (32, 64, 128))
def test_gemm_ring_and_row_invariance(cuda, mode, bn):
    """Deep and shallow rings give the same bits for the same (dtype, BN); rows give the same bits at every M.  Across
    BN, whether the bits agree is printed only: nothing in the code promises it."""
    K = 896 if mode == "bf16" else 1922
    N = 1922
    o = Ops(mode, 1031, N, K, seed=bn)
    full = {}
    for ring in (0, 1):
        full[ring] = torch.empty(1031, N, device=cuda)
        gemm(mode, o, bn=bn, ring=ring, out_f32=full[ring], ldc=N)
    torch.cuda.synchronize()
    assert torch.equal(full[0].view(torch.int32), full[1].view(torch.int32)), "deep and shallow rings differ"
    for M in (1, 7, 128, 129, 300):
        a = Ops.__new__(Ops)
        a.__dict__.update(o.__dict__)
        a.M = M
        out = torch.empty(M, N, device=cuda)
        gemm(mode, a, bn=bn, ring=0, out_f32=out, ldc=N)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), full[0][:M].view(torch.int32)), ("rows depend on M", M)
    others = {}
    for b in (32, 64, 128):
        out = torch.empty(1031, N, device=cuda)
        gemm(mode, o, bn=b, ring=0, out_f32=out, ldc=N)
        torch.cuda.synchronize()
        others[b] = bool(torch.equal(out.view(torch.int32), full[0].view(torch.int32)))
    print(f"GEMM {mode} K={K}: BN={bn} bit-identical to BN 32/64/128: {others}")


# ====================================================================================== PDL ordering
@pytest.mark.gpu
def test_gemm_pdl_chain(cuda):
    """A TF32 GEMM writes the A operand of a second one that may fetch its weights before the PDL wait (w_const), on
    one stream with no host synchronisation between them; the intermediate buffer starts as NaN.  The second result is
    finite and correct, so the A loads come after griddepcontrol.wait."""
    M, K1, K2, N = 129, 1024, 1024, 1922
    o1 = Ops("tf32", M, K2, K1, seed=1)
    mid = torch.full((M + PAD_ROWS, K2 + 4), NAN, device=cuda)
    o2 = Ops("tf32", M, N, K2, seed=2)
    o2.A, o2.lda = mid, K2 + 4
    out = torch.empty(M, N, device=cuda)
    torch.cuda.synchronize()
    gemm("tf32", o1, w_const=1, out_f32=mid, ldc=K2 + 4)
    gemm("tf32", o2, w_const=1, out_f32=out, ldc=N)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all()), "the second GEMM read its A before the first one finished"
    record("tf32-pdl", "tf32", K1, worst(mid[:M, :K2], o1.ref), "first GEMM")
    ref2 = tf32_truncate(mid[:M, :K2]).double() @ tf32_truncate(o2.W32).double().T
    record("tf32-pdl", "tf32", K2, worst(out, ref2), "second GEMM")


# ====================================================================================== the public entry
PUBLIC = [("bf16", 128, 128, 64), ("bf16", 500, 896, 896), ("bf16", 500, 1152, 896), ("bf16", 7, 896, 4864),
          ("bf16", 300, 1922, 1024), ("bf16", 1000, 9728, 896), ("bf16", 64, 2048, 896),
          ("tf32", 256, 1024, 1024), ("tf32", 256, 1922, 1024), ("tf32", 250, 1920, 1922), ("tf32", 77, 3072, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,M,N,K", PUBLIC, ids=[f"{c[0]}-M{c[1]}-N{c[2]}-K{c[3]}" for c in PUBLIC])
def test_gemm_public_entry(cuda, mode, M, N, K):
    """nt_gemm itself, so the dispatcher's own BN and ring: the prefill and codec shapes, plain, and at M = 333 the
    epilogues of the prefill (bias + residual in place, SiLU to bf16, SwiGLU to bf16)."""
    o = Ops(mode, M, N, K, seed=M * 3 + N)
    ldc = N + 4
    out = sentinel(M + PAD_ROWS, ldc)
    before = out.clone()
    gemm(mode, o, out_f32=out, ldc=ldc, public=True)
    torch.cuda.synchronize()
    tag = f"public M={M} N={N} K={K}"
    assert_untouched(out, before, all_rows(M), N, tag)
    check_product(f"{mode}-public", mode, o, out[:M, :N], o.ref, o.ref, tag, o.exact)


@pytest.mark.gpu
def test_gemm_public_epilogues(cuda):
    """The prefill's epilogues through nt_gemm at M = 333: bias + residual in place, SiLU to bf16, SwiGLU to bf16.  A
    bf16-only call is RNE of the fp32-only call of the same shape, since the dispatcher picks the same kernel for both."""
    g = torch.Generator(device=cuda).manual_seed(3)
    M, N, K = 333, 896, 896
    o = Ops("bf16", M, N, K, seed=3)
    bias = torch.randn(N, device=cuda, generator=g)
    out = torch.randn(M, N, device=cuda, generator=g)
    res = out.clone()
    gemm("bf16", o, out_f32=out, ldc=N, bias=bias, residual=out, ldr=N, public=True)
    torch.cuda.synchronize()
    record("bf16-public", "bf16", K, worst(out, o.ref + bias.double() + res.double(), o.ref), "bias+residual in place")
    silu = torch.nn.functional.silu
    for act, ncol, want, scale in ((1, N, silu(o.ref), o.ref),
                                   (2, N // 2, silu(o.ref[:, 0::2]) * o.ref[:, 1::2], swiglu_scale(o.ref))):
        tag = "SiLU" if act == 1 else "SwiGLU"
        ob, of = sentinel(M + PAD_ROWS, ncol, torch.bfloat16), sentinel(M + PAD_ROWS, ncol)
        bb, bf = ob.clone(), of.clone()
        gemm("bf16", o, out_bf16=ob, ldc=ncol, act=act, public=True)
        gemm("bf16", o, out_f32=of, ldc=ncol, act=act, public=True)
        torch.cuda.synchronize()
        assert_untouched(ob, bb, all_rows(M), ncol, tag)
        assert_untouched(of, bf, all_rows(M), ncol, tag)
        assert_bf16_is_rne(ob, of, all_rows(M), ncol, tag)
        record("bf16-public", "bf16", K, worst(of[:M], want, scale), tag)


@pytest.mark.gpu
def test_gemm_public_conv_taps_and_row_mask(cuda):
    """Conv1d(k = 3, pad = 1) over a padded-batch layout expressed as one TF32 GEMM (the codec path), against
    torch's conv1d in float64."""
    g = torch.Generator().manual_seed(5)
    B, T, Cc, Co = 3, 50, 128, 96
    Tp = T + 6
    x = torch.randn(B, Cc, T, generator=g)
    w = torch.randn(Co, Cc, 3, generator=g) / (3 * Cc) ** 0.5
    b = torch.randn(Co, generator=g)
    ref = torch.nn.functional.conv1d(tf32_truncate(x).double(), tf32_truncate(w).double(), b.double(), padding=1)
    buf = torch.zeros(B * Tp + 8, Cc)
    for i in range(B):
        buf[i * Tp + 3: i * Tp + 3 + T] = x[i].T
    o = Ops.__new__(Ops)
    o.mode, o.M, o.N, o.K, o.lda, o.ldw, o.lo_rows = "tf32", B * Tp - 6, Co, 3 * Cc, Cc, 3 * Cc, (0, 0)
    o.A = buf.to(cuda)[2:]                             # first row the tap window of output row 0 touches
    o.W = w.permute(0, 2, 1).reshape(Co, 3 * Cc).contiguous().to(cuda)
    out = sentinel(B * Tp + 8, Co)
    before = out.clone()
    gemm("tf32", o, out_f32=out[3:], ldc=Co, bias=b.to(cuda), valid=(Tp, T), public=True)
    torch.cuda.synchronize()
    rows_ok = torch.zeros(B * Tp + 8, dtype=torch.bool, device=cuda)
    for i in range(B):
        rows_ok[i * Tp + 3: i * Tp + 3 + T] = True
    assert_untouched(out, before, rows_ok, Co, "public conv")
    got = torch.stack([out[i * Tp + 3: i * Tp + 3 + T].T for i in range(B)]).cpu()
    e = float(chunk_errors(got.permute(0, 2, 1).reshape(-1, Co), ref.permute(0, 2, 1).reshape(-1, Co),
                           ref.permute(0, 2, 1).reshape(-1, Co) - b.double()).max())
    record("tf32-public", "tf32", 3 * Cc, e, "conv taps + row mask")


# ====================================================================================== CPU
def test_fault_models_exceed_the_bars():
    """float64, CPU: each fault the checks above exist to catch lands at least 10x past the bar it would be measured
    against, or breaks an exact check."""
    g = torch.Generator().manual_seed(0)
    lines = []

    def past(label, err, mode, K, factor=10.0):
        b = bar_of(mode, K)[1]
        lines.append(f"{label} {err:.2e} ({err / b:.1f}x)")
        assert err > factor * b, (label, err, b)

    def rnd(M, K, N, bf):
        A, W = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
        return (A.bfloat16().float(), W.bfloat16().float()) if bf else (A, W)

    # the last partial k-block dropped
    for mode, K, bk in (("bf16", 72, 64), ("tf32", 40, 32)):
        A, W = rnd(129, K, 130, mode == "bf16")
        A, W = A.double(), W.double()
        good = A @ W.T
        past(f"{mode} K={K} without its partial k-block", worst(A[:, :bk] @ W[:, :bk].T, good), mode, K)
    # split-K: slice z's k-range shifted by one block; the bias added on every slice
    for mode, K, bk, used in (("bf16", 4864, 64, 8), ("tf32", 7168, 32, 8), ("bf16", 896, 64, 3)):
        A, W = rnd(7, K, 896, mode == "bf16")
        A, W = A.double(), W.double()
        bias = torch.randn(896, generator=g, dtype=torch.float64)
        for z in range(1, used):
            c, s = slice_cols(K, bk, used, z), slice_cols(K, bk, used, z, shift=1 if z < used - 1 else -1)
            good = A[:, c] @ W[:, c].T
            past(f"{mode} K={K} slice {z}/{used} shifted one k-block", worst(A[:, s] @ W[:, s].T, good), mode, K)
            past(f"{mode} K={K} slice {z}/{used} with the bias", worst(good + bias, good), mode, K)
    # the last row tile shifted by one row
    for M in (129, 300, 1031):
        A, W = rnd(M + 1, 896, 130, True)
        full = A.double() @ W.double().T
        good = full[:M]
        bad = good.clone()
        t0 = (M - 1) // 128 * 128
        bad[t0:] = full[t0 + 1:M + 1]
        past(f"last row tile shifted one row M={M}", worst(bad, good), "bf16", 896)
    # bf16 output truncated instead of rounded to nearest even
    v = torch.randn(129, 130, generator=g)
    trunc = (v.view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    assert not torch.equal(trunc.view(torch.int16), v.bfloat16().view(torch.int16))
    assert float((trunc.view(torch.int16) != v.bfloat16().view(torch.int16)).double().mean()) > 0.4
    lines.append("bf16 truncated: breaks the RNE equality")
    # the bf16 pair swapped inside pack_bf16x2
    sw = v.bfloat16().view(-1, 2).flip(-1).reshape(129, 130)
    assert not torch.equal(sw.view(torch.int16), v.bfloat16().view(torch.int16))
    # 3xTF32 without its A_lo . W_hi term; plain TF32 operands rounded instead of truncated.  Both are operand faults:
    # the same k-block code runs at every K, so the K <= 40 cases, which every TF32 and 3xTF32 instantiation runs, catch
    # them.  At K >= 1024 the tensor core's accumulation error is of their size, and the factor is only reported.
    for K in KS["tf32"]:
        A, W = rnd(64, K, 130, False)
        (ah, al), (wh, wl) = tf32_split(A), tf32_split(W)
        exact = A.double() @ W.double().T
        d = lambda x: x.double()
        no_lo = d(ah) @ d(wh).T + d(ah) @ d(wl).T
        trunc = d(tf32_truncate(A)) @ d(tf32_truncate(W)).T
        rounded = d(tf32_round(A)) @ d(tf32_round(W)).T
        factor = 10.0 if K <= 40 else 0.0
        past(f"3xTF32 K={K} without A_lo.W_hi", worst(no_lo, exact), "3xtf32", K, factor)
        past(f"TF32 K={K} operands rounded, not truncated", worst(rounded, trunc), "tf32", K, factor)
    print("FAULTS: " + "; ".join(lines))


def test_error_measure_sees_one_chunk():
    """A single wrong 32-column chunk of one row is seen at its own size, not averaged over the matrix."""
    ref = torch.randn(300, 1922, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got = ref.clone()
    got[299, 1920:] += 1e-3 * ref[299].pow(2).mean().sqrt()
    e = chunk_errors(got, ref, ref)
    assert abs(float(e.max()) - 1e-3) < 1e-9 and int((e > 0).sum()) == 1
    got[5, 7] = NAN
    assert math.isinf(float(chunk_errors(got, ref, ref)[5, 0]))
