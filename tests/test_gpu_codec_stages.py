"""Every NeuCodec decoder stage against float64 on its own inputs, in every GEMM precision mode.

``nt_codec_debug_set_stages`` makes a decode run one stage of the fixed stage list (include/neutts_b200.h) and
``nt_codec_debug_ptr`` exposes the workspace buffers.  A stage walk decodes one stage at a time: before each stage it
snapshots the stage's input rows, after it compares the output with a float64 implementation of that stage evaluated
on the snapshot and on the packed device weights (``dec.w``).  An error upstream therefore cannot hide an error
downstream, and the error of each stage is the kernel's own.

Errors are measured where bugs show:
    row and GEMM stages   relative RMS per (item, frame); the first 3 frames, the last 3 and the interior apart
    GEMM + residual       relative to the product alone, so that the residual does not dilute it
    attention             relative RMS per (item, head)
    GroupNorm + swish     relative RMS per (item, group)
    spectrum              per element, relative to its magnitude
    overlap-add           relative RMS per item; the first and the last hop apart
At N >= 1024 the row stages check every edge frame plus a seeded sample of frames.

Each GEMM is held to the bar of the arithmetic its mode claims: 3xTF32 for every GEMM in "3xtf32" and for the head
and inverse-DFT GEMMs in "mixed", TF32 for the rest.  The 3xTF32 bars are per GEMM, because that error grows with K
(see BARS).  In "tf32" mode each GEMM's error must also sit TF32_APART times above its 3xTF32 bar, which shows on the
GPU that the check tells the modes apart.

Conditions of every walk: a decode at (max_batch, max_frames) with other codes runs first, so stale rows exist; then
every named buffer is filled with NaN, so a row a kernel must not read poisons its output; after every stage the pad
rows of x0, x1 and x2 of the call are exactly 0 (the next conv's "same" padding reads them); and the PCM of the walk is
bit-identical to a one-call decode of the same codes.

Crafted inputs go where random ones are too kind: needle keys at the edges of the 32-key tiles, peaked softmax and
items with very different statistics (attention); positions up to 2047 (RoPE); a large DC offset (GroupNorm, final
LayerNorm); log-magnitudes across the clip and large phases (spectrum); poisoned pad frames and fewer frames than
overlap (overlap-add); ids outside the codebook (FSQ).  ``test_fault_models_exceed_the_bars`` (CPU) shows that the
faults these checks exist for land at least 10x past the bars (TF32_APART for TF32 operands in a 3xTF32 GEMM).
"""
from __future__ import annotations

import functools
import math

import pytest
import torch

from oracle import codec_oracle as CO
from tests.helpers import codec_shape, codec_weight_dict, tf32_truncate

# Worst errors measured on one H100 80GB HBM3 (700 W power limit) over the whole GPU matrix, and the bars, ~4x above:
#   fsq affine 7.8e-8; RMSNorm / LayerNorm rows 1.5e-7; GroupNorm + swish per group 4.0e-7; RoPE 4.0e-8;
#   attention per head 1.1e-6 (N = 2048); spectrum per element 2.2e-7; overlap-add per item 1.4e-7
#   crafted: LayerNorm rows with means to 1e4 7.5e-4 (the fp32 mean of 1024 values near 1e4 is off by ~1e-3, the
#   inputs' own ulp); GroupNorm group at mean 1e3, N = 2048, 3.9e-5; needle / peaked attention 4.7e-5
#   plain TF32 GEMMs 9.6e-4 (every op, any K: the tensor core truncates each operand to 10 mantissa bits)
#   3xTF32 GEMMs per op (K): embed (7168) 6.1e-5, conv1 / conv2 (3072) 2.5e-5, fc2 (4096) 3.1e-5, idft (1922) 1.9e-5,
#   qkv / proj / fc1 / head (1024) 6.6e-6 .. 8.9e-6.  The operand split makes every product fp32-grade, but the tensor
#   core's fp32 accumulation does not round to nearest, so the error grows with K instead of staying near 1e-6.
BARS = {
    "fsq": 3e-7, "norm": 6e-7, "norm-mean": 3e-3, "gn": 1.6e-6, "gn-dc": 1.6e-4, "rope": 1.6e-7, "attn": 4.4e-6,
    "attn-crafted": 2e-4, "spec": 9e-7, "ola": 6e-7, "tf32": 4e-3,
    "3xtf32-embed": 2.5e-4, "3xtf32-conv1": 1e-4, "3xtf32-conv2": 1e-4, "3xtf32-qkv": 3e-5, "3xtf32-proj": 3.4e-5,
    "3xtf32-fc1": 3.6e-5, "3xtf32-fc2": 1.25e-4, "3xtf32-head": 2.7e-5, "3xtf32-idft": 8e-5,
}
# In "tf32" mode every GEMM stage's error must be this many times its 3xTF32 bar.  Measured: 3.0x (embed, K = 7168),
# 6x (fc2), 7.5x (conv), 9.4x (idft), 22-25x (K = 1024).  A factor of 10 holds only at K = 1024: at K = 7168 the
# accumulation error of 3xTF32 already sits 12x below plain TF32 before the bar's 4x margin.
TF32_APART = 2.5
WORST: dict = {}
TF32_FLOOR: dict = {}            # GEMM op -> smallest whole-stage error of its plain TF32 form, and where

MODES = ("tf32", "mixed", "3xtf32")
NAN = float("nan")

# stage op -> (input buffers, output buffer, kind)
IO = {
    "fsq": ((), "x0", "fsq"), "embed": (("x0",), "x1", "gemm"),
    "gn1": (("x1",), "x2", "gn"), "conv1": (("x2",), "x3", "gemm"), "gn2": (("x3",), "x2", "gn"),
    "conv2": (("x2", "x1"), "x1", "gemm"),
    "norm1": (("x1",), "xn", "norm"), "qkv": (("xn",), "qkv", "gemm"), "rope": (("qkv",), "qkv", "rope"),
    "attn": (("qkv",), "att", "attn"), "proj": (("att", "x1"), "x1", "gemm"), "norm2": (("x1",), "xn", "norm"),
    "fc1": (("xn",), "hbuf", "gemm"), "fc2": (("hbuf", "x1"), "x1", "gemm"),
    "final_ln": (("x1",), "xn", "norm"), "head": (("xn",), "sp", "gemm"), "spec": (("sp",), "sp", "spec"),
    "idft": (("sp",), "fr", "gemm"), "ola": (("fr",), "pcm", "ola"),
}


def stage_names(depth: int, rope: bool = True) -> list:
    """Copy of the stage list of ``nt_codec_debug_set_stages`` (include/neutts_b200.h)."""
    rn = lambda i: [f"rn{i}.{s}" for s in ("gn1", "conv1", "gn2", "conv2")]
    ops = ("norm1", "qkv") + (("rope",) if rope else ()) + ("attn", "proj", "norm2", "fc1", "fc2")
    blocks = [f"b{l}.{s}" for l in range(depth) for s in ops]
    return ["fsq", "embed", *rn(0), *rn(1), *blocks, *rn(2), *rn(3), "final_ln", "head", "spec", "idft", "ola"]


def widths(cfg) -> dict:
    C = cfg.hidden
    return dict(x0=C, x1=C, x2=C, x3=C, xn=C, qkv=3 * C, hbuf=cfg.mlp_mult * C, att=C,
                sp=(cfg.n_fft + 2 + 31) // 32 * 32, fr=cfg.n_fft)


def gemm_bar(op: str, mode: str) -> str:
    if op in ("head", "idft"):
        return "tf32" if mode == "tf32" else "3xtf32"
    return "3xtf32" if mode == "3xtf32" else "tf32"


# ====================================================================================== float64 stages
class Ref64:
    """The decoder's stages in float64 on the packed weights (layouts of include/neutts_b200.h).  Buffers are the
    item rows of the padded-batch layout, float64 [B, N + 6, width]: frame t of item b at row 3 + t."""

    def __init__(self, cfg, packed: dict):
        self.cfg = cfg
        d = lambda t: t.detach().cpu().double()
        self.w = {k: [d(t) for t in v] if isinstance(v, list) else d(v) for k, v in packed.items()}
        self.C, self.nb = cfg.hidden, cfg.n_fft // 2 + 1
        self.clip = float(torch.tensor(cfg.mag_clip, dtype=torch.float32))

    @staticmethod
    def conv(x, w, b, k: int, f):
        """"same" Conv1d at frames f: output frame t reads rows t + 3 - k // 2 .. of the padded item (tap-major W)."""
        off = 3 - k // 2
        win = torch.stack([x[:, f + off + j] for j in range(k)], dim=2)
        return win.flatten(2) @ w.T + b

    def gn_swish(self, x, N: int, w, b, f, stat_rows=None):
        """GroupNorm + swish over the N frames of every item (``stat_rows``: rows the statistics span instead)."""
        B, C, G = x.shape[0], self.C, self.cfg.groups
        s = x[:, 3:3 + N] if stat_rows is None else x[:, stat_rows]
        s = s.reshape(B, -1, G, C // G)
        mean = s.mean(dim=(1, 3), keepdim=True)
        var = (s - mean).pow(2).mean(dim=(1, 3), keepdim=True)
        v = x[:, 3 + f].reshape(B, len(f), G, C // G)
        y = ((v - mean) / torch.sqrt(var + self.cfg.norm_eps)).reshape(B, len(f), C) * w + b
        return y * torch.sigmoid(y)

    def rms(self, x, w):
        return x / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + self.cfg.norm_eps) * w

    def ln(self, x, w, b):
        m = x.mean(-1, keepdim=True)
        return (x - m) / torch.sqrt((x - m).pow(2).mean(-1, keepdim=True) + self.cfg.norm_eps) * w + b

    def rope(self, rows, pos):
        """Interleaved-pair rotary on q and k of qkv rows [B, F, 3C] at frame positions ``pos`` [F].  The angle
        pos * inv_freq is formed in fp32, as the kernel forms it; cos / sin are taken in float64."""
        B, F, C = rows.shape[0], rows.shape[1], self.C
        inv = (1.0 / self.cfg.rope_base ** (torch.arange(32, dtype=torch.float64) * 2 / 64)).float()
        ang = (pos.float()[:, None] * inv[None, :]).double()                     # [F, 32]
        c, s = ang.cos()[None, :, None], ang.sin()[None, :, None]
        out = rows.clone()
        for part in (0, 1):
            x = rows[..., part * C:(part + 1) * C].reshape(B, F, C // 64, 32, 2)
            y = torch.stack((x[..., 0] * c - x[..., 1] * s, x[..., 1] * c + x[..., 0] * s), dim=-1)
            out[..., part * C:(part + 1) * C] = y.reshape(B, F, C)
        return out

    def attn(self, qkv, N: int, f, keys=None):
        """Bidirectional softmax attention of the queries at frames f over the keys of frames ``keys`` (all N)."""
        B, C = qkv.shape[0], self.C
        H = C // 64
        kr = torch.arange(N) if keys is None else keys
        q = qkv[:, 3 + f, :C].reshape(B, len(f), H, 64)
        k = qkv[:, 3 + kr, C:2 * C].reshape(B, len(kr), H, 64)
        v = qkv[:, 3 + kr, 2 * C:].reshape(B, len(kr), H, 64)
        p = torch.softmax(torch.einsum("bfhd,bnhd->bhfn", q, k) / 8.0, dim=-1)
        return torch.einsum("bhfn,bnhd->bfhd", p, v).reshape(B, len(f), C)

    def spec(self, sp, f, clip=True):
        lm, ph = sp[:, 3 + f, :self.nb], sp[:, 3 + f, self.nb:2 * self.nb]
        mag = lm.exp()
        if clip:
            mag = mag.clamp(max=self.clip)
        return torch.cat((mag * ph.cos(), mag * ph.sin()), -1), mag

    def ola(self, fr, N: int, drop=None):
        """Overlap-add of the windowed frames, "same" trim, / window envelope.  ``drop``: a frame left out of the
        envelope (fault model)."""
        n_fft, hop = self.cfg.n_fft, self.cfg.hop
        B = fr.shape[0]
        out_size = (N - 1) * hop + n_fft
        y = torch.zeros(B, out_size, dtype=torch.float64)
        env = torch.zeros(out_size, dtype=torch.float64)
        wsq = torch.hann_window(n_fft, periodic=True, dtype=torch.float64).pow(2)
        for t in range(N):
            y[:, t * hop:t * hop + n_fft] += fr[:, 3 + t]
            if t != drop:
                env[t * hop:t * hop + n_fft] += wsq
        pad = (n_fft - hop) // 2
        return (y / env)[:, pad:out_size - pad]

    def run(self, name: str, b: dict, f, N: int, codes=None):
        """Expected output rows [B, len(f), width] of stage ``name`` from the item rows ``b`` (buffer -> float64
        [B, N + 6, width]), and the tensor its error is relative to (the product alone for a GEMM with a residual;
        the magnitudes for the spectrum).  ``ola`` returns the PCM [B, hop * N]."""
        w = self.w
        blk, _, op = name.rpartition(".")
        i = int(blk[2:]) if blk.startswith("rn") else int(blk[1:]) if blk else 0
        if op == "fsq":
            z = CO.fsq_dequant(codes[:, f], self.cfg).double()
            y = z @ w["fsq_w"].T + w["fsq_b"]
            return y, y
        if op == "embed":
            y = self.conv(b["x0"], w["embed_w"], w["embed_b"], 7, f)
            return y, y
        if op in ("gn1", "gn2"):
            n = op[2]
            y = self.gn_swish(b["x1" if n == "1" else "x3"], N, w[f"rn_n{n}w"][i], w[f"rn_n{n}b"][i], f)
            return y, y
        if op == "conv1":
            y = self.conv(b["x2"], w["rn_c1w"][i], w["rn_c1b"][i], 3, f)
            return y, y
        if op == "conv2":
            p = self.conv(b["x2"], w["rn_c2w"][i], w["rn_c2b"][i], 3, f)
            return b["x1"][:, 3 + f] + p, p
        if op in ("norm1", "norm2"):
            y = self.rms(b["x1"][:, 3 + f], w["att_norm" if op == "norm1" else "ffn_norm"][i])
            return y, y
        if op == "qkv":
            y = b["xn"][:, 3 + f] @ w["wqkv"][i].T
            return y, y
        if op == "rope":
            y = self.rope(b["qkv"][:, 3 + f], f)
            return y, y
        if op == "attn":
            y = self.attn(b["qkv"], N, f)
            return y, y
        if op == "proj":
            p = b["att"][:, 3 + f] @ w["wproj"][i].T
            return b["x1"][:, 3 + f] + p, p
        if op == "fc1":
            y = torch.nn.functional.silu(b["xn"][:, 3 + f] @ w["fc1"][i].T)
            return y, y
        if op == "fc2":
            p = b["hbuf"][:, 3 + f] @ w["fc2"][i].T
            return b["x1"][:, 3 + f] + p, p
        if op == "final_ln":
            y = self.ln(b["x1"][:, 3 + f], w["final_ln_w"], w["final_ln_b"])
            return y, y
        if op == "head":
            y = b["xn"][:, 3 + f] @ w["head_w"].T + w["head_b"]
            return y, y
        if op == "spec":
            return self.spec(b["sp"], f)
        if op == "idft":
            y = b["sp"][:, 3 + f, :2 * self.nb] @ w["idft_basis"][:, :2 * self.nb].T
            return y, y
        if op == "ola":
            y = self.ola(b["fr"], N)
            return y, y
        raise KeyError(name)


# ====================================================================================== error measures
def _finite(t) -> bool:
    return bool(torch.isfinite(t).all())


def row_errors(got, ref, scale):
    """Relative RMS per leading index over the last dim; inf wherever ``got`` is not finite."""
    e = (got - ref).norm(dim=-1) / scale.norm(dim=-1).clamp_min(1e-300)
    return torch.where(torch.isfinite(got).all(-1), e, torch.full_like(e, math.inf))


def stage_errors(kind: str, got, ref, scale, f, N: int, cfg) -> dict:
    """Named worst errors of one stage: see the module docstring for the measure of each kind."""
    if kind in ("fsq", "gemm", "norm", "rope"):
        e = row_errors(got, ref, scale)                                      # [B, F]
        edge = (f < 3) | (f >= N - 3)
        out = {"edge": float(e[:, edge].max())}
        if (~edge).any():
            out["interior"] = float(e[:, ~edge].max())
        return out
    if kind == "gn":
        B, F, C = got.shape
        G = cfg.groups
        g = lambda t: t.reshape(B, F, G, C // G).permute(0, 2, 1, 3).reshape(B, G, -1)
        return {"group": float(row_errors(g(got), g(ref), g(scale)).max())}
    if kind == "attn":
        B, F, C = got.shape
        h = lambda t: t.reshape(B, F, C // 64, 64).permute(0, 2, 1, 3).reshape(B, C // 64, -1)
        return {"head": float(row_errors(h(got), h(ref), h(scale)).max())}
    if kind == "spec":
        nb = cfg.n_fft // 2 + 1
        d = torch.complex(got[..., :nb] - ref[..., :nb], got[..., nb:] - ref[..., nb:]).abs() / scale
        return {"element": float(d.max()) if _finite(got) else math.inf}
    if kind == "ola":
        hop = cfg.hop
        return {"item": float(row_errors(got, ref, ref).max()),
                "first hop": float(row_errors(got[:, :hop], ref[:, :hop], ref[:, :hop]).max()),
                "last hop": float(row_errors(got[:, -hop:], ref[:, -hop:], ref[:, -hop:]).max())}
    raise KeyError(kind)


def record(key: str, mode: str, errs: dict, tag: str) -> None:
    worst = max(errs.values())
    if worst > WORST.get((key, mode), (-1.0, ""))[0]:
        WORST[(key, mode)] = (worst, tag)
    assert worst < BARS[key], (key, mode, tag, errs)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nCODEC-STAGES worst error per stage kind and mode (bar):")
        for (key, mode), (v, tag) in sorted(WORST.items()):
            print(f"  {key:13s} {mode:7s} {v:.3e}  ({BARS[key]:.0e})  at {tag}")
    for op, (v, tag) in sorted(TF32_FLOOR.items()):
        print(f"  plain TF32 {op:6s} smallest stage error {v:.3e} = {v / BARS[f'3xtf32-{op}']:.1f}x its 3xTF32 bar, at {tag}")


# ====================================================================================== decoders
FULL = dict(depth=2)
MAX_BATCH, MAX_FRAMES = 4, 2048


@functools.lru_cache(maxsize=None)
def _weights(tiny: bool, seed: int):
    cfg = CO.CodecConfig.tiny() if tiny else CO.CodecConfig(**FULL)
    return cfg, CO.random_weights(cfg, seed)


@functools.lru_cache(maxsize=None)
def decoder(mode: str, tiny: bool = False, rope_axis: str = "time"):
    from neutts_air_b200.codec import CodecDecoder

    cfg, w = _weights(tiny, 5)
    cfg = CO.CodecConfig(**{**cfg.__dict__, "rope_axis": rope_axis})
    mb, mf = (3, 300) if tiny else (MAX_BATCH, MAX_FRAMES)
    dec = CodecDecoder(codec_shape(cfg), codec_weight_dict(w), device="cuda:0", max_batch=mb, max_frames=mf,
                       precision=mode)
    return cfg, dec, Ref64(cfg, dec.w)


def buf_rows(dec) -> int:
    return dec.max_batch * (dec.max_frames + 6) + 8


def items(dec, cfg, name: str, B: int, N: int):
    """Float64 CPU copy of the item rows [B, N + 6, width] of workspace buffer ``name``."""
    wd = widths(cfg)[name]
    return dec.debug_buffer(name, (buf_rows(dec), wd))[:B * (N + 6)].cpu().double().view(B, N + 6, wd)


def item_view(dec, cfg, name: str, B: int, N: int):
    """Device view of the item rows [B, N + 6, width] of workspace buffer ``name`` (to write crafted inputs)."""
    wd = widths(cfg)[name]
    return dec.debug_buffer(name, (buf_rows(dec), wd))[:B * (N + 6)].view(B, N + 6, wd)


def pad_rows(B: int, N: int):
    return torch.tensor([b * (N + 6) + r for b in range(B) for r in (0, 1, 2, N + 3, N + 4, N + 5)], device="cuda:0")


def frames_checked(N: int, seed: int):
    """Every frame below N = 1024; above, the edge frames, the 128-frame tile boundaries and a seeded sample."""
    if N < 1024:
        return torch.arange(N)
    g = torch.Generator().manual_seed(seed)
    pick = {0, 1, 2, N - 3, N - 2, N - 1, 127, 128, 1023, 1024} | set(torch.randint(0, N, (54,), generator=g).tolist())
    return torch.tensor(sorted(pick))


def run_stage(dec, s: int, codes):
    dec.debug_set_stages(s, s)
    try:
        return dec.decode_code(codes, validate=False)
    finally:
        dec.debug_set_stages(0, -1)


# ====================================================================================== the stage walk
def walk(mode: str, B: int, N: int, seed: int, tiny: bool = False, rope_axis: str = "time") -> dict:
    cfg, dec, ref = decoder(mode, tiny, rope_axis)
    names = stage_names(cfg.depth, rope_axis == "time")
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, cfg.codebook_size, (B, 1, N), generator=g).cuda()
    other = torch.randint(0, cfg.codebook_size, (dec.max_batch, 1, dec.max_frames), generator=g).cuda()
    want = dec.decode_code(codes, validate=False).clone()
    dec.decode_code(other, validate=False)                 # stale rows everywhere past this call's
    for name, wd in widths(cfg).items():
        dec.debug_buffer(name, (buf_rows(dec), wd)).fill_(NAN)
    f = frames_checked(N, seed)
    pads = pad_rows(B, N)
    worst = {}
    for s, name in enumerate(names):
        op = name.rpartition(".")[2]
        ins, out, kind = IO[op]
        snap = {n: items(dec, cfg, n, B, N) for n in ins}
        pcm = run_stage(dec, s, codes)
        for x in ("x0", "x1", "x2"):
            assert bool((dec.debug_buffer(x, (buf_rows(dec), cfg.hidden))[pads] == 0).all()), (name, x, "pad rows")
        exp, scale = ref.run(name, snap, f, N, codes.cpu()[:, 0].long())
        if out == "pcm":
            got = pcm[:, 0].cpu().double()
        else:
            got = items(dec, cfg, out, B, N)[:, 3 + f, :exp.shape[-1]]
        errs = stage_errors(kind, got, exp, scale, f, N, cfg)
        key = kind if kind != "gemm" else "tf32" if gemm_bar(op, mode) == "tf32" else f"3xtf32-{op}"
        tag = f"{'tiny/' + rope_axis if tiny else 'full'} B={B} N={N} {name}"
        record(key, mode, errs, tag)
        if kind == "gemm" and mode == "tf32":
            # plain TF32 must be told apart from 3xTF32: the whole stage sits 10x above the 3xTF32 bar
            overall = float((got - exp).norm() / scale.norm())
            if overall < TF32_FLOOR.get(op, (math.inf, ""))[0]:
                TF32_FLOOR[op] = (overall, tag)
            assert overall > TF32_APART * BARS[f"3xtf32-{op}"], (tag, overall)
        worst[name] = max(errs.values())
    assert torch.equal(pcm, want), "a stage-by-stage decode differs from the one-call decode"
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("B", (1, 3))
@pytest.mark.parametrize("mode", MODES)
def test_stage_walk_full_width(cuda, mode, B):
    """Full widths (hidden 1024, 16 heads, MLP 4096, n_fft 1920, hop 480) at depth 2 on a decoder sized like the
    facade's (max_frames 2048): edge frame counts, 32-key tile edges and 128-query block edges."""
    for N in (1, 2, 3, 31, 32, 33, 127, 128, 129, 250):
        worst = walk(mode, B, N, seed=100 * B + N)
        print(f"WALK {mode} B={B} N={N}: worst {max(worst.values()):.2e} at {max(worst, key=worst.get)}")


@pytest.mark.gpu
def test_stage_walk_2048_frames(cuda):
    """The largest call the facade makes: N = max_frames = 2048, two items, 3xTF32."""
    worst = walk("3xtf32", 2, 2048, seed=7)
    print(f"WALK 3xtf32 B=2 N=2048: worst {max(worst.values()):.2e} at {max(worst, key=worst.get)}")


@pytest.mark.gpu
@pytest.mark.parametrize("rope_axis", ["time", "head"])
def test_stage_walk_tiny(cuda, rope_axis):
    """The tiny config: 4 channels per group, n_fft 64, hop 16; rope_axis "head" has no rope stage."""
    for N in (1, 2, 33, 129):
        walk("3xtf32", 2, N, seed=N, tiny=True, rope_axis=rope_axis)


@pytest.mark.gpu
def test_stage_range_is_validated(cuda):
    for tiny, axis in ((False, "time"), (True, "head")):
        cfg, dec, _ = decoder("3xtf32", tiny, axis)
        n = len(stage_names(cfg.depth, axis == "time"))
        dec.debug_set_stages(0, n - 1)
        dec.debug_set_stages(n - 1, n - 1)
        for first, last in ((0, n), (n, n), (n, -1), (-1, 0), (3, 2), (0, -2)):
            with pytest.raises(ValueError):
                dec.debug_set_stages(first, last)
        dec.debug_set_stages(0, -1)
        with pytest.raises(KeyError):
            dec.debug_buffer("pcm", (1,))


# ====================================================================================== crafted inputs
def _stage(cfg, name: str, rope: bool = True) -> int:
    return stage_names(cfg.depth, rope).index(name)


def _codes(B: int, N: int):
    return torch.zeros(B, 1, N, dtype=torch.int32, device="cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("N", (1, 33, 129, 2048))
def test_attention_crafted(cuda, N):
    """Needle keys at frames 0, 31, 32 and N-1 (the edges of the 32-key tiles), peaked softmax, and items whose
    values differ by orders of magnitude, so that a dropped tile, an unmasked key or a neighbour item's key is loud."""
    cfg, dec, ref = decoder("3xtf32")
    B, C, H = 3, cfg.hidden, cfg.heads
    g = torch.Generator().manual_seed(N)
    qkv = torch.full((B, N + 6, 3 * C), NAN, dtype=torch.float64)
    u = torch.nn.functional.normalize(torch.randn(H, 64, generator=g, dtype=torch.float64), dim=-1)
    needles = [j for j in (0, 31, 32, N - 1) if j < N]
    for b in range(B):
        q = 0.3 * torch.randn(N, H, 64, generator=g, dtype=torch.float64)
        k = 0.3 * torch.randn(N, H, 64, generator=g, dtype=torch.float64) + 0.5 * b
        v = (torch.randn(N, H, 64, generator=g, dtype=torch.float64) + 50 * b) * 10.0 ** b
        for h in range(H):
            if h < 8:                                  # needle heads: every query points at one key
                j = needles[h % len(needles)]
                q[:, h] += 3 * u[h]
                k[j, h] = 48 * u[h]
                v[j, h] = 1e3 * (b + 1) * torch.sign(u[h])
            else:                                      # peaked heads: scores spread over tens of units
                q[:, h] *= 12
        qkv[b, 3:3 + N] = torch.cat((q.reshape(N, C), k.reshape(N, C), v.reshape(N, C)), -1)
    item_view(dec, cfg, "qkv", B, N).copy_(qkv.float())
    item_view(dec, cfg, "att", B, N).fill_(NAN)
    run_stage(dec, _stage(cfg, "b0.attn"), _codes(B, N))
    snap = items(dec, cfg, "qkv", B, N)
    f = frames_checked(N, N)
    exp = ref.attn(snap, N, f)
    got = items(dec, cfg, "att", B, N)[:, 3 + f]
    record("attn-crafted", "3xtf32", stage_errors("attn", got, exp, exp, f, N, cfg), f"attn crafted N={N}")


@pytest.mark.gpu
def test_rope_positions_to_2047(cuda):
    cfg, dec, ref = decoder("3xtf32")
    B, N, C = 2, 2048, cfg.hidden
    g = torch.Generator().manual_seed(3)
    item_view(dec, cfg, "qkv", B, N)[:, 3:3 + N] = torch.randn(B, N, 3 * C, generator=g).cuda()
    snap = items(dec, cfg, "qkv", B, N)
    run_stage(dec, _stage(cfg, "b1.rope"), _codes(B, N))
    got = items(dec, cfg, "qkv", B, N)
    f = torch.arange(N)
    exp = ref.rope(snap[:, 3 + f], f)
    assert torch.equal(got[:, 3:3 + N, 2 * C:], snap[:, 3:3 + N, 2 * C:])       # v untouched
    record("rope", "3xtf32", stage_errors("rope", got[:, 3 + f], exp, exp, f, N, cfg), "rope t <= 2047")


@pytest.mark.gpu
@pytest.mark.parametrize("N", (1, 2048))
def test_groupnorm_dc_offset(cuda, N):
    """One group with a mean of 1e3 and unit spread: the statistics must not lose the spread."""
    cfg, dec, ref = decoder("3xtf32")
    B, C = 2, cfg.hidden
    cpg = C // cfg.groups
    g = torch.Generator().manual_seed(N)
    x = torch.zeros(B, N + 6, C)
    x[:, 3:3 + N] = torch.randn(B, N, C, generator=g)
    x[:, 3:3 + N, 5 * cpg:6 * cpg] += 1e3
    item_view(dec, cfg, "x1", B, N).copy_(x)
    run_stage(dec, _stage(cfg, "rn0.gn1"), _codes(B, N))
    f = torch.arange(N)
    exp = ref.gn_swish(x.double(), N, ref.w["rn_n1w"][0], ref.w["rn_n1b"][0], f)
    got = items(dec, cfg, "x2", B, N)[:, 3 + f]
    record("gn-dc", "3xtf32", stage_errors("gn", got, exp, exp, f, N, cfg), f"gn1 DC 1e3 N={N}")


@pytest.mark.gpu
def test_final_layernorm_large_mean(cuda):
    cfg, dec, ref = decoder("3xtf32")
    B, N, C = 2, 64, cfg.hidden
    g = torch.Generator().manual_seed(9)
    x = torch.zeros(B, N + 6, C)
    means = torch.tensor([0.0, 1e2, -1e3, 1e3, 3e3, -1e4])
    x[:, 3:3 + N] = torch.randn(B, N, C, generator=g) + means[torch.arange(N) % len(means)][None, :, None]
    item_view(dec, cfg, "x1", B, N).copy_(x)
    run_stage(dec, _stage(cfg, "final_ln"), _codes(B, N))
    f = torch.arange(N)
    exp = ref.ln(x.double()[:, 3 + f], ref.w["final_ln_w"], ref.w["final_ln_b"])
    got = items(dec, cfg, "xn", B, N)[:, 3 + f]
    record("norm-mean", "3xtf32", stage_errors("norm", got, exp, exp, f, N, cfg), "final LN, means to 1e4")


@pytest.mark.gpu
def test_spectrum_clip_edge_and_large_phases(cuda):
    """Log-magnitudes a few ulp either side of ln(mag_clip) and down to -30; phases up to +-1e3 rad."""
    cfg, dec, ref = decoder("3xtf32")
    B, N, nb = 2, 48, cfg.n_fft // 2 + 1
    g = torch.Generator().manual_seed(4)
    edge = torch.tensor(math.log(cfg.mag_clip), dtype=torch.float32)
    steps = torch.arange(-6, 7, dtype=torch.int32)
    near = (edge.view(torch.int32) + steps).view(torch.float32)                 # ln(clip) +- 6 ulp
    lm = torch.rand(B, N, nb, generator=g) * 36 - 30
    lm.view(-1)[:B * N * nb // 4] = near.repeat(B * N * nb // 4 // len(near) + 1)[:B * N * nb // 4]
    lm = lm.view(-1)[torch.randperm(B * N * nb, generator=g)].view(B, N, nb)
    ph = (torch.rand(B, N, nb, generator=g) * 2 - 1) * torch.logspace(0, 3, nb)
    sp = item_view(dec, cfg, "sp", B, N)
    sp[:, 3:3 + N, :nb] = lm.cuda()
    sp[:, 3:3 + N, nb:2 * nb] = ph.cuda()
    snap = items(dec, cfg, "sp", B, N)
    run_stage(dec, _stage(cfg, "spec"), _codes(B, N))
    f = torch.arange(N)
    exp, mag = ref.spec(snap, f)
    got = items(dec, cfg, "sp", B, N)[:, 3 + f, :2 * nb]
    assert float((snap[:, 3 + f, :nb] > math.log(cfg.mag_clip)).double().mean()) > 0.05    # the clip engages
    record("spec", "3xtf32", stage_errors("spec", got, exp, mag, f, N, cfg), "spec clip edge, phases 1e3")


@pytest.mark.gpu
@pytest.mark.parametrize("N", (1, 2, 3, 9))
def test_overlap_add_poisoned_pads_and_short_calls(cuda, N):
    """Every pad frame holds 1e30 (finite, so it survives every product), which must not reach the PCM; N <= 3 has
    fewer frames than the n_fft / hop = 4 that overlap."""
    cfg, dec, ref = decoder("3xtf32")
    B = 3
    g = torch.Generator().manual_seed(N)
    dec.debug_buffer("fr", (buf_rows(dec), cfg.n_fft)).fill_(1e30)
    item_view(dec, cfg, "fr", B, N)[:, 3:3 + N] = (torch.randn(B, N, cfg.n_fft, generator=g) * 0.1).cuda()
    snap = items(dec, cfg, "fr", B, N)
    pcm = run_stage(dec, _stage(cfg, "ola"), _codes(B, N))[:, 0].cpu().double()
    exp = ref.ola(snap, N)
    assert _finite(pcm)
    record("ola", "3xtf32", stage_errors("ola", pcm, exp, exp, torch.arange(N), N, cfg), f"ola poisoned pads N={N}")


@pytest.mark.gpu
def test_fsq_ids_outside_the_codebook(cuda):
    """CUDA codes skip range validation; every int32 id decodes as id mod levels**dims (floor modulo), exactly as the
    oracle's digits.  The digits are recovered from x0 by least squares against the affine and must be exact."""
    cfg, dec, ref = decoder("3xtf32")
    ids = [-1, -65536, -65537, 65536, 2**31 - 1, -2**31, 0, 65535, 12345]
    codes = torch.tensor(ids, dtype=torch.int32).view(1, 1, -1).cuda()
    N = len(ids)
    run_stage(dec, 0, codes)
    f = torch.arange(N)
    got = items(dec, cfg, "x0", 1, N)[:, 3 + f]
    want_z = CO.fsq_dequant(torch.tensor(ids, dtype=torch.int64), cfg).double()
    assert torch.equal(want_z, CO.fsq_dequant(torch.tensor(ids, dtype=torch.int64) % cfg.codebook_size, cfg).double())
    z = torch.linalg.lstsq(ref.w["fsq_w"], (got[0] - ref.w["fsq_b"]).T).solution.T          # [N, dims]
    half = cfg.fsq_levels // 2
    assert torch.equal(torch.round(z * half) / half, want_z), (z, want_z)
    exp = want_z @ ref.w["fsq_w"].T + ref.w["fsq_b"]
    record("fsq", "3xtf32", stage_errors("fsq", got, exp[None], exp[None], f, N, cfg), "fsq ids outside the codebook")


# ====================================================================================== CPU
def _cpu_ref(cfg, w):
    from neutts_air_b200.codec import pack_weights

    return Ref64(cfg, pack_weights(codec_shape(cfg), codec_weight_dict(w), "cpu"))


def emulate(ref: Ref64, codes, rope: bool):
    """The stage list run in float64 on a padded-batch workspace, with the stage references of this file."""
    cfg = ref.cfg
    B, N = codes.shape[0], codes.shape[-1]
    bufs = {n: torch.zeros(B, N + 6, wd, dtype=torch.float64) for n, wd in widths(cfg).items()}
    f = torch.arange(N)
    for name in stage_names(cfg.depth, rope):
        out = IO[name.rpartition(".")[2]][1]
        y, _ = ref.run(name, bufs, f, N, codes[:, 0].long())
        if out == "pcm":
            return y
        bufs[out][:, 3 + f, :y.shape[-1]] = y
    raise AssertionError("no ola stage")


@pytest.mark.parametrize("rope_axis", ["time", "head"])
def test_stage_references_chain_to_the_oracle(rope_axis):
    """The float64 stages of this file, run in the order of the stage list on the padded layout, are the decoder:
    they reproduce the oracle's fp32 decode to its own rounding."""
    cfg = CO.CodecConfig.tiny(rope_axis=rope_axis)
    w = CO.random_weights(cfg, 3)
    codes = torch.randint(0, cfg.codebook_size, (2, 1, 37), generator=torch.Generator().manual_seed(1))
    got = emulate(_cpu_ref(cfg, w), codes, rope_axis == "time")
    with torch.no_grad():
        want = CO.decode_code(codes, w, cfg)[:, 0].double()
    err = float((got - want).norm() / want.norm())
    assert err < 2e-5, err


def test_stage_list_matches_the_header():
    """The stage count per block in the header comment and this file's copy of the list agree."""
    import os

    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "neutts_b200.h")).read()
    assert "norm1 (x1 -> xn) | qkv (xn -> qkv) | rope (qkv in place) | attn (qkv -> att)" in hdr
    for depth, rope in ((2, True), (12, True), (2, False)):
        names = stage_names(depth, rope)
        assert len(names) == 2 + 16 + depth * (8 if rope else 7) + 5 == len(set(names))
        assert names[0] == "fsq" and names[-1] == "ola"


def test_fault_models_exceed_the_bars():
    """float64, CPU: each fault these checks exist to catch lands at least 10x past the bar of the stage that could
    commit it, measured the way the stage is checked."""
    cfg = CO.CodecConfig.tiny(hidden=1024, heads=16, n_fft=1920, hop=480)
    g = torch.Generator().manual_seed(0)
    ref = Ref64(cfg, {})
    lines = []

    def past(label, err, key):
        lines.append(f"{label} {err:.2e} ({err / BARS[key]:.0f}x {key})")
        assert err > 10 * BARS[key], (label, err, BARS[key])

    # a 3xTF32 GEMM computed from TF32 operands, at the K of each GEMM; every row must show it
    C = cfg.hidden
    for op, K in (("embed", 7 * C), ("conv1", 3 * C), ("conv2", 3 * C), ("qkv", C), ("proj", C), ("fc1", C),
                  ("fc2", 4 * C), ("head", C), ("idft", cfg.n_fft + 2)):
        a = torch.randn(32, K, generator=g)
        wt = torch.randn(256, K, generator=g) / math.sqrt(K)
        exact = a.double() @ wt.double().T
        plain = tf32_truncate(a).double() @ tf32_truncate(wt).double().T
        e = float(row_errors(plain, exact, exact).min())
        lines.append(f"TF32 operands in {op} (K={K}) {e:.2e} ({e / BARS['3xtf32-' + op]:.1f}x)")
        assert e > TF32_APART * BARS["3xtf32-" + op], (op, e)
    # the last partial key tile dropped (N = 33: 32 keys kept)
    N, B = 33, 2
    qkv = torch.randn(B, N + 6, 3 * cfg.hidden, generator=g, dtype=torch.float64)
    f = torch.arange(N)
    full = ref.attn(qkv, N, f)
    past("attention without the last key tile", stage_errors("attn", ref.attn(qkv, N, f, keys=torch.arange(32)), full,
                                                             full, f, N, cfg)["head"], "attn")
    # GroupNorm statistics over the N + 6 rows of the padded item (zero pads included)
    for N in (1, 250, 2048):
        x = torch.zeros(B, N + 6, cfg.hidden, dtype=torch.float64)
        x[:, 3:3 + N] = torch.randn(B, N, cfg.hidden, generator=g, dtype=torch.float64) + 0.3
        f = torch.arange(N)
        gw, gb = torch.ones(cfg.hidden, dtype=torch.float64), torch.zeros(cfg.hidden, dtype=torch.float64)
        good = ref.gn_swish(x, N, gw, gb, f)
        bad = ref.gn_swish(x, N, gw, gb, f, stat_rows=torch.arange(N + 6))
        past(f"GroupNorm stats over N+6 rows N={N}", stage_errors("gn", bad, good, good, f, N, cfg)["group"], "gn")
    # RoPE at position t + 1
    N = 2048
    rows = torch.randn(1, N, 3 * cfg.hidden, generator=g, dtype=torch.float64)
    f = torch.arange(N)
    good = ref.rope(rows, f)
    past("RoPE at t + 1", stage_errors("rope", ref.rope(rows, f + 1), good, good, f, N, cfg)["edge"], "rope")
    # the overlap-add envelope missing the first or the last frame
    for N in (1, 2, 5, 250):
        fr = torch.randn(B, N + 6, cfg.n_fft, generator=g, dtype=torch.float64) * 0.1
        good = ref.ola(fr, N)
        for drop, part in ((0, "first hop"), (N - 1, "last hop")):
            e = stage_errors("ola", ref.ola(fr, N, drop=drop), good, good, torch.arange(N), N, cfg)[part]
            past(f"OLA envelope without frame {drop} N={N}", e, "ola")
    # the spectrum without the clip, on log-magnitudes that reach 1 past ln(mag_clip)
    N, nb = 8, cfg.n_fft // 2 + 1
    sp = torch.zeros(B, N + 6, 2 * nb, dtype=torch.float64)
    sp[:, 3:3 + N, :nb] = math.log(cfg.mag_clip) + torch.rand(B, N, nb, generator=g, dtype=torch.float64) * 2 - 1
    sp[:, 3:3 + N, nb:] = torch.randn(B, N, nb, generator=g, dtype=torch.float64) * 10
    f = torch.arange(N)
    good, mag = ref.spec(sp, f)
    bad, _ = ref.spec(sp, f, clip=False)
    past("spectrum without the clip", stage_errors("spec", bad, good, mag, f, N, cfg)["element"], "spec")
    print("FAULTS: " + "; ".join(lines))
