"""Every speech-LM projection path against float64, on a model whose attention is an exact average.

The dense projections (q/k/v, o_proj, gate/up + SwiGLU, down_proj, the lm_head, their split-K slices, the folds that sum
the slices, and the persistent kernel's bf16 hi + lo activation pairs) are most of the arithmetic of a decode step.
The logit-parity tests see them on random weights at 2e-2 .. 3e-2 relative RMS, a bar that plain bf16 activations in
place of hi + lo pass, and that one missing K slice of one tile comes within a few times of.  The attention and sampler
tests take the projections out of the model on purpose.  The tests here put them back, at the precision each path
claims.

The average-attention model: ``wk = 0`` and ``bk = 0`` in every layer, so K is exactly 0 after RoPE, every score is 0
and every probability is ``2^0 = 1``, which bf16 holds exactly.  Every attention kernel (prefill, fp32 and mma decode,
the persistent kernel's split-KV merge) then returns the exact mean of the cached V rows of its context, up to fp32
summation.  Attention becomes a known linear function of the cache, so o_proj and everything after it can carry
random weights, each sublayer adding about as much as the residual it joins.  The untied lm_head has the identity in
rows ``0..H-1``, so ``logits[:H]`` is the final-normed residual and shows which 128-row tile of o_proj or down_proj is
wrong; the vocabulary (160 * 128 + 66) is even, not a multiple of 128, and has more 128-row tiles than the GPU has SMs.

The float64 reference recomputes the model for every token row, taking each layer's attention as the mean of the V
rows that run left in the paged cache: recomputing V would add ~1e-4 of bf16 rounding-flip noise and hide the hi + lo
path.  It rounds activations to bf16 where the path under test does (DESIGN.md §3):

    path                                                   activations rounded to bf16
    per-op chain, batch <= 4 (gemv_kernel)                 none
    persistent kernel, batch <= 8 (hi + lo pairs)          none
    prefill (wgmma GEMMs)                                  xn, attention out, SwiGLU out; lm_head input at batch > 4
    per-op chain at batch > 4, persistent kernel > 8       xn, attention out, SwiGLU out, lm_head input

Every case checks: every K row in the pool is exactly 0; the V row each layer appended, against float64 v rounded to
bf16; ``logits[:H]`` per 128-element tile and ``logits[H:]`` per row (relative RMS); in prefill also the final residual
of every token row at index >= max_batch (lower rows are re-embedded by the sampler).  Decode runs 4 teacher-forced
steps in one call and checks every step.  Slots above the batch hold "loud" tokens (embedding rows scaled by 256), and
a decode call at a larger batch (prefill: a prefill of every slot) runs first, so a leaked idle row moves the error by
orders of magnitude.

The persistent kernel runs the work plan its planner makes for its grid, the device's SM count unless
``debug_set_sms`` sets a smaller one.  ``test_decode_projections_at_every_plan`` runs the decode checks at one CTA
count per plan regime up to the device's count (tests.helpers.regime_representatives), at batches 1, 3 and 12, and
also checks each row's kept sampler window against the float64 sampler.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
import subprocess

import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import (GEMV_MAX_BATCH, decode_branch, gather_kv, gemm_splits, make_lm, plan_regime, plan_summary,
                           regime_representatives, rel_rms, set_decode_impl)
from tests.sampler_ref import prob_err, ref_window

# Worst errors measured on one H100 80GB HBM3 (132 SMs, 400 W power limit) over the whole case matrix, and the bars,
# ~4x above.  Relative RMS of logits[:H] per (row, 128-element tile), of logits[H:] per row and of the prefill residual
# per row; the appended V row per (row, layer) against float64 v rounded to bf16.
#   fp32 GEMV chain (batch <= 4)                                          3.1e-7  -> 1.2e-6
#   persistent kernel, hi + lo activations (batch <= 8)                   6.9e-6  -> 3e-5
#   bf16 activations (chain > 4, persistent > 8), mirrored roundings      3.6e-3  -> 1.5e-2
#   prefill (wgmma GEMMs), mirrored roundings                             3.2e-3  -> 1.3e-2
#   appended V row, fp32 and hi + lo paths (a rare flip of its rounding)  5.6e-4  -> 2.2e-3
#   appended V row, bf16 activations and prefill                          4.2e-3  -> 1.7e-2
# On the bf16 paths the floor is the rounding itself: one flipped bf16 rounding of a SwiGLU output moves the residual
# and flips more roundings downstream (test_fault_models_exceed_the_bars).
BARS = {"fp32": 1.2e-6, "hilo": 3e-5, "bf16": 1.5e-2, "prefill": 1.3e-2, "v-exact": 2.2e-3, "v-bf16": 1.7e-2}

VOCAB = 160 * 128 + 66            # 20546
EOS = VOCAB - 1
N_LOUD = 64
LOUD0 = EOS - N_LOUD              # ids [LOUD0, EOS): embedding rows scaled by 256 (exact in bf16)
N_LAYERS = 3
STEPS = 4
MAX_CTX = 512
# NeuTTS-Air and NeuTTS-Nano widths, a small model, the Nano-like model bench.py measures in its streaming line (8 query
# / 2 KV heads: GQA ratio 4) and Air widths over 16 query / 4 KV heads
SHAPES = {"air": (896, 4864, 14, 2), "nano": (576, 1536, 9, 3), "small": (256, 640, 4, 2), "bench": (512, 2048, 8, 2),
          "air16x4": (896, 4864, 16, 4)}

NONE = frozenset()
PREFILL_GEMV = frozenset({"x", "attn", "act"})
BF16 = frozenset({"x", "attn", "act", "head"})


# ====================================================================================== the model
@functools.lru_cache(maxsize=None)
def avg_model(shape: str, seed: int = 0):
    """(cfg, weights) of the average-attention model at the widths of ``shape`` (bf16-representable float32)."""
    H, I, nh, nkv = SHAPES[shape]
    cfg = O.LMConfig(vocab_size=VOCAB, hidden_size=H, intermediate_size=I, num_layers=N_LAYERS, num_heads=nh,
                     num_kv_heads=nkv, head_dim=64, tie_embeddings=False)
    g = torch.Generator().manual_seed(seed)

    def rn(*shape_, std):
        return (torch.randn(*shape_, generator=g) * std).bfloat16().float()

    layers = []
    for _ in range(N_LAYERS):
        layers.append(dict(
            ln1=1 + 0.1 * torch.randn(H, generator=g), wq=rn(64 * nh, H, std=H ** -0.5), bq=rn(64 * nh, std=0.1),
            wk=torch.zeros(64 * nkv, H), bk=torch.zeros(64 * nkv),
            wv=rn(64 * nkv, H, std=H ** -0.5), bv=rn(64 * nkv, std=1.0), wo=rn(H, 64 * nh, std=(64 * nh) ** -0.5),
            ln2=1 + 0.1 * torch.randn(H, generator=g), wg=rn(I, H, std=H ** -0.5), wu=rn(I, H, std=H ** -0.5),
            wd=rn(H, I, std=2 * I ** -0.5)))
    embed = rn(VOCAB, H, std=1.0)
    embed[LOUD0:EOS] *= 256
    head = rn(VOCAB, H, std=H ** -0.5)
    head[:H] = torch.eye(H)
    w = O.LMWeights(embed=embed, layers=layers, final_norm=1 + 0.1 * torch.randn(H, generator=g), lm_head=head)
    return cfg, w


@functools.lru_cache(maxsize=None)
def weights64(shape: str):
    cfg, w = avg_model(shape)
    d = lambda t: t.double()
    layers = [{k: d(v) for k, v in L.items()} for L in w.layers]
    return cfg, dict(embed=d(w.embed), layers=layers, fn=d(w.final_norm), head=d(w.lm_head))


# ====================================================================================== float64 reference
def _bf(t):
    return t.bfloat16().double()


def _rms(h, w, eps):
    return h / torch.sqrt(h.pow(2).mean(-1, keepdim=True) + eps) * w


def forward64(shape: str, toks, attn_of, rb=NONE, fault=None):
    """The average-attention model in float64 for token rows ``toks`` [R].  ``attn_of(layer, v)`` returns the rows'
    attention output [R, n_heads * 64] given the layer's float64 v [R, n_kv * 64].  ``rb``: which activations are
    rounded to bf16 ("x": both RMSNorm outputs, "attn", "act": SwiGLU out, "head": the lm_head input).  ``fault``:
    (layer, "o" | "d", tile, k0, k1, factor) scales the K range [k0, k1) of that 128-row tile of o_proj / down_proj by
    ``factor`` (0: a dropped slice, 2: a slice counted twice).  Returns dict(h, v: [layers], logits)."""
    cfg, W = weights64(shape)
    r = lambda t, what: _bf(t) if what in rb else t
    h = W["embed"][torch.as_tensor(toks, dtype=torch.long)]
    vs = []

    def proj(x, w, l, ph):
        y = x @ w.T
        if fault and fault[0] == l and fault[1] == ph:
            _, _, t, k0, k1, f = fault
            rows = slice(128 * t, 128 * t + 128)
            y[:, rows] += (f - 1) * (x[:, k0:k1] @ w[rows, k0:k1].T)
        return y

    for l, L in enumerate(W["layers"]):
        x = r(_rms(h, L["ln1"], cfg.rms_eps), "x")
        v = x @ L["wv"].T + L["bv"]
        vs.append(v)
        a = attn_of(l, v)
        h = h + proj(r(a, "attn"), L["wo"], l, "o")
        x = r(_rms(h, L["ln2"], cfg.rms_eps), "x")
        g, u = x @ L["wg"].T, x @ L["wu"].T
        h = h + proj(r(torch.nn.functional.silu(g) * u, "act"), L["wd"], l, "d")
    y = r(_rms(h, W["fn"], cfg.rms_eps), "head")
    return dict(h=h, v=vs, logits=y @ W["head"].T)


def heads_of(mean_v, nrep: int):
    """Attention output [R, n_heads * 64] from the mean V rows [R, n_kv, 64]: query head h reads KV head h // nrep."""
    return mean_v.repeat_interleave(nrep, dim=1).reshape(mean_v.shape[0], -1)


def causal_mean_attn(seq_lens, nrep: int):
    """attn_of for rows that are sequences laid back to back, V taken from the model itself rounded to bf16 (as the
    cache stores it): every row averages the V rows of its sequence up to itself."""
    def attn_of(_, v):
        out, t0 = [], 0
        for n in seq_lens:
            vb = _bf(v[t0: t0 + n]).view(n, -1, 64)
            out.append(vb.cumsum(0) / torch.arange(1, n + 1, dtype=torch.float64)[:, None, None])
            t0 += n
        return heads_of(torch.cat(out), nrep)
    return attn_of


def logit_errors(got, ref, H: int):
    """(worst relative RMS over (row, 128-element tile) of logits[:, :H], worst over rows of logits[:, H:])."""
    if not torch.isfinite(got).all():
        return math.inf, math.inf
    g, r = got.double(), ref.double()
    head = max(rel_rms(g[i, t: t + 128], r[i, t: t + 128]) for i in range(g.shape[0]) for t in range(0, H, 128))
    tail = max(rel_rms(g[i, H:], r[i, H:]) for i in range(g.shape[0]))
    return head, tail


def row_errors(got, ref):
    """Worst relative RMS over rows."""
    return max(rel_rms(got[i], ref[i]) for i in range(got.shape[0]))


# ---------------------------------------------------------------------------------------- CPU tests
def test_average_model_attention_is_the_mean():
    """wk = bk = 0: the oracle's softmax attention equals the plain mean of V (the premise of every case)."""
    cfg, w = avg_model("small")
    g = torch.Generator().manual_seed(1)
    toks = torch.randint(0, LOUD0, (9,), generator=g)
    L0 = w.layers[0]
    x = O.rms_norm(w.embed[toks], L0["ln1"], cfg.rms_eps)
    q = (x @ L0["wq"].T + L0["bq"]).view(9, cfg.num_heads, 64)
    k = (x @ L0["wk"].T + L0["bk"]).view(9, cfg.num_kv_heads, 64)
    v = (x @ L0["wv"].T + L0["bv"]).view(9, cfg.num_kv_heads, 64)
    assert not k.any()
    nrep = cfg.num_heads // cfg.num_kv_heads
    got = O.attention(q, k, v, 0, nrep).reshape(9, -1).double()
    want = heads_of(v.double().cumsum(0) / torch.arange(1, 10, dtype=torch.float64)[:, None, None], nrep)
    assert rel_rms(got, want) < 1e-6


@pytest.mark.parametrize("shape", ["small", "nano"])
def test_forward64_matches_the_oracle(shape):
    """With exact activations and V rounded to bf16 as cached, forward64 over back-to-back sequences is the oracle's
    forward pass of each sequence (its "decode" rounding points: K/V bf16, everything else fp32)."""
    cfg, w = avg_model(shape)
    H = cfg.hidden_size
    g = torch.Generator().manual_seed(2)
    lens = [11, 1, 5]
    toks = torch.randint(0, LOUD0, (sum(lens),), generator=g)
    toks[3] = LOUD0 + 5                        # a loud token: its residual is 256x larger
    ref = forward64(shape, toks, causal_mean_attn(lens, cfg.num_heads // cfg.num_kv_heads))
    want = torch.cat([O.forward(cfg, w, s, mirror="decode")[0] for s in toks.split(lens)])
    assert rel_rms(ref["logits"], want) < 1e-5
    # logits[:H] is the final-normed residual: the identity rows of the lm_head
    assert rel_rms(ref["logits"][:, :H], _rms(ref["h"], weights64(shape)[1]["fn"], cfg.rms_eps)) < 1e-14
    # each sublayer adds about as much as the residual it joins: the final residual of a normal row has RMS ~ 2..4
    rms = ref["h"].pow(2).mean(-1).sqrt()
    assert ((rms > 1.5) & (rms < 6)).sum() == len(toks) - 1 and rms[3] > 100


def _plan_shape(shape: str) -> tuple:
    """(hidden, inter, n_heads, n_kv, vocab): the key of the tests.helpers plan functions."""
    return SHAPES[shape] + (VOCAB,)


def _most_slices(shape: str):
    """(o_proj, down_proj) K slices of the plans that cut them finest, over every plan the planner accepts on 8..256
    CTAs (read from the library, no GPU needed): the smallest slice any decode can run."""
    plans = [p for G in range(8, 257) for flat in (False, True)
             if (p := plan_summary(_plan_shape(shape), G, flat)) is not None]
    return max(p[1] for p in plans), max(p[2] for p in plans)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_fault_models_exceed_the_bars(shape):
    """float64, CPU: the faults these tests exist to catch move the error past the bar of every path that could commit
    them.  Activations rounded to bf16 instead of hi + lo: at least 10x past the hi + lo and fp32 bars.  One K slice of
    one o_proj / down_proj tile dropped, or counted twice, with the slice bounds of the plan that cuts that GEMM finest
    at any CTA count from 8 to 256 (the smallest slice): at least 10x past the hi + lo and fp32 bars, and at
    least 5x past the bf16 and prefill bars.  Those two sit on the noise floor of bf16 activations themselves: a
    rounding flip of one SwiGLU output moves the residual, which flips more roundings in the next layer, so even an fp32
    implementation with the same rounding points is ~4e-3 from the float64 mirror after three layers."""
    cfg, _ = avg_model(shape)
    H = cfg.hidden_size
    nrep = cfg.num_heads // cfg.num_kv_heads
    g = torch.Generator().manual_seed(3)
    lens = [1, 7, 24]
    toks = torch.randint(0, LOUD0, (sum(lens),), generator=g)
    attn_of = causal_mean_attn(lens, nrep)
    exact = forward64(shape, toks, attn_of)
    worst = lambda ref: max(logit_errors(ref["logits"], exact["logits"], H))
    bf16 = worst(forward64(shape, toks, attn_of, rb=BF16))
    lines = [f"bf16 activations {bf16:.2e}"]
    assert bf16 > 10 * max(BARS["hilo"], BARS["fp32"]), bf16
    for ph, KB, S in zip(("o", "d"), (cfg.num_heads, cfg.intermediate_size // 64), _most_slices(shape)):
        for z, t, f in ((S - 1, 0, 0), (S // 2, (H - 1) // 128, 2)):   # the last slice of tile 0; a middle one, last tile
            k0, k1 = 64 * (KB * z // S), 64 * (KB * (z + 1) // S)
            e = worst(forward64(shape, toks, attn_of, fault=(1, ph, t, k0, k1, f)))
            lines.append(f"{ph} tile {t} slice {z}/{S} x{f}: {e:.2e}")
            assert e > 10 * max(BARS["hilo"], BARS["fp32"]), (ph, z, f, e)
            assert e > 5 * max(BARS["bf16"], BARS["prefill"]), (ph, z, f, e)
    print(f"FAULTS {shape}: " + "; ".join(lines))


# ====================================================================================== GPU cases
def _sms() -> int:
    return min(torch.cuda.get_device_properties(0).multi_processor_count, 256)


def _card() -> str:
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "power limit unknown"
    return f"{name}, {_sms()} SMs, {pl}"


def _decode(lm, B: int, steps: int, sp):
    """One nt_lm_decode call over slots 0..B-1 (B may be below the batch the engine was prefilled with)."""
    from neutts_air_b200 import _lib

    logits = torch.empty(steps, B, VOCAB, dtype=torch.float32, device=lm.device)
    n0 = lm.L.nt_launch_count()
    _lib.check(lm.L.nt_lm_decode(lm.handle, C.byref(lm.state), B, steps, C.byref(sp), logits.data_ptr(),
                                 _lib.current_stream_ptr()))
    torch.cuda.synchronize()
    return logits.cpu(), lm.L.nt_launch_count() - n0


# (id, shape, batch, NT_DECODE_IMPL, branch)
DECODE_CASES = [
    ("air-tc-b1", "air", 1, None, "tc-hilo-n16-flat-fold"),
    ("air-tc-b3", "air", 3, None, "tc-hilo-n16-wholeK-phases"),
    ("air-tc-b8", "air", 8, None, "tc-hilo-n16-wholeK-phases"),
    ("air-tc-b9", "air", 9, None, "tc-bf16-n16-wholeK-phases"),
    ("air-tc-b16", "air", 16, None, "tc-bf16-n16-wholeK-phases"),
    ("air-tc-b20", "air", 20, "tc", "tc-bf16-n32-wholeK-phases"),
    ("air-tc-b40", "air", 40, "tc", "tc-bf16-n64-wholeK-phases"),
    ("air-chain-b1", "air", 1, "perop", "gemv"),
    ("air-chain-b4", "air", 4, "perop", "gemv"),
    ("air-chain-b6", "air", 6, "perop", "gemm"),
    ("air-chain-b17", "air", 17, None, "gemm"),
    ("nano-tc-b1", "nano", 1, None, "tc-hilo-n16-wholeK-fold"),
    ("nano-tc-b6", "nano", 6, None, "tc-hilo-n16-wholeK-phases"),
    ("small-tc-b1", "small", 1, None, "tc-hilo-n16-flat-fold"),
    ("small-tc-b12", "small", 12, None, "tc-bf16-n16-wholeK-phases"),
    ("bench-tc-b1", "bench", 1, None, "tc-hilo-n16-wholeK-fold"),
    ("bench-tc-b3", "bench", 3, None, "tc-hilo-n16-wholeK-phases"),
    ("bench-tc-b8", "bench", 8, None, "tc-hilo-n16-wholeK-phases"),
    ("bench-tc-b9", "bench", 9, None, "tc-bf16-n16-wholeK-phases"),
    ("bench-tc-b16", "bench", 16, None, "tc-bf16-n16-wholeK-phases"),
    ("bench-chain-b4", "bench", 4, "perop", "gemv"),
    ("bench-chain-b6", "bench", 6, "perop", "gemm"),
    ("air16x4-tc-b1", "air16x4", 1, None, "tc-hilo-n16-flat-fold"),
    ("air16x4-tc-b8", "air16x4", 8, None, "tc-hilo-n16-wholeK-phases"),
]


def _check_rows(lm, rows, ref):
    """Worst error of the V rows the run appended, over layers and rows = [(slot, position)] in the order of ref's
    rows, against float64 v rounded to bf16."""
    got = _v_rows(lm, rows)
    return max(row_errors(got[l], _bf(ref["v"][l])) for l in range(N_LAYERS))


def _v_rows(lm, rows):
    """The V rows [layers, len(rows), n_kv * 64] at rows = [(slot, position)] of the run's cache."""
    return torch.stack([torch.stack([gather_kv(lm, l, b, p + 1)[1][p] for b, p in rows]).reshape(len(rows), -1)
                        for l in range(N_LAYERS)])


def _mean_v_from_cache(lm, shape, rows):
    """attn_of reading the run's cache: row (slot b, position p) averages slot b's V rows 0..p of the layer."""
    cfg, _ = avg_model(shape)
    nrep = cfg.num_heads // cfg.num_kv_heads
    cache = {}

    def attn_of(l, _):
        out = []
        for b, p in rows:
            if (l, b) not in cache:
                V = gather_kv(lm, l, b, max(pp for bb, pp in rows if bb == b) + 1)[1]
                cache[(l, b)] = V.cumsum(0) / torch.arange(1, V.shape[0] + 1, dtype=torch.float64)[:, None, None]
            out.append(cache[(l, b)][p])
        return heads_of(torch.stack(out), nrep)
    return attn_of


def _path_key(kind: str, B: int) -> str:
    if kind == "tc":
        return "hilo" if B <= 8 else "bf16"
    return "fp32" if B <= GEMV_MAX_BATCH else "bf16"


@pytest.mark.gpu
@pytest.mark.parametrize("case", DECODE_CASES, ids=[c[0] for c in DECODE_CASES])
def test_decode_projections_vs_float64(cuda, case, monkeypatch):
    """4 teacher-forced decode steps in one call at batch B, after a call at B + 2 that decoded the loud slots too;
    every step's logits and every appended V row against the float64 model on the run's own cache."""
    name, shape, B, impl, branch = case
    cfg, w = avg_model(shape)
    H = cfg.hidden_size
    MB = B + 2
    lm = make_lm(cfg, w, max_batch=MB, max_ctx=MAX_CTX, page_shuffle_seed=B)
    g = torch.Generator().manual_seed(1000 + B)
    lens = [int(n) for n in torch.randint(1, 300, (MB,), generator=g)]
    lens[0] = 299   # one slot past 4 pages
    loud = lambda n: torch.randint(LOUD0, EOS, (n,), generator=g)
    normal = lambda n: torch.randint(0, LOUD0, (n,), generator=g)
    prompts = [(normal(n) if b < B else loud(n)).tolist() for b, n in enumerate(lens)]
    forced = torch.stack([normal(STEPS + 2) if b < B else loud(STEPS + 2) for b in range(MB)])
    sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=STEPS + 4, forced=forced)
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    br = decode_branch(_plan_shape(shape), B, _sms(), MAX_CTX, impl)
    persistent = br["kind"] == "tc"
    set_decode_impl(monkeypatch, "tc" if persistent else "perop")
    _decode(lm, MB, 1, sp)                    # the earlier call: every slot, the loud ones included
    set_decode_impl(monkeypatch, impl)
    logits, launches = _decode(lm, B, STEPS, sp)

    # the branch
    assert br["name"] == branch
    assert launches == 1 if persistent else launches > STEPS, launches
    kind = br["kind"]
    key = _path_key(kind, B)
    rb = NONE if key in ("hilo", "fp32") else BF16

    assert not lm.kv[:, 0].any(), "a K row is not 0"
    rows = [(b, lens[b] + 1 + s) for s in range(STEPS) for b in range(B)]
    toks = [int(forced[b, 1 + s]) for s in range(STEPS) for b in range(B)]
    attn_of = _mean_v_from_cache(lm, shape, rows)
    ref = forward64(shape, toks, attn_of, rb=rb)
    got = logits.reshape(STEPS * B, VOCAB)
    head, tail = logit_errors(got, ref["logits"], H)
    vrow = _check_rows(lm, rows, ref)
    msg = (f"PROJ {name} [{branch}, {launches} launches, {_card()}]: logits[:H] tile {head:.2e} logits[H:] {tail:.2e} "
           f"V row {vrow:.2e} (bar {BARS[key]:.1e})")
    if key == "hilo":
        fault = max(logit_errors(forward64(shape, toks, attn_of, rb=BF16)["logits"], ref["logits"], H))
        msg += f"; bf16-activation fault model {fault:.2e} ({fault / max(head, tail, 1e-30):.0f}x)"
        assert max(head, tail) * 100 < fault, (head, tail, fault)
    print(msg)
    assert head < BARS[key] and tail < BARS[key], (head, tail)
    assert vrow < BARS["v-bf16" if key == "bf16" else "v-exact"], vrow


# The CTA-count sweep: one engine per shape, batches run at every count
SWEEP_BATCHES = (1, 3, 12)
SWEEP_MAX_BATCH = 14
# test_gpu_sampler.py's bar on the kept probabilities, max |p - p64| (tests/sampler_ref.py: BARS["prob"])
PROB_BAR = 4e-7


def _sweep_case(lm, shape: str, G: int, B: int, cap, monkeypatch):
    """One case of the sweep at G CTAs and batch B, checked as in test_decode_projections_vs_float64, with the 4
    teacher-forced steps in launches of 1 + 3 at batch 1 (fold counters and ping-pong parity carry across a launch),
    and the last launch's kept sampler windows against the float64 sampler on the returned logits.  Returns the
    logits, the appended V rows and the line to print."""
    cfg, _ = avg_model(shape)
    H = cfg.hidden_size
    MB = B + 2
    g = torch.Generator().manual_seed(3000 + B)
    lens = [int(n) for n in torch.randint(1, 300, (MB,), generator=g)]
    lens[0] = 299   # one slot past 4 pages
    loud = lambda n: torch.randint(LOUD0, EOS, (n,), generator=g)
    normal = lambda n: torch.randint(0, LOUD0, (n,), generator=g)
    prompts = [(normal(n) if b < B else loud(n)).tolist() for b, n in enumerate(lens)]
    forced = torch.stack([normal(STEPS + 2) if b < B else loud(STEPS + 2) for b in range(MB)])
    sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=STEPS + 4, forced=forced)
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    br = decode_branch(_plan_shape(shape), B, G, MAX_CTX)
    persistent = br["kind"] == "tc"
    set_decode_impl(monkeypatch, "tc" if persistent else "perop")
    _decode(lm, MB, 1, sp)                    # the earlier call: every slot, the loud ones included
    set_decode_impl(monkeypatch, None)
    runs = [_decode(lm, B, n, sp) for n in ((1, STEPS - 1) if B == 1 else (STEPS,))]
    logits, launches = torch.cat([r[0] for r in runs]), sum(r[1] for r in runs)
    assert launches == len(runs) if persistent else launches > STEPS, (shape, G, B, br["name"], launches)

    key = _path_key(br["kind"], B)
    assert not lm.kv[:, 0].any(), "a K row is not 0"
    rows = [(b, lens[b] + 1 + s) for s in range(STEPS) for b in range(B)]
    toks = [int(forced[b, 1 + s]) for s in range(STEPS) for b in range(B)]
    ref = forward64(shape, toks, _mean_v_from_cache(lm, shape, rows), rb=NONE if key in ("hilo", "fp32") else BF16)
    head, tail = logit_errors(logits.reshape(STEPS * B, VOCAB), ref["logits"], H)
    v = _v_rows(lm, rows)
    vrow = max(row_errors(v[l], _bf(ref["v"][l])) for l in range(N_LAYERS))
    vbar = BARS["v-bf16" if key == "bf16" else "v-exact"]

    tv, ti, tt = (t.cpu().numpy() for t in cap)
    perr = 0.0
    for b in range(B):
        ids, p = ref_window(logits[-1, b].numpy(), 0, EOS, 0, 50, 1.0)
        assert ti[b, : len(ids)].tolist() == ids.tolist() and (ti[b, len(ids):] == -1).all(), (shape, G, B, b)
        assert tt[b] == forced[b, STEPS + 1], (shape, G, B, b)
        perr = max(perr, prob_err(tv[b, : len(ids)], p))

    line = (f"PROJ-SMS {shape} G={G} B={B} [{br['name']}, split_cap {br['split_cap']}, {launches} launches]: "
            f"logits[:H] tile {head:.2e} logits[H:] {tail:.2e} (bar {BARS[key]:.1e}) V row {vrow:.2e} (bar {vbar:.1e}) "
            f"kept p {perr:.1e} (bar {PROB_BAR:.0e})")
    assert head < BARS[key] and tail < BARS[key], line
    assert vrow < vbar, line
    assert perr < PROB_BAR, line
    return logits, v, br, line


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_decode_projections_at_every_plan(cuda, shape, monkeypatch):
    """The decode cases of test_decode_projections_vs_float64 at one CTA count per plan regime the planner makes up to
    the device's SM count (tests.helpers.regime_representatives), set with ``debug_set_sms``, at batches 1, 3 and 12.
    The engine takes the branch decode_branch predicts, the per-op chain where the persistent kernel has no plan or
    too few CTAs.  The sweep starts and ends at the device's count, and those two runs must agree bit for bit: a change
    of count leaves nothing stale in the plan, the fold counters or the stamps."""
    cfg, w = avg_model(shape)
    dev = _sms()
    card = _card()
    lm = make_lm(cfg, w, max_batch=SWEEP_MAX_BATCH, max_ctx=MAX_CTX, page_shuffle_seed=7)
    cap = lm.debug_capture_sampler()
    reps = sorted(regime_representatives(_plan_shape(shape), dev).values())
    counts = [None] + reps + [0]      # None: the engine as created; 0: the device's count restored
    first, caps, plans, seen = {}, set(), set(), []
    for G in counts:
        if G is not None:
            lm.debug_set_sms(G)
        g_eff = G or dev
        for B in SWEEP_BATCHES:
            logits, v, br, line = _sweep_case(lm, shape, g_eff, B, cap, monkeypatch)
            print(f"{line} [{card}]")
            if br["kind"] == "tc":
                caps.add(br["split_cap"])
                plans.add(br["plan"])
            if G is None:
                first[B] = (logits, v)
            elif G == 0:
                assert torch.equal(logits, first[B][0]) and torch.equal(v, first[B][1]), (shape, B)
        seen.append(g_eff)
    print(f"PROJ-SMS {shape}: {len(reps)} regimes at CTA counts {seen}; split_cap {sorted(caps)}; plans {sorted(plans)}")
    assert {1, 8} <= caps, caps
    regimes = [plan_regime(_plan_shape(shape), G) for G in reps]
    want = {"wholeK"} if any(wk for wk, _ in regimes) else set()
    if any(wk and fl for wk, fl in regimes):
        want.add("flat")
    assert plans == want, (plans, want)


@pytest.mark.gpu
def test_debug_set_sms_refuses_counts_the_device_cannot_run(cuda):
    cfg, w = avg_model("small")
    lm = make_lm(cfg, w, max_batch=1, max_ctx=MAX_CTX)
    top = min(torch.cuda.get_device_properties(0).multi_processor_count, 256)
    for n in (-1, 7, top + 1):
        with pytest.raises(ValueError, match=f"not in 8..{top}"):
            lm.debug_set_sms(n)
    lm.debug_set_sms(8)
    lm.debug_set_sms(top)
    lm.debug_set_sms(0)


# (id, shape, lens, split-K GEMMs)
PREFILL_CASES = [("air-prefill-b3-t70", "air", [17, 1, 52], True),
                 ("air-prefill-b6-t700", "air", [200, 64, 129, 1, 250, 56], False),
                 ("bench-prefill-b5-t90", "bench", [33, 1, 17, 38, 1], True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PREFILL_CASES, ids=[c[0] for c in PREFILL_CASES])
def test_prefill_projections_vs_float64(cuda, case):
    """A ragged prefill after a prefill of every slot with loud prompts: the last-row logits, the final residual of
    every token row at index >= max_batch and every V row, against the float64 model on the run's own cache."""
    name, shape, lens, split = case
    B = len(lens)
    cfg, w = avg_model(shape)
    H, I, nh, nkv = SHAPES[shape]
    MB = B + 2
    lm = make_lm(cfg, w, max_batch=MB, max_ctx=MAX_CTX, page_shuffle_seed=B)
    g = torch.Generator().manual_seed(2000 + B)
    sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=4)
    lm.prefill([torch.randint(LOUD0, EOS, (300,), generator=g).tolist() for _ in range(MB)], sp)
    prompts = [torch.randint(0, LOUD0, (n,), generator=g).tolist() for n in lens]
    T = sum(lens)
    ws = 8 * 128 * max((nh + 2 * nkv) * 64, H)                      # lm->splitk_floats
    splits = [gemm_splits(T, N, K, ws) for N, K in (((nh + 2 * nkv) * 64, H), (H, 64 * nh), (H, I))]
    assert all(s > 1 for s in splits) if split else all(s == 1 for s in splits), splits
    logits = lm.prefill(prompts, sp, return_logits=True)
    torch.cuda.synchronize()
    h_run = lm.debug_buffer("h", (T, H)).double().cpu()
    assert not lm.kv[:, 0].any(), "a K row is not 0"
    rows = [(b, p) for b, n in enumerate(lens) for p in range(n)]
    toks = [t for p in prompts for t in p]
    gemv = B <= GEMV_MAX_BATCH            # the prefill's lm_head runs as a GEMV
    rb = PREFILL_GEMV if gemv else BF16
    ref = forward64(shape, toks, _mean_v_from_cache(lm, shape, rows), rb=rb)
    last = torch.tensor(lens).cumsum(0) - 1
    head, tail = logit_errors(logits.cpu(), ref["logits"][last], H)
    hres = row_errors(h_run[MB:], ref["h"][MB:])
    vrow = _check_rows(lm, rows, ref)
    print(f"PROJ {name} [split-K {splits}, lm_head {'GEMV' if gemv else 'wgmma'}, {_card()}]: logits[:H] tile "
          f"{head:.2e} logits[H:] {tail:.2e} residual rows >= {MB} {hres:.2e} V row {vrow:.2e}")
    assert max(head, tail, hres) < BARS["prefill"], (head, tail, hres)
    assert vrow < BARS["v-bf16"], vrow
