"""Every speech-LM attention kernel against float64 attention over its own paged KV cache.

The whole-layer and logit parity tests see attention only through the residual stream, at bars (6e-3 .. 2e-2
relative RMS) that a skipped page, a dropped split-KV partial or one leaked masked row can hide under: with random
weights, attention over a long context is nearly uniform, so its output is close to the mean of V.  The tests here
compare each kernel's attention itself with float64 attention computed from the very operands the kernel read (its
own query where a buffer exposes it, the K/V rows it left in the paged cache), on inputs built to make such bugs
loud: peaked softmax, "needle" keys on the first, far and last pages, and poison (huge K and V) in every cache row
a kernel must not read.

Kernels and how each is observed:
  * prefill (``attn_prefill_kernel``): the ``attn_bf16`` buffer against ``ref_attention(mirror="mma")`` on the
    ``q`` buffer and the cached K/V, per sequence and head, for GQA ratios 1 to 8;
  * prefill RoPE + KV append (``rope_append_kernel``): the ``q`` buffer and every cached K and V row against the
    float64 projection of the embedding, RoPE'd, with and without split-K slices of the qkv GEMM to sum;
  * per-op decode chain, fp32 (``attn_decode_kernel``, batch <= 4) and tensor-core (``attn_decode_mma_kernel``,
    batch > 4, RoPE + KV append fused), and the persistent kernel's split-KV attention and merge
    (``decode_tc_kernel``): through an attention-transparent model.  One layer with ``wo = I``, a zero MLP,
    ``final_norm = 1`` and an lm_head whose first ``hidden`` rows are ``I`` makes ``logits[:hidden]`` equal to
    ``rmsnorm(e + attn)`` (bf16-rounded on the paths whose GEMM inputs are bf16), so every decode path, the persistent
    kernel included, exposes its attention output.  The decode context is crafted in place: the test writes the
    cache rows and ``seq_lens`` itself, so contexts up to 4095 tokens need no long prefill.  Every path runs at every
    GQA ratio from 1 to 8 (``RATIO_MODELS``): the kernels' query tile, head-to-group mapping, prologue loops and the
    persistent kernel's split count all depend on the ratio and the KV-head count.

Errors are relative RMS per (sequence, head); the tests print them.  BARS lists the worst values measured on the
H100 and the bars, about 4x above them.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import (GEMV_MAX_BATCH, decode_branch, gather_kv, gemm_splits, make_lm, rel_rms, runs_persistent,
                           set_decode_impl)

PAGE = 64
LOG2E = 1.4426950408889634
KV_POISON_K, KV_POISON_V = 64.0, 8192.0   # prefill_slots: every stale row of the pool (exact in bf16)

# Worst relative RMS error per (sequence, head), measured on one H100 80GB HBM3 (132 SMs, 400 W power limit), and the
# bars, ~4x above:
#   prefill, "mma" mirror, attn_bf16 against the mirror rounded to bf16       8.7e-4  -> 3e-3
#   fp32 decode chain (attn_decode_kernel), exact attention                    4.8e-7  -> 2e-6
#   persistent kernel, batch <= 8 (bf16 hi + lo activations), "mma" mirror     1.3e-3  -> 5e-3
#   bf16 activations (mma chain kernel, persistent kernel batch > 8)           3.2e-3  -> 1.2e-2
#   appended K / V row against float64 RoPE'd k / v rounded to bf16           6.5e-4  -> 3e-3
#   prefill q buffer per (row, head) against float64 (rope_append_kernel)                     9.1e-4  -> 4e-3
#   prefill K / V rows per (row, head) against float64 rounded to bf16                        3.0e-3  -> 1.2e-2
# The tensor-core kernels round each probability against the running maximum of its page, the mirror against the
# global one; that and the odd flipped bf16 rounding of the query are what the mirror leaves.  The decode cases at GQA
# ratios 1..8 and the prefill rows were measured on one H100 80GB HBM3 (132 SMs, 700 W power limit): fp32 chain 6.6e-7,
# hi + lo 1.6e-3, bf16 activations 3.2e-3, appended rows 1.3e-3, all under the bars above.  The prefill rows' floor is
# the bf16 rounding of the normalised input: an element whose fp32 and float64 values round to neighbouring bf16 values
# moves its row's q by ~1e-4 .. 1e-3; rows without such a flip sit at 3e-7 (q).
BARS = {"prefill": 3e-3, "decode-fp32": 2e-6, "decode-mma": 5e-3, "decode-bf16": 1.2e-2, "row": 3e-3,
        "prefill-q": 4e-3, "row-head": 1.2e-2}


# ====================================================================================== float64 reference helpers
def ref_attention(q, k, v, n_rep: int, causal_offset: int | None = None, mirror: str | None = None):
    """Attention in float64.  q: [Tq, Hq, 64]; k, v: [Tk, Hkv, 64]; query head h reads KV head h // n_rep.
    ``causal_offset``: key position of q[0]; query i sees keys 0..causal_offset + i (None: every key).

    ``mirror=None`` is exact softmax attention.  ``mirror="mma"`` applies the rounding points of the tensor-core
    kernels (``oracle.lm_oracle.attention(mma_bf16=True)``): the query times d^-1/2 * log2(e) is rounded to bf16 (the
    product taken in fp32, as the kernels do), the probabilities 2^(s - max) are rounded to bf16 before P.V, and the
    normaliser sums the unrounded probabilities."""
    assert mirror in (None, "mma"), mirror
    q, k, v = q.double(), k.double(), v.double()
    Tq, Hq, d = q.shape
    Tk = k.shape[0]
    scale = d ** -0.5 * LOG2E
    mask = None
    if causal_offset is not None:
        mask = torch.arange(Tk)[None, :] > (torch.arange(Tq)[:, None] + causal_offset)
    out = torch.empty(Tq, Hq, d, dtype=torch.float64)
    for h in range(Hq):   # one head at a time: a 2047 x 2047 score matrix per head
        kh, vh = k[:, h // n_rep], v[:, h // n_rep]
        if mirror == "mma":
            qs = (q[:, h].float() * torch.tensor(scale, dtype=torch.float32)).bfloat16().double()
            s = qs @ kh.T
        else:
            s = (q[:, h] @ kh.T) * scale
        if mask is not None:
            s = s.masked_fill(mask, float("-inf"))
        p = torch.exp2(s - s.max(dim=-1, keepdim=True).values)
        pv = p.bfloat16().double() if mirror == "mma" else p
        out[:, h] = (pv @ vh) / p.sum(dim=-1, keepdim=True)
    return out


def rope64(x, pos, theta: float):
    """Half-split RoPE of x [heads, 64] (float64) at position ``pos``, or of x [T, heads, 64] at positions ``pos`` [T].
    The angle pos * inv_freq is formed in fp32, as the reference (modeling_qwen2.py rotary embedding) and the kernels
    form it; cos / sin are taken in float64."""
    inv = (1.0 / theta ** (torch.arange(32, dtype=torch.float64) * 2 / 64)).float()
    if torch.is_tensor(pos):
        ang = (pos.to(torch.float32)[:, None, None] * inv).double()
    else:
        ang = (torch.tensor(float(pos), dtype=torch.float32) * inv).double()
    c, s = ang.cos(), ang.sin()
    x1, x2 = x[..., :32], x[..., 32:]
    return torch.cat((x1 * c - x2 * s, x2 * c + x1 * s), dim=-1)


def rmsnorm64(x, eps: float):
    return x / torch.sqrt(x.pow(2).mean() + eps)


def per_head_err(got, ref) -> float:
    """Worst relative RMS error over heads; got / ref: [..., heads, 64].  inf when ``got`` is not finite."""
    if not torch.isfinite(got).all():
        return math.inf
    g, r = got.double(), ref.double()
    num = (g - r).pow(2).sum(-1).sum(tuple(range(g.dim() - 2)))
    den = r.pow(2).sum(-1).sum(tuple(range(g.dim() - 2))).clamp_min(1e-300)
    return float((num / den).sqrt().max())


# ---------------------------------------------------------------------------------------- CPU tests of the helpers
@pytest.mark.parametrize("causal", [None, 0, 5])
@pytest.mark.parametrize("n_rep", [1, 3])
def test_ref_attention_matches_oracle(causal, n_rep):
    g = torch.Generator().manual_seed(n_rep * 10 + (causal or 0))
    Tq, Tk, n_kv = (9 if causal is not None else 4), 14, 2
    q = torch.randn(Tq, n_kv * n_rep, 64, generator=g) * 2
    k = torch.randn(Tk, n_kv, 64, generator=g).bfloat16().float()
    v = torch.randn(Tk, n_kv, 64, generator=g).bfloat16().float()
    exact = ref_attention(q, k, v, n_rep, causal)
    mma = ref_attention(q, k, v, n_rep, causal, mirror="mma")
    o_exact = O.attention(q, k, v, causal, n_rep)
    o_mma = O.attention(q, k, v, causal, n_rep, mma_bf16=True)
    assert rel_rms(exact, o_exact) < 1e-6
    assert rel_rms(mma, o_mma) < 1e-5
    assert rel_rms(mma, exact) > 1e-4        # the mirror does round: it is not the exact attention again


def test_error_measures_report_non_finite_output():
    ref = torch.ones(3, 2, 64)
    bad = ref.clone()
    bad[1, 0, 5] = float("nan")
    assert rel_rms(bad, ref) == math.inf and per_head_err(bad, ref) == math.inf
    assert max(0.0, per_head_err(bad, ref)) == math.inf      # a NaN would have been dropped by max()
    assert per_head_err(ref, ref) == 0.0 and rel_rms(ref * 1.01, ref) == pytest.approx(0.01)


def test_ref_attention_masks_and_normalises():
    """A key behind the causal horizon carries no weight, whatever its size; a lone visible key returns its V."""
    k = torch.zeros(3, 1, 64)
    v = torch.stack([torch.full((1, 64), float(i + 1)) for i in range(3)])
    k[2] = 1e3
    q = torch.ones(2, 1, 64)
    o = ref_attention(q, k, v, 1, causal_offset=0)
    assert torch.equal(o[0, 0], torch.ones(64, dtype=torch.float64))            # query 0 sees key 0 only
    assert torch.allclose(o[1, 0], torch.full((64,), 1.5, dtype=torch.float64))  # equal scores: the mean
    o = ref_attention(q[:1], k, v, 1)                                            # no mask: the huge key wins
    assert torch.allclose(o[0, 0], torch.full((64,), 3.0, dtype=torch.float64))


def test_gather_kv_follows_a_shuffled_page_table():
    n_pages, n_kv = 7, 2
    kv = torch.zeros(2, 2, n_pages, n_kv, PAGE, 64, dtype=torch.bfloat16)
    pg, hd, row = torch.meshgrid(torch.arange(n_pages), torch.arange(n_kv), torch.arange(PAGE), indexing="ij")
    for which, sign in ((0, 1), (1, -1)):   # dims 0, 1, 2 of every row of layer 1: (page, head, row), exact in bf16
        kv[1, which, ..., 0], kv[1, which, ..., 1], kv[1, which, ..., 2] = sign * pg, sign * hd, sign * row
    table = torch.tensor([[5, 2, 6], [0, 3, 1]], dtype=torch.int32)
    lm = SimpleNamespace(kv=kv, page_table=table)
    n = 2 * PAGE + 17
    K, V = gather_kv(lm, 1, 0, n)
    assert K.shape == V.shape == (n, n_kv, 64) and K.dtype == torch.float64
    for t in range(n):
        want = torch.tensor([[float(table[0, t // PAGE]), h, t % PAGE] for h in range(n_kv)], dtype=torch.float64)
        assert torch.equal(K[t, :, :3], want) and torch.equal(V[t, :, :3], -want), t
    assert not K[:, :, 3:].any()
    K1, _ = gather_kv(lm, 1, 1, 5)
    assert torch.equal(K1[:, 0, 0], torch.zeros(5, dtype=torch.float64)) and torch.equal(K1[:, 0, 2], torch.arange(5.0, dtype=torch.float64))
    K0, _ = gather_kv(lm, 0, 0, 3)   # layer 0 is untouched
    assert not K0.any()


def test_project_rows_matches_project():
    cfg, w = transparent_model(12, 3, seed=4)
    toks, pos = [5, 900, 5, 2047], [0, 3, 700, 2046]
    q, k, v = project_rows(cfg, w, toks, pos)
    for i, (t, p) in enumerate(zip(toks, pos)):
        q1, k1, v1 = project(cfg, w, t, p, rb=True)
        assert rel_rms(q[i], q1) < 1e-14 and rel_rms(k[i], k1) < 1e-14 and rel_rms(v[i], v1) < 1e-14, i


def test_rope64_matches_oracle_rope():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 64, generator=g, dtype=torch.float64)
    for pos in (0, 1, 700, 4095):
        cos, sin = O.rope_cos_sin(torch.tensor([pos]), 64, 1e6)
        want = O.apply_rope(x.float()[None], cos, sin)[0]
        # the oracle computes inv_freq in fp32 arithmetic, the library (and rope64) rounds the float64 value to fp32:
        # at position 4095 the angles differ by a few 1e-6
        assert rel_rms(rope64(x, pos, 1e6), want) < 2e-5
    pos = torch.tensor([0, 1, 700, 4095])
    xs = torch.randn(4, 3, 64, generator=g, dtype=torch.float64)
    assert torch.equal(rope64(xs, pos, 1e6), torch.stack([rope64(xs[i], int(p), 1e6) for i, p in enumerate(pos)]))


# ====================================================================================== attention-transparent model
def transparent_model(n_heads: int, n_kv: int, seed: int, qk_std: float = 1.0, vocab: int = 2048, inter: int = 256):
    """One layer, hidden = n_heads * 64, wo = I, zero MLP, final_norm = 1, lm_head rows 0..hidden-1 = I (untied), small
    embeddings: logits[:hidden] = rmsnorm(e + attention).  q / k elements have standard deviation ~qk_std."""
    H = 64 * n_heads
    cfg = O.LMConfig(vocab_size=vocab, hidden_size=H, intermediate_size=inter, num_layers=1, num_heads=n_heads,
                     num_kv_heads=n_kv, head_dim=64, tie_embeddings=False)
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std):
        return (torch.randn(*shape, generator=g) * std).bfloat16().float()

    s = H ** -0.5
    layer = dict(ln1=torch.ones(H), wq=rn(H, H, std=qk_std * s), bq=rn(H, std=0.1),
                 wk=rn(64 * n_kv, H, std=qk_std * s), bk=rn(64 * n_kv, std=0.1),
                 wv=rn(64 * n_kv, H, std=s), bv=rn(64 * n_kv, std=0.1),
                 wo=torch.eye(H), ln2=torch.ones(H),
                 wg=torch.zeros(inter, H), wu=torch.zeros(inter, H), wd=torch.zeros(H, inter))
    head = torch.zeros(vocab, H)
    head[:H] = torch.eye(H)
    w = O.LMWeights(embed=rn(vocab, H, std=0.01), layers=[layer], final_norm=torch.ones(H), lm_head=head)
    return cfg, w


def project(cfg, w, tok: int, pos: int, rb: bool):
    """float64 q [n_heads, 64], k, v [n_kv, 64] of token ``tok`` at position ``pos`` (q, k RoPE'd); ``rb``: the
    normalised input is rounded to bf16 first, as on the paths whose GEMM inputs are bf16."""
    L0 = w.layers[0]
    x = rmsnorm64(w.embed[tok].double(), cfg.rms_eps) * L0["ln1"].double()
    if rb:
        x = x.bfloat16().double()
    lin = lambda n: x @ L0["w" + n].double().T + L0["b" + n].double()
    q = rope64(lin("q").view(cfg.num_heads, 64), pos, cfg.rope_theta)
    k = rope64(lin("k").view(cfg.num_kv_heads, 64), pos, cfg.rope_theta)
    return q, k, lin("v").view(cfg.num_kv_heads, 64)


def project_rows(cfg, w, toks, pos):
    """``project(..., rb=True)`` of token rows ``toks`` [T] at positions ``pos`` [T] at once: float64 q [T, n_heads,
    64], k, v [T, n_kv, 64] from the bf16-rounded normalised input, as the prefill's wgmma GEMM reads it."""
    L0 = w.layers[0]
    e = w.embed[torch.as_tensor(toks, dtype=torch.long)].double()
    x = (e / torch.sqrt(e.pow(2).mean(-1, keepdim=True) + cfg.rms_eps) * L0["ln1"].double()).bfloat16().double()
    lin = lambda n, heads: (x @ L0["w" + n].double().T + L0["b" + n].double()).view(len(toks), heads, 64)
    pos = torch.as_tensor(pos)
    return (rope64(lin("q", cfg.num_heads), pos, cfg.rope_theta), rope64(lin("k", cfg.num_kv_heads), pos, cfg.rope_theta),
            lin("v", cfg.num_kv_heads))


def transparent_logits(cfg, w, tok: int, attn, rb: bool):
    """What the transparent model's logits[:hidden] are for attention output ``attn`` [n_heads, 64] (float64)."""
    r = (lambda t: t.bfloat16().double()) if rb else (lambda t: t)
    h = w.embed[tok].double() + r(attn.reshape(-1))
    return r(rmsnorm64(h, cfg.rms_eps) * w.final_norm.double())


def craft_slot(lm, b: int, L: int, q, n_rep: int, g):
    """Layer-0 cache rows of slot ``b``: a random haystack in rows 0..L-1 with needle keys at rows 0, 63, 64, the last
    row of a far page and L-1 that raise the score of every query head of their group (scores ~8..10 against a
    haystack of standard deviation 1), and poison in every row from L on (score ~20, V = 1e4)."""
    rows = lm.max_pages * PAGE
    assert len(lm._slot_pages[b]) == lm.max_pages      # every page of the slot is allocated
    n_kv = q.shape[0] // n_rep
    K = torch.randn(rows, n_kv, 64, generator=g, dtype=torch.float64)
    V = torch.randn(rows, n_kv, 64, generator=g, dtype=torch.float64)
    qg = q.view(n_kv, n_rep, 64)
    # q_h . dirn / 8 = 1 + sum over the other heads h' of q_h . q_h' / |q_h'|^2 ~ 1 for each head h of the group
    dirn = 8 * (qg / qg.pow(2).sum(-1, keepdim=True)).sum(1)
    far = ((L - 1) // PAGE // 2) * PAGE + PAGE - 1
    needles = sorted({p for p in (0, 63, 64, far, L - 1) if p < L})
    for j, p in enumerate(needles):
        K[p] = (8.0 + 0.5 * j) * dirn
        V[p] = 2 * torch.randn(n_kv, 64, generator=g, dtype=torch.float64)
    K[L:] = 20 * dirn
    V[L:] = 1e4
    pages = lm.page_table[b].to(device=lm.kv.device, dtype=torch.long)
    as_pages = lambda t: t.view(lm.max_pages, PAGE, n_kv, 64).permute(0, 2, 1, 3).to(lm.kv.device, torch.bfloat16)
    lm.kv[0, 0, pages] = as_pages(K)
    lm.kv[0, 1, pages] = as_pages(V)
    return needles


def tc_geometry(lm, B: int, L: int, sms: int):
    """Split-KV geometry of the persistent kernel for a slot at length L: (split cap, pages per split, splits,
    attention warps per split)."""
    sms = min(sms, 256)
    cap = min(8, sms // (B * lm.shape.num_kv_heads), lm.max_ctx // PAGE)
    n_ctx = min(L + 1, lm.max_ctx)
    npages = -(-n_ctx // PAGE)
    pps = -(-npages // cap)
    aw = 2 if (B == 1 and lm.shape.hidden_size <= 1024) else 4   # batch 1 folds in the CTA: 2 page-walking warps
    return cap, pps, -(-npages // pps), aw


def run_crafted_decode(cfg, w, lens, steps, impl, max_ctx, monkeypatch, seed):
    """Prefill 1-token prompts, craft every slot's context (length lens[b]), decode ``steps`` teacher-forced steps.
    Returns (lm, forced tokens, logits [steps, B, V] on the CPU, kernel launches of the decode call, rb)."""
    B = len(lens)
    lm = make_lm(cfg, w, max_batch=B, max_ctx=max_ctx, page_shuffle_seed=seed)
    g = torch.Generator().manual_seed(seed)
    eos = cfg.vocab_size - 1
    forced = torch.randint(0, eos, (B, steps + 1), generator=g)
    sp = lm.sampling(eos, min_new_tokens=0, forced=forced)
    lm.prefill([[int(t)] for t in torch.randint(0, eos, (B,), generator=g)], sp)
    torch.cuda.synchronize()
    persistent = runs_persistent(impl, B)
    rb = B > 8 if persistent else B > GEMV_MAX_BATCH
    n_rep = cfg.num_heads // cfg.num_kv_heads
    for b, L in enumerate(lens):
        craft_slot(lm, b, L, project(cfg, w, int(forced[b, 0]), L, rb)[0], n_rep, g)
    lm.seq_lens[:B] = torch.tensor(lens, dtype=torch.int32, device=lm.device)
    set_decode_impl(monkeypatch, impl)
    n0 = lm.L.nt_launch_count()
    logits = lm.decode(steps, sp, return_logits=True)
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    return lm, forced, logits.cpu(), launches, rb


def check_decode(cfg, w, lm, forced, logits, lens, steps, mirror, rb):
    """Per step and slot: logits[:hidden] against the transparent model in float64 on the cache rows the kernel saw,
    and the row the step appended against the float64 RoPE'd k / v rounded to bf16.  Returns the worst errors."""
    n_rep = cfg.num_heads // cfg.num_kv_heads
    H = cfg.hidden_size
    worst_attn = worst_row = 0.0
    for b, L in enumerate(lens):
        Kc, Vc = gather_kv(lm, 0, b, L + steps)
        for s in range(steps):
            pos, tok = L + s, int(forced[b, s])
            q, k, v = project(cfg, w, tok, pos, rb)
            o = ref_attention(q[None], Kc[: pos + 1], Vc[: pos + 1], n_rep, mirror=mirror)[0]
            ref = transparent_logits(cfg, w, tok, o, rb)
            got = logits[s, b, :H].double()
            worst_attn = max(worst_attn, per_head_err(got.view(cfg.num_heads, 64), ref.view(cfg.num_heads, 64)))
            row = max(rel_rms(Kc[pos], k.bfloat16()), rel_rms(Vc[pos], v.bfloat16()))
            worst_row = max(worst_row, row)
    return worst_attn, worst_row


# ====================================================================================== prefill
PREFILL_LENS = [1, 15, 16, 17, 63, 64, 65, 129, 700, 2047]   # 16-query / 64-key tile edges and the context limit


def _prefill_errors(lm, cfg, slots, lens):
    """Worst per-(sequence, head) error of attn_bf16 against the "mma" mirror, sequences in call order."""
    T, HD = sum(lens), cfg.num_heads * 64
    n_rep = cfg.num_heads // cfg.num_kv_heads
    q = lm.debug_buffer("q", (T, HD)).double().cpu().view(T, cfg.num_heads, 64)
    got = lm.debug_buffer("attn_bf16", (T, HD), torch.bfloat16).double().cpu().view(T, cfg.num_heads, 64)
    errs, t0 = [], 0
    for s, n in zip(slots, lens):
        K, V = gather_kv(lm, 0, s, n)
        ref = ref_attention(q[t0: t0 + n], K, V, n_rep, causal_offset=0, mirror="mma").bfloat16().double()
        errs.append(per_head_err(got[t0: t0 + n], ref))
        t0 += n
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize("n_heads,n_kv", [(4, 4), (4, 2), (9, 3), (8, 2), (10, 2), (12, 2), (14, 2), (8, 1)],
                         ids=["gqa1", "gqa2", "gqa3", "gqa4", "gqa5", "gqa6", "gqa7", "gqa8"])
def test_prefill_attention_vs_float64(cuda, n_heads, n_kv):
    """attn_prefill_kernel on its own operands: one ragged prefill, lengths on the 16-query / 64-key tile edges up to
    the context limit, shuffled pages, q / k scaled so the softmax is peaked.  Worst per-(sequence, head) error
    against the "mma" mirror, measured: see BARS."""
    cfg, w = transparent_model(n_heads, n_kv, seed=100 + n_heads, qk_std=2.5)
    lm = make_lm(cfg, w, max_batch=len(PREFILL_LENS), max_ctx=2048, page_shuffle_seed=7)
    g = torch.Generator().manual_seed(n_kv)
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in PREFILL_LENS]
    lm.prefill(prompts, lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=2))
    torch.cuda.synchronize()
    errs = _prefill_errors(lm, cfg, range(len(PREFILL_LENS)), PREFILL_LENS)
    print(f"PREFILL-ATTN gqa{n_heads // n_kv} ({n_heads}/{n_kv}): " + " ".join(f"{n}:{e:.2e}" for n, e in zip(PREFILL_LENS, errs)))
    assert max(errs) < BARS["prefill"], errs


# (query heads, KV heads) of the GQA-ratio cases: every ratio from 1 to 8, ratio 4 over 2 and over 3 KV heads, hidden =
# 64 * query heads <= 896 (the widest the persistent kernel plans for).  gqa7 is NeuTTS-Air's attention, gqa4 the Nano
# shape's.
RATIO_MODELS = {"gqa1": (8, 8), "gqa2": (4, 2), "gqa3": (9, 3), "gqa4": (8, 2), "gqa4kv3": (12, 3), "gqa5": (10, 2),
                "gqa6": (12, 2), "gqa7": (14, 2), "gqa8": (8, 1)}


def row_head_err(got, ref) -> float:
    """Worst relative RMS error over (row, head); got / ref: [rows, heads, 64].  inf when ``got`` is not finite."""
    if not torch.isfinite(got).all():
        return math.inf
    g, r = got.double(), ref.double()
    return float(((g - r).pow(2).sum(-1) / r.pow(2).sum(-1).clamp_min(1e-300)).sqrt().max())


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(RATIO_MODELS))
def test_prefill_rope_rows_vs_float64(cuda, model):
    """rope_append_kernel: the prefill's rotated q buffer and every cached K and V row, per (row, head), against
    rope64(bf16(rmsnorm(e) * ln1) @ W + b, pos) in float64 (K and V rounded to bf16 as cached).  Two ragged prefills:
    the first PREFILL_LENS, few rows, where the qkv GEMM splits K into slices that the kernel sums (at hidden >= 512),
    then all of PREFILL_LENS, where it does not."""
    n_heads, n_kv = RATIO_MODELS[model]
    cfg, w = transparent_model(n_heads, n_kv, seed=200 + n_heads + n_kv, qk_std=2.5)
    H, QN = cfg.hidden_size, (n_heads + 2 * n_kv) * 64
    lm = make_lm(cfg, w, max_batch=len(PREFILL_LENS), max_ctx=2048, page_shuffle_seed=n_kv)
    g = torch.Generator().manual_seed(n_heads)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=2)
    for lens in (PREFILL_LENS[:4], PREFILL_LENS):
        T = sum(lens)
        splits = gemm_splits(T, QN, H, 8 * 128 * max(QN, H))          # lm->splitk_floats
        assert (splits > 1) == (T < 100 and H >= 512), splits
        prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
        lm.prefill(prompts, sp)
        torch.cuda.synchronize()
        q = lm.debug_buffer("q", (T, n_heads * 64)).double().cpu().view(T, n_heads, 64)
        K, V = (torch.cat(t) for t in zip(*(gather_kv(lm, 0, b, n) for b, n in enumerate(lens))))
        rq, rk, rv = project_rows(cfg, w, [t for p in prompts for t in p], torch.cat([torch.arange(n) for n in lens]))
        errs = (row_head_err(q, rq), row_head_err(K, rk.bfloat16()), row_head_err(V, rv.bfloat16()))
        print(f"PREFILL-ROPE {model} ({n_heads}/{n_kv}) T={T} split-K {splits}: q {errs[0]:.2e} K {errs[1]:.2e} "
              f"V {errs[2]:.2e}")
        assert errs[0] < BARS["prefill-q"] and max(errs[1:]) < BARS["row-head"], (T, errs)


@pytest.mark.gpu
def test_prefill_slots_attention_ignores_stale_rows(cuda):
    """Refilled slots: after a prefill of long sequences, every layer-0 K/V row of the pool is overwritten with large
    finite poison (K = 64, V = 8192); newcomers prefilled into some slots must attend to their own rows only, so an
    off-by-one in a mask or in the compact slot table shows up at once."""
    cfg, w = transparent_model(14, 2, seed=7, qk_std=2.5)
    lm = make_lm(cfg, w, max_batch=6, max_ctx=2048, page_shuffle_seed=13)
    g = torch.Generator().manual_seed(17)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=2)
    lm.prefill([torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in (2000, 1500, 1800, 900, 1200, 700)], sp)
    torch.cuda.synchronize()
    lm.kv[0, 0] = KV_POISON_K
    lm.kv[0, 1] = KV_POISON_V
    slots, lens = [4, 1, 3], [17, 700, 65]
    lm.prefill_slots(slots, [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in lens], sp, [10, 11, 12])
    torch.cuda.synchronize()
    for s, n in zip(slots, lens):   # the newcomers' pages hold poison right behind their rows
        K, V = gather_kv(lm, 0, s, -(-n // PAGE) * PAGE)
        assert torch.all(K[n:] == KV_POISON_K) and torch.all(V[n:] == KV_POISON_V)
    errs = _prefill_errors(lm, cfg, slots, lens)
    print("PREFILL-SLOTS-ATTN " + " ".join(f"slot{s}/{n}:{e:.2e}" for s, n, e in zip(slots, lens, errs)))
    assert max(errs) < BARS["prefill"], errs


# ====================================================================================== decode
# (id, impl, lens, max_ctx, mirror, branch).  14 query heads over 2 KV heads: NeuTTS-Air's attention shape.
def _lens(B, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    out = [hi] + torch.randint(lo, hi, (B - 1,), generator=g).tolist()
    return out


_RATIO_PATHS = [   # (id, impl, lens, mirror, branch): the paths every RATIO_MODELS shape runs
    ("chain-fp32-b1", "perop", [2047], None, "fp32"),
    ("chain-fp32-b4", "perop", [511, 512, 513, 1000], None, "fp32"),
    ("chain-mma-b6", "perop", [2047, 1000, 513, 512, 511, 64], "mma", "mma"),
    ("persistent-b1", None, [2047], "mma", "tc-b1"),
    ("persistent-b8", None, _lens(8, 900, 2047, 2), "mma", "tc-hilo"),
    ("persistent-b16", None, _lens(16, 1200, 2047, 3), "mma", "tc-bf16"),
]
# (id, model, impl, lens, max_ctx, mirror, branch); model: a RATIO_MODELS key.  8/8 at batch 16 has 128 (sequence, KV
# head) pairs: on a 132-SM H100 each gets one attention split ("tc-bf16-cap1").  8/1 at batch 16 has 8 splits of at most
# 4 pages, one page per attention warp ("tc-bf16-1page").
DECODE_CASES = [
    ("chain-fp32-b1", "gqa7", "perop", [2047], 2048, None, "fp32"),
    ("chain-fp32-b4", "gqa7", "perop", [511, 512, 513, 1000], 2048, None, "fp32"),
    ("chain-mma-b6", "gqa7", "perop", [2047, 1000, 513, 512, 511, 64], 2048, "mma", "mma"),
    ("chain-mma-b34", "gqa7", "perop", [511, 512, 513] + _lens(31, 64, 2047, 1), 2048, "mma", "mma"),
    ("persistent-b1", "gqa7", None, [2047], 2048, "mma", "tc-b1"),
    ("persistent-b4", "gqa7", None, [2047, 1000, 513, 1500], 2048, "mma", "tc-hilo"),
    ("persistent-b8", "gqa7", None, _lens(8, 900, 2047, 2), 2048, "mma", "tc-hilo"),
    ("persistent-b16", "gqa7", None, _lens(16, 1200, 2047, 3), 2048, "mma", "tc-bf16"),
    ("persistent-b34-ctx4096", "gqa7", "tc", _lens(34, 2049, 4095, 4), 4096, "mma", "tc-pagefallback"),
] + [(f"{model}-{name}", model, impl, lens, 2048, mirror,
      {("gqa1", "tc-bf16"): "tc-bf16-cap1", ("gqa8", "tc-bf16"): "tc-bf16-1page"}.get((model, branch), branch))
     for model in RATIO_MODELS if model != "gqa7" for name, impl, lens, mirror, branch in _RATIO_PATHS]


def _assert_branch(lm, branch, lens, launches, steps, impl):
    """The path the case meant to test: decode_branch's prediction, the launch count and the split-KV geometry."""
    B = len(lens)
    s = lm.shape
    sms = min(torch.cuda.get_device_properties(0).multi_processor_count, 256)
    br = decode_branch((s.hidden_size, s.intermediate_size, s.num_heads, s.num_kv_heads, s.vocab_size), B, sms,
                       lm.max_ctx, impl)
    npages = [-(-(L + 1) // PAGE) for L in lens]
    if branch in ("fp32", "mma"):
        assert br["name"] == ("gemv" if branch == "fp32" else "gemm"), br
        assert launches > steps, launches                     # the per-op chain: several kernels per step
        # more than 8 pages: each of the 8 warp pairs (fp32) / warps (mma) walks several pages
        assert max(npages) > 8
        return br
    bf16 = branch.startswith("tc-bf16") or branch == "tc-pagefallback"
    assert br["kind"] == "tc" and br["act"] == ("bf16" if bf16 else "hilo"), br
    assert br["fold"] == (branch == "tc-b1"), br
    assert launches == 1, launches                            # one launch: the persistent kernel
    geo = [tc_geometry(lm, B, L, sms) for L in lens]
    cap = geo[0][0]
    assert cap == br["split_cap"], (cap, br)
    if branch not in ("tc-pagefallback", "tc-bf16-cap1"):
        assert cap > 1 and max(g[2] for g in geo) == cap      # the merge sees split_cap partials
    if branch == "tc-b1":
        assert cap == min(8, sms // lm.shape.num_kv_heads) and geo[0][3] == 2 and geo[0][1] > geo[0][3]
    elif branch == "tc-hilo":
        assert 1 < B <= 8 and max(g[1] for g in geo) > 1
    elif branch == "tc-bf16":
        assert B > 8 and cap == min(8, sms // (B * lm.shape.num_kv_heads)) and max(g[1] for g in geo) > geo[0][3]
    elif branch == "tc-bf16-1page":  # split_cap partials of at most one page per attention warp
        assert B > 8 and cap == min(8, sms // (B * lm.shape.num_kv_heads)) and max(g[1] for g in geo) == geo[0][3]
    elif branch == "tc-bf16-cap1":   # one split per (sequence, KV head): its warps walk every page, no merge
        assert B > 8 and cap == 1 and all(g[2] == 1 for g in geo) and max(g[1] for g in geo) > geo[0][3]
    elif branch == "tc-pagefallback":
        assert cap == 1 and max(g[1] for g in geo) > 32       # pages past the 32-entry cache: page_of's global load
    return br


@pytest.mark.gpu
@pytest.mark.parametrize("case", DECODE_CASES, ids=[c[0] for c in DECODE_CASES])
def test_decode_attention_vs_float64(cuda, case, monkeypatch):
    """Decode attention on a crafted cache, on every decode path, through the attention-transparent model.  Needles on
    the first, far and last pages make every page and every split-KV partial count; poison behind the context makes a
    leaked row blow the error up by orders of magnitude.  Also checks the K/V row the step appended.  Worst errors
    measured: see BARS."""
    name, model, impl, lens, max_ctx, mirror, branch = case
    n_heads, n_kv = RATIO_MODELS[model]
    cfg, w = transparent_model(n_heads, n_kv, seed=5 if model == "gqa7" else 5 + 16 * n_heads + n_kv)
    lm, forced, logits, launches, rb = run_crafted_decode(cfg, w, lens, 1, impl, max_ctx, monkeypatch, seed=len(lens))
    br = _assert_branch(lm, branch, lens, launches, 1, impl)
    attn_err, row_err = check_decode(cfg, w, lm, forced, logits, lens, 1, mirror, rb)
    print(f"DECODE-ATTN {name}: ratio {n_heads // n_kv} ({n_heads}/{n_kv}) [{br['name']}, split_cap {br['split_cap']}, "
          f"launches {launches}]: attention {attn_err:.2e} appended row {row_err:.2e}")
    assert attn_err < BARS["decode-" + ("fp32" if mirror is None else ("bf16" if rb else "mma"))], attn_err
    assert row_err < BARS["row"], row_err


@pytest.mark.gpu
def test_decode_attention_multistep_crosses_a_page(cuda, monkeypatch):
    """L = 62 and 4 teacher-forced steps in ONE persistent-kernel launch: the context crosses the page boundary at
    64 inside the launch, and step s must read the rows that steps 0..s-1 appended."""
    cfg, w = transparent_model(14, 2, seed=9)
    lens, steps = [62, 62], 4
    lm, forced, logits, launches, rb = run_crafted_decode(cfg, w, lens, steps, None, 2048, monkeypatch, seed=21)
    assert launches == 1, launches
    attn_err, row_err = check_decode(cfg, w, lm, forced, logits, lens, steps, "mma", rb)
    print(f"DECODE-ATTN multistep: attention {attn_err:.2e} appended rows {row_err:.2e}")
    assert attn_err < BARS["decode-mma"], attn_err
    assert row_err < BARS["row"], row_err
