"""Shared test plumbing: oracle weights -> HF-style state dicts -> CUDA engines, error measures, and the rule that picks
the decode path."""
from __future__ import annotations

import functools
import math
import warnings

import torch

from oracle import codec_oracle, lm_oracle


def lm_state_dict(w: lm_oracle.LMWeights, tied: bool = True) -> dict:
    sd = {"model.embed_tokens.weight": w.embed, "model.norm.weight": w.final_norm}
    for i, L in enumerate(w.layers):
        p = f"model.layers.{i}."
        sd.update({
            p + "input_layernorm.weight": L["ln1"], p + "post_attention_layernorm.weight": L["ln2"],
            p + "self_attn.q_proj.weight": L["wq"], p + "self_attn.q_proj.bias": L["bq"],
            p + "self_attn.k_proj.weight": L["wk"], p + "self_attn.k_proj.bias": L["bk"],
            p + "self_attn.v_proj.weight": L["wv"], p + "self_attn.v_proj.bias": L["bv"],
            p + "self_attn.o_proj.weight": L["wo"], p + "mlp.gate_proj.weight": L["wg"],
            p + "mlp.up_proj.weight": L["wu"], p + "mlp.down_proj.weight": L["wd"]})
    if not tied:
        sd["lm_head.weight"] = w.lm_head
    return sd


def lm_shape(cfg: lm_oracle.LMConfig):
    from neutts_air_b200.lm import LMShape

    return LMShape(cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_layers, cfg.num_heads,
                   cfg.num_kv_heads, cfg.head_dim, cfg.rms_eps, cfg.rope_theta, cfg.tie_embeddings)


def make_lm(cfg, w, **kw):
    from neutts_air_b200.lm import SpeechLM

    return SpeechLM(lm_shape(cfg), lm_state_dict(w, cfg.tie_embeddings), device="cuda:0", **kw)


def codec_shape(cfg: codec_oracle.CodecConfig):
    from neutts_air_b200.codec import CodecShape

    return CodecShape(cfg.fsq_levels, cfg.fsq_dims, cfg.quant_dim, cfg.hidden, cfg.depth, cfg.heads, cfg.head_dim,
                      cfg.mlp_mult, cfg.groups, cfg.embed_kernel, cfg.n_fft, cfg.hop, cfg.rope_base, cfg.rope_axis,
                      cfg.norm_eps, cfg.mag_clip)


def codec_weight_dict(w: codec_oracle.CodecWeights) -> dict:
    return dict(project_out_w=w.project_out_w, project_out_b=w.project_out_b, fc_post_a_w=w.fc_post_a_w,
                fc_post_a_b=w.fc_post_a_b, embed_w=w.embed_w, embed_b=w.embed_b, prior=w.prior, post=w.post,
                blocks=w.blocks, final_ln_w=w.final_ln_w, final_ln_b=w.final_ln_b, head_w=w.head_w, head_b=w.head_b)


def make_codec(cfg, w, **kw):
    from neutts_air_b200.codec import CodecDecoder

    return CodecDecoder(codec_shape(cfg), codec_weight_dict(w), device="cuda:0", **kw)


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def rel_rms(got, ref) -> float:
    """Relative RMS error of torch tensors, numpy arrays or lists; inf when ``got`` holds a NaN or an inf (so that max()
    over errors cannot drop it)."""
    got, ref = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(ref, dtype=torch.float64)
    if not torch.isfinite(got).all():
        return math.inf
    return float((got - ref).norm() / ref.norm().clamp_min(1e-300))


def tf32_truncate(x):
    """fp32 -> TF32 (10-bit mantissa) by truncation, as the tensor core reads an fp32 operand in a plain TF32 MMA (this
    model gives the 7.4e-4 .. 8.0e-4 per row that plain TF32 GEMMs measure on the H100; round to nearest gives 3e-4)."""
    i = x.float().contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32)


def gather_kv(lm, layer: int, b: int, n: int):
    """Rows 0..n-1 of slot ``b``'s K and V in layer ``layer``, read through ``lm.page_table`` from the paged pool
    ``lm.kv[layer, 0|1, page, kv_head, row, :]`` (pages of 64 rows).  Returns two float64 CPU tensors [n, n_kv, 64]."""
    page = lm.kv.shape[-2]
    npg = (n + page - 1) // page
    pages = lm.page_table[b, :npg].to(device=lm.kv.device, dtype=torch.long)
    out = []
    for which in (0, 1):
        t = lm.kv[layer, which].index_select(0, pages)                     # [npg, n_kv, 64, 64]
        out.append(t.permute(0, 2, 1, 3).reshape(npg * page, t.shape[1], 64)[:n].double().cpu())
    return out[0], out[1]


# The decode path nt_lm_decode (lm_api.cu) takes: with NT_DECODE_IMPL unset, the persistent kernel up to
# kTcDefaultMaxBatch sequences (lm_decode_tc.cuh) and the per-op chain above; "tc" or "perop" forces one.  The chain
# runs its projections, and every lm_head its GEMV, up to kGemvMaxBatch rows (lm_kernels.cuh), wgmma GEMMs above.
# test_decode_plan.py checks both constants against the headers.
TC_DEFAULT_MAX_BATCH = 16
GEMV_MAX_BATCH = 4


def set_decode_impl(monkeypatch, impl):
    """Force the decode path with NT_DECODE_IMPL = ``impl``, or leave the choice to the engine when ``impl`` is None."""
    if impl:
        monkeypatch.setenv("NT_DECODE_IMPL", impl)
    else:
        monkeypatch.delenv("NT_DECODE_IMPL", raising=False)


def runs_persistent(impl, B: int) -> bool:
    """Whether a decode at batch B runs the persistent kernel after ``set_decode_impl(monkeypatch, impl)``."""
    return impl == "tc" or (impl is None and B <= TC_DEFAULT_MAX_BATCH)


# ------------------------------------------------------------------------------- the persistent kernel's work plans
@functools.lru_cache(maxsize=None)
def plan_summary(shape: tuple, G: int, flat: bool):
    """The persistent decode kernel's plan for ``shape`` = (hidden, inter, n_heads, n_kv, vocab) on G CTAs, as (sq, so,
    sd, sg, max_chunks, everybody), or None where the planner rejects it.  ``everybody``: the whole-K plan's gate/up
    layout when fewer than 16 CTAs would be left for the split phases, so that every CTA takes gate/up tiles and split
    items alike (restated from tc_build_plan, lm_decode_tc.cu); False for the flat plan."""
    from neutts_air_b200.lm import debug_decode_plan

    try:
        p = debug_decode_plan(*shape, G, flat)
    except ValueError:
        return None
    Tg = -(-2 * shape[1] // 128)
    return p["sq"], p["so"], p["sd"], p["sg"], p["max_chunks"], not flat and G - min(Tg, G) < 16


def plan_regime(shape: tuple, G: int):
    """(whole-K plan, flat plan) summaries at G CTAs: what a decode of ``shape`` can run there."""
    return plan_summary(shape, G, False), plan_summary(shape, G, True)


@functools.lru_cache(maxsize=None)
def regime_representatives(shape: tuple, max_G: int) -> dict:
    """{regime: the smallest G in 8..max_G that has it}.  A regime recurring at separate counts counts once."""
    reps = {}
    for G in range(8, max_G + 1):
        reps.setdefault(plan_regime(shape, G), G)
    return reps


def decode_branch(shape: tuple, B: int, G: int, max_ctx: int, impl=None) -> dict:
    """The path nt_lm_decode (lm_api.cu) takes after ``set_decode_impl(monkeypatch, impl)``, for B <= max_batch
    sequences of ``shape`` on G CTAs, restated from nt_lm_decode and launch_decode_tc: the persistent kernel when
    ``runs_persistent(impl, B)``, its whole-K plan is accepted at G and B * n_kv <= G, else the per-op chain.  On the
    persistent kernel: the flat plan when it is accepted and the slices are folded in the consumer CTAs (batch 1), bf16
    hi + lo activation pairs up to batch 8, the tile width N and the attention splits per (sequence, kv head)."""
    H, n_kv = shape[0], shape[3]
    whole, flat = plan_regime(shape, G)
    if not runs_persistent(impl, B) or whole is None or B * n_kv > G:
        return dict(kind="chain", name="gemv" if B <= GEMV_MAX_BATCH else "gemm", split_cap=None)
    fold = B == 1 and H * 4 <= 16 * 1024 and H <= 1024          # tc_fold_in_cta
    plan = "flat" if flat is not None and fold else "wholeK"
    nt = 16 if B <= 16 else (32 if B <= 32 else 64)
    act = "hilo" if B <= 8 else "bf16"
    return dict(kind="tc", plan=plan, fold=fold, act=act, nt=nt, split_cap=min(8, G // (B * n_kv), max_ctx // 64),
                name=f"tc-{act}-n{nt}-{plan}-{'fold' if fold else 'phases'}")


def head_list(V: int, eos: int, rng=None) -> tuple:
    """The persistent kernel's lm_head tile list for vocabulary V under the vocabulary range ``rng`` = (lo, hi) (None:
    off), restated from vocab_tiles and nt_lm_decode (lm_api.cu): (head_n, head_lo, head_eos, head_eos_at).  The range's
    tiles head_lo, head_lo + 1, ... in order, with EOS's tile head_eos inserted at position head_eos_at (0 when it lies
    below the range, last when above) when EOS lies outside the range's tiles; head_eos = head_eos_at = -1 otherwise."""
    t_lo = rng[0] // 128 if rng else 0
    t_hi = -(-(rng[1] if rng else V) // 128)
    et = eos // 128
    head_eos = et if rng and (et < t_lo or et >= t_hi) else -1
    head_eos_at = -1 if head_eos < 0 else (0 if head_eos < t_lo else t_hi - t_lo)
    return t_hi - t_lo + (head_eos >= 0), t_lo, head_eos, head_eos_at


def head_partition(head_n: int, head_eos_at: int, G: int, head_lo: int = 0, head_eos: int = -1) -> list:
    """The lm_head work of the persistent kernel on G CTAs, restated from decode_tc_kernel (lm_decode_tc.cu): CTA c
    takes list positions [head_n c / G, head_n (c + 1) / G).  Returns, per CTA, (t0, t1, row tiles of t0..t1-1)."""
    def tile(v):
        return head_eos if v == head_eos_at else head_lo + v - (1 if 0 <= head_eos_at < v else 0)

    out = []
    for c in range(G):
        t0, t1 = head_n * c // G, head_n * (c + 1) // G
        out.append((t0, t1, [tile(v) for v in range(t0, t1)]))
    return out


def head_grid_features(head: tuple, G: int) -> set:
    """What the lm_head partition of ``head`` = head_list(...) looks like on G CTAs: "empty" (some CTA holds no tile),
    "one-each" (G = head_n), "even" / "odd" (some CTA holds an even / odd count above 1), "eos-alone" / "eos-shared"
    (the inserted EOS tile is the only tile of its CTA / shares it with range tiles)."""
    head_n, head_lo, head_eos, head_eos_at = head
    f = set()
    for t0, t1, tiles in head_partition(head_n, head_eos_at, G, head_lo, head_eos):
        n = t1 - t0
        if n == 0:
            f.add("empty")
        elif n > 1:
            f.add("even" if n % 2 == 0 else "odd")
        if head_eos >= 0 and head_eos in tiles:
            f.add("eos-alone" if n == 1 else "eos-shared")
    if G == head_n:
        f.add("one-each")
    return f


def head_grid_counts(shape: tuple, head: tuple, B: int, max_ctx: int, dev: int, impl=None) -> list:
    """CTA counts to run a decode of B sequences of ``shape`` on, with the lm_head tile list ``head``: among the counts
    in [max(8, B n_kv), dev] where ``decode_branch`` takes the persistent kernel, the smallest, the device's count
    ``dev``, every plan regime's representative (``regime_representatives``), at batch 1 a flat-plan and a whole-K-plan
    count, the H100 PCIe's 114 and head_n +- 1 (a CTA count next to the list length), and the smallest count showing
    each ``head_grid_features`` feature some accepted count shows.  Sorted."""
    ok = [G for G in range(max(8, B * shape[3]), dev + 1) if decode_branch(shape, B, G, max_ctx, impl)["kind"] == "tc"]
    assert dev in ok, (shape, B, dev)
    want = {ok[0], dev} | {G for G in regime_representatives(shape, dev).values() if G in ok}
    want |= {G for G in (114, head[0] - 1, head[0] + 1) if G in ok}
    if B == 1:
        for plan in ("flat", "wholeK"):
            want |= {next((G for G in ok if decode_branch(shape, B, G, max_ctx, impl)["plan"] == plan), dev)}
    have = set().union(*(head_grid_features(head, G) for G in want))
    for G in ok:
        new = head_grid_features(head, G) - have
        if new:
            want.add(G)
            have |= new
    return sorted(want)


def gemm_splits(M: int, N: int, K: int, ws_floats: int) -> int:
    """Split-K slices gemm_dispatch (gemm_tc.cu) picks for an M x N x K bf16 GEMM with a split workspace of
    ``ws_floats`` floats, on the device's SM count (restated)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mt = -(-M // 128)
    bn = 128
    if mt * -(-N // 128) < sms * 13 // 16:
        bn = 64
    if mt * -(-N // 64) < sms * 11 // 16:
        bn = 32
    tiles, nkb = mt * -(-N // bn), -(-K // 64)
    if tiles > 48 or nkb < 8:
        return 1
    sk = min((sms - 4) // tiles, nkb // 4, 8)
    return sk if sk > 1 and M * N * sk <= ws_floats else 1


# ------------------------------------------------------------------------------- a small engine and its bar, a facade
SMALL = dict(vocab_size=4096, hidden_size=256, intermediate_size=640, num_layers=3, num_heads=4, num_kv_heads=2)


def _setup(max_batch, max_ctx=256, **kw):
    cfg = lm_oracle.LMConfig.tiny(**SMALL)
    w = lm_oracle.random_weights(cfg, 21, std=0.05, bf16_round=True)
    return cfg, w, make_lm(cfg, w, max_batch=max_batch, max_ctx=max_ctx, **kw)


def _bar(got, mir, tag):
    r = rel_err(got, mir)
    print(f"REFILL-PARITY {tag}: relRMS {r:.2e} max/std {max_err(got, mir) / float(mir.std()):.2e}")
    assert r < 6e-3 and max_err(got, mir) < 5e-2 * float(mir.std()), (tag, r, max_err(got, mir))


def _tts(max_batch=1, seed=7):
    from neutts import NeuTTS
    from tests.fakes import FakePhonemizer, SmallTok

    cfg = lm_oracle.LMConfig.tiny(vocab_size=4096, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4,
                                  num_kv_heads=2)
    w = lm_oracle.random_weights(cfg, 3, std=0.05, bf16_round=True)
    lm = make_lm(cfg, w, max_batch=max_batch, max_ctx=2048, max_new=512)
    ccfg = codec_oracle.CodecConfig.tiny()
    dec = make_codec(ccfg, codec_oracle.random_weights(ccfg, 2), max_batch=max_batch, max_frames=512)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=SmallTok(), phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=max_batch, seed=seed)
    tts.max_context = 2048
    return tts, ccfg
