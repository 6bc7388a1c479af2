"""GPU: the repetition penalty on every lm_head and sampler path, against transformers' RepetitionPenaltyLogitsProcessor.

The model is the logit-programmable one-layer model of ``sampler_ref.py``: a token's logits are the pattern that
owns it, so teacher-forced runs with the table off give the exact fp32 logits every launch of a run with the table on
starts from.  Each check applies transformers' processor (fp32 torch, CPU) to those logits with the history taken
from the forced ids, and compares bit for bit:

  * the logits of every launch (prefill, ``prefill_slots`` and decode), and the tile maxima (processed in the
    persistent kernel, raw behind the chain's GEMM);
  * the captured sampler windows against the float64 chain on the penalised scores (per-slot controls on top);
  * a table with every entry 1 leaves tokens, logits, windows and tile maxima bit-identical to the table off;
  * launch counts: one fix-up launch per chain lm_head and one history launch per prefill, none while off;
  * one multi-step launch at batch 1 and 8 walks out of a greedy loop in exactly the predicted order, which needs the
    token of step t in the bitmap that every CTA reads at step t + 1.

The one bar that is not bit-exact, kept probabilities within 4e-7 of the float64 chain (BARS["prob"] of
sampler_ref.py), measured at most 1.8e-7 in the teacher-forced windows and 1.2e-7 in the sampled runs on one
H100 80GB HBM3 (400 W power limit), with no ambiguous draw.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200 import synthetic
from neutts_air_b200.lm import LMShape, SpeechLM
from tests.fakes import AlignedTok
from tests.helpers import make_lm, runs_persistent, set_decode_impl
from tests.processors_ref import bits_equal, hf_penalty, ranked
from tests.sampler_ref import (BARS, MARGIN, MIN_NEW, PATTERNS, SEED, Checker, _range, prob_err,
                               processed_scores, programmable, ref_window, ref_window_cut, tile_maxima)

pytestmark = pytest.mark.gpu


PENS = [1.3, 0.7, 2.0, 1.0, 1.15, 0.9, 3.0, 1.05]


def _setup(m, B, pats, steps):
    """Prompts (two strong ids of the row's pattern, EOS, then a token of the pattern) and forced tokens (the pattern's
    best ids in order)."""
    prompts, forced = [], []
    for b, p in enumerate(pats):
        r = ranked(m, p)
        prompts.append([int(r[10]), int(r[1]), m.eos, m.token_for(p, b)])
        forced.append(r[: steps + 1])
    return prompts, torch.tensor(np.stack(forced), dtype=torch.int32)


def _run(lm, m, sp, prompts, B, steps):
    """Prefill + ``steps`` single decode steps.  Per launch: logits, captured window, tile maxima, launch count."""
    nt = m.nt
    out = []
    for j in range(steps + 1):
        n0 = lm.L.nt_launch_count()
        lg = lm.prefill(prompts, sp, return_logits=True) if j == 0 else lm.decode(1, sp, return_logits=True)[0]
        torch.cuda.synchronize()
        out.append(dict(logits=lg.cpu().numpy(), launches=lm.L.nt_launch_count() - n0,
                        cap=[t[:B].cpu().numpy().copy() for t in lm._capture],
                        tmax=lm.debug_buffer("tmax", (B, nt)).cpu().numpy().copy(),
                        out=lm.out_tokens[:B, : j + 1].cpu().numpy().copy()))
    return out


# (id, vocabulary, batch, NT_DECODE_IMPL, vocabulary range kind, per-slot controls)
TF_CASES = [
    ("persistent-b1-fold", 217472, 1, None, None, False),
    ("persistent-b3", 217472, 3, None, None, False),
    ("persistent-b8-hilo", 217472, 8, None, None, True),
    ("persistent-b16", 217472, 16, None, None, False),
    ("chain-b4-gemv-radix", 217472, 4, "perop", None, True),
    ("chain-b6-tile", 217472, 6, "perop", None, False),
    ("chain-b17-tile", 217472, 17, "perop", None, True),
    ("chain-b6-radix-v4142", 4142, 6, "perop", None, False),
    ("persistent-b3-range-eos-before", 217472, 3, None, "speech", False),
    ("persistent-b6-range-eos-inside", 217472, 6, None, "around-eos", True),
    ("chain-b2-range-eos-after", 217472, 2, "perop", "below-eos", False),
    ("chain-b7-range-eos-inside", 217472, 7, "perop", "around-eos", False),
]
STEPS = 4


@pytest.mark.parametrize("case", TF_CASES, ids=[c[0] for c in TF_CASES])
def test_penalty_every_path(cuda, case, monkeypatch):
    name, V, B, impl, rkind, ctl = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    persistent = runs_persistent(impl, B)
    pats = (PATTERNS * 3)[:B]
    prompts, forced = _setup(m, B, pats, STEPS)
    rng = _range(m, rkind) if rkind else None
    if rng:
        lm.set_vocab_range(*rng)
    rows = [(PENS[b % len(PENS)], b % 2 == 0) for b in range(B)]
    temps = [(0.7, 1.5, 1.0)[b % 3] for b in range(B)] if ctl else [1.0] * B
    ctl_rows = [(temps[b], (50, 64, 20)[b % 3], (0.9, 1.0, 0.8)[b % 3], (0.0, 0.05, 0.0)[b % 3]) for b in range(B)]
    lm.debug_capture_sampler()
    # 1. sampled: the table off, then on with every entry 1 -- bit-identical
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    runs = {}
    for tag, table in (("off", None), ("ones", [(1.0, True)] * B)):
        lm.set_repetition_penalty(table)
        lm.set_slot_sampling(ctl_rows if ctl else None)
        runs[tag] = _run(lm, m, sp, prompts, B, STEPS)
    for j, (a, b) in enumerate(zip(runs["off"], runs["ones"])):
        for k in ("logits", "tmax", "out"):
            assert bits_equal(a[k], b[k]) if k != "out" else np.array_equal(a[k], b[k]), (name, j, k)
        for x, y in zip(a["cap"], b["cap"]):
            assert np.array_equal(x, y), (name, j)
        extra = (2 if j == 0 else (0 if persistent else 1))   # history + fix-up at prefill, the fix-up per chain step
        assert b["launches"] == a["launches"] + extra, (name, j, a["launches"], b["launches"])
        if j > 0 and persistent:
            assert b["launches"] == 1 + (2 if rng else 0)
    # 2. teacher-forced: per-slot penalties, include_prompt both ways, against transformers' processor
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED, forced=forced)
    res = {}
    for tag, table in (("off", None), ("on", rows)):
        lm.set_repetition_penalty(table)
        lm.set_slot_sampling(ctl_rows if ctl else None)
        res[tag] = _run(lm, m, sp, prompts, B, STEPS)
    worst, moved = 0.0, 0
    for j in range(STEPS + 1):
        off, on = res["off"][j], res["on"][j]
        assert on["launches"] == off["launches"] + (2 if j == 0 else (0 if persistent else 1)), (name, j)
        tv, ti, _ = on["cap"]
        for b in range(B):
            pen, inc = rows[b]
            want = hf_penalty(off["logits"][b], prompts[b], forced[b, :j].tolist(), pen, inc)
            assert bits_equal(on["logits"][b], want), (name, j, b, np.nonzero(on["logits"][b] != want)[0][:5])
            if rng:
                assert np.isneginf(want[: rng[0]][np.arange(rng[0]) != m.eos]).all()
            if inc and pen != 1.0:
                e = off["logits"][b][m.eos]
                if np.isfinite(e) and e != 0:
                    assert on["logits"][b][m.eos] != e, (name, j, b)          # EOS in the prompt history is penalised
            # tile maxima: processed (1/T, EOS mask) in the persistent kernel's decode steps, raw behind every lm_head else
            if j > 0 and persistent:
                assert bits_equal(on["tmax"][b], tile_maxima(processed_scores(want, j, m.eos, MIN_NEW, temps[b]))), (name, j, b)
            else:
                assert bits_equal(on["tmax"][b], tile_maxima(want)), (name, j, b)
            moved += not bits_equal(on["tmax"][b], off["tmax"][b])
            # the captured window: the float64 chain on the penalised scores (penalty -> EOS mask -> 1/T -> cuts)
            if ctl:
                T, k, tp, mp = ctl_rows[b]
                ids, p, margin = ref_window_cut(want, j, m.eos, MIN_NEW, T, k, tp, mp)
                if margin < MARGIN:
                    continue
            else:
                ids, p = ref_window(want, j, m.eos, MIN_NEW, 50, 1.0)
            assert ti[b, : len(ids)].tolist() == ids.tolist(), (name, j, b)
            err = prob_err(tv[b, : len(ids)], p)
            worst = max(worst, err)
            assert err < BARS["prob"], (name, j, b, err)
    assert moved > 0   # the penalty moved tile maxima (below 1 they rise)
    print(f"PENALTY {name}: logits and tile maxima bit-identical to transformers' processor; worst window prob err {worst:.2e}")


@pytest.mark.parametrize("impl,B", [(None, 3), ("perop", 6), ("perop", 4)], ids=["persistent-b3", "chain-b6-tile", "chain-b4-radix"])
def test_penalty_sampled_vs_float64(cuda, impl, B, monkeypatch):
    """Sampled runs with the penalty on: kept ids exact, kept probabilities within the bar, every token on the float64
    inverse CDF of the same Philox draw, computed on the (penalised) logits the launch returned."""
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    lm.set_repetition_penalty([(PENS[b], b % 2 == 1) for b in range(B)])
    ck = Checker(m, lm, sp, False)
    pats = ["gauss", "ties", "stairs", "onetile", "gauss", "flat"][:B]
    prompts, _ = _setup(m, B, pats, 0)
    before = ck.snapshot()
    lg = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    before["ngen"][:] = 0
    before["done"][:] = 0
    ck.check_launch(lg, list(range(B)), list(range(B)), before, after, 0, tag="prefill")
    for step in range(6):
        before = ck.snapshot()
        if before["done"][:B].all():
            break
        lg = lm.decode(1, sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        ck.check_launch(lg, list(range(B)), list(range(B)), before, ck.snapshot(), 1, tag=f"step {step}")
    ck.report(f"penalty-sampled-{impl or 'persistent'}-b{B}")


@pytest.mark.parametrize("impl,B", [(None, 1), (None, 8), ("perop", 6)], ids=["persistent-b1-fold", "persistent-b8-hilo", "chain-b6"])
def test_multistep_launch_breaks_a_greedy_loop(cuda, impl, B, monkeypatch):
    """Greedy decoding repeats one id forever without the penalty (asserted first).  With penalty 2, one decode call of
    40 steps walks through the pattern's ids in exactly the order a float64 prediction gives, where the token of step t
    is penalised at step t + 1; every step's logits are the penalised ones, bit for bit."""
    V, n = 217472, 40
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    # patterns with many strong ids: a set-based penalty walks through them (one dominant id and a cliff would not)
    pats = ["gauss", "ties", "stairs", "gauss", "ties", "stairs", "gauss", "ties"][:B]
    prompts, _ = _setup(m, B, pats, 0)
    sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=64, greedy=True, seed=SEED)
    lm.set_repetition_penalty(None)
    first_off = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    n0 = lm.L.nt_launch_count()
    off = lm.decode(n, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    if impl is None:
        assert lm.L.nt_launch_count() - n0 == 1
    toks_off = lm.out_tokens[:B, : n + 1].cpu().numpy()
    for b in range(B):
        assert (toks_off[b, 1:] == toks_off[b, 1]).all(), (b, toks_off[b])     # stuck on one id
    lm.set_repetition_penalty([(2.0, True)] * B)
    first_on = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    n0 = lm.L.nt_launch_count()
    on = lm.decode(n, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    if impl is None:
        assert lm.L.nt_launch_count() - n0 == 1
    toks = lm.out_tokens[:B, : n + 1].cpu().numpy()
    for b in range(B):
        hist = list(prompts[b])
        want0 = hf_penalty(first_off[b], prompts[b], [], 2.0, True)
        assert bits_equal(first_on[b], want0)
        pred = [int(np.argmax(want0))]
        L = off[0, b]   # every step of the pattern has these logits (bit-identical across the steps of a launch)
        assert all(bits_equal(off[s, b], L) for s in range(n))
        for s in range(n):
            want = hf_penalty(L, hist, pred, 2.0, True)
            assert bits_equal(on[s, b], want), (b, s)
            pred.append(int(np.argmax(want)))
        assert toks[b].tolist() == pred, (b, toks[b].tolist(), pred)
        assert len(set(pred[1:])) > n // 2, pred      # the loop is broken: the walk visits many ids
    print(f"PENALTY multistep {impl or 'persistent'} B={B}: {n} steps in one call follow the predicted walk")


def test_prefill_slots_history_and_survivors(cuda, monkeypatch):
    """A refilled slot's history is its new prompt only; a survivor's logits are bit-identical with or without the
    refill.  Teacher-forced, chain decode (tile sampler) and persistent decode."""
    V, MB = 217472, 6
    m = programmable(V)
    cfg, w = m.oracle()
    pats = PATTERNS[:MB]
    prompts, forced = _setup(m, MB, pats, 8)
    newp = [int(ranked(m, "gauss")[3]), int(ranked(m, "gauss")[0]), m.token_for("gauss", 9)]
    rows = [(1.3, True), (0.8, True), (2.0, False), (1.2, True), (1.0, True), (1.5, True)]
    for impl in ("perop", None):
        set_decode_impl(monkeypatch, impl)
        res = {}
        for tag in ("refill", "plain", "off"):
            lm = make_lm(cfg, w, max_batch=MB, max_ctx=256, max_new=64)
            lm.set_repetition_penalty(None if tag == "off" else rows)
            sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, forced=forced)
            lm.prefill(prompts, sp)
            lm.decode(2, sp)
            slot_lg = None
            if tag != "plain":
                n0 = lm.L.nt_launch_count()
                slot_lg = lm.prefill_slots([2], [newp], sp, [77], return_logits=True).cpu().numpy()
                torch.cuda.synchronize()
                res[tag + "_launches"] = lm.L.nt_launch_count() - n0
            res[tag] = (slot_lg, lm.decode(1, sp, return_logits=True)[0].cpu().numpy())
            torch.cuda.synchronize()
        assert res["refill_launches"] == res["off_launches"] + 2
        # the refilled slot: prompt-only history at its prefill, then prompt + its first (forced) token
        pen, inc = rows[2]
        assert bits_equal(res["refill"][0][0], hf_penalty(res["off"][0][0], newp, [], pen, inc))
        assert bits_equal(res["refill"][1][2], hf_penalty(res["off"][1][2], newp, forced[2, :1].tolist(), pen, inc))
        for s in range(MB):
            if s != 2:
                assert bits_equal(res["refill"][1][s], res["plain"][1][s]), (impl, s)


def test_lifecycle(cuda, monkeypatch):
    """Switching on between prefill and decode leaves that decode bit-identical to off (the slots are unrecorded);
    switching off, then on, then prefilling restores the penalty.  Bad tables are refused and change nothing."""
    V, B = 217472, 3
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    pats = ["gauss", "ties", "onetile"]
    prompts, forced = _setup(m, B, pats, 6)
    rows = [(1.3, True), (0.7, True), (2.0, True)]
    for impl in (None, "perop"):
        set_decode_impl(monkeypatch, impl)
        sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=64, forced=forced)
        lm.set_repetition_penalty(None)
        p_off = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
        d_off = lm.decode(2, sp, return_logits=True).cpu().numpy()
        lm.prefill(prompts, sp)
        lm.set_repetition_penalty(rows)                       # on after the prefill: unrecorded
        d_late = lm.decode(2, sp, return_logits=True).cpu().numpy()
        assert bits_equal(d_late, d_off), impl
        lm.set_repetition_penalty(None)
        lm.set_repetition_penalty(rows)
        p_on = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
        d_on = lm.decode(2, sp, return_logits=True).cpu().numpy()
        torch.cuda.synchronize()
        for b in range(B):
            assert bits_equal(p_on[b], hf_penalty(p_off[b], prompts[b], [], *rows[b]))
            for s in range(2):
                assert bits_equal(d_on[s, b], hf_penalty(d_off[s, b], prompts[b], forced[b, : s + 1].tolist(), *rows[b]))
        # new values in a table that stays on take effect at the next launch; the histories are kept (a row's
        # unpenalised logits are those of its pattern at every step)
        lm.set_repetition_penalty([(1.1, True)] * B)
        d_new = lm.decode(1, sp, return_logits=True).cpu().numpy()
        for b in range(B):
            assert bits_equal(d_new[0, b], hf_penalty(d_off[1, b], prompts[b], forced[b, :3].tolist(), 1.1, True))
    for bad in ([(0.0, True)] * B, [(float("nan"), True)] * B, [(-1.0, True)] * B, [(float("inf"), True)] * B):
        with pytest.raises(ValueError):
            lm.set_repetition_penalty(bad)
    from neutts_air_b200 import _lib

    arr = (_lib.SlotPenalty * B)(*(_lib.SlotPenalty(1.2, 2) for _ in range(B)))
    assert lm.L.nt_lm_set_repetition_penalty(lm.handle, arr, None) != 0 and b"include_prompt" in lm.L.nt_last_error()
    assert lm._penalty_host == [(1.1, True)] * B


# ------------------------------------------------------------------------------------------------ full Air size
@pytest.mark.parametrize("B", [1, 64])
def test_full_size_teacher_forced(cuda, B, monkeypatch):
    """Air shape, synthetic weights: a 500-token prompt and 250 teacher-forced steps with penalty 1.3 (prompt included),
    at batch 1 (persistent kernel) and batch 64 (chain).  Every launch's logits are transformers' processor applied to
    the table-off logits of an identical engine run in lock-step, bit for bit."""
    set_decode_impl(monkeypatch, None)
    shape = LMShape()
    V, eos, steps = shape.vocab_size, 151670, 250
    sd = synthetic.lm_state_dict(shape, 0)
    eng = [SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=1024, max_new=256, max_prefill_tokens=B * 520)
           for _ in range(2)]
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, V, (500,), generator=g).tolist() for _ in range(B)]
    forced = torch.randint(151936, V, (B, steps + 1), generator=g)
    forced[:, 5:40] = forced[:, :1]                      # a loop on one id: the history keeps it once
    forced[:, 40:60] = torch.tensor(prompts)[:, 100:120]  # generated ids that are also in the prompt
    forced[forced == eos] = eos + 1
    eng[1].set_repetition_penalty([(1.3, True)] * B)
    sps = [e.sampling(eos, min_new_tokens=0, max_new_tokens=steps + 1, forced=forced) for e in eng]
    lgs = [e.prefill(prompts, sp, return_logits=True) for e, sp in zip(eng, sps)]
    for s in range(steps + 1):
        off, on = (x.cpu().numpy() for x in lgs)
        for b in range(B):
            assert bits_equal(on[b], hf_penalty(off[b], prompts[b], forced[b, :s].tolist(), 1.3, True)), (B, s, b)
        if s < steps:
            lgs = [e.decode(1, sp, return_logits=True)[0] for e, sp in zip(eng, sps)]
    assert torch.equal(eng[1].out_tokens[:B, : steps + 1].cpu(), forced.int())
    print(f"PENALTY full size B={B}: {steps} teacher-forced steps bit-identical to transformers' processor")


# ------------------------------------------------------------------------------------------------ the facade
class _NoQueue:
    """The engine without ``generate_queue``: the facade then runs chunks of ``max_batch``."""

    def __init__(self, lm):
        self._lm = lm

    def __getattr__(self, k):
        if k == "generate_queue":
            raise AttributeError(k)
        return getattr(self._lm, k)


@pytest.mark.parametrize("mode", ["queue", "chunked", "stream"])
def test_facade_per_utterance_penalty(cuda, mode, monkeypatch):
    """NeuTTS with per-utterance penalty lists (infer_batch on the queue and in chunks, infer_stream_batch): each
    utterance's tokens equal a generate_batch run of its chunk with its own penalty and stream key."""
    import warnings

    from neutts import NeuTTS
    from oracle import codec_oracle as CO
    from oracle import lm_oracle as LO
    from tests.fakes import FakePhonemizer
    from tests.helpers import make_codec

    set_decode_impl(monkeypatch, None)
    tok = AlignedTok()
    V = tok.speech_base + 65536
    eos = tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>")
    cfg = LO.LMConfig.tiny(vocab_size=V, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    lm = make_lm(cfg, LO.random_weights(cfg, 3, std=0.05, bf16_round=True), max_batch=2, max_ctx=2048, max_new=256)
    ccfg = CO.CodecConfig.tiny()
    dec = make_codec(ccfg, CO.random_weights(ccfg, 2), max_batch=4, max_frames=512)
    n = 2 if mode == "stream" else 4
    texts = ["alpha", "beta gamma", "delta", "eps zeta"][:n]
    refs, rts = [torch.arange(10 + 5 * i) for i in range(n)], ["one", "two", "three", "four"][:n]
    pens, incl = [1.0, 1.3, 2.0, 0.8][:n], [True, False, True, True][:n]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=_NoQueue(lm) if mode == "chunked" else lm, codec=dec,
                     max_batch=2, seed=7)
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    tts.max_context = max(len(p) for p in prompts) + 60
    if mode == "stream":
        tts.streaming_frames_per_chunk = 25
        for _ in tts.infer_stream_batch(texts, refs, rts, repetition_penalty=pens, penalize_prompt=incl):
            pass
        torch.cuda.synchronize()
        got = [lm.out_tokens[b, : int(lm.n_generated[b])].cpu() for b in range(n)]
        want = lm.generate_batch(prompts, eos, max_length=tts.max_context, min_new_tokens=50, seed=7, repetition_penalty=pens,
                                 penalize_prompt=incl)
    else:
        # equal caps with EOS masked: the queue's schedule coincides with the chunked one (both decode at batch 2)
        cap = 40
        kw = dict(max_new_tokens=cap, min_new_tokens=cap) if mode == "queue" else {}
        seen = []
        meth = "generate_queue" if mode == "queue" else "generate_batch"
        orig = getattr(lm, meth)

        def rec(*a, **k):
            out = orig(*a, **k)
            seen.append((k, out))
            return out

        monkeypatch.setattr(lm, meth, rec)
        wavs = tts.infer_from_prompt_ids(prompts, repetition_penalty=pens, penalize_prompt=incl, **kw) if mode == "queue" else \
            tts.infer_batch(texts, refs, rts, repetition_penalty=pens, penalize_prompt=incl)
        assert all(len(w_) > 0 and np.isfinite(w_).all() for w_ in wavs)
        assert [k["repetition_penalty"] for k, _ in seen] == ([pens] if mode == "queue" else [pens[0:2], pens[2:4]])
        assert [k["penalize_prompt"] for k, _ in seen] == ([incl] if mode == "queue" else [incl[0:2], incl[2:4]])
        got = [t for _, out in seen for t in out]
        monkeypatch.undo()
        set_decode_impl(monkeypatch, None)
        gkw = dict(min_new_tokens=cap, max_new_tokens=cap) if mode == "queue" else dict(min_new_tokens=50)
        want = []
        for j in range(0, n, 2):
            want += lm.generate_batch(prompts[j: j + 2], eos, max_length=tts.max_context, seed=7, slot_base=j,
                                      repetition_penalty=pens[j: j + 2], penalize_prompt=incl[j: j + 2], **gkw)
        # the penalty does something: without it, utterances 2 and 3 come out differently
        plain = lm.generate_batch(prompts[2:4], eos, max_length=tts.max_context, seed=7, slot_base=2, **gkw)
        assert not torch.equal(plain[0], want[2]) or not torch.equal(plain[1], want[3])
    assert len(got) == n
    for i in range(n):
        assert torch.equal(got[i].long(), want[i].long()), (mode, i, got[i][:10], want[i][:10])
