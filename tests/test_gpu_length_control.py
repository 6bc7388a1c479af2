"""GPU: per-slot length control (min_new_tokens and the exponential decay length penalty) on every lm_head and sampler
path, against transformers' MinNewTokensLengthLogitsProcessor and ExponentialDecayLengthPenalty.

The model is the logit-programmable one-layer model of ``sampler_ref.py``: a token's logits are the pattern that owns
it, so teacher-forced runs with the table off give the exact fp32 logits every launch of a run with the table on starts
from.  Each check applies transformers' processors (fp32 torch, CPU) to those logits and compares bit for bit:

  * the stored logits of every launch hold the decayed EOS score (the mask is not stored, as without the table);
  * the tile maxima: processed (decay, mask, 1/T) in the persistent kernel's decode steps, raw elsewhere;
  * the captured sampler windows against the float64 chain with each slot's own floor;
  * a neutral table (every slot at the launch's floor, factor 1) leaves tokens, logits, windows, tile maxima, state and
    launch counts bit-identical to the table off;
  * one multi-step launch: EOS is never drawn before a slot's floor, and a decaying slot draws it at the predicted step.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200 import synthetic
from neutts_air_b200.lm import LMShape, SpeechLM
from tests.helpers import make_lm, runs_persistent, set_decode_impl
from tests.processors_ref import bits_equal, hf_chain, ranked
from tests.sampler_ref import (BARS, MARGIN, MIN_NEW, PATTERNS, SEED, Checker, _range, draw_u, prob_err,
                               processed_scores, programmable, ref_token, ref_window, ref_window_cut, tile_maxima)

pytestmark = pytest.mark.gpu


# per-slot (min_new_tokens, decay_start, decay_factor): floors 0..3, starts at or after floor - 1, factors on both
# sides of 1 (and 1 itself)
LENGTHS = [(0, 0, 1.3), (2, 1, 0.8), (1, 0, 2.5), (3, 2, 1.0), (0, 1, 1.05), (2, 3, 1.7), (1, 1, 0.5), (3, 4, 3.0)]
STEPS = 5


def _setup(m, B, pats, steps):
    prompts, forced = [], []
    for b, p in enumerate(pats):
        r = ranked(m, p)
        prompts.append([int(r[10]), int(r[1]), m.eos, m.token_for(p, b)])
        forced.append(r[: steps + 1])
    return prompts, torch.tensor(np.stack(forced), dtype=torch.int32)


def _run(lm, m, sp, prompts, B, steps):
    nt = m.nt
    out = []
    for j in range(steps + 1):
        n0 = lm.L.nt_launch_count()
        lg = lm.prefill(prompts, sp, return_logits=True) if j == 0 else lm.decode(1, sp, return_logits=True)[0]
        torch.cuda.synchronize()
        out.append(dict(logits=lg.cpu().numpy(), launches=lm.L.nt_launch_count() - n0,
                        cap=[t[:B].cpu().numpy().copy() for t in lm._capture],
                        tmax=lm.debug_buffer("tmax", (B, nt)).cpu().numpy().copy(),
                        out=lm.out_tokens[:B, : j + 1].cpu().numpy().copy(),
                        state=torch.stack((lm.n_generated[:B], lm.done[:B], lm.seq_lens[:B])).cpu().numpy()))
    return out


# (id, vocabulary, batch, NT_DECODE_IMPL, vocabulary range kind, per-slot controls, penalty)
TF_CASES = [
    ("persistent-b1-fold", 217472, 1, None, None, False, False),
    ("persistent-b3", 217472, 3, None, None, False, True),
    ("persistent-b8-hilo", 217472, 8, None, None, True, False),
    ("persistent-b16", 217472, 16, None, None, False, True),
    ("chain-b2-gemv", 217472, 2, "perop", None, False, False),
    ("chain-b4-gemv", 217472, 4, "perop", None, True, True),
    ("chain-b6-tile", 217472, 6, "perop", None, False, False),
    ("chain-b17-tile", 217472, 17, "perop", None, True, False),
    ("chain-b6-v4142", 4142, 6, "perop", None, False, True),
    ("persistent-b3-range-eos-before", 217472, 3, None, "speech", False, False),
    ("persistent-b6-range-eos-inside", 217472, 6, None, "around-eos", True, True),
    ("chain-b2-range-eos-after", 217472, 2, "perop", "below-eos", False, False),
    ("chain-b7-range-eos-inside", 217472, 7, "perop", "around-eos", False, True),
]


@pytest.mark.parametrize("case", TF_CASES, ids=[c[0] for c in TF_CASES])
def test_length_control_every_path(cuda, case, monkeypatch):
    name, V, B, impl, rkind, ctl, pen = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    persistent = runs_persistent(impl, B)
    pats = (["eos"] + PATTERNS * 3)[:B]
    prompts, forced = _setup(m, B, pats, STEPS)
    rng = _range(m, rkind) if rkind else None
    if rng:
        lm.set_vocab_range(*rng)
    pens = [(1.3, 1.0, 0.8)[b % 3] for b in range(B)] if pen else [1.0] * B
    temps = [(0.7, 1.5, 1.0)[b % 3] for b in range(B)] if ctl else [1.0] * B
    ctl_rows = [(temps[b], (50, 64, 20)[b % 3], (0.9, 1.0, 0.8)[b % 3], (0.0, 0.05, 0.0)[b % 3]) for b in range(B)]
    rows = [LENGTHS[b % len(LENGTHS)] for b in range(B)]
    lm.set_repetition_penalty([(p, True) for p in pens] if pen else None)
    lm.set_slot_sampling(ctl_rows if ctl else None)
    lm.debug_capture_sampler()
    # 1. sampled: the table off, then a neutral table (the launch's floor, no decay) -- bit-identical, same launches
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    runs = {}
    for tag, table in (("off", None), ("neutral", [(MIN_NEW, MIN_NEW - 1, 1.0)] * B)):
        lm.set_length_control(table)
        runs[tag] = _run(lm, m, sp, prompts, B, STEPS)
    for j, (a, b) in enumerate(zip(runs["off"], runs["neutral"])):
        for k in ("logits", "tmax", "out", "state"):
            assert bits_equal(a[k], b[k]) if k in ("logits", "tmax") else np.array_equal(a[k], b[k]), (name, j, k)
        for x, y in zip(a["cap"], b["cap"]):
            assert np.array_equal(x, y), (name, j)
        assert a["launches"] == b["launches"], (name, j)
    # 2. teacher-forced: per-slot floors and decays against transformers' processors on the table-off logits
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED, forced=forced)
    res = {}
    for tag, table in (("off", None), ("on", rows)):
        lm.set_length_control(table)
        res[tag] = _run(lm, m, sp, prompts, B, STEPS)
    worst, decayed = 0.0, 0
    for j in range(STEPS + 1):
        off, on = res["off"][j], res["on"][j]
        # the chain's decode steps add one fix-up launch while some entry decays; prefills and the persistent kernel none
        decays = any(f != 1.0 for _, _, f in rows)
        assert on["launches"] == off["launches"] + (1 if decays and j > 0 and not persistent else 0), (name, j)
        tv, ti, _ = on["cap"]
        for b in range(B):
            mn, start, f = rows[b]
            want = hf_chain(res["off"][j]["logits"][b], prompts[b], forced[b, :j].tolist(), j, 1.0, (start, f), m.eos)
            assert bits_equal(on["logits"][b], want), (name, j, b, np.nonzero(on["logits"][b] != want)[0][:5])
            decayed += not bits_equal(want, off["logits"][b])
            if j > 0 and persistent:
                assert bits_equal(on["tmax"][b], tile_maxima(processed_scores(want, j, m.eos, mn, temps[b]))), (name, j, b)
            else:
                assert bits_equal(on["tmax"][b], tile_maxima(want)), (name, j, b)
            if ctl:
                T, k, tp, mp = ctl_rows[b]
                ids, p, margin = ref_window_cut(want, j, m.eos, mn, T, k, tp, mp)
                if margin < MARGIN:
                    continue
            else:
                ids, p = ref_window(want, j, m.eos, mn, 50, 1.0)
            assert ti[b, : len(ids)].tolist() == ids.tolist(), (name, j, b)
            err = prob_err(tv[b, : len(ids)], p)
            worst = max(worst, err)
            assert err < BARS["prob"], (name, j, b, err)
    assert decayed > 0
    print(f"LENGTH {name}: logits and tile maxima bit-identical to transformers' processors; worst window prob err {worst:.2e}")


def _predict(m, first, steps_logits, prompt, mn, decay, n):
    """Greedy tokens under the length control, from the table-off logits of each draw (valid until EOS: before it
    the on and off runs draw the same ids)."""
    toks = []
    for s in range(n + 1):
        row = first if s == 0 else steps_logits[s - 1]
        want = hf_chain(row, prompt, toks, s, 1.0, decay, m.eos)
        sc = want.astype(np.float64)
        if s < mn:
            sc[m.eos] = -np.inf
        toks.append(int(np.argmax(sc)))
        if toks[-1] == m.eos:
            break
    return toks


@pytest.mark.parametrize("impl,B", [(None, 1), (None, 8), ("perop", 6)], ids=["persistent-b1-fold", "persistent-b8-hilo", "chain-b6"])
def test_multistep_launch_ends_at_the_predicted_step(cuda, impl, B, monkeypatch):
    """Greedy, one decode call of n steps.  Slots on the "eos" pattern (EOS is their largest logit) draw EOS exactly at
    their own floor; the other slots never draw EOS without the table, and with a decay draw it at the step transformers'
    processors predict from the table-off logits."""
    V, n = 217472, 40
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    pats = ["gauss", "eos", "stairs", "eos", "ties", "onetile", "eos", "gauss"][:B] if B > 1 else ["gauss"]
    prompts, _ = _setup(m, B, pats, 0)
    rows = [(5 + 3 * b, 6 + 3 * b, 1.0) if p == "eos" else (b % 3, 4 + b, (1.12, 1.3, 1.08, 1.2)[b % 4])
            for b, p in enumerate(pats)]
    sp = lm.sampling(m.eos, min_new_tokens=n + 5, max_new_tokens=64, greedy=True, seed=SEED)
    lm.set_length_control(None)
    first_off = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    off = lm.decode(n, sp, return_logits=True).cpu().numpy()
    assert not (lm.out_tokens[:B, : n + 1].cpu().numpy() == m.eos).any()
    lm.set_length_control(rows)
    first_on = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    n0 = lm.L.nt_launch_count()
    on = lm.decode(n, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    if impl is None:
        assert lm.L.nt_launch_count() - n0 == 1
    toks = lm.out_tokens[:B].cpu().numpy()
    ngen = lm.n_generated[:B].cpu().tolist()
    for b in range(B):
        mn, start, f = rows[b]
        assert bits_equal(first_on[b], first_off[b])   # a prefill draws at n = 0: nothing decays
        pred = _predict(m, first_off[b], off[:, b], prompts[b], mn, (start, f), n)
        assert pred[-1] == m.eos, (b, pred)
        assert toks[b, : len(pred)].tolist() == pred and ngen[b] == len(pred), (b, toks[b, : len(pred)], pred)
        assert m.eos not in toks[b, : mn].tolist()
        if pats[b] == "eos":
            assert len(pred) == mn + 1, (b, pred)          # EOS at the first draw the floor allows
        for s in range(len(pred) - 1):                     # the stored logits of every step before EOS
            want = hf_chain(off[s, b], prompts[b], pred, s + 1, 1.0, (start, f), m.eos)
            assert bits_equal(on[s, b], want), (b, s)


class SlotFloorChecker(Checker):
    """``Checker`` with each slot's own min_new_tokens: the Philox stream key of a launch row is its slot here
    (slot_base 0, no refill), so the key picks the floor."""

    def __init__(self, m, lm, sp, floors):
        super().__init__(m, lm, sp, False)
        self.floors = floors
        self.eos_live = 0   # draws whose window kept EOS with a non-negligible probability

    def expect_token(self, logits_row, ngen, key):
        sp = self.sp
        win = ref_window(logits_row, ngen, sp.eos_id, self.floors[key], sp.top_k, sp.temperature)
        tok, ok = ref_token(win, draw_u(sp.seed, ngen, key))
        self.draws += 1
        self.ambiguous += len(ok) > 1
        ids, p = win
        self.eos_live += bool(((ids == sp.eos_id) & (p > 1e-3)).any())
        return win, tok, ok


# per-slot (min_new_tokens, decay_start, decay_factor) of the sampled runs: EOS starts at -30 on these patterns, and the
# decays bring it into the window within a few steps (factor 0.7 pushes it further down)
SAMPLED = [(2, 1, 2.0), (0, 0, 1.6), (3, 3, 1.4), (1, 2, 0.7), (0, 1, 1.5), (2, 2, 1.8), (1, 0, 1.3), (0, 0, 1.0)]


@pytest.mark.parametrize("impl,B", [(None, 3), (None, 8), ("perop", 6), ("perop", 17)],
                         ids=["persistent-b3", "persistent-b8-hilo", "chain-b6-tile", "chain-b17-tile"])
def test_sampled_with_decay_vs_float64(cuda, impl, B, monkeypatch):
    """Sampled runs with per-slot floors and decays: kept ids exact, kept probabilities within the bar, every token on
    the float64 inverse CDF of the same Philox draw over the (decayed) logits the launch returned, with each slot's own
    floor; no EOS before a floor, and the decaying slots end on EOS within the run."""
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    rows = [SAMPLED[b % len(SAMPLED)] for b in range(B)]
    lm.set_length_control(rows)
    ck = SlotFloorChecker(m, lm, sp, [r[0] for r in rows])
    pats = (["gauss", "ties", "stairs", "onetile", "plateau", "flat"] * 3)[:B]
    prompts = [[m.token_for("gauss", b), m.token_for(p, b)] for b, p in enumerate(pats)]
    before = ck.snapshot()
    lg = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    before["ngen"][:] = 0
    before["done"][:] = 0
    ck.check_launch(lg, list(range(B)), list(range(B)), before, after, 0, tag="prefill")
    for step in range(16):
        before = ck.snapshot()
        if before["done"][:B].all():
            break
        lg = lm.decode(1, sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        ck.check_launch(lg, list(range(B)), list(range(B)), before, ck.snapshot(), 1, tag=f"step {step}")
    toks, ngen = lm.out_tokens[:B].cpu().numpy(), lm.n_generated[:B].cpu().numpy()
    for b, (mn, start, f) in enumerate(rows):
        assert m.eos not in toks[b, : min(mn, ngen[b])].tolist(), (b, toks[b, : ngen[b]])
        if f > 1.0:
            assert toks[b, ngen[b] - 1] == m.eos, (b, rows[b], toks[b, : ngen[b]])
    assert ck.eos_live > 0
    ck.report(f"length-sampled-{impl or 'persistent'}-b{B} (eos live in {ck.eos_live} windows)")


def test_prefill_slots_and_forks_take_their_entries(cuda, monkeypatch):
    """``prefill_slots`` writes the refilled slots' new entries and leaves the survivors bit-identical; the takes of a
    fork inherit their prompt's entry (every take of an "eos" prompt ends exactly at its prompt's floor)."""
    V, B = 217472, 4
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, "perop")
    eos_prompt = [m.token_for("eos", 0)]
    gauss = [m.token_for("gauss", 1)]
    sp = lm.sampling(m.eos, min_new_tokens=60, max_new_tokens=64, greedy=True, seed=SEED)
    # survivors' reference: slots 0, 2 decode without a refill
    base_rows = [(60, 59, 1.0)] * B
    lm.set_length_control(base_rows)
    lm.prefill([gauss, gauss, gauss, gauss], sp)
    lm.decode(3, sp)
    ref = lm.decode(8, sp, return_logits=True).cpu().numpy()
    ref_tok = lm.out_tokens[:B, :12].cpu().numpy()
    lm.prefill([gauss, gauss, gauss, gauss], sp)
    lm.decode(3, sp)
    lm.set_length_control([(4, 5, 1.0), (7, 8, 1.0)], slots=[1, 3])
    lm.prefill_slots([1, 3], [eos_prompt, eos_prompt], sp, stream_ids=[11, 13])
    got = lm.decode(8, sp, return_logits=True).cpu().numpy()
    toks = lm.out_tokens[:B, :12].cpu().numpy()
    for s in (0, 2):
        assert bits_equal(got[:, s], ref[:, s]) and np.array_equal(toks[s], ref_tok[s]), s
    for s, mn in ((1, 4), (3, 7)):
        assert toks[s, mn] == m.eos and m.eos not in toks[s, :mn].tolist(), (s, toks[s])
    # forks: 2 prompts x 2 takes, the prompts' floors 3 and 6
    outs = lm.generate_batch([eos_prompt, eos_prompt], m.eos, max_length=200, min_new_tokens=[3, 6], max_new_tokens=20,
                             greedy=True, seed=SEED, num_return_sequences=2)
    assert [len(o) for o in outs] == [4, 4, 7, 7] and all(int(o[-1]) == m.eos for o in outs), outs


def test_toggle_and_graph_recapture(cuda, monkeypatch):
    """The chain's cached decode graph follows the table: off, on with decay, new values, neutral, off.  Each multi-step
    launch (graph replay) matches single steps (no graph) under the same table, bit for bit."""
    V, B, n = 4142, 3, 12
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, "perop")
    prompts = [[m.token_for(p, b)] for b, p in enumerate(["gauss", "stairs", "ties"])]
    sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=64, greedy=True, seed=SEED)
    tables = [None, [(0, 2, 1.4)] * B, [(1, 3, 1.9), (0, 0, 1.2), (2, 5, 2.2)], [(0, 0, 1.0)] * B, None]
    for t in tables:
        lm.set_length_control(t)
        lm.prefill(prompts, sp)
        lm.decode(n, sp)                       # graph replay
        torch.cuda.synchronize()
        graph = (lm.out_tokens[:B, : n + 1].cpu().numpy(), lm.n_generated[:B].cpu().numpy())
        lm.prefill(prompts, sp)
        lm.decode(n, sp, return_logits=True)   # no graph: one decode_step per step
        torch.cuda.synchronize()
        single = (lm.out_tokens[:B, : n + 1].cpu().numpy(), lm.n_generated[:B].cpu().numpy())
        assert all(np.array_equal(a, b) for a, b in zip(graph, single)), t
        if t is not None and t[0][2] != 1.0:
            assert (graph[0] == m.eos).any(), t   # the decay ends every slot inside the window


def test_overflow_refused_only_for_sampled_slots(cuda):
    """A c_k that overflows fp32 within a launch's max_new_tokens is refused by the launch that samples its slot; a slot
    the launch never reads may keep an entry of an earlier call with a shorter cap."""
    V = 4142
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=2, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=64, seed=SEED)
    lm.set_length_control([(0, 0, 1.0), (0, 0, 10.0)])   # 10**39 - 1 overflows fp32 at k = 39 <= 64
    with pytest.raises((ValueError, RuntimeError), match="slot 1: .*not finite"):
        lm.prefill([[1], [2]], sp)
    lm.prefill([[1]], sp)                                 # slot 1 is not sampled
    lm.decode(2, sp)
    with pytest.raises((ValueError, RuntimeError), match="slot 1: .*not finite"):
        lm.prefill_slots([1], [[2]], sp, stream_ids=[1])
    sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=30, seed=SEED)
    lm.prefill([[1], [2]], sp)
    # through SpeechLM: a later call with fewer prompts and a larger cap leaves the earlier entry in slot 1 alone
    lm.generate_batch([[1], [2]], m.eos, max_length=200, min_new_tokens=0, max_new_tokens=30, seed=SEED,
                      exponential_decay_length_penalty=(0, 10.0))
    out = lm.generate_batch([[1]], m.eos, max_length=200, min_new_tokens=0, max_new_tokens=64, seed=SEED,
                            exponential_decay_length_penalty=(0, 1.5))
    assert lm._length_host[1] == (0, 0, 10.0) and len(out) == 1
    lm.set_length_control(None)


def test_facade_lists_match_generate_batch(cuda):
    """A pass-through check: ``NeuTTS.infer_batch`` hands its per-utterance floors and decays to
    ``SpeechLM.generate_batch`` unchanged, and a second ``generate_batch`` call with the same ids and settings gives the
    same tokens.  The values themselves are checked against transformers by the tests above."""
    from tests.helpers import _tts

    tts, _ = _tts(max_batch=3, seed=7)
    lm = tts.backbone
    texts, refs, rtexts = ["a b", "c d e", "f"], [np.arange(5) % 7, np.arange(3) % 7, np.arange(4) % 7], ["x", "y", "z"]
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rtexts)]
    mn = [2, 0, 5]
    decay = [(3, 1.05), None, (6, 1.02)]
    seen = {}
    orig = lm.generate_batch

    def spy(*a, **k):
        seen.update(k)
        out = orig(*a, **k)
        seen["out"] = out
        return out

    lm.generate_batch = spy
    tts.infer_batch(texts, refs, rtexts, min_new_tokens=mn, exponential_decay_length_penalty=decay)
    lm.generate_batch = orig
    assert seen["min_new_tokens"] == mn and seen["exponential_decay_length_penalty"] == [(3, 1.05), None, (6, 1.02)]
    eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
    want = lm.generate_batch(prompts, eos, max_length=tts.max_context, min_new_tokens=mn, seed=seen["seed"],
                             exponential_decay_length_penalty=decay, **{k: v for k, v in seen.items() if k in (
                                 "temperature", "top_k", "vocab_range", "slot_base")})
    assert all(torch.equal(a, b) for a, b in zip(seen["out"], want))


# ------------------------------------------------------------------------------------------------ full Air size
@pytest.mark.parametrize("B", [1, 64])
def test_full_size_teacher_forced(cuda, B, monkeypatch):
    """Air shape, synthetic weights: a 500-token prompt and 250 teacher-forced steps with the decay on every slot (starts
    0..4, factors 1.01, 1.02, 0.99 and 1) and floors on some, at batch 1 (persistent kernel) and batch 64 (chain).
    Every launch's logits are transformers' ExponentialDecayLengthPenalty applied to the table-off logits of an
    identical engine run in lock-step, bit for bit; k reaches 250 (c_k up to 140 at factor 1.02)."""
    set_decode_impl(monkeypatch, None)
    shape = LMShape()
    V, eos, steps = shape.vocab_size, 151670, 250
    sd = synthetic.lm_state_dict(shape, 0)
    eng = [SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=1024, max_new=256, max_prefill_tokens=B * 520)
           for _ in range(2)]
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, V, (500,), generator=g).tolist() for _ in range(B)]
    forced = torch.randint(151936, V, (B, steps + 1), generator=g)
    forced[forced == eos] = eos + 1
    rows = [(b % 3, b % 5 + 2, (1.01, 1.02, 0.99, 1.0)[b % 4]) for b in range(B)] if B > 1 else [(1, 0, 1.01)]
    eng[1].set_length_control(rows)
    sps = [e.sampling(eos, min_new_tokens=0, max_new_tokens=steps + 1, forced=forced) for e in eng]
    lgs = [e.prefill(prompts, sp, return_logits=True) for e, sp in zip(eng, sps)]
    moved = 0
    for s in range(steps + 1):
        off, on = (x.cpu().numpy() for x in lgs)
        for b in range(B):
            want = hf_chain(off[b], prompts[b], forced[b, :s].tolist(), s, 1.0, rows[b][1:], eos)
            assert bits_equal(on[b], want), (B, s, b)
            moved += not bits_equal(want[eos], off[b][eos])
        if s < steps:
            lgs = [e.decode(1, sp, return_logits=True)[0] for e, sp in zip(eng, sps)]
    assert torch.equal(eng[1].out_tokens[:B, : steps + 1].cpu(), forced.int())
    assert moved > 0
    print(f"LENGTH full size B={B}: {steps} teacher-forced steps bit-identical to transformers' processor ({moved} decayed)")
