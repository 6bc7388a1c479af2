"""CPU: per-slot length control (min_new_tokens and the exponential decay length penalty).

* The engine's EOS arithmetic -- fp32 c_k = (float)(pow(factor, k) - 1) formed in double, then s + |s| * c_k as an fp32
  product and an fp32 sum -- is bit-identical to transformers' ``ExponentialDecayLengthPenalty``, for negative, zero
  and positive EOS logits, factors below and above 1, and k from 1 to max_new - start.
* The whole chain (penalty -> min-new-tokens mask -> decay -> suppression -> 1/T -> top-k -> top-p -> min-p) keeps the
  ids transformers' processors and warpers keep, on 200+ seeded cases.
* ``check_length`` / ``per_prompt_length`` refuse what ``nt_lm_set_length_control`` and the launches refuse.
* Entries follow utterances through the queue, forks and the streaming queue, and the facade's defaults pass the
  backbone exactly the keyword arguments it had before.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import Settings, check_length, per_prompt_length, resolve_settings
from tests.fakes import EOS, FakeTokenizer, GenerateBackbone, KwBackbone, QueueStub, _facade, _prompts
from tests.sampler_ref import chain64, suppressed_scores


def decayed(s: np.float32, start: int, factor: float, n: int) -> np.float32:
    """The engine's EOS score after the decay at n generated tokens."""
    if n <= start or factor == 1.0:
        return np.float32(s)
    c = np.float32(pow(factor, n - start) - 1)
    with np.errstate(over="ignore"):
        return np.float32(np.float32(s) + np.float32(np.abs(np.float32(s)) * c))


def hf_decay(row, eos, start, factor, plen, n):
    from transformers.generation.logits_process import ExponentialDecayLengthPenalty

    ids = torch.zeros(1, plen + n, dtype=torch.long)
    return ExponentialDecayLengthPenalty((start, factor), eos, plen)(ids, torch.from_numpy(row.copy())[None])[0].numpy()


def test_eos_arithmetic_is_bit_identical():
    rng = np.random.default_rng(3)
    eos, V, checked = 7, 16, 0
    for factor in (0.3, 0.8, 0.97, 1.0001, 1.05, 1.3, 2.5, 10.0):
        for start, max_new in ((0, 30), (4, 40), (17, 64)):
            for s in (-31.7, -2.5, -1e-3, -0.0, 0.0, 1e-3, 0.75, 4.25, 15.0, float(rng.normal(0, 5))):
                for n in sorted({start + 1, start + 2, (start + max_new) // 2, max_new - 1, max_new}):
                    row = rng.normal(0, 3, V).astype(np.float32)
                    row[eos] = np.float32(s)
                    with np.errstate(over="ignore"):
                        c = np.float32(pow(factor, max(n - start, 0)) - 1)
                    if not np.isfinite(c):
                        continue
                    want = hf_decay(row, eos, start, factor, 5, n)
                    got = decayed(row[eos], start, factor, n)
                    assert np.float32(got).view(np.uint32) == want[eos].view(np.uint32), (factor, start, s, n)
                    others = np.arange(V) != eos
                    # transformers adds 0 to every other id, which turns a -0.0 into +0.0; the engine leaves them alone
                    assert np.array_equal(want[others], row[others])
                    checked += 1
    assert checked > 1000


def test_fp32_scalar_product_not_double():
    """transformers multiplies the fp32 |s| by the Python float c_k: torch rounds c_k to fp32 first."""
    x = torch.from_numpy(np.random.default_rng(0).normal(0, 10, 50000).astype(np.float32))
    c = pow(1.37, 21) - 1
    got = (torch.abs(x) * c).numpy()
    assert np.array_equal(got, np.abs(x.numpy()) * np.float32(c))
    assert not np.array_equal(got, (np.abs(x.numpy()).astype(np.float64) * c).astype(np.float32))


def test_length_chain_matches_transformers():
    from transformers.generation.logits_process import (ExponentialDecayLengthPenalty, MinNewTokensLengthLogitsProcessor,
                                                        MinPLogitsWarper, RepetitionPenaltyLogitsProcessor,
                                                        SuppressTokensLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)

    rng = np.random.default_rng(11)
    checked = decays = masked = 0
    for case in range(300):
        V = 1024
        lo = 128 * int(rng.integers(0, 4)) if case % 2 else 0
        hi = min(V, lo + 128 * int(rng.integers(2, 8))) if case % 2 else V
        eos = int(rng.integers(lo, hi)) if case % 4 == 1 else int(rng.integers(0, V))
        pen = float(np.float32(rng.choice([1.0, 0.8, 1.3])))
        T = float(rng.choice([0.5, 1.0, 1.5]))
        k = int(rng.choice([1, 20, 50, 64]))
        top_p = float(rng.choice([1.0, 0.9, 0.6]))
        min_p = float(rng.choice([0.0, 0.05, 0.2]))
        min_new = int(rng.integers(0, 4))
        start = min_new - 1 + int(rng.integers(0, 3)) if min_new else int(rng.integers(0, 3))
        factor = float(rng.choice([0.5, 0.9, 1.0, 1.2, 2.0, 4.0]))
        ngen = int(rng.integers(0, 9))
        logits = rng.normal(0.0, 2.0, V).astype(np.float32)
        logits[eos] = np.float32(rng.choice([-6.0, -1.5, 0.0, 1.0, 3.0]))
        plen = int(rng.integers(1, 20))
        prompt = rng.integers(lo, hi, plen)
        gen = rng.integers(lo, hi, ngen)
        inp = torch.from_numpy(np.concatenate((prompt, gen)).astype(np.int64))[None]
        y = torch.from_numpy(logits.copy())[None]
        if pen != 1.0:
            y = RepetitionPenaltyLogitsProcessor(pen)(inp, y)
        stored = y[0].numpy().copy()       # the engine's chain from here: decay on the stored row, mask in the sampler
        stored[eos] = decayed(stored[eos], start, factor, ngen)
        y = MinNewTokensLengthLogitsProcessor(plen, min_new, eos, device="cpu")(inp, y)
        y = ExponentialDecayLengthPenalty((start, factor), eos, plen)(inp, y)
        # processors: bit-identical, the mask's -inf included
        want = stored.copy()
        if ngen < min_new:
            want[eos] = -np.inf
        assert np.array_equal(y[0].numpy().view(np.uint32), want.view(np.uint32)), case
        ids, p, margin = chain64(suppressed_scores(stored, lo, hi, eos, ngen, min_new, T), k, top_p, min_p)
        if margin < 1e-6:
            continue
        y = y.double()
        if hi - lo < V:
            y = SuppressTokensLogitsProcessor([i for i in range(V) if not (lo <= i < hi or i == eos)], device="cpu")(inp, y)
        y = TemperatureLogitsWarper(T)(inp, y)
        y = TopKLogitsWarper(k)(inp, y)
        if top_p < 1:
            y = TopPLogitsWarper(top_p)(inp, y)
        if min_p > 0:
            y = MinPLogitsWarper(min_p)(inp, y)
        q = torch.softmax(y[0], -1).numpy()
        # a decayed EOS can dwarf the rest of the window: ids whose float64 probability underflows count as dropped
        assert sorted(ids[p > 0].tolist()) == np.nonzero(q > 0)[0].tolist(), case
        assert np.abs(q[ids] - p).max() < 1e-6, case
        checked += 1
        decays += ngen > start and factor != 1.0
        masked += ngen < min_new
    assert checked >= 200 and decays >= 50 and masked >= 30, (checked, decays, masked)


@pytest.mark.parametrize("row,max_new,ok", [
    ((0, 0, 1.0), None, True), ((50, 49, 1.0), None, True), ((3, 10, 0.5), 64, True), ((3, 2, 1.2), 64, True),
    ((-1, 0, 1.0), None, False),                      # min_new_tokens < 0
    ((3, 5, 0.0), None, False), ((3, 5, -1.1), None, False), ((3, 5, math.inf), None, False), ((3, 5, math.nan), None, False),
    ((3, -1, 1.2), None, False),                      # start < 0
    ((5, 3, 1.2), None, False),                       # start < min_new_tokens - 1: -inf + inf
    ((0, 0, 10.0), 38, True), ((0, 0, 10.0), 39, False), ((0, 10, 10.0), 48, True), ((0, 10, 10.0), 49, False),
    ((0, 0, 1e300), 64, False),                       # pow overflows double
    ((2.5, 3, 1.2), None, False), ((True, 3, 1.2), None, False), ((2, 3.0, 1.2), None, False), ((2, 3, "1.2"), None, False),
])
def test_check_length(row, max_new, ok):
    if ok:
        assert check_length(*row, max_new=max_new) == (int(row[0]), int(row[1]), float(row[2]))
    else:
        with pytest.raises(ValueError):
            check_length(*row, max_new=max_new)


def test_per_prompt_length():
    assert per_prompt_length(3, 50, None) is None
    assert per_prompt_length(3, 0, None) is None
    assert per_prompt_length(2, [5, 0], None) == [(5, 4, 1.0), (0, 0, 1.0)]
    assert per_prompt_length(2, 3, (10, 1.5)) == [(3, 10, 1.5), (3, 10, 1.5)]
    assert per_prompt_length(2, np.array([1, 2]), [(4, 1.1), None]) == [(1, 4, 1.1), (2, 1, 1.0)]
    for mn, d in (([1, 2, 3], None), (-1, None), (5, (2, 1.5)), (3, [(4, 1.1)]), (3, (4, 0.0)), (3, "x"), (3, [(4, 1.1), 7])):
        with pytest.raises(ValueError):
            per_prompt_length(2, mn, d)
    with pytest.raises(ValueError, match="overflows"):
        per_prompt_length(1, 0, (0, 10.0), max_new=100)


# ---------------------------------------------------------------------------------------- stub engines
class LenStub(QueueStub):
    """QueueStub that logs the length-control table calls and the launch floor."""

    def set_length_control(self, rows, slots=None):
        self.log.append(("length", None if rows is None else [tuple(r) for r in rows], None if slots is None else list(slots)))
        self._length_host = rows

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, limits=None, slot_base=0):
        self.floor = min_new
        return super().sampling(eos, min_new, max_new, top_k, temperature, seed, greedy, limits, slot_base)


LENS = [5, 6, 7, 8, 9]
CAPS = [3, 4, 2, 5, 3]


def test_defaults_make_no_engine_call():
    a = QueueStub(2)
    a.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=1)
    for kw in ({}, dict(exponential_decay_length_penalty=None), dict(exponential_decay_length_penalty=[None] * 5)):
        b = LenStub(2)
        b.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=1, **kw)
        assert b.log == a.log and b.floor == 1, kw


def test_queue_writes_entries_before_prefills_and_switches_off():
    floors = [1, 0, 2, 1, 0]
    decay = [(2, 1.5), None, (3, 0.9), None, (0, 1.1)]
    st = LenStub(2)
    st.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=floors,
                      exponential_decay_length_penalty=decay)
    rows = [(1, 2, 1.5), (0, 0, 1.0), (2, 3, 0.9), (1, 0, 1.0), (0, 0, 1.1)]
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("length")] == ("length", rows[:2], None)
    assert kinds.index("length") < kinds.index("prefill") and st.floor == 1   # the launch floor: row 0's
    refills = [i for i, e in enumerate(st.log) if e[0] == "refill"]
    assert refills
    for i in refills:
        slots, tags = st.log[i][1], st.log[i][2]
        assert st.log[i - 1] == ("length", [rows[t - 1] for t in tags], slots)
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # the left-over table goes off
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("length")] == ("length", None, None) and kinds.index("length") < kinds.index("prefill")
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # off stays off without a call
    assert "length" not in [e[0] for e in st.log]
    st.log.clear()
    for bad in (dict(min_new_tokens=[1, -1]), dict(min_new_tokens=[1, 2, 3]), dict(exponential_decay_length_penalty=(0, 1.5),
                                                                                    min_new_tokens=4)):
        with pytest.raises(ValueError):
            st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, **bad)
    assert st.log == []


def test_a_queue_floor_of_zero_reads_before_decoding():
    """A newcomer whose floor is 0 may end inside its prefill: the queue reads the state before decoding it."""
    st = LenStub(2, eos_at={3: 0})
    out = st.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=[1, 1, 0, 1, 1])
    assert out[2].tolist() == [EOS]


def test_forks_and_settings_repeat():
    s = resolve_settings(None, 2, min_new_tokens=[3, 6], exponential_decay_length_penalty=[(4, 1.2), None])
    r = s.repeat(3)
    assert r.length == [(3, 4, 1.2)] * 3 + [(6, 5, 1.0)] * 3 and r.min_new_tokens == 3
    assert r.floors(6) == [3, 3, 3, 6, 6, 6]
    off = Settings(None, None, None, 1.0, 50).repeat(4)
    assert off.length is None and off.floors(4) == [50] * 4


def test_generate_seam_takes_transformers_keyword():
    st = LenStub(1)
    seen = {}
    st.generate_batch = lambda prompts, eos, *a, **kw: seen.update(kw) or [torch.tensor([EOS])]
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1, exponential_decay_length_penalty=[4, 1.3])
    assert seen["exponential_decay_length_penalty"] == (4, 1.3)
    seen.clear()
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1)
    assert "exponential_decay_length_penalty" not in seen


# ---------------------------------------------------------------------------------------- facade
def _len(kw):
    return {k: kw[k] for k in ("min_new_tokens", "exponential_decay_length_penalty") if k in kw}


def test_facade_defaults_pass_the_same_kwargs():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    tts = _facade(bb, 3)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, min_new_tokens=50, exponential_decay_length_penalty=None)
    assert [_len(c[2]) for c in bb.calls] == [dict(min_new_tokens=50)] * 2
    gb = GenerateBackbone(tok)
    tts = _facade(gb, 1)
    tts.infer("a b", [1, 2], "r")
    assert _len(gb.kws[0]) == dict(min_new_tokens=50)
    tts.infer("a b", [1, 2], "r", min_new_tokens=7, exponential_decay_length_penalty=(20, 1.05))
    assert _len(gb.kws[1]) == dict(min_new_tokens=7, exponential_decay_length_penalty=(20, 1.05))

    class NoKw:   # a backbone without the decay keyword keeps working with the defaults
        device = torch.device("cpu")

        def generate(self, ids, max_length, eos_token_id, do_sample, use_cache, min_new_tokens, temperature, top_k):
            return torch.cat((ids, torch.tensor([[tok.speech_base + 2]])), dim=1)

    nk = NoKw()
    nk.tok = tok
    _facade(nk, 1).infer("a b", [1, 2], "r")
    # a per-utterance list without any pair asks for no decay: nothing is forwarded, to any backbone
    _facade(nk, 2).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, exponential_decay_length_penalty=[None, None])
    bb = KwBackbone(tok, queue=False)
    _facade(bb, 2).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, exponential_decay_length_penalty=[None, None])
    assert _len(bb.calls[0][2]) == dict(min_new_tokens=50)


def test_facade_lists_follow_their_utterances():
    tok = FakeTokenizer()
    floors = [10 + i for i in range(7)]
    decay = [None if i % 2 else (20 + i, 1.01 + 0.01 * i) for i in range(7)]
    bb = KwBackbone(tok, queue=False)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, min_new_tokens=floors,
                               exponential_decay_length_penalty=decay)
    assert [(c[2]["slot_base"], c[2]["min_new_tokens"], c[2]["exponential_decay_length_penalty"]) for c in bb.calls] == [
        (0, floors[0:3], decay[0:3]), (3, floors[3:6], decay[3:6]), (6, floors[6:], decay[6:])]
    bb = KwBackbone(tok)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, exponential_decay_length_penalty=(30, 1.1))
    assert len(bb.calls) == 1 and bb.calls[0][0] == "queue"
    assert _len(bb.calls[0][2]) == dict(min_new_tokens=50, exponential_decay_length_penalty=(30, 1.1))
    gb = GenerateBackbone(tok)   # one utterance at a time: each gets its own values
    _facade(gb, 3).infer_batch(["a b"] * 3, [[1, 2]] * 3, ["r"] * 3, min_new_tokens=[1, 2, 3],
                               exponential_decay_length_penalty=[(5, 1.1), None, (7, 1.2)])
    assert [_len(k) for k in gb.kws] == [dict(min_new_tokens=1, exponential_decay_length_penalty=(5, 1.1)),
                                         dict(min_new_tokens=2),
                                         dict(min_new_tokens=3, exponential_decay_length_penalty=(7, 1.2))]
    with pytest.raises(ValueError, match="one value per utterance"):
        _facade(bb, 3).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, min_new_tokens=[5])
    with pytest.raises(ValueError, match="exponential_decay_length_penalty"):
        _facade(bb, 3).infer_stream_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, exponential_decay_length_penalty=[(5, 1.1)])
