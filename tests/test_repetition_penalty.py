"""CPU: the repetition penalty -- its fp32 / float64 semantics, validation and host plumbing.

* ``penalized`` (fp32, the kernels' arithmetic) is bit-identical to transformers' RepetitionPenaltyLogitsProcessor on
  the same fp32 logits, with and without ``prompt_ignore_length``, for penalties below and above 1, negative and zero
  logits and repeated ids; the whole chain (penalty -> EOS mask -> suppression -> 1/T -> top-k -> top-p -> min-p)
  keeps the ids and probabilities of transformers' processors and warpers applied in that order.
* ``check_penalty`` / ``per_prompt_penalty`` mirror ``nt_lm_set_repetition_penalty``'s rules.
* Stub engines: a default call never touches the table, a table is written before the first prefill, a left-over
  table is switched off, and ``generate_queue`` writes a newcomer's entry before its refill.
* The facade forwards the (repetition_penalty, penalize_prompt) pair only when it differs from the defaults.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import check_penalty, per_prompt_penalty
from tests.fakes import EOS, FakeTokenizer, GenerateBackbone, KwBackbone, QueueStub, _facade, _prompts
from tests.sampler_ref import chain64, suppressed_scores


def history(prompt, generated, include_prompt: bool = True):
    """The distinct ids a slot's penalty applies to."""
    ids = (list(prompt) if include_prompt else []) + list(generated)
    return np.unique(np.asarray(ids, dtype=np.int64))


def penalized(logits, hist, penalty: float):
    """fp32 logits with every id in ``hist`` penalised once: s < 0 ? s * p : s / p, p and the result in fp32 (an IEEE
    division, as torch's fp32 ``score / penalty``)."""
    s = np.asarray(logits, dtype=np.float32).copy()
    p = np.float32(penalty)
    h = np.asarray(hist, dtype=np.int64)
    v = s[h]
    s[h] = np.where(v < 0, v * p, v / p).astype(np.float32)
    return s


def test_penalty_chain_matches_transformers():
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
                                                        RepetitionPenaltyLogitsProcessor, SuppressTokensLogitsProcessor,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)

    rng = np.random.default_rng(5)
    checked = below = ignored = 0
    for case in range(260):
        V = 1024
        lo = 128 * int(rng.integers(0, 4)) if case % 2 else 0
        hi = min(V, lo + 128 * int(rng.integers(2, 8))) if case % 2 else V
        eos = int(rng.integers(lo, hi)) if case % 4 == 1 else int(rng.integers(0, V))
        pen = float(np.float32(rng.choice([0.5, 0.8, 0.95, 1.1, 1.3, 2.0, 3.7])))
        T = float(rng.choice([0.5, 0.7, 1.0, 1.5]))
        k = int(rng.choice([1, 20, 50, 64]))
        top_p = float(rng.choice([1.0, 0.9, 0.6]))
        min_p = float(rng.choice([0.0, 0.05, 0.2]))
        ngen, min_new = int(rng.integers(0, 5)), 2
        logits = rng.normal(0.0, 2.0, V).astype(np.float32)
        logits[rng.choice(V, 40, replace=False)] = 0.0                   # zero logits: divided, stay +0
        plen = int(rng.integers(1, 30))
        prompt = rng.integers(lo, hi, plen)
        prompt[: plen // 3] = prompt[plen // 3: 2 * (plen // 3)]       # repeated ids
        gen = rng.integers(lo, hi, ngen)
        if ngen:
            gen[-1] = prompt[0]                                         # a generated id that is also in the prompt
        include = bool(case % 3)
        ids_in = np.concatenate((prompt, gen)).astype(np.int64)
        # the processor alone, on fp32 logits: bit-identical
        x = torch.from_numpy(logits.copy())[None]
        proc = RepetitionPenaltyLogitsProcessor(pen, prompt_ignore_length=None if include else plen)
        want = proc(torch.from_numpy(ids_in)[None], x)[0].numpy()
        got = penalized(logits, history(prompt, gen, include), pen)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), case
        # the whole chain
        ids, p, margin = chain64(suppressed_scores(got, lo, hi, eos, ngen, min_new, T), k, top_p, min_p)
        if margin < 1e-6:
            continue
        inp = torch.from_numpy(ids_in)[None]
        y = torch.from_numpy(want.astype(np.float64))[None]
        y = MinNewTokensLengthLogitsProcessor(plen, min_new, eos, device="cpu")(inp, y)
        if hi - lo < V:
            y = SuppressTokensLogitsProcessor([i for i in range(V) if not (lo <= i < hi or i == eos)], device="cpu")(inp, y)
        y = TemperatureLogitsWarper(T)(inp, y)
        y = TopKLogitsWarper(k)(inp, y)
        if top_p < 1:
            y = TopPLogitsWarper(top_p)(inp, y)
        if min_p > 0:
            y = MinPLogitsWarper(min_p)(inp, y)
        q = torch.softmax(y[0], -1).numpy()
        assert sorted(ids.tolist()) == np.nonzero(q > 0)[0].tolist(), case
        assert np.abs(q[ids] - p).max() < 1e-6, case
        checked += 1
        below += pen < 1
        ignored += not include
    assert checked >= 200 and below >= 40 and ignored >= 40, (checked, below, ignored)


def test_penalty_edge_values():
    s = np.array([-np.inf, -2.0, -0.0, 0.0, 3.0, 1e-40], dtype=np.float32)
    got = penalized(s, np.arange(6), 1.3)
    assert got[0] == -np.inf and got[1] == np.float32(-2.0) * np.float32(1.3) and got[4] == np.float32(3.0) / np.float32(1.3)
    assert got[3] == 0.0 and np.signbit(got[2]) and not np.signbit(got[3])
    assert np.array_equal(penalized(s, np.arange(6), 1.0), s)          # 1 changes nothing, bit for bit
    # the reciprocal product would differ from the division on a share of the logits
    x = np.random.default_rng(1).normal(0, 4, 4096).astype(np.float32)
    x = x[x > 0]
    assert (x / np.float32(1.3) != x * (np.float32(1.0) / np.float32(1.3))).any()


@pytest.mark.parametrize("pen,ok", [(1.0, True), (1.3, True), (0.5, True), (2, True), (0.0, False), (-1.2, False),
                                    (float("nan"), False), (float("inf"), False), (1e-50, False), (1e39, False),
                                    (True, False), ("1.2", False)])
def test_check_penalty(pen, ok):
    if ok:
        assert check_penalty(pen) == (float(pen), True)
        assert check_penalty(pen, False) == (float(pen), False)
    else:
        with pytest.raises(ValueError):
            check_penalty(pen)


def test_per_prompt_penalty():
    assert per_prompt_penalty(3, 1.0, True) is None
    assert per_prompt_penalty(3, 1.0, False) is None
    assert per_prompt_penalty(2, [1.0, 1.0], [True, False]) is None
    assert per_prompt_penalty(2, 1.2, True) == [(1.2, True), (1.2, True)]
    assert per_prompt_penalty(2, [1.0, 1.3], False) == [(1.0, False), (1.3, False)]
    assert per_prompt_penalty(2, np.array([1.1, 0.9]), [1, 0]) == [(float(np.float64(1.1)), True), (0.9, False)]
    for pen, inc in (([1.0, 1.3, 1.2], True), (1.2, [True]), ([0.0, 1.2], True), (1.2, "yes"), ([1.2, float("nan")], True)):
        with pytest.raises(ValueError):
            per_prompt_penalty(2, pen, inc)


# ---------------------------------------------------------------------------------------- stub engines
class PenStub(QueueStub):
    """QueueStub that also logs the penalty table calls."""

    def set_repetition_penalty(self, rows, slots=None):
        self.log.append(("penalty", None if rows is None else [tuple(r) for r in rows], None if slots is None else list(slots)))
        self._penalty_host = rows


LENS = [5, 6, 7, 8, 9]


def test_default_calls_make_no_engine_call():
    a = QueueStub(2)
    a.generate_queue(_prompts(LENS), EOS, max_new_tokens=[3, 4, 2, 5, 3], min_new_tokens=1)
    for kw in ({}, dict(repetition_penalty=1.0), dict(repetition_penalty=1.0, penalize_prompt=False),
               dict(repetition_penalty=[1.0] * 5)):
        b = PenStub(2)
        b.generate_queue(_prompts(LENS), EOS, max_new_tokens=[3, 4, 2, 5, 3], min_new_tokens=1, **kw)
        assert b.log == a.log, kw


def test_queue_writes_entries_before_prefills_and_switches_off():
    pens = [1.1, 1.2, 1.3, 1.4, 1.5]
    incl = [True, False, True, False, True]
    st = PenStub(2)
    st.generate_queue(_prompts(LENS), EOS, max_new_tokens=[3, 4, 2, 5, 3], min_new_tokens=1, repetition_penalty=pens,
                      penalize_prompt=incl)
    rows = list(zip(pens, incl))
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("penalty")] == ("penalty", rows[:2], None)
    assert kinds.index("penalty") < kinds.index("prefill")
    refills = [i for i, e in enumerate(st.log) if e[0] == "refill"]
    assert refills
    for i in refills:
        slots, tags = st.log[i][1], st.log[i][2]
        assert st.log[i - 1] == ("penalty", [rows[t - 1] for t in tags], slots)
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # the left-over table goes off
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("penalty")] == ("penalty", None, None) and kinds.index("penalty") < kinds.index("prefill")
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # off stays off without a call
    assert "penalty" not in [e[0] for e in st.log]
    st.log.clear()
    with pytest.raises(ValueError):
        st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, repetition_penalty=[1.2, 0.0])
    with pytest.raises(ValueError):
        st.generate_queue(_prompts(LENS), EOS, max_new_tokens=3, repetition_penalty=[1.2] * 4)
    assert st.log == []


def test_generate_seam_takes_transformers_keyword():
    st = PenStub(1)
    seen = {}
    st.generate_batch = lambda prompts, eos, *a, **kw: seen.update(kw) or [torch.tensor([EOS])]
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1, repetition_penalty=1.25)
    assert seen["repetition_penalty"] == 1.25 and "penalize_prompt" not in seen   # prompt included, as transformers
    seen.clear()
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1, repetition_penalty=1.0)
    assert "repetition_penalty" not in seen


# ---------------------------------------------------------------------------------------- facade
def _pen(kw):
    return {k: kw[k] for k in ("repetition_penalty", "penalize_prompt") if k in kw}


def test_facade_forwards_the_pair_only_when_it_differs():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    tts = _facade(bb, 3)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_penalty=1.0, penalize_prompt=True)
    assert [_pen(c[2]) for c in bb.calls] == [{}, {}]
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_penalty=[1.0, 1.3])
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, penalize_prompt=False, repetition_penalty=1.2)
    assert _pen(bb.calls[2][2]) == dict(repetition_penalty=[1.0, 1.3], penalize_prompt=True)
    assert _pen(bb.calls[3][2]) == dict(repetition_penalty=1.2, penalize_prompt=False)
    # a backbone whose generate has no such keyword keeps working with the defaults
    gb = GenerateBackbone(tok)
    tts = _facade(gb, 1)
    tts.infer("a b", [1, 2], "r")
    tts.infer("a b", [1, 2], "r", repetition_penalty=1.0)
    assert all(not _pen(k) for k in gb.kws)

    class NoKw:
        device = torch.device("cpu")

        def generate(self, ids, max_length, eos_token_id, do_sample, use_cache, min_new_tokens, temperature, top_k):
            return torch.cat((ids, torch.tensor([[tok.speech_base + 2]])), dim=1)

    nk = NoKw()
    nk.tok = tok
    _facade(nk, 1).infer("a b", [1, 2], "r", repetition_penalty=1.0, penalize_prompt=True)


def test_facade_lists_follow_their_utterances():
    tok = FakeTokenizer()
    pens = [1.0 + 0.1 * i for i in range(7)]
    bb = KwBackbone(tok, queue=False)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, repetition_penalty=pens, penalize_prompt=False)
    assert [(c[2]["slot_base"], c[2]["repetition_penalty"], c[2]["penalize_prompt"]) for c in bb.calls] == [
        (0, pens[0:3], False), (3, pens[3:6], False), (6, pens[6:], False)]
    bb = KwBackbone(tok)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, repetition_penalty=pens)
    assert len(bb.calls) == 1 and bb.calls[0][0] == "queue" and bb.calls[0][2]["repetition_penalty"] == pens
    with pytest.raises(ValueError, match="one value per utterance"):
        _facade(bb, 3).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_penalty=[1.2])
    with pytest.raises(ValueError, match="one value per utterance"):
        _facade(bb, 3).infer_stream_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, penalize_prompt=[True])
