"""CPU: the vocabulary range (speech-token-only decoding) -- its float64 semantics, validation and host plumbing.

* The float64 chain with suppression (every id outside [lo, hi) + EOS -> -inf, then the chain of
  ``test_sampling_controls``) equals transformers' SuppressTokensLogitsProcessor, MinNewTokensLengthLogitsProcessor
  and the four warpers applied in order.
* ``check_vocab_range`` mirrors ``nt_lm_set_vocab_range``'s rules.
* Stub engines: a default call never touches the range, a range is set before the first prefill, a range left on is
  switched off, and ``generate_queue`` keeps the range across refills.
* The facade forwards ``vocab_range`` (engines) or ``suppress_tokens`` (transformers-style backbones) only while
  ``speech_tokens_only`` is on.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import check_vocab_range
from tests.test_gpu_sampler import processed_scores
from tests.test_host_logic import FakeTokenizer
from tests.test_queue_host import EOS, QueueStub, _prompts
from tests.test_sampling_controls import GenerateBackbone, KwBackbone, _facade, chain64


def suppressed_scores(logits, lo: int, hi: int, eos: int, ngen: int, min_new: int, temperature: float):
    s = np.asarray(logits, dtype=np.float32).copy()
    keep = np.zeros(s.size, dtype=bool)
    keep[lo:hi] = True
    keep[eos] = True
    s[~keep] = -np.inf
    return processed_scores(s, ngen, eos, min_new, temperature)


def test_suppression_chain_matches_transformers():
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
                                                        SuppressTokensLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)

    rng = np.random.default_rng(0)
    V = 1024
    checked = outside = 0
    for case in range(240):
        lo = 128 * int(rng.integers(0, 6))
        hi = min(V, lo + 128 * int(rng.integers(1, 3)))
        eos = int(rng.integers(0, V))
        T = float(rng.choice([0.5, 0.7, 1.0, 1.5]))
        k = int(rng.choice([1, 20, 50, 64]))
        top_p = float(rng.choice([1.0, 0.9, 0.6]))
        min_p = float(rng.choice([0.0, 0.05, 0.2]))
        ngen, min_new = int(rng.integers(0, 4)), 2
        logits = rng.normal(0.0, 2.0, V).astype(np.float32)
        if case % 3 == 0:   # adversarial: the unconstrained top 64 lie entirely outside the range
            out = np.setdiff1d(np.arange(V), np.arange(lo, hi))
            logits[rng.choice(out, 64, replace=False)] += 20.0
            outside += 1
        ids, p, margin = chain64(suppressed_scores(logits, lo, hi, eos, ngen, min_new, T), k, top_p, min_p)
        if margin < 1e-6:
            continue
        # transformers, in generate()'s order: processors, then the warpers
        x = torch.from_numpy(logits.astype(np.float64))[None]
        inp = torch.zeros(1, 5 + ngen, dtype=torch.long)
        suppress = [i for i in range(V) if not (lo <= i < hi or i == eos)]
        x = SuppressTokensLogitsProcessor(suppress, device="cpu")(inp, x)
        x = MinNewTokensLengthLogitsProcessor(5, min_new, eos, device="cpu")(inp, x)
        x = TemperatureLogitsWarper(T)(inp, x)
        x = TopKLogitsWarper(k)(inp, x)
        if top_p < 1:
            x = TopPLogitsWarper(top_p)(inp, x)
        if min_p > 0:
            x = MinPLogitsWarper(min_p)(inp, x)
        q = torch.softmax(x[0], -1).numpy()
        kept = np.nonzero(q > 0)[0]
        assert sorted(ids.tolist()) == kept.tolist(), case
        assert np.abs(q[ids] - p).max() < 1e-6, case   # fp32 1 / T product against the float64 division
        assert all(lo <= i < hi or i == eos for i in ids)
        checked += 1
    assert checked >= 200 and outside >= 60, (checked, outside)


@pytest.mark.parametrize("lo,hi,ok", [(151936, 217472, True), (0, 217472, True), (0, 128, True), (128, 192, False), (128, 256, True),
                                      (217344, 217472, True), (151936, 217400, False), (100, 1024, False),
                                      (128, 191, False), (256, 128, False), (0, 217474, False), (-128, 256, False),
                                      (1.5, 256, False)])
def test_validation_mirrors_the_library(lo, hi, ok):
    if ok:
        assert check_vocab_range((lo, hi), 217472) == (lo, hi)
    else:
        with pytest.raises(ValueError):
            check_vocab_range((lo, hi), 217472)
    assert check_vocab_range(None, 217472) is None


class RangeStub(QueueStub):
    """QueueStub that also logs the vocabulary range calls."""

    def set_vocab_range(self, lo, hi=None):
        self.log.append(("range", None if lo is None else (lo, hi)))
        self._vocab_range = None if lo is None else (lo, hi)


RNG = (128, 1024)


def _stub(max_batch):
    st = RangeStub(max_batch)
    st.shape = type("S", (), {"vocab_size": 1024})()
    return st


def test_default_calls_log_exactly_what_they_did():
    a, b = QueueStub(2), _stub(2)
    for st in (a, b):
        st.generate_queue(_prompts([5, 6, 7]), EOS, max_new_tokens=[3, 4, 2], min_new_tokens=1)
        st.generate_queue(_prompts([5, 6]), EOS, max_new_tokens=[3, 3], min_new_tokens=1)
    assert a.log == b.log


def test_range_before_first_prefill_kept_across_refills_and_switched_off():
    st = _stub(2)
    st.generate_queue(_prompts([5, 6, 7, 8]), EOS, max_new_tokens=[3, 4, 2, 5], min_new_tokens=1, vocab_range=RNG)
    kinds = [e[0] for e in st.log]
    assert kinds.index("range") < kinds.index("prefill")
    assert [e for e in st.log if e[0] == "range"] == [("range", RNG)] and "refill" in kinds
    st.log.clear()
    st.generate_queue(_prompts([5, 6]), EOS, max_new_tokens=[3, 3], min_new_tokens=1)   # the left-over range goes off
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("range")] == ("range", None) and kinds.index("range") < kinds.index("prefill")
    st.log.clear()
    st.generate_queue(_prompts([5, 6]), EOS, max_new_tokens=[3, 3], min_new_tokens=1)   # off stays off without a call
    assert "range" not in [e[0] for e in st.log]
    with pytest.raises(ValueError):
        st.generate_queue(_prompts([5, 6]), EOS, max_new_tokens=[3, 3], vocab_range=(100, 1024))
    assert "range" not in [e[0] for e in st.log]


def test_facade_forwards_the_speech_range_only_when_on():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    _facade(bb, 3).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    assert "vocab_range" not in bb.calls[0][2]
    tts = _facade(bb, 3)
    tts.speech_tokens_only = True
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    assert bb.calls[1][2]["vocab_range"] == (tok.speech_base, tok.speech_base + 4 ** 8)
    qb = KwBackbone(tok, queue=True)
    tts = _facade(qb, 1)
    tts.speech_tokens_only = True
    tts.infer_batch(["a b"] * 3, [[1, 2]] * 3, ["r"] * 3)
    assert qb.calls[0][0] == "queue" and qb.calls[0][2]["vocab_range"] == (tok.speech_base, tok.speech_base + 4 ** 8)

    class HFBackbone(GenerateBackbone):
        config = type("C", (), {"vocab_size": tok.speech_base + 4 ** 8})()

    gb = HFBackbone(tok)
    _facade(gb, 1).infer("a b", [1, 2], "r")
    assert "suppress_tokens" not in gb.kws[0] and "vocab_range" not in gb.kws[0]
    tts = _facade(gb, 1)
    tts.speech_tokens_only = True
    tts.infer("a b", [1, 2], "r")
    sup = set(gb.kws[1]["suppress_tokens"])
    eos = tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>")
    assert eos not in sup and tok.speech_base not in sup and tok.speech_base - 1 in sup
    assert len(sup) == tok.speech_base - (1 if eos < tok.speech_base else 0)


def test_constructor_keyword_is_kept():
    from neutts import NeuTTS
    import inspect

    p = inspect.signature(NeuTTS.__init__).parameters["speech_tokens_only"]
    assert p.kind == p.KEYWORD_ONLY and p.default is False


def test_set_vocab_range_needs_both_bounds():
    from neutts_air_b200.lm import SpeechLM

    st = _stub(2)
    with pytest.raises(ValueError):
        SpeechLM.set_vocab_range(st, 128)
    with pytest.raises(ValueError):
        SpeechLM.set_vocab_range(st, 128, None)
    with pytest.raises(ValueError):
        check_vocab_range((128, None), 1024)
