"""CPU: the definition of the per-token log-probabilities against live transformers, argument validation, the queue's
harvest of a finished slot's rows, and the facade's plumbing on stub engines."""
import math
import types

import numpy as np
import pytest
import torch
from transformers import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
                          RepetitionPenaltyLogitsProcessor, SuppressTokensLogitsProcessor, TemperatureLogitsWarper,
                          TopKLogitsWarper, TopPLogitsWarper)
from transformers.generation.utils import GenerationMixin

from tests.fakes import EOS, FakeCodec, FakePhonemizer, FakeTokenizer, QueueStub, _prompts


# ----------------------------------------------------------------------------------------- float64 reference
def ref_logprobs(logits, hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p, tok, greedy):
    """(sampled, model) of ``tok`` in float64: penalty -> EOS mask -> range, then model = log-softmax over the whole
    vocabulary; sampled = log-probability in the kept window (1/T, the top_k best by (score desc, id asc), top-p keeps
    entry j iff the mass before it is < top_p, min-p keeps q_j >= min_p q_0), or model for greedy runs."""
    s = np.asarray(logits, dtype=np.float64).copy()
    for i in set(hist):
        s[i] = s[i] * penalty if s[i] < 0 else s[i] / penalty
    if masked:
        s[eos] = -np.inf
    if allowed is not None:
        keep = np.zeros(s.size, dtype=bool)
        keep[allowed] = True
        s[~keep] = -np.inf
    lse = lambda x: x.max() + np.log(np.exp(x - x.max()).sum())
    model = s[tok] - lse(s)
    if greedy:
        return model, model
    p = s / T
    order = np.lexsort((np.arange(p.size), -p))[: min(top_k, 64)]
    sc = p[order]
    q = np.exp(sc - lse(sc))
    before = np.concatenate(([0.0], np.cumsum(q)[:-1]))
    cut = (before < top_p) & (q >= min_p * q[0])
    k = int(np.argmin(cut)) if not cut.all() else cut.size
    k = max(k, 1)
    win = order[:k]
    if tok not in win:
        return -math.inf, model
    w = sc[:k]
    return float(w[list(win).index(tok)] - lse(w)), float(model)


def hf_logprobs(logits, prompt, hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p, tok, greedy, V):
    """transformers' processors (and, sampling, its warpers) on float64 scores; ``sampled`` through
    compute_transition_scores(normalize_logits=True), ``model`` as log_softmax of the processors' output."""
    ids = torch.tensor([prompt + hist])
    procs = LogitsProcessorList([RepetitionPenaltyLogitsProcessor(penalty)])
    if masked:
        procs.append(MinNewTokensLengthLogitsProcessor(len(prompt), len(hist) + 1, eos))
    if allowed is not None:
        procs.append(SuppressTokensLogitsProcessor([i for i in range(V) if i not in set(allowed)]))
    x = procs(ids, torch.tensor(np.asarray(logits, dtype=np.float64))[None].clone())
    model = torch.log_softmax(x, -1)[0, tok].item()
    if not greedy:
        warp = LogitsProcessorList([TemperatureLogitsWarper(T), TopKLogitsWarper(top_k), TopPLogitsWarper(top_p)])
        if min_p > 0:
            warp.append(MinPLogitsWarper(min_p))
        x = warp(ids, x)
    fake = types.SimpleNamespace(config=types.SimpleNamespace(get_text_config=lambda: types.SimpleNamespace(vocab_size=V)))
    seq = torch.tensor([prompt + hist + [tok]])
    sampled = GenerationMixin.compute_transition_scores(fake, seq, (x,), normalize_logits=True)[0, 0].item()
    return sampled, model


def _near_cut(logits, hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p) -> bool:
    """True when the case sits within 1e-6 of a top-p or min-p cut (float rounding may then keep another prefix)."""
    s = np.asarray(logits, dtype=np.float64).copy()
    for i in set(hist):
        s[i] = s[i] * penalty if s[i] < 0 else s[i] / penalty
    if masked:
        s[eos] = -np.inf
    if allowed is not None:
        keep = np.zeros(s.size, dtype=bool)
        keep[allowed] = True
        s[~keep] = -np.inf
    sc = np.sort(s / T)[::-1][: min(top_k, 64)]
    q = np.exp(sc - sc.max())
    q /= q.sum()
    before = np.concatenate(([0.0], np.cumsum(q)[:-1]))
    return bool((np.abs(before - top_p) < 1e-6).any() or (np.abs(q - min_p * q[0]) < 1e-6).any())


def test_reference_matches_transformers():
    rng = np.random.default_rng(11)
    V, eos, n, dropped = 700, 650, 0, 0
    while n < 240:
        logits = rng.normal(0, 2.5, V)
        logits[eos] = rng.normal(3, 1)
        prompt = rng.integers(0, V, 6).tolist()
        hist = rng.integers(0, V, int(rng.integers(0, 8))).tolist()
        penalty = float(rng.choice([1.0, 1.3, 0.8]))
        masked = bool(rng.integers(2))
        allowed = None if rng.integers(3) else list(range(128, 512)) + [eos]
        T = float(rng.choice([1.0, 0.7, 1.4]))
        top_k, top_p, min_p = int(rng.choice([1, 20, 50, 64])), float(rng.choice([1.0, 0.9, 0.6])), float(rng.choice([0.0, 0.05]))
        greedy = n % 7 == 0
        if not greedy and _near_cut(logits, prompt + hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p):
            dropped += 1
            continue
        cand = [i for i in range(V) if not (masked and i == eos) and (allowed is None or i in allowed)]
        tok = int(rng.choice(cand)) if n % 3 else int(np.argmax(logits if allowed is None else
                                                               np.where(np.isin(np.arange(V), cand), logits, -np.inf)))
        want = ref_logprobs(logits, prompt + hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p, tok, greedy)
        got = hf_logprobs(logits, prompt, hist, penalty, eos, masked, allowed, T, top_k, top_p, min_p, tok, greedy, V)
        assert abs(got[1] - want[1]) < 1e-9, (n, got, want)
        if want[0] == -math.inf:
            assert got[0] == -math.inf, (n, got, want)
        else:
            assert abs(got[0] - want[0]) < 1e-9, (n, got, want)
        n += 1
    assert dropped < n // 4


# ----------------------------------------------------------------------------------------- validation
def test_abi_rejects_null_handle():
    from neutts_air_b200 import _lib, build

    build.build()
    L = _lib.lib()
    assert L.nt_lm_set_logprobs(None, None, None) == -1 and b"null handle" in L.nt_last_error()


def test_settings_apply_switches_logprobs():
    from neutts_air_b200.lm import resolve_settings

    calls = []
    lm = types.SimpleNamespace(logprobs=None, set_logprobs=lambda on: calls.append(on))
    resolve_settings(lm, 2).apply(lm, 2)                       # off and off: no call
    resolve_settings(lm, 2, logprobs=True).apply(lm, 2)
    lm.logprobs = object()
    resolve_settings(lm, 2, logprobs=True).apply(lm, 2)        # on and on: no call
    resolve_settings(lm, 2).apply(lm, 2)
    assert calls == [True, False]


# ----------------------------------------------------------------------------------------- the queue
class LogprobQueue(QueueStub):
    """QueueStub whose sampler also writes (sampled, model) = (-tag, -step) next to every token; a refill scribbles
    NaN over its slot's rows first, so a harvest after the refill would see them."""

    def __init__(self, max_batch, eos_at=None):
        super().__init__(max_batch, eos_at)
        self.logprobs = None

    def set_logprobs(self, on=True):
        self.logprobs = torch.zeros(self.max_batch, self.max_new, 2) if on else None
        self.log.append(("logprobs", bool(on)))

    def _start(self, s, prompt, key):
        if self.logprobs is not None:
            self.logprobs[s] = float("nan")
        super()._start(s, prompt, key)

    def _emit(self, s):
        g = int(self.n_generated[s])
        super()._emit(s)
        if self.logprobs is not None:
            self.logprobs[s, g] = torch.tensor([-float(self.who[s]), -float(g)])


def test_queue_harvests_rows_before_refill():
    lens = [90, 80, 95, 70, 99, 85, 60]
    caps = [100 - m for m in lens]
    lm = LogprobQueue(3, eos_at={2: 4, 6: 0})
    ids, lps = lm.generate_queue(_prompts(lens), EOS, max_length=100, min_new_tokens=0, check_every=8, return_logprobs=True)
    assert lm.log[1] == ("logprobs", True)
    for i, (t, lp) in enumerate(zip(ids, lps)):
        n = {2: 5, 6: 1}.get(i + 1, caps[i])
        assert len(t) == n and lp.dtype == torch.float32 and lp.shape == (n, 2)
        assert lp[:, 0].tolist() == [-(i + 1.0)] * n and lp[:, 1].tolist() == [-float(g) for g in range(n)]
    plain = lm.generate_queue(_prompts(lens), EOS, max_length=100, min_new_tokens=0, check_every=8)
    assert lm.log[-1][0] != "logprobs" and ("logprobs", False) in lm.log and lm.logprobs is None
    assert all(torch.equal(a, b) for a, b in zip(plain, ids))
    assert lm.generate_queue([], EOS, max_length=100, return_logprobs=True) == ([], [])


# ----------------------------------------------------------------------------------------- the facade
class BatchStub:
    """generate_batch / set_logprobs stub: prompt i generates [speech 1, text 'A', speech 2, EOS] with rows (i, j)."""
    device = torch.device("cpu")

    def __init__(self, tok):
        self.tok, self.calls = tok, []

    def set_logprobs(self, on=True):
        pass

    def generate_batch(self, prompts, eos, slot_base=0, return_logprobs=False, **kw):
        self.calls.append((slot_base, return_logprobs))
        sb = self.tok.speech_base
        ids = [torch.tensor([sb + 1, 65, sb + 2, eos]) for _ in prompts]
        lps = [torch.tensor([[slot_base + i, j] for j in range(4)], dtype=torch.float32) for i in range(len(prompts))]
        return (ids, lps) if return_logprobs else ids


def _facade(make_backbone, max_batch=2):
    import warnings

    from neutts import NeuTTS

    tok = FakeTokenizer()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=make_backbone(tok), codec=FakeCodec(),
                      max_batch=max_batch, seed=3)


def test_facade_returns_rows_aligned_with_ids():
    tts = _facade(BatchStub)
    wavs, lps = tts.infer_batch(["a", "b", "c"], [[1], [2], [3]], ["x", "y", "z"], return_logprobs=True)
    assert len(wavs) == len(lps) == 3 and all(len(w) == 2 * 480 for w in wavs)   # 2 speech codes per utterance
    for i, lp in enumerate(lps):
        assert isinstance(lp, np.ndarray) and lp.dtype == np.float32 and lp.shape == (4, 2)   # text id and EOS keep rows
        assert lp[:, 0].tolist() == [float(i)] * 4
    assert tts.backbone.calls == [(0, True), (2, True)]
    wav, lp = tts.infer("a", [1], "x", return_logprobs=True)
    assert lp.shape == (4, 2) and len(wav) == 960
    assert isinstance(tts.infer("a", [1], "x"), np.ndarray) and tts.backbone.calls[-1] == (0, False)
    wavs, lps = tts.infer_from_prompt_ids([[5, 6]], return_logprobs=True)
    assert len(wavs) == 1 and lps[0].shape == (4, 2)


def test_facade_rejects_unsupported_logprobs():
    from tests.fakes import FakeBackbone

    tts = _facade(lambda tok: FakeBackbone([3005, 2005]))
    with pytest.raises(ValueError, match="set_logprobs"):
        tts.infer_batch(["a"], [[1]], ["x"], return_logprobs=True)
    with pytest.raises(ValueError, match="set_logprobs"):
        tts.infer_from_prompt_ids([[5]], return_logprobs=True)
    tts.backbone = BatchStub(tts.tokenizer)
    with pytest.raises(ValueError, match="distributed"):
        tts.infer_batch(["a"], [[1]], ["x"], distributed=True, return_logprobs=True)
    assert tts.backbone.calls == []
