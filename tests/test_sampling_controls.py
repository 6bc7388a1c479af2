"""Per-slot sampling controls (temperature, top_k, top_p, min_p) without a GPU: the float64 reference of the whole
processor chain, pinned to transformers' own warpers, and the host plumbing of the engine and the facade on stubs.

The reference (``chain64``, ``ref_window_cut`` in sampler_ref.py) is what tests/test_gpu_sampling_controls.py compares
every sampler path with.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import per_prompt_controls
from tests.fakes import EOS, FakeTokenizer, GenerateBackbone, KwBackbone, QueueStub, _facade, _prompts
from tests.sampler_ref import chain64, ref_token, ref_window_cut


def test_chain_matches_transformers_warpers():
    """TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> MinPLogitsWarper, softmax: the same kept ids
    and probabilities as chain64 on the same float64 scores (logits / T), except within 1e-6 of a cut."""
    from transformers.generation.logits_process import (MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)

    rng = np.random.default_rng(11)
    kept_cases = cut_cases = 0
    for case in range(240):
        V = int(rng.integers(70, 3000))
        logits = rng.normal(0.0, rng.uniform(0.5, 4.0), V)
        T = float(rng.choice([0.3, 0.7, 1.0, 1.3, 2.0]))
        k = int(rng.choice([1, 2, 7, 20, 50, 64]))
        top_p = float(rng.choice([1.0, 0.2, 0.5, 0.8, 0.95]))
        min_p = float(rng.choice([0.0, 0.01, 0.05, 0.3]))
        ids, q, margin = chain64(logits / T, k, top_p, min_p)
        if margin < 1e-6:
            continue
        x = torch.from_numpy(logits)[None, :]
        for w in (TemperatureLogitsWarper(T), TopKLogitsWarper(k), TopPLogitsWarper(top_p) if top_p < 1 else None,
                  MinPLogitsWarper(min_p) if min_p > 0 else None):
            if w is not None:
                x = w(None, x)
        probs = torch.softmax(x, dim=-1)[0].numpy()
        hf_ids = np.nonzero(probs > 0)[0]
        assert sorted(ids.tolist()) == hf_ids.tolist(), (case, V, T, k, top_p, min_p)
        assert np.abs(probs[ids] - q).max() < 1e-12, case
        kept_cases += 1
        cut_cases += len(ids) < min(k, V)
    assert kept_cases >= 200 and cut_cases >= 60, (kept_cases, cut_cases)


def test_chain_defaults_are_plain_top_k():
    """top_p = 1 and min_p = 0 keep the whole top-k window, even where the cumulative sum rounds to 1 early."""
    s = np.array([50.0, 0.0, -1.0, -2.0] + [-3.0] * 60)
    ids, q, margin = chain64(s, 64, 1.0, 0.0)
    assert len(ids) == 64 and margin == np.inf
    assert ids[0] == 0 and (np.diff(ids[4:]) > 0).all()
    ids, q, _ = chain64(s, 64, 0.999999, 0.0)              # the first entry holds all but ~1e-21 of the mass
    assert len(ids) == 1 and q.tolist() == [1.0]


def test_chain_cuts_and_draw():
    s = np.log(np.array([0.4, 0.3, 0.2, 0.06, 0.04]))
    ids, q, _ = chain64(s, 5, 0.75, 0.0)                    # excl: 0, .4, .7, .9 -> three stay
    assert ids.tolist() == [0, 1, 2] and np.allclose(q, [4 / 9, 3 / 9, 2 / 9])
    ids, _, _ = chain64(s, 5, 1.0, 0.6)                     # q_j / q_0 >= 0.6: 1, .75
    assert ids.tolist() == [0, 1]
    ids, _, _ = chain64(s, 5, 0.95, 0.12)                   # min-p (>= .048) keeps 4, top-p keeps 4
    assert ids.tolist() == [0, 1, 2, 3]
    ids, _, _ = chain64(s, 2, 0.99, 0.0)                    # top-k first
    assert ids.tolist() == [0, 1]
    ids, _, _ = chain64(s, 5, 0.01, 0.99)                   # entry 0 always stays
    assert ids.tolist() == [0]
    w = chain64(s, 5, 0.75, 0.0)[:2]
    assert ref_token(w, 0.5)[0] == 1 and ref_token(w, 0.99)[0] == 2


def test_ref_window_cut_uses_inverse_temperature_product():
    x = np.random.default_rng(3).normal(0, 3, 500).astype(np.float32)
    ids, q, _ = ref_window_cut(x, 0, 7, 0, 0.7, 64, 1.0, 0.0)
    s = x * (np.float32(1) / np.float32(0.7))
    assert ids.tolist() == np.lexsort((np.arange(500), -s.astype(np.float64)))[:64].tolist()


# ====================================================================================== host plumbing on stubs
def test_per_prompt_controls_validation():
    assert per_prompt_controls(3, 1.0, 50, 1.0, 0.0) is None
    assert per_prompt_controls(3, 0.7, 20, 1.0, 0.0) is None            # scalars: the launch scalars govern
    assert per_prompt_controls(2, 0.7, 20, 0.9, 0.0) == [(0.7, 20, 0.9, 0.0)] * 2
    assert per_prompt_controls(2, [0.5, 2.0], 50, 1.0, [0.0, 0.1]) == [(0.5, 50, 1.0, 0.0), (2.0, 50, 1.0, 0.1)]
    assert per_prompt_controls(2, torch.tensor([0.5, 1.0]), np.array([3, 4]), 1.0, 0.0)[1] == (1.0, 4, 1.0, 0.0)
    for bad in (dict(temperature=[1.0]), dict(top_k=[1, 2, 3]), dict(top_p=[0.5] * 4)):
        kw = dict(temperature=1.0, top_k=50, top_p=1.0, min_p=0.0) | bad
        with pytest.raises(ValueError, match="one value per prompt"):
            per_prompt_controls(2, **kw)
    for bad in (dict(temperature=[0.0, 1.0]), dict(temperature=[float("nan"), 1.0]), dict(temperature=[float("inf"), 1.0]),
                dict(top_k=[0, 1]), dict(top_k=[65, 1]), dict(top_k=[2.5, 1]), dict(top_p=[0.0, 1.0]),
                dict(top_p=[1.5, 1.0]), dict(top_p=[float("nan"), 1.0]), dict(min_p=[1.0, 0.0]), dict(min_p=[-0.1, 0.0]),
                dict(top_p=0.0), dict(min_p=1.0)):
        kw = dict(temperature=1.0, top_k=50, top_p=1.0, min_p=0.0) | bad
        with pytest.raises(ValueError):
            per_prompt_controls(2, **kw)


class CtlStub(QueueStub):
    """QueueStub that also runs generate_batch and logs the launch scalars and every per-slot table write."""

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, forced=None, limits=None, slot_base=0):
        self.log.append(("scalars", top_k, temperature))
        return super().sampling(eos, min_new, max_new, top_k, temperature, seed, greedy,
                                limits=[] if limits is None else limits, slot_base=slot_base)

    def set_slot_sampling(self, rows, slots=None):
        self.log.append(("table", None if rows is None else [tuple(r) for r in rows], None if slots is None else list(slots)))
        self._slot_sp_host = rows


LENS = [90, 80, 95, 70, 99, 85, 60]


def test_default_calls_are_unchanged():
    """Scalar controls with top_p = 1, min_p = 0: the same call log as the engine without per-slot controls, and the
    table is never touched."""
    plain = QueueStub(3)
    plain.generate_queue(_prompts(LENS), EOS, max_length=100, min_new_tokens=100, check_every=8, slot_base=40)
    for kw in ({}, dict(temperature=1.0, top_k=50, top_p=1.0, min_p=0.0)):
        lm = CtlStub(3)
        lm.generate_queue(_prompts(LENS), EOS, max_length=100, min_new_tokens=100, check_every=8, slot_base=40, **kw)
        assert [e for e in lm.log if e[0] != "scalars"] == plain.log
        assert [e for e in lm.log if e[0] == "scalars"] == [("scalars", 50, 1.0)]
    lm = CtlStub(3)
    lm.generate_batch(_prompts(LENS[:3]), EOS, max_length=100, min_new_tokens=100, temperature=0.7, top_k=20)
    assert lm.log[0] == ("scalars", 20, 0.7) and lm.log[2][0] == "prefill"
    assert not [e for e in lm.log if e[0] == "table"]


def test_default_call_switches_a_left_over_table_off():
    lm = CtlStub(3)
    lm.generate_batch(_prompts(LENS[:2]), EOS, max_length=100, min_new_tokens=100, top_p=[0.9, 0.5])
    assert ("table", [(1.0, 50, 0.9, 0.0), (1.0, 50, 0.5, 0.0)], None) in lm.log
    lm.log.clear()
    lm.generate_batch(_prompts(LENS[:2]), EOS, max_length=100, min_new_tokens=100)
    tables = [i for i, e in enumerate(lm.log) if e[0] == "table"]
    prefill = [i for i, e in enumerate(lm.log) if e[0] == "prefill"]
    assert [lm.log[i] for i in tables] == [("table", None, None)] and tables[0] < prefill[0]


def test_lists_are_validated_before_any_engine_call():
    lm = CtlStub(3)
    with pytest.raises(ValueError):
        lm.generate_batch(_prompts(LENS[:2]), EOS, max_length=100, temperature=[1.0, 0.5, 0.7])
    with pytest.raises(ValueError):
        lm.generate_queue(_prompts(LENS), EOS, max_length=100, min_p=[0.1] * 6 + [1.0])
    assert lm.log == []


def test_queue_writes_newcomers_controls_before_their_prefill():
    temps = [0.5, 0.6, 0.7, 0.8, 0.9, 1.1, 1.2]
    ks = [1, 64, 10, 20, 30, 40, 50]
    lm = CtlStub(3)
    lm.generate_queue(_prompts(LENS), EOS, max_length=100, min_new_tokens=100, check_every=8, temperature=temps, top_k=ks,
                      min_p=0.05)
    rows = [(t, k, 1.0, 0.05) for t, k in zip(temps, ks)]
    assert lm.log[0] == ("scalars", 1, 0.5)
    first = lm.log.index(("table", rows[:3], None))
    assert first < [i for i, e in enumerate(lm.log) if e[0] == "prefill"][0]
    refills = [i for i, e in enumerate(lm.log) if e[0] == "refill"]
    assert refills
    for i in refills:
        slots, tags = lm.log[i][1], lm.log[i][2]
        assert lm.log[i - 1] == ("table", [rows[t - 1] for t in tags], slots)   # only the newcomers' slots
    assert sum(len(lm.log[i][2]) for i in refills) == 4


# ---------------------------------------------------------------------------------------- facade
def _ctl(kw):
    return {k: kw[k] for k in ("temperature", "top_k", "top_p", "min_p") if k in kw}


def test_facade_defaults_forward_what_they_always_did():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    tts = _facade(bb, 3)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, temperature=1.0, top_k=50, top_p=1.0, min_p=0.0)
    assert [_ctl(c[2]) for c in bb.calls] == [dict(temperature=1.0, top_k=50)] * 2
    assert bb.calls[0][2] == bb.calls[1][2]
    gb = GenerateBackbone(tok)
    tts = _facade(gb, 1)
    tts.infer("a b", [1, 2], "r")
    tts.infer("a b", [1, 2], "r", top_p=0.8, min_p=0.1, temperature=0.7)
    assert "top_p" not in gb.kws[0] and "min_p" not in gb.kws[0]
    assert _ctl(gb.kws[1]) == dict(temperature=0.7, top_k=50, top_p=0.8, min_p=0.1)
    assert {k: v for k, v in gb.kws[0].items() if k not in ("temperature", "top_k")} == \
        {k: v for k, v in gb.kws[1].items() if k not in ("temperature", "top_k", "top_p", "min_p")}


def test_facade_lists_follow_their_utterances(monkeypatch):
    tok = FakeTokenizer()
    temps = [0.5 + 0.1 * i for i in range(7)]
    tops = [0.9 - 0.05 * i for i in range(7)]
    kw = dict(temperature=temps, top_p=tops)
    # chunks of max_batch
    bb = KwBackbone(tok, queue=False)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, **kw)
    assert [(c[1], c[2]["slot_base"], c[2]["temperature"], c[2]["top_p"], c[2]["top_k"]) for c in bb.calls] == [
        (3, 0, temps[0:3], tops[0:3], 50), (3, 3, temps[3:6], tops[3:6], 50), (1, 6, temps[6:], tops[6:], 50)]
    assert all("min_p" not in c[2] for c in bb.calls)
    # one queue
    bb = KwBackbone(tok)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, min_p=[0.01 * i for i in range(7)], top_k=20)
    assert len(bb.calls) == 1 and bb.calls[0][0] == "queue"
    assert _ctl(bb.calls[0][2]) == dict(temperature=1.0, top_k=20, min_p=[0.01 * i for i in range(7)])
    # sharded over ranks: this rank's utterances, in shard order, for the queue and for the chunked call
    from neutts_air_b200 import dist

    monkeypatch.setattr(dist, "world", lambda: (1, 2))
    monkeypatch.setattr(dist, "all_gather_waveforms", lambda local, mine, n, device=None: (local, mine, n))
    for shard, what in (([0, 2, 3, 5, 6], "queue"), ([1, 4], "batch")):
        monkeypatch.setattr(dist, "shard_indices", lambda n, lengths, shard=shard: shard)
        bb = KwBackbone(tok)
        _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, distributed=True, **kw)
        assert [(c[0], c[2]["temperature"], c[2]["top_p"]) for c in bb.calls] == [
            (what, [temps[i] for i in shard], [tops[i] for i in shard])]
    # transformers-style backbone: one utterance per generate call, with its own values
    gb = GenerateBackbone(tok)
    _facade(gb, 3).infer_batch(["a b"] * 3, [[1, 2]] * 3, ["r"] * 3, temperature=temps[:3], top_p=tops[:3], min_p=0.05)
    assert [_ctl(k) for k in gb.kws] == [dict(temperature=temps[i], top_k=50, top_p=tops[i], min_p=0.05) for i in range(3)]


def test_facade_rejects_lists_of_the_wrong_length():
    tok = FakeTokenizer()
    bb = KwBackbone(tok)
    tts = _facade(bb, 3)
    with pytest.raises(ValueError, match="one value per utterance"):
        tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, top_k=[10, 20, 30])
    with pytest.raises(ValueError, match="one value per utterance"):
        tts.infer_stream_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, temperature=[1.0])
    assert bb.calls == []
