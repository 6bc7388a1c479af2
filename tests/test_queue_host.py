"""Host logic of continuous batching (SpeechLM.generate_queue) and the facade's use of it, on a CPU stub engine.

The stub keeps SpeechLM's host side (page pool, per-slot page lists, generate_queue, release_pages) and replaces the
device calls: prompt i (every id of it is i + 1) emits the tokens 1000 * (i + 1) + step, or EOS at a chosen step.
"""
import types
import warnings

import numpy as np
import torch

from neutts_air_b200.lm import PagePool, SpeechLM
from tests.test_host_logic import FakeCodec, FakePhonemizer, FakeTokenizer

EOS = 9


class QueueStub(SpeechLM):
    def __init__(self, max_batch, eos_at=None):
        self.max_ctx, self.max_new, self.max_batch, self.device = 2048, 2048, max_batch, torch.device("cpu")
        self.max_pages = self.max_ctx // self.PAGE
        self.num_pages = max_batch * self.max_pages
        self.pool = PagePool(self.num_pages, shuffle_seed=1)
        self._slot_pages = [[] for _ in range(max_batch)]
        self.out_tokens = torch.zeros(max_batch, self.max_new, dtype=torch.int32)
        self.n_generated = torch.zeros(max_batch, dtype=torch.int32)
        self.done = torch.zeros(max_batch, dtype=torch.int32)
        self.eos_at = eos_at or {}
        self.who, self.cap = [None] * max_batch, [0] * max_batch
        self.log, self.admitted = [], 0

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, limits=None, slot_base=0):
        self.limit_table = list(limits) + [max_new] * (self.max_batch - len(limits))
        self.log.append(("sampling", list(limits), slot_base))
        return types.SimpleNamespace(max_new_tokens=max_new, slot_base=slot_base)

    def _start(self, s, prompt, key):
        tag = prompt[0]
        assert all(t == tag for t in prompt)
        assert key == self.slot_base + tag - 1, (key, tag)   # Philox stream = slot_base + input index
        self._slot_pages[s] = self.pool.alloc((len(prompt) + self.limit_table[s] + self.PAGE - 1) // self.PAGE)
        self.who[s], self.cap[s] = tag, self.limit_table[s]
        self.n_generated[s], self.done[s] = 0, 0
        self.admitted += 1
        self._emit(s)

    def _emit(self, s):
        g = int(self.n_generated[s])
        tok = EOS if self.eos_at.get(self.who[s]) == g else 1000 * self.who[s] + g
        self.out_tokens[s, g], self.n_generated[s] = tok, g + 1
        if tok == EOS or g + 1 >= self.cap[s]:
            self.done[s] = 1

    def prefill(self, prompts, sp):
        self.release_pages()
        self.slot_base = sp.slot_base
        self.log.append(("prefill", [p[0] for p in prompts]))
        for s, p in enumerate(prompts):
            self._start(s, p, sp.slot_base + s)
        self._B = len(prompts)

    def prefill_slots(self, slots, prompts, sp, stream_ids, return_logits=False, limits=None):
        assert all(self.done[s] for s in slots)          # only finished slots are refilled
        self.log.append(("refill", list(slots), [p[0] for p in prompts], list(stream_ids), list(limits)))
        self.release_pages(slots)
        for s, p, key, lim in zip(slots, prompts, stream_ids, limits):
            self.limit_table[s] = lim
            self._start(s, p, key)

    def decode(self, n, sp):
        live = [s for s in range(self._B) if not self.done[s]]
        left = [self.cap[s] - int(self.n_generated[s]) for s in live]
        self.log.append(("decode", n, min(left), max(left), self.admitted))
        for _ in range(n):
            for s in live:
                if not self.done[s]:
                    self._emit(s)


def _prompts(lens):
    return [[i + 1] * m for i, m in enumerate(lens)]


def test_queue_fifo_order_streams_limits_and_pages():
    lens = [90, 80, 95, 70, 99, 85, 60]            # max_length 100 -> caps 10, 20, 5, 30, 1, 15, 40
    caps = [100 - m for m in lens]
    lm = QueueStub(3)
    out = lm.generate_queue(_prompts(lens), EOS, max_length=100, min_new_tokens=100, check_every=8, slot_base=40)
    # outputs in input order, each exactly its own tokens up to its cap
    assert [o.tolist() for o in out] == [[1000 * (i + 1) + g for g in range(c)] for i, c in enumerate(caps)]
    assert all(o.dtype == torch.int64 for o in out)
    # FIFO admission, every prompt once: the first wave by prefill, the rest by refills in input order
    assert lm.log[0] == ("sampling", caps[:3], 40)
    assert lm.log[1] == ("prefill", [1, 2, 3])
    refills = [e for e in lm.log if e[0] == "refill"]
    assert [t for e in refills for t in e[2]] == [4, 5, 6, 7]
    for e in refills:
        assert e[3] == [40 + t - 1 for t in e[2]]                 # stream id = slot_base + index
        assert e[4] == [caps[t - 1] for t in e[2]]                # a limits entry at each admission
    # the page pool is whole again
    assert sorted(lm.pool.free) == list(range(lm.num_pages))
    assert all(not p for p in lm._slot_pages)


def test_queue_launches_end_at_the_earliest_due_completion():
    lens = [90, 80, 95, 70, 99, 85, 60]
    lm = QueueStub(3)
    lm.generate_queue(_prompts(lens), EOS, max_length=100, min_new_tokens=100, check_every=8)
    decodes = [e for e in lm.log if e[0] == "decode"]
    assert decodes
    for _, n, lo, hi, admitted in decodes:
        if admitted < len(lens):      # prompts waiting: stop when the first slot reaches its cap
            assert n == min(8, lo), (n, lo)
        else:                         # queue drained: run on, checking every 8 steps
            assert n == min(8, hi), (n, hi)


def test_queue_refills_a_slot_that_finished_at_prefill():
    # prompt 5 has a cap of 1; prompt 6 samples EOS as its first token (min_new_tokens=0)
    lens = [90, 80, 95, 70, 99, 85, 60]
    lm = QueueStub(3, eos_at={6: 0})
    out = lm.generate_queue(_prompts(lens), EOS, max_length=100, min_new_tokens=0, check_every=8)
    assert out[4].tolist() == [5000] and out[5].tolist() == [EOS]
    assert out[6].tolist() == [7000 + g for g in range(40)]
    assert lm.admitted == 7
    # the slot of prompt 5 went straight to prompt 6, and that one straight to prompt 7, with no decode in between
    refills = [i for i, e in enumerate(lm.log) if e[0] == "refill"]
    seq = [lm.log[i][2] for i in refills]
    assert [5] in seq and [6] in seq and [7] in seq
    i5, i6, i7 = (refills[seq.index([t])] for t in (5, 6, 7))
    assert i6 == i5 + 1 and i7 == i6 + 1
    assert sorted(lm.pool.free) == list(range(lm.num_pages))


def test_queue_eos_stops_early_and_fewer_prompts_than_slots():
    lm = QueueStub(4, eos_at={2: 3})
    out = lm.generate_queue(_prompts([10, 20]), EOS, max_length=60, min_new_tokens=0, check_every=5)
    assert out[0].tolist() == [1000 + g for g in range(50)]
    assert out[1].tolist() == [2000, 2001, 2002, EOS]
    assert not [e for e in lm.log if e[0] == "refill"]
    assert lm.generate_queue([], EOS) == []


class BatchBackbone:
    device = torch.device("cpu")

    def __init__(self, tok):
        self.tok, self.calls = tok, []

    def _ids(self, prompts):
        return [torch.tensor([self.tok.speech_base + len(p) % 50, self.tok.speech_base + 3]) for p in prompts]

    def generate_batch(self, prompts, eos, **kw):
        self.calls.append(("batch", len(prompts), kw["slot_base"]))
        return self._ids(prompts)


class QueueBackbone(BatchBackbone):
    def generate_queue(self, prompts, eos, **kw):
        self.calls.append(("queue", len(prompts), kw["slot_base"]))
        return self._ids(prompts)


def _facade(max_batch, queue=True):
    from neutts import NeuTTS

    tok = FakeTokenizer()
    bb = (QueueBackbone if queue else BatchBackbone)(tok)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=bb, codec=FakeCodec(), max_batch=max_batch, seed=1)
    return tts, bb


def test_facade_sends_long_lists_through_the_queue():
    texts, refs, rts = ["a b"] * 7, [[1, 2]] * 7, ["r"] * 7
    tts, bb = _facade(3)
    wavs = tts.infer_batch(texts, refs, rts)
    assert len(wavs) == 7 and bb.calls == [("queue", 7, 0)]
    # a list that fits keeps the chunked call
    bb.calls.clear()
    tts.infer_batch(texts[:3], refs[:3], rts[:3])
    assert bb.calls == [("batch", 3, 0)]
    # a backbone without generate_queue keeps the chunks of max_batch
    tts2, bb2 = _facade(3, queue=False)
    wavs2 = tts2.infer_batch(texts, refs, rts)
    assert bb2.calls == [("batch", 3, 0), ("batch", 3, 3), ("batch", 1, 6)]
    assert all(np.array_equal(a, b) for a, b in zip(wavs, wavs2))


def test_facade_distributed_runs_one_queue_per_rank(monkeypatch):
    from neutts_air_b200 import dist

    monkeypatch.setattr(dist, "world", lambda: (2, 4))
    monkeypatch.setattr(dist, "shard_indices", lambda n, lengths: [0, 2, 3, 5, 6])
    monkeypatch.setattr(dist, "all_gather_waveforms", lambda local, mine, n, device=None: (local, mine, n))
    tts, bb = _facade(3)
    local, mine, n = tts.infer_batch(["a b"] * 8, [[1, 2]] * 8, ["r"] * 8, distributed=True)
    assert bb.calls == [("queue", 5, 2 << 20)] and len(local) == 5 and mine == [0, 2, 3, 5, 6] and n == 8
    bb.calls.clear()
    monkeypatch.setattr(dist, "shard_indices", lambda n, lengths: [1, 4])
    tts.infer_batch(["a b"] * 8, [[1, 2]] * 8, ["r"] * 8, distributed=True)
    assert bb.calls == [("batch", 2, 2 << 20)]
