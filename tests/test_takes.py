"""Host logic of several takes per utterance (SpeechLM.prefill_fork / generate_batch(num_return_sequences=n) and
NeuTTS's ``takes``), on CPU stubs: page-pool reference counts, the page-table layout of a fork, argument validation,
slot and stream-key mapping, per-prompt settings written to every take, the facade's chunking and its choice of take.
"""
import types
import warnings

import numpy as np
import pytest
import torch

from neutts_air_b200 import _lib
from neutts_air_b200.lm import PagePool, Settings, SpeechLM, check_takes, fork_slots, resolve_settings
from tests.fakes import FakeCodec, FakePhonemizer, FakeTokenizer

EOS = 9


# ---------------------------------------------------------------------------------------------- page pool
def test_page_pool_reference_counts():
    pool = PagePool(8, shuffle_seed=3)
    assert pool.num_free == 8
    a = pool.alloc(3)
    b = pool.alloc(2)
    assert pool.num_free == 3 and all(pool.refs[p] == 1 for p in a + b)
    pool.share(a)
    pool.share(a)
    assert all(pool.refs[p] == 3 for p in a)
    pool.release(a + b)                       # b is freed, a is still held twice
    assert pool.num_free == 5 and sorted(set(pool.free) & set(a)) == []
    pool.release(a)
    assert pool.num_free == 5
    pool.release(a)
    assert pool.num_free == 8 and sorted(pool.free) == list(range(8))
    assert all(r == 0 for r in pool.refs)


def test_page_pool_refuses_unheld_pages():
    pool = PagePool(4)
    p = pool.alloc(1)
    with pytest.raises(ValueError):
        pool.share([q for q in range(4) if q not in p][:1])    # a free page
    with pytest.raises(ValueError):
        pool.release(p + p)                                     # held once, released twice
    assert pool.refs[p[0]] == 1 and pool.num_free == 3         # a refused call changes nothing
    pool.release(p)
    with pytest.raises(ValueError):
        pool.release(p)


def test_page_pool_without_sharing_frees_in_the_same_order():
    """Unshared pages go back to the free list exactly as before reference counts existed."""
    a, b = PagePool(16, shuffle_seed=5), PagePool(16, shuffle_seed=5)
    pa, pb = a.alloc(7), b.alloc(7)
    assert pa == pb
    a.release(pa)
    b.free.extend(reversed(pb))
    assert a.free == b.free


# ---------------------------------------------------------------------------------------------- stub engine
class ForkStub(SpeechLM):
    """SpeechLM's host side with the device calls replaced: take j of prompt i (all ids i + 1) emits one token,
    100 * (i + 1) + j, then stops."""

    def __init__(self, max_batch, max_ctx=512):
        self.max_ctx, self.max_new, self.max_batch, self.device = max_ctx, max_ctx, max_batch, torch.device("cpu")
        self.max_pages = self.max_ctx // self.PAGE
        self.num_pages = max_batch * self.max_pages
        self.pool = PagePool(self.num_pages, shuffle_seed=1)
        self._slot_pages = [[] for _ in range(max_batch)]
        self.out_tokens = torch.zeros(max_batch, self.max_new, dtype=torch.int32)
        self.n_generated = torch.zeros(max_batch, dtype=torch.int32)
        self.done = torch.zeros(max_batch, dtype=torch.int32)
        self.shape = types.SimpleNamespace(vocab_size=4096)
        self._slot_sp_host = self._vocab_range = self._penalty_host = self.logprobs = None
        self.log = []

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, forced=None, limits=None, slot_base=0):
        self.log.append(("sampling", None if limits is None else list(limits), slot_base,
                         None if forced is None else forced.shape[0]))
        return types.SimpleNamespace(max_new_tokens=max_new, slot_base=slot_base)

    def set_slot_sampling(self, rows, slots=None):
        self.log.append(("controls", rows))
        self._slot_sp_host = rows

    def set_repetition_penalty(self, rows, slots=None):
        self.log.append(("penalty", rows))
        self._penalty_host = rows

    def set_logprobs(self, on=True):
        self.logprobs = torch.zeros(self.max_batch, self.max_new, 2) if on else None

    def set_vocab_range(self, lo, hi=None):
        self._vocab_range = None if lo is None else (lo, hi)

    def _emit(self, rows):
        for s, tok in rows:
            self.out_tokens[s, 0], self.n_generated[s], self.done[s] = tok, 1, 1
            if self.logprobs is not None:
                self.logprobs[s, 0] = torch.tensor([-0.5, -float(s)])

    def prefill(self, prompts, sp):
        self.log.append(("prefill", len(prompts)))
        self._emit((s, 100 * p[0]) for s, p in enumerate(prompts))
        self._B = len(prompts)

    def prefill_fork(self, prompts, n, sp, return_logits=False):
        n = check_takes(len(prompts), n, self.max_batch)
        self.log.append(("fork", len(prompts), n))
        self.release_pages()
        self.table = np.zeros((self.max_batch, self.max_pages), dtype=np.int32)
        self._alloc_fork_pages(self.table, [len(p) for p in prompts], n, sp.max_new_tokens)
        self._emit((i * n + j, 100 * p[0] + j) for i, p in enumerate(prompts) for j in range(n))
        self._B = len(prompts) * n

    def decode(self, n, sp):
        pass


def _prompts(lens):
    return [[i + 1] * m for i, m in enumerate(lens)]


def test_fork_page_table_layout_and_release():
    """Take j of prompt i holds the prompt's full pages (shared by all its takes) and pages of its own from page P // 64
    on; releasing a take returns only its own pages until its last sibling lets go of the shared ones."""
    lm = ForkStub(8)
    lens, n, cap = [130, 64, 5], 2, 70          # 2 full pages + tail, 1 full page (no tail), no full page
    sp = types.SimpleNamespace(max_new_tokens=cap)
    lm.prefill_fork(_prompts(lens), n, sp)
    t = lm.table
    used = 0
    for i, P in enumerate(lens):
        full, need = P // 64, (P + cap + 63) // 64
        rows = [t[i * n + j] for j in range(n)]
        for r in rows:
            assert (r[:full] == rows[0][:full]).all() and (r[need:] == 0).all()
        own = [set(r[full:need].tolist()) for r in rows]
        assert not own[0] & own[1] and all(len(o) == need - full for o in own)
        assert not own[0] & set(rows[0][:full].tolist())
        used += full + n * (need - full)
    assert lm.pool.num_free == lm.num_pages - used
    shared0 = t[0, :2].tolist()
    before = lm.pool.num_free
    lm.release_pages([1])                                   # prompt 0's second take: its 2 own pages only
    assert lm.pool.num_free == before + (130 + cap + 63) // 64 - 2
    assert all(lm.pool.refs[p] == 1 for p in shared0)
    lm.release_pages([0])
    assert all(lm.pool.refs[p] == 0 for p in shared0)
    lm.release_pages()
    assert sorted(lm.pool.free) == list(range(lm.num_pages))


def test_fork_slots_and_stream_keys():
    assert fork_slots(2, 3, slot_base=10) == [(0, 0, 0, 10), (0, 1, 1, 11), (0, 2, 2, 12),
                                              (1, 0, 3, 13), (1, 1, 4, 14), (1, 2, 5, 15)]
    # the keys are those of generate_batch on the prompts repeated n times (repeat_interleave): slot + slot_base
    for i, j, s, key in fork_slots(3, 4, 7):
        assert s == i * 4 + j and key == s + 7


def test_check_takes():
    assert check_takes(3, 2, 6) == 2 and check_takes(1, np.int64(4), 4) == 4
    for bad in (0, -1, 1.5, "2", True, None):
        with pytest.raises(ValueError):
            check_takes(1, bad, 8)
    with pytest.raises(ValueError):
        check_takes(3, 3, 8)


def test_prefill_argument_errors():
    """SpeechLM.prefill (one take per prompt) raises ValueError for an empty call, an empty or over-long prompt, more
    prompts than slots and an id outside the vocabulary, before it touches the page pool or the device."""
    lm = object.__new__(SpeechLM)            # host fields only: a check that came later would hit a missing attribute
    lm.max_batch, lm.max_ctx, lm.shape = 2, 128, types.SimpleNamespace(vocab_size=4096)
    sp = types.SimpleNamespace(max_new_tokens=8)
    for prompts, msg in (([], "empty prompt"), ([[1], []], "empty prompt"), ([[1] * 128], r"1\.\.127"),
                         ([[1]] * 3, "slots"), ([[1, 4096]], "out of range"), ([[-1]], "out of range")):
        with pytest.raises(ValueError, match=msg):
            lm.prefill(prompts, sp)


def test_generate_batch_validates_before_any_engine_call():
    lm = ForkStub(4)
    for n in (0, -2, 3):                                    # 3: 2 prompts x 3 takes > 4 slots
        with pytest.raises(ValueError):
            lm.generate_batch(_prompts([10, 20]), EOS, max_length=100, num_return_sequences=n)
    assert lm.log == []
    with pytest.raises(ValueError):
        lm.generate_queue(_prompts([10, 20]), EOS, max_length=100, num_return_sequences=2)
    assert lm.log == []


def test_generate_batch_takes_order_settings_caps_and_pages():
    lm = ForkStub(6)
    prompts = _prompts([70, 20, 30])
    ids = lm.generate_batch(prompts, EOS, max_length=100, min_new_tokens=0, num_return_sequences=2, slot_base=5,
                            temperature=[0.5, 1.0, 1.5], top_k=[10, 20, 30], repetition_penalty=[1.0, 1.2, 1.3],
                            max_new_tokens=[5, 50, 60], forced=torch.zeros(6, 3, dtype=torch.int32))
    # results in slot order: take j of prompt i at i * 2 + j
    assert [o.tolist() for o in ids] == [[100 * (i + 1) + j] for i in range(3) for j in range(2)]
    assert all(o.dtype == torch.int64 for o in ids)
    # every per-prompt row went to both of its takes, through the one settings path, before the fork
    ctl = [e for e in lm.log if e[0] == "controls"][0][1]
    assert [(c[0], c[1]) for c in ctl] == [(0.5, 10), (0.5, 10), (1.0, 20), (1.0, 20), (1.5, 30), (1.5, 30)]
    pen = [e for e in lm.log if e[0] == "penalty"][0][1]
    assert [p[0] for p in pen] == [1.0, 1.0, 1.2, 1.2, 1.3, 1.3]
    # caps per take (the prompt's), forced rows per take, and the fork itself
    samp = [e for e in lm.log if e[0] == "sampling"][0]
    assert samp == ("sampling", [5, 5, 50, 50, 60, 60], 5, 6)
    assert ("fork", 3, 2) in lm.log and ("prefill", 3) not in lm.log
    order = [e[0] for e in lm.log]
    assert order.index("controls") < order.index("fork") and order.index("penalty") < order.index("fork")
    lm.release_pages()
    assert lm.pool.num_free == lm.num_pages


def test_generate_batch_one_take_keeps_the_plain_prefill():
    lm = ForkStub(4)
    ids = lm.generate_batch(_prompts([10, 20]), EOS, max_length=100, min_new_tokens=0, num_return_sequences=1)
    assert [o.tolist() for o in ids] == [[100], [200]]
    assert ("prefill", 2) in lm.log and not [e for e in lm.log if e[0] == "fork"]


def test_settings_repeat():
    lm = types.SimpleNamespace(shape=types.SimpleNamespace(vocab_size=4096))
    st = resolve_settings(lm, 2, temperature=[0.7, 1.3], top_k=[5, 9], repetition_penalty=[1.1, 1.0],
                          penalize_prompt=[True, False], logprobs=True)
    r = st.repeat(3)
    assert r.controls == [st.controls[0]] * 3 + [st.controls[1]] * 3
    assert r.penalty == [st.penalty[0]] * 3 + [st.penalty[1]] * 3
    assert (r.vocab_range, r.temperature, r.top_k, r.logprobs) == (st.vocab_range, st.temperature, st.top_k, True)
    off = Settings(None, None, None, 1.0, 50).repeat(4)
    assert off.controls is None and off.penalty is None


def test_generate_seam_rows():
    """generate(num_return_sequences=n): [B * n, P + gen], row b * n + j = prompt b then take j (transformers' layout)."""
    lm = ForkStub(4)
    x = torch.tensor([[1, 1, 1], [2, 2, 2]])
    out = lm.generate(x, max_length=100, eos_token_id=EOS, min_new_tokens=0, num_return_sequences=2, seed=0)
    assert out.shape == (4, 4)
    assert out[:, :3].tolist() == x.repeat_interleave(2, dim=0).tolist()
    assert out[:, 3].tolist() == [100, 101, 200, 201]


# ---------------------------------------------------------------------------------------------- facade
class PlainBackbone:
    """generate_batch with num_return_sequences: take j of a prompt of length P gets the model log-probabilities
    ``scores(P, j)`` (then EOS, scored as the last token)."""
    device = torch.device("cpu")

    def __init__(self, tok, scores):
        self.tok, self.scores, self.calls = tok, scores, []

    def generate_batch(self, prompts, eos, num_return_sequences=1, return_logprobs=False, **kw):
        n = num_return_sequences
        self.calls.append((len(prompts), n, kw["slot_base"], return_logprobs))
        base = self.tok.speech_base
        ids, lps = [], []
        for i, p in enumerate(prompts):
            for j in range(n):
                rows = self.scores(len(p), j)
                ids.append(torch.tensor([base + 10 * j + k for k in range(len(rows))] + [eos]))
                lps.append(torch.tensor([[-1.0, v] for v in rows + [rows[-1]]], dtype=torch.float32))
        return (ids, lps) if return_logprobs else ids


class TakesBackbone(PlainBackbone):
    def set_logprobs(self, on=True):
        pass


def _facade(max_batch, scores=lambda plen, j: [-1.0, -2.0], backbone=None):
    from neutts import NeuTTS

    tok = FakeTokenizer()
    bb = backbone or TakesBackbone(tok, scores)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=bb, codec=FakeCodec(), max_batch=max_batch, seed=1)
    return tts, bb


def test_best_takes_rule_and_ties():
    from neutts.neutts import best_takes

    lp = lambda *v: np.array([[0.0, x] for x in v], dtype=np.float32)
    rows = [lp(-1, -3), lp(-1.5, -1.5), lp(-4),            # prompt 0: means -2, -1.5, -4 -> take 1
            lp(-2, -2), lp(-1, -3), lp(-3, -1)]            # prompt 1: three means of -2 -> the first take
    assert best_takes(rows, 3) == [1, 3]
    assert best_takes([lp(-np.inf), lp(-5)], 2) == [1]
    assert best_takes([lp(-1)], 1) == [0]


def test_take_chunks():
    from neutts import NeuTTS

    ch = NeuTTS.take_chunks(7, 3, 8)                      # 2 utterances x 3 takes per chunk of 8 slots
    assert [(list(r), b) for r, b in ch] == [([0, 1], 0), ([2, 3], 6), ([4, 5], 12), ([6], 18)]
    assert [(list(r), b) for r, b in NeuTTS.take_chunks(3, 4, 4)] == [([0], 0), ([1], 4), ([2], 8)]


def test_facade_keeps_the_most_probable_take():
    # take 2 of every utterance is best; utterance lengths differ so the codes identify the take
    tts, bb = _facade(6, scores=lambda plen, j: [-3.0, -1.0] if j == 2 else [-2.5, -2.5, -2.5])
    texts, refs, rts = ["a b", "c", "d e f", "g"], [[1, 2]] * 4, ["r"] * 4
    wavs, lps = tts.infer_batch(texts, refs, rts, takes=3, return_logprobs=True)
    assert bb.calls == [(2, 3, 0, True), (2, 3, 6, True)]   # 6 // 3 = 2 utterances per chunk, slot_base = 2 x 3
    assert len(wavs) == 4 and len(lps) == 4
    assert all(lp[:, 1].tolist() == [-3.0, -1.0, -1.0] for lp in lps)
    codes = tts._ids_to_codes(torch.tensor([tts.speech_base + 20, tts.speech_base + 21]))
    assert all(np.array_equal(w, tts._decode_codes([codes])[0]) for w in wavs)
    # infer: one utterance through the same path
    bb.calls.clear()
    w1 = tts.infer("a b", [1, 2], "r", takes=3)
    assert bb.calls == [(1, 3, 0, True)] and np.array_equal(w1, wavs[0])


def test_facade_takes_errors():
    tts, bb = _facade(4)
    args = (["a"], [[1]], ["r"])
    for bad in (0, 5, 2.0, True):
        with pytest.raises(ValueError):
            tts.infer_batch(*args, takes=bad)
    with pytest.raises(ValueError):
        tts.infer_batch(*args, takes=2, distributed=True)
    with pytest.raises(ValueError):
        tts.infer_stream("a", [1], "r", takes=2)
    with pytest.raises(ValueError):
        tts.infer_stream_batch(["a"], [[1]], ["r"], takes=2)
    assert bb.calls == []

    nolp = PlainBackbone(FakeTokenizer(), lambda plen, j: [-1.0])
    tts2, _ = _facade(4, backbone=nolp)
    with pytest.raises(ValueError):
        tts2.infer_batch(*args, takes=2)
    assert nolp.calls == []


def test_facade_one_take_is_todays_path():
    """takes=1 makes exactly the calls infer_batch made before takes existed: no num_return_sequences, no logprobs."""
    tts, bb = _facade(3)
    calls = []
    bb.generate_batch = lambda prompts, eos, **kw: calls.append(sorted(kw)) or [torch.tensor([tts.speech_base + 1])] * len(prompts)
    tts.infer_batch(["a", "b"], [[1], [2]], ["r", "s"], takes=1)
    assert calls and all("num_return_sequences" not in c and "return_logprobs" not in c for c in calls)


def test_header_declares_prefill_fork():
    assert "nt_lm_prefill_fork" in _lib.EXPORTS
