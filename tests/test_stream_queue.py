"""CPU: streaming synthesis of more utterances than slots (``infer_stream_batch`` queue mode) on a stub engine.

The stub keeps ``SpeechLM``'s slot semantics: one scripted token stream per Philox stream id, finished slots idle,
per-slot caps, ``prefill_slots`` refills chosen slots while the others keep decoding, and KV pages are held per slot
until released.  Every utterance's streamed audio must equal the reference's single-utterance window procedure
(oracle/stream_oracle.py) over its own reference and generated codes, whatever slot it ran in and whenever it was
admitted."""
import numpy as np
import pytest
import torch

from oracle import stream_oracle as SO
from tests.fakes import BatchRampCodec, FakeBatchStreamLM, RampCodec, _tts


class QueueStreamLM:
    """``SpeechLM``'s prefill / prefill_slots / decode / release_pages / per-slot settings surface on scripted tokens.
    ``scripts[k]``: the tokens stream k emits (EOS after its end).  Every engine call is appended to ``log``."""
    device = torch.device("cpu")

    def __init__(self, scripts, max_batch, log, max_new=4096):
        self.scripts, self.max_batch, self.max_new, self.log = scripts, max_batch, max_new, log
        self.out_tokens = torch.zeros(max_batch, max_new, dtype=torch.int32)
        self.n_generated = torch.zeros(max_batch, dtype=torch.int32)
        self.done = torch.zeros(max_batch, dtype=torch.int32)
        self.stream = [None] * max_batch
        self.held = set()            # slots holding KV pages
        self.admitted = []           # (slot, stream id, controls row, penalty row) at every admission
        self._slot_sp_host = None
        self._penalty_host = None
        self.B = 0

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, limits=None):
        self.eos = eos
        self.limits = [max_new] * self.max_batch
        if limits is not None:
            self.limits[: len(limits)] = list(limits)
        self.log.append(("sampling", None if limits is None else list(limits)))

    def _table(self, name, default, rows, slots):
        if rows is None:
            setattr(self, name, None)
            return
        table = list(getattr(self, name) or [default] * self.max_batch)
        for s, r in zip(range(len(rows)) if slots is None else slots, rows):
            table[s] = tuple(r)
        setattr(self, name, table)

    def set_slot_sampling(self, rows, slots=None):
        self.log.append(("set_slot_sampling", None if slots is None else list(slots)))
        self._table("_slot_sp_host", (1.0, 50, 1.0, 0.0), rows, slots)

    def set_repetition_penalty(self, rows, slots=None):
        self.log.append(("set_repetition_penalty", None if slots is None else list(slots)))
        self._table("_penalty_host", (1.0, True), rows, slots)

    def _seat(self, s, k):
        self.out_tokens[s].zero_()
        self.n_generated[s] = 0
        self.done[s] = 0
        self.stream[s] = k
        self.held.add(s)
        sp = self._slot_sp_host[s] if self._slot_sp_host else None
        pen = self._penalty_host[s] if self._penalty_host else None
        self.admitted.append((s, k, sp, pen))

    def _emit(self, slots):
        for s in slots:
            n = int(self.n_generated[s])
            if self.stream[s] is None or int(self.done[s]) or n >= self.limits[s]:
                continue
            script = self.scripts[self.stream[s]]
            tok = script[n] if n < len(script) else self.eos
            self.out_tokens[s, n] = tok
            self.n_generated[s] = n + 1
            if tok == self.eos or n + 1 >= self.limits[s]:
                self.done[s] = 1

    def live(self):
        return [s for s in range(self.B) if self.stream[s] is not None and not int(self.done[s])]

    def prefill(self, prompts, sp):
        assert 1 <= len(prompts) <= self.max_batch
        self.log.append(("prefill", len(prompts)))
        self.held.clear()
        self.stream = [None] * self.max_batch
        for s in range(len(prompts)):
            self._seat(s, s)
        self.B = len(prompts)
        self._emit(range(self.B))

    def prefill_slots(self, slots, prompts, sp, stream_ids, limits=None):
        assert len(slots) == len(prompts) == len(stream_ids) and limits is not None
        self.log.append(("prefill_slots", list(slots), list(stream_ids), list(limits)))
        for s, k, cap in zip(slots, stream_ids, limits):
            self.limits[s] = min(int(cap), self.max_new)
            self._seat(s, k)
        self.B = max(self.B, max(slots) + 1)
        self._emit(slots)

    def decode(self, steps, sp):
        assert steps >= 1
        self.log.append(("decode", steps, len(self.live())))
        for _ in range(steps):
            self._emit(range(self.B))

    def release_pages(self, slots=None):
        self.log.append(("release_pages",))
        self.held -= set(range(self.max_batch) if slots is None else slots)


def _case(tts, tok, n, seed, cap1=(), gen_len=None, max_new=4096):
    """n utterances with ragged references, ragged generated lengths (some past their cap; all ``gen_len`` when
    given, without junk), junk ids, caps from ``max_context`` (the utterances in ``cap1`` get a cap of 1) -> (refs, scripts, caps)."""
    rng = np.random.default_rng(seed)
    overhead = len(tts._apply_chat_template([], "ref", "hello"))
    tts.max_context = overhead + 130 + 250
    refs, scripts = [], []
    for i in range(n):
        m = tts.max_context - 1 - overhead if i in cap1 else int(rng.integers(40, 131))
        refs.append(rng.integers(0, 65536, m).tolist())
        sc = []
        junk = 0 if gen_len else int(rng.integers(0, 6))
        for j, c in enumerate(rng.integers(0, 65536, gen_len or int(rng.integers(3, 420))).tolist()):
            if junk and j % junk == 0:
                sc.append(65 if j % 2 else tok.speech_base + 70000)   # text id / id past the codebook: dropped
            sc.append(tok.speech_base + c)
        scripts.append(sc)
    caps = [min(tts.max_context - len(tts._apply_chat_template(r, "ref", "hello")), max_new) for r in refs]
    return refs, scripts, caps


def _expected(tts, tok, codec, ref, script, cap, F):
    kept = [t - tok.speech_base for t in script[:cap] if 0 <= t - tok.speech_base < 65536]
    allc = ref + kept
    frames = []
    for (t0, t1, s0, s1) in SO.chunk_plan(len(ref), len(allc), hop=codec.hop, frames=F):
        wav = RampCodec.decode_code(codec, torch.tensor(allc[t0:t1])[None, None, :])[0, 0].numpy()
        frames.append(wav[s0:s1] if s1 is not None else wav[max(s0, 0):])
    return SO.linear_overlap_add(frames, F * codec.hop) if frames else np.zeros(0, np.float32)


def _setup(F, n, seed, log, cap1=(), gen_len=None, max_new=4096):
    """The facade on ``QueueStreamLM`` (MAX_BATCH slots) and the ramp codec, with ``_case``'s utterances."""
    tts, tok = _tts()
    codec = BatchRampCodec()
    tts.codec, tts.hop_length = codec, codec.hop
    tts.streaming_frames_per_chunk = F
    tts.streaming_stride_samples = F * codec.hop
    tts.max_batch = MAX_BATCH
    refs, scripts, caps = _case(tts, tok, n, seed, cap1, gen_len, max_new)
    lm = QueueStreamLM(scripts, MAX_BATCH, log, max_new)
    tts.backbone = lm
    return tts, tok, codec, lm, refs, scripts, caps


def _consume(tts, n, refs, log, limit_yields=None, **kw):
    got = [[] for _ in range(n)]
    gen = tts.infer_stream_batch(["hello"] * n, refs, ["ref"] * n, **kw)
    for k, out in enumerate(gen):
        assert len(out) == n and any(o is not None for o in out)
        log.append(("yield", [u for u, o in enumerate(out) if o is not None]))
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
        if limit_yields is not None and k + 1 == limit_yields:
            break
    gen.close()
    return got


MAX_BATCH = 4


@pytest.mark.parametrize("F", [25, 50])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 9, 14])
def test_stream_queue_matches_reference_window_plan_per_utterance(n, F):
    """Every utterance's audio equals the reference procedure over its own codes; the call log shows FIFO admission,
    stream id = utterance index, the newcomers' caps, refills only after the previous occupant's last chunk went out,
    bounded launches with a live slot each, and every page given back."""
    log = []
    tts, tok, codec, lm, refs, scripts, caps = _setup(F, n, 100 * n + F, log, cap1={1, MAX_BATCH + 2})
    assert n < 2 or caps[1] == 1
    got = _consume(tts, n, refs, log)
    for u in range(n):
        want = _expected(tts, tok, codec, refs[u], scripts[u], caps[u], F)
        have = np.concatenate(got[u]) if got[u] else np.zeros(0, np.float32)
        assert have.shape == want.shape, (u, have.shape, want.shape)
        assert np.abs(have - want).max(initial=0) < 1e-5, u
    S = min(n, MAX_BATCH)
    refills = [e for e in log if e[0] == "prefill_slots"]
    assert [e for e in log if e[0] == "prefill"] == [("prefill", S)]
    assert log[[e[0] for e in log].index("sampling")][1] == (caps[:S] if n > MAX_BATCH else
                                                              (None if min(caps) == max(caps) else caps))
    if n <= MAX_BATCH:
        assert not refills and ("release_pages",) not in log   # the lock-step path makes the same calls as before
    else:
        assert [k for e in refills for k in e[2]] == list(range(S, n))          # FIFO; stream id = utterance index
        assert all(e[3] == [caps[k] for k in e[2]] for e in refills)            # each newcomer's own cap
        assert log[-1] == ("release_pages",) and not lm.held
    # a slot is refilled only after the last chunk of the utterance it held has been yielded
    occupant = {s: s for s in range(S)}
    last_yield = {u: max((i for i, e in enumerate(log) if e[0] == "yield" and u in e[1]), default=-1) for u in range(n)}
    for i, e in enumerate(log):
        if e[0] == "prefill_slots":
            for s, k in zip(e[1], e[2]):
                assert last_yield[occupant[s]] < i, (s, occupant[s], k)
                occupant[s] = k
    decodes = [e for e in log if e[0] == "decode"]
    assert decodes and all(1 <= e[1] <= F + tts.streaming_lookforward and e[2] >= 1 for e in decodes)
    assert {k for _, k, _, _ in lm.admitted} == set(range(n))


@pytest.mark.parametrize("n", [4, 9])
def test_stream_caps_at_the_engine_max_new(n):
    """Caps set by the engine's max_new (the width of out_tokens) on some utterances while others still decode, on
    the lock-step path and in the queue."""
    log = []
    tts, tok, codec, lm, refs, scripts, caps = _setup(25, n, 11, log, gen_len=400, max_new=300)
    assert min(caps) < 300 == max(caps)
    got = _consume(tts, n, refs, log)
    for u in range(n):
        want = _expected(tts, tok, codec, refs[u], scripts[u], caps[u], 25)
        have = np.concatenate(got[u]) if got[u] else np.zeros(0, np.float32)
        assert have.shape == want.shape and np.abs(have - want).max(initial=0) < 1e-5, u


def test_stream_queue_reads_a_cap_of_one_newcomer_before_decoding():
    """The first wave ends together and the one newcomer has a cap of 1: it is done inside its prefill, so the next
    round reads it (and sends its tail) without a decode launch over no live slot."""
    log = []
    tts, tok, codec, lm, refs, scripts, caps = _setup(25, MAX_BATCH + 1, 3, log, cap1={MAX_BATCH}, gen_len=40)
    got = _consume(tts, MAX_BATCH + 1, refs, log)
    assert caps[MAX_BATCH] == 1 and [e[2] for e in log if e[0] == "prefill_slots"] == [[MAX_BATCH]]
    assert all(e[2] >= 1 for e in log if e[0] == "decode")
    i = [e[0] for e in log].index("prefill_slots")
    assert "decode" not in [e[0] for e in log[i:]]
    for u in range(MAX_BATCH + 1):
        want = _expected(tts, tok, codec, refs[u], scripts[u], caps[u], 25)
        have = np.concatenate(got[u]) if got[u] else np.zeros(0, np.float32)
        assert have.shape == want.shape and np.abs(have - want).max(initial=0) < 1e-5, u


def test_stream_queue_per_utterance_settings_follow_their_utterances():
    """Per-utterance control and penalty lists: every slot holds its utterance's row when that utterance is admitted,
    written by ``set_slot_sampling`` / ``set_repetition_penalty`` for exactly the refilled slots."""
    n, log = 11, []
    tts, tok, codec, lm, refs, scripts, caps = _setup(25, n, 5, log)
    temps = [0.5 + 0.1 * i for i in range(n)]
    top_k = [1 + 5 * i for i in range(n)]
    pens = [1.0 + 0.05 * i for i in range(n)]
    keep_prompt = [i % 2 == 0 for i in range(n)]
    _consume(tts, n, refs, log, temperature=temps, top_k=top_k, repetition_penalty=pens, penalize_prompt=keep_prompt)
    assert sorted(k for _, k, _, _ in lm.admitted) == list(range(n))
    for s, k, sp, pen in lm.admitted:
        assert sp == (pytest.approx(temps[k]), top_k[k], 1.0, 0.0), (s, k, sp)
        assert pen == (pytest.approx(pens[k]), keep_prompt[k]), (s, k, pen)
    refills = [e for e in log if e[0] == "prefill_slots"]
    for name in ("set_slot_sampling", "set_repetition_penalty"):
        calls = [e[1] for e in log if e[0] == name]
        assert calls[0] is None and calls[1:] == [e[1] for e in refills]   # apply() for slots 0..S-1, then per refill


def test_stream_queue_needs_prefill_slots():
    """A backbone that cannot refill a slot rejects a list longer than its slots before any engine call."""
    class NoRefill(FakeBatchStreamLM):
        max_batch = 2

        def sampling(self, *a, **kw):
            raise AssertionError("engine call")

        def prefill(self, *a, **kw):
            raise AssertionError("engine call")

    tts, tok = _tts()
    lm = NoRefill([[tok.speech_base + 1]] * 3)
    tts.backbone = lm
    with pytest.raises(ValueError, match="prefill_slots"):
        tts.infer_stream_batch(["a", "b", "c"], [[1, 2]] * 3, ["r"] * 3)
    with pytest.raises(ValueError, match="prefill_slots"):
        next(tts._stream_batch([[1, 2, 3]] * 3, [[1, 2]] * 3))
    assert lm.decode_calls == []


def test_stream_queue_early_close_releases_pages():
    """A consumer that stops after a few chunks gets every page back, and the next stream on the engine is whole."""
    n, log = 10, []
    tts, tok, codec, lm, refs, scripts, caps = _setup(25, n, 9, log)
    _consume(tts, n, refs, log, limit_yields=3)
    assert sum(e[0] == "yield" for e in log) == 3 and log[-1] == ("release_pages",) and not lm.held
    got = _consume(tts, n, refs, log)
    for u in range(n):
        want = _expected(tts, tok, codec, refs[u], scripts[u], caps[u], 25)
        have = np.concatenate(got[u]) if got[u] else np.zeros(0, np.float32)
        assert have.shape == want.shape and np.abs(have - want).max(initial=0) < 1e-5, u
    assert not lm.held
