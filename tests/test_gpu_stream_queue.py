"""GPU: streaming more utterances than slots (``infer_stream_batch`` queue mode) on the H100 engines.

Tiny random LM and codec, as test_gpu_queue.py and test_gpu_facade.py build them.  The tokens each utterance generated
are read back (from ``generate_queue`` where the schedules coincide, else from the engine's ``out_tokens`` row just
before the slot is refilled); the CPU oracles then redo the reference's streaming with them -- every planned window
through the codec oracle, slice, triangular overlap-add -- and the streamed PCM must match within the streaming bar
of test_gpu_facade.py (5e-3 relative RMS)."""
import warnings

import numpy as np
import pytest
import torch

from oracle import codec_oracle as CO
from oracle import lm_oracle as LO
from oracle import stream_oracle as SO
from tests.fakes import AlignedTok, FakePhonemizer
from tests.helpers import make_codec, make_lm

pytestmark = pytest.mark.gpu

MAX_BATCH = 4
F = 25


def _tts(speech_tokens_only=False, seed=7):
    """Facade on a 4-slot engine whose vocabulary is 3072 other ids + 65 536 speech ids (so that the speech range is
    128-aligned), and the tiny codec; returns (tts, codec weights, codec config)."""
    from neutts import NeuTTS

    tok = AlignedTok()
    V = tok.speech_base + 65536
    cfg = LO.LMConfig.tiny(vocab_size=V, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    lm = make_lm(cfg, LO.random_weights(cfg, 3, std=0.05, bf16_round=True), max_batch=MAX_BATCH, max_ctx=2048, max_new=512)
    ccfg = CO.CodecConfig.tiny()
    cw = CO.random_weights(ccfg, 2)
    dec = make_codec(ccfg, cw, max_batch=MAX_BATCH, max_frames=512)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=MAX_BATCH, seed=seed,
                     speech_tokens_only=speech_tokens_only)
    tts.hop_length = ccfg.hop
    tts.streaming_frames_per_chunk = F
    tts.streaming_stride_samples = F * ccfg.hop
    return tts, cw, ccfg


def _stream(tts, texts, refs, rts, stop_after=None, **kw):
    """Streamed PCM per utterance (every yield has one entry per utterance)."""
    got = [[] for _ in texts]
    gen = tts.infer_stream_batch(texts, refs, rts, **kw)
    for k, out in enumerate(gen):
        assert len(out) == len(texts)
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
        if stop_after is not None and k + 1 == stop_after:
            break
    gen.close()
    return [np.concatenate(g) if g else np.zeros(0, np.float32) for g in got]


def _harvest(lm, monkeypatch):
    """Wraps ``lm.prefill_slots`` so that it saves the outgoing occupant's generated ids before each refill; its
    ``stream_ids`` name the utterances.  Returns ``finish()``, which reads the last occupants' rows after the stream
    and gives the ids of every utterance."""
    ids, occ = {}, {s: s for s in range(MAX_BATCH)}
    orig = lm.prefill_slots

    def keep(s):
        ids[occ[s]] = lm.out_tokens[s, : int(lm.n_generated[s])].cpu().long()

    def wrapped(slots, prompts, sp, stream_ids, **kw):
        for s, k in zip(slots, stream_ids):
            keep(s)
            occ[s] = int(k)
        return orig(slots, prompts, sp, stream_ids, **kw)

    monkeypatch.setattr(lm, "prefill_slots", wrapped)

    def finish():
        for s in occ:
            keep(s)
        return ids
    return finish


def _oracle_pcm(tts, ref, gen_ids, cw, ccfg):
    allc = list(ref) + tts._ids_to_codes(gen_ids).tolist()
    frames = []
    for (t0, t1, s0, s1) in SO.chunk_plan(len(ref), len(allc), hop=ccfg.hop, frames=F):
        with torch.no_grad():
            wav = CO.decode_code(torch.tensor(allc[t0:t1])[None, None, :], cw, ccfg)[0, 0].numpy()
        frames.append(wav[s0:s1] if s1 is not None else wav[max(s0, 0):])
    return SO.linear_overlap_add(frames, F * ccfg.hop) if frames else np.zeros(0, np.float32)


def _check_pcm(tag, have, want):
    assert have.shape == want.shape, (tag, have.shape, want.shape)
    if want.size == 0:
        return
    err = float(np.sqrt(np.mean((have - want) ** 2)) / max(np.sqrt(np.mean(want ** 2)), 1e-9))
    print(f"STREAM-QUEUE-PCM {tag}: {want.size} samples, relRMS {err:.2e}")
    assert err < 5e-3, (tag, err)


def _ragged(n, seed):
    """n utterances with ragged texts and reference lengths (so ragged prompts and, through max_context, caps)."""
    rng = np.random.default_rng(seed)
    texts = ["utterance " + "x" * int(rng.integers(1, 60)) for _ in range(n)]
    refs = [rng.integers(0, 65536, int(rng.integers(30, 140))).tolist() for _ in range(n)]
    return texts, refs, ["reference"] * n


def test_stream_queue_coinciding_schedule_matches_generate_queue(cuda):
    """3 x max_batch utterances with equal prompt lengths and equal caps of 40 (EOS stays masked below 50 tokens):
    every slot finishes in the same round, so the stream refills all of them together, exactly as generate_queue
    does.  Each utterance's PCM equals the windowed oracle decode of the tokens generate_queue draws for it."""
    tts, cw, ccfg = _tts(speech_tokens_only=True)
    n = 3 * MAX_BATCH
    rng = np.random.default_rng(1)
    texts = ["utterance %02d" % i for i in range(n)]
    refs = [rng.integers(0, 65536, 60).tolist() for _ in range(n)]
    rts = ["reference"] * n
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    assert len({len(p) for p in prompts}) == 1
    tts.max_context = len(prompts[0]) + 40
    pcm = _stream(tts, texts, refs, rts)
    lm = tts.backbone
    eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
    ids = lm.generate_queue(prompts, eos, max_length=tts.max_context, min_new_tokens=50, seed=tts.seed,
                            vocab_range=tts._speech_range())
    assert [len(i) for i in ids] == [40] * n
    for u in range(n):
        _check_pcm(f"coinciding {u}", pcm[u], _oracle_pcm(tts, refs[u], ids[u], cw, ccfg))
    assert lm.pool.num_free == lm.num_pages


def test_stream_queue_ragged_matches_oracle_and_repeats(cuda, monkeypatch):
    """About 2.5 x max_batch utterances with ragged prompts and caps: each utterance's PCM matches the oracle decode of
    its own tokens, a second run is bit-identical, and every KV page is back in the pool."""
    tts, cw, ccfg = _tts()
    n = 10
    texts, refs, rts = _ragged(n, 4)
    lens = [len(tts._apply_chat_template(c, rt, t)) for t, c, rt in zip(texts, refs, rts)]
    tts.max_context = max(lens) + 60
    caps = [tts.max_context - m for m in lens]
    lm = tts.backbone
    finish = _harvest(lm, monkeypatch)
    pcm = _stream(tts, texts, refs, rts)
    ids = finish()
    assert sorted(ids) == list(range(n))
    assert all(min(50, c) <= len(ids[u]) <= c for u, c in enumerate(caps)), ([len(ids[u]) for u in range(n)], caps)
    assert lm.pool.num_free == lm.num_pages
    for u in range(n):
        _check_pcm(f"ragged {u} ({len(ids[u])} tokens)", pcm[u], _oracle_pcm(tts, refs[u], ids[u], cw, ccfg))
    again = _stream(tts, texts, refs, rts)
    assert all(np.array_equal(a, b) for a, b in zip(pcm, again))
    assert lm.pool.num_free == lm.num_pages


def test_stream_queue_early_close_frees_the_engine(cuda):
    """A consumer that stops after a few chunks: every page is back in the pool, and the next infer_batch on the same
    object is bit-identical to the same call made before the stream."""
    tts, cw, ccfg = _tts()
    texts, refs, rts = _ragged(10, 6)
    tts.max_context = 400
    before = tts.infer_batch(texts[:6], refs[:6], rts[:6])
    pcm = _stream(tts, texts, refs, rts, stop_after=3)
    assert any(p.size for p in pcm)
    lm = tts.backbone
    assert lm.pool.num_free == lm.num_pages
    after = tts.infer_batch(texts[:6], refs[:6], rts[:6])
    assert all(np.array_equal(a, b) for a, b in zip(before, after))


def test_stream_queue_facade_controls_and_speech_tokens_only(cuda, monkeypatch):
    """infer_stream_batch on a list longer than max_batch with per-utterance controls and speech_tokens_only=True:
    every generated id is a speech id or EOS, and each utterance's PCM matches the oracle decode of its tokens."""
    tts, cw, ccfg = _tts(speech_tokens_only=True)
    n = 9
    texts, refs, rts = _ragged(n, 8)
    lens = [len(tts._apply_chat_template(c, rt, t)) for t, c, rt in zip(texts, refs, rts)]
    tts.max_context = max(lens) + 80
    lm = tts.backbone
    finish = _harvest(lm, monkeypatch)
    pcm = _stream(tts, texts, refs, rts, temperature=[0.7 + 0.05 * i for i in range(n)],
                  top_k=[5 + 5 * i for i in range(n)], top_p=[0.9] * n, min_p=[0.0, 0.05] * 4 + [0.0],
                  repetition_penalty=[1.0 + 0.1 * (i % 3) for i in range(n)])
    ids = finish()
    eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
    base = tts.speech_base
    for u in range(n):
        t = ids[u]
        assert len(t) > 0 and bool((((t >= base) & (t < base + 65536)) | (t == eos)).all()), u
        _check_pcm(f"facade {u}", pcm[u], _oracle_pcm(tts, refs[u], t, cw, ccfg))
    assert lm._vocab_range == (base, base + 65536)
    assert lm.pool.num_free == lm.num_pages
