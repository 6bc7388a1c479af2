"""GPU: long-form synthesis (``long_form=True``) on the tiny engines of tests/helpers.py, at a fixed seed.  A text that
fits is one segment and comes back bit for bit as without ``long_form``; texts of 2-4 segments (a short
``max_context``), more of them than slots, equal the seam join of ``infer_batch`` / ``infer_stream_batch`` over the
round-robin flattened segments, bit for bit, in float32 24 kHz, int16 16 kHz and with per-text speeds."""
import warnings

import numpy as np
import pytest
import torch

from neutts_air_b200 import longform as LF
from tests.helpers import _tts

pytestmark = pytest.mark.gpu

TEXTS = ["The first text has a sentence. It has another one, and a clause! A third sentence closes it.",
         "Short one here. Then a second sentence follows it, slowly.",
         "Line one of three.\nLine two of three.\nLine three, the last.",
         "Are you there? Yes. No. Maybe, perhaps, who knows; we will see - later. Bye.",
         "One more text, long enough to need two segments at least, or it would not count."]
RT = "reference voice"


def _pair(sr=24000, fmt="float32", max_batch=2, max_context=260):
    """The tiny facade and a second one on the same engines with another output format."""
    from neutts import NeuTTS

    tts, ccfg = _tts(max_batch=max_batch)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        other = NeuTTS(tokenizer=tts.tokenizer, phonemizer=tts.phonemizer, backbone=tts.backbone, codec=tts.codec,
                       max_batch=max_batch, seed=tts.seed, sample_rate=sr, pcm_format=fmt)
    for t in (tts, other):
        t.watermarker = None
        t.max_context = max_context
        t.hop_length = ccfg.hop
        t.streaming_stride_samples = t.streaming_frames_per_chunk * ccfg.hop
    return tts, other


def _refs(n=len(TEXTS)):
    rng = np.random.default_rng(4)
    return [torch.from_numpy(rng.integers(0, 1024, int(rng.integers(30, 50)))) for _ in range(n)], [RT] * n


def _flat(tts, texts, refs, rts):
    """(owner of each flattened segment, segment texts, their refs and ref texts) in round-robin order."""
    segs = [tts.segments(t, c, rt) for t, c, rt in zip(texts, refs, rts)]
    order = LF.round_robin([len(s) for s in segs])
    return ([t for t, _ in order], [segs[t][k] for t, k in order], [refs[t] for t, _ in order],
            [rts[t] for t, _ in order], segs)


def _joined(tts, owners, per_segment, n, pause=0.0):
    return [LF.join([per_segment[j] for j, o in enumerate(owners) if o == t], tts.sample_rate, pause) for t in range(n)]


def _stream_cat(gen, n):
    got = [[] for _ in range(n)]
    for out in gen:
        assert len(out) == n
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
    return [np.concatenate(g) for g in got]


# ------------------------------------------------------------------------------------------------- every text fits
def test_texts_that_fit_are_unchanged(cuda):
    tts, _ = _pair(max_context=2048)
    refs, rts = _refs()
    assert all(tts.segments(t, c, rt) == [t] for t, c, rt in zip(TEXTS, refs, rts))
    a = tts.infer(TEXTS[0], refs[0], RT)
    assert np.array_equal(tts.infer(TEXTS[0], refs[0], RT, long_form=True, pause=1.0), a)
    plain = tts.infer_batch(TEXTS, refs, rts, temperature=[0.8, 1.0, 1.2, 0.9, 1.1])
    got = tts.infer_batch(TEXTS, refs, rts, temperature=[0.8, 1.0, 1.2, 0.9, 1.1], long_form=True)
    assert all(np.array_equal(x, y) for x, y in zip(got, plain))
    plain = list(tts.infer_stream_batch(TEXTS, refs, rts))
    got = list(tts.infer_stream_batch(TEXTS, refs, rts, long_form=True, pause=0.5))
    assert len(got) == len(plain)
    for a, b in zip(got, plain):
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))
    one = list(tts.infer_stream(TEXTS[1], refs[1], RT))
    assert [c.tobytes() for c in tts.infer_stream(TEXTS[1], refs[1], RT, long_form=True)] == [c.tobytes() for c in one]


# ------------------------------------------------------------------------------------------------- several segments
@pytest.mark.parametrize("fmt", ["f32-24k", "i16-16k", "speeds"])
def test_long_texts_equal_the_join_of_their_segments(cuda, fmt):
    tts, t16 = _pair(16000, "int16")
    t = t16 if fmt == "i16-16k" else tts
    refs, rts = _refs()
    owners, flat, frefs, frts, segs = _flat(t, TEXTS, refs, rts)
    assert all(2 <= len(s) <= 5 for s in segs) and len(flat) > t.max_batch
    kw = dict(speed=[0.75, 1.0, 1.25, 1.0, 1.5]) if fmt == "speeds" else {}
    flat_kw = {k: [v[o] for o in owners] for k, v in kw.items()}
    per_seg = t.infer_batch(flat, frefs, frts, **flat_kw)
    for pause in (0.0, 0.125):
        got = t.infer_batch(TEXTS, refs, rts, long_form=True, pause=pause, **kw)
        want = _joined(t, owners, per_seg, len(TEXTS), pause)
        for g, w in zip(got, want):
            assert g.dtype == (np.int16 if fmt == "i16-16k" else np.float32) and np.array_equal(g, w)
    one = t.infer(TEXTS[0], refs[0], RT, long_form=True, **{k: v[0] for k, v in kw.items()})
    alone = t.infer_batch(segs[0], [refs[0]] * len(segs[0]), [RT] * len(segs[0]),
                          **{k: v[0] for k, v in kw.items()})
    assert np.array_equal(one, LF.join(alone, t.sample_rate))


@pytest.mark.parametrize("fmt", ["f32-24k", "i16-16k"])
def test_long_streams_equal_the_join_of_their_segment_streams(cuda, fmt):
    tts, t16 = _pair(16000, "int16")
    t = t16 if fmt == "i16-16k" else tts
    refs, rts = _refs()
    owners, flat, frefs, frts, segs = _flat(t, TEXTS, refs, rts)
    per_seg = _stream_cat(t.infer_stream_batch(flat, frefs, frts), len(flat))
    got = _stream_cat(t.infer_stream_batch(TEXTS, refs, rts, long_form=True, pause=0.05), len(TEXTS))
    for g, w in zip(got, _joined(t, owners, per_seg, len(TEXTS), 0.05)):
        assert np.array_equal(g, w)
    alone = _stream_cat(t.infer_stream_batch(segs[2], [refs[2]] * len(segs[2]), [RT] * len(segs[2])), len(segs[2]))
    one = np.concatenate(list(t.infer_stream(TEXTS[2], refs[2], RT, long_form=True)))
    assert np.array_equal(one, LF.join(alone, t.sample_rate))


def test_closing_a_long_stream_early_frees_every_page(cuda):
    tts, _ = _pair()
    refs, rts = _refs()
    lm = tts.backbone
    gen = tts.infer_stream_batch(TEXTS, refs, rts, long_form=True)
    for k, _ in enumerate(gen):
        if k == 2:
            break
    gen.close()
    assert lm.pool.num_free == lm.num_pages
    gen = tts.infer_stream(TEXTS[0], refs[0], RT, long_form=True)
    next(gen)
    gen.close()
    assert lm.pool.num_free == lm.num_pages


def test_logprob_rows_concatenate_per_text(cuda):
    tts, _ = _pair()
    refs, rts = _refs()
    owners, flat, frefs, frts, _ = _flat(tts, TEXTS, refs, rts)
    wavs, lps = tts.infer_batch(flat, frefs, frts, return_logprobs=True)
    got_w, got_lp = tts.infer_batch(TEXTS, refs, rts, long_form=True, return_logprobs=True)
    for t in range(len(TEXTS)):
        js = [j for j, o in enumerate(owners) if o == t]
        assert np.array_equal(got_lp[t], np.concatenate([lps[j] for j in js]))
        assert np.array_equal(got_w[t], LF.join([wavs[j] for j in js], tts.sample_rate))
