"""GPU: the output resampler (resample.cu) against the float64 oracle, streams against one-shot calls bit for bit, the
fused 16-bit conversion, and the facade's sample_rate / pcm_format on the tiny engines."""
import warnings

import numpy as np
import pytest
import torch

from oracle import resample_oracle as RO
from tests.helpers import _tts

pytestmark = pytest.mark.gpu

RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 96000]


def _rs(sr, fmt="float32", rows=1):
    from neutts_air_b200.resample import Resampler

    return Resampler(sr, fmt, device="cuda:0", max_rows=rows)


@pytest.mark.parametrize("sr", RATES)
def test_kernel_matches_oracle(cuda, sr):
    rng = np.random.default_rng(sr)
    x = (rng.standard_normal((3, 4801)) * 0.3).astype(np.float32)
    got = _rs(sr).resample(torch.from_numpy(x).to(cuda)).cpu().numpy().astype(np.float64)
    want = RO.resample(x.astype(np.float64), sr)
    assert got.shape == want.shape
    rel = float(np.sqrt(np.mean((got - want) ** 2) / np.mean(want ** 2)))
    mx = float(np.abs(got - want).max()) / float(np.abs(x).max())
    print(f"RESAMPLE-ACCURACY {sr} Hz: relRMS {rel:.2e}, max abs / max|x| {mx:.2e}")
    assert rel <= 1e-6 and mx <= 1e-5, (sr, rel, mx)


def test_ragged_rows_in_one_launch(cuda):
    rs = _rs(22050, rows=5)
    rng = np.random.default_rng(1)
    xs = [(rng.standard_normal(n) * 0.3).astype(np.float32) for n in (1, 90, 173, 4000, 0)]
    got = rs.push(range(5), xs, final=True)
    for x, y in zip(xs, got):
        assert len(y) == RO.out_len(len(x), 22050)
        if len(x):
            assert np.abs(y - RO.resample(x.astype(np.float64), 22050)).max() <= 1e-5 * np.abs(x).max()
            assert np.array_equal(y, rs.resample(torch.from_numpy(x).to(cuda)).cpu().numpy())


@pytest.mark.parametrize("sr", [8000, 11025, 16000, 22050, 44100, 48000])
@pytest.mark.parametrize("fmt", ["float32", "int16"])
def test_chunked_pushes_are_bit_identical_to_one_shot(cuda, sr, fmt):
    rows = 4
    rs = _rs(sr, fmt, rows=rows)
    rng = np.random.default_rng(7 + sr)
    xs = [(rng.standard_normal(int(rng.integers(1, 9000))) * 0.5).astype(np.float32) for _ in range(rows)]
    cuts = [np.split(x, np.sort(rng.integers(0, len(x) + 1, 25))) for x in xs]   # empty and short chunks included
    outs, nxt = [[] for _ in range(rows)], [0] * rows
    for step in range(26):
        live = [r for r in range(rows) if step == 25 or rng.random() < 0.8]   # a row left out keeps its stream
        chunks = []
        for r in live:
            chunks.append(np.concatenate(cuts[r][nxt[r]: step + 1]))
            nxt[r] = step + 1
        for r, y in zip(live, rs.push(live, chunks, final=step == 25)):
            outs[r].append(y)
    for r in range(rows):
        y = np.concatenate(outs[r])
        one = rs.resample(torch.from_numpy(xs[r]).to(cuda)).cpu().numpy()
        assert y.dtype == one.dtype and len(y) == RO.out_len(len(xs[r]), sr)
        assert np.array_equal(y, one), (sr, fmt, r)


@pytest.mark.parametrize("sr", [16000, 24000, 48000])
def test_int16_is_the_oracle_conversion_of_the_float_output(cuda, sr):
    rng = np.random.default_rng(sr)
    x = torch.from_numpy((rng.standard_normal((2, 5000)) * 0.7).astype(np.float32)).to(cuda)   # ~15% beyond +-1
    y32 = _rs(sr).resample(x).cpu().numpy()
    y16 = _rs(sr, "int16").resample(x).cpu().numpy()
    assert y16.dtype == np.int16 and (np.abs(y32) > 1).any()
    assert np.array_equal(y16, RO.to_int16(y32))


def test_wrong_spans_and_rows_are_refused(cuda):
    import ctypes as C

    from neutts_air_b200 import _lib

    rs = _rs(16000, rows=2)
    with pytest.raises(ValueError):
        rs.push([0, 0], [np.zeros(10), np.zeros(10)])
    with pytest.raises(ValueError):
        rs.push([2], [np.zeros(10)])
    x = torch.zeros(10, device=cuda)
    out = torch.empty(100, device=cuda)
    off = (C.c_int64 * 2)(0, 10)
    bad = (C.c_int64 * 2)(0, 99)                           # a span the contract does not give
    rc = rs.L.nt_resampler_push(rs.handle, 1, (C.c_int32 * 1)(0), None, x.data_ptr(), off, out.data_ptr(), bad, None)
    assert rc == -1 and b"span" in rs.L.nt_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)


# ------------------------------------------------------------------------------------------------------------ facade
def _pair(sr, fmt="float32", max_batch=2):
    """A 24 kHz facade and one at (sr, fmt) on the same engines and seed."""
    from neutts import NeuTTS

    tts, ccfg = _tts(max_batch=max_batch)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        other = NeuTTS(tokenizer=tts.tokenizer, phonemizer=tts.phonemizer, backbone=tts.backbone, codec=tts.codec,
                       max_batch=max_batch, seed=tts.seed, sample_rate=sr, pcm_format=fmt)
    for t in (tts, other):
        t.watermarker = None
        t.max_context = 400
        t.hop_length = ccfg.hop
        t.streaming_stride_samples = t.streaming_frames_per_chunk * ccfg.hop
    return tts, other


def _inputs(n):
    rng = np.random.default_rng(n)
    return (["utterance " + "x" * int(rng.integers(1, 30)) for _ in range(n)],
            [torch.from_numpy(rng.integers(0, 1024, int(rng.integers(20, 60)))) for _ in range(n)], ["reference"] * n)


def _at(rate_fmt, wav):
    rs = _rs(*rate_fmt)
    return rs.resample(torch.from_numpy(np.asarray(wav, np.float32)).cuda()).cpu().numpy()


def test_facade_infer_and_batch_equal_resampled_24k(cuda):
    tts, t16 = _pair(16000)
    assert t16.sample_rate == 16000
    texts, refs, rts = _inputs(5)                           # 5 utterances on 2 slots: the queue
    a = tts.infer(texts[0], refs[0], rts[0])
    b = t16.infer(texts[0], refs[0], rts[0])
    assert b.dtype == np.float32 and np.array_equal(b, _at((16000,), a))
    w24 = tts.infer_batch(texts, refs, rts)
    w16 = t16.infer_batch(texts, refs, rts)
    assert len(w16) == 5
    for x, y in zip(w24, w16):
        assert len(y) == RO.out_len(len(x), 16000) and np.array_equal(y, _at((16000,), x))
    d = t16._decode(list(range(30)))
    assert np.array_equal(d, _at((16000,), tts._decode(list(range(30)))))


def _stream_cat(gen, n):
    got = [[] for _ in range(n)]
    for out in gen:
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
    return [np.concatenate(g) for g in got]


@pytest.mark.parametrize("sr,fmt", [(16000, "float32"), (44100, "int16")])
def test_facade_streams_equal_one_shot_of_the_24k_stream(cuda, sr, fmt):
    tts, other = _pair(sr, fmt)
    texts, refs, rts = _inputs(5)
    one24 = np.concatenate(list(tts.infer_stream(texts[0], refs[0], rts[0])))
    one = np.concatenate(list(other.infer_stream(texts[0], refs[0], rts[0])))
    assert one.dtype == np.dtype(fmt) and np.array_equal(one, _at((sr, fmt), one24))
    s24 = _stream_cat(tts.infer_stream_batch(texts, refs, rts), 5)        # queue: 5 utterances on 2 slots
    s = _stream_cat(other.infer_stream_batch(texts, refs, rts), 5)
    for x, y in zip(s24, s):
        assert np.array_equal(y, _at((sr, fmt), x))


@pytest.mark.parametrize("sr", [24000, 48000])
def test_facade_int16(cuda, sr):
    tts, t16 = _pair(sr, "int16")
    texts, refs, rts = _inputs(3)
    w = tts.infer_batch(texts, refs, rts)
    got = t16.infer_batch(texts, refs, rts)
    for x, y in zip(w, got):
        assert y.dtype == np.int16
        want = RO.to_int16(x) if sr == 24000 else _at((sr, "int16"), x)
        assert np.array_equal(y, want)


class _StubMark:
    """Watermark stand-in: scales the waveform and records the rate and lengths it saw."""

    def __init__(self):
        self.seen = []

    def apply_watermark(self, wav, sample_rate):
        self.seen.append((sample_rate, len(wav)))
        return (np.asarray(wav, np.float32) * np.float32(0.5) + np.float32(0.01)).astype(np.float32)


def test_watermark_is_applied_at_24k_before_resampling(cuda):
    tts, t16 = _pair(16000)
    texts, refs, rts = _inputs(3)
    tts.watermarker, t16.watermarker = _StubMark(), _StubMark()
    w24 = tts.infer_batch(texts, refs, rts)                 # watermarked at 24 kHz
    w16 = t16.infer_batch(texts, refs, rts)
    assert t16.watermarker.seen == tts.watermarker.seen and all(r == 24000 for r, _ in t16.watermarker.seen)
    for x, y in zip(w24, w16):
        assert np.array_equal(y, _at((16000,), x))


def test_early_close_leaves_the_resampler_reusable(cuda):
    _, t16 = _pair(22050)
    texts, refs, rts = _inputs(4)
    full = _stream_cat(t16.infer_stream_batch(texts, refs, rts), 4)
    gen = t16.infer_stream_batch(texts, refs, rts)
    next(gen)
    gen.close()
    again = _stream_cat(t16.infer_stream_batch(texts, refs, rts), 4)
    assert all(np.array_equal(a, b) for a, b in zip(full, again))
