"""CPU: the output resampler's float64 oracle against torchaudio, its streaming contract, the 16-bit rule, the geometry
the library reports, and argument validation (resampler and facade)."""
import math

import numpy as np
import pytest

from oracle import resample_oracle as RO

RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 96000]


def _lengths(sr):
    taps = RO.geometry(sr)[3]
    orig = RO.geometry(sr)[0]
    short = max(1, min(taps - 1, 5))                # shorter than the taps
    odd = 2413 if 2413 % orig else 2411             # not a multiple of orig
    return [1, short, odd, 480 * 37]


@pytest.mark.parametrize("sr", RATES)
def test_oracle_equals_torchaudio(sr):
    torch = pytest.importorskip("torch")
    AF = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(sr)
    for n in _lengths(sr):
        x = rng.standard_normal((2, n))
        want = AF.resample(torch.from_numpy(x), 24000, sr).numpy()
        got = RO.resample(x, sr)
        assert got.shape == want.shape == (2, math.ceil(sr * n / 24000)), (sr, n)
        assert np.abs(got - want).max() <= 1e-12, (sr, n)


def test_table_sizes_of_the_documented_rates():
    sizes = {sr: RO.table(sr).size * 4 for sr in (8000, 16000, 22050, 44100, 48000, 11025)}
    assert sizes == {8000: 164, 16000: 184, 22050: 174 * 147 * 4, 44100: 94 * 147 * 4, 48000: 120, 11025: 348 * 147 * 4}
    assert RO.geometry(11025)[3] - 1 == 347        # the most a stream holds at 11025 Hz


@pytest.mark.parametrize("sr", RATES)
def test_stream_oracle_concatenates_to_one_shot(sr):
    rng = np.random.default_rng(100 + sr)
    orig, new, w, taps = RO.geometry(sr)
    for trial in range(4):
        n = int(rng.integers(1, 6000))
        x = rng.standard_normal(n)
        cuts = np.sort(rng.integers(0, n + 1, int(rng.integers(0, 30))))
        parts = np.split(x, cuts)                   # repeated cuts give empty chunks, close cuts chunks < the hold
        s = RO.Stream(sr)
        outs, received, emitted = [], 0, 0
        for p in parts:
            y = s.push(p)
            received += len(p)
            emitted += len(y)
            # frame k is out exactly when k * orig + w + orig <= received
            assert emitted == new * sum(1 for k in range(received + 1) if k * orig + w + orig <= received)
            assert len(s.held) < taps
            outs.append(y)
        outs.append(s.push(np.zeros(0), final=True))
        got = np.concatenate(outs)
        assert len(got) == math.ceil(sr * n / 24000)
        np.testing.assert_allclose(got, RO.resample(x, sr), rtol=0, atol=1e-12)


def _int16_rule(y):
    """Python's round() of the float32 product: round half to even, computed independently of numpy's rint."""
    y = np.float32(min(max(np.float32(y), np.float32(-1)), np.float32(1)))
    return int(round(float(y * np.float32(32767))))


def test_int16_rule():
    to16 = RO.to_int16
    assert to16([1.0, -1.0, 0.0]).tolist() == [32767, -32767, 0]
    assert to16([1.5, -7.0, 1e30, -1e30]).tolist() == [32767, -32767, 32767, -32767]   # clipped, never wrapped
    halves = []
    for k in range(0, 32767, 97):                   # values whose float32 product lies exactly on k + 0.5
        y = np.float32((k + 0.5) / 32767)
        if float(y * np.float32(32767)) == k + 0.5:
            halves.append((y, k))
    assert {k % 2 for _, k in halves} == {0, 1}
    for y, k in halves:
        want = k if k % 2 == 0 else k + 1
        assert to16([y]).tolist() == [want] and to16([-y]).tolist() == [-want], (y, k)
    rng = np.random.default_rng(3)
    y = (rng.standard_normal(20000) * 0.6).astype(np.float32)
    got = to16(y)
    assert got.dtype == np.int16
    assert got.tolist() == [_int16_rule(v) for v in y]
    # unlike the truncating (y * 32767).astype(np.int16) of a host conversion
    assert to16([0.99999]).tolist() == [32767] and int((np.float32(0.99999) * 32767).astype(np.int16)) == 32766


def test_library_geometry_matches_the_oracle():
    from neutts_air_b200.resample import check_args

    for sr in RATES:
        info = check_args(sr)
        assert (info.orig, info.target, info.width, info.taps) == RO.geometry(sr), sr
        assert info.table_bytes >= RO.table(sr).size * 4 and info.row_bytes >= 8 * info.taps


@pytest.mark.parametrize("bad", [16000.0, True, 0, -8000, "16000", None])
def test_rejects_bad_rates(bad):
    from neutts_air_b200.resample import Resampler

    with pytest.raises(ValueError, match="positive integer"):
        Resampler(bad)


def test_rejects_oversize_table_and_unknown_format():
    from neutts_air_b200.resample import Resampler

    with pytest.raises(ValueError, match="232448 bytes"):
        Resampler(44056)                           # gcd 8: 5507 phases of 3014 taps, a 66 MB table
    with pytest.raises(ValueError, match="pcm_format"):
        Resampler(16000, pcm_format="int8")


def test_facade_validates_output_arguments():
    from neutts import NeuTTS
    from tests.fakes import FakeBackbone, FakeCodec, FakePhonemizer, FakeTokenizer

    kw = dict(tokenizer=FakeTokenizer(), phonemizer=FakePhonemizer(), backbone=FakeBackbone([1]), codec=FakeCodec())
    for bad in (dict(sample_rate=44056), dict(sample_rate=16000.0), dict(sample_rate=0), dict(sample_rate=True),
                dict(pcm_format="int8"), dict(sample_rate=16000, pcm_format="float64")):
        with pytest.raises(ValueError):
            NeuTTS(**kw, **bad)
    tts = NeuTTS(**kw, sample_rate=16000, pcm_format="int16")
    assert (tts.sample_rate, tts.pcm_format) == (16000, "int16")


def test_facade_default_rate_is_24k():
    from neutts import NeuTTS
    from tests.fakes import FakeBackbone, FakeCodec, FakePhonemizer, FakeTokenizer

    tts = NeuTTS(tokenizer=FakeTokenizer(), phonemizer=FakePhonemizer(), backbone=FakeBackbone([1]), codec=FakeCodec())
    assert (tts.sample_rate, tts.pcm_format) == (24000, "float32")
    assert tts._output_resampler() is None
