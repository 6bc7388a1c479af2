"""GPU: the loudness meter and normaliser (loudness.cu) against the float64 oracle at every rate, at the lengths where
blocks begin and end, up to the longest stretched utterance, in ragged batches of 1..64 rows, bit for bit across runs;
and the facade's ``loudness`` on tiny engines whose codec has NeuCodec's 480-sample hop, so that utterances are longer
than one 400 ms gating block."""
import warnings

import numpy as np
import pytest
import torch

from neutts_air_b200 import longform as LF
from oracle import codec_oracle, lm_oracle
from oracle import loudness_oracle as LO
from tests.helpers import make_codec, make_lm

pytestmark = pytest.mark.gpu

RATES = [16000, 22050, 24000, 44100, 48000]
LONGEST = 2048 * 480 * 2     # the longest stretched utterance: 2048 frames at speed 0.5


def _program(r, n, seed, span=2.5, silences=True, peak=0.25):
    """Noise under a level that changes every 100 ms over `span` decades, optionally with silent stretches."""
    rng = np.random.default_rng(seed)
    step = r // 10
    x = rng.standard_normal(n) * np.repeat(10 ** rng.uniform(-span, 0, n // step + 1), step)[:n]
    if silences and n > 10 * step:
        x[n // 5: n // 5 + 3 * step] = 0
        x[int(0.7 * n):int(0.7 * n) + 7 * step] = 0
    return (x / max(np.abs(x).max(), 1e-30) * peak).astype(np.float32)


def _measure(rows, r=24000):
    from neutts_air_b200.loudness import measure

    return measure([torch.from_numpy(x).cuda() for x in rows], r)


def _same(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a[~np.isnan(a)], b[~np.isnan(b)], atol=1e-8, rtol=0)


def _ulps(got, want):
    """Largest distance in float32 units in the last place (both arrays float32)."""
    return int(np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max(initial=0))


# ------------------------------------------------------------------------------------------------- meter
@pytest.mark.parametrize("r", RATES)
def test_measure_matches_float64_at_every_rate(cuda, r):
    gate, step = LO.geometry(r)
    rows = [_program(r, n, r + i) for i, n in enumerate([gate - 1, gate, gate + 3 * step + 1, 7 * r + 13, 30 * r])]
    got = _measure(rows, r)
    want = np.array([LO.integrated(x, r) for x in rows])
    assert np.isnan(got[0]) and _same(got, want), (got, want)


def test_measure_at_block_edges_and_the_longest_utterance(cuda):
    k = [1, 2, 5, 37]
    lens = [9599, 9600] + [9600 + j * 2400 + d for j in k for d in (-1, 0, 1)] + [LONGEST - 1, LONGEST]
    rows = [_program(24000, n, n) for n in lens]
    got = _measure(rows)
    want = np.array([LO.integrated(x, 24000) for x in rows])
    assert np.isnan(got[0]) and not np.isnan(got[1:]).any() and _same(got, want), np.abs(got - want)


@pytest.mark.parametrize("B", [1, 7, 64])
def test_ragged_batches_silence_and_quiet_rows(cuda, B):
    rng = np.random.default_rng(B)
    rows = []
    for b in range(B):
        n = int(rng.integers(1, 24000 * 12))
        kind = b % 5
        if kind == 0:
            rows.append(np.zeros(n, np.float32))                                    # silence: NaN
        elif kind == 1:
            rows.append(_program(24000, n, b, peak=3e-3))                          # quiet, near -60 LUFS
        else:
            rows.append(_program(24000, n, b, peak=float(10 ** rng.uniform(-2, 0))))
    got = _measure(rows)
    want = np.array([LO.integrated(x, 24000) for x in rows])
    assert _same(got, want), np.nanmax(np.abs(got - want))
    assert np.array_equal(got, _measure(rows), equal_nan=True)                      # the same bits every run


def test_a_row_alone_equals_the_row_in_a_batch(cuda):
    rows = [_program(24000, 24000 * n + 7 * n, n) for n in range(1, 9)]
    batch = _measure(rows)
    assert np.array_equal(batch, np.concatenate([_measure([x]) for x in rows]))


def test_host_arrays_and_a_2d_tensor(cuda):
    from neutts_air_b200.loudness import measure

    x = np.stack([_program(24000, 48000, s) for s in range(3)])
    a = measure(list(x))
    assert np.array_equal(a, measure(torch.from_numpy(x).cuda())) and _same(a, np.array([LO.integrated(v, 24000) for v in x]))
    assert measure([]).shape == (0,)


# ------------------------------------------------------------------------------------------------- normaliser
def test_normalize_is_float32_of_the_oracle_gain(cuda):
    from neutts_air_b200.loudness import measure, normalize

    # no silent stretches here: a block of the filter's ring-out after one sits near -75 LUFS, and a +12 dB gain would
    # lift it over the -70 gate (the re-measured value then moves, as BS.1770's gating implies)
    rows = [_program(24000, n, n, span=1.0, silences=False) for n in (9600, 24000 * 5 + 3, 24000 * 40)]
    rows += [np.zeros(30000, np.float32), _program(24000, 9599, 1)]
    targets = [-16.0, -23.0, -9.5, -16.0, -16.0]
    got = [y.cpu().numpy() for y in normalize([torch.from_numpy(x).cuda() for x in rows], targets)]
    for x, y, t in zip(rows[:3], got, targets):
        want = (LO.gain(LO.integrated(x, 24000), t) * x.astype(np.float64)).astype(np.float32)
        assert y.dtype == np.float32 and _ulps(y, want) <= 1
    for x, y in zip(rows[3:], got[3:]):
        assert y.tobytes() == x.tobytes()                                            # NaN rows come back unchanged
    again = measure(got)
    assert np.allclose(again[:3], targets[:3], atol=1e-6, rtol=0) and np.isnan(again[3:]).all()


def test_normalize_with_none_targets_and_in_place(cuda):
    import ctypes as C

    from neutts_air_b200 import _lib
    from neutts_air_b200.loudness import normalize

    rows = [_program(24000, 24000 * s, s, span=1.0) for s in (1, 2, 3)]
    got = normalize([torch.from_numpy(x).cuda() for x in rows], [None, -20, None])
    assert got[0].cpu().numpy().tobytes() == rows[0].tobytes() and got[2].cpu().numpy().tobytes() == rows[2].tobytes()
    # out == in through the C ABI: the same bits as a separate output
    x = torch.from_numpy(np.concatenate(rows)).cuda()
    off = np.array([0, 24000, 72000, 144000], np.int64)
    offp = off.ctypes.data_as(C.POINTER(C.c_int64))
    L = _lib.lib()
    ws = torch.empty(L.nt_loudness_workspace_bytes(24000, 3, offp), dtype=torch.uint8, device="cuda")
    lufs = torch.empty(3, dtype=torch.float64, device="cuda")
    tg = (C.c_double * 3)(float("nan"), -20.0, float("nan"))
    _lib.check(L.nt_loudness_run(24000, 3, x.data_ptr(), offp, tg, lufs.data_ptr(), x.data_ptr(), ws.data_ptr(),
                                 ws.numel(), _lib.current_stream_ptr()))
    assert torch.equal(x, torch.cat(got))
    with pytest.raises(RuntimeError, match="workspace"):
        _lib.check(L.nt_loudness_run(24000, 3, x.data_ptr(), offp, tg, lufs.data_ptr(), x.data_ptr(), ws.data_ptr(),
                                     ws.numel() - 1, _lib.current_stream_ptr()))


# ------------------------------------------------------------------------------------------------- facade
TEXTS = ["The first text has a sentence. It has another one, and a clause! A third sentence closes it.",
         "Short one here. Then a second sentence follows it, slowly.",
         "Line one of three.\nLine two of three.\nLine three, the last."]


def _pair(sr=24000, fmt="float32", max_batch=2, max_context=2048):
    """A tiny facade whose codec hops 480 samples per frame, and a second one on the same engines with another output
    format."""
    from neutts import NeuTTS
    from tests.fakes import FakePhonemizer, SmallTok

    cfg = lm_oracle.LMConfig.tiny(vocab_size=4096, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4,
                                  num_kv_heads=2)
    lm = make_lm(cfg, lm_oracle.random_weights(cfg, 3, std=0.05, bf16_round=True), max_batch=max_batch, max_ctx=2048,
                 max_new=512)
    ccfg = codec_oracle.CodecConfig.tiny(n_fft=1920, hop=480)
    dec = make_codec(ccfg, codec_oracle.random_weights(ccfg, 2), max_batch=max_batch, max_frames=512)
    out = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for s, f in ((24000, "float32"), (sr, fmt)):
            t = NeuTTS(tokenizer=SmallTok(), phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=max_batch,
                       seed=7, sample_rate=s, pcm_format=f)
            t.watermarker = None
            t.max_context = max_context
            t.hop_length = ccfg.hop
            out.append(t)
    return out


def _inputs(n):
    rng = np.random.default_rng(n)
    return (["utterance " + "x" * int(rng.integers(1, 30)) for _ in range(n)],
            [torch.from_numpy(rng.integers(0, 1024, int(rng.integers(20, 60)))) for _ in range(n)], ["reference"] * n)


def _gpu_gain(rows, targets):
    from neutts_air_b200.loudness import normalize

    return [x if t is None else y.cpu().numpy()
            for x, t, y in zip(rows, targets, normalize([torch.from_numpy(x).cuda() for x in rows], targets))]


def _check_gained(got, plain, targets):
    """got[i] is plain[i] at its target: bit-identical to the GPU normaliser, within 1 ulp of the oracle's gain, and
    reading the target; rows without a target keep their bytes."""
    assert all(len(x) >= 9600 and np.isfinite(LO.integrated(x, 24000)) for x in plain)
    for y, x, w, t in zip(got, plain, _gpu_gain(plain, targets), targets):
        assert y.tobytes() == w.tobytes()
        if t is None:
            assert y.tobytes() == x.tobytes()
        else:
            assert _ulps(y, (LO.gain(LO.integrated(x, 24000), t) * x.astype(np.float64)).astype(np.float32)) <= 1
    m = _measure([y for y, t in zip(got, targets) if t is not None])
    assert np.allclose(m, [t for t in targets if t is not None], atol=1e-6, rtol=0)


def test_facade_infer_batch_loudness(cuda):
    tts, _ = _pair()
    texts, refs, rts = _inputs(3)
    plain = tts.infer_batch(texts, refs, rts)
    targets = [-16, None, -23]
    _check_gained(tts.infer_batch(texts, refs, rts, loudness=targets), plain, targets)
    _check_gained(tts.infer_batch(texts, refs, rts, loudness=-16), plain, [-16] * 3)
    assert tts.infer(texts[0], refs[0], rts[0], loudness=-16).tobytes() == _gpu_gain([tts.infer(texts[0], refs[0], rts[0])], [-16])[0].tobytes()


def test_facade_loudness_after_the_stretch(cuda):
    from neutts_air_b200.stretch import TimeStretch

    tts, _ = _pair()
    texts, refs, rts = _inputs(3)
    speeds = [0.75, 1.0, 1.5]
    plain = tts.infer_batch(texts, refs, rts)
    ts = TimeStretch("cuda:0")
    slow = [x if s == 1.0 else ts.stretch([torch.from_numpy(x).cuda()], s)[0].cpu().numpy() for x, s in zip(plain, speeds)]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(slow, tts.infer_batch(texts, refs, rts, speed=speeds)))
    targets = [-16, None, -23]
    _check_gained(tts.infer_batch(texts, refs, rts, speed=speeds, loudness=targets), slow, targets)


def test_facade_loudness_of_the_kept_take(cuda):
    tts, _ = _pair()
    texts, refs, rts = _inputs(3)
    plain = tts.infer_batch(texts, refs, rts, takes=2)
    targets = [None, -16, -30]
    _check_gained(tts.infer_batch(texts, refs, rts, takes=2, loudness=targets), plain, targets)


def test_facade_long_form_gains_each_segment(cuda):
    tts, _ = _pair(max_context=260)
    rng = np.random.default_rng(4)
    refs = [torch.from_numpy(rng.integers(0, 1024, int(rng.integers(30, 50)))) for _ in TEXTS]
    rts = ["reference voice"] * len(TEXTS)
    segs = [tts.segments(t, c, rt) for t, c, rt in zip(TEXTS, refs, rts)]
    assert all(len(s) >= 2 for s in segs)
    order = LF.round_robin([len(s) for s in segs])
    owners = [t for t, _ in order]
    per_seg = tts.infer_batch([segs[t][k] for t, k in order], [refs[t] for t in owners], [rts[t] for t in owners])
    targets = [-16, None, -23]
    gained = _gpu_gain(per_seg, [targets[t] for t in owners])
    got = tts.infer_batch(TEXTS, refs, rts, long_form=True, pause=0.125, loudness=targets)
    for t, g in enumerate(got):
        want = LF.join([gained[j] for j, o in enumerate(owners) if o == t], tts.sample_rate, 0.125)
        assert g.tobytes() == want.tobytes()
    assert abs(_measure([got[0]])[0] - (-16)) < 1.0        # near the target, not on it: the seams change its blocks


def test_facade_loudness_then_resample_int16(cuda):
    from neutts_air_b200.resample import Resampler

    tts, t16 = _pair(16000, "int16")
    texts, refs, rts = _inputs(3)
    targets = [-16, None, -23]
    gained = _gpu_gain(tts.infer_batch(texts, refs, rts), targets)
    got = t16.infer_batch(texts, refs, rts, loudness=targets)
    rs = Resampler(16000, "int16", device="cuda:0")
    for y, x in zip(got, gained):
        assert y.dtype == np.int16 and np.array_equal(y, rs.resample(torch.from_numpy(x).cuda()).cpu().numpy())
