"""GPU: the speaking-rate stretch (stretch.cu), each stage against float64 on the GPU's own inputs, end to end against
the oracle on well-conditioned audio (a 60 s row included), streams against one-shot calls bit for bit, and the
facade's ``speed`` on the tiny engines."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from oracle import stretch_oracle as SO
from tests.helpers import _tts

pytestmark = pytest.mark.gpu

SPEEDS = [0.5, 0.7, 0.75, 1 / 0.9, 1.25, 1.5, 2.0]


def _ts(rows=1):
    from neutts_air_b200.stretch import TimeStretch

    return TimeStretch("cuda:0", max_rows=rows)


def _speech_like(L, seed):
    """Noise under a comb of 513 bin-centred tones with quadratic phases: no analysis bin comes near zero."""
    k = np.arange(513)[:, None]
    comb = np.cos(2 * np.pi * k * np.arange(1024)[None, :] / 1024 + np.pi * k ** 2 / 4).sum(0)
    x = np.resize(comb / np.abs(comb).max() * 0.5, L)
    return (x + 0.002 * np.random.default_rng(seed).standard_normal(L)).astype(np.float32)


def _rel_rms(got, want):
    return float(np.sqrt(np.mean((got - want) ** 2) / np.mean(want ** 2)))


# ------------------------------------------------------------------------------------------------- stage twins
@pytest.mark.parametrize("r", SPEEDS)
@pytest.mark.parametrize("L", [300, 5000, 8192])
def test_stages_match_float64_on_their_own_inputs(cuda, r, L):
    ts = _ts()
    info = ts.info
    x = (np.random.default_rng(L).standard_normal(L) * 0.3).astype(np.float32)
    y = ts.stretch([torch.from_numpy(x).to(cuda)], r)[0].cpu().numpy().astype(np.float64)
    T = 1 + L // 256
    K = len(torch.arange(0, T, r, dtype=torch.float64))
    torch.cuda.synchronize()
    # analysis: the GPU's spectra of all T frames against a float64 STFT of the same fp32 row
    sp = ts.debug("spec", T * info.spec_ld).view(T, info.spec_ld).cpu().double()
    S_gpu = torch.complex(sp[:, :513], sp[:, 513:1026]).T
    S_ref = SO.analysis(x.astype(np.float64))
    ea = float((S_gpu - S_ref).abs().max() / S_ref.abs().max())
    # vocoder: the GPU's stretched spectra against the float64 vocoder fed the GPU's analysis spectra
    n2 = info.stretch_lo_rows * info.stretch_ld
    buf = ts.debug("stretch", 2 * n2)
    s2 = (buf[:n2].double() + buf[n2:].double()).view(info.stretch_lo_rows, info.stretch_ld)[:K].cpu()
    S2_gpu = torch.complex(s2[:, :513], s2[:, 513:1026]).T
    S2_ref = SO.phase_vocoder(S_gpu, r)
    ev = float((S2_gpu - S2_ref).abs().max() / S2_ref.abs().max())
    # synthesis: the GPU's PCM against the float64 istft of the GPU's stretched spectra
    want = SO.synthesis(S2_gpu, round(L / r))
    es = _rel_rms(y, want)
    print(f"STRETCH-STAGES r={r:.4f} L={L}: analysis max/max {ea:.2e}, vocoder max/max {ev:.2e}, synthesis relRMS {es:.2e}")
    assert y.shape == want.shape == (round(L / r),)
    assert ea <= 1e-5 and ev <= 1e-6 and es <= 1e-5, (ea, ev, es)


# ------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("r", SPEEDS)
def test_end_to_end_on_well_conditioned_audio(cuda, r):
    rows = [_speech_like(L, i) for i, L in enumerate((1, 700, 24000 + 37, 72000))]
    for x in rows[2:]:
        S = SO.analysis(x.astype(np.float64)).abs()
        assert float((S / S.pow(2).mean(0).sqrt()).min()) >= 1e-3        # no bin near zero: the comparison is fair
    got = _ts().stretch([torch.from_numpy(x).to(cuda) for x in rows], r)
    for x, y in zip(rows, got):
        want = SO.time_stretch(x.astype(np.float64), r)
        y = y.cpu().numpy().astype(np.float64)
        assert y.shape == want.shape
        if len(x) > 1:
            rel = _rel_rms(y, want)
            print(f"STRETCH-E2E r={r:.4f} L={len(x)}: relRMS {rel:.2e}")
            assert rel <= 1e-4, (r, len(x), rel)


@pytest.mark.parametrize("r", [0.75, 1.25])
def test_sixty_seconds_do_not_drift(cuda, r):
    x = _speech_like(60 * 24000, 60)
    S = SO.analysis(x.astype(np.float64)).abs()
    assert float((S / S.pow(2).mean(0).sqrt()).min()) >= 1e-3
    y = _ts().stretch([torch.from_numpy(x).to(cuda)], r)[0].cpu().numpy().astype(np.float64)
    want = SO.time_stretch(x.astype(np.float64), r)
    n = len(want)
    head, tail = _rel_rms(y[: n // 10], want[: n // 10]), _rel_rms(y[-n // 10:], want[-n // 10:])
    print(f"STRETCH-60s r={r}: relRMS first tenth {head:.2e}, last tenth {tail:.2e}, whole {_rel_rms(y, want):.2e}")
    assert y.shape == want.shape and _rel_rms(y, want) <= 1e-4 and tail <= 1e-4


# ------------------------------------------------------------------------------------------------- streams
def _stream(ts, rows, xs, speeds, rng, cuts=20, tiny=True):
    """Push rows' samples in random pieces (1-sample and empty ones included), rows left out at random; the last
    push of every row is final (sometimes with an empty chunk)."""
    pieces = []
    for x in xs:
        c = np.sort(rng.integers(0, len(x) + 1, cuts))
        p = np.split(x, c)
        if tiny and len(x) > 10:
            p = [x[:1], x[1:2], np.zeros(0, np.float32)] + np.split(x[2:], np.sort(rng.integers(0, len(x) - 1, cuts)))
        pieces.append(p + [np.zeros(0, np.float32)] if rng.random() < 0.5 else p)
    out = [[] for _ in rows]
    nxt = [0] * len(rows)
    while any(n < len(p) for n, p in zip(nxt, pieces)):
        live = [i for i in range(len(rows)) if nxt[i] < len(pieces[i]) and rng.random() < 0.8]
        if not live:
            continue
        got = ts.push([rows[i] for i in live], [pieces[i][nxt[i]] for i in live], [speeds[i] for i in live],
                      [nxt[i] == len(pieces[i]) - 1 for i in live])
        for i, y in zip(live, got):
            out[i].append(y)
            nxt[i] += 1
    return [np.concatenate(o) for o in out]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_chunked_streams_are_bit_identical_to_one_shot(cuda, seed):
    rng = np.random.default_rng(seed)
    rows = 4
    ts = _ts(rows)
    xs = [(rng.standard_normal(int(n)) * 0.3).astype(np.float32) for n in rng.integers(1, 30000, rows)]
    speeds = [float(s) for s in rng.choice(SPEEDS, rows)]
    one = [y.cpu().numpy() for y in ts.stretch([torch.from_numpy(x).to(cuda) for x in xs], speeds)]
    got = _stream(ts, list(range(rows)), xs, speeds, rng)
    for x, y, z, s in zip(xs, one, got, speeds):
        assert len(z) == round(len(x) / s) and np.array_equal(z, y), (len(x), s)


def test_row_output_does_not_depend_on_its_neighbours(cuda):
    rng = np.random.default_rng(5)
    ts = _ts(3)
    xs = [(rng.standard_normal(n) * 0.3).astype(np.float32) for n in (20000, 9000, 40000)]
    alone = [ts.push([r], [x], [0.7], final=True)[0] for r, x in enumerate(xs)]
    together = ts.push([0, 1, 2], xs, [0.7, 1.5, 0.7], final=True)
    assert np.array_equal(together[0], alone[0]) and np.array_equal(together[2], alone[2])
    one = ts.stretch([torch.from_numpy(x).to(cuda) for x in xs], 0.7)
    assert all(np.array_equal(a, o.cpu().numpy()) for a, o in zip(alone, one))


def test_reset_mid_stream_and_speed_binding(cuda):
    rng = np.random.default_rng(9)
    ts = _ts(2)
    x = (rng.standard_normal(12000) * 0.3).astype(np.float32)
    ts.push([0], [rng.standard_normal(5000).astype(np.float32)], 1.25)
    with pytest.raises(ValueError, match="speed"):
        ts.push([0], [x[:10]], 0.8)                         # a running stream keeps its speed
    ts.reset([0])
    got = np.concatenate([ts.push([0], [x[:7000]], 0.8)[0], ts.push([0], [x[7000:]], 0.8, final=True)[0]])
    assert np.array_equal(got, ts.stretch([torch.from_numpy(x).to(cuda)], 0.8)[0].cpu().numpy())


def test_push_checks_spans_and_speeds_before_launching(cuda):
    from neutts_air_b200 import _lib

    ts = _ts(1)
    x = torch.zeros(4000, device=cuda)
    out = torch.empty(9000, device=cuda)
    off = (C.c_int64 * 2)(0, 4000)
    sp = (C.c_double * 1)(1.25)
    n0 = ts.L.nt_launch_count()
    rc = ts.L.nt_stretch_push(ts.handle, 1, (C.c_int32 * 1)(0), None, sp, x.data_ptr(), off, out.data_ptr(),
                              (C.c_int64 * 2)(0, 99), None)
    assert rc == -1 and b"span" in ts.L.nt_last_error()
    rc = ts.L.nt_stretch_push(ts.handle, 1, None, None, (C.c_double * 1)(2.5), x.data_ptr(), off, out.data_ptr(),
                              (C.c_int64 * 2)(0, 1600), None)
    assert rc == -1 and b"[0.5, 2.0]" in ts.L.nt_last_error()
    assert ts.L.nt_launch_count() == n0
    with pytest.raises(ValueError):
        _lib.check(rc)


# ------------------------------------------------------------------------------------------------- facade
def _pair(sr=24000, fmt="float32", max_batch=2):
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


def _stretched(x, r):
    return _ts().stretch([torch.from_numpy(np.asarray(x, np.float32)).cuda()], r)[0].cpu().numpy()


def test_facade_infer_batch_speeds(cuda):
    tts, _ = _pair()
    texts, refs, rts = _inputs(3)
    plain = tts.infer_batch(texts, refs, rts)
    speeds = [0.75, 1.0, 1.5]
    got = tts.infer_batch(texts, refs, rts, speed=speeds)
    for x, y, r in zip(plain, got, speeds):
        assert len(y) == round(len(x) / r)
        assert np.array_equal(y, x if r == 1.0 else _stretched(x, r))
    assert got[1].tobytes() == plain[1].tobytes()


def test_facade_stretch_then_resample_int16(cuda):
    from neutts_air_b200.resample import Resampler

    tts, t16 = _pair(16000, "int16")
    texts, refs, rts = _inputs(3)
    plain = tts.infer_batch(texts, refs, rts)
    got = t16.infer_batch(texts, refs, rts, speed=[1.25, 1.0, 0.6])
    rs = Resampler(16000, "int16", device="cuda:0")
    for x, y, r in zip(plain, got, [1.25, 1.0, 0.6]):
        s = x if r == 1.0 else _stretched(x, r)
        assert y.dtype == np.int16 and np.array_equal(y, rs.resample(torch.from_numpy(s).cuda()).cpu().numpy())


def _stream_cat(gen, n):
    got = [[] for _ in range(n)]
    for out in gen:
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
    return [np.concatenate(g) for g in got]


def test_facade_streams_equal_one_shot_stretch_of_the_plain_stream(cuda):
    tts, _ = _pair()
    texts, refs, rts = _inputs(5)
    speeds = [0.75, 1.0, 1.5, 0.5, 2.0]
    plain = _stream_cat(tts.infer_stream_batch(texts, refs, rts), 5)          # queue: 5 utterances on 2 slots
    got = _stream_cat(tts.infer_stream_batch(texts, refs, rts, speed=speeds), 5)
    for x, y, r in zip(plain, got, speeds):
        assert np.array_equal(y, x if r == 1.0 else _stretched(x, r))
    one = np.concatenate(list(tts.infer_stream(texts[0], refs[0], rts[0], speed=0.75)))
    assert np.array_equal(one, _stretched(np.concatenate(list(tts.infer_stream(texts[0], refs[0], rts[0]))), 0.75))
