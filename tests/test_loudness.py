"""CPU: the loudness meter's float64 oracle against torchaudio (and where it departs from it on purpose), BS.1770's
calibration, the gating edge cases, rate and target validation, the library's geometry, and the facade's routing of
``loudness`` on fake engines (a recording stand-in replaces the GPU normaliser)."""
import math

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from oracle import loudness_oracle as LO
from tests.fakes import FakeTokenizer, KwBackbone, _facade

RATES = [16000, 22050, 24000, 44100, 48000]


def _program(r, seconds, seed):
    """Noise under a level that changes every 100 ms, with silent stretches, peak-normalised so that neither
    K-weighting stage reaches +-1."""
    rng = np.random.default_rng(seed)
    n = int(seconds * r)
    step = r // 10
    x = rng.standard_normal(n) * np.repeat(10 ** rng.uniform(-2.5, 0, n // step + 1), step)[:n]
    x[n // 5: n // 5 + 3 * step] = 0
    x[int(0.7 * n):int(0.7 * n) + 7 * step] = 0
    return x / np.abs(x).max() * 0.25


def _stage_peaks(x, r):
    (b1, a1), (b2, a2) = LO.k_weighting(r)
    y1 = lfilter(b1, a1, x)
    return np.abs(y1).max(), np.abs(lfilter(b2, a2, y1)).max()


@pytest.mark.parametrize("r", RATES)
def test_oracle_equals_torchaudio(r):
    AF = pytest.importorskip("torchaudio.functional")
    for seed, seconds in [(0, 0.4), (1, 0.75), (2, 3.3), (3, 11.0)]:
        x = _program(r, seconds, seed + r)
        assert max(_stage_peaks(x, r)) < 1.0
        want = AF.loudness(torch.from_numpy(x)[None], r).item()
        assert abs(LO.integrated(x, r) - want) < 1e-9


def test_no_clamp_departs_from_torchaudio_on_a_full_scale_5khz_sine():
    AF = pytest.importorskip("torchaudio.functional")
    x = np.sin(2 * np.pi * 5000 * np.arange(3 * 48000) / 48000)
    assert max(_stage_peaks(x, 48000)) > 1.0
    ours, theirs = LO.integrated(x, 48000), AF.loudness(torch.from_numpy(x)[None], 48000).item()
    assert abs(ours - 0.27) < 0.01 and abs(theirs - (-2.14)) < 0.01


def test_997_hz_calibration():
    x = np.sin(2 * np.pi * 997 * np.arange(5 * 48000) / 48000)
    assert abs(LO.integrated(x, 48000) - (-3.01)) < 0.1


@pytest.mark.parametrize("r", RATES)
def test_silence_short_rows_and_one_block(r):
    gate, step = LO.geometry(r)
    assert gate == round(0.4 * r) and step * 4 == gate
    assert math.isnan(LO.integrated(np.zeros(3 * gate), r))
    x = _program(r, 1.0, r)
    assert math.isnan(LO.integrated(x[: gate - 1], r))
    z = LO.block_energies(x[:gate], r)
    assert len(z) == 1 and len(LO.block_energies(x[: gate + step - 1], r)) == 1
    assert len(LO.block_energies(x[: gate + step], r)) == 2
    assert LO.integrated(x[:gate], r) == pytest.approx(-0.691 + 10 * math.log10(z[0]), abs=1e-12)


def test_oracle_normalize_and_nan_rows():
    x = _program(24000, 2.0, 5).astype(np.float32)
    L = LO.integrated(x, 24000)
    y = LO.normalize(x, -16.0, 24000)
    assert np.array_equal(y, (10 ** ((-16.0 - L) / 20) * x.astype(np.float64)).astype(np.float32))
    assert LO.integrated(y, 24000) == pytest.approx(-16.0, abs=1e-5)
    short = x[:9599]
    assert np.array_equal(LO.normalize(short, -16.0, 24000), short)


@pytest.mark.parametrize("bad", [7999, 192010, 24005, 0, -24000, 24000.0, True, "24000", None])
def test_rejects_bad_rates(bad):
    from neutts_air_b200.loudness import check_rate

    with pytest.raises(ValueError, match="sample_rate"):
        check_rate(bad)


@pytest.mark.parametrize("r", [8000, 8090, 16000, 22050, 24000, 44100, 48000, 96000, 192000])
def test_library_geometry(r):
    from neutts_air_b200 import loudness

    info = loudness.query(r)
    assert (info.gate, info.step) == LO.geometry(r)
    assert info.step % info.chunk == 0 and info.chunks_per_step * info.chunk == info.step and info.chunk <= 256
    assert info.chunk == max(c for c in range(1, 257) if info.step % c == 0)
    if r == 24000:
        assert (info.chunk, info.chunks_per_step) == (240, 10)


@pytest.mark.parametrize("bad", [7990, 24001, 200000])
def test_library_rejects_bad_rates(bad):
    import ctypes as C

    from neutts_air_b200 import _lib

    L = _lib.lib()
    with pytest.raises(ValueError, match="multiple of 10 Hz"):
        _lib.check(L.nt_loudness_query(bad, C.byref(_lib.LoudnessInfo())))
    off = (C.c_int64 * 2)(0, 24000)
    assert L.nt_loudness_workspace_bytes(bad, 1, off) == 0
    with pytest.raises(ValueError, match="multiple of 10 Hz"):
        _lib.check(L.nt_loudness_run(bad, 1, None, off, None, None, None, None, 0, None))


def test_library_workspace_grows_with_whole_segments():
    import ctypes as C

    from neutts_air_b200 import _lib

    L = _lib.lib()

    def ws(*lens):
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        return L.nt_loudness_workspace_bytes(24000, len(lens), off.ctypes.data_as(C.POINTER(C.c_int64)))

    # a row shorter than one block filters nothing; the tail after the last whole step reaches no block
    assert ws(9599) == ws(100) and ws(9600) == ws(9600 + 2399) < ws(9600 + 2400)


@pytest.mark.parametrize("bad", [-70.5, 0.5, 6, float("nan"), float("inf"), -float("inf"), True, "-16"])
def test_rejects_bad_targets(bad):
    from neutts_air_b200.loudness import check_target

    with pytest.raises(ValueError, match=r"\[-70.0, 0.0\]"):
        check_target(bad)
    bb = KwBackbone(FakeTokenizer())
    with pytest.raises(ValueError, match=r"\[-70.0, 0.0\]"):
        _facade(bb, 2).infer_batch(["a"], [[1]], ["r"], loudness=bad)
    with pytest.raises(ValueError, match=r"\[-70.0, 0.0\]"):
        _facade(bb, 2).infer_batch(["a", "b"], [[1], [2]], ["r"] * 2, loudness=[-16, bad])
    with pytest.raises(ValueError, match=r"\[-70.0, 0.0\]"):
        _facade(bb, 2).infer(["a"], [1], "r", loudness=bad, long_form=True)
    assert bb.calls == []


def test_target_list_of_the_wrong_length():
    bb = KwBackbone(FakeTokenizer())
    with pytest.raises(ValueError, match="one value per utterance"):
        _facade(bb, 2).infer_batch(["a", "b"], [[1], [2]], ["r"] * 2, loudness=[-16, -23, -16])
    assert bb.calls == []


def test_streams_take_no_loudness():
    bb = KwBackbone(FakeTokenizer())
    with pytest.raises(TypeError):
        _facade(bb, 2).infer_stream("a", [1], "r", loudness=-16)
    with pytest.raises(TypeError):
        _facade(bb, 2).infer_stream_batch(["a"], [[1]], ["r"], loudness=-16)


# ---------------------------------------------------------------------------------------------- facade on fakes
class IdBackbone:
    """generate_batch / generate_queue / forks: prompt p yields the one code len(p) (so the waveform names its prompt);
    takes are scored so that take 1 wins."""
    device = torch.device("cpu")

    def __init__(self, tok, queue=True):
        self.tok, self.calls = tok, []
        if queue:
            self.generate_queue = lambda prompts, eos, **kw: self._gen("queue", prompts, kw)

    def set_logprobs(self, on=True):
        pass

    def _gen(self, what, prompts, kw):
        self.calls.append((what, len(prompts), {k: v for k, v in kw.items() if k != "seed"}))
        n = kw.get("num_return_sequences", 1)
        ids = [torch.tensor([self.tok.speech_base + len(p)]) for p in prompts for _ in range(n)]
        if kw.get("return_logprobs"):
            lps = [torch.tensor([[-1.0, -1.0 if j == 1 else -3.0]]) for _ in prompts for j in range(n)]
            return ids, lps
        return ids

    def generate_batch(self, prompts, eos, **kw):
        return self._gen("batch", prompts, kw)


def _utts(n):
    texts = ["w" * (3 * i + 1) for i in range(n)]      # distinct prompt lengths
    return texts, [[1, 2]] * n, ["r"] * n


def _prompt_len(tts, texts, refs, rts):
    return [len(tts._apply_chat_template(c, rt, t)) for t, c, rt in zip(texts, refs, rts)]


class RecNormalize:
    """Stand-in for loudness.normalize: records (first sample, target) of every row and returns the row plus 1000."""

    def __init__(self):
        self.log = []

    def __call__(self, rows, targets, sample_rate=24000):
        assert sample_rate == 24000
        out = []
        for x, t in zip(rows, targets):
            self.log.append((round(float(x[0]) * 65536), t))
            out.append(torch.as_tensor(x) + 1000.0)
        return out


def _rec(monkeypatch):
    from neutts_air_b200 import loudness

    rec = RecNormalize()
    monkeypatch.setattr(loudness, "normalize", rec)
    return rec


def test_default_makes_the_same_engine_calls_and_measures_nothing(monkeypatch):
    from neutts import NeuTTS
    from neutts_air_b200 import loudness

    def boom(*a, **k):
        raise AssertionError("a row was normalised")

    monkeypatch.setattr(loudness, "normalize", boom)
    monkeypatch.setattr(NeuTTS, "_decode_stretched", boom)
    texts, refs, rts = _utts(5)
    runs = []
    for kw in ({}, dict(loudness=None), dict(loudness=[None] * 5)):
        bb = IdBackbone(FakeTokenizer(), queue=False)
        w = _facade(bb, 2).infer_batch(texts, refs, rts, **kw)
        runs.append((bb.calls, w))
        assert all("loudness" not in c[2] for c in bb.calls)
    for calls, w in runs[1:]:
        assert calls == runs[0][0] and all(a.tobytes() == b.tobytes() for a, b in zip(w, runs[0][1]))


@pytest.mark.parametrize("how", ["chunks", "queue", "takes", "shards"])
def test_target_list_follows_its_utterances(monkeypatch, how):
    from neutts_air_b200 import dist

    texts, refs, rts = _utts(5)
    targets = [-16.0, None, -23.0, -30, None]
    bb = IdBackbone(FakeTokenizer(), queue=how in ("queue", "shards"))
    tts = _facade(bb, 2 if how != "takes" else 4)
    rec = _rec(monkeypatch)
    plen = _prompt_len(tts, texts, refs, rts)
    plain = tts.infer_batch(texts, refs, rts, **({"takes": 2} if how == "takes" else {}))
    kw = {}
    mine = list(range(5))
    if how == "takes":
        kw["takes"] = 2
    if how == "shards":
        mine = [0, 2, 3]
        monkeypatch.setattr(dist, "world", lambda: (1, 2))
        monkeypatch.setattr(dist, "shard_indices", lambda n, lengths: mine)
        monkeypatch.setattr(dist, "all_gather_waveforms", lambda local, idx, n, device=None: local)
        kw["distributed"] = True
    wavs = tts.infer_batch(texts, refs, rts, loudness=targets, **kw)
    assert all("loudness" not in c[2] for c in bb.calls)
    assert sorted(rec.log) == sorted((plen[i], float(targets[i])) for i in mine if targets[i] is not None)
    for w, i in zip(wavs, mine):
        if targets[i] is None:
            assert w.tobytes() == plain[i].tobytes()
        else:
            assert np.array_equal(w, plain[i] + np.float32(1000.0))


def test_scalar_target_infer_and_prompt_ids(monkeypatch):
    bb = IdBackbone(FakeTokenizer(), queue=False)
    tts = _facade(bb, 2)
    rec = _rec(monkeypatch)
    texts, refs, rts = _utts(3)
    plen = _prompt_len(tts, texts, refs, rts)
    tts.infer_batch(texts, refs, rts, loudness=-16)
    assert sorted(rec.log) == sorted((p, -16.0) for p in plen)
    rec.log.clear()
    tts.infer(texts[0], refs[0], rts[0], loudness=-23)
    assert rec.log == [(plen[0], -23.0)]
    rec.log.clear()
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    tts.infer_from_prompt_ids(prompts, loudness=[None, -20, None])
    assert rec.log == [(plen[1], -20.0)]
