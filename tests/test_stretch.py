"""CPU: the speaking-rate stretch's float64 oracle against torchaudio, its streaming span rule, speed validation, and
the facade's routing of ``speed`` on fake engines (a recording stand-in replaces the GPU stretcher)."""
import math

import numpy as np
import pytest
import torch

from oracle import stretch_oracle as SO
from tests.fakes import FakeTokenizer, KwBackbone, _facade

SPEEDS = [0.5, 0.7, 1 / 0.9, 1.25, 2.0]
LENGTHS = [1, 255, 256, 257, 1023, 24000, 480 * 37]


@pytest.mark.parametrize("r", SPEEDS)
def test_oracle_equals_torchaudio(r):
    AF = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(int(r * 1000))
    win = torch.hann_window(1024, dtype=torch.float64)
    adv = torch.linspace(0, math.pi * 256, 513, dtype=torch.float64)[:, None]
    for L in LENGTHS:
        x = torch.from_numpy(rng.standard_normal(L))
        S = torch.stft(x, 1024, 256, window=win, center=True, pad_mode="constant", return_complex=True)
        S2 = AF.phase_vocoder(S, r, adv)
        assert S2.shape[-1] == math.ceil(S.shape[-1] / r) == len(torch.arange(0, S.shape[-1], r, dtype=torch.float64))
        got = SO.time_stretch(x.numpy(), r)
        assert len(got) == round(L / r)
        steps = torch.arange(0, S.shape[-1], r, dtype=torch.float64)
        # the restatement is torchaudio's function: fed torch.arange's positions it returns torchaudio's spectra
        assert (SO.phase_vocoder(S, r, steps) - S2).abs().max() <= 1e-12
        # the contract's positions j * r agree with torch.arange's to a few ulps (exactly at dyadic speeds)
        ours = SO.time_steps(S.shape[-1], r)
        assert ours.shape == steps.shape and (ours - steps).abs().max() <= 4 * np.finfo(float).eps * S.shape[-1]
        if r in (0.5, 1.25, 2.0):
            assert torch.equal(ours, steps)
        if round(L / r) == 0 or not torch.equal(ours, steps):
            continue
        want = torch.istft(S2, 1024, 256, window=win, center=True, length=round(L / r)).numpy()
        assert np.abs(got - want).max() <= 1e-12, (r, L)


def test_identity_facts():
    x = np.random.default_rng(0).standard_normal(24000)
    assert np.abs(SO.synthesis(SO.analysis(x), len(x)) - x).max() < 1e-13
    S = SO.analysis(x)
    assert SO.phase_vocoder(S, 1.0) is S


@pytest.mark.parametrize("r", SPEEDS + [0.75, 1.5, 1.0])
def test_span_rule_sums_to_the_whole_row(r):
    from neutts_air_b200.stretch import emitted

    rng = np.random.default_rng(int(r * 977))
    for n in range(0, 20000, 37):      # the library's mirror equals the oracle's plain statement
        assert emitted(n, False, r) == SO.emitted(n, False, r)
        assert emitted(n, False, r) <= max(0, round(n / r) - 511)   # a later length= can never trim an emitted sample
    for L in (0, 1, 300, 1023, 5000, 24000 + 17):
        for _ in range(5):
            cuts = np.sort(rng.integers(0, L + 1, int(rng.integers(0, 12))))
            sizes = np.diff(np.concatenate([[0], cuts, [L]])).tolist() + [0]   # empty pushes, then an empty final one
            recv, total = 0, 0
            for k, m in enumerate(sizes):
                fin = k == len(sizes) - 1
                span = emitted(recv + m, fin, r) - emitted(recv, False, r)
                assert span >= 0
                total += span
                recv += m
            assert total == round(L / r)


@pytest.mark.parametrize("bad", [0.49, 2.01, 0.0, -1.0, float("nan"), float("inf"), True, "1.0", None])
def test_rejects_bad_speeds(bad):
    from neutts_air_b200.stretch import check_speed

    with pytest.raises(ValueError, match=r"\[0.5, 2.0\]"):
        check_speed(bad)
    tts = _facade(KwBackbone(FakeTokenizer()), 2)
    with pytest.raises(ValueError, match=r"\[0.5, 2.0\]"):
        tts.infer_batch(["a"], [[1]], ["r"], speed=bad)
    with pytest.raises(ValueError, match=r"\[0.5, 2.0\]"):
        tts.infer_stream_batch(["a"], [[1]], ["r"], speed=[bad])


def test_speed_list_of_the_wrong_length():
    bb = KwBackbone(FakeTokenizer())
    with pytest.raises(ValueError, match="one value per utterance"):
        _facade(bb, 2).infer_batch(["a", "b"], [[1], [2]], ["r"] * 2, speed=[1.0, 1.5, 2.0])
    assert bb.calls == []


# ---------------------------------------------------------------------------------------------- facade on fakes
class RecStretch:
    """Stand-in for TimeStretch: records (first sample, speed) of every stretched row and returns round(L / speed)
    samples of the input's first value plus the speed."""

    def __init__(self):
        self.log = []

    def stretch(self, rows, speeds):
        out = []
        for x, s in zip(rows, speeds):
            self.log.append((round(float(x[0]) * 65536), s))
            out.append(torch.full((round(len(x) / s),), float(x[0]) + s))
        return out


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


def _tts(bb, max_batch, monkeypatch):
    from neutts import NeuTTS

    tts = _facade(bb, max_batch)
    rec = RecStretch()
    monkeypatch.setattr(NeuTTS, "_time_stretch", lambda self: rec)
    return tts, rec


def _utts(n):
    texts = ["w" * (3 * i + 1) for i in range(n)]      # distinct prompt lengths
    return texts, [[1, 2]] * n, ["r"] * n


def test_defaults_make_the_same_engine_calls_and_build_no_stretcher(monkeypatch):
    from neutts import NeuTTS

    def boom(self):
        raise AssertionError("a stretcher was built")

    monkeypatch.setattr(NeuTTS, "_time_stretch", boom)
    texts, refs, rts = _utts(5)
    runs = []
    for kw in ({}, dict(speed=1.0), dict(speed=[1.0] * 5)):
        bb = IdBackbone(FakeTokenizer(), queue=False)
        w = _facade(bb, 2).infer_batch(texts, refs, rts, **kw)
        runs.append((bb.calls, w))
        assert all("speed" not in c[2] for c in bb.calls)
    for calls, w in runs[1:]:
        assert calls == runs[0][0] and all(np.array_equal(a, b) for a, b in zip(w, runs[0][1]))


def _prompt_len(tts, texts, refs, rts):
    return [len(tts._apply_chat_template(c, rt, t)) for t, c, rt in zip(texts, refs, rts)]


@pytest.mark.parametrize("how", ["chunks", "queue", "takes", "shards"])
def test_speed_list_follows_its_utterances(monkeypatch, how):
    from neutts_air_b200 import dist

    texts, refs, rts = _utts(5)
    speeds = [0.75, 1.0, 1.5, 2.0, 1.0]
    bb = IdBackbone(FakeTokenizer(), queue=how in ("queue", "shards"))
    tts, rec = _tts(bb, 2 if how != "takes" else 4, monkeypatch)
    plen = _prompt_len(tts, texts, refs, rts)
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
    wavs = tts.infer_batch(texts, refs, rts, speed=speeds, **kw)
    assert all("speed" not in c[2] for c in bb.calls)
    assert {"chunks": "batch", "queue": "queue", "takes": "batch", "shards": "queue"}[how] == bb.calls[0][0]
    # every utterance not at 1.0 was stretched once, at its own speed; the 1.0 ones were left alone
    assert sorted(rec.log) == sorted((plen[i], speeds[i]) for i in mine if speeds[i] != 1.0)
    for w, i in zip(wavs, mine):
        assert len(w) == round(480 / speeds[i])
        want = plen[i] / 65536.0 + (speeds[i] if speeds[i] != 1.0 else 0.0)
        assert np.allclose(w, want)


def test_scalar_speed_and_infer(monkeypatch):
    bb = IdBackbone(FakeTokenizer(), queue=False)
    tts, rec = _tts(bb, 2, monkeypatch)
    texts, refs, rts = _utts(3)
    plen = _prompt_len(tts, texts, refs, rts)
    w = tts.infer_batch(texts, refs, rts, speed=1.25)
    assert [len(x) for x in w] == [round(480 / 1.25)] * 3 and sorted(rec.log) == sorted((p, 1.25) for p in plen)
    w1 = tts.infer(texts[0], refs[0], rts[0], speed=0.5)
    assert len(w1) == 960 and rec.log[-1] == (plen[0], 0.5)
