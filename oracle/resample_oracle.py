"""Float64 restatement of the output resampler (TEST INFRASTRUCTURE ONLY).

torchaudio.functional.resample(x, 24000, sample_rate) with its defaults (sinc_interp_hann, lowpass_filter_width 6,
rolloff 0.99), written in numpy straight from the formula of include/neutts_b200.h: with g = gcd(24000, sr),
orig = 24000 / g, new = sr / g, width w = ceil(6 * orig / (0.99 * min(orig, new))), the table has `new` phases of
2w + orig taps, and output k * new + p is phase p dotted with x_pad[k * orig : k * orig + 2w + orig], x_pad being x
with w zeros in front and w + orig behind, cut to ceil(sr * len / 24000) samples.  ``Stream`` restates the streaming
contract; ``to_int16`` the 16-bit conversion, in float32 as the device computes it.  No torchaudio import: the GPU
tests compare against this module alone.
"""
from __future__ import annotations

import math

import numpy as np

SRC_RATE = 24_000
WIDTH, ROLLOFF = 6, 0.99


def geometry(sr: int) -> tuple:
    """(orig, new, w, taps); at 24000 there is no filter: (1, 1, 0, 1)."""
    g = math.gcd(SRC_RATE, sr)
    orig, new = SRC_RATE // g, sr // g
    if orig == new:
        return 1, 1, 0, 1
    w = math.ceil(WIDTH * orig / (min(orig, new) * ROLLOFF))
    return orig, new, w, 2 * w + orig


def table(sr: int) -> np.ndarray:
    """float64 [new, taps] (the identity [[1.0]] at 24000)."""
    orig, new, w, taps = geometry(sr)
    if w == 0:
        return np.ones((1, 1))
    base = min(orig, new) * ROLLOFF
    idx = np.arange(-w, w + orig, dtype=np.float64)[None, :] / orig
    t = np.arange(0, -new, -1, dtype=np.float64)[:, None] / new + idx
    t = np.clip(t * base, -WIDTH, WIDTH)
    window = np.cos(t * math.pi / WIDTH / 2) ** 2
    t = t * math.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(t == 0, 1.0, np.sin(t) / t)
    return k * (window * (base / orig))


def out_len(n: int, sr: int) -> int:
    return -(-sr * n // SRC_RATE)


def _frames(xp: np.ndarray, tab: np.ndarray, orig: int, n_frames: int) -> np.ndarray:
    """Frames 0 .. n_frames-1 of padded input xp (each reads xp[k * orig : k * orig + taps]), interleaved."""
    taps = tab.shape[1]
    if n_frames == 0:
        return np.zeros(0)
    win = np.lib.stride_tricks.sliding_window_view(xp[: (n_frames - 1) * orig + taps], taps)[::orig]
    return (win @ tab.T).reshape(-1)


def resample(x, sr: int) -> np.ndarray:
    """One row (1-D) or rows ([..., L]) of 24 kHz samples -> float64 at sr."""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 1:
        return np.stack([resample(r, sr) for r in x.reshape(-1, x.shape[-1])]).reshape(*x.shape[:-1], -1)
    orig, new, w, taps = geometry(sr)
    tab = table(sr)
    xp = np.concatenate([np.zeros(w), x, np.zeros(w + orig)])
    return _frames(xp, tab, orig, len(x) // orig + 1)[: out_len(len(x), sr)]


class Stream:
    """The streaming contract for one row: frame k is final once k * orig + w + orig <= samples received; ``push``
    returns the final samples not returned before and keeps only the samples the first frame not yet final reads."""

    def __init__(self, sr: int):
        self.sr = sr
        self.orig, self.new, self.w, self.taps = geometry(sr)
        self.tab = table(sr)
        self.reset()

    def reset(self):
        self.held = np.zeros(self.w)      # x_pad from the window start of the first frame not yet final

    def push(self, chunk, final: bool = False) -> np.ndarray:
        comb = np.concatenate([self.held, np.asarray(chunk, dtype=np.float64)])
        if final:
            r = len(comb) - self.w                      # samples after the first open frame's window start
            out = _frames(np.concatenate([comb, np.zeros(self.w + self.orig)]), self.tab, self.orig, r // self.orig + 1)
            self.reset()
            return out[: -(-self.new * r // self.orig)]
        n_frames = (len(comb) - self.taps) // self.orig + 1 if len(comb) >= self.taps else 0
        out = _frames(comb, self.tab, self.orig, n_frames)
        self.held = comb[n_frames * self.orig:]
        return out


def to_int16(y) -> np.ndarray:
    """16-bit PCM in float32: clip to [-1, 1], times 32767, round half to even (the device's __float2int_rn)."""
    y = np.asarray(y, dtype=np.float32)
    return np.rint(np.clip(y, np.float32(-1), np.float32(1)) * np.float32(32767)).astype(np.int16)
