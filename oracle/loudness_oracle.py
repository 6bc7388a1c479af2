"""Float64 restatement of the loudness meter and normalizer (TEST INFRASTRUCTURE ONLY).

ITU-R BS.1770-4 integrated loudness of one mono row at rate r, as ``torchaudio.functional.loudness`` computes it, with
the two differences include/neutts_b200.h states: no stage of the K-weighting is clamped to [-1, 1] (torchaudio's
``lfilter`` clamps by default; BS.1770 and pyloudnorm do not), and a row shorter than one gating block reads NaN
(torchaudio raises).  No torchaudio import: the GPU tests compare against this module alone, and the CPU tests pin it
to torchaudio.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import lfilter

ABS_GATE = -70.0
BIAS = -0.691


def check_rate(r: int) -> None:
    if isinstance(r, bool) or not isinstance(r, (int, np.integer)) or not (8000 <= r <= 192000 and r % 10 == 0):
        raise ValueError(f"sample rate {r!r} must be a multiple of 10 Hz in [8000, 192000]")


def geometry(r: int) -> tuple:
    """(gate, step) in samples: 400 ms blocks every 100 ms."""
    check_rate(r)
    gate = round(0.4 * r)
    return gate, gate // 4


def k_weighting(r: int) -> tuple:
    """(b, a) of the two biquads, torchaudio's treble_biquad(4 dB, 1500 Hz, Q 1/sqrt 2) then highpass_biquad(38 Hz,
    Q 0.5), each normalised by a0."""
    w0 = 2 * math.pi * 1500.0 / r
    alpha = math.sin(w0) / 2 / (1 / math.sqrt(2))
    A = math.exp(4.0 / 40 * math.log(10))
    t1, t2, t3 = 2 * math.sqrt(A) * alpha, (A - 1) * math.cos(w0), (A + 1) * math.cos(w0)
    b = [A * ((A + 1) + t2 + t1), -2 * A * ((A - 1) + t3), A * ((A + 1) + t2 - t1)]
    a = [(A + 1) - t2 + t1, 2 * ((A - 1) - t3), (A + 1) - t2 - t1]
    shelf = (np.array(b) / a[0], np.array(a) / a[0])
    w0 = 2 * math.pi * 38.0 / r
    alpha = math.sin(w0) / 2.0 / 0.5
    b = [(1 + math.cos(w0)) / 2, -1 - math.cos(w0), (1 + math.cos(w0)) / 2]
    a = [1 + alpha, -2 * math.cos(w0), 1 - alpha]
    high = (np.array(b) / a[0], np.array(a) / a[0])
    return shelf, high


def block_energies(x, r: int) -> np.ndarray:
    """z_j, the mean square of the K-weighted row over block j = [j * step, j * step + gate)."""
    gate, step = geometry(r)
    y = np.asarray(x, dtype=np.float64)
    for b, a in k_weighting(r):
        y = lfilter(b, a, y)
    if len(y) < gate:
        return np.zeros(0)
    nb = (len(y) - gate) // step + 1
    y2 = y * y
    return np.array([y2[j * step: j * step + gate].mean() for j in range(nb)])


def integrated(x, r: int) -> float:
    """Gated integrated loudness in LUFS; NaN when no block passes both gates."""
    z = block_energies(x, r)
    with np.errstate(divide="ignore"):
        lj = BIAS + 10 * np.log10(z)
    keep = lj > ABS_GATE
    if not keep.any():
        return math.nan
    rel = BIAS + 10 * math.log10(z[keep].mean()) - 10
    keep &= lj > rel
    return BIAS + 10 * math.log10(z[keep].mean())


def gain(L: float, target: float) -> float:
    return 10 ** ((target - L) / 20)


def normalize(x, target: float, r: int) -> np.ndarray:
    """float32(g * x) with g from the float64 loudness; a row whose loudness is NaN comes back unchanged."""
    x = np.asarray(x, dtype=np.float32)
    L = integrated(x, r)
    if math.isnan(L):
        return x.copy()
    return (gain(L, target) * x.astype(np.float64)).astype(np.float32)
