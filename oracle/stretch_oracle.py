"""Float64 restatement of the speaking-rate stretch (TEST INFRASTRUCTURE ONLY).

librosa.effects.time_stretch(x, rate=r) as torch / torchaudio compute it, for a row x of L samples at 24 kHz:

    S  = torch.stft(x, 1024, 256, window=hann_window(1024), center=True, pad_mode="constant", return_complex=True)
    S2 = torchaudio.functional.phase_vocoder(S, r, linspace(0, pi * 256, 513)[:, None])
    y  = torch.istft(S2, 1024, 256, window=hann_window(1024), center=True, length=round(L / r))

``phase_vocoder`` below restates torchaudio's function line by line, with output frame j at tau_j = j * r (see
``time_steps``; no torchaudio import: the GPU tests compare against this module alone, and the CPU tests pin it to
torchaudio where it is installed).  ``emitted`` is the streaming
contract of include/neutts_b200.h: how many output samples are final after n input samples.
"""
from __future__ import annotations

import math

import numpy as np
import torch

N_FFT, HOP = 1024, 256
BINS = N_FFT // 2 + 1
MIN_SPEED, MAX_SPEED = 0.5, 2.0


def window() -> torch.Tensor:
    return torch.hann_window(N_FFT, dtype=torch.float64)   # periodic


def out_len(L: int, r: float) -> int:
    """Samples of a row of L samples stretched at r: round(L / r), half to even (Python's round)."""
    return round(L / r)


def analysis(x) -> torch.Tensor:
    """complex128 [513, T], T = 1 + L // 256."""
    x = torch.as_tensor(np.asarray(x, dtype=np.float64))
    return torch.stft(x, N_FFT, HOP, window=window(), center=True, pad_mode="constant", return_complex=True)


def time_steps(T: int, r: float) -> torch.Tensor:
    """tau_j = j * r (one fp64 product per frame) for j < torch.arange's count, ceil(T / r).  torch.arange itself
    returns these values except where its vectorised CPU kernel rounds one an ulp away (for speeds such as 0.7 or
    1/0.9, at positions that depend on the CPU's vector width); when that moves tau_j across an integer, torchaudio
    interpolates another frame pair.  The project's contract is the product, the same on every machine."""
    return torch.arange(len(torch.arange(0, T, r, dtype=torch.float64)), dtype=torch.float64) * r


def phase_vocoder(S: torch.Tensor, r: float, steps: torch.Tensor | None = None) -> torch.Tensor:
    """torchaudio.functional.phase_vocoder(S, r, linspace(0, pi * hop, 513)[:, None]) on complex128 [513, T], with
    the output frame positions ``steps`` (default ``time_steps``; torchaudio uses torch.arange(0, T, r))."""
    if r == 1.0:
        return S
    adv = torch.linspace(0, math.pi * HOP, BINS, dtype=torch.float64)[:, None]
    time_steps_ = time_steps(S.shape[-1], r) if steps is None else steps
    alphas = time_steps_ % 1.0
    phase_0 = S[..., :1].angle()
    Sp = torch.nn.functional.pad(S, [0, 2])
    S0 = Sp.index_select(-1, time_steps_.long())
    S1 = Sp.index_select(-1, (time_steps_ + 1).long())
    phase = S1.angle() - S0.angle() - adv
    phase = phase - 2 * math.pi * torch.round(phase / (2 * math.pi))
    phase = torch.cat([phase_0, (phase + adv)[..., :-1]], dim=-1)
    mag = alphas * S1.abs() + (1 - alphas) * S0.abs()
    return torch.polar(mag, torch.cumsum(phase, -1))


def synthesis(S2: torch.Tensor, length: int) -> np.ndarray:
    """istft of complex128 [513, K] with the analysis window, center, cut or zero-padded to ``length`` (torch.istft
    refuses length 0, whose result is empty)."""
    if length == 0:
        return np.zeros(0)
    return torch.istft(S2, N_FFT, HOP, window=window(), center=True, length=length).numpy()


def time_stretch(x, r: float) -> np.ndarray:
    """One row (1-D) -> float64 [round(L / r)]."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return synthesis(phase_vocoder(analysis(x), r), out_len(len(x), r))


def frames_ready(n: int, r: float) -> int:
    """Output frames whose analysis frames are complete after n input samples: j with 256 a1_j + 512 <= n, where
    a1_j = int(j * r + 1) is the later analysis frame output frame j reads."""
    j = 0
    while int(j * r + 1.0) * HOP + N_FFT // 2 <= n:
        j += 1
    return j


def emitted(n: int, final: bool, r: float) -> int:
    """Output samples final after n input samples (all of them, round(n / r), once the stream ends)."""
    return out_len(n, r) if final else max(0, HOP * frames_ready(n, r) - N_FFT // 2)
