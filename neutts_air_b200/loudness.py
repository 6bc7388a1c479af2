"""Loudness on the GPU: ITU-R BS.1770-4 integrated loudness of mono rows, and normalisation to a loudness target
(C-ABI ``nt_loudness_*``, include/neutts_b200.h).

The meter is ``torchaudio.functional.loudness`` in float64 with two deliberate differences: no K-weighting stage is
clamped to [-1, 1] (torchaudio's ``lfilter`` clamps by default, which misreads loud material; BS.1770 does not clamp),
and a row shorter than one 400 ms gating block reads NaN instead of raising.  Silence reads NaN too.

Normalising scales each row by g = 10^((T - L) / 20), each sample rounded once to float32; a row whose loudness is NaN
comes back unchanged, and nothing limits the peaks.  Re-measuring a normalised row gives T, except where the gain
moves a block across the -70 LUFS absolute gate: which blocks count then changes, which BS.1770's gating implies.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib

MIN_RATE, MAX_RATE = 8000, 192000
MIN_TARGET, MAX_TARGET = -70.0, 0.0


def check_rate(sample_rate) -> int:
    """A meter rate as an int: a multiple of 10 Hz in [8000, 192000] (a gating block is then exactly four 100 ms
    steps); ValueError with the reason otherwise."""
    if isinstance(sample_rate, (bool, np.bool_)) or not isinstance(sample_rate, (int, np.integer)):
        raise ValueError(f"sample_rate {sample_rate!r} must be an integer")
    r = int(sample_rate)
    if not MIN_RATE <= r <= MAX_RATE:
        raise ValueError(f"sample_rate {r} must be in [{MIN_RATE}, {MAX_RATE}]")
    if r % 10:
        raise ValueError(f"sample_rate {r} must be a multiple of 10 Hz (a 100 ms step must be whole samples)")
    return r


def check_target(target) -> float:
    """A loudness target as a float: finite, in [-70, 0] LUFS; ValueError otherwise."""
    if isinstance(target, (bool, np.bool_)) or not isinstance(target, (int, float, np.integer, np.floating)):
        raise ValueError(f"loudness target {target!r} must be a number in [{MIN_TARGET}, {MAX_TARGET}] LUFS")
    t = float(target)
    if not (math.isfinite(t) and MIN_TARGET <= t <= MAX_TARGET):
        raise ValueError(f"loudness target {target!r} must be finite and in [{MIN_TARGET}, {MAX_TARGET}] LUFS")
    return t


def query(sample_rate=24000) -> _lib.LoudnessInfo:
    """Gate, step and chunk geometry of a rate (no GPU needed)."""
    info = _lib.LoudnessInfo()
    _lib.check(_lib.lib().nt_loudness_query(check_rate(sample_rate), C.byref(info)))
    return info


def _pack(rows):
    """Rows (device tensors, or host arrays moved to the device) -> packed float32 device buffer and host offsets."""
    rows = list(rows) if not isinstance(rows, torch.Tensor) or rows.dim() > 1 else [rows]
    if not torch.cuda.is_available():
        raise RuntimeError("neutts_air_b200.loudness needs a CUDA device (sm_90a); there is no CPU fallback")
    dev = next((x.device for x in rows if isinstance(x, torch.Tensor) and x.is_cuda), None)
    dev = dev or torch.device("cuda", torch.cuda.current_device())
    xs = [(x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, dtype=np.float32)))
          .reshape(-1).to(device=dev, dtype=torch.float32) for x in rows]
    off = np.concatenate([[0], np.cumsum([x.numel() for x in xs])]).astype(np.int64)
    x = torch.cat(xs).contiguous() if xs else torch.empty(0, dtype=torch.float32, device=dev)
    return x, off, dev


def _run(x, off, dev, sample_rate, targets=None, out=None) -> torch.Tensor:
    r = check_rate(sample_rate)
    L = _lib.lib()
    n = len(off) - 1
    lufs = torch.empty(n, dtype=torch.float64, device=dev)
    if n == 0:
        return lufs
    offp = off.ctypes.data_as(C.POINTER(C.c_int64))
    ws = torch.empty(max(1, L.nt_loudness_workspace_bytes(r, n, offp)), dtype=torch.uint8, device=dev)
    tg = None if targets is None else (C.c_double * n)(*targets)
    with torch.cuda.device(dev):
        _lib.check(L.nt_loudness_run(r, n, x.data_ptr() if x.numel() else None, offp, tg, lufs.data_ptr(),
                                     out.data_ptr() if out is not None and out.numel() else None, ws.data_ptr(),
                                     ws.numel(), _lib.current_stream_ptr()))
    return lufs


@torch.no_grad()
def measure(rows, sample_rate=24000) -> np.ndarray:
    """Integrated loudness in LUFS of each row (device tensors or host arrays, any lengths; a [B, L] tensor is B rows)
    -> float64 host array; NaN for a silent row or one shorter than 400 ms."""
    x, off, dev = _pack(rows)
    return _run(x, off, dev, sample_rate).cpu().numpy()


@torch.no_grad()
def normalize(rows, targets, sample_rate=24000) -> list:
    """Each row scaled to its loudness target (a number, or one per row with None for a row to leave alone; each in
    [-70, 0] LUFS) -> a list of float32 device tensors, views into one packed buffer.  Runs on the current stream
    without synchronising the host.  A row whose loudness is NaN (silent, or shorter than 400 ms) is returned
    unchanged.  The gain can move a block across the -70 LUFS absolute gate, and a row re-measured then reads slightly
    off its target."""
    x, off, dev = _pack(rows)
    n = len(off) - 1
    if isinstance(targets, (list, tuple, np.ndarray)):
        if len(targets) != n:
            raise ValueError(f"targets has {len(targets)} entries for {n} rows")
        tg = [math.nan if t is None else check_target(t) for t in targets]
    else:
        tg = [check_target(targets)] * n
    out = torch.empty_like(x)
    _run(x, off, dev, sample_rate, tg, out)
    return [out[off[k]: off[k + 1]] for k in range(n)]
