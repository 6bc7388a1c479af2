"""Speaking rate on the GPU: a phase-vocoder time stretch of 24 kHz PCM for whole utterances and for streams (C-ABI
``nt_stretch_*``, include/neutts_b200.h).

Semantics of ``librosa.effects.time_stretch(x, rate=speed)`` as torch / torchaudio compute it (stft with n_fft 1024,
hop 256 and a Hann window, ``torchaudio.functional.phase_vocoder``, istft with ``length=round(L / speed)``);
``speed`` > 1 is faster speech, the pitch is kept.  A stream stretched push by push is bit-identical to the same
samples stretched in one call.  A plain phase vocoder (no phase locking) adds some phasiness.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib

N_FFT, HOP = 1024, 256
MIN_SPEED, MAX_SPEED = 0.5, 2.0


def check_speed(speed) -> float:
    """A speed as a float; ValueError for bools, non-numbers, non-finite values and values outside [0.5, 2.0]."""
    if isinstance(speed, (bool, np.bool_)) or not isinstance(speed, (int, float, np.integer, np.floating)):
        raise ValueError(f"speed {speed!r} must be a number in [{MIN_SPEED}, {MAX_SPEED}]")
    s = float(speed)
    if not (math.isfinite(s) and MIN_SPEED <= s <= MAX_SPEED):
        raise ValueError(f"speed {speed!r} must be a finite number in [{MIN_SPEED}, {MAX_SPEED}]")
    return s


def out_len(L: int, speed) -> int:
    """Samples of a row of L samples stretched at ``speed``: round(L / speed), half to even."""
    return round(int(L) / check_speed(speed))


def _frames_ready(n: int, r: float) -> int:
    """Output frames whose analysis frames are complete after n samples (the contract of include/neutts_b200.h)."""
    if n < N_FFT - HOP:
        return 0
    G = (n - N_FFT // 2) // HOP
    j = math.ceil(G / r)
    while j > 0 and int((j - 1) * r + 1.0) > G:
        j -= 1
    while int(j * r + 1.0) <= G:
        j += 1
    return j


def emitted(n: int, final: bool, r: float) -> int:
    """Output samples final after n input samples of a stream at speed r."""
    return round(n / r) if final else max(0, HOP * _frames_ready(n, r) - N_FFT // 2)


class TimeStretch:
    """24 kHz float32 PCM -> the same audio at another speaking rate, on ``device``; ``max_rows`` independent streams."""

    def __init__(self, device="cuda", max_rows: int = 1):
        if isinstance(max_rows, bool) or not isinstance(max_rows, int) or max_rows < 0:
            raise ValueError(f"max_rows {max_rows!r} must be a non-negative integer")
        if not torch.cuda.is_available():
            raise RuntimeError("neutts_air_b200.TimeStretch needs a CUDA device (sm_90a); there is no CPU fallback")
        self.L = _lib.lib()
        self.info = _lib.StretchInfo()
        _lib.check(self.L.nt_stretch_query(C.byref(self.info)))
        self.max_rows = max_rows
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device(self.device.type, torch.cuda.current_device())
        with torch.cuda.device(self.device):
            self.table = torch.empty(self.info.table_bytes, dtype=torch.uint8, device=self.device)
            self.state = torch.empty(max(1, max_rows) * self.info.row_bytes, dtype=torch.uint8, device=self.device)
            self.scratch = torch.empty(self.info.scratch_bytes, dtype=torch.uint8, device=self.device)
            self.handle = C.c_void_p()
            _lib.check(self.L.nt_stretch_create(max_rows, self.table.data_ptr(), self.state.data_ptr(),
                                                self.scratch.data_ptr(), C.byref(self.handle)))
        self._rows = [None] * max_rows     # per row: [samples received, speed] (mirrors the library's contract)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.L.nt_stretch_destroy(self.handle)
        except Exception:
            pass

    @staticmethod
    def out_len(L: int, speed) -> int:
        return out_len(L, speed)

    def _speeds(self, speeds, n: int) -> list:
        if isinstance(speeds, (list, tuple, np.ndarray)):
            if len(speeds) != n:
                raise ValueError(f"speeds has {len(speeds)} entries for {n} rows")
            return [check_speed(s) for s in speeds]
        return [check_speed(speeds)] * n

    def _push(self, n, rows, finals, speeds, x, in_off, out_off) -> torch.Tensor:
        out = torch.empty(int(out_off[-1]), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.nt_stretch_push(
                self.handle, n, rows, finals, (C.c_double * n)(*speeds), x.data_ptr() if x is not None else None,
                in_off.ctypes.data_as(C.POINTER(C.c_int64)), out.data_ptr() if out.numel() else None,
                out_off.ctypes.data_as(C.POINTER(C.c_int64)), _lib.current_stream_ptr()))
        return out

    @torch.no_grad()
    def stretch(self, pcm_rows, speeds) -> list:
        """Rows on the device (a list of 1-D tensors of any lengths, or a [B, L] tensor), each stretched whole at its
        speed (a number or one per row) -> a list of 1-D float32 device tensors of round(L / speed) samples, views
        into one packed buffer.  No stream row is read or written."""
        rows = list(pcm_rows) if not isinstance(pcm_rows, torch.Tensor) or pcm_rows.dim() > 1 else [pcm_rows]
        sp = self._speeds(speeds, len(rows))
        if not rows:
            return []
        for x in rows:
            if x.device != self.device:
                raise ValueError(f"pcm is on {x.device}, the stretcher on {self.device}")
        xs = [x.reshape(-1).to(torch.float32) for x in rows]
        lens = [x.numel() for x in xs]
        spans = [round(n / s) for n, s in zip(lens, sp)]
        in_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        out_off = np.concatenate([[0], np.cumsum(spans)]).astype(np.int64)
        x = torch.cat(xs).contiguous() if in_off[-1] else None
        out = self._push(len(xs), None, None, sp, x, in_off, out_off)
        return [out[out_off[k]: out_off[k + 1]] for k in range(len(xs))]

    def _span(self, row: int, n: int, final: bool, speed: float) -> int:
        recv = self._rows[row][0] if self._rows[row] else 0
        return emitted(recv + n, final, speed) - emitted(recv, False, speed)

    @torch.no_grad()
    def push(self, rows, chunks, speeds, final=False) -> list:
        """Stream: the next 24 kHz samples of each row in ``rows`` (host arrays, any length, empty included) at its speed
        (a number or one per row; a row keeps the speed of its first push until it ends or is reset) -> the output
        samples that became final, as float32 host arrays.  ``final`` (one bool, or one per row) ends a row's stream:
        the rest of its output comes out and the row starts over."""
        rows = [int(r) for r in rows]
        if len(chunks) != len(rows):
            raise ValueError("rows and chunks must have the same length")
        finals = [bool(final)] * len(rows) if isinstance(final, (bool, np.bool_)) else [bool(f) for f in final]
        if len(finals) != len(rows):
            raise ValueError("final must be a bool or one bool per row")
        if len(set(rows)) != len(rows) or any(not 0 <= r < self.max_rows for r in rows):
            raise ValueError(f"rows must be distinct and in 0..{self.max_rows - 1}")
        sp = self._speeds(speeds, len(rows))
        for r, s in zip(rows, sp):
            if self._rows[r] is not None and self._rows[r][1] != s:
                raise ValueError(f"row {r} streams at speed {self._rows[r][1]}, not {s} (reset it to change the speed)")
        if not rows:
            return []
        xs = [np.asarray(c, dtype=np.float32).reshape(-1) for c in chunks]
        spans = [self._span(r, len(x), f, s) for r, x, f, s in zip(rows, xs, finals, sp)]
        in_off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
        out_off = np.concatenate([[0], np.cumsum(spans)]).astype(np.int64)
        with torch.cuda.device(self.device):
            x = torch.from_numpy(np.concatenate(xs)).to(self.device) if in_off[-1] else None
        out = self._push(len(rows), (C.c_int32 * len(rows))(*rows), (C.c_int32 * len(rows))(*finals), sp, x, in_off,
                         out_off)
        host = out.cpu().numpy()
        for r, x, f, s in zip(rows, xs, finals, sp):
            self._rows[r] = None if f else [(self._rows[r][0] if self._rows[r] else 0) + len(x), s]
        return [host[out_off[k]: out_off[k + 1]] for k in range(len(rows))]

    def reset(self, rows) -> None:
        """Rows that start a new stream (a slot given to another utterance, or a stream closed early)."""
        rows = [int(r) for r in rows]
        if any(not 0 <= r < self.max_rows for r in rows):
            raise ValueError(f"rows must be in 0..{self.max_rows - 1}")
        if rows:
            _lib.check(self.L.nt_stretch_reset(self.handle, (C.c_int32 * len(rows))(*rows), len(rows)))
        for r in rows:
            self._rows[r] = None

    def debug(self, name: str, floats: int) -> torch.Tensor:
        """A stage buffer of the last round as a flat float32 device tensor of ``floats`` entries (tests)."""
        p = self.L.nt_stretch_debug_ptr(self.handle, name.encode())
        if not p:
            raise ValueError(f"no stage buffer {name!r}")
        off = p - self.scratch.data_ptr()
        return self.scratch[off: off + 4 * floats].view(torch.float32)
