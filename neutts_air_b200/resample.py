"""Output rate and 16-bit PCM on the GPU: a polyphase resampler for whole utterances and for streams (C-ABI
``nt_resampler_*``, include/neutts_b200.h).

Semantics of ``torchaudio.functional.resample(x, 24000, sample_rate)`` with its defaults; ``pcm_format="int16"`` fuses
``__float2int_rn(clip(y, -1, 1) * 32767)`` (clipped to +-32767, rounded half to even) into the same kernel.  That
conversion differs on purpose from ``(y * 32767).astype(np.int16)``, which truncates and wraps values beyond +-1.
A stream resampled push by push is bit-identical to the same samples resampled in one call.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

SRC_RATE = 24_000
PCM_FORMATS = {"float32": 0, "int16": 1}
_DTYPES = {"float32": torch.float32, "int16": torch.int16}


def check_args(sample_rate, pcm_format="float32") -> _lib.ResamplerInfo:
    """Validate an output rate and format (no GPU needed); returns the geometry.  ValueError for a rate that is not a
    positive integer, one whose filter table does not fit an sm_90 block's shared memory, or an unknown format."""
    if isinstance(sample_rate, bool) or not isinstance(sample_rate, (int, np.integer)) or sample_rate <= 0:
        raise ValueError(f"sample_rate {sample_rate!r} must be a positive integer")
    if pcm_format not in PCM_FORMATS:
        raise ValueError(f"pcm_format {pcm_format!r} must be one of {sorted(PCM_FORMATS)}")
    info = _lib.ResamplerInfo()
    _lib.check(_lib.lib().nt_resampler_query(int(sample_rate), C.byref(info)))
    return info


class Resampler:
    """24 kHz float32 PCM -> ``sample_rate`` as float32 or int16, on ``device``; ``max_rows`` independent streams."""

    def __init__(self, sample_rate: int, pcm_format: str = "float32", device="cuda", max_rows: int = 1):
        self.info = check_args(sample_rate, pcm_format)
        if isinstance(max_rows, bool) or not isinstance(max_rows, int) or max_rows < 0:
            raise ValueError(f"max_rows {max_rows!r} must be a non-negative integer")
        if not torch.cuda.is_available():
            raise RuntimeError("neutts_air_b200.Resampler needs a CUDA device (sm_90a); there is no CPU fallback")
        self.L = _lib.lib()
        self.sample_rate, self.pcm_format, self.max_rows = int(sample_rate), pcm_format, max_rows
        self.dtype = _DTYPES[pcm_format]
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device(self.device.type, torch.cuda.current_device())
        with torch.cuda.device(self.device):
            self.table = torch.empty(self.info.table_bytes, dtype=torch.uint8, device=self.device)
            self.state = torch.empty(max(1, max_rows) * self.info.row_bytes, dtype=torch.uint8, device=self.device)
            self.handle = C.c_void_p()
            _lib.check(self.L.nt_resampler_create(self.sample_rate, PCM_FORMATS[pcm_format], max_rows,
                                                  self.table.data_ptr(), self.state.data_ptr(), C.byref(self.handle)))
        self._held = [self.info.width] * max_rows     # the contract's held samples per row (mirrors the library's)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.L.nt_resampler_destroy(self.handle)
        except Exception:
            pass

    def out_len(self, n):
        """Output samples of ``n`` input samples resampled whole: ceil(sample_rate * n / 24000) (n an int or a list)."""
        if isinstance(n, (list, tuple)):
            return [self.out_len(m) for m in n]
        return -(-self.info.target * int(n) // self.info.orig)

    def _span(self, row: int, n: int, final: bool) -> int:
        """Samples a push of n samples to ``row`` makes final (the contract of include/neutts_b200.h)."""
        i = self.info
        h = self._held[row]
        if final:
            return -(-i.target * (h + n - i.width) // i.orig)
        return ((h + n - i.taps) // i.orig + 1) * i.target if h + n >= i.taps else 0

    @torch.no_grad()
    def resample(self, pcm: torch.Tensor) -> torch.Tensor:
        """Rows of equal length on the device (``[..., L]`` float32) -> ``[..., out_len(L)]`` at the output rate, in
        ``pcm_format``, on the same device.  One launch per 128 rows; no stream state is read or written."""
        if pcm.device != self.device:
            raise ValueError(f"pcm is on {pcm.device}, the resampler on {self.device}")
        n = pcm.shape[-1]
        x = pcm.reshape(-1, n).to(torch.float32).contiguous()
        B, m = x.shape[0], self.out_len(n)
        out = torch.empty(B, m, dtype=self.dtype, device=self.device)
        if B and m:
            in_off = (C.c_int64 * (B + 1))(*range(0, (B + 1) * n, n))
            out_off = (C.c_int64 * (B + 1))(*range(0, (B + 1) * m, m))
            with torch.cuda.device(self.device):
                _lib.check(self.L.nt_resampler_push(self.handle, B, None, None, x.data_ptr(), in_off, out.data_ptr(),
                                                    out_off, _lib.current_stream_ptr()))
        return out.reshape(*pcm.shape[:-1], m)

    @torch.no_grad()
    def push(self, rows, chunks, final=False) -> list:
        """Stream: the next 24 kHz samples of each row in ``rows`` (host arrays, any length, empty included) -> the
        output samples that became final, as host numpy arrays in ``pcm_format``.  ``final`` (one bool, or one per
        row) ends a row's stream: the rest of its output comes out and the row starts over.  One host-to-device copy,
        one launch and one device-to-host copy per call (per 128 rows)."""
        rows = [int(r) for r in rows]
        if len(chunks) != len(rows):
            raise ValueError("rows and chunks must have the same length")
        finals = [bool(final)] * len(rows) if isinstance(final, (bool, np.bool_)) else [bool(f) for f in final]
        if len(finals) != len(rows):
            raise ValueError("final must be a bool or one bool per row")
        if len(set(rows)) != len(rows) or any(not 0 <= r < self.max_rows for r in rows):
            raise ValueError(f"rows must be distinct and in 0..{self.max_rows - 1}")
        if not rows:
            return []
        xs = [np.asarray(c, dtype=np.float32).reshape(-1) for c in chunks]
        spans = [self._span(r, len(x), f) for r, x, f in zip(rows, xs, finals)]
        in_off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
        out_off = np.concatenate([[0], np.cumsum(spans)]).astype(np.int64)
        with torch.cuda.device(self.device):
            x = torch.from_numpy(np.concatenate(xs)).to(self.device) if in_off[-1] else None
            out = torch.empty(int(out_off[-1]), dtype=self.dtype, device=self.device)
            _lib.check(self.L.nt_resampler_push(
                self.handle, len(rows), (C.c_int32 * len(rows))(*rows), (C.c_int32 * len(rows))(*finals),
                x.data_ptr() if x is not None else None, in_off.ctypes.data_as(C.POINTER(C.c_int64)),
                out.data_ptr() if out.numel() else None, out_off.ctypes.data_as(C.POINTER(C.c_int64)),
                _lib.current_stream_ptr()))
            host = out.cpu().numpy()
        i = self.info
        for r, x, f, s in zip(rows, xs, finals, spans):
            self._held[r] = i.width if f else self._held[r] + len(x) - s // i.target * i.orig
        return [host[out_off[k]: out_off[k + 1]] for k in range(len(rows))]

    def reset(self, rows) -> None:
        """Rows that start a new stream (a slot given to another utterance, or a stream closed early)."""
        rows = [int(r) for r in rows]
        if any(not 0 <= r < self.max_rows for r in rows):
            raise ValueError(f"rows must be in 0..{self.max_rows - 1}")
        if rows:
            _lib.check(self.L.nt_resampler_reset(self.handle, (C.c_int32 * len(rows))(*rows), len(rows)))
        for r in rows:
            self._held[r] = self.info.width
