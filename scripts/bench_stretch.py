"""Speaking-rate stretch cost: one-shot rows and streamed pushes, next to a codec decode of the same audio.

  * ``stretch``: 64 utterances of 10 s (64 x 240 000 samples at 24 kHz) stretched whole at 0.75 and 1.25, one
    ``TimeStretch.stretch`` call (rounds of 8192 samples x 32 rows, five launches each), timed with CUDA events;
  * ``push``: 25-codec-frame chunks (12 000 samples, the streaming stride) pushed for 8 and 16 rows at once, 20 pushes
    per row ending in a final one; each push is one host-to-device copy, its rounds and one device-to-host copy, and
    the time is its CUDA-event span.  ``latency_samples`` is how far the stretched output lags the input in a stream:
    samples received minus (samples emitted x speed) after a non-final push, which is what the stretch adds to the
    first audio of a stream;
  * ``codec_decode``: 64 x 500 frames (10 s) with NeuCodec's shape on synthetic weights (3xTF32, the default).

    python scripts/bench_stretch.py [--iters 10] [--warmup 2] [--out FILE.json]

Prints a device line (card name, power limit, maximum SM clock), then one JSON line per measurement.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_queue import device_line  # noqa: E402

B, SECONDS, SRC = 64, 10, 24_000
CHUNK = 12_000
SPEEDS = (0.75, 1.25)


def _events_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stretch.py needs a CUDA device")
    from neutts_air_b200.stretch import TimeStretch, emitted

    dev = torch.device("cuda", torch.cuda.current_device())
    lines = [device_line()]
    print(json.dumps(lines[0]), flush=True)
    n = SECONDS * SRC
    rng = np.random.default_rng(0)
    host = (rng.standard_normal((B, n)) * 0.2).astype(np.float32)
    x = torch.from_numpy(host).to(dev)
    ts = TimeStretch(dev, max_rows=16)
    for r in SPEEDS:
        rows = list(x)
        med, best = _events_ms(lambda: ts.stretch(rows, r), args.iters, args.warmup)
        line = dict(op="stretch", speed=r, rows=B, in_samples=n, out_samples=round(n / r), ms_median=round(med, 3),
                    ms_min=round(best, 3), audio_s_per_ms=round(B * SECONDS / med, 2))
        print(json.dumps(line), flush=True)
        lines.append(line)
        for nrows in (8, 16):
            chunks = [host[:nrows, j: j + CHUNK] for j in range(0, 20 * CHUNK, CHUNK)]

            def stream():
                for k, c in enumerate(chunks):
                    ts.push(range(nrows), list(c), r, final=k == len(chunks) - 1)

            med, best = _events_ms(stream, max(3, args.iters // 2), 1)
            lag = max(m - emitted(m, False, r) * r for m in range(CHUNK, 20 * CHUNK, CHUNK))
            line = dict(op="push", speed=r, rows=nrows, pushes=len(chunks), chunk_samples=CHUNK,
                        ms_per_push_median=round(med / len(chunks), 4), ms_stream_median=round(med, 3),
                        ms_stream_min=round(best, 3), latency_samples=round(lag, 1))
            print(json.dumps(line), flush=True)
            lines.append(line)

    from neutts_air_b200 import synthetic
    from neutts_air_b200.codec import CodecDecoder, CodecShape

    frames = n // 480
    codec = CodecDecoder(CodecShape(), synthetic.codec_weights(CodecShape(), 0), device=dev, max_batch=B, max_frames=frames)
    codes = torch.from_numpy(rng.integers(0, 65536, (B, 1, frames))).to(dev)
    med, best = _events_ms(lambda: codec.decode_code(codes), max(3, args.iters // 2), 1)
    line = dict(op="codec_decode", rows=B, frames=frames, precision="3xtf32", ms_median=round(med, 3), ms_min=round(best, 3))
    print(json.dumps(line), flush=True)
    lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
