"""Output resampler cost: one-shot rows and streamed pushes, next to a codec decode of the same audio.

A batch of 64 utterances of 10 s each (64 x 240 000 samples at 24 kHz) goes to 16 kHz, 22.05 kHz and 48 kHz, as float32
and as int16:
  * ``resample``: one call over the [64, 240000] device tensor (one kernel launch), timed with CUDA events;
  * ``push``: the same audio streamed as 20 pushes of 0.5 s per row (12 000 samples, the stride of 25 codec frames),
    all 64 rows in every push; each push is one host-to-device copy, one launch and one device-to-host copy, and the
    time is its CUDA-event span (it ends in the device-to-host copy).
Bytes are what the algorithm must move: the 24 kHz fp32 input read once and the output written once (the push line adds
nothing for the history, < 2 KB per row).  GB/s is those bytes over the time.  The codec line decodes 64 x 500 frames
(10 s at 50 frames per second) with NeuCodec's shape on synthetic weights (3xTF32, the default precision), so the
resampler's share can be read off.

    python scripts/bench_resample.py [--iters 20] [--warmup 3] [--out FILE.json]

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
RATES = (16_000, 22_050, 48_000)


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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py needs a CUDA device")
    from neutts_air_b200.resample import Resampler

    dev = torch.device("cuda", torch.cuda.current_device())
    lines = [device_line()]
    print(json.dumps(lines[0]), flush=True)
    n = SECONDS * SRC
    rng = np.random.default_rng(0)
    host = (rng.standard_normal((B, n)) * 0.2).astype(np.float32)
    x = torch.from_numpy(host).to(dev)
    for sr in RATES:
        for fmt, size in (("float32", 4), ("int16", 2)):
            rs = Resampler(sr, fmt, device=dev, max_rows=B)
            m = rs.out_len(n)
            nbytes = B * n * 4 + B * m * size
            med, best = _events_ms(lambda: rs.resample(x), args.iters, args.warmup)
            line = dict(op="resample", rate=sr, pcm=fmt, rows=B, in_samples=n, out_samples=m, bytes=nbytes,
                        ms_median=round(med, 4), ms_min=round(best, 4), gb_s=round(nbytes / med / 1e6, 1))
            print(json.dumps(line), flush=True)
            lines.append(line)

            chunks = [host[:, j: j + CHUNK] for j in range(0, n, CHUNK)]
            rows = list(range(B))

            def stream():
                for k, c in enumerate(chunks):
                    rs.push(rows, list(c), final=k == len(chunks) - 1)

            med, best = _events_ms(stream, max(3, args.iters // 4), 1)
            per = med / len(chunks)
            pbytes = nbytes / len(chunks)
            line = dict(op="push", rate=sr, pcm=fmt, rows=B, pushes=len(chunks), chunk_samples=CHUNK,
                        ms_per_push_median=round(per, 4), ms_stream_median=round(med, 3), ms_stream_min=round(best, 3),
                        bytes_per_push=int(pbytes), gb_s=round(pbytes / per / 1e6, 2))
            print(json.dumps(line), flush=True)
            lines.append(line)
            del rs

    from neutts_air_b200 import synthetic
    from neutts_air_b200.codec import CodecDecoder, CodecShape

    frames = n // 480
    codec = CodecDecoder(CodecShape(), synthetic.codec_weights(CodecShape(), 0), device=dev, max_batch=B, max_frames=frames)
    codes = torch.from_numpy(rng.integers(0, 65536, (B, 1, frames))).to(dev)
    med, best = _events_ms(lambda: codec.decode_code(codes), max(3, args.iters // 4), 1)
    line = dict(op="codec_decode", rows=B, frames=frames, precision="3xtf32", ms_median=round(med, 3), ms_min=round(best, 3))
    print(json.dumps(line), flush=True)
    lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
