"""Loudness normalisation cost, next to the codec decode of the same audio, and its share of a whole ``infer_batch``.

  * ``normalize``: ``loudness.normalize`` (measure + gain, one call) over batch 1, 8 and 64 rows of 5 s and 40 s at
    24 kHz (speech-like noise with 100 ms level changes), timed with CUDA events; ``measure`` the meter alone;
  * ``codec_decode``: NeuCodec's shape on synthetic weights (3xTF32, the default) for the same rows: 250 and 2000
    frames per row (batch 64 x 40 s is skipped: 128 000 frames in one decode is far past what a serving batch holds);
  * ``infer_batch``: Air-shaped synthetic LM and codec weights, 8 utterances with EOS masked for 250 tokens (5 s), with
    and without ``loudness=-16``, alternated in one process after a warm-up; medians of ``--repeats`` runs.

    python scripts/bench_loudness.py [--iters 20] [--warmup 3] [--repeats 5]

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

from scripts.bench_long_form import make_tts, timed  # noqa: E402
from scripts.bench_queue import device_line  # noqa: E402
from scripts.bench_stretch import _events_ms  # noqa: E402

SR = 24_000
BATCHES = (1, 8, 64)
SECONDS = (5, 40)


def _rows(B, seconds, seed=0):
    rng = np.random.default_rng(seed)
    n, step = seconds * SR, SR // 10
    lvl = np.repeat(10 ** rng.uniform(-1.5, 0, (B, n // step)), step, axis=1)
    return torch.from_numpy((0.1 * rng.standard_normal((B, n)) * lvl).astype(np.float32)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loudness.py needs a CUDA device")
    from neutts_air_b200 import loudness, synthetic
    from neutts_air_b200.codec import CodecDecoder, CodecShape
    from neutts_air_b200.lm import LMShape, SpeechLM

    print(json.dumps(device_line()), flush=True)
    codec_w = synthetic.codec_weights(CodecShape(), 0)
    codecs = {}
    for s in SECONDS:
        for B in BATCHES:
            x = list(_rows(B, s))
            norm, _ = _events_ms(lambda: loudness.normalize(x, -16.0), args.iters, args.warmup)
            meas, _ = _events_ms(lambda: loudness._run(*loudness._pack(x), SR), args.iters, args.warmup)
            line = dict(op="normalize", rows=B, seconds=s, ms_normalize=round(norm, 4), ms_measure=round(meas, 4))
            frames = s * SR // 480
            if B * frames <= 64 * 250:
                key = (B, frames)
                if key not in codecs:
                    codecs.clear()
                    codecs[key] = CodecDecoder(CodecShape(), codec_w, device="cuda", max_batch=key[0], max_frames=frames)
                codes = torch.randint(0, 65536, (B, 1, frames), device="cuda")
                dec, _ = _events_ms(lambda: codecs[key].decode_code(codes), max(3, args.iters // 4), 1)
                line.update(ms_codec=round(dec, 3), normalize_over_codec=round(norm / dec, 4))
            print(json.dumps(line), flush=True)
    codecs.clear()

    B, T = 8, 250
    shape = LMShape()
    lm = SpeechLM(shape, synthetic.lm_state_dict(shape, 1), device="cuda", max_batch=B, max_ctx=2048, max_new=T)
    tts = make_tts(lm, CodecDecoder(CodecShape(), codec_w, device="cuda", max_batch=B, max_frames=T), B)
    ref = torch.randint(0, 65536, (200,), generator=torch.Generator().manual_seed(1))
    texts = [f"utterance number {i} of the batch, read at an even pace." for i in range(B)]
    kw = dict(min_new_tokens=T)
    modes = {"plain": {}, "loudness": dict(loudness=-16.0)}
    for m in modes.values():
        tts.infer_batch(texts, [ref] * B, ["reference text"] * B, **kw, **m)
    res = {k: [] for k in modes}
    for _ in range(args.repeats):
        for k, m in modes.items():
            res[k].append(timed(lambda: tts.infer_batch(texts, [ref] * B, ["reference text"] * B, **kw, **m))[0])
    med = {k: float(np.median(v)) for k, v in res.items()}
    print(json.dumps(dict(op="infer_batch", rows=B, tokens=T, s_plain=round(med["plain"], 4),
                          s_loudness=round(med["loudness"], 4), spread_plain=[round(min(res["plain"]), 4),
                                                                               round(max(res["plain"]), 4)],
                          spread_loudness=[round(min(res["loudness"]), 4), round(max(res["loudness"]), 4)])),
          flush=True)


if __name__ == "__main__":
    main()
