"""Continuous batching vs fixed chunks on the speech LM: wall time, tokens/s, decode steps and slot occupancy.

64 utterances with 500-token prompts on Air-shaped synthetic weights.  Real speech stops at EOS and output lengths
spread widely; here each utterance gets a seeded cap drawn from U{50..750} and EOS is masked, so it stops exactly at
its cap.  The chunked schedule runs generate_batch per max_batch utterances (each chunk lasts as long as its longest
utterance); the queue runs generate_queue, which refills a slot as soon as its utterance ends.  The two alternate in
one process, on the same engine.

    python scripts/bench_queue.py [--batches 8 16] [--repeats 3] [--n 64]

Prints one JSON line per (max_batch, schedule) and a device line (card name, power limit, maximum SM clock).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EOS = 1000
PROMPT = 500


def device_line() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, pl, clk = [x.strip() for x in out.strip().split(",")]
        return {"device": name, "power_limit_w": float(pl), "sm_max_mhz": float(clk)}
    except Exception:
        return {"device": torch.cuda.get_device_name(), "power_limit_w": None, "sm_max_mhz": None}


class StepCounter:
    """Wraps SpeechLM.decode to count the decode steps each schedule launches."""

    def __init__(self, lm):
        self.lm, self.steps, self._decode = lm, 0, lm.decode
        lm.decode = self

    def __call__(self, n, sp, return_logits=False):
        self.steps += n
        return self._decode(n, sp, return_logits)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--n", type=int, default=64)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    rng = np.random.default_rng(0)
    caps = [int(c) for c in rng.integers(50, 751, size=args.n)]
    g = torch.Generator().manual_seed(1)
    prompts = [torch.randint(2000, shape.vocab_size, (PROMPT,), generator=g).tolist() for _ in range(args.n)]
    total = sum(caps)
    print(json.dumps({**device_line(), "utterances": args.n, "prompt_tokens": PROMPT, "caps": "U{50..750} seed 0",
                      "generated_tokens": total}), flush=True)
    kw = dict(max_length=2048, min_new_tokens=max(caps), temperature=1.0, top_k=50, seed=3)
    for B in args.batches:
        lm = SpeechLM(shape, sd, device="cuda", max_batch=B, max_ctx=2048, max_new=max(caps))
        counter = StepCounter(lm)

        def chunked():
            out = []
            for j in range(0, args.n, B):
                out += lm.generate_batch(prompts[j: j + B], EOS, max_new_tokens=caps[j: j + B], slot_base=j, **kw)
            return out

        def queued():
            return lm.generate_queue(prompts, EOS, max_new_tokens=caps, check_every=32, **kw)

        runs = {"chunked": [], "queue": []}
        for name, fn in (("chunked", chunked), ("queue", queued)):   # warm-up: graph capture, lazy module loads
            fn()
        for _ in range(args.repeats):
            for name, fn in (("chunked", chunked), ("queue", queued)):
                torch.cuda.synchronize()
                counter.steps = 0
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                assert [len(o) for o in out] == caps, name
                runs[name].append((dt, counter.steps))
        for name, r in runs.items():
            times = [t for t, _ in r]
            steps = r[0][1]
            print(json.dumps({"max_batch": B, "schedule": name, "lm_wall_s": [round(t, 3) for t in times],
                              "lm_wall_s_median": round(float(np.median(times)), 3),
                              "tokens_per_s": round(total / float(np.median(times)), 1), "decode_steps": steps,
                              "occupancy": round(total / (B * steps), 3)}), flush=True)
        del lm, counter
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
