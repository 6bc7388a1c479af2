"""Repetition penalty: the decode loop with the per-slot penalty table off and on.

The Air shape with synthetic weights, 500-token prompts and the 249-step decode loop of bench.py (EOS masked, so
every utterance decodes every step), at several batch sizes.  "on" is penalty 1.2 on every slot with the prompt in
the history: the persistent kernel rewrites the history logits in its lm_head epilogue, the per-op chain adds one
fix-up launch after its lm_head, and every sampler step sets one bit.  Off and on alternate in one process, on one
engine, three times each after a warm-up; the decode loop is timed with CUDA events.

    python scripts/bench_repetition_penalty.py [--batches 1 8 16 64] [--repeats 3]

Prints a device line (card name, power limit, maximum SM clock) and one JSON line per (batch, table).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bench_queue import device_line  # noqa: E402

EOS = 151670
PROMPT, STEPS = 500, 249
PENALTY = 1.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 16, 64])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    print(json.dumps(device_line()), flush=True)
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    for B in args.batches:
        lm = SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=1024, max_new=STEPS + 1,
                      max_prefill_tokens=B * PROMPT)
        g = torch.Generator().manual_seed(B)
        prompts = [torch.randint(0, shape.vocab_size, (PROMPT,), generator=g).tolist() for _ in range(B)]
        sp = lm.sampling(EOS, min_new_tokens=STEPS + 1, max_new_tokens=STEPS + 1, seed=1)
        times = {"off": [], "on": []}
        for rep in range(args.repeats + 1):
            for mode in ("off", "on"):
                lm.set_repetition_penalty([(PENALTY, True)] * B if mode == "on" else None)
                lm.prefill(prompts, sp)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                lm.decode(STEPS, sp)
                e1.record()
                torch.cuda.synchronize()
                assert int(lm.n_generated[:B].min()) == STEPS + 1
                if rep:
                    times[mode].append(e0.elapsed_time(e1) * 1e3 / STEPS)
        for mode in ("off", "on"):
            t = sorted(times[mode])
            print(json.dumps({"batch": B, "penalty": mode, "us_per_step_median": round(t[len(t) // 2], 1),
                              "us_per_step_all": [round(x, 1) for x in times[mode]]}), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
