"""Length control: the decode loop with the per-slot length-control table off and with the decay active on every slot.

The Air shape with synthetic weights, 500-token prompts and the 249-step decode loop of bench.py, at several batch
sizes.  Both modes are teacher-forced with the same random non-EOS ids, so every utterance decodes every step whatever
the decay does to EOS.  "on" is min_new_tokens 0 and (start 0, factor 1.01) on every slot, so the decay applies from
the first decode step on: the persistent kernel adds it to the EOS row of its lm_head epilogue, the per-op chain adds
one fix-up launch after its lm_head.  Off and on alternate in one process, on one engine, three times each after a
warm-up; the decode loop is timed with CUDA events.

    python scripts/bench_length_control.py [--batches 1 8 16 64] [--repeats 3]

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
DECAY = (0, 1.01)


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
        forced = torch.randint(0, EOS, (B, STEPS + 1), generator=g)
        sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=STEPS + 1, seed=1, forced=forced)
        times = {"off": [], "on": []}
        for rep in range(args.repeats + 1):
            for mode in ("off", "on"):
                lm.set_length_control([(0,) + DECAY] * B if mode == "on" else None)
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
            print(json.dumps({"batch": B, "length_control": mode, "us_per_step_median": round(t[len(t) // 2], 1),
                              "us_per_step_all": [round(x, 1) for x in times[mode]]}), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
