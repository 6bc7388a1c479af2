"""Repetition-aware sampling: the decode loop with the per-slot RAS table off and on.

The Air shape with synthetic weights, 500-token prompts and the 249-step decode loop of bench.py (EOS masked, so
every utterance decodes every step), at several batch sizes: 1, 8 and 16 run the persistent kernel, 64 the per-op
chain.  "on" is CosyVoice 2's default, (win_size, tau_r) = (10, 0.1), on every slot: every sampled draw counts itself
in the slot's last 10 tokens, and a repeat redraws from the whole row.

Two models per batch:
  * "synthetic": the plain synthetic weights, where the table costs the window count and redraws only the repeats the
    model happens to draw;
  * "forced": one embedding row (tied to the lm_head) is a large constant vector and every prompt ends with it, so
    that id dominates every logits row: every draw repeats and every step after the first redraws (the worst case,
    the full-row pass at every step).
Off and on alternate in one process, on one engine, three times each after a warm-up; after each toggle an untimed
two-step decode rebuilds the chain's decode graph, then the decode loop is timed with CUDA events, and the redraws are
read from the engine's counter.

    python scripts/bench_repetition_aware_sampling.py [--batches 1 8 16 64] [--repeats 3]

Prints a device line (card name, power limit, maximum SM clock) and one JSON line per (model, batch, table).
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
RAS = (10, 0.1)
LOOP_ID = 160000   # the forced model's dominant id (a speech code)


def forced_state_dict(sd: dict) -> dict:
    """The synthetic weights with embedding row LOOP_ID (the tied lm_head row) set to 0.5 in every channel: once it is
    the input, the residual stream points along it and its logit (~0.5 * hidden) dwarfs every other one."""
    sd = dict(sd)
    e = sd["model.embed_tokens.weight"].clone()
    e[LOOP_ID] = 0.5
    sd["model.embed_tokens.weight"] = e
    if "lm_head.weight" in sd:
        h = sd["lm_head.weight"].clone()
        h[LOOP_ID] = 0.5
        sd["lm_head.weight"] = h
    return sd


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
    base = synthetic.lm_state_dict(shape, 0)
    for model in ("synthetic", "forced"):
        sd = base if model == "synthetic" else forced_state_dict(base)
        for B in args.batches:
            lm = SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=1024, max_new=STEPS + 1,
                          max_prefill_tokens=B * PROMPT)
            g = torch.Generator().manual_seed(B)
            prompts = [torch.randint(0, shape.vocab_size, (PROMPT,), generator=g).tolist() for _ in range(B)]
            if model == "forced":
                prompts = [p[:-1] + [LOOP_ID] for p in prompts]
            sp = lm.sampling(EOS, min_new_tokens=STEPS + 1, max_new_tokens=STEPS + 1, seed=1)
            times, redraws = {"off": [], "on": []}, {"off": [], "on": []}
            for rep in range(args.repeats + 1):
                for mode in ("off", "on"):
                    lm.set_repetition_aware_sampling([RAS] * B if mode == "on" else None)
                    lm.prefill(prompts, sp)
                    lm.decode(2, sp)   # untimed: the toggle changed the decode-graph key; the chain captures it here
                    lm.prefill(prompts, sp)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    lm.decode(STEPS, sp)
                    e1.record()
                    torch.cuda.synchronize()
                    assert int(lm.n_generated[:B].min()) == STEPS + 1
                    if rep:
                        times[mode].append(e0.elapsed_time(e1) * 1e3 / STEPS)
                        redraws[mode].append(int(lm.ras_redraws()[:B].sum()))
            for mode in ("off", "on"):
                t = sorted(times[mode])
                print(json.dumps({"model": model, "batch": B, "ras": mode, "us_per_step_median": round(t[len(t) // 2], 1),
                                  "us_per_step_all": [round(x, 1) for x in times[mode]],
                                  "redraw_rate": round(max(redraws[mode]) / (B * STEPS), 4)}), flush=True)
            del lm
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
