"""Classifier-free guidance: the decode step with and without an unconditional partner per utterance.

The Air shape with synthetic weights, 500-token prompts, negative prompts of 350 tokens (the prompt's first 350 ids:
the same reference without the target text) and the 249-step decode loop of bench.py (EOS masked, so every sequence
decodes every step), for U utterances, i.e. 2U slots.  Three cases alternate in one process, on one engine, three
times each after a warm-up, and the decode loop is timed with CUDA events:

  * "default": 2U unguided prompts on the engine's default decode path (the persistent kernel up to 16 slots);
  * "chain": the same 2U unguided prompts on the per-op chain (NT_DECODE_IMPL=perop), the path guidance runs on;
  * "guided": U guided prompts (scale 3) and their U negative prompts.

Then one profiled guided decode (torch.profiler, CUDA activities) gives the share of the combine
(guidance_lse_kernel, guidance_mix_kernel) and follow (guidance_follow_kernel) kernels in the step's kernel time.

    python scripts/bench_guidance.py [--utterances 1 4 8 32] [--repeats 3]

Prints a device line (card name, power limit, maximum SM clock) and one JSON line per (utterances, case), with the
median microseconds per decode step.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bench_queue import device_line  # noqa: E402

EOS = 151670
PROMPT, NEG, STEPS = 500, 350, 249
SCALE = 3.0


def _decode_us(lm, prompts, sp, table, impl):
    """One prefill and the timed decode loop -> microseconds per step."""
    if impl:
        os.environ["NT_DECODE_IMPL"] = impl
    else:
        os.environ.pop("NT_DECODE_IMPL", None)
    lm.set_guidance(table)
    lm.prefill(prompts, sp)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    lm.decode(STEPS, sp)
    e1.record()
    torch.cuda.synchronize()
    assert int(lm.n_generated[: len(prompts)].min()) == STEPS + 1
    return 1e3 * e0.elapsed_time(e1) / STEPS


def _kernel_share(lm, prompts, sp, table):
    """Share of the guidance kernels in the CUDA kernel time of a profiled guided decode."""
    from torch.profiler import ProfilerActivity, profile

    os.environ.pop("NT_DECODE_IMPL", None)
    lm.set_guidance(table)
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lm.decode(STEPS, sp)
        torch.cuda.synchronize()
    total = combine = follow = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        total += t
        if "guidance_lse_kernel" in e.key or "guidance_mix_kernel" in e.key:
            combine += t
        elif "guidance_follow_kernel" in e.key:
            follow += t
    return {"combine_share": combine / total if total else None, "follow_share": follow / total if total else None,
            "combine_us_per_step": combine / STEPS, "follow_us_per_step": follow / STEPS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, nargs="+", default=[1, 4, 8, 32])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    print(json.dumps(device_line()), flush=True)
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    for U in args.utterances:
        S = 2 * U
        lm = SpeechLM(shape, sd, device="cuda:0", max_batch=S, max_ctx=1024, max_new=STEPS + 1,
                      max_prefill_tokens=S * PROMPT)
        g = torch.Generator().manual_seed(U)
        prompts = [torch.randint(0, shape.vocab_size, (PROMPT,), generator=g).tolist() for _ in range(U)]
        guided = prompts + [p[:NEG] for p in prompts]   # c slots 0..U-1, u slots U..2U-1
        table = [(U + i, SCALE) for i in range(U)] + [(-1, 1.0)] * U
        unguided = prompts + [torch.randint(0, shape.vocab_size, (PROMPT,), generator=g).tolist() for _ in range(U)]
        sp = lm.sampling(EOS, min_new_tokens=STEPS + 1, max_new_tokens=STEPS + 1, seed=1)
        cases = {"default": (unguided, None, None), "chain": (unguided, None, "perop"), "guided": (guided, table, None)}
        times = {k: [] for k in cases}
        for rep in range(args.repeats + 1):
            for name, (ps, tab, impl) in cases.items():
                us = _decode_us(lm, ps, sp, tab, impl)
                if rep:
                    times[name].append(us)
        share = _kernel_share(lm, guided, sp, table)
        lm.set_guidance(None)
        for name, ts in times.items():
            row = {"utterances": U, "slots": S, "case": name, "us_per_step": statistics.median(ts), "runs": ts}
            if name == "guided":
                row.update(share)
            print(json.dumps(row), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
