"""Timeline of one batch-1 decode step of the persistent decode kernel, from its %globaltimer marks.

The Air shape with synthetic weights, one 500-token prompt and the 249-step decode loop of bench.py (EOS masked).
``nt_lm_debug_set_profile`` makes thread 0 of CTAs 0 and 1 record a mark at the end of every phase of one chosen step,
and fine marks inside layer 2 and the sampler.  CTA 0 owns qkv, o_proj and down_proj items and the first attention
split; CTA 1 owns gate/up units and the second attention split.  Marks 11 and 12 bracket a tile fold, recorded only when
the CTA stores the last slice of a qkv, o_proj, gate/up or down_proj tile.  The marks cost a global
store each, so the timeline runs in launches of its own, never on the bench path.

    python scripts/profile_decode_tc.py [--repeats 3] [--step 100]

Prints a device line (card name, power limit, maximum SM clock), then per launch and CTA the per-phase averages over
layers 1..L-1 (µs), and the fine marks of layer 2 of the last launch relative to the end of layer 1.
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

# coarse marks (every layer): the end of each phase; 104 closes a layer
COARSE = {100: "qkv (ln1 fold + projection)", 101: "attention", 102: "o_proj (merge + projection)",
          103: "gate/up (ln2 fold + projection)", 104: "down (SwiGLU staging + projection)"}
FINE = {1: "fold: start", 2: "fold: rows read", 4: "fold: staged", 5: "bop ready", 10: "split-K item out", 11: "tile fold: last arrival", 12: "tile fold: rows out", 21: "attention: start", 22: "attention: prologue done", 23: "attention: page in",
        25: "attention: partials out", 31: "o_proj input: staged", 32: "o_proj input: bop ready",
        41: "down input: staged", 42: "down input: bop ready", 50: "gate/up item out", 110: "lm_head done",
        111: "sampler done", 200: "grid barrier passed", 0: "step start"}


def marks_of(buf, cta):
    t, ids = buf[cta, :512].tolist(), buf[cta, 512:].tolist()
    n = next((i for i, v in enumerate(t) if v == 0), 512)
    return list(zip(t[:n], ids[:n]))


def phases(marks, n_layers):
    """Per coarse phase: the time from the previous coarse mark (the step start for layer 0's qkv), one entry per layer."""
    out = {k: [] for k in COARSE}
    prev = marks[0][0]
    layer_ends = []
    for t, i in marks:
        if i in COARSE:
            out[i].append((t - prev) / 1e3)
            prev = t
            if i == 104:
                layer_ends.append(t)
    assert all(len(v) == n_layers for v in out.values()), {k: len(v) for k, v in out.items()}
    return out, layer_ends


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--step", type=int, default=100, help="decode step (of the 249) whose timeline is recorded")
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    print(json.dumps(device_line()), flush=True)
    shape = LMShape()
    L = shape.num_layers
    lm = SpeechLM(shape, synthetic.lm_state_dict(shape, 0), device="cuda:0", max_batch=1, max_ctx=1024,
                  max_new=STEPS + 1, max_prefill_tokens=PROMPT)
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(0, shape.vocab_size, (PROMPT,), generator=g).tolist()
    sp = lm.sampling(EOS, min_new_tokens=STEPS + 1, max_new_tokens=STEPS + 1, seed=1)
    buf = torch.zeros(2, 1024, dtype=torch.int64, device="cuda:0")
    for rep in range(args.repeats + 1):
        buf.zero_()
        lm.prefill([prompt], sp)
        lm.L.nt_lm_debug_set_profile(lm.handle, buf.data_ptr() if rep else None, args.step)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lm.decode(STEPS, sp)
        e1.record()
        torch.cuda.synchronize()
        lm.L.nt_lm_debug_set_profile(lm.handle, None, 0)
        if not rep:
            continue   # warm-up
        host = buf.cpu()
        for cta in (0, 1):
            m = marks_of(host, cta)
            ph, ends = phases(m, L)
            step_us = (m[-1][0] - m[0][0]) / 1e3
            layer_us = (ends[-1] - ends[0]) / 1e3 / (L - 1)
            line = {"launch": rep, "cta": cta, "us_per_step_launch": round(e0.elapsed_time(e1) * 1e3 / STEPS, 1),
                    "step_us": round(step_us, 1), "layer_us": round(layer_us, 2),
                    "phase_us": {COARSE[k]: round(sum(v[1:]) / (L - 1), 2) for k, v in ph.items()},
                    "head_and_sampler_us": round((m[-1][0] - ends[-1]) / 1e3, 1)}
            print(json.dumps(line), flush=True)
            if rep == args.repeats:
                t0 = ends[1]   # end of layer 1 = start of layer 2
                fine = [(round((t - t0) / 1e3, 2), i, FINE.get(i, COARSE.get(i, "?"))) for t, i in m if ends[1] < t <= ends[2]]
                for t, i, name in fine:
                    print(f"  cta {cta} layer 2 +{t:7.2f} us  [{i:3d}] {name}")


if __name__ == "__main__":
    main()
