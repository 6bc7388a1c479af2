"""Several takes of one utterance: one forked prefill (generate_batch(num_return_sequences=n)) vs the prompt repeated n
times (generate_batch([prompt] * n)), on the speech LM.

One Air-sized prompt (reference codes plus phonemes, ~600 tokens) on Air-shaped synthetic weights, n = 1, 2, 4, 8 takes
at batch n.  Each take generates a fixed number of tokens (EOS masked).  Reported per (n, mode):
  prefill_ms        device time of the prefill call alone (CUDA events; it includes the first sampler launch)
  ttft_ms           wall time from the prefill call to the first token of every take on the host
  tokens_per_s      generated tokens / wall time of the whole generate_batch call
  pages             KV pages drawn from the pool by the prefill
The two modes alternate in one process, on the same engine.

    python scripts/bench_takes.py [--takes 1 2 4 8] [--prompt 600] [--gen 250] [--repeats 5]

Prints one JSON line per (n, mode) and a device line (card name, power limit, maximum SM clock).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_queue import device_line  # noqa: E402

EOS = 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--takes", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--prompt", type=int, default=600)
    ap.add_argument("--gen", type=int, default=250)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(2000, shape.vocab_size, (args.prompt,), generator=g).tolist()
    print(json.dumps({**device_line(), "prompt_tokens": args.prompt, "generated_per_take": args.gen}), flush=True)
    kw = dict(max_length=2048, min_new_tokens=args.gen, max_new_tokens=args.gen, temperature=1.0, top_k=50, seed=3)
    for n in args.takes:
        lm = SpeechLM(shape, sd, device="cuda", max_batch=n, max_ctx=2048, max_new=args.gen)
        modes = {"fork": lambda sp: lm.prefill_fork([prompt], n, sp), "repeat": lambda sp: lm.prefill([prompt] * n, sp)}
        gens = {"fork": lambda: lm.generate_batch([prompt], EOS, num_return_sequences=n, **kw),
                "repeat": lambda: lm.generate_batch([prompt] * n, EOS, **kw)}
        for name in modes:                      # warm-up: graph capture, lazy module loads
            gens[name]()
        rec = {m: dict(prefill=[], ttft=[], wall=[], pages=None) for m in modes}
        for _ in range(args.repeats):
            for name, pre in modes.items():
                sp = lm.sampling(EOS, args.gen, args.gen, 50, 1.0, 3)
                lm.release_pages()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                pre(sp)
                e1.record()
                first = lm.cur_token[:n].cpu()       # waits for the first token of every take
                t1 = time.perf_counter()
                assert first.numel() == n
                torch.cuda.synchronize()
                r = rec[name]
                r["prefill"].append(e0.elapsed_time(e1))
                r["ttft"].append((t1 - t0) * 1e3)
                r["pages"] = lm.num_pages - lm.pool.num_free
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = gens[name]()
                torch.cuda.synchronize()
                r["wall"].append(time.perf_counter() - t0)
                assert [len(o) for o in out] == [args.gen] * n, name
        for name, r in rec.items():
            wall = float(np.median(r["wall"]))
            print(json.dumps({"takes": n, "mode": name, "prefill_tokens": args.prompt * (1 if name == "fork" else n),
                              "prefill_ms_median": round(float(np.median(r["prefill"])), 3),
                              "prefill_ms": [round(x, 3) for x in r["prefill"]],
                              "ttft_ms_median": round(float(np.median(r["ttft"])), 3),
                              "tokens_per_s": round(n * args.gen / wall, 1), "wall_s_median": round(wall, 3),
                              "pages": r["pages"]}), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
