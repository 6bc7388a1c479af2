"""Teacher-forced scoring: ``SpeechLM.score`` against the decode-loop route it replaces.

The Air shape with synthetic weights; B sequences of 500 prompt + 250 scored tokens.  "score" is one ``score`` call
(``nt_lm_score``: one prefill pass over all 750 tokens, the lm_head with its log-softmax epilogue over the 250 scored
rows of every sequence).  "decode" is the route that existed before: ``prefill`` of the prompt, then 249 teacher-forced
decode steps with ``set_logprobs`` on, reading the ``model`` column.  The two alternate in one process, three times each
after a warm-up, timed with CUDA events.

    python scripts/bench_score.py [--batches 1 8 32] [--repeats 3]

Prints a device line (card name, power limit, maximum SM clock) and one JSON line per (batch, route).
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
PROMPT, SCORED = 500, 250


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    print(json.dumps(device_line()), flush=True)
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    L = PROMPT + SCORED
    for B in args.batches:
        lm = SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=1024, max_new=SCORED,
                      max_prefill_tokens=B * L)
        g = torch.Generator().manual_seed(B)
        seqs = [torch.randint(0, shape.vocab_size, (L,), generator=g).tolist() for _ in range(B)]
        forced = torch.tensor([s[PROMPT:] for s in seqs], dtype=torch.int32)
        sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=SCORED, forced=forced, seed=1)
        times = {"score": [], "decode": []}
        for rep in range(args.repeats + 1):
            for route in ("score", "decode"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                if route == "score":
                    out = lm.score(seqs, PROMPT)
                else:
                    lm.set_logprobs(True)
                    lm.prefill([s[:PROMPT] for s in seqs], sp)
                    lm.decode(SCORED - 1, sp)
                e1.record()
                torch.cuda.synchronize()
                if route == "decode":
                    assert int(lm.n_generated[:B].min()) == SCORED
                    lm.set_logprobs(False)
                    lm.release_pages()
                else:
                    assert all(o.shape == (SCORED,) and bool(torch.isfinite(o).all()) for o in out)
                if rep:
                    times[route].append(e0.elapsed_time(e1))
        for route in ("score", "decode"):
            t = sorted(times[route])
            med = t[len(t) // 2]
            print(json.dumps({"batch": B, "route": route, "ms_median": round(med, 2), "ms_all": [round(x, 2) for x in times[route]],
                              "scored_tokens_per_s": round(B * SCORED / med * 1e3)}), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
