"""Every engine call SpeechLM.generate_queue makes, pinned call for call on a CPU stub engine.

Each scenario runs generate_queue on ``RecordingStub`` and records the engine calls with their arguments (sampling
params, every per-slot table write, prefill, prefill_slots, decode), what the call returned (or the ValueError it
raised) and whether every KV page went back to the pool.  tests/golden/queue_calls.json holds the expected records.
"""
import json
import os

import pytest
import torch

from neutts_air_b200.lm import LMShape
from tests.fakes import EOS, GuidedStub

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "queue_calls.json")


class RecordingStub(GuidedStub):
    """GuidedStub that records every engine call with its arguments; tables are recorded as written, rows and slots."""

    shape = LMShape(vocab_size=16384)

    def __init__(self, max_batch, eos_at=None):
        super().__init__(max_batch, eos_at)
        self.calls = []

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, forced=None, limits=None, slot_base=0):
        self.calls.append(["sampling", min_new, max_new, top_k, temperature, seed, greedy,
                           None if limits is None else list(limits), slot_base])
        return super().sampling(eos, min_new, max_new, top_k, temperature, seed, greedy, forced, limits, slot_base)

    def _table(self, name, mirror, rows, slots):
        self.calls.append([name, None if rows is None else [list(r) for r in rows], None if slots is None else list(slots)])
        setattr(self, mirror, rows)

    def set_slot_sampling(self, rows, slots=None):
        self._table("set_slot_sampling", "_slot_sp_host", rows, slots)

    def set_repetition_penalty(self, rows, slots=None):
        self._table("set_repetition_penalty", "_penalty_host", rows, slots)

    def set_length_control(self, rows, slots=None):
        self._table("set_length_control", "_length_host", rows, slots)

    def set_vocab_range(self, lo, hi=None):
        self.calls.append(["set_vocab_range", lo, hi])
        self._vocab_range = None if lo is None else (lo, hi)

    def set_logprobs(self, on=True):
        self.calls.append(["set_logprobs", on])
        self.logprobs = torch.zeros(self.max_batch, self.max_new, 2) if on else None

    def set_guidance(self, rows, slots=None):
        self.calls.append(["set_guidance", None if rows is None else [list(r) for r in rows],
                           None if slots is None else list(slots)])
        super().set_guidance(rows, slots)

    def prefill(self, prompts, sp):
        self.calls.append(["prefill", [[p[0], len(p)] for p in prompts]])   # tag (negative: a negative prompt), length
        super().prefill(prompts, sp)

    def prefill_slots(self, slots, prompts, sp, stream_ids, return_logits=False, limits=None):
        self.calls.append(["prefill_slots", list(slots), [[p[0], len(p)] for p in prompts], list(stream_ids),
                           None if limits is None else list(limits)])
        super().prefill_slots(slots, prompts, sp, stream_ids, return_logits, limits)

    def decode(self, n, sp):
        self.calls.append(["decode", n])
        super().decode(n, sp)


def _tagged(lens, sign=1):
    """Prompt i: the id sign * (i + 1), repeated lens[i] times (the stubs read a prompt's index from its ids)."""
    return [[sign * (i + 1)] * m for i, m in enumerate(lens)]


def _negs(lens):
    return [None if m is None else [-(i + 1)] * m for i, m in enumerate(lens)]


LENS7 = [90, 80, 95, 70, 99, 85, 60]   # max_length 100 -> caps 10, 20, 5, 30, 1, 15, 40

SCENARIOS = {
    "unguided_7_on_3": dict(slots=3, calls=[dict(
        prompts=_tagged(LENS7), max_length=100, min_new_tokens=100, check_every=8, slot_base=40)]),
    "unguided_early_eos_2_on_8": dict(slots=8, eos_at={2: 3}, calls=[dict(
        prompts=_tagged([10, 20]), max_length=60, min_new_tokens=0, check_every=5)]),
    "unguided_done_at_prefill": dict(slots=3, eos_at={6: 0}, calls=[dict(
        prompts=_tagged(LENS7), max_length=100, min_new_tokens=0, check_every=8)]),
    "unguided_per_prompt_settings": dict(slots=4, eos_at={3: 7}, calls=[dict(
        prompts=_tagged([40, 55, 30, 62, 48, 35, 50]), max_length=100, check_every=6, slot_base=3,
        temperature=[0.7, 1.0, 1.3, 0.9, 1.1, 0.8, 1.2], top_p=0.9, min_new_tokens=[0, 3, 20, 5, 2, 8, 1],
        repetition_penalty=[1.0, 1.2, 1.0, 1.5, 1.1, 1.0, 1.3], exponential_decay_length_penalty=(30, 1.02),
        vocab_range=(1024, 8192), return_logprobs=True)]),
    "mixed_7_on_4": dict(slots=4, eos_at={2: 4, 6: 10}, calls=[dict(
        prompts=_tagged([90, 80, 95, 70, 60, 85, 75]), max_length=100, min_new_tokens=2, check_every=8, slot_base=40,
        guidance_scale=[2.0, 1.0, 3.0, 3.0, 1.0, 2.0, 1.5], negative_prompt_ids=_negs([5, 3, 7, 2, 4, 6, 1]))]),
    "late_prompt_guided": dict(slots=3, calls=[dict(
        prompts=_tagged([20, 30, 25, 15, 22]), max_length=60, min_new_tokens=1, check_every=4,
        guidance_scale=[1.0, 1.0, 1.0, 1.0, 2.5], negative_prompt_ids=_negs([None] * 4 + [4]))]),
    "all_guided_5_slots": dict(slots=5, eos_at={1: 6, 4: 12}, calls=[dict(
        prompts=_tagged([30, 40, 35, 25, 45, 20]), max_length=80, check_every=5, slot_base=7,
        guidance_scale=[2.0, 3.0, 1.5, 2.0, 4.0, 2.5], negative_prompt_ids=_negs([3, 4, 2, 5, 1, 3]),
        temperature=[0.8, 1.0, 1.2, 0.9, 1.1, 0.7], top_k=[40, 50, 20, 64, 10, 30], repetition_penalty=1.2,
        min_new_tokens=[0, 5, 2, 0, 3, 1])]),
    "guided_on_1_slot": dict(slots=1, calls=[dict(
        prompts=_tagged([10, 12]), guidance_scale=[1.0, 2.0], negative_prompt_ids=_negs([2, 2]))]),
    "unguided_on_1_slot": dict(slots=1, eos_at={2: 5}, calls=[dict(
        prompts=_tagged([30, 20, 40, 10]), max_length=60, min_new_tokens=0, check_every=7)]),
    "guided_then_unguided": dict(slots=4, calls=[
        dict(prompts=_tagged([20, 30, 25]), max_length=50, min_new_tokens=0, check_every=6,
             guidance_scale=[2.0, 1.0, 3.0], negative_prompt_ids=_negs([2, None, 3])),
        dict(prompts=_tagged([10, 15, 12, 18, 9]), max_length=40, min_new_tokens=0, check_every=6)]),
}


def record(spec) -> dict:
    """The engine calls, results and page-pool state of one scenario, in JSON form."""
    lm = RecordingStub(spec["slots"], spec.get("eos_at"))
    results = []
    for kw in spec["calls"]:
        try:
            out = lm.generate_queue(eos_token_id=EOS, **kw)
        except ValueError as e:
            results.append({"error": str(e)})
            continue
        if kw.get("return_logprobs"):
            out, lps = out
            results.append({"ids": [o.tolist() for o in out], "logprobs": [list(lp.shape) for lp in lps]})
        else:
            results.append({"ids": [o.tolist() for o in out]})
    pages_back = sorted(lm.pool.free) == list(range(lm.num_pages)) and all(not p for p in lm._slot_pages)
    return json.loads(json.dumps({"calls": lm.calls, "results": results, "pages_back": pages_back}))


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_queue_engine_calls(name):
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    assert record(SCENARIOS[name]) == want


if __name__ == "__main__":
    # Rewrites the golden; run it only when the call sequence is meant to change:  python -m tests.test_queue_calls
    with open(GOLDEN, "w") as f:   # one scenario per line
        f.write("{\n" + ",\n".join(f"{json.dumps(name)}: {json.dumps(record(spec), separators=(',', ':'))}"
                                   for name, spec in sorted(SCENARIOS.items())) + "\n}\n")
