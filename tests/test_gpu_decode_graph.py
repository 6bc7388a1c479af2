"""GPU: the per-op chain's cached decode graph follows every host setting it bakes into its launches.

``nt_lm_decode`` replays one captured step when the chain runs more than one step with no logits output.  Each case
switches a setting between such launches: the slot sampling table (on, new values, off), the vocabulary range (on,
changed, off), the repetition penalty (on, off), the sampler capture (on, off) and the layer count (1, all).  The
reference is the same sequence on the same engine as single-step ``decode(1)`` calls, which never use the graph.
After every launch, out_tokens, n_generated, done and the capture buffers must be bit-identical between the two.
Every switch must also change the outcome against the same run without it, so that no case passes vacuously.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import lm_oracle as LO
from tests.helpers import make_lm, set_decode_impl

pytestmark = pytest.mark.gpu

V, EOS, K = 2048, 7, 4     # vocabulary, EOS id (masked throughout by min_new_tokens), steps per launch


def _slot_rows(B: int, shift: int) -> list:
    return [(0.6 + 0.1 * ((s + shift) % 8), 64 - (5 * s + shift) % 40, 0.95, 0.01 * ((s + shift) % 3)) for s in range(B)]


# name -> (greedy, the setting's states: state 0 before the prefill, state i before launch i)
CASES = {
    "slot-table": (False, [lambda lm: lm.set_slot_sampling(_slot_rows(lm.max_batch, 0)),
                           lambda lm: lm.set_slot_sampling(_slot_rows(lm.max_batch, 3)),
                           lambda lm: lm.set_slot_sampling(None)]),
    "vocab-range": (False, [lambda lm: lm.set_vocab_range(256, 1024), lambda lm: lm.set_vocab_range(1024, V),
                            lambda lm: lm.set_vocab_range(None)]),
    # greedy: the tied-embedding model repeats tokens, which the penalty breaks
    "penalty": (True, [lambda lm: lm.set_repetition_penalty([(4.0, True)] * lm.max_batch),
                       lambda lm: lm.set_repetition_penalty(None)]),
    "capture": (False, [lambda lm: lm.debug_capture_sampler(True), lambda lm: lm.debug_capture_sampler(False)]),
    "layers": (False, [lambda lm: lm.debug_set_layers(1), lambda lm: lm.debug_set_layers(-1)]),
}


def _reset(lm) -> None:
    lm.set_slot_sampling(None)
    lm.set_vocab_range(None)
    lm.set_repetition_penalty(None)
    lm.debug_capture_sampler(False)
    lm.debug_set_layers(-1)


def _run(lm, prompts, greedy, states, launches, graph) -> list:
    """Applies states[0], prefills, then runs ``launches`` launches of K steps, applying states[i] (when there is one)
    before launch i.  graph: one decode(K) per launch, else K decode(1) calls.  Returns the outcome after each launch."""
    B = len(prompts)
    _reset(lm)
    # a prefill leaves the columns past n_generated as an earlier run wrote them, and after a run on fewer layers the
    # other layers attend over cache rows that no prefill wrote
    lm.out_tokens.zero_()
    lm.kv.zero_()
    sp = lm.sampling(EOS, min_new_tokens=64, max_new_tokens=64, top_k=50, temperature=1.0, seed=11, greedy=greedy)
    states[0](lm)
    cap = lm._capture
    lm.prefill(prompts, sp)
    out = []
    for i in range(launches):
        if 0 < i < len(states):
            states[i](lm)
        cap = lm._capture if lm._capture is not None else cap
        for steps in [K] if graph else [1] * K:
            lm.decode(steps, sp)
        torch.cuda.synchronize()
        got = [lm.out_tokens[:B], lm.n_generated[:B], lm.done[:B]] + list(cap or [])
        out.append([t.cpu().numpy().copy() for t in got])
    return out


def _same(a, b) -> bool:
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("B,impl", [(3, "perop"), (17, None)], ids=["chain-b3", "chain-b17"])
@pytest.mark.parametrize("case", list(CASES))
def test_decode_graph_follows_setting(cuda, case, B, impl, monkeypatch):
    set_decode_impl(monkeypatch, impl)   # batch 17 takes the chain by default
    cfg = LO.LMConfig.tiny(vocab_size=V, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    lm = make_lm(cfg, LO.random_weights(cfg, 5, bf16_round=True), max_batch=B, max_ctx=256, max_new=64)
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(EOS + 1, V, (20 + 3 * b,), generator=g).tolist() for b in range(B)]
    greedy, states = CASES[case]
    n = len(states)
    got = _run(lm, prompts, greedy, states, n, graph=True)
    want = _run(lm, prompts, greedy, states, n, graph=False)
    for i in range(n):
        assert _same(got[i], want[i]), (case, B, f"launch {i}")
    for i in range(1, n):   # the same run without switch i
        without = _run(lm, prompts, greedy, states[:i], i + 1, graph=False)
        assert _same(without[i - 1], want[i - 1]) and not _same(without[i], want[i]), (case, B, f"switch {i}")
