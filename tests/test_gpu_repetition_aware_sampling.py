"""GPU: repetition-aware sampling (VALL-E 2's RAS, CosyVoice 2's ``ras_sampling``) on every sampler path, against the
float64 reference of ``tests/ras_ref.py``.

The model is the logit-programmable one-layer model of ``sampler_ref.py``: a token's logits are the pattern that owns
it, and a pattern's top id owns that pattern again, so at a small top_k every slot loops on one id until a redraw
moves it.  Every token of multi-step single launches is checked: the draw of the top-k window with u1, the trigger on
the window the device holds (its own earlier tokens of the slot), and a triggered draw on the float64 inverse CDF of
the full row with u2.  Also covered: a table that never triggers is bit-identical to the table off, the vocabulary
range and the EOS mask hold for redraws, refills, takes and guided c slots, the sampled log-probability of a redrawn
token, the redraw counter, the graph key, a bad table through the ABI, and the Air shape at batch 1 and 64.
"""
from __future__ import annotations


import numpy as np
import pytest
import torch

from neutts_air_b200 import _lib, synthetic
from neutts_air_b200.lm import LMShape, SpeechLM, check_ras
from tests.helpers import make_lm, runs_persistent, set_decode_impl
from tests.processors_ref import bits_equal
from tests.ras_ref import RasChecker
from tests.sampler_ref import MIN_NEW, SEED, _range, programmable

pytestmark = pytest.mark.gpu

V = 217472
# (win_size, tau_r) per slot, or None: short and long windows, low and high thresholds
RAS = [(10, 0.1), (4, 0.5), (64, 0.05), None, (1, 1.0), (16, 0.25), (8, 0.5), (3, 1.0)]
LOOPS = ["onetile", "gauss", "stairs", "ties", "plateau", "flat", "partial", "gauss"]


def _entries(rows):
    return [None if r is None else check_ras(*r) for r in rows]


def _prompts(m, B, pats=LOOPS):
    return [[m.token_for("gauss", b), m.token_for(pats[b % len(pats)], b)] for b in range(B)]


def _launch(lm, ck, logits, slots, keys, n0, ngen, out, lps=None, top_k=None, allowed=None):
    """Check the tokens one launch wrote: logits [steps, R, V] (row i -> slot slots[i]); n0[s]: the slot's n_generated
    before the launch; ngen / out: the state after it."""
    steps = logits.shape[0]
    for j in range(steps):
        for i, s in enumerate(slots):
            n = int(n0[s]) + j
            if n >= int(ngen[s]):
                continue
            ck.check(logits[j, i], s, n, keys[i], out[s], int(out[s, n]),
                     None if lps is None else lps[s, n, 0], top_k=top_k, allowed=allowed)


def _state(lm, B):
    torch.cuda.synchronize()
    lp = lm.logprobs[:B].cpu().numpy() if lm.logprobs is not None else None
    return lm.n_generated[:B].cpu().numpy().copy(), lm.out_tokens[:B].cpu().numpy().copy(), lp


# ------------------------------------------------------------------------------------------------ sampled launches
CASES = [   # (id, NT_DECODE_IMPL, batch, CTAs (0: the device's), top_k, temperature, log-probabilities)
    ("persistent-b1", None, 1, 0, 1, 1.0, True),
    ("persistent-b3-g8", None, 3, 8, 1, 1.0, False),
    ("persistent-b8-g40", None, 8, 40, 4, 1.3, True),
    ("persistent-b16", None, 16, 0, 1, 0.8, False),
    ("persistent-b6-g17", None, 6, 17, 2, 1.0, True),
    ("chain-b2-gemv", "perop", 2, 0, 1, 1.0, True),
    ("chain-b8-tile", "perop", 8, 0, 3, 1.2, False),
    ("chain-b20-tile", "perop", 20, 0, 1, 1.0, True),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_multistep_launch_vs_float64(cuda, case, monkeypatch):
    """One prefill and one 40-step launch: every token on the float64 sampler with repetition-aware sampling, the
    redraw counter equal to the redraws the reference predicts, and redrawn tokens' sampled log-probabilities within
    2e-4 of float64."""
    name, impl, B, G, top_k, T, lp = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    if G:
        lm.debug_set_sms(G)
    rows = [RAS[b % len(RAS)] for b in range(B)]
    lm.set_repetition_aware_sampling(rows)
    if lp:
        lm.set_logprobs(True)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED)
    ck = RasChecker(sp, _entries(rows), [T] * B, MIN_NEW)
    prompts = _prompts(m, B)
    lg0 = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    ngen, out, lps = _state(lm, B)
    assert (lm.ras_redraws()[:B] == 0).all()
    _launch(lm, ck, lg0[None], list(range(B)), list(range(B)), np.zeros(B, int), ngen, out, lps)
    n0 = ngen.copy()
    lg = lm.decode(40, sp, return_logits=True).cpu().numpy()
    ngen, out, lps = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), list(range(B)), n0, ngen, out, lps)
    assert ck.redraws > 0
    want, got = np.bincount([s for s, _, _ in ck.redrawn], minlength=B), lm.ras_redraws()[:B].numpy()
    assert (got >= want).all() and (ck.skipped > 0 or np.array_equal(got, want)), (got, want)
    ck.report(f"{name} ({'persistent' if runs_persistent(impl, B) else 'chain'})")


@pytest.mark.parametrize("impl,B", [(None, 4), ("perop", 5)], ids=["persistent-b4", "chain-b5"])
def test_table_that_never_triggers_is_bit_identical(cuda, impl, B, monkeypatch):
    """Entries that cannot trigger within the run (64 repeats in 64 tokens, over 30 steps) give tokens, logits, tile
    maxima and log-probabilities bit-identical to the table off, and no redraw."""
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    lm.set_logprobs(True)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=3, temperature=1.1, seed=SEED)
    prompts = _prompts(m, B)
    runs = {}
    for tag, rows in (("off", None), ("on", [(64, 1.0)] * B)):
        lm.set_repetition_aware_sampling(rows)
        l0 = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
        ls = lm.decode(30, sp, return_logits=True).cpu().numpy()
        tm = lm.debug_buffer("tmax", (B, m.nt)).cpu().numpy().copy()
        ngen, out, lps = _state(lm, B)
        runs[tag] = (l0, ls, tm, ngen, out, lps)
    for a, b in zip(runs["off"], runs["on"]):
        assert bits_equal(a, b) if a.dtype == np.float32 else np.array_equal(a, b)
    assert (lm.ras_redraws()[:B] == 0).all()


@pytest.mark.parametrize("impl", [None, "perop"], ids=["persistent", "chain"])
def test_redraws_keep_range_and_eos_mask(cuda, impl, monkeypatch):
    """Under the vocabulary range every redraw stays in the range (EOS is masked for the whole run, so never EOS)."""
    B = 4
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    lo, hi = _range(m, "speech")
    lm.set_vocab_range(lo, hi)
    rows = [(10, 0.1), (4, 0.5), (2, 1.0), (8, 0.25)]
    lm.set_repetition_aware_sampling(rows)
    sp = lm.sampling(m.eos, min_new_tokens=64, max_new_tokens=64, top_k=1, temperature=1.0, seed=SEED)
    ck = RasChecker(sp, _entries(rows), [1.0] * B, 64)
    lm.prefill(_prompts(m, B, ["onetile", "gauss", "stairs", "ties"]), sp)
    ngen, out, _ = _state(lm, B)
    n0 = ngen.copy()
    lg = lm.decode(30, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), list(range(B)), n0, ngen, out, allowed=lambda t: lo <= t < hi)
    assert ck.redraws > 0 and not (out[:, :30] == m.eos).any()
    lm.set_vocab_range(None)
    ck.report(f"range-{impl or 'persistent'}")


@pytest.mark.parametrize("impl", [None, "perop"], ids=["persistent", "chain"])
def test_refills_and_takes_have_their_own_windows(cuda, impl, monkeypatch):
    """``prefill_slots`` refills a looping slot: the newcomer's window starts empty (its stream key is its own) and the
    survivors carry on; ``prefill_fork`` takes of one prompt each keep their own window and stream."""
    B = 4
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    rows = [(6, 0.5), (10, 0.2), (4, 0.75), (12, 0.25)]
    lm.set_repetition_aware_sampling(rows)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=1, temperature=1.0, seed=SEED)
    ck = RasChecker(sp, _entries(rows), [1.0] * B, MIN_NEW)
    keys = list(range(B))
    lm.prefill(_prompts(m, B), sp)
    ngen, out, _ = _state(lm, B)
    n0 = ngen.copy()
    lg = lm.decode(12, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), keys, n0, ngen, out)
    before = ck.redrawn[:]
    assert lm.ras_redraws()[1] > 0
    # refill slot 1 with the same loop: its counter restarts, and its first draws see only its own tokens
    keys[1] = 9
    lgr = lm.prefill_slots([1], [_prompts(m, B)[1]], sp, stream_ids=[9], return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    assert lm.ras_redraws()[1] == 0 and ngen[1] == 1
    _launch(lm, ck, lgr[None], [1], [9], np.zeros(B, int), ngen, out)
    n0 = ngen.copy()
    lg = lm.decode(12, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), keys, n0, ngen, out)
    assert lm.ras_redraws()[1] == sum(1 for s, _, _ in ck.redrawn[len(before):] if s == 1)
    # takes: 2 prompts x 2 takes, each take its own window and Philox stream
    rows = [(6, 0.5), (6, 0.5), (3, 1.0), (3, 1.0)]
    lm.set_repetition_aware_sampling(rows)
    ck = RasChecker(sp, _entries(rows), [1.0] * B, MIN_NEW)
    lg0 = lm.prefill_fork(_prompts(m, 2), 2, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg0[[0, 0, 1, 1]][None], list(range(B)), list(range(B)), np.zeros(B, int), ngen, out)
    n0 = ngen.copy()
    lg = lm.decode(16, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), list(range(B)), n0, ngen, out)
    assert ck.redraws > 0
    ck.report(f"refill-takes-{impl or 'persistent'}")


def test_guided_c_slots_redraw(cuda):
    """Guided pairs (the chain): the c slots' draws follow their own entries on the combined rows; the u slots take
    the c slots' tokens."""
    B = 4
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    rows = [(8, 0.25), (5, 0.4), (8, 0.25), (5, 0.4)]
    lm.set_repetition_aware_sampling(rows)
    lm.set_guidance([(2, 1.5), (3, 3.0), (-1, 1.0), (-1, 1.0)])
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=1, temperature=1.0, seed=SEED)
    ck = RasChecker(sp, _entries(rows), [1.0] * B, MIN_NEW)
    p = _prompts(m, 2, ["onetile", "gauss"])
    lm.prefill(p + [[m.token_for("stairs", 0)], [m.token_for("ties", 1)]], sp)
    ngen, out, _ = _state(lm, B)
    n0 = ngen.copy()
    lg = lm.decode(24, sp, return_logits=True).cpu().numpy()
    ngen, out, _ = _state(lm, B)
    _launch(lm, ck, lg[:, :2], [0, 1], [0, 1], n0, ngen, out)
    assert ck.redraws > 0 and np.array_equal(out[2, : ngen[0]], out[0, : ngen[0]])
    lm.set_guidance(None)
    ck.report("guided")


def test_toggle_rebuilds_graph_and_bad_table_keeps_previous(cuda, monkeypatch):
    """The chain's decode graph (multi-step launch, no logits) follows the table: off, on, off; each graph replay
    equals single steps without a graph under the same table.  A bad table through the ABI is refused with
    NT_ERR_INVALID and the previous one stays in force."""
    B, n = 3, 20
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, "perop")
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=1, temperature=1.0, seed=SEED)
    prompts = _prompts(m, B)
    seen = {}
    for tag, rows in (("off", None), ("on", [(6, 0.5)] * B), ("off2", None)):
        lm.set_repetition_aware_sampling(rows)
        toks = []
        for graph in (True, False):
            lm.prefill(prompts, sp)
            lm.decode(n, sp, return_logits=not graph)
            toks.append(_state(lm, B)[1][:, : n + 1])
        assert np.array_equal(toks[0], toks[1]), tag
        seen[tag] = (toks[0], lm.ras_redraws()[:B].clone())
    assert np.array_equal(seen["off"][0], seen["off2"][0]) and not np.array_equal(seen["off"][0], seen["on"][0])
    assert (seen["on"][1] > 0).all() and (seen["off"][1] == 0).all()
    lm.set_repetition_aware_sampling([(6, 0.5)] * B)
    for bad in ((65, 1), (6, 0), (6, 7), (-1, 1)):
        tab = (_lib.SlotRAS * B)(*[_lib.SlotRAS(*r) for r in [(6, 3), bad, (6, 3)]])
        assert lm.L.nt_lm_set_repetition_aware_sampling(lm.handle, tab, None) == -1, bad
        assert b"slot 1" in lm.L.nt_last_error()
    lm.prefill(prompts, sp)
    lm.decode(n, sp)
    assert np.array_equal(_state(lm, B)[1][:, : n + 1], seen["on"][0])   # still the (6, 0.5) table
    with pytest.raises(ValueError):
        lm.set_repetition_aware_sampling([(6, 0.5), (65, 0.5), (6, 0.5)])
    assert lm._ras_host == [(6, 3)] * B


# ------------------------------------------------------------------------------------------------ full Air size
@pytest.mark.parametrize("B", [1, 64])
def test_full_size_one_launch(cuda, B, monkeypatch):
    """Air shape, synthetic weights: a 100-token prompt and one 12-step launch with every slot's table on, at batch 1
    (persistent kernel) and batch 64 (chain); every token on the float64 sampler with repetition-aware sampling."""
    set_decode_impl(monkeypatch, None)
    shape = LMShape()
    eos = 151670
    sd = synthetic.lm_state_dict(shape, 0)
    lm = SpeechLM(shape, sd, device="cuda:0", max_batch=B, max_ctx=512, max_new=64, max_prefill_tokens=B * 128)
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, shape.vocab_size, (100,), generator=g).tolist() for _ in range(B)]
    rows = [(64, 1 / 64)] * B    # any repeat within the last 64 tokens redraws
    lm.set_repetition_aware_sampling(rows)
    lm.set_logprobs(True)
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=64, top_k=2, temperature=1.0, seed=SEED)
    ck = RasChecker(sp, _entries(rows), [1.0] * B, 0)
    lg0 = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    ngen, out, lps = _state(lm, B)
    _launch(lm, ck, lg0[None], list(range(B)), list(range(B)), np.zeros(B, int), ngen, out, lps)
    n0 = ngen.copy()
    lg = lm.decode(12, sp, return_logits=True).cpu().numpy()
    ngen, out, lps = _state(lm, B)
    _launch(lm, ck, lg, list(range(B)), list(range(B)), n0, ngen, out, lps)
    want, got = np.bincount([s for s, _, _ in ck.redrawn], minlength=B), lm.ras_redraws()[:B].numpy()
    assert (got >= want).all() and (ck.skipped > 0 or np.array_equal(got, want)), (got, want)
    ck.report(f"Air B={B}")
