"""The persistent decode kernel's lm_head epilogue (``epi_head``) and sampler (``sample_phase``) with every per-slot
setting on at once, at every CTA count that changes how the lm_head tile list falls on the grid, and at all four batch
widths of the kernel (hi + lo activations, N = 16, 32 and 64).

The model is the logit-programmable one-layer model of ``sampler_ref.py``: its wo = wd = 0, so the residual stream is
exactly ``embed[tok]`` on every CTA count and work plan, and every stored logit, tile maximum, kept window, token and
log-probability must come out bit-identical at every count.  Each case turns on together the repetition penalty
(penalties on both sides of 1, prompt included or not), per-slot floors and EOS decays, per-slot temperature / top-k /
top-p / min-p, log-probabilities and a vocabulary range, spread over the slots so that some slot has each setting
neutral.  At the device's SM count, a sampled run is checked against the references:

  * stored logits bit-identical to transformers' RepetitionPenaltyLogitsProcessor -> ExponentialDecayLengthPenalty on
    the logits of a teacher-forced run of the same tokens with the penalty and length tables off; suppressed ids -inf;
  * processed tile maxima (penalty, decay, floor mask, 1 / T) bit-identical to those scores' maxima;
  * kept windows against the float64 chain (ids exact, probabilities within BARS["prob"]; a cut closer than MARGIN
    to its threshold is skipped), tokens on the float64 inverse CDF of the same Philox draw;
  * ``model`` and ``sampled`` log-probabilities within the bars of test_gpu_logprobs.py.

At every other count the same run is bit-identical to the device-count run (logits, tile maxima, windows, tokens,
log-probabilities, state and launch counts), and one 6-step launch of greedy decoding gives the tokens of 6 single
steps: the sampler sets history bits that other CTAs' ``epi_head`` reads at the next step, and which CTA owns a
penalised tile changes with the count.  ``helpers.head_grid_counts`` picks the counts; the CPU test below checks they
cover what the lm_head partition can look like.

Measured on one H100 80GB HBM3 (132 SMs, 700 W power limit), the counts per case:
  v217472 b1 [8, 20, 114, 132], b16 [16, 20, 114, 132], b40 [40, 114, 132]; speech b3 [8, 20, 114, 132], b20 [20, 114,
  132]; below-eos b8 [8, 20, 114, 132], b40 [40, 114, 132]; around-eos b1 and b16 [8 | 16, 20, 39, 40, 41, 114, 132];
  narrow b3 [8, 20, 114, 132], b20 [20, 114, 132]; v4142 b8 [8, 20, 32, 33, 34, 114, 132], b40 [40, 114, 132].
  Worst over the 916 checked rows: kept probabilities 2.1e-7 (bar 4e-7), ``model`` 1.1e-6 (bar 5e-5), ``sampled``
  3.7e-7 (bar 2e-5); no window within MARGIN of a cut, one ambiguous draw of 916.  Every other count was bit-identical
  to the device's.  The module takes 78 to 94 s.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from tests.helpers import (TC_DEFAULT_MAX_BATCH, decode_branch, head_grid_counts, head_grid_features, head_list,
                           head_partition, make_lm, regime_representatives, set_decode_impl)
from tests.processors_ref import LOGPROB_BARS, bits_equal, hf_chain, model_ref, ranked, sampled_ref
from tests.sampler_ref import (BARS, INTER, MARGIN, PATTERNS_ALL, SEED, H, _range, controls_for, draw_u, prob_err,
                               processed_scores, programmable, ref_token, ref_window_cut, tile_maxima)

MAX_CTX, MAX_NEW, MIN_NEW = 256, 64, 3
STEPS = 4             # decode steps after the prefill in the checked runs
GREEDY_STEPS = 6      # the multi-step launch at every count
H100_SMS = 132        # the CPU test's device

# Per slot s: slot s % 4 == 1 samples with the reference defaults, s % 4 == 2 has no floor and no decay, and the
# penalty is 1 at s % 8 == 3.
PENALTIES = [(1.3, True), (0.7, False), (2.0, True), (1.0, True), (1.15, False), (0.9, True), (3.0, False), (1.05, True)]
LENGTHS = [(2, 1, 0.8), (1, 0, 2.5), (0, 0, 1.0), (3, 2, 1.3), (0, 1, 1.05), (2, 3, 1.7), (0, 0, 1.0), (3, 4, 3.0)]
NEUTRAL_CONTROLS = (1.0, 50, 1.0, 0.0)

# (id, vocabulary, vocabulary range kind, batch)
CASES = [
    ("v217472-b1", 217472, None, 1),
    ("v217472-b16", 217472, None, 16),
    ("v217472-b40-n64", 217472, None, 40),
    ("speech-b3", 217472, "speech", 3),
    ("speech-b20-n32", 217472, "speech", 20),
    ("below-eos-b8", 217472, "below-eos", 8),
    ("below-eos-b40-n64", 217472, "below-eos", 40),
    ("around-eos-b1", 217472, "around-eos", 1),
    ("around-eos-b16", 217472, "around-eos", 16),
    ("narrow-b3", 217472, "narrow", 3),
    ("narrow-b20-n32", 217472, "narrow", 20),
    ("v4142-b8", 4142, None, 8),
    ("v4142-b40-n64", 4142, None, 40),
]


def vocab_range(m, kind):
    """``sampler_ref._range``, and "narrow": the 3 tiles ending 10 tiles below EOS's (EOS inserted last)."""
    if kind == "narrow":
        t = m.eos // 128
        return (t - 13) * 128, (t - 10) * 128
    return _range(m, kind) if kind else None


def impl_for(B):
    return "tc" if B > TC_DEFAULT_MAX_BATCH else None


def plan_shape(V):
    return (H, INTER, 2, 1, V)


def settings(m, B):
    """Prompts (two strong ids of the slot's pattern, EOS, a token of the pattern) and the per-slot tables."""
    pats = (PATTERNS_ALL * 8)[:B]
    prompts = []
    for b, p in enumerate(pats):
        r = ranked(m, p)
        prompts.append([int(r[10]), int(r[1]), m.eos, m.token_for(p, b)])
    pens = [PENALTIES[b % len(PENALTIES)] for b in range(B)]
    lens = [LENGTHS[b % len(LENGTHS)] for b in range(B)]
    ctl = [NEUTRAL_CONTROLS if b % 4 == 1 else c for b, c in enumerate(controls_for(B))]
    return prompts, pens, lens, ctl


# ============================================================================================== CPU: the chosen counts
def test_head_partition_restatement():
    """``head_partition`` hands out every list position once, in order, and the tiles it names are the range's tiles
    in order with EOS's tile inserted first or last; the head lists of the module's cases."""
    heads = {}
    for _, V, kind, _ in CASES:
        m = programmable(V)
        rng = vocab_range(m, kind)
        head = head_list(V, m.eos, rng)
        heads[(V, kind)] = head
        head_n, head_lo, head_eos, head_eos_at = head
        t_hi = -(-(rng[1] if rng else V) // 128)
        want = list(range(head_lo, t_hi))
        if head_eos >= 0:
            want.insert(head_eos_at, head_eos)
        assert len(want) == head_n
        for G in (8, 9, 20, 33, 97, 114, 132, 256):
            part = head_partition(head_n, head_eos_at, G, head_lo, head_eos)
            assert len(part) == G and part[0][0] == 0 and part[-1][1] == head_n
            assert all(a[1] == b[0] for a, b in zip(part, part[1:]))
            assert [t for _, _, tiles in part for t in tiles] == want, (V, kind, G)
    eos_t = programmable(217472).eos // 128
    assert heads[(217472, None)] == (1699, 0, -1, -1) and heads[(4142, None)] == (33, 0, -1, -1)
    assert heads[(217472, "speech")] == (513, 1187, eos_t, 0)
    assert heads[(217472, "below-eos")][2:] == (eos_t, heads[(217472, "below-eos")][0] - 1)
    assert heads[(217472, "around-eos")] == (40, eos_t - 20, -1, -1)
    assert heads[(217472, "narrow")] == (4, eos_t - 13, eos_t, 3)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cta_counts_cover_the_head_partition(case):
    """The counts a case runs at (on a 132-SM H100): the smallest accepted count, the device's, every plan regime of
    the programmable shape, both plans at batch 1, G = head_n where it fits, and every head-partition feature any
    accepted count has (a CTA with no tile, counts of both parities above 1, the EOS tile alone and shared)."""
    name, V, kind, B = case
    m = programmable(V)
    shape, impl = plan_shape(V), impl_for(B)
    head = head_list(V, m.eos, vocab_range(m, kind))
    counts = head_grid_counts(shape, head, B, MAX_CTX, H100_SMS, impl)
    ok = [G for G in range(8, H100_SMS + 1) if decode_branch(shape, B, G, MAX_CTX, impl)["kind"] == "tc"]
    assert set(counts) <= set(ok) and ok[0] == max(8, B) and {ok[0], H100_SMS} <= set(counts)
    assert {G for G in regime_representatives(shape, H100_SMS).values() if G in ok} <= set(counts)
    if head[0] in ok:
        assert head[0] in counts
    possible = set().union(*(head_grid_features(head, G) for G in ok))
    covered = set().union(*(head_grid_features(head, G) for G in counts))
    assert covered == possible, (name, possible - covered)
    assert {"even", "odd"} <= possible or head[0] < 2 * ok[0]
    if head[2] >= 0:
        assert "eos-alone" in covered or head[0] > 2 * H100_SMS
    if B == 1:
        plans = {decode_branch(shape, B, G, MAX_CTX, impl)["plan"] for G in ok}
        assert {decode_branch(shape, B, G, MAX_CTX, impl)["plan"] for G in counts} == plans
    assert len(counts) <= 8, counts
    print(f"HEAD-GRID {name}: head {head} counts {counts} features {sorted(covered)}")


# ============================================================================================== GPU
def _run(lm, sp, prompts, B, nt, steps, buf=None):
    """prefill + ``steps`` single decode steps.  Per launch: done flags before it, logits, captured window, tile
    maxima, state after it and launch count; then the tokens and (``buf``) the log-probabilities."""
    lm.out_tokens.zero_()      # every run starts from the same buffers: a launch that does not write them leaves
    lm.debug_buffer("tmax", (B, nt)).zero_()   # equal contents in both runs of a comparison
    if buf is not None:
        buf.fill_(float("nan"))
    recs = []
    for j in range(steps + 1):
        done = np.zeros(B, dtype=np.int32) if j == 0 else lm.done[:B].cpu().numpy().copy()
        n0 = lm.L.nt_launch_count()
        lg = lm.prefill(prompts, sp, return_logits=True) if j == 0 else lm.decode(1, sp, return_logits=True)[0]
        torch.cuda.synchronize()
        recs.append(dict(done=done, logits=lg.cpu().numpy(), launches=lm.L.nt_launch_count() - n0,
                         cap=[t[:B].cpu().numpy().copy() for t in lm._capture],
                         tmax=lm.debug_buffer("tmax", (B, nt)).cpu().numpy().copy(),
                         state=torch.stack((lm.n_generated[:B], lm.done[:B], lm.seq_lens[:B],
                                            lm.cur_token[:B])).cpu().numpy()))
    toks = lm.out_tokens[:B, : steps + 1].cpu().numpy().copy()
    lp = buf[:B, : steps + 1].cpu().numpy().copy() if buf is not None else None
    return recs, toks, lp


def _greedy(lm, sp, prompts, B):
    """One launch of GREEDY_STEPS steps and GREEDY_STEPS single steps from the same prefill: tokens, state, launches."""
    out = []
    for multi in (True, False):
        lm.out_tokens.zero_()
        lm.prefill(prompts, sp)
        n0 = lm.L.nt_launch_count()
        for _ in range(1 if multi else GREEDY_STEPS):
            lm.decode(GREEDY_STEPS if multi else 1, sp)
        torch.cuda.synchronize()
        out.append((lm.out_tokens[:B, : GREEDY_STEPS + 1].cpu().numpy().copy(),
                    torch.stack((lm.n_generated[:B], lm.done[:B])).cpu().numpy(), lm.L.nt_launch_count() - n0))
    return out


def _identical(a, b):
    """Two records of ``_run``: bit for bit."""
    recs_a, toks_a, lp_a = a
    recs_b, toks_b, lp_b = b
    assert np.array_equal(toks_a, toks_b) and bits_equal(lp_a, lp_b), "tokens / log-probabilities"
    for j, (x, y) in enumerate(zip(recs_a, recs_b)):
        assert x["launches"] == y["launches"], (j, x["launches"], y["launches"])
        assert np.array_equal(x["state"], y["state"]) and np.array_equal(x["done"], y["done"]), j
        assert bits_equal(x["logits"], y["logits"]), (j, "logits")
        assert bits_equal(x["tmax"], y["tmax"]), (j, "tile maxima")
        assert bits_equal(x["cap"][0], y["cap"][0]) and all(np.array_equal(p, q) for p, q in zip(x["cap"][1:], y["cap"][1:])), j


def _check_references(m, run, off, prompts, pens, lens, ctl, rng, worst):
    """The device-count run ``run`` (settings on) against ``off`` (the same tokens teacher-forced, penalty and length
    tables off): points of the module docstring.  Returns (rows checked, windows skipped, draws, ambiguous draws)."""
    recs, toks, lp = run
    eos = m.eos
    keep = None
    if rng is not None:
        keep = np.zeros(m.V, dtype=bool)
        keep[rng[0]: rng[1]] = True
        keep[eos] = True
    rows = skipped = draws = ambiguous = 0
    for j, rec in enumerate(recs):
        tv, ti, tt = rec["cap"]
        for b in range(len(prompts)):
            if rec["done"][b]:
                continue
            rows += 1
            pen, inc = pens[b]
            floor, start, factor = lens[b]
            T, k, tp, mp = ctl[b]
            want = hf_chain(off[0][j]["logits"][b], prompts[b], toks[b, :j].tolist(), j, pen, (start, factor), eos, inc)
            got = rec["logits"][b]
            assert bits_equal(got, want), (j, b, np.nonzero(got != want)[0][:5])
            if keep is not None:
                assert np.isneginf(got[~keep]).all(), (j, b)
            proc = processed_scores(want, j, eos, floor, T)
            assert bits_equal(rec["tmax"][b], tile_maxima(proc if j > 0 else want)), (j, b)
            ids, q, margin = ref_window_cut(want, j, eos, floor, T, k, tp, mp)
            if margin < MARGIN:
                skipped += 1
                continue
            n = len(ids)
            assert ti[b, :n].tolist() == ids.tolist() and (ti[b, n:] == -1).all(), (j, b, ti[b, :n].tolist(), ids.tolist())
            err = prob_err(tv[b, :n], q)
            worst["prob"] = max(worst["prob"], err)
            assert err < BARS["prob"], (j, b, err)
            tok, ok = ref_token((ids, q), draw_u(SEED, j, b))
            draws += 1
            ambiguous += len(ok) > 1
            assert int(tt[b]) in ok and int(toks[b, j]) == int(tt[b]), (j, b, int(tt[b]), tok, ok)
            sampled, model = (float(v) for v in lp[b, j])
            ref = model_ref(want, int(tt[b]), eos, j < floor)
            assert math.isfinite(ref), (j, b)
            worst["model"] = max(worst["model"], abs(model - ref))
            assert abs(model - ref) < LOGPROB_BARS["model"], (j, b, model, ref)
            ref = sampled_ref(want, ti[b].tolist(), int(tt[b]), T)
            worst["sampled"] = max(worst["sampled"], abs(sampled - ref))
            assert abs(sampled - ref) < LOGPROB_BARS["sampled"], (j, b, sampled, ref)
            assert abs(math.exp(sampled) - float(tv[b, ids.tolist().index(int(tt[b]))])) < LOGPROB_BARS["prob"], (j, b)
    return rows, skipped, draws, ambiguous


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_head_and_sampler_at_every_cta_count(cuda, case, monkeypatch):
    name, V, kind, B = case
    m = programmable(V)
    cfg, w = m.oracle()
    shape, impl = plan_shape(V), impl_for(B)
    dev = torch.cuda.get_device_properties(0).multi_processor_count
    rng = vocab_range(m, kind)
    head = head_list(V, m.eos, rng)
    counts = head_grid_counts(shape, head, B, MAX_CTX, dev, impl)
    lm = make_lm(cfg, w, max_batch=B, max_ctx=MAX_CTX, max_new=MAX_NEW)
    set_decode_impl(monkeypatch, impl)
    prompts, pens, lens, ctl = settings(m, B)
    if rng is not None:
        lm.set_vocab_range(*rng)
    lm.set_slot_sampling(ctl)
    lm.debug_capture_sampler()
    buf = lm.set_logprobs(True)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=MAX_NEW, top_k=50, temperature=1.0, seed=SEED)
    greedy_sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=MAX_NEW, greedy=True, seed=SEED)
    nt = 16 if B <= 16 else (32 if B <= 32 else 64)
    first = greedy_first = None
    worst = {"prob": 0.0, "model": 0.0, "sampled": 0.0}
    branches = set()
    for G in [dev] + [G for G in counts if G != dev]:
        br = decode_branch(shape, B, G, MAX_CTX, impl)
        assert br["kind"] == "tc" and br["nt"] == nt and br["act"] == ("hilo" if B <= 8 else "bf16"), (G, br)
        branches.add(br["name"])
        lm.debug_set_sms(0 if G == dev else G)
        lm.set_repetition_penalty(pens)       # before the prefill, whose prompt tokens the history records
        lm.set_length_control(lens)
        run = _run(lm, sp, prompts, B, m.nt, STEPS, buf)
        greedy = _greedy(lm, greedy_sp, prompts, B)
        (multi_toks, multi_state, multi_launches), (single_toks, single_state, _) = greedy
        assert np.array_equal(multi_toks, single_toks) and np.array_equal(multi_state, single_state), (G, multi_toks, single_toks)
        assert multi_launches == run[0][1]["launches"], (G, multi_launches, run[0][1]["launches"])   # one kernel for 6 steps
        if first is None:
            # the same tokens teacher-forced with the penalty and length tables off: the logits the settings start from
            lm.set_repetition_penalty(None)
            lm.set_length_control(None)
            forced = torch.from_numpy(run[1].astype(np.int32))
            fsp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=MAX_NEW, top_k=50, temperature=1.0, seed=SEED,
                              forced=forced)
            off = _run(lm, fsp, prompts, B, m.nt, STEPS)
            rows, skipped, draws, ambiguous = _check_references(m, run, off, prompts, pens, lens, ctl, rng, worst)
            assert draws > 0 and ambiguous <= max(1, BARS["ambiguous"] * draws), (draws, ambiguous)
            assert any(not bits_equal(a["logits"], b["logits"]) for a, b in zip(run[0], off[0]))   # the settings act
            first, greedy_first = run, multi_toks
        else:
            _identical(first, run)
            assert np.array_equal(multi_toks, greedy_first), (G, multi_toks, greedy_first)
    lm.debug_set_sms(0)
    print(f"HEAD-GRID {name}: {sorted(branches)} head {head} at G = {counts}; rows {rows} windows skipped {skipped} "
          f"draws {draws} ambiguous {ambiguous}; worst prob {worst['prob']:.2e} model {worst['model']:.2e} "
          f"sampled {worst['sampled']:.2e}")
