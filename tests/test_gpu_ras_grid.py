"""Repetition-aware sampling in the persistent decode kernel at every batch width and at every CTA count that changes
how the lm_head tile list falls on the grid, with every other per-slot setting on; and on the chain at V = 4 142.

Every case turns on together, per slot: repetition-aware sampling (short and long windows, (64, 1/64), and entries
that never trigger), the repetition penalty (both sides of 1, prompt included or not), EOS floors and decays,
temperature / top-k / top-p / min-p (some slots at top_k 1 or 2, so that they loop), log-probabilities, and a
vocabulary range (off, "speech", "around-eos" or "narrow"); some slot has each setting neutral.  The model is the
logit-programmable one-layer model of ``sampler_ref.py`` (residual stream exactly ``embed[tok]``), so every output
must be bit-identical at every CTA count.  Persistent cases cover the five table-on instantiations of
``decode_tc_kernel``: batch 1 (FOLD, hi + lo, both plans through the counts), 3 and 8 (hi + lo), 16 (N = 16, bf16),
20 (N = 32), 40 and 64 (N = 64; 64 makes every column of the tile live), each at V = 217 472 and 4 142.  At V = 4 142
a logits row is 16 568 bytes, so odd rows are not 16-byte aligned and take the scalar branch of
``ras_full_row_draw``; its chunks are 20 ids, threads 208..255 hold none, and thread 207 holds the 2-id chunk
[4140, 4142) where the "partial" pattern keeps its winners.  Chain cases: batch 2 (GEMV lm_head + ``tile_max_kernel``),
6 (with a ``prefill_slots`` refill of slot 3 after 4 steps) and 17 (wgmma epilogue maxima).

At the device's SM count (the chain: once), a run of single steps is checked against float64:
  * stored logits bit-identical to transformers' RepetitionPenaltyLogitsProcessor -> ExponentialDecayLengthPenalty
    on the logits of the same tokens teacher-forced with the penalty, length and repetition-aware tables off, over
    each slot's actual history (redrawn tokens included); suppressed ids -inf;
  * processed tile maxima (persistent kernel) bit-identical; kept windows against the float64 chain (ids exact,
    probabilities within BARS["prob"]);
  * every token through ``ras_ref.RasChecker`` with per-slot controls and floors: a draw that does not trigger on the
    kept window's inverse CDF of u1, the trigger decided on the window of the device's own tokens, a redraw on the
    float64 inverse CDF of u2 over the whole processed row times the slot's 1 / T; ``sampled`` and ``model`` within
    the bars of test_gpu_logprobs.py (a redraw's ``sampled`` over the full row within 2e-4);
  * ``ras_redraws()`` equal to the redraws the reference predicts; no EOS while a slot's floor masks it, and a slot
    done exactly when it drew EOS, by a plain draw or a redraw (the measured runs drew no EOS by a redraw).
At every other count the run is bit-identical to the device-count run (logits, tile maxima, windows, tokens,
log-probabilities, state, redraw counters and launch counts).  At every count, one sampled multi-step launch (the
chain: its graph replay) gives the tokens, log-probabilities, state and redraw counters of the single steps.
Coverage is asserted per case, so that no case passes without redraws: the N = 32 / 64 cases redraw in a column
>= 16 / >= 40, the V = 4 142 cases named in COVER redraw on an odd row, into the 2-id last chunk, outside a top-p /
min-p cut, at T != 1, and redraw a token new to a slot's penalty history whose next row is checked penalised.

Measured on one H100 80GB HBM3 (132 SMs, 700 W power limit): 2 679 checked rows, 686 redraws (per case, in the order
of PERSISTENT then CHAIN: 4, 6, 8, 12, 14, 16, 39, 33, 39, 55, 61, 75, 109, 153; 12, 12, 38), no draw skipped or
ambiguous, no window within MARGIN of a cut.  Worst: kept probabilities 9.2e-8 (bar 4e-7), ``model``
2.5e-6 (bar 5e-5), ``sampled`` 3.9e-7 (bar 2e-5), a redrawn token's ``sampled`` 3.5e-6 (bar 2e-4).  Every other count
was bit-identical to the device's, and every multi-step launch to its single steps.  The module takes about 80 s.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import check_ras
from tests.helpers import (TC_DEFAULT_MAX_BATCH, decode_branch, head_grid_counts, head_list, make_lm, set_decode_impl)
from tests.processors_ref import bits_equal, hf_chain, ranked
from tests.ras_ref import RasChecker, chunk_of, window_cut
from tests.sampler_ref import BARS, INTER, MARGIN, SEED, H, _range, prob_err, processed_scores, programmable, tile_maxima

MAX_CTX, MAX_NEW = 256, 64
STEPS = 8             # decode steps after the prefill

# Per slot: pattern (9), controls (8), repetition-aware entry (7), penalty (5) and length entry (6), so that the
# settings meet in every combination over a wide batch.  "partial" sits at slots 0, 4, 9, 13, ...: even and odd rows.
PATTERNS = ["partial", "onetile", "gauss", "stairs", "partial", "ties", "plateau", "flat", "eos"]
CONTROLS = [
    (1.0, 1, 1.0, 0.0),     # top_k 1: loops until a redraw moves it
    (0.7, 64, 0.3, 0.0),    # top-p keeping about one id
    (1.3, 2, 1.0, 0.0),
    (1.0, 50, 1.0, 0.0),    # the reference defaults
    (1.5, 64, 1.0, 0.5),    # min-p
    (0.8, 3, 0.9, 0.05),
    (2.0, 1, 1.0, 0.0),
    (1.0, 8, 0.6, 0.2),
]
RAS = [(4, 0.5), (64, 1 / 64), (10, 0.1), None, (3, 1.0), (64, 1.0), (16, 0.25)]   # (64, 1.0) never triggers here
PENALTIES = [(1.0, True), (0.8, False), (1.3, True), (0.9, True), (1.2, False)]
LENGTHS = [(3, 4, 1.3), (0, 0, 1.0), (5, 4, 1.1), (1, 0, 1.0), (2, 3, 1.5), (0, 0, 1.0)]   # (floor, start, factor)

# (id, vocabulary, range kind, batch)
PERSISTENT = [
    ("v217472-b1", 217472, None, 1),
    ("v4142-b1-speech", 4142, "speech", 1),
    ("v217472-b3-speech", 217472, "speech", 3),
    ("v4142-b3", 4142, None, 3),
    ("v217472-b8-around-eos", 217472, "around-eos", 8),
    ("v4142-b8", 4142, None, 8),
    ("v217472-b16-narrow", 217472, "narrow", 16),
    ("v4142-b16", 4142, None, 16),
    ("v217472-b20-n32", 217472, None, 20),
    ("v4142-b20-n32-speech", 4142, "speech", 20),
    ("v217472-b40-n64-speech", 217472, "speech", 40),
    ("v4142-b40-n64", 4142, None, 40),
    ("v217472-b64-n64", 217472, None, 64),
    ("v4142-b64-n64-narrow", 4142, "narrow", 64),
]
# (id, batch, refill: (after decode step, slot, pattern, stream key) or None)
CHAIN = [
    ("chain-b2-gemv", 2, None),
    ("chain-b6-refill", 6, (4, 3, "onetile", 9)),
    ("chain-b17-tile", 17, None),
]
# coverage each named case must show (see the module docstring)
ALL = ("odd_row", "last_chunk", "outside_cut", "hot_t", "penalised_next")
COVER = {name: ALL for name in ("v4142-b3", "v4142-b8", "v4142-b16", "v4142-b20-n32-speech", "v4142-b40-n64",
                                "chain-b2-gemv", "chain-b6-refill", "chain-b17-tile")}


def vocab_range(m, kind):
    """``sampler_ref._range``, and "narrow": the 3 tiles ending 10 tiles below EOS's (EOS inserted last)."""
    if kind == "narrow":
        t = m.eos // 128
        return (t - 13) * 128, (t - 10) * 128
    return _range(m, kind) if kind else None


def prompt_for(m, pat, b):
    r = ranked(m, pat)
    return [int(r[10]), int(r[1]), m.eos, m.token_for(pat, b)]


def settings(m, B):
    prompts = [prompt_for(m, PATTERNS[b % len(PATTERNS)], b) for b in range(B)]
    ctl = [CONTROLS[b % len(CONTROLS)] for b in range(B)]
    ras = [RAS[b % len(RAS)] for b in range(B)]
    pens = [PENALTIES[b % len(PENALTIES)] for b in range(B)]
    lens = [LENGTHS[b % len(LENGTHS)] for b in range(B)]
    return prompts, ctl, ras, pens, lens


def _state(lm, B):
    return np.stack([t[:B].cpu().numpy() for t in (lm.n_generated, lm.done, lm.seq_lens, lm.cur_token)]
                    + [lm.ras_redraws()[:B].numpy()])


def _run(lm, sp, prompts, B, nt, buf, refill=None, sp_after=None):
    """prefill + STEPS single decode steps (a ``refill`` = (step, slot, prompt, key) runs ``prefill_slots`` after that
    many steps, and ``sp_after`` serves from there on).  Per launch: slots of its rows, done flags and n_generated
    before it, logits, captured window, tile maxima, state after it, launch count.  Returns (records, tokens and
    log-probabilities before the refill, the same at the end)."""
    lm.out_tokens.zero_()
    lm.debug_buffer("tmax", (B, nt)).zero_()
    buf.fill_(float("nan"))
    ops = ["prefill"] + ["decode"] * STEPS
    if refill is not None:
        ops.insert(1 + refill[0], "refill")
    recs, before = [], None
    for op in ops:
        st = _state(lm, B) if recs else np.zeros((5, B), dtype=np.int32)
        n0 = lm.L.nt_launch_count()
        if op == "prefill":
            lg, rows = lm.prefill(prompts, sp, return_logits=True), list(range(B))
        elif op == "refill":
            torch.cuda.synchronize()
            before = (lm.out_tokens[:B].cpu().numpy().copy(), buf[:B].cpu().numpy().copy())
            sp = sp_after
            lg = lm.prefill_slots([refill[1]], [refill[2]], sp, stream_ids=[refill[3]], return_logits=True)
            rows = [refill[1]]
            st[0, refill[1]] = st[1, refill[1]] = 0
        else:
            lg, rows = lm.decode(1, sp, return_logits=True)[0], list(range(B))
        torch.cuda.synchronize()
        R = len(rows)
        recs.append(dict(op=op, rows=rows, ngen=st[0].copy(), done=st[1].copy(), logits=lg.cpu().numpy(),
                         launches=lm.L.nt_launch_count() - n0, cap=[t[:R].cpu().numpy().copy() for t in lm._capture],
                         tmax=lm.debug_buffer("tmax", (R, nt)).cpu().numpy().copy(), state=_state(lm, B)))
    end = (lm.out_tokens[:B].cpu().numpy().copy(), buf[:B].cpu().numpy().copy())
    return recs, before or end, end


def _multi(lm, sp, prompts, B, steps, buf):
    """One launch of ``steps`` decode steps after the prefill: tokens, log-probabilities, state, launches."""
    lm.out_tokens.zero_()
    buf.fill_(float("nan"))
    lm.prefill(prompts, sp)
    n0 = lm.L.nt_launch_count()
    lm.decode(steps, sp)
    torch.cuda.synchronize()
    return (lm.out_tokens[:B, : steps + 1].cpu().numpy().copy(), buf[:B, : steps + 1].cpu().numpy().copy(),
            _state(lm, B), lm.L.nt_launch_count() - n0)


def _identical(a, b):
    """Two results of ``_run``: bit for bit."""
    for x, y in zip(a[1] + a[2], b[1] + b[2]):
        assert bits_equal(x, y) if x.dtype == np.float32 else np.array_equal(x, y), "tokens / log-probabilities"
    for j, (x, y) in enumerate(zip(a[0], b[0])):
        assert x["launches"] == y["launches"], (j, x["launches"], y["launches"])
        assert np.array_equal(x["state"], y["state"]), (j, x["state"], y["state"])
        assert bits_equal(x["logits"], y["logits"]), (j, "logits")
        assert bits_equal(x["tmax"], y["tmax"]), (j, "tile maxima")
        assert bits_equal(x["cap"][0], y["cap"][0]) and all(np.array_equal(p, q) for p, q in zip(x["cap"][1:], y["cap"][1:])), j


def _check_multi(run, multi, persistent):
    """The multi-step launch against the single steps it replaces (up to a refill)."""
    toks, lp, state, launches = multi
    k = toks.shape[1] - 1
    recs, (toks_a, lp_a), _ = run
    assert np.array_equal(toks, toks_a[:, : k + 1]), (toks, toks_a[:, : k + 1])
    assert bits_equal(lp, lp_a[:, : k + 1]), "log-probabilities"
    assert np.array_equal(state, recs[k]["state"]), (state, recs[k]["state"])
    if persistent:
        assert launches == recs[1]["launches"], (launches, recs[1]["launches"])   # one kernel for all the steps


def _check_references(m, run, off, prompts, ctl, ras, pens, lens, rng, refill, persistent, ck, worst):
    """The device-count run against ``off`` (the same tokens teacher-forced, penalty, length and repetition-aware
    tables off): the points of the module docstring.  Returns the coverage counts of the run's redraws."""
    recs, (toks_a, lp_a), (toks_b, lp_b) = run
    eos, B = m.eos, len(prompts)
    keep = None
    if rng is not None:
        keep = np.zeros(m.V, dtype=bool)
        keep[rng[0]: rng[1]] = True
        keep[eos] = True
    cover = dict(rows=0, redraws=0, max_col=-1, odd_row=0, last_chunk=0, outside_cut=0, hot_t=0, penalised_next=0,
                 eos_redraw=0, windows_skipped=0)
    checked, redraws = set(), []
    refilled = False
    for rec, orec in zip(recs, off[0]):
        refilled |= rec["op"] == "refill"
        for i, s in enumerate(rec["rows"]):
            if rec["done"][s]:
                continue
            fresh = refill is not None and s == refill[1] and refilled
            phase = "b" if fresh or refill is None or s != refill[1] else "a"
            toks, lp = (toks_b, lp_b) if phase == "b" else (toks_a, lp_a)
            prompt = refill[2] if fresh else prompts[s]
            key = refill[3] if fresh else s
            n = int(rec["ngen"][s])
            pen, inc = pens[s]
            floor, start, factor = lens[s]
            T, k, tp, mp = ctl[s]
            cover["rows"] += 1
            want = hf_chain(orec["logits"][i], prompt, toks[s, :n].tolist(), n, pen, (start, factor), eos, inc)
            got_lg = rec["logits"][i]
            assert bits_equal(got_lg, want), (s, n, np.nonzero(got_lg != want)[0][:5])
            if keep is not None:
                assert np.isneginf(got_lg[~keep]).all(), (s, n)
            if persistent:
                proc = processed_scores(want, n, eos, floor, T)
                assert bits_equal(rec["tmax"][i], tile_maxima(proc if rec["op"] == "decode" else want)), (s, n)
            tv, ti, tt = (c[i] for c in rec["cap"])
            ids, q, margin = window_cut(want, n, eos, floor, T, k, tp, mp)
            if margin >= MARGIN:
                assert ti[: len(ids)].tolist() == ids.tolist() and (ti[len(ids):] == -1).all(), (s, n, ti[: len(ids)], ids)
                err = prob_err(tv[: len(ids)], q)
                worst["prob"] = max(worst["prob"], err)
                assert err < BARS["prob"], (s, n, err)
            else:
                cover["windows_skipped"] += 1
            got = int(toks[s, n])
            assert int(tt) == got, (s, n, int(tt), got)
            if n < floor:
                assert got != eos, (s, n)
            verdict = ck.check(want, s, n, key, toks[s], got, sampled_lp=lp[s, n, 0], model_lp=lp[s, n, 1])
            after = rec["state"][:, s]
            assert after[0] == n + 1 and after[3] == got and bool(after[1]) == (got == eos), (s, n, got, after)
            checked.add((phase, s, n))
            if verdict:
                hist = (list(prompt) if inc else []) + toks[s, :n].tolist()
                redraws.append((phase, s, n, got, T, tp < 1 or mp > 0, got not in ids, pen != 1.0 and got not in hist))
    for phase, s, n, got, T, cut, outside, new in redraws:
        cover["redraws"] += 1
        cover["max_col"] = max(cover["max_col"], s)
        cover["odd_row"] += m.V % 4 != 0 and s % 2 == 1
        cover["last_chunk"] += chunk_of(m.V, got)[1][1] - chunk_of(m.V, got)[1][0] == 2 and s % 2 == 0
        cover["outside_cut"] += cut and outside
        cover["hot_t"] += T != 1.0
        cover["penalised_next"] += new and (phase, s, n + 1) in checked
        cover["eos_redraw"] += got == eos
    # the redraw counters: since each slot's last prefill
    pred = np.zeros(B, dtype=np.int64)
    for phase, s, *_ in redraws:
        pred[s] += phase == "b"
    got = recs[-1]["state"][4]
    assert (got >= pred).all() and (ck.skipped > 0 or np.array_equal(got, pred)), (got, pred)
    return cover


def _entries(rows):
    return [None if r is None else check_ras(*r) for r in rows]


def _case(cuda, monkeypatch, name, V, kind, B, impl, refill=None):
    m = programmable(V)
    cfg, w = m.oracle()
    shape = (H, INTER, 2, 1, V)
    dev = torch.cuda.get_device_properties(0).multi_processor_count
    rng = vocab_range(m, kind)
    persistent = impl != "perop"
    counts = head_grid_counts(shape, head_list(V, m.eos, rng), B, MAX_CTX, dev, impl) if persistent else [dev]
    lm = make_lm(cfg, w, max_batch=B, max_ctx=MAX_CTX, max_new=MAX_NEW)
    set_decode_impl(monkeypatch, impl)
    prompts, ctl, ras, pens, lens = settings(m, B)
    if refill is not None:
        refill = (refill[0], refill[1], prompt_for(m, refill[2], 100), refill[3])
    if rng is not None:
        lm.set_vocab_range(*rng)
    lm.set_slot_sampling(ctl)
    lm.debug_capture_sampler()
    buf = lm.set_logprobs(True)
    sp = lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=MAX_NEW, top_k=50, temperature=1.0, seed=SEED)
    nt = m.nt
    first, cover, branches = None, None, set()
    worst = {"prob": 0.0}
    ck = RasChecker(sp, _entries(ras), None, 0, controls=ctl, floors=[ln[0] for ln in lens])
    for G in [dev] + [G for G in counts if G != dev]:
        if persistent:
            br = decode_branch(shape, B, G, MAX_CTX, impl)
            assert br["kind"] == "tc" and br["nt"] == (16 if B <= 16 else (32 if B <= 32 else 64)), (G, br)
            branches.add(br["name"])
        lm.debug_set_sms(0 if G == dev else G)
        lm.set_repetition_penalty(pens)       # before the prefill, whose prompt tokens the history records
        lm.set_length_control(lens)
        lm.set_repetition_aware_sampling(ras)
        run = _run(lm, sp, prompts, B, nt, buf, refill, sp)
        k = STEPS if refill is None else refill[0]
        _check_multi(run, _multi(lm, sp, prompts, B, k, buf), persistent)
        if first is None:
            lm.set_repetition_penalty(None)
            lm.set_length_control(None)
            lm.set_repetition_aware_sampling(None)
            forced, keep = [], []   # keep: each forced table's device buffer, alive until the run is over
            for toks in (run[1][0], run[2][0]):
                forced.append(lm.sampling(m.eos, min_new_tokens=0, max_new_tokens=MAX_NEW, top_k=50, temperature=1.0,
                                          seed=SEED, forced=torch.from_numpy(toks.astype(np.int32))))
                keep.append(lm.forced)
            off = _run(lm, forced[0], prompts, B, nt, buf, refill, forced[1])
            del keep
            cover = _check_references(m, run, off, prompts, ctl, ras, pens, lens, rng, refill, persistent, ck, worst)
            first = run
        else:
            _identical(first, run)
    lm.debug_set_sms(0)
    ck.report(name)
    print(f"RAS-GRID {name}: {sorted(branches) or ['chain']} at G = {counts if persistent else '-'}; coverage {cover}; "
          f"worst prob {worst['prob']:.2e}")
    assert cover["redraws"] > 0 and cover["windows_skipped"] <= max(1, 0.02 * cover["rows"]), cover
    nt_width = 16 if B <= 16 else (32 if B <= 32 else 64)
    if persistent and nt_width > 16:   # a redraw beyond the columns of the next narrower tile (N = 64: beyond 40 at 64)
        assert cover["max_col"] >= (16 if nt_width == 32 else (40 if B > 40 else 32)), cover
    for what in COVER.get(name, ()):
        assert cover[what] > 0, (what, cover)
    return cover


@pytest.mark.gpu
@pytest.mark.parametrize("case", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_persistent_at_every_cta_count(cuda, case, monkeypatch):
    name, V, kind, B = case
    _case(cuda, monkeypatch, name, V, kind, B, "tc" if B > TC_DEFAULT_MAX_BATCH else None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHAIN, ids=[c[0] for c in CHAIN])
def test_chain(cuda, case, monkeypatch):
    name, B, refill = case
    _case(cuda, monkeypatch, name, 4142, None, B, "perop", refill)
