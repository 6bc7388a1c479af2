"""Every speech-LM sampler path against a float64 top-k sampler on the same logits and Philox draws.

The logit-parity tests are teacher-forced: the sampler runs, but the forced token overrides whatever it selected, so a
wrong threshold, tie order or EOS mask changes the audio without moving one logit.  The tests here compare what each
sampler path kept and drew with a plain float64 reference that reads the operands the kernel read: its own logits
(returned by the call), its own ``n_generated`` and its own Philox counter.

Sampler paths (both run ``sample_tiles_seq`` and end in ``sample_finish`` in lm_device.cuh):
  * tile-max sampler kernel (``topk_tiles_kernel``): prefill, ``prefill_slots`` with a ``row_slot`` map and the per-op
    decode chain, on raw tile maxima -- from the tensor-core lm_head's epilogue where its GEMM tiles the vocabulary by
    128, from ``tile_max_kernel`` behind the GEMV lm_head (batch <= 4) and narrower GEMM tiles -- with the EOS tile
    patched through ``fix_tile`` while EOS is masked;
  * the persistent decode kernel's sampler (``sample_phase``): processed tile maxima written by ``epi_head``.
Inside ``sample_tiles_seq`` the *direct*, *fast* and *general* paths are chosen from the tile maxima; ``tile_path``
restates that choice so that every case can assert which one its rows took.

The model is programmable: one layer with wo = 0 and down_proj = 0 leaves the residual stream at exactly
``embed[tok]``, and ``embed[t]`` is a one-hot on the pattern that owns ``t mod P``.  Token t's logits are then one
lm_head column (times a common scale), so any bf16 pattern can be written there and exact ties stay exact on every
activation path.  A pattern's strong candidates sit on the ids it owns, so every drawn token selects the same pattern
again and a batch row keeps its pattern for the whole run.  That also tests the hand-off: step s+1's logits must be the
logits of the token drawn at step s.

The float64 reference and the model live in tests/sampler_ref.py; its BARS lists the worst values measured on the
H100 and the bars, about 4x above them.
"""
from __future__ import annotations

import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import make_lm, rel_rms, runs_persistent, set_decode_impl
from tests.sampler_ref import (H, INTER, MASK32, MIN_NEW, PATTERNS, PATTERNS_ALL, PHILOX_M, PHILOX_W, SEED, Checker,
                               _prompts, draw_u, fp32_logits, philox4x32_10, prob_err, processed_scores, programmable,
                               ref_token, ref_window, tile_maxima, tile_path)


# ---------------------------------------------------------------------------------------- CPU tests of the reference
def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10."""
    assert philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    assert philox4x32_10((MASK32,) * 4, (MASK32, MASK32)) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
    assert philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0)) == (
        0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)


def test_philox_constants_match_curand():
    hdr = "/usr/local/cuda/include/curand_philox4x32_x.h"
    if not os.path.exists(hdr):
        pytest.skip("CUDA headers not installed")
    src = open(hdr).read()
    want = {"PHILOX_M4x32_0": PHILOX_M[0], "PHILOX_M4x32_1": PHILOX_M[1], "PHILOX_W32_0": PHILOX_W[0],
            "PHILOX_W32_1": PHILOX_W[1]}
    for name, val in want.items():
        m = re.search(rf"#define\s+{name}\s+\(?(0x[0-9A-Fa-f]+)", src)
        assert m and int(m.group(1), 16) == val, name


def test_draw_u_counter_and_key_layout():
    c0 = philox4x32_10((7, 3, 0, 0), (SEED & MASK32, 1))[0]
    assert draw_u(SEED, 7, 3) == (c0 >> 8) / 16777216.0
    assert 0.0 <= draw_u(SEED, 0, 0) < 1.0
    us = {draw_u(SEED, n, k) for n in range(4) for k in range(4)}
    assert len(us) == 16                                            # counter words 0 and 1 both matter
    assert draw_u(SEED, 5, 2) != draw_u(SEED & MASK32, 5, 2)        # so does the key's high word


def test_ref_window_matches_oracle_topk_probs():
    g = torch.Generator().manual_seed(5)
    V, eos = 5000, 4321
    for top_k, T, ngen in ((50, 0.7, 3), (64, 1.5, 60), (1, 1.0, 0), (17, 1.0, 49)):
        logits = torch.randn(V, generator=g) * 2
        logits[eos] = 20.0
        ids, p = ref_window(logits.numpy(), ngen, eos, 50, top_k, T)
        oi, op = O.topk_probs(logits, ngen, eos, 50, T, top_k)
        assert ids.tolist() == oi.tolist()
        assert prob_err(p, op.double().numpy()) < 1e-6             # HF divides by T: fp32 rounding apart
        assert (eos in ids.tolist()) == (ngen >= 50)


def test_ref_window_ties_keep_smaller_ids():
    logits = np.zeros(300, dtype=np.float32)
    logits[[250, 7, 130, 40, 200]] = 3.0
    logits[299] = 4.0
    ids, p = ref_window(logits, 0, 0, 0, 4, 1.0)
    assert ids.tolist() == [299, 7, 40, 130]
    assert np.allclose(p[1:], p[1]) and p[0] > p[1]


def test_ref_window_eos_mask_and_partial_last_tile():
    V, eos = 16462, 16461                         # 128 full tiles + 78 columns; EOS is the very last id
    logits = np.zeros(V, dtype=np.float32)
    logits[eos], logits[V - 2], logits[5] = 9.0, 8.0, 7.0
    ids, _ = ref_window(logits, 2, eos, 3, 3, 1.0)
    assert ids.tolist() == [V - 2, 5, 0]           # masked while n_generated < min_new_tokens
    ids, _ = ref_window(logits, 3, eos, 3, 3, 1.0)
    assert ids.tolist() == [eos, V - 2, 5]
    tm = tile_maxima(processed_scores(logits, 2, eos, 3, 1.0))
    assert tm.size == 129 and tm[-1] == 8.0        # the padding of the partial tile never wins


def test_inverse_temperature_product_differs_from_division():
    """The kernels multiply by fp32(1/T); transformers divides by T.  For T = 0.7 the two differ in the last bit for a
    sizeable share of logits (never in their order by more than that)."""
    x = np.random.default_rng(0).normal(0, 3, 10000).astype(np.float32)
    mul = x * (np.float32(1) / np.float32(0.7))
    div = x / np.float32(0.7)
    diff = mul != div
    assert 0.05 < diff.mean() < 0.9
    assert np.abs((mul - div)[diff] / div[diff]).max() < 2.5e-7     # one ulp
    assert np.array_equal(processed_scores(x, 0, 0, 0, 0.7)[1:], mul[1:])


def test_ref_token_boundaries():
    w = (np.array([10, 20, 30, 40]), np.array([0.5, 0.25, 0.125, 0.125]))
    assert ref_token(w, 0.0) == (10, {10})
    assert ref_token(w, 0.3) == (10, {10})
    assert ref_token(w, 0.5) == (20, {10, 20})                     # exactly on the boundary: either neighbour
    assert ref_token(w, 0.5 - 2e-6) == (10, {10, 20})
    assert ref_token(w, 0.5 + 2e-5) == (20, {20})
    assert ref_token(w, 0.874999) == (30, {30, 40})
    assert ref_token(w, 0.9) == (40, {40})
    assert ref_token(w, 1.0 - 2.0 ** -24) == (40, {40})           # cumulative sum short of u: the last candidate
    assert ref_token(w, 0.9, greedy=True) == (10, {10})


def test_error_measures_report_non_finite_output():
    assert prob_err([0.5, float("nan")], [0.5, 0.5]) == math.inf
    assert max(0.0, prob_err([math.inf], [1.0])) == math.inf
    assert rel_rms([1.0, float("nan")], [1.0, 1.0]) == math.inf
    assert prob_err([0.5, 0.25], [0.5, 0.5]) == 0.25


def test_odd_vocabulary_is_rejected():
    """The GEMV lm_head works on row pairs, so the library takes even vocabularies only: 16461 and 4141 (the odd sizes
    one would pick for a partial last tile) are refused at configuration; the GPU tests use 16462 and 4142."""
    import ctypes as C

    from neutts_air_b200 import _lib, build

    build.build()
    L = _lib.lib()
    for V in (16461, 4141):
        cfg = _lib.LMConfig(V, H, INTER, 1, 2, 1, 64, 1e-6, 1e6, 4, 256, 64, 16, 256)
        assert L.nt_lm_workspace_bytes(C.byref(cfg)) == 0 and b"even" in L.nt_last_error()
        cfg.vocab_size = V + 1
        assert L.nt_lm_workspace_bytes(C.byref(cfg)) > 0


@pytest.mark.parametrize("V", [217472, 16462, 4142])
def test_patterns_force_their_paths(V):
    """The patterns reach the sample_tiles_seq paths they are meant for (per tile_path on fp32 logits)."""
    m = programmable(V)
    want = {217472: dict(gauss="direct", ties="direct", flat="fast", plateau="general", eos="fast", partial="direct",
                         onetile="direct", stairs="direct"),
            16462: dict(flat="direct", plateau="general", partial="direct"),
            4142: {n: "general" for n in PATTERNS_ALL}}[V]
    for name, path in want.items():
        proc = processed_scores(fp32_logits(m, name), 0, m.eos, 3, 1.0)
        assert tile_path(proc, 50) == path, (name, path)
    # ties: the 84 equal values straddle the 50th and 64th rank; EOS is the largest logit of its pattern
    ids, _ = ref_window(fp32_logits(m, "ties"), 0, m.eos, 0, 64, 1.0)
    vals = fp32_logits(m, "ties")[ids]
    assert (vals[20:] == vals[20]).all() and (np.diff(ids[20:]) > 0).all()
    st = np.sort(fp32_logits(m, "stairs"))[::-1]
    assert (np.diff(st[: min(64, m.nt)]) < 0).all() and st[min(64, m.nt)] < st[min(64, m.nt) - 1]
    lg = fp32_logits(m, "eos")
    assert lg.argmax() == m.eos and (m.eos // 128) != m.nt - 1
    assert [m.pattern_of(m.token_for(n, k)) for n in PATTERNS for k in range(3)] == [j for j in range(7) for _ in range(3)]
    part = fp32_logits(m, "partial")
    assert part[V - 1] == part.max() and part[V - 1] in part[: V - 128]    # V - 1 ties a smaller id


# ====================================================================================== GPU tests
def run_decode_steps(ck: Checker, B: int, steps: int, persistent: bool, tag: str):
    lm = ck.lm
    for step in range(steps):
        before = ck.snapshot()
        if before["done"][:B].all():
            break
        n0 = lm.L.nt_launch_count()
        logits = lm.decode(1, ck.sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        launches = lm.L.nt_launch_count() - n0
        assert (launches == 1) == persistent, (tag, launches)
        after = ck.snapshot()
        ck.check_handoff(logits, range(B), before["cur"], f"{tag} step {step}")
        ck.check_launch(logits, list(range(B)), [ck.sp.slot_base + b for b in range(B)], before, after, 1,
                        tag=f"{tag} step {step}")
        ck.check_tmax(logits, before["ngen"][:B], persistent, f"{tag} step {step}")


# (id, vocabulary, batch, NT_DECODE_IMPL, top_k, temperature, greedy, patterns, per-row limits, expected decode paths)
CASES = [
    ("persistent-b1-eos", 217472, 1, None, 64, 1.0, False, ["eos"], None, {"fast"}),
    ("radix-b3-persistent", 217472, 3, None, 50, 0.7, False, ["ties", "stairs", "partial"], None, {"direct"}),
    ("persistent-b6-hilo", 217472, 6, None, 50, 1.5, False, PATTERNS[:6], [2, 64, 64, 64, 64, 64],
     {"direct", "fast", "general"}),
    ("tile-b9-persistent-bf16", 217472, 9, None, 64, 0.7, False, PATTERNS + ["eos", "flat"], None,
     {"direct", "fast", "general"}),
    ("persistent-b12-partial-tile", 16462, 12, None, 50, 1.0, False, PATTERNS + PATTERNS[:5], None, {"direct", "general"}),
    ("persistent-b20-tc", 217472, 20, "tc", 50, 1.0, False, (PATTERNS_ALL * 3)[:20], None, {"direct", "fast", "general"}),
    ("persistent-b4-top1", 217472, 4, None, 1, 1.0, False, ["gauss", "ties", "flat", "onetile"], None, {"direct"}),
    ("persistent-b6-greedy-v4142", 4142, 6, None, 50, 1.0, True, PATTERNS[:6], None, {"general"}),
    ("chain-b2-radix", 16462, 2, "perop", 1, 1.0, False, ["gauss", "ties"], None, set()),
    ("chain-b7-tile", 217472, 7, "perop", 50, 0.7, False, PATTERNS, [64, 2, 64, 64, 64, 64, 64], set()),
    ("chain-b5-tile-partial", 16462, 5, "perop", 64, 1.5, False, ["partial", "plateau", "eos", "stairs", "flat"], None,
     set()),
    ("chain-b7-radix-v4142", 4142, 7, "perop", 64, 0.7, False, PATTERNS, None, set()),
]
STEPS = 4


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sampler_vs_float64(cuda, case, monkeypatch):
    """Prefill (tile-max kernel with the EOS fix_tile) and STEPS single decode steps on the given path.  At every launch: kept ids, kept probabilities, the drawn token, the state update, the
    hand-off into the next step and (where readable) the tile maxima."""
    name, V, B, impl, top_k, T, greedy, pats, limits, want_paths = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED,
                     greedy=greedy, limits=limits)
    ck = Checker(m, lm, sp, greedy, limits)
    prompts = _prompts(m, pats)
    before = ck.snapshot()
    logits = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    before["ngen"][:] = 0
    before["done"][:] = 0
    ck.check_handoff(logits, range(B), {b: p[-1] for b, p in enumerate(prompts)}, "prefill")
    ck.check_launch(logits, list(range(B)), list(range(B)), before, after, 0, tag="prefill")
    assert after["seq"][:B].tolist() == [len(p) for p in prompts]
    ck.check_tmax(logits, [0] * B, False, "prefill")
    ck.paths.clear()
    set_decode_impl(monkeypatch, impl)
    persistent = runs_persistent(impl, B)
    run_decode_steps(ck, B, STEPS, persistent, name)
    ck.report(name)
    if persistent:
        assert want_paths <= set(ck.paths), (want_paths, ck.paths)
    done = lm.done[:B].cpu()
    if limits is not None:                                    # the capped row stopped, the rest decoded on
        capped = [b for b, c in enumerate(limits) if c < STEPS]
        assert all(int(done[b]) for b in capped) and int(lm.n_generated[capped[0]]) == limits[capped[0]]
        assert int(lm.n_generated[:B].max()) == STEPS + 1
    eos_rows = [b for b, p in enumerate(pats) if p == "eos"]
    if eos_rows:   # EOS, the largest logit, ends a row at the first unmasked step (p(EOS) > 0.9 at every temperature)
        outs, ngen = lm.out_tokens[:B].cpu(), lm.n_generated[:B].cpu()
        stopped = [b for b in eos_rows if int(done[b]) and int(outs[b, int(ngen[b]) - 1]) == m.eos]
        assert stopped and all(int(ngen[b]) == MIN_NEW + 1 for b in stopped), (eos_rows, stopped)


SLOT_CASES = [   # (id, max_batch, first prefill batch, refilled slots, stream ids): GEMV (B = 2) / GEMM (B = 6) lm_head
    ("radix-b2-into-9", 9, 9, [7, 2], [100, 3]),
    ("tile-b6-into-12", 12, 12, [11, 0, 5, 3, 8, 1], [40, 41, 7, 43, 44, 45]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SLOT_CASES, ids=[c[0] for c in SLOT_CASES])
def test_prefill_slots_sampler_vs_float64(cuda, case, monkeypatch):
    """prefill_slots samples logits row i into slot slots[i] with that slot's Philox key; every other slot keeps its
    state.  Then two decode steps on the persistent kernel: refilled slots draw from their own keys."""
    name, MB, B0, slots, keys = case
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=MB, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    ck = Checker(m, lm, sp, False)
    set_decode_impl(monkeypatch, None)
    lm.prefill(_prompts(m, (PATTERNS * 2)[:B0]), sp)
    lm.decode(2, sp)
    torch.cuda.synchronize()
    before = ck.snapshot()
    pats = ["eos", "flat", "ties", "plateau", "partial", "gauss"][: len(slots)]
    prompts = [[m.token_for(p, 5), m.token_for(p, 9)] for p in pats]
    logits = lm.prefill_slots(slots, prompts, sp, keys, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    for s in slots:
        before["ngen"][s], before["done"][s] = 0, 0
    touched = ck.check_launch(logits, slots, keys, before, after, 0, tag="prefill_slots")
    assert [int(after["seq"][s]) for s in slots] == [len(p) for p in prompts]
    for s in set(range(MB)) - touched:                      # every other slot is untouched
        for f in ("ngen", "done", "seq", "cur"):
            assert after[f][s] == before[f][s], (s, f)
        assert (after["out"][s] == before["out"][s]).all(), s
    ck.check_tmax(logits, [0] * len(slots), False, "prefill_slots")
    key_of = {s: k for s, k in zip(slots, keys)}
    for step in range(2):
        before = ck.snapshot()
        lg = lm.decode(1, sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        after = ck.snapshot()
        ck.check_handoff(lg, range(MB), before["cur"], f"after slots, step {step}")
        ck.check_launch(lg, list(range(MB)), [key_of.get(s, s) for s in range(MB)], before, after, 1,
                        tag=f"after slots, step {step}")
    ck.report(name)


@pytest.mark.gpu
@pytest.mark.parametrize("impl,B", [(None, 6), ("perop", 7)], ids=["persistent-b6", "chain-b7"])
def test_multistep_launch_tokens_vs_float64(cuda, impl, B, monkeypatch):
    """decode(n) in one call: every step's drawn token against the reference on that step's returned logits (the
    window is the last step's only), including the persistent kernel's in-kernel step transitions.  The chain then
    reruns the same generation without logits, on its CUDA-graph path: identical tokens."""
    V, n = 217472, 6
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED,
                     limits=[3] + [64] * (B - 1))
    ck = Checker(m, lm, sp, False, [3] + [64] * (B - 1))
    set_decode_impl(monkeypatch, impl)
    prompts = _prompts(m, PATTERNS[:B])
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    st = ck.snapshot()
    n0 = lm.L.nt_launch_count()
    logits = lm.decode(n, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    assert (launches == 1) == runs_persistent(impl, B), launches
    fin = ck.snapshot()
    ngen, done, cur = st["ngen"].copy(), st["done"].copy(), st["cur"].copy()
    for s in range(n):
        if done[:B].all():
            break
        ck.check_handoff(logits[s], [b for b in range(B)], cur, f"step {s}")
        for b in range(B):
            if done[b]:
                continue
            _, tok, ok = ck.expect_token(logits[s, b], int(ngen[b]), b)
            got = int(fin["out"][b, ngen[b]])
            assert got in ok, (s, b, got, tok, ok)
            ngen[b] += 1
            cur[b] = got
            done[b] = got == m.eos or ngen[b] >= ck.lim(b)
    assert fin["ngen"][:B].tolist() == ngen[:B].tolist() and fin["done"][:B].tolist() == done[:B].astype(int).tolist()
    ck.report(f"multistep-{impl or 'persistent'}")
    if impl == "perop":
        toks = fin["out"][:B].copy()
        lm.prefill(prompts, sp)
        lm.decode(n, sp)
        torch.cuda.synchronize()
        assert np.array_equal(lm.out_tokens[:B].cpu().numpy(), toks)
        assert lm.n_generated[:B].cpu().tolist() == fin["ngen"][:B].tolist()


@pytest.mark.gpu
def test_capture_off_and_graph_rebuilt(cuda, monkeypatch):
    """Switching the capture off stops the writes, and a decode graph captured while it was on is not replayed."""
    V, B = 16462, 7
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    set_decode_impl(monkeypatch, "perop")
    tv, ti, tt = lm.debug_capture_sampler()
    lm.prefill(_prompts(m, PATTERNS), sp)
    lm.decode(3, sp)                               # graph captured with the capture on
    torch.cuda.synchronize()
    assert (tt[:B] >= 0).all()
    lm.debug_capture_sampler(False)
    tt.fill_(-7)
    ti.fill_(-7)
    lm.decode(3, sp)
    torch.cuda.synchronize()
    assert (tt == -7).all() and (ti == -7).all()
