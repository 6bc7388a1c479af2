"""CPU: the persistent decode kernel's work plan is a partition of every GEMM phase, for every SM count it may meet.

``tc_build_plan`` (lm_decode_tc.cu) cuts the qkv, o_proj, gate/up and down_proj GEMMs of a layer into (tile, k-block
range, slice) items and hands each CTA at most ``kTcMaxItems`` of them per phase.  The kernel trusts the plan: a tile
slice listed twice is summed twice, one left out is never computed, and neither faults.  The plan depends on the shape
and on the CTA count, the device's SM count unless ``nt_lm_debug_set_sms`` sets a smaller one.  These tests read the
plan through ``nt_debug_decode_plan`` (host code, no CUDA call) and check it for every count from 8 to 256.  They also
pin the list of plan regimes (``tests.helpers.regime_representatives``): one CTA count per distinct plan, at which
test_gpu_projections.py runs the kernel against float64.
"""
from __future__ import annotations

import pytest

MAX_ITEMS, MAX_GU_SLICES, MAX_CHUNKS = 4, 4, 14   # kTcMaxItems, kTcMaxGuSlices, the staging area's k-blocks

# (hidden, inter, n_heads, n_kv, vocab): NeuTTS-Air and NeuTTS-Nano widths, a small model, the Nano-like model bench.py
# measures in its streaming line (8 query / 2 KV heads, GQA ratio 4), Air widths over 16 / 4 heads, and the
# attention-transparent models of test_gpu_attention.py at every GQA ratio (hidden = 64 * query heads, inter 256)
SHAPES = {"air": (896, 4864, 14, 2, 20546), "nano": (576, 1536, 9, 3, 20546), "small": (256, 640, 4, 2, 20546),
          "bench": (512, 2048, 8, 2, 217472), "air16x4": (896, 4864, 16, 4, 20546)}
RATIO_HEADS = {"gqa1": (8, 8), "gqa2": (4, 2), "gqa3": (9, 3), "gqa4": (8, 2), "gqa4kv3": (12, 3), "gqa5": (10, 2),
               "gqa6": (12, 2), "gqa7": (14, 2), "gqa8": (8, 1)}
SHAPES.update({f"attn-{k}": (64 * nh, 256, nh, nkv, 2048) for k, (nh, nkv) in RATIO_HEADS.items()})
# which plans the planner accepts on an H100 SXM (132 SMs): (whole-K, flat).  Of the transparent models only the
# hidden-256 one has a flat plan there.
ACCEPTED_AT_132 = {"air": (True, True), "nano": (True, False), "small": (True, True), "bench": (True, False),
                   "air16x4": (True, True), **{f"attn-{k}": (True, k == "gqa2") for k in RATIO_HEADS}}
# SM counts at which the Air shape has no whole-K plan (so no persistent-kernel plan at all: every decode takes the
# per-op chain).  114 is the H100 PCIe.  DESIGN.md §2 records this performance cliff.
AIR_WHOLE_K_REJECTED = set(range(8, 42)) | set(range(92, 118))
# The bench shape has a whole-K plan from 12 CTAs up, and no flat plan at 132.
BENCH_WHOLE_K_REJECTED = set(range(8, 12))
# Plan regimes up to 132 CTAs (see test_plan_regimes_up_to_132_ctas)
REGIMES_AT_132 = {"air": 33, "nano": 52, "small": 14, "bench": 47, "air16x4": 30, "attn-gqa1": 17, "attn-gqa2": 6,
                  "attn-gqa3": 20, "attn-gqa4": 19, "attn-gqa4kv3": 25, "attn-gqa5": 22, "attn-gqa6": 27,
                  "attn-gqa7": 31, "attn-gqa8": 18}


def plan_or_none(shape, n_sms, flat):
    from neutts_air_b200.lm import debug_decode_plan

    try:
        return debug_decode_plan(*shape, n_sms, flat)
    except ValueError as e:
        msg = str(e)
        assert msg.startswith("neutts_b200: ") and len(msg) > len("neutts_b200: ") + 10, msg
        return None


def check_plan(shape, n_sms, flat, p):
    """Every invariant the kernel relies on; raises AssertionError naming the first one broken."""
    hidden, inter, n_heads, n_kv, vocab = shape
    qkv_n = (n_heads + 2 * n_kv) * 64
    G = n_sms
    assert len(p["items"]) == G
    geo = {"qkv": (-(-qkv_n // 128), hidden // 64, p["sq"]), "o": (-(-hidden // 128), n_heads, p["so"]),
           "d": (-(-hidden // 128), inter // 64, p["sd"])}
    for ph, (T, KB, S) in geo.items():
        assert 1 <= S <= min(KB, 16), (ph, S)
        got = sorted(it for c in range(G) for it in p["items"][c][ph])
        want = sorted((t, KB * z // S, KB * (z + 1) // S - KB * z // S, z) for t in range(T) for z in range(S))
        assert got == want, f"{ph}: the items are not tiles 0..{T - 1} x slices 0..{S - 1}"
    Tg, KBh = -(-2 * inter // 128), hidden // 64
    gu = [(c, it) for c in range(G) for it in p["items"][c]["gu"]]
    if not flat:
        assert p["sg"] == 1 and p["gu_split"] == 0 and p["gu_nsl"] is None
        assert sorted(it for _, it in gu) == [(t, 0, KBh, 0) for t in range(Tg)], "whole-K gate/up"
    else:
        assert p["gu_split"] == 1 and all(p["gu_split_cta"])
        U = Tg * KBh
        for c in range(G):   # CTA c owns the units [U c / G, U (c + 1) / G) of the tile-major (tile, k-block) order
            units = [t * KBh + k for t, kb0, nkb, _ in p["items"][c]["gu"] for k in range(kb0, kb0 + nkb)]
            assert units == list(range(U * c // G, U * (c + 1) // G)), f"flat gate/up: CTA {c}"
        for t in range(Tg):
            sl = sorted((z, kb0, nkb) for _, (tt, kb0, nkb, z) in gu if tt == t)
            nsl = len(sl)
            assert 1 <= nsl <= MAX_GU_SLICES and nsl == p["gu_nsl"][t], (t, nsl, p["gu_nsl"][t])
            assert [z for z, _, _ in sl] == list(range(nsl)), (t, sl)
            k = 0
            for _, kb0, nkb in sl:      # slices contiguous in K, in slice order, covering 0..KBh
                assert kb0 == k and nkb >= 1, (t, sl)
                k += nkb
            assert k == KBh, (t, sl)
        assert p["sg"] == max(p["gu_nsl"])
    worst = 0
    for c in range(G):
        for ph in ("qkv", "o", "gu", "d"):
            assert len(p["items"][c][ph]) <= MAX_ITEMS
            if ph != "gu" or flat:
                worst = max(worst, sum(it[2] for it in p["items"][c][ph]))
    assert p["max_chunks"] == worst <= MAX_CHUNKS, (p["max_chunks"], worst)
    assert sum(p["fold_q"]) == 1 and sum(p["fold_g"]) == 1
    assert p["items"][p["fold_q"].index(1)]["qkv"] and p["items"][p["fold_g"].index(1)]["gu"]
    assert p["ntiles"] == -(-vocab // 128)


@pytest.mark.parametrize("flat", [False, True], ids=["whole-k", "flat"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_every_accepted_plan_is_a_partition(name, flat):
    shape = SHAPES[name]
    accepted = []
    for n_sms in range(8, 257):
        p = plan_or_none(shape, n_sms, flat)
        if p is None:
            continue
        accepted.append(n_sms)
        check_plan(shape, n_sms, flat, p)
    rejected = sorted(set(range(8, 257)) - set(accepted))
    print(f"PLAN {name} {'flat' if flat else 'whole-K'}: accepted at {len(accepted)} SM counts; rejected at "
          f"{_ranges(rejected) or 'none'}")
    assert (132 in accepted) == ACCEPTED_AT_132[name][flat]
    if name == "air" and not flat:
        assert set(rejected) == AIR_WHOLE_K_REJECTED, _ranges(rejected)
    if name == "bench" and not flat:
        assert set(rejected) == BENCH_WHOLE_K_REJECTED, _ranges(rejected)


def _ranges(xs):
    out, i = [], 0
    while i < len(xs):
        j = i
        while j + 1 < len(xs) and xs[j + 1] == xs[j] + 1:
            j += 1
        out.append(f"{xs[i]}-{xs[j]}" if j > i else str(xs[i]))
        i = j + 1
    return ", ".join(out)


def test_nano_batch1_plan_at_132_sms():
    """At 132 SMs the Nano shape has no flat plan, so batch-1 decode runs the in-CTA fold on the whole-K plan (SwiGLU
    output handed over through act2), a combination the Air shape never takes."""
    assert plan_or_none(SHAPES["nano"], 132, True) is None
    p = plan_or_none(SHAPES["nano"], 132, False)
    assert p is not None and p["gu_split"] == 0 and p["sg"] == 1


def test_plan_regimes_up_to_132_ctas():
    """The regimes a 132-SM H100 can be made to run, one representative CTA count each (the smallest): a regime is the
    (whole-K plan, flat plan) pair of (sq, so, sd, sg, max_chunks, gate/up layout) summaries, None where rejected."""
    from tests.helpers import decode_branch, plan_regime, regime_representatives

    reps = {name: regime_representatives(shape, 132) for name, shape in SHAPES.items()}
    print("REGIMES " + "; ".join(f"{n} {len(r)}: {sorted(r.values())}" for n, r in reps.items()))
    assert {n: len(r) for n, r in reps.items()} == REGIMES_AT_132
    for name, r in reps.items():
        assert len(set(r.values())) == len(r)
        for regime, G in r.items():
            assert plan_regime(SHAPES[name], G) == regime
            assert all(plan_regime(SHAPES[name], g) != regime for g in range(8, G)), (name, G)
        assert min(r.values()) == 8
    air, nano, small = (regime_representatives(SHAPES[n], 132) for n in ("air", "nano", "small"))
    everybody = lambda r: [G for (whole, _), G in r.items() if whole is not None and whole[5]]
    # Air: the whole-K plan in the "everybody does everything" branch (42..91), also with no flat plan, where batch 1
    # folds in the CTAs on the whole-K plan; o_proj in 13 slices (91); no whole-K plan at 92..117 (114: H100 PCIe)
    assert everybody(air) and all(42 <= G <= 91 for G in everybody(air))
    assert any(w is not None and w[5] and f is None for w, f in air)
    assert any(w is not None and w[1] == 13 for w, _ in air)
    assert sum(w is None and 92 <= G <= 117 for (w, _), G in air.items()) >= 2
    assert all(decode_branch(SHAPES["air"], B, G, 512)["kind"] == "chain" for G in range(92, 118) for B in (1, 3, 12))
    # Nano: the flat gate/up plan with the in-CTA fold, and the everybody branch
    assert any(w is not None and f is not None for w, f in nano)
    assert decode_branch(SHAPES["nano"], 1, 16, 512)["plan"] == "flat"
    assert everybody(nano) and all(10 <= G <= 39 for G in everybody(nano))
    # hidden 256: the everybody branch (8..25), attention in one split at batch 3
    assert everybody(small) and all(8 <= G <= 25 for G in everybody(small))
    assert any(decode_branch(SHAPES["small"], 3, G, 512)["split_cap"] == 1 for G in small.values())


def test_bench_and_ratio_shapes_at_132_sms():
    """The paths the GPU tests expect at 132 CTAs.  The bench shape: batch 1 folds in the CTAs on the whole-K plan (no
    flat plan), batch 8, the streaming line's batch, runs the phases on hi + lo activations.  Air widths over 16 / 4
    heads: batch 1 takes the flat plan.  8 / 8 heads at batch 9..16: one attention split per (sequence, KV head)."""
    from tests.helpers import decode_branch

    bench = lambda B: decode_branch(SHAPES["bench"], B, 132, 2048)
    assert [bench(B)["name"] for B in (1, 3, 8, 9, 16)] == [
        "tc-hilo-n16-wholeK-fold", "tc-hilo-n16-wholeK-phases", "tc-hilo-n16-wholeK-phases",
        "tc-bf16-n16-wholeK-phases", "tc-bf16-n16-wholeK-phases"]
    assert decode_branch(SHAPES["air16x4"], 1, 132, 512)["name"] == "tc-hilo-n16-flat-fold"
    assert decode_branch(SHAPES["air16x4"], 8, 132, 512)["name"] == "tc-hilo-n16-wholeK-phases"
    gqa1 = SHAPES["attn-gqa1"]
    assert all(decode_branch(gqa1, B, 132, 2048)["split_cap"] == 1 for B in range(9, 17))
    assert decode_branch(gqa1, 8, 132, 2048)["split_cap"] == 2
    for k in RATIO_HEADS:   # every transparent model runs the persistent kernel at batch 1, 8 and 16
        assert all(decode_branch(SHAPES[f"attn-{k}"], B, 132, 2048)["kind"] == "tc" for B in (1, 8, 16)), k


def test_bad_arguments_are_refused():
    from neutts_air_b200.lm import debug_decode_plan

    for n_sms in (7, 257):
        with pytest.raises(ValueError, match="SMs unsupported"):
            debug_decode_plan(*SHAPES["air"], n_sms, False)
    with pytest.raises(ValueError, match="does not fit the shared-memory plan"):
        debug_decode_plan(960, 4864, 15, 5, 20546, 132, False)     # hidden 960 > 896
    with pytest.raises(ValueError, match="multiples of 64"):
        debug_decode_plan(896, 4800 + 32, 14, 2, 20546, 132, False)


def test_decode_path_constants_match_the_headers():
    """The batch limits the GPU tests predict the decode path with (tests/helpers.py) are the library's own."""
    import os
    import re

    from tests.helpers import GEMV_MAX_BATCH, TC_DEFAULT_MAX_BATCH

    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neutts_air_b200", "csrc")
    for header, name, want in (("lm_decode_tc.cuh", "kTcDefaultMaxBatch", TC_DEFAULT_MAX_BATCH),
                               ("lm_kernels.cuh", "kGemvMaxBatch", GEMV_MAX_BATCH)):
        m = re.search(rf"constexpr\s+int\s+{name}\s*=\s*(\d+)\s*;", open(os.path.join(csrc, header)).read())
        assert m and int(m.group(1)) == want, (header, name, m and m.group(1), want)
