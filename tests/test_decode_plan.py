"""CPU: the persistent decode kernel's work plan is a partition of every GEMM phase, for every SM count it may meet.

``tc_build_plan`` (lm_decode_tc.cu) cuts the qkv, o_proj, gate/up and down_proj GEMMs of a layer into (tile, k-block
range, slice) items and hands each CTA at most ``kTcMaxItems`` of them per phase.  The kernel trusts the plan: a tile
slice listed twice is summed twice, one left out is never computed, and neither faults.  The plan depends on the shape
and on the SM count, and a GPU run only ever sees one SM count, so these tests read the plan through
``nt_debug_decode_plan`` (host code, no CUDA call) and check it for every count from 8 to 256.
"""
from __future__ import annotations

import pytest

MAX_ITEMS, MAX_GU_SLICES, MAX_CHUNKS = 4, 4, 14   # kTcMaxItems, kTcMaxGuSlices, the staging area's k-blocks

# (hidden, inter, n_heads, n_kv, vocab): NeuTTS-Air and NeuTTS-Nano widths, and a small model
SHAPES = {"air": (896, 4864, 14, 2, 20546), "nano": (576, 1536, 9, 3, 20546), "small": (256, 640, 4, 2, 20546)}
# which plans the planner accepts on an H100 SXM (132 SMs): (whole-K, flat)
ACCEPTED_AT_132 = {"air": (True, True), "nano": (True, False), "small": (True, True)}
# SM counts at which the Air shape has no whole-K plan (so no persistent-kernel plan at all: every decode takes the
# per-op chain).  114 is the H100 PCIe.  DESIGN.md §2 records this performance cliff.
AIR_WHOLE_K_REJECTED = set(range(8, 42)) | set(range(92, 118))


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


def test_bad_arguments_are_refused():
    from neutts_air_b200.lm import debug_decode_plan

    for n_sms in (7, 257):
        with pytest.raises(ValueError, match="SMs unsupported"):
            debug_decode_plan(*SHAPES["air"], n_sms, False)
    with pytest.raises(ValueError, match="does not fit the shared-memory plan"):
        debug_decode_plan(960, 4864, 15, 5, 20546, 132, False)     # hidden 960 > 896
    with pytest.raises(ValueError, match="multiples of 64"):
        debug_decode_plan(896, 4800 + 32, 14, 2, 20546, 132, False)
