"""CPU: repetition-aware sampling (VALL-E 2's RAS, CosyVoice 2's ``ras_sampling``).

* The float64 reference (``tests/ras_ref.py``): the slot entry's ``min_count = ceil(win_size * tau_r)`` decides
  exactly as CosyVoice's ``rep_num >= win_size * tau_r`` for every window 1..64, a grid of tau_r and every count; the
  window holds generated tokens only; the redraw's uniform is Philox word 1 of the draw's block; the kernel's chunked
  fp32 full-row draw lands on the float64 inverse CDF.
* ``check_ras`` / ``per_prompt_ras`` refuse what ``nt_lm_set_repetition_aware_sampling`` refuses.
* Entries follow prompts through the queue, refills, takes, guided pairs, long-form and the facade; the default makes
  no engine call and forwards nothing.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import RAS_OFF, Settings, check_ras, per_prompt_ras, ras_entry, resolve_settings
from tests.fakes import EOS, FakeTokenizer, GenerateBackbone, GuidedStub, KwBackbone, QueueStub, _facade, _prompts
from tests.processors_ref import model_ref
from tests.ras_ref import (RasChecker, chunk_of, chunk_per, cosyvoice_redraws, draw_u2, full_logprobs, full_scores,
                           kernel_full_draw, min_count, ref_full_token, window_count, window_cut)
from tests.sampler_ref import SEED, draw_u, philox4x32_10, ref_token, ref_window_cut

TAUS = [1e-9, 0.01, 0.05, 0.1, 1 / 3, 0.2, 0.25, 0.3, 0.5, 0.7, 0.75, 0.9, 0.99, 1.0, 0.1 + 0.2, 2 / 3]


# ---------------------------------------------------------------------------------------- the float64 reference
def test_min_count_is_cosyvoice_comparison():
    """Over every window 1..64, a grid of tau_r and every repeat count 0..W: count >= ceil(W * tau) (what the slot
    entry holds) decides exactly as CosyVoice's float comparison, and check_ras stores that ceil."""
    for W in range(1, 65):
        for tau in TAUS:
            W_, m = check_ras(W, tau)
            assert W_ == W and m == min_count(W, tau) and 1 <= m <= W, (W, tau, m)
            for c in range(W + 1):
                hist = [7] * c + [3] * (W - c)
                assert cosyvoice_redraws(hist, 7, W, tau) == (c >= m), (W, tau, c)


def test_window_counts_generated_tokens_only():
    hist = [5, 5, 1, 5, 2, 5]
    assert window_count(hist, 6, 3, 5) == 2 and window_count(hist, 6, 64, 5) == 4 and window_count(hist, 2, 10, 5) == 2
    assert window_count(hist, 0, 10, 5) == 0                     # token 0: empty window, never a redraw
    assert window_count(hist + [5] * 10, 6, 3, 5) == 2           # positions >= n (a refill's old tokens) never count


def test_u2_is_word_one_of_the_same_block():
    for n, key in ((0, 0), (1, 3), (17, 5), (63, 1 << 20)):
        w = philox4x32_10((n, key, 0, 0), (SEED & 0xFFFFFFFF, SEED >> 32))
        assert draw_u(SEED, n, key) == (w[0] >> 8) * 2.0 ** -24
        assert draw_u2(SEED, n, key) == (w[1] >> 8) * 2.0 ** -24
        assert 0.0 <= draw_u2(SEED, n, key) < 1.0


def test_full_row_inverse_cdf_ascending_ids():
    s = np.array([-np.inf, 0.0, np.log(3.0), -np.inf, 0.0], dtype=np.float32)   # p = 0, .2, .6, 0, .2
    assert ref_full_token(s, 0.1)[0] == 1 and ref_full_token(s, 0.5)[0] == 2 and ref_full_token(s, 0.9)[0] == 4
    assert ref_full_token(s, 0.8 - 1e-7)[1] == {2, 4}            # at a boundary either neighbour with mass
    assert ref_full_token(s, 0.5)[1] == {2}
    lp = full_logprobs(s)
    assert lp[0] == -np.inf and abs(math.exp(lp[2]) - 0.6) < 1e-7   # log(3) rounded to fp32


@pytest.mark.parametrize("V", [1000, 4142, 217472])
def test_kernel_draw_lands_on_float64_cdf(V):
    """The kernel's chunked fp32 draw (per-thread chunks, block scan, one chunk walked again) picks the float64
    inverse-CDF token, or a neighbour at an ambiguous boundary, on seeded rows with suppressed ids and a masked EOS."""
    rng = np.random.default_rng(V)
    for case in range(12 if V < 100000 else 3):
        s = (rng.normal(0, 1 + case % 4, V) / (0.7 + 0.1 * case)).astype(np.float32)
        if case % 3 == 1:
            s[: V // 3] = -np.inf                                 # a vocabulary range
        if case % 3 == 2:
            s[rng.integers(V)] = -np.inf                          # a masked EOS
        m = float(s[np.isfinite(s)].max())
        for u2 in (0.0, 1e-6, 0.25, 0.5, 0.9999, float(rng.random()), 1 - 2 ** -24):
            tok, ok = ref_full_token(s, u2)
            got = kernel_full_draw(s, m, u2)
            assert got in ok and np.isfinite(s[got]), (V, case, u2, got, tok, ok)


def _sp(eos, top_k=1):
    return SimpleNamespace(eos_id=eos, seed=SEED, top_k=top_k)


def _device_token(row, s, n, key, history, entry, floor, ctl):
    """What a correct sampler draws: the cut window's inverse CDF of u1, or on a trigger the full row's of u2."""
    T, k, tp, mp = ctl
    ids, q, _ = ref_window_cut(row, n, EOS_V, floor, T, k, tp, mp)
    t = ref_token((ids, q), draw_u(SEED, n, key))[0]
    if entry is not None and n > 0 and window_count(history, n, entry[0], t) >= entry[1]:
        return ref_full_token(full_scores(row, n, EOS_V, floor, T), draw_u2(SEED, n, key))[0], True
    return t, False


EOS_V = 4000   # the EOS id of the CPU rows below (V = 4142)


def _loop_row(rng, V=4142, top=1234):
    row = rng.normal(0.0, 1.5, V).astype(np.float32)
    row[top] = 6.0
    return row


def test_neutral_controls_reduce_to_the_launch_checker():
    """Per-slot entries (T, top_k, 1.0, 0.0) and floors equal to min_new check exactly as the launch-wide checker: the
    same verdicts, redraws and windows over looping slots at several temperatures and top_k."""
    rng = np.random.default_rng(5)
    entries = [(4, 2), (1, 1), None, (10, 1)]
    temps, top_k, min_new = [1.0, 0.7, 1.3, 2.0], 3, 2
    old = RasChecker(_sp(EOS_V, top_k), entries, temps, min_new)
    new = RasChecker(_sp(EOS_V, top_k), entries, temps, min_new, controls=[(T, top_k, 1.0, 0.0) for T in temps],
                     floors=[min_new] * 4)
    rows = [_loop_row(rng, top=100 + 7 * s) for s in range(4)]
    hist = [[] for _ in range(4)]
    for n in range(12):
        for s in range(4):
            got, _ = _device_token(rows[s], s, n, s, hist[s], entries[s], min_new, (temps[s], top_k, 1.0, 0.0))
            hist[s].append(got)
            verdict = old.check(rows[s], s, n, s, hist[s], got)
            assert verdict is not None and new.check(rows[s], s, n, s, hist[s], got) == verdict, (s, n)
    assert old.redrawn == new.redrawn and old.redraws > 0 and old.skipped == new.skipped == 0
    assert old.windows.keys() == new.windows.keys()
    assert all(np.array_equal(old.windows[x], new.windows[x]) for x in old.windows)


def test_top_p_redraw_reads_the_whole_row():
    """A slot whose top-p keeps one id (q0 > top_p): the draw is that id, and a triggered redraw lands on the full
    row's inverse CDF of u2, outside the kept window; the window's id is refused there."""
    rng = np.random.default_rng(7)
    row = rng.normal(0.0, 1.0, 4142).astype(np.float32)
    row[[50, 900, 3000]] = [9.0, 7.5, 8.0]
    ctl = (0.9, 64, 0.3, 0.0)
    ids, _, margin = ref_window_cut(row, 5, EOS_V, 0, *ctl)
    assert ids.tolist() == [50] and margin > 1e-2
    ck = RasChecker(_sp(EOS_V), [(2, 1)], [1.0], 0, controls=[ctl], floors=[0])
    seen = 0
    for n in range(1, 40):
        tok, redrawn = _device_token(row, 0, n, 0, [50] * n, (2, 1), 0, ctl)
        assert redrawn
        ok = ref_full_token(full_scores(row, n, EOS_V, 0, ctl[0]), draw_u2(SEED, n, 0))[1]
        if 50 in ok:
            continue
        assert ck.check(row, 0, n, 0, [50] * n, tok, sampled_lp=full_logprobs(full_scores(row, n, EOS_V, 0, ctl[0]))[tok],
                        model_lp=model_ref(row, tok, EOS_V, False)) is True
        with pytest.raises(AssertionError):
            ck.check(row, 0, n, 0, [50] * n, 50)
        seen += tok not in ids
    assert seen >= 3 and ck.worst_lp == 0.0


def test_floor_masks_eos_in_the_redraw():
    """Below a slot's floor the redraw's row leaves EOS out: where the unmasked full row draws EOS, the checker wants
    the next id with mass and refuses EOS; at or above the floor it accepts EOS."""
    row = np.full(4142, -30.0, dtype=np.float32)
    row[EOS_V - 10], row[EOS_V] = 6.0, 5.0              # EOS (19 % of the mass) sorts after the looping id
    row[EOS_V + 7] = 5.5
    ctl = (1.0, 1, 1.0, 0.0)
    for floor in (3, 30):
        ck = RasChecker(_sp(EOS_V), [(3, 1)], [1.0], 0, controls=[ctl], floors=[floor])
        hits = 0
        for n in range(1, 30):
            hist = [EOS_V - 10] * n
            open_tok = ref_full_token(full_scores(row, n, EOS_V, 0, 1.0), draw_u2(SEED, n, 0))[0]
            tok, redrawn = _device_token(row, 0, n, 0, hist, (3, 1), floor, ctl)
            assert redrawn and (tok != EOS_V if n < floor else tok == open_tok)
            if open_tok == EOS_V and n < floor:
                hits += 1
                assert ck.check(row, 0, n, 0, hist, tok) is True
                with pytest.raises(AssertionError):
                    ck.check(row, 0, n, 0, hist, EOS_V)
            elif open_tok == EOS_V:
                hits += 1
                assert ck.check(row, 0, n, 0, hist, EOS_V) is True
        assert hits >= 2, floor


def test_full_row_chunks_at_v4142():
    """V = 4142: 20 ids per thread, threads 208..255 hold no id and thread 207 the 2-id chunk [4140, 4142).  The
    kernel's fp32 draw restated (``kernel_full_draw``) lands on the float64 CDF when the mass sits in that last chunk,
    in a chunk boundary's neighbours and in an empty thread's range; ``window_cut`` equals ``ref_window_cut``."""
    V = 4142
    assert chunk_per(V) == 20 and chunk_of(V, 4141) == (207, (4140, 4142)) and chunk_of(V, 4139) == (206, (4120, 4140))
    assert all(chunk_of(V, 0)[0] == 0 and min(V, t * 20) == V for t in range(208, 256))
    rng = np.random.default_rng(11)
    for hot in ([4140], [4141], [4140, 4141], [4139, 4140], [19, 20], [4100, 4141]):
        s = (rng.normal(0, 1, V) - 8).astype(np.float32)
        s[hot] = 4.0
        m = float(s.max())
        for u2 in (0.0, 0.3, 0.5, 0.97, 1 - 2 ** -24, float(rng.random())):
            tok, ok = ref_full_token(s, u2)
            assert kernel_full_draw(s, m, u2) in ok, (hot, u2, tok, ok)
    for case in range(6):
        row = rng.normal(0, 2, V).astype(np.float32)
        row[rng.integers(V, size=5)] = 3.0                  # ties across the window's edge
        args = (case, EOS_V, 2, (0.7, 1.3)[case % 2], (1, 8, 64)[case % 3], (1.0, 0.6)[case % 2], (0.0, 0.1)[case % 3 == 2])
        a, b = window_cut(row, *args), ref_window_cut(row, *args)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


# ---------------------------------------------------------------------------------------- host validation
@pytest.mark.parametrize("row,ok", [
    ((10, 0.1), (10, 1)), ((1, 1.0), (1, 1)), ((64, 1.0), (64, 64)), ((64, 0.1), (64, 7)), ((3, 1 / 3), (3, 1)),
    ((10, 0.3), (10, 3)), ((np.int64(8), np.float32(0.5)), (8, 4)), ((5, 1), (5, 5)),
    ((0, 0.1), None), ((65, 0.1), None), ((-1, 0.1), None), ((10.0, 0.1), None), ((True, 0.1), None),
    ((10, 0.0), None), ((10, -0.1), None), ((10, 1.01), None), ((10, math.nan), None), ((10, math.inf), None),
    ((10, True), None), ((10, "0.1"), None), ((10, None), None)])
def test_check_ras(row, ok):
    if ok is None:
        with pytest.raises(ValueError, match="repetition_aware_sampling"):
            check_ras(*row)
    else:
        assert check_ras(*row) == ok


def test_per_prompt_ras():
    assert per_prompt_ras(3, None) is None
    assert per_prompt_ras(3, [None] * 3) is None
    assert per_prompt_ras(2, (10, 0.1)) == [(10, 0.1)] * 2
    assert per_prompt_ras(2, [10, 0.1]) == [(10, 0.1)] * 2
    assert per_prompt_ras(2, [(10, 0.1), None]) == [(10, 0.1), None]
    assert per_prompt_ras(2, [(10, 0.1), (4, 0.5)]) == [(10, 0.1), (4, 0.5)]
    for bad in ((10, 0.1, 3), [(10, 0.1)], [(10, 0.1)] * 3, [(99, 0.1), None], (10, 2.0), [None, (1, 0)], "10"):
        with pytest.raises(ValueError, match="repetition_aware_sampling"):
            per_prompt_ras(2, bad)
    assert ras_entry(None) == RAS_OFF and ras_entry((10, 0.1)) == (10, 1)


def test_abi_refuses_a_null_handle():
    from neutts_air_b200 import _lib

    L = _lib.lib()
    tab = (_lib.SlotRAS * 1)(_lib.SlotRAS(10, 1))
    assert L.nt_lm_set_repetition_aware_sampling(None, tab, None) == -1   # NT_ERR_INVALID
    assert b"nt_lm_set_repetition_aware_sampling: null handle" in L.nt_last_error()


# ---------------------------------------------------------------------------------------- call logs
class RasStub(QueueStub):
    def __init__(self, max_batch, eos_at=None):
        super().__init__(max_batch, eos_at)
        self._ras_host = None

    def set_repetition_aware_sampling(self, rows, slots=None):
        self.log.append(("ras", None if rows is None else list(rows), None if slots is None else list(slots)))
        self._ras_host = None if rows is None else list(rows)


class GuidedRasStub(GuidedStub):
    def __init__(self, max_batch, eos_at=None):
        super().__init__(max_batch, eos_at)
        self._ras_host = None

    def set_repetition_aware_sampling(self, rows, slots=None):
        self.log.append(("ras", None if rows is None else list(rows), None if slots is None else list(slots)))
        self._ras_host = None if rows is None else list(rows)


LENS = [2, 3, 1, 2, 4]
CAPS = [3, 4, 2, 5, 3]


def test_defaults_make_no_engine_call():
    a = QueueStub(2)
    a.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=1)
    for kw in ({}, dict(repetition_aware_sampling=None), dict(repetition_aware_sampling=[None] * 5)):
        b = RasStub(2)
        b.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=1, **kw)
        assert b.log == a.log, kw


def test_queue_writes_entries_before_prefills_and_refills():
    ras = [(10, 0.1), None, (4, 0.5), (64, 1.0), None]
    st = RasStub(2)
    st.generate_queue(_prompts(LENS), EOS, max_new_tokens=CAPS, min_new_tokens=1, repetition_aware_sampling=ras)
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("ras")] == ("ras", ras[:2], None) and kinds.index("ras") < kinds.index("prefill")
    refills = [i for i, e in enumerate(st.log) if e[0] == "refill"]
    assert refills
    for i in refills:
        slots, tags = st.log[i][1], st.log[i][2]
        assert st.log[i - 1] == ("ras", [ras[t - 1] for t in tags], slots)
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # the left-over table goes off
    kinds = [e[0] for e in st.log]
    assert st.log[kinds.index("ras")] == ("ras", None, None) and kinds.index("ras") < kinds.index("prefill")
    st.log.clear()
    st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, min_new_tokens=1)      # off stays off without a call
    assert "ras" not in [e[0] for e in st.log]
    for bad in (dict(repetition_aware_sampling=[(10, 0.1)]), dict(repetition_aware_sampling=(0, 0.1)),
                dict(repetition_aware_sampling=(10, 0.0))):
        st.log.clear()
        with pytest.raises(ValueError, match="repetition_aware_sampling"):
            st.generate_queue(_prompts(LENS[:2]), EOS, max_new_tokens=3, **bad)
        assert st.log == []


def test_takes_and_guided_pairs_repeat_entries():
    s = resolve_settings(None, 2, repetition_aware_sampling=[(10, 0.1), None])
    assert s.ras == [(10, 0.1), None]
    assert s.repeat(3).ras == [(10, 0.1)] * 3 + [None] * 3
    p = s.pair([(1, 2, 3.0)])                # prompt 1 guided: its u slot (2) repeats its entry
    assert p.ras == [(10, 0.1), None, None]
    p = resolve_settings(None, 2, repetition_aware_sampling=(8, 0.25)).pair([(0, 2, 2.0), (1, 3, 2.0)])
    assert p.ras == [(8, 0.25)] * 4
    off = Settings(None, None, None, 1.0, 50).repeat(4)
    assert off.ras is None


def test_guided_queue_entries_follow_c_and_u():
    st = GuidedRasStub(4)
    ras = [(10, 0.1), (5, 0.4), None]
    st.generate_queue(_prompts([2, 2, 2]), EOS, max_new_tokens=3, min_new_tokens=1, guidance_scale=[2.0, 1.0, 3.0],
                      negative_prompt_ids=[[-(i + 1)] * 2 for i in range(3)], repetition_aware_sampling=ras)
    writes = [e for e in st.log if e[0] == "ras"]
    assert writes[0] == ("ras", [(10, 0.1), (5, 0.4), (10, 0.1)], None)   # c slots 0, 1, then prompt 0's u slot
    assert writes[1][1] == [None, None] and len(writes[1][2]) == 2         # prompt 2's c and u slots, at its refill


def test_generate_seam_takes_the_keyword():
    st = RasStub(1)
    seen = {}
    st.generate_batch = lambda prompts, eos, *a, **kw: seen.update(kw) or [torch.tensor([EOS])]
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1, repetition_aware_sampling=[10, 0.1])
    assert seen["repetition_aware_sampling"] == (10, 0.1)
    seen.clear()
    st.generate(torch.tensor([[3, 3, 3]]), max_length=10, eos_token_id=EOS, seed=1)
    assert "repetition_aware_sampling" not in seen


# ---------------------------------------------------------------------------------------- facade
class RasKwBackbone(KwBackbone):
    def set_repetition_aware_sampling(self, rows, slots=None):   # marks an engine that runs RAS
        raise AssertionError("the facade hands the setting to generate_batch / generate_queue")


def _ras(kw):
    return kw.get("repetition_aware_sampling", "absent")


def test_facade_default_forwards_nothing():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    tts = _facade(bb, 3)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_aware_sampling=None)
    tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_aware_sampling=[None, None])
    assert [c[2] for c in bb.calls[1:]] == [bb.calls[0][2]] * 2 and _ras(bb.calls[0][2]) == "absent"
    gb = GenerateBackbone(tok)
    _facade(gb, 1).infer("a b", [1, 2], "r", repetition_aware_sampling=None)
    assert _ras(gb.kws[0]) == "absent"


def test_facade_refuses_backbones_without_it():
    tok = FakeTokenizer()
    gb = GenerateBackbone(tok)
    tts = _facade(gb, 2)
    for call in (lambda: tts.infer("a b", [1, 2], "r", repetition_aware_sampling=(10, 0.1)),
                 lambda: tts.infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, repetition_aware_sampling=[None, (10, 0.1)]),
                 lambda: tts.infer_from_prompt_ids([[1, 2]], repetition_aware_sampling=(10, 0.1)),
                 lambda: tts.infer_batch(["a b"], [[1, 2]], ["r"], long_form=True, repetition_aware_sampling=(10, 0.1))):
        with pytest.raises(ValueError, match="set_repetition_aware_sampling"):
            call()
    assert gb.kws == []   # refused before any generation
    with pytest.raises(ValueError, match="set_repetition_aware_sampling"):
        next(iter(tts.infer_stream("a b", [1, 2], "r", repetition_aware_sampling=(10, 0.1))))
    with pytest.raises(ValueError, match="repetition_aware_sampling"):
        _facade(RasKwBackbone(tok, queue=False), 2).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2,
                                                               repetition_aware_sampling=[(10, 0.1)])


def test_facade_lists_follow_their_utterances():
    tok = FakeTokenizer()
    ras = [None if i % 3 == 1 else (10 + i, 0.1 * (1 + i % 4)) for i in range(7)]
    bb = RasKwBackbone(tok, queue=False)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, repetition_aware_sampling=ras)
    assert [(c[2]["slot_base"], c[2]["repetition_aware_sampling"]) for c in bb.calls] == [
        (0, ras[0:3]), (3, ras[3:6]), (6, ras[6:])]
    bb = RasKwBackbone(tok)
    _facade(bb, 3).infer_batch(["a b"] * 7, [[1, 2]] * 7, ["r"] * 7, repetition_aware_sampling=(10, 0.1))
    assert len(bb.calls) == 1 and bb.calls[0][0] == "queue" and _ras(bb.calls[0][2]) == (10, 0.1)
    bb = RasKwBackbone(tok, queue=False)   # takes: every take of an utterance gets its entry (generate_batch repeats it)
    bb.set_logprobs = lambda on=True: None
    bb._call = lambda what, prompts, kw: bb.calls.append((what, len(prompts), kw)) or (
        [torch.tensor([tok.speech_base + 1])] * (len(prompts) * kw.get("num_return_sequences", 1)),
        [np.zeros((1, 2), np.float32)] * (len(prompts) * kw.get("num_return_sequences", 1)))
    _facade(bb, 4).infer_batch(["a b"] * 2, [[1, 2]] * 2, ["r"] * 2, takes=2, repetition_aware_sampling=[(6, 0.5), None])
    assert [(c[2]["num_return_sequences"], c[2]["repetition_aware_sampling"]) for c in bb.calls] == [(2, [(6, 0.5), None])]


def test_long_form_segments_take_their_texts_entry():
    tok = FakeTokenizer()
    bb = RasKwBackbone(tok, queue=False)
    tts = _facade(bb, 8)
    tts.segments = lambda text, c, rt: text.split("|")
    tts.infer_batch(["a|b|c", "d", "e|f"], [[1, 2]] * 3, ["r"] * 3, long_form=True,
                    repetition_aware_sampling=[(10, 0.1), None, (3, 1.0)])
    # round-robin order: a d e b f c
    assert bb.calls[0][2]["repetition_aware_sampling"] == [(10, 0.1), None, (3, 1.0), (10, 0.1), (3, 1.0), (10, 0.1)]
    bb.calls.clear()
    tts.infer_batch(["a|b", "d"], [[1, 2]] * 2, ["r"] * 2, long_form=True, repetition_aware_sampling=(10, 0.1))
    assert bb.calls[0][2]["repetition_aware_sampling"] == (10, 0.1)
