"""Per-slot sampling controls on every speech-LM sampler path, against the float64 chain of test_sampling_controls.

The programmable one-layer model, the Philox restatement and the float64 top-k helpers come from test_gpu_sampler.py;
every path that file covers is run here with the per-slot table on:
  * identity: a table whose entries equal the launch scalars (top_p = 1, min_p = 0) gives bit-identical tokens,
    captured windows and tile maxima to the table off;
  * mixed controls in one batch: every slot its own (temperature, top_k, top_p, min_p); kept ids exact, kept
    probabilities within BARS["prob"], the token on the float64 inverse CDF of the same Philox draw.  Every cut stays
    at least MARGIN away from its threshold (asserted on the kernel's own logits), so fp32 rounding cannot move it;
  * the persistent kernel's processed tile maxima, fp32(logit) * fp32(1 / T_b) per row, bit for bit;
  * prefill into chosen slots: newcomers sample with their own entries, survivors keep theirs;
  * the C validation of nt_lm_set_slot_sampling and the decode graph when the table is toggled;
  * the facade on synthetic engines.
"""
from __future__ import annotations

import warnings

import numpy as np
import pytest
import torch

from tests.helpers import make_lm
from tests.test_gpu_sampler import (BARS, MIN_NEW, PATTERNS, PATTERNS_ALL, SEED, _prompts, _set_impl, _tile_sampler, draw_u,
                                    fp32_logits, prob_err, processed_scores, programmable, ref_token, tile_maxima, tile_path)
from tests.test_sampling_controls import chain64, ref_window_cut

MARGIN = 1e-4
STEPS = 3

# (temperature, top_k, top_p, min_p): k = 1 and 64, T < 1 and > 1, top-p cutting inside the window, min-p cutting
# before top-p does, and a plain entry
PALETTE = [
    (0.7, 64, 0.5, 0.0),
    (1.5, 1, 1.0, 0.0),
    (1.0, 64, 1.0, 0.2),
    (1.3, 50, 0.9, 0.3),
    (0.5, 20, 0.3, 0.0),
    (2.0, 64, 0.95, 0.01),
    (1.0, 8, 0.6, 0.05),
    (0.8, 33, 1.0, 0.0),
]


def controls_for(B: int, shift: int = 0):
    return [PALETTE[(b + shift) % len(PALETTE)] for b in range(B)]


# (id, vocabulary, batch, NT_DECODE_IMPL, patterns, palette shift, expected paths of sample_tiles_seq)
CASES = [
    ("radix-b2", 16462, 2, "perop", ["gauss", "ties"], 0, set()),
    ("persistent-b1-fold", 217472, 1, None, ["gauss"], 0, {"direct"}),
    ("persistent-b6-hilo-tile-prefill", 217472, 6, None, PATTERNS[:6], 1, {"direct", "fast", "general"}),
    ("persistent-b12-plain", 16462, 12, None, PATTERNS + PATTERNS[:5], 2, {"direct", "general"}),
    ("persistent-b16-plain", 217472, 16, None, PATTERNS_ALL * 2, 0, {"direct", "fast", "general"}),
    ("chain-b20", 217472, 20, None, (PATTERNS_ALL * 3)[:20], 4, set()),
    ("chain-b7-tile", 217472, 7, "perop", PATTERNS, 5, set()),
]


def _windows(m, pat: str, ctl):
    """Reference windows of a pattern row under controls ctl, with EOS masked and unmasked."""
    lg = fp32_logits(m, pat)
    return [ref_window_cut(lg, ngen, m.eos, MIN_NEW, *ctl) for ngen in (0, MIN_NEW)]


SLOT_CASES = [   # (id, max_batch, refilled slots, stream ids): radix (B = 2) / tile kernel (B = 6)
    ("radix-b2-into-9", 9, [7, 2], [100, 3]),
    ("tile-b6-into-12", 12, [11, 0, 5, 3, 8, 1], [40, 41, 7, 43, 44, 45]),
]
SLOT_PATS = ["gauss", "flat", "ties", "plateau", "partial", "gauss"]


def _all_rows():
    """(case, vocabulary, pattern, controls) of every row the GPU tests below check."""
    for name, V, B, impl, pats, shift, _ in CASES:
        for pat, ctl in zip(pats, controls_for(B, shift)):
            yield name, V, pat, ctl
    for name, MB, slots, _ in SLOT_CASES:
        pats, ctl = (PATTERNS * 2)[:MB], controls_for(MB)
        for s, pat, c in zip(slots, SLOT_PATS, controls_for(len(slots), 3)):
            pats[s], ctl[s] = pat, c
        for pat, c in zip(pats, ctl):
            yield name, 217472, pat, c
    for B in (6, 7):
        for pat, ctl in zip(PATTERNS[:B], controls_for(B, 2)):
            yield f"multistep-b{B}", 217472, pat, ctl


def test_cases_keep_clear_of_cut_thresholds():
    """On fp32 logits of the patterns (the kernels reproduce them to ~1e-5), every cut of every case is MARGIN away
    from its threshold, several rows cut inside their window, min-p cuts before top-p somewhere, and the persistent
    cases reach the sample_tiles_seq paths they list."""
    cut = minp_first = 0
    for name, V, pat, ctl in _all_rows():
        m = programmable(V)
        T, k, p, mp = ctl
        for (ids, _, margin), ngen in zip(_windows(m, pat, ctl), (0, MIN_NEW)):
            assert margin >= 2 * MARGIN, (name, pat, ctl, margin)
            s = processed_scores(fp32_logits(m, pat), ngen, m.eos, MIN_NEW, T)
            cut += len(ids) < len(chain64(s, k, 1.0, 0.0)[0])
            if p < 1 and mp > 0:
                minp_first += len(chain64(s, k, 1.0, mp)[0]) < len(chain64(s, k, p, 0.0)[0])
    assert cut >= 20 and minp_first >= 2, (cut, minp_first)
    for name, V, B, impl, pats, shift, want in CASES:
        m = programmable(V)
        paths = {tile_path(processed_scores(fp32_logits(m, pat), ngen, m.eos, MIN_NEW, c[0]), c[1])
                 for pat, c in zip(pats, controls_for(B, shift)) for ngen in (0, MIN_NEW)}
        assert want <= paths, (name, want, paths)


# ====================================================================================== GPU driver
def _snap(lm):
    return dict(ngen=lm.n_generated.cpu().numpy().copy(), done=lm.done.cpu().numpy().copy(),
                seq=lm.seq_lens.cpu().numpy().copy(), out=lm.out_tokens.cpu().numpy().copy())


def _record(lm, cap, logits, before, rows, keys, nt, tag):
    torch.cuda.synchronize()
    R = len(rows)
    return dict(tag=tag, logits=logits.cpu().numpy(), before=before, after=_snap(lm), rows=list(rows), keys=list(keys),
                tv=cap[0][:R].cpu().numpy().copy(), ti=cap[1][:R].cpu().numpy().copy(), tt=cap[2][:R].cpu().numpy().copy(),
                tmax=lm.debug_buffer("tmax", (R, nt)).cpu().numpy().copy())


def drive(lm, sp, prompts, steps, monkeypatch, impl, nt, table=None):
    """prefill + `steps` single decode steps; per launch: logits, captured window, tile maxima, state before / after."""
    cap = lm.debug_capture_sampler()
    _set_impl(monkeypatch, None)
    lm.set_slot_sampling(table)
    B = len(prompts)
    lm.out_tokens.zero_()                           # every run starts from the same buffers: a launch that does not
    lm.debug_buffer("tmax", (B, nt)).zero_()        # write them leaves equal contents in both runs of a comparison
    before = _snap(lm)
    before["ngen"][:], before["done"][:] = 0, 0
    recs = [_record(lm, cap, lm.prefill(prompts, sp, return_logits=True), before, range(B), range(B), nt, "prefill")]
    _set_impl(monkeypatch, impl)
    for step in range(steps):
        before = _snap(lm)
        if before["done"][:B].all():
            break
        lg = lm.decode(1, sp, return_logits=True)[0]
        recs.append(_record(lm, cap, lg, before, range(B), range(B), nt, f"step {step}"))
    return recs


def check_launch(m, rec, ctl, stats, tmax_processed=None):
    """One launch against the float64 chain with the per-slot controls ctl[slot]."""
    tag = rec["tag"]
    for i, (s, key) in enumerate(zip(rec["rows"], rec["keys"])):
        T, k, p, mp = ctl[s]
        lg = rec["logits"][i]
        ngen = int(rec["before"]["ngen"][s])
        ids, q, margin = ref_window_cut(lg, ngen, m.eos, MIN_NEW, T, k, p, mp)
        assert margin >= MARGIN, (tag, i, ctl[s], margin)
        n = len(ids)
        assert rec["ti"][i, :n].tolist() == ids.tolist(), (tag, i, ctl[s], rec["ti"][i, :n].tolist(), ids.tolist())
        assert (rec["ti"][i, n:] == -1).all() and (rec["tv"][i, n:] == 0).all(), (tag, i)
        err = prob_err(rec["tv"][i, :n], q)
        stats["prob"] = max(stats["prob"], err)
        assert err < BARS["prob"], (tag, i, err)
        tok, ok = ref_token((ids, q), draw_u(SEED, ngen, key))
        stats["draws"] += 1
        stats["ambiguous"] += len(ok) > 1
        assert int(rec["tt"][i]) in ok, (tag, i, int(rec["tt"][i]), tok, ok)
        if not rec["before"]["done"][s]:
            assert int(rec["after"]["out"][s, ngen]) == int(rec["tt"][i]), (tag, s)
        stats["cut"] += n < min(k, 64)
        proc = processed_scores(lg, ngen, m.eos, MIN_NEW, T)
        stats["paths"].add(tile_path(proc, k))
        if tmax_processed is not None:
            want = tile_maxima(proc) if tmax_processed else tile_maxima(lg)
            assert np.array_equal(rec["tmax"][i], want), (tag, i, np.nonzero(rec["tmax"][i] != want)[0][:5])


def _engine(V, B, max_batch=None):
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=max_batch or B, max_ctx=256, max_new=64)
    return m, lm


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_identity_and_mixed_controls(cuda, case, monkeypatch):
    name, V, B, impl, pats, shift, want_paths = case
    m, lm = _engine(V, B)
    nt = m.nt
    prompts = _prompts(m, pats)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=0.7, seed=SEED)
    # 1. identity: entries equal to the launch scalars, top-p and min-p off
    off = drive(lm, sp, prompts, STEPS, monkeypatch, impl, nt)
    on = drive(lm, sp, prompts, STEPS, monkeypatch, impl, nt, table=[(0.7, 50, 1.0, 0.0)] * B)
    assert len(off) == len(on)
    for a, b in zip(off, on):
        for f in ("logits", "tv", "ti", "tt", "tmax"):
            assert np.array_equal(a[f], b[f]), (name, a["tag"], f)
        for f in ("ngen", "done", "seq", "out"):
            assert np.array_equal(a["after"][f], b["after"][f]), (name, a["tag"], f)
    # 2. mixed controls, one entry per slot
    ctl = controls_for(B, shift)
    recs = drive(lm, sp, prompts, STEPS, monkeypatch, impl, nt, table=ctl)
    persistent = impl is None and B <= 16
    stats = dict(prob=0.0, draws=0, ambiguous=0, cut=0, paths=set())
    for r in recs:
        tm = None
        if r["tag"] != "prefill" and persistent:
            tm = True                                   # 3. processed maxima of the persistent epilogue, per-row T
        elif _tile_sampler(V, B):
            tm = False                                  # raw maxima of the chain's lm_head GEMM
        check_launch(m, r, ctl, stats, tm)
    if persistent:
        assert want_paths <= stats["paths"], (want_paths, stats["paths"])
    print(f"CONTROLS {name}: draws {stats['draws']} ambiguous {stats['ambiguous']} cut {stats['cut']} "
          f"worst prob err {stats['prob']:.2e} paths {sorted(stats['paths'])}")
    assert stats["cut"] > 0
    assert stats["ambiguous"] <= max(1, BARS["ambiguous"] * stats["draws"])
    lm.set_slot_sampling(None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SLOT_CASES, ids=[c[0] for c in SLOT_CASES])
def test_refilled_slots_sample_with_their_own_controls(cuda, case, monkeypatch):
    """4. The survivors' entries stay, the newcomers' entries are written before their prefill_slots."""
    name, MB, slots, keys = case
    V = 217472
    m, lm = _engine(V, MB)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    cap = lm.debug_capture_sampler()
    _set_impl(monkeypatch, None)
    ctl = controls_for(MB)
    lm.set_slot_sampling(ctl)
    lm.prefill(_prompts(m, (PATTERNS * 2)[:MB]), sp)
    lm.decode(2, sp)
    new = controls_for(len(slots), shift=3)
    lm.set_slot_sampling(new, slots=slots)
    for s, c in zip(slots, new):
        ctl[s] = c
    assert lm._slot_sp_host == ctl
    before = _snap(lm)
    for s in slots:
        before["ngen"][s], before["done"][s] = 0, 0
    pats = SLOT_PATS[: len(slots)]
    prompts = [[m.token_for(p, 5), m.token_for(p, 9)] for p in pats]
    lg = lm.prefill_slots(slots, prompts, sp, keys, return_logits=True)
    stats = dict(prob=0.0, draws=0, ambiguous=0, cut=0, paths=set())
    check_launch(m, _record(lm, cap, lg, before, slots, keys, m.nt, "prefill_slots"), ctl, stats,
                 False if _tile_sampler(V, len(slots)) else None)
    key_of = dict(zip(slots, keys))
    for step in range(2):
        before = _snap(lm)
        lg = lm.decode(1, sp, return_logits=True)[0]
        rec = _record(lm, cap, lg, before, range(MB), [key_of.get(s, s) for s in range(MB)], m.nt, f"after slots {step}")
        check_launch(m, rec, ctl, stats, True)
    assert stats["cut"] > 0 and stats["ambiguous"] <= max(1, BARS["ambiguous"] * stats["draws"])
    print(f"CONTROLS {name}: draws {stats['draws']} cut {stats['cut']} worst prob err {stats['prob']:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("impl,B", [(None, 6), ("perop", 7)], ids=["persistent-b6", "chain-b7"])
def test_multistep_launch_with_controls(cuda, impl, B, monkeypatch):
    """decode(n) in one call with mixed controls: every step's token against the float64 chain on that step's logits;
    the chain then reruns the generation on its CUDA-graph path (no logits) with identical tokens."""
    V, n = 217472, 6
    m, lm = _engine(V, B)
    ctl = controls_for(B, shift=2)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    _set_impl(monkeypatch, impl)
    lm.set_slot_sampling(ctl)
    prompts = _prompts(m, PATTERNS[:B])
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    st = _snap(lm)
    logits = lm.decode(n, sp, return_logits=True).cpu().numpy()
    fin = _snap(lm)
    ngen, done = st["ngen"].copy(), st["done"].copy()
    ambiguous = draws = 0
    for s in range(n):
        for b in range(B):
            if done[b]:
                continue
            ids, q, margin = ref_window_cut(logits[s, b], int(ngen[b]), m.eos, MIN_NEW, *ctl[b])
            assert margin >= MARGIN, (s, b, margin)
            tok, ok = ref_token((ids, q), draw_u(SEED, int(ngen[b]), b))
            got = int(fin["out"][b, ngen[b]])
            assert got in ok, (s, b, got, tok, ok)
            draws += 1
            ambiguous += len(ok) > 1
            ngen[b] += 1
            done[b] = got == m.eos
    assert fin["ngen"][:B].tolist() == ngen[:B].tolist()
    assert ambiguous <= max(1, BARS["ambiguous"] * draws)
    if impl == "perop":
        toks = fin["out"][:B].copy()
        lm.prefill(prompts, sp)
        lm.decode(n, sp)
        torch.cuda.synchronize()
        assert np.array_equal(lm.out_tokens[:B].cpu().numpy(), toks)


@pytest.mark.gpu
def test_validation_and_decode_graph(cuda, monkeypatch):
    """5. The library refuses every bad entry and keeps the previous table; switching the table on replaces a decode
    graph captured without it, and new values in a table that stays on reach the cached graph's next replay."""
    from neutts_air_b200 import _lib

    V, B = 16462, 7
    m, lm = _engine(V, B)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    _set_impl(monkeypatch, "perop")
    tv, ti, tt = lm.debug_capture_sampler()
    prompts = _prompts(m, PATTERNS)
    lm.prefill(prompts, sp)
    lm.decode(3, sp)                                   # graph captured with the table off
    torch.cuda.synchronize()
    assert ((ti[:B] >= 0).sum(1) == 50).all()
    lm.set_slot_sampling([(1.0, 1, 1.0, 0.0)] * B)
    lm.decode(3, sp)                                   # the graph is rebuilt with the table: one kept id per row
    torch.cuda.synchronize()
    assert ((ti[:B] >= 0).sum(1) == 1).all()
    lm.set_slot_sampling([(1.0, 2, 1.0, 0.0)] * B)     # new values, table stays on
    lm.decode(3, sp)
    torch.cuda.synchronize()
    assert ((ti[:B] >= 0).sum(1) == 2).all()
    good = [(1.0, 3, 1.0, 0.0)] * B
    lm.set_slot_sampling(good)
    bads = [(0.0, 3, 1.0, 0.0), (float("nan"), 3, 1.0, 0.0), (float("inf"), 3, 1.0, 0.0), (-1.0, 3, 1.0, 0.0),
            (1.0, 0, 1.0, 0.0), (1.0, 65, 1.0, 0.0), (1.0, 3, 0.0, 0.0), (1.0, 3, 1.5, 0.0), (1.0, 3, float("nan"), 0.0),
            (1.0, 3, 1.0, 1.0), (1.0, 3, 1.0, -0.5), (1.0, 3, 1.0, float("nan"))]
    for bad in bads:
        rows = list(good)
        rows[B - 1] = bad
        arr = (_lib.SlotSampling * B)(*(_lib.SlotSampling(*r) for r in rows))
        with pytest.raises(ValueError):
            _lib.check(lm.L.nt_lm_set_slot_sampling(lm.handle, arr, _lib.current_stream_ptr()))
        with pytest.raises(ValueError):
            lm.set_slot_sampling(rows)
    lm.decode(3, sp)                                   # the last good table is still in force
    torch.cuda.synchronize()
    assert ((ti[:B] >= 0).sum(1) == 3).all()
    lm.set_slot_sampling(None)
    lm.decode(3, sp)                                   # off again: the scalars, on a rebuilt graph
    torch.cuda.synchronize()
    assert ((ti[:B] >= 0).sum(1) == 50).all()
    assert lm.L.nt_lm_set_slot_sampling(lm.handle, None, _lib.current_stream_ptr()) == 0
    assert lm.L.nt_lm_set_slot_sampling(None, None, None) == -1


@pytest.mark.gpu
def test_facade_lists_match_per_utterance_runs(cuda, monkeypatch):
    """6. infer_batch with per-utterance lists: utterance i's ids are those of a generate_batch call on the same prompts
    with every slot set to utterance i's controls (same seed, same stream ids).  Explicit defaults change nothing."""
    from oracle import codec_oracle as CO
    from oracle import lm_oracle as LO
    from tests.helpers import make_codec
    from tests.test_gpu_facade import SmallTok
    from tests.test_host_logic import FakePhonemizer
    from neutts import NeuTTS

    cfg = LO.LMConfig.tiny(vocab_size=4096, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    lm = make_lm(cfg, LO.random_weights(cfg, 3, std=0.05, bf16_round=True), max_batch=3, max_ctx=2048, max_new=512)
    ccfg = CO.CodecConfig.tiny()
    dec = make_codec(ccfg, CO.random_weights(ccfg, 2), max_batch=3, max_frames=512)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=SmallTok(), phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=3, seed=7)
    tts.max_context = 2048
    texts, refs, rts = ["alpha", "beta gamma", "delta"], [torch.arange(10 + 5 * i) for i in range(3)], ["one", "two", "three"]
    plain = tts.infer_batch(texts, refs, rts)
    explicit = tts.infer_batch(texts, refs, rts, temperature=1.0, top_k=50, top_p=1.0, min_p=0.0)
    assert all(np.array_equal(a, b) for a, b in zip(plain, explicit))
    seen = []
    orig = lm.generate_batch

    def rec(*a, **kw):
        out = orig(*a, **kw)
        seen.append([o.clone() for o in out])
        return out

    monkeypatch.setattr(lm, "generate_batch", rec)
    ctl = dict(temperature=[0.6, 1.0, 1.4], top_k=[64, 5, 30], top_p=[0.8, 1.0, 0.5], min_p=[0.0, 0.1, 0.02])
    tts.infer_batch(texts, refs, rts, **ctl)
    got = seen[0]
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
    for i in range(3):
        one = {k: [v[i]] * 3 for k, v in ctl.items()}
        want = orig(prompts, eos, max_length=tts.max_context, min_new_tokens=50, max_new_tokens=None, seed=7, slot_base=0, **one)
        assert torch.equal(got[i], want[i]), i
    assert lm._slot_sp_host is not None
    again = tts.infer_batch(texts, refs, rts)          # a default call after controls: the table is off again
    assert lm._slot_sp_host is None
    assert all(np.array_equal(a, b) for a, b in zip(plain, again))
