"""GPU: per-token log-probabilities (``SpeechLM.set_logprobs``) on every sampler path, against float64.

Runs on the logit-programmable one-layer model of sampler_ref.py (the lm_head writes chosen logits for every input
token), so each case reaches the sampler path it names.  Every case runs twice on one engine, with the feature off and
on, from the same prefill and seed:
  1. tokens, returned logits, captured windows, tile maxima, state and ``nt_launch_count`` deltas are bit-identical;
  2. ``model`` of every token against float64 log_softmax over the kernel's own returned logits row (EOS left out
     while it is masked);
  3. ``sampled`` at the steps whose window is captured (the last step of each launch) against float64 over that
     window's processed scores, ``exp(sampled)`` against the captured kept probability, and -inf for forced ids
     outside the window.  Greedy runs: ``sampled`` equals ``model``.
BARS (LOGPROB_BARS of processors_ref.py) lists the worst values measured on the H100 and the bars.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from neutts_air_b200 import synthetic
from neutts_air_b200.lm import LMShape, SpeechLM
from tests.helpers import _tts, make_lm, set_decode_impl
from tests.processors_ref import LOGPROB_BARS as BARS
from tests.processors_ref import model_ref, sampled_ref
from tests.sampler_ref import PATTERNS, PATTERNS_ALL, SEED, _prompts, programmable

pytestmark = pytest.mark.gpu

MIN_NEW = 3
WORST = {k: 0.0 for k in BARS}


def _note(key, err, tag):
    WORST[key] = max(WORST[key], err)
    assert err < BARS[key], (key, err, tag)


def _snap(lm):
    return {k: getattr(lm, k).cpu().numpy().copy() for k in ("n_generated", "done", "seq_lens", "cur_token", "out_tokens")}


def run_once(lm, sp, prompts, launches, tmax_rows):
    """prefill + decode launches of ``launches`` steps each, all returning logits.  Per launch: the state before and
    after, the logits [steps][R][V], the capture, the tile maxima (``tmax_rows(kind)`` rows, 0 = not read) and the
    launch count."""
    cap = lm.debug_capture_sampler()
    lm.out_tokens.zero_()   # entries past a row's count keep whatever an earlier run wrote
    recs = []
    for n in [0] + list(launches):
        before = _snap(lm)
        c0 = lm.L.nt_launch_count()
        lg = lm.prefill(prompts, sp, return_logits=True)[None] if n == 0 else lm.decode(n, sp, return_logits=True)
        torch.cuda.synchronize()
        rows = tmax_rows("prefill" if n == 0 else "decode")
        recs.append(dict(n=n, before=before, after=_snap(lm), logits=lg.cpu().numpy(), launches=lm.L.nt_launch_count() - c0,
                         cap=[t.cpu().numpy().copy() for t in cap],
                         tmax=lm.debug_buffer("tmax", (rows, programmable(lm.shape.vocab_size).nt)).cpu().numpy().copy()
                         if rows else None))
    return recs


def check_logprobs(recs, lp, B, eos, temps, greedy, forced, tag):
    """Points 2 and 3 of the module docstring over every token the launches wrote."""
    kinds = {"in": 0, "out": 0}
    for r in recs:
        ngen, done = r["before"]["n_generated"].copy(), r["before"]["done"].copy()
        if r["n"] == 0:
            ngen[:], done[:] = 0, 0
        out = r["after"]["out_tokens"]
        for j in range(r["logits"].shape[0]):
            for b in range(B):
                if done[b]:
                    continue
                tok, g = int(out[b, ngen[b]]), int(ngen[b])
                row = r["logits"][j, b]
                sampled, model = (float(v) for v in lp[b, g])
                want = model_ref(row, tok, eos, g < MIN_NEW)
                if want == -math.inf:
                    assert model == -math.inf, (tag, b, g)
                else:
                    _note("model", abs(model - want), (tag, b, g))
                if greedy and not forced:
                    assert sampled == model, (tag, b, g)
                elif j == r["logits"].shape[0] - 1:     # the launch's last step: its window is captured
                    tv, ti, _ = r["cap"]
                    ids = ti[b].tolist()
                    ws = sampled_ref(row, ids, tok, temps[b])
                    if ws == -math.inf:
                        assert sampled == -math.inf, (tag, b, g, sampled)
                        kinds["out"] += 1
                    else:
                        kinds["in"] += 1
                        _note("sampled", abs(sampled - ws), (tag, b, g))
                        _note("prob", abs(math.exp(sampled) - float(tv[b, ids.index(tok)])), (tag, b, g))
                else:   # a forced id may lie outside the window (-inf)
                    assert (forced or math.isfinite(sampled)) and sampled <= 1e-6, (tag, b, g, sampled)
                ngen[b] += 1
                done[b] = tok == eos
    return kinds


def assert_identical(off, on, tag):
    """Point 1: the feature changes nothing but the log-probability buffer."""
    for a, b in zip(off, on):
        assert a["launches"] == b["launches"], (tag, a["launches"], b["launches"])
        assert np.array_equal(a["logits"], b["logits"]), tag
        for k in a["after"]:
            assert np.array_equal(a["after"][k], b["after"][k]), (tag, k)
        for x, y in zip(a["cap"], b["cap"]):
            assert np.array_equal(x, y), tag
        if a["tmax"] is not None:
            assert np.array_equal(a["tmax"], b["tmax"]), tag


CTL = [(0.7, 50, 0.9, 0.0), (1.3, 64, 1.0, 0.05), (1.0, 20, 0.8, 0.02)]
# (id, vocabulary, batch, NT_DECODE_IMPL, top_k, temperature, greedy, forced, patterns, per-slot controls,
#  vocabulary range (lm_head tiles), penalty, decode launches)
CASES = [
    ("persistent-b1-fold", 217472, 1, None, 50, 1.0, False, False, ["eos"], None, None, None, [1, 1, 3]),
    ("persistent-b3-controls", 217472, 3, None, 50, 0.7, False, False, ["ties", "gauss", "flat"], CTL, None, None,
     [1, 2, 2]),
    ("persistent-b8-hilo-penalty", 217472, 8, None, 64, 1.0, False, False, PATTERNS + ["eos"], None, None, 1.3, [1, 3]),
    ("persistent-b16-range-eos-inside", 217472, 16, None, 50, 1.0, False, False, (PATTERNS_ALL * 2)[:16], None,
     (800, 900), None, [1, 3]),
    ("persistent-b3-greedy-penalty", 217472, 3, None, 50, 1.0, True, False, ["eos", "ties", "gauss"], None, None, 1.3,
     [1, 2]),
    ("persistent-b8-forced", 217472, 8, None, 50, 0.7, False, True, PATTERNS + ["eos"], None, None, None, [1, 2]),
    ("chain-b2-radix", 217472, 2, "perop", 50, 1.0, False, False, ["eos", "gauss"], None, None, None, [1, 3]),
    ("chain-b4-radix-range-eos-before", 217472, 4, "perop", 50, 1.0, False, False, ["eos", "ties", "gauss", "flat"],
     None, (900, 1000), 1.3, [1, 2]),
    ("chain-b6-tiles-controls", 217472, 6, "perop", 50, 1.0, False, False, PATTERNS[:6], CTL * 2, None, None, [1, 3]),
    ("chain-b6-tiles-forced", 217472, 6, "perop", 50, 1.0, False, True, PATTERNS[:6], None, None, 1.3, [1, 2]),
    ("chain-b17-tiles-range-eos-after", 217472, 17, None, 50, 1.0, False, False, (PATTERNS_ALL * 3)[:17], None,
     (100, 200), None, [1, 2]),
    ("radix-v4142-b3", 4142, 3, "perop", 64, 1.0, False, False, ["eos", "plateau", "ties"], None, None, None, [1, 2]),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_logprobs_every_path(cuda, case, monkeypatch):
    name, V, B, impl, top_k, T, greedy, forced, pats, ctl, rng, pen, launches = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, impl)
    if ctl is not None:
        lm.set_slot_sampling(ctl[:B])
    if rng is not None:
        lm.set_vocab_range(rng[0] * 128, rng[1] * 128)
    if pen is not None:
        lm.set_repetition_penalty([(pen, True)] * B)
    temps = [ctl[b][0] for b in range(B)] if ctl is not None else [T] * B
    prompts = _prompts(m, pats)
    tmax_rows = lambda kind: B   # every launch leaves the tile maxima of its rows
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED,
                     greedy=greedy)
    if forced:   # the free run's first two tokens (inside the window), then random ids (almost surely outside it)
        free = run_once(lm, sp, prompts, launches, lambda kind: 0)[-1]["after"]["out_tokens"][:B]
        f = torch.from_numpy(free.astype(np.int64))
        g = torch.Generator().manual_seed(3)
        f[:, 2::2] = torch.randint(0, V, (B, f[:, 2::2].shape[1]), generator=g)
        f[f == m.eos] = m.eos + 1
        sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED,
                         greedy=greedy, forced=f)
    off = run_once(lm, sp, prompts, launches, tmax_rows)
    buf = lm.set_logprobs(True)
    buf.fill_(float("nan"))
    on = run_once(lm, sp, prompts, launches, tmax_rows)
    assert_identical(off, on, name)
    lp = buf.cpu().numpy()
    ngen = on[-1]["after"]["n_generated"][:B]
    kinds = check_logprobs(on, lp, B, m.eos, temps, greedy, forced, name)
    for b in range(B):   # written exactly where tokens were, nothing else
        assert not np.isnan(lp[b, : ngen[b]]).any() and np.isnan(lp[b, ngen[b]:]).all(), (name, b)
    if forced:
        assert kinds["in"] > 0 and kinds["out"] > 0, kinds
    eos_rows = [b for b, p in enumerate(pats) if p == "eos" and rng is None and not forced]
    assert all(on[-1]["after"]["done"][b] for b in eos_rows)   # EOS drawn once unmasked: both EOS states covered
    lm.set_logprobs(False)
    assert lm.logprobs is None
    print(f"LOGPROBS {name}: worst {WORST} window kinds {kinds}")


@pytest.mark.parametrize("slots", [[2, 0], [5, 1, 3, 0, 6]], ids=["radix-b2", "tiles-b5"])
def test_prefill_slots_entries(cuda, slots, monkeypatch):
    """prefill_slots writes entry [s][0] of each refilled slot (logits row i -> slot slots[i]) and nothing else."""
    V, MB = 217472, 7
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=MB, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, None)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    buf = lm.set_logprobs(True)
    lm.prefill(_prompts(m, PATTERNS[:MB]), sp)
    lm.decode(2, sp)
    torch.cuda.synchronize()
    old = buf.cpu().numpy().copy()
    cap = lm.debug_capture_sampler()
    prompts = [[m.token_for(p, 5), m.token_for(p, 9)] for p in ["gauss", "ties", "flat", "eos", "partial"][: len(slots)]]
    lg = lm.prefill_slots(slots, prompts, sp, [40 + i for i in range(len(slots))], return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    new = buf.cpu().numpy()
    tv, ti, _ = (t.cpu().numpy() for t in cap)
    out = lm.out_tokens.cpu().numpy()
    for i, s in enumerate(slots):
        tok = int(out[s, 0])
        _note("model", abs(float(new[s, 0, 1]) - model_ref(lg[i], tok, m.eos, True)), ("slots", s))
        _note("sampled", abs(float(new[s, 0, 0]) - sampled_ref(lg[i], ti[i].tolist(), tok, 1.0)), ("slots", s))
    mask = np.ones(new.shape[:2], dtype=bool)
    mask[slots, 0] = False
    assert np.array_equal(old[mask], new[mask], equal_nan=True)


def test_decode_graph_recaptured_on_toggle(cuda, monkeypatch):
    """The per-op chain's decode graph: a graph captured with the feature off never replays with it on, or the reverse."""
    V, B = 217472, 3
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, "perop")
    sp = lm.sampling(m.eos, min_new_tokens=64, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    lm.prefill(_prompts(m, ["gauss", "ties", "flat"]), sp)
    lm.decode(3, sp)                                  # graph captured with the feature off
    buf = lm.set_logprobs(True)
    buf.fill_(float("nan"))
    lm.decode(3, sp)
    torch.cuda.synchronize()
    assert np.isfinite(buf[:B, 4:7].cpu().numpy()).all() and np.isnan(buf[:B, 7:].cpu().numpy()).all()
    lm.set_logprobs(False)
    buf.fill_(float("nan"))
    lm.decode(3, sp)
    torch.cuda.synchronize()
    assert np.isnan(buf.cpu().numpy()).all()
    assert int(lm.n_generated[0]) == 10


def test_queue_rows(cuda, monkeypatch):
    """generate_queue: a buffer pre-filled with NaN returns one finite row per token for every prompt, each equal to
    the same prompt's row of a generate_batch run of its chunk."""
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=3, max_ctx=256, max_new=64)
    set_decode_impl(monkeypatch, None)
    pats = ["eos", "gauss", "ties", "eos", "flat", "partial", "eos"]
    prompts = _prompts(m, pats)
    lm.set_logprobs(True).fill_(float("nan"))
    ids, lps = lm.generate_queue(prompts, m.eos, max_length=40, min_new_tokens=MIN_NEW, seed=SEED, check_every=4,
                                 return_logprobs=True)
    assert lm.logprobs is not None and len(ids) == len(lps) == len(prompts)
    for i, (t, lp) in enumerate(zip(ids, lps)):
        assert lp.dtype == torch.float32 and lp.shape == (len(t), 2), (i, lp.shape)
        assert torch.isfinite(lp).all(), i
        assert (lp <= 1e-6).all(), i
    assert any(len(t) < len(ids[1]) for t in ids)    # EOS rows finished early and their slots were refilled
    plain = lm.generate_queue(prompts, m.eos, max_length=40, min_new_tokens=MIN_NEW, seed=SEED, check_every=4)
    assert lm.logprobs is None and all(torch.equal(a, b) for a, b in zip(plain, ids))


@pytest.mark.parametrize("B", [1, 64])
def test_full_size_model_logprobs(cuda, B, monkeypatch):
    """Air shape, synthetic weights: 500-token prompts and 249 decode steps with EOS masked, at batch 1 (persistent
    kernel) and 64 (chain); ``model`` against float64 log_softmax of the returned logits at several steps."""
    set_decode_impl(monkeypatch, None)
    shape = LMShape()
    V, eos, steps = shape.vocab_size, 151670, 250
    lm = SpeechLM(shape, synthetic.lm_state_dict(shape, 0), device="cuda:0", max_batch=B, max_ctx=1024, max_new=256,
                  max_prefill_tokens=B * 520)
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, V, (500,), generator=g).tolist() for _ in range(B)]
    sp = lm.sampling(eos, min_new_tokens=steps, max_new_tokens=steps, seed=SEED)
    buf = lm.set_logprobs(True)
    buf.fill_(float("nan"))
    lg = lm.prefill(prompts, sp, return_logits=True)
    checks = {0: lg}
    done = 1
    for s in (1, 100, 249):
        if s > done:
            lm.decode(s - done, sp)
        checks[s] = lm.decode(1, sp, return_logits=True)[0]
        done = s + 1
    torch.cuda.synchronize()
    out, lp = lm.out_tokens.cpu().numpy(), buf.cpu().numpy()
    assert np.isfinite(lp[:B, :steps]).all()
    worst = 0.0
    for s, l in checks.items():
        l = l.cpu().numpy()
        for b in range(B):
            err = abs(float(lp[b, s, 1]) - model_ref(l[b], int(out[b, s]), eos, True))
            worst = max(worst, err)
            assert err < BARS["model"], (B, s, b, err)
    print(f"LOGPROBS full size B={B}: worst model err {worst:.2e}")


def test_facade_returns_arrays(cuda, monkeypatch):
    """infer_batch(return_logprobs=True): one float32 [n_generated, 2] array per utterance, equal to the engine's rows
    for the same (seeded) generation."""
    set_decode_impl(monkeypatch, None)
    tts, _ = _tts(max_batch=3)
    texts, refs, rts = ["alpha", "beta gamma", "delta"], [torch.arange(10 + 5 * i) for i in range(3)], ["a", "b c", "d"]
    wavs, lps = tts.infer_batch(texts, refs, rts, return_logprobs=True)
    assert len(wavs) == len(lps) == 3
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    ids, want = tts._generate_ids(prompts, logprobs=True)
    for lp, t, wl in zip(lps, ids, want):
        assert isinstance(lp, np.ndarray) and lp.dtype == np.float32 and lp.shape == (len(t), 2)
        assert np.array_equal(lp, wl.numpy())
    plain = tts.infer_batch(texts, refs, rts)
    assert all(np.array_equal(a, b) for a, b in zip(plain, wavs))
