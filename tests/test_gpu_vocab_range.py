"""GPU: the vocabulary range (``nt_lm_set_vocab_range``, speech-token-only decoding) on every sampler path.

Reuses the logit-programmable one-layer model and the float64 sampler of ``sampler_ref.py``.  Every case runs the
same prompts twice on one path, with the range off and on.  With the range on, at every launch:
  * every suppressed logit reads -inf, and every allowed logit equals the range-off launch bit for bit (a row keeps
    its pattern, and a pattern's logits depend on nothing else);
  * the kept window, its probabilities and the drawn token match the float64 sampler on the kernel's own logits (the
    -inf rows are exactly transformers' SuppressTokensLogitsProcessor);
  * no drawn token lies outside [lo, hi) + EOS.
At the full Air size the engine generates 250 tokens per utterance with the range on, and teacher-forced logits of
the allowed rows equal the range-off logits bit for bit.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200 import synthetic
from neutts_air_b200.lm import LMShape, SpeechLM
from tests.fakes import AlignedTok
from tests.helpers import make_lm, runs_persistent, set_decode_impl
from tests.sampler_ref import (MARGIN, MIN_NEW, PATTERNS, SEED, Checker, _prompts, _range, check_launch, controls_for,
                               drive, programmable)

pytestmark = pytest.mark.gpu


def allowed_mask(V: int, lo: int, hi: int, eos: int):
    a = np.zeros(V, dtype=bool)
    a[lo:hi] = True
    a[eos] = True
    return a


def check_range(tag, logits_on, logits_off, allowed, rows=None):
    """Suppressed -> -inf; allowed rows bit-identical to the range-off logits (rows: which rows to compare)."""
    assert np.isneginf(logits_on[:, ~allowed]).all(), tag
    for i in range(logits_on.shape[0]) if rows is None else rows:
        assert np.array_equal(logits_on[i, allowed], logits_off[i, allowed]), (tag, i)


# (id, vocabulary, batch, NT_DECODE_IMPL, top_k, temperature, patterns, range: "speech" = [lo, V) with EOS outside |
#  "around-eos" = 40 tiles holding EOS, expected sample_tiles_seq paths of the persistent kernel)
CASES = [
    ("persistent-b1-fold", 217472, 1, None, 50, 1.0, ["flat"], "speech", {"fast"}),
    ("persistent-b6-hilo", 217472, 6, None, 50, 0.7, PATTERNS[:6], "speech", {"direct", "fast"}),
    ("persistent-b12-eos-inside", 217472, 12, None, 64, 1.0, PATTERNS + PATTERNS[:5], "around-eos", {"general"}),
    ("persistent-b3-partial-tile", 16462, 3, None, 50, 1.5, ["partial", "gauss", "onetile"], "speech", set()),
    ("persistent-b6-v4142", 4142, 6, None, 50, 1.0, PATTERNS[:6], "speech", {"general"}),
    ("chain-b2-radix", 217472, 2, "perop", 50, 1.0, ["onetile", "ties"], "speech", set()),
    ("chain-b7-tile", 217472, 7, "perop", 64, 0.7, PATTERNS, "speech", set()),
    ("chain-b5-tile-eos-inside", 217472, 5, "perop", 50, 1.0, ["eos", "flat", "gauss", "ties", "stairs"], "around-eos",
     set()),
    # EOS tile after the range's tiles (the last entry of the persistent kernel's lm_head tile list)
    ("persistent-b6-eos-after", 217472, 6, None, 50, 1.0, PATTERNS[:6], "below-eos", {"direct", "fast"}),
    ("chain-b2-radix-eos-after", 217472, 2, "perop", 50, 1.0, ["gauss", "flat"], "below-eos", set()),
    ("chain-b7-tile-eos-after", 217472, 7, "perop", 64, 1.0, PATTERNS, "below-eos", set()),
    # the tied values of the "ties" pattern lie on both sides of lo
    ("persistent-b3-ties-lo", 217472, 3, None, 64, 1.0, ["ties", "ties", "ties"], "ties-lo", set()),
    ("chain-b2-radix-ties-lo", 217472, 2, "perop", 64, 1.0, ["ties", "ties"], "ties-lo", set()),
    ("chain-b5-tile-ties-lo", 217472, 5, "perop", 64, 1.0, ["ties"] * 5, "ties-lo", set()),
]
STEPS = 4


def _run(m, B, impl, top_k, T, pats, rng, monkeypatch):
    """Prefill + STEPS single decode steps; returns (logits per launch, tokens, checker paths, engine)."""
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED)
    if rng is not None:
        lm.set_vocab_range(*rng)
    ck = Checker(m, lm, sp, False)
    prompts = _prompts(m, pats)
    before = ck.snapshot()
    launches = [lm.prefill(prompts, sp, return_logits=True).cpu().numpy()]
    torch.cuda.synchronize()
    after = ck.snapshot()
    before["ngen"][:] = 0
    before["done"][:] = 0
    ck.check_launch(launches[0], list(range(B)), list(range(B)), before, after, 0, tag="prefill")
    ck.check_tmax(launches[0], [0] * B, False, "prefill")
    ck.paths.clear()
    set_decode_impl(monkeypatch, impl)
    persistent = runs_persistent(impl, B)
    curs = [lm.cur_token[:B].cpu().numpy().copy()]
    for step in range(STEPS):
        before = ck.snapshot()
        n0 = lm.L.nt_launch_count()
        lg = lm.decode(1, sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        # under the range a launch first fills its logits rows and tile maxima with -inf (two small kernels)
        assert ((lm.L.nt_launch_count() - n0 - (2 if rng else 0)) == 1) == persistent
        after = ck.snapshot()
        ck.check_launch(lg, list(range(B)), [b for b in range(B)], before, after, 1, tag=f"step {step}")
        ck.check_tmax(lg, before["ngen"][:B], persistent, f"step {step}")
        launches.append(lg)
        curs.append(lm.cur_token[:B].cpu().numpy().copy())
    ck.report("vocab-range" if rng else "range-off")
    toks = [lm.out_tokens[b, : int(lm.n_generated[b])].cpu().numpy() for b in range(B)]
    return launches, curs, ck.paths, toks


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_vocab_range_sampler_paths(cuda, case, monkeypatch):
    name, V, B, impl, top_k, T, pats, kind, want_paths = case
    m = programmable(V)
    lo, hi = _range(m, kind)
    allowed = allowed_mask(V, lo, hi, m.eos)
    off, curs_off, _, _ = _run(m, B, impl, top_k, T, pats, None, monkeypatch)
    on, curs_on, paths, toks = _run(m, B, impl, top_k, T, pats, (lo, hi), monkeypatch)
    compared = 0
    for i, (a, b) in enumerate(zip(on, off)):
        # launch i reads the tokens drawn at launch i - 1 (the prompts' last ids at the prefill)
        rows = [r for r in range(B) if i == 0 or m.pattern_of(int(curs_on[i - 1][r])) == m.pattern_of(int(curs_off[i - 1][r]))]
        compared += len(rows)
        check_range(f"{name} launch {i}", a, b, allowed, rows)
    assert compared >= B * (STEPS + 1) // 2, compared
    for t in toks:
        assert allowed[t].all(), (name, t[~allowed[t]])
    assert want_paths <= set(paths), (want_paths, paths)


@pytest.mark.parametrize("impl,B", [(None, 6), ("perop", 3)], ids=["persistent-b6", "chain-b3"])
def test_vocab_range_multistep_and_toggle(cuda, impl, B, monkeypatch):
    """decode(n) in one launch with the range on, then the range off and on again between launches: every launch's
    logits suppress exactly while the range is on, and the tokens stay in range."""
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    set_decode_impl(monkeypatch, impl)
    lo, hi = 1187 * 128, V
    allowed = allowed_mask(V, lo, hi, m.eos)
    prompts = _prompts(m, PATTERNS[:B])
    lm.set_vocab_range(lo, hi)
    lm.prefill(prompts, sp)
    lg = lm.decode(5, sp, return_logits=True).cpu().numpy()
    assert np.isneginf(lg[:, :, ~allowed]).all() and np.isfinite(lg[:, :, allowed]).all()
    lm.set_vocab_range(None)
    lg = lm.decode(2, sp, return_logits=True).cpu().numpy()
    assert np.isfinite(lg).all()
    lm.set_vocab_range(lo, hi)
    lg = lm.decode(2, sp, return_logits=True).cpu().numpy()
    assert np.isneginf(lg[:, :, ~allowed]).all()
    lm.decode(3, sp)   # the chain's decode graph was captured under the range
    torch.cuda.synchronize()
    for b in range(B):
        t = lm.out_tokens[b, : int(lm.n_generated[b])].cpu().numpy()
        assert allowed[t[:6]].all() and allowed[t[8:]].all(), (b, t)


def test_vocab_range_validation(cuda):
    V = 4142
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=2, max_ctx=256, max_new=64)
    for lo, hi in ((0, V + 2), (128, 128), (256, 128), (128, 191), (100, 1024), (128, 1000), (-128, 1024)):
        with pytest.raises(ValueError):
            lm.set_vocab_range(lo, hi)
        assert lm.L.nt_lm_set_vocab_range(lm.handle, lo, hi, None) != 0
    assert lm.L.nt_lm_set_vocab_range(lm.handle, 3968, V, None) == 0   # hi == V: partial last tile (V % 128 != 0)
    lm.set_vocab_range(0, V)                                           # the whole vocabulary is "off"
    assert lm._vocab_range is None


# ------------------------------------------------------------------------------------------------ full Air size
@pytest.fixture(scope="module")
def air_lm(cuda):
    shape = LMShape()
    return SpeechLM(shape, synthetic.lm_state_dict(shape, 0), device="cuda:0", max_batch=64, max_ctx=1024, max_new=256,
                    max_prefill_tokens=64 * 120)


@pytest.mark.parametrize("B", [1, 8, 16, 64])
def test_full_size_speech_only_generation(air_lm, B, monkeypatch):
    """250 tokens per utterance at the Air shape with the range [speech_base, V): only speech ids or EOS.  Then
    teacher-forced logits with the range on equal the range-off logits on every allowed row, bit for bit."""
    set_decode_impl(monkeypatch, None)
    lm, V, eos, base = air_lm, 217472, 151670, 151936
    allowed = allowed_mask(V, base, V, eos)
    g = torch.Generator().manual_seed(B)
    prompts = [torch.randint(0, V, (100,), generator=g).tolist() for _ in range(B)]
    outs = lm.generate_batch(prompts, eos, max_length=1024, min_new_tokens=250, max_new_tokens=250, seed=3,
                             vocab_range=(base, V))
    assert all(len(o) == 250 for o in outs)
    for o in outs:
        assert allowed[o.numpy()].all()
    forced = torch.stack(outs)[:, :8]
    res = {}
    for rng in ((base, V), None):
        lm.set_vocab_range(*(rng or (None,)))
        sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8, forced=forced)
        first = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
        res[rng is None] = (first, lm.decode(4, sp, return_logits=True).cpu().numpy())
    on, off = res[False], res[True]
    check_range(f"B={B} prefill", on[0], off[0], allowed)
    for s in range(4):
        check_range(f"B={B} step {s}", on[1][s], off[1][s], allowed)
    print(f"VOCAB RANGE full size B={B}: 250 tokens per utterance, all speech ids or EOS; allowed logits bit-identical")


@pytest.mark.parametrize("rng", [(151936, 217472), None], ids=["range-on", "range-off"])
def test_full_size_queue_matches_chunked(cuda, rng, monkeypatch):
    """Equal caps (EOS masked) make the two schedules coincide (as in test_gpu_queue): generate_queue with the range,
    two slots refilled twice, gives exactly the tokens of generate_batch per chunk with the range."""
    set_decode_impl(monkeypatch, None)
    shape = LMShape()
    lm = SpeechLM(shape, synthetic.lm_state_dict(shape, 0), device="cuda:0", max_batch=2, max_ctx=256, max_new=64)
    V, eos, base, cap = 217472, 151670, 151936, 20
    g = torch.Generator().manual_seed(11)
    prompts = [torch.randint(0, V, (int(n),), generator=g).tolist() for n in (40, 90, 60, 75, 50, 33)]
    kw = dict(max_length=256, min_new_tokens=cap, max_new_tokens=cap, seed=5, vocab_range=rng)
    q = lm.generate_queue(prompts, eos, check_every=8, **kw)
    chunked = []
    for i in range(0, 6, 2):
        chunked += lm.generate_batch(prompts[i:i + 2], eos, slot_base=i, **kw)
    assert [len(o) for o in q] == [cap] * 6
    for a, b in zip(q, chunked):
        assert torch.equal(a, b)
        assert rng is None or ((a >= base) | (a == eos)).all()


# ------------------------------------------------------------------------------------ per-slot controls on top
# Inside the speech range the "plateau" pattern keeps only its clipped background, dozens of values tied at 3.0: a
# window of equal probabilities puts top-p's cumulative mass exactly on its threshold, which no reference can decide.
NO_PLATEAU = [p for p in PATTERNS if p != "plateau"]
CTL_CASES = [   # (id, vocabulary, batch, NT_DECODE_IMPL, patterns, palette shift)
    ("radix-b2", 16462, 2, "perop", ["gauss", "ties"], 0),
    ("persistent-b1-fold", 217472, 1, None, ["gauss"], 0),
    ("persistent-b6-hilo", 217472, 6, None, NO_PLATEAU[:6], 1),
    ("persistent-b12-plain", 217472, 12, None, NO_PLATEAU + NO_PLATEAU[:6], 2),
    ("chain-b7-tile", 217472, 7, "perop", PATTERNS, 5),
]


@pytest.mark.parametrize("case", CTL_CASES, ids=[c[0] for c in CTL_CASES])
def test_vocab_range_with_slot_controls(cuda, case, monkeypatch):
    """Per-slot temperature, top_k, top_p and min_p combine with the range unchanged: (1) a table equal to the launch
    scalars is bit-identical to the table off under the range; (2) mixed controls per slot match the float64 chain on
    the kernel's own logits (suppressed ids -inf), with the kept probabilities and tile maxima held to the bars of
    test_gpu_sampling_controls."""
    name, V, B, impl, pats, shift = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    lo, hi = _range(m, "speech")
    allowed = allowed_mask(V, lo, hi, m.eos)
    lm.set_vocab_range(lo, hi)
    nt = m.nt
    prompts = _prompts(m, pats)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=0.7, seed=SEED)
    off = drive(lm, sp, prompts, 3, monkeypatch, impl, nt)
    same = drive(lm, sp, prompts, 3, monkeypatch, impl, nt, table=[(0.7, 50, 1.0, 0.0)] * B)
    for a, b in zip(off, same):
        for f in ("logits", "tv", "ti", "tt", "tmax"):
            assert np.array_equal(a[f], b[f]), (name, a["tag"], f)
    ctl = controls_for(B, shift)
    recs = drive(lm, sp, prompts, 3, monkeypatch, impl, nt, table=ctl)
    persistent = runs_persistent(impl, B)
    stats = dict(prob=0.0, draws=0, ambiguous=0, cut=0, paths=set())
    for r in recs:
        assert np.isneginf(r["logits"][:, ~allowed]).all(), (name, r["tag"])
        check_launch(m, r, ctl, stats, r["tag"] != "prefill" and persistent)
        assert allowed[r["tt"]].all(), (name, r["tag"], r["tt"])
    print(f"CONTROLS+RANGE {name}: draws {stats['draws']} ambiguous {stats['ambiguous']} cut {stats['cut']} "
          f"worst prob err {stats['prob']:.2e} (margin bar {MARGIN}) paths {sorted(stats['paths'])}")
    assert stats["cut"] > 0
    assert stats["ambiguous"] <= max(1, 0.01 * stats["draws"])
    lm.set_slot_sampling(None)


# ------------------------------------------------------------------------------------ prefill into chosen slots
SLOT_CASES = [   # (id, max_batch, first prefill batch, refilled slots, stream ids): GEMV (B = 2) / GEMM (B = 6) lm_head
    ("radix-b2-into-9", 9, 9, [7, 2], [100, 3]),
    ("tile-b6-into-12", 12, 12, [11, 0, 5, 3, 8, 1], [40, 41, 7, 43, 44, 45]),
]


@pytest.mark.parametrize("case", SLOT_CASES, ids=[c[0] for c in SLOT_CASES])
def test_vocab_range_prefill_slots(cuda, case, monkeypatch):
    """prefill_slots under the range: its logits suppress exactly and equal the range-off call on every allowed id, the
    window and token of every row match the float64 sampler, and the refilled slots then decode inside the range."""
    name, MB, B0, slots, keys = case
    V = 217472
    m = programmable(V)
    lo, hi = _range(m, "speech")
    allowed = allowed_mask(V, lo, hi, m.eos)
    pats = ["eos", "flat", "ties", "plateau", "partial", "gauss"][: len(slots)]
    prompts = [[m.token_for(p, 5), m.token_for(p, 9)] for p in pats]
    got = {}
    set_decode_impl(monkeypatch, None)
    for rng in (None, (lo, hi)):
        cfg, w = m.oracle()
        lm = make_lm(cfg, w, max_batch=MB, max_ctx=256, max_new=64)
        sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
        if rng:
            lm.set_vocab_range(*rng)
        ck = Checker(m, lm, sp, False)
        lm.prefill(_prompts(m, (PATTERNS * 2)[:B0]), sp)
        lm.decode(2, sp)
        torch.cuda.synchronize()
        before = ck.snapshot()
        logits = lm.prefill_slots(slots, prompts, sp, keys, return_logits=True).cpu().numpy()
        torch.cuda.synchronize()
        after = ck.snapshot()
        for s in slots:
            before["ngen"][s], before["done"][s] = 0, 0
        ck.check_launch(logits, slots, keys, before, after, 0, tag=f"prefill_slots {rng}")
        ck.check_tmax(logits, [0] * len(slots), False, f"prefill_slots {rng}")
        got[rng is not None] = logits
        if rng:
            assert allowed[[int(after["out"][s, 0]) for s in slots]].all()
            lm.decode(2, sp)
            torch.cuda.synchronize()
            for s in slots:
                t = lm.out_tokens[s, : int(lm.n_generated[s])].cpu().numpy()
                assert allowed[t].all(), (s, t)
        ck.report(f"prefill_slots {name} {rng}")
    check_range(name, got[True], got[False], allowed)


# ------------------------------------------------------------------------------------ the facade end to end
@pytest.mark.parametrize("stream", [False, True], ids=["infer_batch", "infer_stream_batch"])
def test_facade_speech_tokens_only_end_to_end(cuda, stream, monkeypatch):
    """NeuTTS(speech_tokens_only=True) on a random-weight engine (which otherwise emits mostly non-speech ids): every
    generated id is a speech id or EOS, for infer_batch and for infer_stream_batch, and the flag off still lets other
    ids through (so the check has teeth)."""
    import warnings

    from neutts import NeuTTS
    from oracle import codec_oracle as CO
    from oracle import lm_oracle as LO
    from tests.fakes import FakePhonemizer
    from tests.helpers import make_codec

    set_decode_impl(monkeypatch, None)
    tok = AlignedTok()
    V = tok.speech_base + 65536
    cfg = LO.LMConfig.tiny(vocab_size=V, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    lm = make_lm(cfg, LO.random_weights(cfg, 3, std=0.05, bf16_round=True), max_batch=3, max_ctx=2048, max_new=256)
    ccfg = CO.CodecConfig.tiny()
    dec = make_codec(ccfg, CO.random_weights(ccfg, 2), max_batch=3, max_frames=512)
    eos = tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>")
    texts, refs, rts = ["alpha", "beta gamma", "delta"], [torch.arange(10 + 5 * i) for i in range(3)], ["one", "two", "three"]
    seen = []
    orig = lm.generate_batch

    def rec(*a, **kw):
        out = orig(*a, **kw)
        seen.extend(out)
        return out

    monkeypatch.setattr(lm, "generate_batch", rec)
    for only in (False, True):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=3, seed=7,
                         speech_tokens_only=only)
        tts.max_context = 2048
        tts.streaming_frames_per_chunk = 25
        seen.clear()
        if stream:
            for _ in tts.infer_stream_batch(texts, refs, rts):
                pass
            torch.cuda.synchronize()
            ids = [lm.out_tokens[b, : int(lm.n_generated[b])].cpu() for b in range(3)]
        else:
            wavs = tts.infer_batch(texts, refs, rts)
            assert all(len(w_) > 0 and np.isfinite(w_).all() for w_ in wavs)
            ids = list(seen)
        assert len(ids) == 3 and all(len(i) > 0 for i in ids)
        flat = torch.cat(ids)
        in_range = ((flat >= tok.speech_base) & (flat < V)) | (flat == eos)
        if only:
            assert bool(in_range.all()), flat[~in_range][:10]
            assert lm._vocab_range == (tok.speech_base, V)
        else:
            assert not bool(in_range.all())   # random weights: without the flag, non-speech ids do come out
            assert lm._vocab_range is None
