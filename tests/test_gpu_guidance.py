"""GPU: classifier-free guidance (``set_guidance``) on every launch kind of the per-op chain.

Twin runs: the same teacher-forced tokens in the same slots, once with guidance off (the unconditional slot forced to
its c's tokens) and once on.  The twin's raw logits rows give the float64 combination every guided c row must match;
u rows and unguided slots must be bit-identical to the twin (logits, tokens, tile maxima).  Covered: prefill, decode
with the GEMV lm_head (<= 4 rows) and the GEMM lm_head, and ``prefill_slots`` into scattered slots.  Then sampled runs
with per-slot controls, repetition penalty, length control and log-probabilities: every captured window against the
float64 chain on the engine's own processed row, u's state mirroring c's after every launch; routing and launch counts;
the decode graph; the C-level refusals; the queue against per-prompt generate_batch calls; transformers' greedy
guided generate against SpeechLM.generate; and the NeuTTS facade on the synthetic engines.

BARS["combine"] bounds max |got - ref| / max |ref| of a guided row against the float64 combination of the twin's rows:
the worst case measured 3.0e-7 (B = 7, scales up to 4) on one H100 80GB HBM3 (700 W power limit); the bar is 5x that.
BARS["prob"] is sampler_ref's bar on kept probabilities.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200 import _lib
from oracle import lm_oracle as O
from tests.helpers import SMALL, make_lm, set_decode_impl
from tests.sampler_ref import MARGIN, draw_u, prob_err, ref_token, ref_window_cut, tile_maxima

pytestmark = pytest.mark.gpu

BARS = {"combine": 1.5e-6, "prob": 4e-7}


@pytest.fixture(scope="module")
def model():
    cfg = O.LMConfig.tiny(**SMALL)
    w = O.random_weights(cfg, 3, std=0.05, bf16_round=True)
    return cfg, w


def ls64(row):
    x = np.asarray(row, dtype=np.float64)
    m = x.max()
    return x - (m + np.log(np.exp(x - m).sum()))


def combine64(c_row, u_row, g):
    lc, lu = ls64(c_row), ls64(u_row)
    return g * (lc - lu) + lu


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _prompts(rng, V, lens):
    return [rng.integers(0, V - 1, L).tolist() for L in lens]


def _run(lm, prompts, forced, table, steps, refill=None):
    """Teacher-forced prefill + decode (+ optional refill and decode) -> per-launch logits, tokens and tile maxima."""
    lm.set_guidance(table)
    eos = lm.shape.vocab_size - 1
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=1 + 2 * steps, forced=forced)
    out = [lm.prefill(prompts, sp, return_logits=True).cpu()]
    out += list(lm.decode(steps, sp, return_logits=True).cpu())
    if refill is not None:
        slots, new_prompts, new_table = refill
        if table is not None:
            lm.set_guidance(new_table)
        out.append(lm.prefill_slots(slots, new_prompts, sp, stream_ids=[500 + s for s in slots], return_logits=True).cpu())
        out += list(lm.decode(steps, sp, return_logits=True).cpu())
    torch.cuda.synchronize()
    nt = -(-lm.shape.vocab_size // 128)
    tm = lm.debug_buffer("tmax", (lm.max_batch, nt)).clone().cpu()
    return out, lm.out_tokens.clone().cpu(), lm.n_generated.clone().cpu(), tm


@pytest.mark.parametrize("B", [4, 7])
def test_combine_against_twin(model, monkeypatch, B):
    """Prefill and decode at B rows (GEMV lm_head at 4, GEMM at 7), then a refill of two scattered slots as a new
    pair: guided rows against the float64 combination of the twin's rows, everything else bit-identical."""
    set_decode_impl(monkeypatch, "perop")
    cfg, w = model
    V = cfg.vocab_size
    lm = make_lm(cfg, w, max_batch=8, max_ctx=256)
    rng = np.random.default_rng(B)
    lens = [37, 50, 21, 64, 9, 30, 44][:B]
    prompts = _prompts(rng, V, lens)
    # B = 4: pair (0, 3) and (1, 2);  B = 7: pairs (0, 5), (3, 6), slots 1, 2, 4 unguided
    pairs = [(0, 3, 3.0), (1, 2, 0.6)] if B == 4 else [(0, 5, 2.5), (3, 6, 1.7)]
    table = [(-1, 1.0)] * 8
    for c, u, g in pairs:
        table[c] = (u, g)
    steps = 3
    forced = torch.from_numpy(rng.integers(0, V - 1, (8, 1 + 2 * steps))).int()
    for c, u, _ in pairs:
        forced[u] = forced[c]
    refill = None
    if B == 7:   # slots 6 and 1 refilled as a new pair (c = 6, u = 1); pair (3, 6) ends
        new_table = list(table)
        new_table[3] = (-1, 1.0)
        new_table[6] = (1, 4.0)
        refill = ([6, 1], _prompts(rng, V, [25, 12]), new_table)
        forced[1] = forced[6]
    twin = _run(lm, prompts, forced, None, steps, refill)
    got = _run(lm, prompts, forced, table, steps, refill)
    assert torch.equal(twin[1][:B], got[1][:B]) and torch.equal(twin[2][:B], got[2][:B])
    worst = 0.0
    for launch, (lt, lg) in enumerate(zip(twin[0], got[0])):
        if refill is not None and launch == 1 + steps:   # the refill's rows are in call order: (c = 6, u = 1)
            ref = combine64(lt[0].numpy(), lt[1].numpy(), 4.0)
            worst = max(worst, float(np.abs(lg[0].numpy() - ref).max() / np.abs(ref).max()))
            assert np.array_equal(bits(lt[1]), bits(lg[1]))
            continue
        cur = pairs if (refill is None or launch <= steps) else [(0, 5, 2.5), (6, 1, 4.0)]
        guided = {c for c, _, _ in cur}
        for r in range(lt.shape[0]):
            if r in guided:
                c, u, g = next(p for p in cur if p[0] == r)
                ref = combine64(lt[c].numpy(), lt[u].numpy(), g)
                worst = max(worst, float(np.abs(lg[c].numpy() - ref).max() / np.abs(ref).max()))
            else:
                assert np.array_equal(bits(lt[r]), bits(lg[r])), (launch, r)
    print(f"B={B}: worst relative combine error {worst:.3e}")
    assert worst < BARS["combine"], worst
    # tile maxima of the last launch: the combined rows' raw maxima, the others as the twin's
    last = got[0][-1]
    cur = pairs if refill is None else [(0, 5, 2.5), (6, 1, 4.0)]
    for r in range(last.shape[0]):
        if r in {c for c, _, _ in cur}:
            assert np.array_equal(bits(got[3][r]), bits(tile_maxima(last[r].numpy()))), r
        else:
            assert np.array_equal(bits(got[3][r]), bits(twin[3][r])), r


def test_against_float64_model(model, monkeypatch):
    """The guided row at prefill against the float64 model's rows of the prompt and the negative prompt, and u's next
    logits after one forced step against the float64 model on the negative prompt plus c's token."""
    set_decode_impl(monkeypatch, "perop")
    from tests.sampler_ref import forward64

    cfg, w = model
    V = cfg.vocab_size
    lm = make_lm(cfg, w, max_batch=2, max_ctx=128)
    rng = np.random.default_rng(5)
    p, q = _prompts(rng, V, [40, 23])
    forced = torch.from_numpy(rng.integers(0, V - 1, (2, 4))).int()
    lm.set_guidance([(1, 2.0), (-1, 1.0)])
    sp = lm.sampling(V - 1, min_new_tokens=0, max_new_tokens=4, forced=forced)
    l0 = lm.prefill([p, q], sp, return_logits=True).cpu()
    l1 = lm.decode(1, sp, return_logits=True).cpu()
    torch.cuda.synchronize()
    f_p = forward64(cfg, w, torch.tensor(p))[-1].numpy()
    f_q = forward64(cfg, w, torch.tensor(q))[-1].numpy()
    ref = combine64(f_p, f_q, 2.0)
    d = l0[0].numpy() - ref
    assert float(np.linalg.norm(d - d.mean()) / np.linalg.norm(ref - ref.mean())) < 2e-2
    t0 = int(forced[0, 0])
    f_q1 = forward64(cfg, w, torch.tensor(q + [t0]))[-1].numpy()
    assert float(np.linalg.norm(l1[0, 1].numpy() - f_q1) / np.linalg.norm(f_q1)) < 6e-3
    assert lm.out_tokens[1, :2].tolist() == forced[0, :2].tolist()


@pytest.mark.parametrize("V", [217472, 4096])
def test_draws_and_mirror(monkeypatch, V):
    """Sampled guided runs with per-slot controls, penalty, length control, a speech vocabulary range and
    log-probabilities: every window against the float64 chain on the engine's processed row, the token against the
    Philox draw, and u's state equal to c's after every launch."""
    set_decode_impl(monkeypatch, "perop")
    cfg = O.LMConfig.tiny(vocab_size=V, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    w = O.random_weights(cfg, 9, std=0.05, bf16_round=True)
    lm = make_lm(cfg, w, max_batch=6, max_ctx=256)
    rng = np.random.default_rng(V)
    prompts = _prompts(rng, V, [30, 45, 12, 28, 8, 19])
    ctrl = [(0.8, 40, 0.9, 0.0), (1.0, 64, 1.0, 0.05), (1.3, 20, 1.0, 0.0)]
    lm.set_slot_sampling(ctrl + ctrl)
    lm.set_repetition_penalty([(1.2, True), (1.0, True), (0.9, False)] * 2)
    lm.set_length_control([(2, 3, 1.1), (0, 0, 1.0), (1, 4, 1.05)] * 2)
    if V > 4096:
        lm.set_vocab_range(128, V - 128 * 64)
    lm.set_logprobs(True)
    table = [(3, 3.0), (4, 0.5), (-1, 1.0), (-1, 1.0), (-1, 1.0), (-1, 1.0)]
    lm.set_guidance(table)
    cap = lm.debug_capture_sampler(True)
    seed = 77
    eos = V - 1
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=12, seed=seed)
    rows = [lm.prefill(prompts, sp, return_logits=True).cpu()]
    checked = 0
    for step in range(11):
        ngen = lm.n_generated.cpu().tolist()
        st = [lm.cur_token.cpu(), lm.seq_lens.cpu(), lm.done.cpu()]
        for c, u in ((0, 3), (1, 4)):
            assert lm.n_generated[u] == lm.n_generated[c] and lm.cur_token[u] == lm.cur_token[c]
            assert lm.done[u] == lm.done[c]
            assert torch.equal(lm.out_tokens[u, : ngen[c]], lm.out_tokens[c, : ngen[c]])
            assert int(st[1][u]) - int(st[1][c]) == len(prompts[u]) - len(prompts[c])
        lg = rows[-1]
        for s in (0, 1, 2):
            if step > 0 and int(prev_done[s]):
                continue
            n = ngen[s] - 1
            T, k, tp, mp = ctrl[s]
            floor = (2, 0, 1)[s]
            ids, q, margin = ref_window_cut(lg[s].numpy(), n, eos, floor, T, k, tp, mp)
            if margin < MARGIN:
                continue
            got_ids = cap[1][s].cpu().numpy()
            got_ids = got_ids[got_ids >= 0]
            assert got_ids.tolist() == ids.tolist(), (step, s)
            assert prob_err(cap[0][s].cpu().numpy()[: len(ids)], q) < BARS["prob"]
            _, ok = ref_token((ids, q), draw_u(seed, n, s))
            tok = int(cap[2][s])
            assert tok in ok
            # the model log-probability: log-softmax of the processed row, EOS left out while masked
            row = lg[s].numpy().astype(np.float64)
            if n < floor:
                row[eos] = -np.inf
            m = row[np.isfinite(row)].max()
            model_lp = row[tok] - (m + np.log(np.exp(row[np.isfinite(row)] - m).sum()))
            assert abs(float(lm.logprobs[s, n, 1]) - model_lp) < 1e-4
            checked += 1
        prev_done = st[2]
        if bool(lm.done[:3].all()):
            break
        rows.append(lm.decode(1, sp, return_logits=True)[0].cpu())
    assert checked >= 12, checked
    lm.set_logprobs(False)
    lm.debug_capture_sampler(False)


def test_routing_and_launch_counts(model, monkeypatch):
    """Guided decode runs the chain at every batch with three launches per step on top of the chain's; tc refuses."""
    cfg, w = model
    V = cfg.vocab_size
    L = _lib.lib()
    lm = make_lm(cfg, w, max_batch=16, max_ctx=256)
    rng = np.random.default_rng(1)
    for B in (2, 4, 9, 16):
        prompts = _prompts(rng, V, [10 + b for b in range(B)])
        sp = lm.sampling(V - 1, min_new_tokens=0, max_new_tokens=8)
        per = {}
        for on in (False, True):
            set_decode_impl(monkeypatch, None if on else "perop")
            lm.set_guidance([(B - 1, 2.0)] + [(-1, 1.0)] * 15 if on else None)
            lm.prefill(prompts, sp)
            lm.decode(1, sp)
            n0 = L.nt_launch_count()
            lm.decode(1, sp)
            torch.cuda.synchronize()
            per[on] = L.nt_launch_count() - n0
        assert per[True] == per[False] + 3, (B, per)
        set_decode_impl(monkeypatch, "tc")
        with pytest.raises(ValueError):
            lm.decode(1, sp)
    lm.set_guidance(None)


def test_graph_reads_new_scales_and_refusals(model, monkeypatch):
    """A graph captured with one scale replays a new scale written into a table that stays on; each bad table is
    refused by the library and the previous one stays in force."""
    set_decode_impl(monkeypatch, "perop")
    cfg, w = model
    V = cfg.vocab_size
    lm = make_lm(cfg, w, max_batch=4, max_ctx=128)
    rng = np.random.default_rng(2)
    prompts = _prompts(rng, V, [20, 31, 17, 9])
    forced = torch.from_numpy(rng.integers(0, V - 1, (4, 8))).int()
    forced[2] = forced[0]
    sp = lm.sampling(V - 1, min_new_tokens=0, max_new_tokens=8, forced=forced)
    lm.set_guidance(None)
    lm.prefill(prompts, sp)
    raw = lm.decode(3, sp, return_logits=True)[-1].cpu()
    for g in (2.0, 5.0):
        lm.set_guidance([(2, g), (-1, 1.0), (-1, 1.0), (-1, 1.0)])
        lm.prefill(prompts, sp)
        lm.decode(3, sp)   # graph path: the table is read at replay
        torch.cuda.synchronize()
        got = lm.debug_buffer("logits", (4, V)).cpu()
        ref = combine64(raw[0].numpy(), raw[2].numpy(), g)
        assert np.abs(got[0].numpy() - ref).max() / np.abs(ref).max() < BARS["combine"], g
        assert np.array_equal(bits(got[1]), bits(raw[1]))
    L = _lib.lib()
    bad = [[(0, 2.0)] + [(-1, 1.0)] * 3,                   # its own partner
           [(4, 2.0)] + [(-1, 1.0)] * 3,                   # out of range
           [(2, 2.0), (2, 3.0), (-1, 1.0), (-1, 1.0)],     # one u for two c
           [(2, 2.0), (-1, 1.0), (3, 2.0), (-1, 1.0)],     # the partner has a partner
           [(2, 1.0)] + [(-1, 1.0)] * 3,                   # scale 1
           [(2, -1.0)] + [(-1, 1.0)] * 3,                  # scale <= 0
           [(2, float("inf"))] + [(-1, 1.0)] * 3]          # not finite
    for t in bad:
        arr = (_lib.SlotGuidance * 4)(*(_lib.SlotGuidance(*e) for e in t))
        assert L.nt_lm_set_guidance(lm.handle, arr, _lib.current_stream_ptr()) == -1, t
        with pytest.raises(ValueError):
            lm.set_guidance(t)
    lm.prefill(prompts, sp)
    lm.decode(3, sp)
    torch.cuda.synchronize()
    got = lm.debug_buffer("logits", (4, V)).cpu()
    ref = combine64(raw[0].numpy(), raw[2].numpy(), 5.0)   # the last good table is still in force
    assert np.abs(got[0].numpy() - ref).max() / np.abs(ref).max() < BARS["combine"]
    with pytest.raises(ValueError):
        lm.prefill_fork(prompts[:2], 2, sp)


def test_queue_mixed(model, monkeypatch):
    """generate_queue over 3 x max_batch mixed prompts (pairs admitted by prefill_slots into freed slots) against a
    generate_batch call of each prompt with the same stream key (slot_base = its index) at the same lm_head width on
    the same decode path: the first wave's tokens are equal, and at least half of the refilled prompts' tokens; every
    page is back in the pool."""
    set_decode_impl(monkeypatch, None)
    cfg, w = model
    V = cfg.vocab_size
    M = 6
    lm = make_lm(cfg, w, max_batch=M, max_ctx=256)
    rng = np.random.default_rng(4)
    n = 3 * M
    prompts = _prompts(rng, V, rng.integers(5, 60, n).tolist())
    scales = [(2.0, 1.0, 3.0)[i % 3] for i in range(n)]
    negs = [None if i % 2 else _prompts(rng, V, [int(rng.integers(3, 30))])[0] for i in range(n)]
    caps = rng.integers(3, 30, n).tolist()
    kw = dict(eos_token_id=V - 1, min_new_tokens=0, seed=3)
    out = lm.generate_queue(prompts, max_new_tokens=caps, guidance_scale=scales, negative_prompt_ids=negs, check_every=4,
                            **kw)
    assert lm.pool.num_free == lm.num_pages
    # the reference runs prompt i in slot 0 (stream key i) padded with unguided fillers to the queue's width, so its
    # rows take the same lm_head path (GEMM, bf16-normalised rows) as in the queue; alone it would take the GEMV, and
    # an unguided call at this width would take the persistent kernel
    fill = _prompts(rng, V, [20] * M)
    set_decode_impl(monkeypatch, "perop")   # the queue ran every slot on the chain (guidance was on); so do the references
    first = 0   # prompts 0 .. first - 1 went in by the queue's first prefill, in the generate_batch layout
    while first < n and first + 1 + sum(g != 1.0 for g in scales[: first + 1]) <= M:
        first += 1
    refilled = exact = 0
    for i in range(n):
        f = M - 1 - (scales[i] != 1.0)
        one = lm.generate_batch([prompts[i]] + fill[:f], max_new_tokens=[caps[i]] + [max(caps)] * f,
                                guidance_scale=[scales[i]] + [1.0] * f, negative_prompt_ids=[negs[i]] + [None] * f,
                                slot_base=i, **kw)[0]
        if i < first:
            assert torch.equal(out[i], one), i
            continue
        # a refill's prefill shares its call with other prompts, and the prefill GEMMs split K by the call's token
        # count, so its KV matches the reference's only to rounding (bf16 activations) and a draw may part; the
        # admission itself (partner, negative prompt, key, cap) is checked exactly on the CPU stub (test_guidance.py)
        refilled += 1
        exact += bool(torch.equal(out[i], one))
    print(f"queue: {first} first-wave prompts equal, {exact} of {refilled} refilled prompts equal to the end")
    assert exact * 2 >= refilled
    assert refilled > 0
    lm.set_guidance(None)


def test_transformers_greedy_end_to_end(model, monkeypatch):
    """transformers' float64 Qwen2ForCausalLM, greedy, with guidance_scale and negative_prompt_ids (explicit, and the
    default of the prompt's last token), against greedy SpeechLM.generate: while the two sequences agree, every step
    whose float64 guided top-2 margin is at least MARGIN_BAR draws the same token; where they part, the margin was
    below the bar."""
    set_decode_impl(monkeypatch, None)
    from transformers import Qwen2Config, Qwen2ForCausalLM

    from tests.helpers import lm_state_dict

    MARGIN_BAR = 0.05   # guided log-probability units; the engine's guided rows sit ~1e-2 from float64 at most here
    cfg, w = model
    V = cfg.vocab_size
    hc = Qwen2Config(vocab_size=V, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                     num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.num_heads,
                     num_key_value_heads=cfg.num_kv_heads, rms_norm_eps=cfg.rms_eps, max_position_embeddings=256,
                     tie_word_embeddings=True, rope_parameters={"rope_type": "default", "rope_theta": cfg.rope_theta})
    hf = Qwen2ForCausalLM(hc).double().eval()
    hf.config._attn_implementation = "eager"
    missing, _ = hf.load_state_dict({k: v.double() for k, v in lm_state_dict(w).items()}, strict=False)
    assert set(missing) <= {"lm_head.weight"}
    hf.tie_weights()
    lm = make_lm(cfg, w, max_batch=2, max_ctx=256)
    rng = np.random.default_rng(8)
    N = 16
    checked = 0
    for explicit in (True, False):
        p = _prompts(rng, V - 1, [33])[0]
        neg = _prompts(rng, V - 1, [14])[0] if explicit else None
        ids = torch.tensor([p])
        extra = dict(negative_prompt_ids=torch.tensor([neg])) if explicit else {}
        with torch.no_grad():
            r = hf.generate(ids, do_sample=False, guidance_scale=2.0, max_new_tokens=N, min_new_tokens=N, eos_token_id=V - 1,
                            pad_token_id=0, output_scores=True, return_dict_in_generate=True, **extra)
        ref = r.sequences[0, len(p):].tolist()
        got = lm.generate(ids.cuda(), max_length=256, eos_token_id=V - 1, do_sample=False, min_new_tokens=N,
                          max_new_tokens=N, guidance_scale=2.0, **extra)[0, len(p):].cpu().tolist()
        for t in range(N):
            top2 = torch.topk(r.scores[t][0], 2).values
            margin = float(top2[0] - top2[1])
            if got[t] != ref[t]:
                assert margin < MARGIN_BAR, (explicit, t, margin)
                break
            checked += margin >= MARGIN_BAR
    print(f"transformers greedy: {checked} steps checked")
    assert checked >= 12, checked
    lm.set_guidance(None)


def test_facade_on_engines():
    """NeuTTS.infer_batch with per-utterance scales and negative texts on the synthetic engines, chunked (fits) and
    queued (does not): the same waveforms as the codec on SpeechLM's own guided generation of the template prompts."""
    from tests.helpers import _tts

    for max_batch, n in ((4, 2), (3, 4)):
        tts, _ = _tts(max_batch=max_batch, seed=5)
        refs = [torch.arange(10 + 3 * i, dtype=torch.int32) for i in range(n)]
        rts, texts = [f"reference {i}" for i in range(n)], [f"say {i}" for i in range(n)]
        scales = [2.0, 1.0, 3.0, 1.5][:n]
        negs = ["", None, "other words", None][:n]
        wavs = tts.infer_batch(texts, refs, rts, guidance_scale=scales, negative_text=negs, min_new_tokens=5)
        prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
        neg_ids = [tts._apply_chat_template(c, rt, t or "") for t, c, rt in zip(negs, refs, rts)]
        eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
        gen = (tts.backbone.generate_queue if n + sum(g != 1 for g in scales) > max_batch else tts.backbone.generate_batch)(
            prompts, eos, max_length=tts.max_context, min_new_tokens=5, seed=tts.seed, slot_base=0, temperature=1.0,
            top_k=50, guidance_scale=scales, negative_prompt_ids=neg_ids)
        ref = tts._decode_codes([tts._ids_to_codes(g) for g in gen], watermark=True)
        assert len(wavs) == n and all(np.array_equal(a, b) for a, b in zip(wavs, ref)), max_batch
        tts.backbone.set_guidance(None)
