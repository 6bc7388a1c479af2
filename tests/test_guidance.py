"""Classifier-free guidance without a GPU: the float64 reference of the guided processor chain, pinned to transformers'
UnbatchedClassifierFreeGuidanceLogitsProcessor and the processors that follow it, and the host logic on stubs.

tests/test_gpu_guidance.py compares the engine with the same combination (``combine64`` there restates ``guided64``).
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from neutts_air_b200.lm import (NO_GUIDANCE, Settings, check_guidance_scale, check_guidance_table, guided_caps,
                                guided_layout, per_prompt_guidance)
from tests.sampler_ref import chain64


def ls64(x):
    x = np.asarray(x, dtype=np.float64)
    fin = np.isfinite(x)
    m = x[fin].max()
    return x - (m + np.log(np.exp(x[fin] - m).sum()))


def guided64(c_row, u_row, g):
    """The engine's combination in float64: g * (ls_c - ls_u) + ls_u, -inf where c's logit is -inf."""
    lc, lu = ls64(c_row), ls64(u_row)
    with np.errstate(invalid="ignore"):
        out = g * (lc - lu) + lu
    out[~np.isfinite(np.asarray(c_row, dtype=np.float64))] = -np.inf
    return out


def chain_after(scores, hist, penalty, ngen, eos, min_new, decay, T, k, top_p, min_p):
    """Everything after the combine, in the engine's order: penalty, EOS mask, length decay, 1/T, top-k, top-p, min-p."""
    s = np.array(scores, dtype=np.float64)
    for t in set(hist):
        s[t] = s[t] * penalty if s[t] < 0 else s[t] / penalty
    if ngen < min_new:
        s[eos] = -np.inf
    if decay is not None and ngen > decay[0]:
        s[eos] = s[eos] + abs(s[eos]) * (decay[1] ** (ngen - decay[0]) - 1)
    return chain64(s / T, k, top_p, min_p)


def tiny_qwen2(V=300, seed=0):
    from transformers import Qwen2Config, Qwen2ForCausalLM

    torch.manual_seed(seed)
    cfg = Qwen2Config(vocab_size=V, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=256, tie_word_embeddings=False)
    m = Qwen2ForCausalLM(cfg).double().eval()
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0.0, 0.2)
    return m


@pytest.mark.parametrize("negative", [True, False])
def test_reference_matches_transformers(negative):
    """transformers' guidance processor over forced continuations, followed by its repetition penalty, min-new-tokens,
    exponential decay, temperature, top-k, top-p and min-p: the float64 reference gives the same rows and windows."""
    from transformers.generation.logits_process import (ExponentialDecayLengthPenalty, MinNewTokensLengthLogitsProcessor,
                                                        MinPLogitsWarper, RepetitionPenaltyLogitsProcessor,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper,
                                                        UnbatchedClassifierFreeGuidanceLogitsProcessor)

    V, eos = 300, 299
    m = tiny_qwen2(V)
    rng = np.random.default_rng(1)
    prompt = rng.integers(0, V - 1, 17).tolist()
    neg = rng.integers(0, V - 1, 9).tolist() if negative else None
    forced = rng.integers(0, V - 1, 12).tolist()
    g, pen, T, k, top_p, min_p, min_new, decay = 2.5, 1.3, 0.8, 40, 0.9, 0.02, 3, (5, 1.2)
    cfg = UnbatchedClassifierFreeGuidanceLogitsProcessor(g, m, torch.tensor([neg]) if negative else None)
    rest = [RepetitionPenaltyLogitsProcessor(pen), MinNewTokensLengthLogitsProcessor(len(prompt), min_new, eos),
            ExponentialDecayLengthPenalty(decay, eos, len(prompt)), TemperatureLogitsWarper(T), TopKLogitsWarper(k),
            TopPLogitsWarper(top_p), MinPLogitsWarper(min_p)]
    u_seq = list(neg) if negative else [prompt[-1]]
    checked = 0
    with torch.no_grad():
        for t in range(len(forced)):
            ids = torch.tensor([prompt + forced[:t]])
            x = m(ids).logits[:, -1]
            hf = cfg(ids, x.clone())
            u_row = m(torch.tensor([u_seq])).logits[0, -1].numpy()
            ref = guided64(x[0].numpy(), u_row, g)
            assert np.abs(hf[0].numpy() - ref).max() < 1e-10, t
            y = hf
            for p in rest:
                y = p(ids, y)
            probs = torch.softmax(y, -1)[0].numpy()
            wid, q, margin = chain_after(ref, prompt + forced[:t], pen, t, eos, min_new, decay, T, k, top_p, min_p)
            u_seq.append(forced[t])
            if margin < 1e-6:
                continue
            assert sorted(wid.tolist()) == np.nonzero(probs > 0)[0].tolist(), t
            assert np.abs(probs[wid] - q).max() < 1e-10, t
            checked += 1
    assert checked >= 8, checked


def test_vocabulary_range_orders():
    """With every id outside a range suppressed: transformers with the suppression before the guidance processor and
    after it, and the engine (both rows restricted to the range), give rows that differ by a per-row constant on the
    allowed ids, so softmax and every warper agree; the penalty and the decay would see the shift."""
    from transformers.generation.logits_process import SuppressTokensLogitsProcessor

    rng = np.random.default_rng(3)
    V, lo, hi, eos, g = 512, 128, 384, 511, 3.0
    c, u = rng.normal(0, 3, V), rng.normal(0, 3, V)
    allowed = np.zeros(V, dtype=bool)
    allowed[lo:hi] = True
    allowed[eos] = True
    sup = SuppressTokensLogitsProcessor(np.nonzero(~allowed)[0].tolist(), device="cpu")
    ct = torch.from_numpy(c)[None]
    # suppression first: transformers' processor takes c's suppressed row and u's full row (it runs the model itself)
    before = g * (torch.log_softmax(sup(None, ct.clone()), -1) - torch.log_softmax(torch.from_numpy(u)[None], -1))
    before = (before + torch.log_softmax(torch.from_numpy(u)[None], -1))[0].numpy()
    after = sup(None, torch.from_numpy(guided64(c, u, g))[None])[0].numpy()
    cr, ur = np.where(allowed, c, -np.inf), np.where(allowed, u, -np.inf)
    engine = guided64(cr, ur, g)
    for other in (before, after):
        assert np.array_equal(np.isfinite(other), allowed) and np.array_equal(np.isfinite(engine), allowed)
        d = engine[allowed] - other[allowed]
        assert np.ptp(d) < 1e-9
        pe, po = np.exp(engine[allowed] - engine[allowed].max()), np.exp(other[allowed] - other[allowed].max())
        assert np.abs(pe / pe.sum() - po / po.sum()).max() < 1e-12
    assert abs(np.mean(engine[allowed] - before[allowed])) > 1e-3   # a real shift, not zero


def test_scale_and_table_validation():
    assert check_guidance_scale(3) == 3.0 and check_guidance_scale(1.0) == 1.0
    assert check_guidance_scale(1 + 1e-9) == 1.0            # 1 in fp32: no guidance, as the library would store it
    for bad in (0, -1.0, float("inf"), float("nan"), "2", True, None):
        with pytest.raises(ValueError):
            check_guidance_scale(bad)
    ok = [(2, 2.0), (-1, 1.0), (-1, 7.0), (-1, 1.0)]
    assert check_guidance_table(ok, 4) == ok
    for bad in ([(0, 2.0)] + [NO_GUIDANCE] * 3, [(4, 2.0)] + [NO_GUIDANCE] * 3, [(-2, 2.0)] + [NO_GUIDANCE] * 3,
                [(2, 2.0), (2, 3.0), NO_GUIDANCE, NO_GUIDANCE], [(2, 2.0), NO_GUIDANCE, (3, 2.0), NO_GUIDANCE],
                [(2, 1.0)] + [NO_GUIDANCE] * 3, [(2, 0.0)] + [NO_GUIDANCE] * 3, [(2, 2.0)] * 1):
        with pytest.raises(ValueError):
            check_guidance_table(bad, 4)


def test_per_prompt_guidance_and_layout():
    prompts = [[5, 6, 7], [8, 9], [1], [2, 3]]
    assert per_prompt_guidance(prompts, 1.0, None) is None
    assert per_prompt_guidance(prompts, 1.0, [[1]] * 4) is None
    gd = per_prompt_guidance(prompts, [2.0, 1.0, 3.0, 1.0], [None, [4], [9, 9], None])
    assert gd == [(2.0, [7]), (1.0, None), (3.0, [9, 9]), (1.0, None)]   # default: the prompt's last token
    assert guided_layout(4, gd) == [(0, 4, 2.0), (2, 5, 3.0)]          # prompts keep their slots, u slots above
    assert guided_caps([10, 10, 10, 10], gd, 12) == [10, 10, 10, 10]
    assert guided_caps([10, 10, 10, 10], [(2.0, [1] * 5)] + gd[1:], 12) == [7, 10, 10, 10]
    with pytest.raises(ValueError):
        guided_caps([10] * 4, [(2.0, [1] * 12)] + gd[1:], 12)          # no room left for the pair
    with pytest.raises(ValueError):
        per_prompt_guidance(prompts, 2.0, [[], None, None, None])      # empty negative prompt
    with pytest.raises(ValueError):
        per_prompt_guidance(prompts, [2.0, 1.0], None)                 # one scale per prompt
    with pytest.raises(ValueError):
        per_prompt_guidance(prompts, 2.0, [[1]])                       # one negative prompt per prompt


class Recorder:
    """The settings mirrors of SpeechLM, recording every setter call."""

    max_batch = 8

    def __init__(self):
        self.calls = []
        self._slot_sp_host = self._vocab_range = self._penalty_host = self._length_host = None
        self._guidance_host = None
        self.logprobs = None

    def __getattr__(self, name):
        if not name.startswith("set_"):
            raise AttributeError(name)

        def rec(*a, **kw):
            self.calls.append((name, a, kw))
            if name == "set_guidance":
                self._guidance_host = a[0]
        return rec


def test_settings_apply_and_pair():
    off = Settings(None, None, None, 1.0, 50)
    lm = Recorder()
    off.apply(lm, 4)
    assert lm.calls == []                                     # guidance off: no call at all
    st = Settings([(1.0, 50, 1.0, 0.0), (0.5, 20, 1.0, 0.0)], [(1.2, True), (1.0, True)], None, 1.0, 50,
                  length=[(3, 2, 1.0), (0, 0, 1.0)])
    paired = st.pair([(1, 2, 2.0)])
    assert paired.controls[2] == st.controls[1] and paired.penalty[2] == st.penalty[1] and paired.length[2] == st.length[1]
    assert paired.guidance == [NO_GUIDANCE, (2, 2.0), NO_GUIDANCE]
    paired.apply(lm, 3)
    assert lm.calls[-1] == ("set_guidance", ([NO_GUIDANCE, (2, 2.0)] + [NO_GUIDANCE] * 6,), {})
    lm.calls.clear()
    off.apply(lm, 2)                                          # a later call without guidance switches it off
    assert ("set_guidance", (None,), {}) in lm.calls
    assert st.pair([]) is st


def test_admit_writes_pair_entries():
    lm = Recorder()
    st = Settings(None, None, None, 1.0, 50)
    st.admit(lm, [3, 5], [7, 7], guide={3: (5, 2.0), 5: NO_GUIDANCE, 1: NO_GUIDANCE})
    assert lm.calls == [("set_guidance", ([(5, 2.0), NO_GUIDANCE, NO_GUIDANCE],), {"slots": [3, 5, 1]})]


# ---------------------------------------------------------------------------------------------- engine host on stubs
from tests.fakes import EOS, FakeTokenizer, GenerateBackbone, GuidedStub, KwBackbone, _facade  # noqa: E402


def _negs(lens):
    return [[-(i + 1)] * m for i, m in enumerate(lens)]


def test_queue_admits_pairs_fifo_with_their_negative_prompts():
    lens = [90, 80, 95, 70, 60, 85, 75]
    caps = [100 - m for m in lens]
    scales = [2.0, 1.0, 3.0, 3.0, 1.0, 2.0, 1.5]
    negs = _negs([5] * 7)
    lm = GuidedStub(4)
    out = lm.generate_queue(_prompts_tagged(lens), EOS, max_length=100, min_new_tokens=100, check_every=8, slot_base=40,
                            guidance_scale=scales, negative_prompt_ids=negs)
    assert [o.tolist() for o in out] == [[1000 * (i + 1) + g for g in range(c)] for i, c in enumerate(caps)]
    # first wave: prompts 0 (+u), 1, and prompt 2 would need two more slots: it waits (FIFO), nothing overtakes it
    assert lm.log[1][0] == "guide" and lm.log[2] == ("prefill", [1, 2, -1])
    assert lm.log[1][1][0] == (2, 2.0) and lm.log[1][1][1:] == [NO_GUIDANCE] * 3
    refills = [e for e in lm.log if e[0] == "refill"]
    tags = [t for e in refills for t in e[2] if t > 0]
    assert tags == sorted(tags) == [3, 4, 5, 6, 7]
    for e in refills:
        slots, got = e[1], e[2]
        guide = next(x for x in reversed(lm.log[: lm.log.index(e)]) if x[0] == "guide")[1]
        for s, t in zip(slots, got):
            if t > 0 and scales[t - 1] != 1.0:
                u = guide[s][0]
                assert guide[s][1] == scales[t - 1] and u in slots and got[slots.index(u)] == -t   # its own negative
            elif t > 0:
                assert guide[s] == NO_GUIDANCE
        assert e[3] == [40 + abs(t) - 1 for t in got]                # both slots of a pair: the prompt's stream key
        assert e[4] == [caps[abs(t) - 1] for t in got]
    assert sorted(lm.pool.free) == list(range(lm.num_pages))


def _prompts_tagged(lens):
    return [[i + 1] * m for i, m in enumerate(lens)]


def test_batch_layout_keeps_unguided_stream_keys():
    lm = GuidedStub(6)
    out = lm.generate_batch(_prompts_tagged([10, 12, 9, 11]), EOS, max_length=30, min_new_tokens=100, slot_base=7,
                            guidance_scale=[1.0, 2.0, 1.0, 4.0], negative_prompt_ids=_negs([3] * 4))
    assert [o.tolist()[:2] for o in out] == [[1000 * (i + 1), 1000 * (i + 1) + 1] for i in range(4)]
    assert ("prefill", [1, 2, 3, 4, -2, -4]) in lm.log            # prompts in slots 0..3, u slots 4 and 5 above
    assert lm.u_at == {4: 2, 5: 4}                                # keys checked by the stub: slot_base + slot
    guide = [e for e in lm.log if e[0] == "guide"][-1][1]
    assert guide[:6] == [NO_GUIDANCE, (4, 2.0), NO_GUIDANCE, (5, 4.0), NO_GUIDANCE, NO_GUIDANCE]
    with pytest.raises(ValueError):                               # 5 prompts + 2 guided > 6 slots
        lm.generate_batch(_prompts_tagged([4] * 5), EOS, guidance_scale=[2.0, 2.0, 1.0, 1.0, 1.0])
    with pytest.raises(ValueError):
        lm.generate_batch(_prompts_tagged([4] * 2), EOS, guidance_scale=2.0, num_return_sequences=2)


def test_guidance_off_call_log():
    """Without guidance, generate_batch and generate_queue make no guidance call and the same prefill/decode calls
    as a run that never heard of guidance (the parent's sequence: sampling, prefill, decode...)."""
    for run in ("batch", "queue"):
        lm = GuidedStub(3)
        f = lm.generate_batch if run == "batch" else lm.generate_queue
        f(_prompts_tagged([90, 80, 95]), EOS, max_length=100, min_new_tokens=100, check_every=8, slot_base=2)
        assert not any(e[0] == "guide" for e in lm.log)
        assert [e[0] for e in lm.log][:2] == ["sampling", "prefill"] and lm.log[1] == ("prefill", [1, 2, 3])
        assert all(e[0] == "decode" for e in lm.log[2:])


def test_generate_negative_rows_and_mask():
    from neutts_air_b200.lm import SpeechLM

    lm = SpeechLM.__new__(SpeechLM)
    seen = []
    lm.generate_batch = lambda prompts, eos, *a, **kw: seen.append(kw) or [torch.tensor([eos])] * len(prompts)
    ids = torch.tensor([[5, 6, 7], [8, 9, 10]])
    lm.generate(ids, eos_token_id=1, guidance_scale=2.0, negative_prompt_ids=torch.tensor([[3, 4]]), seed=0)
    assert seen[-1]["guidance_scale"] == 2.0 and seen[-1]["negative_prompt_ids"] == [[3, 4], [3, 4]]   # one row: all
    lm.generate(ids, eos_token_id=1, guidance_scale=2.0, negative_prompt_ids=torch.tensor([[3, 4], [1, 2]]), seed=0)
    assert seen[-1]["negative_prompt_ids"] == [[3, 4], [1, 2]]
    lm.generate(ids, eos_token_id=1, guidance_scale=2.0, seed=0,
                negative_prompt_attention_mask=torch.ones(1, 2, dtype=torch.long))
    assert seen[-1]["negative_prompt_ids"] is None                # the engine's default: each prompt's last token
    for off in (None, 1.0):
        lm.generate(ids, eos_token_id=1, guidance_scale=off, negative_prompt_ids=torch.tensor([[3]]), seed=0)
        assert "guidance_scale" not in seen[-1]
    with pytest.raises(ValueError):
        lm.generate(ids, eos_token_id=1, guidance_scale=2.0, negative_prompt_ids=torch.tensor([[3, 4]]),
                    negative_prompt_attention_mask=torch.tensor([[0, 1]]), seed=0)
    with pytest.raises(ValueError):
        lm.generate(ids, eos_token_id=1, guidance_scale=2.0, negative_prompt_ids=torch.ones(3, 2, dtype=torch.long), seed=0)


# ---------------------------------------------------------------------------------------------------- facade on stubs
def test_facade_forwards_guidance_and_builds_negative_prompts():
    tok = FakeTokenizer()
    bb = KwBackbone(tok, queue=False)
    tts = _facade(bb, 3)
    refs, rts = [[1, 2], [3], [4, 5]], ["a", "b", "c"]
    tts.infer_batch(["x", "y", "z"], refs, rts)
    assert all("guidance_scale" not in kw and "negative_prompt_ids" not in kw for _, _, kw in bb.calls)   # off: as today
    bb.calls.clear()
    tts.infer_batch(["x", "y", "z"], refs, rts, guidance_scale=[2.0, 1.0, 3.0], negative_text=["no", None, None])
    # 3 prompts + 2 guided need 5 slots of 3: chunks [0, 1] and [2] (slot_base 0 and 2)
    assert [(n, kw["slot_base"]) for _, n, kw in bb.calls] == [(2, 0), (1, 2)]
    kw0, kw1 = bb.calls[0][2], bb.calls[1][2]
    assert kw0["guidance_scale"] == [2.0, 1.0] and kw1["guidance_scale"] == [3.0]
    assert kw0["negative_prompt_ids"][0] == tts._apply_chat_template(refs[0], "a", "no")
    assert kw1["negative_prompt_ids"][0] == tts._apply_chat_template(refs[2], "c", "")   # None: the voice alone
    bb.calls.clear()
    tts.infer("x", refs[0], "a", guidance_scale=2.0)
    assert bb.calls[0][2]["negative_prompt_ids"] == [tts._apply_chat_template(refs[0], "a", "")]
    bb.calls.clear()
    tts.infer_from_prompt_ids([[7, 8], [9]], guidance_scale=1.5, negative_prompt_ids=[[1], None])
    assert bb.calls[0][2]["guidance_scale"] == 1.5 and bb.calls[0][2]["negative_prompt_ids"] == [[1], None]
    qb = KwBackbone(tok, queue=True)
    tq = _facade(qb, 3)
    tq.infer_batch(["x", "y"], refs[:2], rts[:2], guidance_scale=2.0)    # 4 slots > 3: the queue takes them
    assert qb.calls[0][0] == "queue" and qb.calls[0][1] == 2


def test_facade_injected_transformers_backbone_receives_guidance():
    tok = FakeTokenizer()
    bb = GenerateBackbone(tok)
    tts = _facade(bb, 2)
    tts.infer_batch(["x", "y"], [[1], [2]], ["a", "b"])
    assert all("guidance_scale" not in kw and "negative_prompt_ids" not in kw for kw in bb.kws)
    bb.kws.clear()
    tts.infer_batch(["x", "y"], [[1], [2]], ["a", "b"], guidance_scale=[3.0, 1.0], negative_text="n")
    assert bb.kws[0]["guidance_scale"] == 3.0
    assert bb.kws[0]["negative_prompt_ids"].tolist() == [tts._apply_chat_template([1], "a", "n")]
    assert "guidance_scale" not in bb.kws[1] and "negative_prompt_ids" not in bb.kws[1]
    bb.kws.clear()
    tts.infer_from_prompt_ids([[4, 5]], guidance_scale=2.0)             # default negative prompt: not passed
    assert bb.kws[0]["guidance_scale"] == 2.0 and "negative_prompt_ids" not in bb.kws[0]


def test_facade_refuses_guidance_where_unsupported():
    tok = FakeTokenizer()
    tts = _facade(KwBackbone(tok), 4)
    with pytest.raises(ValueError):
        tts.infer_stream("x", [1], "a", guidance_scale=2.0)
    with pytest.raises(ValueError):
        tts.infer_stream_batch(["x"], [[1]], ["a"], guidance_scale=[2.0])
    with pytest.raises(ValueError):
        tts.infer_batch(["x"], [[1]], ["a"], guidance_scale=2.0, takes=2)
    with pytest.raises(ValueError):
        tts.infer_batch(["x"], [[1]], ["a"], guidance_scale=0.0)
