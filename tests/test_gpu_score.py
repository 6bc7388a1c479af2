"""GPU: teacher-forced scoring (``nt_lm_score`` / ``SpeechLM.score`` / ``NeuTTS.score``).

  * exact logits: on the logit-programmable model of sampler_ref.py the lm_head input of every scored row is one
    bf16 value on one pattern's column, so each row's logits are known exactly and the scores are checked against a
    float64 log-softmax of them, at a vocabulary with a partial last tile and at the Air vocabulary, across the row-block
    boundary of the lm_head;
  * a random 3-layer model against the oracle with the scoring path's rounding points (``mirror="batched"``), against
    the unrounded float64 reference and against transformers' ``labels=`` loss;
  * invariance: a sequence's scores are bit-identical alone, in a batch, in another order, in a second call, and with
    every sampling setting switched on;
  * agreement with the ``model`` log-probabilities of generation on the three decode paths;
  * the engine state a call leaves, the Air shape, and the facade.

BARS lists the worst values measured on one H100 80GB HBM3 (700 W power limit) and the bars, about 4x above them.
"""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import make_lm
from tests.sampler_ref import PATTERNS_ALL, programmable, score64

pytestmark = pytest.mark.gpu

# worst |score - reference| measured on the H100 -> bar
BARS = {
    "exact": 5e-5,          # 2.1e-6: programmable model against float64 log-softmax of its exact logits
    "mirror": 6e-2,         # 1.4e-2: random 3-layer model against the oracle with the scoring path's rounding points
    "unrounded": 8e-2,      # 1.8e-2: ... against the float64 reference without them (bf16 operands)
    "loss": 3e-2,           # 7.2e-3: ... -mean against transformers' labels= loss
    "generation": 7e-2,     # 1.7e-2: against the `model` column of generation (decode vs prefill rounding)
    "air": 6e-2,            # 1.5e-2: Air shape against the oracle with the scoring path's rounding points
}
SMALL = dict(vocab_size=4096, hidden_size=256, intermediate_size=640, num_layers=3, num_heads=4, num_kv_heads=2)


def _worst(got, ref) -> float:
    got = np.asarray(got, dtype=np.float64)
    if not np.isfinite(got).all():
        return float("inf")
    return float(np.abs(got - np.asarray(ref, dtype=np.float64)).max())


# ====================================================================================== exact logits
def _pattern_sequences(m, n_long: int):
    """Sequences whose scored rows walk every pattern, with targets at the pattern's winners, ties, V - 1, V - 2, EOS,
    one id per tile edge and random ids; the first one is n_long tokens long."""
    rng = np.random.default_rng(7)
    V = m.V
    seqs = []
    for j, name in enumerate(PATTERNS_ALL):
        row = m.target[j]
        top = np.argsort(-row, kind="stable")[:6].tolist()
        targets = top + [V - 1, V - 2, m.eos, 127, 128, V - (V % 128 or 128)] + rng.integers(0, V, 6).tolist()
        seq = []
        for n, t in enumerate(targets):
            seq += [m.token_for(name, n), int(t)]
        seqs.append(seq)
    long = rng.integers(0, V, n_long).tolist()
    return [long] + seqs


def _exact_scores(m, seq, start):
    xs_b = float(torch.tensor(m.xs, dtype=torch.float32).bfloat16())   # the bf16 lm_head input of every row
    out = []
    for t in range(start, len(seq)):
        z = xs_b * m.W[m.pattern_of(seq[t - 1])].numpy()
        z = z - z.max()
        out.append(z[seq[t]] - np.log(np.exp(z).sum()))
    return np.asarray(out)


@pytest.mark.parametrize("V", [4142, 217472])
def test_score_exact_logits(cuda, V):
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=4, max_ctx=1088, max_prefill_tokens=2048)
    seqs = _pattern_sequences(m, 1030)            # 1029 scored rows: the lm_head runs blocks of 1024 + 5 rows
    starts = [1] + [1 + (i % 3) for i in range(len(seqs) - 1)]
    got = lm.score(seqs, starts)
    worst = 0.0
    for s, st, g in zip(seqs, starts, got):
        assert g.shape == (len(s) - st,)
        worst = max(worst, _worst(g, _exact_scores(m, s, st)))
    print(f"SCORE exact logits V={V}: worst |err| {worst:.2e}")
    assert worst < BARS["exact"], worst


# ====================================================================================== random 3-layer model
@pytest.fixture(scope="module")
def small(cuda):
    cfg = O.LMConfig.tiny(**SMALL)
    w = O.random_weights(cfg, 21, std=0.05, bf16_round=True)
    return cfg, w, make_lm(cfg, w, max_batch=17, max_ctx=512, max_prefill_tokens=2048, max_new=128)


def _seqs(n, seed, lo=20, hi=200):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(lo, hi, (n,), generator=g).tolist()
    return [torch.randint(0, SMALL["vocab_size"], (L,), generator=g).tolist() for L in lens]


def test_score_random_model_against_oracle(small):
    cfg, w, lm = small
    seqs = _seqs(6, 1)
    starts = [1, 5, len(seqs[2]) - 1, 30, 2, 11]
    got = lm.score(seqs, starts)
    w_mirror = w_unr = w_loss = 0.0
    model = None
    try:
        model = O.to_hf_model(cfg, w, attn_implementation="sdpa").double()
    except ImportError:
        pass
    for s, st, g in zip(seqs, starts, got):
        ids = torch.tensor(s)
        logits, _ = O.forward(cfg, w, ids, mirror="batched")
        lp = torch.log_softmax(logits.double(), -1)
        t = torch.arange(st, len(s))
        w_mirror = max(w_mirror, _worst(g, lp[t - 1, ids[t]]))
        ref64 = score64(cfg, w, ids, st)
        w_unr = max(w_unr, _worst(g, ref64))
        if model is not None:
            labels = ids.clone()
            labels[:st] = -100
            with torch.no_grad():
                loss = float(model(ids[None], labels=labels[None]).loss)
            w_loss = max(w_loss, abs(-float(g.double().mean()) - loss))
    print(f"SCORE random model: worst |err| vs mirror {w_mirror:.2e}, vs float64 {w_unr:.2e}, mean vs HF loss {w_loss:.2e}")
    assert w_mirror < BARS["mirror"] and w_unr < BARS["unrounded"] and w_loss < BARS["loss"], (w_mirror, w_unr, w_loss)


def test_score_invariance(small):
    cfg, w, lm = small
    seqs = _seqs(7, 2)
    starts = [3, 1, 9, 4, 17, 2, 6]
    alone = lm.score(seqs[3:4], starts[3:4])[0]
    batch = lm.score(seqs, starts)
    rev = lm.score(seqs[::-1], starts[::-1])
    again = lm.score(seqs, starts)
    for i in range(7):
        assert torch.equal(batch[i], rev[6 - i]) and torch.equal(batch[i], again[i]), i
    assert torch.equal(alone, batch[3])
    # every sampling setting on: the scores are the model's alone
    lm.set_repetition_penalty([(1.7, True)] * lm.max_batch)
    lm.set_vocab_range(128, 1024)
    lm.set_slot_sampling([(0.5, 7, 0.8, 0.1)] * lm.max_batch)
    lm.set_logprobs(True)
    try:
        on = lm.score(seqs, starts)
    finally:
        lm.set_repetition_penalty(None)
        lm.set_vocab_range(None)
        lm.set_slot_sampling(None)
        lm.set_logprobs(False)
    for i in range(7):
        assert torch.equal(on[i], batch[i]), i


@pytest.mark.parametrize("B", [1, 8, 17])   # persistent kernel (FOLD at batch 1), persistent kernel, per-op chain
def test_score_agrees_with_generation(small, B):
    cfg, w, lm = small
    prompts = _seqs(B, 10 + B, 10, 120)
    ids, lps = lm.generate_batch(prompts, cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=40, seed=B, top_k=50,
                                 return_logprobs=True)
    full = [p + g.tolist() for p, g in zip(prompts, ids)]
    keep = [i for i, g in enumerate(ids) if len(g) >= 1]
    got = lm.score([full[i] for i in keep], [len(prompts[i]) for i in keep])
    worst = max(_worst(got[k], lps[i][:, 1]) for k, i in enumerate(keep))
    print(f"SCORE vs generation B={B}: worst |err| {worst:.2e} over {sum(len(ids[i]) for i in keep)} tokens")
    assert worst < BARS["generation"], worst


def test_score_engine_state(small):
    cfg, w, lm = small
    eos = cfg.vocab_size - 1
    lm.set_logprobs(True)
    try:
        sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8, seed=3)
        lm.prefill(_seqs(3, 4), sp)
        lm.decode(4, sp)
        torch.cuda.synchronize()
        before = (lm.out_tokens.clone(), lm.logprobs.clone(), lm.cur_token.clone())
        seqs = _seqs(3, 5)
        lm.score(seqs, 2)
        torch.cuda.synchronize()
        assert torch.equal(lm.out_tokens, before[0]) and torch.equal(lm.logprobs, before[1])
        assert torch.equal(lm.cur_token, before[2])
        assert lm.seq_lens[:3].tolist() == [len(s) for s in seqs] and lm.seq_lens[3:].abs().sum() == 0
        assert int(lm.n_generated.abs().sum()) == 0 and bool((lm.done == 1).all())
        assert lm.pool.num_free == lm.num_pages
        with pytest.raises(RuntimeError, match="before nt_lm_prefill"):
            lm.decode(1, sp)
        with pytest.raises(RuntimeError, match="before nt_lm_prefill"):
            lm.prefill_slots([0], [[1, 2, 3]], sp, stream_ids=[0])
        lm.prefill(_seqs(2, 6), sp)       # a new prefill makes the engine decode again
        lm.decode(2, sp)
        torch.cuda.synchronize()
        assert int(lm.n_generated[:2].min()) >= 1
    finally:
        lm.set_logprobs(False)
        lm.release_pages()
    with pytest.raises(ValueError, match="start"):
        lm.score([[1, 2, 3]], 3)
    with pytest.raises(ValueError, match="out of range"):
        lm.score([[1, cfg.vocab_size]], 1)
    with pytest.raises(ValueError, match="sequence 0"):
        lm.score([list(range(600))], 1)


def test_score_facade_matches_engine(small):
    import warnings

    from neutts import NeuTTS
    from tests.fakes import FakeCodec, FakePhonemizer, FakeTokenizer

    cfg, w, lm = small
    tok = FakeTokenizer()
    tok.speech_base, tok.special_base = 1000, 900   # ids inside the tiny vocabulary
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=lm, codec=FakeCodec(), max_batch=17, seed=1)
    tts._n_codes = lambda: 3000
    codes = [[5, 17, 2999, 0], [44]]
    got = tts.score_batch(["hello", "a b"], [[1, 2], [3]], ["ref", "x"], codes)
    prompts = [tts._apply_chat_template(c, r, t) for t, c, r in (("hello", [1, 2], "ref"), ("a b", [3], "x"))]
    sge = tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>")
    want = lm.score([p + [1000 + c for c in cs] + [sge] for p, cs in zip(prompts, codes)], [len(p) for p in prompts])
    for g, wv, cs in zip(got, want, codes):
        assert g.shape == (len(cs) + 1,) and np.array_equal(g, wv.numpy())
    one = tts.score("hello", [1, 2], "ref", codes[0], include_eos=False)
    assert np.array_equal(one, got[0][:-1])


# ====================================================================================== Air shape
def test_score_air_shape(cuda):
    from neutts_air_b200 import synthetic
    from neutts_air_b200.lm import LMShape, SpeechLM

    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 0)
    lm = SpeechLM(shape, sd, device="cuda:0", max_batch=2, max_ctx=1024, max_new=16, max_prefill_tokens=1600)
    g = torch.Generator().manual_seed(9)
    seq = torch.randint(0, shape.vocab_size, (750,), generator=g).tolist()
    got = lm.score([seq], 500)[0]
    del lm
    cfg = O.LMConfig()
    f = lambda k: sd[k].float().cuda()
    layers = [dict(ln1=f(p + "input_layernorm.weight"), wq=f(p + "self_attn.q_proj.weight"), bq=f(p + "self_attn.q_proj.bias"),
                   wk=f(p + "self_attn.k_proj.weight"), bk=f(p + "self_attn.k_proj.bias"), wv=f(p + "self_attn.v_proj.weight"),
                   bv=f(p + "self_attn.v_proj.bias"), wo=f(p + "self_attn.o_proj.weight"), ln2=f(p + "post_attention_layernorm.weight"),
                   wg=f(p + "mlp.gate_proj.weight"), wu=f(p + "mlp.up_proj.weight"), wd=f(p + "mlp.down_proj.weight"))
              for p in (f"model.layers.{i}." for i in range(cfg.num_layers))]
    emb = f("model.embed_tokens.weight")
    w = O.LMWeights(embed=emb, layers=layers, final_norm=f("model.norm.weight"), lm_head=emb)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.device("cuda"):
            ids = torch.tensor(seq)
            logits, _ = O.forward(cfg, w, ids, mirror="batched")
            t = torch.arange(500, 750)
            ref = torch.log_softmax(logits[t - 1].double(), -1)[torch.arange(250), ids[t]].cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    worst = _worst(got, ref)
    print(f"SCORE Air shape (500 + 250 tokens): worst |err| {worst:.2e}, mean score {float(got.double().mean()):.3f}")
    assert worst < BARS["air"], worst
