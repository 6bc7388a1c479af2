"""GPU parity of the speech-LM path (prefill + decode + sampler state machine) against the CPU oracle.

Two oracles, both on the same bf16-valued weights:
  * "mirrored"  = oracle/lm_oracle.py with the rounding points DESIGN.md lists for the CUDA path
                  (bf16 KV cache; bf16 GEMM A-operands in the tensor-core path);
  * "reference" = the pure fp32 semantics of transformers Qwen2 (what the reference runs).
bf16 rounding points make the comparison chaotic at the 2^-9 level — one flipped rounding of a GEMM
input element shifts a whole output row — so the bars are stated as relative RMS error plus a max
error in units of the logit spread (see _check_logits); the decode path, which keeps fp32
activations, is held to 1e-3 relative RMS.
"""
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import make_lm, max_err, rel_err, set_decode_impl

pytestmark = pytest.mark.gpu

SMALL = dict(vocab_size=4096, hidden_size=256, intermediate_size=640, num_layers=3, num_heads=4, num_kv_heads=2)
# full NeuTTS-Air widths, fewer layers and a smaller vocabulary so the CPU oracle finishes in seconds
WIDE = dict(vocab_size=8192, hidden_size=896, intermediate_size=4864, num_layers=2, num_heads=14, num_kv_heads=2)


def _setup(cfgkw, seed, std=0.05, **lmkw):
    cfg = O.LMConfig.tiny(**cfgkw)
    w = O.random_weights(cfg, seed, std=std, bf16_round=True)
    lm = make_lm(cfg, w, **lmkw)
    return cfg, w, lm


def _teacher_forced(cfg, w, lm, prompts, forced, n_new, eos):
    """Run prefill + n_new-1 decode steps with teacher-forced tokens; return per-step logits [B][n_new, V]."""
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=n_new, forced=forced)
    l0 = lm.prefill(prompts, sp, return_logits=True)
    ls = lm.decode(n_new - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    return torch.cat((l0[None], ls), 0).permute(1, 0, 2).cpu()       # [B, n_new, V]


def _check_logits(got, mir, ref, tag):
    """relative RMS error <= 6e-3 against the mirrored oracle and <= 2e-2 against the pure-fp32
    reference semantics; max error <= 5% / 10% of the logit spread."""
    spread = float(ref.std())
    r_m, r_r = rel_err(got, mir), rel_err(got, ref)
    m_m, m_r = max_err(got, mir) / spread, max_err(got, ref) / spread
    print(f"LOGITS-PARITY {tag}: relRMS mirrored {r_m:.2e} reference {r_r:.2e}; max/spread mirrored {m_m:.2e} reference {m_r:.2e}")
    assert r_m < 6e-3 and m_m < 5e-2, (r_m, m_m)
    assert r_r < 2e-2 and m_r < 1e-1, (r_r, m_r)


@pytest.mark.parametrize("cfgkw,P,n_new", [(SMALL, 70, 12), (WIDE, 200, 6)])
def test_lm_b1_logits_vs_oracle(cuda, cfgkw, P, n_new):
    cfg, w, lm = _setup(cfgkw, 11, max_batch=1, max_ctx=512, page_shuffle_seed=3)
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, cfg.vocab_size, (P,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, n_new), generator=g)
    eos = cfg.vocab_size - 1
    got = _teacher_forced(cfg, w, lm, [prompt.tolist()], forced, n_new, eos)[0]
    _, mir = O.generate(cfg, w, prompt, eos, max_length=512, max_new_tokens=n_new, forced=forced[0], mirror=True)
    _, ref = O.generate(cfg, w, prompt, eos, max_length=512, max_new_tokens=n_new, forced=forced[0], mirror=False)
    # step 0 comes out of the tensor-core prefill path, the rest out of the persistent decode kernel
    _check_logits(got, mir, ref, f"H{cfg.hidden_size} P{P}")
    # state machine: forced tokens were recorded, counters advanced
    assert lm.out_tokens[0, :n_new].cpu().tolist() == forced[0].tolist()
    assert int(lm.n_generated[0]) == n_new and int(lm.seq_lens[0]) == P + n_new - 1


@pytest.mark.parametrize("persistent", [True, False], ids=["persistent-kernel", "per-op-chain"])
@pytest.mark.parametrize("cfgkw", [SMALL, WIDE])
def test_lm_decode_path_tight(cuda, cfgkw, persistent, monkeypatch):
    """Both decode implementations for batch <= 4: the persistent wgmma kernel (default) and the per-op
    CUDA-core chain (NT_DECODE_IMPL=perop).  A 1-token prompt followed by 70 teacher-forced steps exercises only the
    decode kernels (fp32-grade activations, bf16 KV; crosses the 64-token page boundary): against the mirrored
    oracle the only noise left is the rare flip of a bf16 K/V rounding -> 1e-3 relative RMS."""
    set_decode_impl(monkeypatch, None if persistent else "perop")
    cfg, w, lm = _setup(cfgkw, 13, max_batch=1, max_ctx=256, page_shuffle_seed=5)
    g = torch.Generator().manual_seed(6)
    n_new, eos = 71, cfg.vocab_size - 1
    prompt = torch.randint(0, cfg.vocab_size, (1,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, n_new), generator=g)
    got = _teacher_forced(cfg, w, lm, [prompt.tolist()], forced, n_new, eos)[0]
    # the persistent wgmma kernel keeps fp32-grade activations (bf16 hi + lo pairs) but runs the attention products
    # on bf16 tensor-core operands like the prefill kernel: mirror "decode_tc"; the per-op chain is all fp32: "decode"
    _, mir = O.generate(cfg, w, prompt, eos, max_length=256, max_new_tokens=n_new, forced=forced[0], mirror=True,
                        decode_mirror="decode_tc" if persistent else None)
    r = rel_err(got, mir)
    print(f"DECODE-PATH-PARITY H{cfg.hidden_size} persistent={persistent}: relRMS {r:.2e} max {max_err(got, mir):.2e}")
    assert r < 1e-3, r


@pytest.mark.parametrize("persistent", [True, False], ids=["persistent-kernel", "per-op-chain"])
def test_lm_ragged_batch_prefill_and_decode(cuda, persistent, monkeypatch):
    """Ragged prompts packed back to back (no left padding); batch 3 decodes on the persistent wgmma kernel
    (default) or on the per-op CUDA-core chain (NT_DECODE_IMPL=perop)."""
    set_decode_impl(monkeypatch, None if persistent else "perop")
    cfg, w, lm = _setup(SMALL, 21, max_batch=4, max_ctx=256)
    g = torch.Generator().manual_seed(9)
    lens, n_new, eos = [33, 64, 7], 5, cfg.vocab_size - 1
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g) for n in lens]
    forced = torch.randint(0, cfg.vocab_size, (3, n_new), generator=g)
    got = _teacher_forced(cfg, w, lm, [p.tolist() for p in prompts], forced, n_new, eos)
    for b, p in enumerate(prompts):
        _, mir = O.generate(cfg, w, p, eos, max_length=256, max_new_tokens=n_new, forced=forced[b], mirror=True)
        assert rel_err(got[b], mir) < 6e-3 and max_err(got[b], mir) < 5e-2 * float(mir.std()), (b, rel_err(got[b], mir))


def test_lm_decode_impl_rejects_unknown_value(cuda, monkeypatch):
    """NT_DECODE_IMPL takes tc or perop; any other value, such as "mega", fails instead of silently picking a path."""
    cfg, w, lm = _setup(SMALL, 23, max_batch=1, max_ctx=128)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=4)
    lm.prefill([[1, 2, 3]], sp)
    set_decode_impl(monkeypatch, "mega")
    with pytest.raises(ValueError, match="tc and perop"):
        lm.decode(2, sp)


@pytest.mark.parametrize("B,impl", [(6, None), (10, None), (18, None), (18, "tc"), (34, "tc"), (7, "perop")],
                         ids=["persistent-b6-hilo", "persistent-b10-bf16", "chain-b18", "persistent-b18-n32", "persistent-b34-n64", "chain-b7"])
def test_lm_batched_decode(cuda, B, impl, monkeypatch):
    """Batched decode, every kernel variant: the persistent wgmma kernel with bf16 hi+lo activations (batch <= 8),
    with plain bf16 activations on N = 16 / 32 / 64 token columns (the default up to batch 16; larger batches forced
    with NT_DECODE_IMPL=tc), and the per-op chain (default from batch 17; forced at batch 7).  Prefill is the
    tensor-core path in every case, so the bar is the pure-reference one."""
    set_decode_impl(monkeypatch, impl)
    cfg, w, lm = _setup(SMALL, 31, max_batch=36, max_ctx=256)
    g = torch.Generator().manual_seed(2)
    lens = ([20, 41, 64, 65, 9, 30, 17, 80, 33, 5, 12, 70, 3, 44, 27, 90, 61, 8] * 2)[:B]
    n_new, eos = 4, cfg.vocab_size - 1
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g) for n in lens]
    forced = torch.randint(0, cfg.vocab_size, (B, n_new), generator=g)
    got = _teacher_forced(cfg, w, lm, [p.tolist() for p in prompts], forced, n_new, eos)
    for b, p in enumerate(prompts):
        _, ref = O.generate(cfg, w, p, eos, max_length=256, max_new_tokens=n_new, forced=forced[b], mirror=False)
        assert rel_err(got[b], ref) < 2e-2 and max_err(got[b], ref) < 1e-1 * float(ref.std()), (b, rel_err(got[b], ref))
    assert lm.out_tokens[:B, :n_new].cpu().tolist() == forced.tolist()
    # run-to-run reproducibility, bit for bit: concurrent instances and the split-K GEMMs (slices folded in
    # slice order by the following RMSNorm) must not introduce order-dependent sums
    again = _teacher_forced(cfg, w, lm, [p.tolist() for p in prompts], forced, n_new, eos)
    assert torch.equal(got, again)


def test_lm_generate_stops_and_graph_replay(cuda):
    """EOS handling (min_new_tokens mask, stop flag), max_length stop, CUDA-graph replay == eager."""
    cfg, w, lm = _setup(SMALL, 41, max_batch=2, max_ctx=128)
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in (30, 50)]
    eos = 7
    outs = lm.generate_batch(prompts, eos, max_length=128, min_new_tokens=5, temperature=1.0, top_k=50, seed=99)
    for o, p in zip(outs, prompts):
        assert 1 <= len(o) <= 128 - len(p)                    # max_length counts the sequence's own prompt (per-sequence cap)
        assert eos not in o[:5].tolist()                      # masked during the first min_new_tokens
        if eos in o.tolist():
            assert o.tolist().index(eos) == len(o) - 1        # nothing is emitted after EOS
    # same seed -> same tokens (Philox keyed by seed/slot/step), with and without graph replay
    outs2 = lm.generate_batch(prompts, eos, max_length=128, min_new_tokens=5, temperature=1.0, top_k=50, seed=99, check_every=1)
    assert [o.tolist() for o in outs] == [o.tolist() for o in outs2]
    # greedy decoding: every emitted token is (near-)argmax of the oracle's logits along the same path.
    # Random weights leave top-1/top-2 gaps below the bf16 noise floor now and then, so the check is
    # "oracle logit of the chosen token within 5% of the spread of the oracle maximum".
    o_greedy = lm.generate_batch(prompts[:1], eos, max_length=128, min_new_tokens=0, max_new_tokens=6, greedy=True)[0]
    assert 1 <= len(o_greedy) <= 6
    cache = O.KVCache(cfg.num_layers)
    logits, _ = O.forward(cfg, w, torch.tensor(prompts[0]), cache, mirror="prefill")
    for t in o_greedy.tolist():
        row = logits[-1]
        assert float(row.max() - row[t]) < 5e-2 * float(row.std()), (t, int(row.argmax()))
        logits, _ = O.forward(cfg, w, torch.tensor([t]), cache, mirror="decode")


def test_hf_generate_seam(cuda):
    """The transformers-style .generate() the facade calls (neutts/neutts.py:338-347)."""
    cfg, w, lm = _setup(SMALL, 51, max_batch=1, max_ctx=128)
    prompt = torch.arange(40)[None]
    out = lm.generate(prompt, max_length=128, eos_token_id=3, do_sample=True, temperature=1.0, top_k=50,
                      use_cache=True, min_new_tokens=10, seed=1)
    assert out.shape[0] == 1 and out.shape[1] > 40 + 10 - 1 and out.shape[1] <= 128
    assert out[0, :40].tolist() == list(range(40))
    with pytest.raises(ValueError):
        lm.generate(torch.arange(200)[None], max_length=128, eos_token_id=3)


def _kv_rows(lm, layer, which, b, T):
    """K or V of slot b, positions 0..T-1, gathered through the page table -> [T, n_kv, 64] fp32."""
    table = lm.page_table[b].cpu().tolist()
    pages = torch.stack([lm.kv[layer, which, table[t // 64], :, t % 64, :] for t in range(T)])
    return pages.float().cpu()


@pytest.mark.parametrize("cfgkw,P", [(SMALL, 70), (WIDE, 130)])
def test_lm_prefill_stages_vs_oracle(cuda, cfgkw, P):
    """Per-stage parity of the tensor-core prefill path, layer by layer (SURVEY.md §7 step 2):
    q after RoPE, cached K/V, attention output, SwiGLU output, residual stream."""
    cfg, w, lm = _setup(cfgkw, 61, max_batch=1, max_ctx=256, page_shuffle_seed=1)
    g = torch.Generator().manual_seed(8)
    prompt = torch.randint(0, cfg.vocab_size, (P,), generator=g)
    col = {}
    O.forward(cfg, w, prompt, O.KVCache(cfg.num_layers), mirror="prefill", collect=col)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=4)
    errs = {}
    HD, I, H = cfg.num_heads * 64, cfg.intermediate_size, cfg.hidden_size
    for nl in range(1, cfg.num_layers + 1):
        lm.debug_set_layers(nl)
        lm.prefill([prompt.tolist()], sp)
        torch.cuda.synchronize()
        o, li = col[nl - 1], nl - 1
        errs[f"L{li}.q"] = rel_err(lm.debug_buffer("q", (P, HD)), o["q"])
        errs[f"L{li}.k"] = rel_err(_kv_rows(lm, li, 0, 0, P), o["k"])
        errs[f"L{li}.v"] = rel_err(_kv_rows(lm, li, 1, 0, P), o["v"])
        errs[f"L{li}.attn"] = rel_err(lm.debug_buffer("attn_bf16", (P, HD), torch.bfloat16).float(), o["attn"])
        errs[f"L{li}.act"] = rel_err(lm.debug_buffer("act_bf16", (P, I), torch.bfloat16).float(), o["act"])
        errs[f"L{li}.h"] = rel_err(lm.debug_buffer("h", (P, H))[1:], o["h"][1:])   # row 0 is reused by the sampler
    lm.debug_set_layers(-1)
    print("PREFILL-STAGE-ERRORS", cfg.hidden_size, {k: f"{v:.2e}" for k, v in errs.items()})
    # relative RMS error per stage: layer 0's q is exact up to fp32 accumulation order and the odd flipped
    # bf16 rounding of its input; everything downstream carries the rounding-flip noise described above
    assert errs["L0.q"] < 1e-4, errs
    bad = {k: v for k, v in errs.items() if v > 1e-2}
    assert not bad, bad
