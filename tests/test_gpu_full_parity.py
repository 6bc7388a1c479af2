"""GPU: the BASELINE model shape (24 layers, hidden 896, vocabulary 217 472) pinned to the oracle.

VERDICT r1 "next round" item 1: the full NeuTTS-Air shape is compared with ``oracle/lm_oracle.py`` (pure fp32
reference semantics) AND with the real ``transformers.Qwen2ForCausalLM`` forward on the same bf16-valued weights:

  (a) configs[1]: 500-token prompt + 16 teacher-forced decode steps, batch 1;
  (b) configs[2]: batch 64 with ragged prompts U{200..1400}, 4 of the 64 slots checked against the oracle;
  (c) context limit: a 2040-token prompt decoded to the max_ctx = 2048 stop (``done``, ``seq_lens``, logits);
  (d) a Nano-like shape (hidden 576, 9 heads / 3 KV heads, inter 1536) to show the kernels are config-driven;
  (e) the Nano-like shape bench.py streams (hidden 512, 8 / 2 heads, inter 2048, 28 layers, V = 217 472) at batch 8.

Bars (relative RMS error of the logits / max error in units of the logit spread), stated per test:
vs the pure-fp32 reference 2e-2 / 1e-1 — the CUDA path keeps bf16 weights (shared with the oracle), a bf16 KV
cache and bf16 GEMM inputs on the tensor-core path; those roundings are the whole difference.
The oracle runs on the GPU box's host cores (a 500-token fp32 prefill takes well under a second there).
"""
import os

import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import decode_branch, make_lm, max_err, rel_err

pytestmark = pytest.mark.gpu

EOS = 151670


@pytest.fixture(scope="module")
def full(cuda):
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = O.LMConfig()
    assert (cfg.num_layers, cfg.hidden_size, cfg.vocab_size) == (24, 896, 217472)
    w = O.random_weights(cfg, 7, std=0.02, bf16_round=True)
    return cfg, w


def _tf(lm, prompts, forced, n_new, eos=EOS):
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=n_new, forced=forced)
    l0 = lm.prefill(prompts, sp, return_logits=True)
    ls = lm.decode(n_new - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    return torch.cat((l0[None], ls), 0).permute(1, 0, 2).float().cpu()       # [B, n_new, V]


def _bars(got, ref, tag, r_bar=2e-2, m_bar=1e-1):
    spread = float(ref.std())
    r, m = rel_err(got, ref), max_err(got, ref) / spread
    print(f"FULL-PARITY {tag}: relRMS {r:.2e} max/spread {m:.2e} (spread {spread:.3f})")
    assert torch.isfinite(got).all()
    assert r < r_bar and m < m_bar, (tag, r, m)
    return r, m


def test_full_b1_500_prefill_16_decode_vs_oracle_and_hf(full):
    cfg, w = full
    lm = make_lm(cfg, w, max_batch=1, max_ctx=2048, max_new=32, max_prefill_tokens=512, page_shuffle_seed=2)
    g = torch.Generator().manual_seed(5)
    P, n_new = 500, 17
    prompt = torch.randint(0, cfg.vocab_size, (P,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, n_new), generator=g)
    got = _tf(lm, [prompt.tolist()], forced, n_new)[0]
    # state machine at the end of the teacher-forced run
    assert lm.out_tokens[0, :n_new].cpu().tolist() == forced[0].tolist()
    assert int(lm.seq_lens[0]) == P + n_new - 1
    # (1) restated oracle, pure fp32 reference semantics
    _, ref = O.generate(cfg, w, prompt, EOS, max_length=2048, max_new_tokens=n_new, forced=forced[0], mirror=False)
    _bars(got[:1], ref[:1], "b1 prefill(500) vs oracle")
    _bars(got[1:], ref[1:], "b1 16 decode steps vs oracle")
    # (2) the real transformers model (what neutts/neutts.py:164 loads), eager attention, fp32
    hf = O.to_hf_model(cfg, w)
    with torch.no_grad():
        out = hf(prompt[None], use_cache=True, logits_to_keep=1)
        rows = [out.logits[0, -1]]
        past = out.past_key_values
        for t in forced[0, :-1].tolist():
            out = hf(torch.tensor([[t]]), past_key_values=past, use_cache=True)
            past = out.past_key_values
            rows.append(out.logits[0, -1])
    hf_logits = torch.stack(rows)
    r_o = rel_err(ref, hf_logits)
    print(f"FULL-PARITY oracle vs transformers at full size: relRMS {r_o:.2e}")
    assert r_o < 1e-4
    _bars(got, hf_logits, "b1 all 17 steps vs transformers")
    # per-layer hidden state of the prefill (residual stream after each layer), rows 1.. (row 0 is reused by the sampler)
    _, hid = O.forward(cfg, w, prompt, O.KVCache(cfg.num_layers), collect_hidden=True, last_only=True)
    sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=4)
    errs = []
    for nl in (1, 6, 12, 18, 24):
        lm.debug_set_layers(nl)
        lm.prefill([prompt.tolist()], sp)
        torch.cuda.synchronize()
        errs.append((nl, rel_err(lm.debug_buffer("h", (P, cfg.hidden_size))[1:], hid[nl][1:])))
    lm.debug_set_layers(-1)
    print("FULL-PARITY prefill hidden relRMS by layer:", ", ".join(f"L{n}: {e:.2e}" for n, e in errs))
    assert max(e for _, e in errs) < 2e-2


def test_full_context_limit_stop(full):
    """P = 2040 -> 8 new tokens reach max_ctx = 2048: done flag, seq_lens, logits at contexts 2040..2047."""
    cfg, w = full
    lm = make_lm(cfg, w, max_batch=1, max_ctx=2048, max_new=32, max_prefill_tokens=2048)
    g = torch.Generator().manual_seed(8)
    P = 2040
    prompt = torch.randint(0, cfg.vocab_size, (P,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, 8), generator=g)
    sp = lm.sampling(EOS, min_new_tokens=0, max_new_tokens=32, forced=forced)
    l0 = lm.prefill([prompt.tolist()], sp, return_logits=True)
    ls = lm.decode(12, sp, return_logits=True)       # asks for more steps than the context allows
    torch.cuda.synchronize()
    assert int(lm.done[0]) == 1
    assert int(lm.n_generated[0]) == 8, int(lm.n_generated[0])          # 2040 + 8 = max_ctx (stopping_criteria.py:73-84)
    assert int(lm.seq_lens[0]) == 2047
    got = torch.cat((l0[None], ls[:7]), 0)[:, 0].float().cpu()
    _, ref = O.generate(cfg, w, prompt, EOS, max_length=2048, max_new_tokens=8, forced=forced[0], mirror=False)
    assert ref.shape[0] == 8
    _bars(got, ref, "ctx 2040..2047 vs oracle")
    # generate_batch applies the same stop through the public seam
    outs = lm.generate_batch([prompt.tolist()], EOS, max_length=2048, min_new_tokens=0, seed=3)
    assert len(outs[0]) <= 8


def test_full_batch64_ragged_vs_oracle(full):
    """configs[2]: 64 ragged prompts U{200..1400}; prefill + 3 decode steps; slots 0, longest, shortest and 37 vs the oracle."""
    cfg, w = full
    g = torch.Generator().manual_seed(21)
    lens = torch.randint(200, 1401, (64,), generator=g).tolist()
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g) for n in lens]
    n_new = 4
    forced = torch.randint(0, cfg.vocab_size, (64, n_new), generator=g)
    lm = make_lm(cfg, w, max_batch=64, max_ctx=2048, max_new=8, max_prefill_tokens=sum(lens))
    got = _tf(lm, [p.tolist() for p in prompts], forced, n_new)
    again = _tf(lm, [p.tolist() for p in prompts], forced, n_new)
    assert torch.equal(got, again), "batch-64 decode is not run-to-run reproducible"
    check = sorted({0, 37, max(range(64), key=lambda i: lens[i]), min(range(64), key=lambda i: lens[i])})
    for b in check:
        _, ref = O.generate(cfg, w, prompts[b], EOS, max_length=2048, max_new_tokens=n_new, forced=forced[b], mirror=False)
        _bars(got[b, :1], ref[:1], f"b64 slot {b} (P={lens[b]}) prefill")
        _bars(got[b, 1:], ref[1:], f"b64 slot {b} (P={lens[b]}) decode")
    assert lm.out_tokens[:64, :n_new].cpu().tolist() == forced.tolist()
    assert lm.seq_lens[:64].cpu().tolist() == [n + n_new - 1 for n in lens]


NANO = dict(vocab_size=16384, hidden_size=576, intermediate_size=1536, num_layers=6, num_heads=9, num_kv_heads=3)


@pytest.mark.parametrize("B", [1, 8])
def test_nano_like_shape(cuda, B):
    """hidden 576 (not a multiple of 128), 9 query / 3 KV heads (GQA ratio 3), qkv rows 960: nothing is hard-coded to Air."""
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = O.LMConfig.tiny(**NANO)
    w = O.random_weights(cfg, 17, std=0.04, bf16_round=True)
    lm = make_lm(cfg, w, max_batch=B, max_ctx=512, max_new=16, page_shuffle_seed=4)
    g = torch.Generator().manual_seed(6)
    lens = [150, 64, 65, 200, 31, 129, 90, 255][:B]
    prompts = [torch.randint(0, cfg.vocab_size, (n,), generator=g) for n in lens]
    n_new = 10
    forced = torch.randint(0, cfg.vocab_size, (B, n_new), generator=g)
    got = _tf(lm, [p.tolist() for p in prompts], forced, n_new, eos=cfg.vocab_size - 1)
    for b in range(B):
        _, ref = O.generate(cfg, w, prompts[b], cfg.vocab_size - 1, max_length=512, max_new_tokens=n_new, forced=forced[b], mirror=False)
        _bars(got[b], ref, f"nano-like B={B} slot {b}")


# The Nano-like model bench.py measures in its streaming line: hidden 512, 8 query / 2 KV heads (GQA ratio 4), inter 2048
BENCH_NANO = dict(vocab_size=217472, hidden_size=512, intermediate_size=2048, num_layers=28, num_heads=8, num_kv_heads=2)


def test_bench_nano_shape_b8(cuda):
    """The benchmark's streaming shape end to end: 28 layers, V = 217 472, batch 8, 500-token prompts, then 16
    teacher-forced steps in one launch of the persistent kernel (hi + lo activations, whole-K plan); slots 0 and 5
    against the oracle, prefill and decode rows."""
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = O.LMConfig.tiny(**BENCH_NANO)
    w = O.random_weights(cfg, 23, std=0.02, bf16_round=True)
    B, P, n_new = 8, 500, 17
    lm = make_lm(cfg, w, max_batch=B, max_ctx=2048, max_new=32, max_prefill_tokens=B * P, page_shuffle_seed=5)
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
    forced = torch.randint(0, cfg.vocab_size, (B, n_new), generator=g)
    eos = cfg.vocab_size - 1
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=n_new, forced=forced)
    l0 = lm.prefill([p.tolist() for p in prompts], sp, return_logits=True)
    torch.cuda.synchronize()
    n0 = lm.L.nt_launch_count()
    ls = lm.decode(n_new - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    got = torch.cat((l0[None], ls), 0).permute(1, 0, 2).float().cpu()
    sms = min(torch.cuda.get_device_properties(0).multi_processor_count, 256)
    br = decode_branch((cfg.hidden_size, cfg.intermediate_size, cfg.num_heads, cfg.num_kv_heads, cfg.vocab_size), B, sms,
                       2048)
    print(f"FULL-PARITY bench-nano B={B}: decode [{br['name']}, {launches} launches]")
    assert br["name"] == "tc-hilo-n16-wholeK-phases" and launches == 1, (br, launches)
    assert lm.out_tokens[:B, :n_new].cpu().tolist() == forced.tolist()
    for b in (0, 5):
        _, ref = O.generate(cfg, w, prompts[b], eos, max_length=2048, max_new_tokens=n_new, forced=forced[b], mirror=False)
        _bars(got[b, :1], ref[:1], f"bench-nano B={B} slot {b} prefill(500)")
        _bars(got[b, 1:], ref[1:], f"bench-nano B={B} slot {b} 16 decode steps")
