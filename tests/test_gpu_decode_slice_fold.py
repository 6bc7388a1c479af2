"""GPU: the batch-1 persistent decode kernel's qkv and gate/up slice folds.

At batch 1 the last CTA to store a split-K slice of a qkv or gate/up row tile folds the tile (lm_decode_tc.cu,
``tile_fold``): it adds the slices (and, for qkv, the bias and RoPE; for gate/up, SwiGLU) and publishes finished rows
that the attention prologue and the down_proj staging poll, one stamped pair per element.  Each such tile has a
self-resetting arrival counter in the grid-barrier block, and each published buffer holds one version whose reuse rests
on the layer's chain of hand-offs.  A counter left off by one, or a version overwritten before all its readers are
through, would change results only across launches, at some layer counts or at the end of the context; these tests run
those cases at the NeuTTS-Air widths (9 qkv row tiles of 7 slices, 76 gate/up tiles of up to 4 slices):

* two identical launches give bit-identical tokens and logits;
* ``decode(5)`` then ``decode(7)`` gives the same tokens and logits as one ``decode(12)``, so the counters carry over
  from one launch to the next;
* with 1 and 2 layers, a launch that asks for more steps than the context holds stops at max_ctx, and its logits up
  to the last position match the float64 oracle (mirrored roundings) at test_gpu_lm's bar for multi-token prompts.

test_gpu_decode_tile_fold's 1-token float64 check at 1 and 2 layers runs the same kernel path and covers the 1e-3 bar.
"""
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import decode_branch, make_lm, max_err, rel_err, runs_persistent, set_decode_impl

pytestmark = pytest.mark.gpu

WIDE = dict(vocab_size=8192, hidden_size=896, intermediate_size=4864, num_heads=14, num_kv_heads=2)


def _engine(n_layers, seed, max_ctx=256, **kw):
    cfg = O.LMConfig.tiny(num_layers=n_layers, **WIDE)
    w = O.random_weights(cfg, seed, std=0.05, bf16_round=True)
    return cfg, w, make_lm(cfg, w, max_batch=1, max_ctx=max_ctx, page_shuffle_seed=5, **kw)


def _flat_fold(cfg, max_ctx):
    """The batch-1 decode of ``cfg`` runs the persistent kernel's flat plan with the in-CTA folds on this device."""
    G = torch.cuda.get_device_properties(0).multi_processor_count
    shape = (cfg.hidden_size, cfg.intermediate_size, cfg.num_heads, cfg.num_kv_heads, cfg.vocab_size)
    br = decode_branch(shape, 1, G, max_ctx)
    return br["kind"] == "tc" and br["plan"] == "flat" and br["fold"]


def _sampled_run(lm, cfg, prompt, chunks):
    eos = cfg.vocab_size - 1
    total = sum(chunks)
    sp = lm.sampling(eos, min_new_tokens=total + 2, max_new_tokens=total + 2, top_k=50, temperature=1.0, seed=11)
    lm.prefill([prompt], sp)
    logits = torch.cat([lm.decode(n, sp, return_logits=True) for n in chunks], 0)
    torch.cuda.synchronize()
    return lm.out_tokens[0, : total + 1].cpu().clone(), logits[:, 0].cpu()


def test_identical_launches_are_bit_identical(cuda, monkeypatch):
    set_decode_impl(monkeypatch, None)
    assert runs_persistent(None, 1)
    cfg, _, lm = _engine(2, 51)
    assert _flat_fold(cfg, 256)
    prompt = torch.randint(0, cfg.vocab_size - 1, (75,), generator=torch.Generator().manual_seed(3)).tolist()
    t0, l0 = _sampled_run(lm, cfg, prompt, [12])
    t1, l1 = _sampled_run(lm, cfg, prompt, [12])
    assert torch.equal(t0, t1)
    assert torch.equal(l0, l1), [int((l0[s] != l1[s]).sum()) for s in range(l0.shape[0])]


def test_split_launches_match_one_launch(cuda, monkeypatch):
    set_decode_impl(monkeypatch, None)
    cfg, _, lm = _engine(3, 52)
    prompt = torch.randint(0, cfg.vocab_size - 1, (60,), generator=torch.Generator().manual_seed(4)).tolist()
    t_one, l_one = _sampled_run(lm, cfg, prompt, [12])
    t_two, l_two = _sampled_run(lm, cfg, prompt, [5, 7])
    assert torch.equal(t_one, t_two), (t_one.tolist(), t_two.tolist())
    assert torch.equal(l_one, l_two), [int((l_one[s] != l_two[s]).sum()) for s in range(l_one.shape[0])]


@pytest.mark.parametrize("n_layers", [1, 2])
def test_context_fills_during_the_launch(cuda, monkeypatch, n_layers):
    """A 120-token prompt, max_ctx 128: one launch of 12 steps reaches the context limit after 8 new tokens.  The bar is
    test_gpu_lm's for mirrored multi-token prompts (the prefill's bf16 roundings enter every row)."""
    set_decode_impl(monkeypatch, None)
    max_ctx, P = 128, 120
    cfg, w, lm = _engine(n_layers, 61 + n_layers, max_ctx=max_ctx, max_new=32)
    assert _flat_fold(cfg, max_ctx)
    g = torch.Generator().manual_seed(10)
    n_new, eos = max_ctx - P, cfg.vocab_size - 1
    prompt = torch.randint(0, cfg.vocab_size, (P,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, n_new), generator=g)
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=32, forced=forced)
    l0 = lm.prefill([prompt.tolist()], sp, return_logits=True)
    ls = lm.decode(12, sp, return_logits=True)
    torch.cuda.synchronize()
    assert int(lm.done[0]) == 1
    assert int(lm.n_generated[0]) == n_new, int(lm.n_generated[0])
    assert int(lm.seq_lens[0]) == max_ctx - 1
    got = torch.cat((l0[None], ls[: n_new - 1]), 0)[:, 0].cpu()
    _, mir = O.generate(cfg, w, prompt, eos, max_length=max_ctx, max_new_tokens=n_new, forced=forced[0], mirror=True,
                        decode_mirror="decode_tc")
    assert mir.shape[0] == n_new
    r, m = rel_err(got, mir), max_err(got, mir)
    print(f"SLICE-FOLD L{n_layers} context limit: relRMS {r:.2e} max {m:.2e}")
    assert r < 6e-3 and m < 5e-2 * float(mir.std()), (r, m)
