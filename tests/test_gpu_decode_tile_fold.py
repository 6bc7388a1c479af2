"""GPU: the batch-1 persistent decode kernel's tile fold.

At batch 1 the last CTA to store a split-K slice of an o_proj or down_proj row tile folds the tile into the residual
stream (lm_decode_tc.cu, ``tile_fold``): it counts arrivals on one self-resetting counter per tile and writes into a
two-buffer ping-pong indexed by the fold number.  A counter left off by one after a launch, or a buffer parity that
does not follow the fold count, would change results only across launches or at some layer counts; these tests run
those cases:

* two identical launches give bit-identical logits at every step;
* ``decode(5)`` then ``decode(7)`` gives the same tokens and logits as one ``decode(12)`` from the same prefill and
  seed, so the counters and the ping-pong carry over from one launch to the next;
* models with 1 and 2 layers (an odd and an even number of folds per layer loop) match the float64 oracle at the
  decode-path bar of test_gpu_lm (1e-3 relative RMS, mirrored roundings).
"""
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import make_lm, max_err, rel_err, runs_persistent, set_decode_impl

pytestmark = pytest.mark.gpu

# NeuTTS-Air widths (7 row tiles of o_proj and down_proj, 7 and 16 K slices), a small vocabulary
WIDE = dict(vocab_size=8192, hidden_size=896, intermediate_size=4864, num_heads=14, num_kv_heads=2)


def _engine(n_layers, seed, max_ctx=256):
    cfg = O.LMConfig.tiny(num_layers=n_layers, **WIDE)
    w = O.random_weights(cfg, seed, std=0.05, bf16_round=True)
    return cfg, w, make_lm(cfg, w, max_batch=1, max_ctx=max_ctx, page_shuffle_seed=3)


def _sampled_run(lm, cfg, prompt, chunks):
    """Prefill, then decode launches of ``chunks`` steps each (sampled, EOS masked); tokens and per-step logits."""
    eos = cfg.vocab_size - 1
    total = sum(chunks)
    sp = lm.sampling(eos, min_new_tokens=total + 2, max_new_tokens=total + 2, top_k=50, temperature=1.0, seed=7)
    lm.prefill([prompt], sp)
    logits = torch.cat([lm.decode(n, sp, return_logits=True) for n in chunks], 0)
    torch.cuda.synchronize()
    return lm.out_tokens[0, : total + 1].cpu().clone(), logits[:, 0].cpu()


def test_identical_launches_are_bit_identical(cuda, monkeypatch):
    set_decode_impl(monkeypatch, None)
    assert runs_persistent(None, 1)
    cfg, _, lm = _engine(2, 31)
    prompt = torch.randint(0, cfg.vocab_size - 1, (90,), generator=torch.Generator().manual_seed(1)).tolist()
    t0, l0 = _sampled_run(lm, cfg, prompt, [12])
    t1, l1 = _sampled_run(lm, cfg, prompt, [12])
    assert torch.equal(t0, t1)
    assert torch.equal(l0, l1), [int((l0[s] != l1[s]).sum()) for s in range(l0.shape[0])]


def test_split_launches_match_one_launch(cuda, monkeypatch):
    set_decode_impl(monkeypatch, None)
    cfg, _, lm = _engine(2, 32)
    prompt = torch.randint(0, cfg.vocab_size - 1, (70,), generator=torch.Generator().manual_seed(2)).tolist()
    t_one, l_one = _sampled_run(lm, cfg, prompt, [12])
    t_two, l_two = _sampled_run(lm, cfg, prompt, [5, 7])
    assert torch.equal(t_one, t_two), (t_one.tolist(), t_two.tolist())
    assert torch.equal(l_one, l_two), [int((l_one[s] != l_two[s]).sum()) for s in range(l_one.shape[0])]


@pytest.mark.parametrize("n_layers", [1, 2])
def test_layer_counts_match_float64(cuda, monkeypatch, n_layers):
    """A 1-token prompt and 40 teacher-forced steps: every logit row but the first comes out of the persistent kernel."""
    set_decode_impl(monkeypatch, None)
    cfg, w, lm = _engine(n_layers, 40 + n_layers)
    g = torch.Generator().manual_seed(8)
    n_new, eos = 41, cfg.vocab_size - 1
    prompt = torch.randint(0, cfg.vocab_size, (1,), generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, n_new), generator=g)
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=n_new, forced=forced)
    l0 = lm.prefill([prompt.tolist()], sp, return_logits=True)
    ls = lm.decode(n_new - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    got = torch.cat((l0[None], ls), 0)[:, 0].cpu()
    _, mir = O.generate(cfg, w, prompt, eos, max_length=256, max_new_tokens=n_new, forced=forced[0], mirror=True,
                        decode_mirror="decode_tc")
    r = rel_err(got, mir)
    print(f"TILE-FOLD L{n_layers}: relRMS {r:.2e} max {max_err(got, mir):.2e}")
    assert r < 1e-3, r
