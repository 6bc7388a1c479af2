"""GPU: the full NeuTTS-Air shape (24 layers, vocabulary 217 472 — the BASELINE workload's model), where the CPU
oracle would take minutes per forward.  Parity there is checked through size-independent properties:

  * prefill / decode consistency: the logits after prefill(P) + k teacher-forced decode steps equal the logits at
    the last position of prefill(P + k) — two different kernel families (tensor-core GEMMs + flash attention vs the
    persistent wgmma decode kernel with split-KV attention) over the same paged KV cache, RoPE positions and weights;
  * batch invariance: a sequence decoded alone and inside a batch of 6 agrees (both on the persistent wgmma kernel,
    which folds the split-K slices in every CTA at batch 1 and in dedicated fold phases at batch 6);
  * reproducibility: the same seed gives the same sampled tokens twice.
"""
import pytest
import torch

from neutts_air_b200 import synthetic
from neutts_air_b200.lm import LMShape, SpeechLM
from tests.helpers import max_err, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def full_lm(cuda):
    shape = LMShape()
    assert (shape.num_layers, shape.hidden_size, shape.vocab_size) == (24, 896, 217472)
    return SpeechLM(shape, synthetic.lm_state_dict(shape, 0), device="cuda:0", max_batch=6, max_ctx=1024, max_new=16,
                    max_prefill_tokens=6 * 400)


def _prompt(n, seed):
    return torch.randint(0, 217472, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


def test_full_size_prefill_decode_consistency(full_lm):
    lm, P, k = full_lm, 300, 3
    ids = _prompt(P + k, 5)
    eos = 151670
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8, forced=torch.tensor([ids[P:P + k] + [0] * 5]))
    lm.prefill([ids[:P]], sp)
    stepped = lm.decode(k, sp, return_logits=True)[-1, 0].float().cpu()      # after feeding ids[P..P+k-1]
    sp2 = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8)
    whole = lm.prefill([ids], sp2, return_logits=True)[0].float().cpu()      # last position of prefill(P + k)
    r, m = rel_err(stepped, whole), max_err(stepped, whole) / float(whole.std())
    print(f"FULL-SIZE prefill/decode consistency: relRMS {r:.2e}, max/spread {m:.2e}, spread {float(whole.std()):.3f}")
    assert torch.isfinite(stepped).all() and torch.isfinite(whole).all()
    assert r < 3e-2 and m < 2e-1, (r, m)
    assert int(stepped.argmax()) in torch.topk(whole, 5).indices.tolist()


def test_full_size_batch_invariance_and_reproducibility(full_lm):
    lm = full_lm
    eos = 151670
    prompts = [_prompt(n, 10 + i) for i, n in enumerate((120, 333, 64, 200, 257, 90))]
    forced = torch.randint(0, 217472, (6, 8), generator=torch.Generator().manual_seed(3))
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8, forced=forced)
    lm.prefill(prompts, sp)
    batch = lm.decode(4, sp, return_logits=True)[:, 1].float().cpu()          # slot 1, persistent kernel at batch 6
    sp1 = lm.sampling(eos, min_new_tokens=0, max_new_tokens=8, forced=forced[1:2])
    lm.prefill(prompts[1:2], sp1)
    solo = lm.decode(4, sp1, return_logits=True)[:, 0].float().cpu()          # same sequence alone (persistent kernel, batch 1)
    r = rel_err(batch, solo)
    print(f"FULL-SIZE batch invariance: relRMS {r:.2e}")
    assert r < 3e-2, r
    outs = [lm.generate_batch(prompts[:2], eos, max_length=1024, min_new_tokens=4, max_new_tokens=12, seed=77) for _ in range(2)]
    assert [o.tolist() for o in outs[0]] == [o.tolist() for o in outs[1]]


@pytest.mark.parametrize("B,impl", [(1, None), (3, None), (6, None), (6, "perop")],
                         ids=["persistent-b1", "persistent-b3", "persistent-b6", "chain-b6-tile-sampler"])
def test_decode_kernel_sampler_matches_standalone_sampler(full_lm, B, impl, monkeypatch):
    """The persistent decode kernel samples inside the kernel (tile maxima -> candidate tiles -> exact top-k ->
    Philox draw); the per-op chain runs the same scheme as a kernel of its own behind the lm_head GEMM.  Given the logits it returns for a step, the stand-alone sampler op (``nt_op_topk_sample``, pinned
    to the HF processors + multinomial by tests/test_gpu_kernels.py) must pick the very same token: same top-50 set,
    same probabilities, same Philox counter (seed, slot, n_generated).  Covers the EOS mask (min_new_tokens) too."""
    import ctypes as C

    from neutts_air_b200 import _lib

    if impl:   # the per-op chain: tensor-core lm_head with tile maxima in its epilogue + topk_tiles_kernel
        monkeypatch.setenv("NT_DECODE_IMPL", impl)
    lm, eos, n_steps = full_lm, 151670, 9
    L = _lib.lib()
    prompts = [_prompt(40 + 17 * i, 30 + i) for i in range(B)]
    sp = lm.sampling(eos, min_new_tokens=5, max_new_tokens=16, top_k=50, temperature=0.8, seed=4242)
    lm.prefill(prompts, sp)
    logits = lm.decode(n_steps, sp, return_logits=True).float()            # [n_steps, B, V]; step s draws token s + 1
    torch.cuda.synchronize()
    toks = lm.out_tokens[:B, : n_steps + 1].cpu()
    V = logits.shape[-1]
    ws = torch.empty(1 << 24, dtype=torch.uint8, device=logits.device)
    tok = torch.zeros(B, dtype=torch.int32, device=logits.device)
    tv = torch.zeros(B, 64, device=logits.device)
    ti = torch.zeros(B, 64, dtype=torch.int32, device=logits.device)
    for s in range(n_steps):
        ngen = s + 1
        ng = torch.full((B,), ngen, dtype=torch.int32, device=logits.device)
        row = logits[s].contiguous()
        _lib.check(L.nt_op_topk_sample(row.data_ptr(), B, V, C.byref(sp), ng.data_ptr(), ngen, tok.data_ptr(), tv.data_ptr(),
                                       ti.data_ptr(), ws.data_ptr(), ws.numel(), _lib.current_stream_ptr()))
        torch.cuda.synchronize()
        assert tok.cpu().tolist() == toks[:, ngen].tolist(), (s, tok.cpu().tolist(), toks[:, ngen].tolist())
        if ngen < 5:
            assert eos not in ti[:, :50].cpu().flatten().tolist()
