"""Checkpoints that transformers' Qwen2, Llama and Mistral classes write, loaded through ``loader.load_speech_lm`` and run
on the kernels: ragged prefill and teacher-forced decode on every decode path, against the oracle and transformers.

The checkpoints (written at test time by tests/checkpoints.py's ``write_checkpoint``; 3 layers, peaked attention, norm
weights and biases away from 1 and 0, even vocabularies that are not multiples of 128):

    air-qwen2            hidden 896, 14/2 heads, inter 4864, q/k/v biases, theta 1e6, eps 1e-6, tied, bf16 safetensors
    nano-llama           hidden 576, 9/3 heads, inter 1536, no biases, theta 1e5, eps 1e-5, tied, fp32 in 3+ shards
    mistral              hidden 256, 4/2 heads, inter 640, no biases, theta 1e4, eps 1e-5, untied, fp16 pytorch_model.bin
    qwen2-distinct-head  hidden 256, 4/2 heads, a tied config whose checkpoint carries its own lm_head.weight

Prompts are ragged (one of 318 tokens, the others on the 64-token page edges) and 6 teacher-forced decode steps cross
a page boundary.  Decode paths: the persistent kernel at batch 1 (in-CTA fold), 3 (hi + lo activations) and 12 (bf16
activations); ``NT_DECODE_IMPL=perop`` at batch 2 (GEMV chain) and 6 (wgmma chain); the path is asserted from the
launch count.  Each case compares
  (a) against lm_oracle with the path's rounding points (prefill: "prefill", "batched" above batch 4 where the lm_head
      input is bf16; decode: "decode_tc" on the persistent kernel up to batch 8, "decode" on the GEMV chain, "batched"
      on the bf16 paths), on weights read from transformers' model and rounded to bf16 as the engine streams them;
  (b) against transformers' float64 model on the same directory, its Linear and Embedding weights rounded to bf16.
A 1-token prompt with 70 decode steps on the two batch-1 paths checks decode where it alone wrote the cache.  The bars
and the measured errors are in checkpoints.GPU_BARS; test_loader_faults_exceed_the_gpu_bars in test_loader_families.py
shows that each loader fault moves these logits by 10x the decode-only bar and 4x the widest ragged bar.
"""
from __future__ import annotations

import subprocess

import pytest
import torch

from oracle import lm_oracle as O
from tests.checkpoints import GPU_BARS, Ckpt, hf_model64, oracle_of, write_checkpoint
from tests.helpers import GEMV_MAX_BATCH, max_err, rel_rms, runs_persistent, set_decode_impl

pytestmark = pytest.mark.gpu

CHECKPOINTS = {
    "air-qwen2": Ckpt("qwen2", hidden=896, inter=4864, heads=14, kv=2, vocab=64 * 128 + 62, theta=1e6, eps=1e-6,
                      tied=True, fmt="bf16", seed=21),
    "nano-llama": Ckpt("llama", hidden=576, inter=1536, heads=9, kv=3, vocab=48 * 128 + 94, theta=1e5, eps=1e-5,
                       tied=True, fmt="fp32-shards", seed=22),
    "mistral": Ckpt("mistral", hidden=256, inter=640, heads=4, kv=2, vocab=40 * 128 + 66, theta=1e4, eps=1e-5,
                    tied=False, fmt="fp16-bin", seed=23),
    "qwen2-distinct-head": Ckpt("qwen2", hidden=256, inter=640, heads=4, kv=2, vocab=40 * 128 + 2, theta=1e6, eps=1e-6,
                                tied=True, distinct_head=True, fmt="bf16", seed=24),
}
# (id, batch, NT_DECODE_IMPL): the path
PATHS = [("tc-b1-fold", 1, None), ("tc-b3-hilo", 3, None), ("tc-b12-bf16", 12, None),
         ("perop-b2-gemv", 2, "perop"), ("perop-b6-wgmma", 6, "perop")]
LENS = [318, 63, 64, 62, 127, 128, 1, 190, 191, 192, 255, 65]
N_NEW = 7                  # the prefill's logits + 6 decode steps
MAX_CTX = 512

BARS = GPU_BARS


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    """name -> (directory, transformers float64 model with bf16 Linear / Embedding weights, oracle cfg, oracle weights)."""
    out = {}

    def get(name):
        if name not in out:
            ck = CHECKPOINTS[name]
            root = write_checkpoint(ck, tmp_path_factory.mktemp(name))
            model = hf_model64(root, ck.family, bf16_weights=True)
            out[name] = (root, model, *oracle_of(model))
        return out[name]
    return get


def _card() -> str:
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "power limit unknown"
    return f"{name}, {pl}"


def _mirrors(B: int, impl):
    """(prefill mirror, decode mirror, decode bar key) of the path at batch B."""
    persistent = runs_persistent(impl, B)
    gemv = B <= GEMV_MAX_BATCH
    pm = "prefill" if gemv else "batched"
    if persistent:
        return pm, ("decode_tc" if B <= 8 else "batched"), ("decode-exact" if B <= 8 else "decode-bf16")
    return pm, ("decode" if gemv else "batched"), ("decode-exact" if gemv else "decode-bf16")


def _oracle(cfg, w, prompt, forced, pm, dm):
    cache = O.KVCache(cfg.num_layers)
    rows = [O.forward(cfg, w, prompt, cache, mirror=pm, last_only=True)[0][-1]]
    for s in range(N_NEW - 1):
        rows.append(O.forward(cfg, w, forced[s: s + 1], cache, mirror=dm)[0][-1])
    return torch.stack(rows)


@pytest.mark.parametrize("path", PATHS, ids=[p[0] for p in PATHS])
@pytest.mark.parametrize("name", list(CHECKPOINTS))
def test_loaded_checkpoint_vs_oracle_and_transformers(cuda, checkpoints, name, path, monkeypatch):
    from neutts_air_b200 import loader

    pid, B, impl = path
    root, model, cfg, w = checkpoints(name)
    V = cfg.vocab_size
    set_decode_impl(monkeypatch, impl)
    lm = loader.load_speech_lm(str(root), device="cuda:0", max_batch=B, max_ctx=MAX_CTX, page_shuffle_seed=B)
    assert lm.shape.tie_embeddings == (CHECKPOINTS[name].tied and not CHECKPOINTS[name].distinct_head)
    g = torch.Generator().manual_seed(100 + B)
    prompts = [torch.randint(0, V - 1, (n,), generator=g) for n in LENS[:B]]
    forced = torch.randint(0, V - 1, (B, N_NEW), generator=g)
    sp = lm.sampling(V - 1, min_new_tokens=0, max_new_tokens=N_NEW, forced=forced)
    l0 = lm.prefill([p.tolist() for p in prompts], sp, return_logits=True)
    torch.cuda.synchronize()
    n0 = lm.L.nt_launch_count()
    ls = lm.decode(N_NEW - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    got = torch.cat((l0[None], ls), 0).permute(1, 0, 2).double().cpu()          # [B, N_NEW, V]
    if runs_persistent(impl, B):
        assert launches == 1, launches                   # one launch: the persistent kernel
    else:
        assert launches > N_NEW - 1, launches            # the per-op chain: several kernels per step
    assert lm.out_tokens[:B, :N_NEW].cpu().tolist() == forced.tolist()

    pm, dm, dkey = _mirrors(B, impl)
    e = {"prefill": 0.0, "decode": 0.0, "reference": 0.0, "reference-max": 0.0}
    for b, p in enumerate(prompts):
        mir = _oracle(cfg, w, p, forced[b], pm, dm)
        with torch.no_grad():
            ref = model(torch.cat((p, forced[b, : N_NEW - 1]))[None]).logits[0, len(p) - 1:]
        e["prefill"] = max(e["prefill"], rel_rms(got[b, 0], mir[0]))
        e["decode"] = max(e["decode"], rel_rms(got[b, 1:], mir[1:]))
        e["reference"] = max(e["reference"], rel_rms(got[b], ref))
        e["reference-max"] = max(e["reference-max"], max_err(got[b], ref) / float(ref.std()))
    print(f"LOADER {name} {pid} [{launches} launches, {_card()}]: (a) prefill {e['prefill']:.2e} (bar {BARS['prefill']:.1e}) "
          f"decode {e['decode']:.2e} (bar {BARS[dkey]:.1e}); (b) relRMS {e['reference']:.2e} (bar {BARS['reference']:.1e}) "
          f"max/spread {e['reference-max']:.2e} (bar {BARS['reference-max']:.1e})")
    assert e["prefill"] < BARS["prefill"], e
    assert e["decode"] < BARS[dkey], e
    assert e["reference"] < BARS["reference"] and e["reference-max"] < BARS["reference-max"], e


DECODE_ONLY = [("tc-b1-fold", None), ("perop-b1-gemv", "perop")]


@pytest.mark.parametrize("path", DECODE_ONLY, ids=[p[0] for p in DECODE_ONLY])
@pytest.mark.parametrize("name", list(CHECKPOINTS))
def test_loaded_checkpoint_decode_only(cuda, checkpoints, name, path, monkeypatch):
    """A 1-token prompt and 70 teacher-forced steps (past the first page): the KV cache is almost all written by the
    decode path, whose activations are fp32-grade, so the mirrored oracle sits at the K/V rounding flips alone."""
    from neutts_air_b200 import loader

    pid, impl = path
    root, model, cfg, w = checkpoints(name)
    V, n_new = cfg.vocab_size, 71
    set_decode_impl(monkeypatch, impl)
    lm = loader.load_speech_lm(str(root), device="cuda:0", max_batch=1, max_ctx=256, page_shuffle_seed=5)
    g = torch.Generator().manual_seed(6)
    prompt = torch.randint(0, V - 1, (1,), generator=g)
    forced = torch.randint(0, V - 1, (1, n_new), generator=g)
    sp = lm.sampling(V - 1, min_new_tokens=0, max_new_tokens=n_new, forced=forced)
    l0 = lm.prefill([prompt.tolist()], sp, return_logits=True)
    n0 = lm.L.nt_launch_count()
    ls = lm.decode(n_new - 1, sp, return_logits=True)
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    assert launches == 1 if impl is None else launches > n_new - 1, launches
    got = torch.cat((l0[None], ls), 0)[:, 0].double().cpu()
    _, mir = O.generate(cfg, w, prompt, V - 1, max_length=256, max_new_tokens=n_new, forced=forced[0], mirror=True,
                        decode_mirror="decode_tc" if impl is None else None)
    with torch.no_grad():
        ref = model(torch.cat((prompt, forced[0, : n_new - 1]))[None]).logits[0]
    e_m, e_r = rel_rms(got[1:], mir[1:]), rel_rms(got, ref)
    print(f"LOADER-DECODE {name} {pid} [{launches} launches, {_card()}]: (a) {e_m:.2e} (bar {BARS['decode-only']:.1e}); "
          f"(b) {e_r:.2e} (bar {BARS['decode-only-reference']:.1e})")
    assert e_m < BARS["decode-only"], e_m
    assert e_r < BARS["decode-only-reference"], e_r
