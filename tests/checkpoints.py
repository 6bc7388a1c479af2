"""Tiny Qwen2, Llama and Mistral checkpoints written at test time by transformers' own classes, transformers' float64
model read back from them, and the oracle weights taken from that model; the bars of the GPU tests that load them.

The weights make loader faults visible: norm weights 1 + N(0, 0.1) and biases N(0, 0.1) (transformers' init leaves 1
and 0, under which a swapped norm or a dropped bias changes nothing), q/k projections large enough for attention scores
of standard deviation > 2, and embeddings of std 0.005, so that eps matters.
"""
from __future__ import annotations

import dataclasses
import math
from pathlib import Path

import pytest
import torch

pytest.importorskip("transformers")
import transformers  # noqa: E402

from oracle import lm_oracle as O  # noqa: E402

transformers.logging.set_verbosity_error()

CLASSES = {"qwen2": ("Qwen2Config", "Qwen2ForCausalLM"), "llama": ("LlamaConfig", "LlamaForCausalLM"),
           "mistral": ("MistralConfig", "MistralForCausalLM"), "qwen3": ("Qwen3Config", "Qwen3ForCausalLM"),
           "qwen2_moe": ("Qwen2MoeConfig", "Qwen2MoeForCausalLM")}
QK_GAIN = 1.8          # q/k weights of std QK_GAIN / sqrt(H): attention scores of std > 2 after the norm weights
# Bars of test_gpu_loader_families.py: relative RMS per slot ("reference-max": max error in units of the logit
# spread), ~4x above the worst errors measured on one H100 80GB HBM3 (700 W) over its 28 cases:
#   ragged prefill, lm_oracle with the prefill's rounding points                     2.2e-2 -> 8e-2
#   6 decode steps after it, fp32-grade paths (persistent batch <= 8, GEMV chain)     1.4e-2 -> 5e-2
#   6 decode steps after it, bf16-activation paths                                    1.8e-2 -> 7e-2
#   those 7 logit rows against transformers' float64 model (bf16 weights)            4.0e-2 -> 1.5e-1; max 0.23 -> 0.9
#   1-token prompt + 70 decode steps, against the mirrored oracle                     3.5e-3 -> 1.4e-2
#   the same against transformers' float64 model                                      1.5e-2 -> 6e-2
# Peaked attention amplifies the flips of bf16 roundings (activations before the prefill GEMMs, the K/V cache, the
# tensor-core attention operands) that these paths carry by design (test_gpu_projections.py, whose attention is an
# exact average, measures 3.6e-3 on its bf16 paths).  After a ragged prefill the decode steps inherit the prefill's
# flips through the cache, hence the 1-token cases, where the decode path writes the cache.
GPU_BARS = {"prefill": 8e-2, "decode-exact": 5e-2, "decode-bf16": 7e-2, "reference": 1.5e-1, "reference-max": 0.9,
            "decode-only": 1.4e-2, "decode-only-reference": 6e-2}


@dataclasses.dataclass(frozen=True)
class Ckpt:
    """A tiny checkpoint: family, widths, RoPE theta, RMSNorm eps, tying, on-disk format and extra config keys.
    ``fmt``: "bf16" (one safetensors file), "fp32-shards" (several safetensors shards), "fp16-bin" (pytorch_model.bin).
    ``distinct_head``: a tied config whose checkpoint still carries its own ``lm_head.weight`` (bf16 only)."""
    family: str
    hidden: int = 128
    inter: int = 256
    heads: int = 2
    kv: int = 1
    vocab: int = 2 * 128 + 62
    layers: int = 3
    theta: float = 1e4
    eps: float = 1e-5
    tied: bool = False
    fmt: str = "bf16"
    distinct_head: bool = False
    extra: tuple = ()
    seed: int = 0


def hf_config(ck: Ckpt):
    kw = dict(vocab_size=ck.vocab, hidden_size=ck.hidden, intermediate_size=ck.inter, num_hidden_layers=ck.layers,
              num_attention_heads=ck.heads, num_key_value_heads=ck.kv, head_dim=64, rms_norm_eps=ck.eps,
              tie_word_embeddings=ck.tied, max_position_embeddings=4096, rope_theta=ck.theta)
    kw.update(dict(ck.extra))
    if "rope_parameters" in kw:
        kw.pop("rope_theta")
    return getattr(transformers, CLASSES[ck.family][0])(**kw)


def _randomise(model, ck: Ckpt) -> None:
    g = torch.Generator().manual_seed(ck.seed)
    rn = lambda shape, std: torch.randn(*shape, generator=g) * std
    with torch.no_grad():
        for name, p in model.named_parameters():          # a tied lm_head is the embedding (listed once)
            if name.endswith("norm.weight"):
                p.copy_(1 + rn(p.shape, 0.1))
            elif name.endswith(".bias"):
                p.copy_(rn(p.shape, 0.1))
            elif name.endswith("embed_tokens.weight"):
                p.copy_(rn(p.shape, 0.005))
            elif name.endswith(("q_proj.weight", "k_proj.weight")):
                p.copy_(rn(p.shape, QK_GAIN / math.sqrt(p.shape[1])))
            elif p.dim() == 2:
                p.copy_(rn(p.shape, 1 / math.sqrt(p.shape[1])))


def write_checkpoint(ck: Ckpt, root: Path) -> Path:
    """Writes ``ck`` with transformers' own class into ``root`` and returns ``root``."""
    from safetensors.torch import load_file, save_file

    root.mkdir(parents=True, exist_ok=True)
    model = getattr(transformers, CLASSES[ck.family][1])(hf_config(ck))
    _randomise(model, ck)
    if ck.fmt == "bf16":
        model.to(torch.bfloat16).save_pretrained(root)
    elif ck.fmt == "fp32-shards":
        total = sum(p.numel() * 4 for p in model.parameters())
        model.save_pretrained(root, max_shard_size=total // 3)
        assert len(list(root.glob("*.safetensors"))) >= 3
    elif ck.fmt == "fp16-bin":
        model.config.save_pretrained(root)
        sd = {k: v.half() for k, v in model.state_dict().items()}
        if ck.tied:
            del sd["lm_head.weight"]
        sd["model.layers.0.self_attn.rotary_emb.inv_freq"] = torch.ones(32)    # older .bin files keep this buffer
        torch.save(sd, root / "pytorch_model.bin")
    else:
        raise ValueError(ck.fmt)
    if ck.distinct_head:
        assert ck.fmt == "bf16" and ck.tied
        sd = load_file(str(root / "model.safetensors"))
        assert "lm_head.weight" not in sd
        g = torch.Generator().manual_seed(ck.seed + 1)
        sd["lm_head.weight"] = (torch.randn(ck.vocab, ck.hidden, generator=g) / math.sqrt(ck.hidden)).bfloat16()
        save_file(sd, str(root / "model.safetensors"), metadata={"format": "pt"})
    return root


def hf_model64(root: Path, family: str, bf16_weights: bool = False):
    """transformers' float64 model from ``root`` (eager attention); ``bf16_weights`` rounds every Linear and Embedding
    weight to bf16, as the engine streams them (norms and biases stay as stored)."""
    model = getattr(transformers, CLASSES[family][1]).from_pretrained(root, dtype=torch.float64, attn_implementation="eager")
    if bf16_weights:
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, (torch.nn.Linear, torch.nn.Embedding)):
                    m.weight.copy_(m.weight.bfloat16().double())
    return model.eval()


def oracle_of(model) -> tuple:
    """(lm_oracle.LMConfig, lm_oracle.LMWeights in fp32) read from a transformers model's state_dict, independently of
    pack_weights: absent q/k/v biases are zeros, the lm_head is whatever tensor the model's lm_head holds."""
    c = model.config
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    sd["lm_head.weight"] = model.lm_head.weight.detach().float()
    H, d = c.hidden_size, c.head_dim
    cfg = O.LMConfig(vocab_size=c.vocab_size, hidden_size=H, intermediate_size=c.intermediate_size,
                     num_layers=c.num_hidden_layers, num_heads=c.num_attention_heads, num_kv_heads=c.num_key_value_heads,
                     head_dim=d, rms_eps=c.rms_norm_eps, rope_theta=float(c.rope_parameters["rope_theta"]),
                     tie_embeddings=bool(torch.equal(sd["lm_head.weight"], sd["model.embed_tokens.weight"])))
    w = O.LMWeights(embed=sd["model.embed_tokens.weight"], final_norm=sd["model.norm.weight"], lm_head=sd["lm_head.weight"])
    for i in range(cfg.num_layers):
        p = f"model.layers.{i}."
        a = lambda n: sd[p + n]
        b = lambda n, rows: sd.get(p + n, torch.zeros(rows))
        w.layers.append(dict(
            ln1=a("input_layernorm.weight"), ln2=a("post_attention_layernorm.weight"),
            wq=a("self_attn.q_proj.weight"), bq=b("self_attn.q_proj.bias", cfg.num_heads * d),
            wk=a("self_attn.k_proj.weight"), bk=b("self_attn.k_proj.bias", cfg.num_kv_heads * d),
            wv=a("self_attn.v_proj.weight"), bv=b("self_attn.v_proj.bias", cfg.num_kv_heads * d),
            wo=a("self_attn.o_proj.weight"), wg=a("mlp.gate_proj.weight"), wu=a("mlp.up_proj.weight"),
            wd=a("mlp.down_proj.weight")))
    return cfg, w
