"""Seeded synthetic weights at the (inferred) NeuTTS-Air / NeuCodec shapes.

No checkpoint, tokenizer or codec source exists offline (SURVEY.md fact 2), so benchmarks and the
smoke test run on these.  Plain tensors only: the LM comes out as an HF-named Qwen2 state_dict, the
codec as the dict layout ``codec.pack_weights`` consumes.  Both arms of bench.py (the GPU and the CPU
reference) are built from the same tensors.
"""
from __future__ import annotations

import math

import torch


def lm_state_dict(shape, seed: int = 0, dtype=torch.bfloat16, std: float = 0.02) -> dict:
    """transformers' default init: N(0, 0.02) matrices and biases, unit norms."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: (torch.randn(*s, generator=g) * std).to(dtype)
    H, I, d = shape.hidden_size, shape.intermediate_size, shape.head_dim
    sd = {"model.embed_tokens.weight": rn(shape.vocab_size, H), "model.norm.weight": torch.ones(H)}
    for i in range(shape.num_layers):
        p = f"model.layers.{i}."
        sd.update({
            p + "input_layernorm.weight": torch.ones(H), p + "post_attention_layernorm.weight": torch.ones(H),
            p + "self_attn.q_proj.weight": rn(shape.num_heads * d, H), p + "self_attn.q_proj.bias": rn(shape.num_heads * d),
            p + "self_attn.k_proj.weight": rn(shape.num_kv_heads * d, H), p + "self_attn.k_proj.bias": rn(shape.num_kv_heads * d),
            p + "self_attn.v_proj.weight": rn(shape.num_kv_heads * d, H), p + "self_attn.v_proj.bias": rn(shape.num_kv_heads * d),
            p + "self_attn.o_proj.weight": rn(H, shape.num_heads * d),
            p + "mlp.gate_proj.weight": rn(I, H), p + "mlp.up_proj.weight": rn(I, H), p + "mlp.down_proj.weight": rn(H, I)})
    if not getattr(shape, "tie_embeddings", True):
        sd["lm_head.weight"] = rn(shape.vocab_size, H)
    return sd


def codec_weights(shape, seed: int = 0) -> dict:
    """Scales keep activations O(1) through the stack and give the PCM a speech-like level
    (RMS ~0.1, no clip at mag 1e2), so the 1e-3 RMS parity bar is meaningful."""
    g = torch.Generator().manual_seed(seed)
    C = shape.hidden
    rn = lambda *s, std: torch.randn(*s, generator=g) * std
    lin = lambda o, i, gain=1.0: rn(o, i, std=gain / math.sqrt(i))

    def resnet():
        return dict(n1w=1.0 + rn(C, std=0.05), n1b=rn(C, std=0.05), c1w=rn(C, C, 3, std=1.0 / math.sqrt(3 * C)), c1b=rn(C, std=0.02),
                    n2w=1.0 + rn(C, std=0.05), n2b=rn(C, std=0.05), c2w=rn(C, C, 3, std=0.5 / math.sqrt(3 * C)), c2b=rn(C, std=0.02))

    w = dict(project_out_w=lin(shape.quant_dim, shape.fsq_dims, 1.5), project_out_b=rn(shape.quant_dim, std=0.1),
             fc_post_a_w=lin(C, shape.quant_dim), fc_post_a_b=rn(C, std=0.05),
             embed_w=rn(C, C, shape.embed_kernel, std=1.0 / math.sqrt(shape.embed_kernel * C)), embed_b=rn(C, std=0.02))
    w["prior"] = [resnet() for _ in range(2)]
    w["blocks"] = [dict(att_norm=1.0 + rn(C, std=0.05), wqkv=lin(3 * C, C, 1.5), wproj=lin(C, C, 0.5), ffn_norm=1.0 + rn(C, std=0.05),
                        fc1=lin(shape.mlp_mult * C, C), fc2=lin(C, shape.mlp_mult * C, 0.5)) for _ in range(shape.depth)]
    w["post"] = [resnet() for _ in range(2)]
    w["final_ln_w"], w["final_ln_b"] = 1.0 + rn(C, std=0.05), rn(C, std=0.05)
    nb = shape.n_fft // 2 + 1
    hw, hb = lin(2 * nb, C), torch.zeros(2 * nb)
    hw[:nb] *= 0.5
    hb[:nb] = 2.5 - 3.5 * torch.linspace(0, 1, nb)
    hw[nb:] *= 2.0
    w["head_w"], w["head_b"] = hw, hb
    return w
