"""Shared test plumbing: oracle weights -> HF-style state dicts -> CUDA engines."""
from __future__ import annotations

import math

import torch

from oracle import codec_oracle, lm_oracle


def lm_state_dict(w: lm_oracle.LMWeights, tied: bool = True) -> dict:
    sd = {"model.embed_tokens.weight": w.embed, "model.norm.weight": w.final_norm}
    for i, L in enumerate(w.layers):
        p = f"model.layers.{i}."
        sd.update({
            p + "input_layernorm.weight": L["ln1"], p + "post_attention_layernorm.weight": L["ln2"],
            p + "self_attn.q_proj.weight": L["wq"], p + "self_attn.q_proj.bias": L["bq"],
            p + "self_attn.k_proj.weight": L["wk"], p + "self_attn.k_proj.bias": L["bk"],
            p + "self_attn.v_proj.weight": L["wv"], p + "self_attn.v_proj.bias": L["bv"],
            p + "self_attn.o_proj.weight": L["wo"], p + "mlp.gate_proj.weight": L["wg"],
            p + "mlp.up_proj.weight": L["wu"], p + "mlp.down_proj.weight": L["wd"]})
    if not tied:
        sd["lm_head.weight"] = w.lm_head
    return sd


def lm_shape(cfg: lm_oracle.LMConfig):
    from neutts_air_b200.lm import LMShape

    return LMShape(cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_layers, cfg.num_heads,
                   cfg.num_kv_heads, cfg.head_dim, cfg.rms_eps, cfg.rope_theta, cfg.tie_embeddings)


def make_lm(cfg, w, **kw):
    from neutts_air_b200.lm import SpeechLM

    return SpeechLM(lm_shape(cfg), lm_state_dict(w, cfg.tie_embeddings), device="cuda:0", **kw)


def codec_shape(cfg: codec_oracle.CodecConfig):
    from neutts_air_b200.codec import CodecShape

    return CodecShape(cfg.fsq_levels, cfg.fsq_dims, cfg.quant_dim, cfg.hidden, cfg.depth, cfg.heads, cfg.head_dim,
                      cfg.mlp_mult, cfg.groups, cfg.embed_kernel, cfg.n_fft, cfg.hop, cfg.rope_base, cfg.rope_axis,
                      cfg.norm_eps, cfg.mag_clip)


def codec_weight_dict(w: codec_oracle.CodecWeights) -> dict:
    return dict(project_out_w=w.project_out_w, project_out_b=w.project_out_b, fc_post_a_w=w.fc_post_a_w,
                fc_post_a_b=w.fc_post_a_b, embed_w=w.embed_w, embed_b=w.embed_b, prior=w.prior, post=w.post,
                blocks=w.blocks, final_ln_w=w.final_ln_w, final_ln_b=w.final_ln_b, head_w=w.head_w, head_b=w.head_b)


def make_codec(cfg, w, **kw):
    from neutts_air_b200.codec import CodecDecoder

    return CodecDecoder(codec_shape(cfg), codec_weight_dict(w), device="cuda:0", **kw)


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def rel_rms(got, ref) -> float:
    """Relative RMS error; inf when ``got`` holds a NaN or an inf (so that max() over errors cannot drop it)."""
    if not torch.isfinite(got).all():
        return math.inf
    return float((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-300))


def gather_kv(lm, layer: int, b: int, n: int):
    """Rows 0..n-1 of slot ``b``'s K and V in layer ``layer``, read through ``lm.page_table`` from the paged pool
    ``lm.kv[layer, 0|1, page, kv_head, row, :]`` (pages of 64 rows).  Returns two float64 CPU tensors [n, n_kv, 64]."""
    page = lm.kv.shape[-2]
    npg = (n + page - 1) // page
    pages = lm.page_table[b, :npg].to(device=lm.kv.device, dtype=torch.long)
    out = []
    for which in (0, 1):
        t = lm.kv[layer, which].index_select(0, pages)                     # [npg, n_kv, 64, 64]
        out.append(t.permute(0, 2, 1, 3).reshape(npg * page, t.shape[1], 64)[:n].double().cpu())
    return out[0], out[1]
