"""Checkpoint readers (SURVEY.md §8f N2): HF safetensors / .bin -> the packed device layouts.

Nothing here is exercised against the real ``neuphonic/*`` checkpoints in this environment (offline,
no cache); the Qwen2 reader is tested against checkpoints written by ``transformers.save_pretrained``
and the codec reader against a state_dict laid out with the upstream ``neucodec`` names.
"""
from __future__ import annotations

import json
import os
from pathlib import Path

import torch

from .codec import CodecDecoder, CodecShape
from .lm import LMShape, SpeechLM


def resolve_repo(repo: str) -> Path:
    """Local directory, or a snapshot in the HF cache (offline: ``local_files_only``)."""
    p = Path(str(repo))
    if p.exists():
        return p
    try:
        from huggingface_hub import snapshot_download

        return Path(snapshot_download(str(repo), local_files_only=bool(os.environ.get("HF_HUB_OFFLINE"))))
    except Exception as e:  # no network / not cached
        raise FileNotFoundError(f"checkpoint {repo!r} is neither a local directory nor available from the HF hub: {e}") from e


def read_state_dict(root: Path) -> dict:
    files = sorted(root.glob("*.safetensors"))
    sd: dict = {}
    if files:
        from safetensors.torch import load_file

        for f in files:
            sd.update(load_file(str(f)))
        return sd
    for name in ("pytorch_model.bin", "model.bin", "model.pt"):
        if (root / name).exists():
            return torch.load(root / name, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no safetensors / pytorch_model.bin under {root}")


def load_tokenizer(repo: str):
    from transformers import AutoTokenizer

    return AutoTokenizer.from_pretrained(str(resolve_repo(repo)))


def load_speech_lm(repo: str, device="cuda", **kw) -> SpeechLM:
    """``AutoModelForCausalLM.from_pretrained`` replacement (neutts/neutts.py:163-166): config.json decides
    every dimension (NeuTTS-Nano and Air differ), weights are cast to bf16."""
    root = resolve_repo(repo)
    cfg = json.loads((root / "config.json").read_text())
    arch = (cfg.get("architectures") or ["Qwen2ForCausalLM"])[0]
    # the kernels implement the pre-norm RMSNorm / RoPE (half-split) / GQA / SwiGLU decoder that Qwen2, Llama and
    # Mistral share; q/k/v biases are optional (absent in Llama-style checkpoints -> zeros)
    family = ("Qwen2", "Llama", "Mistral", "Qwen3")
    if not any(f in arch for f in family) and cfg.get("model_type") not in ("qwen2", "llama", "mistral"):
        raise ValueError(f"unsupported backbone architecture {arch!r}: the sm_90a kernels implement the "
                         f"Qwen2/Llama-family decoder (RMSNorm, RoPE, GQA, SwiGLU)")
    if cfg.get("rope_scaling") not in (None, {}) and (cfg["rope_scaling"] or {}).get("rope_type", "default") != "default":
        raise ValueError("scaled RoPE variants are not implemented")
    sd = read_state_dict(root)
    shape = LMShape.from_hf_config(cfg)
    # tied embeddings: trust the tensors, not a missing config key (a real lm_head must not be dropped silently)
    if "lm_head.weight" in sd and "model.embed_tokens.weight" in sd:
        same = sd["lm_head.weight"].shape == sd["model.embed_tokens.weight"].shape and bool(
            torch.equal(sd["lm_head.weight"], sd["model.embed_tokens.weight"]))
        shape.tie_embeddings = same
    elif "lm_head.weight" not in sd:
        shape.tie_embeddings = True
    return SpeechLM(shape, sd, device=device, **kw)


# ---- NeuCodec decoder: upstream module names (neucodec / XCodec2 lineage) -> oracle-style dict ----
_RES = (("norm1.weight", "n1w"), ("norm1.bias", "n1b"), ("conv1.weight", "c1w"), ("conv1.bias", "c1b"),
        ("norm2.weight", "n2w"), ("norm2.bias", "n2b"), ("conv2.weight", "c2w"), ("conv2.bias", "c2b"))


def codec_weights_from_state_dict(sd: dict) -> tuple:
    """Returns (CodecShape, weights dict).  Keys follow the upstream decoder:
    ``generator.quantizer.project_out.*`` (or ``...quantizer.layers.0.project_out``), ``fc_post_a.*``,
    ``generator.backbone.{embed,prior_net.N,transformers.N,post_net.N,final_layer_norm}.*``,
    ``generator.head.out.*``."""
    def find(*cands):
        for c in cands:
            if c in sd:
                return sd[c]
        raise KeyError(f"none of {cands} in codec checkpoint")

    bb = "generator.backbone."
    w = dict(
        project_out_w=find("generator.quantizer.project_out.weight", "generator.quantizer.fsqs.0.project_out.weight"),
        project_out_b=find("generator.quantizer.project_out.bias", "generator.quantizer.fsqs.0.project_out.bias"),
        fc_post_a_w=find("fc_post_a.weight"), fc_post_a_b=find("fc_post_a.bias"),
        embed_w=find(bb + "embed.weight"), embed_b=find(bb + "embed.bias"),
        final_ln_w=find(bb + "final_layer_norm.weight"), final_ln_b=find(bb + "final_layer_norm.bias"),
        head_w=find("generator.head.out.weight"), head_b=find("generator.head.out.bias"))
    for grp, key in (("prior_net", "prior"), ("post_net", "post")):
        w[key] = [{short: sd[f"{bb}{grp}.{i}.{long}"] for long, short in _RES} for i in range(2)]
    depth = 1 + max(int(k.split(".")[3]) for k in sd if k.startswith(bb + "transformers."))
    w["blocks"] = [dict(att_norm=sd[f"{bb}transformers.{i}.att_norm.weight"], wqkv=sd[f"{bb}transformers.{i}.att.c_attn.weight"],
                        wproj=sd[f"{bb}transformers.{i}.att.c_proj.weight"], ffn_norm=sd[f"{bb}transformers.{i}.ffn_norm.weight"],
                        fc1=sd[f"{bb}transformers.{i}.mlp.fc1.weight"], fc2=sd[f"{bb}transformers.{i}.mlp.fc2.weight"])
                   for i in range(depth)]
    hidden = w["embed_w"].shape[0]
    n_fft = w["head_w"].shape[0] - 2
    shape = CodecShape(fsq_dims=w["project_out_w"].shape[1], quant_dim=w["project_out_w"].shape[0], hidden=hidden, depth=depth,
                       heads=hidden // 64, mlp_mult=w["blocks"][0]["fc1"].shape[0] // hidden,
                       embed_kernel=w["embed_w"].shape[2], n_fft=n_fft, hop=n_fft // 4,
                       rope_axis=os.environ.get("NEUTTS_CODEC_ROPE_AXIS", "head"))
    return shape, w


def load_codec_decoder(repo: str, device="cuda", **kw) -> CodecDecoder:
    root = resolve_repo(repo)
    shape, w = codec_weights_from_state_dict(read_state_dict(root))
    dec = CodecDecoder(shape, w, device=device, **kw)
    dec.repo = str(repo)     # encode_code() delegates to neucodec.from_pretrained(repo)
    return dec
