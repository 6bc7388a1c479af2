"""Checkpoint readers (SURVEY.md §8f N2): HF safetensors / .bin -> the packed device layouts.

The speech-LM reader takes Qwen2, Llama and Mistral checkpoints and refuses, before any CUDA work, every config or
tensor the kernels would compute differently than transformers does (``check_lm_config``, ``lm.check_tensors``).
It is tested end to end against checkpoints that transformers' own classes write (bf16 and sharded fp32 safetensors,
fp16 ``pytorch_model.bin``; tests/test_loader_families.py on the CPU, tests/test_gpu_loader_families.py through the
kernels); the real ``neuphonic/*`` checkpoints are not available offline.  The codec reader is tested against a
state_dict laid out with the upstream ``neucodec`` names.
"""
from __future__ import annotations

import json
import os
from pathlib import Path

import torch

from .codec import CodecDecoder, CodecShape
from .lm import LMShape, SpeechLM, check_tensors


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


# the kernels implement the pre-norm RMSNorm / RoPE (half-split) / GQA / SwiGLU decoder that these three share; q/k/v
# biases are optional (absent in Llama and Mistral checkpoints -> zeros)
ARCHITECTURES = {"Qwen2ForCausalLM": "qwen2", "LlamaForCausalLM": "llama", "MistralForCausalLM": "mistral"}


def _binding_window(cfg: dict) -> int | None:
    """The attention window some layer of the transformers model attends within, or None when every layer attends to
    its whole context.  ``layer_types`` (transformers 5) names the sliding layers; without it Qwen2 slides from layer
    ``max_window_layers`` on when ``use_sliding_window`` is set, and Mistral slides in every layer."""
    window = cfg.get("sliding_window")
    if window is None:
        return None
    if cfg.get("layer_types") is not None:
        return window if "sliding_attention" in cfg["layer_types"] else None
    if cfg.get("model_type") == "qwen2":
        slides = cfg.get("use_sliding_window", False) and cfg.get("max_window_layers", 28) < cfg["num_hidden_layers"]
        return window if slides else None
    return window


def check_lm_config(cfg: dict, max_ctx: int) -> None:
    """Raises ValueError, naming the key, for a config.json whose model the kernels would compute differently than
    transformers does: another architecture, scaled or partial RoPE, an activation other than SiLU, or an attention
    window shorter than the engine's context ``max_ctx``."""
    archs = cfg.get("architectures") or []
    mtype = cfg.get("model_type")
    # one allowlisted family, named by the architecture, the model_type or both (and then the same one)
    families = {ARCHITECTURES.get(a) for a in archs} | ({mtype} if mtype is not None else set())
    if len(families) != 1 or not families <= set(ARCHITECTURES.values()):
        raise ValueError(f"unsupported backbone (architectures={archs!r}, model_type={mtype!r}): the sm_90a kernels "
                         f"implement {', '.join(ARCHITECTURES)} (RMSNorm, RoPE, GQA, SwiGLU)")
    for key in ("rope_scaling", "rope_parameters"):
        rope = cfg.get(key) or {}
        kind = rope.get("rope_type", rope.get("type", "default"))
        if kind != "default":
            raise ValueError(f"{key}.rope_type = {kind!r}: scaled RoPE variants are not implemented")
        if float(rope.get("partial_rotary_factor", 1.0)) != 1.0:
            raise ValueError(f"{key}.partial_rotary_factor = {rope['partial_rotary_factor']}: partial RoPE is not implemented")
    if float(cfg.get("partial_rotary_factor", 1.0)) != 1.0:
        raise ValueError(f"partial_rotary_factor = {cfg['partial_rotary_factor']}: partial RoPE is not implemented")
    act = cfg.get("hidden_act", "silu")
    if act != "silu":
        raise ValueError(f"hidden_act = {act!r}: the MLP kernels compute SwiGLU (silu)")
    window = _binding_window(cfg)
    if window is not None and window < max_ctx:
        raise ValueError(f"sliding_window = {window} < max_ctx = {max_ctx}: the attention kernels attend to the whole "
                         f"context; load with max_ctx <= {window}")


def read_speech_lm(repo: str, max_ctx: int = 2048) -> tuple:
    """Everything ``load_speech_lm`` does short of the device: (LMShape, state_dict) of a checked checkpoint.

    The lm_head follows the tensors the way ``from_pretrained`` does: an ``lm_head.weight`` in the checkpoint is used
    even under ``tie_word_embeddings = true`` (shared with the embedding only when equal to it); without one the head
    is the embedding, and an untied config without one is refused (transformers would initialise a random head)."""
    root = resolve_repo(repo)
    cfg = json.loads((root / "config.json").read_text())
    check_lm_config(cfg, max_ctx)
    sd = read_state_dict(root)
    shape = LMShape.from_hf_config(cfg)
    check_tensors(shape, sd)
    if "lm_head.weight" in sd:
        shape.tie_embeddings = sd["lm_head.weight"].shape == sd["model.embed_tokens.weight"].shape and bool(
            torch.equal(sd["lm_head.weight"], sd["model.embed_tokens.weight"]))
    elif not shape.tie_embeddings:
        raise ValueError("tie_word_embeddings is false (or absent) and the checkpoint has no lm_head.weight")
    return shape, sd


def load_speech_lm(repo: str, device="cuda", **kw) -> SpeechLM:
    """``AutoModelForCausalLM.from_pretrained`` replacement (neutts/neutts.py:163-166) for Qwen2, Llama and Mistral
    checkpoints: config.json decides every dimension (NeuTTS-Nano and Air differ), weights are cast to bf16.  Every
    refusal of ``read_speech_lm`` happens before any CUDA work."""
    shape, sd = read_speech_lm(repo, kw.get("max_ctx", 2048))
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
