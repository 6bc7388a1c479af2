"""The speech-LM loader against checkpoints that transformers' own Qwen2, Llama and Mistral classes write.

``loader.load_speech_lm`` -> ``LMShape.from_hf_config`` -> ``lm.pack_weights`` is the route a real checkpoint takes to
the kernels; the other speech-LM tests build their engines from oracle weights and skip it.  Every checkpoint here is
written at test time by ``save_pretrained`` (or ``torch.save`` of the state_dict for an fp16 ``pytorch_model.bin``),
with weights that make loader faults visible: norm weights 1 + N(0, 0.1) and biases N(0, 0.1) (transformers' init
leaves 1 and 0, under which a swapped norm or a dropped bias changes nothing), q/k projections large enough for
attention scores of standard deviation > 2 (a peaked softmax, so a RoPE error moves the output), and embeddings of
std 0.005, so that ``mean(x^2)`` of the first layer's input is comparable to ``eps = 1e-5``.

CPU only: the config the loader reads against transformers' config object, the packed tensors against the checkpoint,
the oracle against transformers' float64 model for each family, every refusal (before any CUDA work), and a float64
check that each loader fault the GPU tests (test_gpu_loader_families.py) claim to catch moves the logits far past their
bars.
"""
from __future__ import annotations

import json
import math
from pathlib import Path

import pytest
import torch

pytest.importorskip("transformers")
import transformers  # noqa: E402

from neutts_air_b200 import loader  # noqa: E402
from neutts_air_b200.lm import LMShape, _rope_pair_perm, pack_weights  # noqa: E402
from oracle import lm_oracle as O  # noqa: E402
from tests.checkpoints import GPU_BARS, Ckpt, hf_model64, oracle_of, write_checkpoint  # noqa: E402
from tests.helpers import rel_rms  # noqa: E402


def edit_config(root: Path, fn) -> None:
    cfg = json.loads((root / "config.json").read_text())
    fn(cfg)
    (root / "config.json").write_text(json.dumps(cfg, indent=2))


def v4_layout(cfg: dict) -> None:
    """config.json as transformers 4 writes it: ``rope_theta`` at the top level, no ``rope_parameters``."""
    cfg["rope_theta"] = cfg.pop("rope_parameters")["rope_theta"]


def no_theta(cfg: dict) -> None:
    cfg.pop("rope_parameters", None)
    cfg.pop("rope_theta", None)


# ====================================================================================== float64 restatement
FAULTS = ("theta-1e6", "eps-1e-6", "ln1-ln2", "perm-q-only", "gate-up", "no-qkv-bias", "tied-head")


def forward64(cfg: O.LMConfig, w: O.LMWeights, ids, fault: str | None = None) -> dict:
    """The decoder in float64 over one sequence (causal), with one loader fault applied as the engine would compute it:
    the wrong theta / eps, ln1 and ln2 exchanged, k packed without the RoPE pair permutation (the kernel then rotates k's
    rows in the wrong pairs: k as if its rows were in the inverse permutation), gate and up exchanged, q/k/v biases
    dropped, or the embedding as lm_head.  Returns dict(logits [T, V], score_std: per layer)."""
    d, nh, nkv = cfg.head_dim, cfg.num_heads, cfg.num_kv_heads
    theta = 1e6 if fault == "theta-1e6" else cfg.rope_theta
    eps = 1e-6 if fault == "eps-1e-6" else cfg.rms_eps
    D = lambda t: t.double()
    ids = torch.as_tensor(ids, dtype=torch.long)
    T = ids.shape[0]
    inv = torch.argsort(_rope_pair_perm(nkv))
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64) / d))
    emb = torch.cat([torch.arange(T, dtype=torch.float64)[:, None] * inv_freq] * 2, dim=-1)
    cos, sin = emb.cos()[:, None, :], emb.sin()[:, None, :]
    rope = lambda x: x * cos + torch.cat((-x[..., d // 2:], x[..., : d // 2]), -1) * sin
    rms = lambda x, g: x / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + eps) * D(g)
    mask = torch.triu(torch.ones(T, T, dtype=torch.bool), 1)
    h = D(w.embed)[ids]
    stds = []
    for L in w.layers:
        ln1, ln2 = (L["ln2"], L["ln1"]) if fault == "ln1-ln2" else (L["ln1"], L["ln2"])
        wk, bk = D(L["wk"]), D(L["bk"])
        if fault == "perm-q-only":
            wk, bk = wk[inv], bk[inv]
        bq, bv = D(L["bq"]), D(L["bv"])
        if fault == "no-qkv-bias":
            bq, bk, bv = bq * 0, bk * 0, bv * 0
        x = rms(h, ln1)
        q = rope((x @ D(L["wq"]).T + bq).view(T, nh, d))
        k = rope((x @ wk.T + bk).view(T, nkv, d)).repeat_interleave(nh // nkv, 1)
        v = (x @ D(L["wv"]).T + bv).view(T, nkv, d).repeat_interleave(nh // nkv, 1)
        s = torch.einsum("qhd,khd->hqk", q, k) / math.sqrt(d)
        stds.append(float(s.masked_select(~mask).std()))
        a = torch.einsum("hqk,khd->qhd", torch.softmax(s.masked_fill(mask, -math.inf), -1), v).reshape(T, -1)
        h = h + a @ D(L["wo"]).T
        x = rms(h, ln2)
        wg, wu = (L["wu"], L["wg"]) if fault == "gate-up" else (L["wg"], L["wu"])
        h = h + (torch.nn.functional.silu(x @ D(wg).T) * (x @ D(wu).T)) @ D(L["wd"]).T
    head = w.embed if fault == "tied-head" else w.lm_head
    return dict(logits=rms(h, w.final_norm) @ D(head).T, score_std=stds)


# ====================================================================================== config
CONFIG_CASES = {
    "qwen2-tied": Ckpt("qwen2", tied=True, theta=1e6, eps=1e-6),
    "qwen2-distinct-head": Ckpt("qwen2", tied=True, distinct_head=True),
    "llama-untied": Ckpt("llama", theta=1e5, heads=4, kv=2, fmt="fp32-shards"),
    "llama-tied": Ckpt("llama", tied=True, theta=5e5, heads=4, kv=4),
    "mistral-untied": Ckpt("mistral", fmt="fp16-bin"),
}
LAYOUTS = {"v5": None, "v4": v4_layout, "no-theta": no_theta}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", list(CONFIG_CASES))
def test_config_matches_transformers(tmp_path, name, layout):
    """LMShape from config.json equals transformers' own config object (both config.json layouts, and with no theta
    at all), and the lm_head the loader keeps is the one ``from_pretrained`` uses."""
    ck = CONFIG_CASES[name]
    root = write_checkpoint(ck, tmp_path)
    if LAYOUTS[layout]:
        edit_config(root, LAYOUTS[layout])
    c = transformers.AutoConfig.from_pretrained(root)
    shape, sd = loader.read_speech_lm(str(root))
    want = (c.vocab_size, c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.num_attention_heads,
            c.num_key_value_heads, c.head_dim, c.rms_norm_eps, float(c.rope_parameters["rope_theta"]))
    got = (shape.vocab_size, shape.hidden_size, shape.intermediate_size, shape.num_layers, shape.num_heads,
           shape.num_kv_heads, shape.head_dim, shape.rms_eps, shape.rope_theta)
    assert got == want
    assert shape.rope_theta == (1e4 if layout == "no-theta" else ck.theta)
    assert LMShape.from_hf_config(json.loads((root / "config.json").read_text())).tie_embeddings == c.tie_word_embeddings
    model = hf_model64(root, ck.family)
    hf_tied = bool(torch.equal(model.lm_head.weight, model.model.embed_tokens.weight))
    assert shape.tie_embeddings == hf_tied == (ck.tied and not ck.distinct_head)
    pk = pack_weights(shape, sd, "cpu")
    assert torch.equal(pk["lm_head"].double(), model.lm_head.weight.bfloat16().double())


# ====================================================================================== packing
PACK_CASES = {
    "qwen2-bf16": Ckpt("qwen2", hidden=256, inter=640, heads=4, kv=2, theta=1e6),
    "llama-fp32-shards": Ckpt("llama", hidden=192, inter=384, heads=3, kv=3, fmt="fp32-shards"),
    "mistral-fp16-bin": Ckpt("mistral", hidden=256, inter=512, heads=4, kv=2, fmt="fp16-bin"),
}


@pytest.mark.parametrize("name", list(PACK_CASES))
def test_packing_undone_equals_the_checkpoint(tmp_path, name):
    """Undo pack_weights (the q/k RoPE pair permutation, the gate/up interleave, the qkv concatenation): every packed
    tensor equals the checkpoint tensor rounded to bf16 (fp32 for norms and biases), exactly, in every layer; absent
    biases come back as exact zeros."""
    ck = PACK_CASES[name]
    root = write_checkpoint(ck, tmp_path)
    shape, sd = loader.read_speech_lm(str(root))
    pk = pack_weights(shape, sd, "cpu")
    ref = {k: v.detach().float() for k, v in hf_model64(root, ck.family).state_dict().items()}
    bf = lambda t: t.bfloat16()
    nq, nk = 64 * ck.heads, 64 * ck.kv
    iq, ik = torch.argsort(_rope_pair_perm(ck.heads)), torch.argsort(_rope_pair_perm(ck.kv))
    for i in range(ck.layers):
        p = f"model.layers.{i}."
        wqkv, bqkv = pk["wqkv"][i], pk["bqkv"][i]
        assert wqkv.dtype == torch.bfloat16 and bqkv.dtype == torch.float32 and wqkv.shape[0] == nq + 2 * nk
        parts = {"q": (wqkv[:nq][iq], bqkv[:nq][iq]), "k": (wqkv[nq: nq + nk][ik], bqkv[nq: nq + nk][ik]),
                 "v": (wqkv[nq + nk:], bqkv[nq + nk:])}
        for n, (wt, bt) in parts.items():
            assert torch.equal(wt, bf(ref[p + f"self_attn.{n}_proj.weight"])), (i, n)
            bias = ref.get(p + f"self_attn.{n}_proj.bias")
            assert torch.equal(bt, bias if bias is not None else torch.zeros(bt.shape[0])), (i, n)
            assert (bias is not None) == (ck.family == "qwen2")
        gu = pk["wgu"][i].view(ck.inter, 2, ck.hidden)
        assert torch.equal(gu[:, 0], bf(ref[p + "mlp.gate_proj.weight"])) and torch.equal(gu[:, 1], bf(ref[p + "mlp.up_proj.weight"]))
        assert torch.equal(pk["wo"][i], bf(ref[p + "self_attn.o_proj.weight"]))
        assert torch.equal(pk["wd"][i], bf(ref[p + "mlp.down_proj.weight"]))
        assert pk["ln1"][i].dtype == torch.float32 and torch.equal(pk["ln1"][i], ref[p + "input_layernorm.weight"])
        assert torch.equal(pk["ln2"][i], ref[p + "post_attention_layernorm.weight"])
    assert torch.equal(pk["embed"], bf(ref["model.embed_tokens.weight"]))
    assert torch.equal(pk["final_norm"], ref["model.norm.weight"])
    assert torch.equal(pk["lm_head"], bf(ref["lm_head.weight"])) and pk["lm_head"] is not pk["embed"]


# ====================================================================================== oracle per family
ORACLE_CASES = {f"{fam}-theta{int(th)}-{'tied' if tied else 'untied'}": Ckpt(fam, theta=th, tied=tied, heads=4, kv=2,
                                                                              hidden=256, inter=512, seed=3)
                for fam in ("llama", "mistral") for th in (1e4, 1e5) for tied in (True, False)}
ORACLE_CASES["qwen2-theta1000000-tied"] = Ckpt("qwen2", theta=1e6, eps=1e-6, tied=True, heads=4, kv=2, hidden=256, inter=512)


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_oracle_matches_transformers_per_family(tmp_path, name):
    """lm_oracle.forward (fp32, mirror=None) on weights read from the checkpoint equals transformers' float64 model on
    the same directory, and so does the float64 restatement here; attention is peaked."""
    ck = ORACLE_CASES[name]
    root = write_checkpoint(ck, tmp_path)
    model = hf_model64(root, ck.family)
    cfg, w = oracle_of(model)
    ids = torch.randint(0, ck.vocab, (150,), generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        ref = model(ids[None]).logits[0]
    got = O.forward(cfg, w, ids)[0]
    f64 = forward64(cfg, w, ids)
    e, e64 = rel_rms(got, ref), rel_rms(f64["logits"], ref)
    print(f"ORACLE {name}: fp32 oracle {e:.2e}, float64 restatement {e64:.2e}, score std {min(f64['score_std']):.2f}")
    # transformers' float64 model still takes its RMSNorm and its RoPE tables in fp32, hence ~3e-6 for both
    assert e < 1e-5, e
    assert e64 < 1e-5, e64
    assert min(f64["score_std"]) > 2


# ====================================================================================== refusals
def _qwen2_moe():
    return Ckpt("qwen2_moe", extra=(("num_experts", 4), ("num_experts_per_tok", 2), ("moe_intermediate_size", 64),
                                    ("shared_expert_intermediate_size", 64)))


def _rename_arch(cfg):
    cfg["architectures"] = ["LlamaForCausalLMWithValueHead"]


def _partial_rotary(cfg):
    cfg["rope_parameters"]["partial_rotary_factor"] = 0.5


def _rope_scaling_v4(cfg):
    v4_layout(cfg)
    cfg["rope_scaling"] = {"type": "linear", "factor": 2.0}


# (id, checkpoint, config edit, max_ctx, match)
REFUSALS = [
    ("qwen3", Ckpt("qwen3"), None, 2048, "Qwen3ForCausalLM"),
    ("qwen2-moe", _qwen2_moe(), None, 2048, "Qwen2MoeForCausalLM"),
    ("renamed-architecture", Ckpt("llama"), _rename_arch, 2048, "LlamaForCausalLMWithValueHead"),
    ("llama-attention-bias", Ckpt("llama", extra=(("attention_bias", True),)), None, 2048, r"o_proj\.bias"),
    ("llama-mlp-bias", Ckpt("llama", extra=(("mlp_bias", True),)), None, 2048, r"gate_proj\.bias"),
    ("llama-gelu", Ckpt("llama", extra=(("hidden_act", "gelu"),)), None, 2048, "hidden_act"),
    ("llama3-rope", Ckpt("llama", extra=(("rope_parameters", dict(
        rope_type="llama3", rope_theta=5e5, factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
        original_max_position_embeddings=256)),)), None, 2048, "rope_type"),
    ("linear-rope-v4", Ckpt("llama"), _rope_scaling_v4, 2048, "rope_scaling"),
    ("partial-rotary", Ckpt("llama"), _partial_rotary, 2048, "partial_rotary_factor"),
    ("mistral-window-64", Ckpt("mistral", extra=(("sliding_window", 64),)), None, 2048, "sliding_window"),
    ("mistral-window-4096-ctx-8192", Ckpt("mistral"), None, 8192, "sliding_window"),
    ("qwen2-sliding-window", Ckpt("qwen2", extra=(("use_sliding_window", True), ("sliding_window", 64),
                                                  ("max_window_layers", 0))), None, 2048, "sliding_window"),
    ("untied-without-lm-head", Ckpt("llama", fmt="fp16-bin", tied=True),
     lambda c: c.update(tie_word_embeddings=False), 2048, "lm_head"),
    ("no-tie-key-without-lm-head", Ckpt("llama", tied=True), lambda c: c.pop("tie_word_embeddings"), 2048, "lm_head"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_loader_refuses(tmp_path, case):
    """load_speech_lm raises ValueError naming the key or setting, before any CUDA work, for every checkpoint the
    kernels would compute differently than transformers does."""
    _, ck, edit, max_ctx, match = case
    root = write_checkpoint(ck, tmp_path)
    if edit:
        edit_config(root, edit)
    with pytest.raises(ValueError, match=match):
        loader.load_speech_lm(str(root), device="cpu", max_ctx=max_ctx)


ACCEPTED = [
    ("mistral-window-4096-ctx-2048", Ckpt("mistral"), 2048),
    ("mistral-window-64-ctx-64", Ckpt("mistral", extra=(("sliding_window", 64),)), 64),
    ("qwen2-sliding-above-the-last-layer", Ckpt("qwen2", extra=(("use_sliding_window", True), ("sliding_window", 64),
                                                                ("max_window_layers", 3))), 2048),
]


@pytest.mark.parametrize("case", ACCEPTED, ids=[c[0] for c in ACCEPTED])
def test_loader_accepts_windows_that_do_not_bind(tmp_path, case):
    """A window no shorter than the engine's context, or one no layer uses, changes nothing: the checkpoint loads."""
    _, ck, max_ctx = case
    root = write_checkpoint(ck, tmp_path)
    shape, sd = loader.read_speech_lm(str(root), max_ctx)
    pack_weights(shape, sd, "cpu")


def test_pack_weights_refuses_unused_tensors():
    """pack_weights accounts for every tensor under model. and lm_head.: an extra layer, an o_proj bias or a q_norm is
    refused with its name; rotary inv_freq buffers and names outside those prefixes are ignored."""
    from tests.helpers import lm_state_dict

    cfg = O.LMConfig.tiny()
    w = O.random_weights(cfg, 0)
    shape = LMShape(cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_layers, cfg.num_heads, cfg.num_kv_heads)
    sd = lm_state_dict(w, tied=False)
    sd["model.layers.0.self_attn.rotary_emb.inv_freq"] = torch.ones(32)
    sd["optimizer.step"] = torch.zeros(1)
    pack_weights(shape, sd, "cpu")
    for extra in ("model.layers.2.input_layernorm.weight", "model.layers.1.self_attn.o_proj.bias",
                  "model.layers.0.self_attn.q_norm.weight", "lm_head.bias"):
        with pytest.raises(ValueError, match=extra.replace(".", r"\.")):
            pack_weights(shape, {**sd, extra: torch.zeros(4)}, "cpu")


# ====================================================================================== sensitivity
SENSITIVITY_CASES = {
    "qwen2-biases-untied": Ckpt("qwen2", hidden=256, inter=640, heads=4, kv=2, theta=1e5, seed=5),
    "llama-nano-heads": Ckpt("llama", hidden=576, inter=1536, heads=9, kv=3, theta=1e5, seed=6),
    "mistral-untied": Ckpt("mistral", hidden=256, inter=640, heads=4, kv=2, theta=1e4, seed=7),
}


@pytest.mark.parametrize("name", list(SENSITIVITY_CASES))
def test_loader_faults_exceed_the_gpu_bars(tmp_path, name):
    """float64: each loader fault moves the logits past the GPU bars.  On a 71-token sequence (the 1-token-prompt
    decode cases) by at least 10x the mirrored bar and 4x the bar against transformers; on a 300-token sequence (the
    ragged cases) by at least 4x their widest relative-RMS bar.  Faults that cannot apply to a checkpoint (biases it
    lacks) are skipped."""
    ck = SENSITIVITY_CASES[name]
    root = write_checkpoint(ck, tmp_path)
    cfg, w = oracle_of(hf_model64(root, ck.family))
    g = torch.Generator().manual_seed(11)
    lines = []
    for T, bars in ((71, (10 * GPU_BARS["decode-only"], 4 * GPU_BARS["decode-only-reference"])),
                    (300, (4 * max(v for k, v in GPU_BARS.items() if k != "reference-max"),))):
        ids = torch.randint(0, ck.vocab, (T,), generator=g)
        exact = forward64(cfg, w, ids)["logits"]
        for fault in FAULTS:
            if fault == "no-qkv-bias" and ck.family != "qwen2":
                continue
            e = rel_rms(forward64(cfg, w, ids, fault)["logits"], exact)
            lines.append(f"T{T} {fault} {e:.2e}")
            assert e > max(bars), (T, fault, e)
    print(f"FAULTS {name}: " + "; ".join(lines))
