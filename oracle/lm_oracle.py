"""CPU oracle for hot path A (speech-LM prefill + decode + sampler).

TEST INFRASTRUCTURE ONLY.  Nothing under ``neutts_air_b200/``, ``neutts/`` or
``neuttsair/`` may import this module; only ``tests/``, ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs and ``__graft_entry__.smoke()`` do.

This is a plain-PyTorch fp32 restatement of the arithmetic the reference reaches
through ``neutts/neutts.py:334-352`` (``self.backbone.generate``), i.e. the
``transformers`` Qwen2 decoder and the HF sampling loop.  Each function cites the
file:line it follows (paths under ``site-packages/transformers`` are the
third-party module that holds the arithmetic; the reference pins
``transformers==4.56.1`` in ``requirements.txt:8``, this container has 5.5.0).

Pinning: ``oracle/make_golden.py`` runs this restatement against the real
``transformers.Qwen2ForCausalLM`` (eager attention, fp32) on seeded weights and
commits the resulting vectors under ``tests/golden/``; ``tests/test_oracle_lm.py``
re-checks both against the fixtures (and against transformers itself when it is
importable).  The reference's own tests pin no numerical result
(``tests/test_neutts.py:55-58`` only asserts type/finite), so the transformers
cross-check is the strongest pin available offline.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch


@dataclass
class LMConfig:
    """Shape of the decoder.  Defaults = NeuTTS-Air as inferred in SURVEY.md §8
    (Qwen2.5-0.5B base per TRAINING.md:33, vocab 151936 + 65536)."""

    vocab_size: int = 217472
    hidden_size: int = 896
    intermediate_size: int = 4864
    num_layers: int = 24
    num_heads: int = 14
    num_kv_heads: int = 2
    head_dim: int = 64
    rms_eps: float = 1e-6
    rope_theta: float = 1e6
    tie_embeddings: bool = True

    @staticmethod
    def tiny(**kw) -> "LMConfig":
        base = dict(vocab_size=512, hidden_size=128, intermediate_size=256, num_layers=2,
                    num_heads=2, num_kv_heads=1, head_dim=64)
        base.update(kw)
        return LMConfig(**base)


@dataclass
class LMWeights:
    """fp32 tensors in HF layout ([out, in] for every Linear)."""

    embed: torch.Tensor                      # [V, H]
    layers: list = field(default_factory=list)  # dicts: ln1, wq,bq, wk,bk, wv,bv, wo, ln2, wg, wu, wd
    final_norm: torch.Tensor = None          # [H]
    lm_head: torch.Tensor = None             # [V, H] (== embed when tied)


def random_weights(cfg: LMConfig, seed: int = 0, std: float = 0.02, bf16_round: bool = False) -> LMWeights:
    """HF default init (normal(0, 0.02), norms = 1); biases get the same normal so
    the bias path is exercised.  ``bf16_round`` rounds every matrix to bf16 values
    (kept in fp32) so the oracle and the bf16 kernel path see identical weights."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape):
        t = torch.randn(*shape, generator=g) * std
        return t.bfloat16().float() if bf16_round else t

    H, I, d = cfg.hidden_size, cfg.intermediate_size, cfg.head_dim
    w = LMWeights(embed=rn(cfg.vocab_size, H))
    for _ in range(cfg.num_layers):
        w.layers.append(dict(
            ln1=1.0 + rn(H), wq=rn(cfg.num_heads * d, H), bq=rn(cfg.num_heads * d),
            wk=rn(cfg.num_kv_heads * d, H), bk=rn(cfg.num_kv_heads * d),
            wv=rn(cfg.num_kv_heads * d, H), bv=rn(cfg.num_kv_heads * d),
            wo=rn(H, cfg.num_heads * d), ln2=1.0 + rn(H),
            wg=rn(I, H), wu=rn(I, H), wd=rn(H, I)))
    w.final_norm = 1.0 + rn(H)
    w.lm_head = w.embed if cfg.tie_embeddings else rn(cfg.vocab_size, H)
    return w


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """models/qwen2/modeling_qwen2.py:258-263 — fp32 variance, cast, then *weight."""
    var = x.float().pow(2).mean(-1, keepdim=True)
    return weight * (x.float() * torch.rsqrt(var + eps)).to(x.dtype)


def rope_cos_sin(positions: torch.Tensor, head_dim: int, theta: float):
    """modeling_qwen2.py:95-113 — inv_freq = theta^(-2i/d), emb = cat(freqs, freqs), fp32."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).float() / head_dim))
    freqs = positions.float()[..., None] * inv_freq          # [..., d/2]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """modeling_qwen2.py:116-146 — half-split rotation: x*cos + cat(-x2, x1)*sin.
    x: [..., T, heads, d]; cos/sin: [..., T, d]."""
    d = x.shape[-1]
    x1, x2 = x[..., : d // 2], x[..., d // 2:]
    rot = torch.cat((-x2, x1), dim=-1)
    return x * cos[..., None, :] + rot * sin[..., None, :]


def attention(q, k, v, causal_offset: int | None, n_rep: int, mma_bf16: bool = False):
    """modeling_qwen2.py:149-183 (eager path of record): repeat_kv, QK^T * d^-1/2,
    additive causal mask, fp32 softmax, PV.
    q: [Tq, Hq, d], k/v: [Tk, Hkv, d].  causal_offset = absolute position of q[0]
    minus position of k[0] (None = bidirectional).

    mma_bf16 (mirror of the CUDA tensor-core prefill kernel, not reference semantics): the query is
    scaled by d^-1/2 * log2(e) and rounded to bf16, the probabilities 2^(s - max) are rounded to bf16
    before P.V, the normaliser sums the unrounded probabilities."""
    Tq, Hq, d = q.shape
    Tk = k.shape[0]
    k = k.repeat_interleave(n_rep, dim=1)
    v = v.repeat_interleave(n_rep, dim=1)
    mask = None
    if causal_offset is not None:
        qi = torch.arange(Tq)[:, None] + causal_offset
        kj = torch.arange(Tk)[None, :]
        mask = kj > qi
    if mma_bf16:
        qs = (q * (d ** -0.5 * 1.4426950408889634)).bfloat16().float()
        s = torch.einsum("qhd,khd->hqk", qs, k)
        if mask is not None:
            s = s.masked_fill(mask, float("-inf"))
        pr = torch.exp2(s - s.max(dim=-1, keepdim=True).values)
        o = torch.einsum("hqk,khd->qhd", pr.bfloat16().float(), v)
        return o / pr.sum(dim=-1).T[:, :, None]
    s = torch.einsum("qhd,khd->hqk", q, k) * (d ** -0.5)
    if mask is not None:
        s = s.masked_fill(mask, float("-inf"))
    p = torch.softmax(s.float(), dim=-1).to(q.dtype)
    return torch.einsum("hqk,khd->qhd", p, v)


class KVCache:
    """cache_utils.py:88-121 DynamicLayer.update — concatenation along the sequence."""

    def __init__(self, num_layers: int):
        self.k = [None] * num_layers
        self.v = [None] * num_layers

    def update(self, layer: int, k: torch.Tensor, v: torch.Tensor):
        if self.k[layer] is None:
            self.k[layer], self.v[layer] = k, v
        else:
            self.k[layer] = torch.cat((self.k[layer], k), dim=0)
            self.v[layer] = torch.cat((self.v[layer], v), dim=0)
        return self.k[layer], self.v[layer]

    def length(self) -> int:
        return 0 if self.k[0] is None else self.k[0].shape[0]


def forward(cfg: LMConfig, w: LMWeights, ids: torch.Tensor, cache: KVCache | None = None,
            collect_hidden: bool = False, mirror: str | None = None, collect: dict | None = None,
            last_only: bool = False):
    """One sequence.  ids: int64 [T] (prompt for prefill, one id for a decode step).
    Follows Qwen2Model.forward modeling_qwen2.py:353-413 and the decoder layer
    :280-309 (pre-norm, residual add after attention and after the MLP); the
    lm_head (:475, tied :418) is applied to every position here and callers slice.

    ``mirror`` switches on the rounding points the CUDA path states in DESIGN.md, so
    the kernels can be checked to ~fp32 accuracy against their own specification (it is
    not part of the reference semantics; ``mirror=None`` is the reference):
      "decode"  (CUDA-core GEMV chain): K/V rounded to bf16 when cached, all else fp32;
      "decode_tc" (persistent wgmma decode kernel, batch <= 8): as "decode" (activations travel as bf16 hi + lo
                pairs, fp32-grade), but attention runs on bf16 tensor-core operands (scaled query, probabilities);
      "prefill" (tensor-core path): additionally the normalised activations, the
                attention output and the SwiGLU output are rounded to bf16 (GEMM A operands), and
                attention runs on bf16 tensor-core operands (scaled query and probabilities);
      "batched" (tensor-core decode, batch > 4): as "prefill" plus a bf16 lm_head input.

    ``last_only`` applies the lm_head to the last position only (what generate needs,
    modeling_qwen2.py:474-475 ``logits_to_keep``); full-size tests use it to skip a [T, V] product.

    Returns (logits [T, V] (or [1, V]), hiddens list or None).
    """
    cache = cache if cache is not None else KVCache(cfg.num_layers)
    past = cache.length()
    T = ids.shape[0]
    pos = torch.arange(past, past + T)
    cos, sin = rope_cos_sin(pos, cfg.head_dim, cfg.rope_theta)
    n_rep = cfg.num_heads // cfg.num_kv_heads
    assert mirror in (None, "decode", "decode_tc", "prefill", "batched")
    kv_round_bf16 = mirror is not None
    rb = (lambda t: t.bfloat16().float()) if mirror in ("prefill", "batched") else (lambda t: t)
    rb_head = (lambda t: t.bfloat16().float()) if mirror == "batched" else (lambda t: t)

    h = w.embed[ids]                                               # :367
    hiddens = [h.clone()] if collect_hidden else None
    for li, L in enumerate(w.layers):
        x = rb(rms_norm(h, L["ln1"], cfg.rms_eps))                 # :291
        q = (x @ L["wq"].T + L["bq"]).view(T, cfg.num_heads, cfg.head_dim)      # :217
        k = (x @ L["wk"].T + L["bk"]).view(T, cfg.num_kv_heads, cfg.head_dim)   # :218
        v = (x @ L["wv"].T + L["bv"]).view(T, cfg.num_kv_heads, cfg.head_dim)   # :219
        q = apply_rope(q, cos, sin)                                # :222
        k = apply_rope(k, cos, sin)
        if kv_round_bf16:
            k, v = k.bfloat16().float(), v.bfloat16().float()
        kk, vv = cache.update(li, k, v)                            # :225
        a = attention(q, kk, vv, causal_offset=past, n_rep=n_rep, mma_bf16=(mirror in ("prefill", "batched", "decode_tc")))  # :231
        a = rb(a.reshape(T, -1))
        h = h + a @ L["wo"].T                                      # :244, :302
        h_mid = h
        x = rb(rms_norm(h, L["ln2"], cfg.rms_eps))                 # :306
        act = torch.nn.functional.silu(x @ L["wg"].T) * (x @ L["wu"].T)  # :47
        h = h + rb(act) @ L["wd"].T                                # :308
        if collect is not None:
            collect[li] = dict(q=q.reshape(T, -1).clone(), k=k.clone(), v=v.clone(), attn=a.clone(),
                               h_mid=h_mid.clone(), act=rb(act).clone(), h=h.clone())
        if collect_hidden:
            hiddens.append(h.clone())
    hn = rms_norm(h[-1:] if last_only else h, w.final_norm, cfg.rms_eps)   # :409
    logits = rb_head(hn) @ w.lm_head.T                             # :475
    return logits, hiddens


# ----------------------------------------------------------------------------------------------
# sampler semantics (generation/logits_process.py:224-233, 296-299, 580-586; utils.py:2762-2805)
# ----------------------------------------------------------------------------------------------

def process_logits(logits: torch.Tensor, n_generated: int, eos_id: int, min_new_tokens: int,
                   temperature: float, top_k: int) -> torch.Tensor:
    """Processor order generation/utils.py:1134,1214,1219: MinNewTokensLength ->
    Temperature -> TopK.  logits: fp32 [V].  Returns filtered scores (−inf outside top-k)."""
    s = logits.float().clone()
    if n_generated < min_new_tokens:                 # logits_process.py:224-233
        s[eos_id] = float("-inf")
    s = s / temperature                              # :296-299
    k = min(top_k, s.shape[-1])                      # :580-586: remove scores < k-th largest
    kth = torch.topk(s, k).values[-1]
    return s.masked_fill(s < kth, float("-inf"))


def topk_probs(logits: torch.Tensor, n_generated: int, eos_id: int, min_new_tokens: int = 50,
               temperature: float = 1.0, top_k: int = 50):
    """Distribution torch.multinomial samples from at generation/utils.py:2789-2791:
    softmax of the processed scores.  Returns (token ids sorted by prob desc, probs)."""
    s = process_logits(logits, n_generated, eos_id, min_new_tokens, temperature, top_k)
    p = torch.softmax(s, dim=-1)
    idx = torch.nonzero(p > 0).flatten()
    order = torch.argsort(p[idx], descending=True, stable=True)
    return idx[order], p[idx][order]


def generate(cfg: LMConfig, w: LMWeights, prompt: torch.Tensor, eos_id: int, max_length: int = 2048,
             min_new_tokens: int = 50, temperature: float = 1.0, top_k: int = 50,
             max_new_tokens: int | None = None, seed: int = 0, forced: torch.Tensor | None = None,
             mirror: bool = False, decode_mirror: str | None = None):
    """The hot loop generation/utils.py:2743-2805 for one sequence: prefill, then
    decode one token at a time until EOS (after min_new_tokens) or max_length
    (prompt + generated, stopping_criteria.py:73-84).  ``forced`` teacher-forces
    the emitted tokens (for logits parity; sampling RNG streams cannot match).
    ``mirror`` applies the CUDA path's stated rounding points ("prefill" for the prompt, "decode" for the
    steps; ``decode_mirror="batched"`` selects the batch > 8 decode roundings instead).
    Returns (generated ids [N], per-step logits [N, V])."""
    g = torch.Generator().manual_seed(seed)
    cache = KVCache(cfg.num_layers)
    logits, _ = forward(cfg, w, prompt, cache, mirror="prefill" if mirror else None, last_only=True)
    step_logits, out = [], []
    cur = logits[-1]
    limit = max_length - prompt.shape[0]
    if max_new_tokens is not None:
        limit = min(limit, max_new_tokens)
    while len(out) < limit:
        step_logits.append(cur.clone())
        if forced is not None:
            tok = int(forced[len(out)])
        else:
            s = process_logits(cur, len(out), eos_id, min_new_tokens, temperature, top_k)
            tok = int(torch.multinomial(torch.softmax(s, -1), 1, generator=g))
        out.append(tok)
        if tok == eos_id and forced is None:
            break
        if len(out) >= limit:
            break
        logits, _ = forward(cfg, w, torch.tensor([tok]), cache,
                            mirror=decode_mirror if decode_mirror else ("decode" if mirror else None))
        cur = logits[-1]
    return torch.tensor(out, dtype=torch.int64), torch.stack(step_logits)


# ----------------------------------------------------------------------------------------------
# bridge to the real third-party implementation (used by make_golden.py, tests and the CPU baseline)
# ----------------------------------------------------------------------------------------------

def to_hf_model(cfg: LMConfig, w: LMWeights, attn_implementation: str = "eager"):
    """Build transformers.Qwen2ForCausalLM (what neutts/neutts.py:164 loads) holding ``w``."""
    from transformers import Qwen2Config, Qwen2ForCausalLM

    hf_cfg = Qwen2Config(
        vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
        num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.num_heads,
        num_key_value_heads=cfg.num_kv_heads, rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta,
        max_position_embeddings=32768, tie_word_embeddings=cfg.tie_embeddings,
        attn_implementation=attn_implementation, use_sliding_window=False)
    hf_cfg.head_dim = cfg.head_dim
    try:
        hf_cfg.rope_parameters = {"rope_type": "default", "rope_theta": cfg.rope_theta}
    except Exception:
        pass
    with torch.device("meta"):
        model = Qwen2ForCausalLM(hf_cfg)
    model = model.to_empty(device="cpu").float()
    sd = {"model.embed_tokens.weight": w.embed, "model.norm.weight": w.final_norm}
    for i, L in enumerate(w.layers):
        p = f"model.layers.{i}."
        sd.update({
            p + "input_layernorm.weight": L["ln1"], p + "post_attention_layernorm.weight": L["ln2"],
            p + "self_attn.q_proj.weight": L["wq"], p + "self_attn.q_proj.bias": L["bq"],
            p + "self_attn.k_proj.weight": L["wk"], p + "self_attn.k_proj.bias": L["bk"],
            p + "self_attn.v_proj.weight": L["wv"], p + "self_attn.v_proj.bias": L["bv"],
            p + "self_attn.o_proj.weight": L["wo"],
            p + "mlp.gate_proj.weight": L["wg"], p + "mlp.up_proj.weight": L["wu"],
            p + "mlp.down_proj.weight": L["wd"]})
    if not cfg.tie_embeddings:
        sd["lm_head.weight"] = w.lm_head
    missing, unexpected = model.load_state_dict(sd, strict=False, assign=True)
    assert not unexpected, unexpected
    if cfg.tie_embeddings:
        model.lm_head.weight = model.model.embed_tokens.weight
    # rotary inv_freq is a non-persistent buffer: rebuild it after to_empty()
    rot = model.model.rotary_emb
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, dtype=torch.int64).float() / cfg.head_dim))
    rot.inv_freq = inv
    if hasattr(rot, "original_inv_freq"):
        rot.original_inv_freq = inv.clone()
    return model.eval()


def speech_prompt(cfg: LMConfig, n_text: int, ref_codes: torch.Tensor, speech_base: int, seed: int = 0):
    """Synthetic prompt of SURVEY.md §8d: n_text uniform ids in the text range followed by
    speech_base + ref_codes (the layout neutts/neutts.py:303-332 produces)."""
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, max(1, min(151643, speech_base)), (n_text,), generator=g)
    return torch.cat((text, speech_base + ref_codes.long()))
