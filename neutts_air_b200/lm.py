"""Speech-LM engine on the C-ABI: weight packing, paged KV pool, prefill + device-side decode loop.

Host-side mirror of inner seam 1 of the reference (``neutts/neutts.py:334-352``): an object with
``.device`` and ``.generate(LongTensor[1,P], max_length=, eos_token_id=, do_sample=, temperature=,
top_k=, use_cache=, min_new_tokens=) -> LongTensor[1,P+N]``, plus a batched ``generate_batch``.
All arithmetic happens in ``libneutts_b200.so``; torch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from collections import Counter
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib


@dataclass
class LMShape:
    """Decoder shape; read from the checkpoint's config.json at load time (never hard-coded:
    SURVEY.md §8).  Defaults = NeuTTS-Air as inferred from TRAINING.md:33 / README.md:44-45."""

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
    def from_hf_config(cfg: dict) -> "LMShape":
        """The shape a transformers config.json describes, read as transformers' Qwen2 / Llama / Mistral config classes
        read it: ``rope_theta`` from ``rope_parameters`` (transformers 5) or the top level (transformers 4), else
        10 000; ``tie_word_embeddings`` false when absent (the checkpoint's tensors may still tie: loader.py)."""
        rope = cfg.get("rope_theta")
        if rope is None and isinstance(cfg.get("rope_parameters"), dict):
            rope = cfg["rope_parameters"].get("rope_theta")
        heads = cfg["num_attention_heads"]
        return LMShape(
            vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"], intermediate_size=cfg["intermediate_size"],
            num_layers=cfg["num_hidden_layers"], num_heads=heads,
            num_kv_heads=cfg.get("num_key_value_heads") or heads,
            head_dim=cfg.get("head_dim") or cfg["hidden_size"] // heads,
            rms_eps=cfg.get("rms_norm_eps", 1e-6), rope_theta=float(rope if rope is not None else 1e4),
            tie_embeddings=bool(cfg.get("tie_word_embeddings", False)))


def _rope_pair_perm(n_heads: int) -> torch.Tensor:
    """Row order that puts RoPE partners (i, i+32) of every 64-row head next to each other."""
    one = torch.stack((torch.arange(32), torch.arange(32) + 32), dim=1).reshape(-1)
    return (torch.arange(n_heads)[:, None] * 64 + one[None, :]).reshape(-1)


_LAYER_TENSORS = ("input_layernorm.weight", "post_attention_layernorm.weight", "self_attn.q_proj.weight",
                  "self_attn.q_proj.bias", "self_attn.k_proj.weight", "self_attn.k_proj.bias", "self_attn.v_proj.weight",
                  "self_attn.v_proj.bias", "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
                  "mlp.down_proj.weight")


def check_tensors(shape: LMShape, sd: dict) -> None:
    """Raises ValueError listing the names under ``model.`` and ``lm_head.`` that ``pack_weights`` would not read: an
    o_proj or MLP bias, per-head q/k norms, a layer beyond ``num_layers``.  The kernels have no place for them, so a
    checkpoint holding one describes a different model.  ``rotary_emb.inv_freq`` buffers (older .bin files) are
    derived from the config and ignored."""
    known = {"model.embed_tokens.weight", "model.norm.weight", "lm_head.weight"}
    known.update(f"model.layers.{i}.{n}" for i in range(shape.num_layers) for n in _LAYER_TENSORS)
    extra = sorted(k for k in sd if k.startswith(("model.", "lm_head.")) and k not in known
                   and not k.endswith("rotary_emb.inv_freq"))
    if extra:
        raise ValueError(f"checkpoint tensors the speech-LM kernels do not implement: {', '.join(extra[:8])}"
                         + (f" (+{len(extra) - 8} more)" if len(extra) > 8 else ""))


def pack_weights(shape: LMShape, sd: dict, device) -> dict:
    """HF Qwen2 / Llama / Mistral state_dict (``model.layers.N.self_attn.q_proj.weight`` ...) -> the packed bf16/fp32
    device tensors the kernels stream (layouts documented in include/neutts_b200.h).  Raises ValueError when the
    state_dict holds a tensor the kernels would not use (``check_tensors``)."""
    check_tensors(shape, sd)
    dev = torch.device(device)
    bf = lambda t: t.to(device=dev, dtype=torch.bfloat16).contiguous()
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
    pq = _rope_pair_perm(shape.num_heads)
    pk = _rope_pair_perm(shape.num_kv_heads)
    g = lambda k: sd[k]
    out = dict(ln1=[], wqkv=[], bqkv=[], wo=[], ln2=[], wgu=[], wd=[])
    for i in range(shape.num_layers):
        p = f"model.layers.{i}."
        wq, wk, wv = g(p + "self_attn.q_proj.weight"), g(p + "self_attn.k_proj.weight"), g(p + "self_attn.v_proj.weight")
        zb = lambda w_: torch.zeros(w_.shape[0], dtype=torch.float32)     # Llama-style checkpoints carry no q/k/v bias
        bq = sd.get(p + "self_attn.q_proj.bias", None)
        bk = sd.get(p + "self_attn.k_proj.bias", None)
        bv = sd.get(p + "self_attn.v_proj.bias", None)
        bq, bk, bv = (bq if bq is not None else zb(wq)), (bk if bk is not None else zb(wk)), (bv if bv is not None else zb(wv))
        out["wqkv"].append(bf(torch.cat((wq[pq], wk[pk], wv), dim=0)))
        out["bqkv"].append(f32(torch.cat((bq.float()[pq], bk.float()[pk], bv.float()), dim=0)))
        out["wo"].append(bf(g(p + "self_attn.o_proj.weight")))
        wg, wu = g(p + "mlp.gate_proj.weight"), g(p + "mlp.up_proj.weight")
        out["wgu"].append(bf(torch.stack((wg, wu), dim=1).reshape(2 * wg.shape[0], wg.shape[1])))
        out["wd"].append(bf(g(p + "mlp.down_proj.weight")))
        out["ln1"].append(f32(g(p + "input_layernorm.weight")))
        out["ln2"].append(f32(g(p + "post_attention_layernorm.weight")))
    out["embed"] = bf(g("model.embed_tokens.weight"))
    if shape.tie_embeddings or "lm_head.weight" not in sd:
        out["lm_head"] = out["embed"]
    else:
        out["lm_head"] = bf(g("lm_head.weight"))
    out["final_norm"] = f32(g("model.norm.weight"))
    return out


class PagePool:
    """Free-list allocator over the KV page ids (host side; one id addresses every layer).  Every allocated page has a
    reference count: several slots may hold one page (the takes of one prompt share its full prompt pages), and a
    page returns to the free list when its last holder releases it."""

    def __init__(self, num_pages: int, shuffle_seed: int | None = None):
        order = list(range(num_pages))
        if shuffle_seed is not None:
            rng = np.random.default_rng(shuffle_seed)
            rng.shuffle(order)
        self.free = order[::-1]
        self.refs = [0] * num_pages

    @property
    def num_free(self) -> int:
        """Pages no slot holds."""
        return len(self.free)

    def alloc(self, n: int) -> list:
        if n > len(self.free):
            raise RuntimeError(f"KV page pool exhausted: need {n}, have {len(self.free)}")
        pages = [self.free.pop() for _ in range(n)]
        for p in pages:
            self.refs[p] = 1
        return pages

    def _check_held(self, pages, verb: str) -> list:
        pages = list(pages)
        for p, k in Counter(pages).items():
            if not 0 <= p < len(self.refs) or self.refs[p] < k:
                raise ValueError(f"cannot {verb} page {p}: it is held {self.refs[p] if 0 <= p < len(self.refs) else 0} "
                                 f"time(s), asked {k}")
        return pages

    def share(self, pages) -> None:
        """One more reference to each of ``pages`` (allocated ones only)."""
        for p in self._check_held(pages, "share"):
            self.refs[p] += 1

    def release(self, pages) -> None:
        """Drops one reference to each of ``pages``; a page whose count reaches zero is free again."""
        freed = []
        for p in self._check_held(pages, "release"):
            self.refs[p] -= 1
            if self.refs[p] == 0:
                freed.append(p)
        self.free.extend(reversed(freed))


DEFAULT_CONTROLS = (1.0, 50, 1.0, 0.0)   # temperature, top_k, top_p, min_p: the reference's (neutts/neutts.py:338-347)


def per_item(n: int, noun: str, **values) -> dict:
    """Each keyword a scalar (kept as it is) or a sequence with one value per ``noun`` (made a list of Python
    scalars); raises ValueError for a sequence of another length."""
    out = {}
    for name, v in values.items():
        if isinstance(v, (list, tuple, np.ndarray, torch.Tensor)):
            v = [x.item() if hasattr(x, "item") else x for x in v]
            if len(v) != n:
                raise ValueError(f"{name} needs one value per {noun} ({n}), got {len(v)}")
        out[name] = v
    return out


def _rows(n: int, cols: dict):
    """The n rows of ``per_item``'s columns (a scalar repeats in every row)."""
    return zip(*(v if isinstance(v, list) else [v] * n for v in cols.values()))


def check_controls(temperature, top_k, top_p, min_p) -> tuple:
    """One slot's sampling controls, validated as ``nt_lm_set_slot_sampling`` does -> (float, int, float, float)."""
    t, p, m = float(temperature), float(top_p), float(min_p)
    if not (math.isfinite(t) and t > 0):
        raise ValueError(f"temperature {temperature} must be finite and > 0")
    if int(top_k) != top_k or not 1 <= int(top_k) <= 64:
        raise ValueError(f"top_k {top_k} must be an integer in 1..64")
    if not 0 < p <= 1:
        raise ValueError(f"top_p {top_p} must be in (0, 1]")
    if not 0 <= m < 1:
        raise ValueError(f"min_p {min_p} must be in [0, 1)")
    return t, int(top_k), p, m


def per_prompt_controls(n: int, temperature, top_k, top_p, min_p):
    """Sampling controls of n prompts.  Each control is a scalar or a sequence with one value per prompt.  Returns None
    when every control is a scalar and top-p / min-p are off (``sampling``'s scalars then govern, exactly as without
    per-slot controls), else one validated (temperature, top_k, top_p, min_p) per prompt."""
    cols = per_item(n, "prompt", temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p)
    if not any(isinstance(v, list) for v in cols.values()) and top_p == 1 and min_p == 0:
        return None
    return [check_controls(*row) for row in _rows(n, cols)]


def check_vocab_range(vocab_range, vocab_size: int):
    """A vocabulary range (lo, hi), validated as ``nt_lm_set_vocab_range`` does -> (int, int); None -> None (off).
    Rules: 0 <= lo < hi <= vocab_size, hi - lo >= 64 (top_k <= 64 always finds k allowed ids), lo % 128 == 0 and
    hi % 128 == 0 unless hi == vocab_size."""
    if vocab_range is None:
        return None
    lo, hi = vocab_range
    if not all(isinstance(v, (int, float, np.integer)) for v in (lo, hi)) or int(lo) != lo or int(hi) != hi:
        raise ValueError(f"vocab range {vocab_range} must be two integers")
    lo, hi = int(lo), int(hi)
    if not 0 <= lo < hi <= vocab_size:
        raise ValueError(f"vocab range [{lo}, {hi}) not inside [0, {vocab_size})")
    if hi - lo < 64:
        raise ValueError(f"vocab range [{lo}, {hi}) holds fewer than 64 ids")
    if lo % 128 or (hi % 128 and hi != vocab_size):
        raise ValueError(f"vocab range [{lo}, {hi}): lo must be a multiple of 128, hi too unless it is {vocab_size}")
    return lo, hi


def check_takes(n_prompts: int, n, max_batch: int) -> int:
    """Takes per prompt (``num_return_sequences``), validated: an integer >= 1 with n_prompts * n <= max_batch."""
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError(f"num_return_sequences {n!r} must be an integer >= 1")
    if n_prompts * int(n) > max_batch:
        raise ValueError(f"{n_prompts} prompt(s) x {int(n)} takes need {n_prompts * int(n)} slots; the engine has {max_batch}")
    return int(n)


def fork_slots(n_prompts: int, n: int, slot_base: int = 0) -> list:
    """(prompt, take, slot, Philox stream key) of every slot ``prefill_fork`` fills: take j of prompt i in slot i * n + j
    (transformers' repeat_interleave order), drawing from stream slot + slot_base."""
    return [(i, j, i * n + j, i * n + j + slot_base) for i in range(n_prompts) for j in range(n)]


def score_starts(lens, start) -> list:
    """The start of every sequence ``score`` takes: ``start`` is an int or one value per sequence, each in 1..L - 1."""
    starts = per_item(len(lens), "sequence", start=start)["start"]
    starts = starts if isinstance(starts, list) else [starts] * len(lens)
    out = []
    for b, (L, s) in enumerate(zip(lens, starts)):
        if isinstance(s, bool) or int(s) != s or not 1 <= int(s) < L:
            raise ValueError(f"sequence {b}: start {s!r} must be an integer in 1..{L - 1} (its length is {L})")
        out.append(int(s))
    return out


def pack_score_calls(lens, max_batch: int, max_tokens: int, max_ctx: int) -> list:
    """Sequences of lengths ``lens`` packed greedily, in input order, into ``nt_lm_score`` calls of at most
    ``max_batch`` sequences and ``max_tokens`` tokens -> a list of index lists.  A sequence longer than ``max_ctx`` or
    ``max_tokens`` fits no call and raises ValueError."""
    calls, cur, tok = [], [], 0
    for i, L in enumerate(lens):
        if L > max_ctx or L > max_tokens:
            raise ValueError(f"sequence {i} has {L} tokens; one scoring call takes at most {min(max_ctx, max_tokens)}")
        if cur and (len(cur) == max_batch or tok + L > max_tokens):
            calls.append(cur)
            cur, tok = [], 0
        cur.append(i)
        tok += L
    if cur:
        calls.append(cur)
    return calls


DEFAULT_PENALTY = (1.0, True)   # repetition penalty, prompt included: transformers' RepetitionPenaltyLogitsProcessor


def check_penalty(penalty, include_prompt=True) -> tuple:
    """One slot's repetition penalty, validated as ``nt_lm_set_repetition_penalty`` does -> (float, bool).  The penalty
    must be finite and > 0 in fp32 (1 = none); ``include_prompt``: the prompt's ids count (transformers' default)."""
    if isinstance(penalty, bool) or not isinstance(penalty, (int, float, np.integer, np.floating)):
        raise ValueError(f"repetition penalty {penalty!r} must be a number")
    p = float(penalty)
    with np.errstate(over="ignore"):
        f = float(np.float32(p)) if math.isfinite(p) else p   # the value the library stores
    if not (math.isfinite(f) and f > 0):
        raise ValueError(f"repetition penalty {penalty} must be finite and > 0")
    if not isinstance(include_prompt, (bool, int, np.integer, np.bool_)) or int(include_prompt) not in (0, 1):
        raise ValueError(f"penalize_prompt {include_prompt!r} must be a bool")
    return p, bool(include_prompt)


def per_prompt_penalty(n: int, penalty, include_prompt):
    """Repetition penalties of n prompts, each argument a scalar or one value per prompt.  Returns None when every
    penalty is 1 (nothing to penalise: no engine call), else one validated (penalty, include_prompt) per prompt."""
    cols = per_item(n, "prompt", repetition_penalty=penalty, penalize_prompt=include_prompt)
    rows = [check_penalty(p, i) for p, i in _rows(n, cols)]
    return None if all(r[0] == 1.0 for r in rows) else rows


DEFAULT_LENGTH = (50, 49, 1.0)   # min_new_tokens, decay start, decay factor: the reference's floor, no decay


def _is_int(v) -> bool:
    return not isinstance(v, (bool, np.bool_)) and isinstance(v, (int, np.integer))


def check_length(min_new_tokens, decay_start, decay_factor, max_new: int | None = None) -> tuple:
    """One slot's length control, validated as ``nt_lm_set_length_control`` does -> (int, int, float):
    ``min_new_tokens`` >= 0 (transformers' MinNewTokensLengthLogitsProcessor), ``decay_start`` >= 0 and >=
    min_new_tokens - 1 (the decay never meets the mask's -inf, which transformers would turn into NaN) and
    ``decay_factor`` finite and > 0, 1 = no decay (ExponentialDecayLengthPenalty).  ``max_new``: also refuse a decay
    whose c_k = pow(factor, k) - 1 is not finite in fp32 for some k <= max_new - decay_start, as every launch does."""
    if not _is_int(min_new_tokens) or min_new_tokens < 0:
        raise ValueError(f"min_new_tokens {min_new_tokens!r} must be an integer >= 0")
    if not _is_int(decay_start) or decay_start < 0:
        raise ValueError(f"exponential_decay_length_penalty start {decay_start!r} must be an integer >= 0")
    if isinstance(decay_factor, bool) or not isinstance(decay_factor, (int, float, np.integer, np.floating)):
        raise ValueError(f"exponential_decay_length_penalty factor {decay_factor!r} must be a number")
    f = float(decay_factor)
    if not (math.isfinite(f) and f > 0):
        raise ValueError(f"exponential_decay_length_penalty factor {decay_factor} must be finite and > 0")
    if decay_start < min_new_tokens - 1:
        raise ValueError(f"exponential_decay_length_penalty start {decay_start} must be >= min_new_tokens - 1 = "
                         f"{min_new_tokens - 1}: the decay would meet the -inf of the min_new_tokens mask")
    k = (max_new or 0) - int(decay_start)
    if f > 1 and k >= 1:   # c_k grows with k: the largest reachable one decides
        try:
            c = pow(f, k) - 1
        except OverflowError:
            c = math.inf
        with np.errstate(over="ignore"):
            if not math.isfinite(float(np.float32(c))):
                raise ValueError(f"exponential_decay_length_penalty factor {f} overflows fp32 within {k} steps "
                                 f"after its start (pow({f}, {k}) - 1)")
    return int(min_new_tokens), int(decay_start), f


def per_prompt_decay(n: int, decay) -> list:
    """``exponential_decay_length_penalty`` of n prompts: None, one (start, factor) pair, or one None / pair per
    prompt -> a list of n entries."""
    pair = lambda d: isinstance(d, (list, tuple)) and len(d) == 2 and all(
        isinstance(x, (int, float, np.integer, np.floating)) and not isinstance(x, bool) for x in d)
    if decay is None or pair(decay):
        return [decay] * n
    if isinstance(decay, (list, tuple)) and len(decay) == n and all(d is None or pair(d) for d in decay):
        return list(decay)
    raise ValueError(f"exponential_decay_length_penalty must be None, one (start, factor) pair, or one of those per "
                     f"prompt ({n}); got {decay!r}")


def per_prompt_length(n: int, min_new_tokens, decay, max_new: int | None = None):
    """Length control of n prompts: ``min_new_tokens`` an int or one per prompt, ``decay`` as ``per_prompt_decay``.
    Returns None when ``min_new_tokens`` is one int and no prompt decays (the launch scalar then governs, exactly as without
    the table), else one validated (min_new_tokens, decay_start, decay_factor) per prompt (``check_length``; a prompt
    without decay gets factor 1 and start max(min_new_tokens - 1, 0))."""
    floors = per_item(n, "prompt", min_new_tokens=min_new_tokens)["min_new_tokens"]
    decays = per_prompt_decay(n, decay)
    if not isinstance(floors, list):
        check_length(floors, max(floors - 1, 0) if _is_int(floors) else 0, 1.0)
        if all(d is None for d in decays):
            return None
        floors = [floors] * n
    return [check_length(m, *(d if d is not None else (max(m - 1, 0) if _is_int(m) else 0, 1.0)), max_new=max_new)
            for m, d in zip(floors, decays)]


RAS_OFF = (0, 0)   # (window, min_count) of a slot without repetition-aware sampling
RAS_MAX_WINDOW = 64   # the generated tokens each slot keeps on the device for its window


def check_ras(win_size, tau_r) -> tuple:
    """One prompt's repetition-aware sampling (VALL-E 2's RAS, CosyVoice 2's ``ras_sampling(win_size, tau_r)``),
    validated as ``nt_lm_set_repetition_aware_sampling`` does -> the slot entry (window, min_count).  ``win_size``: an
    int in 1..64, the generated tokens the window looks back over; ``tau_r``: finite in (0, 1], not a bool.  A draw
    is redrawn from the whole distribution when it occurs at least ``min_count = ceil(win_size * tau_r)`` times in the
    window (float64, exactly CosyVoice's ``rep_num >= win_size * tau_r``)."""
    if not _is_int(win_size) or not 1 <= win_size <= RAS_MAX_WINDOW:
        raise ValueError(f"repetition_aware_sampling win_size {win_size!r} must be an integer in 1..{RAS_MAX_WINDOW}")
    if isinstance(tau_r, (bool, np.bool_)) or not isinstance(tau_r, (int, float, np.integer, np.floating)):
        raise ValueError(f"repetition_aware_sampling tau_r {tau_r!r} must be a number")
    t = float(tau_r)
    if not (math.isfinite(t) and 0 < t <= 1):
        raise ValueError(f"repetition_aware_sampling tau_r {tau_r} must be finite and in (0, 1]")
    return int(win_size), int(math.ceil(int(win_size) * t))


def ras_entry(row) -> tuple:
    """The slot entry of one prompt's setting: None -> ``RAS_OFF``, a (win_size, tau_r) pair -> ``check_ras``."""
    if row is None:
        return RAS_OFF
    if not isinstance(row, (list, tuple)) or len(row) != 2:
        raise ValueError(f"repetition_aware_sampling must be None or one (win_size, tau_r) pair; got {row!r}")
    return check_ras(*row)


def per_prompt_ras(n: int, ras):
    """``repetition_aware_sampling`` of n prompts: None, one (win_size, tau_r) pair, or one None / pair per prompt.
    Returns None when no prompt has it (no engine call), else one validated pair (a tuple) or None per prompt."""
    pair = lambda r: isinstance(r, (list, tuple)) and len(r) == 2 and not any(isinstance(x, (list, tuple)) or x is None
                                                                             for x in r)
    if ras is None:
        return None
    if pair(ras):
        rows = [tuple(ras)] * n
    elif isinstance(ras, (list, tuple)) and len(ras) == n and all(r is None or pair(r) for r in ras):
        rows = [None if r is None else tuple(r) for r in ras]
    else:
        raise ValueError(f"repetition_aware_sampling must be None, one (win_size, tau_r) pair, or one None / pair per "
                         f"prompt ({n}); got {ras!r}")
    for r in rows:
        ras_entry(r)
    return None if all(r is None for r in rows) else rows


NO_GUIDANCE = (-1, 1.0)   # (partner, scale) of a slot outside every guided pair


def check_guidance_scale(scale) -> float:
    """One prompt's ``guidance_scale``: a number, finite and > 0 in fp32 (the value the library stores) -> float.
    1 means no guidance, as in transformers, which adds no processor then."""
    if isinstance(scale, bool) or not isinstance(scale, (int, float, np.integer, np.floating)):
        raise ValueError(f"guidance_scale {scale!r} must be a number")
    g = float(scale)
    with np.errstate(over="ignore"):
        f = float(np.float32(g)) if math.isfinite(g) else g
    if not (math.isfinite(f) and f > 0):
        raise ValueError(f"guidance_scale {scale} must be finite and > 0")
    return g if f != 1.0 else 1.0


def check_guidance_table(table, max_batch: int) -> list:
    """A whole slot table of (partner, scale) entries, validated as ``nt_lm_set_guidance`` does -> a list of
    (int, float): partner -1 or another slot in 0..max_batch - 1; a partner serves one slot and has no partner of its
    own; scale finite, > 0 and != 1 (in fp32) wherever partner >= 0."""
    table = [(int(p), float(g)) for p, g in table]
    if len(table) != max_batch:
        raise ValueError(f"the guidance table needs {max_batch} entries, got {len(table)}")
    served = {}
    for s, (p, g) in enumerate(table):
        if not (p == -1 or (0 <= p < max_batch and p != s)):
            raise ValueError(f"slot {s}: partner {p} must be -1 or another slot in 0..{max_batch - 1}")
        if p < 0:
            continue
        if check_guidance_scale(g) == 1.0:
            raise ValueError(f"slot {s}: guidance scale {g} must be != 1")
        if p in served:
            raise ValueError(f"slot {p} is the partner of both slot {served[p]} and slot {s}")
        if table[p][0] >= 0:
            raise ValueError(f"slot {s}: its partner {p} has a partner of its own")
        served[p] = s
    return table


def per_prompt_guidance(prompts, guidance_scale, negative_prompt_ids):
    """Guidance of the prompts: ``guidance_scale`` a number or one per prompt, ``negative_prompt_ids`` None or one id
    list per prompt (None entries: transformers' default, the prompt's last token).  Returns None when no prompt is
    guided (scale 1), else one (scale, negative prompt) per prompt, (1.0, None) for an unguided one."""
    n = len(prompts)
    scales = per_item(n, "prompt", guidance_scale=guidance_scale)["guidance_scale"]
    scales = [check_guidance_scale(g) for g in (scales if isinstance(scales, list) else [scales] * n)]
    if negative_prompt_ids is None:
        negs = [None] * n
    elif isinstance(negative_prompt_ids, (list, tuple)) and len(negative_prompt_ids) == n:
        negs = [None if q is None else [int(t) for t in (q.tolist() if hasattr(q, "tolist") else q)]
                for q in negative_prompt_ids]
    else:
        raise ValueError(f"negative_prompt_ids must be None or one id list per prompt ({n})")
    if all(g == 1.0 for g in scales):
        return None
    out = []
    for p, g, q in zip(prompts, scales, negs):
        if g == 1.0:
            out.append((1.0, None))
            continue
        if q is not None and len(q) == 0:
            raise ValueError("an empty negative prompt gives the unconditional sequence nothing to start from")
        out.append((g, list(q) if q is not None else [int(p[-1])]))
    return out


def guided_layout(n: int, guidance) -> list:
    """(c slot, u slot, scale) of every guided prompt of a batch: prompt i in slot i, the unconditional sequences in
    slots n, n + 1, ... in prompt order, so that unguided prompts keep their slots and Philox streams."""
    if guidance is None:
        return []
    pairs = [(i, g) for i, (g, _) in enumerate(guidance) if g != 1.0]
    return [(i, n + k, g) for k, (i, g) in enumerate(pairs)]


def guided_caps(caps, guidance, max_ctx: int) -> list:
    """The generated-token cap of every prompt with guidance: a guided pair stops together, so its cap is
    min(c's cap, max_ctx - len(negative prompt)).  A negative prompt that leaves no room raises ValueError."""
    out = list(caps)
    for i, (g, neg) in enumerate(guidance or []):
        if g == 1.0:
            continue
        room = max_ctx - len(neg)
        if room < 1:
            raise ValueError(f"prompt {i}: its negative prompt of {len(neg)} tokens leaves no room in the context of {max_ctx}")
        out[i] = min(out[i], room)
    return out


@dataclass
class Settings:
    """The per-prompt generation settings of one call, resolved and validated before any engine call
    (``resolve_settings``)."""

    controls: list | None      # one (temperature, top_k, top_p, min_p) per prompt; None: the launch scalars govern
    penalty: list | None       # one (penalty, include_prompt) per prompt; None: no penalty
    vocab_range: tuple | None  # (lo, hi); None: the whole vocabulary
    temperature: float         # the launch scalars, taken from the first row while the controls table is on (the
    top_k: int                 # sampler then reads every slot's own row)
    logprobs: bool = False     # per-token log-probabilities on (``SpeechLM.set_logprobs``)
    length: list | None = None # one (min_new_tokens, decay_start, decay_factor) per prompt; None: the launch scalar
    min_new_tokens: int = 50   # the launch scalar, row 0's while the length table is on
    guidance: list | None = None  # one (partner slot, scale) per slot of the prefill (NO_GUIDANCE outside a pair);
                                  # None: guidance off
    ras: list | None = None    # one (win_size, tau_r) or None per prompt; None: repetition-aware sampling off

    def floors(self, n: int) -> list:
        """The min_new_tokens of each of the n prompts."""
        return [r[0] for r in self.length] if self.length is not None else [self.min_new_tokens] * n

    def apply(self, lm, n: int) -> None:
        """Before a prefill of prompts 0..n-1 into slots 0..n-1, on its stream: controls, then range, then penalty, then
        length control, then repetition-aware sampling, then log-probabilities.  Each setting is applied, or switched off when an earlier call left it on, or makes no call when it is off and
        stays off.  ``lm`` needs the ``set_*`` methods only when a call is due; a missing mirror counts as off."""
        if self.controls is not None or getattr(lm, "_slot_sp_host", None) is not None:
            lm.set_slot_sampling(None if self.controls is None else self.controls[:n])
        if self.vocab_range is not None:
            lm.set_vocab_range(*self.vocab_range)
        elif getattr(lm, "_vocab_range", None) is not None:
            lm.set_vocab_range(None)
        if self.penalty is not None or getattr(lm, "_penalty_host", None) is not None:
            lm.set_repetition_penalty(None if self.penalty is None else self.penalty[:n])
        if self.length is not None or getattr(lm, "_length_host", None) is not None:
            lm.set_length_control(None if self.length is None else self.length[:n])
        if self.ras is not None or getattr(lm, "_ras_host", None) is not None:
            lm.set_repetition_aware_sampling(None if self.ras is None else self.ras[:n])
        if self.logprobs != (getattr(lm, "logprobs", None) is not None):
            lm.set_logprobs(self.logprobs)
        if self.guidance is not None:   # the whole table: no pair of an earlier call survives
            lm.set_guidance(self.guidance[:n] + [NO_GUIDANCE] * (lm.max_batch - n))
        elif getattr(lm, "_guidance_host", None) is not None:
            lm.set_guidance(None)

    def pair(self, pairs, n: int | None = None) -> "Settings":
        """The settings of a batch with guided pairs ((c, u, scale) from ``guided_layout``): the u slots, above the
        prompts in pair order, repeat their c's rows (they are never sampled, but every launch checks their entries),
        and ``guidance`` holds the table of every slot.  ``n``: the batch holds only the first n prompts (a queue's
        first wave of a call with guidance); their table is on even without a pair."""
        if n is None:
            if not pairs:
                return self
            n = pairs[0][1]
        rows = lambda r: None if r is None else list(r[:n]) + [r[c] for c, _, _ in pairs]
        table = [NO_GUIDANCE] * (n + len(pairs))
        for c, u, g in pairs:
            table[c] = (u, g)
        return dataclasses.replace(self, controls=rows(self.controls), penalty=rows(self.penalty), length=rows(self.length),
                                   ras=rows(self.ras), guidance=table)

    def repeat(self, n: int) -> "Settings":
        """The settings of n takes of every prompt: each prompt's row repeated n times, in slot order (take j of prompt
        i in slot i * n + j), so that ``apply`` writes it into all of the prompt's take slots."""
        rows = lambda r: None if r is None else [x for x in r for _ in range(n)]
        return dataclasses.replace(self, controls=rows(self.controls), penalty=rows(self.penalty), length=rows(self.length),
                                   ras=rows(self.ras))

    def admit(self, lm, slots, idx, guide=None) -> None:
        """Before a refill of prompts ``idx`` into ``slots``: writes their rows; every other slot keeps its own, and
        the range holds.  ``guide`` (queue with guidance): {slot: (partner, scale)} for the refilled slots (a pair's u
        slot is in ``slots`` with its prompt's index repeated in ``idx``) and every slot freed since the last refill."""
        if self.controls is not None:
            lm.set_slot_sampling([self.controls[i] for i in idx], slots=slots)
        if self.penalty is not None:
            lm.set_repetition_penalty([self.penalty[i] for i in idx], slots=slots)
        if self.length is not None:
            lm.set_length_control([self.length[i] for i in idx], slots=slots)
        if self.ras is not None:
            lm.set_repetition_aware_sampling([self.ras[i] for i in idx], slots=slots)
        if guide is not None:
            lm.set_guidance(list(guide.values()), slots=list(guide))


def resolve_settings(lm, n: int, temperature=1.0, top_k=50, top_p=1.0, min_p=0.0, vocab_range=None,
                     repetition_penalty=1.0, penalize_prompt=True, logprobs=False, min_new_tokens=50,
                     exponential_decay_length_penalty=None, max_new: int | None = None,
                     repetition_aware_sampling=None) -> Settings:
    """The settings of n prompts on engine ``lm``, each control a scalar or one value per prompt
    (``per_prompt_controls``, ``per_prompt_penalty``, ``per_prompt_length``, ``per_prompt_ras``,
    ``check_vocab_range``; ``lm.shape`` is read only for a range).  ``max_new``: the call's largest generated-token cap, against which a decay is checked."""
    if vocab_range is not None:
        vocab_range = check_vocab_range(vocab_range, lm.shape.vocab_size)
    penalty = per_prompt_penalty(n, repetition_penalty, penalize_prompt)
    length = per_prompt_length(n, min_new_tokens, exponential_decay_length_penalty, max_new)
    ras = per_prompt_ras(n, repetition_aware_sampling)
    controls = per_prompt_controls(n, temperature, top_k, top_p, min_p)
    if controls:
        temperature, top_k = controls[0][0], controls[0][1]
    floor = length[0][0] if length else int(min_new_tokens)
    return Settings(controls, penalty, vocab_range, temperature, top_k, bool(logprobs), length, floor, ras=ras)


PLAN_PHASES = ("qkv", "o", "gu", "d")   # phase order of the persistent kernel's work plan


def debug_decode_plan(hidden: int, inter: int, n_heads: int, n_kv: int, vocab: int, n_sms: int, flat: bool) -> dict:
    """The persistent decode kernel's work plan for a model shape on ``n_sms`` CTAs, built by the library's host planner
    (no GPU needed): ``items[c][phase]`` lists CTA c's (tile, first k-block, k-blocks, slice) items of each phase
    (``PLAN_PHASES``), ``fold_q`` / ``fold_g`` / ``gu_split`` its flags, ``gu_nsl`` the K slices of every gate/up tile
    (flat plan), and ``sq, so, sd, sg, ntiles, max_chunks`` the plan summary.  Raises ValueError when the kernel cannot
    take the shape (the engine then decodes on the per-op chain)."""
    L = _lib.lib()
    items = np.zeros((n_sms, 4, 4, 4), dtype=np.int16)
    counts = np.zeros((n_sms, 4), dtype=np.int32)
    flags = np.zeros((n_sms, 3), dtype=np.int32)
    tg = (2 * inter + 127) // 128
    nsl = np.zeros(tg, dtype=np.uint8)
    info = np.zeros(7, dtype=np.int32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(L.nt_debug_decode_plan(hidden, inter, n_heads, n_kv, vocab, n_sms, int(bool(flat)), ptr(items),
                                      ptr(counts), ptr(flags), ptr(nsl), tg, ptr(info)))
    out = dict(zip(("sq", "so", "sd", "sg", "ntiles", "max_chunks", "gu_split"), info.tolist()))
    out["items"] = [{ph: [tuple(int(v) for v in items[c, p, i]) for i in range(counts[c, p])]
                     for p, ph in enumerate(PLAN_PHASES)} for c in range(n_sms)]
    out["fold_q"], out["fold_g"] = flags[:, 0].tolist(), flags[:, 1].tolist()
    out["gu_split_cta"] = flags[:, 2].tolist()
    out["gu_nsl"] = nsl.tolist() if flat else None
    return out


class SpeechLM:
    PAGE = 64

    def __init__(self, shape: LMShape, state_dict: dict, device="cuda", max_batch: int = 1, max_ctx: int = 2048,
                 max_new: int | None = None, max_prefill_tokens: int | None = None, page_shuffle_seed: int | None = None):
        if not torch.cuda.is_available():
            raise RuntimeError("neutts_air_b200.SpeechLM needs a CUDA device (sm_90a); there is no CPU fallback")
        self.L = _lib.lib()
        self.shape = shape
        self.device = torch.device(device)
        self.max_batch, self.max_ctx = max_batch, max_ctx
        self.max_new = max_new or max_ctx
        self.max_pages = max_ctx // self.PAGE
        self.num_pages = max_batch * self.max_pages
        self.max_prefill_tokens = max_prefill_tokens or max_batch * max_ctx
        with torch.cuda.device(self.device):
            self.w = pack_weights(shape, state_dict, self.device)
            cfg = _lib.LMConfig(shape.vocab_size, shape.hidden_size, shape.intermediate_size, shape.num_layers,
                                shape.num_heads, shape.num_kv_heads, shape.head_dim, shape.rms_eps, shape.rope_theta,
                                max_batch, max_ctx, self.PAGE, self.num_pages, self.max_prefill_tokens)
            self.cfg = cfg
            ws_bytes = self.L.nt_lm_workspace_bytes(C.byref(cfg))
            if ws_bytes == 0:
                _lib.check(-1)
            self.workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
            self._ptrs = {k: _lib.ptr_array(self.w[k]) for k in ("ln1", "wqkv", "bqkv", "wo", "ln2", "wgu", "wd")}
            wts = _lib.LMWeights(self.w["embed"].data_ptr(), self.w["lm_head"].data_ptr(), self.w["final_norm"].data_ptr(),
                                 self._ptrs["ln1"], self._ptrs["wqkv"], self._ptrs["bqkv"], self._ptrs["wo"],
                                 self._ptrs["ln2"], self._ptrs["wgu"], self._ptrs["wd"])
            self.handle = C.c_void_p()
            _lib.check(self.L.nt_lm_create(C.byref(cfg), C.byref(wts), self.workspace.data_ptr(), ws_bytes,
                                           C.byref(self.handle)))
            # caller-owned state (zeroed KV pool: masked keys must hold finite values)
            i32 = dict(dtype=torch.int32, device=self.device)
            self.kv = torch.zeros(shape.num_layers, 2, self.num_pages, shape.num_kv_heads, self.PAGE, 64,
                                  dtype=torch.bfloat16, device=self.device)
            self.page_table = torch.zeros(max_batch, self.max_pages, **i32)
            self.seq_lens = torch.zeros(max_batch, **i32)
            self.cur_token = torch.zeros(max_batch, **i32)
            self.out_tokens = torch.zeros(max_batch, self.max_new, **i32)
            self.n_generated = torch.zeros(max_batch, **i32)
            self.done = torch.zeros(max_batch, **i32)
            self.forced = None
        self.state = _lib.LMState(self.kv.data_ptr(), self.page_table.data_ptr(), self.seq_lens.data_ptr(),
                                  self.cur_token.data_ptr(), self.out_tokens.data_ptr(), self.n_generated.data_ptr(),
                                  self.done.data_ptr(), self.max_new)
        self.pool = PagePool(self.num_pages, page_shuffle_seed)
        self._table_host = None
        self._slot_pages = [[] for _ in range(max_batch)]
        self._slot_sp_host = None   # host mirror of the per-slot sampling controls (None: off)
        self._vocab_range = None    # (lo, hi) while the vocabulary range is on
        self._penalty_host = None   # host mirror of the per-slot repetition penalties (None: off)
        self._length_host = None    # host mirror of the per-slot length control (None: off)
        self._ras_host = None       # host mirror of the per-slot repetition-aware sampling (None: off)
        self.logprobs = None        # per-token log-probabilities, [max_batch][max_new][2] on the device (None: off)
        self._guidance_host = None  # host mirror of the guidance table (None: off)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.L.nt_lm_destroy(self.handle)
        except Exception:
            pass

    # ------------------------------------------------------------------ low-level steps
    def sampling(self, eos_id: int, min_new_tokens: int = 50, max_new_tokens: int | None = None, top_k: int = 50,
                 temperature: float = 1.0, seed: int = 0, greedy: bool = False, forced: torch.Tensor | None = None,
                 limits=None, slot_base: int = 0):
        """``limits``: optional per-sequence caps on generated tokens (list / tensor, one per slot);
        ``slot_base``: global index of slot 0, so that chunks of a larger batch and ranks of a distributed job
        draw from independent Philox streams under one seed."""
        mnt = min(max_new_tokens or self.max_new, self.max_new)
        lptr = None
        if limits is not None:
            lt = torch.full((self.max_batch,), mnt, dtype=torch.int32)
            lt[: len(limits)] = torch.as_tensor(list(limits), dtype=torch.int32)
            self.limits = lt.to(self.device)
            lptr = self.limits.data_ptr()
        fptr = None
        if forced is not None:
            f = torch.zeros(self.max_batch, self.max_new, dtype=torch.int32, device=self.device)
            f[: forced.shape[0], : forced.shape[1]] = forced.to(self.device, torch.int32)
            self.forced = f
            fptr = f.data_ptr()
        return _lib.Sampling(int(eos_id), int(min_new_tokens), int(mnt), int(top_k), float(temperature), int(seed),
                             int(bool(greedy)), fptr, lptr, int(slot_base))

    def set_slot_sampling(self, rows, slots=None) -> None:
        """Per-slot sampling controls.  ``rows``: one (temperature, top_k, top_p, min_p) per slot of ``slots`` (default:
        slots 0..len(rows) - 1); every other slot keeps its entry, or the reference defaults (1.0, 50, 1.0, 0.0) when
        the table was off.  ``None`` switches the table off, and ``sampling``'s temperature and top_k govern every
        slot again.  The table is copied on the current stream, so it is ordered before the next prefill or decode."""
        self._write_slot_table("_slot_sp_host", self.L.nt_lm_set_slot_sampling, _lib.SlotSampling, check_controls,
                               DEFAULT_CONTROLS, rows, slots)

    def _write_slot_table(self, mirror: str, setter, entry, check, default, rows, slots, check_table=None) -> None:
        """Behind the ``set_*`` methods of per-slot tables: validates ``rows`` (``check``) and ``slots``, merges them
        into the host mirror (attribute ``mirror``; ``default`` fills a table that was off), validates the merged table
        (``check_table(table, max_batch)``, when given), and hands the whole table of ``entry`` structs to the C
        ``setter`` on the current stream.  ``rows=None``: the table goes off.  A bad table raises before anything is
        written."""
        table = arr = None
        if rows is not None:
            rows = [check(*r) for r in rows]
            slots = list(range(len(rows))) if slots is None else [int(s) for s in slots]
            if len(slots) != len(rows) or len(set(slots)) != len(slots) or any(not 0 <= s < self.max_batch for s in slots):
                raise ValueError(f"slots must be distinct, in 0..{self.max_batch - 1} and one per row")
            table = list(getattr(self, mirror) or [default] * self.max_batch)
            for s, r in zip(slots, rows):
                table[s] = r
            if check_table is not None:
                table = check_table(table, self.max_batch)
            arr = (entry * self.max_batch)(*(entry(*r) for r in table))
        with torch.cuda.device(self.device):
            _lib.check(setter(self.handle, arr, _lib.current_stream_ptr()))
        setattr(self, mirror, table)

    def set_vocab_range(self, lo, hi=None) -> None:
        """Restrict every later sampler launch to ids in [lo, hi) plus the launch's EOS id (transformers'
        ``suppress_tokens`` with every other id suppressed; the min-new-tokens EOS mask still applies).  The lm_head
        then computes only the range's 128-row tiles and the EOS tile, and every suppressed logit reads -inf.  The
        range holds for every slot.  ``set_vocab_range(None)`` switches it off; a bad range raises ValueError and leaves
        the previous one in force (rules: ``check_vocab_range``)."""
        if lo is not None and hi is None:
            raise ValueError("set_vocab_range needs both lo and hi (or None to switch the range off)")
        rng = None if lo is None else check_vocab_range((lo, hi), self.shape.vocab_size)
        if rng is not None and rng == (0, self.shape.vocab_size):
            rng = None
        lo_, hi_ = rng if rng is not None else (0, self.shape.vocab_size)
        with torch.cuda.device(self.device):
            _lib.check(self.L.nt_lm_set_vocab_range(self.handle, lo_, hi_, _lib.current_stream_ptr()))
        self._vocab_range = rng

    def set_repetition_penalty(self, rows, slots=None) -> None:
        """Per-slot repetition penalty (transformers' ``RepetitionPenaltyLogitsProcessor``).  ``rows``: one
        (penalty, include_prompt) per slot of ``slots`` (default: slots 0..len(rows) - 1); every other slot keeps its
        entry, or (1.0, True) when the table was off.  A slot's history is its prompt (when include_prompt) plus every
        token generated for it since; it is recorded from the slot's next prefill, so switch the table on before the
        prefill whose tokens should count.  ``None`` switches the table off.  The table is copied on the current stream,
        so it is ordered before the next prefill or decode."""
        self._write_slot_table("_penalty_host", self.L.nt_lm_set_repetition_penalty, _lib.SlotPenalty, check_penalty,
                               DEFAULT_PENALTY, rows, slots)

    def set_length_control(self, rows, slots=None) -> None:
        """Per-slot length control (transformers' ``MinNewTokensLengthLogitsProcessor`` and
        ``ExponentialDecayLengthPenalty``).  ``rows``: one (min_new_tokens, decay_start, decay_factor) per slot of
        ``slots`` (default: slots 0..len(rows) - 1); every other slot keeps its entry, or (50, 49, 1.0) when the table
        was off.  While on, a slot's min_new_tokens replaces ``sampling``'s, and once it has generated n > decay_start
        tokens its EOS score s becomes s + |s| * (decay_factor ** (n - decay_start) - 1) before the vocabulary range,
        the temperature and the warpers; greedy and teacher-forced runs see it too.  ``None`` switches the table off.
        Rules: ``check_length``.  The table is copied on the current stream, so it is ordered before the next prefill
        or decode."""
        self._write_slot_table("_length_host", self.L.nt_lm_set_length_control, _lib.SlotLength, check_length,
                               DEFAULT_LENGTH, rows, slots)

    def set_repetition_aware_sampling(self, rows, slots=None) -> None:
        """Per-slot Repetition Aware Sampling (VALL-E 2; CosyVoice 2's ``ras_sampling``).  ``rows``: one
        (win_size, tau_r) pair or None (off) per slot of ``slots`` (default: slots 0..len(rows) - 1); every other slot
        keeps its entry, or none when the table was off.  While a slot's entry is on, a sampled draw that occurs at
        least ceil(win_size * tau_r) times among the slot's last win_size generated tokens (never its prompt) is
        replaced by one draw from the whole distribution: the softmax of the processed scores times 1 / T, without the
        top-k, top-p and min-p cuts.  Greedy and teacher-forced runs, and every slot's first token, never redraw.
        ``None`` switches the table off.  Rules: ``check_ras``.  The table is copied on the current stream, so it is
        ordered before the next prefill or decode."""
        self._write_slot_table("_ras_host", self.L.nt_lm_set_repetition_aware_sampling, _lib.SlotRAS, ras_entry,
                               RAS_OFF, None if rows is None else [(r,) for r in rows], slots)

    def ras_redraws(self) -> torch.Tensor:
        """Each slot's repetition-aware redraws since the prefill that filled it (int32 CPU tensor [max_batch])."""
        return self.debug_buffer("ras_redraws", (self.max_batch,), torch.int32).cpu()

    def set_logprobs(self, on: bool = True):
        """Per-token log-probabilities.  While on, every later sampler launch writes, for each token it writes to
        ``out_tokens[s][n]``, the pair ``logprobs[s][n] = (sampled, model)`` into ``self.logprobs`` (device float32
        [max_batch][max_new][2], allocated here and kept while on): ``sampled`` is the token's log-probability in the
        kept window the sampler drew from (transformers' ``compute_transition_scores(normalize_logits=True)``; greedy
        runs: equal to ``model``; teacher-forced ids outside the window: -inf), ``model`` its log-softmax over the whole
        vocabulary after the repetition penalty, the min-new-tokens EOS mask and the vocabulary range, before
        temperature and the warpers.  ``on=False`` switches it off and frees the buffer.  Returns the buffer or None."""
        buf = (self.logprobs if self.logprobs is not None else
               torch.zeros(self.max_batch, self.max_new, 2, dtype=torch.float32, device=self.device)) if on else None
        with torch.cuda.device(self.device):
            _lib.check(self.L.nt_lm_set_logprobs(self.handle, None if buf is None else buf.data_ptr(),
                                                 _lib.current_stream_ptr()))
        self.logprobs = buf
        return buf

    def set_guidance(self, rows, slots=None) -> None:
        """Classifier-free guidance (transformers' ``guidance_scale`` with ``negative_prompt_ids``).  ``rows``: one
        (partner, scale) per slot of ``slots`` (default: slots 0..len(rows) - 1); every other slot keeps its entry, or
        (-1, 1.0) (no partner) when the table was off.  Slot c with partner u >= 0 is guided: at every sampler launch
        its logits row becomes ``scale * (ls_c - ls_u) + ls_u`` (log-softmaxes) before the penalty, the length control
        and the warpers, and u, which holds the negative prompt, takes every token c draws and is never sampled.
        ``None`` switches guidance off.  ``generate_batch`` / ``generate_queue`` leave their table on when they return
        (the next call's settings replace it); a caller that then prefills or decodes directly switches it off first,
        or its launches must include both slots of every pair still in the table.  The merged table is validated first (``check_guidance_table``); a bad one
        raises ValueError and leaves the previous table in force.  Copied on the current stream."""
        self._write_slot_table("_guidance_host", self.L.nt_lm_set_guidance, _lib.SlotGuidance,
                               lambda p, g: (int(p), float(g)), NO_GUIDANCE, rows, slots, check_guidance_table)

    def _stage_ids(self, prompts) -> torch.Tensor:
        """The prompts' ids, range-checked, back to back in a persistent pinned buffer (so their H2D copy is
        asynchronous)."""
        flat = np.concatenate([np.asarray(p, dtype=np.int64) for p in prompts])
        if flat.min() < 0 or flat.max() >= self.shape.vocab_size:
            raise ValueError("token id out of range")
        if getattr(self, "_ids_pinned", None) is None or self._ids_pinned.numel() < flat.size:
            self._ids_pinned = torch.empty(max(flat.size, self.max_prefill_tokens), dtype=torch.int32).pin_memory()
        staged = self._ids_pinned[: flat.size]
        staged.copy_(torch.from_numpy(flat.astype(np.int32)))
        return staged

    def _alloc_pages(self, table, slots, lens, caps) -> None:
        """KV pages for prompt + cap tokens of every listed slot, written into its row of the page table ``table``."""
        for s, n, cap in zip(slots, lens, caps):
            need = (min(n + cap, self.max_ctx) + self.PAGE - 1) // self.PAGE
            pages = self.pool.alloc(need)
            self._slot_pages[s] = pages
            table[s] = 0
            table[s, :need] = pages

    def _alloc_fork_pages(self, table, lens, n: int, cap: int) -> None:
        """KV pages of n takes of every prompt, written into the page table ``table``: take j of prompt i (slot i * n + j)
        holds the prompt's P // 64 full pages, shared by all n takes, then pages of its own from page P // 64 on (the
        partly filled last prompt page, if any, and room for ``cap`` generated tokens)."""
        need = [(min(P + cap, self.max_ctx) + self.PAGE - 1) // self.PAGE for P in lens]
        total = sum(P // self.PAGE + n * (m - P // self.PAGE) for P, m in zip(lens, need))
        if total > self.pool.num_free:
            raise RuntimeError(f"KV page pool exhausted: need {total}, have {self.pool.num_free}")
        for i, j, s, _ in fork_slots(len(lens), n):
            if j == 0:
                shared = self.pool.alloc(lens[i] // self.PAGE)
            else:
                self.pool.share(shared)
            pages = shared + self.pool.alloc(need[i] - len(shared))
            self._slot_pages[s] = pages
            table[s] = 0
            table[s, : need[i]] = pages

    def prefill(self, prompts, sp, return_logits: bool = False):
        """prompts: list of 1-D int sequences.  Fills the KV cache and samples the first token of every prompt, prompt b
        in slot b: ``prefill_fork`` with one take per prompt."""
        return self.prefill_fork(prompts, 1, sp, return_logits)

    def prefill_fork(self, prompts, n: int, sp, return_logits: bool = False):
        """n takes of every prompt from one prefill (``nt_lm_prefill_fork``).  Take j of prompt i lives in slot i * n + j
        and draws from Philox stream i * n + j + slot_base, as in ``prefill`` on the prompts each repeated n times; the
        prompts are prefilled once, and all n takes read one copy of each full prompt page (``_alloc_fork_pages``).
        Resets every slot; afterwards ``decode`` continues all len(prompts) * n takes.  Returns the [len(prompts), vocab]
        last-position logits (the same for every n) when ``return_logits``."""
        B = len(prompts)
        n = check_takes(B, n, self.max_batch)
        lens = [len(p) for p in prompts]
        if not lens or min(lens) < 1:
            raise ValueError("empty prompt")
        if max(lens) >= self.max_ctx:
            raise ValueError(f"prompt lengths must be in 1..{self.max_ctx - 1}")
        staged = self._stage_ids(prompts)
        self.release_pages()
        table = np.zeros((self.max_batch, self.max_pages), dtype=np.int32)
        self._alloc_fork_pages(table, lens, n, sp.max_new_tokens)
        cu = np.zeros(B + 1, dtype=np.int32)
        cu[1:] = np.cumsum(lens)
        with torch.cuda.device(self.device):
            ids = staged.to(self.device, non_blocking=True)
            if self._table_host is None or not np.array_equal(self._table_host, table):
                self.page_table.copy_(torch.from_numpy(table))
                self._table_host = table
            logits = torch.empty(B, self.shape.vocab_size, dtype=torch.float32, device=self.device) if return_logits else None
            cu_p, lg_p = cu.ctypes.data_as(C.POINTER(C.c_int32)), logits.data_ptr() if return_logits else None
            if n == 1 and self._guidance_host is not None:   # the fork entry is refused while guidance is on
                _lib.check(self.L.nt_lm_prefill(self.handle, C.byref(self.state), ids.data_ptr(), cu_p, B, C.byref(sp), lg_p,
                                                _lib.current_stream_ptr()))
            else:
                _lib.check(self.L.nt_lm_prefill_fork(self.handle, C.byref(self.state), ids.data_ptr(), cu_p, B, n,
                                                     C.byref(sp), lg_p, _lib.current_stream_ptr()))
        self._B = B * n
        return logits

    def release_pages(self, slots=None) -> None:
        """Return the KV pages of ``slots`` (default: every slot) to the pool.  A page shared with another slot (the
        full prompt pages of ``prefill_fork``'s takes) stays held until its last holder releases it."""
        for b in range(self.max_batch) if slots is None else slots:
            if self._slot_pages[b]:
                self.pool.release(self._slot_pages[b])
                self._slot_pages[b] = []

    def prefill_slots(self, slots, prompts, sp, stream_ids, return_logits: bool = False, limits=None):
        """Prefill ``prompts`` into the listed ``slots`` while every other slot keeps its KV pages, tokens and counters
        (so its decoding simply continues).  Needs an earlier ``prefill``.  Samples the first token of each listed slot.
        ``stream_ids``: the Philox stream key of each prompt (>= 0), used for its slot instead of slot + slot_base
        until the next ``prefill``.  ``limits``: optional cap on generated tokens per prompt, written into the slots'
        entries of the per-slot limits (``sp`` must come from ``sampling(..., limits=...)``).  Afterwards ``decode``
        continues every live slot below the widest batch prefilled so far.  Returns the [len(slots), vocab]
        logits in call order when ``return_logits``."""
        slots = [int(s) for s in slots]
        B = len(slots)
        if B == 0 or B != len(prompts) or B != len(stream_ids):
            raise ValueError("slots, prompts and stream_ids must be non-empty and of equal length")
        if len(set(slots)) != B or min(slots) < 0 or max(slots) >= self.max_batch:
            raise ValueError(f"slots must be distinct and in 0..{self.max_batch - 1}")
        if getattr(self, "_B", None) is None:
            raise RuntimeError("prefill_slots needs an earlier prefill")
        lens = [len(p) for p in prompts]
        if min(lens) < 1 or max(lens) >= self.max_ctx:
            raise ValueError(f"prompt lengths must be in 1..{self.max_ctx - 1}")
        if min(int(s) for s in stream_ids) < 0:
            raise ValueError("stream ids must be >= 0")
        caps = [min(int(c), sp.max_new_tokens) for c in limits] if limits is not None else [sp.max_new_tokens] * B
        if limits is not None and (getattr(self, "limits", None) is None or sp.limits != self.limits.data_ptr()):
            raise ValueError("per-prompt limits need sampling params built with limits=")
        staged = self._stage_ids(prompts)
        self.release_pages(slots)
        table = self._table_host.copy()
        self._alloc_pages(table, slots, lens, caps)
        cu = np.zeros(B + 1, dtype=np.int32)
        cu[1:] = np.cumsum(lens)
        slots_h = np.asarray(slots, dtype=np.int32)
        keys_h = np.asarray([int(k) for k in stream_ids], dtype=np.int32)
        i32p = C.POINTER(C.c_int32)
        with torch.cuda.device(self.device):
            ids = staged.to(self.device, non_blocking=True)
            self.page_table.copy_(torch.from_numpy(table))   # same stream as the prefill below
            self._table_host = table
            if limits is not None:
                self.limits.index_copy_(0, torch.tensor(slots, device=self.device),
                                        torch.tensor(caps, dtype=torch.int32, device=self.device))
            logits = torch.empty(B, self.shape.vocab_size, dtype=torch.float32, device=self.device) if return_logits else None
            _lib.check(self.L.nt_lm_prefill_slots(self.handle, C.byref(self.state), slots_h.ctypes.data_as(i32p),
                                                  keys_h.ctypes.data_as(i32p), ids.data_ptr(), cu.ctypes.data_as(i32p), B,
                                                  C.byref(sp), logits.data_ptr() if return_logits else None,
                                                  _lib.current_stream_ptr()))
        self._B = max(self._B, max(slots) + 1)
        return logits

    @torch.no_grad()
    def score(self, sequences, start) -> list:
        """Teacher-forced scoring (``nt_lm_score``): for every sequence x_0 .. x_{L-1} and its start s, the
        log-probability of each token x_t (s <= t < L) under the model given x_0 .. x_{t-1}, from one prefill pass -- the
        model alone, with no repetition penalty, EOS mask, vocabulary range, temperature or warper (the settings stay as
        they are).  transformers' ``-cross_entropy(logits[s-1:L-1], ids[s:L], reduction="none")``.

        ``sequences``: 1-D int sequences (at least 2 ids each); ``start``: an int or one per sequence.  Returns one
        float32 CPU tensor [L - s] per sequence, in input order.  Sequences go into calls of at most ``max_batch``
        sequences and ``max_prefill_tokens`` tokens (``pack_score_calls``); each call takes KV pages as ``prefill`` does
        and gives them all back.  A sequence's scores do not depend on the others in its call.  Every slot is reset:
        ``decode`` and ``prefill_slots`` need a new ``prefill`` afterwards."""
        seqs = [np.asarray(s, dtype=np.int64).reshape(-1) for s in sequences]
        lens = [len(s) for s in seqs]
        starts = score_starts(lens, start)
        calls = pack_score_calls(lens, self.max_batch, self.max_prefill_tokens, self.max_ctx)
        if seqs:
            self._stage_ids(seqs)   # range check of every id before any engine call
        if getattr(self, "_score_scratch", None) is None:
            n = self.L.nt_lm_score_scratch_bytes(C.byref(self.cfg))
            if n == 0:
                _lib.check(-1)
            self._score_scratch = torch.empty(n, dtype=torch.uint8, device=self.device)
        out = [None] * len(seqs)
        i32p = C.POINTER(C.c_int32)
        for idx in calls:
            B = len(idx)
            clens = [lens[i] for i in idx]
            staged = self._stage_ids([seqs[i] for i in idx])
            self.release_pages()
            table = np.zeros((self.max_batch, self.max_pages), dtype=np.int32)
            self._alloc_pages(table, range(B), clens, [0] * B)
            cu = np.zeros(B + 1, dtype=np.int32)
            cu[1:] = np.cumsum(clens)
            st = np.asarray([starts[i] for i in idx], dtype=np.int32)
            n = sum(L - s for L, s in zip(clens, st.tolist()))
            try:
                with torch.cuda.device(self.device):
                    ids = staged.to(self.device, non_blocking=True)
                    if self._table_host is None or not np.array_equal(self._table_host, table):
                        self.page_table.copy_(torch.from_numpy(table))
                        self._table_host = table
                    res = torch.empty(n, dtype=torch.float32, device=self.device)
                    _lib.check(self.L.nt_lm_score(self.handle, C.byref(self.state), ids.data_ptr(), cu.ctypes.data_as(i32p),
                                                  st.ctypes.data_as(i32p), B, res.data_ptr(), self._score_scratch.data_ptr(),
                                                  self._score_scratch.numel(), _lib.current_stream_ptr()))
                    res = res.cpu()
            finally:
                self.release_pages()
            o = 0
            for i, L, s in zip(idx, clens, st.tolist()):
                out[i] = res[o: o + L - s].clone()
                o += L - s
        return out

    def decode(self, n_steps: int, sp, return_logits: bool = False):
        B = self._B
        with torch.cuda.device(self.device):
            logits = (torch.empty(n_steps, B, self.shape.vocab_size, dtype=torch.float32, device=self.device)
                      if return_logits else None)
            _lib.check(self.L.nt_lm_decode(self.handle, C.byref(self.state), B, n_steps, C.byref(sp),
                                           logits.data_ptr() if return_logits else None, _lib.current_stream_ptr()))
        return logits

    def head_gemv(self, h: torch.Tensor) -> torch.Tensor:
        """lm_head (+ final RMSNorm) GEMV alone: the kernel bench.py puts on the roofline."""
        B = h.shape[0]
        logits = torch.empty(B, self.shape.vocab_size, dtype=torch.float32, device=self.device)
        _lib.check(self.L.nt_lm_head_gemv(self.handle, h.data_ptr(), B, logits.data_ptr(), _lib.current_stream_ptr()))
        return logits

    # ------------------------------------------------------------------ per-stage parity hooks (tests)
    def debug_set_layers(self, n: int) -> None:
        _lib.check(self.L.nt_lm_debug_set_layers(self.handle, n))

    def debug_set_sms(self, n: int) -> None:
        """Decode on ``n`` CTAs (8 .. min(device SMs, 256)) as if the device had that many SMs: the persistent kernel's
        grid and work plans, its batch gate and the GEMV grids; 0 restores the device's count."""
        _lib.check(self.L.nt_lm_debug_set_sms(self.handle, n))

    def debug_buffer(self, name: str, shape, dtype=torch.float32) -> torch.Tensor:
        """View of an internal activation buffer (lives inside ``self.workspace``)."""
        ptr = self.L.nt_lm_debug_ptr(self.handle, name.encode())
        if not ptr:
            raise KeyError(name)
        off = ptr - self.workspace.data_ptr()
        n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        return self.workspace[off: off + n].view(dtype).view(*shape)

    def debug_capture_sampler(self, on: bool = True):
        """Every later sampler launch writes, per logits row, its kept window (probabilities [64] fp32, ids [64] int32,
        -1 padded) and the token it selected into buffers owned here; returns them as (topk_val, topk_idx, token), or
        None when ``on`` is False (capture off).  Each launch overwrites the rows it samples."""
        if not on:
            _lib.check(self.L.nt_lm_debug_capture_sampler(self.handle, None, None, None))
            self._capture = None
            return None
        B = self.max_batch
        self._capture = (torch.zeros(B, 64, dtype=torch.float32, device=self.device),
                         torch.full((B, 64), -2, dtype=torch.int32, device=self.device),
                         torch.full((B,), -2, dtype=torch.int32, device=self.device))
        _lib.check(self.L.nt_lm_debug_capture_sampler(self.handle, *(t.data_ptr() for t in self._capture)))
        return self._capture

    # ------------------------------------------------------------------ generation
    def _caps(self, lens, max_length: int, max_new_tokens) -> list:
        """Generated-token cap per prompt; ``max_new_tokens``: None, one int, or one int per prompt."""
        if max_new_tokens is None or isinstance(max_new_tokens, int):
            max_new_tokens = [max_new_tokens or max_length] * len(lens)
        if len(max_new_tokens) != len(lens):
            raise ValueError("max_new_tokens needs one entry per prompt")
        return [min(max_length - n, int(m), self.max_new) for n, m in zip(lens, max_new_tokens)]

    def _results(self, rows, ngen, logprobs: bool):
        """Generated ids of ``rows`` (slots) as int64 CPU tensors, cut at ``ngen`` per row; with ``logprobs`` also
        each row's float32 CPU ``[n, 2]`` (sampled, model) log-probabilities, read before any refill overwrites them."""
        toks = self.out_tokens[rows].cpu()
        ids = [toks[r, : int(n)].long() for r, n in enumerate(ngen)]
        if not logprobs:
            return ids, None
        lp = self.logprobs[rows].cpu()
        return ids, [lp[r, : int(n)].clone() for r, n in enumerate(ngen)]

    def _prepare(self, prompts, max_length, max_new_tokens, guidance_scale=1.0, negative_prompt_ids=None, **settings) -> tuple:
        """Shared preamble of ``generate_batch`` / ``generate_queue``, run before any engine call: the max_length
        checks, the generated-token cap per prompt and the resolved ``settings`` -> (caps, Settings, guidance), with
        guidance as ``per_prompt_guidance`` and every guided prompt's cap shortened so its negative prompt fits."""
        guidance = per_prompt_guidance(prompts, guidance_scale, negative_prompt_ids)
        max_length = max_length or self.max_ctx
        if max_length > self.max_ctx:
            raise ValueError(f"max_length {max_length} exceeds the engine context {self.max_ctx}")
        lens = [len(p) for p in prompts]
        if any(max_length - n < 1 for n in lens):
            raise ValueError("prompt already at max_length")
        # max_length counts prompt + generated PER SEQUENCE (stopping_criteria.py:73-84): a long prompt in the batch
        # must not shorten its neighbours, so every slot gets its own cap and the loop runs to the largest one
        caps = self._caps(lens, max_length, max_new_tokens)
        st = resolve_settings(self, len(prompts), max_new=max(caps, default=0), **settings)
        return guided_caps(caps, guidance, self.max_ctx), st, guidance

    def generate_batch(self, prompts, eos_token_id: int, max_length: int | None = None, min_new_tokens: int = 50,
                       temperature: float = 1.0, top_k: int = 50, max_new_tokens: int | None = None, seed: int = 0,
                       greedy: bool = False, forced: torch.Tensor | None = None, check_every: int = 64, slot_base: int = 0,
                       top_p: float = 1.0, min_p: float = 0.0, vocab_range=None, repetition_penalty=1.0,
                       penalize_prompt=True, return_logprobs: bool = False, num_return_sequences: int = 1,
                       exponential_decay_length_penalty=None, guidance_scale=1.0, negative_prompt_ids=None,
                       repetition_aware_sampling=None):
        """Returns a list of int64 CPU tensors with the generated ids of each prompt (EOS included
        when it was sampled), following transformers' stopping rules (stopping_criteria.py:73-84,
        467-471): stop at EOS or when prompt + generated reaches max_length.  ``max_new_tokens`` may also be a
        list with one cap per prompt.  ``temperature``, ``top_k``, ``top_p`` and ``min_p`` are each a scalar or one
        value per prompt (per-slot controls, ``set_slot_sampling``).  ``vocab_range``: (lo, hi) restricts every draw to
        [lo, hi) plus EOS (``set_vocab_range``); None leaves the range off.  ``repetition_penalty`` (> 0, 1 = off) and
        ``penalize_prompt`` (the prompt's ids count) are each a scalar or one value per prompt
        (``set_repetition_penalty``); they apply to greedy and teacher-forced runs too.  ``return_logprobs``: returns
        ``(ids, logprobs)`` instead, ``logprobs[i]`` a float32 CPU tensor [len(ids[i]), 2] of (sampled, model)
        log-probabilities per generated token (``set_logprobs``, switched on for the call and off by a later call
        without it).  ``min_new_tokens`` is an int or one per prompt, and ``exponential_decay_length_penalty`` None,
        transformers' (start, factor) or one None / pair per prompt (``set_length_control``): per-prompt floors or any
        decay switch the per-slot table on for the call.  ``num_return_sequences`` n > 1: n takes of every prompt from one prefill (``prefill_fork``;
        len(prompts) * n <= max_batch), returned in slot order, take j of prompt i at index i * n + j, each drawing
        from the Philox stream the prompt repeated n times would give it; every per-prompt setting (and cap) applies
        to all n takes of its prompt, while ``forced`` has one row per take.

        ``guidance_scale`` (a number or one per prompt; 1 = off) and ``negative_prompt_ids`` (None, or one id list or
        None per prompt) add classifier-free guidance as transformers' ``UnbatchedClassifierFreeGuidanceLogitsProcessor``
        (``set_guidance``): prompt i stays in slot i and the unconditional sequence of each guided prompt, its negative
        prompt (default: the prompt's last token) followed by its draws, takes a slot above the prompts, so
        len(prompts) + guided prompts <= max_batch.  A guided prompt's cap is at most max_ctx - len(negative prompt).
        Guidance with ``num_return_sequences`` > 1 raises ValueError.

        ``repetition_aware_sampling``: None, one (win_size, tau_r) pair or one None / pair per prompt
        (``set_repetition_aware_sampling``): a sampled token that repeats at least ceil(win_size * tau_r) times among
        the prompt's last win_size generated tokens is redrawn once from the whole distribution.  It follows its
        prompt into every take and into a guided prompt's slot."""
        n_takes = check_takes(len(prompts), num_return_sequences, self.max_batch)
        caps, settings, guidance = self._prepare(
            prompts, max_length, max_new_tokens, guidance_scale, negative_prompt_ids, temperature=temperature, top_k=top_k,
            top_p=top_p, min_p=min_p, vocab_range=vocab_range, repetition_penalty=repetition_penalty,
            penalize_prompt=penalize_prompt, logprobs=return_logprobs, min_new_tokens=min_new_tokens,
            exponential_decay_length_penalty=exponential_decay_length_penalty,
            repetition_aware_sampling=repetition_aware_sampling)
        pairs = guided_layout(len(prompts), guidance)
        if pairs and n_takes > 1:
            raise ValueError("classifier-free guidance takes one sequence per prompt (num_return_sequences=1)")
        if len(prompts) + len(pairs) > self.max_batch:
            raise ValueError(f"{len(prompts)} prompt(s) with {len(pairs)} guided need {len(prompts) + len(pairs)} slots; "
                             f"the engine has {self.max_batch}")
        if n_takes > 1:
            caps = [c for c in caps for _ in range(n_takes)]
            settings = settings.repeat(n_takes)
        caps = caps + [caps[c] for c, _, _ in pairs]
        settings = settings.pair(pairs)
        limit = max(caps)
        sp = self.sampling(eos_token_id, settings.min_new_tokens, limit, settings.top_k, settings.temperature, seed, greedy,
                           forced, limits=caps if min(caps) < limit else None, slot_base=slot_base)
        B = len(prompts) * n_takes
        settings.apply(self, B + len(pairs))
        if n_takes > 1:
            self.prefill_fork(prompts, n_takes, sp)
        else:
            self.prefill(list(prompts) + [guidance[c][1] for c, _, _ in pairs], sp)
        remaining = limit - 1
        while remaining > 0:
            n = min(check_every, remaining)
            self.decode(n, sp)
            remaining -= n
            if remaining > 0 and bool(self.done[:B].all()):  # one small D2H read per `check_every` steps
                break
        ids, lps = self._results(slice(0, B), self.n_generated[:B].cpu().tolist(), return_logprobs)
        return (ids, lps) if return_logprobs else ids

    def generate_queue(self, prompts, eos_token_id: int, max_length: int | None = None, min_new_tokens: int = 50,
                       temperature: float = 1.0, top_k: int = 50, max_new_tokens: int | None = None, seed: int = 0,
                       greedy: bool = False, check_every: int = 32, slot_base: int = 0, top_p: float = 1.0,
                       min_p: float = 0.0, vocab_range=None, repetition_penalty=1.0, penalize_prompt=True,
                       return_logprobs: bool = False, num_return_sequences: int = 1,
                       exponential_decay_length_penalty=None, guidance_scale=1.0, negative_prompt_ids=None,
                       repetition_aware_sampling=None):
        """Continuous batching over any number of prompts: ``generate_batch``'s results and stopping rules, but a slot
        whose sequence finished is refilled with the next waiting prompt while the other slots keep decoding.

        Prompts are admitted FIFO into ``min(len(prompts), max_batch)`` slots; prompt i draws from Philox stream
        ``slot_base + i``, the stream the chunked loop (``generate_batch`` per ``max_batch`` prompts with
        ``slot_base`` = the chunk's first index) gives it.  Decoding runs in launches of at most ``check_every``
        steps, each cut short so that it ends with the earliest cap-driven completion while prompts wait.  After each
        launch one small read of (n_generated, done) finds the finished slots; their tokens are copied out and the next
        prompts go into all freed slots with one ``prefill_slots`` call.  Returns the generated ids per prompt (int64
        CPU tensors, EOS included when sampled) in input order; every KV page is back in the pool afterwards.
        ``temperature``, ``top_k``, ``top_p`` and ``min_p`` are each a scalar or one value per prompt; a newcomer's
        controls are written into its slot before its prefill, and the other slots keep theirs.  ``vocab_range`` as in
        ``generate_batch``: set once before the first prefill, it holds across every refill.  ``repetition_penalty`` and
        ``penalize_prompt`` as in ``generate_batch``; a newcomer's entry is written before its prefill.
        ``return_logprobs`` as in ``generate_batch``: a finished slot's rows are copied out with its tokens, before
        the refill that reuses the slot.  ``min_new_tokens`` and ``exponential_decay_length_penalty`` as in
        ``generate_batch``; a newcomer's entry is written before its prefill.  One sequence per prompt: ``num_return_sequences`` > 1 raises ValueError
        (``generate_batch`` takes several per prompt).

        ``guidance_scale`` and ``negative_prompt_ids`` as in ``generate_batch``.  A guided prompt needs two free slots,
        filled by one ``prefill_slots`` call with the others admitted at that read; admission stays FIFO (the head of
        the queue waits for room), and the pair's slots free together.  ``repetition_aware_sampling`` as in
        ``generate_batch``; a newcomer's entry is written before its prefill."""
        if num_return_sequences != 1:
            raise ValueError("generate_queue returns one sequence per prompt; use generate_batch(num_return_sequences=n) "
                             "for several takes of each prompt")
        caps, settings, guidance = self._prepare(
            prompts, max_length, max_new_tokens, guidance_scale, negative_prompt_ids, temperature=temperature, top_k=top_k,
            top_p=top_p, min_p=min_p, vocab_range=vocab_range, repetition_penalty=repetition_penalty,
            penalize_prompt=penalize_prompt, logprobs=return_logprobs, min_new_tokens=min_new_tokens,
            exponential_decay_length_penalty=exponential_decay_length_penalty,
            repetition_aware_sampling=repetition_aware_sampling)
        n, M = len(prompts), self.max_batch
        if n == 0:
            return ([], []) if return_logprobs else []
        if check_every < 1:
            raise ValueError("check_every must be >= 1")
        guided = guidance is not None
        need = [1 + (g != 1.0) for g, _ in guidance] if guided else [1] * n   # slots per prompt: c, and u when guided
        if max(need) > M:
            raise ValueError(f"a guided prompt needs 2 slots; the engine has {M}")
        k = 0   # the first wave: prompts 0..k-1 and their u slots, in the generate_batch layout
        while k < n and sum(need[: k + 1]) <= M:
            k += 1
        pairs = guided_layout(k, guidance[:k]) if guided else []
        slot_caps = caps[:k] + [caps[c] for c, _, _ in pairs]
        sp = self.sampling(eos_token_id, settings.min_new_tokens, max(caps), settings.top_k, settings.temperature, seed,
                           greedy, limits=slot_caps, slot_base=slot_base)
        # with guidance the table is on from the first prefill, pair or not: the decode path depends on it, so switching
        # it on at a later refill would change the kernels of the slots already decoding
        (settings.pair(pairs, k) if guided else settings).apply(self, len(slot_caps))
        self.prefill(list(prompts[:k]) + [guidance[c][1] for c, _, _ in pairs], sp)
        occ = list(range(k)) + [None] * (M - k)   # prompt held by each c slot, None once harvested
        partner = {c: u for c, u, _ in pairs}     # c slot -> its u slot
        busy = set(range(k)) | set(partner.values())
        ngen = [1] * M   # generated tokens per slot, as of the last read
        nxt = k          # next prompt to admit
        out, out_lp = [None] * n, [None] * n
        # a sequence can finish inside its prefill: a cap of 1, or EOS when it is not masked at step 0
        floors = settings.floors(n)
        at_prefill = lambda idx: min(floors[i] for i in idx) <= 0 or min(caps[i] for i in idx) <= 1
        read = at_prefill(range(k))
        while True:
            if read:
                ngen, done = torch.stack((self.n_generated, self.done)).cpu().tolist()   # the one small D2H read per launch
                fin = [s for s in range(M) if occ[s] is not None and done[s]]
                freed = []
                if fin:
                    ids, lps = self._results(fin, [ngen[s] for s in fin], return_logprobs)
                    for r, s in enumerate(fin):
                        out[occ[s]] = ids[r]
                        if return_logprobs:
                            out_lp[occ[s]] = lps[r]
                        occ[s] = None
                        freed += [s] + ([partner.pop(s)] if s in partner else [])
                    busy -= set(freed)
                # FIFO, the head of the queue waiting for room: each prompt takes the lowest free slot, its u slot the next
                free, room = (s for s in range(M) if s not in busy), M - len(busy)
                new = []   # (c slot, u slot or None, prompt) of every admitted prompt
                while nxt < n and need[nxt] <= room:
                    new.append((next(free), next(free) if need[nxt] == 2 else None, nxt))
                    room -= need[nxt]
                    nxt += 1
                if new:
                    new_pairs = [(c, u, i) for c, u, i in new if u is not None]
                    slots = [c for c, _, _ in new] + [u for _, u, _ in new_pairs]
                    idx = [i for _, _, i in new] + [i for _, _, i in new_pairs]
                    guide = None
                    if guided:   # every freed slot's entry is rewritten in the same call, so no finished pair survives
                        guide = {s: NO_GUIDANCE for s in freed + slots}
                        guide.update((c, (u, guidance[i][0])) for c, u, i in new_pairs)
                    settings.admit(self, slots, idx, guide=guide)   # before their prefill, on the same stream
                    self.prefill_slots(slots, [prompts[i] for _, _, i in new] + [guidance[i][1] for _, _, i in new_pairs],
                                       sp, [slot_base + i for i in idx], limits=[caps[i] for i in idx])
                    for c, u, i in new:
                        occ[c], ngen[c] = i, 1
                        if u is not None:
                            partner[c] = u
                    busy |= set(slots)
                    if at_prefill([i for _, _, i in new]):
                        continue   # read again before decoding: a newcomer may be done already
            live = [s for s in range(M) if occ[s] is not None]
            if not live:
                break
            left = [caps[occ[s]] - ngen[s] for s in live]
            steps = max(1, min(check_every, min(left) if nxt < n else max(left)))
            self.decode(steps, sp)
            read = True
        self.release_pages()
        return (out, out_lp) if return_logprobs else out

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, max_length: int = 2048, eos_token_id: int | None = None,
                 do_sample: bool = True, temperature: float = 1.0, top_k: int = 50, use_cache: bool = True,
                 min_new_tokens: int = 0, max_new_tokens: int | None = None, seed: int | None = None,
                 top_p: float = 1.0, min_p: float = 0.0, vocab_range=None, repetition_penalty: float = 1.0,
                 num_return_sequences: int = 1, exponential_decay_length_penalty=None, guidance_scale=None,
                 negative_prompt_ids=None, negative_prompt_attention_mask=None, repetition_aware_sampling=None, **_):
        """transformers-compatible seam used by ``NeuTTS._infer_torch`` (neutts/neutts.py:338-347).  ``top_p`` and
        ``min_p`` act as transformers' TopPLogitsWarper / MinPLogitsWarper; ``vocab_range`` (lo, hi) suppresses every
        id outside [lo, hi) and EOS (``set_vocab_range``); ``repetition_penalty`` acts as transformers'
        RepetitionPenaltyLogitsProcessor (prompt included); ``exponential_decay_length_penalty`` (start, factor) acts as
        transformers' ExponentialDecayLengthPenalty (``set_length_control``); ``num_return_sequences`` n returns n takes of every prompt
        from one prefill, [B * n, P + gen] with take j of row b at row b * n + j, as transformers; ``guidance_scale``
        with ``negative_prompt_ids`` ([1 or B, L]; default: each prompt's last token) acts as transformers'
        UnbatchedClassifierFreeGuidanceLogitsProcessor (``generate_batch``), and ``negative_prompt_attention_mask`` must
        be None or all ones; ``repetition_aware_sampling`` (win_size, tau_r) redraws repeating tokens
        (``set_repetition_aware_sampling``); other generation kwargs are ignored."""
        if eos_token_id is None:
            raise ValueError("eos_token_id is required")
        if input_ids.dim() != 2:
            raise ValueError("input_ids must be [B, P]")
        prompts = [row.tolist() for row in input_ids.cpu()]
        guided = {}
        if guidance_scale is not None and guidance_scale != 1:
            if negative_prompt_attention_mask is not None and not bool(torch.as_tensor(negative_prompt_attention_mask).eq(1).all()):
                raise ValueError("negative_prompt_attention_mask must be all ones: padded negative prompts are not supported")
            negs = None
            if negative_prompt_ids is not None:
                q = torch.as_tensor(negative_prompt_ids)
                q = q[None] if q.dim() == 1 else q
                if q.shape[0] not in (1, len(prompts)):
                    raise ValueError(f"negative_prompt_ids has {q.shape[0]} rows for {len(prompts)} prompts")
                negs = [q[min(b, q.shape[0] - 1)].tolist() for b in range(len(prompts))]
            guided = dict(guidance_scale=guidance_scale, negative_prompt_ids=negs)
        if seed is None:
            seed = int(torch.randint(0, 2**31 - 1, (1,)).item())  # reference sampling is unseeded
        cuts = {} if top_p == 1.0 and min_p == 0.0 else dict(top_p=top_p, min_p=min_p)
        if vocab_range is not None:
            cuts["vocab_range"] = vocab_range
        if repetition_penalty is not None and repetition_penalty != 1.0:
            cuts["repetition_penalty"] = repetition_penalty
        if num_return_sequences != 1:
            cuts["num_return_sequences"] = num_return_sequences
        if exponential_decay_length_penalty is not None:
            cuts["exponential_decay_length_penalty"] = tuple(exponential_decay_length_penalty)
        if repetition_aware_sampling is not None:
            cuts["repetition_aware_sampling"] = tuple(repetition_aware_sampling)
        outs = self.generate_batch(prompts, eos_token_id, max_length, min_new_tokens, temperature, top_k,
                                   max_new_tokens, seed, greedy=not do_sample, **cuts, **guided)
        n = max(len(o) for o in outs)
        takes = len(outs) // len(prompts)
        res = torch.full((len(outs), input_ids.shape[1] + n), int(eos_token_id), dtype=torch.long)
        for b, o in enumerate(outs):
            res[b, : input_ids.shape[1]] = input_ids[b // takes].cpu()
            res[b, input_ids.shape[1]: input_ids.shape[1] + len(o)] = o
        return res.to(input_ids.device)
