"""Speech-LM engine on the C-ABI: weight packing, paged KV pool, prefill + device-side decode loop.

Host-side mirror of inner seam 1 of the reference (``neutts/neutts.py:334-352``): an object with
``.device`` and ``.generate(LongTensor[1,P], max_length=, eos_token_id=, do_sample=, temperature=,
top_k=, use_cache=, min_new_tokens=) -> LongTensor[1,P+N]``, plus a batched ``generate_batch``.
All arithmetic happens in ``libneutts_b200.so``; torch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
import math
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
        rope = cfg.get("rope_theta")
        if rope is None and isinstance(cfg.get("rope_parameters"), dict):
            rope = cfg["rope_parameters"].get("rope_theta")
        heads = cfg["num_attention_heads"]
        return LMShape(
            vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"], intermediate_size=cfg["intermediate_size"],
            num_layers=cfg["num_hidden_layers"], num_heads=heads,
            num_kv_heads=cfg.get("num_key_value_heads", heads),
            head_dim=cfg.get("head_dim") or cfg["hidden_size"] // heads,
            rms_eps=cfg.get("rms_norm_eps", 1e-6), rope_theta=float(rope if rope is not None else 1e6),
            tie_embeddings=bool(cfg.get("tie_word_embeddings", True)))


def _rope_pair_perm(n_heads: int) -> torch.Tensor:
    """Row order that puts RoPE partners (i, i+32) of every 64-row head next to each other."""
    one = torch.stack((torch.arange(32), torch.arange(32) + 32), dim=1).reshape(-1)
    return (torch.arange(n_heads)[:, None] * 64 + one[None, :]).reshape(-1)


def pack_weights(shape: LMShape, sd: dict, device) -> dict:
    """HF Qwen2 state_dict (``model.layers.N.self_attn.q_proj.weight`` ...) -> the packed bf16/fp32
    device tensors the kernels stream (layouts documented in include/neutts_b200.h)."""
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
    """Free-list allocator over the KV page ids (host side; one id addresses every layer)."""

    def __init__(self, num_pages: int, shuffle_seed: int | None = None):
        order = list(range(num_pages))
        if shuffle_seed is not None:
            rng = np.random.default_rng(shuffle_seed)
            rng.shuffle(order)
        self.free = order[::-1]

    def alloc(self, n: int) -> list:
        if n > len(self.free):
            raise RuntimeError(f"KV page pool exhausted: need {n}, have {len(self.free)}")
        return [self.free.pop() for _ in range(n)]

    def release(self, pages) -> None:
        self.free.extend(reversed(list(pages)))


DEFAULT_CONTROLS = (1.0, 50, 1.0, 0.0)   # temperature, top_k, top_p, min_p: the reference's (neutts/neutts.py:338-347)


def _is_seq(v) -> bool:
    return isinstance(v, (list, tuple, np.ndarray, torch.Tensor))


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
    cols = []
    for name, v in (("temperature", temperature), ("top_k", top_k), ("top_p", top_p), ("min_p", min_p)):
        if _is_seq(v):
            v = [x.item() if hasattr(x, "item") else x for x in v]
            if len(v) != n:
                raise ValueError(f"{name} needs one value per prompt ({n}), got {len(v)}")
            cols.append(v)
        else:
            cols.append(None)
    if all(c is None for c in cols) and top_p == 1 and min_p == 0:
        return None
    vals = [c if c is not None else [v] * n for c, v in zip(cols, (temperature, top_k, top_p, min_p))]
    return [check_controls(*row) for row in zip(*vals)]


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
        if rows is None:
            _lib.check(self.L.nt_lm_set_slot_sampling(self.handle, None, _lib.current_stream_ptr()))
            self._slot_sp_host = None
            return
        rows = [check_controls(*r) for r in rows]
        slots = list(range(len(rows))) if slots is None else [int(s) for s in slots]
        if len(slots) != len(rows) or len(set(slots)) != len(slots) or any(not 0 <= s < self.max_batch for s in slots):
            raise ValueError(f"slots must be distinct, in 0..{self.max_batch - 1} and one per row")
        table = list(self._slot_sp_host or [DEFAULT_CONTROLS] * self.max_batch)
        for s, r in zip(slots, rows):
            table[s] = r
        arr = (_lib.SlotSampling * self.max_batch)(*(_lib.SlotSampling(*r) for r in table))
        with torch.cuda.device(self.device):
            _lib.check(self.L.nt_lm_set_slot_sampling(self.handle, arr, _lib.current_stream_ptr()))
        self._slot_sp_host = table

    def _use_controls(self, rows) -> None:
        """Slots 0..len(rows) - 1 take ``rows``; None leaves the table off (switching it off only if an earlier call
        left it on)."""
        if rows is not None or getattr(self, "_slot_sp_host", None) is not None:
            self.set_slot_sampling(rows)

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

    def _use_vocab_range(self, vocab_range) -> None:
        """The engine takes ``vocab_range``; None leaves the range off (switching it off only if an earlier call left
        it on), so a default call makes no engine call."""
        if vocab_range is not None:
            self.set_vocab_range(*vocab_range)
        elif getattr(self, "_vocab_range", None) is not None:
            self.set_vocab_range(None)

    def prefill(self, prompts, sp, return_logits: bool = False):
        """prompts: list of 1-D int sequences.  Fills the KV cache and samples the first token."""
        lens = [len(p) for p in prompts]
        if not lens or min(lens) < 1:
            raise ValueError("empty prompt")
        flat = np.concatenate([np.asarray(p, dtype=np.int64) for p in prompts])
        if flat.min() < 0 or flat.max() >= self.shape.vocab_size:
            raise ValueError("token id out of range")
        # stage through a persistent pinned buffer: the H2D copy of the prompt ids is asynchronous and DMA-able
        if getattr(self, "_ids_pinned", None) is None or self._ids_pinned.numel() < flat.size:
            self._ids_pinned = torch.empty(max(flat.size, self.max_prefill_tokens), dtype=torch.int32).pin_memory()
        staged = self._ids_pinned[: flat.size]
        staged.copy_(torch.from_numpy(flat.astype(np.int32)))
        return self.prefill_packed(staged, lens, sp, return_logits)

    def prefill_packed(self, ids_host: torch.Tensor, lens, sp, return_logits: bool = False):
        """ids_host: int32 host tensor (pinned memory makes the H2D copy asynchronous) holding the
        prompts back to back; lens: their lengths."""
        B = len(lens)
        if not 1 <= B <= self.max_batch:
            raise ValueError(f"batch {B} not in 1..{self.max_batch}")
        if ids_host.dtype != torch.int32 or ids_host.numel() != sum(lens):
            raise ValueError("ids_host must be int32 with sum(lens) elements")
        self.release_pages()
        table = np.zeros((self.max_batch, self.max_pages), dtype=np.int32)
        for b, n in enumerate(lens):
            if not 1 <= n < self.max_ctx:
                raise ValueError(f"prompt {b} has length {n}; must be in 1..{self.max_ctx - 1}")
            need = (min(n + sp.max_new_tokens, self.max_ctx) + self.PAGE - 1) // self.PAGE
            pages = self.pool.alloc(need)
            self._slot_pages[b] = pages
            table[b, :need] = pages
        cu = np.zeros(B + 1, dtype=np.int32)
        cu[1:] = np.cumsum(lens)
        with torch.cuda.device(self.device):
            ids = ids_host.to(self.device, non_blocking=True)
            if self._table_host is None or not np.array_equal(self._table_host, table):
                self.page_table.copy_(torch.from_numpy(table))
                self._table_host = table
            self.n_generated.zero_()
            self.done.zero_()
            logits = torch.empty(B, self.shape.vocab_size, dtype=torch.float32, device=self.device) if return_logits else None
            _lib.check(self.L.nt_lm_prefill(self.handle, C.byref(self.state), ids.data_ptr(),
                                            cu.ctypes.data_as(C.POINTER(C.c_int32)), B, C.byref(sp),
                                            logits.data_ptr() if return_logits else None, _lib.current_stream_ptr()))
        self._B = B
        return logits

    def release_pages(self, slots=None) -> None:
        """Return the KV pages of ``slots`` (default: every slot) to the pool."""
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
        flat = np.concatenate([np.asarray(p, dtype=np.int64) for p in prompts])
        if flat.min() < 0 or flat.max() >= self.shape.vocab_size:
            raise ValueError("token id out of range")
        self.release_pages(slots)
        table = self._table_host.copy()
        for s, n, cap in zip(slots, lens, caps):
            need = (min(n + cap, self.max_ctx) + self.PAGE - 1) // self.PAGE
            pages = self.pool.alloc(need)
            self._slot_pages[s] = pages
            table[s] = 0
            table[s, :need] = pages
        if getattr(self, "_ids_pinned", None) is None or self._ids_pinned.numel() < flat.size:
            self._ids_pinned = torch.empty(max(flat.size, self.max_prefill_tokens), dtype=torch.int32).pin_memory()
        staged = self._ids_pinned[: flat.size]
        staged.copy_(torch.from_numpy(flat.astype(np.int32)))
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

    def generate_batch(self, prompts, eos_token_id: int, max_length: int | None = None, min_new_tokens: int = 50,
                       temperature: float = 1.0, top_k: int = 50, max_new_tokens: int | None = None, seed: int = 0,
                       greedy: bool = False, forced: torch.Tensor | None = None, check_every: int = 64, slot_base: int = 0,
                       top_p: float = 1.0, min_p: float = 0.0, vocab_range=None):
        """Returns a list of int64 CPU tensors with the generated ids of each prompt (EOS included
        when it was sampled), following transformers' stopping rules (stopping_criteria.py:73-84,
        467-471): stop at EOS or when prompt + generated reaches max_length.  ``max_new_tokens`` may also be a
        list with one cap per prompt.  ``temperature``, ``top_k``, ``top_p`` and ``min_p`` are each a scalar or one
        value per prompt (per-slot controls, ``set_slot_sampling``).  ``vocab_range``: (lo, hi) restricts every draw to
        [lo, hi) plus EOS (``set_vocab_range``); None leaves the range off."""
        if vocab_range is not None:   # validated before any engine call
            vocab_range = check_vocab_range(vocab_range, self.shape.vocab_size)
        max_length = max_length or self.max_ctx
        if max_length > self.max_ctx:
            raise ValueError(f"max_length {max_length} exceeds the engine context {self.max_ctx}")
        lens = [len(p) for p in prompts]
        if min(max_length - n for n in lens) < 1:
            raise ValueError("prompt already at max_length")
        # max_length counts prompt + generated PER SEQUENCE (stopping_criteria.py:73-84): a long prompt in the batch
        # must not shorten its neighbours, so every slot gets its own cap and the loop runs to the largest one
        caps = self._caps(lens, max_length, max_new_tokens)
        limit = max(caps)
        rows = per_prompt_controls(len(prompts), temperature, top_k, top_p, min_p)
        if rows is not None:   # the launch scalars are validated but not used while the table is on
            temperature, top_k = rows[0][0], rows[0][1]
        sp = self.sampling(eos_token_id, min_new_tokens, limit, top_k, temperature, seed, greedy, forced,
                           limits=caps if min(caps) < limit else None, slot_base=slot_base)
        self._use_controls(rows)
        self._use_vocab_range(vocab_range)
        self.prefill(prompts, sp)
        remaining = limit - 1
        B = len(prompts)
        while remaining > 0:
            n = min(check_every, remaining)
            self.decode(n, sp)
            remaining -= n
            if remaining > 0 and bool(self.done[:B].all()):  # one small D2H read per `check_every` steps
                break
        ngen = self.n_generated[:B].cpu()
        toks = self.out_tokens[:B].cpu()
        return [toks[b, : int(ngen[b])].long() for b in range(B)]

    def generate_queue(self, prompts, eos_token_id: int, max_length: int | None = None, min_new_tokens: int = 50,
                       temperature: float = 1.0, top_k: int = 50, max_new_tokens: int | None = None, seed: int = 0,
                       greedy: bool = False, check_every: int = 32, slot_base: int = 0, top_p: float = 1.0,
                       min_p: float = 0.0, vocab_range=None):
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
        ``generate_batch``: set once before the first prefill, it holds across every refill."""
        if vocab_range is not None:   # validated before any engine call
            vocab_range = check_vocab_range(vocab_range, self.shape.vocab_size)
        max_length = max_length or self.max_ctx
        if max_length > self.max_ctx:
            raise ValueError(f"max_length {max_length} exceeds the engine context {self.max_ctx}")
        n = len(prompts)
        if n == 0:
            return []
        if check_every < 1:
            raise ValueError("check_every must be >= 1")
        lens = [len(p) for p in prompts]
        if min(max_length - m for m in lens) < 1:
            raise ValueError("prompt already at max_length")
        caps = self._caps(lens, max_length, max_new_tokens)
        S = min(n, self.max_batch)
        ctl_rows = per_prompt_controls(n, temperature, top_k, top_p, min_p)
        if ctl_rows is not None:
            temperature, top_k = ctl_rows[0][0], ctl_rows[0][1]
        sp = self.sampling(eos_token_id, min_new_tokens, max(caps), top_k, temperature, seed, greedy,
                           limits=caps[:S], slot_base=slot_base)
        self._use_controls(ctl_rows[:S] if ctl_rows is not None else None)
        self._use_vocab_range(vocab_range)
        self.prefill([prompts[i] for i in range(S)], sp)
        occ = list(range(S))   # prompt held by each slot, None once harvested
        ngen = [1] * S         # generated tokens per slot, as of the last read
        nxt = S                # next prompt to admit
        out = [None] * n
        # a sequence can finish inside its prefill: a cap of 1, or EOS when it is not masked at step 0
        at_prefill = lambda idx: min_new_tokens <= 0 or min(caps[i] for i in idx) <= 1
        read = at_prefill(range(S))
        while True:
            if read:
                st = torch.stack((self.n_generated[:S], self.done[:S])).cpu()   # the one small D2H read per launch
                ngen = st[0].tolist()
                fin = [s for s in range(S) if occ[s] is not None and int(st[1, s])]
                if fin:
                    rows = self.out_tokens[fin].cpu()
                    for r, s in enumerate(fin):
                        out[occ[s]] = rows[r, : ngen[s]].long()
                        occ[s] = None
                    take = fin[: n - nxt]
                    if take:
                        idx = list(range(nxt, nxt + len(take)))
                        nxt += len(take)
                        if ctl_rows is not None:   # the newcomers' controls, before their prefill on the same stream
                            self.set_slot_sampling([ctl_rows[i] for i in idx], slots=take)
                        self.prefill_slots(take, [prompts[i] for i in idx], sp, [slot_base + i for i in idx],
                                           limits=[caps[i] for i in idx])
                        for s, i in zip(take, idx):
                            occ[s], ngen[s] = i, 1
                        if at_prefill(idx):
                            continue   # read again before decoding: a newcomer may be done already
            live = [s for s in range(S) if occ[s] is not None]
            if not live:
                break
            left = [caps[occ[s]] - ngen[s] for s in live]
            steps = max(1, min(check_every, min(left) if nxt < n else max(left)))
            self.decode(steps, sp)
            read = True
        self.release_pages()
        return out

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, max_length: int = 2048, eos_token_id: int | None = None,
                 do_sample: bool = True, temperature: float = 1.0, top_k: int = 50, use_cache: bool = True,
                 min_new_tokens: int = 0, max_new_tokens: int | None = None, seed: int | None = None,
                 top_p: float = 1.0, min_p: float = 0.0, vocab_range=None, **_):
        """transformers-compatible seam used by ``NeuTTS._infer_torch`` (neutts/neutts.py:338-347).  ``top_p`` and
        ``min_p`` act as transformers' TopPLogitsWarper / MinPLogitsWarper; ``vocab_range`` (lo, hi) suppresses every
        id outside [lo, hi) and EOS (``set_vocab_range``); other generation kwargs are ignored."""
        if eos_token_id is None:
            raise ValueError("eos_token_id is required")
        if input_ids.dim() != 2:
            raise ValueError("input_ids must be [B, P]")
        prompts = [row.tolist() for row in input_ids.cpu()]
        if seed is None:
            seed = int(torch.randint(0, 2**31 - 1, (1,)).item())  # reference sampling is unseeded
        cuts = {} if top_p == 1.0 and min_p == 0.0 else dict(top_p=top_p, min_p=min_p)
        if vocab_range is not None:
            cuts["vocab_range"] = vocab_range
        outs = self.generate_batch(prompts, eos_token_id, max_length, min_new_tokens, temperature, top_k,
                                   max_new_tokens, seed, greedy=not do_sample, **cuts)
        n = max(len(o) for o in outs)
        res = torch.full((len(outs), input_ids.shape[1] + n), int(eos_token_id), dtype=torch.long)
        for b, o in enumerate(outs):
            res[b, : input_ids.shape[1]] = input_ids[b].cpu()
            res[b, input_ids.shape[1]: input_ids.shape[1] + len(o)] = o
        return res.to(input_ids.device)
