"""The float64 reference of repetition-aware sampling (VALL-E 2's RAS, CosyVoice 2's ``ras_sampling``) the tests compare
the engine with, built on ``sampler_ref``'s sampler: the window count over a slot's generated tokens, the redraw's
Philox uniform, the full-row inverse CDF, the full-row pass's chunk geometry, and a checker for the tokens of one
sampler launch, with per-slot sampling controls and EOS floors when given.
"""
from __future__ import annotations

import math

import numpy as np

from tests.processors_ref import LOGPROB_BARS, model_ref, sampled_ref
from tests.sampler_ref import MARGIN, MASK32, chain64, draw_u, philox4x32_10, processed_scores, ref_token, ref_window

V_THREADS = 256   # consumer threads of the sampler CTA: the full-row pass gives each a chunk of ceil(V / 256) ids
REDRAW_SAMPLED_BAR = 2e-4   # |sampled - float64| of a redrawn token: fp32 sums over the whole row


def chunk_per(V: int) -> int:
    """Ids per thread chunk of ``ras_full_row_draw``: ceil(V / 256) rounded up to a multiple of 4."""
    return (-(-V // V_THREADS) + 3) // 4 * 4


def chunk_of(V: int, tok: int):
    """(thread, [lo, hi)) of the chunk that holds id ``tok``."""
    per = chunk_per(V)
    t = tok // per
    return t, (t * per, min(V, (t + 1) * per))


def window_cut(logits, ngen: int, eos: int, min_new: int, temperature: float, top_k: int, top_p: float, min_p: float):
    """``sampler_ref.ref_window_cut`` on the ids that can enter the window (every id at or above the min(top_k, 64)-th
    largest processed score, ties included): the same result, without sorting the whole row."""
    s = processed_scores(logits, ngen, eos, min_new, temperature)
    k = min(top_k, 64, s.size)
    cand = np.nonzero(s >= np.partition(s, s.size - k)[s.size - k])[0]
    ids, q, margin = chain64(s[cand], top_k, top_p, min_p)
    return cand[ids], q, margin


def cosyvoice_redraws(window_tokens, top_id: int, win_size: int, tau_r: float) -> bool:
    """CosyVoice 2's test, restated: ``rep_num = (tensor(decoded_tokens[-win_size:]) == top_ids).sum()`` then
    ``rep_num >= win_size * tau_r`` (a float64 product)."""
    rep = sum(int(t) == int(top_id) for t in list(window_tokens)[-win_size:]) if win_size > 0 else 0
    return rep >= win_size * tau_r


def min_count(win_size: int, tau_r: float) -> int:
    return int(math.ceil(win_size * tau_r))


def draw_u2(seed: int, ngen: int, stream_key: int) -> float:
    """The redraw's uniform: word 1 of the same Philox block whose word 0 gives ``draw_u``."""
    c1 = philox4x32_10((ngen, stream_key, 0, 0), (seed & MASK32, seed >> 32))[1]
    return (c1 >> 8) * 2.0 ** -24


def window_count(history, n: int, window: int, tok: int) -> int:
    """Occurrences of ``tok`` among the slot's generated tokens [max(0, n - window), n)."""
    return int(sum(int(t) == int(tok) for t in history[max(0, n - window): n]))


def full_scores(logits, ngen: int, eos: int, min_new: int, temperature: float):
    """The scores the redraw samples from: fp32 logit * fp32 (1 / T), EOS -> -inf while ngen < min_new (as ``sample_finish``
    forms them; ids the vocabulary range suppresses already read -inf)."""
    return processed_scores(logits, ngen, eos, min_new, temperature)


def full_logprobs(scores):
    """float64 log-softmax over the whole row of ``scores`` (-inf stays -inf)."""
    s = np.asarray(scores, dtype=np.float64)
    m = s[np.isfinite(s)].max()
    return s - (m + math.log(np.exp(s - m).sum()))


FULL_AMBIG = 2e-5   # |cumulative probability - u2| below this on the full row: fp32 sums of ~1e5 terms drift this far


def ref_full_token(scores, u2: float):
    """Inverse CDF in ascending id order over softmax(scores) in float64: the first id whose cumulative probability
    exceeds u2.  Returns (token, the set of acceptable tokens): every id with mass whose CDF interval comes within
    FULL_AMBIG of u2 (the kernel sums the row in fp32)."""
    p = np.exp(full_logprobs(scores))
    c = np.cumsum(p)
    above = np.nonzero(c > u2)[0]
    pos = np.nonzero(p > 0)[0]
    j = int(above[0]) if above.size else int(pos[-1])
    lo = c - p
    near = pos[(c[pos] > u2 - FULL_AMBIG) & (lo[pos] <= u2 + FULL_AMBIG)]
    return j, {j} | {int(i) for i in near} | ({int(pos[-1])} if u2 + FULL_AMBIG >= c[-1] else set())


def _warp_scan(x):
    """The kernel's inclusive warp scan (Hillis-Steele, shfl_up by 1, 2, 4, 8, 16) of 32 fp32 values."""
    c = np.asarray(x, dtype=np.float32).copy()
    off = 1
    while off < 32:
        c[off:] = (c[off:] + c[:-off]).astype(np.float32)
        off *= 2
    return c


def kernel_full_draw(scores_fp32, m: float, u2: float) -> int:
    """``ras_full_row_draw`` restated in numpy fp32: per-thread chunks of ceil(V / 256) ids rounded up to a multiple
    of 4, each summed in id order; the chunk sums scanned per warp and the 8 warp totals summed in order; the chunk
    that holds u2 * total (else the last chunk with mass) walked 32 ids at a time with a warp scan; when the walk never
    passes the target, its last id with mass.  (The kernel's exp is ``__expf``; here it is numpy's fp32 exp.)"""
    s = np.asarray(scores_fp32, dtype=np.float32)
    V = s.size
    per = chunk_per(V)
    e = np.exp((s - np.float32(m)).astype(np.float32)).astype(np.float32)
    part = np.zeros(V_THREADS, dtype=np.float32)
    for t in range(V_THREADS):
        acc = np.float32(0)
        for x in e[min(V, t * per): min(V, (t + 1) * per)]:
            acc = np.float32(acc + x)
        part[t] = acc
    incl = np.concatenate([_warp_scan(part[w * 32:(w + 1) * 32]) for w in range(V_THREADS // 32)])
    excl = np.concatenate([np.concatenate(([np.float32(0)], incl[w * 32: w * 32 + 31])) for w in range(V_THREADS // 32)])
    base, total = np.zeros(V_THREADS // 32, dtype=np.float32), np.float32(0)
    for w in range(V_THREADS // 32):
        base[w] = total
        total = np.float32(total + incl[w * 32 + 31])
    target = np.float32(np.float32(u2) * total)
    last_t = int(np.nonzero(part > 0)[0][-1])
    sel = [t for t in range(V_THREADS) if part[t] > 0 and np.float32(base[t // 32] + excl[t]) <= target
           and (target < np.float32(base[t // 32] + incl[t]) or t == last_t)]
    assert len(sel) == 1, sel
    t = sel[0]
    cum = np.float32(base[t // 32] + excl[t])
    lo, hi = min(V, t * per), min(V, (t + 1) * per)
    last = -1
    for i0 in range(lo, hi, 32):
        ids = np.arange(i0, i0 + 32)
        ev = np.where(ids < hi, e[np.minimum(ids, V - 1)], np.float32(0)).astype(np.float32)
        c = _warp_scan(ev)
        hit = np.nonzero((ev > 0) & (np.float32(cum) + c > target))[0]
        if hit.size:
            return int(i0 + hit[0])
        pos = np.nonzero(ev > 0)[0]
        if pos.size:
            last = int(i0 + pos[-1])
        cum = np.float32(cum + c[31])
    return last


class RasChecker:
    """Checks every token of sampler launches against the float64 sampler with repetition-aware sampling.

    The trigger is decided on the window the device holds (its own earlier tokens of the slot); a redraw must lie on
    the full-row inverse CDF of u2.  A draw whose top-k token is ambiguous and whose candidates disagree on the
    trigger is skipped (counted); a draw that lands on a neighbour of the float64 token inside the ambiguity band
    counts as ambiguous.  ``entries[s]`` = (window, min_count) or None per slot.

    Per-slot settings (optional): ``controls[s]`` = (T, top_k, top_p, min_p) replaces ``temps[s]`` and the launch's
    top_k, and the window is the float64 chain with the slot's top-p / min-p cut (a window whose cut lies within
    ``sampler_ref.MARGIN`` of its threshold is skipped, counted); ``floors[s]`` replaces ``min_new`` as the slot's EOS
    floor.  ``logits_row`` is the processed row the device sampled from: its stored logits, i.e. transformers'
    penalty and length decay over the slot's actual history (redrawn tokens included) and the vocabulary range.  A
    redraw samples that whole row times the slot's 1 / T with EOS masked below the floor, and no top-k / top-p / min-p
    cut."""

    def __init__(self, sp, entries, temps, min_new: int, greedy: bool = False, controls=None, floors=None):
        self.sp, self.entries, self.temps, self.min_new, self.greedy = sp, entries, temps, min_new, greedy
        self.controls, self.floors = controls, floors
        self.draws = self.redraws = self.skipped = self.ambiguous = 0
        self.worst_lp = 0.0                          # redrawn tokens' sampled log-probabilities
        self.worst = {"sampled": 0.0, "model": 0.0}  # every other checked log-probability (``model_lp`` given)
        self.redrawn = []   # (slot, n, token) of every checked redraw
        self.windows = {}   # (slot, n) -> the kept window ids of every checked draw

    def check(self, logits_row, s: int, n: int, key: int, history, got: int, sampled_lp=None, top_k=None,
              allowed=None, model_lp=None):
        """Slot s drew ``got`` at n_generated n from ``logits_row`` (Philox stream ``key``); ``history``: the slot's
        generated tokens [0, n).  ``sampled_lp``: the device's sampled log-probability of ``got`` (optional; checked
        for redraws, and for every draw when ``model_lp``, the device's model log-probability, is given too).
        Returns True for a redraw, False for a draw that does not trigger, None for a skipped one."""
        sp = self.sp
        floor = self.min_new if self.floors is None else self.floors[s]
        if self.controls is None:
            T = self.temps[s]
            win = ref_window(logits_row, n, sp.eos_id, floor, top_k or sp.top_k, T)
        else:
            T, k, tp, mp = self.controls[s]
            ids, q, margin = window_cut(logits_row, n, sp.eos_id, floor, T, k, tp, mp)
            if margin < MARGIN:
                self.draws += 1
                self.skipped += 1
                return None
            win = (ids, q)
        self.windows[(s, n)] = win[0]
        t, ok1 = ref_token(win, draw_u(sp.seed, n, key), self.greedy)
        self.draws += 1
        e = self.entries[s]
        trig = {e is not None and n > 0 and window_count(history, n, e[0], c) >= e[1] for c in ok1}
        if len(trig) > 1:
            self.skipped += 1
            return None
        if model_lp is not None:
            ref = model_ref(logits_row, got, sp.eos_id, n < floor)
            assert math.isfinite(ref), (s, n, got)
            self.worst["model"] = max(self.worst["model"], abs(float(model_lp) - ref))
            assert abs(float(model_lp) - ref) < LOGPROB_BARS["model"], (s, n, got, model_lp, ref)
        if not trig.pop():
            assert got in ok1, (s, n, got, t, ok1)
            self.ambiguous += got != t
            if model_lp is not None and sampled_lp is not None:
                ref = sampled_ref(logits_row, win[0].tolist(), got, T)
                self.worst["sampled"] = max(self.worst["sampled"], abs(float(sampled_lp) - ref))
                assert abs(float(sampled_lp) - ref) < LOGPROB_BARS["sampled"], (s, n, got, sampled_lp, ref)
            return False
        scores = full_scores(logits_row, n, sp.eos_id, floor, T)
        tok, ok2 = ref_full_token(scores, draw_u2(sp.seed, n, key))
        assert got in ok2, (s, n, got, tok, ok2)
        self.ambiguous += got != tok
        if allowed is not None:
            assert allowed(got), (s, n, got)
        self.redraws += 1
        self.redrawn.append((s, n, got))
        if sampled_lp is not None:
            err = abs(float(sampled_lp) - float(full_logprobs(scores)[got]))
            self.worst_lp = max(self.worst_lp, err)
            assert err < REDRAW_SAMPLED_BAR, (s, n, got, sampled_lp, err)
        return True

    def report(self, name: str):
        print(f"RAS {name}: draws {self.draws}, redraws checked {self.redraws}, skipped {self.skipped}, ambiguous "
              f"{self.ambiguous}, worst redraw log-prob err {self.worst_lp:.2e}, sampled {self.worst['sampled']:.2e}, "
              f"model {self.worst['model']:.2e}")
        assert self.skipped + self.ambiguous <= max(2, 0.02 * self.draws), (self.skipped, self.ambiguous, self.draws)
