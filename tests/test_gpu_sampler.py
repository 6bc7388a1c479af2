"""Every speech-LM sampler path against a float64 top-k sampler on the same logits and Philox draws.

The logit-parity tests are teacher-forced: the sampler runs, but the forced token overrides whatever it selected, so a
wrong threshold, tie order or EOS mask changes the audio without moving one logit.  The tests here compare what each
sampler path kept and drew with a plain float64 reference that reads the operands the kernel read: its own logits
(returned by the call), its own ``n_generated`` and its own Philox counter.

Sampler paths (both run ``sample_tiles_seq`` and end in ``sample_finish`` in lm_device.cuh):
  * tile-max sampler kernel (``topk_tiles_kernel``): prefill, ``prefill_slots`` with a ``row_slot`` map and the per-op
    decode chain, on raw tile maxima -- from the tensor-core lm_head's epilogue where its GEMM tiles the vocabulary by
    128, from ``tile_max_kernel`` behind the GEMV lm_head (batch <= 4) and narrower GEMM tiles -- with the EOS tile
    patched through ``fix_tile`` while EOS is masked;
  * the persistent decode kernel's sampler (``sample_phase``): processed tile maxima written by ``epi_head``.
Inside ``sample_tiles_seq`` the *direct*, *fast* and *general* paths are chosen from the tile maxima; ``tile_path``
restates that choice so that every case can assert which one its rows took.

The model is programmable: one layer with wo = 0 and down_proj = 0 leaves the residual stream at exactly
``embed[tok]``, and ``embed[t]`` is a one-hot on the pattern that owns ``t mod P``.  Token t's logits are then one
lm_head column (times a common scale), so any bf16 pattern can be written there and exact ties stay exact on every
activation path.  A pattern's strong candidates sit on the ids it owns, so every drawn token selects the same pattern
again and a batch row keeps its pattern for the whole run.  That also tests the hand-off: step s+1's logits must be the
logits of the token drawn at step s.

BARS lists the worst values measured on the H100 and the bars, about 4x above them.
"""
from __future__ import annotations

import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O
from tests.helpers import make_lm

# Worst errors measured on one H100 80GB HBM3 (132 SMs, 700 W power limit) over the whole GPU matrix, and the bars:
#   kept probabilities, max |p - p64| (__expf, fp32 sums and division)                  8.8e-8 -> 4e-7
#   next step's logits against the float64 logits of the drawn token (relative RMS)     4.3e-5 -> 2e-4
#   draws within AMBIG of a boundary: 4 of ~610 (0.7 %); a case may have one, or 1 % of its draws
BARS = {"prob": 4e-7, "handoff": 2e-4, "ambiguous": 0.01}
AMBIG = 1e-5          # |cumulative probability - u| below this: either neighbour is accepted

MASK32 = 0xFFFFFFFF
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
SEED = (1 << 32) + 0x5EED   # the key's high word is 1: a sampler that drops it draws differently


# ====================================================================================== float64 reference sampler
def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) as ``philox4x32_10`` in lm_device.cuh: ten rounds, each two 32x32->64
    multiplies whose high halves are xored with the other counter words and the key, the key bumped by the Weyl
    constants after every round.  ctr: 4 ints, key: 2 ints (uint32).  Returns the 4 output words."""
    c0, c1, c2, c3 = (int(x) & MASK32 for x in ctr)
    k0, k1 = (int(x) & MASK32 for x in key)
    for _ in range(10):
        p0, p1 = PHILOX_M[0] * c0, PHILOX_M[1] * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & MASK32, (p0 >> 32) ^ c3 ^ k1, p0 & MASK32
        k0, k1 = (k0 + PHILOX_W[0]) & MASK32, (k1 + PHILOX_W[1]) & MASK32
    return c0, c1, c2, c3


def draw_u(seed: int, ngen: int, stream_key: int) -> float:
    """The uniform ``sample_finish`` draws: counter {n_generated, stream key, 0, 0}, key (seed low, seed high word),
    u = (word 0 >> 8) * 2^-24.  The stream key is slot + slot_base, or the key ``prefill_slots`` gave the slot."""
    c0 = philox4x32_10((ngen, stream_key, 0, 0), (seed & MASK32, seed >> 32))[0]
    return (c0 >> 8) * 2.0 ** -24


def processed_scores(logits, ngen: int, eos: int, min_new: int, temperature: float):
    """The kernels' logits processors: EOS -> -inf while ngen < min_new_tokens, then fp32(logit) * fp32(1 / T) (the
    reciprocal formed in fp32, as ``1.0f / temperature``).  HF divides by T instead; see
    ``test_inverse_temperature_product_differs_from_division``."""
    s = np.asarray(logits, dtype=np.float32).copy()
    s *= np.float32(1.0) / np.float32(temperature)
    if ngen < min_new:
        s[eos] = -np.inf
    return s


def ref_window(logits, ngen: int, eos: int, min_new: int, top_k: int, temperature: float):
    """Kept window of the kernels: processed scores ordered by (score desc, id asc), the first min(top_k, 64); softmax
    in float64 over the kept scores.  Returns (ids int64 [k], probabilities float64 [k])."""
    s = processed_scores(logits, ngen, eos, min_new, temperature)
    k = min(top_k, 64, s.size)
    ids = np.arange(s.size)
    order = np.lexsort((ids, -s.astype(np.float64)))[:k]
    sc = s[order].astype(np.float64)
    p = np.exp(sc - sc[0])
    return order.astype(np.int64), p / p.sum()


def ref_token(window, u: float, greedy: bool = False):
    """Inverse CDF over the window: the first j whose float64 cumulative probability exceeds u.  Returns (token, the set
    of acceptable tokens): a draw within AMBIG of a boundary accepts either neighbour.  Greedy takes window[0]."""
    ids, p = window
    if greedy:
        return int(ids[0]), {int(ids[0])}
    c = np.cumsum(p)
    above = np.nonzero(c > u)[0]
    j = int(above[0]) if above.size else len(ids) - 1
    ok = {int(ids[j])}
    if j > 0 and abs(c[j - 1] - u) < AMBIG:
        ok.add(int(ids[j - 1]))
    if j + 1 < len(ids) and abs(c[j] - u) < AMBIG:
        ok.add(int(ids[j + 1]))
    return int(ids[j]), ok


def prob_err(got, ref) -> float:
    """max |got - ref|; inf when ``got`` holds a NaN or an inf (so that max() over errors cannot drop it)."""
    got = np.asarray(got, dtype=np.float64)
    if not np.isfinite(got).all():
        return math.inf
    return float(np.abs(got - np.asarray(ref, dtype=np.float64)).max(initial=0.0))


def rel_rms(got, ref) -> float:
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    if not np.isfinite(got).all():
        return math.inf
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-300))


def tile_maxima(scores):
    """Per-128-column maxima of a score row (a partial last tile is padded with -inf)."""
    nt = -(-scores.size // 128)
    pad = np.full(nt * 128, -np.inf, dtype=np.float32)
    pad[: scores.size] = scores
    return pad.reshape(nt, 128).max(axis=1)


def tile_path(proc, top_k: int) -> str:
    """Which path ``sample_tiles_seq`` takes for processed scores ``proc`` [V] (restated from lm_device.cuh):
    "direct" when the top_k-th of the 256 per-thread maxima, L, is finite, at most 256 tiles reach it and at most 512
    logits of those tiles do; else the k = min(top_k, 64, tiles) best tiles (value desc, index asc) are scanned for
    logits >= the k-th tile maximum (every logit when there are fewer tiles than top_k): "fast" for <= 512 such
    candidates, "general" (the global candidate arrays) beyond."""
    V = proc.size
    nt = -(-V // 128)
    tm = tile_maxima(proc)
    rows = np.full(nt * 128, -np.inf, dtype=np.float32)
    rows[:V] = proc
    rows = rows.reshape(nt, 128)
    ktop = min(top_k, 64)
    if nt <= 2048:
        best = np.array([tm[t::256].max() if t < nt else -np.inf for t in range(256)], dtype=np.float32)
        L = best[np.lexsort((np.arange(256), -best.astype(np.float64)))[ktop - 1]]
        if L > -np.inf:
            hit = tm >= L
            if hit.sum() <= 256 and (rows[hit] >= L).sum() <= 512:
                return "direct"
    k = min(ktop, nt)
    order = np.lexsort((np.arange(nt), -tm.astype(np.float64)))
    chosen = order[:k]
    if nt < top_k:
        nc = sum(min(128, V - 128 * int(t)) for t in chosen)
    else:
        nc = int((rows[chosen] >= tm[order[k - 1]]).sum())
    return "fast" if nc <= 512 else "general"


# ====================================================================================== logit-programmable model
P = 16                      # token t reads the pattern that owns t mod P
H, INTER = 128, 256
BACKGROUND = -30.0          # every id a pattern does not own
PATTERNS = ["gauss", "ties", "flat", "plateau", "eos", "partial", "onetile"]
PATTERNS_ALL = PATTERNS + ["stairs"]   # stairs: top-k winners alone in the tiles of distinct threads


class Programmable:
    """Patterns -> residue owners, EOS id, target logits; the oracle weights of the model that realises them."""

    def __init__(self, V: int, seed: int = 0):
        self.V, self.nt = V, -(-V // 128)
        rng = np.random.default_rng(seed)
        free = list(range(P))
        own = {"partial": [(V - 1) % P, (V - 2) % P]}
        for r in own["partial"]:
            free.remove(r)
        for name, n in (("ties", 1), ("flat", 1), ("plateau", 4), ("eos", 1), ("onetile", 1), ("stairs", 1)):
            own[name], free = free[:n], free[n:]
        own["gauss"] = free
        self.owner = np.zeros(P, dtype=np.int64)
        for j, name in enumerate(PATTERNS_ALL):
            self.owner[own[name]] = j
        ids = np.arange(V)
        self.owned = {name: ids[np.isin(ids % P, own[name])] for name in PATTERNS_ALL}
        r_eos = own["eos"][0]
        base = (self.nt // 2) * 128 + 40
        self.eos = base - base % P + r_eos
        self.target = np.full((len(PATTERNS_ALL), V), BACKGROUND, dtype=np.float64)
        for j, name in enumerate(PATTERNS_ALL):
            self.target[j, self.owned[name]] = self._pattern(name, self.owned[name], rng)
        # what the lm_head holds: the targets over the common activation scale, rounded to bf16 (ties stay ties)
        self.xs = 1.0 / math.sqrt(1.0 / H + 1e-6)
        self.W = torch.from_numpy(self.target / self.xs).float().bfloat16().double()   # [n_pat, V]

    def _pattern(self, name, owned, rng):
        V, nt = self.V, self.nt
        tile = owned // 128
        low = np.clip(rng.normal(0.0, 1.0, owned.size), -4.0, 3.0)
        pos = {int(i): n for n, i in enumerate(owned)}

        def first_per_tile(tiles, skip=()):
            out = []
            for t in tiles:
                c = owned[(tile == t) & ~np.isin(owned, list(skip))]
                if c.size:
                    out.append(int(c[rng.integers(c.size)]))
            return out

        if name == "gauss":
            return rng.normal(0.0, 2.0, owned.size)
        v = low
        if name == "ties":            # 20 distinct winners, then 84 values tied at 10 (smaller ids must win)
            sel = rng.choice(owned, min(104, owned.size), replace=False)
            for n, i in enumerate(sel):
                v[pos[int(i)]] = 12.0 + 0.25 * n if n < 20 else 10.0
        elif name in ("flat", "eos"):  # every tile's maximum is 5: > 256 tiles reach L, the direct path gives up
            eos_tile = self.eos // 128 if name == "eos" else -1
            tiles = [t for t in range(nt) if t != eos_tile]
            for i in first_per_tile(tiles):
                v[pos[i]] = 5.0
            hi_tiles = tiles[3: 3 + 10 * max(1, nt // 12): max(1, nt // 12)][:10]
            for n, i in enumerate(first_per_tile(hi_tiles)):   # a few larger maxima: candidates above the tie
                v[pos[i]] = 6.0 + 0.2 * n
            if name == "eos":              # EOS is the largest logit, next to strong candidates of its own tile
                v[pos[self.eos]] = 15.0
                for n, i in enumerate(first_per_tile([eos_tile] * 2, skip=(self.eos,))):
                    v[pos[i]] = 4.5 - 0.25 * n
        elif name == "plateau":        # > 512 equal values in the best tiles: the general path
            T = min(40, nt)
            v[tile < T] = 5.0
            for n, i in enumerate(first_per_tile(range(min(3, nt)))):
                v[pos[i]] = 6.0 + 0.5 * n
        elif name == "partial":        # winners in the last (partial) tile, including V - 1 and V - 2
            last = owned[tile == nt - 1]
            v[pos[V - 1]], v[pos[V - 2]] = 9.0, 8.5
            for n, i in enumerate([i for i in last if i < V - 2][-3:]):
                v[pos[int(i)]] = 8.0 - 0.5 * n
            v[pos[int(owned[0])]] = 9.0    # a tie with V - 1 at a smaller id
            for n, i in enumerate(first_per_tile(range(0, nt, max(1, nt // 60)))[:60]):
                v[pos[i]] = max(v[pos[i]], 6.0 + 0.01 * n)
        elif name == "stairs":         # 64 distinct winners, one per tile in tiles 0..63 (threads 0..63): the top_k-th
            for n, i in enumerate(first_per_tile(range(min(64, nt)))):   # thread maximum is exactly the top_k-th logit
                v[pos[i]] = 10.0 + 0.1 * n
        elif name == "onetile":        # every winner inside one tile
            hot = owned[tile == min(5, nt - 1)]
            for n, i in enumerate(hot):
                v[pos[int(i)]] = 10.0 - 0.5 * n
        return v

    def token_for(self, name: str, n: int = 0) -> int:
        """An id whose logits are pattern ``name`` (never EOS)."""
        ids = self.owned[name]
        ids = ids[ids != self.eos]
        return int(ids[(7 + 3 * n) % ids.size])

    def pattern_of(self, tok: int) -> int:
        return int(self.owner[tok % P])

    def ref_logits(self, tok: int):
        """float64 logits of the step whose input token is ``tok``."""
        return self.xs * self.W[self.pattern_of(tok)].numpy()

    def oracle(self):
        cfg = O.LMConfig(vocab_size=self.V, hidden_size=H, intermediate_size=INTER, num_layers=1, num_heads=2,
                         num_kv_heads=1, head_dim=64, tie_embeddings=False)
        z = torch.zeros
        layer = dict(ln1=torch.ones(H), wq=z(128, H), bq=z(128), wk=z(64, H), bk=z(64), wv=z(64, H), bv=z(64),
                     wo=z(H, 128), ln2=torch.ones(H), wg=z(INTER, H), wu=z(INTER, H), wd=z(H, INTER))
        embed = torch.zeros(self.V, H)
        embed[torch.arange(self.V), torch.from_numpy(self.owner[np.arange(self.V) % P])] = 1.0
        head = torch.zeros(self.V, H)
        head[:, : len(PATTERNS_ALL)] = self.W.T.float()
        return cfg, O.LMWeights(embed=embed, layers=[layer], final_norm=torch.ones(H), lm_head=head)


_MODELS = {}


def programmable(V: int) -> Programmable:
    if V not in _MODELS:
        _MODELS[V] = Programmable(V)
    return _MODELS[V]


def fp32_logits(m: Programmable, name: str):
    """The logits a kernel computes for pattern ``name``, to fp32 accuracy (CPU path checks)."""
    return (np.float32(m.xs) * m.W[PATTERNS_ALL.index(name)].numpy().astype(np.float32)).astype(np.float32)


# ---------------------------------------------------------------------------------------- CPU tests of the reference
def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10."""
    assert philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    assert philox4x32_10((MASK32,) * 4, (MASK32, MASK32)) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
    assert philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0)) == (
        0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)


def test_philox_constants_match_curand():
    hdr = "/usr/local/cuda/include/curand_philox4x32_x.h"
    if not os.path.exists(hdr):
        pytest.skip("CUDA headers not installed")
    src = open(hdr).read()
    want = {"PHILOX_M4x32_0": PHILOX_M[0], "PHILOX_M4x32_1": PHILOX_M[1], "PHILOX_W32_0": PHILOX_W[0],
            "PHILOX_W32_1": PHILOX_W[1]}
    for name, val in want.items():
        m = re.search(rf"#define\s+{name}\s+\(?(0x[0-9A-Fa-f]+)", src)
        assert m and int(m.group(1), 16) == val, name


def test_draw_u_counter_and_key_layout():
    c0 = philox4x32_10((7, 3, 0, 0), (SEED & MASK32, 1))[0]
    assert draw_u(SEED, 7, 3) == (c0 >> 8) / 16777216.0
    assert 0.0 <= draw_u(SEED, 0, 0) < 1.0
    us = {draw_u(SEED, n, k) for n in range(4) for k in range(4)}
    assert len(us) == 16                                            # counter words 0 and 1 both matter
    assert draw_u(SEED, 5, 2) != draw_u(SEED & MASK32, 5, 2)        # so does the key's high word


def test_ref_window_matches_oracle_topk_probs():
    g = torch.Generator().manual_seed(5)
    V, eos = 5000, 4321
    for top_k, T, ngen in ((50, 0.7, 3), (64, 1.5, 60), (1, 1.0, 0), (17, 1.0, 49)):
        logits = torch.randn(V, generator=g) * 2
        logits[eos] = 20.0
        ids, p = ref_window(logits.numpy(), ngen, eos, 50, top_k, T)
        oi, op = O.topk_probs(logits, ngen, eos, 50, T, top_k)
        assert ids.tolist() == oi.tolist()
        assert prob_err(p, op.double().numpy()) < 1e-6             # HF divides by T: fp32 rounding apart
        assert (eos in ids.tolist()) == (ngen >= 50)


def test_ref_window_ties_keep_smaller_ids():
    logits = np.zeros(300, dtype=np.float32)
    logits[[250, 7, 130, 40, 200]] = 3.0
    logits[299] = 4.0
    ids, p = ref_window(logits, 0, 0, 0, 4, 1.0)
    assert ids.tolist() == [299, 7, 40, 130]
    assert np.allclose(p[1:], p[1]) and p[0] > p[1]


def test_ref_window_eos_mask_and_partial_last_tile():
    V, eos = 16462, 16461                         # 128 full tiles + 78 columns; EOS is the very last id
    logits = np.zeros(V, dtype=np.float32)
    logits[eos], logits[V - 2], logits[5] = 9.0, 8.0, 7.0
    ids, _ = ref_window(logits, 2, eos, 3, 3, 1.0)
    assert ids.tolist() == [V - 2, 5, 0]           # masked while n_generated < min_new_tokens
    ids, _ = ref_window(logits, 3, eos, 3, 3, 1.0)
    assert ids.tolist() == [eos, V - 2, 5]
    tm = tile_maxima(processed_scores(logits, 2, eos, 3, 1.0))
    assert tm.size == 129 and tm[-1] == 8.0        # the padding of the partial tile never wins


def test_inverse_temperature_product_differs_from_division():
    """The kernels multiply by fp32(1/T); transformers divides by T.  For T = 0.7 the two differ in the last bit for a
    sizeable share of logits (never in their order by more than that)."""
    x = np.random.default_rng(0).normal(0, 3, 10000).astype(np.float32)
    mul = x * (np.float32(1) / np.float32(0.7))
    div = x / np.float32(0.7)
    diff = mul != div
    assert 0.05 < diff.mean() < 0.9
    assert np.abs((mul - div)[diff] / div[diff]).max() < 2.5e-7     # one ulp
    assert np.array_equal(processed_scores(x, 0, 0, 0, 0.7)[1:], mul[1:])


def test_ref_token_boundaries():
    w = (np.array([10, 20, 30, 40]), np.array([0.5, 0.25, 0.125, 0.125]))
    assert ref_token(w, 0.0) == (10, {10})
    assert ref_token(w, 0.3) == (10, {10})
    assert ref_token(w, 0.5) == (20, {10, 20})                     # exactly on the boundary: either neighbour
    assert ref_token(w, 0.5 - 2e-6) == (10, {10, 20})
    assert ref_token(w, 0.5 + 2e-5) == (20, {20})
    assert ref_token(w, 0.874999) == (30, {30, 40})
    assert ref_token(w, 0.9) == (40, {40})
    assert ref_token(w, 1.0 - 2.0 ** -24) == (40, {40})           # cumulative sum short of u: the last candidate
    assert ref_token(w, 0.9, greedy=True) == (10, {10})


def test_error_measures_report_non_finite_output():
    assert prob_err([0.5, float("nan")], [0.5, 0.5]) == math.inf
    assert max(0.0, prob_err([math.inf], [1.0])) == math.inf
    assert rel_rms([1.0, float("nan")], [1.0, 1.0]) == math.inf
    assert prob_err([0.5, 0.25], [0.5, 0.5]) == 0.25


def test_odd_vocabulary_is_rejected():
    """The GEMV lm_head works on row pairs, so the library takes even vocabularies only: 16461 and 4141 (the odd sizes
    one would pick for a partial last tile) are refused at configuration; the GPU tests use 16462 and 4142."""
    import ctypes as C

    from neutts_air_b200 import _lib, build

    build.build()
    L = _lib.lib()
    for V in (16461, 4141):
        cfg = _lib.LMConfig(V, H, INTER, 1, 2, 1, 64, 1e-6, 1e6, 4, 256, 64, 16, 256)
        assert L.nt_lm_workspace_bytes(C.byref(cfg)) == 0 and b"even" in L.nt_last_error()
        cfg.vocab_size = V + 1
        assert L.nt_lm_workspace_bytes(C.byref(cfg)) > 0


@pytest.mark.parametrize("V", [217472, 16462, 4142])
def test_patterns_force_their_paths(V):
    """The patterns reach the sample_tiles_seq paths they are meant for (per tile_path on fp32 logits)."""
    m = programmable(V)
    want = {217472: dict(gauss="direct", ties="direct", flat="fast", plateau="general", eos="fast", partial="direct",
                         onetile="direct", stairs="direct"),
            16462: dict(flat="direct", plateau="general", partial="direct"),
            4142: {n: "general" for n in PATTERNS_ALL}}[V]
    for name, path in want.items():
        proc = processed_scores(fp32_logits(m, name), 0, m.eos, 3, 1.0)
        assert tile_path(proc, 50) == path, (name, path)
    # ties: the 84 equal values straddle the 50th and 64th rank; EOS is the largest logit of its pattern
    ids, _ = ref_window(fp32_logits(m, "ties"), 0, m.eos, 0, 64, 1.0)
    vals = fp32_logits(m, "ties")[ids]
    assert (vals[20:] == vals[20]).all() and (np.diff(ids[20:]) > 0).all()
    st = np.sort(fp32_logits(m, "stairs"))[::-1]
    assert (np.diff(st[: min(64, m.nt)]) < 0).all() and st[min(64, m.nt)] < st[min(64, m.nt) - 1]
    lg = fp32_logits(m, "eos")
    assert lg.argmax() == m.eos and (m.eos // 128) != m.nt - 1
    assert [m.pattern_of(m.token_for(n, k)) for n in PATTERNS for k in range(3)] == [j for j in range(7) for _ in range(3)]
    part = fp32_logits(m, "partial")
    assert part[V - 1] == part.max() and part[V - 1] in part[: V - 128]    # V - 1 ties a smaller id


# ====================================================================================== GPU driver
class Checker:
    """Compares the sampler launches of one engine with the float64 reference and keeps score."""

    def __init__(self, m: Programmable, lm, sp, greedy: bool, limits=None):
        self.m, self.lm, self.sp, self.greedy = m, lm, sp, greedy
        self.limits = limits
        self.worst_prob = self.worst_handoff = 0.0
        self.draws = self.ambiguous = 0
        self.paths = {}
        self.cap = lm.debug_capture_sampler()

    def snapshot(self):
        lm = self.lm
        return dict(ngen=lm.n_generated.cpu().numpy().copy(), done=lm.done.cpu().numpy().copy(),
                    seq=lm.seq_lens.cpu().numpy().copy(), cur=lm.cur_token.cpu().numpy().copy(),
                    out=lm.out_tokens.cpu().numpy().copy())

    def lim(self, s):
        cap = self.sp.max_new_tokens
        return min(cap, self.limits[s]) if self.limits is not None and s < len(self.limits) else cap

    def expect_token(self, logits_row, ngen, key):
        sp = self.sp
        win = ref_window(logits_row, ngen, sp.eos_id, sp.min_new_tokens, sp.top_k, sp.temperature)
        tok, ok = ref_token(win, draw_u(sp.seed, ngen, key), self.greedy)
        self.draws += 1
        self.ambiguous += len(ok) > 1
        return win, tok, ok

    def check_launch(self, logits, rows_slots, keys, before, after, advance, windows=True, tag=""):
        """One sampler launch: logits [R, V] (row i -> slot rows_slots[i], Philox stream keys[i]); state before/after."""
        sp, m = self.sp, self.m
        tv, ti, tt = (t.cpu().numpy() for t in self.cap)
        touched = set()
        for i, s in enumerate(rows_slots):
            touched.add(s)
            lg = logits[i]
            ngen = int(before["ngen"][s])
            win, tok, ok = self.expect_token(lg, ngen, keys[i])
            if windows:
                k = len(win[0])
                assert ti[i, :k].tolist() == win[0].tolist(), (tag, i, ti[i, :k].tolist(), win[0].tolist())
                assert (ti[i, k:] == -1).all() and (tv[i, k:] == 0).all(), (tag, i)
                err = prob_err(tv[i, :k], win[1])
                self.worst_prob = max(self.worst_prob, err)
                assert err < BARS["prob"], (tag, i, err)
                assert int(tt[i]) in ok, (tag, i, int(tt[i]), tok, ok)
                proc = processed_scores(lg, ngen, sp.eos_id, sp.min_new_tokens, sp.temperature)
                path = tile_path(proc, sp.top_k)
                self.paths[path] = self.paths.get(path, 0) + 1
            if before["done"][s]:                       # a finished slot is left untouched
                for f in ("ngen", "done", "seq", "cur"):
                    assert after[f][s] == before[f][s], (tag, s, f)
                assert (after["out"][s] == before["out"][s]).all(), (tag, s)
                continue
            got = int(after["out"][s, ngen])
            assert got in ok, (tag, s, got, tok, ok)
            assert after["ngen"][s] == ngen + 1 and after["cur"][s] == got, (tag, s)
            seq = int(before["seq"][s]) + advance if advance else int(after["seq"][s])
            assert after["seq"][s] == seq, (tag, s, after["seq"][s], seq)
            stop = got == sp.eos_id or ngen + 1 >= self.lim(s) or ngen + 1 >= self.lm.max_new or seq + 1 >= self.lm.max_ctx
            assert bool(after["done"][s]) == stop, (tag, s, got, ngen)
        return touched

    def check_handoff(self, logits, slots, cur_tokens, tag=""):
        """Row i of ``logits`` must be the float64 logits of token cur_tokens[slot i] (the token drawn before)."""
        for i, s in enumerate(slots):
            err = rel_rms(logits[i], self.m.ref_logits(int(cur_tokens[s])))
            self.worst_handoff = max(self.worst_handoff, err)
            assert err < BARS["handoff"], (tag, i, s, err)

    def check_tmax(self, logits, ngens, processed: bool, tag=""):
        """"tmax" rows: the persistent kernel's processed per-tile maxima (times fp32 1/T, EOS masked while
        n_generated < min_new_tokens), or the chain GEMM's raw maxima.  Bit-exact."""
        sp = self.sp
        R, nt = logits.shape[0], self.m.nt
        tm = self.lm.debug_buffer("tmax", (R, nt)).cpu().numpy()
        for i in range(R):
            want = tile_maxima(processed_scores(logits[i], ngens[i], sp.eos_id, sp.min_new_tokens, sp.temperature)
                               if processed else logits[i])
            assert np.array_equal(tm[i], want), (tag, i, np.nonzero(tm[i] != want)[0][:5])

    def report(self, name):
        print(f"SAMPLER {name}: draws {self.draws} ambiguous {self.ambiguous} worst prob err {self.worst_prob:.2e} "
              f"hand-off {self.worst_handoff:.2e} paths {dict(sorted(self.paths.items()))}")
        assert self.ambiguous <= max(1, BARS["ambiguous"] * self.draws), (self.ambiguous, self.draws)


def _set_impl(monkeypatch, impl):
    if impl:
        monkeypatch.setenv("NT_DECODE_IMPL", impl)
    else:
        monkeypatch.delenv("NT_DECODE_IMPL", raising=False)


def _prompts(m, pats):
    return [[m.token_for("gauss", b), m.token_for(p, b)] for b, p in enumerate(pats)]


def run_decode_steps(ck: Checker, B: int, steps: int, persistent: bool, tag: str):
    lm = ck.lm
    for step in range(steps):
        before = ck.snapshot()
        if before["done"][:B].all():
            break
        n0 = lm.L.nt_launch_count()
        logits = lm.decode(1, ck.sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        launches = lm.L.nt_launch_count() - n0
        assert (launches == 1) == persistent, (tag, launches)
        after = ck.snapshot()
        ck.check_handoff(logits, range(B), before["cur"], f"{tag} step {step}")
        ck.check_launch(logits, list(range(B)), [ck.sp.slot_base + b for b in range(B)], before, after, 1,
                        tag=f"{tag} step {step}")
        ck.check_tmax(logits, before["ngen"][:B], persistent, f"{tag} step {step}")


# (id, vocabulary, batch, NT_DECODE_IMPL, top_k, temperature, greedy, patterns, per-row limits, expected decode paths)
CASES = [
    ("persistent-b1-eos", 217472, 1, None, 64, 1.0, False, ["eos"], None, {"fast"}),
    ("radix-b3-persistent", 217472, 3, None, 50, 0.7, False, ["ties", "stairs", "partial"], None, {"direct"}),
    ("persistent-b6-hilo", 217472, 6, None, 50, 1.5, False, PATTERNS[:6], [2, 64, 64, 64, 64, 64],
     {"direct", "fast", "general"}),
    ("tile-b9-persistent-bf16", 217472, 9, None, 64, 0.7, False, PATTERNS + ["eos", "flat"], None,
     {"direct", "fast", "general"}),
    ("persistent-b12-partial-tile", 16462, 12, None, 50, 1.0, False, PATTERNS + PATTERNS[:5], None, {"direct", "general"}),
    ("persistent-b20-tc", 217472, 20, "tc", 50, 1.0, False, (PATTERNS_ALL * 3)[:20], None, {"direct", "fast", "general"}),
    ("persistent-b4-top1", 217472, 4, None, 1, 1.0, False, ["gauss", "ties", "flat", "onetile"], None, {"direct"}),
    ("persistent-b6-greedy-v4142", 4142, 6, None, 50, 1.0, True, PATTERNS[:6], None, {"general"}),
    ("chain-b2-radix", 16462, 2, "perop", 1, 1.0, False, ["gauss", "ties"], None, set()),
    ("chain-b7-tile", 217472, 7, "perop", 50, 0.7, False, PATTERNS, [64, 2, 64, 64, 64, 64, 64], set()),
    ("chain-b5-tile-partial", 16462, 5, "perop", 64, 1.5, False, ["partial", "plateau", "eos", "stairs", "flat"], None,
     set()),
    ("chain-b7-radix-v4142", 4142, 7, "perop", 64, 0.7, False, PATTERNS, None, set()),
]
STEPS = 4
MIN_NEW = 3


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sampler_vs_float64(cuda, case, monkeypatch):
    """Prefill (tile-max kernel with the EOS fix_tile) and STEPS single decode steps on the given path.  At every launch: kept ids, kept probabilities, the drawn token, the state update, the
    hand-off into the next step and (where readable) the tile maxima."""
    name, V, B, impl, top_k, T, greedy, pats, limits, want_paths = case
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=top_k, temperature=T, seed=SEED,
                     greedy=greedy, limits=limits)
    ck = Checker(m, lm, sp, greedy, limits)
    prompts = _prompts(m, pats)
    before = ck.snapshot()
    logits = lm.prefill(prompts, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    before["ngen"][:] = 0
    before["done"][:] = 0
    ck.check_handoff(logits, range(B), {b: p[-1] for b, p in enumerate(prompts)}, "prefill")
    ck.check_launch(logits, list(range(B)), list(range(B)), before, after, 0, tag="prefill")
    assert after["seq"][:B].tolist() == [len(p) for p in prompts]
    ck.check_tmax(logits, [0] * B, False, "prefill")
    ck.paths.clear()
    _set_impl(monkeypatch, impl)
    persistent = impl == "tc" or (impl is None and B <= 16)
    run_decode_steps(ck, B, STEPS, persistent, name)
    ck.report(name)
    if persistent:
        assert want_paths <= set(ck.paths), (want_paths, ck.paths)
    done = lm.done[:B].cpu()
    if limits is not None:                                    # the capped row stopped, the rest decoded on
        capped = [b for b, c in enumerate(limits) if c < STEPS]
        assert all(int(done[b]) for b in capped) and int(lm.n_generated[capped[0]]) == limits[capped[0]]
        assert int(lm.n_generated[:B].max()) == STEPS + 1
    eos_rows = [b for b, p in enumerate(pats) if p == "eos"]
    if eos_rows:   # EOS, the largest logit, ends a row at the first unmasked step (p(EOS) > 0.9 at every temperature)
        outs, ngen = lm.out_tokens[:B].cpu(), lm.n_generated[:B].cpu()
        stopped = [b for b in eos_rows if int(done[b]) and int(outs[b, int(ngen[b]) - 1]) == m.eos]
        assert stopped and all(int(ngen[b]) == MIN_NEW + 1 for b in stopped), (eos_rows, stopped)


SLOT_CASES = [   # (id, max_batch, first prefill batch, refilled slots, stream ids): GEMV (B = 2) / GEMM (B = 6) lm_head
    ("radix-b2-into-9", 9, 9, [7, 2], [100, 3]),
    ("tile-b6-into-12", 12, 12, [11, 0, 5, 3, 8, 1], [40, 41, 7, 43, 44, 45]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SLOT_CASES, ids=[c[0] for c in SLOT_CASES])
def test_prefill_slots_sampler_vs_float64(cuda, case, monkeypatch):
    """prefill_slots samples logits row i into slot slots[i] with that slot's Philox key; every other slot keeps its
    state.  Then two decode steps on the persistent kernel: refilled slots draw from their own keys."""
    name, MB, B0, slots, keys = case
    V = 217472
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=MB, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    ck = Checker(m, lm, sp, False)
    _set_impl(monkeypatch, None)
    lm.prefill(_prompts(m, (PATTERNS * 2)[:B0]), sp)
    lm.decode(2, sp)
    torch.cuda.synchronize()
    before = ck.snapshot()
    pats = ["eos", "flat", "ties", "plateau", "partial", "gauss"][: len(slots)]
    prompts = [[m.token_for(p, 5), m.token_for(p, 9)] for p in pats]
    logits = lm.prefill_slots(slots, prompts, sp, keys, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    after = ck.snapshot()
    for s in slots:
        before["ngen"][s], before["done"][s] = 0, 0
    touched = ck.check_launch(logits, slots, keys, before, after, 0, tag="prefill_slots")
    assert [int(after["seq"][s]) for s in slots] == [len(p) for p in prompts]
    for s in set(range(MB)) - touched:                      # every other slot is untouched
        for f in ("ngen", "done", "seq", "cur"):
            assert after[f][s] == before[f][s], (s, f)
        assert (after["out"][s] == before["out"][s]).all(), s
    ck.check_tmax(logits, [0] * len(slots), False, "prefill_slots")
    key_of = {s: k for s, k in zip(slots, keys)}
    for step in range(2):
        before = ck.snapshot()
        lg = lm.decode(1, sp, return_logits=True)[0].cpu().numpy()
        torch.cuda.synchronize()
        after = ck.snapshot()
        ck.check_handoff(lg, range(MB), before["cur"], f"after slots, step {step}")
        ck.check_launch(lg, list(range(MB)), [key_of.get(s, s) for s in range(MB)], before, after, 1,
                        tag=f"after slots, step {step}")
    ck.report(name)


@pytest.mark.gpu
@pytest.mark.parametrize("impl,B", [(None, 6), ("perop", 7)], ids=["persistent-b6", "chain-b7"])
def test_multistep_launch_tokens_vs_float64(cuda, impl, B, monkeypatch):
    """decode(n) in one call: every step's drawn token against the reference on that step's returned logits (the
    window is the last step's only), including the persistent kernel's in-kernel step transitions.  The chain then
    reruns the same generation without logits, on its CUDA-graph path: identical tokens."""
    V, n = 217472, 6
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED,
                     limits=[3] + [64] * (B - 1))
    ck = Checker(m, lm, sp, False, [3] + [64] * (B - 1))
    _set_impl(monkeypatch, impl)
    prompts = _prompts(m, PATTERNS[:B])
    lm.prefill(prompts, sp)
    torch.cuda.synchronize()
    st = ck.snapshot()
    n0 = lm.L.nt_launch_count()
    logits = lm.decode(n, sp, return_logits=True).cpu().numpy()
    torch.cuda.synchronize()
    launches = lm.L.nt_launch_count() - n0
    assert (launches == 1) == (impl is None), launches
    fin = ck.snapshot()
    ngen, done, cur = st["ngen"].copy(), st["done"].copy(), st["cur"].copy()
    for s in range(n):
        if done[:B].all():
            break
        ck.check_handoff(logits[s], [b for b in range(B)], cur, f"step {s}")
        for b in range(B):
            if done[b]:
                continue
            _, tok, ok = ck.expect_token(logits[s, b], int(ngen[b]), b)
            got = int(fin["out"][b, ngen[b]])
            assert got in ok, (s, b, got, tok, ok)
            ngen[b] += 1
            cur[b] = got
            done[b] = got == m.eos or ngen[b] >= ck.lim(b)
    assert fin["ngen"][:B].tolist() == ngen[:B].tolist() and fin["done"][:B].tolist() == done[:B].astype(int).tolist()
    ck.report(f"multistep-{impl or 'persistent'}")
    if impl == "perop":
        toks = fin["out"][:B].copy()
        lm.prefill(prompts, sp)
        lm.decode(n, sp)
        torch.cuda.synchronize()
        assert np.array_equal(lm.out_tokens[:B].cpu().numpy(), toks)
        assert lm.n_generated[:B].cpu().tolist() == fin["ngen"][:B].tolist()


@pytest.mark.gpu
def test_capture_off_and_graph_rebuilt(cuda, monkeypatch):
    """Switching the capture off stops the writes, and a decode graph captured while it was on is not replayed."""
    V, B = 16462, 7
    m = programmable(V)
    cfg, w = m.oracle()
    lm = make_lm(cfg, w, max_batch=B, max_ctx=256, max_new=64)
    sp = lm.sampling(m.eos, min_new_tokens=MIN_NEW, max_new_tokens=64, top_k=50, temperature=1.0, seed=SEED)
    _set_impl(monkeypatch, "perop")
    tv, ti, tt = lm.debug_capture_sampler()
    lm.prefill(_prompts(m, PATTERNS), sp)
    lm.decode(3, sp)                               # graph captured with the capture on
    torch.cuda.synchronize()
    assert (tt[:B] >= 0).all()
    lm.debug_capture_sampler(False)
    tt.fill_(-7)
    ti.fill_(-7)
    lm.decode(3, sp)
    torch.cuda.synchronize()
    assert (tt == -7).all() and (ti == -7).all()
