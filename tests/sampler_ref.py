"""The float64 references the speech-LM sampler tests compare the kernels with, and the model they run them on.

* The reference sampler: the Philox draw of every launch, the logits processors, the kept top-k window and the
  inverse CDF over it, the tile maxima and the ``sample_tiles_seq`` path a score row takes; the per-slot chain (top-p,
  min-p) and the vocabulary-range suppression on top of it; the teacher-forced score.
* The logit-programmable one-layer model (``programmable``: one instance per vocabulary size in a process), whose
  token logits are chosen patterns (test_gpu_sampler.py describes it), and the drivers that check kernel launches on
  it: ``Checker``, and ``drive`` with ``check_launch`` for per-slot controls.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import lm_oracle as O
from tests.helpers import rel_rms, set_decode_impl

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


def _prompts(m, pats):
    return [[m.token_for("gauss", b), m.token_for(p, b)] for b, p in enumerate(pats)]


MIN_NEW = 3


# ====================================================================================== float64 reference chain
def chain64(scores, top_k: int, top_p: float, min_p: float):
    """Processed scores [V] -> kept window of the kernels: (score desc, id asc), the first min(top_k, 64); its float64
    softmax q; top-p keeps entry j iff sum_{i<j} q_i < top_p (off at 1), min-p iff q_j >= min_p * q_0 (off at 0); the
    kept prefix renormalised.  Returns (ids int64 [k'], probabilities float64 [k'], margin): margin is the distance of
    the cut quantities (exclusive cumulative mass, q_j / q_0) to their thresholds over the window (inf: no cut)."""
    s = np.asarray(scores, dtype=np.float64)
    k = min(top_k, 64, s.size)
    order = np.lexsort((np.arange(s.size), -s))[:k]
    p = np.exp(s[order] - s[order[0]])
    q = p / p.sum()
    keep = np.ones(k, dtype=bool)
    margin = np.inf
    if top_p < 1:
        excl = np.concatenate(([0.0], np.cumsum(q)[:-1]))
        keep &= excl < top_p
        margin = min(margin, float(np.abs(excl - top_p).min()))
    if min_p > 0:
        ratio = q / q[0]
        keep &= ratio >= min_p
        margin = min(margin, float(np.abs(ratio - min_p).min()))
    kp = int(np.argmin(keep)) if not keep.all() else k
    kp = max(kp, 1)
    return order[:kp].astype(np.int64), q[:kp] / q[:kp].sum(), margin


def ref_window_cut(logits, ngen: int, eos: int, min_new: int, temperature: float, top_k: int, top_p: float, min_p: float):
    """The kernels' chain on logits: EOS mask and fp32(logit) * fp32(1 / T) (``processed_scores``), then ``chain64``."""
    return chain64(processed_scores(logits, ngen, eos, min_new, temperature), top_k, top_p, min_p)


def suppressed_scores(logits, lo: int, hi: int, eos: int, ngen: int, min_new: int, temperature: float):
    s = np.asarray(logits, dtype=np.float32).copy()
    keep = np.zeros(s.size, dtype=bool)
    keep[lo:hi] = True
    keep[eos] = True
    s[~keep] = -np.inf
    return processed_scores(s, ngen, eos, min_new, temperature)


# ====================================================================================== float64 teacher-forced score
def forward64(cfg: O.LMConfig, w: O.LMWeights, ids) -> torch.Tensor:
    """Qwen2 logits [T, V] in float64, causal attention; the rotary angles and the RMSNorm statistics in fp32, as
    transformers forms them in a float64 model."""
    d = lambda t: t.double()
    ids = torch.as_tensor(ids, dtype=torch.long)
    T = ids.shape[0]
    cos, sin = O.rope_cos_sin(torch.arange(T), cfg.head_dim, cfg.rope_theta)
    cos, sin = cos.double(), sin.double()

    def norm(x, wt):
        return O.rms_norm(x, d(wt), cfg.rms_eps)

    n_rep = cfg.num_heads // cfg.num_kv_heads
    mask = torch.triu(torch.ones(T, T, dtype=torch.bool), 1)
    h = d(w.embed)[ids]
    for L in w.layers:
        x = norm(h, L["ln1"])
        q = (x @ d(L["wq"]).T + d(L["bq"])).view(T, cfg.num_heads, cfg.head_dim)
        k = (x @ d(L["wk"]).T + d(L["bk"])).view(T, cfg.num_kv_heads, cfg.head_dim)
        v = (x @ d(L["wv"]).T + d(L["bv"])).view(T, cfg.num_kv_heads, cfg.head_dim)
        q, k = O.apply_rope(q, cos, sin), O.apply_rope(k, cos, sin)
        k, v = k.repeat_interleave(n_rep, 1), v.repeat_interleave(n_rep, 1)
        s = torch.einsum("qhd,khd->hqk", q, k) * cfg.head_dim ** -0.5
        p = torch.softmax(s.masked_fill(mask, float("-inf")), -1)
        h = h + torch.einsum("hqk,khd->qhd", p, v).reshape(T, -1) @ d(L["wo"]).T
        x = norm(h, L["ln2"])
        h = h + (torch.nn.functional.silu(x @ d(L["wg"]).T) * (x @ d(L["wu"]).T)) @ d(L["wd"]).T
    return norm(h, w.final_norm) @ d(w.lm_head).T


def score64(cfg, w, ids, start: int) -> np.ndarray:
    """score[t] = log_softmax(z_{t-1})[x_t] for start <= t < len(ids), float64."""
    ids = torch.as_tensor(ids, dtype=torch.long)
    lp = torch.log_softmax(forward64(cfg, w, ids), -1)
    t = torch.arange(start, ids.shape[0])
    return lp[t - 1, ids[t]].numpy()


# ================================================================================== GPU driver of the per-slot controls
MARGIN = 1e-4

# (temperature, top_k, top_p, min_p): k = 1 and 64, T < 1 and > 1, top-p cutting inside the window, min-p cutting
# before top-p does, and a plain entry
PALETTE = [
    (0.7, 64, 0.5, 0.0),
    (1.5, 1, 1.0, 0.0),
    (1.0, 64, 1.0, 0.2),
    (1.3, 50, 0.9, 0.3),
    (0.5, 20, 0.3, 0.0),
    (2.0, 64, 0.95, 0.01),
    (1.0, 8, 0.6, 0.05),
    (0.8, 33, 1.0, 0.0),
]


def controls_for(B: int, shift: int = 0):
    return [PALETTE[(b + shift) % len(PALETTE)] for b in range(B)]


def _snap(lm):
    return dict(ngen=lm.n_generated.cpu().numpy().copy(), done=lm.done.cpu().numpy().copy(),
                seq=lm.seq_lens.cpu().numpy().copy(), out=lm.out_tokens.cpu().numpy().copy())


def _record(lm, cap, logits, before, rows, keys, nt, tag):
    torch.cuda.synchronize()
    R = len(rows)
    return dict(tag=tag, logits=logits.cpu().numpy(), before=before, after=_snap(lm), rows=list(rows), keys=list(keys),
                tv=cap[0][:R].cpu().numpy().copy(), ti=cap[1][:R].cpu().numpy().copy(), tt=cap[2][:R].cpu().numpy().copy(),
                tmax=lm.debug_buffer("tmax", (R, nt)).cpu().numpy().copy())


def drive(lm, sp, prompts, steps, monkeypatch, impl, nt, table=None):
    """prefill + `steps` single decode steps; per launch: logits, captured window, tile maxima, state before / after."""
    cap = lm.debug_capture_sampler()
    set_decode_impl(monkeypatch, None)
    lm.set_slot_sampling(table)
    B = len(prompts)
    lm.out_tokens.zero_()                           # every run starts from the same buffers: a launch that does not
    lm.debug_buffer("tmax", (B, nt)).zero_()        # write them leaves equal contents in both runs of a comparison
    before = _snap(lm)
    before["ngen"][:], before["done"][:] = 0, 0
    recs = [_record(lm, cap, lm.prefill(prompts, sp, return_logits=True), before, range(B), range(B), nt, "prefill")]
    set_decode_impl(monkeypatch, impl)
    for step in range(steps):
        before = _snap(lm)
        if before["done"][:B].all():
            break
        lg = lm.decode(1, sp, return_logits=True)[0]
        recs.append(_record(lm, cap, lg, before, range(B), range(B), nt, f"step {step}"))
    return recs


def check_launch(m, rec, ctl, stats, tmax_processed=None):
    """One launch against the float64 chain with the per-slot controls ctl[slot]."""
    tag = rec["tag"]
    for i, (s, key) in enumerate(zip(rec["rows"], rec["keys"])):
        T, k, p, mp = ctl[s]
        lg = rec["logits"][i]
        ngen = int(rec["before"]["ngen"][s])
        ids, q, margin = ref_window_cut(lg, ngen, m.eos, MIN_NEW, T, k, p, mp)
        assert margin >= MARGIN, (tag, i, ctl[s], margin)
        n = len(ids)
        assert rec["ti"][i, :n].tolist() == ids.tolist(), (tag, i, ctl[s], rec["ti"][i, :n].tolist(), ids.tolist())
        assert (rec["ti"][i, n:] == -1).all() and (rec["tv"][i, n:] == 0).all(), (tag, i)
        err = prob_err(rec["tv"][i, :n], q)
        stats["prob"] = max(stats["prob"], err)
        assert err < BARS["prob"], (tag, i, err)
        tok, ok = ref_token((ids, q), draw_u(SEED, ngen, key))
        stats["draws"] += 1
        stats["ambiguous"] += len(ok) > 1
        assert int(rec["tt"][i]) in ok, (tag, i, int(rec["tt"][i]), tok, ok)
        if not rec["before"]["done"][s]:
            assert int(rec["after"]["out"][s, ngen]) == int(rec["tt"][i]), (tag, s)
        stats["cut"] += n < min(k, 64)
        proc = processed_scores(lg, ngen, m.eos, MIN_NEW, T)
        stats["paths"].add(tile_path(proc, k))
        if tmax_processed is not None:
            want = tile_maxima(proc) if tmax_processed else tile_maxima(lg)
            assert np.array_equal(rec["tmax"][i], want), (tag, i, np.nonzero(rec["tmax"][i] != want)[0][:5])


# ====================================================================================== vocabulary ranges of the model
def ties_ids(m):
    """Ids of the "ties" pattern's 84 values tied at 10."""
    j = PATTERNS.index("ties")
    return np.nonzero(m.target[j] == 10.0)[0]


def _range(m, kind):
    if kind == "speech":   # the Air layout: [1187 * 128, V), EOS below it
        lo = 1187 * 128 if m.V == 217472 else (m.nt - 3) * 128
        return lo, m.V
    t = m.eos // 128
    if kind == "below-eos":   # [0, (t - 5) * 128): EOS lies above the range
        return 0, (t - 5) * 128
    if kind == "ties-lo":     # lo at the tile edge nearest the median tied id
        ids = ties_ids(m)
        lo = int(round(float(np.median(ids)) / 128)) * 128
        assert (ids < lo).sum() >= 10 and (ids >= lo).sum() >= 10, lo
        return lo, m.V
    return (t - 20) * 128, (t + 20) * 128   # 40 tiles with EOS in the middle
