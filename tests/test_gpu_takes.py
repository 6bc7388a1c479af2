"""GPU: several takes per prompt from one prefill (SpeechLM.prefill_fork, generate_batch(num_return_sequences=n),
NeuTTS.infer_batch(takes=n)).

The takes of a prompt share its full KV pages; each has a private copy of the partly filled last prompt page and pages
of its own for generated tokens.  Checked here: the fork's prefill logits are those of one take (a plain prefill), bit
for bit, and the C entry nt_lm_prefill is that one take; the page-table rows and the copied tail rows; decoding over
shared pages gives exactly the logits of private copies and never writes a shared page; the first draw of every take is the float64 reference draw on its prompt's logits with its
own Philox stream; a refill of one take leaves its siblings alone; the public outputs keep transformers' layout.
Prompt lengths cross page boundaries and include a multiple of 64; B * n covers the GEMV decode (<= 4), the persistent
kernel (<= 16) and the per-op chain (> 16).
"""
import ctypes as C
import math
import warnings

import numpy as np
import pytest
import torch

from neutts_air_b200 import _lib
from neutts_air_b200.lm import fork_slots
from oracle import lm_oracle as O
from tests.helpers import _bar, _setup, _tts, gather_kv, set_decode_impl
from tests.sampler_ref import draw_u, ref_token, ref_window_cut

pytestmark = pytest.mark.gpu

LENS = [70, 64, 5, 130]
CASES = [(2, 2), (3, 4), (3, 6)]          # B * n = 4 (GEMV), 12 (persistent kernel), 18 (chain)
STEPS = 6


def _prompts(B, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 4096, (m,), generator=g).tolist() for m in LENS[:B]]


def _forced(B, n, seed=5):
    """One row per take; every take of the last prompt gets the same row (their logits must then agree)."""
    g = torch.Generator().manual_seed(seed)
    f = torch.randint(0, 4095, (B * n, 1 + STEPS), generator=g)   # never EOS (4095)
    f[(B - 1) * n:] = f[(B - 1) * n]
    return f


def _privatise(lm, B, n, lens):
    """Give every take of every prompt its own copy of each shared full prompt page (the control layout)."""
    table = lm._table_host.copy()
    for i, P in enumerate(lens):
        for j in range(1, n):
            s = i * n + j
            for k in range(P // 64):
                old = int(table[s, k])
                new = lm.pool.alloc(1)[0]
                lm.kv[:, :, new] = lm.kv[:, :, old]
                lm.pool.release([old])
                lm._slot_pages[s][k] = new
                table[s, k] = new
    lm.page_table.copy_(torch.from_numpy(table))
    lm._table_host = table


@pytest.mark.parametrize("impl", ["tc", "perop"], ids=["persistent-kernel", "per-op-chain"])
@pytest.mark.parametrize("B,n", CASES, ids=[f"{b}x{n}" for b, n in CASES])
def test_fork_prefill_kv_and_decode(cuda, B, n, impl, monkeypatch):
    set_decode_impl(monkeypatch, impl)
    N = B * n
    cfg, w, lm = _setup(N, page_shuffle_seed=7)
    _, _, plain = _setup(N, page_shuffle_seed=7)
    _, _, ctl = _setup(N, page_shuffle_seed=7)
    eos = cfg.vocab_size - 1
    prompts, forced = _prompts(B), _forced(B, n)
    lens = [len(p) for p in prompts]
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=1 + STEPS, forced=forced)
    lf = lm.prefill_fork(prompts, n, sp, return_logits=True)
    # 1. the prefill logits are those of a plain prefill (one take) of the same prompts, bit for bit
    lp = plain.prefill(prompts, plain.sampling(eos, min_new_tokens=0, max_new_tokens=1 + STEPS), return_logits=True)
    assert torch.equal(lf, lp)
    # 2. page-table rows: shared full pages, private tail page with the parent's rows, private pages after it
    torch.cuda.synchronize()
    table = lm.page_table.cpu()
    for i, P in enumerate(lens):
        full, parent = P // 64, i * n
        for j in range(1, n):
            s = i * n + j
            assert torch.equal(table[s, :full], table[parent, :full]), (i, j)
            others = {p for r in range(N) if r != s for p in lm._slot_pages[r]}
            tail = int(table[s, full])
            assert tail not in others and lm.pool.refs[tail] == 1, (i, j)
            if P % 64:
                for layer in range(cfg.num_layers):
                    kp, vp = gather_kv(lm, layer, parent, P)
                    kc, vc = gather_kv(lm, layer, s, P)
                    assert torch.equal(kp, kc) and torch.equal(vp, vc), (i, j, layer)
    shared = sorted({int(p) for i, P in enumerate(lens) for p in table[i * n, : P // 64]})
    before = lm.kv[:, :, shared].clone()
    # 3. decoding over shared pages: the logits of private copies, bit for bit; no shared page changes
    ld = lm.decode(STEPS, sp, return_logits=True)
    sc = ctl.sampling(eos, min_new_tokens=0, max_new_tokens=1 + STEPS, forced=forced)
    ctl.prefill_fork(prompts, n, sc)
    _privatise(ctl, B, n, lens)
    lc = ctl.decode(STEPS, sc, return_logits=True)
    assert torch.equal(ld, lc)
    assert torch.equal(lm.kv[:, :, shared], before)
    torch.cuda.synchronize()
    got = {s: torch.cat((lf[s // n: s // n + 1], ld[:, s])).cpu() for s in range(N)}
    last = range((B - 1) * n, N)
    for s in last:
        assert torch.equal(got[s], got[last[0]]), s
    for i, j, s, _ in fork_slots(B, n):
        if s in last and s != last[0]:
            continue
        _, mir = O.generate(cfg, w, torch.tensor(prompts[i]), eos, max_length=256, max_new_tokens=1 + STEPS, forced=forced[s],
                            mirror=True)
        _bar(got[s], mir, f"take {j} of prompt {i} (slot {s})")
    out, ngen, seq = lm.out_tokens.cpu(), lm.n_generated.cpu(), lm.seq_lens.cpu()
    for i, j, s, _ in fork_slots(B, n):
        assert out[s, : 1 + STEPS].tolist() == forced[s].tolist()
        assert int(ngen[s]) == 1 + STEPS and int(seq[s]) == lens[i] + STEPS


def test_c_prefill_is_one_take(cuda):
    """The C entry nt_lm_prefill is nt_lm_prefill_fork with one take: on the pages SpeechLM.prefill laid out, it gives
    the same logits, first tokens and slot state, resets every slot's counters itself, and refuses a batch outside
    1..max_batch with its own message."""
    B = 3
    cfg, w, lm = _setup(B + 1, page_shuffle_seed=7)
    prompts = _prompts(B)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=1 + STEPS, seed=4)
    want = lm.prefill(prompts, sp, return_logits=True)
    state = lambda: [t.clone() for t in (lm.out_tokens, lm.cur_token, lm.seq_lens, lm.n_generated, lm.done)]
    before = state()
    ids = torch.tensor([t for p in prompts for t in p], dtype=torch.int32, device=lm.device)
    cu = np.cumsum([0] + [len(p) for p in prompts]).astype(np.int32)
    got = torch.empty_like(want)
    call = lambda b: lm.L.nt_lm_prefill(lm.handle, C.byref(lm.state), ids.data_ptr(), cu.ctypes.data_as(C.POINTER(C.c_int32)),
                                        b, C.byref(sp), got.data_ptr(), _lib.current_stream_ptr())
    lm.n_generated.fill_(7)
    lm.done.fill_(1)
    _lib.check(call(B))
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert all(torch.equal(a, b) for a, b in zip(state(), before))
    for b in (0, B + 2):
        with pytest.raises(ValueError, match=rf"batch {b} not in 1\.\.{B + 1}"):
            _lib.check(call(b))


PALETTE = [(0.8, 40, 0.9, 0.0), (1.3, 64, 1.0, 0.02), (1.0, 20, 0.7, 0.05)]


@pytest.mark.parametrize("B,n", CASES, ids=[f"{b}x{n}" for b, n in CASES])
def test_first_draws(cuda, B, n):
    """4. Each take's first token is the float64 draw on its prompt's (penalised) logits row with stream key
    i * n + j + slot_base, under per-prompt top-p / min-p and repetition penalty; each take gets its own log-prob row."""
    N, slot_base, seed, min_new = B * n, 11, 1234, 50
    cfg, w, lm = _setup(N)
    eos = cfg.vocab_size - 1
    prompts = _prompts(B, seed=9)
    ctl = [PALETTE[i % len(PALETTE)] for i in range(B)]
    lm.set_slot_sampling([c for c in ctl for _ in range(n)])
    lm.set_repetition_penalty([(1.3 + 0.2 * i, True) for i in range(B) for _ in range(n)])
    lm.set_logprobs(True)
    cap = lm.debug_capture_sampler()
    sp = lm.sampling(eos, min_new_tokens=min_new, max_new_tokens=8, seed=seed, slot_base=slot_base)
    logits = lm.prefill_fork(prompts, n, sp, return_logits=True)
    torch.cuda.synchronize()
    lg, tok, lp = logits.cpu().numpy(), cap[2].cpu().numpy(), lm.logprobs[:, 0].cpu().numpy()
    checked = 0
    for i, j, s, key in fork_slots(B, n, slot_base):
        T, k, p, mp = ctl[i]
        ids, q, margin = ref_window_cut(lg[i], 0, eos, min_new, T, k, p, mp)
        _, ok = ref_token((ids, q), draw_u(seed, 0, key))
        if margin > 1e-6:
            assert int(tok[s]) in ok, (i, j, int(tok[s]), ok)
            checked += 1
        assert int(lm.out_tokens[s, 0]) == int(tok[s]) and int(lm.n_generated[s]) == 1
        row = lg[i].astype(np.float64)
        row[eos] = -np.inf
        m = row.max()
        model = row[int(tok[s])] - (m + math.log(np.exp(row - m).sum()))
        assert abs(float(lp[s, 1]) - model) < 1e-4 * max(1.0, abs(model)), (s, float(lp[s, 1]), model)
    assert checked >= N // 2
    # different streams: the takes of one prompt do not all draw the same token
    assert any(len({int(tok[i * n + j]) for j in range(n)}) > 1 for i in range(B))


@pytest.mark.parametrize("impl", ["tc", "perop"], ids=["persistent-kernel", "per-op-chain"])
def test_refill_one_take(cuda, impl, monkeypatch):
    """5. prefill_slots into one take's slot returns only that take's private pages and leaves its siblings' logits
    bit-identical; after generate_batch(num_return_sequences=n) every page goes back to the pool."""
    set_decode_impl(monkeypatch, impl)
    B, n = 2, 3
    N = B * n
    cfg, w, lm = _setup(N, page_shuffle_seed=7)
    eos = cfg.vocab_size - 1
    prompts, forced = _prompts(B), _forced(B, n)
    runs = []
    for refill in (False, True):
        sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=1 + 2 * STEPS, forced=forced)
        lm.prefill_fork(prompts, n, sp)
        l1 = lm.decode(STEPS, sp, return_logits=True)
        if refill:
            child = 1
            own = lm._slot_pages[child][len(prompts[0]) // 64:]
            free = lm.pool.num_free
            lm.prefill_slots([child], [prompts[1][:40]], sp, stream_ids=[99])
            assert lm.pool.num_free == free + len(own) - len(lm._slot_pages[child])
        l2 = lm.decode(STEPS, sp, return_logits=True)
        torch.cuda.synchronize()
        runs.append(torch.cat((l1, l2)).cpu())
    for s in range(N):
        if s != 1:
            assert torch.equal(runs[0][:, s], runs[1][:, s]), s
    ids = lm.generate_batch(prompts, eos, max_length=256, min_new_tokens=0, max_new_tokens=20, seed=3, num_return_sequences=n)
    assert len(ids) == N
    lm.release_pages()
    assert lm.pool.num_free == lm.num_pages and sorted(lm.pool.free) == list(range(lm.num_pages))


def test_public_outputs(cuda):
    """6. generate(num_return_sequences=n): [B * n, P + gen], row b * n + j = prompt b, then the ids of take j of
    generate_batch(num_return_sequences=n) under the same seed."""
    B, n = 2, 2
    cfg, w, lm = _setup(B * n)
    eos = cfg.vocab_size - 1
    g = torch.Generator().manual_seed(2)
    x = torch.randint(0, 4095, (B, 67), generator=g)
    out = lm.generate(x.cuda(), max_length=120, eos_token_id=eos, min_new_tokens=10, num_return_sequences=n, seed=5)
    ids = lm.generate_batch(x.tolist(), eos, max_length=120, min_new_tokens=10, seed=5, num_return_sequences=n)
    assert out.shape == (B * n, 67 + max(len(o) for o in ids))
    assert torch.equal(out[:, :67].cpu(), x.repeat_interleave(n, dim=0))
    for r, o in enumerate(ids):
        assert out[r, 67: 67 + len(o)].cpu().tolist() == o.tolist()


def test_facade_keeps_the_most_probable_take(cuda):
    from neutts.neutts import best_takes

    takes = 2
    tts, _ = _tts(max_batch=4)
    texts, refs, rts = ["alpha", "beta gamma", "delta"], [torch.arange(10 + 5 * i) for i in range(3)], ["one", "two", "three"]
    wavs, lps = tts.infer_batch(texts, refs, rts, takes=takes, return_logprobs=True)
    assert len(wavs) == 3 and len(lps) == 3
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    eos = tts._tok_id("<|SPEECH_GENERATION_END|>")
    kept = []
    for idx, base in tts.take_chunks(3, takes, 4):       # 2 utterances per chunk, slot_base = first x takes
        ids, lp = tts.backbone.generate_batch([prompts[i] for i in idx], eos, max_length=tts.max_context, min_new_tokens=50,
                                              seed=tts.seed, slot_base=base, temperature=1.0, top_k=50,
                                              num_return_sequences=takes, return_logprobs=True)
        means = [float(r[:, 1].double().mean()) for r in lp]
        keep = best_takes(lp, takes)
        for u, k in enumerate(keep):
            assert means[k] == max(means[u * takes: (u + 1) * takes])
        kept += [(ids[k], lp[k]) for k in keep]
    for wv, lpk, (ids, lpr) in zip(wavs, lps, kept):
        assert np.array_equal(lpk, lpr.numpy())
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = tts._watermark(tts._decode_codes([tts._ids_to_codes(ids)])[0])
        assert np.array_equal(wv, ref)
