"""GPU: continuous batching -- prefill into chosen slots while the others keep decoding, and the queue built on it.

Refill parity holds newcomers (and the survivors of a batch of 4) to the bar of test_lm_ragged_batch_prefill_and_decode
against the mirrored oracle, and the survivors of larger batches to test_lm_batched_decode's; refilling must not
disturb the survivors by a single bit; the queue must reproduce the chunked schedule's
tokens exactly when the two schedules coincide.
"""
import warnings

import numpy as np
import pytest
import torch

from oracle import codec_oracle as CO
from oracle import lm_oracle as O
from tests.fakes import FakePhonemizer, SmallTok
from tests.helpers import SMALL, _bar, _setup, make_codec, make_lm, max_err, rel_err, set_decode_impl

pytestmark = pytest.mark.gpu

N1, N2 = 6, 8   # decode steps before / after the refill


def _refill_run(cfg, lm, prompts, forced, slots, new_prompts, new_forced):
    """Prefill every slot, decode N1 steps, refill `slots` with `new_prompts`, decode N2 steps (all teacher-forced).
    Returns per-slot logits: the survivors' [1 + N1 + N2, V] and the newcomers' [1 + N2, V]."""
    eos = cfg.vocab_size - 1
    sp = lm.sampling(eos, min_new_tokens=0, max_new_tokens=1 + N1 + N2, forced=forced)
    l0 = lm.prefill(prompts, sp, return_logits=True)
    l1 = lm.decode(N1, sp, return_logits=True)
    for s, f in zip(slots, new_forced):
        lm.forced[s].zero_()
        lm.forced[s, : len(f)] = f.to(lm.device, torch.int32)
    ln = lm.prefill_slots(slots, new_prompts, sp, stream_ids=[1000 + s for s in slots], return_logits=True)
    l2 = lm.decode(N2, sp, return_logits=True)
    torch.cuda.synchronize()
    B = len(prompts)
    surv = {b: torch.cat((l0[b: b + 1], l1[:, b], l2[:, b])).cpu() for b in range(B) if b not in slots}
    new = {s: torch.cat((ln[i: i + 1], l2[:, s])).cpu() for i, s in enumerate(slots)}
    return surv, new


def _case(max_batch, seed):
    g = torch.Generator().manual_seed(seed)
    lens = [20, 41, 64, 65, 9, 30, 17, 80, 33, 5, 12, 70, 3, 44, 27, 90, 61, 8][:max_batch]   # test_lm_batched_decode's
    prompts = [torch.randint(0, SMALL["vocab_size"], (n,), generator=g) for n in lens]
    forced = torch.randint(0, SMALL["vocab_size"] - 1, (max_batch, 1 + N1 + N2), generator=g)   # never EOS
    slots = [max_batch - 1, 1]          # call order differs from slot order; newcomer 0 spans two KV pages
    new_lens = [90, 17]
    return prompts, forced, slots, new_lens


def _newcomers(new_lens, seed):
    g = torch.Generator().manual_seed(seed)
    p = [torch.randint(0, SMALL["vocab_size"], (n,), generator=g) for n in new_lens]
    f = torch.randint(0, SMALL["vocab_size"] - 1, (len(new_lens), 1 + N2), generator=g)
    return p, f


@pytest.mark.parametrize("impl", ["tc", "perop"], ids=["persistent-kernel", "per-op-chain"])
@pytest.mark.parametrize("max_batch", [4, 10, 18])
def test_refill_parity(cuda, max_batch, impl, monkeypatch):
    """Survivors decode across a refill of two other slots; newcomers (one longer than a 64-token page) start from
    their own prompts on a shuffled page pool.  Every sequence meets the oracle bar of its batch; the slot state
    (recorded tokens, counters, lengths) is each slot's own."""
    set_decode_impl(monkeypatch, impl)
    cfg, w, lm = _setup(max_batch, page_shuffle_seed=7)
    prompts, forced, slots, new_lens = _case(max_batch, 3)
    new_prompts, new_forced = _newcomers(new_lens, 4)
    surv, new = _refill_run(cfg, lm, [p.tolist() for p in prompts], forced, slots, [p.tolist() for p in new_prompts], new_forced)
    eos = cfg.vocab_size - 1
    for b, got in surv.items():
        if max_batch <= 4:
            _, mir = O.generate(cfg, w, prompts[b], eos, max_length=256, max_new_tokens=1 + N1 + N2, forced=forced[b], mirror=True)
            _bar(got, mir, f"survivor {b}")
        else:
            # a survivor's logits are bit-identical to those of a batch that saw no refill (next test), so they are held
            # to the bar test_lm_batched_decode sets for that batched prefill + decode: against the pure reference
            _, ref = O.generate(cfg, w, prompts[b], eos, max_length=256, max_new_tokens=1 + N1 + N2, forced=forced[b], mirror=False)
            assert rel_err(got, ref) < 2e-2 and max_err(got, ref) < 1e-1 * float(ref.std()), (b, rel_err(got, ref))
    for i, s in enumerate(slots):
        _, mir = O.generate(cfg, w, new_prompts[i], eos, max_length=256, max_new_tokens=1 + N2, forced=new_forced[i], mirror=True)
        _bar(new[s], mir, f"newcomer in slot {s}")
    out, ngen, lens = lm.out_tokens.cpu(), lm.n_generated.cpu(), lm.seq_lens.cpu()
    for b in range(max_batch):
        if b in slots:
            i = slots.index(b)
            n, f, P = 1 + N2, new_forced[i], len(new_prompts[i])
        else:
            n, f, P = 1 + N1 + N2, forced[b], len(prompts[b])
        assert out[b, :n].tolist() == f.tolist(), b
        assert int(ngen[b]) == n and int(lens[b]) == P + n - 1, (b, int(ngen[b]), int(lens[b]))
    # survivors reached the cap of 1 + N1 + N2 tokens; the newcomers, N1 tokens short of it, are still live
    assert lm.done[:max_batch].cpu().tolist() == [int(b not in slots) for b in range(max_batch)]


@pytest.mark.parametrize("impl", ["tc", "perop"], ids=["persistent-kernel", "per-op-chain"])
@pytest.mark.parametrize("max_batch", [4, 10, 18])
def test_refill_leaves_survivors_bit_identical(cuda, max_batch, impl, monkeypatch):
    """Different newcomers (same lengths) in the refilled slots change nothing in any other slot, bit for bit; nor does
    the refill itself: the survivors' logits equal those of a run in which no slot was refilled."""
    set_decode_impl(monkeypatch, impl)
    cfg, w, lm = _setup(max_batch, page_shuffle_seed=7)
    prompts, forced, slots, new_lens = _case(max_batch, 3)
    sp = lm.sampling(cfg.vocab_size - 1, min_new_tokens=0, max_new_tokens=1 + N1 + N2, forced=forced)
    l0 = lm.prefill([p.tolist() for p in prompts], sp, return_logits=True)
    ls = lm.decode(N1 + N2, sp, return_logits=True)
    plain = {b: torch.cat((l0[b: b + 1], ls[:, b])).cpu() for b in range(max_batch) if b not in slots}
    runs = []
    for seed in (4, 5):
        new_prompts, new_forced = _newcomers(new_lens, seed)
        runs.append(_refill_run(cfg, lm, [p.tolist() for p in prompts], forced, slots, [p.tolist() for p in new_prompts], new_forced))
    (s1, n1), (s2, n2) = runs
    assert s1.keys() == s2.keys()
    for b in s1:
        assert torch.equal(s1[b], s2[b]), b
        assert torch.equal(s1[b], plain[b]), b
    assert not torch.equal(n1[slots[0]], n2[slots[0]])   # the newcomers did differ


@pytest.mark.parametrize("max_batch", [4, 18])
def test_queue_matches_chunked_schedule(cuda, max_batch):
    """Equal caps (EOS masked) make the two schedules coincide: every slot ends together and the queue refills all of
    them with the next max_batch prompts in slot order.  Each prompt keeps its Philox stream, so the sampled tokens
    are exactly those of generate_batch per chunk with slot_base = the chunk's first index."""
    cfg, w, lm = _setup(max_batch)
    g = torch.Generator().manual_seed(8)
    n, cap, eos = 3 * max_batch, 40, 5
    prompts = [torch.randint(0, cfg.vocab_size, (int(m),), generator=g).tolist() for m in torch.randint(3, 90, (n,), generator=g)]
    kw = dict(max_length=256, min_new_tokens=cap, max_new_tokens=cap, temperature=1.0, top_k=50, seed=1234)
    chunked = []
    for j in range(0, n, max_batch):
        chunked += lm.generate_batch(prompts[j: j + max_batch], eos, slot_base=j, **kw)
    queued = lm.generate_queue(prompts, eos, **kw)
    assert [len(o) for o in queued] == [cap] * n
    assert [o.tolist() for o in queued] == [o.tolist() for o in chunked]
    assert sorted(lm.pool.free) == list(range(lm.num_pages))


def test_queue_end_to_end(cuda):
    """Ragged caps with EOS masked: every utterance stops exactly at its cap, a second run is bit-identical, and a
    greedy run of a refilled utterance follows the oracle's (near-)argmax along its own path."""
    cfg, w, lm = _setup(4, max_ctx=256)
    g = torch.Generator().manual_seed(12)
    eos, max_length = 5, 128
    lens = [30, 118, 60, 100, 45, 121, 80, 110, 20, 95]
    prompts = [torch.randint(0, cfg.vocab_size, (m,), generator=g).tolist() for m in lens]
    caps = [max_length - m for m in lens]
    kw = dict(max_length=max_length, min_new_tokens=max_length, seed=77, check_every=16)
    a = lm.generate_queue(prompts, eos, **kw)
    assert [len(o) for o in a] == caps
    b = lm.generate_queue(prompts, eos, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert sorted(lm.pool.free) == list(range(lm.num_pages))
    greedy = lm.generate_queue(prompts, eos, max_length=max_length, min_new_tokens=max_length, greedy=True, check_every=16)
    i = 7                      # admitted after the first wave of four finished
    assert len(greedy[i]) == caps[i]
    cache = O.KVCache(cfg.num_layers)
    logits, _ = O.forward(cfg, w, torch.tensor(prompts[i]), cache, mirror="prefill")
    for t in greedy[i].tolist():
        row = logits[-1]
        assert float(row.max() - row[t]) < 5e-2 * float(row.std()), (t, int(row.argmax()))
        logits, _ = O.forward(cfg, w, torch.tensor([t]), cache, mirror="decode")


def test_facade_infer_batch_queues_long_lists(cuda):
    """Seven utterances at max_batch 3 run as one queue: seven waveforms of hop x codes samples, reproducible."""
    from neutts import NeuTTS

    cfg = O.LMConfig.tiny(vocab_size=4096, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=4, num_kv_heads=2)
    w = O.random_weights(cfg, 3, std=0.05, bf16_round=True)
    lm = make_lm(cfg, w, max_batch=3, max_ctx=2048, max_new=512)
    ccfg = CO.CodecConfig.tiny()
    dec = make_codec(ccfg, CO.random_weights(ccfg, 2), max_batch=3, max_frames=512)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = NeuTTS(tokenizer=SmallTok(), phonemizer=FakePhonemizer(), backbone=lm, codec=dec, max_batch=3, seed=7)
    tts.max_context = 2048
    texts = ["alpha", "beta gamma", "delta", "epsilon zeta eta", "theta", "iota kappa", "lambda"]
    refs = [torch.arange(10 + 5 * i) for i in range(7)]
    rts = ["one", "two words", "three", "four", "five", "six", "seven"]
    calls = []
    orig = lm.generate_queue
    lm.generate_queue = lambda *a, **k: calls.append(len(a[0])) or orig(*a, **k)
    wavs = tts.infer_batch(texts, refs, rts)
    assert calls == [7]
    assert len(wavs) == 7 and all(isinstance(x, np.ndarray) and np.isfinite(x).all() for x in wavs)
    prompts = [tts._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, refs, rts)]
    gen = tts._generate_ids(prompts)
    for x, ids in zip(wavs, gen):
        assert len(x) == ccfg.hop * len(tts._ids_to_codes(ids)) > 0
    again = tts.infer_batch(texts, refs, rts)
    assert all(np.array_equal(x, y) for x, y in zip(wavs, again))
