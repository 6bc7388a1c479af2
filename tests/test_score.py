"""CPU: teacher-forced scoring -- the definition against transformers, the packing of sequences into calls, the facade
on stub backbones and the scratch-size query of the C ABI."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O
from tests.fakes import FakeCodec, FakePhonemizer, FakeTokenizer
from tests.sampler_ref import score64


def _tiny():
    cfg = O.LMConfig.tiny(vocab_size=300, hidden_size=128, intermediate_size=256, num_layers=2, num_heads=4, num_kv_heads=2)
    return cfg, O.random_weights(cfg, 5, std=0.08)


def test_score64_matches_transformers_cross_entropy_and_loss():
    """Per-token cross-entropy of transformers in float64 to 1e-9; its labels= loss (computed in float32) to 1e-6."""
    pytest.importorskip("transformers")
    cfg, w = _tiny()
    model = O.to_hf_model(cfg, w, attn_implementation="sdpa").double()   # eager attention takes its softmax in float32
    g = torch.Generator().manual_seed(1)
    worst = 0.0
    for L, s in ((2, 1), (9, 1), (17, 5), (17, 16), (40, 23)):
        ids = torch.randint(0, cfg.vocab_size, (L,), generator=g)
        ref = score64(cfg, w, ids, s)
        assert ref.shape == (L - s,)
        with torch.no_grad():
            logits = model(ids[None]).logits[0]
            ce = torch.nn.functional.cross_entropy(logits[s - 1: L - 1], ids[s:L], reduction="none")
            labels = ids.clone()
            labels[:s] = -100
            loss = model(ids[None], labels=labels[None]).loss
        worst = max(worst, float(np.abs(ref + ce.numpy()).max()))
        # transformers' loss upcasts the logits to float32 (ForCausalLMLoss), so it agrees to fp32 rounding only
        assert abs(-ref.mean() - float(loss)) < 1e-6 * max(1.0, float(loss))
    assert worst < 1e-9


# ====================================================================================== packing
def test_pack_score_calls_respects_limits_and_order():
    from neutts_air_b200.lm import pack_score_calls

    lens = [5, 7, 3, 10, 2, 2, 2, 9, 1 + 1]
    calls = pack_score_calls(lens, max_batch=3, max_tokens=12, max_ctx=64)
    assert [i for c in calls for i in c] == list(range(len(lens)))
    for c in calls:
        assert 1 <= len(c) <= 3 and sum(lens[i] for i in c) <= 12
    assert calls == [[0, 1], [2], [3, 4], [5, 6], [7, 8]]
    assert pack_score_calls([], 4, 100, 64) == []
    assert pack_score_calls([12], 1, 12, 64) == [[0]]
    with pytest.raises(ValueError, match="sequence 1"):
        pack_score_calls([4, 13], 4, 12, 64)
    with pytest.raises(ValueError, match="sequence 0"):
        pack_score_calls([65], 4, 1000, 64)


def test_score_starts():
    from neutts_air_b200.lm import score_starts

    assert score_starts([4, 6], 1) == [1, 1]
    assert score_starts([4, 6], [3, 5]) == [3, 5]
    assert score_starts([4], np.array([2])) == [2]
    for bad in (0, 4, 2.5, True, [1]):
        with pytest.raises(ValueError):
            score_starts([4, 6], bad)


# ====================================================================================== facade on stubs
class ScoreStub:
    """A backbone with ``score``: records what it was handed and returns -(position) for every scored token."""

    def __init__(self, tok):
        self.tok, self.calls = tok, []

    def score(self, seqs, starts):
        self.calls.append(([list(s) for s in seqs], list(starts)))
        return [torch.arange(s, len(q), dtype=torch.float32).neg() for q, s in zip(seqs, starts)]


def _facade(backbone=ScoreStub):
    from neutts import NeuTTS

    tok = FakeTokenizer()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=backbone(tok), codec=FakeCodec(), max_batch=2,
                      seed=3)


def test_facade_builds_prompt_codes_and_eos():
    tts = _facade()
    tok = tts.tokenizer
    sge = tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>")
    prompt = tts._apply_chat_template([1, 2], "ref text", "hello")
    out = tts.score("hello", [1, 2], "ref text", [7, 0, 65535])
    (seqs, starts), = tts.backbone.calls
    assert seqs == [prompt + [3007, 3000, 3000 + 65535, sge]] and starts == [len(prompt)]
    assert isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == (4,)
    assert out.tolist() == [-float(len(prompt) + i) for i in range(4)]
    assert tts.score("hello", [1, 2], "ref text", np.array([7]), include_eos=False).shape == (1,)
    assert tts.backbone.calls[-1][0][0][-1] == 3007
    outs = tts.score_batch(["a", "bb", "c"], [[1], [2, 3], []], ["x", "y", "z"], [[1, 2], [3], torch.tensor([4, 5, 6])])
    assert [o.shape for o in outs] == [(3,), (2,), (4,)]
    seqs, starts = tts.backbone.calls[-1]
    assert starts == [len(tts._apply_chat_template(c, r, t)) for t, c, r in (("a", [1], "x"), ("bb", [2, 3], "y"), ("c", [], "z"))]
    outs = tts.score_from_prompt_ids([[5, 6, 7]], [[8, 9]])
    assert tts.backbone.calls[-1] == ([[5, 6, 7, 8, 9]], [3]) and outs[0].shape == (2,)


def test_facade_score_errors():
    from tests.fakes import FakeBackbone

    tts = _facade()
    with pytest.raises(ValueError, match="empty"):
        tts.score("a", [1], "x", [])
    with pytest.raises(ValueError, match="0..65535"):
        tts.score("a", [1], "x", [65536])
    with pytest.raises(ValueError, match="0..65535"):
        tts.score("a", [1], "x", [-1])
    with pytest.raises(ValueError, match="same length"):
        tts.score_batch(["a", "b"], [[1]], ["x"], [[1]])
    with pytest.raises(ValueError, match="empty"):
        tts.score_from_prompt_ids([[5]], [[]])
    assert tts.backbone.calls == []
    tts = _facade(lambda tok: FakeBackbone([3005, 2005]))
    with pytest.raises(ValueError, match=r"needs a backbone with score \(neutts_air_b200.SpeechLM\)"):
        tts.score("a", [1], "x", [3])
    with pytest.raises(ValueError, match="backbone with score"):
        tts.score_from_prompt_ids([[5]], [[6]])


# ====================================================================================== C ABI
def test_score_scratch_bytes_without_gpu():
    from neutts_air_b200 import _lib, build

    build.build()
    L = _lib.lib()
    a = lambda x: (x + 255) // 256 * 256
    for V, P in ((217472, 2048), (4142, 300), (4096, 5000)):
        cfg = _lib.LMConfig(V, 896, 4864, 24, 14, 2, 64, 1e-6, 1e6, 4, 2048, 64, 128, P)
        R = min(1024, P)
        assert L.nt_lm_score_scratch_bytes(C.byref(cfg)) == a(8 * R * -(-V // 128)) + a(4 * R) + 2 * a(4 * P)
    bad = _lib.LMConfig(217472, 896, 4864, 24, 14, 2, 128, 1e-6, 1e6, 1, 2048, 64, 32, 2048)
    assert L.nt_lm_score_scratch_bytes(C.byref(bad)) == 0 and b"head_dim" in L.nt_last_error()
