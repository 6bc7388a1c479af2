"""CPU stand-ins for what the facade and the engine's host side talk to: tokenizers, a phonemizer (the HF tokenizer and
espeak are not available offline), codecs and backbones, and ``QueueStub``, a ``SpeechLM`` that keeps its host side
(page pool, per-slot page lists, generate_queue, release_pages) and replaces the device calls: prompt i (every id of it
is i + 1) emits the tokens 1000 * (i + 1) + step, or EOS at a chosen step.  ``GuidedStub`` adds guidance to it."""
import types
import warnings

import torch

from neutts_air_b200.lm import NO_GUIDANCE, PagePool, SpeechLM, check_guidance_table


class FakeTokenizer:
    """Character-level tokenizer with the special tokens the reference adds (TRAINING.md:33-57)."""
    SPECIALS = ["<|TEXT_REPLACE|>", "<|TEXT_PROMPT_START|>", "<|TEXT_PROMPT_END|>", "<|SPEECH_REPLACE|>",
                "<|SPEECH_GENERATION_START|>", "<|SPEECH_GENERATION_END|>"]

    def __init__(self, n_speech=65536):
        self.chars = {chr(c): c for c in range(32, 1024)}
        self.chars["\n"] = 10
        self.special_base = 2000
        self.speech_base = 3000
        self.n_speech = n_speech

    def convert_tokens_to_ids(self, tok):
        if tok in self.SPECIALS:
            return self.special_base + self.SPECIALS.index(tok)
        if tok.startswith("<|speech_"):
            return self.speech_base + int(tok[9:-2])
        raise KeyError(tok)

    def encode(self, text, add_special_tokens=True):
        import re

        out = []
        for part in re.split(r"(<\|[A-Za-z_0-9]+\|>)", text):
            if not part:
                continue
            if part.startswith("<|") and part.endswith("|>"):
                out.append(self.convert_tokens_to_ids(part))
            else:
                out += [self.chars[c] for c in part]
        return out

    def decode(self, ids, add_special_tokens=False):
        inv = {v: k for k, v in self.chars.items()}
        s = ""
        for i in ids:
            if i >= self.speech_base:
                s += f"<|speech_{i - self.speech_base}|>"
            elif i >= self.special_base:
                s += self.SPECIALS[i - self.special_base]
            else:
                s += inv[i]
        return s


class FakePhonemizer:
    def phonemize(self, texts):
        return [t.lower().replace(",", " ,") for t in texts]


class FakeCodec:
    device = torch.device("cpu")
    max_batch = 4

    def decode_code(self, codes):
        return torch.zeros(codes.shape[0], 1, 480 * codes.shape[2]) + codes[:, :, :1].float() / 65536.0


class FakeBackbone:
    """transformers-style .generate(): appends fixed ids (some non-speech) and EOS."""
    device = torch.device("cpu")

    def __init__(self, tail):
        self.tail = tail

    def generate(self, ids, **kw):
        self.kw = kw
        return torch.cat((ids, torch.tensor([self.tail])), dim=1)


def _tts(tail=None):
    from neutts import NeuTTS

    tok = FakeTokenizer()
    tail = tail if tail is not None else [tok.speech_base + 5, 65, tok.speech_base + 70000, tok.speech_base + 9, tok.special_base + 5]
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), backbone=FakeBackbone(tail), codec=FakeCodec()), tok


class RampCodec:
    """Deterministic 'codec': frame i of the window becomes hop samples of code/1000 + 0.01 * position-in-window,
    so a wrong window start, slice or cross-fade weight changes the output."""
    device = torch.device("cpu")
    max_batch = 1
    hop = 8

    def decode_code(self, codes):
        c = codes[0, 0].float()
        frames = c[:, None] / 1000.0 + 0.01 * torch.arange(len(c))[:, None] + torch.zeros(1, self.hop)
        return frames.reshape(1, 1, -1)


class FakeBatchStreamLM:
    """Batched prefill()/decode() surface of SpeechLM: one scripted token stream per slot, lock-step decoding,
    finished slots idle (as inside the persistent kernel)."""
    device = torch.device("cpu")

    def __init__(self, scripts, max_new=4096):
        self.scripts, self.max_new = [list(s) for s in scripts], max_new
        B = len(scripts)
        self.out_tokens = torch.zeros(B, max_new, dtype=torch.int32)
        self.n_generated = torch.zeros(B, dtype=torch.int32)
        self.done = torch.zeros(B, dtype=torch.int32)
        self.decode_calls = []

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, limits=None):
        self.eos = eos
        self.limits = list(limits) if limits is not None else [max_new] * len(self.scripts)
        return None

    def _emit(self):
        for b, script in enumerate(self.scripts):
            n = int(self.n_generated[b])
            if int(self.done[b]) or n >= self.limits[b]:
                continue
            tok = script[n] if n < len(script) else self.eos
            self.out_tokens[b, n] = tok
            self.n_generated[b] = n + 1
            if tok == self.eos or n + 1 >= self.limits[b]:
                self.done[b] = 1

    def prefill(self, prompts, sp):
        self._emit()

    def decode(self, steps, sp):
        assert steps >= 1
        self.decode_calls.append(steps)
        for _ in range(steps):
            self._emit()


class BatchRampCodec(RampCodec):
    max_batch = 2          # smaller than the batch: same-length windows are split over several codec calls

    def decode_code(self, codes):
        assert codes.shape[0] <= self.max_batch
        return torch.cat([RampCodec.decode_code(self, codes[r: r + 1]) for r in range(codes.shape[0])])


EOS = 9


class QueueStub(SpeechLM):
    def __init__(self, max_batch, eos_at=None):
        self.max_ctx, self.max_new, self.max_batch, self.device = 2048, 2048, max_batch, torch.device("cpu")
        self.max_pages = self.max_ctx // self.PAGE
        self.num_pages = max_batch * self.max_pages
        self.pool = PagePool(self.num_pages, shuffle_seed=1)
        self._slot_pages = [[] for _ in range(max_batch)]
        self.out_tokens = torch.zeros(max_batch, self.max_new, dtype=torch.int32)
        self.n_generated = torch.zeros(max_batch, dtype=torch.int32)
        self.done = torch.zeros(max_batch, dtype=torch.int32)
        self.eos_at = eos_at or {}
        self.who, self.cap = [None] * max_batch, [0] * max_batch
        self.log, self.admitted = [], 0

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, limits=None, slot_base=0):
        self.limit_table = list(limits) + [max_new] * (self.max_batch - len(limits))
        self.log.append(("sampling", list(limits), slot_base))
        return types.SimpleNamespace(max_new_tokens=max_new, slot_base=slot_base)

    def _start(self, s, prompt, key):
        tag = prompt[0]
        assert all(t == tag for t in prompt)
        assert key == self.slot_base + tag - 1, (key, tag)   # Philox stream = slot_base + input index
        self._slot_pages[s] = self.pool.alloc((len(prompt) + self.limit_table[s] + self.PAGE - 1) // self.PAGE)
        self.who[s], self.cap[s] = tag, self.limit_table[s]
        self.n_generated[s], self.done[s] = 0, 0
        self.admitted += 1
        self._emit(s)

    def _emit(self, s):
        g = int(self.n_generated[s])
        tok = EOS if self.eos_at.get(self.who[s]) == g else 1000 * self.who[s] + g
        self.out_tokens[s, g], self.n_generated[s] = tok, g + 1
        if tok == EOS or g + 1 >= self.cap[s]:
            self.done[s] = 1

    def prefill(self, prompts, sp):
        self.release_pages()
        self.slot_base = sp.slot_base
        self.log.append(("prefill", [p[0] for p in prompts]))
        for s, p in enumerate(prompts):
            self._start(s, p, sp.slot_base + s)
        self._B = len(prompts)

    def prefill_slots(self, slots, prompts, sp, stream_ids, return_logits=False, limits=None):
        assert all(self.done[s] for s in slots)          # only finished slots are refilled
        self.log.append(("refill", list(slots), [p[0] for p in prompts], list(stream_ids), list(limits)))
        self.release_pages(slots)
        for s, p, key, lim in zip(slots, prompts, stream_ids, limits):
            self.limit_table[s] = lim
            self._start(s, p, key)

    def decode(self, n, sp):
        live = [s for s in range(self._B) if not self.done[s]]
        left = [self.cap[s] - int(self.n_generated[s]) for s in live]
        self.log.append(("decode", n, min(left), max(left), self.admitted))
        for _ in range(n):
            for s in live:
                if not self.done[s]:
                    self._emit(s)


class GuidedStub(QueueStub):
    """QueueStub with guidance: prompt i is i + 1 repeated, its negative prompt -(i + 1) repeated.  A u slot emits
    nothing itself (it mirrors its c on the device); the stub records where each negative prompt went."""

    def __init__(self, max_batch, eos_at=None):
        super().__init__(max_batch, eos_at)
        self._guidance_host = None
        self.u_at = {}   # u slot -> tag of the prompt whose negative prompt it holds
        self.done[:] = 1   # a slot no prefill has filled yet holds nothing to decode: the queue may fill it

    def sampling(self, eos, min_new, max_new, top_k, temperature, seed, greedy, forced=None, limits=None, slot_base=0):
        return super().sampling(eos, min_new, max_new, top_k, temperature, seed, greedy,
                                limits=list(limits) if limits is not None else [max_new] * self.max_batch,
                                slot_base=slot_base)

    def set_guidance(self, rows, slots=None):
        if rows is not None:
            slots = list(range(len(rows))) if slots is None else list(slots)
            table = list(self._guidance_host or [NO_GUIDANCE] * self.max_batch)
            for s, r in zip(slots, rows):
                table[s] = r
            rows = check_guidance_table(table, self.max_batch)
        self.log.append(("guide", None if rows is None else list(rows)))
        self._guidance_host = rows

    def _start(self, s, prompt, key):
        if prompt[0] > 0:
            self.u_at.pop(s, None)
            return super()._start(s, prompt, key)
        tag = -prompt[0]   # u is never sampled: its key is whatever the launch gives its slot
        self._slot_pages[s] = self.pool.alloc((len(prompt) + self.limit_table[s] + self.PAGE - 1) // self.PAGE)
        self.u_at[s] = tag
        self.who[s], self.cap[s] = None, self.limit_table[s]
        self.n_generated[s], self.done[s] = 1, 1   # u never emits here; the queue only reads c slots

    def prefill_slots(self, slots, prompts, sp, stream_ids, return_logits=False, limits=None):
        super().prefill_slots(slots, prompts, sp, stream_ids, return_logits, limits)
        self._B = max(self._B, max(slots) + 1)   # as SpeechLM.prefill_slots: decode covers every slot filled so far

    def set_logprobs(self, on=True):
        self.logprobs = None


def _prompts(lens):
    return [[i + 1] * m for i, m in enumerate(lens)]


class KwBackbone:
    device = torch.device("cpu")

    def __init__(self, tok, queue=True):
        self.tok, self.calls = tok, []
        if queue:
            self.generate_queue = lambda prompts, eos, **kw: self._call("queue", prompts, kw)

    def _call(self, what, prompts, kw):
        self.calls.append((what, len(prompts), kw))
        return [torch.tensor([self.tok.speech_base + 1]) for _ in prompts]

    def generate_batch(self, prompts, eos, **kw):
        return self._call("batch", prompts, kw)


class GenerateBackbone:
    """transformers-style backbone: records the generate kwargs of every utterance."""
    device = torch.device("cpu")

    def __init__(self, tok):
        self.tok, self.kws = tok, []

    def generate(self, ids, **kw):
        self.kws.append(kw)
        return torch.cat((ids, torch.tensor([[self.tok.speech_base + 2]])), dim=1)


def _facade(bb, max_batch):
    from neutts import NeuTTS

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return NeuTTS(tokenizer=bb.tok, phonemizer=FakePhonemizer(), backbone=bb, codec=FakeCodec(), max_batch=max_batch, seed=1)


class SmallTok(FakeTokenizer):
    """FakeTokenizer squeezed into a 4096-token vocabulary: 1024 speech codes from id 3000."""

    def __init__(self):
        super().__init__(n_speech=1024)


class AlignedTok:
    """FakeTokenizer whose 65 536 speech ids start at a 128-aligned id (3072) and end at the vocabulary's end."""

    def __new__(cls):
        tok = FakeTokenizer(n_speech=65536)
        tok.speech_base = 3072
        return tok
