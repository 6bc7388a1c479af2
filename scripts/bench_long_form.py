"""Long-form synthesis vs the loop a user writes without it: one text of 24 sentences, too long for one prompt.

Air-shaped synthetic LM and NeuCodec weights, the character tokenizer and phonemizer of tests/fakes.py, a 400-code
reference.  ``long_form`` runs ``infer(text, long_form=True)``: its segments decode side by side in the engine's slots.
``loop`` runs ``infer`` once per segment of ``segments(text)``, in order, one slot busy at a time.  EOS is masked
through ``min_new_tokens`` so every segment runs to its cap (max_context - prompt length), and both modes generate
the same number of tokens.  As in bench.py, every generated id is folded into the codebook, so each token is one
codec frame.  Streaming: the same pair through ``infer_stream`` (time to the first chunk, wall time to the end).
The modes alternate in one process after a warm-up; medians of ``--repeats`` runs.

    python scripts/bench_long_form.py [--batches 8 16] [--repeats 3]

Prints a device line (card name, power limit, maximum SM clock), the segmentation, and one JSON line per
(max_batch, mode): wall seconds, audio seconds per second, segments, and for streams the time to the first chunk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_queue import device_line  # noqa: E402
from tests.fakes import FakePhonemizer, FakeTokenizer  # noqa: E402

SR = 24_000
REF = 400
REF_TEXT = ("This is the voice we copy, read at an easy pace by a calm speaker in a quiet room, "
            "so the model can hear how it sounds.")
WORDS = ("the a river morning quietly station letter window garden across under before after music small bright "
         "evening table city north thousand paper simple open careful story winter").split()


def long_text(n=24, seed=0) -> str:
    """n sentences of 6..18 seeded words, three paragraphs."""
    rng = np.random.default_rng(seed)
    sents = []
    for i in range(n):
        words = [WORDS[k] for k in rng.integers(0, len(WORDS), int(rng.integers(6, 19)))]
        if len(words) > 9:
            words[len(words) // 2] += ","
        sents.append(" ".join(words).capitalize() + (".", "?", "!")[i % 7 % 3])
    per = n // 3
    return "\n".join(" ".join(sents[k: k + per]) for k in range(0, n, per))


def make_tts(lm, codec, batch):
    from neutts import NeuTTS

    class BenchTTS(NeuTTS):   # a random-weight LM emits arbitrary ids: fold them into the codebook, as bench.py does
        def _ids_to_codes(self, ids):
            return (ids.long() - self.speech_base) % 65536

        def _ids_to_codes_masked(self, ids):
            return (ids.long() - self.speech_base) % 65536, torch.ones_like(ids, dtype=torch.bool)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tts = BenchTTS(backbone=lm, codec=codec, tokenizer=FakeTokenizer(), phonemizer=FakePhonemizer(), max_batch=batch,
                       seed=5)
    tts.watermarker = None
    return tts


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def stream_timed(gens):
    """Consumes the generators in order -> (wall s, first chunk s, samples)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first, samples = None, 0
    for gen in gens:
        for chunk in gen:
            if first is None:
                first = time.perf_counter() - t0
            samples += len(chunk)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, first, samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    from neutts_air_b200 import build, synthetic
    from neutts_air_b200.codec import CodecDecoder, CodecShape
    from neutts_air_b200.lm import LMShape, SpeechLM

    build.build()
    text = long_text()
    ref = torch.randint(0, 65536, (REF,), generator=torch.Generator().manual_seed(1))
    shape = LMShape()
    sd = synthetic.lm_state_dict(shape, 1)
    codec_w = synthetic.codec_weights(CodecShape(), 0)
    print(json.dumps({**device_line(), "sentences": 24, "text_chars": len(text), "ref_codes": REF}), flush=True)
    for B in args.batches:
        lm = SpeechLM(shape, sd, device="cuda", max_batch=B, max_ctx=2048, max_new=2048)
        codec = CodecDecoder(CodecShape(), codec_w, device="cuda", max_batch=B, max_frames=2048)
        tts = make_tts(lm, codec, B)
        segs = tts.segments(text, ref, REF_TEXT)
        caps = [tts.max_context - len(tts._apply_chat_template(ref, REF_TEXT, s)) for s in segs]
        floor = dict(min_new_tokens=tts.max_context)                 # EOS masked: every segment runs to its cap
        if B == args.batches[0]:
            print(json.dumps({"segments": len(segs), "segment_chars": [len(s) for s in segs], "caps": caps}), flush=True)
        modes = {
            "long_form": lambda: [tts.infer(text, ref, REF_TEXT, long_form=True, **floor)],
            "loop": lambda: [tts.infer(s, ref, REF_TEXT, **floor) for s in segs],
        }
        streams = {
            "long_form": lambda: [tts.infer_stream(text, ref, REF_TEXT, long_form=True, **floor)],
            "loop": lambda: [tts.infer_stream(s, ref, REF_TEXT, **floor) for s in segs],
        }
        for fn in list(modes.values()) + list(streams.values()):    # warm-up: graph capture, lazy module loads
            out = fn()
            if not isinstance(out[0], np.ndarray):
                stream_timed(out)
        res = {("whole", m): [] for m in modes}
        res.update({("stream", m): [] for m in streams})
        for _ in range(args.repeats):
            for m, fn in modes.items():
                wall, out = timed(fn)
                res[("whole", m)].append((wall, None, sum(len(w) for w in out)))
            for m, fn in streams.items():
                res[("stream", m)].append(stream_timed(fn()))
        for (kind, m), r in res.items():
            walls = [x[0] for x in r]
            k = int(np.argsort(walls)[len(walls) // 2])
            wall, first, samples = r[k]
            line = {"max_batch": B, "kind": kind, "mode": m, "segments": len(segs), "wall_s": [round(w, 3) for w in walls],
                    "wall_s_median": round(wall, 3), "audio_s": round(samples / SR, 2),
                    "audio_s_per_s": round(samples / SR / wall, 1)}
            if kind == "stream":
                firsts = sorted(x[1] for x in r)
                line["first_chunk_ms_median"] = round(firsts[len(firsts) // 2] * 1e3, 1)
            print(json.dumps(line), flush=True)
        del lm, codec, tts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
