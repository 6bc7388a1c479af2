"""Drop-in ``neutts.NeuTTS`` on the H100 engine.

Same public surface as the reference facade (``/root/reference/neutts/neutts.py:73-465``):
constructor signature and attributes (``:75-98``), ``infer`` (``:216``), ``infer_stream`` (``:245``),
``encode_reference`` (``:266``), the private seams ``_apply_chat_template`` / ``_infer_torch`` /
``_decode`` / ``_to_phones``, and the same error convention (``ValueError`` / ``ImportError`` /
``NotImplementedError``).  Behind it, hot path A (speech-LM prefill + decode) and hot path B
(NeuCodec decoder) run in ``libneutts_b200.so`` on an sm_90a GPU; there is no CPU fallback and no
llama.cpp / ONNX / vLLM dispatch.

What differs from the reference, on purpose:
  * generated ids go straight from the device to the codec (``speech id = token id - id(<|speech_0|>)``)
    instead of ``tokenizer.decode`` + regex; ``_infer_torch`` / ``_decode`` still speak the string
    protocol so code written against the reference keeps working;
  * ``infer_batch`` takes lists and shards utterances over ranks (one NCCL all-gather of waveforms);
  * ``infer_stream`` works on this backend (the reference raises for torch backbones) with the
    reference's streaming window geometry (``:87-91``) and an incremental cross-fade;
  * tokenizer, phonemizer, backbone and codec can be injected, so the facade runs offline.
"""
from __future__ import annotations

import re
import warnings
from pathlib import Path
from typing import Generator, Sequence

import numpy as np
import torch

from neutts_air_b200 import longform
from neutts_air_b200.lm import check_guidance_scale, per_item, per_prompt_decay, per_prompt_ras, resolve_settings

SPEECH_RE = re.compile(r"<\|speech_(\d+)\|>")
CHAT = "user: Convert the text to speech:<|TEXT_REPLACE|>\nassistant:<|SPEECH_REPLACE|>"
CONTROL_DEFAULTS = dict(temperature=1.0, top_k=50, top_p=1.0, min_p=0.0)   # the reference's (neutts/neutts.py:338-347)
PENALTY_DEFAULTS = dict(repetition_penalty=1.0, penalize_prompt=True)       # no repetition penalty, as the reference


def _ras_arg(n: int, ras):
    """``repetition_aware_sampling`` of n utterances, validated: None when no utterance has it (nothing is forwarded),
    one (win_size, tau_r) tuple, or a list with one None / tuple per utterance."""
    per = per_prompt_ras(n, ras)
    if per is None:
        return None
    return per[0] if not isinstance(ras[0], (list, tuple, type(None))) else per   # one pair, or one entry per utterance


def _controls(n: int, temperature, top_k, top_p, min_p, repetition_penalty=1.0, penalize_prompt=True, min_new_tokens=50,
              exponential_decay_length_penalty=None, repetition_aware_sampling=None) -> dict:
    """Sampling controls of n utterances: each a scalar or one value per utterance (a list then).  The length decay and
    the repetition-aware sampling are each None, one pair (a tuple), or a list with one None / pair per utterance."""
    ctl = per_item(n, "utterance", temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p,
                   repetition_penalty=repetition_penalty, penalize_prompt=penalize_prompt, min_new_tokens=min_new_tokens)
    decay = exponential_decay_length_penalty
    if decay is not None:
        per = per_prompt_decay(n, decay)
        if all(d is None for d in per):   # a list with no pair asks for no decay: forward nothing
            decay = None
        else:
            decay = tuple(decay) if per[0] is decay else [None if d is None else tuple(d) for d in per]
    ctl["exponential_decay_length_penalty"] = decay
    ctl["repetition_aware_sampling"] = _ras_arg(n, repetition_aware_sampling)
    return ctl


def _guided(n: int, guidance_scale) -> bool:
    """Whether any of n utterances is guided: ``guidance_scale`` a number or one per utterance, each finite and > 0
    (1 = off; ValueError otherwise)."""
    g = per_item(n, "utterance", guidance_scale=guidance_scale)["guidance_scale"]
    return any(check_guidance_scale(x) != 1.0 for x in (g if isinstance(g, list) else [g]))


def _add_guidance(ctl: dict, n: int, guidance_scale, negatives) -> dict:
    """The controls of n utterances with classifier-free guidance: ``negatives`` None or one negative prompt (id list,
    or None for the prompt's last token) per utterance.  Nothing is added when no utterance is guided, so the engine
    calls stay exactly those of a run without guidance."""
    if _guided(n, guidance_scale):
        g = per_item(n, "utterance", guidance_scale=guidance_scale)["guidance_scale"]
        if negatives is not None and len(negatives) != n:
            raise ValueError(f"negative prompts need one entry per utterance ({n}), got {len(negatives)}")
        ctl["guidance_scale"] = g
        ctl["negative_prompt_ids"] = None if negatives is None else [None if q is None else list(q) for q in negatives]
    return ctl


def _speeds(n: int, speed):
    """One speaking rate per utterance (``speed`` a number or one per utterance, each in [0.5, 2.0]; ValueError
    otherwise), or None when every one is 1.0: then nothing is stretched and no stretcher is built."""
    from neutts_air_b200.stretch import check_speed

    s = per_item(n, "utterance", speed=speed)["speed"]
    s = [check_speed(x) for x in s] if isinstance(s, list) else [check_speed(s)] * n
    return s if any(x != 1.0 for x in s) else None


def _targets(n: int, loudness):
    """One loudness target per utterance (``loudness`` None, a number, or one number / None per utterance, each finite
    and in [-70, 0] LUFS; ValueError otherwise), or None when no utterance has one: then nothing is measured."""
    from neutts_air_b200.loudness import check_target

    if loudness is None:
        return None
    t = per_item(n, "utterance", loudness=loudness)["loudness"]
    t = [None if x is None else check_target(x) for x in t] if isinstance(t, list) else [check_target(t)] * n
    return t if any(x is not None for x in t) else None


def _pick(ctl: dict, idx) -> dict:
    """The controls of the utterances ``idx`` (lists are indexed, scalars stay)."""
    return {k: [v[i] for i in idx] if isinstance(v, list) else v for k, v in ctl.items()}


def _backbone_kw(ctl: dict) -> dict:
    """generate kwargs: temperature and top_k always (as the reference passes them), top_p / min_p only when they are
    in use, and the repetition penalty pair only when it differs from the defaults, so that backbones without them keep
    working."""
    kw = dict(temperature=ctl["temperature"], top_k=ctl["top_k"])
    kw.update({k: ctl[k] for k in ("top_p", "min_p") if isinstance(ctl[k], list) or ctl[k] != CONTROL_DEFAULTS[k]})
    pen = {k: ctl.get(k, v) for k, v in PENALTY_DEFAULTS.items()}
    if any(isinstance(v, list) or v != PENALTY_DEFAULTS[k] for k, v in pen.items()):
        kw.update(pen)
    if ctl.get("exponential_decay_length_penalty") is not None:
        kw["exponential_decay_length_penalty"] = ctl["exponential_decay_length_penalty"]
    if ctl.get("repetition_aware_sampling") is not None:
        kw["repetition_aware_sampling"] = ctl["repetition_aware_sampling"]
    if "guidance_scale" in ctl:
        kw["guidance_scale"] = ctl["guidance_scale"]
        kw["negative_prompt_ids"] = ctl["negative_prompt_ids"]
    return kw


def best_takes(logprobs, n: int) -> list:
    """Index of the kept take of every prompt, given its n takes' log-probability rows in slot order (take j of prompt i
    at index i * n + j, rows [n_generated, 2] of (sampled, model)): the take with the highest mean ``model``
    log-probability over its generated tokens, EOS included; ties go to the lowest take index."""
    keep = []
    for i in range(len(logprobs) // n):
        means = [float(np.mean(np.asarray(logprobs[i * n + j], dtype=np.float64)[:, 1])) for j in range(n)]
        keep.append(i * n + max(range(n), key=lambda j: (means[j], -j)))
    return keep


class _CrossFade:
    """Incremental equivalent of the reference's ``_linear_overlap_add`` (``neutts/neutts.py:46-70``):
    triangular weights over every chunk, weighted sum / weight sum, but only the samples a new chunk
    can still change are kept (the reference re-sums the whole history on every chunk)."""

    def __init__(self, stride: int):
        self.stride = stride
        self.acc = np.zeros(0, dtype=np.float32)
        self.wsum = np.zeros(0, dtype=np.float32)

    def push(self, frame: np.ndarray, final: bool = False) -> np.ndarray:
        n = frame.shape[-1]
        t = np.linspace(0, 1, n + 2, dtype=np.float32)[1:-1]
        w = np.abs(0.5 - (t - 0.5))
        if n > self.acc.shape[0]:
            grow = n - self.acc.shape[0]
            self.acc = np.concatenate([self.acc, np.zeros(grow, np.float32)])
            self.wsum = np.concatenate([self.wsum, np.zeros(grow, np.float32)])
        self.acc[:n] += w * frame.astype(np.float32)
        self.wsum[:n] += w
        take = self.acc.shape[0] if final else min(self.stride, self.acc.shape[0])
        out = self.acc[:take] / self.wsum[:take]
        self.acc, self.wsum = self.acc[take:], self.wsum[take:]
        return out


class NeuTTS:
    def __init__(self, backbone_repo="neuphonic/neutts-nano", backbone_device="cpu", codec_repo="neuphonic/neucodec",
                 codec_device="cpu", *, tokenizer=None, phonemizer=None, backbone=None, codec=None,
                 max_batch: int = 1, seed: int | None = None, speech_tokens_only: bool = False,
                 sample_rate: int = 24_000, pcm_format: str = "float32"):
        """Same positional signature and defaults as the reference (``neutts/neutts.py:75-81``), so
        ``examples/basic_example.py:12-17`` runs unmodified.  The device strings keep their reference
        meaning for the CALLER -- ``"cpu"`` = results come back as host arrays, which this facade always
        does -- but the engines themselves only exist for sm_90a: a ``"cpu"`` request runs on the current
        CUDA device and says so once (there is no CPU fallback).  ``speech_tokens_only``: generation may only draw
        ``<|speech_N|>`` ids and ``<|SPEECH_GENERATION_END|>`` (every other id suppressed, as transformers'
        ``suppress_tokens``); the engine then skips the lm_head rows of every other id.

        ``sample_rate`` and ``pcm_format`` ("float32" or "int16") choose what every waveform comes back as.  NeuCodec
        synthesises 24 kHz float32; any other setting resamples on the GPU before the copy to the host, with
        torchaudio's ``resample`` semantics (``neutts_air_b200.resample.Resampler``), streams included.  "int16" is
        ``rint(clip(y, -1, 1) * 32767)`` (clipped, rounded half to even), not the truncating ``astype`` that wraps
        samples beyond +-1.  The watermark, when there is one, is applied at 24 kHz first, as the reference does."""
        if not (type(sample_rate) is int and sample_rate == 24_000 and pcm_format == "float32"):
            from neutts_air_b200.resample import check_args

            check_args(sample_rate, pcm_format)   # ValueError for a rate or format the resampler cannot serve
        self.sample_rate = int(sample_rate)       # the rate of every waveform returned (the codec's is 24 kHz)
        self.pcm_format = pcm_format
        self._resampler = None
        self._stretcher = None
        # constants the reference exposes (neutts/neutts.py:84-91)
        self.max_context = 2048
        self.hop_length = 480
        self.streaming_overlap_frames = 1
        self.streaming_frames_per_chunk = 25
        self.streaming_lookforward = 5
        self.streaming_lookback = 50
        self.streaming_stride_samples = self.streaming_frames_per_chunk * self.hop_length
        self._is_quantized_model = False
        self._is_onnx_codec = False
        self.tokenizer = tokenizer
        self.max_batch = max_batch
        self.seed = seed
        self.speech_tokens_only = bool(speech_tokens_only)
        self.phonemizer = phonemizer if phonemizer is not None else self._load_phonemizer()
        self._load_backbone(backbone_repo, backbone_device, backbone)
        self._load_codec(codec_repo, codec_device, codec)
        try:  # optional watermark, exactly as the reference (neutts/neutts.py:110-121)
            import perth

            self.watermarker = perth.PerthImplicitWatermarker()
        except (ImportError, AttributeError) as e:
            warnings.warn(f"Perth watermarking unavailable: {e}. Audio will not be watermarked.")
            self.watermarker = None
        self._speech_base = None

    # ------------------------------------------------------------------ loading
    @staticmethod
    def _load_phonemizer():
        try:
            from phonemizer.backend import EspeakBackend
        except ImportError as e:
            raise ImportError("phonemizer (and espeak-ng) are required for text input; "
                              "pass phonemizer=... to NeuTTS to inject one") from e
        return EspeakBackend(language="en-us", preserve_punctuation=True, with_stress=True)

    def _load_backbone(self, backbone_repo, backbone_device, backbone=None):
        if backbone is not None:
            self.backbone = backbone
            return
        if str(backbone_repo).endswith("gguf"):
            raise ValueError("GGUF / llama.cpp backbones are not dispatched by the H100 build; "
                             "use the safetensors checkpoint (e.g. neuphonic/neutts-air)")
        backbone_device = self._engine_device(backbone_device, "backbone")
        from neutts_air_b200 import loader

        if self.tokenizer is None:
            self.tokenizer = loader.load_tokenizer(backbone_repo)
        self.backbone = loader.load_speech_lm(backbone_repo, backbone_device, max_batch=self.max_batch,
                                              max_ctx=self.max_context)

    def _load_codec(self, codec_repo, codec_device, codec=None):
        if codec is not None:
            self.codec = codec
            return
        if str(codec_repo).endswith(".onnx") or codec_repo == "neuphonic/neucodec-onnx-decoder":
            raise ValueError("ONNX codec decoders are not dispatched by the H100 build; use 'neuphonic/neucodec'")
        if codec_repo not in ("neuphonic/neucodec", "neuphonic/distill-neucodec") and not Path(str(codec_repo)).exists():
            raise ValueError("Invalid codec repo! Must be one of: 'neuphonic/neucodec', 'neuphonic/distill-neucodec' "
                             "(or a local checkpoint directory).")
        codec_device = self._engine_device(codec_device, "codec")
        from neutts_air_b200 import loader

        self.codec = loader.load_codec_decoder(codec_repo, codec_device, max_batch=self.max_batch,
                                               max_frames=self.max_context)

    @staticmethod
    def _engine_device(requested, what: str):
        """Reference device string -> the CUDA device the H100 engine runs on."""
        dev = torch.device(requested)
        if dev.type == "cuda":
            return dev
        if dev.type != "cpu":
            raise ValueError(f"unsupported {what}_device {requested!r}")
        if not torch.cuda.is_available():
            raise RuntimeError(f"neutts (H100 build): {what}_device={requested!r} was requested, but the engines exist only for "
                               "CUDA sm_90a and no CUDA device is visible (there is no CPU fallback)")
        warnings.warn(f"neutts (H100 build): {what}_device={requested!r} -> running on cuda:{torch.cuda.current_device()}; "
                      "outputs are returned on the host as with the reference's CPU path", stacklevel=3)
        return torch.device("cuda", torch.cuda.current_device())

    # ------------------------------------------------------------------ prompt construction (N1)
    def _to_phones(self, text: str) -> str:
        return " ".join(self.phonemizer.phonemize([text])[0].split())

    def _tok_id(self, name: str) -> int:
        return self.tokenizer.convert_tokens_to_ids(name)

    @property
    def speech_base(self) -> int:
        """Token id of ``<|speech_0|>``; speech ids are contiguous above it (TRAINING.md:52-57 adds
        them with one ``add_tokens`` call), which is checked once here."""
        if self._speech_base is None:
            base = self._tok_id("<|speech_0|>")
            probe = (1, 4095, 65535)
            if any(self._tok_id(f"<|speech_{i}|>") != base + i for i in probe):
                raise ValueError("tokenizer does not map <|speech_N|> to consecutive ids")
            self._speech_base = base
        return self._speech_base

    def _apply_chat_template(self, ref_codes, ref_text: str, input_text: str) -> list:
        """Same id sequence as the reference builds (``neutts/neutts.py:303-332``):
        ``user: Convert the text to speech: [TPS] phones [TPE] \\nassistant: [SGS] ref speech ids``."""
        phones = self._to_phones(ref_text) + " " + self._to_phones(input_text)
        text_ids = self.tokenizer.encode(phones, add_special_tokens=False)
        ids = list(self.tokenizer.encode(CHAT))
        t = ids.index(self._tok_id("<|TEXT_REPLACE|>"))
        ids = ids[:t] + [self._tok_id("<|TEXT_PROMPT_START|>")] + list(text_ids) + [self._tok_id("<|TEXT_PROMPT_END|>")] + ids[t + 1:]
        s = ids.index(self._tok_id("<|SPEECH_REPLACE|>"))
        codes = [int(c) for c in (ref_codes.tolist() if hasattr(ref_codes, "tolist") else ref_codes)]
        base = self.speech_base
        return ids[:s] + [self._tok_id("<|SPEECH_GENERATION_START|>")] + [base + c for c in codes]

    # ------------------------------------------------------------------ hot path A
    def _check_logprobs(self, distributed: bool = False) -> None:
        """``return_logprobs`` needs an engine that writes them (``SpeechLM.set_logprobs``) and a single process."""
        if distributed:
            raise ValueError("return_logprobs is not supported with distributed=True")
        if not hasattr(self.backbone, "set_logprobs"):
            raise ValueError("return_logprobs needs a backbone with set_logprobs (neutts_air_b200.SpeechLM)")

    def _check_takes(self, takes, distributed: bool = False) -> int:
        """``takes`` per utterance: an integer in 1..max_batch; more than one needs a single process and an engine that
        writes log-probabilities (the best take is chosen by them) and forks a prefill (``generate_batch``'s
        ``num_return_sequences``)."""
        if isinstance(takes, bool) or not isinstance(takes, (int, np.integer)) or not 1 <= takes <= self.max_batch:
            raise ValueError(f"takes {takes!r} must be an integer in 1..max_batch ({self.max_batch})")
        if takes > 1:
            if distributed:
                raise ValueError("takes > 1 is not supported with distributed=True")
            if not hasattr(self.backbone, "set_logprobs"):
                raise ValueError("takes > 1 needs a backbone with set_logprobs (neutts_air_b200.SpeechLM)")
        return int(takes)

    def _generate_ids(self, prompts: Sequence[Sequence[int]], max_new_tokens: int | None = None,
                      min_new_tokens: int = 50, slot_base: int = 0, ctl: dict | None = None, logprobs: bool = False,
                      takes: int = 1):
        """Batched device-side generation; returns generated token ids per prompt (CPU int64 tensors), or with
        ``logprobs`` (ids, per-prompt float32 CPU tensors [n, 2] of (sampled, model) log-probabilities).
        Sampling parameters default to the reference's (``neutts/neutts.py:338-347``); ``ctl`` (see ``_controls``)
        overrides them, per prompt where a control is a list; ``min_new_tokens`` is an int or one per prompt.  ``takes`` > 1: that many takes of every prompt from
        one prefill (len(prompts) * takes <= max_batch), of which the one ``best_takes`` picks is returned."""
        eos = self._tok_id("<|SPEECH_GENERATION_END|>")
        seed = self.seed if self.seed is not None else int(torch.randint(0, 2**31 - 1, (1,)).item())
        kw = _backbone_kw(ctl if ctl is not None else CONTROL_DEFAULTS)
        if logprobs:
            self._check_logprobs()
            kw["return_logprobs"] = True
        rng = self._speech_range()
        if rng is not None:
            kw["vocab_range"] = rng
        if takes > 1 and "guidance_scale" in kw:
            raise ValueError("classifier-free guidance generates one take per utterance (takes=1)")
        if takes > 1:
            kw["return_logprobs"] = True
            ids, lps = self.backbone.generate_batch(list(prompts), eos, max_length=self.max_context, min_new_tokens=min_new_tokens,
                                                    max_new_tokens=max_new_tokens, seed=seed, slot_base=slot_base,
                                                    num_return_sequences=takes, **kw)
            keep = best_takes(lps, takes)
            ids, lps = [ids[k] for k in keep], [lps[k] for k in keep]
            return (ids, lps) if logprobs else ids
        if self._slots(len(prompts), kw) > self.max_batch and hasattr(self.backbone, "generate_queue"):
            # more prompts than slots: refill each slot as soon as its utterance ends (prompt i keeps the Philox
            # stream slot_base + i that the chunked loop gives it)
            return self.backbone.generate_queue(list(prompts), eos, max_length=self.max_context, min_new_tokens=min_new_tokens,
                                                max_new_tokens=max_new_tokens, seed=seed, slot_base=slot_base, **kw)
        if hasattr(self.backbone, "generate_batch"):
            return self.backbone.generate_batch(list(prompts), eos, max_length=self.max_context, min_new_tokens=min_new_tokens,
                                                max_new_tokens=max_new_tokens, seed=seed, slot_base=slot_base, **kw)
        outs = []  # injected transformers-style backbone: one sequence at a time, as the reference does
        suppress = {}
        if rng is not None:   # the same allowed set as transformers' suppress_tokens list
            del kw["vocab_range"]
            vocab = getattr(getattr(self.backbone, "config", None), "vocab_size", None) or len(self.tokenizer)
            suppress["suppress_tokens"] = [i for i in range(vocab) if not (rng[0] <= i < rng[1] or i == eos)]
        for i, p in enumerate(prompts):
            t = torch.tensor(list(p)).unsqueeze(0).to(self.backbone.device)
            one = {k: v[i] if isinstance(v, list) else v for k, v in kw.items()}
            if one.get("exponential_decay_length_penalty", ()) is None:   # this utterance has no decay: pass nothing
                del one["exponential_decay_length_penalty"]
            one.update(suppress)
            g, neg = one.pop("guidance_scale", 1.0), one.pop("negative_prompt_ids", None)
            if g != 1.0:   # transformers' UnbatchedClassifierFreeGuidanceLogitsProcessor; None: the prompt's last token
                one["guidance_scale"] = g
                if neg is not None:
                    one["negative_prompt_ids"] = torch.tensor([list(neg)]).to(self.backbone.device)
            with torch.no_grad():
                o = self.backbone.generate(t, max_length=self.max_context, eos_token_id=eos, do_sample=True, use_cache=True,
                                           min_new_tokens=min_new_tokens[i] if isinstance(min_new_tokens, list) else min_new_tokens,
                                           **one)
            outs.append(o[0, t.shape[-1]:].cpu().long())
        return outs

    @staticmethod
    def _slots(n: int, ctl: dict) -> int:
        """Engine slots n prompts take at once: one each, and one more for every guided prompt's negative prompt."""
        g = ctl.get("guidance_scale", 1.0)
        return n + (sum(x != 1.0 for x in g) if isinstance(g, list) else (n if g != 1.0 else 0))

    def _negatives(self, n: int, guidance_scale, negative_text, ref_codes, ref_texts):
        """The negative prompts of n utterances: the chat template with the utterance's reference codes and text and
        ``negative_text`` (a string or one per utterance; None is "", the voice without the words) as the input text.
        None when no utterance is guided."""
        if not _guided(n, guidance_scale):
            return None
        neg = per_item(n, "utterance", negative_text=negative_text)["negative_text"]
        neg = neg if isinstance(neg, list) else [neg] * n
        return [self._apply_chat_template(c, rt, t if t is not None else "") for c, rt, t in zip(ref_codes, ref_texts, neg)]

    @staticmethod
    def _no_guidance(guidance_scale, what: str) -> None:
        if _guided(len(guidance_scale) if isinstance(guidance_scale, (list, tuple)) else 1, guidance_scale):
            raise ValueError(f"classifier-free guidance is not supported by {what} (guidance_scale must be 1)")

    def _n_codes(self) -> int:
        shape = getattr(self.codec, "shape", None)
        return getattr(shape, "fsq_levels", 4) ** getattr(shape, "fsq_dims", 8)

    def _speech_range(self):
        """[speech_base, speech_base + n_codes) while ``speech_tokens_only`` is on, else None."""
        return (self.speech_base, self.speech_base + self._n_codes()) if self.speech_tokens_only else None

    def _ids_to_codes(self, ids: torch.Tensor) -> torch.Tensor:
        """Drop every token that is not ``<|speech_N|>`` (the reference's regex does the same, ``:276``)."""
        base = self.speech_base
        n_codes = getattr(getattr(self.codec, "shape", None), "fsq_levels", 4) ** getattr(getattr(self.codec, "shape", None), "fsq_dims", 8)
        c = ids.long() - base
        return c[(c >= 0) & (c < n_codes)]

    def _ids_to_codes_masked(self, ids: torch.Tensor):
        """Tensor form of ``_ids_to_codes`` for the device-side code history: (codes, keep mask), same shape as ids."""
        shape = getattr(self.codec, "shape", None)
        n_codes = getattr(shape, "fsq_levels", 4) ** getattr(shape, "fsq_dims", 8)
        c = ids.long() - self.speech_base
        return c, (c >= 0) & (c < n_codes)

    def _infer_torch(self, prompt_ids: list) -> str:
        """String protocol of the reference seam (``neutts/neutts.py:334-352``)."""
        out = self._generate_ids([prompt_ids])[0]
        return self.tokenizer.decode(out.numpy().tolist(), add_special_tokens=False)

    # ------------------------------------------------------------------ hot path B
    def _output_resampler(self):
        """The GPU resampler to ``sample_rate`` / ``pcm_format`` (one row per slot), or None for 24 kHz float32."""
        if self._resampler is None and (self.sample_rate, self.pcm_format) != (24_000, "float32"):
            from neutts_air_b200.resample import Resampler

            rows = max(self.max_batch, getattr(self.backbone, "max_batch", 1))
            self._resampler = Resampler(self.sample_rate, self.pcm_format, device=self.codec.device, max_rows=rows)
        return self._resampler

    def _time_stretch(self):
        """The GPU speaking-rate stretcher (one stream row per slot), built on first use."""
        if self._stretcher is None:
            from neutts_air_b200.stretch import TimeStretch

            rows = max(self.max_batch, getattr(self.backbone, "max_batch", 1))
            self._stretcher = TimeStretch(device=self.codec.device, max_rows=rows)
        return self._stretcher

    def _decode_codes(self, codes: Sequence[torch.Tensor], watermark: bool = False, speeds=None, targets=None) -> list:
        """codes: list of 1-D int tensors -> list of numpy waveforms at ``sample_rate`` in ``pcm_format`` (batched by
        equal length).  ``watermark``: each waveform is watermarked at 24 kHz, before any resampling.  ``speeds``: None
        or one speaking rate per waveform; a waveform whose rate is not 1.0 is stretched at 24 kHz right after the
        codec, before the watermark and the resampler.  ``targets``: None or one loudness target (LUFS, or None) per
        waveform; a waveform with one is normalised to it at 24 kHz after the stretch, before the watermark."""
        if speeds is not None or targets is not None:
            return self._decode_stretched(codes, watermark, speeds, targets)
        rs = self._output_resampler()
        out = [None] * len(codes)
        by_len: dict = {}
        for i, c in enumerate(codes):
            if len(c) == 0:
                raise ValueError("No valid speech tokens found in the output.")
            by_len.setdefault(len(c), []).append(i)
        cap = getattr(self.codec, "max_batch", 1)
        for n, idxs in by_len.items():
            for j in range(0, len(idxs), cap):
                grp = idxs[j: j + cap]
                batch = torch.stack([codes[i].long() for i in grp])[:, None, :].to(self.codec.device)
                if rs is None:
                    with torch.no_grad():
                        pcm = self.codec.decode_code(batch).cpu().numpy()
                    for r, i in enumerate(grp):
                        out[i] = pcm[r, 0, :]
                    continue
                with torch.no_grad():
                    pcm = self.codec.decode_code(batch)[:, 0, :]
                if watermark and self.watermarker is not None:
                    wm = np.stack([self._watermark(w) for w in pcm.cpu().numpy()]).astype(np.float32)
                    pcm = torch.from_numpy(wm).to(rs.device)
                pcm = rs.resample(pcm).cpu().numpy()
                for r, i in enumerate(grp):
                    out[i] = pcm[r]
        if watermark and rs is None:
            out = [self._watermark(w) for w in out]
        return out

    def _decode_stretched(self, codes, watermark: bool, speeds, targets=None) -> list:
        """``_decode_codes`` with speaking rates or loudness targets (either may be None): per waveform codec -> stretch
        (rate != 1.0) -> loudness (a target) -> watermark -> resample, all but the watermark on the device; a waveform
        at 1.0 without a target gets the bytes it gets without either."""
        from neutts_air_b200.loudness import normalize

        rs = self._output_resampler()
        ts = self._time_stretch() if speeds is not None else None
        out = [None] * len(codes)
        by_len: dict = {}
        for i, c in enumerate(codes):
            if len(c) == 0:
                raise ValueError("No valid speech tokens found in the output.")
            by_len.setdefault(len(c), []).append(i)
        cap = getattr(self.codec, "max_batch", 1)
        for n, idxs in by_len.items():
            for j in range(0, len(idxs), cap):
                grp = idxs[j: j + cap]
                batch = torch.stack([codes[i].long() for i in grp])[:, None, :].to(self.codec.device)
                with torch.no_grad():
                    pcm = self.codec.decode_code(batch)[:, 0, :]
                rows = list(pcm)
                fast = [r for r, i in enumerate(grp) if speeds is not None and speeds[i] != 1.0]
                if fast:
                    for r, y in zip(fast, ts.stretch([rows[r] for r in fast], [speeds[grp[r]] for r in fast])):
                        rows[r] = y
                level = [r for r, i in enumerate(grp) if targets is not None and targets[i] is not None]
                if level:
                    for r, y in zip(level, normalize([rows[r] for r in level], [targets[grp[r]] for r in level])):
                        rows[r] = y
                for r, i in enumerate(grp):
                    w = rows[r]
                    if watermark and self.watermarker is not None:
                        w = self._watermark(w.cpu().numpy())
                        w = torch.from_numpy(np.asarray(w, dtype=np.float32)).to(pcm.device) if rs is not None else w
                    if rs is not None:
                        w = rs.resample(w)
                    out[i] = w.cpu().numpy() if isinstance(w, torch.Tensor) else w
        return out

    def _decode(self, codes) -> np.ndarray:
        """``codes``: the ``<|speech_N|>`` string of the reference seam (``neutts/neutts.py:273-295``) or a 1-D int sequence."""
        if isinstance(codes, str):
            ids = [int(n) for n in SPEECH_RE.findall(codes)]
            codes = torch.tensor(ids, dtype=torch.long)
        else:
            codes = torch.as_tensor(codes, dtype=torch.long).flatten()
        if len(codes) == 0:
            raise ValueError("No valid speech tokens found in the output.")
        return self._decode_codes([codes])[0]

    def _watermark(self, wav: np.ndarray) -> np.ndarray:
        return wav if self.watermarker is None else self.watermarker.apply_watermark(wav, sample_rate=24_000)

    # ------------------------------------------------------------------ public API
    def infer(self, text: str, ref_codes, ref_text: str, *, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0,
              min_p: float = 0.0, repetition_penalty: float = 1.0, penalize_prompt: bool = True,
              return_logprobs: bool = False, takes: int = 1, min_new_tokens: int = 50,
              exponential_decay_length_penalty=None, guidance_scale: float = 1.0, negative_text: str | None = None,
              speed: float = 1.0, long_form: bool = False, pause: float = 0.0, repetition_aware_sampling=None,
              loudness=None):
        """Text + reference voice -> 24 kHz float32 waveform (``neutts/neutts.py:216-243``).  The sampling controls
        default to the reference's values; see ``infer_batch``.  ``return_logprobs``: returns (waveform, log-probs).
        ``takes``: generate that many takes and keep the most probable one (``infer_batch``).  ``guidance_scale`` and
        ``negative_text``: classifier-free guidance (``infer_batch``).  ``speed``: speaking rate (``infer_batch``).
        ``long_form`` and ``pause``: a text longer than the context, in segments (``infer_batch``).
        ``repetition_aware_sampling``: redraw a token that loops (``infer_batch``).  ``loudness``: a target in LUFS
        (``infer_batch``)."""
        out = self.infer_batch([text], [ref_codes], [ref_text], temperature=temperature, top_k=top_k, top_p=top_p,
                               min_p=min_p, repetition_penalty=repetition_penalty, penalize_prompt=penalize_prompt,
                               return_logprobs=return_logprobs, takes=takes, min_new_tokens=min_new_tokens,
                               exponential_decay_length_penalty=exponential_decay_length_penalty,
                               guidance_scale=guidance_scale, negative_text=negative_text, speed=speed,
                               long_form=long_form, pause=pause, repetition_aware_sampling=repetition_aware_sampling,
                               loudness=loudness)
        return (out[0][0], out[1][0]) if return_logprobs else out[0]

    def infer_from_prompt_ids(self, prompts: Sequence[Sequence[int]], max_new_tokens: int | None = None,
                              min_new_tokens: int = 50, slot_base: int = 0, *, temperature=1.0, top_k=50, top_p=1.0,
                              min_p=0.0, repetition_penalty=1.0, penalize_prompt=True, return_logprobs: bool = False,
                              takes: int = 1, exponential_decay_length_penalty=None, guidance_scale=1.0,
                              negative_prompt_ids=None, speed=1.0, repetition_aware_sampling=None, loudness=None):
        """Hot path only: prompt ids (host) -> waveforms (host).  Used by bench.py's end-to-end leg.
        ``slot_base`` offsets the sampler's Philox slot index so chunks / ranks under one seed draw independently.
        More prompts than ``max_batch`` go through the backbone's ``generate_queue`` when it has one.  Sampling
        controls, length controls, ``return_logprobs`` and ``takes`` as in ``infer_batch`` (here len(prompts) * takes <=
        max_batch, and ``slot_base`` counts takes).  ``guidance_scale`` (a number or one per prompt, 1 = off) and
        ``negative_prompt_ids`` (None, or one id list or None per prompt; None: the prompt's last token) add
        classifier-free guidance (``SpeechLM.generate_batch``; transformers' ``guidance_scale`` and
        ``negative_prompt_ids`` on an injected transformers backbone).  ``speed``: speaking rate of each waveform (a
        number or one per prompt, ``infer_batch``); it acts on the PCM alone and never reaches the backbone.
        ``repetition_aware_sampling`` and ``loudness`` (a target or one per prompt) as in ``infer_batch``."""
        speeds = _speeds(len(prompts), speed)
        targets = _targets(len(prompts), loudness)
        ctl = _controls(len(prompts), temperature, top_k, top_p, min_p, repetition_penalty, penalize_prompt, min_new_tokens,
                        exponential_decay_length_penalty, repetition_aware_sampling)
        self._check_ras(ctl)
        ctl = _add_guidance(ctl, len(prompts), guidance_scale, negative_prompt_ids)
        min_new_tokens = ctl.pop("min_new_tokens")
        takes = self._check_takes(takes)
        if takes > 1 and return_logprobs:
            self._check_logprobs()
        gen = self._generate_ids(prompts, max_new_tokens, min_new_tokens, slot_base, ctl, logprobs=return_logprobs,
                                 takes=takes)
        if return_logprobs:
            gen, lps = gen
        wavs = self._decode_codes([self._ids_to_codes(g) for g in gen], watermark=True, speeds=speeds, targets=targets)
        return (wavs, [lp.numpy() for lp in lps]) if return_logprobs else wavs

    def infer_batch(self, texts: Sequence[str], ref_codes: Sequence, ref_texts: Sequence[str], distributed: bool = False, *,
                    temperature=1.0, top_k=50, top_p=1.0, min_p=0.0, repetition_penalty=1.0, penalize_prompt=True,
                    return_logprobs: bool = False, takes: int = 1, min_new_tokens=50, exponential_decay_length_penalty=None,
                    guidance_scale=1.0, negative_text=None, speed=1.0, long_form: bool = False, pause: float = 0.0,
                    repetition_aware_sampling=None, loudness=None):
        """List in / list out.  With ``distributed=True`` (inside an initialised torch.distributed job) the
        utterances are sharded over ranks and every rank returns all waveforms (one all-gather).

        A list longer than ``max_batch`` (per rank when distributed) runs as one queue on a backbone that has
        ``generate_queue``: a slot whose utterance ended takes the next one while the others keep decoding, so a
        short utterance does not hold its slot until the longest of its chunk ends.  Utterance i keeps the random
        stream it has in the chunked schedule.  Shorter lists, and backbones without ``generate_queue``, run in
        chunks of ``max_batch``.  The codec then decodes the finished code lists either way.

        Sampling controls (keyword-only; the defaults are the reference's): ``temperature`` (logits times 1 / T),
        ``top_k`` (1..64), ``top_p`` (nucleus, (0, 1]) and ``min_p`` ([0, 1)), applied in transformers' order.  Each
        is a scalar or a list with one value per utterance; a list follows its utterances through chunking, the queue
        and the sharding over ranks.  ``repetition_penalty`` (transformers' RepetitionPenaltyLogitsProcessor: > 0, 1 =
        off) divides the positive logits and multiplies the negative ones of every id already in the utterance, which
        breaks loops of one repeated codec id; ``penalize_prompt=False`` leaves the prompt (the reference codes) out of
        that history.  Both are scalars or one value per utterance too.

        Length controls (transformers' processors, acting on the end-of-speech score alone): ``min_new_tokens``
        (default 50, the reference's one second of audio) masks the end of speech until that many tokens exist, an int
        or one per utterance, so a short line need not run a whole second.  ``exponential_decay_length_penalty``
        (start, factor), factor > 0 (ExponentialDecayLengthPenalty), is a soft cap: after ``start`` generated tokens the
        end-of-speech score s becomes s + |s| * (factor ** k - 1) at step k past it, so an utterance that runs on ends
        at a point the model picks near the length the caller expects, instead of being cut at the hard cap.  None, one
        pair, or one None / pair per utterance; start must be >= min_new_tokens - 1.

        ``repetition_aware_sampling`` (VALL-E 2's Repetition Aware Sampling, CosyVoice 2's ``ras_sampling``): None (the
        default), one (win_size, tau_r) pair, or one None / pair per utterance, win_size an int in 1..64 and tau_r in
        (0, 1].  A drawn code that already occurs at least ceil(win_size * tau_r) times among the utterance's last
        win_size generated codes is thrown away and drawn again from the whole distribution (no top-k / top-p / min-p
        cut), which breaks a loop of one repeated code where it happens and leaves every other step alone.  Needs a
        ``SpeechLM`` backbone (ValueError otherwise: transformers' ``generate`` has no such option).

        ``return_logprobs=True`` (not with ``distributed``; needs a ``SpeechLM`` backbone) returns (waveforms,
        log-probs): per utterance a float32 array [n_generated, 2] with the (sampled, model) log-probability of every
        generated token, EOS included (``SpeechLM.set_logprobs``).  Its rows follow the generated ids, not the codec
        frames: a non-speech id the codec never sees keeps its row.  ``sampled`` is the token's log-probability in the
        distribution it was drawn from (after every control above), ``model`` its log-softmax over the whole
        vocabulary after the repetition penalty and before temperature and the warpers; their mean or minimum over an
        utterance flags a bad take, or picks the best of several.  Streaming does not return them.

        ``takes`` > 1 (at most ``max_batch``; not with ``distributed``; needs a ``SpeechLM`` backbone): every utterance
        is generated ``takes`` times from one prefill of its prompt (``generate_batch``'s ``num_return_sequences``:
        the takes share the prompt's KV pages), and only the take with the highest mean ``model`` log-probability over
        its generated tokens (EOS included; ties: the first take) goes through the codec.  Utterances run in chunks of
        ``max_batch // takes``; ``return_logprobs`` returns the kept takes' rows.

        Classifier-free guidance (transformers' ``guidance_scale`` with a negative prompt): ``guidance_scale`` (a number
        or one per utterance, > 0; 1 = off) and ``negative_text`` (a string or one per utterance).  The negative prompt
        is the chat template with the utterance's own reference codes and reference text and ``negative_text`` as the
        input text; None means "", the voice without the words, which steers the draws toward the text.  Each guided
        utterance decodes its negative prompt in a second engine slot, so a chunk or the queue holds fewer of them at
        once.  Not with ``takes`` > 1 (ValueError); ``distributed`` works, every rank guiding its own utterances.

        ``speed`` (a number or one per utterance, in [0.5, 2.0]; > 1 is faster) is the speaking rate: each waveform is
        time-stretched at 24 kHz on the GPU right after the codec (librosa's ``time_stretch``, a phase vocoder: the
        pitch is kept, a waveform of L samples becomes round(L / speed)), before the watermark and any resampling.  A
        list follows its utterances through chunking, the queue, takes (the kept take is stretched) and the sharding
        over ranks.  An utterance at exactly 1.0 is not stretched; with every speed at 1.0 nothing changes.

        ``loudness`` (None, a target in LUFS, or one target or None per utterance; each finite and in [-70, 0], e.g.
        -16 for podcasts and streaming, -23 for EBU R128 broadcast) normalises each waveform on the GPU to that
        ITU-R BS.1770-4 integrated loudness (``neutts_air_b200.loudness``), measured at 24 kHz after the stretch and
        before the watermark and any resampling: the waveform is scaled by 10^((target - L) / 20).  There is no limiter,
        so float32 samples may exceed +-1 (int16 output clips).  A waveform that is silent or shorter than 400 ms has no
        loudness and comes back unchanged; one where the gain moves a 400 ms block across the -70 LUFS absolute gate
        re-measures slightly off its target.  A list follows its utterances through chunking, the queue, takes (the kept
        take is normalised), long-form segments and the sharding over ranks.  With ``loudness=None`` nothing changes.

        ``long_form=True``: a text too long for one prompt is split into segments that fit (``segments``); the
        segments of all texts run as one batch (segment 0 of every text first, then segment 1 of every text that has
        one, and so on; segment j of that order draws from random stream j), each with its text's controls, and each
        text's waveforms are joined after the codec, stretch, watermark and resampler with 10 ms fades at every seam
        and ``pause`` seconds (in [0, 10]) of silence between segments.  A text that fits is one segment and comes back
        as without ``long_form``.  With ``return_logprobs`` a text's rows are its segments' rows, concatenated.  Each
        segment is normalised to its text's ``loudness`` target before the join, so a joined text sits near its target
        but not exactly on it (the fades and pauses change its blocks)."""
        if not (len(texts) == len(ref_codes) == len(ref_texts)):
            raise ValueError("texts, ref_codes and ref_texts must have the same length")
        pause = longform.check_pause(pause, long_form)
        targets = _targets(len(texts), loudness)
        if long_form:
            owners, flat, refs, rts, kw = self._long_form_plan(
                texts, ref_codes, ref_texts, temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p,
                repetition_penalty=repetition_penalty, penalize_prompt=penalize_prompt, min_new_tokens=min_new_tokens,
                exponential_decay_length_penalty=exponential_decay_length_penalty, guidance_scale=guidance_scale,
                negative_text=negative_text, speed=speed, repetition_aware_sampling=repetition_aware_sampling,
                loudness=targets)
            out = self.infer_batch(flat, refs, rts, distributed, return_logprobs=return_logprobs, takes=takes, **kw)
            wavs, lps = out if return_logprobs else (out, None)
            idx = [[j for j, o in enumerate(owners) if o == t] for t in range(len(texts))]
            joined = [longform.join([wavs[j] for j in js], self.sample_rate, pause) for js in idx]
            return (joined, [np.concatenate([lps[j] for j in js]) for js in idx]) if return_logprobs else joined
        speeds = _speeds(len(texts), speed)
        ctl = _controls(len(texts), temperature, top_k, top_p, min_p, repetition_penalty, penalize_prompt, min_new_tokens,
                        exponential_decay_length_penalty, repetition_aware_sampling)
        self._check_ras(ctl)
        ctl = _add_guidance(ctl, len(texts), guidance_scale,
                            self._negatives(len(texts), guidance_scale, negative_text, ref_codes, ref_texts))
        if takes != 1 and "guidance_scale" in ctl:
            raise ValueError("classifier-free guidance generates one take per utterance (takes=1)")
        takes = self._check_takes(takes, distributed)
        if return_logprobs:
            self._check_logprobs(distributed)
        prompts = [self._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, ref_codes, ref_texts)]
        if takes > 1:
            return self._infer_takes(prompts, ctl, takes, return_logprobs, speeds, targets)
        queue = hasattr(self.backbone, "generate_queue")

        def run(idx, slot_base):
            c = _pick(ctl, idx)
            g, neg = c.pop("guidance_scale", 1.0), c.pop("negative_prompt_ids", None)
            return self.infer_from_prompt_ids([prompts[i] for i in idx], slot_base=slot_base, return_logprobs=return_logprobs,
                                              guidance_scale=g, negative_prompt_ids=neg,
                                              speed=1.0 if speeds is None else [speeds[i] for i in idx],
                                              loudness=None if targets is None else [targets[i] for i in idx], **c)

        # chunks of prompts whose slots (two for a guided one) fit the engine; prompt i keeps Philox stream i
        chunks, j = [], 0
        while j < len(prompts):
            k = j + 1
            while k < len(prompts) and self._slots(k + 1 - j, _pick(ctl, range(j, k + 1))) <= self.max_batch:
                k += 1
            chunks.append(range(j, k))
            j = k
        if not distributed:
            if queue and len(chunks) > 1:
                return run(range(len(prompts)), 0)
            out, lps = [], []
            for idx in chunks:
                r = run(idx, idx[0])
                out += r[0] if return_logprobs else r
                lps += r[1] if return_logprobs else []
            return (out, lps) if return_logprobs else out
        from neutts_air_b200 import dist

        mine = dist.shard_indices(len(prompts), [len(p) for p in prompts])
        local = []
        rank = dist.world()[0]
        if queue and self._slots(len(mine), _pick(ctl, mine)) > self.max_batch:
            local = run(mine, rank << 20)
        else:
            for j in range(0, len(mine), self.max_batch):
                local += run(mine[j: j + self.max_batch], (rank << 20) + j)
        out = dist.all_gather_waveforms(local, mine, len(prompts), device=self.codec.device)
        # 16-bit samples are exact in the float32 gather buffer
        return [w.astype(np.int16) for w in out] if self.pcm_format == "int16" else out

    @staticmethod
    def take_chunks(n_utterances: int, takes: int, max_batch: int) -> list:
        """(utterance indices, slot_base) of every chunk ``infer_batch`` runs with ``takes`` > 1: ``max_batch // takes``
        utterances per chunk, slot_base = the chunk's first utterance x takes, so that take j of utterance u draws from
        the Philox stream u * takes + j under one seed whatever the chunking."""
        per = max_batch // takes
        return [(range(j, min(j + per, n_utterances)), j * takes) for j in range(0, n_utterances, per)]

    def _infer_takes(self, prompts, ctl: dict, takes: int, return_logprobs: bool, speeds=None, targets=None):
        out, lps = [], []
        for idx, slot_base in self.take_chunks(len(prompts), takes, self.max_batch):
            r = self.infer_from_prompt_ids([prompts[i] for i in idx], slot_base=slot_base, return_logprobs=return_logprobs,
                                           takes=takes, speed=1.0 if speeds is None else [speeds[i] for i in idx],
                                           loudness=None if targets is None else [targets[i] for i in idx],
                                           **_pick(ctl, idx))
            out += r[0] if return_logprobs else r
            lps += r[1] if return_logprobs else []
        return (out, lps) if return_logprobs else out

    # ------------------------------------------------------------------ long-form synthesis
    def segments(self, text: str, ref_codes, ref_text: str) -> list:
        """The segments ``long_form=True`` synthesises ``text`` in, with the voice (``ref_codes``, ``ref_text``):
        ``[text]`` when it fits whole, else its sentences packed greedily per line (``neutts_air_b200.longform``).  A
        segment fits when the room ``max_context`` leaves after its prompt covers its text at the reference's pace
        (reference codes per reference-text token) with a 1.25 margin; every candidate is measured on the prompt that
        would run.  ValueError when a single word does not fit."""
        codes = ref_codes.tolist() if hasattr(ref_codes, "tolist") else list(ref_codes)
        lens = {}

        def prompt_len(s: str) -> int:
            if s not in lens:
                lens[s] = len(self._apply_chat_template(codes, ref_text, s))
            return lens[s]

        return longform.segment(text, longform.fit_rule(prompt_len, ref_text, len(codes), self.max_context))

    def _long_form_plan(self, texts, ref_codes, ref_texts, **controls):
        """The flattened segments of ``texts`` in round-robin order -> (owning text of each segment, segment texts,
        reference codes, reference texts, controls): every per-text control list becomes one entry per segment,
        scalars stay."""
        segs = [self.segments(t, c, rt) for t, c, rt in zip(texts, ref_codes, ref_texts)]
        order = longform.round_robin([len(s) for s in segs])
        owners = [t for t, _ in order]
        n = len(texts)
        decay = controls.pop("exponential_decay_length_penalty")
        per = per_prompt_decay(n, decay)
        ras = _ras_arg(n, controls.pop("repetition_aware_sampling", None))
        kw = {k: [v[t] for t in owners] if isinstance(v, list) else v for k, v in per_item(n, "text", **controls).items()}
        kw["exponential_decay_length_penalty"] = decay if per[0] is decay else [per[t] for t in owners]
        kw["repetition_aware_sampling"] = [ras[t] for t in owners] if isinstance(ras, list) else ras
        return (owners, [segs[t][k] for t, k in order], [ref_codes[t] for t in owners], [ref_texts[t] for t in owners],
                kw)

    def _long_form_stream(self, texts, ref_codes, ref_texts, pause: float, **controls) -> Generator[list, None, None]:
        """``infer_stream_batch`` with ``long_form=True``: the flattened segments stream through ``_stream_batch`` and
        ``longform.StreamJoin`` turns the rounds into one stream per text.  Planned here, streamed lazily."""
        owners, flat, refs, rts, kw = self._long_form_plan(texts, ref_codes, ref_texts, **controls)
        speeds = _speeds(len(flat), kw.pop("speed"))
        ctl = _controls(len(flat), **kw)
        self._check_ras(ctl)
        prompts = [self._apply_chat_template(c, rt, t) for t, c, rt in zip(flat, refs, rts)]
        ids = [[int(c) for c in (rc.tolist() if hasattr(rc, "tolist") else rc)] for rc in refs]
        seams = longform.StreamJoin(owners, self.sample_rate, pause, np.int16 if self.pcm_format == "int16" else np.float32)

        def run():
            ends = []
            rounds = self._stream_batch(prompts, ids, ctl, speeds, ends=ends)
            try:
                for out in rounds:
                    got = seams.push(out, ends)
                    if any(g is not None for g in got):
                        yield got
            finally:
                rounds.close()   # every KV page back in the pool when the consumer stops early

        return run()

    # ------------------------------------------------------------------ scoring
    def score(self, text: str, ref_codes, ref_text: str, codes, *, include_eos: bool = True) -> np.ndarray:
        """How likely the speech codes ``codes`` are as this model's rendering of ``text`` in the voice of
        (``ref_codes``, ``ref_text``): float32 log-probabilities, one per code and one more for
        ``<|SPEECH_GENERATION_END|>`` when ``include_eos``, each token's log-softmax over the whole vocabulary given
        the prompt and every earlier code, from one prefill pass (``SpeechLM.score``).  No sampling control applies,
        and ``speech_tokens_only`` does not change the scores.  Their negated mean is the finetuning recipe's loss over
        the speech tokens; a low mean flags a transcript that does not match its audio, and ranks takes or clips."""
        return self.score_batch([text], [ref_codes], [ref_text], [codes], include_eos=include_eos)[0]

    def score_batch(self, texts: Sequence[str], ref_codes: Sequence, ref_texts: Sequence[str], codes: Sequence, *,
                    include_eos: bool = True) -> list:
        """``score`` over lists, one entry per utterance; returns a list of float32 arrays."""
        if not (len(texts) == len(ref_codes) == len(ref_texts) == len(codes)):
            raise ValueError("texts, ref_codes, ref_texts and codes must have the same length")
        self._check_score()
        n_codes = self._n_codes()
        conts = []
        for c in codes:
            c = [int(x) for x in (c.tolist() if hasattr(c, "tolist") else c)]
            if not c:
                raise ValueError("codes to score must not be empty")
            if min(c) < 0 or max(c) >= n_codes:
                raise ValueError(f"codes must lie in 0..{n_codes - 1}")
            conts.append(c)
        prompts = [self._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, ref_codes, ref_texts)]
        base = self.speech_base
        eos = [self._tok_id("<|SPEECH_GENERATION_END|>")] if include_eos else []
        return self.score_from_prompt_ids(prompts, [[base + x for x in c] + eos for c in conts])

    def score_from_prompt_ids(self, prompts: Sequence[Sequence[int]], continuations: Sequence[Sequence[int]]) -> list:
        """Hot path only: the log-probability of every id of each continuation after its prompt (host ids in, float32
        arrays out, one value per continuation id)."""
        if len(prompts) != len(continuations):
            raise ValueError("prompts and continuations must have the same length")
        self._check_score()
        if any(len(c) == 0 for c in continuations) or any(len(p) == 0 for p in prompts):
            raise ValueError("prompts and continuations must not be empty")
        seqs = [list(p) + list(c) for p, c in zip(prompts, continuations)]
        out = self.backbone.score(seqs, [len(p) for p in prompts])
        return [np.asarray(o, dtype=np.float32) for o in out]

    def _check_ras(self, ctl: dict) -> None:
        """Repetition-aware sampling needs an engine that runs it (``SpeechLM.set_repetition_aware_sampling``):
        transformers' ``generate`` has no such option, so asking for it elsewhere fails before any generation."""
        if ctl.get("repetition_aware_sampling") is not None and not hasattr(self.backbone, "set_repetition_aware_sampling"):
            raise ValueError("repetition_aware_sampling needs a backbone with set_repetition_aware_sampling "
                             "(neutts_air_b200.SpeechLM)")

    def _check_score(self) -> None:
        """Scoring needs an engine that scores (``SpeechLM.score``)."""
        if not hasattr(self.backbone, "score"):
            raise ValueError("score needs a backbone with score (neutts_air_b200.SpeechLM)")

    @staticmethod
    def _no_takes(takes) -> None:
        if takes != 1:
            raise ValueError("streaming synthesis generates one take per utterance (takes=1)")

    def infer_stream(self, text: str, ref_codes, ref_text: str, *, temperature: float = 1.0, top_k: int = 50,
                     top_p: float = 1.0, min_p: float = 0.0, repetition_penalty: float = 1.0,
                     penalize_prompt: bool = True, takes: int = 1, min_new_tokens: int = 50,
                     exponential_decay_length_penalty=None, guidance_scale=1.0,
                     speed: float = 1.0, long_form: bool = False, pause: float = 0.0,
                     repetition_aware_sampling=None) -> Generator[np.ndarray, None, None]:
        """Streaming synthesis with the reference's window geometry (``neutts/neutts.py:373-465``):
        every 25 new frames (once 5 look-ahead frames exist) the codec re-decodes
        [n - 50 - 1, n + 25 + 5 + 1) and the chunk is cross-faded with triangular weights.  Sampling controls as in
        ``infer_batch``; streaming returns no per-token log-probabilities (``return_logprobs`` is not supported here)
        and generates one take per utterance (``takes`` other than 1 raises ValueError); classifier-free guidance is not
        supported (``guidance_scale`` other than 1 raises ValueError).  ``speed``: speaking rate (``infer_batch``); each
        cross-faded chunk goes through the stretcher's stream, so the chunks concatenate to the stretched stream.
        ``long_form`` and ``pause``: a text longer than the context, in segments (``infer_stream_batch``).  There is
        no ``loudness``: integrated loudness needs the whole utterance before its first sample can be scaled."""
        self._no_takes(takes)
        self._no_guidance(guidance_scale, "streaming synthesis")
        if self._is_quantized_model:  # kept for signature parity; never true on this build
            raise NotImplementedError("GGUF streaming is not part of the H100 build")
        pause = longform.check_pause(pause, long_form)
        if long_form:
            rounds = self._long_form_stream([text], [ref_codes], [ref_text], pause, temperature=temperature, top_k=top_k,
                                            top_p=top_p, min_p=min_p, repetition_penalty=repetition_penalty,
                                            penalize_prompt=penalize_prompt, min_new_tokens=min_new_tokens,
                                            exponential_decay_length_penalty=exponential_decay_length_penalty, speed=speed,
                                            repetition_aware_sampling=repetition_aware_sampling)
            return self._only_text(rounds)
        ctl = _controls(1, temperature, top_k, top_p, min_p, repetition_penalty, penalize_prompt, min_new_tokens,
                        exponential_decay_length_penalty, repetition_aware_sampling)
        self._check_ras(ctl)
        speeds = _speeds(1, speed)
        prompt = self._apply_chat_template(ref_codes, ref_text, text)
        return self._stream(prompt, [int(c) for c in (ref_codes.tolist() if hasattr(ref_codes, "tolist") else ref_codes)], ctl,
                            speeds)

    def infer_stream_batch(self, texts: Sequence[str], ref_codes: Sequence, ref_texts: Sequence[str], *, temperature=1.0,
                           top_k=50, top_p=1.0, min_p=0.0, repetition_penalty=1.0,
                           penalize_prompt=True, takes: int = 1, min_new_tokens=50,
                           exponential_decay_length_penalty=None, guidance_scale=1.0, speed=1.0, long_form: bool = False,
                           pause: float = 0.0, repetition_aware_sampling=None) -> Generator[list, None, None]:
        """Streaming synthesis of many utterances at once (BASELINE.json configs[4]; the reference streams one
        utterance, ``neutts/neutts.py:373-465``).  Every yield is a list with one entry per utterance, as many entries
        as ``texts``: the next audio chunk (float32, cross-faded exactly as in ``infer_stream``) or ``None`` when that
        utterance has nothing new.  The sequences decode in lock-step in ONE persistent-kernel launch per round; the
        windows that are due are gathered on the device from the code history and go through the codec as one batch.

        A list longer than the engine's ``max_batch`` streams as a queue: utterances take the slots in list order, and
        a slot whose utterance has sent its last chunk takes the next waiting one while the others keep decoding, so
        a late utterance starts as soon as a slot frees up instead of after whole chunks of the list.  Utterance i
        draws from random stream i, the stream it has when the list fits into the slots, and its sampling controls
        (scalars or one value per utterance) follow it into whichever slot it takes.  The queue needs a backbone with
        ``prefill_slots`` (ValueError otherwise), and every KV page is given back when the generator ends or is
        closed early.

        Streaming returns no per-token log-probabilities (``infer_batch``'s ``return_logprobs``) and generates one take
        per utterance (``takes`` other than 1 raises ValueError); ``guidance_scale`` other than 1 raises ValueError.
        ``speed`` (a number or one per utterance): speaking rate, as in ``infer_batch``; it follows its utterance into
        whichever slot it takes.  Chunks go codec -> cross-fade -> stretch -> resample, and concatenate to the stretched
        stream.  Streams take no ``loudness`` target: integrated loudness needs the whole utterance before its first
        sample can be scaled (normalise the finished waveforms with ``neutts_air_b200.loudness.normalize`` instead).

        ``long_form=True``: the texts are split and their segments ordered as in ``infer_batch``, and all segments stream
        as one queue; each text still gets one entry per yield.  A text plays its segments in order: chunks of a later
        segment, decoding in another slot already, are held until every earlier segment of the text has ended, and each
        segment holds back its last 10 ms until its next chunk or its end, for the seam's fade-out and ``pause``.  The
        chunks of a text concatenate to ``infer_batch``'s join of its segments' streams."""
        self._no_takes(takes)
        self._no_guidance(guidance_scale, "streaming synthesis")
        if not (len(texts) == len(ref_codes) == len(ref_texts)):
            raise ValueError("texts, ref_codes and ref_texts must have the same length")
        pause = longform.check_pause(pause, long_form)
        if long_form:
            return self._long_form_stream(texts, ref_codes, ref_texts, pause, temperature=temperature, top_k=top_k,
                                          top_p=top_p, min_p=min_p, repetition_penalty=repetition_penalty,
                                          penalize_prompt=penalize_prompt, min_new_tokens=min_new_tokens,
                                          exponential_decay_length_penalty=exponential_decay_length_penalty, speed=speed,
                                          repetition_aware_sampling=repetition_aware_sampling)
        self._stream_slots(len(texts))
        ctl = _controls(len(texts), temperature, top_k, top_p, min_p, repetition_penalty, penalize_prompt, min_new_tokens,
                        exponential_decay_length_penalty, repetition_aware_sampling)
        self._check_ras(ctl)
        prompts = [self._apply_chat_template(c, rt, t) for t, c, rt in zip(texts, ref_codes, ref_texts)]
        refs = [[int(c) for c in (rc.tolist() if hasattr(rc, "tolist") else rc)] for rc in ref_codes]
        return self._stream_batch(prompts, refs, ctl, _speeds(len(texts), speed))

    @staticmethod
    def _only_text(rounds) -> Generator[np.ndarray, None, None]:
        """The chunks of a one-text long-form stream (its rounds yield only when the text has new audio)."""
        try:
            for out in rounds:
                yield out[0]
        finally:
            rounds.close()

    def _stream(self, prompt, ref_codes, ctl: dict | None = None, speeds=None) -> Generator[np.ndarray, None, None]:
        for out in self._stream_batch([prompt], [list(ref_codes)], ctl, speeds):
            if out[0] is not None:
                yield out[0]

    def _stream_slots(self, n: int) -> int:
        """Slots that stream n utterances: the engine's ``max_batch`` (n when it has none).  More utterances than slots
        run as a queue, which needs an engine that refills single slots (``prefill_slots``)."""
        slots = getattr(self.backbone, "max_batch", n)
        if n > slots and not hasattr(self.backbone, "prefill_slots"):
            raise ValueError(f"streaming {n} utterances through {slots} slots needs a backbone with prefill_slots "
                             "(neutts_air_b200.SpeechLM)")
        return min(n, slots)

    def _stream_batch(self, prompts, refs, ctl: dict | None = None, speeds=None, ends: list | None = None
                      ) -> Generator[list, None, None]:
        """Window geometry of the reference (``neutts/neutts.py:87-91,401-421,443-465``): once F + LA undecoded frames
        exist, the codec decodes [n_dec - LB - OV, n_dec + F + LA) and the slice [n_dec - OV, n_dec + F + OV) is
        cross-faded at stride F * hop; a ragged tail closes the stream.  ``streaming_frames_per_chunk`` may be set to
        50 for the "codec every 50 tokens" configuration BASELINE.json names.

        State per slot: the code history (reference codes, then generated ones) lives ON THE DEVICE next to the
        engine's ``out_tokens``; a round is  absorb the new tokens into the history with device ops -> one small D2H
        read of (n_generated, done, history length) -> batched codec call -> yield -> refill -> decode(k steps, all
        slots).  Cross-fade state and decode position belong to the utterance.

        More utterances than the engine's ``max_batch`` run as a queue on its S slots: utterance i is admitted FIFO and
        draws from Philox stream i (the first S through ``prefill``, later ones through ``prefill_slots``); a slot is
        refilled once its utterance's tail has been decoded from its history row.  Every KV page is back in the pool
        when the generator ends, closed early included.

        ``ends``: None, or a list that holds, at every yield, the utterances whose stream ends with it; a round in which
        one ends is then yielded even when it has no new audio."""
        hop, F, LA, LB, OV = self.hop_length, self.streaming_frames_per_chunk, self.streaming_lookforward, \
            self.streaming_lookback, self.streaming_overlap_frames
        eos = self._tok_id("<|SPEECH_GENERATION_END|>")
        seed = self.seed if self.seed is not None else int(torch.randint(0, 2**31 - 1, (1,)).item())
        lm = self.backbone
        if not hasattr(lm, "prefill"):
            raise NotImplementedError("Streaming needs the neutts_air_b200.SpeechLM backbone")
        N = len(prompts)
        B = self._stream_slots(N)
        queue = N > B
        limits = [min(self.max_context - len(p), lm.max_new) for p in prompts]
        if min(limits) < 1:
            raise ValueError("prompt already at max_length")
        limit = max(limits)
        st = resolve_settings(lm, N, vocab_range=self._speech_range(), max_new=limit,
                              **(ctl if ctl is not None else CONTROL_DEFAULTS))
        top_k, temp, floor = st.top_k, st.temperature, st.min_new_tokens
        if queue or min(limits) < limit:   # a refill writes its newcomer's cap into the per-slot limits
            sp = lm.sampling(eos, floor, limit, top_k, temp, seed, limits=limits[:B])
        else:
            sp = lm.sampling(eos, floor, limit, top_k, temp, seed)
        st.apply(lm, B)   # before the prefill, on the same stream
        dev = lm.out_tokens.device
        cap = max(len(r) for r in refs) + limit
        hist = torch.zeros(B, cap + 1, dtype=torch.long, device=dev)          # column `cap` is a scratch slot for masked writes
        hlen = torch.zeros(B, dtype=torch.long, device=dev)
        absorbed = torch.zeros(B, dtype=torch.long, device=dev)                # generated tokens already looked at
        n_dec = [len(r) for r in refs]
        fades = [_CrossFade(self.streaming_stride_samples) for _ in range(N)]
        tail_done = [False] * N
        occ = list(range(B))   # utterance held by each slot; None once its tail is out and nobody waits
        nxt = B                # next utterance to admit
        rs = self._output_resampler()
        ts = self._time_stretch() if speeds is not None else None

        def at_speed(out, ends=()):
            """the round's cross-faded chunks at each utterance's speaking rate: one push over the slots whose utterance
            is not at 1.0 and has new audio or ends; a chunk whose samples are all still held becomes None"""
            if ts is None:
                return out
            us = [u for u in range(N) if speeds[u] != 1.0 and (out[u] is not None or u in ends)]
            if not us:
                return out
            slot = {occ[b]: b for b in range(B) if occ[b] is not None}
            got = ts.push([slot[u] for u in us], [np.zeros(0, np.float32) if out[u] is None else out[u] for u in us],
                          [speeds[u] for u in us], [u in ends for u in us])
            res = list(out)
            for u, y in zip(us, got):
                res[u] = y if y.size else None
            return res

        def at_rate(out, ends=()):
            """the round's 24 kHz chunks at ``sample_rate``: one push over the slots with new audio or an ending stream
            (utterances ``ends``); a chunk whose samples are all still held becomes None"""
            if rs is None:
                return out
            us = [u for u in range(N) if out[u] is not None or u in ends]
            slot = {occ[b]: b for b in range(B) if occ[b] is not None}
            got = rs.push([slot[u] for u in us], [np.zeros(0, np.float32) if out[u] is None else out[u] for u in us],
                          [u in ends for u in us])
            res = [None] * N
            for u, y in zip(us, got):
                res[u] = y if y.size else None
            return res

        def seat(slots, idx):
            """history rows of ``slots`` := the reference codes of utterances ``idx``, nothing absorbed yet"""
            rows = torch.zeros(len(slots), max(len(refs[i]) for i in idx), dtype=torch.long)
            for r, i in enumerate(idx):
                rows[r, : len(refs[i])] = torch.as_tensor(refs[i], dtype=torch.long)
            sl = torch.tensor(slots, device=dev)
            hist[sl, : rows.shape[1]] = rows.to(dev)
            hlen[sl] = torch.tensor([len(refs[i]) for i in idx], device=dev)
            absorbed[sl] = 0
            if rs is not None:
                rs.reset(slots)
            if ts is not None:
                ts.reset(slots)

        def absorb(lo: int, hi: int):
            """tokens [lo, hi) of every slot -> history (non-speech ids dropped, as the reference's regex does)"""
            hi = min(hi, lm.out_tokens.shape[1])   # a slot that stopped at max_new may lead the round's bound
            if hi <= lo:
                return
            ngen = lm.n_generated[:B].long()
            seg, ok = self._ids_to_codes_masked(lm.out_tokens[:B, lo:hi].long())
            cols = torch.arange(lo, hi, device=dev)[None, :]
            valid = (cols >= absorbed[:, None]) & (cols < ngen[:, None]) & ok
            pos = hlen[:, None] + torch.cumsum(valid, 1) - 1
            hist.scatter_(1, torch.where(valid, pos, torch.full_like(pos, cap)), seg)
            hlen.add_(valid.sum(1))
            absorbed.copy_(torch.minimum(ngen, torch.full_like(ngen, hi)))

        def decode_windows(jobs):
            """jobs: (slot, t0, t1, s0, s1 | None).  Same-length windows share one codec call."""
            out = {}
            by_len = {}
            for j in jobs:
                by_len.setdefault(j[2] - j[1], []).append(j)
            cbatch = max(1, getattr(self.codec, "max_batch", 1))
            for n, grp in by_len.items():
                for g0 in range(0, len(grp), cbatch):
                    g = grp[g0: g0 + cbatch]
                    rows = torch.tensor([j[0] for j in g], device=dev)
                    idx = torch.tensor([j[1] for j in g], device=dev)[:, None] + torch.arange(n, device=dev)[None, :]
                    codes = hist[rows[:, None], idx][:, None, :]
                    with torch.no_grad():
                        pcm = self.codec.decode_code(codes.to(self.codec.device))
                    pcm = pcm[:, 0, :].cpu().numpy()
                    for r, (b, t0, t1, s0, s1) in enumerate(g):
                        wav = self._watermark(pcm[r])
                        out.setdefault(b, []).append(wav[max(s0, 0):] if s1 is None else wav[s0:s1])
            return out

        seat(list(range(B)), list(range(B)))
        try:
            lm.prefill(prompts[:B], sp)             # samples the first token of every slot
            lo, hi = 0, 1
            while True:
                absorb(lo, hi)
                rd = torch.stack((lm.n_generated[:B].long(), lm.done[:B].long(), hlen)).cpu()   # the round's one D2H read
                ngen_h, done_h, hlen_h = rd[0].tolist(), rd[1].tolist(), rd[2].tolist()
                held = [b for b in range(B) if occ[b] is not None]
                finished = {b: bool(done_h[b]) or ngen_h[b] >= limits[occ[b]] for b in held}
                jobs = []
                for b in held:
                    u = occ[b]
                    while hlen_h[b] - n_dec[u] >= F + LA:
                        t0 = max(n_dec[u] - LB - OV, 0)
                        # the reference slices up to n_dec + F + LA + OV, but tokens arrive one at a time there, so
                        # its cache never holds more than n_dec + F + LA entries when a chunk fires (:401-415)
                        t1 = n_dec[u] + F + LA
                        s0 = (n_dec[u] - t0) * hop
                        jobs.append((b, t0, t1, s0, s0 + (F + 2 * OV) * hop))
                        n_dec[u] += F
                out = [None] * N
                if jobs:
                    for b, wavs in decode_windows(jobs).items():
                        out[occ[b]] = np.concatenate([fades[occ[b]].push(w) for w in wavs])
                # ragged tail of an utterance that finished (neutts/neutts.py:443-465), once its regular chunks are out
                tails, ending = [], []
                all_finished = nxt == N and all(finished.values())
                if ends is not None:
                    ends.clear()
                for b in held:
                    u = occ[b]
                    if finished[b] and not tail_done[u] and (all_finished or out[u] is None):
                        tail_done[u] = True
                        ending.append(u)
                        n = hlen_h[b]
                        if n > n_dec[u]:
                            rem = n - n_dec[u]
                            t0 = max(n - (LB + OV + rem), 0)
                            tails.append((b, t0, n, (n - t0 - rem - OV) * hop, None))
                        elif fades[u].acc.shape[0]:
                            flush = fades[u].push(np.zeros(0, np.float32), final=True)
                            out[u] = flush if out[u] is None else np.concatenate((out[u], flush))
                if all_finished and any(o is not None for o in out) and tails:
                    first = at_rate(at_speed(out))   # regular chunks first: a tail is its own yield, as in the reference
                    if any(o is not None for o in first):
                        yield first
                    out = [None] * N
                if tails:
                    for b, wavs in decode_windows(tails).items():
                        t = fades[occ[b]].push(wavs[0], final=True)
                        out[occ[b]] = t if out[occ[b]] is None else np.concatenate((out[occ[b]], t))
                out = at_rate(at_speed(out, ending), ending)
                if ends is not None:
                    ends += ending
                if any(o is not None for o in out) or (ends is not None and ending):
                    yield out
                if all_finished:
                    break
                # refill every slot whose utterance's tail is out (its history row has been read), FIFO
                new = []
                for b in held:
                    if tail_done[occ[b]]:
                        occ[b] = None
                        if nxt < N:
                            occ[b], nxt = nxt, nxt + 1
                            new.append(b)
                if new:
                    idx = [occ[b] for b in new]
                    st.admit(lm, new, idx)   # before their prefill, on the same stream
                    seat(new, idx)
                    lm.prefill_slots(new, [prompts[i] for i in idx], sp, stream_ids=idx, limits=[limits[i] for i in idx])
                    for b, i in zip(new, idx):
                        ngen_h[b], hlen_h[b], finished[b] = 1, len(refs[i]), False
                # decode just enough steps for the next chunk of the most advanced unfinished stream to fire (non-speech
                # ids may make it take another pass), and no further than the earliest cap-driven completion; finished
                # slots idle inside the kernel.  A newcomer's first token is not in its history yet.
                live = [b for b in range(B) if occ[b] is not None and not finished[b]]
                steps = 0
                if live and not any(limits[occ[b]] <= 1 for b in new):   # a cap of 1 ends inside the prefill: read first
                    need = min(F + LA - (hlen_h[b] + (b in new) - n_dec[occ[b]]) for b in live)
                    room = min(limits[occ[b]] - ngen_h[b] for b in live)
                    steps = max(1, min(need, room))
                    lm.decode(steps, sp)
                # every slot's tokens up to its last read count are in its history; a newcomer's start at 0
                lo = min((0 if b in new else ngen_h[b] for b in live), default=0)
                hi = max(ngen_h) + steps
        finally:
            if queue:
                lm.release_pages()   # also when the consumer stops early (generator close)
            if ts is not None:
                ts.reset(range(B))

    def encode_reference(self, ref_audio_path):
        """wav -> NeuCodec codes (``neutts/neutts.py:266-271``).  The encoder is outside the hot path; this
        delegates to ``codec.encode_code`` (the real ``neucodec`` when installed) or loads pre-encoded
        ``.pt`` / ``.npy`` codes saved by ``examples/encode_reference.py``."""
        p = Path(ref_audio_path)
        if p.suffix == ".pt":
            return torch.load(p)
        if p.suffix == ".npy":
            return torch.from_numpy(np.load(p))
        try:
            import librosa

            wav, _ = librosa.load(ref_audio_path, sr=16000, mono=True)
            wav_tensor = torch.from_numpy(wav).float().unsqueeze(0).unsqueeze(0)
            with torch.no_grad():
                return self.codec.encode_code(audio_or_path=wav_tensor).squeeze(0).squeeze(0)
        except ImportError as e:
            # neither librosa nor the neucodec encoder is installed: use the pre-encoded codes that sit next to
            # the audio (the reference ships samples/dave.wav + samples/dave.pt, examples/README.md:15-23)
            for ext in (".pt", ".npy"):
                q = p.with_suffix(ext)
                if q.exists():
                    warnings.warn(f"{e}; using the pre-encoded reference codes {q.name}")
                    return torch.load(q) if ext == ".pt" else torch.from_numpy(np.load(q))
            raise ImportError(f"cannot encode {p.name}: {e} (and no pre-encoded {p.stem}.pt / .npy next to it)") from e
