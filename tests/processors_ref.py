"""The references the speech-LM logits-processor tests compare the kernels with: transformers' processors on one fp32
row (repetition penalty, EOS length decay), float64 log-probabilities, bit-exact comparison, and the forced tokens that
keep a row of the logit-programmable model (``sampler_ref.py``) on its pattern."""
from __future__ import annotations

import math

import numpy as np
import torch

from tests.sampler_ref import fp32_logits

# Worst errors measured on one H100 80GB HBM3 over test_gpu_logprobs.py (DESIGN.md §4, per-token log-probabilities),
# and the bars: |model - float64|, |sampled - float64|, |exp(sampled) - kept probability|
LOGPROB_BARS = {"model": 5e-5, "sampled": 2e-5, "prob": 4e-7}


def hf_penalty(logits_row, prompt, gen, penalty: float, include: bool):
    """transformers' RepetitionPenaltyLogitsProcessor on one fp32 logits row (torch, CPU)."""
    x = torch.from_numpy(np.asarray(logits_row, dtype=np.float32).copy())[None]
    if penalty == 1.0:
        return x[0].numpy()
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor

    ids = torch.tensor([int(t) for t in list(prompt) + list(gen)], dtype=torch.long)[None]
    proc = RepetitionPenaltyLogitsProcessor(float(np.float32(penalty)), prompt_ignore_length=None if include else len(prompt))
    return proc(ids, x)[0].numpy()


def hf_chain(row, prompt, gen, n, penalty=1.0, decay=None, eos=None, include=True):
    """transformers' RepetitionPenaltyLogitsProcessor then ExponentialDecayLengthPenalty (EOS id ``eos``) on one fp32
    logits row (torch, CPU): the scores the engine stores.  n: tokens generated before this draw; gen: those tokens;
    include: whether the prompt counts in the penalty's history."""
    from transformers.generation.logits_process import ExponentialDecayLengthPenalty, RepetitionPenaltyLogitsProcessor

    x = torch.from_numpy(np.asarray(row, dtype=np.float32).copy())[None]
    ids = torch.tensor([int(t) for t in list(prompt) + list(gen)][: len(prompt) + n], dtype=torch.long)
    ids = torch.cat((ids, torch.zeros(len(prompt) + n - ids.numel(), dtype=torch.long)))[None]
    if penalty != 1.0:
        x = RepetitionPenaltyLogitsProcessor(float(np.float32(penalty)),
                                             prompt_ignore_length=None if include else len(prompt))(ids, x)
    if decay is not None and decay[1] != 1.0:
        x = ExponentialDecayLengthPenalty(decay, eos, len(prompt))(ids, x)
    return x[0].numpy()


def bits_equal(a, b) -> bool:
    return np.array_equal(np.asarray(a, dtype=np.float32).view(np.uint32), np.asarray(b, dtype=np.float32).view(np.uint32))


def ranked(m, name):
    """The ids a pattern owns (EOS excluded), by fp32 logit descending: forced tokens that keep a row on its pattern."""
    lg = fp32_logits(m, name)
    ids = m.owned[name]
    ids = ids[ids != m.eos]
    return ids[np.lexsort((ids, -lg[ids].astype(np.float64)))]


def lse64(x) -> float:
    x = np.asarray(x, dtype=np.float64)
    m = x.max()
    return float(m + np.log(np.exp(x - m).sum())) if m > -np.inf else -math.inf


def model_ref(row, tok: int, eos: int, masked: bool) -> float:
    """float64 log-softmax of ``tok`` over the processed logits row (EOS left out while masked)."""
    s = np.asarray(row, dtype=np.float64).copy()
    if masked:
        s[eos] = -np.inf
    return float(s[tok] - lse64(s)) if s[tok] > -np.inf else -math.inf


def sampled_ref(row, ids, tok: int, temperature: float) -> float:
    """float64 log-probability of ``tok`` in the kept window ``ids`` (processed scores fp32(logit * fp32(1 / T)))."""
    ids = [int(i) for i in ids if i >= 0]
    if tok not in ids:
        return -math.inf
    sc = (np.asarray(row, dtype=np.float32)[ids] * (np.float32(1) / np.float32(temperature))).astype(np.float64)
    return float(sc[ids.index(tok)] - lse64(sc))
