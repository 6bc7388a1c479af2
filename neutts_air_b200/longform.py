"""Long-form synthesis on the host: split a text that outgrows the LM context into segments that fit, and join the
segments' waveforms (whole, or as streams) into one per text.

Every function here is pure host code.  The facade (``NeuTTS.segments`` and ``long_form=True``) supplies the prompt
lengths; the segments themselves run through the existing batched, queued and streaming paths.

The fit rule is calibrated by the voice's own pace: ``K = len(ref_codes) / T_ref`` reference frames per input token,
where ``T_ref`` is the number of prompt tokens the reference text adds.  A segment whose prompt is ``P`` tokens long,
``T`` of them its own text, fits when ``max_context - P >= ceil(MARGIN * K * T)``: the room left for generation covers
the segment at the reference's pace with ``MARGIN`` to spare.
"""
from __future__ import annotations

import math
import re
from fractions import Fraction
from typing import Callable, Sequence

import numpy as np

MARGIN = 1.25          # room for a segment spoken slower than the reference (not yet measured on a real checkpoint)
FADE_S = 0.010         # length of each seam's fade-in and fade-out, in seconds
MAX_PAUSE_S = 10.0

ABBREVIATIONS = frozenset({"mr", "mrs", "ms", "dr", "prof", "st", "jr", "sr", "vs", "etc", "e.g", "i.e", "no"})
_END = re.compile(r"[.!?…]+[\"'”’)\]]*(?=\s)")
_WORD = re.compile(r"\w(?:[\w.]*\w)?$")
_CLAUSE = re.compile(r"(?<=[,;:—–])\s+")


# ------------------------------------------------------------------------------------------------- segmentation
def _abbreviation(before: str) -> bool:
    """Whether a period after ``before`` belongs to a single letter or an abbreviation rather than ending a sentence."""
    m = _WORD.search(before)
    if m is None:
        return False
    w = m.group(0)
    return (len(w) == 1 and w.isalpha()) or w.lower() in ABBREVIATIONS


def split_sentences(text: str) -> list:
    """The sentences of ``text``, stripped, empty ones dropped.  A line break always ends one; inside a line a run of
    ``. ! ? …`` and any closing ``" ' ” ’ ) ]`` ends one when whitespace follows, except a lone period after a single
    letter or an abbreviation of ``ABBREVIATIONS`` (case ignored)."""
    out = []
    for line in text.splitlines():
        start = 0
        for m in _END.finditer(line):
            if m.group(0).rstrip("\"'”’)]") == "." and _abbreviation(line[:m.start()]):
                continue
            out.append(line[start:m.end()])
            start = m.end()
        out.append(line[start:])
    return [s for s in (p.strip() for p in out) if s]


def fit_rule(prompt_len: Callable[[str], int], ref_text: str, n_ref: int, max_context: int) -> Callable[[str], bool]:
    """``fits(text)``: whether the prompt with input ``text`` leaves room for its speech at the reference's pace.
    ``prompt_len(text)`` is the length of the prompt whose input text is ``text``; ``n_ref`` the number of reference
    codes.  Exact arithmetic, so a segment on the boundary is decided the same way everywhere."""
    p0 = prompt_len("")
    t_ref = prompt_len(ref_text) - p0
    if t_ref <= 0:
        raise ValueError("long-form synthesis needs a reference text: its length against the reference codes sets the "
                         "pace a segment is fitted to")
    k = Fraction(MARGIN) * n_ref / t_ref

    def fits(text: str) -> bool:
        p = prompt_len(text)
        return max_context - p >= math.ceil(k * (p - p0))

    return fits


def _pack(pieces: Sequence[str], fits: Callable[[str], bool]) -> list:
    """Greedy: consecutive pieces joined with one space while the joined text still fits; each piece fits alone."""
    out = []
    for s in pieces:
        if out and fits(out[-1] + " " + s):
            out[-1] += " " + s
        else:
            out.append(s)
    return out


def _cut(sentence: str, fits: Callable[[str], bool]) -> list:
    """The pieces of a sentence too long to fit: its clauses (cut after ``, ; : — –`` followed by whitespace), and
    the words of a clause too long to fit.  ValueError for a word that does not fit alone."""
    pieces = []
    for clause in _CLAUSE.split(sentence):
        if fits(clause):
            pieces.append(clause)
            continue
        for word in clause.split():
            if not fits(word):
                raise ValueError(f"the word {word!r} does not fit into the context: the reference leaves no room for it "
                                 "(use a shorter reference)")
            pieces.append(word)
    return pieces


def plan_segments(sentences: Sequence[str], fits: Callable[[str], bool]) -> list:
    """Segments of consecutive ``sentences`` (of one line): greedy, joined with one space while the joined text fits;
    a sentence that does not fit alone is cut at clause punctuation, then at whitespace, and its pieces are packed
    greedily again.  ``fits`` is asked once per candidate."""
    pieces = []
    for s in sentences:
        pieces += [s] if fits(s) else _cut(s, fits)
    return _pack(pieces, fits)


def segment(text: str, fits: Callable[[str], bool]) -> list:
    """The segments of ``text``: ``[text]`` itself when it fits whole, else ``plan_segments`` over each line's
    sentences (a line break always ends a segment)."""
    if fits(text):
        return [text]
    out = []
    for line in text.splitlines():
        out += plan_segments(split_sentences(line), fits)
    if not out:
        raise ValueError("the reference leaves no room in the context for any text")
    return out


def round_robin(counts: Sequence[int]) -> list:
    """(text, segment) of every segment, segment 0 of every text first, then segment 1 of every text that has one,
    and so on.  Position j of this list is utterance j of the flattened batch."""
    return [(t, k) for k in range(max(counts, default=0)) for t in range(len(counts)) if k < counts[t]]


# ------------------------------------------------------------------------------------------------- seams
def check_pause(pause, long_form: bool) -> float:
    """``pause``: seconds of silence between segments, a finite number in [0, MAX_PAUSE_S]; non-zero needs
    ``long_form``."""
    if isinstance(pause, bool) or not isinstance(pause, (int, float, np.integer, np.floating)):
        raise ValueError(f"pause {pause!r} must be a number of seconds")
    p = float(pause)
    if not (math.isfinite(p) and 0.0 <= p <= MAX_PAUSE_S):
        raise ValueError(f"pause {pause} must be finite and in [0, {MAX_PAUSE_S:g}] seconds")
    if p != 0.0 and not long_form:
        raise ValueError("pause separates the segments of long-form synthesis: it needs long_form=True")
    return p


def fade_window(sample_rate: int) -> np.ndarray:
    """The seam's fade-in, float32: ``w(i) = sin^2(pi (i + 0.5) / (2 Fd))`` for i < Fd = round(FADE_S * rate) (the
    fade-out is its reverse, so a fade-out overlapping the next fade-in sums to one)."""
    fd = round(FADE_S * sample_rate)
    return (np.sin(np.pi * (np.arange(fd) + 0.5) / (2 * fd)) ** 2).astype(np.float32)


def _pcm(y: np.ndarray, dtype) -> np.ndarray:
    """float32 samples -> the output format (int16: rounded half to even; the faded samples never leave the range)."""
    return np.rint(y).astype(np.int16) if dtype == np.int16 else y


def join(waves: Sequence[np.ndarray], sample_rate: int, pause: float = 0.0) -> np.ndarray:
    """One text's segment waveforms (float32 or int16, at ``sample_rate``) -> one waveform.  Sample i of segment j (of
    L) is multiplied in float32 by w(i) when j > 0 and i < Fd, then by w(L - 1 - i) when j is not the last and
    L - 1 - i < Fd (``fade_window``); int16 is rounded back half to even.  round(pause * rate) zeros go between
    segments.  A single segment comes back untouched."""
    if len(waves) == 1:
        return waves[0]
    dtype = waves[0].dtype
    w = fade_window(sample_rate)
    gap = np.zeros(round(pause * sample_rate), dtype)
    parts = []
    for j, x in enumerate(waves):
        y = x.astype(np.float32)
        n = min(len(w), len(y))
        if j > 0:
            y[:n] *= w[:n]
        if j < len(waves) - 1:
            y[len(y) - n:] *= w[:n][::-1]
        parts.append(_pcm(y, dtype))
        if j < len(waves) - 1:
            parts.append(gap)
    return np.concatenate(parts)


class StreamJoin:
    """Re-sequences the streams of the flattened segments into one stream per text, with ``join``'s seams.

    ``push(chunks, ended)`` takes one round of the segment streams (one entry per segment, a chunk or None) and the
    segments whose stream ended with that round, and returns one entry per text (its new audio, or None).  A text
    plays its segments in order: chunks of a later segment, decoding in another slot already, are held until every
    earlier segment of the text has ended.  A segment with a successor holds back its last Fd samples until its next
    chunk or its end, where they get the fade-out and the pause follows; the fade-in goes by sample index from the
    segment's start.  A text of one segment passes its chunks through untouched."""

    def __init__(self, owners: Sequence[int], sample_rate: int, pause: float, dtype):
        self.owners = list(owners)
        n = max(self.owners) + 1
        self.segs = [[j for j, o in enumerate(self.owners) if o == t] for t in range(n)]
        self.w = fade_window(sample_rate)
        self.gap = np.zeros(round(pause * sample_rate), dtype)
        self.dtype = dtype
        self.cur = [0] * n                                     # index into segs[t] of the segment now playing
        self.pos = [0] * n                                     # samples of that segment seen so far
        self.held = [np.zeros(0, np.float32) for _ in range(n)]  # its last samples, awaiting the fade-out
        self.early = {}                                        # segment -> chunks that came before its turn
        self.ended = set()

    def _play(self, t: int, x: np.ndarray) -> np.ndarray:
        k, segs = self.cur[t], self.segs[t]
        if len(segs) == 1:
            return x
        y, fd, p = x, len(self.w), self.pos[t]
        if k > 0 and p < fd:
            y = x.astype(np.float32)
            n = min(fd - p, len(y))
            y[:n] *= self.w[p:p + n]
        self.pos[t] += len(x)
        if k == len(segs) - 1:
            return _pcm(y, self.dtype) if y is not x else x
        buf = np.concatenate((self.held[t], y.astype(np.float32)))
        cut = max(len(buf) - fd, 0)
        self.held[t] = buf[cut:]
        return _pcm(buf[:cut], self.dtype)

    def _finish(self, t: int) -> list:
        """The current segment of text t has ended: its faded-out tail and the pause, then the chunks its successor
        already sent (and so on while successors have ended too)."""
        out, segs = [], self.segs[t]
        while self.cur[t] < len(segs) and segs[self.cur[t]] in self.ended:
            if self.cur[t] < len(segs) - 1:
                h = self.held[t]
                out += [_pcm(h * self.w[:len(h)][::-1], self.dtype), self.gap]
            self.cur[t] += 1
            self.pos[t] = 0
            self.held[t] = np.zeros(0, np.float32)
            if self.cur[t] < len(segs):
                out += [self._play(t, x) for x in self.early.pop(segs[self.cur[t]], [])]
        return out

    def push(self, chunks: Sequence, ended=()) -> list:
        outs = [[] for _ in self.segs]
        for j, x in enumerate(chunks):
            if x is None:
                continue
            t = self.owners[j]
            if self.segs[t][self.cur[t]] == j:
                outs[t].append(self._play(t, x))
            else:
                self.early.setdefault(j, []).append(x)
        self.ended.update(ended)
        for t in {self.owners[j] for j in ended}:
            outs[t] += self._finish(t)
        return [None if not sum(len(x) for x in o) else o[0] if len(o) == 1 else np.concatenate(o) for o in outs]
