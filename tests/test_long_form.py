"""CPU: long-form synthesis (neutts_air_b200/longform.py and ``long_form=True`` on the facade) with the fakes: sentence
splitting, the fit rule, greedy packing, the seams of whole waveforms and of streams, argument checks, and that the
defaults leave every backbone call as it was."""
import collections
import math
import warnings

import numpy as np
import pytest
import torch

from neutts_air_b200 import longform as LF
from tests.fakes import FakeBatchStreamLM, FakeCodec, FakePhonemizer, KwBackbone, RampCodec, _facade, _tts


# ------------------------------------------------------------------------------------------------- sentences
@pytest.mark.parametrize("text, want", [
    ("One. Two! Three? Four… Five", ["One.", "Two!", "Three?", "Four…", "Five"]),
    ("Wait... what?! Really?!? yes", ["Wait...", "what?!", "Really?!?", "yes"]),
    ('He said "stop." Then left. (Quietly.) [Done!] ’Twas “so.” End',
     ['He said "stop."', "Then left.", "(Quietly.)", "[Done!]", "’Twas “so.”", "End"]),
    ("Mr. and Mrs. Smith met Dr. Who, Prof. X and St. John Jr. and Sr. vs. them etc. and more. Next",
     ["Mr. and Mrs. Smith met Dr. Who, Prof. X and St. John Jr. and Sr. vs. them etc. and more.", "Next"]),
    ("MR. BIG, ms. Jones; e.g. this, i.e. that, No. 5 is here. Next", ["MR. BIG, ms. Jones; e.g. this, i.e. that, No. 5 is here.", "Next"]),
    ("Plan A. B is next. J. R. R. Tolkien wrote. 1. Not a letter", ["Plan A. B is next.", "J. R. R. Tolkien wrote.", "1.", "Not a letter"]),
    ("a.b.c is a name.Really? No space after the period", ["a.b.c is a name.Really?", "No space after the period"]),
    ("Line one\nline two. Still two\r\n\n  \nlast line  ", ["Line one", "line two.", "Still two", "last line"]),
    ("  \n\n . \n", ["."]),
    ("", []),
    ("Dr. Mr.\nSt.", ["Dr. Mr.", "St."]),
])
def test_split_sentences(text, want):
    assert LF.split_sentences(text) == want


# ------------------------------------------------------------------------------------------------- fit rule
def _lens(p0, per_char=1):
    """prompt_len of a prompt whose input text adds ``per_char`` tokens per character to ``p0``."""
    return lambda s: p0 + per_char * len(s)


def test_fit_rule_on_hand_computed_lengths():
    # T_ref = 10, 40 codes: K = 4, 1.25 K = 5.  P = 300 + T: fits iff 360 - 300 - T >= 5 T, i.e. T <= 10
    fits = LF.fit_rule(_lens(300), "r" * 10, 40, 360)
    assert fits("x" * 10) and not fits("x" * 11) and fits("")
    # 41 codes: 1.25 K = 5.125; T = 9 needs ceil(46.125) = 47 <= 51, T = 10 needs ceil(51.25) = 52 > 50
    fits = LF.fit_rule(_lens(300), "r" * 10, 41, 360)
    assert fits("x" * 9) and not fits("x" * 10)
    # exact arithmetic on the boundary: 1.25 * 8 / 10 * T = T exactly, fits iff 2 T <= room
    fits = LF.fit_rule(_lens(100), "r" * 10, 8, 100 + 2 * 7)
    assert fits("x" * 7) and not fits("x" * 8)
    # two tokens per character: T_ref = 20, K = 2, 1.25 K = 2.5, T = 2 len; 60 - 2 len >= ceil(5 len) -> len <= 8
    fits = LF.fit_rule(_lens(500, 2), "r" * 10, 40, 560)
    assert fits("x" * 8) and not fits("x" * 9)
    with pytest.raises(ValueError, match="reference text"):
        LF.fit_rule(_lens(300), "", 40, 360)


def test_segments_measure_the_prompt_that_runs():
    """The facade's fit check on the fake tokenizer (one id per phoneme character): the hand-computed cut point."""
    tts, tok = _tts()
    ref = list(range(40))
    p0 = len(tts._apply_chat_template(ref, "abcdefghij", ""))
    assert len(tts._apply_chat_template(ref, "abcdefghij", "x" * 7)) == p0 + 7
    tts.max_context = p0 + 60           # T_ref = 10, K = 4: a segment of up to 10 phoneme characters fits
    assert tts.segments("aaa. bbbbb", ref, "abcdefghij") == ["aaa. bbbbb"]
    assert tts.segments("aaaa. bbbbbb", ref, "abcdefghij") == ["aaaa.", "bbbbbb"]
    assert tts.segments("Aa, bb, cc, dd", ref, "abcdefghij") == ["Aa, bb,", "cc, dd"]   # "," phonemizes to " ,"
    with pytest.raises(ValueError, match="no room"):
        tts.segments("x" * 11, ref, "abcdefghij")


def test_a_text_that_fits_whole_is_itself():
    fits = lambda s: len(s) <= 60
    for text in ["One. Two.", "  spaced   out  \n\nlines  ", "", "A\nB\nC"]:
        assert LF.segment(text, fits) == [text]


def test_greedy_packing_per_line():
    fits = lambda s: len(s) <= 20
    sents = ["aaa.", "bbbb.", "cc.", "dddddddddd.", "eeeeeeeeeeeeeeeeeeee", "f."]
    assert LF.plan_segments(sents, fits) == ["aaa. bbbb. cc.", "dddddddddd.", "eeeeeeeeeeeeeeeeeeee", "f."]
    # a line break ends a segment even when the next line would fit after it
    assert LF.segment("aaaa. bbbb.\ncc. dd. " + "e" * 20, fits) == ["aaaa. bbbb.", "cc. dd.", "e" * 20]
    assert LF.segment("a b c d e f g h i j k l m n o", lambda s: len(s) <= 10) == ["a b c d e", "f g h i j", "k l m n o"]


def test_cut_at_clauses_then_whitespace():
    fits = lambda s: len(s) <= 12
    s = "one two three, four five six seven; eight"
    assert LF.plan_segments([s], fits) == ["one two", "three, four", "five six", "seven; eight"]
    assert LF.plan_segments(["ab: cd — ef – gh; ij, kl"], lambda s: len(s) <= 9) == ["ab: cd —", "ef – gh;", "ij, kl"]
    # punctuation without whitespace after it is not a cut; the last piece packs with the next sentence
    assert LF.plan_segments(["aa,bb cc,dd", "ee."], lambda s: len(s) <= 9) == ["aa,bb", "cc,dd ee."]
    with pytest.raises(ValueError, match="reference leaves no room"):
        LF.plan_segments(["ok then, a verylongword here"], lambda s: len(s) <= 8)


def test_segments_phonemize_each_candidate_once():
    tts, tok = _tts()
    ref = list(range(40))
    tts.max_context = len(tts._apply_chat_template(ref, "abcdefghij", "")) + 72     # up to 12 characters fit
    seen = collections.Counter()

    class Counting(FakePhonemizer):
        def phonemize(self, texts):
            seen.update(texts)
            return super().phonemize(texts)

    tts.phonemizer = Counting()
    got = tts.segments("One two three four five six seven eight. Nine.", ref, "abcdefghij")
    assert got == ["One two", "three four", "five six", "seven eight.", "Nine."]
    assert max(n for t, n in seen.items() if t != "abcdefghij") == 1


def test_round_robin_order():
    assert LF.round_robin([3, 1, 2]) == [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1), (0, 2)]
    assert LF.round_robin([1, 1, 1]) == [(0, 0), (1, 0), (2, 0)]


# ------------------------------------------------------------------------------------------------- seams
def _join64(waves, rate, pause):
    """float64 restatement of the seam formula."""
    if len(waves) == 1:
        return waves[0].astype(np.float64)
    fd = round(0.010 * rate)
    w = lambda i: math.sin(math.pi * (i + 0.5) / (2 * fd)) ** 2
    out = []
    for j, x in enumerate(waves):
        L = len(x)
        y = x.astype(np.float64)
        for i in range(L):
            if j > 0 and i < fd:
                y[i] *= w(i)
            if j < len(waves) - 1 and L - 1 - i < fd:
                y[i] *= w(L - 1 - i)
        out.append(y)
        if j < len(waves) - 1:
            out.append(np.zeros(round(pause * rate)))
    return np.concatenate(out)


def _waves(rng, lens, dtype):
    if dtype == np.int16:
        return [rng.integers(-32768, 32768, n).astype(np.int16) for n in lens]
    return [(rng.standard_normal(n) * 0.3).astype(np.float32) for n in lens]


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("rate, pause", [(24000, 0.0), (24000, 0.35), (16000, 0.0), (22050, 1.0)])
def test_join_against_float64(dtype, rate, pause):
    rng = np.random.default_rng(rate + int(pause * 100))
    fd = round(0.010 * rate)
    lens = [5000, 3 * fd // 2, 7, 2 * fd, fd, 4000]     # shorter than 2 Fd: the two fades overlap
    waves = _waves(rng, lens, dtype)
    got = LF.join(waves, rate, pause)
    want = _join64(waves, rate, pause)
    assert got.dtype == dtype and got.shape == want.shape == (sum(lens) + 5 * round(pause * rate),)
    if dtype == np.int16:
        assert np.abs(got.astype(np.float64) - want).max() <= 0.5 + 1e-6
    else:
        assert np.abs(got - want).max() <= 2e-7 * np.abs(want).max()
    gaps = np.cumsum(lens)[:-1] + np.arange(5) * round(pause * rate)
    for g in gaps:
        assert not np.any(got[g: g + round(pause * rate)])
    # samples away from every seam are untouched
    assert np.array_equal(got[fd: lens[0] - fd], waves[0][fd: lens[0] - fd])


def test_join_one_segment_is_untouched():
    x = np.arange(10, dtype=np.float32)
    assert LF.join([x], 24000, 0.5) is x


def _feed(seams, waves, owners, rng, max_chunk=700):
    """The segments' waveforms cut into chunks of assorted sizes (1 sample and whole segments included), delivered
    in rounds as concurrent slots would: a segment starts when a slot is free (3 slots, FIFO), sends its chunks over
    later rounds and ends with its last chunk or a round after it.  Returns per-text lists of emitted chunks and, per
    round, the emitted lengths and the segments that had ended."""
    pieces = []
    for x in waves:
        cuts = np.sort(rng.integers(0, len(x) + 1, rng.integers(0, 6)))
        p = [c for c in np.split(x, cuts) if len(c)]
        if len(x) > 3 and rng.random() < 0.5:
            p = [x[:1]] + [c for c in np.split(x[1:], np.sort(rng.integers(0, len(x) - 1, 3))) if len(c)]
        pieces.append(p + ([None] if rng.random() < 0.4 else []))    # None: the end comes a round after the audio
    out = [[] for _ in range(max(owners) + 1)]
    waiting, live, log = list(range(len(waves))), [], []
    ended = set()
    while waiting or live:
        while waiting and len(live) < 3:
            live.append(waiting.pop(0))
        chunks, ends = [None] * len(waves), []
        for j in list(live):
            if rng.random() < 0.7:
                x = pieces[j].pop(0)
                chunks[j] = x
                if not pieces[j]:
                    ends.append(j)
                    live.remove(j)
        got = seams.push(chunks, ends)
        ended.update(ends)
        for t, g in enumerate(got):
            if g is not None:
                out[t].append(g)
        log.append(([sum(len(c) for c in o) for o in out], set(ended)))
    return out, log


@pytest.mark.parametrize("dtype", [np.float32, np.int16])
@pytest.mark.parametrize("seed", range(6))
def test_stream_join_equals_whole_join(dtype, seed):
    rng = np.random.default_rng(seed)
    rate = [24000, 16000][seed % 2]
    pause = [0.0, 0.05][seed // 3 % 2]
    counts = [3, 1, 4, 2]
    owners = [t for t, _ in LF.round_robin(counts)]
    fd = round(0.010 * rate)
    waves = _waves(rng, [int(rng.choice([1, 5, fd - 1, fd, fd + 1, 2 * fd - 3, 900, 3000])) for _ in owners], dtype)
    seams = LF.StreamJoin(owners, rate, pause, dtype)
    out, log = _feed(seams, waves, owners, rng)
    segs = [[j for j, o in enumerate(owners) if o == t] for t in range(len(counts))]
    for t, js in enumerate(segs):
        want = LF.join([waves[j] for j in js], rate, pause)
        have = np.concatenate(out[t]) if out[t] else np.zeros(0, dtype)
        assert have.dtype == dtype and np.array_equal(have, want), t
    # hold-back: while segment k of a text is playing, the text has sent nothing of segment k + 1, and a segment with
    # a successor keeps its last Fd samples (or all of them, when shorter) until it ends
    gap = round(pause * rate)
    for emitted, ended in log:
        for t, js in enumerate(segs):
            done = 0
            while done < len(js) and js[done] in ended:
                done += 1
            if done == len(js):
                continue
            before = sum(len(waves[j]) for j in js[:done]) + done * gap
            bound = before + len(waves[js[done]]) - (min(fd, len(waves[js[done]])) if done < len(js) - 1 else 0)
            assert emitted[t] <= bound, (t, emitted[t], bound)


def test_stream_join_holds_a_later_segment_until_its_turn():
    seams = LF.StreamJoin([0, 0], 1000, 0.0, np.float32)      # Fd = 10
    a, b = np.ones(30, np.float32), np.full(25, 2.0, np.float32)
    got = seams.push([a[:12], b], [1])                            # segment 1 finished before segment 0 got far
    assert len(got[0]) == 2                                       # a's last 10 samples held back, nothing of b
    got = seams.push([a[12:], None], [])
    assert len(got[0]) == 18
    got = seams.push([None, None], [0])                           # a ends: its faded tail, then all of b
    assert len(got[0]) == 10 + 25
    assert np.array_equal(np.concatenate([np.ones(2), np.ones(18), got[0]]).astype(np.float32), LF.join([a, b], 1000))


def test_stream_join_passes_one_segment_texts_through():
    seams = LF.StreamJoin([0, 1], 24000, 0.0, np.float32)
    x, y = np.arange(5, dtype=np.float32), np.arange(7, dtype=np.float32)
    got = seams.push([x, y], [0])
    assert got[0] is x and got[1] is y


# ------------------------------------------------------------------------------------------------- the facade
LONG = "First sentence here. Second one follows, with a clause. Third is short.\nA new line starts. And ends."


def _long_tts(max_context_room=60):
    """The fake facade with max_context set so that LONG needs several segments."""
    tts, tok = _tts()
    tts.watermarker = None
    ref = list(range(40))
    p0 = len(tts._apply_chat_template(ref, "abcdefghij", ""))
    tts.max_context = p0 + max_context_room
    return tts, tok, ref


def test_infer_batch_joins_round_robin_segments():
    tts, tok, ref = _long_tts(350)
    texts = [LONG, "Short.", LONG.replace("First", "Another")]
    segs = [tts.segments(t, ref, "abcdefghij") for t in texts]
    assert [len(s) for s in segs] == [3, 1, 3]
    bb = KwBackbone(tok)
    prompts = []
    bb.generate_batch = lambda p, eos, **kw: prompts.append(p) or [torch.tensor([tok.speech_base + 1 + i]) for i in range(len(p))]
    tts.backbone, tts.max_batch = bb, 8
    got = tts.infer_batch(texts, [ref] * 3, ["abcdefghij"] * 3, long_form=True, pause=0.02, temperature=[0.5, 0.7, 0.9])
    order = [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1), (0, 2), (2, 2)]
    assert prompts == [[tts._apply_chat_template(ref, "abcdefghij", segs[t][k]) for t, k in order]]
    flat = tts.infer_batch([segs[t][k] for t, k in order], [ref] * 7, ["abcdefghij"] * 7)
    for t in range(3):
        assert np.array_equal(got[t], LF.join([flat[j] for j, (o, _) in enumerate(order) if o == t], 24000, 0.02))


def test_controls_follow_their_text_into_every_segment():
    tts, tok, ref = _long_tts(350)
    bb = KwBackbone(tok, queue=False)
    tts.backbone, tts.max_batch = bb, 8
    tts.infer_batch([LONG, "Short."], [ref] * 2, ["abcdefghij"] * 2, long_form=True, temperature=[0.5, 0.9], top_k=20,
                    min_new_tokens=[3, 7], exponential_decay_length_penalty=[(10, 1.1), None], speed=[1.0, 1.0])
    (what, n, kw), = bb.calls
    owners = [0, 1, 0, 0]                     # LONG is three segments here, "Short." one
    assert n == 4 and kw["temperature"] == [[0.5, 0.9][t] for t in owners] and kw["top_k"] == 20
    assert kw["min_new_tokens"] == [[3, 7][t] for t in owners]
    assert kw["exponential_decay_length_penalty"] == [[(10, 1.1), None][t] for t in owners]


def test_long_form_logprob_rows_concatenate_per_text():
    tts, tok, ref = _long_tts(350)

    class LpBackbone(KwBackbone):
        def set_logprobs(self, on=True):
            pass

        def generate_batch(self, prompts, eos, **kw):
            ids = [torch.tensor([tok.speech_base + 1]) for _ in prompts]
            return ids, [torch.full((1 + i, 2), float(i)) for i in range(len(prompts))]

    tts.backbone, tts.max_batch = LpBackbone(tok, queue=False), 8
    wavs, lps = tts.infer_batch([LONG, "Short."], [ref] * 2, ["abcdefghij"] * 2, long_form=True, return_logprobs=True)
    assert [lp[:, 0].tolist() for lp in lps] == [[0.0, 2.0, 2.0, 2.0, 3.0, 3.0, 3.0, 3.0], [1.0, 1.0]]
    w, lp = tts.infer(LONG, ref, "abcdefghij", long_form=True, return_logprobs=True)
    assert lp[:, 0].tolist() == [0.0, 1.0, 1.0, 2.0, 2.0, 2.0]


def _stream_setup(room):
    tts, tok, ref = _long_tts(room)
    codec = RampCodec()
    tts.codec, tts.hop_length = codec, codec.hop
    tts.streaming_stride_samples = tts.streaming_frames_per_chunk * codec.hop
    rng = np.random.default_rng(3)
    scripts = [[tok.speech_base + int(c) for c in rng.integers(0, 65536, int(n))] for n in rng.integers(20, 200, 16)]
    return tts, tok, ref, scripts


def _cat(gen, n):
    got = [[] for _ in range(n)]
    for out in gen:
        assert len(out) == n and any(o is not None for o in out)
        for u, o in enumerate(out):
            if o is not None:
                got[u].append(o)
    return [np.concatenate(g) if g else np.zeros(0, np.float32) for g in got]


@pytest.mark.parametrize("pause", [0.0, 0.01])
def test_stream_batch_long_form_equals_join_of_segment_streams(pause):
    tts, tok, ref, scripts = _stream_setup(350)
    texts = [LONG, "Short.", LONG.replace("First", "Another")]
    segs = [tts.segments(t, ref, "abcdefghij") for t in texts]
    order = LF.round_robin([len(s) for s in segs])
    flat = [segs[t][k] for t, k in order]
    tts.backbone = FakeBatchStreamLM(scripts[: len(flat)])
    per_seg = _cat(tts.infer_stream_batch(flat, [ref] * len(flat), ["abcdefghij"] * len(flat)), len(flat))
    tts.backbone = FakeBatchStreamLM(scripts[: len(flat)])
    got = _cat(tts.infer_stream_batch(texts, [ref] * 3, ["abcdefghij"] * 3, long_form=True, pause=pause), 3)
    for t in range(3):
        want = LF.join([per_seg[j] for j, (o, _) in enumerate(order) if o == t], 24000, pause)
        assert np.array_equal(got[t], want), t
    # one text: its segments in slots 0, 1, 2
    tts.backbone = FakeBatchStreamLM(scripts[:3])
    alone = _cat(tts.infer_stream_batch(segs[0], [ref] * 3, ["abcdefghij"] * 3), 3)
    tts.backbone = FakeBatchStreamLM(scripts[:3])
    one = np.concatenate(list(tts.infer_stream(LONG, ref, "abcdefghij", long_form=True, pause=pause)))
    assert np.array_equal(one, LF.join(alone, 24000, pause))


def test_stream_long_form_that_fits_is_the_plain_stream_chunk_by_chunk():
    tts, tok, ref, scripts = _stream_setup(2000)
    texts = [LONG, "Short.", "Third text."]
    tts.backbone = FakeBatchStreamLM(scripts[:3])
    plain = list(tts.infer_stream_batch(texts, [ref] * 3, ["abcdefghij"] * 3))
    tts.backbone = FakeBatchStreamLM(scripts[:3])
    got = list(tts.infer_stream_batch(texts, [ref] * 3, ["abcdefghij"] * 3, long_form=True))
    assert len(got) == len(plain)
    for a, b in zip(got, plain):
        assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------- arguments
@pytest.mark.parametrize("method", ["infer", "infer_batch", "infer_stream", "infer_stream_batch"])
def test_pause_checks(method):
    tts, tok = _tts()
    one = method in ("infer", "infer_stream")
    args = ("hello", [1, 2], "ref") if one else (["hello"], [[1, 2]], ["ref"])
    call = getattr(tts, method)
    with pytest.raises(ValueError, match="long_form"):
        call(*args, pause=0.5)
    for bad in (-0.1, 10.5, float("nan"), float("inf"), True, False, "1", None):
        with pytest.raises(ValueError, match="pause"):
            call(*args, long_form=True, pause=bad)


@pytest.mark.parametrize("method", ["infer_stream", "infer_stream_batch"])
def test_streams_refuse_guidance_and_takes_with_long_form(method):
    tts, tok = _tts()
    one = method == "infer_stream"
    args = ("hello", [1, 2], "ref") if one else (["hello"], [[1, 2]], ["ref"])
    with pytest.raises(ValueError, match="guidance"):
        getattr(tts, method)(*args, long_form=True, guidance_scale=2.0)
    with pytest.raises(ValueError, match="takes"):
        getattr(tts, method)(*args, long_form=True, takes=2)


def test_long_form_checks_the_reference_text():
    tts, tok = _tts()
    with pytest.raises(ValueError, match="reference text"):
        tts.infer("hello", [1, 2], "", long_form=True)


# ------------------------------------------------------------------------------------------------- defaults
CALLS = [
    dict(),
    dict(temperature=[0.5, 0.8, 1.1], top_p=0.9, min_new_tokens=[0, 5, 9]),
    dict(guidance_scale=[2.0, 1.0, 1.5], negative_text="x"),
    dict(exponential_decay_length_penalty=(60, 1.05), speed=[1.0, 1.0, 1.0], repetition_penalty=1.3),
]


@pytest.mark.parametrize("queue", [True, False])
@pytest.mark.parametrize("kw", range(len(CALLS)))
def test_defaults_leave_every_backbone_call_unchanged(queue, kw):
    """With long_form=False (given or not) the backbone gets exactly the calls it got before, and with long_form=True
    on texts that fit whole it gets those calls too."""
    texts, refs, rts = ["one. two.", "three", "four, five."], [[1, 2, 3]] * 3, ["ref"] * 3

    def record(**extra):
        bb = KwBackbone(_tts()[1], queue=queue)
        tts = _facade(bb, 2)
        tts.watermarker = None
        tts.infer_batch(texts, refs, rts, **CALLS[kw], **extra)
        tts.infer(texts[0], refs[0], rts[0], **{k: v[0] if isinstance(v, list) else v for k, v in CALLS[kw].items()},
                  **extra)
        return bb.calls

    plain = record()
    assert plain and record(long_form=False) == plain and record(long_form=False, pause=0.0) == plain
    assert record(long_form=True) == plain
    assert record(long_form=True, pause=3.0) == plain
