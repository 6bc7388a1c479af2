"""CPU, world_size 2, gloo: the one collective of the path (all-gather of finished waveforms) and
the sharded facade call, without a GPU."""
import os
import socket

import numpy as np
import torch
import torch.distributed as td
import torch.multiprocessing as mp


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from neutts_air_b200 import dist

        lens = [30, 10, 50, 20, 40]
        mine = dist.shard_indices(len(lens), lens)
        wavs = [np.full(480 * lens[i], float(i), dtype=np.float32) for i in mine]     # ragged lengths
        allw = dist.all_gather_waveforms(wavs, mine, len(lens), device="cpu", lengths=lens)
        ok = all(len(allw[i]) == 480 * lens[i] and float(allw[i][0]) == float(i) and float(allw[i][-1]) == float(i) for i in range(5))
        # bounded job (bench.py, fixed-length utterances): t_max known -> the all-gather is the ONLY collective; tensors
        # (as a device engine returns them) are accepted as well as numpy arrays; over-long waveforms are refused
        wt = [torch.full((480 * lens[i],), float(i)) for i in mine]
        allt = dist.all_gather_waveforms(wt, mine, len(lens), device="cpu", t_max=480 * 50)
        ok = ok and all(len(allt[i]) == 480 * lens[i] and float(allt[i][-1]) == float(i) for i in range(5))
        try:
            dist.all_gather_waveforms(wt, mine, len(lens), device="cpu", t_max=100)
            ok = False
        except ValueError:
            pass

        # facade path: every rank ends up with every waveform
        import warnings

        from neutts import NeuTTS
        from tests.fakes import FakeBackbone, FakeCodec, FakePhonemizer, FakeTokenizer

        tok = FakeTokenizer()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            tts = NeuTTS(tokenizer=tok, phonemizer=FakePhonemizer(), codec=FakeCodec(),
                         backbone=FakeBackbone([tok.speech_base + 7, tok.speech_base + 8, tok.special_base + 5]))
        texts = ["a", "bb bb", "ccc ccc ccc"]
        outs = tts.infer_batch(texts, [[1, 2]] * 3, ["r"] * 3, distributed=True)
        ok = ok and len(outs) == 3 and all(len(o) == 960 for o in outs)
        q.put((rank, ok, mine))
    finally:
        td.destroy_process_group()


def test_all_gather_waveforms_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(30)
    assert all(r[1] for r in res), res
    assert sorted(res[0][2] + res[1][2]) == [0, 1, 2, 3, 4]            # the two shards partition the utterances
