"""CPU: the measurement harness's own arithmetic (bench.py) -- workload shape, algorithmic bytes of a decode step,
the tokenizer stub the end-to-end leg gives the facade, CLI defaults the driver relies on."""
import sys

import bench
from neutts_air_b200.lm import LMShape


def test_workload_and_algorithmic_bytes():
    assert (bench.PREFILL, bench.DECODE, bench.HOP, bench.SR) == (500, 250, 480, 24000) and bench.AUDIO_S == 5.0
    p = bench.synth_prompts(3, 217472, bench.SPEECH_BASE, 1)
    assert all(len(x) == 500 for x in p)
    assert all(t < 151643 for t in p[0][:128]) and all(bench.SPEECH_BASE <= t < bench.SPEECH_BASE + 65536 for t in p[0][128:])
    m = bench.synth_prompts(16, 217472, bench.SPEECH_BASE, 2, mixed=True)
    assert all(200 <= len(x) <= 1400 for x in m) and len({len(x) for x in m}) > 4
    # BASELINE.md section 2: every bf16 weight once + KV of the mean context + the token's activations
    sb = bench.step_bytes(LMShape(), 1, 500)
    assert abs(sb - 1.1132e9) < 2e6, sb
    assert abs((bench.step_bytes(LMShape(), 64, 500) - sb) - 63 * (12288 * 626 + 1792)) < 1e3


def test_bench_tokenizer_and_cli_defaults(monkeypatch):
    tok = bench._BenchTokenizer()
    assert tok.convert_tokens_to_ids("<|SPEECH_GENERATION_END|>") == bench.EOS
    assert tok.convert_tokens_to_ids("<|speech_0|>") == bench.SPEECH_BASE
    assert tok.convert_tokens_to_ids("<|speech_65535|>") == bench.SPEECH_BASE + 65535
    monkeypatch.setattr(sys, "argv", ["bench.py"])
    a = bench.parse()
    assert (a.gpus, a.impl, a.batch) == (1, "b200", 0) and a.warmup >= 3 and a.steps >= 1     # contract: W >= 3, default N = 1


def test_dump_outputs_writes_float_arrays_within_the_cap(tmp_path, monkeypatch):
    import numpy as np
    import torch

    pcm = torch.randn(6, 1000)
    ids = torch.arange(6 * 250, dtype=torch.int32).reshape(6, 250)
    bench.dump_outputs(str(tmp_path / "a"), {"pcm": pcm, "generated_ids": ids})
    got = np.load(tmp_path / "a" / "pcm.npy"), np.load(tmp_path / "a" / "generated_ids.npy")
    assert got[0].dtype == np.float32 and np.array_equal(got[0], pcm.numpy())
    assert got[1].dtype == np.float64 and np.array_equal(got[1], ids.double().numpy())
    # over the cap: the same seeded rows of every array, recorded next to them
    monkeypatch.setattr(bench, "DUMP_BYTES", 3 * 1000 * 4)
    for d in ("b", "c"):
        bench.dump_outputs(str(tmp_path / d), {"pcm": pcm, "generated_ids": ids})
    rows = np.load(tmp_path / "b" / "sampled_rows.npy").astype(int)
    assert 0 < len(rows) < 6 and np.array_equal(rows, np.load(tmp_path / "c" / "sampled_rows.npy"))
    assert np.array_equal(np.load(tmp_path / "b" / "pcm.npy"), pcm.numpy()[rows])
    assert sum((tmp_path / "b" / f).stat().st_size for f in ("pcm.npy", "generated_ids.npy")) <= 3 * 1000 * 4 + 1024


def test_steps_flag_sets_the_timed_steps(monkeypatch):
    monkeypatch.setattr(sys, "argv", ["bench.py", "--steps", "7", "--warmup", "3", "--dump-outputs", "/tmp/x"])
    a = bench.parse()
    assert (a.steps, a.warmup, a.dump_outputs) == (7, 3, "/tmp/x")
