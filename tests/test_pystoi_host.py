"""CPU checks of pystoi's STOI and ESTOI: the float64 restatement (tests/pystoi_ref64.py) against the reference CI's STOI
known answers (df/scripts/test_df.py, on the reference's own CPU enhance() with the pretrained checkpoints, where the
reference tree exists) and against tests/golden/pystoi_ref.json (made by oracle/gen_golden_pystoi.py); its counts and
values at the edges of pystoi's rules; the names and bits of deepfilternet_b200.evaluation_utils."""
import json
import math
import os

import numpy as np
import pytest

import pystoi_ref64 as P
from deepfilternet_b200 import evaluation_utils as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF = json.load(open(os.path.join(GOLDEN, "pystoi_ref.json")))


def signal(rng, n, sr):
    """oracle/gen_golden_pystoi.py's seeded pairs: speech-like bursts and a scaled, noisy copy."""
    blk = max(1, sr // 20)
    env = np.repeat(rng.uniform(0, 1, n // blk + 1) ** 3 * (rng.uniform(0, 1, n // blk + 1) > 0.2), blk)[:n]
    c = (0.3 * env * rng.standard_normal(n)).astype(np.float32)
    d = (rng.uniform(0.3, 1.2) * c + rng.uniform(0.001, 0.1) * rng.standard_normal(n)).astype(np.float32)
    return c, d


def stationary(rng, n10):
    """A pair of n10 samples at 10 kHz with no frame 40 dB below the loudest: every frame is kept."""
    c = (0.1 * rng.standard_normal(n10)).astype(np.float32)
    return c, (0.7 * c + 0.05 * rng.standard_normal(n10)).astype(np.float32)


@pytest.mark.parametrize("name", sorted(REF["cases"]))
def test_restatement_matches_fixture(name):
    case = REF["cases"][name]
    c, d = signal(np.random.default_rng(case["seed"]), case["n"], case["sr"])
    r = P.pystoi10(P.rows10(c, case["sr"]), P.rows10(d, case["sr"]))
    assert {k: r[k] for k in case["counts"]} == case["counts"]
    # the fixture's rows come from torchaudio's float32 resampler, these from the float64 one rounded to float32: the last
    # bits of the rows differ, which moves the values by up to about 1e-7
    assert abs(r["stoi"] - case["stoi"]) < 1e-6 and abs(r["estoi"] - case["estoi"]) < 1e-6, (r["stoi"], r["estoi"], case)


def test_fixture_known_answers():
    """The restatement on the reference's CPU enhance() of the full assets (the fixture's "pretrained" rows) reproduces
    test_df.py's STOI targets to 1e-5 (its own tolerance is 1e-4)."""
    assert sorted(REF["ci_stoi"]) == sorted(REF["pretrained"]) == sorted(REF["seeded"])
    for m, target in REF["ci_stoi"].items():
        assert abs(REF["pretrained"][m]["stoi"] - target) < 1e-5, (m, REF["pretrained"][m]["stoi"], target)
        assert 0 < REF["pretrained"][m]["estoi"] < REF["pretrained"][m]["stoi"]
        assert REF["seeded"][m]["counts"]["J"] == REF["seeded"][m]["counts"]["nf"] - 29


@pytest.mark.parametrize("model", ["DeepFilterNet3", "DeepFilterNet2", "DeepFilterNet"])
def test_restatement_reproduces_ci_targets_live(model):
    """Live: the reference's CPU enhance() of noisy_snr0.wav with the pretrained checkpoint, df.io.resample to 10 kHz,
    then the restatement, against df/scripts/test_df.py's STOI target."""
    import ref_harness as rh
    if not rh.available():
        pytest.skip("reference tree not present")
    import torch
    rh.import_reference()
    import df.io as df_io
    from df.enhance import enhance, init_df
    model_dir = os.path.join(rh.unpack_models(), model)
    clean, noisy = (rh.read_wav(os.path.join(rh.REF_ROOT, "assets", a))[0]
                    for a in ("clean_freesound_33711.wav", "noisy_snr0.wav"))
    net, st, _, _ = init_df(model_dir, log_file=None, log_level="ERROR", config_allow_defaults=True)
    enh = enhance(net, st, torch.from_numpy(noisy[None]), pad=True)[0].numpy()
    x10, y10 = (df_io.resample(torch.as_tensor(a), 48000, 10000, method="sinc_fast").numpy() for a in (clean, enh))
    assert abs(P.pystoi10(x10, y10)["stoi"] - REF["ci_stoi"][model]) < 1e-5


def test_edges_no_frame_and_too_short():
    rng = np.random.default_rng(1)
    for n, F in ((1, 0), (256, 0), (257, 1), (384, 1), (385, 2)):
        c, d = stationary(rng, n)
        r = P.pystoi10(c, d)
        assert r["F"] == F == P.n_frames(n)
        if F == 0:
            assert math.isnan(r["stoi"]) and math.isnan(r["estoi"]) and r["K"] == 0
        else:
            assert r["stoi"] == r["estoi"] == 1e-5 and r["K"] == F and r["nf"] == F - 1


def test_edges_k_30_31_32():
    """K = 30 leaves 29 STFT frames (1e-5); K = 31 one segment; K = 32 two."""
    rng = np.random.default_rng(2)
    for K, J in ((30, 0), (31, 1), (32, 2)):
        for extra in (1, 64, 128):   # F = K for 128 (K - 1) + 256 < L10 <= 128 K + 256
            n = 128 * (K - 1) + 256 + extra
            c, d = stationary(rng, n)
            r = P.pystoi10(c, d)
            assert (r["F"], r["K"], r["lc"], r["nf"], r["J"]) == (K, K, (K - 1) * 128 + 256, K - 1, J)
            assert r["X"].shape == (15, K - 1)
            if J == 0:
                assert r["stoi"] == r["estoi"] == 1e-5
            else:
                assert 0.5 < r["stoi"] < 1 and 0 < r["estoi"] < 1


def test_silence_mask_and_silent_degraded():
    rng = np.random.default_rng(3)
    c, d = stationary(rng, 20000)
    c[5000:12000] *= 1e-3   # 60 dB down: those frames are dropped
    r = P.pystoi10(c, d)
    assert r["K"] < r["F"] and r["lc"] == (r["K"] - 1) * 128 + 256
    # a silent degraded signal: every band row of y is constant (0); pystoi's noise would make ESTOI random there,
    # without it both measures are exactly 0
    z = P.pystoi10(c, np.zeros_like(d))
    assert z["stoi"] == 0.0 and z["estoi"] == 0.0


def test_constant_band_row_normalises_to_zero():
    a = np.arange(15 * 30, dtype=np.float64).reshape(1, 15, 30) % 7
    a[0, 4] = 2.5   # a constant band row
    n = P._normalise(a, 2)
    assert np.all(n[0, 4] == 0) and np.isfinite(n).all()
    assert np.allclose(np.linalg.norm(np.delete(n[0], 4, axis=0), axis=1), 1.0)
    col = P._normalise(n, 1)
    assert np.isfinite(col).all() and np.allclose(col.sum(1), 0.0)


def test_names_and_bits():
    assert E.METRICS["pystoi"] == (128, "PYSTOI") and E.METRICS["estoi"] == (256, "ESTOI")
    assert E.metric_bits(["PYSTOI", "estoi"]) == 384 and E.metric_bits(["estoi", "stoi"]) == 258
    assert E.bit_names(511 & ~8 & ~64) == ["sisdr", "stoi", "ssnr", "llr", "wss", "pystoi", "estoi"]
    assert E.bit_names(256 | 2) == ["stoi", "estoi"]
    assert E._split_composite(["pystoi", "composite"], lambda r, d: 1.0)[1] == 128 | 4 | 16 | 32
