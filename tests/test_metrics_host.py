"""CPU checks of the metrics: the float64 restatement (tests/metrics_ref64.py) against the reference's fixtures and, where
the reference tree exists, against live reference calls; the layout and validation logic of
deepfilternet_b200.evaluation_utils; the metric names evaluation_loop refuses."""
import json
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import metrics_ref64 as R
from deepfilternet_b200 import evaluation_utils as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_cases():
    """{name: (sr, clean, degraded, expected)} of metrics_ref.json, the asset inputs resampled by the float64 resampler."""
    from deepfilternet_b200.io import _read_wav
    with open(os.path.join(GOLDEN, "metrics_ref.json")) as f:
        ref = json.load(f)
    npz = np.load(os.path.join(GOLDEN, "metrics_inputs.npz"))
    wav = [_read_wav(os.path.join(GOLDEN, "assets", a))[0][0] for a in ref["assets"]]
    out = {}
    for name, exp in ref["cases"].items():
        if exp["stored"]:
            c, d = npz[f"{name}.clean"], npz[f"{name}.degraded"]
        else:
            c, d = (R.resample64(w, 48000, exp["sr"]).astype(np.float32) for w in wav)
        out[name] = (exp["sr"], c, d, exp)
    return out


def close(a, b, tol=1e-4):
    if math.isnan(b):
        return math.isnan(a)
    return abs(a - b) <= tol + tol * abs(b)


@pytest.mark.parametrize("name", sorted(json.load(open(os.path.join(GOLDEN, "metrics_ref.json")))["cases"]))
def test_restatement_matches_fixture(name):
    sr, c, d, exp = load_cases()[name]
    assert c.size == exp["length"]
    v, counts, margin = R.stoi(c, d, sr)
    assert list(counts) == exp["counts"]
    assert margin > 1e-3
    assert close(v, exp["stoi"]), (v, exp["stoi"])
    assert close(R.si_sdr(c, d), exp["sisdr"]), (R.si_sdr(c, d), exp["sisdr"])
    assert close(R.ssnr(c, d, sr), exp["ssnr"]), (R.ssnr(c, d, sr), exp["ssnr"])


def _reference():
    import ref_harness
    if not ref_harness.available():
        pytest.skip("reference tree not present")
    sys.modules.setdefault("pesq", types.SimpleNamespace(pesq=None))
    ref_harness.import_reference()
    import df.io
    import df.sepm
    import df.stoi
    return ref_harness, df


@pytest.mark.parametrize("sr,seconds,seed", [(48000, 1.3, 1), (44100, 0.9, 2), (16000, 2.1, 3), (8000, 0.7, 4),
                                             (22050, 1.0, 5)])
def test_restatement_matches_live_reference(sr, seconds, seed):
    ref_harness, df = _reference()
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    env = np.repeat(rng.uniform(0.0, 1.0, n // 800 + 1) ** 3, 800)[:n]
    c = (env * rng.standard_normal(n)).astype(np.float32)
    d = (0.7 * c + 0.05 * rng.standard_normal(n)).astype(np.float32)
    v, counts, margin = R.stoi(c, d, sr)
    if margin < 1e-3:
        pytest.skip("a frame lies at the silence threshold")
    ref = float(df.stoi.stoi(torch.from_numpy(c[None]), torch.from_numpy(d[None]), sr)[0])
    assert close(v, ref), (v, ref)
    c16 = df.io.resample(torch.from_numpy(c[None]), sr, 16000)[0].numpy() if sr != 16000 else c
    d16 = df.io.resample(torch.from_numpy(d[None]), sr, 16000)[0].numpy() if sr != 16000 else d
    assert close(R.ssnr(c, d, sr), float(df.sepm.SNRseg(c16, d16, 16000)))
    assert close(R.si_sdr(c, d), ref_harness.si_sdr(c, d))


def test_metric_bits_and_rows():
    assert E.metric_bits(["sisdr"]) == 1 and E.metric_bits(["STOI", "ssnr"]) == 6 and E.metric_bits("stoi") == 2
    assert E.bit_names(7) == ["sisdr", "stoi", "ssnr"] and E.bit_names(5) == ["sisdr", "ssnr"]
    for bad in ([], ["pesqq"]):
        with pytest.raises(ValueError):
            E.metric_bits(bad)


@pytest.mark.parametrize("name,needs", [("composite", "PESQ"), ("composite-octave", "PESQ"), ("pesq", "PESQ"),
                                        ("pesq-nb", "PESQ"), ("dnsmos5", "DNSMOS")])
def test_unsupported_metrics_say_what_they_need(name, needs):
    with pytest.raises(ValueError, match=needs):
        E.metric_bits(["stoi", name])
    with pytest.raises(ValueError, match="does not provide"):
        E.evaluation_loop(None, None, [], [], metrics=[name])


def test_rates():
    assert E.check_sr(48000) == 48000 and E.check_sr(10000) == 10000 and E.check_sr(np.int64(44100)) == 44100
    assert E.tap_floats(16000, 16000) == 0
    assert E.tap_floats(48000, 10000) == 5 * (2 * 78 + 24)
    for bad in (0, -8000, 16000.0, True, 11025):
        with pytest.raises(ValueError):
            E.check_sr(bad)


def test_lengths_and_layout():
    lens = E.check_pair_lengths([3, 5, 2], np.array([3, 5, 2]))
    assert lens.dtype == np.int64 and lens.tolist() == [3, 5, 2]
    off, n = E.packed_offsets(lens)
    assert off.tolist() == [0, 3, 8] and n == 10
    with pytest.raises(ValueError, match="entry 1: clean has 5 samples, degraded 4"):
        E.check_pair_lengths([3, 5], [3, 4])
    for c, d in (([], []), ([0], [0]), ([3, -1], [3, -1]), ([1, 2], [1])):
        with pytest.raises(ValueError):
            E.check_pair_lengths(c, d)
    with pytest.raises(ValueError, match="at most"):
        E.check_pair_lengths(np.ones(E.MAX_ENTRIES + 1), np.ones(E.MAX_ENTRIES + 1))


def test_restatement_counts_follow_the_definition():
    """Counts of silence removal from the framing rule alone: all frames kept, length T10 exactly."""
    x = np.random.default_rng(0).standard_normal(256 * 20).astype(np.float32)
    v, (nk, lc, nf), _ = R.stoi(x, x, 10000)
    assert (nk, lc, nf) == (20 * 2 + 1, 256 * 20, 1 + (256 * 20 - 256) // 128)
    assert abs(v - 1.0) < 1e-9
