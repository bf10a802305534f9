"""CPU checks of LLR, WSS and the composite measure: the float64 restatement (tests/composite_ref64.py) against the
reference's fixtures (tests/golden/composite_ref.json, made by oracle/gen_golden_composite.py) and, where the reference
tree exists, against live df.sepm calls; the regression constants against the reference CI's composite known answers;
the names, bits and composite plumbing of deepfilternet_b200.evaluation_utils.

The largest restatement-vs-reference difference seen is about 2e-7 in LLR (the reference's float32 products in its
quadratic forms, which the restatement evaluates in fp64); WSS agrees to about 1e-14.  So close()'s 1e-4 holds with
margin."""
import json
import math
import os
import sys
import types

import numpy as np
import pytest

import composite_ref64 as C
import metrics_ref64 as M
from deepfilternet_b200 import evaluation_utils as E
from test_metrics_host import close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF = json.load(open(os.path.join(GOLDEN, "composite_ref.json")))


def load_cases():
    """{name: (sr, clean, degraded, expected)} of composite_ref.json; the asset inputs resampled by the float64
    resampler."""
    from deepfilternet_b200.io import _read_wav
    npz = np.load(os.path.join(GOLDEN, "composite_inputs.npz"))
    wav = [_read_wav(os.path.join(GOLDEN, "assets", a))[0][0] for a in REF["assets"]]
    out = {}
    for name, exp in REF["cases"].items():
        if exp["stored"]:
            c, d = npz[f"{name}.clean"], npz[f"{name}.degraded"]
        elif name == "assets_twice_48k":
            c, d = (np.concatenate([w, w]) for w in wav)
        else:
            c, d = (M.resample64(w, 48000, exp["sr"]).astype(np.float32) for w in wav)
        out[name] = (exp["sr"], c, d, exp)
    return out


def to16(x, sr):
    return np.asarray(x, np.float32) if sr == 16000 else M.resample64(x, sr, 16000).astype(np.float32)


@pytest.mark.parametrize("name", sorted(REF["cases"]))
def test_restatement_matches_fixture(name):
    sr, c, d, exp = load_cases()[name]
    assert c.size == exp["length"]
    c16, d16 = to16(c, sr), to16(d, sr)
    assert c16.size == exp["n16"] and C.n_frames(c16.size) == exp["frames"] and C.keep_count(exp["frames"]) == exp["keep"]
    assert close(C.wss(c16, d16), exp["wss"]), (C.wss(c16, d16), exp["wss"])
    got = C.composite(c16, d16, REF["stub_pesq"])
    # LLR (and CSIG / COVL through it) only where it is well conditioned: rows upsampled from 8 kHz have an empty upper half
    # band, their order-16 LPC models are near-singular, and the reference's value is set by the rounding of its float32
    # quadratic forms (the restatement's fp64 forms give another value from the same rows), and it follows the last bits
    # of the resampler
    llr_ok = sr != 8000
    if llr_ok:
        assert close(C.llr(c16, d16), exp["llr"]), (C.llr(c16, d16), exp["llr"])
    for q, (g, e) in enumerate(zip(got, exp["composite"])):
        if llr_ok or q not in (1, 3):
            assert close(g, e), (q, got, exp["composite"])


def test_fixture_edges():
    """The frame count and the 0.95 cut at the edges the fixture pins."""
    cases = REF["cases"]
    assert [cases[f"len{n}_16k"]["frames"] for n in (599, 600, 601, 719, 720)] == [0, 1, 1, 1, 2]
    assert [cases[f"frames{T}_16k"]["keep"] for T in (10, 30, 50)] == [10, 28, 48]
    assert cases["zero_clean_16k"]["llr"] == pytest.approx(math.log(1000.0), abs=1e-12)
    assert cases["zero_zero_16k"]["wss"] == 0.0
    assert all(math.isnan(v) for v in cases["len599_16k"]["composite"])
    assert cases["assets_twice_48k"]["length"] == 20 * 48000


def _reference():
    import ref_harness
    if not ref_harness.available():
        pytest.skip("reference tree not present")
    sys.modules.setdefault("pesq", types.SimpleNamespace(pesq=None))
    ref_harness.import_reference()
    import df.sepm
    return df.sepm


def _pair(rng, n):
    env = np.repeat(rng.uniform(0.0, 1.0, n // 400 + 1) ** 3 * (rng.uniform(0, 1, n // 400 + 1) > 0.15), 400)[:n]
    c = (0.3 * env * rng.standard_normal(n)).astype(np.float32)
    d = (rng.uniform(0.3, 1.2) * c + rng.uniform(0.001, 0.1) * rng.standard_normal(n)).astype(np.float32)
    return c, d


@pytest.mark.parametrize("n,seed", [(600, 1), (1680, 2), (4080, 3), (6480, 4), (16000, 5), (37001, 6)])
def test_restatement_matches_live_reference(n, seed):
    sepm = _reference()
    c, d = _pair(np.random.default_rng(seed), n)
    if C.wss_frames(c, d)[1] < 1e-6:
        pytest.skip("a band energy lies at a slope or clamp edge")
    assert close(C.llr(c, d), float(sepm.llr(c, d, 16000)), 1e-6)
    assert close(C.wss(c, d), float(sepm.wss(c, d, 16000)), 1e-9)


def test_composite_matches_sepm_with_a_stub_pesq(monkeypatch):
    sepm = _reference()
    monkeypatch.setattr(sepm, "pesq", lambda fs, r, d, mode: 3.25)
    rng = np.random.default_rng(12)
    for n in (600, 5000, 24000):
        c, d = _pair(rng, n)
        ref = [float(v) for v in sepm.composite(c, d, 16000)]
        got = C.composite(c, d, 3.25)
        for g, e in zip(got, ref):
            assert close(g, e, 1e-6), (got, ref)


@pytest.mark.parametrize("model", sorted(REF["ci_composite"]))
def test_regression_constants_reproduce_the_ci_known_answers(model):
    """df/scripts/test_df.py's composite known answers (PESQ, CSIG, CBAK, COVL, SSNR of noisy_snr0 enhanced by each
    pretrained model): WSS follows from CBAK and LLR from CSIG (neither is clipped there), and then the COVL regression
    reproduces the CI's COVL to its float32 rounding."""
    p, csig, cbak, covl, ssnr = REF["ci_composite"][model]
    assert 1 < csig < 5 and 1 < cbak < 5 and 1 < covl < 5
    wss = (C.CBAK[0] + C.CBAK[1] * p + C.CBAK[3] * ssnr - cbak) / -C.CBAK[2]
    llr = (C.CSIG[0] + C.CSIG[2] * p + C.CSIG[3] * wss - csig) / -C.CSIG[1]
    assert 0 < llr < 2 and 10 < wss < 100
    assert C.regress(p, llr, wss, ssnr) == pytest.approx((csig, cbak, covl), abs=1e-5)


def test_names_bits_and_rows():
    assert E.METRICS["llr"] == (16, "LLR") and E.METRICS["wss"] == (32, "WSS")
    assert E.metric_bits(["llr", "WSS"]) == 48 and E.metric_bits(["wss", "sisdr"]) == 33
    assert E.bit_names(1 | 2 | 4 | 16 | 32) == ["sisdr", "stoi", "ssnr", "llr", "wss"]
    assert E.bit_names(16 | 4) == ["ssnr", "llr"]
    for bad in (["composite"], ["llr", "composite"]):
        with pytest.raises(ValueError, match="PESQ") as ei:
            E.metric_bits(bad)
        assert "does not provide" in str(ei.value)
    names, bits = E._split_composite(["STOI", "composite"], lambda r, d: 1.0)
    assert names == ["stoi", "composite"] and bits == 2 | 4 | 16 | 32
    assert E._split_composite("composite", lambda r, d: 1.0)[1] == 4 | 16 | 32
    with pytest.raises(ValueError, match="does not provide"):
        E._split_composite(["composite"], None)
    with pytest.raises(ValueError, match="callable"):
        E._split_composite(["composite"], 3.0)
    for name in ("composite-octave", "pesq", "pesq-nb", "dnsmos5"):
        with pytest.raises(ValueError, match="does not provide"):
            E._split_composite([name], lambda r, d: 1.0)


def test_composite_values():
    calls = []

    def pesq(r, d):
        calls.append((r, d))
        return 2.0

    short = np.zeros(599, np.float32)
    assert np.isnan(E.composite_values(pesq, short, short, 0.1, 10.0, 5.0)).all() and not calls
    x = np.zeros(600, np.float32)
    v = E.composite_values(pesq, x, x, 0.5, 30.0, 4.0)
    assert v.dtype == np.float32 and len(calls) == 1 and calls[0][0] is x
    exp = (2.0,) + C.regress(2.0, 0.5, 30.0, 4.0) + (4.0,)
    assert np.array_equal(v, np.asarray(exp, np.float64).astype(np.float32))
    lo = E.composite_values(lambda r, d: -1.0, x, x, 6.9, 120.0, -10.0)
    assert lo[1] == 1.0 and lo[2] == 1.0 and lo[3] == 1.0
    hi = E.composite_values(lambda r, d: 4.6, x, x, 0.0, 0.0, 35.0)
    assert hi[1] == 5.0 and hi[2] == 5.0 and hi[3] == 5.0

    def boom(r, d):
        raise RuntimeError("pesq failed")
    with pytest.raises(RuntimeError, match="pesq failed"):
        E.composite_values(boom, x, x, 0.5, 30.0, 4.0)


def test_restatement_trim_and_peaks():
    assert [C.keep_count(T) for T in (1, 10, 30, 50, 20, 100)] == [1, 10, 28, 48, 19, 95]
    assert C.trimmed_mean(np.array([3.0, 1.0, 2.0, 100.0] + [0.5] * 16)) == pytest.approx((0.5 * 16 + 1 + 2 + 3) / 19)
    e = np.array([[0.0, 1, 2, 1, 0, -1, 3, 4, 4, 2] + [0.0] * 15])
    s = np.diff(e, axis=1)
    pk = C._loc_peaks(s, e)[0]
    # findLocPeaks: rising at band 0 walks to band 2 (slope 2 falls) and takes energy[1]; falling at band 4 walks down to
    # band 1 (the last rise) and takes energy[2]
    assert pk[0] == 1 and pk[1] == 1 and pk[2] == 2 and pk[4] == 2
