"""CPU: streaming handles at other sample rates (dfb_stream_set_sample_rate).  The Python-side checks of DfStream's ``sr``,
the C ABI's declarations, and the resamplers' delays D_r / E_r recomputed from the tap geometry and the causality rule
(every call forms its model hops, and returns its output hops, from the input received so far) against the closed form
the library uses and the table in include/dfb200.h."""
import math
import os
import re
from types import SimpleNamespace

import pytest

from deepfilternet_b200 import _lib
from deepfilternet_b200.streaming import MODEL_SR, STREAM_RATES, DfStream, rate_delays, rate_taps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["dfb_stream_set_sample_rate", "dfb_stream_latency_samples", "dfb_debug_resample_stream"]


def test_new_entry_points_are_declared_and_bound():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES, name
    assert len(_lib.SIGNATURES["dfb_stream_set_sample_rate"][1]) == 10
    assert len(_lib.SIGNATURES["dfb_debug_resample_stream"][1]) == 12


@pytest.mark.parametrize("sr", [11025, 22050, 96000, 0, -16000, 16000.0, "16000", True, None])
def test_unsupported_rates_are_refused_before_the_library(sr):
    with pytest.raises(_lib.DfbError) as e:
        rate_taps(sr)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    fake = SimpleNamespace(_h=None, spectral=False)     # no library call can succeed on it
    with pytest.raises(_lib.DfbError) as e:
        DfStream.set_sample_rate(fake, sr)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED


@pytest.mark.parametrize("sr", [16000, MODEL_SR])
def test_a_spectral_handle_takes_no_rate(sr):
    fake = SimpleNamespace(_h=None, spectral=True)
    with pytest.raises(_lib.DfbError) as e:
        DfStream.set_sample_rate(fake, sr)
    assert e.value.code == _lib.DFB_ERR_INVALID


def causal_delays(sr):
    """D_r and E_r by search: the smallest D (a multiple of nw_up, in 48 kHz samples) with which the last 48 kHz sample of
    every hop boundary a needs only rate-r input before a * h_r, and the smallest E (rate-r samples) with which the last
    rate-r output sample of every boundary needs only 48 kHz samples before a * 480.  Tap k of output t = i * nw + j reads
    input i * og - width + k, k < 2 * width + og."""
    (_, wu, ou, nu), (_, wd, od, nd) = rate_taps(sr)
    hr = sr // 100
    boundaries = range(1, 2 * 48000 // hr + 2)

    def ok(delay, og, nw, width, hop_out, hop_in):
        for a in boundaries:
            t = a * hop_out - delay - 1
            if t >= 0 and (t // nw) * og - width + 2 * width + og - 1 >= a * hop_in:
                return False
        return True

    D = next(m * nu for m in range(1000) if ok(m * nu, ou, nu, wu, 480, hr))
    E = next(e for e in range(10000) if ok(e, od, nd, wd, hr, 480))
    return D, E, (ou, nu, wu), (od, nd, wd)


def header_table():
    hdr = open(os.path.join(ROOT, "include", "dfb200.h")).read()
    rows = re.findall(r"^ \*\s+(\d+)\s+(\d+)\s+(\d+)/(\d+)/(\d+)\s+(\d+)\s+(\d+)/(\d+)/(\d+)\s+(\d+)\s+(\d+) / ([\d.]+)$", hdr, re.M)
    return {int(r[0]): [int(v) for v in r[1:11]] + [float(r[11])] for r in rows}


@pytest.mark.parametrize("sr", STREAM_RATES)
def test_delays_follow_from_the_taps(sr):
    D, E, up, down = causal_delays(sr)
    assert D % (MODEL_SR // math.gcd(sr, MODEL_SR)) == 0 and D * sr % MODEL_SR == 0
    delay = D * sr // MODEL_SR + E
    assert rate_delays(*up, *down) == (D, E, delay)
    assert 0 < delay < sr // 100                      # below one hop at every listed rate
    assert D <= 480                                   # the one extra hop of a session's end covers the zeros in front
    tab = header_table()[sr]
    assert tab == [sr // 100, *up, D, *down, E, delay, tab[10]]
    assert abs(tab[10] - 1000.0 * delay / sr) < 5e-4 + 1e-9    # ms, rounded to 3 decimals


def test_header_table_lists_every_rate():
    assert sorted(header_table()) == list(STREAM_RATES)
