"""CPU: rated ragged batches (enhance_batch / enhance_device_ragged with sr=, dfb_enhance_ragged with rates).  Output lengths
against io.resample's composition, the supported-rate bound, the Python-side refusals, and the new C ABI's declarations,
bindings and exports."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from deepfilternet_b200 import _lib, io, ragged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOP = 480
RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 88200, 96000)
NEW = {"dfb_model_add_rate": 10, "dfb_enhance_ragged": 22, "dfb_enhance_ragged_host": 21,
       "dfb_enhance_out_len_at": 4, "dfb_debug_resample_rows": 12}


def resampled_len(t, orig, new):
    """io.resample's output length"""
    g = math.gcd(orig, new)
    return int(math.ceil((new // g) * t / (orig // g)))


def composition_len(t, r, pad):
    t48 = resampled_len(t, r, 48000)
    return resampled_len(ragged.out_len(t48, HOP, pad), 48000, r)


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("pad", [True, False])
def test_out_len_at_is_the_composition_length(rate, pad):
    hop_r = HOP * rate // 48000
    for t in (1, hop_r - 1, hop_r, hop_r + 1, hop_r + 2, 60 * rate, 60 * rate + 7):
        if not pad and ragged.len_48k(t, rate) < HOP:
            continue   # no frame: refused, as enhance() refuses it
        assert ragged.len_48k(t, rate) == resampled_len(t, rate, 48000)
        assert ragged.out_len_at(t, rate, HOP, pad) == composition_len(t, rate, pad), (t, rate, pad)
    assert ragged.out_len_at(12345, 48000, HOP, pad) == ragged.out_len(12345, HOP, pad)


@pytest.mark.parametrize("rate", RATES)
def test_tap_bound_accepts_the_listed_rates(rate):
    p = io.get_resample_params("sinc_fast")
    n = sum(io.resample_kernel(a, b, **p)[0].numel() for a, b in ((rate, 48000), (48000, rate)))
    assert ragged.rate_tap_floats(rate) == n
    assert n <= ragged.MAX_RATE_TAPS
    assert ragged.check_rate(rate) == rate


def test_tap_bound_rejects_47999_and_names_it():
    assert ragged.rate_tap_floats(11025) == 230794
    assert ragged.rate_tap_floats(47999) > 4e9
    for bad in (47999, 0, -16000, 16000.0, "16000", True):
        with pytest.raises(ValueError, match=re.escape(repr(bad))):
            ragged.check_rate(bad)


def test_rates_arg():
    assert ragged.rates_arg(None, 3) is None
    assert ragged.rates_arg(48000, 3) is None
    assert ragged.rates_arg([48000, 48000], 2) is None
    assert ragged.rates_arg(16000, 2).tolist() == [16000, 16000]
    assert ragged.rates_arg([8000, 48000, 44100], 3).dtype == np.int32
    with pytest.raises(ValueError, match="2 sample rates for 3"):
        ragged.rates_arg([8000, 16000], 3)
    with pytest.raises(ValueError, match="47999"):
        ragged.rates_arg([8000, 47999], 2)


def test_packed_layout_with_rates():
    shapes = [(2, 16000), (1, 4801), (1, 30)]
    rates = np.array([16000, 48000, 8000], np.int32)
    lens, in_off, out_off, n_in, n_out, slices, sr = ragged.packed_layout(shapes, HOP, True, rates)
    assert lens.tolist() == [16000, 16000, 4801, 30]
    assert sr.tolist() == [16000, 16000, 48000, 8000]
    olens = [ragged.out_len_at(t, r, HOP, True) for t, r in zip(lens, sr)]
    assert out_off.tolist() == [0, olens[0], 2 * olens[0], 2 * olens[0] + olens[2]]
    assert (n_in, n_out) == (sum(lens), sum(olens))
    assert slices == [(0, 2, olens[0]), (2 * olens[0], 1, olens[2]), (2 * olens[0] + olens[2], 1, olens[3])]
    # 100 samples at 16 kHz are 300 at 48 kHz: no frame without pad, as enhance() refuses a stream shorter than a hop
    with pytest.raises(RuntimeError, match="shorter than one hop"):
        ragged.packed_layout([(1, 100)], HOP, False, np.array([16000], np.int32))
    ragged.packed_layout([(1, 160)], HOP, False, np.array([16000], np.int32))


def test_padded_layout_with_rates_and_group_rates():
    lens, in_off, out_off, ow = ragged.padded_layout([16000, 8000, 300], 16000, HOP, True, np.array([16000, 8000, 48000]))
    assert ow == 16000 and in_off.tolist() == [0, 16000, 32000] and out_off.tolist() == [0, ow, 2 * ow]
    with pytest.raises(ValueError, match="exceeds"):
        ragged.padded_layout([16001], 16000, HOP, True, np.array([16000]))
    ragged.check_group_rates([2, 1], np.array([16000, 16000, 8000]))
    with pytest.raises(ValueError, match="different sample rates"):
        ragged.check_group_rates([2, 1], np.array([16000, 8000, 8000]))


def test_new_entry_points_are_declared_bound_and_exported():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    so = ctypes.CDLL(_lib.SO_PATH)
    for name, nargs in NEW.items():
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES and len(_lib.SIGNATURES[name][1]) == nargs, name
        assert hasattr(so, name), name
