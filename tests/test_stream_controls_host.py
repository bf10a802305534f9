"""CPU: the Python-side argument checks of DfStream.set_atten_lim / set_post_filter_beta (deepfilternet_b200.streaming)
and the C ABI of per-slot settings and LSNR output."""
import math
import os
import re

import pytest

from deepfilternet_b200 import _lib
from deepfilternet_b200.streaming import DfStream, atten_lim_arg, pf_beta_arg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["dfb_stream_set_atten_lim", "dfb_stream_set_post_filter_beta", "dfb_stream_process_lsnr", "dfb_stream_flush_lsnr",
       "dfb_stream_process_host_lsnr"]


@pytest.mark.parametrize("db,want", [(None, 0.0), (0, 0.0), (12, 12.0), (-6.5, -6.5), (float("inf"), math.inf)])
def test_atten_lim_accepts(db, want):
    assert atten_lim_arg(db) == want


@pytest.mark.parametrize("db", [float("nan"), "12", True])
def test_atten_lim_rejects(db):
    with pytest.raises(ValueError):
        atten_lim_arg(db)


@pytest.mark.parametrize("beta,want", [(0, 0.0), (0.02, 0.02), (1, 1.0)])
def test_pf_beta_accepts(beta, want):
    assert pf_beta_arg(beta) == want


@pytest.mark.parametrize("beta", [-0.01, float("nan"), float("inf"), None, "0.02", False])
def test_pf_beta_rejects(beta):
    with pytest.raises(ValueError):
        pf_beta_arg(beta)


def test_setters_validate_before_the_library():
    """Bad values and slot lists are refused in Python, before any call into the library (none is made here)."""
    s = DfStream.__new__(DfStream)
    s.batch, s._h = 4, None
    for call in (lambda: s.set_atten_lim(float("nan"), [0]), lambda: s.set_post_filter_beta(-1.0, [0]),
                 lambda: s.set_atten_lim(6.0, [4]), lambda: s.set_post_filter_beta(0.02, [1, 1]),
                 lambda: s.set_atten_lim(6.0, [0.5])):
        with pytest.raises(ValueError):
            call()


def test_new_entry_points_are_declared_and_bound():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES, name
    # the LSNR variants take the output buffers of the plain ones plus the LSNR buffer
    assert _lib.SIGNATURES["dfb_stream_process_lsnr"][1][:4] == _lib.SIGNATURES["dfb_stream_process"][1][:4]
    assert len(_lib.SIGNATURES["dfb_stream_process_host_lsnr"][1]) == len(_lib.SIGNATURES["dfb_stream_process_host"][1]) + 1
