"""CPU: the C ABI of the spectral streaming handle (dfb_stream_*_spec) and the Python-side checks of DfStream.process_spec
(deepfilternet_b200.streaming.spec_arg), which refuse a bad input before any call into the library."""
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from deepfilternet_b200 import _lib
from deepfilternet_b200.streaming import DfStream, SpecFrames, spec_arg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["dfb_stream_create_spec", "dfb_stream_process_spec", "dfb_stream_flush_spec", "dfb_stream_process_spec_host",
       "dfb_debug_analysis_erb", "dfb_debug_spec_ingest"]


def test_new_entry_points_are_declared_and_bound():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    for name in NEW:
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES, name
    # process_spec: handle, spectrum, frames, four outputs, stream; the host variant without the stream
    assert len(_lib.SIGNATURES["dfb_stream_process_spec"][1]) == 8
    assert _lib.SIGNATURES["dfb_stream_process_spec_host"][1] == _lib.SIGNATURES["dfb_stream_process_spec"][1][:-1]
    assert len(_lib.SIGNATURES["dfb_stream_flush_spec"][1]) == 6


@pytest.mark.parametrize("make", [lambda: torch.zeros((2, 3, 481), dtype=torch.complex64),
                                  lambda: np.zeros((2, 1, 481), np.complex64)])
def test_spec_arg_accepts(make):
    x = spec_arg(make(), 2, 481)
    assert isinstance(x, torch.Tensor) and x.dtype == torch.complex64 and x.is_contiguous()


@pytest.mark.parametrize("make,exc,msg", [
    (lambda: torch.zeros((2, 3, 480), dtype=torch.complex64), RuntimeError, "DF shape error: expected 481 frequency bins"),
    (lambda: torch.zeros((2, 481, 3), dtype=torch.complex64).transpose(1, 2), RuntimeError, "not contiguous"),
    (lambda: torch.zeros((2, 3, 481), dtype=torch.complex128), ValueError, "complex64"),
    (lambda: torch.zeros((2, 3, 481, 2)), ValueError, "complex64"),
    (lambda: torch.zeros((3, 3, 481), dtype=torch.complex64), ValueError, "shape"),
    (lambda: torch.zeros((2, 0, 481), dtype=torch.complex64), ValueError, "shape"),
    (lambda: torch.zeros((2, 481), dtype=torch.complex64), ValueError, "shape"),
    (lambda: [[0j]], ValueError, "tensor"),
])
def test_spec_arg_rejects(make, exc, msg):
    with pytest.raises(exc, match=msg):
        spec_arg(make(), 2, 481)


def test_process_spec_validates_before_the_library():
    """A fake handle (no library call can succeed): bad inputs raise the argument errors, an audio handle DfbError."""
    fake = SimpleNamespace(batch=2, _h=None, spectral=True, freq_bins=481)
    for bad in (torch.zeros((2, 3, 480), dtype=torch.complex64), torch.zeros((2, 3, 481))):
        with pytest.raises((RuntimeError, ValueError)) as e:
            DfStream.process_spec(fake, bad)
        assert not isinstance(e.value, _lib.DfbError)
    audio = SimpleNamespace(batch=2, _h=None, spectral=False, freq_bins=481)
    for call in (lambda: DfStream.process_spec(audio, torch.zeros((2, 3, 481), dtype=torch.complex64)),
                 lambda: DfStream.flush_spec(audio)):
        with pytest.raises(_lib.DfbError) as e:
            call()
        assert e.value.code == _lib.DFB_ERR_INVALID


def test_spec_frames_is_a_named_tuple():
    assert SpecFrames._fields == ("gains", "coefs", "lsnr", "stage")
