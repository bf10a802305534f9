"""Host: held sessions (DfStream.hold / held_slots, include/dfb200.h dfb_stream_hold_slots) without a GPU.  The Python
argument checks run before the library is called; the new C entry points are declared, bound and exported."""
import ctypes
import os
import re
import types

import numpy as np
import pytest

from deepfilternet_b200 import _lib
from deepfilternet_b200.streaming import DfStream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {"dfb_stream_hold_slots": 4, "dfb_stream_held_slots": 2, "dfb_debug_stream_rows_moved": 2}


def fake_handle(batch=4):
    """what DfStream.hold reads before it calls the library"""
    return types.SimpleNamespace(batch=batch, spectral=False, _h=None)


@pytest.mark.parametrize("slots", [[0, 0], [4], [-1], [0.5], [[0, 1]], np.array([1.0, 2.0])])
def test_hold_refuses_malformed_slots(slots):
    for held in (True, False):
        with pytest.raises(ValueError):
            DfStream.hold(fake_handle(), slots, held)


def test_hold_passes_the_list_and_flag_to_the_library(monkeypatch):
    seen = []

    class Lib:
        def dfb_stream_hold_slots(self, h, ptr, n, hold):
            seen.append(([ptr[i] for i in range(n)], hold))
            return 0

        def dfb_stream_held_slots(self, h, ptr):
            ptr[1] = 1
            ptr[3] = 1
            return 0

    monkeypatch.setattr(_lib, "lib", lambda: Lib())
    DfStream.hold(fake_handle(), [3, 1])
    DfStream.hold(fake_handle(), 2, held=False)
    DfStream.hold(fake_handle(), [])
    assert seen == [([3, 1], 1), ([2], 0), ([], 1)]
    got = DfStream.held_slots(fake_handle())
    assert got.dtype == bool and got.tolist() == [False, True, False, True]


def test_new_entry_points_are_declared_bound_and_exported():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    so = ctypes.CDLL(_lib.SO_PATH)
    for name, nargs in NEW.items():
        m = re.search(rf"\b{name}\s*\(([^)]*)\)", hdr)
        assert m and len(m.group(1).split(",")) == nargs, name
        assert name in _lib.SIGNATURES and len(_lib.SIGNATURES[name][1]) == nargs, name
        assert hasattr(so, name), name
