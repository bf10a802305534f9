"""CPU: the Python-side validation of DfStream.open_linked (deepfilternet_b200.streaming.group_list), which refuses a bad
slot list before the C call."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from deepfilternet_b200.streaming import DfStream, group_list


@pytest.mark.parametrize("slots,want", [(3, [3]), ([7, 0], [7, 0]), ((5, 1, 2), [5, 1, 2]), (np.array([2, 6], np.int32), [2, 6]),
                                        (torch.tensor([6, 0]), [6, 0]), (np.uint8(1), [1])])
def test_group_list_accepts(slots, want):
    a = group_list(slots, 8)
    assert a.dtype == np.int64 and a.flags.c_contiguous and a.tolist() == want   # channel order as given


@pytest.mark.parametrize("slots,msg", [([], "at least one"), ([8], "outside"), ([-1, 2], "outside"), ([1, 4, 1], "listed twice"),
                                       ([1.0, 2.0], "integers"), ([True], "integers"), (["1"], "integers"),
                                       ([[1, 2]], "flat")])
def test_group_list_rejects(slots, msg):
    with pytest.raises(ValueError, match=msg):
        group_list(slots, 8)


@pytest.mark.parametrize("slots", [[], [0, 0], [4], [0.5]])
def test_open_linked_validates_before_the_c_call(slots):
    fake = SimpleNamespace(batch=4, _h=None)   # no handle and no library: the call must not get that far
    with pytest.raises(ValueError):
        DfStream.open_linked(fake, slots)
