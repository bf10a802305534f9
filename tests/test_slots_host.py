"""CPU: the Python-side validation of the slot lists of DfStream.open / close (deepfilternet_b200.streaming.slot_list)."""
import numpy as np
import pytest
import torch

from deepfilternet_b200.streaming import SLOT_CLOSING, SLOT_FREE, SLOT_OPEN, slot_list


@pytest.mark.parametrize("slots,want", [(3, [3]), ([0, 7], [0, 7]), ((5, 1), [5, 1]), (np.array([2], np.int32), [2]),
                                        (torch.tensor([6, 0]), [6, 0]), ([], []), (np.uint8(1), [1])])
def test_slot_list_accepts(slots, want):
    a = slot_list(slots, 8)
    assert a.dtype == np.int64 and a.flags.c_contiguous and a.tolist() == want


@pytest.mark.parametrize("slots,msg", [([8], "outside"), ([-1], "outside"), ([1, 4, 1], "listed twice"), ([1.0], "integers"),
                                       ([True], "integers"), (["1"], "integers"), ([[1, 2]], "flat")])
def test_slot_list_rejects(slots, msg):
    with pytest.raises(ValueError, match=msg):
        slot_list(slots, 8)


def test_slot_state_codes_match_the_c_abi():
    assert (SLOT_FREE, SLOT_OPEN, SLOT_CLOSING) == (0, 1, 2)   # dfb_stream_slot_states
