"""CPU: the host-side layout of ragged batches (deepfilternet_b200.ragged) -- lengths, offsets, output lengths and the
errors the wrappers raise before anything reaches the device."""
import numpy as np
import pytest

from deepfilternet_b200 import ragged

HOP = 480


def test_out_len_matches_enhance():
    assert ragged.out_len(12345, HOP, True) == 12345
    assert ragged.out_len(12345, HOP, False) == 12000
    assert ragged.out_len(480, HOP, False) == 480


def test_check_lengths():
    lens = ragged.check_lengths([1, 480, 4801], HOP, True)
    assert lens.dtype == np.int64 and lens.flags.c_contiguous and lens.tolist() == [1, 480, 4801]
    assert ragged.check_lengths(np.array([[960, 961]]), HOP, False, 961).tolist() == [960, 961]
    assert ragged.check_lengths(np.arange(10)[1::3], HOP, True).flags.c_contiguous
    with pytest.raises(ValueError):
        ragged.check_lengths([480, 0], HOP, True)
    with pytest.raises(ValueError):
        ragged.check_lengths([480, -5], HOP, True)
    with pytest.raises(ValueError):
        ragged.check_lengths([], HOP, True)
    with pytest.raises(ValueError):
        ragged.check_lengths([480, 1000], HOP, True, max_len=999)
    with pytest.raises(RuntimeError):
        ragged.check_lengths([4800, 479], HOP, False)


def test_padded_layout():
    lens, in_off, out_off, ow = ragged.padded_layout([100, 1000, 481], 1000, HOP, True)
    assert lens.tolist() == [100, 1000, 481] and in_off.tolist() == [0, 1000, 2000]
    assert ow == 1000 and out_off.tolist() == [0, 1000, 2000]
    lens, in_off, out_off, ow = ragged.padded_layout([500, 1000, 960], 1000, HOP, False)
    assert ow == 960 and out_off.tolist() == [0, 960, 1920]


def test_packed_layout_at_48k():
    lens, in_off, out_off, n_in, n_out, sl, sr = ragged.packed_layout([(2, 1000), (1, 481), (3, 50)], HOP, True)
    assert lens.tolist() == [1000, 1000, 481, 50, 50, 50]
    assert sr.dtype == np.int32 and sr.tolist() == [48000] * 6
    assert in_off.tolist() == [0, 1000, 2000, 2481, 2531, 2581] and n_in == 2631
    assert out_off.tolist() == in_off.tolist() and n_out == n_in
    assert sl == [(0, 2, 1000), (2000, 1, 481), (2481, 3, 50)]
    lens, in_off, out_off, n_in, n_out, sl, _ = ragged.packed_layout([(2, 1000), (1, 481)], HOP, False)
    assert out_off.tolist() == [0, 960, 1920] and n_out == 2400 and n_in == 2481
    assert sl == [(0, 2, 960), (1920, 1, 480)]
    with pytest.raises(ValueError):
        ragged.packed_layout([(1000,)], HOP, True)
    with pytest.raises(ValueError):
        ragged.packed_layout([(0, 1000)], HOP, True)
    with pytest.raises(ValueError):
        ragged.packed_layout([(1, 1000), (1, 0)], HOP, True)
    with pytest.raises(ValueError):
        ragged.packed_layout([], HOP, True)
    with pytest.raises(RuntimeError):
        ragged.packed_layout([(1, 1000), (2, 100)], HOP, False)
