"""CPU: linked channels without the library -- the link-group layout and the reduce_mask names (deepfilternet_b200.ragged),
the CLI's --reduce-mask, and the oracle restatement of the shared mask (tests/linked_oracle.py) that the GPU tests
compare against."""
import numpy as np
import pytest
import torch

import dfnet_oracle as O
import linked_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import ragged
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.weights import random_state_dict


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean()))


def test_reduce_code():
    assert [ragged.reduce_code(r) for r in (None, "none", "max", "mean", "MEAN")] == [0, 0, 1, 2, 2]
    for bad in ("avg", 1, "", 2.0):
        with pytest.raises(ValueError):
            ragged.reduce_code(bad)


def test_link_groups():
    sizes = ragged.link_groups([2, 3, 1], [100, 100, 7, 7, 7, 5])
    assert sizes.dtype == np.int64 and sizes.flags.c_contiguous and sizes.tolist() == [2, 3, 1]
    assert ragged.link_groups(np.array([1, 1]), [5, 6]).tolist() == [1, 1]
    with pytest.raises(ValueError):     # members of one group differ in length
        ragged.link_groups([2, 1], [100, 101, 7])
    with pytest.raises(ValueError):     # sizes do not sum to the batch
        ragged.link_groups([2, 2], [100, 100, 7])
    with pytest.raises(ValueError):
        ragged.link_groups([2], [100, 100, 7])
    with pytest.raises(ValueError):
        ragged.link_groups([2, 0, 1], [100, 100, 7])
    with pytest.raises(ValueError):
        ragged.link_groups([], [100])
    assert ragged.packed_groups([(2, 1000), (1, 481), (3, 50)]).tolist() == [2, 1, 3]


def test_cli_reduce_mask():
    from deepfilternet_b200.enhance import REDUCE_MASK_CLI, cli_parser
    p = cli_parser()
    assert p.parse_args(["a.wav"]).reduce_mask == 0
    assert p.parse_args(["--reduce-mask", "2", "a.wav"]).reduce_mask == 2
    assert REDUCE_MASK_CLI == {0: None, 1: "max", 2: "mean"}
    for bad in ("3", "-1", "mean"):
        with pytest.raises(SystemExit):
            p.parse_args(["--reduce-mask", bad, "a.wav"])


@pytest.fixture(scope="module")
def dfn3():
    cfg = ModelConfig(model="deepfilternet3", conv_ch=64, conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                      lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", df_pathway_kernel_size_t=5)
    return random_state_dict(cfg, seed=41), cfg.as_dict()


def test_reduce_mask_values():
    m = torch.tensor([[0.1, 0.9], [0.3, 0.2], [0.7, 0.5], [0.4, 0.4]], dtype=torch.float32).view(4, 1, 1, 2)
    mx = LO.reduce_mask(m, 2, "max").view(4, 2)
    assert mx.tolist() == [[0.30000001192092896, 0.8999999761581421]] * 2 + [[0.699999988079071, 0.5]] * 2
    mean = LO.reduce_mask(m, 2, "mean").view(4, 2)
    want = (np.float32(0.1) + np.float32(0.3)) * (np.float32(1) / np.float32(2))
    assert mean[0, 0].item() == float(want) and torch.equal(mean[0], mean[1])
    assert LO.reduce_mask(m, 2, None) is m and LO.reduce_mask(m, 1, "max") is m


def test_oracle_none_is_the_oracle(dfn3):
    sd, cfg = dfn3
    x = synth_audio(2, 9600 + 123, seed=51)
    ref = O.enhance(sd, cfg, x)
    for r in (None, "none"):
        assert torch.equal(LO.enhance(sd, cfg, x, reduce=r), ref)
    assert torch.equal(LO.enhance(sd, cfg, x, pad=False, reduce="max", channels=1), O.enhance(sd, cfg, x, pad=False))


@pytest.mark.parametrize("channels", [2, 3])
def test_oracle_identical_channels_give_the_mono_result(dfn3, channels):
    sd, cfg = dfn3
    x = synth_audio(1, 9600 + 123, seed=52)
    mono = O.enhance(sd, cfg, x)[0]
    for r in ("max", "mean"):
        out = LO.enhance(sd, cfg, x.repeat(channels, 1), reduce=r)
        for c in range(channels):
            assert rms(out[c], mono) < 1e-7, (r, c, rms(out[c], mono))


def test_oracle_linking_changes_different_channels(dfn3):
    sd, cfg = dfn3
    x = synth_audio(2, 9600 + 123, seed=53)
    ref = O.enhance(sd, cfg, x)
    for r in ("max", "mean"):
        out, aux = LO.enhance(sd, cfg, x, reduce=r, return_all=True)
        assert torch.equal(aux["m_link"][0], aux["m_link"][1])
        for c in range(2):
            assert rms(out[c], ref[c]) > 1e-4, (r, c, rms(out[c], ref[c]))
