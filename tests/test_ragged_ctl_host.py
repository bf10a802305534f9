"""CPU: the host side of per-entry settings and LSNR rows of ragged batches -- the dfb_enhance_settings table the batch
calls build, the combinations refused before the library is called, the LSNR row lengths, the deepFilter flags, and the
argument errors of enhance / enhance_batch / enhance_device_ragged."""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from deepfilternet_b200 import _lib, ragged
from deepfilternet_b200 import enhance_batch
from deepfilternet_b200.enhance import cli_parser, cli_settings
from deepfilternet_b200.enhance import enhance as enhance_fn

HOP = 480


class SettingsC(C.Structure):
    """include/dfb200.h dfb_enhance_settings"""
    _fields_ = [("atten_lim_db", C.c_float), ("post_filter_beta", C.c_float), ("lsnr_gating", C.c_int32),
                ("min_db_thresh", C.c_float), ("max_db_erb_thresh", C.c_float), ("max_db_df_thresh", C.c_float)]


def test_settings_dtype_is_the_c_struct():
    assert ragged.SETTINGS_DTYPE.itemsize == C.sizeof(SettingsC)
    for name, _ in SettingsC._fields_:
        assert ragged.SETTINGS_DTYPE.fields[name][1] == getattr(SettingsC, name).offset


def test_no_table_for_the_plain_call():
    for lim in (None, 6, 12.5, -3.0, np.float32(4)):
        assert ragged.settings_table(4, lim, None, None, 0.02) is None


def test_per_entry_values():
    t = ragged.settings_table(3, [None, -6, 12], None, None, 0.02)
    assert t["atten_lim_db"].tolist() == [0.0, 6.0, 12.0]          # |db|, as enhance() takes it; None is off
    assert np.allclose(t["post_filter_beta"], 0.02) and not t["lsnr_gating"].any()
    t = ragged.settings_table(3, 6.0, [0.0, 0.05, None], None, 0.0)
    assert t["atten_lim_db"].tolist() == [6.0] * 3 and np.allclose(t["post_filter_beta"], [0.0, 0.05, 0.0])
    t = ragged.settings_table(2, None, torch.tensor([0.1, 0.2]), None, 0.0)
    assert np.allclose(t["post_filter_beta"], [0.1, 0.2])
    one = ragged.settings_table(3, None, None, (-10, 30, 20), 0.0)
    assert one["lsnr_gating"].tolist() == [1, 1, 1] and one["min_db_thresh"].tolist() == [-10] * 3
    assert one["max_db_erb_thresh"].tolist() == [30] * 3 and one["max_db_df_thresh"].tolist() == [20] * 3
    assert (ragged.settings_table(3, None, None, np.array([-10.0, 30.0, 20.0]), 0.0) == one).all()
    per = ragged.settings_table(3, None, None, [(-10, 30, 20), None, np.array([-5.0, 25.0, 15.0])], 0.0)
    assert per["lsnr_gating"].tolist() == [1, 0, 1] and per["min_db_thresh"][2] == -5 and per["max_db_df_thresh"][2] == 15
    # three entries of three triples are per entry, not one triple
    per3 = ragged.settings_table(3, None, None, [(-1, 2, 3), (-4, 5, 6), (-7, 8, 9)], 0.0)
    assert per3["min_db_thresh"].tolist() == [-1, -4, -7]


@pytest.mark.parametrize("args", [
    ([1, 2], None, None),                      # wrong count
    (None, [0.1], None),
    (None, None, [(-10, 30, 20)] * 2),
    ([float("nan"), 1, 2], None, None),        # NaN limit
    ("6", None, None),
    (None, -0.1, None),                        # beta < 0 / not finite / not a number
    (None, [0, math.inf, 0], None),
    (None, "0.1", None),
    (None, None, (-10, 30)),                   # not a triple
    (None, None, (-10, float("nan"), 20)),     # NaN threshold
    (None, None, [(-10, 30, 20), (1, 2, float("nan")), None]),
])
def test_settings_errors(args):
    with pytest.raises(ValueError):
        ragged.settings_table(3, *args, 0.0)


def test_model_refusals():
    gate = ragged.settings_table(2, None, None, (-10, 30, 20), 0.0)
    beta = ragged.settings_table(2, None, [0.0, 0.02], None, 0.0)
    lim = ragged.settings_table(2, [3, 6], None, None, 0.0)
    for model in ("deepfilternet3",):
        for t in (gate, beta, lim):
            ragged.check_settings_model(model, 32, 96, 5, t, True)
    ragged.check_settings_model("deepfilternet2", 32, 96, 5, lim, True)              # the limit works on DeepFilterNet2
    ragged.check_settings_model("deepfilternet2", 32, 96, 5, ragged.settings_table(2, None, [0.0, 0.0], None, 0.0), False)
    ragged.check_settings_model("deepfilternet", 32, 96, 5, None, False)
    refused = [("deepfilternet2", 32, 96, 5, gate, False), ("deepfilternet2", 32, 96, 5, beta, False),
               ("deepfilternet", 32, 96, 5, lim, False), ("deepfilternet", 32, 96, 5, None, True),
               ("deepfilternet3", 24, 96, 5, lim, False), ("deepfilternet3", 32, 64, 5, lim, False),
               ("deepfilternet3", 32, 96, 3, lim, False)]
    for args in refused:
        with pytest.raises(_lib.DfbError) as e:
            ragged.check_settings_model(*args)
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED, args


def test_lsnr_lens():
    """ceil(out48 / hop): with pad the 48 kHz length's hops, partial last hop included; without, its whole hops."""
    lens = np.array([1, 479, 480, 481, 4801, 48000])
    assert ragged.lsnr_lens(lens, 48000, HOP, True).tolist() == [1, 1, 1, 2, 11, 100]
    assert ragged.lsnr_lens(lens, 48000, HOP, False).tolist() == [0, 0, 1, 1, 10, 100]
    # at 16 kHz: ceil(T * 3) samples at 48 kHz; at 44.1 kHz: ceil(T * 160 / 147)
    assert ragged.lsnr_lens(np.array([160, 161, 16000]), 16000, HOP, True).tolist() == [1, 2, 100]
    assert ragged.lsnr_lens(np.array([441, 44100, 44101]), 44100, HOP, True).tolist() == [1, 100, 101]
    r = np.array([48000, 16000, 8000])
    assert ragged.lsnr_lens(np.array([4800, 1600, 800]), r, HOP, False).tolist() == [10, 10, 10]


def test_cli_flags():
    """The deep-filter binary's flag names (enhance_wav.rs): --pf-beta 0.02 and the three thresholds, which turn gating on
    when any of them is given, the others at -15 / 35 / 35 dB."""
    model = SimpleNamespace(cfg=SimpleNamespace(model="deepfilternet3"), post_filter_beta=0.02)
    a = cli_parser().parse_args(["x.wav"])
    assert a.pf_beta == 0.02 and cli_settings(a, model) == {}
    a = cli_parser().parse_args(["--min-db-thresh", "-20", "x.wav"])
    assert cli_settings(a, model) == {"lsnr_thresholds": (-20.0, 35.0, 35.0)}
    a = cli_parser().parse_args(["--max-db-erb-thresh", "40", "--max-db-df-thresh", "-1", "x.wav"])
    assert cli_settings(a, model) == {"lsnr_thresholds": (-15.0, 40.0, -1.0)}
    a = cli_parser().parse_args(["--pf", "--pf-beta", "0.05", "x.wav"])
    assert cli_settings(a, model) == {"post_filter_beta": 0.05}
    assert cli_settings(cli_parser().parse_args(["--pf", "x.wav"]), model) == {}     # the model's beta: the plain call
    assert cli_settings(cli_parser().parse_args(["--pf-beta", "0.05", "x.wav"]), model) == {}   # without --pf: no post filter
    dfn2 = SimpleNamespace(cfg=SimpleNamespace(model="deepfilternet2"), post_filter_beta=0.02)
    assert cli_settings(cli_parser().parse_args(["--pf", "--pf-beta", "0.05", "x.wav"]), dfn2) == {}


class _Model:
    """Enough of a DfNet for the argument checks that run before the library is called."""
    def __init__(self, kind="deepfilternet3", post_filter=False):
        self.cfg = SimpleNamespace(model=kind, nb_erb=32, nb_df=96, df_order=5)
        self.post_filter, self.post_filter_beta = post_filter, 0.02

    def eval(self):
        return self


def test_python_argument_errors():
    a = [torch.zeros(1, 4800), torch.zeros(2, 960)]
    with pytest.raises(ValueError):
        enhance_batch(_Model(), None, a, atten_lim_db=[1, 2, 3])
    with pytest.raises(ValueError):
        enhance_batch(_Model(), None, a, lsnr_thresholds=(1, 2))
    with pytest.raises(ValueError):
        enhance_batch(_Model(), None, a, post_filter_beta=[0.1, float("nan")])
    for kw in (dict(post_filter_beta=0.1), dict(lsnr_thresholds=(-10, 30, 20))):
        with pytest.raises(_lib.DfbError) as e:
            enhance_batch(_Model("deepfilternet2"), None, a, **kw)
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError):
        enhance_batch(_Model("deepfilternet"), None, a, return_lsnr=True)
    # enhance() takes one value of each
    with pytest.raises(ValueError):
        enhance_fn(_Model(), None, a[0], atten_lim_db=[1.0])
    with pytest.raises(ValueError):
        enhance_fn(_Model(), None, a[0], post_filter_beta=[0.1])
    with pytest.raises(ValueError):
        enhance_fn(_Model(), None, a[0], lsnr_thresholds=[(-10, 30, 20)])
