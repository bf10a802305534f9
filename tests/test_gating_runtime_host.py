"""CPU: the runtime gating mode's oracle (tests/gating_runtime_oracle.py) and the argument checks that run before any
library call (DfNet.set_gating_mode, gating_mode= of enhance / enhance_batch / enhance_device_ragged / DfStream, the
deepFilter command's --gating-mode)."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

import dfnet_oracle as O
import gating_runtime_oracle as GO
import linked_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import _lib, ragged
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import cli_parser, cli_settings, enhance, enhance_batch, enhance_device_ragged
from deepfilternet_b200.weights import random_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def small_cfg(ll=False):
    if ll:
        return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), conv_ch=16,
                           emb_hidden_dim=64, df_hidden_dim=64, emb_num_layers=2, df_num_layers=2, lin_groups=8, enc_lin_groups=8,
                           df_gru_skip="groupedlinear", df_pathway_kernel_size_t=5)
    return ModelConfig(model="deepfilternet3", conv_lookahead=2, df_lookahead=2, conv_ch=16, emb_hidden_dim=64, df_hidden_dim=64,
                       emb_num_layers=2, df_num_layers=2, lin_groups=8, enc_lin_groups=8, df_gru_skip="groupedlinear",
                       df_pathway_kernel_size_t=5)


@pytest.mark.parametrize("ll", [False, True])
def test_oracle_without_gating_is_the_plain_oracle(ll):
    """Thresholds that never gate (and no thresholds) give linked_oracle.enhance's output: both decoders run every frame."""
    cfg = small_cfg(ll)
    sd = random_state_dict(cfg, seed=3)
    a = synth_audio(2, 48000, seed=5)
    want = LO.enhance(sd, cfg.as_dict(), a, pad=False, reduce="mean")
    for stages in (None, (-1e9, 1e9, 1e9)):
        got = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=stages, reduce="mean")
        assert torch.allclose(got, want, atol=1e-6, rtol=0), stages


def test_oracle_runs_no_decoder_on_fully_gated_streams(monkeypatch):
    """Every frame gated: the decoders never run, and the output is the stage rule's alone (zeros below min)."""
    cfg = small_cfg()
    sd = random_state_dict(cfg, seed=3)
    a = synth_audio(1, 24000, seed=6)
    ref = LO.enhance(sd, cfg.as_dict(), a, pad=False, stages=dict(min_db_thresh=-1e9, max_db_erb_thresh=-1e8, max_db_df_thresh=-1e8))
    calls = []
    monkeypatch.setattr(O, "erb_decoder", lambda *x, **k: calls.append("erb"))
    monkeypatch.setattr(O, "df_decoder", lambda *x, **k: calls.append("df"))
    out = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=(1e9, 2e9, 2e9))
    assert calls == [] and torch.count_nonzero(out) == 0
    out = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=(-1e9, -1e8, -1e8))   # every frame passes unprocessed
    assert calls == [] and torch.allclose(out, ref, atol=1e-6, rtol=0)


def test_oracle_decoders_see_only_their_frames():
    """The ERB decoder's masks equal apply mode's (every frame run) up to the first gated frame, and differ at run frames
    after it: the decoder's state has not seen the gated frames.  A DF decoder that never runs leaves no coefficients."""
    cfg = small_cfg()
    sd = random_state_dict(cfg, seed=4)
    a = synth_audio(1, 48000, seed=7)
    _, ref = LO.enhance(sd, cfg.as_dict(), a, pad=False, return_all=True)
    l = ref["lsnr"][0, :, 0]
    mid = float(l.sort().values[len(l) // 2])
    _, aux = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=(-1e9, mid, -1e9), return_all=True)
    e, d = aux["erb_run"][0], aux["df_run"][0]
    assert e.any() and (~e).any() and not d.any()
    g = int(torch.nonzero(~e)[0])
    m_rt, m_ap = aux["m"][0, 0], ref["m"][0, 0]
    assert torch.allclose(m_rt[:g], m_ap[:g], atol=1e-6, rtol=0)
    later = e.clone()
    later[:g + 1] = False
    assert (m_rt[later] - m_ap[later]).abs().max() > 1e-4
    assert torch.count_nonzero(aux["coefs"]) == 0
    assert GO.gated_runs(torch.tensor([True, False, True, False, False, True, False])) == [1, 2, 1]


def test_run_flags_follow_the_apply_kernel():
    """min <= lsnr <= max_erb runs the ERB decoder, and lsnr <= max_df also the DF decoder; NaN runs both (the apply
    kernel's comparisons: a NaN LSNR is stage "gains + deep filter")."""
    l = torch.tensor([-20.0, -10.0, 0.0, 20.0, 25.0, 30.0, 31.0, float("nan")])
    e, d = GO.run_flags(l, (-10.0, 30.0, 20.0))
    assert e.tolist() == [False, True, True, True, True, True, False, True]
    assert d.tolist() == [False, True, True, True, False, False, False, True]


class _Model:
    """Enough of a DfNet for the checks that run before the library is called."""
    def __init__(self):
        self.cfg = SimpleNamespace(model="deepfilternet3", nb_erb=32, nb_df=96, df_order=5)
        self.post_filter, self.post_filter_beta, self.gating_mode = False, 0.02, "apply"

    def eval(self):
        return self


@pytest.mark.parametrize("bad", ["Runtime", "tract", "", None, 1, True])
def test_bad_modes_are_refused_before_the_library(bad):
    if bad is None:
        return   # None means "the model's" wherever a mode is optional
    with pytest.raises(ValueError):
        ragged.gating_mode_code(bad)
    x = torch.zeros(1, 4800)
    with pytest.raises(ValueError):
        enhance(_Model(), None, x, gating_mode=bad)
    with pytest.raises(ValueError):
        enhance_batch(_Model(), None, [x], gating_mode=bad)
    with pytest.raises(ValueError):
        enhance_device_ragged(_Model(), None, x, [4800], gating_mode=bad)
    from deepfilternet_b200 import DfStream
    with pytest.raises(ValueError):
        DfStream(_Model(), None, gating_mode=bad)
    assert ragged.gating_mode_code("apply") == 0 and ragged.gating_mode_code("runtime") == 1


def test_cli_gating_mode():
    """--gating-mode: apply by default; runtime reaches the call only when a threshold flag turns gating on."""
    model = SimpleNamespace(cfg=SimpleNamespace(model="deepfilternet3"), post_filter_beta=0.02)
    assert cli_parser().parse_args(["x.wav"]).gating_mode == "apply"
    assert cli_settings(cli_parser().parse_args(["--gating-mode", "runtime", "x.wav"]), model) == {}
    a = cli_parser().parse_args(["--gating-mode", "runtime", "--min-db-thresh", "-10", "x.wav"])
    assert cli_settings(a, model) == {"lsnr_thresholds": (-10.0, 35.0, 35.0), "gating_mode": "runtime"}
    with pytest.raises(SystemExit):
        cli_parser().parse_args(["--gating-mode", "skip", "x.wav"])


def test_entry_points_declared_bound_and_exported():
    """The new C entry points are in include/dfb200.h, bound by _lib.SIGNATURES with their argument counts, and the
    gating mode constants match the header."""
    hdr = open(os.path.join(ROOT, "include", "dfb200.h")).read()
    for name, nargs in (("dfb_model_set_gating_mode", 2), ("dfb_stream_set_gating_mode", 2), ("dfb_debug_gru_tc_hold", 21)):
        m = re.search(r"\b" + name + r"\(([^)]*)\)", hdr)
        assert m and len(m.group(1).split(",")) == nargs, name
        assert name in _lib.SIGNATURES and len(_lib.SIGNATURES[name][1]) == nargs, name
    assert "DFB_GATING_APPLY = 0" in hdr and "DFB_GATING_RUNTIME = 1" in hdr
    assert ragged.GATING_MODES == {"apply": 0, "runtime": 1}
