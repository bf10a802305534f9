"""GPU: the fused df_conv1 -> df_fc_emb kernel (k_dwpw_gl) element by element against a float64 restatement of
df_conv1 + df_fc_emb (+ e3), built from the c0 / e3 the forward itself produced.  The kernel writes only the BF16 hi / lo
planes of emb_in; they are fetched through the emb_in_hi / emb_in_lo debug entries and compared as hi + lo."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet_oracle as O
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict


def cfg_of(kind):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5)
    if kind == "dfn3":   # df_fc_emb: 32 groups of 96 inputs
        return ModelConfig(model="deepfilternet3", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", **base)
    if kind == "dfn2":   # 8 groups of 384, emb_in = concat(e3, cemb)
        return ModelConfig(model="deepfilternet2", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=8, enc_lin_groups=8, enc_concat=True, **base)
    # DeepFilterNet3_ll: kt = 2 (previous-frame tap), 16 groups of 192
    return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), emb_hidden_dim=512,
                       df_hidden_dim=512, emb_num_layers=3, df_num_layers=3, lin_groups=16, enc_lin_groups=16,
                       df_gru_skip="groupedlinear", **base)


def fetch(model, name, n, dtype=np.float32):
    out = np.empty(n, dtype=np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), out.ctypes.data, out.size)
    assert got == out.size, (name, got, out.size)
    return out.view(dtype)


def bf16_pair_to_f64(hi, lo):
    """BF16 bit patterns (uint16) -> float64 value hi + lo"""
    f = lambda u: (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f(hi) + f(lo)


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "dfn3_ll"])
@pytest.mark.parametrize("B,frames", [(1, 1), (2, 77), (3, 300)])
def test_df_emb_vs_float64(kind, B, frames):
    """Row counts below, at and past the row tile (128; 127 for kt = 2), a one-frame window, and every bin slice (each
    output column of emb_in's df half is checked)."""
    cfg = cfg_of(kind)
    sd = random_state_dict(cfg, seed=7)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    audio = synth_audio(B, frames * cfg.hop_size, seed=21)
    sp, fe, fs = df_features(audio, st, cfg.nb_df, alpha=cfg.norm_alpha)
    T = sp.shape[2]
    model(sp, fe, fs)
    # the fused kernel ran: it writes only emb_in's planes, so the fp32 emb_in activation is not there to fetch
    scratch = np.empty(16, np.float32)
    assert _lib.lib().dfb_model_debug_fetch(model.handle, b"emb_in", scratch.ctypes.data, scratch.size) < 0
    Fd, E, C = cfg.nb_df, cfg.nb_erb, 64
    ED = E // 4 * C
    emb_in_dim = 2 * ED if cfg.enc_concat else ED
    M = B * T
    c0 = fetch(model, "c0", M * Fd * C).reshape(B, T, Fd, C)
    hi = fetch(model, "emb_in_hi", M * emb_in_dim // 2, np.uint16).reshape(B, T, emb_in_dim)
    lo = fetch(model, "emb_in_lo", M * emb_in_dim // 2, np.uint16).reshape(B, T, emb_in_dim)
    got = bf16_pair_to_f64(hi, lo)
    # float64 restatement: df_conv1 (depthwise stride 2, 1x1, BN, ReLU) -> df_fc_emb (grouped linear, ReLU) (+ e3)
    sd64 = {k: v.double() for k, v in sd.items()}
    x = torch.from_numpy(c0).double().permute(0, 3, 1, 2)          # [B, C, T, Fd]
    c1 = O.conv_norm_act(x, sd64, "enc.df_conv1", fstride=2)        # [B, C, T, Fd / 2]
    cemb = torch.relu(O.grouped_linear(c1.permute(0, 2, 3, 1).flatten(2), sd64["enc.df_fc_emb.0.weight"])).numpy()
    if cfg.enc_concat:
        got = got[..., ED:]
        ref = cemb
    else:
        e3 = fetch(model, "e3", M * ED).reshape(B, T, ED).astype(np.float64)
        ref = cemb + e3
    assert got.shape == ref.shape
    assert np.isfinite(got).all()
    # fp32 accumulation of BF16x3 products (~2^-17 relative each) over K = 64 and K = Ig, BN folded into the 1x1 weights in
    # fp32 (measured: <= 5e-6 of max|ref|)
    tol = 2e-5 * (np.abs(ref) + np.abs(ref).max())
    bad = np.abs(got - ref) > tol
    assert not bad.any(), (int(bad.sum()), float(np.abs(got - ref).max()), float(np.abs(ref).max()))

