"""GPU: DeepFilterNet v1 (forward_v1) layer by layer against float64 (tests/model_ref64.py, its v1 section), at every shape
dfb_model_create accepts for it.

Each row of ROWS changes the shipped v1 shape (test_gpu_parity.cfg_v1) to send work down a path the shipped model does not
take (the row's comment names it).  For every row and frame count, dfb_model_forward runs once; each layer's input and
output are fetched with dfb_model_debug_fetch and the layer is recomputed in float64 from the fetched input (teacher
forcing): erb_conv0 and df_conv0 from the features with the conv's own look-ahead padding, the encoder and decoder blocks
(decoder blocks from dec_emb / d* plus the fetched pathways p*), the pathways, cemb from c1, every GRU layer from its
fetched input and its own h[t-1], dec_emb from emb, the mask from p0 and d1, lsnr, alpha and coefs.  emb_in, emb and dfc
are plain fp32 sums of gathered values (k_gather_sum) and must match an fp32 restatement bit for bit.  Everything else
must lie within its bound, element by element, K = 1; the worst err / bound of every layer is printed.  Frame counts:
shorter than the look-ahead plus the taps, and at and past the 8-frame k_conv_in tile and the 4 / 8 / 16-frame k_dwpw
tiles (NF = 128 / Fout).  Every row's enhance() must also stay within RMS 1e-4 of oracle/dfnet1_oracle.py.

Worst err / bound over all rows and frame counts on an H100 80GB HBM3 (700 W): erb_conv0 0.49, df_conv0 0.36, erb_conv1 0.026,
erb_conv2 0.072, erb_conv3 0.083, df_conv1 0.098, cemb 0.11, encoder GRU layers 0.045 / 0.038 / 0.045, DF GRU layers
0.048 / 0.038, lsnr 0.011, alpha 0.023, dec_emb 0.12, conv0p-conv3p 0.16 / 0.15 / 0.18 / 0.20, convt3 0.10, convt2
0.049, convt1 0.047, mask 0.006, coefs 0.037; emb_in, emb and dfc bit-exact; enhance() against the oracle at most RMS
6.4e-8.  No row needed a kernel or packing fix.  This file and the v1 cases of tests/test_gpu_dsp_kernels.py take 35 s
together there."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet1_oracle as O1
import model_ref64 as M
from test_gpu_gru_tc import C1, C2
from test_gpu_model_shapes import check, fetch, fetchable, forward
from test_gpu_parity import RMS_TOL, cfg_v1, rms
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, enhance, libdf
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

R3 = dataclasses.replace
# name: (config, streams)
ROWS = {
    "v1": (cfg_v1(), 2),                                                 # baseline: FFMA df_fc_out, specialised apply
    "v1_df64": (R3(cfg_v1(), nb_df=64), 2),                              # df_fc_out on the BF16x3 GEMM (N = 640)
    "v1_df128": (R3(cfg_v1(), nb_df=128), 3),                            # GEMM at N = 1280; widest c0 / df_fc_emb
    "v1_df8_la0": (R3(cfg_v1(), nb_df=8, df_lookahead=0), 2),            # smallest DF branch (Fd / 2 = 4)
    "v1_e16": (R3(cfg_v1(), nb_erb=16, emb_hidden_dim=256, df_hidden_dim=256), 2),   # H = 256; E / 4 = 4 bins; NF 16
    "v1_dense": (R3(cfg_v1(), gru_groups=1, lin_groups=1, group_shuffle=False), 2),  # identity gathers, dense GRU
    "v1_noshuffle": (R3(cfg_v1(), group_shuffle=False), 2),              # shuffles off except df_fc_emb's
    "v1_l11_la3": (R3(cfg_v1(), emb_num_layers=1, df_num_layers=1, df_lookahead=3), 2),   # one-source gather-sum
    "v1_l2_g4_lg16": (R3(cfg_v1(), emb_num_layers=2, gru_groups=4, lin_groups=16), 2),    # two-source gather-sum
}
FRAMES = [1, 2, 3, 8, 9, 17, 33, 130]


@pytest.fixture(scope="module")
def built():
    cache = {}

    def get(name):
        if name not in cache:
            cfg, _ = ROWS[name]
            sd = random_state_dict(cfg, seed=31)
            st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
            cache[name] = (cfg, sd, st, DfNet(cfg, sd, st)) + M.state64(sd)
        return cache[name]
    return get


def prev_state(h):
    """h[t-1] of every frame, 0 before the first: the state a recurrence step starts from"""
    return torch.cat([torch.zeros_like(h[:, :1]), h[:, :-1]], 1)


@pytest.mark.parametrize("T", FRAMES)
@pytest.mark.parametrize("row", list(ROWS))
def test_layers_against_float64(built, row, T):
    cfg, sd, st, model, sd64, ab = built(row)
    B = ROWS[row][1]
    E, Fd, H, C = cfg.nb_erb, cfg.nb_df, cfg.emb_hidden_dim, 64
    G, LG, shuf = cfg.gru_groups, cfg.lin_groups, cfg.group_shuffle
    audio = synth_audio(B, T * cfg.hop_size, seed=40 + T)
    _, fe, fs = df_features(audio, st, Fd, alpha=cfg.norm_alpha)
    assert fe.shape[2] == T
    m, coefs, lsnr, alpha = forward(model, cfg, fe, fs)
    for l in range(3):
        assert fetchable(model, f"y{l}") == (l < cfg.emb_num_layers)
    for l in range(2):
        assert fetchable(model, f"z{l}") == (l < cfg.df_num_layers)
    act = lambda name, F_: M.channel_last(fetch(model, name, B * T * F_ * C).reshape(B, T, F_, C))
    vec = lambda name: fetch(model, name, B * T * H).reshape(B, T, H)
    e0, e1, e2, e3 = act("e0", E), act("e1", E // 2), act("e2", E // 4), act("e3", E // 4)
    c0, c1 = act("c0", Fd), act("c1", Fd // 2)
    p0, p1, p2, p3 = act("p0", E), act("p1", E // 2), act("p2", E // 4), act("p3", E // 4)
    dec, d3, d2, d1 = act("dec_emb", E // 4), act("d3", E // 4), act("d2", E // 2), act("d1", E)
    cemb, emb_in, emb, dfc = vec("cemb"), vec("emb_in"), vec("emb"), vec("dfc")
    ys = [vec(f"y{l}") for l in range(cfg.emb_num_layers)]
    zs = [vec(f"z{l}") for l in range(cfg.df_num_layers)]
    t64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    r = {}
    check("erb_conv0", r, e0, M.v1_input_conv(sd64, ab, "enc.erb_conv0", fe.double(), 1))
    check("df_conv0", r, c0, M.v1_input_conv(sd64, ab, "enc.df_conv0", fs.double()[:, 0].permute(0, 3, 1, 2), cfg.conv_lookahead))
    check("erb_conv1", r, e1, M.v1_block(sd64, ab, "enc.erb_conv1", e0, lookahead=1, ffma=True))
    check("erb_conv2", r, e2, M.v1_block(sd64, ab, "enc.erb_conv2", e1))
    check("erb_conv3", r, e3, M.v1_block(sd64, ab, "enc.erb_conv3", e2, fstride=1))
    check("df_conv1", r, c1, M.v1_block(sd64, ab, "enc.df_conv1", c0))
    check("cemb", r, cemb, M.v1_cemb(sd64, ab, c1, LG))
    check("emb_in", r, emb_in, M.v1_emb_in(e3.permute(0, 2, 3, 1).numpy(), cemb, LG))
    x = t64(emb_in)
    for l, y in enumerate(ys):
        check(f"emb_gru.{l}", r, y, M.v1_gru_layer(sd64, ab, f"enc.emb_gru.grus.{l}", G, x, prev_state(t64(y)), C1, C2))
        x = M.v1_gru_input(t64(y), G, shuf)
    check("emb", r, emb, M.v1_layer_sum(ys, G, shuf))
    x = t64(emb)
    for l, z in enumerate(zs):
        check(f"df_gru.{l}", r, z, M.v1_gru_layer(sd64, ab, f"df_dec.df_gru.grus.{l}", G, x, prev_state(t64(z)), C1, C2))
        x = M.v1_gru_input(t64(z), G, shuf)
    check("dfc", r, dfc, M.v1_layer_sum(zs, G, shuf))
    check("lsnr", r, lsnr[..., None], M.lsnr_head(sd64, cfg, t64(emb)))
    check("alpha", r, alpha[..., None], M.alpha_head(sd64, t64(dfc)))
    check("dec_emb", r, dec, M.v1_dec_emb(sd64, ab, t64(emb), LG, shuf, E // 4))
    for n, (p, src) in enumerate(((p0, e0), (p1, e1), (p2, e2), (p3, e3))):
        check(f"conv{n}p", r, p, M.v1_block(sd64, ab, f"erb_dec.conv{n}p", src, kt=1, fstride=1))
    check("convt3", r, d3, M.v1_block(sd64, ab, "erb_dec.convt3", dec, fstride=1, path=p3))
    check("convt2", r, d2, M.v1_block(sd64, ab, "erb_dec.convt2", d3, transposed=True, path=p2, ffma=True))
    check("convt1", r, d1, M.v1_block(sd64, ab, "erb_dec.convt1", d2, transposed=True, path=p1, ffma=True))
    check("mask", r, m[:, None], M.v1_mask(sd64, ab, p0, d1))
    check("coefs", r, coefs, M.v1_coefs(sd64, ab, cfg, t64(dfc), c0, M.v1_df_out_on_gemm(cfg)))
    print(f"{row} T={T}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    bad = {k: v for k, v in r.items() if v > 1}
    assert not bad, (row, T, bad)


@pytest.mark.parametrize("row", list(ROWS))
def test_enhance_against_oracle(built, row):
    """enhance(pad=False) of every row within RMS 1e-4 of the v1 CPU oracle, as test_gpu_parity.py requires of the
    shipped shape."""
    cfg, sd, st, model, _, _ = built(row)
    audio = synth_audio(ROWS[row][1], 130 * cfg.hop_size + 77, seed=90)
    got = enhance(model, st, audio, pad=False)
    e = rms(got, O1.enhance(sd, cfg.as_dict(), audio, pad=False))
    print(f"{row}: rms {e:.3g}")
    assert e < RMS_TOL, (row, e)
