"""GPU: every model shape dfb_model_create accepts, layer by layer against float64 (tests/model_ref64.py), and the shapes it
refuses.

Each row of ROWS is a configuration that sends work down a path the shipped models do not take (the row's comment names
it).  For every row and frame count, dfb_model_forward runs once; each layer's input and output are fetched with
dfb_model_debug_fetch and the layer is recomputed in float64 from the fetched input (teacher forcing), so an error in one
layer is not diluted by the others.  |gpu - ref| <= bound element by element, K = 1; the worst err / bound of every layer
is printed.  Worst err / bound over all rows and frame counts on an H100 80GB HBM3 (700 W): erb_conv0 0.59, df_conv0
0.41, erb_conv1 0.14, erb_conv2 0.12, erb_conv3 0.18, df_emb 0.047, convt3 0.091, convt2 0.11, convt1 0.12, mask
0.010, fused convt1 + mask 0.0045, lsnr 0.12, alpha 0.043, coefs 0.053; enhance() against the oracle at most RMS 1.8e-7.
The whole file takes about 30 s there.

The df_emb check found that where df_conv1 and df_fc_emb are not fused and df_fc_emb's shape has no tensor-core geometry
(ll_e40_df104, dfn2_e56_df48_la1), the FFMA grouped linear read a c1 that df_conv1 no longer wrote (enhance() RMS 1e-3 to
3e-3 from the oracle, and chunked runs different from one-shot ones); df_conv1 now writes it there."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet_oracle as O
import dsp_ref64 as R
import model_ref64 as M
from test_gpu_parity import RMS_TOL, cfg_of, rms
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, enhance, libdf
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

R3 = dataclasses.replace
# name: (config, streams).  Tile geometry of k_dwpw_bx: NF = 128 // Fout frames per tile for Fout = E, E / 2, E / 4.
ROWS = {
    "dfn3": (cfg_of("dfn3"), 2),                                    # shipped baseline: fused mask head, fused df_emb
    "dfn3_ll": (cfg_of("ll"), 2),                                   # k_mask_out at kt = 2, the kt = 2 block instances
    "dfn2": (cfg_of("dfn2"), 2),                                    # alpha head, e3 at the row stride 2 ED (enc_concat)
    "e24": (R3(cfg_of("dfn3"), nb_erb=24), 2),                      # k_mask_out at kt = 1; NF 5 / 10 / 21; unfused df_emb
    "e48_df64_inp1": (R3(cfg_of("dfn3"), nb_erb=48, nb_df=64, conv_kernel_inp=(1, 3)), 2),   # one-tap k_conv_in; 96-row tiles
    "e64_df128_inp2": (R3(cfg_of("dfn3"), nb_erb=64, nb_df=128, conv_kernel_inp=(2, 3)), 3),  # fused mask at NF = 2; two taps
    "ll_e8_df16": (R3(cfg_of("ll"), nb_erb=8, nb_df=16, lin_groups=8), 2),        # Fout 2, NF 64; the smallest DF branch
    "ll_e40_df104": (R3(cfg_of("ll"), nb_erb=40, nb_df=104, lin_groups=4), 2),    # NF 3 / 6 / 12; FFMA df_fc_emb
    "dfn2_e56_df48_la1": (R3(cfg_of("dfn2"), nb_erb=56, nb_df=48, conv_lookahead=1, df_lookahead=1), 2),  # look-ahead 1; FFMA df_fc_emb
    "e16_h512": (R3(cfg_of("dfn3"), nb_erb=16, emb_hidden_dim=512, df_hidden_dim=512), 2),  # H = 512 at E = 16, fused mask
}
FRAMES = [1, 9, 33, 130]
# df_out (Hd -> nb_df * 2 order) has no tensor-core geometry at these widths and runs on the FFMA grouped linear, which
# reads the fp32 dfc
FFMA_DF_OUT = {"e64_df128_inp2", "ll_e40_df104"}
# df_conv1 -> df_fc_emb is not fused into k_dwpw_gl at these shapes (df_emb_geometry): df_conv1 on k_dwpw_bx, then the
# grouped linear on whichever kernel takes its shape
UNFUSED_EMB = {"e24", "ll_e40_df104", "dfn2_e56_df48_la1"}


def fused_mask(cfg):
    """convt1's epilogue evaluates the mask head (d1 never written) for kt = 1 and E dividing the 128-row tile"""
    return cfg.conv_kernel[0] == 1 and 128 % cfg.nb_erb == 0


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


def fetch(model, name, n):
    out = np.empty(n, dtype=np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), out.ctypes.data, out.size)
    assert got == out.size, (name, got, out.size)
    return out


def fetchable(model, name):
    scratch = np.empty(1, np.float32)
    return _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), scratch.ctypes.data, 1) == 1


def planes(hi, lo):
    """BF16 hi / lo bit patterns (uint16) -> float64 hi + lo"""
    f = lambda u: (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f(hi) + f(lo)


def forward(model, cfg, fe, fs):
    """dfb_model_forward on the device: m [B,T,E], coefs [B,T,Fd,2 O], lsnr [B,T], alpha [B,T]"""
    B, _, T, E = fe.shape
    d_fe, d_fs = fe.cuda().contiguous(), fs.cuda().contiguous()
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")
    m, c, l, a = nan(B, T, E), nan(B, T, cfg.nb_df, 2 * cfg.df_order), nan(B, T), nan(B, T)
    _lib.check(_lib.lib().dfb_model_forward(model.handle, d_fe.data_ptr(), d_fs.data_ptr(), B, T, m.data_ptr(), c.data_ptr(),
                                            l.data_ptr(), a.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return m.cpu().double(), c.cpu().double(), l.cpu().double(), a.cpu().double()


def check(name, ratios, got, ref_bound):
    ref, bound = ref_bound
    got = np.asarray(got, np.float64)
    ref, bound = np.asarray(ref, np.float64), np.asarray(bound, np.float64)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert np.isfinite(got).all(), name
    ratios[name] = R.err_ratio(got, ref, bound)


@pytest.mark.parametrize("T", FRAMES)
@pytest.mark.parametrize("row", list(ROWS))
def test_layers_against_float64(built, row, T):
    """Teacher-forced layers of one forward pass: erb_conv0, df_conv0, erb_conv1-3, df_conv1 + df_fc_emb (fused or not),
    convt3, convt2, convt1 (+ the mask head, fused or k_mask_out), the LSNR head, df_out + df_convp, DeepFilterNet2's alpha
    head.  Also asserts the path the row claims: d1 is fetchable exactly when the mask head is not fused, emb_in exactly when df_emb is not fused, the fp32
    dfc exactly when df_out runs on the FFMA kernel (or DeepFilterNet2's alpha head reads it)."""
    cfg, sd, st, model, sd64, ab = built(row)
    B = ROWS[row][1]
    E, Fd, C = cfg.nb_erb, cfg.nb_df, 64
    ED = E // 4 * C
    audio = synth_audio(B, T * cfg.hop_size, seed=40 + T)
    _, fe, fs = df_features(audio, st, Fd, alpha=cfg.norm_alpha)
    assert fe.shape[2] == T
    m, coefs, lsnr, alpha = forward(model, cfg, fe, fs)
    assert fetchable(model, "d1") != fused_mask(cfg)
    assert fetchable(model, "dfc") == (cfg.model == "deepfilternet2" or row in FFMA_DF_OUT)
    assert fetchable(model, "emb_in") == (row in UNFUSED_EMB)
    act = lambda name, F_: M.channel_last(fetch(model, name, B * T * F_ * C).reshape(B, T, F_, C))
    e0, e1, e2, c0 = act("e0", E), act("e1", E // 2), act("e2", E // 4), act("c0", Fd)
    e3w = 2 * ED if cfg.enc_concat else ED   # DeepFilterNet2: e3 is the first half of each emb_in row
    e3 = M.channel_last(fetch(model, "e3", B * T * e3w).reshape(B, T, e3w)[:, :, :ED].reshape(B, T, E // 4, C))
    dec_emb, d3, d2 = act("dec_emb", E // 4), act("d3", E // 4), act("d2", E // 2)
    emb_dim = cfg.emb_hidden_dim if cfg.model == "deepfilternet2" else ED
    emb = torch.from_numpy(fetch(model, "emb", B * T * emb_dim).reshape(B, T, emb_dim)).double()
    r = {}
    la = cfg.conv_lookahead
    check("erb_conv0", r, e0, M.input_conv(sd64, ab, "enc.erb_conv0", M.shift(fe.double(), la)))
    check("df_conv0", r, c0, M.input_conv(sd64, ab, "enc.df_conv0", M.shift(fs.double()[:, 0].permute(0, 3, 1, 2), la)))
    check("erb_conv1", r, e1, M.block(sd64, ab, "enc.erb_conv1", e0, fstride=2))
    check("erb_conv2", r, e2, M.block(sd64, ab, "enc.erb_conv2", e1, fstride=2))
    check("erb_conv3", r, e3, M.block(sd64, ab, "enc.erb_conv3", e2))
    D = 2 * ED if cfg.enc_concat else ED
    hi, lo = (fetch(model, f"emb_in_{p}", B * T * D // 2).view(np.uint16).reshape(B, T, D) for p in ("hi", "lo"))
    emb_in = planes(hi, lo)
    if cfg.enc_concat:
        check("df_emb", r, emb_in[..., ED:], M.df_emb(sd64, ab, c0))
    else:
        check("df_emb", r, emb_in, M.df_emb(sd64, ab, c0, e3))
    check("convt3", r, d3, M.block(sd64, ab, "erb_dec.convt3", dec_emb, path=("erb_dec.conv3p", e3)))
    check("convt2", r, d2, M.block(sd64, ab, "erb_dec.convt2", d3, fstride=2, transposed=True, path=("erb_dec.conv2p", e2)))
    d1_ref = M.block(sd64, ab, "erb_dec.convt1", d2, fstride=2, transposed=True, path=("erb_dec.conv1p", e1))
    if fused_mask(cfg):
        check("convt1+mask", r, m[:, None], M.mask_head(sd64, ab, e0, *d1_ref))
    else:
        d1 = act("d1", E)
        check("convt1", r, d1, d1_ref)
        check("mask", r, m[:, None], M.mask_head(sd64, ab, e0, d1))
    check("lsnr", r, lsnr[..., None], M.lsnr_head(sd64, cfg, emb))
    if fetchable(model, "dfc"):
        dfc = torch.from_numpy(fetch(model, "dfc", B * T * cfg.df_hidden_dim).reshape(B, T, -1)).double()
    else:   # the DF GRU's output (+ skip) exists only as the BF16 planes df_out reads: hi + lo is the value it multiplies
        n = B * T * cfg.df_hidden_dim
        hi, lo = (fetch(model, f"dfc_{p}", n // 2).view(np.uint16).reshape(B, T, -1) for p in ("hi", "lo"))
        dfc = torch.from_numpy(planes(hi, lo))
    if cfg.model == "deepfilternet2":
        check("alpha", r, alpha[..., None], M.alpha_head(sd64, dfc))
    check("coefs", r, coefs, M.coefs(sd64, ab, cfg, dfc, c0))
    print(f"{row} T={T}: " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    bad = {k: v for k, v in r.items() if v > 1}
    assert not bad, (row, T, bad)


@pytest.mark.parametrize("row", list(ROWS))
def test_enhance_against_oracle(built, row):
    """enhance(pad=False) of every row within RMS 1e-4 of the CPU oracle, as test_gpu_parity.py requires of the shipped
    models."""
    cfg, sd, st, model, _, _ = built(row)
    audio = synth_audio(ROWS[row][1], 130 * cfg.hop_size + 77, seed=90)
    got = enhance(model, st, audio, pad=False)
    e = rms(got, O.enhance(sd, cfg.as_dict(), audio, pad=False))
    print(f"{row}: rms {e:.3g}")
    assert e < RMS_TOL, (row, e)


# ----------------------------------------------------------------------------------------------------- refusals ----
@pytest.mark.parametrize("change,match", [
    (dict(conv_lookahead=-1), "look-ahead"), (dict(df_lookahead=-1), "look-ahead"),
    (dict(conv_lookahead=4), "look-ahead"), (dict(df_lookahead=4), "look-ahead"),
    (dict(nb_erb=8, nb_df=16), "group width"),   # df_out: 160 outputs in 16 groups of 10
])
def test_refused_shapes(change, match, monkeypatch):
    """Shapes the kernels do not build are refused at creation, by the Python layer before it calls the library and by
    dfb_model_create itself (DFB_ERR_UNSUPPORTED, naming what is built)."""
    from deepfilternet_b200 import model as model_module
    cfg = R3(cfg_of("ll"), **change)
    sd = random_state_dict(R3(cfg, conv_lookahead=0, df_lookahead=0), seed=1)
    st = libdf.DF(48000, 960, 480, cfg.nb_erb, 2)
    with pytest.raises(NotImplementedError, match=match):
        DfNet(cfg, sd, st)
    monkeypatch.setattr(model_module, "check_model_shape", lambda *a: None)
    with pytest.raises(_lib.DfbError) as e:
        DfNet(cfg, sd, st)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED and match in str(e.value), str(e.value)


@pytest.mark.parametrize("change", [dict(df_order=4), dict(df_pathway_kernel_size_t=6)])
def test_df_pathway_refused_at_first_forward(change):
    """df_order != 5 and df_pathway_kernel_size_t outside 1..5 are accepted at creation and refused by the first forward
    pass (DFB_ERR_UNSUPPORTED naming the built kernels), by design: their weights bind only when the pathway conv is built."""
    cfg = R3(cfg_of("dfn3"), **change)
    st = libdf.DF(48000, 960, 480, 32, 2)
    model = DfNet(cfg, random_state_dict(cfg, seed=2), st)
    _, fe, fs = df_features(synth_audio(1, 9 * 480, seed=3), st, cfg.nb_df, alpha=cfg.norm_alpha)
    with pytest.raises(_lib.DfbError) as e:
        forward(model, cfg, fe, fs)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED and "built kernels" in str(e.value)
