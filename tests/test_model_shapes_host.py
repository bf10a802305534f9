"""CPU: the element-wise bounds of tests/model_ref64.py, which tests/test_gpu_model_shapes.py holds the DNN's layers to, reject
plausible kernel mistakes.  Each mistake is applied to the float64 reference on the same inputs; its worst err / bound
must exceed 1, while the reference rounded to fp32 stays within the bound.  Shipped baseline (32 ERB bands, kt = 1) and
one non-32 row (24 bands, NF = 5 / 10 / 21 tiles); DeepFilterNet v1's shipped shape (model_ref64's v1 section)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dfnet1_oracle as O1
import dfnet_oracle as O
import dsp_ref64 as R
import model_ref64 as M
from deepfilternet_b200.config import ModelConfig, check_model_shape
from deepfilternet_b200.weights import random_state_dict
from test_gpu_gru_tc import C1, C2    # the GRU recurrence bound's constants

B, T = 2, 33


def ratio(got, ref_bound):
    ref, bound = ref_bound
    return R.err_ratio(got.numpy(), ref.numpy(), bound.numpy())


def conv_index(sd, prefix, i=0):
    """name of the i-th conv weight of a Conv2dNormAct sequence"""
    return f"{prefix}.{[k for k, kind in O._seq_entries(sd, prefix) if kind == 'conv'][i]}.weight"


def mutated(sd, name, fn):
    sd = dict(sd)
    sd[name] = fn(sd[name].clone())
    return sd


def replicate_edges(x):
    """the f = -1 / f = F padding taps read the edge bins instead of zeros: pad with the neighbouring bin, run the conv
    (which pads with zeros outside), crop"""
    return F.pad(x, (1, 1, 0, 0), mode="replicate")


@pytest.fixture(scope="module", params=[32, 24], ids=["e32", "e24"])
def row(request):
    cfg = ModelConfig(model="deepfilternet3", nb_erb=request.param, conv_ch=64, df_pathway_kernel_size_t=5, conv_lookahead=2,
                      df_lookahead=2, emb_num_layers=3, df_num_layers=2, lin_groups=16, enc_lin_groups=32,
                      df_gru_skip="groupedlinear")
    sd64, ab = M.state64(random_state_dict(cfg, seed=31))
    g = torch.Generator().manual_seed(request.param)
    E = cfg.nb_erb
    act = lambda f: torch.relu(torch.randn(B, 64, T, f, generator=g, dtype=torch.float64))
    x = dict(fe=torch.randn(B, 1, T, E, generator=g, dtype=torch.float64), e0=act(E), e1=act(E // 2), e2=act(E // 4),
             e3=act(E // 4), dec=act(E // 4), d3=act(E // 4), d1=act(E))
    return cfg, sd64, ab, x


def test_fp32_rounding_of_reference_meets_bounds(row):
    """The bounds are not below fp32 resolution: the float64 reference rounded to fp32 meets every one of them."""
    cfg, sd, ab, x = row
    for rb in (M.input_conv(sd, ab, "enc.erb_conv0", x["fe"]), M.block(sd, ab, "enc.erb_conv1", x["e0"], fstride=2),
               M.block(sd, ab, "erb_dec.convt3", x["dec"], path=("erb_dec.conv3p", x["e3"])),
               M.block(sd, ab, "erb_dec.convt2", x["d3"], fstride=2, transposed=True, path=("erb_dec.conv2p", x["e2"])),
               M.mask_head(sd, ab, x["e0"], x["d1"])):
        assert ratio(rb[0].float().double(), rb) <= 1


def test_time_tap_shifted_by_one_frame(row):
    """erb_conv0's current-frame tap reads the previous frame (k_conv_in's staged rows off by one)."""
    cfg, sd, ab, x = row
    name = conv_index(sd, "enc.erb_conv0")

    def shift_tap(w):
        w[:, :, -2] += w[:, :, -1]
        w[:, :, -1] = 0
        return w
    ref = M.input_conv(sd, ab, "enc.erb_conv0", x["fe"])
    assert ratio(O.conv_norm_act(x["fe"], mutated(sd, name, shift_tap), "enc.erb_conv0"), ref) > 1


def test_padding_tap_reads_neighbouring_bin(row):
    """The f = -1 and f = F taps read the edge bins instead of zeros: the input conv, a stride-1 block, the mask head."""
    cfg, sd, ab, x = row
    ref = M.input_conv(sd, ab, "enc.erb_conv0", x["fe"])
    assert ratio(O.conv_norm_act(replicate_edges(x["fe"]), sd, "enc.erb_conv0")[..., 1:-1], ref) > 1
    ref = M.block(sd, ab, "enc.erb_conv3", x["e2"])
    assert ratio(O.conv_norm_act(replicate_edges(x["e2"]), sd, "enc.erb_conv3")[..., 1:-1], ref) > 1
    ref = M.mask_head(sd, ab, x["e0"], x["d1"])
    xin = O.conv_norm_act(x["e0"], sd, "erb_dec.conv0p") + x["d1"]
    assert ratio(O.conv_norm_act(replicate_edges(xin), sd, "erb_dec.conv0_out", act="sigmoid")[..., 1:-1], ref) > 1


def test_pathway_relu_dropped(row):
    """convt3's input is dec_emb + conv3p(e3) with conv3p's ReLU left out."""
    cfg, sd, ab, x = row
    ref = M.block(sd, ab, "erb_dec.convt3", x["dec"], path=("erb_dec.conv3p", x["e3"]))
    bad = O.conv_norm_act(x["dec"] + O.conv_norm_act(x["e3"], sd, "erb_dec.conv3p", act="none"), sd, "erb_dec.convt3")
    assert ratio(bad, ref) > 1


def test_transposed_taps_swapped(row):
    """convt2 (T2): out[2j] and out[2j+1]'s outer taps exchanged."""
    cfg, sd, ab, x = row
    name = conv_index(sd, "erb_dec.convt2")
    ref = M.block(sd, ab, "erb_dec.convt2", x["d3"], fstride=2, transposed=True, path=("erb_dec.conv2p", x["e2"]))
    swapped = mutated(sd, name, lambda w: w.flip(-1))
    xin = x["d3"] + O.conv_norm_act(x["e2"], sd, "erb_dec.conv2p")
    assert ratio(O.conv_norm_act(xin, swapped, "erb_dec.convt2", fstride=2, transposed=True), ref) > 1


def test_mask_bias_dropped(row):
    """conv0_out's folded bias (BN beta - mean * scale) left out of the mask head."""
    cfg, sd, ab, x = row
    bn = f"erb_dec.conv0_out.{O._seq_entries(sd, 'erb_dec.conv0_out')[-1][0]}"
    s = sd[bn + ".weight"] / torch.sqrt(sd[bn + ".running_var"] + 1e-5)
    ref = M.mask_head(sd, ab, x["e0"], x["d1"])
    nobias = mutated(sd, bn + ".bias", lambda b: sd[bn + ".running_mean"] * s)
    assert ratio(M.mask_head(nobias, ab, x["e0"], x["d1"])[0], ref) > 1


@pytest.mark.parametrize("layer", ["erb_conv0", "erb_conv1", "mask"])
def test_one_channel_weight_perturbed(row, layer):
    """One output channel's folded weights off by 2^-12 relative: the FFMA input conv and mask head, and the BF16x3 1x1
    conv of a separable block (whose bound is 2^-14.6 of the absolute-value chain)."""
    cfg, sd, ab, x = row
    up = lambda w: torch.cat([w[:1] * (1 + 2.0 ** -12), w[1:]])
    if layer == "erb_conv0":
        name = conv_index(sd, "enc.erb_conv0")
        ref, bad = M.input_conv(sd, ab, "enc.erb_conv0", x["fe"]), M.input_conv(mutated(sd, name, up), ab, "enc.erb_conv0", x["fe"])[0]
    elif layer == "erb_conv1":
        name = conv_index(sd, "enc.erb_conv1", 1)
        ref = M.block(sd, ab, "enc.erb_conv1", x["e0"], fstride=2)
        bad = M.block(mutated(sd, name, up), ab, "enc.erb_conv1", x["e0"], fstride=2)[0]
    else:
        name = conv_index(sd, "erb_dec.conv0_out")
        ref = M.mask_head(sd, ab, x["e0"], x["d1"])
        bad = M.mask_head(mutated(sd, name, lambda w: w * (1 + 2.0 ** -12)), ab, x["e0"], x["d1"])[0]
    assert ratio(bad, ref) > 1


@pytest.mark.parametrize("model,change", [("deepfilternet3", dict(conv_lookahead=-1)), ("deepfilternet3", dict(df_lookahead=4)),
                                          ("deepfilternet2", dict(conv_lookahead=4)), ("deepfilternet", dict(conv_lookahead=3))])
def test_look_ahead_refused_before_the_library(model, change):
    """Look-aheads outside 0..3 (DeepFilterNet v1: a conv look-ahead other than 2) are refused before dfb_model_create."""
    with pytest.raises(NotImplementedError, match="look-ahead"):
        check_model_shape(ModelConfig(model=model, **change), {})
    check_model_shape(ModelConfig(model=model, conv_lookahead=2), {})


# ------------------------------------------------------------------------------------------- DeepFilterNet v1 ----
# The bounds of model_ref64's v1 section (tests/test_gpu_v1_layers.py) against the mistakes a v1 kernel or its packing
# could make: same rule, each mistake above 1, the fp32 rounding of the reference within 1.
@pytest.fixture(scope="module")
def v1():
    cfg = ModelConfig(model="deepfilternet", conv_lookahead=2, df_lookahead=1, conv_ch=64, conv_kernel=(2, 3),
                      convt_kernel=(2, 3), conv_kernel_inp=(2, 3), conv_k_enc=2, conv_k_dec=2, emb_hidden_dim=512,
                      df_hidden_dim=512, emb_num_layers=3, df_num_layers=2, gru_groups=8, lin_groups=8, group_shuffle=True)
    sd64, ab = M.state64(random_state_dict(cfg, seed=31))
    g = torch.Generator().manual_seed(1)
    E, Fd, H = cfg.nb_erb, cfg.nb_df, cfg.emb_hidden_dim
    act = lambda f: torch.relu(torch.randn(B, 64, T, f, generator=g, dtype=torch.float64))
    sym = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64) * 2 - 1
    x = dict(fe=torch.randn(B, 1, T, E, generator=g, dtype=torch.float64), fs=torch.randn(B, 2, T, Fd, generator=g, dtype=torch.float64),
             e0=act(E), c0=act(Fd), c1=act(Fd // 2), d3=act(E // 4), d2=act(E // 2), p2=act(E // 4), p1=act(E // 2), d1=act(E), p0=act(E),
             e3=act(E // 4).float(), cemb=torch.randn(B, T, H, generator=g), y0=sym(B, T, H), y1=sym(B, T, H), dfc=sym(B, T, H))
    return cfg, sd64, ab, x


def test_v1_fp32_rounding_of_reference_meets_bounds(v1):
    cfg, sd, ab, x = v1
    prev = torch.cat([torch.zeros(B, 1, 512, dtype=torch.float64), x["y1"][:, :-1]], 1)
    for rb in (M.v1_input_conv(sd, ab, "enc.erb_conv0", x["fe"], 1), M.v1_input_conv(sd, ab, "enc.df_conv0", x["fs"], 2),
               M.v1_block(sd, ab, "enc.erb_conv1", x["e0"], lookahead=1, ffma=True), M.v1_block(sd, ab, "enc.df_conv1", x["c0"]),
               M.v1_block(sd, ab, "erb_dec.convt2", x["d3"], transposed=True, path=x["p2"], ffma=True),
               M.v1_cemb(sd, ab, x["c1"], cfg.lin_groups),
               M.v1_gru_layer(sd, ab, "enc.emb_gru.grus.1", 8, M.v1_gru_input(x["y0"], 8, True), prev, C1, C2),
               M.v1_dec_emb(sd, ab, x["dfc"], cfg.lin_groups, True, 8), M.v1_mask(sd, ab, x["p0"], x["d1"]),
               M.v1_coefs(sd, ab, cfg, x["dfc"], x["c0"], gemm=False), M.v1_coefs(sd, ab, cfg, x["dfc"], x["c0"], gemm=True)):
        assert ratio(rb[0].float().double(), rb) <= 1


def test_v1_look_ahead_padding_off_by_one_frame(v1):
    """erb_conv1's look-ahead 1 and df_conv0's 2 (which crops the first frame), each taken one frame short or long."""
    cfg, sd, ab, x = v1
    ref = M.v1_block(sd, ab, "enc.erb_conv1", x["e0"], lookahead=1, ffma=True)
    for la in (0, 2):
        assert ratio(M.v1_block(sd, ab, "enc.erb_conv1", x["e0"], lookahead=la)[0], ref) > 1
    ref = M.v1_input_conv(sd, ab, "enc.df_conv0", x["fs"], 2)
    for la in (1, 3):
        assert ratio(M.v1_input_conv(sd, ab, "enc.df_conv0", x["fs"], la)[0], ref) > 1


def test_v1_transposed_taps_not_reversed(v1):
    """convt2 / convt1 (two time taps, FFMA k_dwpw) with the ConvTranspose2d's time taps used in causal order."""
    cfg, sd, ab, x = v1
    for name, inp, path in (("erb_dec.convt2", x["d3"], x["p2"]), ("erb_dec.convt1", x["d2"], x["p1"])):
        ref = M.v1_block(sd, ab, name, inp, transposed=True, path=path, ffma=True)
        bad = mutated(sd, name + ".sconvt.weight", lambda w: w.flip(2))
        assert ratio(M.v1_block(bad, ab, name, inp, transposed=True, path=path)[0], ref) > 1


def test_v1_emb_in_order(v1):
    """The GRU input e3 + shuffle(cemb), exact: e3 flattened channel-last instead of channel-major (a wrong idx_e3), or
    df_fc_emb's shuffle dropped (a wrong idx_shuf)."""
    cfg, sd, ab, x = v1
    e3 = x["e3"].permute(0, 2, 3, 1).numpy()            # device layout [B,T,F8,C]
    cemb = x["cemb"].numpy()
    rb = M.v1_emb_in(e3, cemb, cfg.lin_groups)
    assert ratio(torch.from_numpy(rb[0]), tuple(torch.from_numpy(v) for v in rb)) == 0
    channel_last = e3.reshape(B, T, -1) + M.group_shuffle(cemb, cfg.lin_groups)
    no_shuffle = np.ascontiguousarray(e3.swapaxes(-1, -2)).reshape(B, T, -1) + cemb
    for bad in (channel_last, no_shuffle):
        assert R.err_ratio(bad.astype(np.float64), *rb) > 1


def test_v1_gru_input_shuffle_dropped(v1):
    """Encoder GRU layer 1 fed the previous layer's output without the group shuffle that weights.py folds into W_ih."""
    cfg, sd, ab, x = v1
    prev = torch.cat([torch.zeros(B, 1, 512, dtype=torch.float64), x["y1"][:, :-1]], 1)
    ref = M.v1_gru_layer(sd, ab, "enc.emb_gru.grus.1", 8, M.v1_gru_input(x["y0"], 8, True), prev, C1, C2)
    assert ratio(M.v1_gru_layer(sd, ab, "enc.emb_gru.grus.1", 8, x["y0"], prev, C1, C2)[0], ref) > 1


def test_v1_alpha_blend_with_unmasked_spectrum():
    """The alpha blend taken with the noisy DF bins instead of the masked ones."""
    rng = np.random.default_rng(3)
    widths = np.full(32, 15)
    widths[-1] += 1                                      # 481 bins
    spec = ((rng.standard_normal((1, 12, 481)) + 1j * rng.standard_normal((1, 12, 481))) * 0.1)
    m = rng.random((1, 12, len(widths)))
    c = (rng.standard_normal((1, 12, 96, 5)) + 1j * rng.standard_normal((1, 12, 96, 5))) * 0.5
    alpha = rng.random((1, 12))
    ref, b = R.apply(spec, m, c, widths, mode=2, nb_df=96, order=5, lookahead=1, alpha=alpha)
    yd, _ = R.apply(spec, m, c, widths, mode=2, nb_df=96, order=5, lookahead=1)
    bad = ref.copy()
    a = alpha[..., None]
    bad[..., :96] = yd[..., :96] * a + spec[..., :96] * (1 - a)
    assert R.err_ratio(bad, ref, b) > 1


def test_v1_coefs_activation_dropped(v1):
    """df_fc_out's tanh dropped, or df_convp's ReLU dropped, at both df_fc_out kernels' bounds."""
    cfg, sd, ab, x = v1
    B_, T_, H = x["dfc"].shape
    lin = (x["dfc"] @ sd["df_dec.df_fc_out.0.weight"].T + sd["df_dec.df_fc_out.0.bias"]).view(B_, T_, 10, -1)
    p = O1.convkxf(x["c0"], sd, "df_dec.df_convp", 1).permute(0, 2, 1, 3)
    bn = "df_dec.df_convp.norm"
    s = sd[bn + ".weight"] / torch.sqrt(sd[bn + ".running_var"] + 1e-5)
    p_lin = F.conv2d(x["c0"], sd["df_dec.df_convp.sconv.weight"]) * s.view(1, -1, 1, 1) + (sd[bn + ".bias"] - sd[bn + ".running_mean"] * s).view(1, -1, 1, 1)
    p_lin = p_lin.permute(0, 2, 1, 3)
    for gemm in (False, True):
        ref = M.v1_coefs(sd, ab, cfg, x["dfc"], x["c0"], gemm)
        for bad in (lin + p, torch.tanh(lin) + p_lin):
            assert ratio(bad.permute(0, 1, 3, 2), ref) > 1
