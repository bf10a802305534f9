"""Float64 restatement of the DNN's convolution layers and heads, with an element-wise error bound for the kernels that
evaluate each.

Every function takes the fp32 values a kernel reads (promoted to float64, in the oracle's [B, C, T, F] layout) and returns
  (reference value in float64, bound)
so that |device result - reference| <= bound element by element.  The reference is oracle/dfnet_oracle.py on the float64
state dict (BatchNorm unfolded); the bound is built from the absolute-value chain of the layer (the same layer on |x|,
|w| and the folded |BN scale| / |BN bias|, without activations):
  * FFMA layers (input convs, mask head, N = 1 heads): gamma_{n+1} * chain for n products per output, the extra rounding
    being the host's fp32 rounding of the folded weights (deepfilternet_b200/weights.py);
  * BF16x3 tensor-core contractions (separable blocks' 1x1 convs, grouped linears, DF pathway conv): bf16x3_bound(chain);
  * a sigmoid output: its argument's bound times 1/4 (the sigmoid's largest slope), plus 4 u of the value (expf, add,
    divide).
DeepFilterNet v1 has its own section at the end (oracle/dfnet1_oracle.py, the same convention).
numpy / torch on the CPU only.
"""
import numpy as np
import torch
import torch.nn.functional as F

import dfnet1_oracle as O1
import dfnet_oracle as O
from dsp_ref64 import U, gamma

# BF16x3 products (hi * hi + hi * lo + lo * hi, ~2^-16 relative each) accumulated in fp32, BN folded in fp32: the relative
# bound the tensor-core kernels meet against the absolute-value chain of the contraction
BF16X3_REL, BF16X3_ABS = 4e-5, 1e-6


def bf16x3_bound(chain):
    return BF16X3_REL * chain + BF16X3_ABS


def state64(sd):
    """(float64 state dict, its absolute-value twin): in the twin every weight is |w| and every BatchNorm computes
    x * |scale| + |beta - mean * scale|, so O.conv_norm_act(|x|, abs_sd, p, act="none") is layer p's absolute-value chain."""
    sd64 = {k: v.double() for k, v in sd.items()}
    ab = {k: v.abs() for k, v in sd64.items()}
    for k in sd64:
        if k.endswith(".running_mean"):
            p = k[:-len(".running_mean")]
            s = sd64[p + ".weight"] / torch.sqrt(sd64[p + ".running_var"] + 1e-5)
            ab[p + ".weight"] = s.abs()
            ab[p + ".bias"] = (sd64[p + ".bias"] - sd64[p + ".running_mean"] * s).abs()
            ab[p + ".running_mean"] = torch.zeros_like(s)
            ab[p + ".running_var"] = torch.full_like(s, 1 - 1e-5)
    return sd64, ab


def channel_last(x):
    """device layout [B, T, F, C] -> oracle layout [B, C, T, F], float64"""
    return torch.as_tensor(np.asarray(x, np.float64)).permute(0, 3, 1, 2)


def shift(x, lookahead):
    """the look-ahead shift of the input features, ConstantPad2d((0, 0, -la, la)) (deepfilternet3.py:359,409-410)"""
    out = torch.zeros_like(x)
    out[:, :, :max(x.shape[2] - lookahead, 0)] = x[:, :, lookahead:]
    return out


def _n_taps(sd, prefix):
    w = sd[f"{prefix}.{O._seq_entries(sd, prefix)[0][0]}.weight"]
    return w.shape[1] * w.shape[2] * w.shape[3]


def input_conv(sd, ab, prefix, x):
    """erb_conv0 (x = shifted feat_erb [B,1,T,E]) / df_conv0 (x = shifted feat_spec [B,2,T,Fd]): k_conv_in, FFMA.
    df_conv0's grouped conv and 1x1 are composed into one 2 x kt x 3 tap conv on the host, whose weights the chain bounds."""
    ref = O.conv_norm_act(x, sd, prefix)
    chain = O.conv_norm_act(x.abs(), ab, prefix, act="none")
    n = _n_taps(sd, prefix) * (x.shape[1] if prefix.endswith("df_conv0") else 1)
    return ref, gamma(n + 2) * chain


def pathway(sd, ab, prefix, x):
    """relu(conv_p(x)): the decoders' depthwise 1x1 pathway (value, absolute value chain)"""
    return O.conv_norm_act(x, sd, prefix), O.conv_norm_act(x.abs(), ab, prefix, act="none")


def block(sd, ab, prefix, x, fstride=1, transposed=False, path=None):
    """separable block (depthwise kt x 3 -> 1x1 -> BN -> ReLU) on x (+ relu(path conv) for the decoder blocks: path is
    (prefix, tensor)): k_dwpw_bx, FFMA depthwise prologue and BF16x3 1x1 conv"""
    xa = x.abs()
    if path is not None:
        p, pa = pathway(sd, ab, *path)
        x, xa = x + p, xa + pa
    ref = O.conv_norm_act(x, sd, prefix, fstride=fstride, transposed=transposed)
    chain = O.conv_norm_act(xa, ab, prefix, fstride=fstride, act="none", transposed=transposed)
    return ref, bf16x3_bound(chain)


def df_emb(sd, ab, c0, e3=None):
    """emb_in's DF half relu(df_fc_emb(df_conv1(c0))), + e3 when the two are summed (DeepFilterNet3), [B,T,ED]
    (deepfilternet3.py:175-183): the fused k_dwpw_gl, or df_conv1 on k_dwpw_bx followed by a grouped linear.  Two BF16x3
    contractions, c1's bound carried through |W|; the result is compared as the BF16 hi + lo planes the GRU projection
    reads (2^-16 of the value)."""
    flat = lambda x: x.permute(0, 2, 3, 1).flatten(2)
    c1, b_c1 = block(sd, ab, "enc.df_conv1", c0, fstride=2)
    w, wa = sd["enc.df_fc_emb.0.weight"], ab["enc.df_fc_emb.0.weight"]
    ref = torch.relu(O.grouped_linear(flat(c1), w))
    bound = bf16x3_bound(O.grouped_linear(flat(c1.abs()), wa)) + O.grouped_linear(flat(b_c1), wa)
    if e3 is not None:
        ref = ref + flat(e3)
        bound = bound + U * ref.abs()
    return ref, bound + 2.0 ** -16 * ref.abs()


def mask_head(sd, ab, e0, d1, b_d1=None):
    """m = sigmoid(conv0_out(relu(conv0p(e0)) + d1)) [B,1,T,E] (deepfilternet3.py:253), k_mask_out or the fused epilogue
    of convt1 (FFMA).  b_d1: bound of d1 when d1 itself is a float64 reference (fused head), carried through |w|."""
    p, pa = pathway(sd, ab, "erb_dec.conv0p", e0)
    x = p + d1
    ref = O.conv_norm_act(x, sd, "erb_dec.conv0_out", act="sigmoid")
    chain = O.conv_norm_act(pa + d1.abs(), ab, "erb_dec.conv0_out", act="none")
    arg = gamma(_n_taps(sd, "erb_dec.conv0_out") + 2) * chain
    if b_d1 is not None:
        bias = ab[f"erb_dec.conv0_out.{O._seq_entries(sd, 'erb_dec.conv0_out')[-1][0]}.bias"].view(1, -1, 1, 1)
        arg = arg + O.conv_norm_act(b_d1, ab, "erb_dec.conv0_out", act="none") - bias
    return ref, 0.25 * arg + 4 * U * ref


def sigmoid_head(x, w, b):
    """sigmoid(x @ w.T + b) for x [B,T,K], w [1,K]: k_grouped_linear with N = 1 (FFMA)"""
    z = x @ w.T + b
    s = torch.sigmoid(z)
    return s, 0.25 * gamma(x.shape[-1] + 2) * (x.abs() @ w.abs().T + b.abs()) + 4 * U * s


def lsnr_head(sd, cfg, emb):
    """enc.lsnr_fc: sigmoid(emb @ w.T + b) * (lsnr_max - lsnr_min) + lsnr_min [B,T,1]"""
    s, bs = sigmoid_head(emb, sd["enc.lsnr_fc.0.weight"], sd["enc.lsnr_fc.0.bias"])
    scale = cfg.lsnr_max - cfg.lsnr_min
    ref = s * scale + cfg.lsnr_min
    return ref, scale * bs + 2 * U * (scale * s + abs(cfg.lsnr_min))


def alpha_head(sd, dfc):
    """DeepFilterNet2's df_fc_a: sigmoid(dfc @ w.T + b) [B,T,1] (deepfilternet2.py:368)"""
    return sigmoid_head(dfc, sd["df_dec.df_fc_a.0.weight"], sd["df_dec.df_fc_a.0.bias"])


def coefs(sd, ab, cfg, dfc, c0):
    """tanh(df_out(dfc)) + relu(df_convp(c0)) [B,T,Fd,2*order] (deepfilternet3.py:323-331): k_gl_bx and k_df_convp_tc,
    both BF16x3; tanhf adds 2 u of the value, the sum one rounding"""
    B, T, _ = dfc.shape
    shape = (B, T, cfg.nb_df, 2 * cfg.df_order)
    lin = O.grouped_linear(dfc, sd["df_dec.df_out.0.weight"]).view(shape)
    lin_chain = O.grouped_linear(dfc.abs(), ab["df_dec.df_out.0.weight"]).view(shape)
    p = O.conv_norm_act(c0, sd, "df_dec.df_convp").permute(0, 2, 3, 1)
    p_chain = O.conv_norm_act(c0.abs(), ab, "df_dec.df_convp", act="none").permute(0, 2, 3, 1)
    t = torch.tanh(lin)
    ref = t + p
    return ref, bf16x3_bound(lin_chain) + 2 * U * t.abs() + bf16x3_bound(p_chain) + U * ref.abs()


# ------------------------------------------------------------------------------------------- DeepFilterNet v1 ----
# Restated with oracle/dfnet1_oracle.py on the float64 / absolute-value state dicts of state64 (v1's BatchNorms are the
# `<layer>.norm` entries; a conv's own bias, conv0_out's, is made |b| there too).  convkxf's ReLU is the identity on the
# non-negative absolute-value chain, so O1.convkxf(|x|, abs_sd, ...) is a layer's chain.  Kernels (csrc/dfb_model.cu
# forward_v1): k_conv_in for erb_conv0 / df_conv0; k_dwpw_bx for blocks without look-ahead that are not two-tap transposed,
# the FFMA k_dwpw for erb_conv1 (look-ahead 1), convt2 and convt1; the FFMA k_grouped_linear for df_fc_emb, erb_dec.fc_emb
# and the N = 1 heads; df_fc_out on k_gemm_bf16x3 where nb_df * 2 order is a multiple of 128, else k_grouped_linear;
# k_convp_v1; k_mask_out.
V1_KT = 2   # every time kernel of the v1 topology dfb_model_create builds (conv_k_enc = conv_k_dec = 2)


def ffma_dwpw_bound(chain, kt):
    """k_dwpw in fp32: the pathway add, kt x 3 depthwise taps, then 64 products + bias of the 1x1 conv with BN folded on
    the host (one more rounding): gamma of the nested sums' total length"""
    return gamma(3 * kt + 64 + 5) * chain


def v1_input_conv(sd, ab, prefix, x, lookahead):
    """erb_conv0 (x = feat_erb [B,1,T,E], look-ahead 1) / df_conv0 (x = feat_spec [B,2,T,Fd], look-ahead conv_lookahead):
    convkxf with its own time padding (kt - 1 - la, la), k_conv_in in FFMA.  df_conv0's grouped conv, 1x1 and BN are one
    2 x kt x 3 tap conv on the host, bounded by the chain of the three."""
    ref = O1.convkxf(x, sd, prefix, V1_KT, fstride=1, lookahead=lookahead)
    chain = O1.convkxf(x.abs(), ab, prefix, V1_KT, fstride=1, lookahead=lookahead)
    return ref, gamma(V1_KT * 3 * x.shape[1] + 2) * chain


def v1_block(sd, ab, prefix, x, kt=V1_KT, fstride=2, lookahead=0, transposed=False, path=None, ffma=False):
    """separable convkxf block (depthwise kt x 3 -> 1x1 -> BN -> ReLU) on x, + path (the fetched, already ReLU'd pathway
    output) for the decoder blocks.  ffma: the FFMA k_dwpw, else k_dwpw_bx (BF16x3 1x1 conv)."""
    xa = x.abs()
    if path is not None:
        x, xa = x + path, xa + path.abs()
    mode = "transposed" if transposed else "normal"
    ref = O1.convkxf(x, sd, prefix, kt, fstride=fstride, lookahead=lookahead, mode=mode)
    chain = O1.convkxf(xa, ab, prefix, kt, fstride=fstride, lookahead=lookahead, mode=mode)
    return ref, ffma_dwpw_bound(chain, kt) if ffma else bf16x3_bound(chain)


def v1_flat(x):
    """[B,C,T,F] -> [B,T,C*F]: the reference's channel-major flattening (deepfilternet.py:135-139)"""
    return x.permute(0, 2, 1, 3).flatten(2)


def group_shuffle(y, groups):
    """GroupedLinear / GroupedGRU's output interleave (modules.py:651-654, 807-812) along the last axis"""
    hs = y.shape[-1] // groups
    return y.reshape(*y.shape[:-1], hs, groups).swapaxes(-1, -2).reshape(y.shape)


def v1_cemb(sd, ab, c1, lin_groups):
    """df_fc_emb(c1 flattened channel-major) before its shuffle [B,T,H]: k_grouped_linear with bias, FFMA"""
    flat = v1_flat(c1)
    ref = O1.grouped_linear(flat, sd, "enc.df_fc_emb", lin_groups, False)
    chain = O1.grouped_linear(flat.abs(), ab, "enc.df_fc_emb", lin_groups, False)
    return ref, gamma(flat.shape[-1] // lin_groups + 2) * chain


def v1_emb_in(e3, cemb, lin_groups):
    """The GRU input e3 (channel-major) + shuffle(cemb) as k_gather_sum computes it: one fp32 add of two gathered
    values, so exact against fp32.  e3 [B,T,F8,C], cemb [B,T,H], both fp32 as fetched -> (value, zero bound)."""
    e3 = np.asarray(e3, np.float32)
    ref = np.ascontiguousarray(e3.swapaxes(-1, -2)).reshape(*e3.shape[:2], -1) + group_shuffle(np.asarray(cemb, np.float32), lin_groups)
    return ref.astype(np.float64), np.zeros(ref.shape)


def v1_layer_sum(ys, groups, shuffle):
    """GroupedGRU's output (add_outputs, modules.py:655-656): sum of the layer outputs, each but the last shuffled, added in
    layer order in fp32 as k_gather_sum does -> (value, zero bound)"""
    acc = np.zeros_like(np.asarray(ys[0], np.float32))
    for l, y in enumerate(ys):
        y = np.asarray(y, np.float32)
        acc = acc + (group_shuffle(y, groups) if shuffle and groups > 1 and l < len(ys) - 1 else y)
    return acc.astype(np.float64), np.zeros(acc.shape)


def v1_gru_input(y_prev, groups, shuffle):
    """layer l > 0's input: the previous layer's output, shuffled (modules.py:651-654); the device folds the shuffle into
    the columns of W_ih"""
    return group_shuffle(y_prev, groups) if shuffle and groups > 1 else y_prev


def v1_gru_layer(sd, ab, prefix, groups, x, prev, c1, c2):
    """One GroupedGRULayer step per frame from the kernel's own previous state (teacher forcing): x [B,T,I] the layer's
    input, prev [B,T,H] the fetched h[t-1] (0 at t = 0) -> (h[t], bound) [B,T,H].
    Bound: the recurrence bound of tests/test_gpu_gru_tc.check_teacher_forced, c1 S + c2, with S from |x proj| and the
    |W_hh| |h| products, plus the BF16x3 projection's error d_g = bf16x3_bound(|W_ih| |x| + |b_ih|) carried through the
    gates: d_n + d_r P_n / 4 + d_z / 2 (sigmoid' <= 1/4, tanh' <= 1, |h_prev - n| <= 2)."""
    B, T, I = x.shape
    H = prev.shape[-1]
    ig, hg = I // groups, H // groups
    ref, bound = torch.empty(B, T, H, dtype=torch.float64), torch.empty(B, T, H, dtype=torch.float64)
    gate = lambda v, k: v[..., k * hg:(k + 1) * hg]
    for g in range(groups):
        q = f"{prefix}.layers.{g}"
        xg, hp = x[..., g * ig:(g + 1) * ig], prev[..., g * hg:(g + 1) * hg]
        xp = xg @ sd[q + ".weight_ih_l0"].T + sd[q + ".bias_ih_l0"]
        dx = bf16x3_bound(xg.abs() @ ab[q + ".weight_ih_l0"].T + ab[q + ".bias_ih_l0"])
        hh = hp @ sd[q + ".weight_hh_l0"].T + sd[q + ".bias_hh_l0"]
        P = hp.abs() @ ab[q + ".weight_hh_l0"].T + ab[q + ".bias_hh_l0"]
        r = torch.sigmoid(gate(xp, 0) + gate(hh, 0))
        z = torch.sigmoid(gate(xp, 1) + gate(hh, 1))
        n = torch.tanh(gate(xp, 2) + r * gate(hh, 2))
        X = xp.abs()
        S = (gate(P, 2) + gate(X, 2)) + (gate(P, 0) + gate(X, 0)) * gate(P, 2) / 4 + (gate(P, 1) + gate(X, 1)) / 2
        ref[..., g * hg:(g + 1) * hg] = (1 - z) * n + z * hp
        bound[..., g * hg:(g + 1) * hg] = c1 * S + c2 + gate(dx, 2) + gate(dx, 0) * gate(P, 2) / 4 + gate(dx, 1) / 2
    return ref, bound


def v1_dec_emb(sd, ab, emb, lin_groups, shuffle, f8):
    """relu(erb_dec.fc_emb(emb)) viewed [B,C,T,F8] (deepfilternet.py:181-183): k_grouped_linear with bias, FFMA, then a
    k_gather_sum re-ordering"""
    B, T, H = emb.shape
    lin = O1.grouped_linear(emb, sd, "erb_dec.fc_emb.0", lin_groups, shuffle)
    chain = O1.grouped_linear(emb.abs(), ab, "erb_dec.fc_emb.0", lin_groups, shuffle)
    view = lambda v: v.reshape(B, T, -1, f8).permute(0, 2, 1, 3)
    return view(torch.relu(lin)), view(gamma(H // lin_groups + 2) * chain)


def v1_mask(sd, ab, p0, d1):
    """m = sigmoid(conv0_out(p0 + d1)) [B,1,T,E] (deepfilternet.py:186-188) from the fetched pathway p0 and d1: k_mask_out,
    FFMA over kt x 3 x 64 products; its argument's bound times 1/4, plus 4 u of the value"""
    ref = O1.convkxf(p0 + d1, sd, "erb_dec.conv0_out", V1_KT, fstride=1, act="sigmoid")
    chain = O1.convkxf(p0.abs() + d1.abs(), ab, "erb_dec.conv0_out", V1_KT, fstride=1)
    return ref, 0.25 * gamma(V1_KT * 3 * p0.shape[1] + 3) * chain + 4 * U * ref


def v1_coefs(sd, ab, cfg, dfc, c0, gemm):
    """tanh(df_fc_out(dfc)) + relu(df_convp(c0)) in the device layout [B,T,Fd,2 O] (deepfilternet.py:224-228): df_fc_out
    on k_gemm_bf16x3 (gemm) or k_grouped_linear (FFMA, H products + bias), tanhf within 2 ulp (4 u of the value), the
    dense 1x1 df_convp in FFMA (64 products + bias, BN folded on the host) and the sum, all in k_convp_v1"""
    B, T, H = dfc.shape
    O2, Fd = 2 * cfg.df_order, cfg.nb_df
    w, b = sd["df_dec.df_fc_out.0.weight"], sd["df_dec.df_fc_out.0.bias"]
    lin = (dfc @ w.T + b).view(B, T, O2, Fd)
    lin_chain = (dfc.abs() @ ab["df_dec.df_fc_out.0.weight"].T + ab["df_dec.df_fc_out.0.bias"]).view(B, T, O2, Fd)
    b_lin = bf16x3_bound(lin_chain) if gemm else gamma(H + 2) * lin_chain
    p = O1.convkxf(c0, sd, "df_dec.df_convp", 1).permute(0, 2, 1, 3)
    p_chain = O1.convkxf(c0.abs(), ab, "df_dec.df_convp", 1).permute(0, 2, 1, 3)
    t = torch.tanh(lin)
    ref = t + p
    bound = b_lin + 4 * U * t.abs() + gamma(c0.shape[1] + 2) * p_chain + U * ref.abs()
    return ref.permute(0, 1, 3, 2), bound.permute(0, 1, 3, 2)


def v1_df_out_on_gemm(cfg):
    """df_fc_out runs on k_gemm_bf16x3 when its N = nb_df * 2 order is a multiple of the GEMM's 128-column slice"""
    return cfg.nb_df * 2 * cfg.df_order % 128 == 0
