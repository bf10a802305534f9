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
numpy / torch on the CPU only.
"""
import numpy as np
import torch
import torch.nn.functional as F

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
