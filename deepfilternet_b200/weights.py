"""Weight packer: reference ``state_dict`` -> the flat fp32 tensors libdfb200 consumes.

Source tensor names/shapes: SURVEY.md Appendix B (dumped from the shipped checkpoints of
``DeepFilterNet/df/deepfilternet3.py`` / ``deepfilternet2.py``).  All activations on the device are
channel-last ``[B, T, F, C=64]``, so conv weights are stored tap-major with the channel fastest.
Eval-mode BatchNorm (eps 1e-5, modules.py:68-69) is folded into the bias-free conv in front of it:
``scale = gamma / sqrt(var + eps)``, ``w' = w * scale[out]``, ``b' = beta - mean * scale``.

Packed tensors (name -> layout):
  enc.erb_conv0.w   [kt][3][C]        dense 1->C conv (kt = conv_kernel_inp[0]), BN folded
  enc.erb_conv0.b   [C]
  <blk>.dw          [kt][3][C]        depthwise taps of erb_conv1-3, df_conv1, convt3 (conv) and
                                      convt2, convt1 (ConvTranspose2d taps as stored, kt = 1)
  <blk>.pw          [C_in][C_out]     1x1 conv, transposed, BN folded
  <blk>.pw_sw                         BF16 hi | lo image of the same 1x1 weight for the tensor-core kernel (umma_sw128_image)
  <blk>.b           [C]
  enc.df_conv0.w    [kt][3][2][C]     grouped 2->C conv composed with its 1x1 conv and BN (direct K = 18 conv)
  enc.df_conv0.b    [C]
  erb_dec.conv{3,2,1,0}p.s / .b  [C]  depthwise 1x1 + BN folded: relu(x * s + b)
  erb_dec.conv0_out.w [kt][3][C]      C->1 conv, BN folded;  erb_dec.conv0_out.b [1]
  df_dec.df_convp.w_sw                BF16 hi | lo image of the grouped (2) temporal conv as one 64 x 64 product
                                      (row g*32 + dt*5 + o, column = channel; zero outside group g)
  df_dec.df_convp.w2 [10][10]         1x1 (in, out), BN folded;  df_dec.df_convp.b [10]
  *.gl              [G][I/G][H/G]     GroupedLinearEinsum weight as stored (modules.py:752-757)
  *.gl_bx           BF16 hi | lo image of the same weight in the tensor-core kernel's operand layout (gl_bx_image)
  <gru>.l{n}.w_ih_t [I][3H] (transposed), .w_ih_hi / .w_ih_lo ([3H][I] BF16 planes for the projection GEMM),
                    .w_hh [3H][H], .b_ih [3H], .b_hh [3H]   torch.nn.GRU gate order (r,z,n)
  enc.lsnr.w [emb_out], enc.lsnr.b [1]
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
import torch

from .config import ModelConfig

EPS = 1e-5


def _np(t) -> np.ndarray:
    return np.ascontiguousarray(t.detach().cpu().to(torch.float32).numpy())


def _seq(sd, prefix: str) -> Tuple[List[int], List[int]]:
    idx = sorted({int(k[len(prefix) + 1:].split(".")[0]) for k in sd if k.startswith(prefix + ".")})
    convs = [i for i in idx if f"{prefix}.{i}.running_mean" not in sd]
    bns = [i for i in idx if f"{prefix}.{i}.running_mean" in sd]
    return convs, bns


def _bn_fold(sd, p: str) -> Tuple[np.ndarray, np.ndarray]:
    g, b = _np(sd[p + ".weight"]).astype(np.float64), _np(sd[p + ".bias"]).astype(np.float64)
    mu, var = _np(sd[p + ".running_mean"]).astype(np.float64), _np(sd[p + ".running_var"]).astype(np.float64)
    scale = g / np.sqrt(var + EPS)
    return scale, b - mu * scale


def bf16_planes(w: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """fp32 -> (hi, lo) BF16 planes with w ~= hi + lo (both round-to-nearest-even), each returned as a
    float32 array holding two BF16 values per element (the C ABI moves fp32 tensors only)."""
    t = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float32))
    hi = t.to(torch.bfloat16)
    lo = (t - hi.to(torch.float32)).to(torch.bfloat16)
    pack = lambda b: np.ascontiguousarray(b.contiguous().view(torch.int16).numpy().view(np.float32))
    return pack(hi), pack(lo)


def umma_sw128_image(w_nk: np.ndarray) -> np.ndarray:
    """[N][64] fp32 -> the shared-memory image of the K-major, 128-byte-swizzled tensor-core B operand: BF16 hi plane
    then lo plane, each N rows of 128 bytes with 16-byte chunk j of row n stored at chunk j ^ (n & 7)."""
    hi, lo = bf16_planes(w_nk)
    n = w_nk.shape[0]
    assert w_nk.shape[1] == 64 and n % 8 == 0
    planes = []
    for pl in (hi, lo):
        c = pl.reshape(n, 8, 4)  # [row][16-byte chunk][4 floats = 8 bf16]
        o = np.empty_like(c)
        rows = np.arange(n)
        for j in range(8):
            o[rows, j ^ (rows & 7)] = c[rows, j]
        planes.append(o.reshape(-1))
    return np.ascontiguousarray(np.concatenate(planes))


def gl_bx_image(w: np.ndarray) -> np.ndarray:
    """GroupedLinearEinsum weight [G][Ig][Hg] -> the shared-memory image of the tensor-core grouped-linear kernel's B operand
    (csrc/dfb_gl.cu): BF16 hi plane then lo plane, each [G][Ig/8][Hgp/8][8 n][8 i] -- K-major 8 x 16-byte core matrices,
    Hg zero-padded to a multiple of 16 (Hgp).  Returned as float32 words (two BF16 per element)."""
    G, Ig, Hg = w.shape
    assert Ig % 8 == 0
    Hgp = (Hg + 15) // 16 * 16
    wp = np.zeros((G, Ig, Hgp), dtype=np.float32)
    wp[:, :, :Hg] = w
    t = torch.from_numpy(wp)
    hi = t.to(torch.bfloat16)
    lo = (t - hi.to(torch.float32)).to(torch.bfloat16)
    planes = []
    for pl in (hi, lo):
        a = pl.view(torch.int16).numpy().reshape(G, Ig // 8, 8, Hgp // 8, 8)   # [g][kc][i8][rg][n8]
        planes.append(np.ascontiguousarray(a.transpose(0, 1, 3, 4, 2)).reshape(-1))  # [g][kc][rg][n8][i8]
    return np.ascontiguousarray(np.concatenate(planes)).view(np.float32)


def gru_layers(sd, prefix: str) -> int:
    n = 0
    while f"{prefix}.weight_ih_l{n}" in sd:
        n += 1
    return n


def pack_state_dict(sd: Dict[str, torch.Tensor], cfg: ModelConfig) -> Tuple[Dict[str, np.ndarray], dict]:
    """Returns (packed tensors, derived integer config for dfb_model_config)."""
    if cfg.model == "deepfilternet":
        return pack_state_dict_v1(sd, cfg)
    C = cfg.conv_ch
    out: Dict[str, np.ndarray] = {}

    def f32(a):
        return np.ascontiguousarray(np.asarray(a, dtype=np.float32))

    # --- erb_conv0: dense 1->C (kt,3) + BN
    convs, bns = _seq(sd, "enc.erb_conv0")
    w = _np(sd[f"enc.erb_conv0.{convs[0]}.weight"]).astype(np.float64)  # [C,1,kt,3]
    s, b = _bn_fold(sd, f"enc.erb_conv0.{bns[0]}")
    inp_kt = w.shape[2]
    out["enc.erb_conv0.w"] = f32((w[:, 0] * s[:, None, None]).transpose(1, 2, 0))
    out["enc.erb_conv0.b"] = f32(b)

    def dwpw(prefix: str, transposed: bool = False):
        convs, bns = _seq(sd, prefix)
        dw = _np(sd[f"{prefix}.{convs[0]}.weight"]).astype(np.float64)  # [C,1,kt,3] (conv and convT alike)
        assert dw.shape[0] == C and dw.shape[1] == 1 and dw.shape[3] == 3, (prefix, dw.shape)
        pw = _np(sd[f"{prefix}.{convs[1]}.weight"]).astype(np.float64)[:, :, 0, 0]  # [out,in]
        s, b = _bn_fold(sd, f"{prefix}.{bns[0]}")
        out[prefix + ".dw"] = f32(dw[:, 0].transpose(1, 2, 0))
        out[prefix + ".pw"] = f32((pw * s[:, None]).T)
        pw_nk = f32(pw * s[:, None])  # [C_out][C_in]: B operand of the tensor-core kernel
        out[prefix + ".pw_sw"] = umma_sw128_image(pw_nk)  # BF16x3 tensor-core path
        out[prefix + ".b"] = f32(b)
        return dw.shape[2]

    kts = [dwpw(p) for p in ("enc.erb_conv1", "enc.erb_conv2", "enc.erb_conv3", "enc.df_conv1",
                             "erb_dec.convt3")]
    conv_kt = kts[0]
    assert all(k == conv_kt for k in kts)
    for p in ("erb_dec.convt2", "erb_dec.convt1"):
        assert dwpw(p, transposed=True) == 1, "ConvTranspose2d with kt > 1 not supported"
    # --- df_conv0: 2->C groups=2 (kt,3), 1x1, BN
    convs, bns = _seq(sd, "enc.df_conv0")
    dw = _np(sd[f"enc.df_conv0.{convs[0]}.weight"]).astype(np.float64)  # [C,1,kt,3]
    assert dw.shape[2] == inp_kt
    pw = _np(sd[f"enc.df_conv0.{convs[1]}.weight"]).astype(np.float64)[:, :, 0, 0]
    s, b = _bn_fold(sd, f"enc.df_conv0.{bns[0]}")
    # composed weights of the direct 2 -> C conv: W[dt][df][ri][n] = sum_{c in group ri} dw[c][dt][df] * pw'[n][c]
    g = C // 2
    pws = pw * s[:, None]                                 # [n][c], BN folded
    weff = np.stack([np.einsum("ctf,nc->tfn", dw[ri * g:(ri + 1) * g, 0], pws[:, ri * g:(ri + 1) * g]) for ri in range(2)], axis=2)
    out["enc.df_conv0.w"] = f32(weff)                     # [kt][3][2][C]
    out["enc.df_conv0.b"] = f32(b)
    # --- decoder pathway convs (depthwise 1x1 + BN + ReLU)
    for n in (3, 2, 1, 0):
        p = f"erb_dec.conv{n}p"
        convs, bns = _seq(sd, p)
        w = _np(sd[f"{p}.{convs[0]}.weight"]).astype(np.float64)[:, 0, 0, 0]
        s, b = _bn_fold(sd, f"{p}.{bns[0]}")
        out[p + ".s"] = f32(w * s)
        out[p + ".b"] = f32(b)
    # --- conv0_out: C->1 (kt,3) + BN + sigmoid
    convs, bns = _seq(sd, "erb_dec.conv0_out")
    w = _np(sd[f"erb_dec.conv0_out.{convs[0]}.weight"]).astype(np.float64)  # [1,C,kt,3]
    s, b = _bn_fold(sd, f"erb_dec.conv0_out.{bns[0]}")
    assert w.shape[2] == conv_kt
    out["erb_dec.conv0_out.w"] = f32((w[0] * s[0]).transpose(1, 2, 0))
    out["erb_dec.conv0_out.b"] = f32(b)
    # --- df_convp: C->10 groups=2 (kt5,1), 1x1 10x10, BN, ReLU
    convs, bns = _seq(sd, "df_dec.df_convp")
    w1 = _np(sd[f"df_dec.df_convp.{convs[0]}.weight"]).astype(np.float64)  # [10, C/2, kt5, 1]
    w2 = _np(sd[f"df_dec.df_convp.{convs[1]}.weight"]).astype(np.float64)[:, :, 0, 0]  # [out,in]
    s, b = _bn_fold(sd, f"df_dec.df_convp.{bns[0]}")
    assert w1.shape[0] == 2 * cfg.df_order and w1.shape[1] == C // 2
    # tensor-core form (k_df_convp_tc): W2[n = g*32 + dt*O + o][k = channel] = w1[g*O + o][k - 32 g][dt] inside group g, else 0
    O, ktp = cfg.df_order, w1.shape[2]
    if C == 64 and ktp * O <= 32:
        w2x = np.zeros((64, 64), dtype=np.float32)
        for g_ in range(2):
            for dt in range(ktp):
                for o in range(O):
                    w2x[g_ * 32 + dt * O + o, g_ * 32:(g_ + 1) * 32] = w1[g_ * O + o, :, dt, 0]
        out["df_dec.df_convp.w_sw"] = umma_sw128_image(w2x)
    out["df_dec.df_convp.w2"] = f32((w2 * s[:, None]).T)
    out["df_dec.df_convp.b"] = f32(b)
    pathway_kt = w1.shape[2]

    # --- grouped linears
    def gl(dst: str, src: str) -> int:
        w = _np(sd[src])
        out[dst] = f32(w)
        if w.shape[1] % 16 == 0 and w.shape[2] % 4 == 0:
            out[dst + "_bx"] = gl_bx_image(w)   # tensor-core grouped linear (BF16x3)
        return w.shape[0]

    g = {}
    g["g_df_fc_emb"] = gl("enc.df_fc_emb.gl", "enc.df_fc_emb.0.weight")
    g["g_enc_in"] = gl("enc.emb_gru.in.gl", "enc.emb_gru.linear_in.0.weight")
    g["g_enc_out"] = gl("enc.emb_gru.out.gl", "enc.emb_gru.linear_out.0.weight") \
        if "enc.emb_gru.linear_out.0.weight" in sd else 0
    g["g_erb_in"] = gl("erb_dec.emb_gru.in.gl", "erb_dec.emb_gru.linear_in.0.weight")
    g["g_erb_out"] = gl("erb_dec.emb_gru.out.gl", "erb_dec.emb_gru.linear_out.0.weight")
    g["g_df_in"] = gl("df_dec.df_gru.in.gl", "df_dec.df_gru.linear_in.0.weight")
    g["g_df_skip"] = gl("df_dec.df_skip.gl", "df_dec.df_skip.weight") if "df_dec.df_skip.weight" in sd else 0
    g["g_df_out"] = gl("df_dec.df_out.gl", "df_dec.df_out.0.weight")

    # --- GRUs
    def gru(dst: str, src: str) -> int:
        n = gru_layers(sd, src)
        for l in range(n):
            out[f"{dst}.l{l}.w_ih_t"] = f32(_np(sd[f"{src}.weight_ih_l{l}"]).T)
            hi, lo = bf16_planes(_np(sd[f"{src}.weight_ih_l{l}"]))              # [3H][I] BF16 hi / lo, two per float
            out[f"{dst}.l{l}.w_ih_hi"], out[f"{dst}.l{l}.w_ih_lo"] = hi, lo
            out[f"{dst}.l{l}.w_hh"] = f32(_np(sd[f"{src}.weight_hh_l{l}"]))
            out[f"{dst}.l{l}.b_ih"] = f32(_np(sd[f"{src}.bias_ih_l{l}"]))
            out[f"{dst}.l{l}.b_hh"] = f32(_np(sd[f"{src}.bias_hh_l{l}"]))
        return n

    n_enc = gru("enc.emb_gru", "enc.emb_gru.gru")
    n_erb = gru("erb_dec.emb_gru", "erb_dec.emb_gru.gru")
    n_df = gru("df_dec.df_gru", "df_dec.df_gru.gru")
    out["enc.lsnr.w"] = f32(_np(sd["enc.lsnr_fc.0.weight"]).reshape(-1))
    out["enc.lsnr.b"] = f32(_np(sd["enc.lsnr_fc.0.bias"]).reshape(-1))
    if "df_dec.df_fc_a.0.weight" in sd:
        out["df_dec.df_fc_a.w"] = f32(_np(sd["df_dec.df_fc_a.0.weight"]).reshape(-1))
        out["df_dec.df_fc_a.b"] = f32(_np(sd["df_dec.df_fc_a.0.bias"]).reshape(-1))

    derived = dict(
        model_kind=2 if cfg.model == "deepfilternet2" else 3,
        nb_erb=cfg.nb_erb, nb_df=cfg.nb_df, df_order=cfg.df_order, df_lookahead=cfg.df_lookahead,
        conv_lookahead=cfg.conv_lookahead, conv_ch=C, conv_kt=conv_kt, inp_kt=inp_kt,
        emb_hidden=int(sd["enc.emb_gru.gru.weight_hh_l0"].shape[1]),
        df_hidden=int(sd["df_dec.df_gru.gru.weight_hh_l0"].shape[1]),
        enc_gru_layers=n_enc, erb_gru_layers=n_erb, df_gru_layers=n_df,
        df_pathway_kt=pathway_kt, enc_concat=int(cfg.enc_concat), **g,
        lsnr_scale=float(cfg.lsnr_max - cfg.lsnr_min), lsnr_offset=float(cfg.lsnr_min),
    )
    return out, derived


# ---------------------------------------------------------------------------------- DeepFilterNet v1 ----
def shuffle_index(n: int, groups: int) -> np.ndarray:
    """Group shuffle of modules.py:651-654 / :807-812 as a gather: shuffled[r] = x[idx[r]].  x index o = a * G + b is viewed
    as [n / G][G] and transposed, so r = b * (n / G) + a."""
    hs = n // groups
    r = np.arange(n)
    return ((r % hs) * groups + r // hs).astype(np.int32)


def _i32(a) -> np.ndarray:
    """int32 table in the fp32 container of the C ABI (bit pattern, like the BF16 planes)."""
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32)).view(np.float32)


def pack_state_dict_v1(sd: Dict[str, torch.Tensor], cfg: ModelConfig) -> Tuple[Dict[str, np.ndarray], dict]:
    """DeepFilterNet v1 (deepfilternet.py:64-279; checkpoint keys with `clc` already renamed to `df`).

    Device activations are channel-last [B,T,F,C]; the reference flattens channel-major ([C][F]) into its grouped linears
    and GRUs and interleaves (`shuffle`) their outputs.  All of that is expressed with gather tables (v1.idx_*) consumed by
    k_gather_sum, so every packed weight keeps the reference's index order, except:
      enc.df_fc_emb.gl     [G][Ig][Hg], input index inside a group i' = f * (C / G) + c (rows gathered from [F][C])
      <gru>.g{l}.l0.*      GroupedGRULayer l as ONE dense GRU of width H: block-diagonal W_ih / W_hh [3H][H] in torch gate order;
                           layers l > 0 have the shuffle of their input folded into the columns of W_ih
      df_dec.df_fc_out.w_t [H][Fd * 2 O] with output column f * 2 O + k (device coefs layout) from reference row k * Fd + f
    """
    C, E, Fd, O2 = cfg.conv_ch, cfg.nb_erb, cfg.nb_df, 2 * cfg.df_order
    G, LG, H = cfg.gru_groups, cfg.lin_groups, cfg.emb_hidden_dim
    out: Dict[str, np.ndarray] = {}

    def f32(a):
        return np.ascontiguousarray(np.asarray(a, dtype=np.float32))

    def t64(k):
        return _np(sd[k]).astype(np.float64)

    def bn(p):
        if p + ".norm.weight" not in sd:
            return None, None
        g_, b_ = t64(p + ".norm.weight"), t64(p + ".norm.bias")
        scale = g_ / np.sqrt(t64(p + ".norm.running_var") + EPS)
        return scale, b_ - t64(p + ".norm.running_mean") * scale

    # erb_conv0: dense 1 -> C (k0 x 3) + BN
    w = t64("enc.erb_conv0.sconv.weight")
    s, b = bn("enc.erb_conv0")
    inp_kt = w.shape[2]
    out["enc.erb_conv0.w"] = f32((w[:, 0] * s[:, None, None]).transpose(1, 2, 0))
    out["enc.erb_conv0.b"] = f32(b)

    def dwpw(p: str, transposed: bool = False) -> int:
        dw = t64(p + (".sconvt.weight" if transposed else ".sconv.weight"))   # [C,1,kt,kf] (Conv2d and ConvTranspose2d alike)
        assert dw.shape[0] == C and dw.shape[1] == 1, (p, dw.shape)
        if dw.shape[3] == 1:   # pathway convs: depthwise 1 x 1 = per-channel scale, as the centre tap of a 1 x 3 kernel
            dw = np.concatenate([np.zeros_like(dw), dw, np.zeros_like(dw)], axis=3)
        taps = dw[:, 0].transpose(1, 2, 0)                  # [kt][3][C]
        if transposed:
            # ConvTranspose2d over time with padding kt - 1 behind a (kt - 1)-frame front pad (modules.py:151-154,172-181):
            # out[t] = sum_j w[j] x[t - j] -- the causal kernel with its time taps reversed
            taps = taps[::-1]
        pw = t64(p + ".1x1conv.weight")[:, :, 0, 0]         # [out][in]
        s, b = bn(p)
        out[p + ".dw"] = f32(taps)
        out[p + ".pw"] = f32((pw * s[:, None]).T)
        out[p + ".pw_sw"] = umma_sw128_image(f32(pw * s[:, None]))
        out[p + ".b"] = f32(b)
        return dw.shape[2]

    kts = [dwpw(p) for p in ("enc.erb_conv1", "enc.erb_conv2", "enc.erb_conv3", "enc.df_conv1")]
    assert all(k == cfg.conv_k_enc for k in kts), kts
    kts = [dwpw("erb_dec.convt3"), dwpw("erb_dec.convt2", True), dwpw("erb_dec.convt1", True)]
    assert all(k == cfg.conv_k_dec for k in kts), kts
    for n in (3, 2, 1, 0):
        assert dwpw(f"erb_dec.conv{n}p") == 1
    # df_conv0: 2 -> C groups = 2 (k0 x 3), 1x1, BN: composed into the direct 2 -> C conv like DeepFilterNet2 / 3
    dw = t64("enc.df_conv0.sconv.weight")
    assert dw.shape == (C, 1, inp_kt, 3), dw.shape
    pw = t64("enc.df_conv0.1x1conv.weight")[:, :, 0, 0]
    s, b = bn("enc.df_conv0")
    g2 = C // 2
    pws = pw * s[:, None]
    weff = np.stack([np.einsum("ctf,nc->tfn", dw[ri * g2:(ri + 1) * g2, 0], pws[:, ri * g2:(ri + 1) * g2]) for ri in range(2)], axis=2)
    out["enc.df_conv0.w"] = f32(weff)
    out["enc.df_conv0.b"] = f32(b)
    # conv0_out: C -> 1 (kt x 3) with bias, sigmoid
    w = t64("erb_dec.conv0_out.sconv.weight")               # [1,C,kt,3]
    assert w.shape[2] == cfg.conv_k_dec
    out["erb_dec.conv0_out.w"] = f32(w[0].transpose(1, 2, 0))
    out["erb_dec.conv0_out.b"] = f32(t64("erb_dec.conv0_out.sconv.bias"))
    # df_convp: dense 1x1 C -> 2 O + BN + ReLU
    w = t64("df_dec.df_convp.sconv.weight")
    assert w.shape == (O2, C, 1, 1), w.shape
    s, b = bn("df_dec.df_convp")
    out["df_dec.df_convp.w"] = f32((w[:, :, 0, 0] * s[:, None]).T)   # [C][O2]
    out["df_dec.df_convp.b"] = f32(b)

    # grouped linears (nn.Linear per group, with bias): [G][Ig][Hg]
    def glin(dst: str, src: str, in_perm=None):
        ws = np.stack([t64(f"{src}.layers.{g_}.weight").T for g_ in range(LG)])     # [G][Ig][Hg]
        if in_perm is not None:
            ws = ws[:, in_perm, :]
        out[dst + ".gl"] = f32(ws)
        out[dst + ".bias"] = f32(np.concatenate([t64(f"{src}.layers.{g_}.bias") for g_ in range(LG)]))

    Fh, cg = Fd // 2, C // LG
    # group g reads channels [g cg, (g + 1) cg) at all Fh bins; reference index inside the group c * Fh + f, device f * cg + c
    ip = np.array([(i % cg) * Fh + i // cg for i in range(cg * Fh)])
    glin("enc.df_fc_emb", "enc.df_fc_emb", ip)
    glin("erb_dec.fc_emb", "erb_dec.fc_emb.0")
    ED = C * E // 4
    assert ED == H, "emb_dim must equal emb_hidden_dim (the grouped GRU keeps the width)"
    F8 = E // 4
    # gather tables (out[k] = src[idx[k]])
    k = np.arange(C * Fh)
    g_, rem = k // (cg * Fh), k % (cg * Fh)
    out["v1.idx_c1"] = _i32((rem // cg) * C + g_ * cg + rem % cg)                   # [F][C] rows -> group-contiguous
    r = np.arange(ED)
    out["v1.idx_e3"] = _i32((r % F8) * C + r // F8)                                 # reference r = c * F8 + f <- device f * C + c
    out["v1.idx_shuf"] = _i32(shuffle_index(ED, LG))
    out["v1.idx_id"] = _i32(r)
    p_ = np.arange(ED)
    rr = (p_ % C) * F8 + p_ // C                                                    # device p = f * C + c -> reference r
    shuf = shuffle_index(ED, LG) if cfg.group_shuffle and LG > 1 else r
    out["v1.idx_dec"] = _i32(shuf[rr])
    if G > 1 and cfg.group_shuffle:
        out["v1.idx_gshuf"] = _i32(shuffle_index(H, G))
    else:
        out["v1.idx_gshuf"] = _i32(np.arange(H))

    # grouped GRUs as dense block-diagonal GRUs
    def ggru(dst: str, src: str) -> int:
        n = 0
        while f"{src}.grus.{n}.layers.0.weight_ih_l0" in sd:
            n += 1
        hg = H // G
        for l in range(n):
            w_ih, w_hh = np.zeros((3 * H, H)), np.zeros((3 * H, H))
            b_ih, b_hh = np.zeros(3 * H), np.zeros(3 * H)
            for g_ in range(G):
                q = f"{src}.grus.{l}.layers.{g_}"
                wi, wh, bi, bh = t64(q + ".weight_ih_l0"), t64(q + ".weight_hh_l0"), t64(q + ".bias_ih_l0"), t64(q + ".bias_hh_l0")
                assert wi.shape == (3 * hg, hg), (q, wi.shape)
                for gate in range(3):
                    rows = slice(gate * H + g_ * hg, gate * H + (g_ + 1) * hg)
                    w_ih[rows, g_ * hg:(g_ + 1) * hg] = wi[gate * hg:(gate + 1) * hg]
                    w_hh[rows, g_ * hg:(g_ + 1) * hg] = wh[gate * hg:(gate + 1) * hg]
                    b_ih[rows] = bi[gate * hg:(gate + 1) * hg]
                    b_hh[rows] = bh[gate * hg:(gate + 1) * hg]
            if l > 0 and G > 1 and cfg.group_shuffle:
                # x_l[r] = y_{l-1}[idx[r]]  =>  W x_l = W'[:, o] y_{l-1}[o] with W'[:, idx[r]] = W[:, r]
                idx = shuffle_index(H, G)
                wp = np.zeros_like(w_ih)
                wp[:, idx] = w_ih
                w_ih = wp
            base = f"{dst}.g{l}.l0"
            out[base + ".w_ih_t"] = f32(w_ih.T)
            out[base + ".w_ih_hi"], out[base + ".w_ih_lo"] = bf16_planes(f32(w_ih))
            out[base + ".w_hh"] = f32(w_hh)
            out[base + ".b_ih"] = f32(b_ih)
            out[base + ".b_hh"] = f32(b_hh)
        return n

    n_enc = ggru("enc.emb_gru", "enc.emb_gru")
    n_df = ggru("df_dec.df_gru", "df_dec.df_gru")
    assert n_enc == cfg.emb_num_layers and n_df == cfg.df_num_layers, (n_enc, n_df)
    out["enc.lsnr.w"] = f32(t64("enc.lsnr_fc.0.weight").reshape(-1))
    out["enc.lsnr.b"] = f32(t64("enc.lsnr_fc.0.bias").reshape(-1))
    out["df_dec.df_fc_a.w"] = f32(t64("df_dec.df_fc_a.0.weight").reshape(-1))
    out["df_dec.df_fc_a.b"] = f32(t64("df_dec.df_fc_a.0.bias").reshape(-1))
    w = t64("df_dec.df_fc_out.0.weight")                     # [O2 * Fd][H], row k * Fd + f
    assert w.shape == (O2 * Fd, H)
    n = np.arange(Fd * O2)
    src = (n % O2) * Fd + n // O2                            # device column f * O2 + k
    out["df_dec.df_fc_out.w_t"] = f32(w[src].T)              # [H][Fd * O2]
    out["df_dec.df_fc_out.b"] = f32(t64("df_dec.df_fc_out.0.bias")[src])
    out["df_dec.df_fc_out.w_hi"], out["df_dec.df_fc_out.w_lo"] = bf16_planes(f32(w[src]))   # [N][K] B operand of the BF16x3 GEMM
    out["v1.ones"] = np.ones(C, dtype=np.float32)
    out["v1.zeros"] = np.zeros(C, dtype=np.float32)
    derived = dict(
        model_kind=1, nb_erb=E, nb_df=Fd, df_order=cfg.df_order, df_lookahead=cfg.df_lookahead,
        conv_lookahead=cfg.conv_lookahead, conv_ch=C, conv_kt=cfg.conv_k_enc, inp_kt=inp_kt,
        emb_hidden=H, df_hidden=cfg.df_hidden_dim, enc_gru_layers=n_enc, erb_gru_layers=0, df_gru_layers=n_df,
        df_pathway_kt=1, enc_concat=0, g_df_fc_emb=LG, g_enc_in=G, g_enc_out=0, g_erb_in=LG, g_erb_out=0, g_df_in=G,
        g_df_skip=0, g_df_out=1,
        lsnr_scale=float(cfg.lsnr_max - cfg.lsnr_min), lsnr_offset=float(cfg.lsnr_min),
    )
    return out, derived


def random_state_dict_v1(cfg: ModelConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Random-init DeepFilterNet v1 weights with the shipped checkpoint's tensor names (after the clc -> df rename)."""
    g = torch.Generator().manual_seed(seed)
    C, E, Fd, O2 = cfg.conv_ch, cfg.nb_erb, cfg.nb_df, 2 * cfg.df_order
    G, LG, H = cfg.gru_groups, cfg.lin_groups, cfg.emb_hidden_dim
    ke, kd, k0 = cfg.conv_k_enc, cfg.conv_k_dec, cfg.conv_kernel_inp[0]
    sd: Dict[str, torch.Tensor] = {}

    def rnd(*shape, scale=1.0):
        return (torch.rand(*shape, generator=g) * 2 - 1) * scale

    def bn(p, n):
        sd[p + ".norm.weight"] = 1.0 + rnd(n, scale=0.3)
        sd[p + ".norm.bias"] = rnd(n, scale=0.2)
        sd[p + ".norm.running_mean"] = rnd(n, scale=0.2)
        sd[p + ".norm.running_var"] = 0.5 + torch.rand(n, generator=g)
        sd[p + ".norm.num_batches_tracked"] = torch.tensor(1)

    def conv(p, name, shape):
        fan = shape[1] * shape[2] * shape[3]
        sd[f"{p}.{name}.weight"] = rnd(*shape, scale=(1.5 / fan) ** 0.5 * 1.7)

    def sep(p, kt, kf=3, transposed=False):
        conv(p, "sconvt" if transposed else "sconv", (C, 1, kt, kf))
        conv(p, "1x1conv", (C, C, 1, 1))
        bn(p, C)

    conv("enc.erb_conv0", "sconv", (C, 1, k0, 3)); bn("enc.erb_conv0", C)
    for p in ("enc.erb_conv1", "enc.erb_conv2", "enc.erb_conv3", "enc.df_conv1"):
        sep(p, ke)
    conv("enc.df_conv0", "sconv", (C, 1, k0, 3)); conv("enc.df_conv0", "1x1conv", (C, C, 1, 1)); bn("enc.df_conv0", C)
    sep("erb_dec.convt3", kd); sep("erb_dec.convt2", kd, transposed=True); sep("erb_dec.convt1", kd, transposed=True)
    for n in (3, 2, 1, 0):
        sep(f"erb_dec.conv{n}p", 1, 1)
    conv("erb_dec.conv0_out", "sconv", (1, C, kd, 3)); sd["erb_dec.conv0_out.sconv.bias"] = rnd(1, scale=0.1)
    conv("df_dec.df_convp", "sconv", (O2, C, 1, 1)); bn("df_dec.df_convp", O2)

    def glin(p, i, h):
        for j in range(LG):
            sd[f"{p}.layers.{j}.weight"] = rnd(h // LG, i // LG, scale=(3.0 / (i // LG)) ** 0.5)
            sd[f"{p}.layers.{j}.bias"] = rnd(h // LG, scale=0.1)

    glin("enc.df_fc_emb", C * Fd // 2, C * E // 4)
    glin("erb_dec.fc_emb.0", H, C * E // 4)

    def ggru(p, layers):
        hg = H // G
        for l in range(layers):
            for j in range(G):
                k_ = (1.0 / hg) ** 0.5
                q = f"{p}.grus.{l}.layers.{j}"
                sd[q + ".weight_ih_l0"] = rnd(3 * hg, hg, scale=k_); sd[q + ".weight_hh_l0"] = rnd(3 * hg, hg, scale=k_)
                sd[q + ".bias_ih_l0"] = rnd(3 * hg, scale=k_); sd[q + ".bias_hh_l0"] = rnd(3 * hg, scale=k_)

    ggru("enc.emb_gru", cfg.emb_num_layers)
    ggru("df_dec.df_gru", cfg.df_num_layers)
    sd["enc.lsnr_fc.0.weight"] = rnd(1, H, scale=0.05); sd["enc.lsnr_fc.0.bias"] = rnd(1, scale=0.1)
    sd["df_dec.df_fc_out.0.weight"] = rnd(O2 * Fd, H, scale=(3.0 / H) ** 0.5); sd["df_dec.df_fc_out.0.bias"] = rnd(O2 * Fd, scale=0.1)
    sd["df_dec.df_fc_a.0.weight"] = rnd(1, H, scale=0.05); sd["df_dec.df_fc_a.0.bias"] = rnd(1, scale=0.1)
    return sd


def random_state_dict(cfg: ModelConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Random-init weights with the shipped architecture's tensor names / shapes (for benchmarks
    and parity tests that must not depend on a checkpoint).  BatchNorm statistics are randomised
    too so that folding is exercised."""
    if cfg.model == "deepfilternet":
        return random_state_dict_v1(cfg, seed)
    g = torch.Generator().manual_seed(seed)
    C, E, Fd = cfg.conv_ch, cfg.nb_erb, cfg.nb_df
    kt, kti = cfg.conv_kernel[0], cfg.conv_kernel_inp[0]
    H, Hd = cfg.emb_hidden_dim, cfg.df_hidden_dim
    sd: Dict[str, torch.Tensor] = {}

    def rnd(*shape, scale=1.0):
        return (torch.rand(*shape, generator=g) * 2 - 1) * scale

    def bn(p, n):
        sd[p + ".weight"] = 1.0 + rnd(n, scale=0.3)
        sd[p + ".bias"] = rnd(n, scale=0.2)
        sd[p + ".running_mean"] = rnd(n, scale=0.2)
        sd[p + ".running_var"] = 0.5 + torch.rand(n, generator=g)
        sd[p + ".num_batches_tracked"] = torch.tensor(1)

    def conv_seq(p, shapes, n_bn, pad):
        i = 1 if pad else 0
        for s in shapes:
            fan = s[1] * s[2] * s[3]
            sd[f"{p}.{i}.weight"] = rnd(*s, scale=(1.5 / fan) ** 0.5 * 1.7)
            i += 1
        bn(f"{p}.{i}", n_bn)

    conv_seq("enc.erb_conv0", [(C, 1, kti, 3)], C, kti > 1)
    for n in ("enc.erb_conv1", "enc.erb_conv2", "enc.erb_conv3", "enc.df_conv1", "erb_dec.convt3"):
        conv_seq(n, [(C, 1, kt, 3), (C, C, 1, 1)], C, kt > 1)
    conv_seq("enc.df_conv0", [(C, 1, kti, 3), (C, C, 1, 1)], C, kti > 1)
    for n in ("erb_dec.convt2", "erb_dec.convt1"):
        conv_seq(n, [(C, 1, 1, 3), (C, C, 1, 1)], C, False)
    for n in (3, 2, 1, 0):
        conv_seq(f"erb_dec.conv{n}p", [(C, 1, 1, 1)], C, False)
    conv_seq("erb_dec.conv0_out", [(1, C, kt, 3)], 1, kt > 1)
    ktp = cfg.df_pathway_kernel_size_t
    conv_seq("df_dec.df_convp", [(2 * cfg.df_order, C // 2, ktp, 1), (2 * cfg.df_order, 2 * cfg.df_order, 1, 1)],
             2 * cfg.df_order, ktp > 1)

    def glw(name, i, h, groups):
        sd[name] = rnd(groups, i // groups, h // groups, scale=(3.0 / (i // groups)) ** 0.5)

    def gruw(p, i, h, layers):
        for l in range(layers):
            k = (1.0 / h) ** 0.5
            sd[f"{p}.weight_ih_l{l}"] = rnd(3 * h, i if l == 0 else h, scale=k)
            sd[f"{p}.weight_hh_l{l}"] = rnd(3 * h, h, scale=k)
            sd[f"{p}.bias_ih_l{l}"] = rnd(3 * h, scale=k)
            sd[f"{p}.bias_hh_l{l}"] = rnd(3 * h, scale=k)

    emb_dim = C * E // 4
    if cfg.model == "deepfilternet3":
        glw("enc.df_fc_emb.0.weight", C * Fd // 2, emb_dim, cfg.enc_lin_groups)
        glw("enc.emb_gru.linear_in.0.weight", emb_dim, H, cfg.lin_groups)
        gruw("enc.emb_gru.gru", H, H, 1)
        glw("enc.emb_gru.linear_out.0.weight", H, emb_dim, cfg.lin_groups)
        sd["enc.lsnr_fc.0.weight"] = rnd(1, emb_dim, scale=0.05)
        glw("erb_dec.emb_gru.linear_in.0.weight", emb_dim, H, cfg.lin_groups)
        gruw("erb_dec.emb_gru.gru", H, H, cfg.emb_num_layers - 1)
        glw("erb_dec.emb_gru.linear_out.0.weight", H, emb_dim, cfg.lin_groups)
        glw("df_dec.df_gru.linear_in.0.weight", emb_dim, Hd, 8)  # SqueezedGRU_S default groups
        gruw("df_dec.df_gru.gru", Hd, Hd, cfg.df_num_layers)
        if cfg.df_gru_skip == "groupedlinear":
            glw("df_dec.df_skip.weight", emb_dim, Hd, cfg.lin_groups)
        glw("df_dec.df_out.0.weight", Hd, Fd * cfg.df_order * 2, cfg.lin_groups)
    else:
        G = cfg.lin_groups
        glw("enc.df_fc_emb.0.weight", C * Fd // 2, emb_dim, G)
        glw("enc.emb_gru.linear_in.0.weight", emb_dim * (2 if cfg.enc_concat else 1), H, G)
        gruw("enc.emb_gru.gru", H, H, 1)
        sd["enc.lsnr_fc.0.weight"] = rnd(1, H, scale=0.05)
        glw("erb_dec.emb_gru.linear_in.0.weight", H, H, G)
        gruw("erb_dec.emb_gru.gru", H, H, cfg.emb_num_layers - 1)
        glw("erb_dec.emb_gru.linear_out.0.weight", H, emb_dim, G)
        glw("df_dec.df_gru.linear_in.0.weight", H, Hd, 8)
        gruw("df_dec.df_gru.gru", Hd, Hd, cfg.df_num_layers)
        glw("df_dec.df_out.0.weight", Hd, Fd * cfg.df_order * 2, G)
    sd["enc.lsnr_fc.0.bias"] = rnd(1, scale=0.1)
    sd["df_dec.df_fc_a.0.weight"] = rnd(1, Hd, scale=0.05)
    sd["df_dec.df_fc_a.0.bias"] = rnd(1, scale=0.1)
    return sd
