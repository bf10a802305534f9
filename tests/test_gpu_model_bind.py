"""GPU: dfb_model_create binds every weight tensor the configured forward pass reads.  A weight set that lacks one, or has
one of the wrong size, is refused at creation with DFB_ERR_INVALID and the tensor's name; a missing tensor-core image only
changes which kernel runs a layer.  The tensor array is built from pack_state_dict as DfNet.__init__ builds it, so that
single entries can be dropped or cut short first."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_parity import cfg_of, cfg_v1

from deepfilternet_b200 import _lib
from deepfilternet_b200._lib import DFB_ERR_INVALID, DfbError, ModelConfigC, TensorC, check
from deepfilternet_b200.weights import pack_state_dict, random_state_dict


def config(kind):
    return cfg_v1() if kind == "v1" else cfg_of(kind)


def packed_weights(kind):
    cfg = config(kind)
    packed, derived = pack_state_dict(random_state_dict(cfg, seed=5), cfg)
    return cfg, packed, derived


def create(cfg, packed, derived):
    cc = ModelConfigC()
    for k, v in derived.items():
        setattr(cc, k, v)
    cc.norm_alpha = cfg.norm_alpha
    names = [n.encode() for n in packed]
    arr = (TensorC * len(packed))()
    for i, (n, a) in enumerate(packed.items()):
        arr[i].name = names[i]
        arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
        arr[i].numel = a.size
    h = C.c_void_p()
    check(_lib.lib().dfb_model_create(C.byref(h), 0, C.byref(cc), arr, len(packed), None))
    return h


def refused(kind, packed, derived, name):
    with pytest.raises(DfbError) as e:
        _lib.lib().dfb_model_free(create(config(kind), packed, derived))
    assert e.value.code == DFB_ERR_INVALID and f"'{name}'" in str(e.value), str(e.value)


@pytest.mark.parametrize("kind,name", [
    ("dfn3", "enc.erb_conv0.w"),                 # input conv
    ("dfn3", "enc.erb_conv2.pw_sw"),             # separable block
    ("dfn3", "df_dec.df_gru.l1.w_ih_hi"),        # GRU layer
    ("dfn3", "erb_dec.emb_gru.out.gl"),          # grouped linear, fp32 weight
    ("dfn2", "enc.df_conv0.b"),
    ("dfn2", "erb_dec.convt1.dw"),
    ("dfn2", "df_dec.df_fc_a.w"),                # DeepFilterNet2's alpha head
    ("ll", "enc.emb_gru.l0.w_ih_lo"),
    ("ll", "erb_dec.conv1p.s"),                  # decoder pathway
    ("v1", "v1.idx_e3"),                         # index table
    ("v1", "enc.emb_gru.g1.l0.w_ih_hi"),
    ("v1", "erb_dec.conv0p.pw"),
    ("v1", "erb_dec.fc_emb.gl"),
])
def test_missing_tensor_is_refused(kind, name):
    _, packed, derived = packed_weights(kind)
    assert name in packed
    del packed[name]
    refused(kind, packed, derived, name)


@pytest.mark.parametrize("kind,name", [
    ("dfn3", "enc.emb_gru.l0.w_hh"),
    ("dfn2", "erb_dec.conv0_out.w"),
    ("ll", "df_dec.df_out.gl"),
    ("v1", "df_dec.df_gru.g0.l0.w_hh"),
    ("v1", "v1.idx_c1"),
])
def test_short_tensor_is_refused(kind, name):
    _, packed, derived = packed_weights(kind)
    packed[name] = np.ascontiguousarray(packed[name].reshape(-1)[:-1])
    refused(kind, packed, derived, name)


@pytest.mark.parametrize("kind,name", [
    ("dfn3", "erb_dec.emb_gru.out.gl_bx"),
    ("dfn2", "df_dec.df_out.gl_bx"),
    ("ll", "df_dec.df_gru.in.gl_bx"),
    ("v1", "df_dec.df_fc_out.w_hi"),
])
def test_optional_image_changes_kernel_only(kind, name):
    """Without the image the layer runs on the FFMA kernel; the forward pass still completes."""
    cfg, packed, derived = packed_weights(kind)
    del packed[name]
    h = create(cfg, packed, derived)
    try:
        B, T, E, Fd, O = 2, 37, cfg.nb_erb, cfg.nb_df, cfg.df_order
        g = torch.Generator(device="cuda").manual_seed(11)
        fe = torch.randn(B, T, E, device="cuda", generator=g) * 0.5 - 0.5
        fs = torch.randn(B, T, Fd, 2, device="cuda", generator=g) * 0.1
        m = torch.full((B, T, E), float("nan"), device="cuda")
        coefs = torch.full((B, T, Fd, 2 * O), float("nan"), device="cuda")
        lsnr = torch.full((B, T), float("nan"), device="cuda")
        alpha = torch.full((B, T), float("nan"), device="cuda") if kind in ("dfn2", "v1") else None
        stream = torch.cuda.current_stream().cuda_stream
        check(_lib.lib().dfb_model_forward(h, fe.data_ptr(), fs.data_ptr(), B, T, m.data_ptr(), coefs.data_ptr(), lsnr.data_ptr(),
                                           alpha.data_ptr() if alpha is not None else None, stream))
        torch.cuda.synchronize()
        for t in (m, coefs, lsnr) + ((alpha,) if alpha is not None else ()):
            assert torch.isfinite(t).all()
        assert ((m >= 0) & (m <= 1)).all()
    finally:
        _lib.lib().dfb_model_free(h)
