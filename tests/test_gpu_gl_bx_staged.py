"""GPU: k_gl_bx's staged BF16-plane epilogue (planes written 64 columns at a time into shared memory and stored with TMA
tensor stores) against float64, and against the register-store path it falls back to.

The staged path clips rows >= M and must leave a wider plane pitch's pad columns alone; the fallbacks named in
launch_gl_bx (pitch not a multiple of 8 elements, plane base not 16-byte aligned, Hg % 16 or gpc * Hg % 64, a ring that
would drop below 2 stages) must give the same bits."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench_gl  # noqa: E402
from test_gpu_gl_bx import bench_m, check  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 0x3C3C   # plane sentinel (int16), outside every row / column the kernel owns
ENC_IN = (16, 32, 16)     # DeepFilterNet3 enc.emb_gru.in / erb_dec.emb_gru.in / df_dec.df_skip: planes staged, 4 blocks
ENC_OUT = (16, 16, 32)    # DeepFilterNet3 enc.emb_gru.out: with fp32 output the ring leaves no room for staged planes
BOTH = (8, 16, 16)        # small weights: fp32 rows and planes both staged
PLANE_SHAPES = [ENC_IN, (8, 64, 32), (8, 128, 32), (8, 32, 32), (16, 32, 32), (8, 64, 64)]


def launch(case, act, res, oscale, ooffset, planes=True, pad=0, extra_rows=0, shift=0):
    """One launch on case's X / W with the planes at pitch N + pad, base shifted by `shift` elements and `extra_rows`
    sentinel rows past M.  res: None or "y" (in place; needs case.y).  Returns (y or None, hi, lo) as full host arrays."""
    import torch
    from deepfilternet_b200 import _lib
    K, N, M = case.G * case.Ig, case.G * case.Hg, case.M
    ldp = N + pad
    rows = M + extra_rows
    hi = lo = None
    if planes:
        hi = torch.full((rows * ldp + shift,), SENT, dtype=torch.int16, device="cuda")
        lo = torch.full((rows * ldp + shift,), SENT, dtype=torch.int16, device="cuda")
    ptr = lambda t, o=0: None if t is None else t.data_ptr() + 2 * o
    resp = case.y.data_ptr() if res == "y" else None
    rc = _lib.lib().dfb_debug_gl_bx(case.x_hi.data_ptr(), case.x_lo.data_ptr(), K, case.w_img.data_ptr(), resp, N,
                                    ptr(case.y), N, ptr(hi, shift), ptr(lo, shift), ldp, M, case.G, case.Ig, case.Hg, act,
                                    oscale, ooffset, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().dfb_last_error().decode()
    torch.cuda.synchronize()
    y = case.y.cpu().numpy().copy() if case.y is not None else None
    if not planes:
        return y, None, None
    unpack = lambda t: t.cpu().numpy()[shift:].reshape(rows, ldp)
    return y, unpack(hi), unpack(lo)


def new_case(shape, M, fp32=False, seed=5):
    return bench_gl.GlCase(*shape, M, fp32=fp32, planes=False, seed=seed)


def split_bf16(y):
    """the RNE hi / lo BF16 split of fp32 y, as int16 planes"""
    import torch
    t = torch.from_numpy(y)
    h = t.to(torch.bfloat16)
    lo = (t - h.float()).to(torch.bfloat16)
    return h.view(torch.int16).numpy(), lo.view(torch.int16).numpy()


@pytest.mark.parametrize("M", [1, 15, 16, 17, 127, 128, 129, 300, "bench"])
def test_staged_planes_rows(M):
    """planes only (DeepFilterNet3 enc.emb_gru.in's shape) at row counts around the warp's 16 rows and the 128-row tile;
    rows past M stay untouched"""
    M = bench_m() if M == "bench" else M
    case = new_case(ENC_IN, M)
    _, hi, lo = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0, extra_rows=17)
    check(case, None, (hi[:M], lo[:M]), bench_gl.ACT_RELU, None, 1.0, 0.0)
    assert (hi[M:] == SENT).all() and (lo[M:] == SENT).all()


@pytest.mark.parametrize("shape", PLANE_SHAPES, ids=lambda s: "G%d_Ig%d_Hg%d" % s)
def test_staged_planes_shapes(shape):
    """every plane-writing shape of the shipped models, tanh with scale / offset, against float64"""
    case = new_case(shape, 300)
    _, hi, lo = launch(case, bench_gl.ACT_TANH, None, 0.75, -0.125)
    check(case, None, (hi, lo), bench_gl.ACT_TANH, None, 0.75, -0.125)


@pytest.mark.parametrize("M", [129, 300])
def test_staged_planes_wide_pitch(M):
    """plane pitch 8 columns wider than the data: the pad columns and the rows past M keep their sentinels, and the data
    has the bits of the dense pitch"""
    case = new_case(ENC_IN, M)
    N = case.G * case.Hg
    _, hi0, lo0 = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0)
    _, hi, lo = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0, pad=8, extra_rows=5)
    assert (hi[:M, :N] == hi0).all() and (lo[:M, :N] == lo0).all()
    assert (hi[:, N:] == SENT).all() and (lo[:, N:] == SENT).all()
    assert (hi[M:] == SENT).all() and (lo[M:] == SENT).all()


@pytest.mark.parametrize("M", [17, 300])
@pytest.mark.parametrize("res", [None, "y"])
def test_staged_both_outputs(M, res):
    """fp32 rows and planes staged together, with the residual added in place (res = y, as df_out does): float64, and
    the planes are the BF16 split of y bit for bit"""
    case = new_case(BOTH, M, fp32=True)
    if res:
        case.set_residual()
    y, hi, lo = launch(case, bench_gl.ACT_TANH, res, 0.75, -0.125, extra_rows=3)
    check(case, y, (hi[:M], lo[:M]), bench_gl.ACT_TANH, res, 0.75, -0.125)
    sh, sl = split_bf16(y)
    assert (hi[:M] == sh).all() and (lo[:M] == sl).all()
    assert (hi[M:] == SENT).all() and (lo[M:] == SENT).all()


@pytest.mark.parametrize("how", ["pitch_not_x8", "base_not_16B"])
def test_fallback_pitch_and_alignment(how):
    """planes that TMA cannot store (pitch N + 4, or a base 8 bytes off 16-byte alignment) come from registers with the
    bits of the staged path, and the pad columns keep their sentinels"""
    M = 300
    case = new_case(ENC_IN, M)
    N = case.G * case.Hg
    _, hi0, lo0 = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0, pad=8)
    kw = dict(pad=4) if how == "pitch_not_x8" else dict(pad=8, shift=4)
    _, hi, lo = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0, extra_rows=2, **kw)
    assert (hi[:M, :N] == hi0[:, :N]).all() and (lo[:M, :N] == lo0[:, :N]).all()
    assert (hi[:, N:] == SENT).all() and (hi[M:] == SENT).all()


def test_fallback_ring():
    """DeepFilterNet3 enc.emb_gru.out writes fp32 and planes: its planes stay register stores (the ring would drop below 2
    stages) and have the bits of the same shape's staged planes-only launch and of the split of y"""
    M = 300
    case = new_case(ENC_OUT, M)
    _, hi0, lo0 = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0)
    case_y = new_case(ENC_OUT, M, fp32=True)
    y, hi, lo = launch(case_y, bench_gl.ACT_RELU, None, 1.0, 0.0)
    assert (hi == hi0).all() and (lo == lo0).all()
    sh, sl = split_bf16(y)
    assert (hi == sh).all() and (lo == sl).all()


@pytest.mark.parametrize("shape", [(4, 16, 12), (2, 32, 16)], ids=lambda s: "G%d_Ig%d_Hg%d" % s)
def test_fallback_shape(shape):
    """Hg % 16 != 0 (a chunk straddles groups) or gpc * Hg % 64 != 0 (the slice ends inside a 64-column block): register
    stores, against float64 and, bit for bit, the BF16 split of the same launch's fp32 output"""
    M = 300
    case = new_case(shape, M, fp32=True)
    y, hi, lo = launch(case, bench_gl.ACT_RELU, None, 1.0, 0.0)
    check(case, y, (hi, lo), bench_gl.ACT_RELU, None, 1.0, 0.0)
    sh, sl = split_bf16(y)
    assert (hi == sh).all() and (lo == sl).all()
