"""GPU: the DSP kernels around the DNN, element by element against the float64 reference of tests/dsp_ref64.py.

Each test asserts |gpu - ref64| <= K * bound for every element, where bound is ref64's bound for an fp32 evaluation of the
same formula (the fp32 CPU oracle meets the same bounds with K = 1, tests/test_dsp_ref64.py), at the shapes where the kernels
switch paths: the one-thread and the time-segmented normalisation scan, the analysis kernel's 8-frame CTA tiles, the apply
kernel's 8 / 16-frame warp tiles with the re-synthesised frame before each and the preloaded deep-filter history, the
specialised and the generic apply kernel, DeepFilterNet v1's alpha blend in both.  Inputs come from seeds only."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dsp_ref64 as R
from test_gpu_parity import cfg_of, cfg_v1
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, enhance, libdf
from deepfilternet_b200._lib import check
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

HOP = 480
ALPHA = 0.99


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, HOP, 32, 2)


def assert_within(name, got, ref, bound, k):
    r = R.err_ratio(got, ref, bound)
    print(f"err/bound {name}: {r:.3g}")
    assert r <= k, (name, r)


def noisy(C, T, seed):
    x = synth_audio(C, T, seed=seed).numpy()
    x[0, 2000:3500] = 0.0       # digital silence over whole frames: |X| = 0 bins and the 1e-10 floor of the dB
    return np.ascontiguousarray(x)


def complex_of(t):
    return torch.view_as_complex(t.contiguous()).numpy().astype(np.complex128)


# ------------------------------------------------------------------ feature normalisation ----
@pytest.mark.parametrize("nb_df", [96, 104])
@pytest.mark.parametrize("Tf", [127, 128, 129, 136, 1001, 3001])
def test_df_features_against_ref64(st, Tf, nb_df):
    """df_features (dfb_features: analysis + both normalisations) for 3 channels.  nb_df = 96 puts E + Fd at 128, the
    segmented scan's limit: k_feat_norm_seg from 128 frames on (129 and 1001 leave a short last segment, 136 = 8 x 17),
    k_feat_norm below; nb_df = 104 runs k_feat_norm<4>.  K = 1 (worst err / bound on an H100 80GB HBM3: spectrum 0.09, ERB
    features 0.20, DF features 0.06)."""
    x = noisy(3, Tf * HOP + 77, seed=Tf)
    sp, fe, fs = df_features(torch.from_numpy(x), st, nb_df, alpha=ALPHA)
    X, bX = R.stft(x, st.fft_window(), HOP)
    assert_within("spec", complex_of(sp[:, 0]), X, bX, 1)
    db, bdb = R.erb_db(X, bX, st.erb_widths())
    ref, b = R.mean_norm(db, ALPHA, None, bdb)
    assert_within("erb", fe[:, 0].numpy(), ref, b, 1)
    ref, b = R.unit_norm(X[..., :nb_df], ALPHA, None, bX[..., :nb_df])
    assert_within("unit", complex_of(fs[:, 0]), ref, b, 1)


# ------------------------------------------------------------------ analysis ----
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("Tf", [1, 7, 8, 9, 17])
def test_analysis_tile_edges(st, Tf, C):
    """dfb_analysis (device pointers) and the ERB dB of df_features (through ref64's normalisation) at frame counts around
    the analysis kernel's 8-frame CTA, with a signal length that is not a multiple of the hop.  K = 1 (worst err / bound on
    an H100 80GB HBM3: spectrum 0.07, ERB features 0.22)."""
    T = Tf * HOP + 1 + (37 * Tf) % 479
    x = noisy(C, T, seed=100 + Tf)
    d = torch.from_numpy(x).cuda()
    spec = torch.full((C, Tf, 481, 2), float("nan"), device="cuda")
    check(_lib.lib().dfb_analysis(st.handle, d.data_ptr(), C, T, spec.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    X, bX = R.stft(x, st.fft_window(), HOP)
    assert_within("spec", complex_of(spec.cpu()), X, bX, 1)
    _, fe, _ = df_features(torch.from_numpy(x), st, 96, alpha=ALPHA)
    db, bdb = R.erb_db(X, bX, st.erb_widths())
    ref, b = R.mean_norm(db, ALPHA, None, bdb)
    assert_within("erb", fe[:, 0].numpy(), ref, b, 1)


# ------------------------------------------------------------------ apply (dfb_apply) ----
KINDS = {   # name: (test_gpu_parity config, nb_df, apply mode, df look-ahead)
    "dfn3": ("dfn3", 96, 1, 2), "ll": ("ll", 96, 1, 0), "dfn2": ("dfn2", 96, 2, 2),
    # nb_df != 96: the generic apply kernel
    "dfn3_df64": ("dfn3", 64, 1, 2), "dfn2_df64": ("dfn2", 64, 2, 2),
    # 24 ERB bands: the generic apply kernel at another band count
    "dfn3_e24": ("e24", 96, 1, 2),
    # DeepFilterNet v1: the masked deep filter blended with the masked bins by alpha (specialised / generic kernel)
    "v1": ("v1", 96, 2, 1), "v1_df64": ("v1", 64, 2, 1),
}
OPTS = {"plain": (False, False), "pf": (True, False), "mask_only": (False, True)}


@pytest.fixture(scope="module")
def models(st):
    out = {}
    for name, (kind, nb_df, _, _) in KINDS.items():
        cfg = dataclasses.replace(cfg_v1() if kind == "v1" else cfg_of(kind), nb_df=nb_df)
        out[name] = DfNet(cfg, random_state_dict(cfg, seed=3), st if cfg.nb_erb == 32 else libdf.DF(48000, 960, HOP, cfg.nb_erb, 2))
    return out


def apply_inputs(B, T, nb_df, seed, E=32):
    """Random spectra with exact-zero bins, masks with exact 0 and 1 entries, random deep-filter coefficients."""
    rng = np.random.default_rng(seed)
    spec = ((rng.standard_normal((B, T, 481)) + 1j * rng.standard_normal((B, T, 481))) * 0.1).astype(np.complex64)
    spec[rng.random(spec.shape) < 0.1] = 0
    m = rng.random((B, T, E)).astype(np.float32)
    m[rng.random(m.shape) < 0.1] = 0
    m[rng.random(m.shape) < 0.1] = 1
    c = ((rng.standard_normal((B, T, nb_df, 5)) + 1j * rng.standard_normal((B, T, nb_df, 5))) * 0.5).astype(np.complex64)
    return spec, m, c


def dfb_apply(model, st, spec, m, c, pf, mask_only):
    """A thin ctypes call of the C entry point dfb_apply (spec_e = the model's apply stages on given outputs)."""
    L = _lib.lib()
    B, T = m.shape[:2]
    d_spec, d_m, d_c = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (spec.view(np.float32), m, c.view(np.float32)))
    out = torch.full_like(d_spec, float("nan"))
    check(L.dfb_model_set_options(model.handle, int(pf), C.c_float(0.02), int(mask_only)))
    try:
        check(L.dfb_apply(model.handle, st.handle, d_spec.data_ptr(), d_m.data_ptr(), d_c.data_ptr(), B, T, out.data_ptr(),
                          torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    finally:
        check(L.dfb_model_set_options(model.handle, int(model.post_filter), C.c_float(model.post_filter_beta), int(not model.run_df)))
    return out.cpu().numpy().view(np.complex64).astype(np.complex128)


def run_apply_case(st, models, kind, opt, B, Tf, seed, rows=None):
    _, nb_df, mode, la = KINDS[kind]
    pf, mask_only = OPTS[opt]
    st = models[kind].df_state
    spec, m, c = apply_inputs(B, Tf, nb_df, seed, st.nb_erb())
    got = dfb_apply(models[kind], st, spec, m, c, pf, mask_only)
    rows = list(range(B)) if rows is None else rows
    ref, b = R.apply(spec[rows], m[rows], c[rows], st.erb_widths(), mode=mode, nb_df=nb_df, order=5, lookahead=la,
                     post_filter=pf, mask_only=mask_only)
    assert_within(f"{kind} {opt} Tf={Tf}", got[rows], ref, b, 1)


@pytest.mark.parametrize("Tf", [1, 2, 3, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2"])
def test_apply_against_ref64(st, models, kind, opt, Tf):
    """The specialised k_apply_synthesis through dfb_apply: DeepFilterNet3 (look-ahead 2), DeepFilterNet3_ll (look-ahead 0)
    and DeepFilterNet2 (masked deep filter), with and without the post filter and with mask_only, at frame counts around the
    8-frame warp tile and the 32-frame CTA (every warp re-synthesises the frame before its first and preloads the deep
    filter's history there).  K = 1 (worst err / bound on an H100 80GB HBM3: 0.994, a gain bin's single rounded product
    against its u |x g| bound; 0.64 with the post filter)."""
    run_apply_case(st, models, kind, opt, 3, Tf, seed=Tf)


def forward_full(model, st, sp, fe, fs, pf, mask_only):
    """dfb_model_forward_full with every output pointer (DeepFilterNet v1 has no dfb_apply): spec_e, m, coefs (complex
    [B,T,nb_df,O]) and alpha of one call"""
    L = _lib.lib()
    B, _, T, E = fe.shape
    d_sp, d_fe, d_fs = (t.cuda().contiguous() for t in (sp, fe, fs))
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")
    spec_e, m, lsnr, c, a = nan(*d_sp.shape), nan(B, T, E), nan(B, T), nan(B, T, model.nb_df, 10), nan(B, T)
    check(L.dfb_model_set_options(model.handle, int(pf), C.c_float(0.02), int(mask_only)))
    try:
        check(L.dfb_model_forward_full(model.handle, st.handle, d_sp.data_ptr(), d_fe.data_ptr(), d_fs.data_ptr(), B, T,
                                       spec_e.data_ptr(), m.data_ptr(), lsnr.data_ptr(), c.data_ptr(), a.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    finally:
        check(L.dfb_model_set_options(model.handle, int(model.post_filter), C.c_float(model.post_filter_beta), int(not model.run_df)))
    return (complex_of(spec_e.cpu()[:, 0]), m.cpu().numpy(), complex_of(c.cpu().reshape(B, T, model.nb_df, 5, 2)),
            a.cpu().numpy())


@pytest.mark.parametrize("Tf", [1, 2, 3, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("kind", ["v1", "v1_df64"])
def test_alpha_blend_against_ref64(st, models, kind, opt, Tf):
    """DeepFilterNet v1's apply stage (mode 2 with alpha: the deep filter of the masked spectrum blended with the masked
    bins by alpha), with and without Mask.pf and with mask_only: the specialised kernel at nb_df = 96, the generic one
    at 64.  dfb_apply refuses v1, so dfb_model_forward_full runs the whole model and spec_e is compared with ref64's apply
    of that call's own m, coefs and alpha, at frame counts around the 8-frame warp tile and the 32-frame CTA.  K = 1 (worst
    err / bound on an H100 80GB HBM3: 0.995 plain, 0.997 with mask_only, 0.65 with the post filter, at either nb_df)."""
    _, nb_df, mode, la = KINDS[kind]
    pf, mask_only = OPTS[opt]
    model = models[kind]
    x = torch.from_numpy(noisy(2, Tf * HOP + 131, seed=300 + Tf))
    sp, fe, fs = df_features(x, st, nb_df, alpha=model.cfg.norm_alpha)
    got, m, c, a = forward_full(model, st, sp, fe, fs, pf, mask_only)
    assert np.isfinite(a).all() and ((a >= 0) & (a <= 1)).all()
    ref, b = R.apply(complex_of(sp[:, 0]), m, c, st.erb_widths(), mode=mode, nb_df=nb_df, order=5, lookahead=la,
                     post_filter=pf, mask_only=mask_only, alpha=a)
    assert_within(f"{kind} {opt} Tf={Tf}", got, ref, b, 1)


@pytest.mark.parametrize("opt", ["plain", "pf"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2"])
def test_apply_16_frame_warps(st, models, kind, opt):
    """B * Tf / 16 >= 6000 switches the apply kernel to 16 frames per warp: 64 streams of 1501 frames, three of them
    compared in full (the first, one inside, the last).  K = 1 (worst err / bound on an H100 80GB HBM3: 0.998; 0.65 with
    the post filter)."""
    run_apply_case(st, models, kind, opt, 64, 1501, seed=7, rows=[0, 37, 63])


@pytest.mark.parametrize("Tf", [1, 8, 9, 17, 33, 64, 65])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("kind", ["dfn3_df64", "dfn2_df64", "dfn3_e24"])
def test_generic_apply_against_ref64(st, models, kind, opt, Tf):
    """nb_df = 64, or 24 ERB bands: dfb_apply runs k_apply_synthesis_generic.  K = 1 (worst err / bound on an H100 80GB HBM3:
    0.996, 0.60 with the post filter at nb_df = 64; 0.991, 0.56 with the post filter at 24 bands)."""
    run_apply_case(st, models, kind, opt, 2, Tf, seed=50 + Tf)


# ------------------------------------------------------------------ fused synthesis ----
@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2", "v1"])
def test_fused_synthesis_against_ref64(st, models, kind):
    """enhance(pad=False) in one time chunk against the float64 ISTFT of the spec_e that DfNet.forward returns for the same
    df_features: the irFFT, window and overlap-add of k_apply_synthesis, including the tail of each warp's frame t0 - 1,
    at lengths that end inside and on a warp / CTA tile; and the attenuation limit mixed in before the ISTFT.  One-chunk
    enhance and forward compute the same model outputs, so the bound is ref64's ISTFT bound alone.  K = 1 (worst
    err / bound on an H100 80GB HBM3: 0.10, with the limit 0.05; DeepFilterNet v1 0.05, with the limit 0.04)."""
    model = models[kind]
    model.set_chunking(1, 1, 1)
    lim_db = 12.0
    lim = 10 ** (-lim_db / 20)
    try:
        for Tf in (8, 9, 31, 32, 33, 63, 64, 65):
            x = torch.from_numpy(noisy(2, Tf * HOP + 211, seed=200 + Tf))
            sp, fe, fs = df_features(x, st, model.nb_df)
            spec_e = complex_of(model(sp, fe, fs)[0][:, 0])
            ref, b = R.istft(spec_e, st.fft_window(), HOP)
            assert_within(f"{kind} Tf={Tf}", enhance(model, st, x, pad=False).numpy(), ref, b, 1)
            mixed, bm = R.atten_limit(complex_of(sp[:, 0]), spec_e, np.zeros(spec_e.shape), lim)
            ref, b = R.istft(mixed, st.fft_window(), HOP, bm)
            assert_within(f"{kind} Tf={Tf} atten", enhance(model, st, x, pad=False, atten_lim_db=lim_db).numpy(), ref, b, 1)
    finally:
        model.set_chunking()
