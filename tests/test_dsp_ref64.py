"""CPU: the float64 DSP reference (tests/dsp_ref64.py) and its error bounds against the fp32 CPU oracle.

The fp32 oracle (oracle/libdf_oracle.c for the STFT, ERB and norms; the oracle's torch formulas for the apply stages) is an
fp32 evaluation of the same formulas, so it has to lie within the bounds the GPU tests use, element by element, with the
same k = 1.  The bounds must also stay tight enough that a small change of a formula falls outside them."""
import numpy as np
import pytest
import torch

import dfnet1_oracle as O1
import dfnet_oracle as O
import dsp_ref64 as R
import libdf_oracle as LO
from tests_common import synth_audio

HOP = 480


@pytest.fixture(scope="module")
def ost():
    return LO.DF(48000, 960, HOP, 32, 2)


within = R.err_ratio


def features(ost, C, T, seed):
    x = synth_audio(C, T, seed=seed).numpy()
    x[0, 1000:1960] = 0.0          # whole frames of digital silence: the 1e-10 floor and |X| = 0 bins
    X, bX = R.stft(x, ost.fft_window(), HOP)
    return x, X, bX


@pytest.mark.parametrize("T", [480, 479 + 480 * 9, 480 * 150 + 17])
def test_stft_and_erb_db(ost, T):
    """Oracle spectrum and ERB dB within the ref64 bounds (measured max err / bound: STFT 0.05, dB 0.16)."""
    x, X, bX = features(ost, 2, T, seed=3)
    spec = ost.analysis(x)
    assert spec.shape == X.shape
    assert within(spec, X, bX) <= 1
    db, bdb = R.erb_db(X, bX, ost.erb_widths())
    assert within(LO.erb(spec, ost.erb_widths()), db, bdb) <= 1
    assert np.median(bX / np.maximum(np.abs(X), 1e-30)) < 1e-4     # not vacuous


@pytest.mark.parametrize("T", [50, 128, 300])
def test_norms(ost, T):
    """erb_norm / unit_norm of the oracle within the bounds chained through ref64's STFT and dB, from the init states and
    from given states (measured max err / bound: mean norm 0.20, unit norm 0.11, mean norm of exact fp32 inputs 0.66)."""
    x, X, bX = features(ost, 2, T * HOP, seed=4)
    spec = ost.analysis(x)
    w = ost.erb_widths()
    db, bdb = R.erb_db(X, bX, w)
    for st in (None, np.random.default_rng(1).uniform(-90, -20, (2, 32)).astype(np.float32)):
        ref, b = R.mean_norm(db, 0.99, st, bdb)
        assert within(LO.erb_norm(LO.erb(spec, w), 0.99, st), ref, b) <= 1
    for F, st in ((96, None), (481, np.random.default_rng(2).uniform(1e-4, 1e-2, (2, 481)).astype(np.float32))):
        ref, b = R.unit_norm(X[..., :F], 0.99, st, bX[..., :F])
        assert within(LO.unit_norm(np.ascontiguousarray(spec[..., :F]), 0.99, st), ref, b) <= 1
    # the exact fp32 inputs (no carried input error): libdf.erb_norm's own contract
    e = LO.erb(spec, w)
    ref, b = R.mean_norm(e.astype(np.float64), 0.9)
    assert within(LO.erb_norm(e, 0.9), ref, b) <= 1


def random_apply_inputs(B, T, nb_df, order, seed):
    rng = np.random.default_rng(seed)
    spec = (rng.standard_normal((B, T, 481)) + 1j * rng.standard_normal((B, T, 481))).astype(np.complex64) * 0.1
    spec[rng.random((B, T, 481)) < 0.1] = 0
    m = rng.random((B, T, 32)).astype(np.float32)
    m[rng.random(m.shape) < 0.1] = 0
    m[rng.random(m.shape) < 0.1] = 1
    c = (rng.standard_normal((B, T, nb_df, order)) + 1j * rng.standard_normal((B, T, nb_df, order))).astype(np.complex64) * 0.5
    return spec, m, c


def oracle_apply(spec, m, c, widths, mode, nb_df, order, la, pf, mask_only):
    """dfnet_oracle.dfnet_forward's apply stages (its lines, in fp32 torch) on given model outputs."""
    s = torch.view_as_real(torch.from_numpy(spec)).unsqueeze(1)
    mt = torch.from_numpy(m).unsqueeze(1)
    coefs = torch.view_as_real(torch.from_numpy(c)).reshape(*c.shape[:3], 2 * order)
    inv = O.erb_inv_matrix(widths)
    m_app = mt
    if pf and mode == 2:
        beta = 0.02
        m_sin = mt * torch.sin(np.pi * mt / 2)
        m_app = (1 + beta) * mt / (1 + beta * mt.div(m_sin.clamp_min(1e-12)).pow(2))
    spec_m = O.apply_mask(s, m_app, inv)
    if mode == 2:
        e = spec_m if mask_only else O.deep_filter(spec_m, coefs, nb_df, order, la)
    else:
        if mask_only:
            e = spec_m
        else:
            e = O.deep_filter(s, coefs, nb_df, order, la)
            e[..., nb_df:, :] = spec_m[..., nb_df:, :]
        if pf:
            beta, eps = 0.02, 1e-12
            mask = (torch.view_as_complex(e.contiguous()).abs() / torch.view_as_complex(s.contiguous()).abs().add(eps)).clamp(eps, 1)
            mask_sin = mask * torch.sin(np.pi * mask / 2).clamp_min(eps)
            g = (1 + beta) / (1 + beta * mask.div(mask_sin).pow(2))
            e = e * g.unsqueeze(-1)
    return torch.view_as_complex(e.squeeze(1).contiguous()).numpy()


@pytest.mark.parametrize("mode,la", [(1, 2), (1, 0), (2, 2)])
@pytest.mark.parametrize("pf,mask_only", [(False, False), (True, False), (False, True), (True, True)])
def test_apply_stages(ost, mode, la, pf, mask_only):
    """Gains, deep filter, DeepFilterNet2's masked deep filter and both post filters of the fp32 oracle within ref64's bound
    (measured max err / bound: 0.98, a single rounded product against its u |x g| bound)."""
    w = ost.erb_widths()
    spec, m, c = random_apply_inputs(2, 19, 96, 5, seed=mode * 10 + la)
    ref, b = R.apply(spec, m, c, w, mode=mode, nb_df=96, order=5, lookahead=la, post_filter=pf, mask_only=mask_only)
    assert within(oracle_apply(spec, m, c, w, mode, 96, 5, la, pf, mask_only), ref, b) <= 1


def oracle_df_alpha(spec, m, c, alpha, widths, nb_df, order, la, pf):
    """DeepFilterNet v1's apply stages in fp32 torch: the (optionally post-filtered) mask, then dfnet1_oracle's DfOp
    real_unfold blended by alpha with the masked bins."""
    s = torch.view_as_real(torch.from_numpy(spec)).unsqueeze(1)
    mt = torch.from_numpy(m).unsqueeze(1)
    if pf:
        beta = 0.02
        m_sin = mt * torch.sin(np.pi * mt / 2)
        mt = (1 + beta) * mt / (1 + beta * mt.div(m_sin.clamp_min(1e-12)).pow(2))
    spec_m = O.apply_mask(s, mt, O.erb_inv_matrix(widths))
    coefs = torch.view_as_real(torch.from_numpy(c)).permute(0, 1, 3, 2, 4)      # [B,T,O,Fd,2]
    e = O1.df_op_real_unfold(spec_m, coefs, torch.from_numpy(alpha).unsqueeze(-1), nb_df, order, la)
    return torch.view_as_complex(e.squeeze(1).contiguous()).numpy()


def random_alpha(B, T, seed):
    rng = np.random.default_rng(seed)
    a = rng.random((B, T)).astype(np.float32)
    a[:, ::5] = 0.0     # exact 0 and 1: only one of the blend's terms remains
    a[:, 1::5] = 1.0
    return a


@pytest.mark.parametrize("la", [0, 1, 3])
@pytest.mark.parametrize("pf", [False, True])
def test_alpha_blend(ost, la, pf):
    """DeepFilterNet v1's alpha blend (mode 2 with alpha) of the fp32 oracle within ref64's bound, with and without Mask.pf,
    at look-aheads 0, 1 (shipped) and 3 (measured max err / bound: 0.99, a gain bin's single rounded product; 0.34 over
    the blended DF bins)."""
    w = ost.erb_widths()
    spec, m, c = random_apply_inputs(2, 19, 96, 5, seed=70 + la)
    alpha = random_alpha(2, 19, seed=la)
    ref, b = R.apply(spec, m, c, w, mode=2, nb_df=96, order=5, lookahead=la, post_filter=pf, alpha=alpha)
    assert within(oracle_df_alpha(spec, m, c, alpha, w, 96, 5, la, pf), ref, b) <= 1


def test_bounds_see_small_formula_changes(ost):
    """The bounds are tight enough for the changes the GPU tests must catch: a deep-filter tap one frame off, and the post
    filter's sine argument scaled by 1 + 2^-10, each leave their bound somewhere."""
    w = ost.erb_widths()
    spec, m, c = random_apply_inputs(1, 12, 96, 5, seed=1)
    ref, b = R.apply(spec, m, c, w, mode=1, nb_df=96, order=5, lookahead=2)
    off, _ = R.apply(spec, m, c, w, mode=1, nb_df=96, order=5, lookahead=3)
    assert within(off, ref, b) > 1e3
    g, bg = R.pf_gain_mask(m.astype(np.float64))
    beta, mm = 0.02, m.astype(np.float64)
    s = np.sin(np.pi * mm / 2 * (1 + 2.0 ** -10))
    gm = (1 + beta) * mm / (1 + beta * np.divide(mm, np.maximum(mm * s, 1e-12)) ** 2)
    assert within(gm, g, np.maximum(bg, 1e-300)) > 10


@pytest.mark.parametrize("Tf", [1, 2, 17, 64])
def test_istft_and_atten_limit(ost, Tf):
    """The oracle's ISTFT with overlap-add, and the attenuation-limit mix, within ref64's bounds (measured max err / bound:
    ISTFT 0.01, limit 0.54)."""
    rng = np.random.default_rng(Tf)
    X = ((rng.standard_normal((2, Tf, 481)) + 1j * rng.standard_normal((2, Tf, 481))) * 0.05).astype(np.complex64)
    ref, b = R.istft(X, ost.fft_window(), HOP)
    assert within(ost.synthesis(X.copy()), ref, b) <= 1
    Y = (X * rng.random(X.shape)).astype(np.complex64)
    lim = 10 ** (-12 / 20)
    got = torch.from_numpy(X) * lim + torch.from_numpy(Y) * (1 - lim)
    out, bo = R.atten_limit(X.astype(np.complex128), Y.astype(np.complex128), np.zeros(X.shape), lim)
    assert within(got.numpy(), out, bo) <= 1


F32 = np.float32
TH = (-10.0, 30.0, 20.0)        # tract's default min / max_erb / max_df thresholds (fp32-exact)


def stage_lsnr(B, T, seed, th=TH):
    """LSNR rows that visit every stage, with values exactly at each threshold and one fp32 ulp either side."""
    rng = np.random.default_rng(seed)
    pick = [x for v in th for x in (np.nextafter(F32(v), F32(-np.inf)), F32(v), np.nextafter(F32(v), F32(np.inf)))]
    pick += [F32(th[0] - 5), F32((th[0] + th[2]) / 2), F32((th[1] + th[2]) / 2), F32(th[1] + 5)]
    return np.asarray(rng.choice(pick, (B, T)), np.float32)


def linked_oracle_rows(spec, m, c, lsnr, w, channels, reduce, la, lim):
    """tests/linked_oracle.py's fp32 torch statement: the link reduction, the DeepFilterNet3 apply stages on the shared mask,
    the stage gating from each group's first channel, then the limit."""
    import linked_oracle as LK
    s = torch.view_as_real(torch.from_numpy(spec)).unsqueeze(1)
    ml = LK.reduce_mask(torch.from_numpy(m).unsqueeze(1), channels, reduce)
    e = oracle_apply(spec, ml.squeeze(1).numpy(), c, w, 1, 96, 5, la, False, False)
    e = torch.view_as_real(torch.from_numpy(e)).unsqueeze(1)
    out = LK.apply_stages(s, e, ml, torch.from_numpy(lsnr)[..., None], w, channels, *TH)
    out = torch.view_as_complex(out.squeeze(1).contiguous())
    if lim:
        out = torch.from_numpy(spec) * lim + out * (1 - lim)
    return out.numpy()


@pytest.mark.parametrize("lim", [0.0, float(F32(10 ** (-12 / 20)))])
@pytest.mark.parametrize("channels,reduce", [(1, "max"), (2, "max"), (2, "mean"), (3, "mean"), (5, "mean"), (3, "max")])
def test_apply_rows_against_linked_oracle(ost, channels, reduce, lim):
    """ref64's row-level apply (stages, link reduction, limit, ISTFT) and linked_oracle's fp32 torch restatement of the same
    step agree within the bounds with K = 1, at every stage, with LSNR values exactly at each threshold and one ulp either
    side (measured max err / bound: spectrum 0.99, 0.54 with the limit; audio 0.012)."""
    w = ost.erb_widths()
    B, T = 2 * channels, 23
    spec, m, c = random_apply_inputs(B, T, 96, 5, seed=channels * 7 + len(reduce))
    lsnr = stage_lsnr(B, T, seed=channels)
    links = [(b - b % channels, channels) for b in range(B)]
    (Y, bY, wY), (a, ba, wa) = R.apply_rows(spec, m, c, w, ost.fft_window(), mode=1, nb_df=96, order=5, lookahead=2, Tf=T,
                                            n_audio=B * T * HOP, lsnr=lsnr, th=TH, atten_lim=lim, links=links, reduce=reduce,
                                            out_len=T * HOP)
    assert wY.all() and wa.all()
    st = R.stage_of(lsnr[::channels].repeat(channels, 0), *TH)
    assert all((st == k).any() for k in range(4))
    got = linked_oracle_rows(spec, m, c, lsnr, w, channels, reduce, 2, lim)
    rs, ra = within(got, Y, bY), within(ost.synthesis(got.astype(np.complex64)).reshape(-1), a, ba)
    print(f"err/bound spectrum {rs:.3g} audio {ra:.3g}")
    assert rs <= 1 and ra <= 1


def test_apply_rows_bounds_see_stage_and_switch_errors(ost):
    """The row-level bounds are tight enough for the errors the GPU tests must catch: an LSNR exactly at a threshold taken
    to the other side (a comparison written with <= / >=), a settings switch one frame late, a slot's first frame
    zeroed, and a link mean summed in another order, each leave the bound of the correct reference."""
    w, win = ost.erb_widths(), ost.fft_window()
    B, T = 3, 20
    spec, m, c = random_apply_inputs(B, T, 96, 5, seed=5)
    lsnr = np.full((B, T), F32(0.0), np.float32)
    kw = dict(mode=1, nb_df=96, order=5, lookahead=2, Tf=T, n_audio=B * T * HOP, th=TH, out_len=T * HOP)
    ref = R.apply_rows(spec, m, c, w, win, lsnr=lsnr, **kw)
    for th, side in zip(TH, (-np.inf, np.inf, np.inf)):
        eq = lsnr.copy()
        eq[:, 7] = F32(th)
        (Y, bY, _), (a, ba, _) = R.apply_rows(spec, m, c, w, win, lsnr=eq, **kw)
        moved = eq.copy()
        moved[:, 7] = np.nextafter(F32(th), F32(side))      # what the flipped comparison computes at equality
        (Ym, _, _), (am, _, _) = R.apply_rows(spec, m, c, w, win, lsnr=moved, **kw)
        assert within(Ym, Y, bY) > 1e3 and within(am, a, ba) > 1e3
    ctl = [dict(lim=0.25, beta=0.0, lim0=0.0, beta0=0.02, sw=9, th_min=0.0, th_erb=0.0, th_df=0.0, gate=0)] * B
    rows = [(b * T * HOP, T * HOP, 100) for b in range(B)]
    (Y, bY, _), (a, ba, _) = R.apply_rows(spec, m, c, w, win, ctl=ctl, rows=rows, **kw)
    late = [dict(ctl[0], sw=10)] * B
    (Ym, _, _), (am, _, _) = R.apply_rows(spec, m, c, w, win, ctl=late, rows=rows, **kw)
    assert within(Ym, Y, bY) > 1e3 and within(am, a, ba) > 1e3
    first = [4] * B
    (Y, bY, _), _ = R.apply_rows(spec, m, c, w, win, rows=rows, first=first, **kw)
    (Ym, _, _), _ = R.apply_rows(spec, m, c, w, win, rows=rows, first=[5] * B, **kw)
    assert within(Ym, Y, bY) > 1e3
    links = [(0, 3)] * 3
    m = m.copy()
    m[0, 1::4], m[1:, 1::4] = 1.0, F32(0.4 * 2.0 ** -23)      # the reordered sum rounds 1 up by one ulp
    (Y, bY, _), _ = R.apply_rows(spec, m, c, w, win, links=links, reduce="mean", **kw)
    rev = np.ascontiguousarray(m[::-1])
    mean_rev = ((rev[0] + rev[1]).astype(np.float32) + rev[2]).astype(np.float32) * (F32(1) / F32(3))
    assert (mean_rev != R.reduce_link_mask(m, links, "mean")[0]).any()
    (Ym, _, _), _ = R.apply_rows(spec, np.broadcast_to(mean_rev, m.shape).copy(), c, w, win, **kw)
    assert within(Ym, Y, bY) > 1.5
