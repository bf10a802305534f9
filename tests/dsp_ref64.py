"""Float64 restatement of the DSP stages around the DNN, with an element-wise error bound for an fp32 evaluation of each.

Every function takes the fp32 values a kernel reads (promoted to float64) and returns
  (reference value in float64, bound)
where ``bound`` has the reference's shape and bounds |fp32 result - reference| element by element for any evaluation that
performs the same operations in fp32 (any summation order, with or without FMA): u = 2^-24 per rounding, gamma_n = n u / (1 - n u)
for a sum of n products (Higham, Accuracy and Stability of Numerical Algorithms, 3.1), plus the error of the inputs carried
through (the ``b*`` arguments).  The formulas follow the CPU oracle (oracle/libdf_oracle.c) and cite the same libDF /
DeepFilterNet lines (paths relative to the reference project).  numpy only, no GPU.
"""
import numpy as np

U = 2.0 ** -24                 # fp32 unit round-off
SINF_ABS = 2.0 ** -21          # __sinf absolute error for |x| <= pi (CUDA C Programming Guide, intrinsic functions: 2^-21.41)
PI_F32 = float(np.float32(3.14159265358979))
F32 = np.float32


def gamma(n):
    return n * U / (1.0 - n * U)


# fp32 FFT of length <= 1024 (forward and inverse): every output is a sum of the N inputs, each of which passes through at
# most 2 log2(N) roundings (a butterfly add and a rounded twiddle product per stage)
G_FFT = gamma(20)


def err_ratio(got, ref, bound):
    """max over elements of |got - ref| / bound (an exact match counts 0, a mismatch against a zero bound inf)."""
    err = np.abs(np.asarray(got, np.complex128) - ref)
    assert err.shape == np.shape(bound), (err.shape, np.shape(bound))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(r.max()) if r.size else 0.0


def band_of_bin(widths):
    return np.repeat(np.arange(len(widths)), np.asarray(widths, dtype=np.int64))


def wnorm_f32(fft, hop):
    """lib.rs:133, in fp32 as the library computes it."""
    return float(F32(1) / (F32(fft * fft) / F32(2 * hop)))


def stft(x, window, hop):
    """frame_analysis (libDF/src/lib.rs:356-394) over a whole signal from zero memory (pyDF/src/lib.rs:41-72):
    x [C, T] -> X [C, T // hop, N/2 + 1];  X[t, k] = wnorm * sum_n w[n] x[(t-1) hop + n] e^{-2 pi i k n / N}."""
    x = np.asarray(x, np.float64)
    w = np.asarray(window, np.float64)
    N = len(w)
    C, T = x.shape
    Tf = T // hop
    xp = np.concatenate([np.zeros((C, N - hop)), x[:, :Tf * hop]], 1)
    frames = np.lib.stride_tricks.sliding_window_view(xp, N, axis=1)[:, ::hop][:, :Tf] * w
    wn = wnorm_f32(N, hop)
    X = np.fft.rfft(frames, axis=-1) * wn
    # window products (1 rounding) + FFT + wnorm product
    bound = (wn * G_FFT * np.abs(frames).sum(-1))[..., None] + U * np.abs(X)
    return X, np.broadcast_to(bound, X.shape).copy()


def erb_db(X, bX, widths):
    """compute_band_corr with x == p (lib.rs:280-295: sum of |X|^2 * (1 / width) in band order) and the dB of
    lib.rs:207-210 (10 log10(e + 1e-10)): X [..., F] -> [..., E]."""
    widths = np.asarray(widths, np.int64)
    P = np.abs(X) ** 2
    # |X|^2 from re^2 + im^2 (3 roundings) and from the input error of X
    bP = gamma(3) * P + 2 * np.abs(X) * bX + bX ** 2
    edges = np.concatenate([[0], np.cumsum(widths)])
    E = np.add.reduceat(P, edges[:-1], axis=-1) / widths
    bE = np.add.reduceat(bP, edges[:-1], axis=-1) / widths
    # the band sum of w products with the rounded 1 / w (w + 1 roundings), then + 1e-10
    bE += gamma(widths + 2) * E
    e = E + 1e-10
    db = 10.0 * np.log10(e)
    be = bE + U * e
    # d(10 log10 e) = 10 / ln 10 * de / e, evaluated at the smallest e the fp32 sum can have; log10f (2 ulp) and * 10
    bdb = 10.0 / np.log(10.0) * be / np.maximum(e - be, e * 0.5) + 6 * U * np.abs(db)
    return db, bdb


def mean_norm_init(E):
    """linspace(-60, -90, E) in fp32 (transforms.rs:310 / oracle dfo_mean_norm_init)."""
    if E == 1:
        return np.full(1, -60.0)
    return (F32(-60) + np.arange(E, dtype=F32) * (F32(-30) / F32(E - 1))).astype(np.float64)


def unit_norm_init(F):
    """linspace(0.001, 0.0001, F) in fp32 (transforms.rs:341 / oracle dfo_unit_norm_init)."""
    if F == 1:
        return np.full(1, float(F32(0.001)))
    return (F32(0.001) + np.arange(F, dtype=F32) * ((F32(0.0001) - F32(0.001)) / F32(F - 1))).astype(np.float64)


def _alpha(alpha):
    a = F32(alpha)
    return float(a), float(F32(1) - a)     # 1 - alpha is exact in fp32 for alpha in [0.5, 1]


def mean_norm(x, alpha, state=None, bx=None):
    """band_mean_norm_erb (lib.rs:244-251): s = x (1 - a) + s a;  out = (x - s) / 40, per channel from `state` [C, E] or
    the linspace init.  x [C, T, E].  The EMA error decays by a per frame and gains at most 3 roundings (two products and
    the sum) plus the input error times (1 - a): accumulated, u |s| / (1 - a) order."""
    x = np.asarray(x, np.float64)
    C, T, E = x.shape
    a, oma = _alpha(alpha)
    bx = np.zeros_like(x) if bx is None else bx
    s = np.broadcast_to(mean_norm_init(E) if state is None else np.asarray(state, np.float64), (C, E)).copy()
    es = np.zeros((C, E))
    out, bout = np.empty_like(x), np.empty_like(x)
    for t in range(T):
        xt = x[:, t]
        sn = xt * oma + s * a
        es = a * es + oma * bx[:, t] + U * (np.abs(xt) * oma + np.abs(s) * a + np.abs(sn))
        s = sn
        out[:, t] = (xt - s) / 40.0
        bout[:, t] = (bx[:, t] + es) / 40.0 + 2 * U * np.abs(out[:, t])
    return out, bout


def unit_norm(X, alpha, state=None, bX=None):
    """band_unit_norm (lib.rs:253-259): s = |x| (1 - a) + s a;  out = x / sqrt(s).  X [C, T, F] complex."""
    X = np.asarray(X, np.complex128)
    C, T, F = X.shape
    a, oma = _alpha(alpha)
    bX = np.zeros(X.shape) if bX is None else bX
    s = np.broadcast_to(unit_norm_init(F) if state is None else np.asarray(state, np.float64), (C, F)).copy()
    es = np.zeros((C, F))
    out, bout = np.empty_like(X), np.empty(X.shape)
    for t in range(T):
        n = np.abs(X[:, t])
        sn = n * oma + s * a
        # hypotf within 2 ulp (4 u), then the EMA's 3 roundings
        es = a * es + oma * (bX[:, t] + 4 * U * n) + U * (n * oma + np.abs(s) * a + sn)
        s = sn
        d = np.sqrt(s)
        out[:, t] = X[:, t] / d
        # 1 / sqrt(s) moves by at most es / (2 (s - es)) relatively; sqrt and the divide round once each
        rel = es / (2 * np.maximum(s - es, s * 0.5)) + 2 * U
        bout[:, t] = bX[:, t] / d + np.abs(out[:, t]) * rel * (1 + rel)
    return out, bout


def _sin_err(theta):
    """|__sinf(fl(fl(pi_f * m) / 2)) - sin(pi m / 2)| for theta = pi m / 2 in [0, pi / 2]: the intrinsic's absolute error
    plus the argument's (pi_f and one product: 1.5 u relative)."""
    return SINF_ABS + 1.5 * U * theta * np.cos(theta)


def pf_gain_mask(m):
    """Mask.pf on ERB gains (DeepFilterNet/df/modules.py:234-245, beta = 0.02, deepfilternet2.py):
    m' = (1 + b) m / (1 + b (m / max(m sin(pi m / 2), 1e-12))^2).  Returns (m', bound) for the exact m given."""
    beta = 0.02
    m = np.asarray(m, np.float64)
    th = np.pi * m / 2
    s = np.sin(th)
    ms = np.maximum(m * s, 1e-12)
    q = np.divide(m, ms)
    g = (1 + beta) * m / (1 + beta * q * q)
    w = beta * q * q / (1 + beta * q * q)
    # sin's error moves q^2 by 2 e_s / sin relatively (only while m sin > 1e-12), and g by w times that; 7 roundings
    rel_sin = np.where(m * s > 1e-12, 2 * _sin_err(th) / np.maximum(s, 1e-30), 0.0)
    return g, g * (w * (rel_sin + 6 * U) + 4 * U)


def pf_gain_spec(y, x, by, beta):
    """DeepFilterNet3's post filter (deepfilternet3.py:448-454): mask = clamp(|y| / (|x| + 1e-12), 1e-12, 1),
    g = (1 + b) / (1 + b (mask / (mask max(sin(pi mask / 2), 1e-12)))^2);  returns (y g, bound) given the bound `by` of y."""
    eps = 1e-12
    ay, ax = np.abs(y), np.abs(x)
    raw = ay / (ax + eps)
    mask = np.clip(raw, eps, 1.0)
    th = np.pi * mask / 2
    s = np.maximum(np.sin(th), eps)
    q2 = 1.0 / (s * s)
    g = (1 + beta) / (1 + beta * q2)
    # mask: two sqrtf of sums of squares (2 u each), the + eps and the divide, plus the input error of y
    bmask = (by + 2 * U * ay) / (ax + eps) + 4 * U * np.minimum(raw, 1.0)
    # clamped at 1 (where dg / dmask = 0), a perturbed |y| may still land below 1
    bmask = np.where((raw >= 1.0) & ((ay - by) / (ax + eps) * (1 - 4 * U) >= 1.0), 0.0, bmask)

    def slope(mk):   # |dg / dmask| = (1 + b) b pi cos / sin^3 (pi mk / 2) / (1 + b / sin^2)^2
        sn = np.maximum(np.sin(np.pi * mk / 2), eps)
        return (1 + beta) * beta * np.pi * np.cos(np.pi * mk / 2) / sn ** 3 / (1 + beta / (sn * sn)) ** 2

    # the slope is smooth in mask and bmask is narrow: take the largest of its values at both ends and the middle
    lo, hi = np.clip(mask - bmask, eps, 1.0), np.clip(mask + bmask, eps, 1.0)
    slope = np.maximum(np.maximum(slope(lo), slope(hi)), slope(mask))
    w = beta * q2 / (1 + beta * q2)
    rel_sin = 2 * _sin_err(th) / s
    bg = slope * bmask + g * (w * (rel_sin + 6 * U) + 4 * U)
    return y * g, by * g + ay * bg + U * ay * g


def _deep_filter(S, bS, coefs, nb_df, order, lookahead, Tv):
    """MF.DF (DeepFilterNet/df/multiframe.py:72-74,126-136,169-180): Y[t, k] = sum_o S[t + o - (O - 1 - L), k] W[t, k, o]
    for k < nb_df, rows outside [0, Tv) zero.  S [B, T, F], coefs [B, T, nb_df, O] complex."""
    B, T, _ = S.shape
    back = order - 1 - lookahead
    Y = np.zeros((B, T, nb_df), np.complex128)
    acc = np.zeros((B, T, nb_df))
    inb = np.zeros((B, T, nb_df))
    for o in range(order):
        tt = np.arange(T) + o - back
        ok = (tt >= 0) & (tt < Tv)
        src = np.zeros((B, T, nb_df), np.complex128)
        bsrc = np.zeros((B, T, nb_df))
        src[:, ok] = S[:, tt[ok], :nb_df]
        bsrc[:, ok] = bS[:, tt[ok], :nb_df]
        w = coefs[..., o]
        Y += src * w
        l1s = np.abs(src.real) + np.abs(src.imag)
        l1w = np.abs(w.real) + np.abs(w.imag)
        acc += l1s * l1w
        inb += bsrc * np.abs(w)
    return Y, gamma(2 * order) * acc + inb


def apply(spec, m, coefs, widths, *, mode, nb_df, order, lookahead, post_filter=False, pf_beta=0.02, mask_only=False,
          Tv=None, alpha=None):
    """The enhanced spectrum of one model output (deepfilternet3.py:438-454 / deepfilternet2.py:481-505):
      mode 1 (DeepFilterNet3): k < nb_df: deep filter of the noisy spectrum; k >= nb_df (or mask_only): spec * erb_inv(m)
        (lib.rs:314-326 == Mask.forward modules.py:266-269); then the optional post filter on every bin.
      mode 2 (DeepFilterNet2): spec * erb_inv(m') first, m' = Mask.pf(m) with the post filter, then the deep filter of
        that masked spectrum for k < nb_df (unless mask_only).
      mode 2 with alpha [B, T] (DeepFilterNet v1, DfOp real_unfold + assign_df, DeepFilterNet/df/modules.py:388-406,
        470-478): the deep-filtered DF bins blended with the masked bins, Y a + X_masked (1 - a).
    spec [B, T, F] complex, m [B, T, E], coefs [B, T, nb_df, O] complex -> (spec_e, bound)."""
    assert alpha is None or mode == 2, "the alpha blend filters the masked spectrum (mode 2)"
    spec = np.asarray(spec, np.complex128)
    m = np.asarray(m, np.float64)
    B, T, F = spec.shape
    Tv = T if Tv is None else Tv
    g, bg = m, np.zeros_like(m)
    if post_filter and mode == 2:
        g, bg = pf_gain_mask(m)
    bob = band_of_bin(widths)
    gb, bgb = g[..., bob], bg[..., bob]
    ax = np.abs(spec)
    xm = spec * gb
    bxm = U * ax * gb + ax * bgb
    if mask_only:
        y, by = xm, bxm
    elif mode == 1:
        Yd, bYd = _deep_filter(spec, np.zeros(spec.shape), coefs, nb_df, order, lookahead, Tv)
        y, by = xm.copy(), bxm.copy()
        y[..., :nb_df], by[..., :nb_df] = Yd, bYd
    else:
        Yd, bYd = _deep_filter(xm, bxm, coefs, nb_df, order, lookahead, Tv)
        if alpha is not None:
            # the blend's roundings: 1 - a, the masked bin's products with g and (1 - a) in either association, Y a and
            # the sum; the inputs' bounds carried through the weights a and 1 - a (both in [0, 1])
            a = np.asarray(alpha, np.float64)[..., None]
            xd, bxd = xm[..., :nb_df], bxm[..., :nb_df]
            bYd = a * bYd + (1 - a) * bxd + gamma(4) * (a * np.abs(Yd) + (1 - a) * np.abs(xd))
            Yd = Yd * a + xd * (1 - a)
        y, by = xm.copy(), bxm.copy()
        y[..., :nb_df], by[..., :nb_df] = Yd, bYd
    if post_filter and mode == 1:
        y, by = pf_gain_spec(y, spec, by, pf_beta)
    return y, by


def atten_limit(x, y, by, lim):
    """enhance.py:238-240: noisy * lim + enhanced * (1 - lim).  lim is exact here; the library's fp32 powf(10, -db / 20)
    is within 4 u of it (the rounded exponent and powf), which moves the result by at most 4 u lim |x - y|."""
    ax, ay = np.abs(x), np.abs(y)
    out = x * lim + y * (1 - lim)
    return out, (1 - lim) * by + 4 * U * lim * np.abs(x - y) + 3 * U * (ax * lim + ay * (1 - lim))


def istft(X, window, hop, bX=None):
    """frame_synthesis (libDF/src/lib.rs:396-427) from zero memory (pyDF/src/lib.rs:74-107): the unnormalised inverse real
    DFT of every frame (imaginary parts of DC and Nyquist ignored, lib.rs:402), windowed, overlap-added:
    out[t hop + i] = w[i] x_t[i] + w[hop + i] x_{t-1}[hop + i].  X [C, Tf, F] -> [C, Tf hop]."""
    X = np.array(X, np.complex128)
    w = np.asarray(window, np.float64)
    N = len(w)
    C, Tf, F = X.shape
    X[..., 0] = X[..., 0].real
    X[..., -1] = X[..., -1].real
    y = np.fft.irfft(X, n=N, axis=-1) * N
    yw = y * w
    # each sample is a sum over the Hermitian spectrum: |X_0| + 2 sum_{0<k<F-1} |X_k| + |X_{F-1}|
    herm = np.full(F, 2.0)
    herm[0] = herm[-1] = 1.0
    l1 = np.abs(X) @ herm
    by = (G_FFT * l1)[..., None] * w + U * np.abs(yw)
    if bX is not None:
        by = by + ((bX @ herm)[..., None] * w)
    out = yw[..., :hop].copy()
    bout = by[..., :hop].copy()
    out[:, 1:] += yw[:, :-1, hop:]
    bout[:, 1:] += by[:, :-1, hop:]
    bout += U * np.abs(out)
    return out.reshape(C, Tf * hop), bout.reshape(C, Tf * hop)


def stage_of(lsnr, th_min, th_erb, th_df):
    """tract.rs:658-672 (DfTract::apply_stages), element-wise: 0 zero gains (lsnr < min), 1 unprocessed (> max_erb), 2 ERB
    gains only (> max_df), 3 gains and deep filter."""
    l = np.asarray(lsnr)
    return np.where(l < th_min, 0, np.where(l > th_erb, 1, np.where(l > th_df, 2, 3)))


def reduce_link_mask(m, links, reduce):
    """The ERB mask each stream applies: its link group's (first, n) max, or the mean as the fp32 sum in channel order times
    fl32(1 / n) (tract.rs:881-898), computed in numpy float32 and then exact.  m [B, T, E] fp32; links None: m itself."""
    m = np.asarray(m, np.float32)
    if links is None:
        return m.astype(np.float64)
    out = np.empty(m.shape, np.float64)
    for b, (f, n) in enumerate(links):
        v = m[f].copy()
        for c in range(1, n):
            v = np.maximum(v, m[f + c]) if reduce == "max" else (v + m[f + c]).astype(np.float32)
        if reduce != "max":
            v = (v * (F32(1) / F32(n))).astype(np.float32)
        out[b] = v
    return out


def apply_rows(spec, m, coefs, widths, window, *, mode, nb_df, order, lookahead, Tf, n_audio, post_filter=False,
               pf_beta=0.02, mask_only=False, alpha=None, Tv=None, lsnr=None, th=(-15.0, 35.0, 35.0), atten_lim=0.0,
               rows=None, first=None, links=None, reduce="max", ctl=None, w0=0, t_first=0, t_emit=None, out_offset=0,
               out_len=None, hop=480):
    """The apply + synthesis step of one window of a ragged batch or of streaming slots, row by row (the contract of
    include/dfb200.h dfb_debug_apply_rows).  spec [B, spec_T, F] with Tv (None: spec_T) existing rows, m [B, mc_T, E],
    coefs [B, mc_T, nb_df, O] complex, alpha / lsnr [B, mc_T] or None.  Per stream b, window frames t = 0 .. Tf - 1 are
    absolute frames w0 + t:
      geometry   rows[b] = (out_off, out_len, row_Tf): the stream ends at tfb = row_Tf - w0; it synthesises frames
                 [0, Te), Te = tfb if tfb <= Tf else t_emit, and its deep-filter taps read spectrum rows [0, min(Tv, tfb)).
                 DeepFilterNet2's masked taps apply the mask only to rows below mc_T.  rows None: Te = Tf, output row
                 b is audio[b out_len, (b + 1) out_len);
      link       links[b] = (first, n): the mask is the group's reduction (reduce_link_mask) and the stage follows the LSNR
                 of the group's first stream;
      stage      stage_of its LSNR with ctl[b]'s thresholds (gating only where ctl[b]["gate"]) or th (every row), when lsnr
                 is given; frames before the slot's first frame (first[b] - w0) are stage 0.  Stage 0: zeros; 1: the noisy
                 bins; 2: ERB gains on every bin; 3: the model's apply (apply).  The DeepFilterNet3 post filter applies at
                 stages 2 and 3 only (tract.rs:617), then the limit;
      settings   ctl[b] = dict(lim, beta, lim0, beta0, sw, th_min, th_erb, th_df, gate): from absolute frame sw on the
                 limit lim and DeepFilterNet3 post-filter beta (0: off) are lim / beta, before it lim0 / beta0.  ctl None:
                 atten_lim and (post_filter, pf_beta) on every frame;
      output     the ISTFT of frames [0, Te) from zero memory: frame t's samples t hop + i - out_offset for t >= t_first,
                 those in [0, out_len) of the row.
    -> (Y [B, Tf, F], bound, Y written [B, Tf] bool), (audio [n_audio], bound, written [n_audio] bool)."""
    spec = np.asarray(spec, np.complex128)
    B, spec_T, F = spec.shape
    mc_T = m.shape[1]
    Tv = spec_T if Tv is None else Tv
    t_emit = Tf if t_emit is None else t_emit
    ml = reduce_link_mask(m, links, reduce)
    bob = band_of_bin(widths)
    Y = np.zeros((B, Tf, F), np.complex128)
    bY = np.zeros((B, Tf, F))
    wY = np.zeros((B, Tf), bool)
    audio, baudio, waudio = np.zeros(n_audio), np.zeros(n_audio), np.zeros(n_audio, bool)
    for b in range(B):
        if rows is not None:
            off, olen, rtf = rows[b]
            tfb = rtf - w0
            Te = tfb if tfb <= Tf else t_emit
            Tvb = min(Tv, tfb)
        else:
            off, olen, Te, Tvb = b * out_len, out_len, Tf, Tv
        if Te <= 0:
            continue
        lb = links[b][0] if links is not None else b
        tz = max(first[b] - w0, 0) if first is not None else 0
        X = spec[b, :Te]
        g, bg = ml[b], np.zeros(ml[b].shape)
        if post_filter and mode == 2:
            g, bg = pf_gain_mask(ml[b])
        gb, bgb = g[:Te][:, bob], bg[:Te][:, bob]
        ax = np.abs(X)
        xm, bxm = X * gb, U * ax * gb + ax * bgb
        y, by = xm.copy(), bxm.copy()
        if not mask_only:
            Tn = max(Te, Tvb)
            src = np.zeros((Tn, F), np.complex128)
            bsrc = np.zeros((Tn, F))
            src[:Tvb] = spec[b, :Tvb]
            if mode == 2:       # the masked spectrum below mc_T, the bare one above
                k = min(Tvb, mc_T)
                gk, bgk = g[:k][:, bob], bg[:k][:, bob]
                a = np.abs(src[:k])
                bsrc[:k] = U * a * gk + a * bgk
                src[:k] = src[:k] * gk
            c = np.zeros((Tn, nb_df, order), np.complex128)
            c[:Te] = coefs[b, :Te]
            Yd, bYd = _deep_filter(src[None], bsrc[None], c[None], nb_df, order, lookahead, Tvb)
            Yd, bYd = Yd[0, :Te], bYd[0, :Te]
            if mode == 2 and alpha is not None:
                a = np.asarray(alpha[b, :Te], np.float64)[:, None]
                xd, bxd = xm[:, :nb_df], bxm[:, :nb_df]
                bYd = a * bYd + (1 - a) * bxd + gamma(4) * (a * np.abs(Yd) + (1 - a) * np.abs(xd))
                Yd = Yd * a + xd * (1 - a)
            y[:, :nb_df], by[:, :nb_df] = Yd, bYd
        # stages, per frame
        stage = np.full(Te, 3)
        c = ctl[b] if ctl is not None else None
        if lsnr is not None and (c is None or c["gate"]):
            t3 = (c["th_min"], c["th_erb"], c["th_df"]) if c is not None else th
            stage = stage_of(np.asarray(lsnr[lb, :Te], np.float64), *t3)
        stage[:min(tz, Te)] = 0
        s2 = (stage == 2)[:, None]
        y, by = np.where(s2, xm, y), np.where(s2, bxm, by)
        s1 = (stage == 1)[:, None]
        y, by = np.where(s1, X, y), np.where(s1, 0.0, by)
        s0 = (stage == 0)[:, None]
        y, by = np.where(s0, 0.0, y), np.where(s0, 0.0, by)
        now = (w0 + np.arange(Te) >= c["sw"]) if c is not None else np.ones(Te, bool)
        for t in range(Te):
            if c is not None:
                lim, beta = (c["lim"], c["beta"]) if now[t] else (c["lim0"], c["beta0"])
                pf1 = mode == 1 and beta > 0
            else:
                lim, beta, pf1 = atten_lim, pf_beta, post_filter and mode == 1
            if pf1 and stage[t] >= 2:
                y[t], by[t] = pf_gain_spec(y[t], X[t], by[t], beta)
            if lim > 0:
                y[t], by[t] = atten_limit(X[t], y[t], by[t], lim)
        Y[b, :Te], bY[b, :Te], wY[b, :Te] = y, by, True
        o, bo = istft(y[None], window, hop, by[None])
        for t in range(max(t_first, 0), Te):
            gpos = t * hop + np.arange(hop) - out_offset
            ok = (gpos >= 0) & (gpos < olen)
            audio[off + gpos[ok]] = o[0, t * hop:(t + 1) * hop][ok]
            baudio[off + gpos[ok]] = bo[0, t * hop:(t + 1) * hop][ok]
            waudio[off + gpos[ok]] = True
    return (Y, bY, wY), (audio, baudio, waudio)
