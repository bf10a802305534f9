"""Float64 restatement of df/sepm.py's LLR, WSS and composite measure on 16 kHz rows, written from their definitions
(DESIGN.md section 5m), vectorised over frames; numpy only.

* Frame i is samples [120 i, 120 i + 480) for i < T = (L16 - 480) // 120, times w_n = 0.5 (1 - cos(2 pi n / 481)),
  n = 1 .. 480.
* LLR: autocorrelation lags 0 .. 16 and Levinson-Durbin in fp64 (the error floored at eps = 2^-52); R and the LPC
  polynomial A = [1, -a] rounded to float32 as the reference returns them; the ratio
  A_d' toeplitz(R_c) A_d / (A_c' toeplitz(R_c) A_c + eps) in fp64, 1000 where it is <= 0, its natural log.
* WSS: x + eps in fp64, windowed, the power of bins 0 .. 511 of a 1024-point FFT, Klatt's 25 critical-band energies in
  dB clamped at -100, their 24 slopes, the weights Kmax / (Kmax + max - E) * Klocmax / (Klocmax + peak - E) with the
  reference's local-peak rule, averaged over both signals; the weighted squared slope difference over the weights.
* Both per-entry values are the mean of the round(0.95 T) smallest frame values.
* composite: CSIG / CBAK / COVL are Hu & Loizou's regressions (IEEE TASLP 16(1), 2008) clipped to [1, 5].

wss_frames also returns a margin: the smallest |slope| between two bands not both clamped, and the smallest distance of
an unclamped band energy from -100 dB; a frame value can only change discontinuously (a local peak moves, a clamp
engages) when one of them crosses zero.
"""
from __future__ import annotations

import numpy as np

EPS = float(np.finfo(np.float64).eps)
WIN, HOP, P, NFFT, NBANDS = 480, 120, 16, 1024, 25
KMAX, KLOCMAX = 20.0, 1.0
# Klatt, "Prediction of perceived phonetic distance from critical-band spectra: a first step", ICASSP 1982: the 25
# critical bands' centre frequencies and bandwidths in Hz.
CENTRE = np.array([50.0, 120.0, 190.0, 260.0, 330.0, 400.0, 470.0, 540.0, 617.372, 703.378, 798.717, 904.128, 1020.38,
                   1148.30, 1288.72, 1442.54, 1610.70, 1794.16, 1993.93, 2211.08, 2446.71, 2701.97, 2978.04, 3276.17,
                   3597.63])
WIDTH = np.array([70.0, 70.0, 70.0, 70.0, 70.0, 70.0, 70.0, 77.3724, 86.0056, 95.3398, 105.411, 116.256, 127.914, 140.423,
                  153.823, 168.154, 183.457, 199.776, 217.153, 235.631, 255.255, 276.072, 298.126, 321.465, 346.136])
# Hu & Loizou, "Evaluation of objective quality measures for speech enhancement", IEEE TASLP 16(1):229-238, 2008
CSIG = (3.093, -1.029, 0.603, -0.009)          # const, LLR, PESQ, WSS
CBAK = (1.634, 0.478, -0.007, 0.063)           # const, PESQ, WSS, segSNR
COVL = (1.594, 0.805, -0.512, -0.007)          # const, PESQ, LLR, WSS


def n_frames(n16: int) -> int:
    return max(0, (n16 - WIN) // HOP)


def keep_count(T: int) -> int:
    """round(0.95 T), Python's round (half to even) of the double T * 0.95."""
    return int(round(T * 0.95))


def window() -> np.ndarray:
    return 0.5 * (1 - np.cos(2 * np.pi * np.arange(1, WIN + 1) / (WIN + 1)))


def frames(x: np.ndarray, T: int) -> np.ndarray:
    return np.lib.stride_tricks.sliding_window_view(x, WIN)[:T * HOP:HOP][:T]


def _levinson(R: np.ndarray) -> np.ndarray:
    """[F, 17] fp64 lags -> [F, 17] float32 A = [1, -a]."""
    F = R.shape[0]
    a = np.zeros((F, P))
    E = R[:, 0].copy()
    for i in range(P):
        s = (a[:, :i] * R[:, i:0:-1]).sum(1) if i else 0.0
        k = (R[:, i + 1] - s) / np.maximum(E, EPS)
        if i:
            a[:, :i] = a[:, :i] - k[:, None] * a[:, i - 1::-1]
        a[:, i] = k
        E = (1 - k * k) * E
    return np.concatenate([np.ones((F, 1)), -a], 1).astype(np.float32)


def llr_frames(c16: np.ndarray, d16: np.ndarray) -> np.ndarray:
    """The T per-frame log-likelihood ratios."""
    T = n_frames(c16.size)
    w = window()
    out = []
    Rs, As = [], []
    for x in (c16, d16):
        fr = frames(np.asarray(x, np.float32).astype(np.float64), T) * w
        R = np.stack([(fr[:, :WIN - k] * fr[:, k:]).sum(1) for k in range(P + 1)], 1)
        Rs.append(R.astype(np.float32))
        As.append(_levinson(R))
    idx = np.abs(np.arange(P + 1)[:, None] - np.arange(P + 1)[None, :])
    Tc = Rs[0].astype(np.float64)[:, idx]                          # [T, 17, 17] toeplitz(R_c)
    Ac, Ad = As[0].astype(np.float64), As[1].astype(np.float64)
    num = np.einsum("fi,fij,fj->f", Ad, Tc, Ad)
    den = np.einsum("fi,fij,fj->f", Ac, Tc, Ac) + EPS
    frac = num / den
    frac[frac <= 0] = 1000.0
    out = np.log(frac)
    return out


def crit_filters() -> np.ndarray:
    """[25, 512] critical-band filters over the kept bins at 16 kHz."""
    j = np.arange(NFFT // 2)
    f0 = np.floor(CENTRE / 8000.0 * (NFFT // 2))
    bw = WIDTH / 8000.0 * (NFFT // 2)
    norm = np.log(WIDTH[0]) - np.log(WIDTH)
    g = np.exp(-11 * ((j[None, :] - f0[:, None]) / bw[:, None]) ** 2 + norm[:, None])
    return g * (g > np.exp(-30.0 / (2.0 * 2.303)))


def _loc_peaks(slope: np.ndarray, energy: np.ndarray) -> np.ndarray:
    """[F, 24], [F, 25] -> [F, 24]: for a rising slope the energy just before the first band (from this one, up to band
    24) whose slope does not rise; otherwise the energy just after the last band at or below this one whose slope rises
    (band 0 when none does)."""
    F, S = slope.shape
    rise = slope > 0
    ii = np.arange(S)
    # first non-rising index >= ii (S when none)
    nr = np.where(~rise, ii[None, :], S)
    first_nr = np.minimum.accumulate(nr[:, ::-1], axis=1)[:, ::-1]
    # last rising index <= ii (-1 when none)
    r = np.where(rise, ii[None, :], -1)
    last_r = np.maximum.accumulate(r, axis=1)
    src = np.where(rise, first_nr - 1, last_r + 1)
    return np.take_along_axis(energy, src, axis=1)


def wss_frames(c16: np.ndarray, d16: np.ndarray):
    """(the T per-frame weighted spectral slope distances, margin)."""
    T = n_frames(c16.size)
    w = window()
    g = crit_filters()
    L, slopes, margin = [], [], np.inf
    for x in (c16, d16):
        fr = frames(np.asarray(x, np.float32).astype(np.float64) + EPS, T) * w
        p = np.abs(np.fft.rfft(fr, NFFT, axis=1)[:, :NFFT // 2]) ** 2
        raw = 10 * np.log10(p @ g.T)                                   # [T, 25]
        e = np.maximum(raw, -100.0)
        unclamped = raw > -100.0
        if unclamped.any():
            margin = min(margin, float(np.abs(raw[unclamped] + 100.0).min()))
        s = np.diff(e, axis=1)
        live = unclamped[:, 1:] | unclamped[:, :-1]
        if live.any():
            margin = min(margin, float(np.abs(s[live]).min()))
        L.append(e)
        slopes.append(s)
    W = []
    for e, s in zip(L, slopes):
        pk = _loc_peaks(s, e)
        W.append(KMAX / (KMAX + e.max(1, keepdims=True) - e[:, :-1]) * (KLOCMAX / (KLOCMAX + pk - e[:, :-1])))
    W = (W[0] + W[1]) / 2.0
    dist = (W * (slopes[0] - slopes[1]) ** 2).sum(1) / W.sum(1)
    return dist, margin


def trimmed_mean(v: np.ndarray) -> float:
    if v.size == 0:
        return float("nan")
    return float(np.sort(v)[:keep_count(v.size)].mean())


def llr(c16, d16) -> float:
    return trimmed_mean(llr_frames(c16, d16))


def wss(c16, d16) -> float:
    return trimmed_mean(wss_frames(c16, d16)[0])


def ssnr16(c16, d16) -> float:
    """sepm.SNRseg at 16 kHz."""
    c, d = np.asarray(c16, np.float64), np.asarray(d16, np.float64)
    nfr = (c.size - WIN + HOP) // HOP
    if nfr - 1 <= 0:
        return float("nan")
    cw = frames(c, nfr - 1) * window()
    dw = frames(d, nfr - 1) * window()
    v = np.clip(10 * np.log10((cw ** 2).sum(1) / (((cw - dw) ** 2).sum(1) + EPS) + EPS), -10.0, 35.0)
    return float(v.mean())


def regress(pesq: float, llr_: float, wss_: float, ssnr_: float):
    """(CSIG, CBAK, COVL), each clipped to [1, 5]."""
    csig = CSIG[0] + CSIG[1] * llr_ + CSIG[2] * pesq + CSIG[3] * wss_
    cbak = CBAK[0] + CBAK[1] * pesq + CBAK[2] * wss_ + CBAK[3] * ssnr_
    covl = COVL[0] + COVL[1] * pesq + COVL[2] * llr_ + COVL[3] * wss_
    return tuple(float(min(5.0, max(1.0, v))) for v in (csig, cbak, covl))


def composite(c16, d16, pesq: float):
    """(PESQ, CSIG, CBAK, COVL, SSNR) of a 16 kHz pair given its PESQ-WB; NaN for fewer than 600 samples."""
    if np.asarray(c16).size < WIN + HOP:
        return (float("nan"),) * 5
    lv, wv, sv = llr(c16, d16), wss(c16, d16), ssnr16(c16, d16)
    return (float(pesq),) + regress(float(pesq), lv, wv, sv) + (sv,)
