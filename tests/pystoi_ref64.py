"""Float64 restatement of pystoi 0.4.1's STOI and extended STOI (``pystoi.stoi(x, y, 10000, extended)``), as the
reference's ``df.evaluation_utils.stoi`` calls it after a sinc_fast resample to 10 kHz (DESIGN.md section 5n).  numpy
only.  pystoi's ESTOI adds ``eps * N(0, 1)`` noise before each normalisation; this restatement omits it, and a centred
row or column of norm 0 normalises to 0, as the device does.  Also exposes the integer counts of the silence removal, the
STFT and the segments, and the band magnitudes.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

import metrics_ref64 as M

EPS = float(np.finfo(np.float64).eps)
FRAME, HOP, NFFT, BANDS, SEG = 256, 128, 512, 15, 30
TOO_SHORT = 1e-5   # pystoi's value when fewer than 30 STFT frames remain (it warns)


def window() -> np.ndarray:
    """np.hanning(258)[1:-1]: 0.5 - 0.5 cos(2 pi n / 257), n = 1 .. 256."""
    return np.hanning(FRAME + 2)[1:-1]


def n_frames(n: int) -> int:
    """Frames of range(0, n - 256, 128): ceil((n - 256) / 128), 0 when n <= 256."""
    return max(0, -(-(n - FRAME) // HOP))


def obm() -> np.ndarray:
    """thirdoct(10000, 512, 15, 150) as a [15, 257] 0/1 matrix."""
    m = np.zeros((BANDS, NFFT // 2 + 1))
    for b, (lo, hi) in enumerate(M.third_octave_bins()):
        m[b, lo:hi] = 1.0
    return m


def _normalise(a: np.ndarray, axis: int) -> np.ndarray:
    a = a - a.mean(axis=axis, keepdims=True)
    n = np.sqrt(np.square(a).sum(axis=axis, keepdims=True))
    return np.divide(a, n, out=np.zeros_like(a), where=n > 0)


def pystoi10(x10: np.ndarray, y10: np.ndarray) -> Dict[str, object]:
    """Both measures of one pair of 10 kHz rows (float32 values, computed in float64): a dict with "stoi", "estoi" (NaN
    when the rows have no frame, 1e-5 when fewer than 30 STFT frames remain), the counts "F" (frames), "K" (kept frames),
    "lc" (silence-free length), "nf" (STFT frames), "J" (segments), "margin" (the smallest distance in dB of a frame
    energy from the 40 dB threshold) and the band magnitudes "X", "Y" [15, nf]."""
    x = np.asarray(x10, np.float64).reshape(-1)
    y = np.asarray(y10, np.float64).reshape(-1)
    F = n_frames(x.size)
    out: Dict[str, object] = dict(F=F, K=0, lc=0, nf=0, J=0, margin=float("inf"), stoi=float("nan"),
                                  estoi=float("nan"), X=np.zeros((BANDS, 0)), Y=np.zeros((BANDS, 0)))
    if F == 0:
        return out
    w = window()
    idx = np.arange(F)[:, None] * HOP + np.arange(FRAME)[None]
    xf, yf = x[idx] * w, y[idx] * w
    en = 20 * np.log10(np.sqrt(np.square(xf).sum(1)) + EPS)
    d = en.max() - 40 - en
    keep = np.nonzero(d < 0)[0]
    K = keep.size
    lc = (K - 1) * HOP + FRAME
    xs, ys = np.zeros(lc), np.zeros(lc)
    for j, i in enumerate(keep):
        xs[j * HOP:j * HOP + FRAME] += xf[i]
        ys[j * HOP:j * HOP + FRAME] += yf[i]
    nf = K - 1
    out.update(K=K, lc=lc, nf=nf, margin=float(np.abs(d).min()))
    sidx = np.arange(nf)[:, None] * HOP + np.arange(FRAME)[None]
    ob = obm()
    X = np.sqrt(ob @ np.square(np.abs(np.fft.rfft(xs[sidx] * w, NFFT, axis=1))).T)   # [15, nf]
    Y = np.sqrt(ob @ np.square(np.abs(np.fft.rfft(ys[sidx] * w, NFFT, axis=1))).T)
    out.update(X=X, Y=Y)
    if nf < SEG:
        out.update(stoi=TOO_SHORT, estoi=TOO_SHORT)
        return out
    J = nf - SEG + 1
    xa = np.stack([X[:, m:m + SEG] for m in range(J)])   # [J, 15, 30]
    ya = np.stack([Y[:, m:m + SEG] for m in range(J)])
    yn = ya * (np.linalg.norm(xa, axis=2, keepdims=True) / (np.linalg.norm(ya, axis=2, keepdims=True) + EPS))
    yp = np.minimum(yn, xa * (1 + 10 ** (15 / 20)))
    yp = yp - yp.mean(2, keepdims=True)
    xc = xa - xa.mean(2, keepdims=True)
    yp = yp / (np.linalg.norm(yp, axis=2, keepdims=True) + EPS)
    xc = xc / (np.linalg.norm(xc, axis=2, keepdims=True) + EPS)
    xe = _normalise(_normalise(xa, 2), 1)
    ye = _normalise(_normalise(ya, 2), 1)
    out.update(J=J, stoi=float(np.sum(yp * xc) / (J * BANDS)), estoi=float(np.sum(xe * ye / SEG) / J))
    return out


def rows10(x: np.ndarray, sr: int) -> np.ndarray:
    """io.resample(x, sr, 10000) in float64, rounded to float32 (the device's rows agree to the last bit or so)."""
    return np.asarray(x, np.float32) if sr == 10000 else M.resample64(x, sr, 10000).astype(np.float32)


def pystoi(x: np.ndarray, y: np.ndarray, sr: int, extended: bool = False, rows: Optional[tuple] = None) -> float:
    """df.evaluation_utils.stoi(x, y, sr, extended) with the float64 resampler (or the given 10 kHz rows)."""
    x10, y10 = rows if rows is not None else (rows10(x, sr), rows10(y, sr))
    return float(pystoi10(x10, y10)["estoi" if extended else "stoi"])
