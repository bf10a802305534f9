"""Float64 restatement of the three metrics of deepfilternet_b200.evaluation_utils, written from their definitions
(DESIGN.md section 5j, deepfilternet_b200/stoi.py): SI-SDR, df/stoi.py's STOI after a sinc_fast resample to 10 kHz, and
sepm.SNRseg after a sinc_fast resample to 16 kHz.  numpy only, apart from the resampler taps, which are
io.resample_kernel's (torchaudio's) float32 taps.  Also exposes the integer counts of STOI's silence removal and STFT.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np

EPS64 = float(np.finfo(np.float64).eps)
EPS32 = float(np.finfo(np.float32).eps)
_TAPS: Dict[Tuple[int, int], Tuple[np.ndarray, int, int, int]] = {}


def taps(sr: int, to: int):
    """(taps float64 [nw][K], width, og, nw) of io.resample_kernel(sr, to) with the sinc_fast parameters."""
    if (sr, to) not in _TAPS:
        from deepfilternet_b200.io import get_resample_params, resample_kernel
        k, width, og, nw = resample_kernel(sr, to, **get_resample_params("sinc_fast"))
        _TAPS[(sr, to)] = (k.numpy().astype(np.float64), width, og, nw)
    return _TAPS[(sr, to)]


def resample64(x: np.ndarray, sr: int, to: int) -> np.ndarray:
    """io.resample(x, sr, to) in float64: output i nw + j = sum_k taps[j][k] x[i og - width + k] (x zero outside),
    ceil(nw T / og) outputs."""
    x = np.asarray(x, dtype=np.float64)
    if sr == to:
        return x.copy()
    k, width, og, nw = taps(sr, to)
    T = x.size
    n_out = -(-nw * T // og)
    n_i = -(-n_out // nw)
    K = k.shape[1]
    xp = np.zeros(n_i * og + K, dtype=np.float64)
    xp[width:width + T] = x
    y = np.zeros((n_i, nw), dtype=np.float64)
    idx = np.arange(n_i) * og
    for kk in range(K):
        y += xp[idx + kk][:, None] * k[None, :, kk]
    return y.reshape(-1)[:n_out]


def si_sdr(reference: np.ndarray, estimate: np.ndarray) -> float:
    """si_sdr_speechmetrics with float32's eps, in float64."""
    r = np.asarray(reference, dtype=np.float64).reshape(-1)
    e = np.asarray(estimate, dtype=np.float64).reshape(-1)
    a = (EPS32 + r @ e) / (r @ r + EPS32)
    t = a * r
    return float(10 * np.log10((EPS32 + t @ t) / (EPS32 + (e - t) @ (e - t))))


def stoi_window() -> np.ndarray:
    """hann_window(258, periodic=False)[1:-1]: 0.5 - 0.5 cos(2 pi (n + 1) / 257), n = 0 .. 255."""
    return 0.5 - 0.5 * np.cos(2 * np.pi * (np.arange(256) + 1) / 257)


def third_octave_bins(fs=10000, nfft=512, num_bands=15, min_freq=150):
    """thirdoct: [(lo, hi)] FFT bin ranges of the bands, each edge the bin nearest to min_freq 2^((2 k -+ 1) / 6)."""
    f = np.arange(nfft // 2 + 1) * (fs / nfft)
    out = []
    for k in range(num_bands):
        lo = int(np.argmin((f - min_freq * 2.0 ** ((2 * k - 1) / 6)) ** 2))
        hi = int(np.argmin((f - min_freq * 2.0 ** ((2 * k + 1) / 6)) ** 2))
        out.append((lo, hi))
    return out


def silence_frames(x10: np.ndarray):
    """remove_silent_frames' framing of the 10 kHz clean row: (energies dB [nfr], threshold dB, pad_front, pad_end)."""
    T = x10.size
    pad = 256 - T % 256
    pf, pe = pad // 2, pad - pad // 2
    xp = np.concatenate([np.zeros(pf), x10, np.zeros(pe)])
    nfr = xp.size // 128 - 1
    w = stoi_window()
    fr = np.lib.stride_tricks.sliding_window_view(xp, 256)[::128][:nfr] * w
    en = 20 * np.log10(np.sqrt((fr ** 2).sum(1)) / 16 + EPS64)
    return en, en.max() - 40, pf, pe


def stoi(x: np.ndarray, y: np.ndarray, sr: int) -> Tuple[float, Tuple[int, int, int], float]:
    """df/stoi.py stoi of one pair: (value, (kept frames, length after silence removal, STFT frames), the smallest distance
    in dB of a frame energy from the 40 dB threshold).  value is NaN when fewer than 512 samples remain."""
    x10, y10 = resample64(x, sr, 10000), resample64(y, sr, 10000)
    en, thr, pf, pe = silence_frames(x10)
    keep = np.nonzero(en > thr)[0]
    margin = float(np.abs(en - thr).min())
    w = stoi_window()
    nk = keep.size
    n = (nk - 1) * 128 + 256
    xp = np.concatenate([np.zeros(pf), x10, np.zeros(pe)])
    yp = np.concatenate([np.zeros(pf), y10, np.zeros(pe)])
    xs, ys, ws = np.zeros(n), np.zeros(n), np.zeros(n)
    for j, i in enumerate(keep):
        xs[j * 128:j * 128 + 256] += xp[i * 128:i * 128 + 256] * w
        ys[j * 128:j * 128 + 256] += yp[i * 128:i * 128 + 256] * w
        ws[j * 128:j * 128 + 256] += w
    xs, ys = xs / ws, ys / ws
    s0 = pf if en[0] > thr else 0
    s1 = n - (pe if en[-1] > thr else 0)
    xs, ys = xs[s0:s1], ys[s0:s1]
    lc = xs.size
    if lc < 512:
        return float("nan"), (nk, lc, 0), margin
    L = 1 + (lc - 256) // 128
    bins = third_octave_bins()

    def bands(sig):
        fr = np.lib.stride_tricks.sliding_window_view(sig, 256)[::128][:L] * (w / w.sum())
        p = np.abs(np.fft.rfft(fr, 512, axis=1)) ** 2
        return np.stack([np.sqrt(p[:, lo:hi].sum(1)) for lo, hi in bins])   # [15, L]

    X, Y = bands(xs), bands(ys)
    N = 30 if L > 30 else L
    J = L - N + 1
    c = 10 ** (15 / 20)
    xa = np.lib.stride_tricks.sliding_window_view(X, N, axis=1)   # [15, J, N]
    ya = np.lib.stride_tricks.sliding_window_view(Y, N, axis=1)
    ya = ya * (np.linalg.norm(xa, axis=2, keepdims=True) / (np.linalg.norm(ya, axis=2, keepdims=True) + EPS64))
    ya = np.minimum(ya, xa * (1 + c))
    xa = xa - xa.mean(2, keepdims=True)
    ya = ya - ya.mean(2, keepdims=True)
    xa = xa / (np.linalg.norm(xa, axis=2, keepdims=True) + EPS64)
    ya = ya / (np.linalg.norm(ya, axis=2, keepdims=True) + EPS64)
    total = float((xa * ya).sum())
    return total / (15 * J), (nk, lc, L), margin


def ssnr(x: np.ndarray, y: np.ndarray, sr: int) -> float:
    """sepm.SNRseg(c16, d16, 16000) after a resample to 16 kHz: 480-sample frames at hop 120 times
    0.5 (1 - cos(2 pi n / 481)), n = 1 .. 480; 10 log10(S / (N + eps) + eps) clipped to [-10, 35]; the last frame
    dropped; the mean (NaN when no frame is left)."""
    c, d = resample64(x, sr, 16000), resample64(y, sr, 16000)
    wl, hop = round(0.03 * 16000), int(math.floor(0.25 * 0.03 * 16000))
    nfr = (c.size - wl + hop) // hop
    if nfr - 1 <= 0:
        return float("nan")
    w = 0.5 * (1 - np.cos(2 * np.pi * np.arange(1, wl + 1) / (wl + 1)))
    cw = np.lib.stride_tricks.sliding_window_view(c, wl)[:(nfr - 1) * hop:hop] * w
    dw = np.lib.stride_tricks.sliding_window_view(d, wl)[:(nfr - 1) * hop:hop] * w
    vals = np.clip(10 * np.log10((cw ** 2).sum(1) / (((cw - dw) ** 2).sum(1) + EPS64) + EPS64), -10.0, 35.0)
    return float(np.mean(vals))
