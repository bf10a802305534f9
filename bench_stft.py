"""Throughput of libdf's STFT / ISTFT at several (sr, fft, hop) against torch / cuFFT computing the same transforms.

  analysis:  ours = dfb_analysis (device pointers): frames [t hop - (N - hop), t hop + hop), window, real FFT, wnorm,
             written as [B, Tf, F];
             torch = F.pad(N - hop zeros on the left) + torch.stft(center=False, window) * wnorm + transpose to [B, Tf, F].
  synthesis: ours = dfb_synthesis: inverse real FFT, window, overlap-add of every earlier frame;
             torch = torch.fft.irfft(X, n=N) * N * window + overlap-add with F.fold.
Both sides run device resident on the same inputs (10 s per stream of a seeded signal), warmed up, timed with CUDA
events, median of 5, alternating ours / torch in one process.  Achieved GB/s counts compulsory bytes only: 4 T read plus
8 F per frame written for the analysis, the reverse for the synthesis; the share of peak is against the H100 SXM data
sheet's 3.35 TB/s.  Prints one JSON line per workload, then one with the card's name and power limit.

    python bench_stft.py [--seconds 10] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from deepfilternet_b200 import _lib, libdf  # noqa: E402
from deepfilternet_b200._lib import check  # noqa: E402

PEAK_BPS = 3.35e12
WORKLOADS = [   # (sr, fft, hop, streams, note)
    (16000, 320, 160, 512, "generic"),
    (48000, 512, 128, 128, "generic"),
    (48000, 2048, 512, 128, "generic"),
    (48000, 960, 240, 128, "generic"),
    (48000, 960, 480, 128, "specialised 960 / 480 kernels"),
]


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, plim = [s.strip() for s in out[0].split(",")]
        return {"gpu": name, "power_limit": plim}
    except Exception as e:   # the numbers stand without it, but say why it is missing
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})"}


def run(sr, N, H, B, seconds, reps):
    L = _lib.lib()
    st = libdf.DF(sr, N, H, 32, 1)
    T = int(sr * seconds)
    Tf, F = T // H, N // 2 + 1
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.rand((B, T), device="cuda", generator=g) - 0.5) * 0.2
    w = torch.from_numpy(st.fft_window()).cuda()
    wn = 1.0 / (float(N * N) / float(2 * H))
    spec = torch.empty((B, Tf, F, 2), device="cuda")
    y = torch.empty((B, Tf * H), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def ours_ana():
        check(L.dfb_analysis(st.handle, x.data_ptr(), B, T, spec.data_ptr(), stream))

    def torch_ana():
        xp = Fn.pad(x[:, :Tf * H], (N - H, 0))
        return (torch.stft(xp, n_fft=N, hop_length=H, window=w, center=False, return_complex=True) * wn).transpose(1, 2).contiguous()

    def ours_syn():
        check(L.dfb_synthesis(st.handle, spec.data_ptr(), B, Tf, y.data_ptr(), stream))

    Xc = torch.view_as_complex(spec)

    def torch_syn():
        fr = torch.fft.irfft(Xc, n=N) * (N * w)                       # [B, Tf, N]
        ola = Fn.fold(fr.transpose(1, 2), output_size=(1, (Tf - 1) * H + N), kernel_size=(1, N), stride=(1, H))
        return ola.reshape(B, -1)[:, :Tf * H]

    for f in (ours_ana, torch_ana, ours_syn, torch_syn):   # warm-up (module load, cuFFT plans)
        f()
        f()
    torch.cuda.synchronize()
    # same transform: compare once, outside the timed regions
    ours_ana()
    ref = torch_ana()
    torch.cuda.synchronize()
    ana_err = float((torch.view_as_complex(spec) - ref).abs().max() / ref.abs().max())
    ours_syn()
    ref_y = torch_syn()
    torch.cuda.synchronize()
    syn_err = float((y - ref_y).abs().max() / ref_y.abs().max())
    res = {}
    for name, a, b in (("analysis", ours_ana, torch_ana), ("synthesis", ours_syn, torch_syn)):
        t_ours, t_torch = [], []
        for _ in range(reps):   # alternate
            t_ours.append(timed(a, 1))
            t_torch.append(timed(b, 1))
        t_ours.sort()
        t_torch.sort()
        res[name] = (t_ours[reps // 2], t_torch[reps // 2])
    nbytes = 4 * B * T + 8 * B * Tf * F   # analysis reads 4 T, writes 8 F per frame; synthesis the reverse (4 Tf H)
    nbytes_syn = 8 * B * Tf * F + 4 * B * Tf * H
    out = {"sr": sr, "fft": N, "hop": H, "streams": B, "seconds": seconds, "kernels": "generic" if (N, H) != (960, 480) else "960/480"}
    for name, nb in (("analysis", nbytes), ("synthesis", nbytes_syn)):
        ms_o, ms_t = res[name]
        out[name] = {"ours_ms": round(ms_o, 4), "torch_ms": round(ms_t, 4), "speedup": round(ms_t / ms_o, 3),
                     "ours_GBps": round(nb / ms_o / 1e6, 1), "ours_peak_frac": round(nb / ms_o / 1e-3 / PEAK_BPS, 3),
                     "torch_GBps": round(nb / ms_t / 1e6, 1)}
    out["max_rel_diff_vs_torch"] = {"analysis": ana_err, "synthesis": syn_err}
    del st
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stft.py needs a CUDA device")
    info = card()
    for sr, N, H, B, _ in WORKLOADS:
        print(json.dumps(run(sr, N, H, B, a.seconds, a.reps)), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps({"card": info, "peak_GBps_assumed": PEAK_BPS / 1e9}), flush=True)


if __name__ == "__main__":
    main()
