#!/usr/bin/env python3
"""Ragged-batch throughput: DeepFilterNet3, 128 streams on one GPU with seeded-uniform lengths in [1 s, 20 s].

Useful audio-seconds per second (the sum of the streams' true lengths over the time) of
  (a) enhance_device_ragged on the padded [B, S] device tensor,
  (b) zero-padding every stream to the longest and enhance_device (what a caller had to do before),
  (c) enhance_batch end to end from CPU tensors (pack into page-locked memory, copies, compute, results on the host),
and, on 128 x 10 s of equal length, the ragged API against enhance_device.  Device rates are timed with CUDA events,
(c) with a host clock around the synchronous call; every variant is warmed up and timed --repeats times, interleaved, and
the median with min / max is reported.  Parity: 4 streams against per-stream enhance_device calls and the CPU oracle.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_ragged.py [--streams 128] [--repeats 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import load_weights, model_config  # noqa: E402

SR = 48000


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info.update(power_limit_w=float(q[0]), sm_mhz=float(q[1]), sm_max_mhz=float(q[2]))
    except Exception as e:  # noqa: BLE001 -- the numbers are still reported, without the card's settings
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def stats(xs):
    xs = sorted(xs)
    return {"median": xs[len(xs) // 2], "min": xs[0], "max": xs[-1], "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    import numpy as np
    import torch
    from deepfilternet_b200 import DfNet, enhance_batch, enhance_device, enhance_device_ragged, libdf
    from tests_common import synth_audio
    assert torch.cuda.is_available(), "bench_ragged.py measures on a GPU"
    before = card()
    cfg = model_config("DeepFilterNet3")
    sd, weights_kind = load_weights("DeepFilterNet3", cfg)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    B = a.streams
    lens = np.random.default_rng(a.seed).integers(SR, 20 * SR + 1, size=B).astype(np.int64)
    S = int(lens.max())
    x = synth_audio(B, S, seed=1234, device="cuda")
    for b in range(B):
        x[b, lens[b]:] = 0
    hosts = [x[b:b + 1, :lens[b]].cpu() for b in range(B)]
    useful_s = float(lens.sum()) / SR
    hop, fft = cfg.hop_size, cfg.fft_size
    true_frames = int(((lens + fft) // hop).sum())
    padded_frames = B * ((S + fft) // hop)
    eq = synth_audio(B, 10 * SR, seed=99, device="cuda")
    eq_s = B * 10.0

    def dev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def host_time(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    out_r = torch.zeros(B, S, device="cuda")
    out_p = torch.empty(B, S, device="cuda")
    out_e = torch.empty_like(eq)
    out_er = torch.zeros_like(eq)
    variants = {
        "a_ragged_device": (lambda: dev_time(lambda: enhance_device_ragged(model, st, x, lens, out=out_r)), useful_s),
        "b_zero_pad_device": (lambda: dev_time(lambda: enhance_device(model, st, x, out=out_p)), useful_s),
        "c_ragged_host_e2e": (lambda: host_time(lambda: enhance_batch(model, st, hosts)), useful_s),
        "equal_ragged_device": (lambda: dev_time(lambda: enhance_device_ragged(model, st, eq, [10 * SR] * B, out=out_er)), eq_s),
        "equal_enhance_device": (lambda: dev_time(lambda: enhance_device(model, st, eq, out=out_e)), eq_s),
    }
    for _ in range(a.warmup):
        for fn, _s in variants.values():
            fn()
    times = {k: [] for k in variants}
    for _ in range(a.repeats):   # interleaved, so that drift of the shared host hits every variant alike
        for k, (fn, _s) in variants.items():
            times[k].append(fn())
    rates = {k: stats([variants[k][1] / t for t in v]) for k, v in times.items()}
    after = card()
    # parity: 4 streams (the shortest, the longest and two between) against per-stream calls and the CPU oracle
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import dfnet_oracle
    order = np.argsort(lens)
    rows = [int(order[0]), int(order[B // 3]), int(order[B // 2]), int(order[-1])]
    got = out_r.cpu()
    par = []
    for b in rows:
        t = int(lens[b])
        alone = enhance_device(model, st, x[b:b + 1, :t].contiguous())[0].cpu()
        ref = dfnet_oracle.enhance(sd, cfg.as_dict(), x[b:b + 1, :t].cpu())[0]
        par.append({"stream": b, "samples": t,
                    "rms_vs_alone": float((got[b, :t] - alone).double().pow(2).mean().sqrt()),
                    "rms_vs_oracle": float((got[b, :t] - ref).double().pow(2).mean().sqrt())})
    eq_rms = float((out_er - out_e).double().pow(2).mean().sqrt())
    print(json.dumps({
        "metric": "useful audio-s/s, DeepFilterNet3, ragged batch", "weights": weights_kind, "card": before, "card_after": after,
        "streams": B, "length_s": {"min": float(lens.min()) / SR, "max": float(lens.max()) / SR, "sum": useful_s},
        "frames": {"true": true_frames, "zero_padded": padded_frames, "ratio": padded_frames / true_frames},
        "rates": rates, "speedup_a_over_b": rates["a_ragged_device"]["median"] / rates["b_zero_pad_device"]["median"],
        "equal_length_ragged_over_enhance_device": rates["equal_ragged_device"]["median"] / rates["equal_enhance_device"]["median"],
        "parity": {"streams": par, "equal_length_rms_ragged_vs_enhance_device": eq_rms,
                   "ok": all(p["rms_vs_alone"] < 1e-6 and p["rms_vs_oracle"] < 1e-4 for p in par) and eq_rms < 1e-6},
    }))


if __name__ == "__main__":
    main()
