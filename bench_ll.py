#!/usr/bin/env python3
"""Low-latency models side by side: DeepFilterNet3 (2 hops of look-ahead), DeepFilterNet3_ll (0 hops, H = 512
recurrences) and DeepFilterNet2_ll (0 hops, H = 256), with seeded random weights of each shipped configuration
(tests/golden/models/<name>/config.ini; bench.py's model_config knows only the four older names).

Per model, alternating the models within each of --runs passes (median and min-max over the passes):
  * the bench_slots.py server: 256 slots, about half open, 1 / 4 / 16 hops per call, modes "slots" and "all_computed":
    device time per call p50 / p99 and useful audio-s/s (the "controls" mode sets per-slot post-filter beta, which
    DeepFilterNet2 does not support);
  * a device-resident batch of 128 x 10 s through enhance_device: audio-s/s;
  * a profile of one such batch (torch.profiler, in a run of its own after the timed passes): the DF pathway conv's
    kernel time and its share of all kernel time, for DeepFilterNet2_ll (k_df_convp_tc<5, 3>) and DeepFilterNet2
    (k_df_convp_tc<5, 5>, same batch).
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_ll.py [--runs 5] [--calls 400] [--hops 1 4 16] [--batch 128] [--seconds 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_slots  # noqa: E402
from bench_ragged import card  # noqa: E402

SR = 48000
MODELS = ("DeepFilterNet3", "DeepFilterNet3_ll", "DeepFilterNet2_ll")


def golden_config(name: str):
    from deepfilternet_b200.config import load_config
    return load_config(os.path.join(ROOT, "tests", "golden", "models", name, "config.ini"), env={})


# bench_slots.run builds its model from this name -> config function
bench_slots.model_config = golden_config


def model_of(name: str):
    from deepfilternet_b200 import DfNet, libdf
    from deepfilternet_b200.weights import random_state_dict
    cfg = golden_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    return DfNet(cfg, random_state_dict(cfg, seed=1), st), st


def batch_rate(model, st, x, reps: int = 3) -> float:
    import torch
    from deepfilternet_b200 import enhance_device
    out = enhance_device(model, st, x)   # warm-up: workspace, tensor maps
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        enhance_device(model, st, x, out=out)
    e1.record()
    torch.cuda.synchronize()
    return reps * x.numel() / SR / (e0.elapsed_time(e1) / 1e3)


def convp_share(model, st, x) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile
    from deepfilternet_b200 import enhance_device
    enhance_device(model, st, x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        enhance_device(model, st, x)
        torch.cuda.synchronize()
    tot = convp = 0.0
    names = set()
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "emcpy" in e.name or "emset" in e.name:
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        tot += us
        if "k_df_convp_tc" in e.name:
            convp += us
            names.add(e.name)
    return {"kernel_ms": tot / 1e3, "df_convp_ms": convp / 1e3, "df_convp_share": convp / tot if tot else None,
            "instances": sorted(names)}


def summary(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--hops", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--models", nargs="+", default=list(MODELS))
    a = ap.parse_args()
    import torch
    from deepfilternet_b200 import DfStream
    assert torch.cuda.is_available(), "bench_ll.py measures on a GPU"
    before = card()
    x = torch.randn(a.batch, int(a.seconds * SR), generator=torch.Generator().manual_seed(3)).mul_(0.1).cuda()
    models = {n: model_of(n) for n in a.models}
    raw = {n: {"batch": []} for n in a.models}
    for _ in range(a.runs):
        for name in a.models:   # alternated within each pass
            for hops in a.hops:
                calls = a.calls if hops == 1 else max(a.calls // hops, 40)
                r = bench_slots.run(name, a.slots, calls, hops, a.warmup, a.seed, modes=("slots", "all_computed"))
                for mode in ("slots", "all_computed"):
                    for k in ("p50_ms", "p99_ms", "useful_audio_s_per_s"):
                        raw[name].setdefault(f"{hops}hop/{mode}/{k}", []).append(r[mode][k])
            raw[name]["batch"].append(batch_rate(*models[name], x))
    res = {n: {k: summary(v) for k, v in d.items()} for n, d in raw.items()}
    prof = {}
    for name in ("DeepFilterNet2_ll", "DeepFilterNet2"):
        prof[name] = convp_share(*model_of(name), x)
    print(json.dumps({"metric": "low-latency models: slot server (p50 / p99 ms per call, useful audio-s/s) and a "
                                f"device-resident {a.batch} x {a.seconds:g} s batch (audio-s/s); median and min-max of "
                                f"{a.runs} alternated passes", "weights": "random (seed 1)",
                      "latency_hops": {n: DfStream(*models[n], batch=1).latency_frames for n in a.models},
                      "card": before, "card_after": card(), "slots": a.slots, "results": res, "df_convp_profile": prof}))


if __name__ == "__main__":
    main()
