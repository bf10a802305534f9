#!/usr/bin/env python3
"""Cost of per-entry settings and LSNR rows on a ragged batch: DeepFilterNet3, 128 streams on one GPU with seeded-uniform
lengths in [1 s, 20 s], device-resident (enhance_device_ragged on a padded [B, S] tensor) and from CPU tensors
(enhance_batch, end to end).  Three calls on each path, alternated in one session:
  1 plain       one attenuation limit for every entry (the call without a settings table)
  2 settings    a limit and a post-filter beta per entry (the settings table: the CTL apply kernel)
  3 gating      per-entry LSNR stage gating plus the LSNR rows (the LSNR head, k_lsnr_rows, the copies back)
Useful audio-seconds per second (the streams' true lengths over the time): device calls timed with CUDA events around
synchronised work, host calls with a host clock around the synchronous call; every call is warmed up, then timed --repeats
times interleaved, reported as median with min / max.  --profile adds one torch.profiler pass per call (outside the timed
runs) and reports the CUDA time per kernel name.  Prints one JSON line with the card's name, power limit and SM clock.

    python bench_ragged_ctl.py [--streams 128] [--repeats 5] [--warmup 2] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import load_weights, model_config  # noqa: E402
from bench_ragged import card, stats  # noqa: E402

SR = 48000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch
    from deepfilternet_b200 import DfNet, enhance_batch, enhance_device_ragged, libdf
    from tests_common import synth_audio
    assert torch.cuda.is_available(), "bench_ragged_ctl.py measures on a GPU"
    before = card()
    cfg = model_config("DeepFilterNet3")
    sd, weights_kind = load_weights("DeepFilterNet3", cfg)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    B = a.streams
    rng = np.random.default_rng(a.seed)
    lens = rng.integers(SR, 20 * SR + 1, size=B).astype(np.int64)
    S = int(lens.max())
    x = synth_audio(B, S, seed=1234, device="cuda")
    for b in range(B):
        x[b, lens[b]:] = 0
    hosts = [x[b:b + 1, :lens[b]].cpu() for b in range(B)]
    useful_s = float(lens.sum()) / SR
    lims = rng.uniform(3.0, 30.0, size=B).tolist()
    betas = rng.uniform(0.0, 0.05, size=B).tolist()
    # thresholds around the runtime's defaults (tract.rs:180-185), so that every stage occurs
    ths = [(-10.0 + d, 30.0 + d, 20.0 + d) for d in rng.uniform(-5.0, 5.0, size=B).tolist()]

    def dev_time(fn):
        torch.cuda.synchronize()
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

    out = torch.zeros(B, S, device="cuda")
    calls = {
        "device_1_plain": lambda: enhance_device_ragged(model, st, x, lens, atten_lim_db=12.0, out=out),
        "device_2_settings": lambda: enhance_device_ragged(model, st, x, lens, atten_lim_db=lims, out=out, post_filter_beta=betas),
        "device_3_gating_lsnr": lambda: enhance_device_ragged(model, st, x, lens, atten_lim_db=12.0, out=out, lsnr_thresholds=ths,
                                                              return_lsnr=True),
        "host_1_plain": lambda: enhance_batch(model, st, hosts, atten_lim_db=12.0),
        "host_2_settings": lambda: enhance_batch(model, st, hosts, atten_lim_db=lims, post_filter_beta=betas),
        "host_3_gating_lsnr": lambda: enhance_batch(model, st, hosts, atten_lim_db=12.0, lsnr_thresholds=ths, return_lsnr=True),
    }
    timer = {k: (dev_time if k.startswith("device") else host_time) for k in calls}
    for _ in range(a.warmup):
        for k, fn in calls.items():
            timer[k](fn)
    times = {k: [] for k in calls}
    for _ in range(a.repeats):   # interleaved, so that drift of the shared host hits every call alike
        for k, fn in calls.items():
            times[k].append(timer[k](fn))
    rates = {k: stats([useful_s / t for t in v]) for k, v in times.items()}
    after = card()
    rel = {}
    for path in ("device", "host"):
        p = rates[f"{path}_1_plain"]
        spread = (p["max"] - p["min"]) / p["median"]
        for c in ("2_settings", "3_gating_lsnr"):
            q = rates[f"{path}_{c}"]["median"]
            rel[f"{path}_{c}"] = {"median_vs_plain": q / p["median"], "plain_spread": spread,
                                  "within_spread_plus_3pct": q >= p["median"] * (1 - spread - 0.03)}
    res = {"metric": "useful audio-s/s, DeepFilterNet3, ragged batch with per-entry settings", "weights": weights_kind,
           "card": before, "card_after": after, "streams": B,
           "length_s": {"min": float(lens.min()) / SR, "max": float(lens.max()) / SR, "sum": useful_s},
           "rates": rates, "relative": rel}
    if a.profile:   # a separate pass per call, after the timed ones
        from torch.profiler import ProfilerActivity, profile
        prof = {}
        for k, fn in calls.items():
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as pr:
                fn()
                torch.cuda.synchronize()
            ks = {}
            for e in pr.key_averages():
                t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
                if t > 0:
                    ks[e.key[:60]] = round(t / 1e3, 3)
            prof[k] = dict(sorted(ks.items(), key=lambda kv: -kv[1])[:12])
        res["profile_ms"] = prof
    print(json.dumps(res))


if __name__ == "__main__":
    main()
