#!/usr/bin/env python3
"""Cost of pystoi's STOI and ESTOI (metric bits 64 and 128) in the device metrics call, on bench_metrics.py's two 48 kHz
sets: 824 seeded recordings of 1.5-5 s and 128 x 10 s.

Per set: the device call (evaluate_device_ragged on padded CUDA tensors, CUDA events) and the host call (evaluate_batch
from CPU tensors, host clock around the synchronous call) for {"stoi"}, {"pystoi"}, {"pystoi", "estoi"} and the existing
three-bit {"sisdr", "stoi", "ssnr"}, alternated, median and min / max of --repeats; each kernel's share of the two-bit
device call (torch.profiler, a separate pass); the CPU time of the float64 restatement (tests/pystoi_ref64.py, its float64
resampler included) on the same set; and the distribution of PYSTOI - STOI over the set.  Prints one JSON line, with the
card's name, power limit and SM clock read in the same run.

    python bench_pystoi.py [--repeats 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from bench_metrics import SR, recordings  # noqa: E402
from bench_ragged import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import torch
    from deepfilternet_b200 import evaluation_utils as E
    import pystoi_ref64 as P

    assert torch.cuda.is_available(), "bench_pystoi.py measures on a GPU"
    info = card()
    rng = np.random.default_rng(2026)   # bench_metrics.py's seed and sets
    sets = {"vbd_824x1.5-5s": recordings(rng, 824, 1.5, 5.0), "128x10s": recordings(rng, 128, 10.0, 10.0)}
    res = {"card": info, "sets": {}}
    calls = {"stoi": ("stoi",), "pystoi": ("pystoi",), "pystoi_estoi": ("pystoi", "estoi"),
             "sisdr_stoi_ssnr": ("sisdr", "stoi", "ssnr")}

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

    for name, recs in sets.items():
        lens = np.array([c.size for c, _ in recs], dtype=np.int64)
        S = int(lens.max())
        xc = torch.zeros(len(recs), S)
        xd = torch.zeros(len(recs), S)
        for i, (c, d) in enumerate(recs):
            xc[i, :c.size] = torch.from_numpy(c)
            xd[i, :d.size] = torch.from_numpy(d)
        xc, xd = xc.cuda(), xd.cuda()
        hc = [torch.from_numpy(c) for c, _ in recs]
        hd = [torch.from_numpy(d) for _, d in recs]
        audio_s = float(lens.sum()) / SR
        variants = {}
        for k, m in calls.items():
            variants[f"device_{k}"] = lambda m=m: dev_time(lambda: E.evaluate_device_ragged(xc, xd, lens, SR, m))
            variants[f"host_{k}"] = lambda m=m: host_time(lambda: E.evaluate_batch(hc, hd, SR, m))
        for _ in range(a.warmup):
            for fn in variants.values():
                fn()
        times = {k: [] for k in variants}
        for _ in range(a.repeats):
            for k, fn in variants.items():
                times[k].append(fn())
        r = {"entries": len(recs), "audio_s": audio_s}
        for k, t in times.items():
            r[f"{k}_call_s"] = stats(t)
            r[f"{k}_audio_s_per_s"] = audio_s / stats(t)["median"]
        r["ratio_pystoi_estoi_over_sisdr_stoi_ssnr"] = (stats(times["device_pystoi_estoi"])["median"]
                                                       / stats(times["device_sisdr_stoi_ssnr"])["median"])
        r["workspace_bytes"] = E.metrics_handle(SR).workspace_bytes()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            E.evaluate_device_ragged(xc, xd, lens, SR, calls["pystoi_estoi"])
            torch.cuda.synchronize()
        kt = {}
        for ev in prof.key_averages():
            dt = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if dt > 0 and "Memcpy" not in ev.key and "Memset" not in ev.key:
                m = re.search(r"\b(k_\w+)", ev.key)
                key = m.group(1) if m else ev.key
                kt[key] = kt.get(key, 0.0) + dt
        tot = sum(kt.values()) or 1.0
        r["kernel_share_pystoi_estoi"] = {k: round(v / tot, 4) for k, v in sorted(kt.items(), key=lambda kv: -kv[1])}
        r["kernel_total_ms_pystoi_estoi"] = tot / 1e3
        both = E.evaluate_batch(hc, hd, SR, ("stoi", "pystoi", "estoi"))
        diff = (both["pystoi"].double() - both["stoi"].double()).numpy()
        diff = diff[np.isfinite(diff)]
        r["pystoi_minus_stoi"] = {"n": int(diff.size), "mean": float(diff.mean()), "std": float(diff.std()),
                                  **{f"p{q}": float(np.percentile(diff, q)) for q in (0, 5, 50, 95, 100)}}
        t0 = time.perf_counter()
        ref = [P.pystoi10(P.rows10(c, SR), P.rows10(d, SR)) for c, d in recs]
        r["ref64_cpu_s"] = time.perf_counter() - t0
        got_p, got_e = both["pystoi"].numpy(), both["estoi"].numpy()
        r["max_abs_vs_ref64"] = {"pystoi": float(max(abs(got_p[i] - v["stoi"]) for i, v in enumerate(ref))),
                                 "estoi": float(max(abs(got_e[i] - v["estoi"]) for i, v in enumerate(ref)))}
        res["sets"][name] = r
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
