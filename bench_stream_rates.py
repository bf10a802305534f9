#!/usr/bin/env python3
"""Streaming slots at other sample rates: bench_slots.py's server (256 slots, about half of them open, sessions of 2-30 s,
seeded random weights) run by a 48 kHz, a 16 kHz and an 8 kHz handle on the same traffic, for DeepFilterNet3 and
DeepFilterNet3_ll and calls of 1, 4 and 16 hops.  Reported per model and call size:
  * device time per call (CUDA events around each process call, slot operations included), mean over the pass; the
    rates alternate pass by pass, and each figure is the median of --reps passes with their min and max;
  * the share of the kernel time of a call that k_resample_up and k_resample_down take (torch.profiler, a separate pass
    per rate);
and the card's name, power limit and max SM clock, read in the same run.  Prints one JSON line.

    python bench_stream_rates.py [--slots 256] [--calls 200] [--hops 1 4 16] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import model_config  # noqa: E402
from bench_ragged import card  # noqa: E402
from bench_slots import traffic  # noqa: E402

RATES = (48000, 16000, 8000)


def start_pass(s, start):
    s.reset()
    s.flush()          # every slot free, then the steady state the plan starts from
    s.open(start)


def one_pass(s, x, start, plan):
    import torch
    start_pass(s, start)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in plan]
    torch.cuda.synchronize()
    for (closes, opens, _), (e0, e1) in zip(plan, ev):
        e0.record()
        if closes:
            s.close(closes)
        if opens:
            s.open(opens)
        s.process(x)
        e1.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def kernel_share(s, x, start, plan):
    """(share of kernel time in k_resample_up / _down, kernel ms per call) over one profiled pass"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    start_pass(s, start)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for closes, opens, _ in plan:
            if closes:
                s.close(closes)
            if opens:
                s.open(opens)
            s.process(x)
        torch.cuda.synchronize()
    tot, rs = 0.0, 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if e.key.startswith("k_") or "kernel" in e.key.lower() or "<<<" in e.key or "void " in e.key:
            tot += t
        if "k_resample_up" in e.key or "k_resample_down" in e.key:
            rs += t
    return (rs / tot if tot else float("nan")), tot / 1e3 / len(plan)


def run(name, slots, calls, hops, reps, warmup, seed):
    import torch
    from deepfilternet_b200 import DfNet, DfStream, libdf
    from deepfilternet_b200.weights import random_state_dict
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
    start, plan = traffic(slots, calls, hops, seed)
    handles = {sr: DfStream(model, st, batch=slots, sr=sr) for sr in RATES}
    xs = {sr: torch.randn(slots, hops * sr // 100, device="cuda") * 0.1 for sr in RATES}
    for sr in RATES:
        for _ in range(warmup):
            handles[sr].process(xs[sr])
    times = {sr: [] for sr in RATES}
    for r in range(reps):
        order = RATES if r % 2 == 0 else RATES[::-1]
        for sr in order:
            times[sr].append(one_pass(handles[sr], xs[sr], start, plan))
    res = {"mean_open_slots": float(np.mean([live for _, _, live in plan]))}
    for sr in RATES:
        t = np.array(times[sr])
        res[f"{sr}"] = {"call_ms_median": float(np.median(t)), "call_ms_min": float(t.min()), "call_ms_max": float(t.max())}
        if sr != 48000:
            res[f"{sr}"]["vs_48k"] = float(np.median(t) / np.median(times[48000]))
            share, kms = kernel_share(handles[sr], xs[sr], start, plan)
            res[f"{sr}"]["resample_kernel_share"] = share
            res[f"{sr}"]["kernel_ms_per_call"] = kms
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--hops", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_stream_rates.py measures on a GPU"
    before = card()
    rows = {}
    for name in a.models:
        for hops in a.hops:
            calls = max(a.calls // hops, 40)
            rows[f"{name}/{hops}hop"] = run(name, a.slots, calls, hops, a.reps, a.warmup, a.seed)
    print(json.dumps({"metric": "streaming slots at 16 and 8 kHz vs 48 kHz on the same traffic: device ms per call (median of "
                                "passes, min / max) and the resamplers' share of kernel time", "weights": "random (seed 1)",
                      "card": before, "card_after": card(), "slots": a.slots, "results": rows}))


if __name__ == "__main__":
    main()
