#!/usr/bin/env python3
"""Cost of the runtime gating mode (DfNet.set_gating_mode("runtime"): each decoder runs only on the frames LSNR stage
gating lets through) against apply mode, at the Rust runtime's default thresholds (-10 / 30 / 20 dB, tract.rs:180-185).

Two workloads, each run in both modes, alternated pass by pass (--passes, 5 by default) in one session:
  * the bench_slots.py server: one DfStream of 256 slots, sessions of 2-30 s arriving so that about half of the slots are
    open, every slot gating with the default thresholds, fed in calls of 1, 4 and 16 hops, DeepFilterNet3 and
    DeepFilterNet3_ll.  The slots carry synthetic noisy speech (tests_common.synth_audio), so every stage occurs.  Per
    pass: the mean device time per call (CUDA events around each process call) and useful audio-s/s;
  * bench_ragged_ctl.py's gating batch: DeepFilterNet3, 128 streams of 1-20 s, per-entry thresholds around the defaults
    and LSNR rows, device resident (enhance_device_ragged) and from CPU tensors (enhance_batch).
Reported as the median of the passes with min / max, and the runtime / apply ratio of the medians.  --profile adds one
torch.profiler pass per workload and mode (outside the timed passes): the CUDA time per kernel, and the share of the
runtime mode's own kernels (k_gate_*) and of k_df_convp_tc.  Pretrained weights when models/_ref travelled with the tree
(bench.load_weights), else seeded random ones.  Prints one JSON line with the card's name, power limit and SM clock.

    python bench_gating_runtime.py [--passes 5] [--calls 200] [--hops 1 4 16] [--models ...] [--streams 128] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import load_weights, model_config  # noqa: E402
from bench_ragged import card, stats  # noqa: E402
from bench_slots import traffic  # noqa: E402

SR, HOP = 48000, 480
TH = (-10.0, 30.0, 20.0)
MODES = ("apply", "runtime")


def kernel_times(fn):
    """CUDA time per kernel name (ms) of one call of fn under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as pr:
        fn()
        torch.cuda.synchronize()
    ks = {}
    for e in pr.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
        if t > 0:
            ks[e.key[:60]] = ks.get(e.key[:60], 0.0) + t / 1e3
    total = sum(ks.values())
    share = lambda p: sum(v for k, v in ks.items() if p in k) / total if total else 0.0  # noqa: E731
    top = dict(sorted(((k, round(v, 3)) for k, v in ks.items()), key=lambda kv: -kv[1])[:10])
    return {"kernel_ms": round(total, 3), "k_gate_share": round(share("k_gate_"), 4),
            "k_df_convp_tc_share": round(share("k_df_convp_tc"), 4), "top_ms": top}


def slots_workload(name, slots, calls, hops_list, warmup, passes, seed, profile):
    import torch
    from deepfilternet_b200 import DfNet, DfStream, libdf
    from tests_common import synth_audio
    cfg = model_config(name)
    sd, kind = load_weights(name, cfg)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    n_hops = 4 * SR // HOP                      # 4 s of synthetic speech per slot, fed round and round
    speech = synth_audio(slots, n_hops * HOP, seed=seed, device="cuda")
    out = {"weights": kind}
    for hops in hops_list:
        n = n_hops // hops
        buf = speech[:, :n * hops * HOP].reshape(slots, n, hops * HOP).permute(1, 0, 2).contiguous()   # call i: buf[i % n]
        start, plan = traffic(slots, calls, hops, seed)
        useful = sum(live for _, _, live in plan) * hops * HOP / SR
        handles = {}
        for mode in MODES:
            s = DfStream(model, st, batch=slots, gating_mode=mode)
            s.set_lsnr_thresholds(*TH)
            for i in range(warmup):
                s.process(buf[i % n])
            handles[mode] = s

        def one_pass(s):
            s.flush()
            s.open(start)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in plan]
            torch.cuda.synchronize()
            for i, ((closes, opens, _), (e0, e1)) in enumerate(zip(plan, ev)):
                e0.record()
                if closes:
                    s.close(closes)
                if opens:
                    s.open(opens)
                s.process(buf[i % n])
                e1.record()
            torch.cuda.synchronize()
            return float(np.mean([a.elapsed_time(b) for a, b in ev]))

        ms = {m: [] for m in MODES}
        for _ in range(passes):
            for m in MODES:
                ms[m].append(one_pass(handles[m]))
        r = {m: {"mean_ms_per_call": stats(ms[m]), "useful_audio_s_per_s": useful / (stats(ms[m])["median"] * len(plan) / 1e3)}
             for m in MODES}
        r["runtime_vs_apply_ms"] = r["runtime"]["mean_ms_per_call"]["median"] / r["apply"]["mean_ms_per_call"]["median"]
        r["mean_open_slots"] = float(np.mean([live for _, _, live in plan]))
        if profile:
            for m in MODES:
                s = handles[m]
                s.flush()
                s.open(start)

                def calls10(s=s):
                    for i in range(10):
                        s.process(buf[i % n])
                r[m]["profile_10_calls"] = kernel_times(calls10)
        out[f"hops_{hops}"] = r
        del handles
    return out


def batch_workload(streams, warmup, passes, seed, profile):
    import torch
    from deepfilternet_b200 import DfNet, enhance_batch, enhance_device_ragged, libdf
    from tests_common import synth_audio
    cfg = model_config("DeepFilterNet3")
    sd, kind = load_weights("DeepFilterNet3", cfg)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    rng = np.random.default_rng(seed)
    lens = rng.integers(SR, 20 * SR + 1, size=streams).astype(np.int64)
    S = int(lens.max())
    x = synth_audio(streams, S, seed=1234, device="cuda")
    for b in range(streams):
        x[b, lens[b]:] = 0
    hosts = [x[b:b + 1, :lens[b]].cpu() for b in range(streams)]
    useful_s = float(lens.sum()) / SR
    ths = [(-10.0 + d, 30.0 + d, 20.0 + d) for d in rng.uniform(-5.0, 5.0, size=streams).tolist()]
    out_t = torch.zeros(streams, S, device="cuda")

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

    calls = {}
    for m in MODES:
        calls[f"device_{m}"] = lambda m=m: enhance_device_ragged(model, st, x, lens, atten_lim_db=12.0, out=out_t, lsnr_thresholds=ths,
                                                                  return_lsnr=True, gating_mode=m)
        calls[f"host_{m}"] = lambda m=m: enhance_batch(model, st, hosts, atten_lim_db=12.0, lsnr_thresholds=ths, return_lsnr=True,
                                                       gating_mode=m)
    timer = {k: (dev_time if k.startswith("device") else host_time) for k in calls}
    for _ in range(warmup):
        for k, fn in calls.items():
            timer[k](fn)
    times = {k: [] for k in calls}
    for _ in range(passes):
        for k, fn in calls.items():
            times[k].append(timer[k](fn))
    rates = {k: stats([useful_s / t for t in v]) for k, v in times.items()}
    res = {"weights": kind, "streams": streams, "length_s_sum": useful_s, "useful_audio_s_per_s": rates,
           "runtime_vs_apply_rate": {p: rates[f"{p}_runtime"]["median"] / rates[f"{p}_apply"]["median"] for p in ("device", "host")}}
    if profile:
        res["profile"] = {k: kernel_times(calls[k]) for k in ("device_apply", "device_runtime")}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--hops", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--no-batch", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_gating_runtime.py measures on a GPU"
    res = {"metric": "runtime vs apply gating mode, default thresholds", "card": card()}
    res["slots"] = {name: slots_workload(name, a.slots, a.calls, a.hops, a.warmup, a.passes, a.seed, a.profile) for name in a.models}
    if not a.no_batch:
        res["batch"] = batch_workload(a.streams, 2, a.passes, a.seed, a.profile)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
