#!/usr/bin/env python3
"""Rated ragged batches: recordings at their own sample rates enhanced in one call, resampled to and from 48 kHz on the
device (enhance_batch(..., sr=rates) / enhance_device_ragged(..., sr=rates); DESIGN.md section 5i).

Workload: DeepFilterNet3 with seeded random weights, 128 recordings of seeded-uniform 1-20 s, each at a rate drawn from a
mix (default 30 % 8 kHz, 40 % 16 kHz, 30 % 48 kHz, the mix bench_slot_rates.py uses), and the same durations all at
16 kHz.  Legs:
  * end to end from CPU tensors: the composition a caller writes today (io.resample of every entry to 48 kHz,
    enhance_batch, io.resample of every result back) against one enhance_batch(..., sr=rates); the two alternate pass by
    pass, each figure the median of --reps passes with its min and max, and useful audio-s/s at the recordings' own
    durations;
  * device resident: enhance_device_ragged(..., sr=rates) against enhance_device_ragged of the same batch resampled to
    48 kHz beforehand, which shows what the resamplers add;
  * kernel share: one torch.profiler pass of the rated device call for k_resample_rows' share of kernel time, and its
    achieved GB/s (each resampled stream's input read once and output written once, both directions) against 3.35 TB/s;
and the card's name, power limit and max SM clock, read in the same run.  Prints one JSON line.

    python bench_ragged_rates.py [--batch 128] [--reps 5] [--mix 8000:0.3 16000:0.4 48000:0.3]
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

from bench import model_config  # noqa: E402
from bench_ragged import card  # noqa: E402
from bench_slot_rates import parse_mix  # noqa: E402

MODEL_SR = 48000
HBM_TBS = 3.35   # H100 SXM data sheet, HBM3


def workload(batch, seed, mix):
    """[(CPU tensor [1, T] at its rate, rate)]: seeded-uniform 1-20 s durations, rates drawn from `mix`"""
    import torch
    rng = np.random.default_rng(seed)
    rates, p = list(mix), np.array(list(mix.values()), np.float64)
    out = []
    for _ in range(batch):
        r = rates[int(rng.choice(len(rates), p=p / p.sum()))]
        n = int(rng.uniform(1.0, 20.0) * r)
        out.append((torch.from_numpy((rng.standard_normal((1, n)) * 0.1).astype(np.float32)), r))
    return out


def composition(model, st, entries):
    from deepfilternet_b200 import enhance_batch, io
    x48 = [io.resample(a, r, MODEL_SR) for a, r in entries]
    y48 = enhance_batch(model, st, x48)
    return [io.resample(y, MODEL_SR, r) for y, (_, r) in zip(y48, entries)]


def rated(model, st, entries):
    from deepfilternet_b200 import enhance_batch
    return enhance_batch(model, st, [a for a, _ in entries], sr=[r for _, r in entries])


def padded(entries, resample_to_48k):
    """[B, S] CUDA tensor of the entries (at their rates, or resampled to 48 kHz) and the row lengths"""
    import torch
    from deepfilternet_b200 import io
    rows = [io.resample(a, r, MODEL_SR)[0] if resample_to_48k else a[0] for a, r in entries]
    lens = [int(x.numel()) for x in rows]
    x = torch.zeros(len(rows), max(lens))
    for b, v in enumerate(rows):
        x[b, :lens[b]] = v
    return x.cuda(), lens


def timed(fa, fb, reps):
    """alternating passes of two callables: {"a": [seconds], "b": [seconds]}"""
    import torch
    t = {"a": [], "b": []}
    for i in range(reps):
        for k in (("a", "b") if i % 2 == 0 else ("b", "a")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            (fa if k == "a" else fb)()
            torch.cuda.synchronize()
            t[k].append(time.perf_counter() - t0)
    return t


def summary(ts, audio_s):
    t = np.array(ts)
    return {"s_median": float(np.median(t)), "s_min": float(t.min()), "s_max": float(t.max()),
            "audio_s_per_s": audio_s / float(np.median(t))}


def kernel_share(fn, entries, st):
    """(k_resample_rows' share of kernel time, its achieved GB/s, kernel ms) over one profiled call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from deepfilternet_b200 import ragged
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot, rs = 0.0, 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if e.key.startswith("k_") or "kernel" in e.key.lower() or "<<<" in e.key or "void " in e.key:
            tot += t
        if "k_resample_rows" in e.key:
            rs += t
    nbytes = 0
    for a, r in entries:
        if r == MODEL_SR:
            continue
        n, n48 = a.shape[-1], ragged.len_48k(a.shape[-1], r)
        o48 = ragged.out_len(n48, st.hop_size(), True)
        nbytes += 4 * (n + n48 + o48 + ragged.out_len_at(n, r, st.hop_size(), True))
    return (rs / tot if tot else float("nan")), (nbytes / (rs * 1e-6) / 1e9 if rs else float("nan")), tot / 1e3


def run(name, batch, reps, seed, mix):
    import torch
    from deepfilternet_b200 import DfNet, enhance_device_ragged, libdf
    from deepfilternet_b200.weights import random_state_dict
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
    entries = workload(batch, seed, mix)
    audio_s = float(sum(a.shape[-1] / r for a, r in entries))
    rates = [r for _, r in entries]
    # warm-up: every shape of the timed window, and every rate's registration
    comp, rat = composition(model, st, entries), rated(model, st, entries)
    err = max(float((x - y).abs().max()) for x, y in zip(comp, rat))
    t = timed(lambda: composition(model, st, entries), lambda: rated(model, st, entries), reps)
    res = {"audio_s": audio_s, "max_abs_diff_rated_vs_composition": err,
           "end_to_end": {"composition": summary(t["a"], audio_s), "rated": summary(t["b"], audio_s)}}
    res["end_to_end"]["rated_vs_composition"] = res["end_to_end"]["rated"]["s_median"] / res["end_to_end"]["composition"]["s_median"]
    xr, lr = padded(entries, False)
    x48, l48 = padded(entries, True)
    dev_rated = lambda: enhance_device_ragged(model, st, xr, lr, sr=rates)   # noqa: E731
    dev_48k = lambda: enhance_device_ragged(model, st, x48, l48)            # noqa: E731
    dev_rated(), dev_48k()
    t = timed(dev_48k, dev_rated, reps)
    res["device"] = {"pre_resampled_48k": summary(t["a"], audio_s), "rated": summary(t["b"], audio_s)}
    res["device"]["rated_vs_48k"] = res["device"]["rated"]["s_median"] / res["device"]["pre_resampled_48k"]["s_median"]
    sh, gbs, kms = kernel_share(dev_rated, entries, st)
    res["k_resample_rows"] = {"kernel_time_share": sh, "achieved_GB_s": gbs, "fraction_of_3.35_TB_s": gbs / (HBM_TBS * 1e3),
                              "kernel_ms_per_call": kms}
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--model", default="DeepFilterNet3")
    ap.add_argument("--mix", nargs="+", default=["8000:0.3", "16000:0.4", "48000:0.3"])
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_ragged_rates.py measures on a GPU"
    before = card()
    mixes = {"mix": parse_mix(a.mix), "all_16k": {16000: 1.0}}
    rows = {k: run(a.model, a.batch, a.reps, a.seed, m) for k, m in mixes.items()}
    print(json.dumps({"metric": "rated ragged batch vs resample + 48 kHz batch + resample: seconds per call (median of "
                                "alternated passes, min / max), useful audio-s/s at the recordings' own durations, and the "
                                "resampler kernel's share of kernel time", "model": a.model, "weights": "random (seed 1)",
                      "batch": a.batch, "mixes": {k: {str(r): p for r, p in m.items()} for k, m in mixes.items()},
                      "card": before, "card_after": card(), "results": rows}))


if __name__ == "__main__":
    main()
