#!/usr/bin/env python3
"""Spectral streaming handle (DfStream(spectral=True)) against the audio handle on the same serving traffic: the
bench_slots.py server -- one handle of 256 slots (seeded random weights), Poisson arrivals that keep about half of the
slots open, sessions of 2-30 s -- fed in calls of --frames frames (1, 4 and 16 by default), DeepFilterNet3 and
DeepFilterNet3_ll.  Both handles get the same slot operations; the audio handle takes n * hop samples per slot and call,
the spectral one n spectrum frames (CUDA tensors in and out for both).

Reported per model and call size, for each handle:
  * per-call device time (CUDA events around each process call): the median over --calls calls, as the median and
    min-max of --reps repetitions;
  * useful frames/s: frames of open sessions per second of device time;
  * (spectral) the time share of k_spec_ingest and k_spec_emit among all kernels of the same traffic, from the library's
    per-kernel CUDA-event profile (dfb_profile_enable), in a run of its own.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_stream_spec.py [--slots 256] [--calls 200] [--frames 1 4 16] [--reps 5] [--warmup 20]
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

HOP, F = 480, 481


def profile(fn, names):
    """Share of each kernel in `names` among all kernels the library launched during fn()."""
    import ctypes as C
    from deepfilternet_b200 import _lib
    L = _lib.lib()
    L.dfb_profile_report(None, 0)
    L.dfb_profile_enable(1, None)
    try:
        fn()
    finally:
        buf = C.create_string_buffer(1 << 20)
        n = L.dfb_profile_report(buf, len(buf))
        L.dfb_profile_enable(0, None)
    per = {}
    for line in buf.raw[:max(n, 0)].decode().splitlines():
        p = line.split()
        if len(p) >= 3:
            per[p[0]] = per.get(p[0], 0.0) + float(p[2])
    total = sum(per.values()) or 1.0
    return {k: per.get(k, 0.0) / total for k in names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    args = ap.parse_args()
    import torch
    from deepfilternet_b200 import DfNet, DfStream, libdf
    from deepfilternet_b200.weights import random_state_dict
    from tests_common import synth_audio

    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_spec.py measures on the GPU: no CUDA device")
    B = args.slots
    st = libdf.DF(48000, 960, HOP, 32, 2)
    src = synth_audio(1, 200 * HOP, seed=5)[0]
    results = []
    for name in args.models:
        cfg = model_config(name)
        model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
        for n in args.frames:
            start, plan = traffic(B, args.warmup + args.calls, n, seed=100 + n)
            audio = src[: n * HOP].repeat(B, 1).contiguous().cuda()
            spec = torch.from_numpy(st.analysis(np.ascontiguousarray(src[None, : (n + 1) * HOP].numpy()))[:, 1:n + 1])
            spec = spec.repeat(B, 1, 1).contiguous().cuda()

            def session(spectral, timed):
                s = DfStream(model, st, batch=B, spectral=spectral)
                s.close([b for b in range(B) if b not in set(start)])
                times, frames = [], 0
                for i, (closes, opens, live) in enumerate(plan):
                    if closes:
                        s.close(closes)
                    if opens:
                        s.open(opens)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    s.process_spec(spec) if spectral else s.process(audio)
                    b.record()
                    if i >= args.warmup and timed:
                        times.append((a, b))
                        frames += live * n
                torch.cuda.synchronize()
                ms = [x.elapsed_time(y) for x, y in times]
                return (float(np.median(ms)), frames / (sum(ms) / 1e3)) if timed else None

            row = {"model": name, "frames_per_call": n, "slots": B}
            runs = {False: [], True: []}
            for _ in range(args.reps):   # the two handles alternate within each repetition
                for spectral in (False, True):
                    runs[spectral].append(session(spectral, True))
            for spectral in (False, True):
                meds, rates = [r[0] for r in runs[spectral]], [r[1] for r in runs[spectral]]
                key = "spectral" if spectral else "audio"
                row[key] = {"call_ms_median": float(np.median(meds)), "call_ms_min": min(meds), "call_ms_max": max(meds),
                            "useful_frames_per_s": float(np.median(rates))}
            row["speedup"] = row["audio"]["call_ms_median"] / row["spectral"]["call_ms_median"]
            row["kernel_share"] = profile(lambda: session(True, False), ["k_spec_ingest", "k_spec_emit"])
            results.append(row)
            print(f"{name:18s} n={n:2d}  audio {row['audio']['call_ms_median']:.3f} ms "
                  f"({row['audio']['useful_frames_per_s']:.3g} fr/s)  spectral {row['spectral']['call_ms_median']:.3f} ms "
                  f"[{row['spectral']['call_ms_min']:.3f}-{row['spectral']['call_ms_max']:.3f}] "
                  f"({row['spectral']['useful_frames_per_s']:.3g} fr/s)  x{row['speedup']:.2f}  "
                  f"ingest {100 * row['kernel_share']['k_spec_ingest']:.1f}% emit {100 * row['kernel_share']['k_spec_emit']:.1f}%",
                  flush=True)
    print(json.dumps({"bench": "stream_spec", "card": card(), "results": results}))


if __name__ == "__main__":
    main()
