#!/usr/bin/env python3
"""Cost of LLR and WSS (df/sepm.py's composite measure) in the device metrics call, on bench_metrics.py's two 48 kHz
sets: 824 seeded recordings of 1.5-5 s and 128 x 10 s.

Per set: the device call (evaluate_device_ragged on padded CUDA tensors, CUDA events) with the 3 existing metric bits
(SI-SDR, STOI, SSNR) against all 5 (plus LLR and WSS), alternated, median and min / max of --repeats; the 5-bit host call
(evaluate_batch from CPU tensors, host clock around the synchronous call); each kernel's share of the 5-bit device call
(torch.profiler, a separate pass).  Then an evaluation_loop-style pass over the 824 set with "composite" and a constant
stub PESQ (enhance_batch with DeepFilterNet3 on seeded weights, the clean STFT round trip, one metrics call per batch, the
16 kHz resample of every pair handed to PESQ; file I/O excluded).  Prints one JSON line, with the card's name, power limit
and SM clock read in the same run.

    python bench_composite.py [--repeats 5] [--warmup 2] [--batch-size 64]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench import model_config  # noqa: E402
from bench_metrics import SR, recordings  # noqa: E402
from bench_ragged import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch-size", type=int, default=64, help="files per enhance / metrics call in the loop pass")
    a = ap.parse_args()
    import numpy as np
    import torch
    from deepfilternet_b200 import DfNet, enhance_batch, libdf
    from deepfilternet_b200 import evaluation_utils as E
    from deepfilternet_b200.weights import random_state_dict

    assert torch.cuda.is_available(), "bench_composite.py measures on a GPU"
    info = card()
    rng = np.random.default_rng(2026)   # bench_metrics.py's seed and sets
    sets = {"vbd_824x1.5-5s": recordings(rng, 824, 1.5, 5.0), "128x10s": recordings(rng, 128, 10.0, 10.0)}
    res = {"card": info, "sets": {}}
    three, five = ("sisdr", "stoi", "ssnr"), ("sisdr", "stoi", "ssnr", "llr", "wss")

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
        variants = {"device_3bits": lambda: dev_time(lambda: E.evaluate_device_ragged(xc, xd, lens, SR, three)),
                    "device_5bits": lambda: dev_time(lambda: E.evaluate_device_ragged(xc, xd, lens, SR, five)),
                    "host_5bits": lambda: host_time(lambda: E.evaluate_batch(hc, hd, SR, five))}
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
        r["ratio_5_over_3_bits"] = stats(times["device_5bits"])["median"] / stats(times["device_3bits"])["median"]
        r["workspace_bytes"] = E.metrics_handle(SR).workspace_bytes()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            E.evaluate_device_ragged(xc, xd, lens, SR, five)
            torch.cuda.synchronize()
        kt = {}
        for ev in prof.key_averages():
            dt = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if dt > 0 and "Memcpy" not in ev.key and "Memset" not in ev.key:
                m = re.search(r"\b(k_\w+)", ev.key)
                key = m.group(1) if m else ev.key
                kt[key] = kt.get(key, 0.0) + dt
        tot = sum(kt.values()) or 1.0
        r["kernel_share_5bits"] = {k: round(v / tot, 4) for k, v in sorted(kt.items(), key=lambda kv: -kv[1])}
        r["kernel_total_ms_5bits"] = tot / 1e3
        res["sets"][name] = r

    # evaluation_loop's steps with "composite" and a constant stub PESQ
    cfg = model_config("DeepFilterNet3")
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=11), st)
    recs = sets["vbd_824x1.5-5s"]
    noisy = [torch.from_numpy(d)[None] for _, d in recs]
    clean = [c[None] for c, _ in recs]
    stub = lambda r, d: 3.0  # noqa: E731

    def loop():
        t = {"enhance": 0.0, "clean_stft": 0.0, "metrics_composite": 0.0}
        for i in range(0, len(recs), a.batch_size):
            t0 = time.perf_counter()
            enh = [e[0] for e in enhance_batch(model, st, noisy[i:i + a.batch_size], pad=False)]
            t1 = time.perf_counter()
            cl = [torch.from_numpy(st.synthesis(st.analysis(c))[0]) for c in clean[i:i + a.batch_size]]
            t2 = time.perf_counter()
            E.evaluate_batch(cl, enh, SR, ("stoi", "composite", "sisdr"), pesq=stub)
            t3 = time.perf_counter()
            t["enhance"] += t1 - t0
            t["clean_stft"] += t2 - t1
            t["metrics_composite"] += t3 - t2
        return t

    loop()
    runs = [loop() for _ in range(max(1, a.repeats // 2))]
    tots = [sum(r.values()) for r in runs]
    med = runs[tots.index(stats(tots)["median"])]
    audio_s = sum(c.size for c, _ in recs) / SR
    res["loop_vbd_dfn3_seeded_composite_stub_pesq"] = {
        "batch_size": a.batch_size, "total_s": stats(tots), "audio_s_per_s": audio_s / stats(tots)["median"],
        "share": {k: round(v / sum(med.values()), 4) for k, v in med.items()}}
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
