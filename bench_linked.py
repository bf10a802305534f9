#!/usr/bin/env python3
"""Cost of linked channels: DeepFilterNet3 (seeded random weights), 64 recordings x 2 channels x 10 s, device resident.

enhance_device_ragged with every recording's two channels linked (reduce_mask="mean": they share one ERB mask) against the
same batch unlinked.  Device time with CUDA events; both variants are warmed up and timed --repeats times, alternating, and
the median with min / max is reported.  A separate, profiled run of each gives the time of the apply + synthesis kernel
(k_apply_synthesis), the only kernel linking changes.  Parity: the linked recordings equal each recording linked and
enhanced alone.  Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_linked.py [--recordings 64] [--seconds 10] [--repeats 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import model_config  # noqa: E402
from bench_ragged import card, stats  # noqa: E402

SR = 48000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=64)
    ap.add_argument("--channels", type=int, default=2)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from deepfilternet_b200 import DfNet, _lib, enhance_device_ragged, libdf
    from deepfilternet_b200.weights import random_state_dict
    from tests_common import synth_audio
    assert torch.cuda.is_available(), "bench_linked.py measures on a GPU"
    before = card()
    cfg = model_config("DeepFilterNet3")
    sd = random_state_dict(cfg, seed=1)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, sd, st)
    R, C, T = a.recordings, a.channels, int(a.seconds * SR)
    B = R * C
    x = synth_audio(B, T, seed=1234, device="cuda")
    lens, groups = [T] * B, [C] * R
    audio_s = B * T / SR
    out_l = torch.zeros(B, T, device="cuda")
    out_i = torch.zeros(B, T, device="cuda")
    runs = {
        "linked_mean": lambda: enhance_device_ragged(model, st, x, lens, out=out_l, group_sizes=groups, reduce_mask="mean"),
        "independent": lambda: enhance_device_ragged(model, st, x, lens, out=out_i),
    }

    def dev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    for _ in range(a.warmup):
        for fn in runs.values():
            dev_time(fn)
    times = {k: [] for k in runs}
    for _ in range(a.repeats):   # alternating, so that drift of the shared host hits both alike
        for k, fn in runs.items():
            times[k].append(dev_time(fn))
    rates = {k: stats([audio_s / t for t in v]) for k, v in times.items()}
    ms = {k: stats([t * 1e3 for t in v]) for k, v in times.items()}
    # k_apply_synthesis alone, in profiled runs (events around every launch) kept apart from the timed ones
    L = _lib.lib()
    apply_ms = {}
    buf = ctypes.create_string_buffer(1 << 16)
    for k, fn in runs.items():
        torch.cuda.synchronize()
        L.dfb_profile_report(buf, len(buf))   # drop anything recorded before
        L.dfb_profile_enable(1, b"k_apply_synthesis")
        fn()
        torch.cuda.synchronize()
        L.dfb_profile_enable(0, None)
        n = L.dfb_profile_report(buf, len(buf))
        launches, total = 0, 0.0
        for line in buf.value.decode()[:max(n, 0)].splitlines():
            name, cnt, t = line.split()
            if name == "k_apply_synthesis":
                launches, total = int(cnt), float(t)
        apply_ms[k] = {"ms": total, "launches": launches}
    after = card()
    # parity: the first, a middle and the last recording against themselves linked and enhanced alone
    par = []
    for r in (0, R // 2, R - 1):
        xr = x[r * C:(r + 1) * C].contiguous()
        alone = enhance_device_ragged(model, st, xr, [T] * C, group_sizes=[C], reduce_mask="mean")
        par.append(float((out_l[r * C:(r + 1) * C] - alone).double().pow(2).mean().sqrt()))
    med = {k: v["median"] for k, v in ms.items()}
    print(json.dumps({
        "metric": "device time, DeepFilterNet3, linked channels (mean) vs independent", "weights": "random (seed 1)",
        "card": before, "card_after": after, "recordings": R, "channels": C, "seconds": a.seconds,
        "ms": ms, "audio_s_per_s": rates, "linked_over_independent_time": med["linked_mean"] / med["independent"],
        "k_apply_synthesis": apply_ms,
        "k_apply_synthesis_linked_over_independent": (apply_ms["linked_mean"]["ms"] / apply_ms["independent"]["ms"]
                                                      if apply_ms["independent"]["ms"] > 0 else None),
        "parity": {"rms_vs_alone": par, "ok": all(p < 1e-6 for p in par)},
    }))


if __name__ == "__main__":
    main()
