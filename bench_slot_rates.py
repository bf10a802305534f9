#!/usr/bin/env python3
"""Streaming slots at mixed rates: bench_slots.py's server (256 slots, about half of them open, sessions of 2-30 s,
seeded random weights), each session at a rate drawn from a mix (default 30 % 8 kHz, 40 % 16 kHz, 30 % 48 kHz), run
  * by one mixed-rate handle of 256 slots (DfStream(slot_rates=...), each session opened at its rate), and
  * by one handle per rate, 256 slots each, each session in the handle of its rate; a tick is the three handles' calls,
timed as one.
For DeepFilterNet3 and DeepFilterNet3_ll and calls of 1, 4 and 16 hops it reports:
  * device time per call (CUDA events around each tick, slot operations included), mean over the pass; the two set-ups
    alternate pass by pass, and each figure is the median of --reps passes with their min and max;
  * useful audio-s/s: seconds of open sessions' audio per second of device time;
  * the share of the kernel time that k_resample_up and k_resample_down take (torch.profiler, a separate pass each);
and the card's name, power limit and max SM clock, read in the same run.  Prints one JSON line.

    python bench_slot_rates.py [--slots 256] [--calls 200] [--hops 1 4 16] [--reps 5] [--mix 8000:0.3 16000:0.4 48000:0.3]
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

MODEL_SR = 48000


def rated_traffic(slots, calls, hops, seed, mix):
    """traffic() with a rate per session drawn from `mix` {rate: probability}: (start {rate: slots}, and per call:
    {rate: slots to close}, {rate: slots to open}, open slots)."""
    start, plan = traffic(slots, calls, hops, seed)
    rng = np.random.default_rng(seed + 1)
    rates, p = list(mix), np.array(list(mix.values()), np.float64)
    rate_of = {}

    def by_rate(ss, assign):
        out = {r: [] for r in rates}
        for b in ss:
            if assign:
                rate_of[b] = rates[int(rng.choice(len(rates), p=p / p.sum()))]
            out[rate_of[b]].append(b)
        return out

    s0 = by_rate(start, True)
    return s0, [(by_rate(closes, False), by_rate(opens, True), live) for closes, opens, live in plan]


class Mixed:
    """one handle whose slots open at their sessions' rates"""

    def __init__(self, model, st, slots, rates, hops):
        import torch
        from deepfilternet_b200 import DfStream
        self.s = DfStream(model, st, batch=slots, slot_rates=[r for r in rates if r != MODEL_SR])
        self.x = torch.randn(slots, hops * 480, device="cuda") * 0.1

    def start(self, s0):
        self.s.reset()
        self.s.flush()
        for r, ss in s0.items():
            if ss:
                self.s.open(ss, sr=r)

    def tick(self, closes, opens):
        cl = sorted(b for ss in closes.values() for b in ss)
        if cl:
            self.s.close(cl)
        for r, ss in opens.items():
            if ss:
                self.s.open(ss, sr=r)
        self.s.process(self.x)


class PerRate:
    """one handle per rate, each session in the handle of its rate"""

    def __init__(self, model, st, slots, rates, hops):
        import torch
        from deepfilternet_b200 import DfStream
        self.h = {r: DfStream(model, st, batch=slots, **({} if r == MODEL_SR else {"sr": r})) for r in rates}
        self.x = {r: torch.randn(slots, hops * r // 100, device="cuda") * 0.1 for r in rates}

    def start(self, s0):
        for r, s in self.h.items():
            s.reset()
            s.flush()
            if s0[r]:
                s.open(s0[r])

    def tick(self, closes, opens):
        for r, s in self.h.items():
            if closes[r]:
                s.close(closes[r])
            if opens[r]:
                s.open(opens[r])
            s.process(self.x[r])


def one_pass(setup, s0, plan):
    import torch
    setup.start(s0)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in plan]
    torch.cuda.synchronize()
    for (closes, opens, _), (e0, e1) in zip(plan, ev):
        e0.record()
        setup.tick(closes, opens)
        e1.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def share(setup, s0, plan):
    """(share of kernel time in k_resample_up / _down, kernel ms per call) over one profiled pass"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    setup.start(s0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for closes, opens, _ in plan:
            setup.tick(closes, opens)
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


def run(name, slots, calls, hops, reps, warmup, seed, mix):
    from deepfilternet_b200 import DfNet, libdf
    from deepfilternet_b200.weights import random_state_dict
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
    s0, plan = rated_traffic(slots, calls, hops, seed, mix)
    setups = {"mixed": Mixed(model, st, slots, list(mix), hops), "per_rate": PerRate(model, st, slots, list(mix), hops)}
    for su in setups.values():
        su.start(s0)
        for closes, opens, _ in plan[:warmup]:
            su.tick(closes, opens)
    times = {k: [] for k in setups}
    for r in range(reps):
        for k in (list(setups) if r % 2 == 0 else list(setups)[::-1]):
            times[k].append(one_pass(setups[k], s0, plan))
    audio_s = float(np.mean([live for _, _, live in plan])) * hops * 0.01      # per call
    res = {"mean_open_slots": float(np.mean([live for _, _, live in plan]))}
    for k, su in setups.items():
        t = np.array(times[k])
        sh, kms = share(su, s0, plan)
        res[k] = {"call_ms_median": float(np.median(t)), "call_ms_min": float(t.min()), "call_ms_max": float(t.max()),
                  "ms_per_10ms_tick": float(np.median(t) / hops), "audio_s_per_s": audio_s / (float(np.median(t)) / 1e3),
                  "resample_kernel_share": sh, "kernel_ms_per_call": kms}
    res["mixed_vs_per_rate"] = res["mixed"]["call_ms_median"] / res["per_rate"]["call_ms_median"]
    return res


def parse_mix(items):
    mix = {}
    for it in items:
        r, p = it.split(":")
        mix[int(r)] = float(p)
    assert abs(sum(mix.values()) - 1) < 1e-6, "the mix's probabilities add up to 1"
    return mix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--hops", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--mix", nargs="+", default=["8000:0.3", "16000:0.4", "48000:0.3"])
    a = ap.parse_args()
    mix = parse_mix(a.mix)
    import torch
    assert torch.cuda.is_available(), "bench_slot_rates.py measures on a GPU"
    before = card()
    rows = {}
    for name in a.models:
        for hops in a.hops:
            calls = max(a.calls // hops, 40)
            rows[f"{name}/{hops}hop"] = run(name, a.slots, calls, hops, a.reps, a.warmup, a.seed, mix)
    print(json.dumps({"metric": "streaming slots at mixed rates: one mixed-rate handle vs one handle per rate on the same "
                                "traffic: device ms per call (median of passes, min / max), useful audio-s/s and the "
                                "resamplers' share of kernel time", "mix": {str(k): v for k, v in mix.items()},
                      "weights": "random (seed 1)", "card": before, "card_after": card(), "slots": a.slots,
                      "results": rows}))


if __name__ == "__main__":
    main()
