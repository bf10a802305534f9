#!/usr/bin/env python3
"""Serving simulation for streaming slots: one DfStream handle of 256 slots (seeded random weights) serves calls that
start and end at seeded times, for DeepFilterNet3 and DeepFilterNet3_ll.

Sessions last 2-30 s (uniform); arrivals (Poisson, at the rate that keeps about half of the slots open) open a free
slot, and a session closes its slot after its last hop.  The handle is fed in calls of --hops hops (1 and 10 by
default).  Reported per model and call size:
  * device time per call (CUDA events around each process call, which includes the slot bookkeeping of that call),
    p50 and p99;
  * useful audio-s/s: audio of the open sessions per second of device time;
  * the same traffic with all 256 slots computed on every call (no slot operations: the only option before slots);
  * the same traffic with per-session settings ("controls"): every session gets its own random attenuation limit
    (6-40 dB) and post-filter beta (0-0.05) when it opens, about 2 % of the calls change one live slot's settings, and
    every call asks for the LSNR of its output hops;
  * stereo traffic ("linked"): the same arrival process, but each arrival is a stereo call with probability 0.5 and
    takes two free slots as one slot group (open_linked) on a handle with reduce_mask="mean", so its channels share one
    ERB mask; "linked_as_mono" runs the identical traffic with every channel opened as its own mono slot.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_slots.py [--slots 256] [--calls 400] [--hops 1 10] [--warmup 20] [--modes ...]
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

SR, HOP = 48000, 480
MODES = ("slots", "all_computed", "controls", "linked", "linked_as_mono")
STEREO = ("linked", "linked_as_mono")


def traffic(slots: int, calls: int, hops: int, seed: int):
    """(slots open at the start, and per call: slots to close, slots to open, open slots after the operations).  Starts
    in steady state: half of the slots open, with uniformly distributed remaining lengths."""
    rng = np.random.default_rng(seed)
    lo, hi = 2 * SR // HOP, 30 * SR // HOP                     # session length in hops
    rate = (slots / 2) / ((lo + hi) / 2)                     # arrivals per hop that keep half the slots busy
    left = np.full(slots, -1, np.int64)                      # hops a session still has; -1: free
    start = rng.permutation(slots)[:slots // 2]
    left[start] = rng.integers(1, hi + 1, slots // 2)
    plan = []
    for _ in range(calls):
        closes = np.flatnonzero(left == 0).tolist()
        left[closes] = -1
        free = np.flatnonzero(left < 0)
        k = min(int(rng.poisson(rate * hops)), free.size)
        opens = rng.choice(free, k, replace=False).tolist() if k else []
        left[opens] = rng.integers(lo, hi + 1, k)
        live = int((left > 0).sum())
        left[left > 0] = np.maximum(left[left > 0] - hops, 0)
        plan.append((closes, opens, live))
    return sorted(start.tolist()), plan


def stereo_traffic(slots: int, calls: int, hops: int, seed: int):
    """traffic() with sessions of one or two channels (probability 0.5 each): (sessions open at the start, and per call:
    sessions to close, sessions to open, open channels after the operations); a session is its list of slots."""
    rng = np.random.default_rng(seed)
    lo, hi = 2 * SR // HOP, 30 * SR // HOP
    rate = (slots / 2) / ((lo + hi) / 2) / 1.5               # 1.5 channels per session: about half the slots busy
    left = {}                                                # session (tuple of slots) -> hops it still has
    free = list(rng.permutation(slots))

    def arrive(n_hops):
        c = 2 if rng.random() < 0.5 else 1
        if len(free) < c:
            return None
        ses = tuple(int(free.pop()) for _ in range(c))
        left[ses] = n_hops
        return ses

    start = []
    while sum(len(k) for k in left) < slots // 2:
        start.append(arrive(int(rng.integers(1, hi + 1))))
    plan, cooling = [], []                                   # a closed session's slots return once its tail is out
    for i in range(calls):
        closes = [k for k, v in left.items() if v == 0]
        for k in closes:
            del left[k]
            cooling.append((i + 1 + -(-4 // hops), k))         # 4 hops: the longest latency (DeepFilterNet2)
        free.extend(b for j, k in cooling if j <= i for b in k)
        cooling = [(j, k) for j, k in cooling if j > i]
        rng.shuffle(free)
        opens = [o for o in (arrive(int(rng.integers(lo, hi + 1))) for _ in range(int(rng.poisson(rate * hops)))) if o]
        live = sum(len(k) for k, v in left.items() if v > 0)
        for k in left:
            left[k] = max(left[k] - hops, 0)
        plan.append(([list(k) for k in closes], [list(k) for k in opens], live))
    return [list(k) for k in start], plan


def run_stereo(model, st, x, slots: int, calls: int, hops: int, warmup: int, seed: int, mode: str):
    """One pass of stereo_traffic: "linked" opens each stereo session as a slot group, "linked_as_mono" as two mono slots."""
    import torch
    from deepfilternet_b200 import DfStream
    start, plan = stereo_traffic(slots, calls, hops, seed)
    linked = mode == "linked"
    s = DfStream(model, st, batch=slots, reduce_mask="mean" if linked else None)
    for _ in range(warmup):
        s.process(x)
    s.flush()

    def open_(ses):
        if linked and len(ses) > 1:
            s.open_linked(ses)
        else:
            s.open(ses)

    for ses in start:
        open_(ses)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in plan]
    torch.cuda.synchronize()
    for (closes, opens, _), (e0, e1) in zip(plan, ev):
        e0.record()
        for ses in closes:
            s.close(ses)
        for ses in opens:
            open_(ses)
        s.process(x)
        e1.record()
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    useful = sum(live for _, _, live in plan) * hops * HOP / SR
    return {"p50_ms": float(np.percentile(ms, 50)), "p99_ms": float(np.percentile(ms, 99)), "mean_ms": float(ms.mean()),
            "useful_audio_s_per_s": useful / (ms.sum() / 1e3), "mean_open_channels": float(np.mean([v for _, _, v in plan])),
            "stereo_share": float(np.mean([len(k) == 2 for _, o, _ in plan for k in o] or [0]))}


def run(name: str, slots: int, calls: int, hops: int, warmup: int, seed: int, modes=("slots", "all_computed", "controls")):
    import torch
    from deepfilternet_b200 import DfNet, DfStream, libdf
    from deepfilternet_b200.weights import random_state_dict
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
    x = torch.randn(slots, hops * HOP, device="cuda") * 0.1
    start, plan = traffic(slots, calls, hops, seed)
    rng = np.random.default_rng(seed + 1)
    setting = lambda: (float(rng.uniform(6, 40)), float(rng.uniform(0, 0.05)))   # (atten_lim_db, beta) of a session
    start_set = [setting() for _ in start]
    open_set = [[setting() for _ in opens] for _, opens, _ in plan]
    change = [(rng.random() < 0.02, rng.random(), setting()) for _ in plan]        # (change?, which live slot, to what)
    res = {}
    for mode in [m for m in modes if m not in STEREO]:
        s = DfStream(model, st, batch=slots)
        for _ in range(warmup):
            s.process(x)
        s.reset()
        live = set()
        if mode != "all_computed":   # the steady state the plan starts from: flush frees every slot, then half of them open
            s.flush()
            s.open(start)
            live = set(start)
        if mode == "controls":
            for b, (db, beta) in zip(start, start_set):
                s.set_atten_lim(db, [b])
                s.set_post_filter_beta(beta, [b])
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in plan]
        torch.cuda.synchronize()
        for (closes, opens, _), (e0, e1), sets, (chg, which, to) in zip(plan, ev, open_set, change):
            e0.record()
            if mode != "all_computed":
                if closes:
                    s.close(closes)
                if opens:
                    s.open(opens)
                live.difference_update(closes)
                live.update(opens)
            if mode == "controls":
                for b, (db, beta) in zip(opens, sets):
                    s.set_atten_lim(db, [b])
                    s.set_post_filter_beta(beta, [b])
                if chg and live:
                    b = sorted(live)[int(which * len(live))]
                    s.set_atten_lim(to[0], [b])
                    s.set_post_filter_beta(to[1], [b])
                s.process(x, return_lsnr=True)
            else:
                s.process(x)
            e1.record()
        torch.cuda.synchronize()
        ms = np.array([a.elapsed_time(b) for a, b in ev])
        useful = sum(live for _, _, live in plan) * hops * HOP / SR
        res[mode] = {"p50_ms": float(np.percentile(ms, 50)), "p99_ms": float(np.percentile(ms, 99)),
                     "mean_ms": float(ms.mean()), "useful_audio_s_per_s": useful / (ms.sum() / 1e3)}
        del s
    for mode in [m for m in modes if m in STEREO]:
        res[mode] = run_stereo(model, st, x, slots, calls, hops, warmup, seed, mode)
    res["mean_open_slots"] = float(np.mean([live for _, _, live in plan]))
    useful = {k: v["useful_audio_s_per_s"] for k, v in res.items() if isinstance(v, dict)}
    if "slots" in useful and "all_computed" in useful:
        res["speedup_useful"] = useful["slots"] / useful["all_computed"]
    if "slots" in useful and "controls" in useful:
        res["controls_vs_slots_useful"] = useful["controls"] / useful["slots"]
    if "linked" in useful and "linked_as_mono" in useful:
        res["linked_vs_mono_useful"] = useful["linked"] / useful["linked_as_mono"]
        res["linked_vs_mono_p50"] = res["linked"]["p50_ms"] / res["linked_as_mono"]["p50_ms"]
        res["linked_vs_mono_p99"] = res["linked"]["p99_ms"] / res["linked_as_mono"]["p99_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--hops", type=int, nargs="+", default=[1, 10])
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--modes", nargs="+", default=list(MODES), choices=MODES)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_slots.py measures on a GPU"
    before = card()
    rows = {}
    for name in a.models:
        for hops in a.hops:
            calls = a.calls if hops == 1 else max(a.calls // hops, 40)
            rows[f"{name}/{hops}hop"] = run(name, a.slots, calls, hops, a.warmup, a.seed, a.modes)
    print(json.dumps({"metric": "serving simulation, streaming slots vs every slot computed vs slots with per-session "
                                "settings and LSNR output vs stereo slot groups", "weights": "random (seed 1)",
                      "card": before, "card_after": card(), "slots": a.slots, "session_s": [2, 30], "results": rows}))


if __name__ == "__main__":
    main()
