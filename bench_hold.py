#!/usr/bin/env python3
"""Held sessions on the bench_slots.py server: one 256-slot DfStream handle (seeded random weights) with about half of its
slots open, for DeepFilterNet3 and DeepFilterNet3_ll, one hop per tick.  On each tick every open session has its hop
ready with probability p (0.9: network jitter; 0.5: discontinuous transmission).  The open set is the bench_slots.py
starting set and stays fixed over the measured ticks (sessions of 2 - 30 s rarely end within them).  Three set-ups:
  * A (hold): one call per tick; the ready sessions advance, the others are held (DfStream.hold).
  * B (export / resume): the exact alternative without holds.  Sessions that become not ready are exported with
    release=True into one device blob per tick; a blob whose sessions are all ready again is resumed, one whose sessions
    are partly ready is resumed and its still-unready sessions exported again, around the tick's one call.
  * C (lower bound): a handle whose live sessions are exactly the ready ones (as many open slots, nothing held).
Per set-up and p: per-tick time p50 / p99 (host clock around the tick's calls and a device synchronise) and useful
audio-seconds per second (ready session-hops * 10 ms over the time), each as median (min - max) over --passes passes
alternated between the set-ups.  What A's ticks add to C's: the host time of A's two DfStream.hold calls per tick
(host clock, they run no device work), and, from a separate torch.profiler pass over each set-up, the kernel time and
the device copy / memset time per tick, k_slot_rows' share of A's kernel time and the state bytes it moves per call
(rows moved x row bytes x 4: read and written once through its scratch rows; a fresh row is written once).  Prints one
JSON line with the card's name and power limit read in the same run.

    python bench_hold.py [--ticks 300] [--passes 5] [--p 0.9 0.5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import model_config  # noqa: E402
from bench_ragged import card  # noqa: E402
from bench_slots import traffic  # noqa: E402

HOP = 480


def stat(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return {"median": float(np.median(xs)), "min": float(xs.min()), "max": float(xs.max())}


def rows_moved(s):
    from deepfilternet_b200 import _lib
    n = C.c_int64()
    _lib.check(_lib.lib().dfb_debug_stream_rows_moved(s._h, C.byref(n)))
    return n.value


class Setup:
    """one set-up's handle(s) and its tick; tick(ready) runs one tick for the boolean ready mask over `live`"""

    def __init__(self, kind, model, st, slots, live, x, warmup):
        self.kind, self.model, self.st, self.slots, self.live, self.x = kind, model, st, slots, np.asarray(live), x
        self.handles = {}
        if kind != "C":
            self.s = self._handle(live, warmup)
        self.ready = np.ones(len(live), bool)
        self.blobs = []   # B: [(blob, slots)] of exported sessions
        self.hold_ms = 0.0   # A: host time of the hold calls so far

    def _handle(self, live, warmup):
        from deepfilternet_b200 import DfStream
        s = DfStream(self.model, self.st, batch=self.slots)
        for _ in range(warmup):
            s.process(self.x)
        s.flush()
        s.open(list(live))
        for _ in range(warmup):
            s.process(self.x)
        return s

    def tick(self, ready):
        if self.kind == "C":   # a handle of exactly len(ready) live sessions
            m = int(ready.sum())
            if m not in self.handles:
                self.handles[m] = self._handle(self.live[:m], 2)
            self.handles[m].process(self.x)
            return
        leave = self.live[self.ready & ~ready].tolist()
        join = self.live[~self.ready & ready]
        if self.kind == "A":
            t0 = time.perf_counter()
            if leave:
                self.s.hold(leave)
            if join.size:
                self.s.hold(join.tolist(), False)
            self.hold_ms += (time.perf_counter() - t0) * 1e3
        else:
            if join.size:
                keep = []
                want = set(join.tolist())
                for blob, slots in self.blobs:
                    if want.isdisjoint(slots):
                        keep.append((blob, slots))
                        continue
                    self.s.resume(blob, slots)
                    rest = [b for b in slots if b not in want]
                    if rest:
                        keep.append((self.s.export(rest, release=True), rest))
                self.blobs = keep
            if leave:
                self.blobs.append((self.s.export(leave, release=True), leave))
        self.ready = ready.copy()
        self.s.process(self.x)


def run_pass(setup, masks):
    """(p50, p99, audio-s/s, host ms of the hold calls per tick)"""
    import torch
    ms = []
    setup.hold_ms = 0.0
    for ready in masks:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        setup.tick(ready)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    ms = np.asarray(ms)
    useful = sum(int(r.sum()) for r in masks) * 0.01
    return (float(np.percentile(ms, 50)), float(np.percentile(ms, 99)), useful / (ms.sum() / 1e3),
            setup.hold_ms / len(masks))


def profile_ticks(setup, masks):
    """per tick: kernel ms, device copy + memset ms, k_slot_rows' share of the kernel time; and (A) rows moved per call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    moved = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ready in masks:
            setup.tick(ready)
            if setup.kind == "A":
                moved.append(rows_moved(setup.s))
        torch.cuda.synchronize()
    kern = copy = slot = 0.0   # us
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if e.key.startswith("cuda"):   # runtime API rows
            continue
        if "Memcpy" in e.key or "Memset" in e.key:
            copy += t
            continue
        kern += t
        if "k_slot_rows" in e.key:
            slot += t
    n = len(masks)
    return {"kernel_ms_per_tick": kern / 1e3 / n, "copy_memset_ms_per_tick": copy / 1e3 / n,
            "k_slot_rows_kernel_share": slot / kern if kern else float("nan"),
            "rows_moved_per_call": float(np.mean(moved)) if moved else 0.0}


def run(name, slots, ticks, passes, ps, warmup, seed):
    import torch
    from deepfilternet_b200 import DfNet, libdf
    from deepfilternet_b200.streaming import _BLOB_HEADER, _BLOB_SESSION, session_info
    from deepfilternet_b200.weights import random_state_dict
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, seed=1), st)
    x = torch.randn(slots, HOP, device="cuda") * 0.1
    live, _ = traffic(slots, 1, 1, seed)
    live = sorted(int(b) for b in live)
    out = {"live_sessions": len(live)}
    for p in ps:
        rng = np.random.default_rng(seed + int(p * 100))
        masks = rng.random((ticks, len(live))) < p
        warm = rng.random((20, len(live))) < p
        setups = {k: Setup(k, model, st, slots, live, x, warmup) for k in "ABC"}
        for s in setups.values():   # every shape the timed ticks use, and C's handles
            for r in warm:
                s.tick(r)
            if s.kind == "C":
                for r in masks:
                    s.tick(r)
        res = {k: {"p50": [], "p99": [], "audio_s_per_s": []} for k in setups}
        res["A"]["hold_calls_host_ms_per_tick"] = []
        for _ in range(passes):
            for k, s in setups.items():
                p50, p99, rate, hold_ms = run_pass(s, masks)
                res[k]["p50"].append(p50); res[k]["p99"].append(p99); res[k]["audio_s_per_s"].append(rate)
                if k == "A":
                    res[k]["hold_calls_host_ms_per_tick"].append(hold_ms)
        row = {k: {m: stat(v) for m, v in r.items()} for k, r in res.items()}
        for k in ("A", "C"):
            row[k]["profile"] = profile_ticks(setups[k], masks[:100])
        info = session_info(setups["A"].s.export([live[0]]))
        row_bytes = (info.nbytes - _BLOB_HEADER.itemsize - _BLOB_SESSION.itemsize * len(info.sessions)) / info.rows
        row["A"]["profile"]["k_slot_rows_bytes_per_call"] = row["A"]["profile"]["rows_moved_per_call"] * row_bytes * 4
        row["A_over_C_p50"] = row["A"]["p50"]["median"] / row["C"]["p50"]["median"]
        row["A_over_B_p50"] = row["A"]["p50"]["median"] / row["B"]["p50"]["median"]
        out[f"p={p}"] = row
        del setups
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--p", type=float, nargs="+", default=[0.9, 0.5])
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_hold.py measures on a GPU"
    before = card()
    rows = {name: run(name, a.slots, a.ticks, a.passes, a.p, a.warmup, a.seed) for name in a.models}
    print(json.dumps({"metric": "per-tick time (ms) and useful audio-s/s of a 256-slot handle whose ~128 sessions each have "
                                "a hop ready with probability p: A holds the others, B exports / resumes them, C runs only "
                                "the ready ones (lower bound)", "weights": "random (seed 1)", "card": before,
                      "card_after": card(), "ticks": a.ticks, "passes": a.passes, "results": rows}))


if __name__ == "__main__":
    main()
