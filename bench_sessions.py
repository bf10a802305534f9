#!/usr/bin/env python3
"""Session migration on the bench_slots.py server: one DfStream handle of 256 slots (seeded random weights) with about
half of them open, for DeepFilterNet3 and DeepFilterNet3_ll.

Reported per model, each as median (min - max) of --reps runs, host clock around the call and a device synchronise:
  * export_d2d_ms / import_d2d_ms: DfStream.export of 128 sessions to a device blob (a snapshot: release=False) and
    DfStream.resume of that blob into a second, long-lived 256-slot handle with no live session;
  * export_host_ms / import_host_ms: the same through a host blob (device="cpu", page-locked);
  * slot_call_ms: one process call of one hop on the source handle, the per-call path the sessions leave and join;
  * bytes_per_session: the blob's size over its sessions (header and records included), and the state row alone.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.

    python bench_sessions.py [--slots 256] [--sessions 128] [--reps 5] [--warmup 20]
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

from bench import model_config  # noqa: E402
from bench_ragged import card  # noqa: E402
from bench_slots import traffic  # noqa: E402

HOP = 480


def stat(ms):
    ms = np.asarray(ms)
    return {"median": float(np.median(ms)), "min": float(ms.min()), "max": float(ms.max())}


def run(name: str, slots: int, n_ses: int, reps: int, warmup: int, seed: int):
    import torch
    from deepfilternet_b200 import DfNet, DfStream, libdf
    from deepfilternet_b200.streaming import session_info
    cfg = model_config(name)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict_of(cfg), st)
    x = torch.randn(slots, HOP, device="cuda") * 0.1
    start, _ = traffic(slots, 1, 1, seed)                    # about half of the slots open
    s = DfStream(model, st, batch=slots)
    for _ in range(warmup):
        s.process(x)
    s.flush()
    s.open(start)
    for _ in range(warmup):
        s.process(x)
    moved = start[:n_ses]

    def timed(fn, before=None):
        out = []
        for _ in range(reps):
            if before:
                before()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
        return out

    res = {"slot_call_ms": stat(timed(lambda: s.process(x)))}
    blobs = {}
    for where in ("d2d", "host"):
        dev = None if where == "d2d" else "cpu"
        s.export(moved, device=dev)                          # warm
        res[f"export_{where}_ms"] = stat(timed(lambda: blobs.__setitem__(where, s.export(moved, device=dev))))
        # a long-lived destination of as many slots, idle: each run's sessions leave it again (untimed) before the next
        dst = DfStream(model, st, batch=slots)
        dst.flush()
        land = list(range(len(moved)))
        release = lambda: dst.export(land, release=True)
        dst.resume(blobs[where], land)                      # warm
        res[f"import_{where}_ms"] = stat(timed(lambda: dst.resume(blobs[where], land), before=release))
        dst.process(x)
    info = session_info(blobs["d2d"])
    res["bytes_per_session"] = info.nbytes / len(info.sessions)
    res["state_row_bytes"] = (info.nbytes - 192 - 112 * len(info.sessions)) / info.rows
    res["live_slots"] = len(start)
    res["sessions_moved"] = len(moved)
    res["d2d_vs_slot_call"] = (res["export_d2d_ms"]["median"] + res["import_d2d_ms"]["median"]) / res["slot_call_ms"]["median"]
    return res


def random_state_dict_of(cfg):
    from deepfilternet_b200.weights import random_state_dict
    return random_state_dict(cfg, seed=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--sessions", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--models", nargs="+", default=["DeepFilterNet3", "DeepFilterNet3_ll"])
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_sessions.py measures on a GPU"
    before = card()
    rows = {name: run(name, a.slots, a.sessions, a.reps, a.warmup, a.seed) for name in a.models}
    print(json.dumps({"metric": "session export / import of 128 sessions on a 256-slot handle, device and host blobs, next to "
                                "one slot-path call (ms, median / min / max)", "weights": "random (seed 1)", "card": before,
                      "card_after": card(), "slots": a.slots, "reps": a.reps, "results": rows}))


if __name__ == "__main__":
    main()
