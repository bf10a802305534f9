"""Where k_gl_bx's time goes inside a real bench.py step, next to its time alone on an idle GPU.

    python scripts/gl_timeline.py [--config 2] [--warmup 3] [--out DIR]

Runs the bench.py config (default 2: DeepFilterNet3, 128 streams x 10 s) through enhance_device, warms it up, then takes a
torch.profiler trace with CUDA activities of one step (DIR/trace.json).  Every k_gl_bx launch of the traced step is named
after forward_body's call (launch order = bench_gl.gl_calls order, once per time chunk) and printed with its duration, its
stream, the kernels of other streams that overlap it (e.g. the other decoder's k_gru_tc) and its bench_gl.py time alone
on the idle GPU.  Per time chunk, the decoder whose last grouped linear ends later is the one on the critical path.
Also prints the card, its power limit and SM clocks, and every call's shared-memory budget (launch_gl_bx's choice)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import bench_gl  # noqa: E402

BOX, MAX_STAGES, PLANE_BYTES = 128 * 128, 6, 8 * 2 * 4096


def smem_budget(c: dict) -> dict:
    """launch_gl_bx's shared-memory layout for a call at the dense pitches forward_body uses"""
    G, Ig, Hg = c["G"], c["Ig"], c["Hg"]
    Hgp = (Hg + 15) // 16 * 16
    gpc = max(g for g in range(1, G + 1) if G % g == 0 and g * Hgp <= 256 and (g * Hgp) % 32 == 0 and (g * Ig) % 64 == 0
              and g * Ig * Hgp * 4 <= 100 * 1024)
    w, yb = gpc * Ig * Hgp * 4, 128 * gpc * Hg * 4
    ring = lambda staged: min(MAX_STAGES, (227 * 1024 - 2048 - w - staged - 256) // (2 * BOX))
    fp32 = c["fp32"] or c["res"]
    stage_y = fp32 and ring(yb) >= 2
    stage_p = (c["planes"] and Hg % 16 == 0 and (gpc * Hg) % 64 == 0 and (stage_y if fp32 else not c["res"])
               and ring((yb if stage_y else 0) + PLANE_BYTES) >= 2)
    staged = (yb if stage_y else 0) + (PLANE_BYTES if stage_p else 0)
    stages = ring(staged)
    return {"gpc": gpc, "weights_KB": w // 1024, "fp32_tile_KB": yb // 1024 if stage_y else 0,
            "plane_blocks_KB": PLANE_BYTES // 1024 if stage_p else 0, "ring_stages": stages,
            "smem_KB": round((1024 + stages * 2 * BOX + w + staged + 384) / 1024, 1),
            "planes": "staged" if stage_p else ("registers" if c["planes"] else "-")}


def idle_ms(c: dict, M: int, iters: int = 20) -> float:
    import torch
    case = bench_gl.GlCase(c["G"], c["Ig"], c["Hg"], M, fp32=c["fp32"] or c["res"], planes=c["planes"], seed=1)
    if c["res"]:
        case.set_residual()
    res = "y" if c["res"] else None
    for _ in range(3):
        case.launch(c["act"], res)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        case.launch(c["act"], res)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, choices=[2, 3, 4])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "gl_timeline"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gl_timeline.py needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    from deepfilternet_b200 import DfNet, enhance_device, libdf
    from deepfilternet_b200.weights import pack_state_dict, random_state_dict
    from tests_common import synth_audio
    print(json.dumps(bench_gl.card_info()))
    model_name, streams, seconds, _ = bench.CONFIGS[a.config]
    cfg = bench.model_config(model_name)
    _, g = pack_state_dict(random_state_dict(cfg, seed=0), cfg)
    calls = bench_gl.gl_calls(cfg, g)
    M = bench_gl.bench_rows(cfg, streams, seconds)
    for c in calls:
        print(json.dumps({"call": c["name"], "G": c["G"], "Ig": c["Ig"], "Hg": c["Hg"], **smem_budget(c)}))

    sd, _ = bench.load_weights(model_name, cfg)
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs, device=0)
    model = DfNet(cfg, sd, st, device=0)
    audio = synth_audio(streams, bench.SR * seconds, seed=1234, device="cuda:0")
    out = torch.empty_like(audio)
    for _ in range(a.warmup):
        enhance_device(model, st, audio, out=out)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        enhance_device(model, st, audio, out=out)
        torch.cuda.synchronize()
    trace = os.path.join(a.out, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    t0 = ev[0]["ts"]
    step_ms = (max(e["ts"] + e["dur"] for e in ev) - t0) / 1e3
    gl = sorted((e for e in ev if "k_gl_bx" in e["name"]), key=lambda e: e["args"].get("correlation", 0))
    idle = {c["name"]: idle_ms(c, M) for c in calls}
    print(json.dumps({"config": a.config, "model": model_name, "rows_per_call": M, "step_ms_traced": round(step_ms, 3),
                      "k_gl_bx_launches": len(gl), "k_gl_bx_ms_sum": round(sum(e["dur"] for e in gl) / 1e3, 3),
                      "k_gl_bx_idle_ms_sum": round(sum(idle.values()) * len(gl) / max(1, len(calls)), 3), "trace": trace}))
    ends = {}
    for i, e in enumerate(gl):
        name, chunk = calls[i % len(calls)]["name"], i // len(calls)
        s, d = e["ts"], e["dur"]
        stream = e["args"].get("stream")
        over = {}
        for o in ev:
            if o is e or o["args"].get("stream") == stream:
                continue
            ov = min(s + d, o["ts"] + o["dur"]) - max(s, o["ts"])
            if ov > 0:
                k = o["name"].split("(")[0].split("<")[0].replace("void ", "").replace("dfb::", "")
                over[k] = over.get(k, 0.0) + ov
        ends[(chunk, name)] = s + d
        print(json.dumps({"chunk": chunk, "call": name, "start_ms": round((s - t0) / 1e3, 3), "ms": round(d / 1e3, 4),
                          "idle_ms": round(idle[name], 4), "stream": stream, "grid": e["args"].get("grid"),
                          "overlapped_by_ms": {k: round(v / 1e3, 3) for k, v in sorted(over.items(), key=lambda kv: -kv[1])[:4]}}))
    for chunk in range(len(gl) // max(1, len(calls))):
        df_end, erb_end = ends.get((chunk, "df_dec.df_out")), ends.get((chunk, "erb_dec.emb_gru.out"))
        if df_end and erb_end:
            print(json.dumps({"chunk": chunk, "critical_decoder": "df_dec" if df_end > erb_end else "erb_dec",
                              "df_dec_ends_ms": round((df_end - t0) / 1e3, 3), "erb_dec_ends_ms": round((erb_end - t0) / 1e3, 3)}))


if __name__ == "__main__":
    main()
