"""Times the tensor-core grouped linear (k_gl_bx, csrc/dfb_gl.cu) alone, once per call that bench.py's models make.

    python bench_gl.py [--iters 50] [--warmup 5] [--models DeepFilterNet3,DeepFilterNet2,DeepFilterNet3_ll]

For every GroupedLinearEinsum layer that forward_body (csrc/dfb_model.cu) runs on k_gl_bx -- with the shape, output kinds
(fp32, BF16 hi / lo planes or both), residual and activation it has there -- one launch is timed on seeded data at the
row count of the model's bench.py config (rows per call = streams x (frames per time chunk + halo)).  Reported per call:
ms per launch (CUDA events over --iters launches after --warmup), the bytes the kernel has to move (input planes, outputs,
residual) and that rate against the H100 SXM data-sheet 3.35 TB/s.  DeepFilterNet v1 is not listed: its GroupedLinear
layers carry a bias and run on the FFMA kernel.  Writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes/s
SR, HALO = 48000, 8         # bench.py sample rate; kHalo (dfb_model.cu): frames of context before a time chunk
# bench.py config per model: (streams, seconds)
BENCH = {"DeepFilterNet3": (128, 10), "DeepFilterNet2": (512, 10), "DeepFilterNet3_ll": (256, 10)}
ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2


def bx_shape_ok(G: int, I: int, O: int) -> bool:
    """gl_bx_geometry (dfb_gl.cu): the shapes k_gl_bx builds"""
    if not G or I % G or O % G:
        return False
    Ig, Hg = I // G, O // G
    if Ig % 16 or Hg % 4:
        return False
    Hgp = (Hg + 15) // 16 * 16
    return any(G % c == 0 and c * Hgp <= 256 and (c * Hgp) % 32 == 0 and (c * Ig) % 64 == 0 and c * Ig * Hgp * 4 <= 100 * 1024
               for c in range(1, G + 1))


def gl_calls(cfg, g: dict) -> list:
    """The k_gl_bx launches of one forward_body pass, in launch order: dicts with name, G, Ig, Hg, act, fp32 (writes y),
    planes (writes BF16 hi / lo planes of y), res (adds a residual read from y itself, in place).  Mirrors forward_body:
    df_fc_emb runs fused with df_conv1 (k_dwpw_gl), fp32 outputs that only feed planes are not written."""
    E, Fd, O2 = cfg.nb_erb, cfg.nb_df, 2 * cfg.df_order
    H, Hd = g["emb_hidden"], g["df_hidden"]
    ED = E // 4 * 64
    dfn2 = g["model_kind"] == 2
    emb_in = 2 * ED if g["enc_concat"] else ED
    emb = H if dfn2 else ED
    calls = []

    def add(name, G, I, O, act, fp32, planes, res=False):
        if G and bx_shape_ok(G, I, O):
            calls.append(dict(name=name, G=G, Ig=I // G, Hg=O // G, act=act, fp32=fp32, planes=planes, res=res))

    add("enc.emb_gru.in", g["g_enc_in"], emb_in, H, ACT_RELU, False, True)
    if g["g_enc_out"]:
        add("enc.emb_gru.out", g["g_enc_out"], H, ED, ACT_RELU, True, True)
    if g["g_df_skip"] and not dfn2:
        add("df_dec.df_skip", g["g_df_skip"], emb, Hd, ACT_NONE, True, False)
    add("df_dec.df_gru.in", g["g_df_in"], emb, Hd, ACT_RELU, dfn2, True)
    if g["g_df_skip"] and dfn2:
        add("df_dec.df_skip", g["g_df_skip"], emb, Hd, ACT_NONE, True, False, res=True)
    add("df_dec.df_out", g["g_df_out"], Hd, Fd * O2, ACT_TANH, True, False, res=True)
    add("erb_dec.emb_gru.in", g["g_erb_in"], emb, H, ACT_RELU, dfn2, True)
    add("erb_dec.emb_gru.out", g["g_erb_out"], H, ED, ACT_RELU, True, False)
    return calls


def bench_rows(cfg, streams: int, seconds: int) -> int:
    """rows of one time chunk of the bench config: the default chunk plan (dfb200.h dfb_model_set_chunking: 3 chunks up to
    8 streams, 2 up to 256, else 1) plus the halo frames before every chunk after the first"""
    frames = (SR * seconds + cfg.fft_size) // cfg.hop_size
    chunks = 3 if streams <= 8 else 2 if streams <= 256 else 1
    per = -(-frames // chunks)
    return streams * (per + (HALO if chunks > 1 else 0))


def call_bytes(c: dict, M: int) -> int:
    K, N = c["G"] * c["Ig"], c["G"] * c["Hg"]
    return M * (4 * K + 4 * N * (int(c["fp32"]) + int(c["planes"]) + int(c["res"])))


class GlCase:
    """Seeded device buffers of one launch: X planes, weight image, y (+ residual in place) and output planes.  Rows
    past the first `block` repeat the seeded block (bench-sized M without gigabytes of host-side random numbers)."""

    def __init__(self, G, Ig, Hg, M, fp32=True, planes=True, seed=0, device="cuda", block=4096):
        import torch
        from deepfilternet_b200.weights import gl_bx_image
        rng = np.random.default_rng(seed)
        self.G, self.Ig, self.Hg, self.M = G, Ig, Hg, M
        K, N = G * Ig, G * Hg
        mb = min(M, block)
        self.w = (rng.standard_normal((G, Ig, Hg)) / np.sqrt(Ig)).astype(np.float32)
        self.x = rng.standard_normal((mb, K)).astype(np.float32)
        self.r = rng.standard_normal((mb, N)).astype(np.float32)
        if mb < M:
            self.x, self.r = np.resize(self.x, (M, K)), np.resize(self.r, (M, N))
        xt = torch.from_numpy(self.x)
        hi = xt.to(torch.bfloat16)
        lo = (xt - hi.float()).to(torch.bfloat16)
        self.x_hi, self.x_lo = hi.view(torch.int16).to(device), lo.view(torch.int16).to(device)
        self.w_img = torch.from_numpy(gl_bx_image(self.w)).to(device)
        self.y = torch.zeros((M, N), dtype=torch.float32, device=device) if fp32 else None
        self.y_hi = torch.zeros((M, N), dtype=torch.int16, device=device) if planes else None
        self.y_lo = torch.zeros((M, N), dtype=torch.int16, device=device) if planes else None

    def set_residual(self):
        """y := the seeded residual (launches with res = y then add it in place)"""
        import torch
        self.y.copy_(torch.from_numpy(self.r))

    def launch(self, act=ACT_NONE, res=None, oscale=1.0, ooffset=0.0, stream=None):
        """res: None, "y" (in place) or a device tensor [M][G*Hg]"""
        import torch
        from deepfilternet_b200 import _lib
        K, N = self.G * self.Ig, self.G * self.Hg
        resp = None if res is None else (self.y if isinstance(res, str) else res).data_ptr()
        ptr = lambda t: None if t is None else t.data_ptr()
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream
        rc = _lib.lib().dfb_debug_gl_bx(self.x_hi.data_ptr(), self.x_lo.data_ptr(), K, self.w_img.data_ptr(), resp, N,
                                        ptr(self.y), N, ptr(self.y_hi), ptr(self.y_lo), N, self.M, self.G, self.Ig, self.Hg,
                                        act, oscale, ooffset, st)
        if rc:
            raise RuntimeError(f"dfb_debug_gl_bx: {rc} {_lib.lib().dfb_last_error().decode()}")


def card_info() -> dict:
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit, sm_clock, max_sm_clock"] = q
    except Exception as e:   # the query is informational only
        out["nvidia-smi"] = f"unavailable ({e})"
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--models", default="DeepFilterNet3,DeepFilterNet2,DeepFilterNet3_ll")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gl.py needs a CUDA device")
    import bench
    from deepfilternet_b200.weights import pack_state_dict, random_state_dict
    print(json.dumps(card_info()))
    total = {}
    for model in a.models.split(","):
        cfg = bench.model_config(model)
        _, g = pack_state_dict(random_state_dict(cfg, seed=0), cfg)
        streams, seconds = BENCH[model]
        M = bench_rows(cfg, streams, seconds)
        for c in gl_calls(cfg, g):
            case = GlCase(c["G"], c["Ig"], c["Hg"], M, fp32=c["fp32"] or c["res"], planes=c["planes"], seed=1)
            if c["res"]:
                case.set_residual()
            res = "y" if c["res"] else None
            for _ in range(a.warmup):
                case.launch(c["act"], res)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                case.launch(c["act"], res)
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / a.iters
            nb = call_bytes(c, M)
            total[model] = total.get(model, 0.0) + ms
            print(json.dumps({"model": model, "call": c["name"], "G": c["G"], "Ig": c["Ig"], "Hg": c["Hg"], "M": M,
                              "out": "+".join(k for k in ("fp32", "planes") if c[k]), "res": c["res"], "act": c["act"],
                              "ms": round(ms, 4), "MB": round(nb / 1e6, 2), "GB/s": round(nb / ms / 1e6, 1),
                              "of_peak": round(nb / ms / 1e-3 / HBM_PEAK, 3)}))
            del case
    print(json.dumps({"ms_per_pass": {k: round(v, 4) for k, v in total.items()}}))


if __name__ == "__main__":
    main()
