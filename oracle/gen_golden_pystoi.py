"""Writes tests/golden/pystoi_ref.json: pystoi's STOI and extended STOI, as the reference's df.evaluation_utils.stoi
reports them (df.io.resample to 10 kHz with sinc_fast, then pystoi.stoi), computed by the float64 restatement
tests/pystoi_ref64.py (pystoi is not a dependency):

* "ci_stoi": the STOI known answers of the reference's CI (df/scripts/test_df.py TARGET_METRICS), read as data;
* "pretrained": the restatement on the reference's own CPU enhance() of the full noisy_snr0.wav with each pretrained
  checkpoint, against clean_freesound_33711.wav (what test_df.py scores);
* "seeded": the same on the first 10 s of the assets (tests/golden/assets) enhanced by the reference modules with the
  seeded weights of oracle/synth_models.py (the weights of kat.json);
* "cases": short pairs at 8, 16, 44.1 and 48 kHz, each made by signal() from its seed (tests/test_pystoi_host.py makes
  them the same way), with their values and counts.

    python oracle/gen_golden_pystoi.py      (needs the reference tree)
"""
from __future__ import annotations

import ast
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "tests")]

import pystoi_ref64 as P  # noqa: E402
import ref_harness as rh  # noqa: E402
import synth_models  # noqa: E402

MODELS = ("DeepFilterNet3", "DeepFilterNet2", "DeepFilterNet")


def ci_targets():
    src = open(os.path.join(rh.REF_ROOT, "DeepFilterNet", "df", "scripts", "test_df.py")).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "TARGET_METRICS" for t in node.targets):
            return {m: v["stoi"] for m, v in ast.literal_eval(node.value).items()}
    raise RuntimeError("TARGET_METRICS not found")


def score(df_io, clean: np.ndarray, enhanced: np.ndarray, sr: int):
    """evaluation_utils.stoi's resample, then the restatement: (stoi, estoi, counts)."""
    x10, y10 = (df_io.resample(torch.as_tensor(np.ascontiguousarray(a, np.float32)), sr, 10000, method="sinc_fast").numpy()
                for a in (clean, enhanced))
    r = P.pystoi10(x10, y10)
    return r["stoi"], r["estoi"], {k: r[k] for k in ("F", "K", "lc", "nf", "J")}


def enhance_pair(model_dir: str, noisy: np.ndarray):
    from df.enhance import enhance, init_df
    model, st, _, _ = init_df(model_dir, log_file=None, log_level="ERROR", config_allow_defaults=True)
    return enhance(model, st, torch.from_numpy(noisy[None]), pad=True)[0].numpy()


def signal(rng, n, sr):
    blk = max(1, sr // 20)
    env = np.repeat(rng.uniform(0, 1, n // blk + 1) ** 3 * (rng.uniform(0, 1, n // blk + 1) > 0.2), blk)[:n]
    c = (0.3 * env * rng.standard_normal(n)).astype(np.float32)
    d = (rng.uniform(0.3, 1.2) * c + rng.uniform(0.001, 0.1) * rng.standard_normal(n)).astype(np.float32)
    return c, d


def main():
    rh.import_reference()
    import df.io as df_io

    out = {"ci_stoi": ci_targets(), "pretrained": {}, "seeded": {}, "cases": {}}
    full = [rh.read_wav(os.path.join(rh.REF_ROOT, "assets", a))[0] for a in ("clean_freesound_33711.wav", "noisy_snr0.wav")]
    short = [rh.read_wav(os.path.join(GOLDEN, "assets", a))[0] for a in ("clean_freesound_33711.wav", "noisy_snr0.wav")]
    pre = rh.unpack_models()
    seeded = synth_models.make_model_dirs(os.path.join(rh.SCRATCH, "synth"))
    for name in MODELS:
        for key, d, (clean, noisy) in (("pretrained", pre, full), ("seeded", seeded, short)):
            s, e, cnt = score(df_io, clean, enhance_pair(os.path.join(d, name), noisy), 48000)
            out[key][name] = {"stoi": s, "estoi": e, "counts": cnt}
            print(key, name, s, e, cnt)
    for seed, (sr, n) in enumerate(((8000, 6000), (16000, 12000), (44100, 40000), (48000, 52000), (48000, 2000))):
        c, d = signal(np.random.default_rng(seed), n, sr)
        s, e, cnt = score(df_io, c, d, sr)
        out["cases"][f"sr{sr}_n{n}"] = {"sr": sr, "n": n, "seed": seed, "stoi": s, "estoi": e, "counts": cnt}
        print(sr, n, s, e, cnt)
    with open(os.path.join(GOLDEN, "pystoi_ref.json"), "w") as f:
        json.dump(out, f, indent=1, allow_nan=True)


if __name__ == "__main__":
    main()
