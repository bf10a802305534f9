"""Writes tests/golden/composite_ref.json and tests/golden/composite_inputs.npz: LLR, WSS and the composite measure of the
reference's own functions (df.sepm.llr / wss / composite on df.io.resample(x, sr, 16000), PESQ replaced by a constant
stub) on:

* the two asset WAVs (clean against noisy_snr0) at 48 kHz, and resampled to 16 kHz and 8 kHz with df.io.resample (not
  stored: the tests load the WAVs and resample them);
* the 48 kHz assets twice over, a 20 s entry (not stored);
* 16 kHz entries of 599, 600, 601, 719 and 720 samples (T = 0, 1, 1, 1 and 2 frames);
* 16 kHz entries of T = 10, 30 and 50 frames, where T * 0.95 lands on .5 (k = 10, 28 and 48);
* an all-zero clean against noise, and zero against zero (16 kHz);
* an 8 kHz entry.

Entries with fewer than 600 samples at 16 kHz have no composite value (the reference's wss raises): NaN.  The file also
keeps the composite known answers of the reference's CI (df/scripts/test_df.py: PESQ, CSIG, CBAK, COVL, SSNR of
noisy_snr0 enhanced by each pretrained model, against clean_freesound_33711), as data.

    python oracle/gen_golden_composite.py      (needs the reference tree; writes the two files)
"""
from __future__ import annotations

import ast
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, "tests")]

import composite_ref64 as R  # noqa: E402
import ref_harness  # noqa: E402

ASSETS = ("clean_freesound_33711.wav", "noisy_snr0.wav")
STUB_PESQ = 2.5


def synthetic_cases(clean48: np.ndarray, df_io):
    rng = np.random.default_rng(20261019)
    c16 = df_io.resample(torch.from_numpy(clean48[None]), 48000, 16000)[0].numpy()
    c8 = df_io.resample(torch.from_numpy(clean48[None]), 48000, 8000)[0].numpy()
    cases = {}

    def noisy(x, s):
        return (0.8 * x + s * rng.standard_normal(x.size)).astype(np.float32)

    for n in (599, 600, 601, 719, 720):
        x = c16[30000:30000 + n]
        cases[f"len{n}_16k"] = (16000, x, noisy(x, 0.01))
    for T in (10, 30, 50):
        x = c16[40000:40000 + 480 + 120 * T]
        cases[f"frames{T}_16k"] = (16000, x, noisy(x, 0.02))
    cases["zero_clean_16k"] = (16000, np.zeros(16000, np.float32), (0.1 * rng.standard_normal(16000)).astype(np.float32))
    cases["zero_zero_16k"] = (16000, np.zeros(16000, np.float32), np.zeros(16000, np.float32))
    x = c8[12000:28000]
    cases["speech_8k"] = (8000, x, noisy(x, 0.01))
    return cases


def ci_targets():
    """TARGET_METRICS' "composite" lists of df/scripts/test_df.py, read as data."""
    src = open(os.path.join(ref_harness.REF_ROOT, "DeepFilterNet", "df", "scripts", "test_df.py")).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "TARGET_METRICS" for t in node.targets):
            tm = ast.literal_eval(node.value)
            return {m: v["composite"] for m, v in tm.items()}
    raise RuntimeError("TARGET_METRICS not found")


def main():
    sys.modules.setdefault("pesq", types.SimpleNamespace(pesq=None))
    ref_harness.import_reference()
    import df.io as df_io
    import df.sepm as sepm

    sepm.pesq = lambda fs, r, d, mode: STUB_PESQ   # composite's PESQ-WB, a constant
    wav = [ref_harness.read_wav(os.path.join(GOLDEN, "assets", a))[0] for a in ASSETS]
    cases = {}
    for sr in (48000, 16000, 8000):
        c, d = wav
        if sr != 48000:
            c = df_io.resample(torch.from_numpy(c[None]), 48000, sr)[0].numpy()
            d = df_io.resample(torch.from_numpy(d[None]), 48000, sr)[0].numpy()
        cases[f"assets_{sr // 1000}k"] = (sr, c, d)
    cases["assets_twice_48k"] = (48000, np.concatenate([wav[0], wav[0]]), np.concatenate([wav[1], wav[1]]))
    synth = synthetic_cases(wav[0], df_io)
    cases.update(synth)

    out = {}
    for name, (sr, c, d) in cases.items():
        c = np.ascontiguousarray(c, np.float32)
        d = np.ascontiguousarray(d, np.float32)
        c16 = c if sr == 16000 else df_io.resample(torch.from_numpy(c[None]), sr, 16000)[0].numpy()
        d16 = d if sr == 16000 else df_io.resample(torch.from_numpy(d[None]), sr, 16000)[0].numpy()
        T = R.n_frames(c16.size)
        lv = sepm.llr(c16, d16, 16000) if T > 0 else None
        lv = float("nan") if lv is None else float(lv)
        if c16.size >= 600:
            wv = float(sepm.wss(c16, d16, 16000))
            comp = [float(v) for v in sepm.composite(c16, d16, 16000)]
            margin = R.wss_frames(c16, d16)[1]
            assert margin > 1e-6, (name, margin)
        else:
            wv, comp, margin = float("nan"), [float("nan")] * 5, float("nan")
        out[name] = {"sr": sr, "length": int(c.size), "n16": int(c16.size), "frames": T, "keep": R.keep_count(T),
                     "llr": lv, "wss": wv, "composite": comp, "stored": name in synth}
        print(f"{name:18s} sr {sr:5d} T {T:5d} llr {lv:.6f} wss {wv:.6f} composite {np.round(comp, 5)} margin {margin:.2e}")
    arrays = {f"{k}.{s}": v for k, (_, c, d) in synth.items() for s, v in (("clean", c), ("degraded", d))}
    np.savez_compressed(os.path.join(GOLDEN, "composite_inputs.npz"), **arrays)
    with open(os.path.join(GOLDEN, "composite_ref.json"), "w") as f:
        json.dump({"assets": list(ASSETS), "stub_pesq": STUB_PESQ, "cases": out, "ci_composite": ci_targets()}, f,
                  indent=1, allow_nan=True)


if __name__ == "__main__":
    main()
