"""Writes tests/golden/metrics_ref.json and tests/golden/metrics_inputs.npz: SI-SDR, STOI and SSNR of the reference's own
functions (df.stoi.stoi, df.sepm.SNRseg after df.io.resample to 16 kHz, and the si_sdr_speechmetrics formula) on:

* the two asset WAVs (clean against noisy_snr0) at 48 kHz, and resampled to 16 kHz and 8 kHz with df.io.resample
  (the inputs are not stored: the tests load the WAVs and resample them the same way);
* clean against 0.5 clean plus seeded noise 30 dB below it (16 kHz);
* clean with 2 s of digital silence at the start and in the middle (8 kHz);
* a 10 kHz entry whose length is an exact multiple of 256;
* a 0.35 s entry (at most 30 STFT frames: one STOI segment);
* a 0.06 s entry (STOI NaN: under 512 samples after silence removal; SSNR valid) and a 0.02 s entry (both NaN);
* an all-zero clean.

A value the reference cannot compute (STOI's skipped entries, SNRseg with no frame) is stored as NaN.  Every case is
checked to have no frame energy within 1e-3 dB of its 40 dB threshold, so that no mask decision can flip on rounding.

    python oracle/gen_golden_metrics.py      (needs the reference tree; writes the two files)
"""
from __future__ import annotations

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

import metrics_ref64 as R  # noqa: E402
import ref_harness  # noqa: E402

ASSETS = ("clean_freesound_33711.wav", "noisy_snr0.wav")


def synthetic_cases(clean48: np.ndarray, df_io):
    rng = np.random.default_rng(20261018)
    c16 = df_io.resample(torch.from_numpy(clean48[None]), 48000, 16000)[0].numpy()
    c8 = df_io.resample(torch.from_numpy(clean48[None]), 48000, 8000)[0].numpy()
    cases = {}
    x = c16[16000:48000]
    n = rng.standard_normal(x.size).astype(np.float32)
    n *= np.sqrt((x.astype(np.float64) ** 2).mean() / 10 ** 3) / np.sqrt((n.astype(np.float64) ** 2).mean())
    cases["scaled_noise_16k"] = (16000, x, (0.5 * x + n).astype(np.float32))
    sp = c8[8000:20000]
    x = np.concatenate([np.zeros(16000), sp[:6000], np.zeros(16000), sp[6000:]]).astype(np.float32)
    cases["silence_8k"] = (8000, x, (x + 0.01 * rng.standard_normal(x.size)).astype(np.float32))
    x = (0.1 * rng.standard_normal(256 * 60)).astype(np.float32)
    cases["mult256_10k"] = (10000, x, (x + 0.05 * rng.standard_normal(x.size)).astype(np.float32))
    x = c16[20000:20000 + 5600]
    cases["short_0.35s_16k"] = (16000, x, (x + 0.02 * rng.standard_normal(x.size)).astype(np.float32))
    x = np.concatenate([0.3 * rng.standard_normal(480), 1e-5 * rng.standard_normal(480)]).astype(np.float32)
    cases["tiny_0.06s_16k"] = (16000, x, (x + 0.01 * rng.standard_normal(x.size)).astype(np.float32))
    x = (0.2 * rng.standard_normal(320)).astype(np.float32)
    cases["tiny_0.02s_16k"] = (16000, x, (x + 0.05 * rng.standard_normal(x.size)).astype(np.float32))
    cases["zero_clean_16k"] = (16000, np.zeros(16000, np.float32), (0.1 * rng.standard_normal(16000)).astype(np.float32))
    return cases


def main():
    sys.modules.setdefault("pesq", types.SimpleNamespace(pesq=None))   # df.sepm imports it; only SNRseg is called
    df = ref_harness.import_reference()
    import df.io as df_io
    import df.sepm as sepm
    import df.stoi as df_stoi

    wav = [ref_harness.read_wav(os.path.join(GOLDEN, "assets", a))[0] for a in ASSETS]
    cases = {}
    for sr in (48000, 16000, 8000):
        c, d = wav
        if sr != 48000:
            c = df_io.resample(torch.from_numpy(c[None]), 48000, sr)[0].numpy()
            d = df_io.resample(torch.from_numpy(d[None]), 48000, sr)[0].numpy()
        cases[f"assets_{sr // 1000}k"] = (sr, c, d)
    synth = synthetic_cases(wav[0], df_io)
    cases.update(synth)

    out = {}
    for name, (sr, c, d) in cases.items():
        c = np.ascontiguousarray(c, np.float32)
        d = np.ascontiguousarray(d, np.float32)
        v64, counts, margin = R.stoi(c, d, sr)
        assert margin > 1e-3, (name, margin)
        st = float(df_stoi.stoi(torch.from_numpy(c[None]), torch.from_numpy(d[None]), sr)[0]) if counts[1] >= 512 else float("nan")
        c16 = c if sr == 16000 else df_io.resample(torch.from_numpy(c[None]), sr, 16000)[0].numpy()
        d16 = d if sr == 16000 else df_io.resample(torch.from_numpy(d[None]), sr, 16000)[0].numpy()
        try:
            ss = float(sepm.SNRseg(c16, d16, 16000))
        except ValueError:   # negative frame count: no frame
            ss = float("nan")
        out[name] = {"sr": sr, "length": int(c.size), "sisdr": ref_harness.si_sdr(c, d), "stoi": st, "ssnr": ss,
                     "counts": list(counts), "stored": name in synth}
        print(f"{name:18s} sr {sr:5d} T {c.size:7d} sisdr {out[name]['sisdr']:9.4f} stoi {st:.6f} ssnr {ss:9.4f} "
              f"counts {counts} margin {margin:.3f} dB")
    np.savez_compressed(os.path.join(GOLDEN, "metrics_inputs.npz"),
                        **{f"{k}.{s}": v for k, (_, c, d) in synth.items() for s, v in (("clean", c), ("degraded", d))})
    with open(os.path.join(GOLDEN, "metrics_ref.json"), "w") as f:
        json.dump({"assets": list(ASSETS), "cases": out}, f, indent=1, allow_nan=True)


if __name__ == "__main__":
    main()
