"""Device LLR and WSS (dfb_metrics_compute's bits 16 and 32) and the composite measure of deepfilternet_b200.evaluation_utils
against the reference's fixtures, frame by frame and per entry against the float64 restatement (tests/composite_ref64.py)
on the device's own 16 kHz rows, their bit-exact batching invariants, the evaluation loop with a caller's PESQ and the
CLI."""
import csv
import os
import sys
import types

import numpy as np
import pytest
import torch

import composite_ref64 as R
from test_composite_host import REF, load_cases
from test_metrics_host import close

pytestmark = pytest.mark.gpu

from deepfilternet_b200 import _lib, evaluation_utils as E, init_df  # noqa: E402
from deepfilternet_b200.io import resample, save_audio  # noqa: E402

OLD = ("sisdr", "stoi", "ssnr")
NEW = ("llr", "wss")


def signal(rng, n, sr):
    blk = max(1, sr // 20)
    env = np.repeat(rng.uniform(0, 1, n // blk + 1) ** 3 * (rng.uniform(0, 1, n // blk + 1) > 0.2), blk)[:n]
    c = (0.3 * env * rng.standard_normal(n)).astype(np.float32)
    d = (rng.uniform(0.3, 1.2) * c + rng.uniform(0.001, 0.1) * rng.standard_normal(n)).astype(np.float32)
    return c, d


def rows16(x, sr):
    """io.resample's 16 kHz row: bit for bit what the device scores."""
    return x if sr == 16000 else resample(torch.from_numpy(x).reshape(1, -1), sr, 16000)[0].numpy()


def batch(rng, B, sr, smin=0.03, smax=8.0):
    """B seeded entries, none with a band energy within 1e-6 dB of a slope sign change or the -100 dB clamp."""
    out = []
    while len(out) < B:
        n = max(1, int(sr * np.exp(rng.uniform(np.log(smin), np.log(smax)))))
        c, d = signal(rng, n, sr)
        c16, d16 = rows16(c, sr), rows16(d, sr)
        if R.n_frames(c16.size) == 0 or R.wss_frames(c16, d16)[1] > 1e-6:
            out.append((c, d))
    return out


def score(entries, sr, metrics):
    r = E.evaluate_batch([torch.from_numpy(c) for c, _ in entries], [torch.from_numpy(d) for _, d in entries], sr, metrics)
    return {k: v.numpy() for k, v in r.items()}


def frames(entries, sr):
    h = E.metrics_handle(sr)
    lens = np.array([c.size for c, _ in entries], dtype=np.int64)
    off, n = E.packed_offsets(lens)
    xc = np.ascontiguousarray(np.concatenate([c for c, _ in entries]))
    xd = np.ascontiguousarray(np.concatenate([d for _, d in entries]))
    cap = n // 100 + 16
    T = np.zeros(lens.size, np.int64)
    llr, wss = np.zeros(cap), np.zeros(cap)
    _lib.check(_lib.lib().dfb_debug_metrics_frames(h.handle, xc.ctypes.data, xd.ctypes.data, n, off.ctypes.data,
                                                   lens.ctypes.data, lens.size, T.ctypes.data, llr.ctypes.data,
                                                   wss.ctypes.data, cap))
    o = np.concatenate(([0], np.cumsum(T)))
    return [(llr[o[i]:o[i + 1]], wss[o[i]:o[i + 1]]) for i in range(lens.size)]


def test_fixtures():
    """Device against the reference's values; LLR of rows upsampled from 8 kHz is not compared (near-singular LPC
    models, see test_composite_host)."""
    cases = load_cases()
    for sr in sorted({v[0] for v in cases.values()}):
        names = [k for k, v in cases.items() if v[0] == sr]
        got = score([(cases[k][1], cases[k][2]) for k in names], sr, NEW)
        for i, k in enumerate(names):
            exp = cases[k][3]
            assert close(float(got["wss"][i]), exp["wss"]), (k, float(got["wss"][i]), exp["wss"])
            if sr != 8000:
                assert close(float(got["llr"][i]), exp["llr"]), (k, float(got["llr"][i]), exp["llr"])


@pytest.mark.parametrize("sr,B,seed", [(16000, 20, 1), (48000, 12, 2)])
def test_frames_against_float64(sr, B, seed):
    entries = batch(np.random.default_rng(seed), B, sr)
    got = frames(entries, sr)
    worst = [0.0, 0.0]
    for (c, d), (gl, gw) in zip(entries, got):
        c16, d16 = rows16(c, sr), rows16(d, sr)
        el, ew = R.llr_frames(c16, d16), R.wss_frames(c16, d16)[0]
        assert gl.size == R.n_frames(c16.size) == el.size
        for q, (g, e) in enumerate(((gl, el), (gw, ew))):
            err = np.abs(g - e) / (1e-4 + 1e-4 * np.abs(e))
            worst[q] = max(worst[q], float(err.max(initial=0.0)))
    assert worst[0] <= 1.0 and worst[1] <= 1.0, worst


@pytest.mark.parametrize("sr,B,seed", [(8000, 7, 3), (16000, 33, 4), (22050, 9, 5), (44100, 12, 6), (48000, 40, 7)])
def test_against_float64(sr, B, seed):
    entries = batch(np.random.default_rng(seed), B, sr)
    got = score(entries, sr, NEW + ("ssnr",))
    for i, (c, d) in enumerate(entries):
        c16, d16 = rows16(c, sr), rows16(d, sr)
        assert close(float(got["wss"][i]), R.wss(c16, d16)), (i, c.size, float(got["wss"][i]), R.wss(c16, d16))
        if sr != 8000:
            assert close(float(got["llr"][i]), R.llr(c16, d16)), (i, c.size, float(got["llr"][i]), R.llr(c16, d16))
        assert close(float(got["ssnr"][i]), R.ssnr16(c16, d16)), (i, float(got["ssnr"][i]), R.ssnr16(c16, d16))


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("sr", [16000, 44100])
def test_bit_exact_invariants(sr):
    rng = np.random.default_rng(17)
    entries = batch(rng, 16, sr, smax=6.0)
    allm = OLD + NEW
    base = score(entries, sr, allm)
    old_only = score(entries, sr, OLD)
    perm = rng.permutation(len(entries))
    permuted = score([entries[i] for i in perm], sr, allm)
    others = batch(np.random.default_rng(18), 20, sr, smax=6.0)
    mixed = score(others[:9] + entries + others[9:], sr, allm)
    for m in allm:
        assert np.array_equal(bits(base[m]), bits(score(entries, sr, allm)[m]))
        assert np.array_equal(bits(base[m][perm]), bits(permuted[m]))
        assert np.array_equal(bits(base[m]), bits(mixed[m][9:9 + len(entries)]))
    for m in OLD:   # requesting the new rows changes no bit of the old ones
        assert np.array_equal(bits(base[m]), bits(old_only[m]))
    for i in (0, 7, 15):
        for subset in (("llr",), ("wss",), ("wss", "stoi"), ("sisdr", "llr")):
            sub = score([entries[i]], sr, subset)
            for m in subset:
                assert bits(sub[m][0]) == bits(base[m][i]), (i, subset, m)


def test_device_ragged_equals_batch():
    sr = 48000
    entries = batch(np.random.default_rng(19), 9, sr, smax=4.0)
    S = max(c.size for c, _ in entries)
    xc = torch.zeros(len(entries), S)
    xd = torch.full((len(entries), S), 3.0)
    for i, (c, d) in enumerate(entries):
        xc[i, :c.size] = torch.from_numpy(c)
        xd[i, :d.size] = torch.from_numpy(d)
    dev = E.evaluate_device_ragged(xc.cuda(), xd.cuda(), [c.size for c, _ in entries], sr, NEW + OLD)
    host = score(entries, sr, NEW + OLD)
    for m in NEW + OLD:
        assert dev[m].is_cuda and np.array_equal(bits(dev[m].cpu().numpy()), bits(host[m]))


def test_composite_batch_and_errors():
    sr = 22050
    rng = np.random.default_rng(20)
    entries = [signal(rng, n, sr) for n in (300, 826, 827, 20000, 60000)]   # 16 kHz: 218, 600, 601, ...
    seen = []

    def pesq(r, d):
        seen.append((r.copy(), d.copy()))
        return 1.5 + 0.01 * len(seen)

    cs, ds = [torch.from_numpy(c) for c, _ in entries], [torch.from_numpy(d) for _, d in entries]
    got = E.evaluate_batch(cs, ds, sr, ("stoi", "composite"), pesq=pesq)
    assert list(got) == ["stoi", "composite"] and got["composite"].shape == (5, 5) and got["composite"].dtype == torch.float32
    rows = score(entries, sr, ("ssnr", "llr", "wss"))
    assert len(seen) == 4 and torch.isnan(got["composite"][0]).all()
    for j, i in enumerate(range(1, 5)):
        c16, d16 = rows16(entries[i][0], sr), rows16(entries[i][1], sr)
        assert c16.size >= 600 and np.array_equal(seen[j][0], c16) and np.array_equal(seen[j][1], d16)
        exp = E.composite_values(lambda r, d: 1.5 + 0.01 * (j + 1), c16, d16, rows["llr"][i], rows["wss"][i], rows["ssnr"][i])
        assert np.array_equal(got["composite"][i].numpy(), exp)
    with pytest.raises(ValueError, match="does not provide"):
        E.evaluate_batch(cs, ds, sr, ("composite",))

    def boom(r, d):
        raise RuntimeError("no licence")
    with pytest.raises(RuntimeError, match="no licence"):
        E.evaluate_batch(cs, ds, sr, ("composite",), pesq=boom)
    for bad in ("composite-octave", "pesq", "pesq-nb", "dnsmos5"):
        with pytest.raises(ValueError, match="does not provide"):
            E.evaluate_batch(cs, ds, sr, (bad,), pesq=pesq)
    L = _lib.lib()
    h = E.metrics_handle(16000)
    x = np.zeros(1000, np.float32)
    out = np.zeros(3, np.float32)
    lens, off = np.array([1000], np.int64), np.zeros(1, np.int64)
    for b_ in (8, 64, 16 | 8):
        assert L.dfb_metrics_compute_host(h.handle, x.ctypes.data, x.ctypes.data, 1000, off.ctypes.data, lens.ctypes.data,
                                          lens.ctypes.data, 1, b_, out.ctypes.data) == _lib.DFB_ERR_INVALID
    assert L.dfb_metrics_compute_host(h.handle, x.ctypes.data, x.ctypes.data, 1000, off.ctypes.data, lens.ctypes.data,
                                      lens.ctypes.data, 1, 16 | 32, out.ctypes.data) == 0


def _dataset(tmp_path, sr, n=4):
    rng = np.random.default_rng(21)
    root = tmp_path / "ds"
    for sub in ("clean_testset_wav", "noisy_testset_wav"):
        (root / sub).mkdir(parents=True)
    for i in range(n):
        c, d = signal(rng, int(sr * rng.uniform(0.8, 3.0)), sr)
        save_audio(str(root / "clean_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(c), sr)
        save_audio(str(root / "noisy_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(d), sr)
    return root


def test_evaluation_loop_with_pesq(tmp_path, model_dir):
    from deepfilternet_b200.io import load_audio
    model, df_state, _, _ = init_df(os.path.join(model_dir, "DeepFilterNet3"), log_level="ERROR")
    sr = df_state.sr()
    root = _dataset(tmp_path, sr)
    cl = sorted(str(p) for p in (root / "clean_testset_wav").iterdir())
    no = sorted(str(p) for p in (root / "noisy_testset_wav").iterdir())
    calls, saved = [], []

    def pesq(r, d):
        calls.append((r.copy(), d.copy()))
        return 2.0 + 0.001 * float(np.abs(d.astype(np.float64)).sum() % 7.0)

    got = E.evaluation_loop(df_state, model, cl, no, metrics=["stoi", "composite", "sisdr"], batch_size=3,
                            save_audio_callback=lambda fn, a: saved.append(a[0].numpy().copy()),
                            csv_path_enh=str(tmp_path / "enh.csv"), csv_path_noisy=str(tmp_path / "noisy.csv"),
                            noisy_metric=True, pesq=pesq)
    labels = ["STOI", "PESQ", "CSIG", "CBAK", "COVL", "SSNR", "SISDR"]
    assert list(got) == [f"{p} {m}" for m in labels for p in ("Noisy   ", "Enhanced")]
    # the pairs the loop scored: per batch of 3 files its enhanced entries (the audio handed to save_audio_callback), then
    # its noisy ones; pesq gets io.resample of each, bit for bit
    pairs, rows_e, rows_n = [], {}, {}
    for b0 in range(0, len(cl), 3):
        for kind in ("enh", "noisy"):
            for i in range(b0, min(b0 + 3, len(cl))):
                clean = df_state.synthesis(df_state.analysis(load_audio(cl[i], sr, method="sinc_fast")[0].numpy()))[0]
                if kind == "enh":
                    deg = saved[i]
                else:
                    deg = df_state.synthesis(df_state.analysis(load_audio(no[i], sr, method="sinc_fast")[0].numpy()))[0]
                c16 = rows16(np.ascontiguousarray(clean, np.float32), sr)
                d16 = rows16(np.ascontiguousarray(deg, np.float32), sr)
                pairs.append((c16, d16))
                p = 2.0 + 0.001 * float(np.abs(d16.astype(np.float64)).sum() % 7.0)
                vals = dict(zip(("PESQ", "CSIG", "CBAK", "COVL", "SSNR"), R.composite(c16, d16, p)))
                (rows_e if kind == "enh" else rows_n)[os.path.basename(no[i])] = vals
    assert len(calls) == len(pairs)
    for (r, d), (a, b) in zip(calls, pairs):
        assert np.array_equal(r, a) and np.array_equal(d, b)
    for path, rows, prefix in ((tmp_path / "enh.csv", rows_e, "Enhanced"), (tmp_path / "noisy.csv", rows_n, "Noisy   ")):
        with open(path) as f:
            r = list(csv.reader(f))
        assert r[0] == ["filename"] + labels
        assert [x[0] for x in r[1:]] == [os.path.basename(p) for p in no]
        for x in r[1:]:
            for j, m in enumerate(labels[1:6]):
                assert close(float(x[2 + j]), rows[x[0]][m]), (path, x[0], m, x[2 + j], rows[x[0]][m])
        for m in labels[1:6]:
            assert close(got[f"{prefix} {m}"], float(np.mean([v[m] for v in rows.values()])))
    with pytest.raises(ValueError, match="PESQ"):
        E.evaluation_loop(df_state, model, cl, no, metrics=["stoi", "composite"])


def test_cli_with_a_pesq_module(tmp_path, model_dir, capsys, monkeypatch):
    seen = []

    def fake_pesq(fs, ref, deg, mode):
        seen.append((fs, mode, ref.dtype, ref.shape == deg.shape))
        return 3.0

    monkeypatch.setitem(sys.modules, "pesq", types.SimpleNamespace(pesq=fake_pesq))
    m = os.path.join(model_dir, "DeepFilterNet3")
    root = _dataset(tmp_path, 48000, n=3)
    args = E.cli_parser().parse_args([str(root), "-m", m, "--csv-path-enh", str(tmp_path / "e.csv"), "--batch-size", "2",
                                      "--metrics", "composite", "stoi", "--log-level", "error"])
    res = E.main(args)
    assert list(res) == [f"Enhanced {k}" for k in ("PESQ", "CSIG", "CBAK", "COVL", "SSNR", "STOI")]
    assert res["Enhanced PESQ"] == 3.0 and len(seen) == 3 and all(s[:2] == (16000, "wb") and s[3] for s in seen)
    printed = capsys.readouterr().out.strip().splitlines()[-1]
    assert [float(v) for v in printed.split(",")] == pytest.approx([v for k, v in res.items() if "SSNR" not in k])
    assert next(csv.reader(open(tmp_path / "e.csv"))) == ["filename", "PESQ", "CSIG", "CBAK", "COVL", "SSNR", "STOI"]
    monkeypatch.setitem(sys.modules, "pesq", None)   # import pesq fails: today's error
    with pytest.raises(ValueError, match="does not provide"):
        E.main(args)
