"""Device metrics (dfb_metrics_compute, deepfilternet_b200.evaluation_utils / stoi) against the reference's fixtures and
the float64 restatement, their integer counts, their bit-exact batching invariants, the evaluation loop and its CLI."""
import csv
import ctypes as C
import os

import numpy as np
import pytest
import torch

import metrics_ref64 as R
from test_metrics_host import close, load_cases

pytestmark = pytest.mark.gpu

from deepfilternet_b200 import _lib, enhance, evaluation_utils as E, init_df, stoi  # noqa: E402
from deepfilternet_b200.io import save_audio  # noqa: E402

NAMES = ("sisdr", "stoi", "ssnr")


def signal(rng, n, sr):
    """Seeded speech-like pair: noise under a blocky envelope with silent stretches, and a scaled noisy copy."""
    blk = max(1, sr // 20)
    env = np.repeat(rng.uniform(0, 1, n // blk + 1) ** 3 * (rng.uniform(0, 1, n // blk + 1) > 0.2), blk)[:n]
    c = (0.3 * env * rng.standard_normal(n)).astype(np.float32)
    d = (rng.uniform(0.3, 1.2) * c + rng.uniform(0.001, 0.1) * rng.standard_normal(n)).astype(np.float32)
    return c, d


def batch(rng, B, sr, smin=0.02, smax=20.0):
    """B seeded entries of smin .. smax s (log-uniform), none with a frame within 1e-3 dB of STOI's threshold."""
    out = []
    while len(out) < B:
        n = max(1, int(sr * np.exp(rng.uniform(np.log(smin), np.log(smax)))))
        c, d = signal(rng, n, sr)
        if R.stoi(c, d, sr)[2] > 1e-3:
            out.append((c, d))
    return out


def score(entries, sr, metrics=NAMES):
    r = E.evaluate_batch([torch.from_numpy(c) for c, _ in entries], [torch.from_numpy(d) for _, d in entries], sr, metrics)
    return {k: v.numpy() for k, v in r.items()}


def counts(entries, sr):
    h = E.metrics_handle(sr)
    lens = np.array([c.size for c, _ in entries], dtype=np.int64)
    off, n = E.packed_offsets(lens)
    xc = np.ascontiguousarray(np.concatenate([c for c, _ in entries]))
    xd = np.ascontiguousarray(np.concatenate([d for _, d in entries]))
    out = np.zeros((lens.size, 3), dtype=np.int64)
    _lib.check(_lib.lib().dfb_debug_metrics_counts(h.handle, xc.ctypes.data, xd.ctypes.data, n, off.ctypes.data,
                                                   lens.ctypes.data, lens.size, out.ctypes.data))
    return out


def test_fixtures():
    cases = load_cases()
    for sr in sorted({v[0] for v in cases.values()}):
        names = [k for k, v in cases.items() if v[0] == sr]
        entries = [(cases[k][1], cases[k][2]) for k in names]
        got = score(entries, sr)
        cnt = counts(entries, sr)
        for i, k in enumerate(names):
            exp = cases[k][3]
            for m in NAMES:
                assert close(float(got[m][i]), exp[m]), (k, m, float(got[m][i]), exp[m])
            assert cnt[i].tolist() == exp["counts"], (k, cnt[i], exp["counts"])


@pytest.mark.parametrize("sr,B,seed", [(8000, 1, 1), (16000, 33, 2), (44100, 12, 3), (48000, 96, 4), (10000, 5, 5)])
def test_against_float64(sr, B, seed):
    rng = np.random.default_rng(seed)
    entries = batch(rng, B, sr, smax=20.0 if B <= 33 else 6.0)
    got = score(entries, sr)
    cnt = counts(entries, sr)
    for i, (c, d) in enumerate(entries):
        v, k, _ = R.stoi(c, d, sr)
        assert cnt[i].tolist() == list(k), (i, c.size, cnt[i], k)
        assert close(float(got["stoi"][i]), v), (i, c.size, float(got["stoi"][i]), v)
        assert close(float(got["sisdr"][i]), R.si_sdr(c, d)), (i, float(got["sisdr"][i]), R.si_sdr(c, d))
        assert close(float(got["ssnr"][i]), R.ssnr(c, d, sr)), (i, float(got["ssnr"][i]), R.ssnr(c, d, sr))


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("sr", [16000, 48000])
def test_bit_exact_invariants(sr):
    rng = np.random.default_rng(7)
    entries = batch(rng, 24, sr, smax=8.0)
    base = score(entries, sr)
    again = score(entries, sr)
    perm = rng.permutation(len(entries))
    permuted = score([entries[i] for i in perm], sr)
    others = batch(np.random.default_rng(8), 40, sr, smax=8.0)
    mixed = score(others[:17] + entries + others[17:], sr)
    for m in NAMES:
        assert np.array_equal(bits(base[m]), bits(again[m]))
        assert np.array_equal(bits(base[m][perm]), bits(permuted[m]))
        assert np.array_equal(bits(base[m]), bits(mixed[m][17:17 + len(entries)]))
    for i in (0, 5, 23):   # alone, and a metric subset
        solo = score([entries[i]], sr)
        sub = score([entries[i]], sr, ("ssnr", "stoi"))
        for m in NAMES:
            assert bits(solo[m][0]) == bits(base[m][i])
        assert bits(sub["stoi"][0]) == bits(base["stoi"][i]) and bits(sub["ssnr"][0]) == bits(base["ssnr"][i])


def test_device_ragged_and_stoi_module():
    sr = 16000
    entries = batch(np.random.default_rng(9), 9, sr, smax=5.0)
    S = max(c.size for c, _ in entries)
    xc = torch.zeros(len(entries), S)
    xd = torch.full((len(entries), S), 3.0)   # padding must not be read
    for i, (c, d) in enumerate(entries):
        xc[i, :c.size] = torch.from_numpy(c)
        xd[i, :d.size] = torch.from_numpy(d)
    lens = [c.size for c, _ in entries]
    dev = E.evaluate_device_ragged(xc.cuda(), xd.cuda(), lens, sr)
    host = score(entries, sr)
    for m in NAMES:
        assert dev[m].is_cuda
        assert np.array_equal(bits(dev[m].cpu().numpy()), bits(host[m]))
    # stoi.stoi on equal-length rows: CPU and CUDA inputs, against evaluate_*
    T = min(lens)
    x, y = xc[:, :T].contiguous(), xd[:, :T].contiguous()
    s_cpu, s_gpu = stoi.stoi(x, y, sr), stoi.stoi(x.cuda(), y.cuda(), sr)
    ref = score([(c[:T], d[:T]) for c, d in entries], sr, ("stoi",))["stoi"]
    assert not s_cpu.is_cuda and s_gpu.is_cuda
    assert np.array_equal(bits(s_cpu.numpy()), bits(ref)) and np.array_equal(bits(s_gpu.cpu().numpy()), bits(ref))
    assert float(E.si_sdr_speechmetrics(entries[0][0], entries[0][1])) == pytest.approx(float(host["sisdr"][0]), abs=0)


def test_errors():
    L = _lib.lib()
    h = E.metrics_handle(16000)
    x = np.zeros(100, np.float32)
    out = np.zeros(3, np.float32)

    def call(lc, ld, bits_):
        lc, ld = np.array(lc, np.int64), np.array(ld, np.int64)
        off = np.zeros(lc.size, np.int64)
        return L.dfb_metrics_compute_host(h.handle, x.ctypes.data, x.ctypes.data, 100, off.ctypes.data, lc.ctypes.data,
                                          ld.ctypes.data, lc.size, bits_, out.ctypes.data)
    assert call([50], [50], 7) == 0
    assert call([50], [49], 7) == _lib.DFB_ERR_INVALID and b"degraded" in L.dfb_last_error()
    assert call([0], [0], 7) == _lib.DFB_ERR_INVALID
    assert call([50], [50], 8) == _lib.DFB_ERR_INVALID and b"unknown metric" in L.dfb_last_error()
    assert call([50], [50], 0) == _lib.DFB_ERR_INVALID
    assert call([101], [101], 1) == _lib.DFB_ERR_INVALID
    from deepfilternet_b200.io import get_resample_params, resample_kernel
    k10, w10, og10, nw10 = resample_kernel(11025, 10000, **get_resample_params("sinc_fast"))
    k16, w16, og16, nw16 = resample_kernel(11025, 16000, **get_resample_params("sinc_fast"))
    hh = C.c_void_p()
    rc = L.dfb_metrics_create(C.byref(hh), 0, 11025, k10.data_ptr(), og10, nw10, w10, k16.data_ptr(), og16, nw16, w16)
    assert rc == _lib.DFB_ERR_UNSUPPORTED and not hh.value
    with pytest.raises(ValueError):
        E.evaluate_batch([torch.zeros(10)], [torch.zeros(11)], 16000)
    with pytest.raises(ValueError):
        E.evaluate_batch([torch.zeros(10)], [torch.zeros(10)], 11025)


def _dataset(tmp_path, sr, n=5):
    rng = np.random.default_rng(11)
    root = tmp_path / "ds"
    for sub in ("clean_testset_wav", "noisy_testset_wav"):
        (root / sub).mkdir(parents=True)
    for i in range(n):
        c, d = signal(rng, int(sr * rng.uniform(0.8, 3.0)), sr)
        save_audio(str(root / "clean_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(c), sr)
        save_audio(str(root / "noisy_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(d), sr)
    return root


def test_evaluation_loop_against_per_file(tmp_path, model_dir):
    from deepfilternet_b200.io import load_audio
    model, df_state, _, _ = init_df(os.path.join(model_dir, "DeepFilterNet3"), log_level="ERROR")
    root = _dataset(tmp_path, df_state.sr())
    cl = sorted(str(p) for p in (root / "clean_testset_wav").iterdir())
    no = sorted(str(p) for p in (root / "noisy_testset_wav").iterdir())
    saved = []
    got = E.evaluation_loop(df_state, model, cl, no, metrics=["stoi", "sisdr", "ssnr"], batch_size=2,
                            save_audio_callback=lambda fn, a: saved.append((fn, a.shape)),
                            csv_path_enh=str(tmp_path / "enh.csv"), csv_path_noisy=str(tmp_path / "noisy.csv"),
                            noisy_metric=True)
    assert list(got) == ["Noisy    STOI", "Enhanced STOI", "Noisy    SISDR", "Enhanced SISDR", "Noisy    SSNR", "Enhanced SSNR"]
    sr = df_state.sr()
    rows_e, rows_n = {}, {}
    for cf, nf in zip(cl, no):
        noisy = load_audio(nf, sr, method="sinc_fast")[0]
        clean = df_state.synthesis(df_state.analysis(load_audio(cf, sr, method="sinc_fast")[0].numpy()))[0]
        enh = enhance(model, df_state, noisy, pad=False)[0].numpy()
        nsy = df_state.synthesis(df_state.analysis(noisy.numpy()))[0]
        rows_e[os.path.basename(nf)] = {"STOI": R.stoi(clean, enh, sr)[0], "SISDR": R.si_sdr(clean, enh), "SSNR": R.ssnr(clean, enh, sr)}
        rows_n[os.path.basename(nf)] = {"STOI": R.stoi(clean, nsy, sr)[0], "SISDR": R.si_sdr(clean, nsy), "SSNR": R.ssnr(clean, nsy, sr)}
    for path, rows, prefix in ((tmp_path / "enh.csv", rows_e, "Enhanced"), (tmp_path / "noisy.csv", rows_n, "Noisy   ")):
        with open(path) as f:
            r = list(csv.reader(f))
        assert r[0] == ["filename", "STOI", "SISDR", "SSNR"]
        assert [x[0] for x in r[1:]] == [os.path.basename(p) for p in no]
        for x in r[1:]:
            for j, m in enumerate(("STOI", "SISDR", "SSNR")):
                assert close(float(x[1 + j]), rows[x[0]][m]), (path, x[0], m, x[1 + j], rows[x[0]][m])
        for m in ("STOI", "SISDR", "SSNR"):
            assert close(got[f"{prefix} {m}"], float(np.mean([v[m] for v in rows.values()])))
    assert [s[0] for s in saved] == cl
    with pytest.raises(ValueError, match="PESQ"):
        E.evaluation_loop(df_state, model, cl, no, metrics=["stoi", "composite"])


def test_cli(tmp_path, model_dir, capsys):
    m = os.path.join(model_dir, "DeepFilterNet3")
    root = _dataset(tmp_path, 48000, n=3)
    args = E.cli_parser().parse_args([str(root), "-m", m, "--csv-path-enh", str(tmp_path / "e.csv"), "--batch-size", "2",
                                      "--metrics", "sisdr", "stoi", "-o", str(tmp_path / "out"), "--log-level", "error"])
    res = E.main(args)
    assert list(res) == ["Enhanced SISDR", "Enhanced STOI"]
    printed = capsys.readouterr().out.strip().splitlines()[-1]
    assert [float(v) for v in printed.split(",")] == pytest.approx(list(res.values()))
    assert len(list(csv.reader(open(tmp_path / "e.csv")))) == 4
    assert len(os.listdir(tmp_path / "out")) == 3
