"""Device PYSTOI and ESTOI (dfb_metrics_compute's bits 128 and 256) against the float64 restatement (tests/pystoi_ref64.py)
on the device's own 10 kHz rows: counts exactly, band magnitudes and values element by element, at every rate and the
edges of pystoi's rules; the known answers of tests/golden/pystoi_ref.json (seeded weights) and, where build() unpacked
the pretrained checkpoints, of the reference's CI; the bit-exact batching invariants; the evaluation loop; refusals."""
import csv
import json
import math
import os

import numpy as np
import pytest
import torch

import pystoi_ref64 as P
from test_pystoi_host import REF, signal

pytestmark = pytest.mark.gpu

from deepfilternet_b200 import _lib, evaluation_utils as E, init_df  # noqa: E402
from deepfilternet_b200.enhance import enhance  # noqa: E402
from deepfilternet_b200.io import resample, save_audio  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OLD = ("sisdr", "stoi", "ssnr", "llr", "wss")
NEW = ("pystoi", "estoi")


def rows10(x, sr):
    """io.resample's 10 kHz row: bit for bit what the device scores."""
    return x if sr == 10000 else resample(torch.from_numpy(x).reshape(1, -1), sr, 10000)[0].numpy()


def len_for(sr, n10):
    """An input length at sr whose 10 kHz row has n10 samples (ceil(10000 T / sr))."""
    T = max(1, (n10 * sr) // 10000 - 2)
    while -(-10000 * T // sr) < n10:
        T += 1
    assert -(-10000 * T // sr) == n10
    return T


def edge_entries(rng, sr):
    """Stationary entries whose 10 kHz rows sit at pystoi's edges: no frame (256), one (257), K = 30 / 31 / 32."""
    out = []
    for n10 in (256, 257, 128 * 29 + 257, 128 * 30 + 300, 128 * 31 + 384):
        T = len_for(sr, n10)
        c = (0.1 * rng.standard_normal(T)).astype(np.float32)
        out.append((c, (0.7 * c + 0.05 * rng.standard_normal(T)).astype(np.float32)))
    return out


def batch(rng, B, sr, smin=0.03, smax=6.0):
    out = []
    while len(out) < B:
        n = max(1, int(sr * np.exp(rng.uniform(np.log(smin), np.log(smax)))))
        out.append(signal(rng, n, sr))
    return out


def score(entries, sr, metrics):
    r = E.evaluate_batch([torch.from_numpy(c) for c, _ in entries], [torch.from_numpy(d) for _, d in entries], sr, metrics)
    return {k: v.numpy() for k, v in r.items()}


def debug(entries, sr):
    """dfb_debug_metrics_pystoi: ([B][5] counts, [(X [15, nf], Y [15, nf])] per entry)."""
    h = E.metrics_handle(sr)
    lens = np.array([c.size for c, _ in entries], dtype=np.int64)
    off, n = E.packed_offsets(lens)
    xc = np.ascontiguousarray(np.concatenate([c for c, _ in entries]))
    xd = np.ascontiguousarray(np.concatenate([d for _, d in entries]))
    cnt = np.zeros((lens.size, 5), np.int64)
    cap = 2 * 15 * (n // 10 + 16)
    bands = np.zeros(cap)
    _lib.check(_lib.lib().dfb_debug_metrics_pystoi(h.handle, xc.ctypes.data, xd.ctypes.data, n, off.ctypes.data,
                                                   lens.ctypes.data, lens.size, cnt.ctypes.data, bands.ctypes.data, cap))
    out, o = [], 0
    for b in range(lens.size):
        nf = int(cnt[b, 3])
        X = bands[o:o + 15 * nf].reshape(15, nf)
        Y = bands[o + 15 * nf:o + 30 * nf].reshape(15, nf)
        out.append((X, Y))
        o += 30 * nf
    return cnt, out


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("sr,B,seed", [(8000, 1, 1), (16000, 33, 2), (44100, 17, 3), (48000, 96, 4)])
def test_element_level_against_float64(sr, B, seed):
    rng = np.random.default_rng(seed)
    entries = (edge_entries(rng, sr) + batch(rng, B, sr))[:max(B, 5)] if B > 1 else batch(rng, 1, sr)
    cnt, bands = debug(entries, sr)
    got = score(entries, sr, NEW)
    checked = 0
    for i, (c, d) in enumerate(entries):
        r = P.pystoi10(rows10(c, sr), rows10(d, sr))
        if r["margin"] < 1e-9:   # a frame energy at the 40 dB threshold: the summation order decides
            continue
        checked += 1
        assert tuple(cnt[i]) == (r["F"], r["K"], r["lc"], r["nf"], r["J"]), (i, c.size, tuple(cnt[i]))
        # both signals share one complex FFT, so a band's rounding is relative to the frame's larger signal: a silent
        # clean frame gets about 1e-16 of the degraded one's bands
        frame = np.maximum(r["X"].max(axis=0, keepdims=True, initial=0.0), r["Y"].max(axis=0, keepdims=True, initial=0.0))
        for g, e in zip(bands[i], (r["X"], r["Y"])):
            assert g.shape == e.shape
            scale = np.maximum(np.abs(e), frame)
            assert np.all(np.abs(g - e) <= 1e-12 * scale + 1e-300), (i, float(np.max(np.abs(g - e) / (scale + 1e-300))))
        for m, k in (("pystoi", "stoi"), ("estoi", "estoi")):
            if math.isnan(r[k]):
                assert math.isnan(got[m][i]), (i, m)
            else:
                assert abs(float(got[m][i]) - r[k]) <= 2e-7, (i, m, float(got[m][i]), r[k])
    assert checked >= len(entries) - 1


def test_edges_on_the_device():
    for sr in (16000, 48000):
        entries = edge_entries(np.random.default_rng(5), sr)
        cnt, _ = debug(entries, sr)
        assert [tuple(c) for c in cnt] == [(0, 0, 0, 0, 0), (1, 1, 256, 0, 0), (30, 30, 29 * 128 + 256, 29, 0),
                                           (31, 31, 30 * 128 + 256, 30, 1), (32, 32, 31 * 128 + 256, 31, 2)]
        got = score(entries, sr, NEW)
        for m in NEW:
            assert math.isnan(got[m][0])
            assert got[m][1] == got[m][2] == np.float32(1e-5)
            assert 0 < got[m][3] < 1 and 0 < got[m][4] < 1
    # silence against silence: every band row is constant (0), ESTOI's rows and columns normalise to 0, both are 0
    z = score([(np.zeros(20000, np.float32), np.zeros(20000, np.float32))], 10000, NEW)
    assert z["pystoi"][0] == 0.0 and z["estoi"][0] == 0.0


def test_seeded_known_answers(model_dir, golden_dir):
    import ref_harness as rh
    clean, noisy = (rh.read_wav(os.path.join(golden_dir, "assets", a))[0]
                    for a in ("clean_freesound_33711.wav", "noisy_snr0.wav"))
    for name, exp in REF["seeded"].items():
        model, st, _, _ = init_df(os.path.join(model_dir, name), log_level="ERROR")
        out = enhance(model, st, torch.from_numpy(noisy[None]), pad=True)[0].numpy()
        s, e = E.stoi(clean, out, 48000), E.stoi(clean, out, 48000, extended=True)
        assert abs(s - exp["stoi"]) < 1e-4 and abs(e - exp["estoi"]) < 1e-4, (name, s, e, exp)


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet2", "DeepFilterNet"])
def test_pretrained_ci_targets(name):
    """df/scripts/test_df.py's STOI known answers on the device: enhance() with the pretrained checkpoint, then stoi(),
    within the CI's 1e-4.  Needs what build() unpacks from the reference (checkpoints and full-length assets)."""
    d = os.path.join(ROOT, "models", "_ref")
    assets = [os.path.join(d, "assets", a) for a in ("clean_freesound_33711.wav", "noisy_snr0.wav")]
    if not (os.path.isdir(os.path.join(d, name)) and all(os.path.isfile(a) for a in assets)):
        pytest.skip("pretrained checkpoints not unpacked")
    import ref_harness as rh
    clean, noisy = (rh.read_wav(a)[0] for a in assets)
    model, st, _, _ = init_df(os.path.join(d, name), log_level="ERROR")
    out = enhance(model, st, torch.from_numpy(noisy[None]), pad=True)[0].numpy()
    s = E.stoi(clean, out, 48000)
    assert abs(s - REF["ci_stoi"][name]) < 1e-4, (name, s, REF["ci_stoi"][name])


@pytest.mark.parametrize("sr", [16000, 44100])
def test_bit_exact_invariants(sr):
    rng = np.random.default_rng(17)
    entries = batch(rng, 16, sr)
    allm = OLD + NEW
    base = score(entries, sr, allm)
    old_only = score(entries, sr, OLD)
    perm = rng.permutation(len(entries))
    permuted = score([entries[i] for i in perm], sr, allm)
    others = batch(np.random.default_rng(18), 20, sr)
    mixed = score(others[:9] + entries + others[9:], sr, allm)
    for m in allm:
        assert np.array_equal(bits(base[m]), bits(score(entries, sr, allm)[m]))
        assert np.array_equal(bits(base[m][perm]), bits(permuted[m]))
        assert np.array_equal(bits(base[m]), bits(mixed[m][9:9 + len(entries)]))
    for m in OLD:   # requesting the new rows changes no bit of the old ones
        assert np.array_equal(bits(base[m]), bits(old_only[m]))
    for i in (0, 7, 15):
        for subset in (("pystoi",), ("estoi",), ("estoi", "stoi"), ("sisdr", "pystoi", "wss")):
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
    dev = E.evaluate_device_ragged(xc.cuda(), xd.cuda(), [c.size for c, _ in entries], sr, NEW + ("stoi",))
    host = score(entries, sr, NEW + ("stoi",))
    for m in NEW + ("stoi",):
        assert dev[m].is_cuda and np.array_equal(bits(dev[m].cpu().numpy()), bits(host[m]))


def test_evaluation_loop_csv(tmp_path, model_dir):
    from deepfilternet_b200.io import load_audio
    model, df_state, _, _ = init_df(os.path.join(model_dir, "DeepFilterNet3"), log_level="ERROR")
    sr = df_state.sr()
    rng = np.random.default_rng(21)
    root = tmp_path / "ds"
    for sub in ("clean_testset_wav", "noisy_testset_wav"):
        (root / sub).mkdir(parents=True)
    for i in range(4):
        c, d = signal(rng, int(sr * rng.uniform(0.8, 3.0)), sr)
        save_audio(str(root / "clean_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(c), sr)
        save_audio(str(root / "noisy_testset_wav" / f"p{i:03d}.wav"), torch.from_numpy(d), sr)
    cl = sorted(str(p) for p in (root / "clean_testset_wav").iterdir())
    no = sorted(str(p) for p in (root / "noisy_testset_wav").iterdir())
    saved = []
    got = E.evaluation_loop(df_state, model, cl, no, metrics=["pystoi", "estoi"], batch_size=3,
                            save_audio_callback=lambda fn, a: saved.append(a[0].numpy().copy()),
                            csv_path_enh=str(tmp_path / "enh.csv"))
    assert list(got) == ["Enhanced PYSTOI", "Enhanced ESTOI"]
    clean = [df_state.synthesis(df_state.analysis(load_audio(f, sr, method="sinc_fast")[0].numpy()))[0] for f in cl]
    exp = score([(np.ascontiguousarray(c, np.float32), e) for c, e in zip(clean, saved)], sr, NEW)
    with open(tmp_path / "enh.csv") as f:
        r = list(csv.reader(f))
    assert r[0] == ["filename", "PYSTOI", "ESTOI"]
    for j, x in enumerate(r[1:]):
        assert x[0] == os.path.basename(no[j])
        assert float(x[1]) == float(exp["pystoi"][j]) and float(x[2]) == float(exp["estoi"][j])
    assert got["Enhanced PYSTOI"] == pytest.approx(float(np.mean(exp["pystoi"].astype(np.float64))))


def test_refusals():
    L = _lib.lib()
    h = E.metrics_handle(16000)
    x = np.zeros(1000, np.float32)
    out = np.zeros(4, np.float32)
    lens, off = np.array([1000], np.int64), np.zeros(1, np.int64)
    for b_ in (8, 64, 512, 128 | 8, 256 | 64, 128 | 1024):
        assert L.dfb_metrics_compute_host(h.handle, x.ctypes.data, x.ctypes.data, 1000, off.ctypes.data, lens.ctypes.data,
                                          lens.ctypes.data, 1, b_, out.ctypes.data) == _lib.DFB_ERR_INVALID
    assert L.dfb_metrics_compute_host(h.handle, x.ctypes.data, x.ctypes.data, 1000, off.ctypes.data, lens.ctypes.data,
                                      lens.ctypes.data, 1, 128 | 256, out.ctypes.data) == 0
    cnt = np.zeros(5, np.int64)
    assert L.dfb_debug_metrics_pystoi(h.handle, x.ctypes.data, x.ctypes.data, 1000, off.ctypes.data, lens.ctypes.data, 1,
                                      cnt.ctypes.data, np.zeros(1).ctypes.data, 1) == _lib.DFB_ERR_INVALID   # 30 nf bands
    with pytest.raises(ValueError):
        E.stoi(np.zeros((2, 100), np.float32), np.zeros((2, 100), np.float32), 16000)
