"""GPU: streaming handles at 8 - 44.1 kHz (DfStream(sr=...), dfb_stream_set_sample_rate).  The resamplers alone are bit for
bit io.resample of the concatenated signal, delayed by D_r / E_r; a session equals the composition of include/dfb200.h:
io.resample up, an unchanged 48 kHz handle fed the same call sizes plus one hop and flushed, io.resample down.  Slots,
linked groups, per-slot settings, LSNR rows and stage gating behave as at 48 kHz; a 48 kHz handle runs no new kernel."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, io, libdf
from deepfilternet_b200.streaming import SLOT_CLOSING, SLOT_FREE, SLOT_OPEN, STREAM_RATES, rate_delays, rate_taps
from deepfilternet_b200.weights import random_state_dict
from test_gpu_slots import cfg_of, rms, schedule

TOL = 1e-6          # RMS, as the streaming tests
SIZES = [1, 2, 3, 7, 40]


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_models = {}


def model_of(kind, st, **kw):
    key = (kind, tuple(sorted(kw.items())))
    if key not in _models:
        cfg = cfg_of(kind, **kw)
        _models[key] = DfNet(cfg, random_state_dict(cfg, seed=191), st)
    return _models[key]


def delays(sr):
    (_, wu, ou, nu), (_, wd, od, nd) = rate_taps(sr)
    return rate_delays(ou, nu, wu, od, nd, wd)


# ------------------------------------------------------------------------------------------ resamplers alone ----
@pytest.mark.parametrize("sr", STREAM_RATES)
@pytest.mark.parametrize("up", [1, 0])
def test_resamplers_alone_are_io_resample(sr, up):
    (ku, wu, ou, nu), (kd, wd, od, nd) = rate_taps(sr)
    taps, og, nw, width = (ku, ou, nu, wu) if up else (kd, od, nd, wd)
    D, E, _ = delays(sr)
    z = D if up else E
    hin, hout = (sr // 100, 480) if up else (480, sr // 100)
    calls = np.array(SIZES, np.int64)
    H = int(calls.sum())
    g = torch.Generator().manual_seed(sr + up)
    x = torch.randn((3, H * hin), generator=g) * 0.3
    out = torch.full((3, H * hout), float("nan"), device="cuda")
    xd, td = x.cuda(), taps.cuda()
    _lib.check(_lib.lib().dfb_debug_resample_stream(up, sr, td.data_ptr(), og, nw, width, xd.data_ptr(), 3,
                                                    calls.ctypes.data_as(C.POINTER(C.c_int64)), len(calls), out.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
    out = out.cpu()
    ref = io.resample(x, sr, 48000) if up else io.resample(x, 48000, sr)
    assert out[:, :z].abs().max().item() == 0
    assert torch.equal(out[:, z:], ref[:, :H * hout - z]), (sr, up, (out[:, z:] - ref[:, :H * hout - z]).abs().max())


# ------------------------------------------------------------------------------------------ the composition ----
def composition(model, st, x, sizes, sr, lsnr=False, make=None, **kw):
    """Output (and LSNR rows) of the session x [B, a1 * h_r] in `sizes` per include/dfb200.h: D zeros + io.resample up, a
    48 kHz handle fed the same calls, one more hop and its flush, then E zeros + io.resample down, cropped."""
    hr, a1 = sr // 100, sum(sizes)
    D, E, _ = delays(sr)
    s48 = make() if make else DfStream(model, st, batch=x.shape[0], **kw)
    L = s48.latency_frames
    up = io.resample(torch.cat([x, torch.zeros(x.shape[0], hr)], 1), sr, 48000)
    u = torch.cat([torch.zeros(x.shape[0], D), up], 1)[:, :(a1 + 1) * 480]
    outs, ls, pos = [], [], 0
    for n in list(sizes) + [1]:
        y = s48.process(u[:, pos * 480:(pos + n) * 480], return_lsnr=lsnr)
        outs.append(y[0] if lsnr else y)
        if lsnr:
            ls.append(y[1])
        pos += n
    y = s48.flush(return_lsnr=lsnr)
    outs.append(y[0] if lsnr else y)
    if lsnr:
        ls.append(y[1])
    y48 = torch.cat(outs, 1)
    z = torch.cat([torch.zeros(x.shape[0], E), io.resample(y48, 48000, sr)], 1)[:, :(a1 + L + 1) * hr]
    return (z, torch.cat(ls, 1)) if lsnr else z


def run_rate(s, x, sizes, lsnr=False):
    hr, outs, ls, pos = s.hop, [], [], 0
    for i, n in enumerate(sizes):
        chunk = x[:, pos * hr:(pos + n) * hr]
        y = s.process(chunk.cuda() if i % 2 else chunk, return_lsnr=lsnr)
        outs.append((y[0] if lsnr else y).cpu())
        if lsnr:
            ls.append(y[1].cpu())
        pos += n
    y = s.flush(return_lsnr=lsnr)
    outs.append(y[0] if lsnr else y)
    if lsnr:
        ls.append(y[1])
    return (torch.cat(outs, 1), torch.cat(ls, 1)) if lsnr else torch.cat(outs, 1)


def assert_close(got, ref, sr, what=""):
    edge = sr // 10     # first / last 100 ms on their own
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    for b in range(got.shape[0]):
        assert rms(got[b], ref[b]) < TOL, (what, b, rms(got[b], ref[b]))
        assert rms(got[b, :edge], ref[b, :edge]) < TOL and rms(got[b, -edge:], ref[b, -edge:]) < TOL, (what, b)


def assert_lsnr(got, ref):
    assert got.shape == ref.shape and torch.equal(got.isnan(), ref.isnan()), (got, ref)
    ok = ~ref.isnan()
    assert (got[ok] - ref[ok]).abs().max().item() < 1e-3 if ok.any() else True


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
@pytest.mark.parametrize("sr", [8000, 16000, 44100])
def test_sessions_equal_the_composition(st, kind, sr):
    model = model_of(kind, st)
    rng = np.random.default_rng(sr + len(kind))
    sizes = [int(v) for v in rng.choice(SIZES, 9)]
    hr, a1 = sr // 100, sum(sizes)
    x = synth_audio(2, a1 * hr, seed=sr, sr=sr)
    s = DfStream(model, st, batch=2, sr=sr)
    L = {"dfn3": 2, "dfn2": 4, "ll": 0}[kind]
    D, E, delay = delays(sr)
    assert (s.sr, s.hop, s.latency_frames, s.latency_samples) == (sr, hr, L + 1, delay)
    got = run_rate(s, x, sizes)
    assert got.shape == (2, (a1 + L + 1) * hr)
    assert_close(got, composition(model, st, x, sizes, sr), sr, (kind, sr, sizes))
    assert np.array_equal(s.slot_states(), [SLOT_FREE] * 2)


# ------------------------------------------------------------------------------------------ slot server ----
def test_slot_server_at_16k(st):
    """test_gpu_slots's schedule on one 16 kHz handle of 8 slots: every session equals a fresh single-slot 16 kHz handle fed
    the same calls and flushed; free slots and closing slots past their L + 1 drain hops return exact zeros."""
    sr, B = 16000, 8
    hr = sr // 100
    model = model_of("dfn3", st)
    calls = schedule(seed=17, n_random=16)
    s = DfStream(model, st, batch=B, sr=sr)
    lat = s.latency_frames
    total = sum(n for _, _, n in calls) + 1
    sessions, live, seed = [], {}, 3000

    def new_session(b):
        nonlocal seed
        ses = dict(slot=b, src=synth_audio(1, total * hr, seed=seed, sr=sr)[0], sizes=[], outs=[], closing=False, left=0,
                   dropped=False)
        seed += 1
        live[b] = ses
        sessions.append(ses)

    for b in range(B):
        new_session(b)
    noise = torch.Generator().manual_seed(11)
    for i in range(len(calls) + 1):
        flush = i == len(calls)
        if not flush:
            opens, closes, n = calls[i]
            if closes:
                s.close(closes)
                for b in closes:
                    if b in live and not live[b]["closing"]:
                        live[b]["closing"], live[b]["left"] = True, lat
            if opens:
                s.open(opens)
                for b in opens:
                    if b in live:
                        live[b]["dropped"] = True
                    new_session(b)
            want = [SLOT_FREE if b not in live else (SLOT_CLOSING if live[b]["closing"] else SLOT_OPEN) for b in range(B)]
            assert np.array_equal(s.slot_states(), want), (i, s.slot_states(), want)
            x = torch.randn((B, n * hr), generator=noise) * 0.3
            for b, ses in live.items():
                if not ses["closing"]:
                    pos = sum(ses["sizes"])
                    x[b] = ses["src"][pos * hr:(pos + n) * hr]
                    ses["sizes"].append(n)
            y = s.process(x.cuda() if i % 2 else x).cpu()
        else:
            for ses in live.values():
                if not ses["closing"]:
                    ses["closing"], ses["left"] = True, lat
            y = s.flush()
            n = lat
        used = set()
        for b, ses in list(live.items()):
            row = y[b]
            if not ses["closing"]:
                ses["outs"].append(row)
            else:
                k = min(n, ses["left"])
                ses["outs"].append(row[:k * hr])
                assert k == n or row[k * hr:].abs().max().item() == 0, (i, b)
                ses["left"] -= k
                if ses["left"] == 0:
                    del live[b]
            used.add(b)
        for b in range(B):
            if b not in used:
                assert y[b].abs().max().item() == 0, ("free slot output", i, b)
    assert not live and np.array_equal(s.slot_states(), np.zeros(B))
    checked = 0
    for ses in sessions:
        if not ses["sizes"]:
            continue
        got = torch.cat(ses["outs"])
        r = DfStream(model, st, batch=1, sr=sr)
        ref = run_rate(r, ses["src"][None, :sum(ses["sizes"]) * hr], ses["sizes"])[0]
        if ses["dropped"]:
            ref = ref[:got.numel()]
        assert got.shape == ref.shape, (ses["slot"], got.shape, ref.shape)
        assert rms(got, ref) < TOL and rms(got[:sr // 10], ref[:sr // 10]) < TOL and rms(got[-sr // 10:], ref[-sr // 10:]) < TOL
        checked += 1
    assert checked >= 12 and any(ses["dropped"] for ses in sessions)


def test_only_live_rows_are_computed_at_16k(st):
    sr, B = 16000, 32
    hr = sr // 100
    model = model_of("dfn3", st)
    s = DfStream(model, st, batch=B, sr=sr)
    x = synth_audio(B, 12 * hr, seed=4, sr=sr)
    s.process(x)
    s.close([b for b in range(B) if b not in (3, 20)])
    s.process(x[:, :hr * s.latency_frames])           # the tails, L + 1 hops, come out
    assert (s.slot_states() == SLOT_OPEN).sum() == 2 and (s.slot_states() == SLOT_FREE).sum() == B - 2
    y = s.process(x[:, :3 * hr])
    buf = np.zeros(B * 64 * 1024, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, b"emb", buf.ctypes.data, buf.size)
    assert got == 2 * (8 + 3) * (model.cfg.nb_erb // 4 * 64)
    assert y[[b for b in range(B) if b not in (3, 20)]].abs().max() == 0 and y[[3, 20]].abs().max() > 0


# ------------------------------------------------------------------------------------------ groups and settings ----
def test_linked_group_and_slot_settings_at_16k(st):
    """One 16 kHz handle: a mean-linked session of 2 channels (open_linked), one slot with its own attenuation limit and
    one with its own post-filter beta, all with LSNR rows; each equals the composition with the same settings at 48 kHz."""
    sr = 16000
    hr = sr // 100
    model = model_of("dfn3", st)
    sizes = [3, 1, 7, 2, 40, 1]
    a1 = sum(sizes)
    x = synth_audio(4, a1 * hr, seed=21, sr=sr)
    s = DfStream(model, st, batch=4, reduce_mask="mean", sr=sr)
    s.open_linked([0, 1])
    s.set_atten_lim(12.0, [2])
    s.set_post_filter_beta(0.03, [3])
    got, gl = run_rate(s, x, sizes, lsnr=True)

    def one(make, rows):
        return composition(model, st, x[rows], sizes, sr, lsnr=True, make=make)

    def with_setting(fn):
        def make():
            r = DfStream(model, st, batch=1)
            fn(r)
            return r
        return make

    ref = [one(lambda: DfStream(model, st, batch=2, channels=2, reduce_mask="mean"), [0, 1]),
           one(with_setting(lambda r: r.set_atten_lim(12.0, [0])), [2]),
           one(with_setting(lambda r: r.set_post_filter_beta(0.03, [0])), [3])]
    assert_close(got, torch.cat([r[0] for r in ref]), sr, "linked / settings")
    assert_lsnr(gl, torch.cat([r[1] for r in ref]))
    assert not torch.equal(got[2], got[3])


@pytest.mark.parametrize("sr", [16000, 44100])
def test_stage_gating_and_lsnr_at_other_rates(st, sr):
    model = model_of("dfn3", st)
    sizes = [2, 7, 1, 40]
    x = synth_audio(3, sum(sizes) * (sr // 100), seed=31, sr=sr)
    x[1] *= 30.0                                             # a loud row: other stages than 1
    s = DfStream(model, st, batch=3, sr=sr)
    s.set_lsnr_thresholds(-5.0, 20.0, 10.0)

    def make():
        r = DfStream(model, st, batch=3)
        r.set_lsnr_thresholds(-5.0, 20.0, 10.0)
        return r

    got, gl = run_rate(s, x, sizes, lsnr=True)
    ref, rl = composition(model, st, x, sizes, sr, lsnr=True, make=make)
    assert_close(got, ref, sr, "gating")
    assert_lsnr(gl, rl)
    assert gl[:, :s.latency_frames - 1].isnan().all()


# ------------------------------------------------------------------------------------------ argument checks ----
def test_rate_setting_rules(st):
    model = model_of("dfn3", st)
    s = DfStream(model, st, batch=2, sr=16000)
    x = synth_audio(2, 4 * 160, seed=1, sr=16000)
    s.process(x)
    for sr in (8000, 48000):                                 # after the first frame
        with pytest.raises(_lib.DfbError) as e:
            s.set_sample_rate(sr)
        assert e.value.code == _lib.DFB_ERR_INVALID
    assert s.hop == 160 and s.process(x).shape == x.shape    # still usable, still at 16 kHz
    s.reset()
    assert s.hop == int(_lib.lib().dfb_stream_frame_length(s._h)) == 160   # the rate survives a reset
    s.close([1])                                             # after a slot operation
    with pytest.raises(_lib.DfbError) as e:
        s.set_sample_rate(8000)
    assert e.value.code == _lib.DFB_ERR_INVALID
    s.reset()
    s.set_sample_rate(8000)
    assert (s.hop, s.latency_samples) == (80, delays(8000)[2])
    s.set_sample_rate(48000)
    assert (s.hop, s.latency_frames, s.latency_samples) == (480, 2, 0)
    L = _lib.lib()
    (ku, wu, ou, nu), (kd, wd, od, nd) = rate_taps(16000)
    for bad in (11025, 96000, 0):
        assert L.dfb_stream_set_sample_rate(s._h, bad, ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd) == _lib.DFB_ERR_UNSUPPORTED
    # taps of another rate
    assert L.dfb_stream_set_sample_rate(s._h, 8000, ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd) == _lib.DFB_ERR_INVALID
    spec = DfStream(model, st, batch=2, spectral=True)
    assert L.dfb_stream_set_sample_rate(spec._h, 16000, ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd) == _lib.DFB_ERR_INVALID
    with pytest.raises(_lib.DfbError):
        DfStream(model, st, batch=2, spectral=True, sr=16000)
    with pytest.raises(_lib.DfbError):
        DfStream(model, st, batch=2, sr=22050)
    for sr in STREAM_RATES:
        r = DfStream(model, st, batch=1, sr=sr)
        assert (r.hop, r.latency_frames, r.latency_samples) == (sr // 100, 3, delays(sr)[2])
        assert r.latency_samples < r.hop


# ------------------------------------------------------------------------------------------ 48 kHz untouched ----
def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages()}


def test_48k_handles_run_no_new_kernel(st):
    model = model_of("dfn3", st)
    x = synth_audio(2, 20 * 480, seed=5)
    outs = []
    names = []
    for kw in ({}, {"sr": 48000}):
        s = DfStream(model, st, batch=2, **kw)
        res = []
        names.append(kernel_names(lambda: res.extend([s.process(x[:, :3 * 480].cuda()).cpu(), s.process(x[:, 3 * 480:]), s.flush()])))
        outs.append(torch.cat(res, 1))
    assert torch.equal(outs[0], outs[1])
    for n in names:
        assert any("k_apply_synthesis" in k for k in n) and not any("k_resample" in k for k in n), n
    s = DfStream(model, st, batch=2, sr=16000)
    n16 = kernel_names(lambda: s.process(synth_audio(2, 3 * 160, seed=5, sr=16000).cuda()))
    assert any("k_resample_up" in k for k in n16) and any("k_resample_down" in k for k in n16)
