"""GPU: mixed-rate streaming handles (DfStream(slot_rates=...), dfb_stream_add_slot_rate), whose slots each run at their own
rate in one pass through the slot path.  The resamplers with mixed rows are bit for bit io.resample of each row (48 kHz
rows: copies); every session equals a handle at its own rate; groups, settings, LSNR rows and gating behave as there; a
handle whose slots all run at 48 kHz computes what a 48 kHz handle does.  No test here opens a profiler session: kernel
launches are counted by the library (dfb_kernel_launches)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests_common import synth_audio

from deepfilternet_b200 import DfStream, _lib, io, libdf
from deepfilternet_b200.streaming import MODEL_SR, SLOT_CLOSING, SLOT_FREE, SLOT_OPEN, STREAM_RATES, rate_delays, rate_taps
from test_gpu_slots import rms, schedule
from test_gpu_stream_rates import assert_lsnr, model_of, run_rate

TOL = 1e-6          # RMS, as the streaming tests
SIZES = [1, 2, 3, 7, 40]
ALL = (MODEL_SR,) + STREAM_RATES
HOP = 480


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


def delays(sr):
    (_, wu, ou, nu), (_, wd, od, nd) = rate_taps(sr)
    return rate_delays(ou, nu, wu, od, nd, wd)


def single(model, st, sr, batch=1, **kw):
    """A handle at one rate: the reference of a session at sr."""
    return DfStream(model, st, batch=batch, **kw) if sr == MODEL_SR else DfStream(model, st, batch=batch, sr=sr, **kw)


def launches(fn):
    """kernels the library launches in fn()"""
    n0 = _lib.lib().dfb_kernel_launches()
    fn()
    return _lib.lib().dfb_kernel_launches() - n0


def close_enough(got, ref, sr, what=""):
    edge = sr // 10     # first / last 100 ms on their own
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert rms(got, ref) < TOL, (what, rms(got, ref))
    assert rms(got[:edge], ref[:edge]) < TOL and rms(got[-edge:], ref[-edge:]) < TOL, what


# ------------------------------------------------------------------------------------------ resamplers alone ----
@pytest.mark.parametrize("up", [1, 0])
def test_resamplers_with_mixed_rows_are_io_resample(st, up):
    model = model_of("dfn3", st)
    s = DfStream(model, st, batch=1, slot_rates=STREAM_RATES)
    rates = np.array(ALL * 2, np.int32)                 # every rate, 48 kHz included, twice in one launch
    R = len(rates)
    calls = np.array(SIZES, np.int64)
    H = int(calls.sum())
    g = torch.Generator().manual_seed(17 + up)
    x = torch.randn((R, H * HOP), generator=g) * 0.3
    out = torch.full((R, H * HOP), float("nan"), device="cuda")
    xd = x.cuda()
    _lib.check(_lib.lib().dfb_debug_resample_slots(up, s._h, rates.ctypes.data_as(C.POINTER(C.c_int32)), xd.data_ptr(), R,
                                                   calls.ctypes.data_as(C.POINTER(C.c_int64)), len(calls), out.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream))
    out = out.cpu()
    for c, sr in enumerate(rates.tolist()):
        if sr == MODEL_SR:
            assert torch.equal(out[c], x[c]), c
            continue
        hin, hout = (sr // 100, HOP) if up else (HOP, sr // 100)
        D, E, _ = delays(sr)
        z = D if up else E
        ref = io.resample(x[c:c + 1, :H * hin], sr, MODEL_SR) if up else io.resample(x[c:c + 1, :H * hin], MODEL_SR, sr)
        assert out[c, :z].abs().max().item() == 0
        assert torch.equal(out[c, z:H * hout], ref[0, :H * hout - z]), (sr, up)
        assert out[c, H * hout:].abs().max().item() == 0 if H * hout < H * HOP else True


# ------------------------------------------------------------------------------------------ slot server ----
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_mixed_slot_server(st, kind):
    """test_gpu_slots's schedule on one 8-slot handle with every rate registered, the sessions opened at the rates of a
    cycle over all seven: each equals a fresh single-slot handle at its rate, rows past a session's samples, free slots
    and closing slots past their own drain are exact zeros, and slot_rates / slot_states follow the schedule."""
    B = 8
    model = model_of(kind, st)
    calls = schedule(seed=23, n_random=16)
    s = DfStream(model, st, batch=B, slot_rates=STREAM_RATES)
    L = {"dfn3": 2, "dfn2": 4, "ll": 0}[kind]
    assert s.latency_frames == L + 1 and s.hop == HOP
    for sr in ALL:
        ref = single(model, st, sr)
        assert s.rate_latency(sr) == (ref.latency_frames, ref.latency_samples)
    total = sum(n for _, _, n in calls) + 1
    sessions, live, seed, cyc = [], {}, 5000, [0]

    def new_session(b):
        nonlocal seed
        sr = ALL[cyc[0] % len(ALL)]
        cyc[0] += 1
        ses = dict(slot=b, sr=sr, src=synth_audio(1, total * sr // 100, seed=seed, sr=sr)[0], sizes=[], outs=[],
                   closing=False, left=0, dropped=False)
        seed += 1
        live[b] = ses
        sessions.append(ses)
        return sr

    def drain(ses):
        return L if ses["sr"] == MODEL_SR else L + 1

    def end(b):
        live[b]["closing"], live[b]["left"] = True, drain(live[b])
        if live[b]["left"] == 0:            # a 48 kHz slot without look-ahead is free at once
            del live[b]

    def check_states(when):
        want = [SLOT_FREE if b not in live else (SLOT_CLOSING if live[b]["closing"] else SLOT_OPEN) for b in range(B)]
        assert np.array_equal(s.slot_states(), want), (when, s.slot_states(), want)
        assert np.array_equal(s.slot_rates(), [live[b]["sr"] if b in live else 0 for b in range(B)]), (when, s.slot_rates())

    assert np.array_equal(s.slot_rates(), [MODEL_SR] * B)
    for b in range(B):                      # the sessions at creation are re-opened at the cycle's rates
        s.open([b], sr=new_session(b))
    noise = torch.Generator().manual_seed(13)
    for i in range(len(calls) + 1):
        flush = i == len(calls)
        if not flush:
            opens, closes, n = calls[i]
            if closes:
                s.close(closes)
                for b in closes:
                    if b in live and not live[b]["closing"]:
                        end(b)
            for b in opens:                 # one call per rate, as a server opens calls
                if b in live:
                    live[b]["dropped"] = True
                s.open([b], sr=new_session(b))
            check_states(("before", i))
            x = torch.randn((B, n * HOP), generator=noise) * 0.3     # what a row ignores is noise
            for b, ses in live.items():
                if not ses["closing"]:
                    hr, pos = ses["sr"] // 100, sum(ses["sizes"])
                    x[b, :n * hr] = ses["src"][pos * hr:(pos + n) * hr]
                    ses["sizes"].append(n)
            y = s.process(x.cuda() if i % 2 else x).cpu()
        else:
            for b in list(live):
                if not live[b]["closing"]:
                    end(b)
            y = s.flush()
            n = L + 1
        assert y.shape == (B, n * HOP)
        used = set()
        for b, ses in list(live.items()):
            hr = ses["sr"] // 100
            k = min(n, ses["left"]) if ses["closing"] else n
            ses["outs"].append(y[b, :k * hr])
            assert y[b, k * hr:].abs().max().item() == 0 if k * hr < n * HOP else True, ("past the row's samples", i, b)
            if ses["closing"]:
                ses["left"] -= k
                if ses["left"] == 0:
                    del live[b]
            used.add(b)
        for b in range(B):
            if b not in used:
                assert y[b].abs().max().item() == 0, ("free slot output", i, b)
        check_states(("after", i))
    assert not live and np.array_equal(s.slot_states(), np.zeros(B))
    checked = set()
    for ses in sessions:
        if not ses["sizes"]:
            continue
        sr, hr = ses["sr"], ses["sr"] // 100
        got = torch.cat(ses["outs"])
        ref = run_rate(single(model, st, sr), ses["src"][None, :sum(ses["sizes"]) * hr], ses["sizes"])[0]
        if ses["dropped"]:
            ref = ref[:got.numel()]
        close_enough(got, ref, sr, (kind, ses["slot"], sr, ses["sizes"]))
        checked.add(sr)
    assert checked == set(ALL) and any(ses["dropped"] for ses in sessions)


# ------------------------------------------------------------------------------------------ groups and settings ----
def test_groups_settings_lsnr_and_gating_on_one_mixed_handle(st):
    """A mean-linked 16 kHz pair, an 8 kHz slot with its own attenuation limit, a 44.1 kHz slot with its own post-filter
    beta and a 48 kHz slot, stage gating on and LSNR rows: each session equals its own handle with the same settings."""
    model = model_of("dfn3", st)
    sizes = [3, 1, 7, 2, 40, 1]
    a1 = sum(sizes)
    th = (-5.0, 20.0, 10.0)
    s = DfStream(model, st, batch=5, reduce_mask="mean", slot_rates=(8000, 16000, 44100))
    s.set_lsnr_thresholds(*th)
    s.open_linked([0, 1], sr=16000)
    s.open([2], sr=8000)
    s.open([3], sr=44100)
    s.set_atten_lim(12.0, [2])
    s.set_post_filter_beta(0.03, [3])
    rates = [16000, 16000, 8000, 44100, MODEL_SR]
    assert np.array_equal(s.slot_rates(), rates)
    src = [synth_audio(2, a1 * 160, seed=41, sr=16000)] + [synth_audio(1, a1 * (r // 100), seed=42 + i, sr=r)
                                                             for i, r in enumerate(rates[2:])]
    src[2][0] *= 30.0                                         # a loud row: other stages than 1
    rows = [src[0][0], src[0][1], src[1][0], src[2][0], src[3][0]]
    L = s.latency_frames - 1
    outs, ls, pos = [[] for _ in rows], [[] for _ in rows], 0
    for i, n in enumerate(sizes + [None]):
        if n is None:
            y, l = s.flush(return_lsnr=True)
            n = L + 1
        else:
            x = torch.zeros((5, n * HOP))
            for b, r in enumerate(rates):
                x[b, :n * (r // 100)] = rows[b][pos * (r // 100):(pos + n) * (r // 100)]
            y, l = s.process(x.cuda() if i % 2 else x, return_lsnr=True)
            y, l = y.cpu(), l.cpu()
            pos += n
        for b, r in enumerate(rates):
            k = n - 1 if (r == MODEL_SR and i == len(sizes)) else n   # a 48 kHz slot drains for L hops
            outs[b].append(y[b, :k * (r // 100)])
            ls[b].append(l[b, :k])
            assert y[b, k * (r // 100):].abs().max().item() == 0 if k * (r // 100) < n * HOP else True, (i, b)
            assert l[b, k:].isnan().all()

    def ref(rows_x, sr, batch=1, setup=None, **kw):
        r = single(model, st, sr, batch=batch, **kw)
        r.set_lsnr_thresholds(*th)
        if setup:
            setup(r)
        return run_rate(r, rows_x, sizes, lsnr=True)

    refs = [ref(src[0], 16000, batch=2, channels=2, reduce_mask="mean"),
            ref(src[1], 8000, setup=lambda r: r.set_atten_lim(12.0, [0])),
            ref(src[2], 44100, setup=lambda r: r.set_post_filter_beta(0.03, [0])),
            ref(src[3], MODEL_SR)]
    ref_rows = [(refs[0][0][0], refs[0][1][0]), (refs[0][0][1], refs[0][1][1])] + [(r[0][0], r[1][0]) for r in refs[1:]]
    for b, r in enumerate(rates):
        close_enough(torch.cat(outs[b]), ref_rows[b][0], r, ("row", b, r))
        assert_lsnr(torch.cat(ls[b]), ref_rows[b][1])


def test_only_live_rows_are_computed_at_three_rates(st):
    B = 32
    model = model_of("dfn3", st)
    s = DfStream(model, st, batch=B, slot_rates=(8000, 16000, 44100))
    keep = {3: 8000, 20: 16000, 27: 44100}
    for b, r in keep.items():
        s.open([b], sr=r)
    x = synth_audio(B, 12 * HOP, seed=4)
    s.process(x)
    s.close([b for b in range(B) if b not in keep])
    s.process(x[:, :HOP * s.latency_frames])            # the tails, L or L + 1 hops, come out
    assert (s.slot_states() == SLOT_OPEN).sum() == 3 and (s.slot_states() == SLOT_FREE).sum() == B - 3
    y = s.process(x[:, :3 * HOP])
    buf = np.zeros(B * 64 * 1024, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, b"emb", buf.ctypes.data, buf.size)
    assert got == 3 * (8 + 3) * (model.cfg.nb_erb // 4 * 64)
    rest = [b for b in range(B) if b not in keep]
    assert y[rest].abs().max() == 0
    for b, r in keep.items():
        assert y[b, :3 * r // 100].abs().max() > 0 and y[b, 3 * r // 100:].abs().max() == 0


# ------------------------------------------------------------------------------------------ 48 kHz untouched ----
@pytest.mark.parametrize("kind", ["dfn3", "ll"])
def test_a_mixed_handle_at_48k_is_a_48k_handle(st, kind):
    model = model_of(kind, st)
    sizes = [3, 17, 1, 40, 2]
    x = synth_audio(3, sum(sizes) * HOP, seed=8)
    plain = DfStream(model, st, batch=3)
    mixed = DfStream(model, st, batch=3, slot_rates=(8000, 44100))
    L = plain.latency_frames
    assert mixed.latency_frames == L + 1 and mixed.latency_samples == 0
    pos = 0
    for i, n in enumerate(sizes):
        chunk = x[:, pos * HOP:(pos + n) * HOP]
        if i == 3:                                      # a close and a re-open on the way
            for h in (plain, mixed):
                h.close([1])
        if i == 4:
            for h in (plain, mixed):
                h.open([1])
        a, b = plain.process(chunk.cuda()).cpu(), mixed.process(chunk.cuda()).cpu()
        assert torch.equal(a, b), (kind, i)
        pos += n
    a, b = plain.flush(), mixed.flush()
    assert b.shape == (3, (L + 1) * HOP)
    assert rms(a, b[:, :L * HOP]) < TOL and b[:, L * HOP:].abs().max().item() == 0
    # The resamplers' launches, counted by the library rather than by a profiler session, whose late records could reach
    # a later test's session: a call of a mixed-rate handle launches what the same call of a 48 kHz handle launches, and
    # k_resample_up and k_resample_down once each.
    plain, m = DfStream(model, st, batch=2), DfStream(model, st, batch=2, slot_rates=(16000,))
    plain.open([0])
    m.open([0], sr=16000)
    x2 = x[:2, :2 * HOP].cuda()
    for h in (plain, m):                                # the opens' row moves and table uploads
        h.process(x2)
    assert launches(lambda: m.process(x2)) == launches(lambda: plain.process(x2)) + 2


# ------------------------------------------------------------------------------------------ rules ----
def test_slot_rate_rules(st):
    model = model_of("dfn3", st)
    L = _lib.lib()
    (ku, wu, ou, nu), (kd, wd, od, nd) = rate_taps(16000)
    (k8, w8, o8, n8), (k8d, w8d, o8d, n8d) = rate_taps(8000)
    one = np.array([0], np.int64)
    p1 = one.ctypes.data_as(C.POINTER(C.c_int64))

    def add(s, sr, taps=None):
        t = taps or ((ku, wu, ou, nu), (kd, wd, od, nd))
        (a, b, c, d), (e, f, g, h) = t
        return L.dfb_stream_add_slot_rate(s._h, sr, a.data_ptr(), c, d, b, e.data_ptr(), g, h, f)

    s = DfStream(model, st, batch=2, slot_rates=(8000, 16000))
    assert s.registered_rates == (8000, 16000) and s.sr == MODEL_SR
    assert add(s, 16000) == 0                               # twice is once
    assert add(s, 8000) == _lib.DFB_ERR_INVALID             # 16 kHz taps for 8 kHz
    assert add(s, 22050) == _lib.DFB_ERR_UNSUPPORTED
    for sr in (12000, 44100):                               # not registered
        assert L.dfb_stream_open_slots_at(s._h, p1, 1, sr) == _lib.DFB_ERR_INVALID
    assert L.dfb_stream_open_slots_at(s._h, p1, 1, 22050) == _lib.DFB_ERR_UNSUPPORTED
    assert L.dfb_stream_open_linked_at(s._h, p1, 1, 11025) == _lib.DFB_ERR_UNSUPPORTED
    assert L.dfb_stream_set_sample_rate(s._h, 16000, ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd) == _lib.DFB_ERR_INVALID
    s.set_sample_rate(MODEL_SR)                             # changes nothing
    assert s.latency_frames == 3 and s.hop == HOP
    s.open([0], sr=16000)
    assert add(s, 44100) == _lib.DFB_ERR_INVALID             # after a slot operation
    s.process(synth_audio(2, 2 * HOP, seed=3))
    assert add(s, 44100) == _lib.DFB_ERR_INVALID             # after the first frame
    s.reset()                                               # registrations survive, every slot at 48 kHz again
    assert np.array_equal(s.slot_rates(), [MODEL_SR] * 2) and s.latency_frames == 3
    s.open_linked([0, 1], sr=8000)
    assert np.array_equal(s.slot_rates(), [8000, 8000]) and np.array_equal(s.slot_groups(), [0, 0])
    with pytest.raises(_lib.DfbError):                      # a group opens as a unit
        s.open([1], sr=16000)
    s.flush()
    assert np.array_equal(s.slot_rates(), [0, 0])
    plain, at16 = DfStream(model, st, batch=2), DfStream(model, st, batch=2, sr=16000)
    for h in (plain, at16):
        for sr in (MODEL_SR, 16000):                        # no registered rates
            assert L.dfb_stream_open_slots_at(h._h, p1, 1, sr) == _lib.DFB_ERR_INVALID
    assert add(at16, 8000, ((k8, w8, o8, n8), (k8d, w8d, o8d, n8d))) == _lib.DFB_ERR_INVALID
    with pytest.raises(_lib.DfbError):
        DfStream(model, st, batch=2, sr=16000, slot_rates=(8000,))
    spec = DfStream(model, st, batch=2, spectral=True)
    assert add(spec, 16000) == _lib.DFB_ERR_INVALID
    with pytest.raises(_lib.DfbError):
        DfStream(model, st, batch=2, spectral=True, slot_rates=(16000,))
    for sr in STREAM_RATES:
        r = DfStream(model, st, batch=1, sr=sr)
        m = DfStream(model, st, batch=1, slot_rates=(sr,))
        assert m.rate_latency(sr) == (r.latency_frames, r.latency_samples) == r.rate_latency(sr)
        assert m.rate_latency(MODEL_SR) == (plain.latency_frames, 0)
