"""GPU: the runtime gating mode (include/dfb200.h dfb_gating_mode, DfNet.set_gating_mode, gating_mode=...), in which each
decoder runs only on the frames LSNR stage gating lets through, as the Rust runtime's decoders do (tract.rs:478-503).

* The recurrence alone (dfb_debug_gru_tc_hold): held steps keep the state; every built k_gru_tc instance equals the plain
  kernel run on each row's compacted steps, bit for bit.
* End to end against tests/gating_runtime_oracle.py (the decoders run on their own frames only) at the gating tolerance of
  5e-6 RMS, on DeepFilterNet3 and DeepFilterNet3_ll: ragged batches with a linked pair, 1 / 6 / 8 chunks on one or two
  lanes, streaming handles with ragged call sizes, slots opened and closed mid-run with their own thresholds, slot
  groups, spectral handles of all four models.  The thresholds come from each stream's own LSNR, with a margin from every
  value, and give gated runs of 1, 2-4, more than 8 frames and more than a time chunk; runtime and apply mode differ by
  far more than the tolerance.
* Bit-exact invariants: thresholds that never gate give apply mode's bits; the LSNR is the same in both modes; entry i of
  a mixed batch equals the batch with entry i's settings everywhere; a stream switched from apply to runtime mode equals
  the oracle with every frame before the switch a run frame."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import gating_runtime_oracle as GO
import linked_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, enhance_batch, enhance_device_ragged, io, libdf
from deepfilternet_b200.config import ModelConfig, load_config
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TOL = 5e-6            # RMS against the oracle: the gating tolerance of tests/test_gpu_ragged_ctl.py
CHUNK_TOL = 1e-6      # RMS between chunkings, as tests/test_gpu_parity.py
SEED = 23
NEVER = (-1e9, 1e9, 1e9)
KINDS = ["dfn3", "dfn3_ll"]


def cfg_of(kind):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5)
    if kind == "dfn3":
        return ModelConfig(model="deepfilternet3", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", **base)
    if kind == "dfn2":
        return ModelConfig(model="deepfilternet2", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=8, enc_lin_groups=8, enc_concat=True, **base)
    if kind == "dfn2_ll":
        import os
        return load_config(os.path.join(os.path.dirname(__file__), "golden", "models", "DeepFilterNet2_ll", "config.ini"), env={})
    return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), emb_hidden_dim=512,
                       df_hidden_dim=512, emb_num_layers=3, df_num_layers=3, lin_groups=16, enc_lin_groups=16,
                       df_gru_skip="groupedlinear", **base)


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean())) if a.size else 0.0


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_MODELS = {}


def model_of(st, kind):
    if kind not in _MODELS:
        _MODELS[kind] = (DfNet(cfg_of(kind), random_state_dict(cfg_of(kind), seed=SEED), st), random_state_dict(cfg_of(kind), seed=SEED))
    return _MODELS[kind]


def signal(seed, secs=6.0, channels=1):
    """Synthetic noisy speech with 1.5 s of near silence from 2 s on: a long stretch of one LSNR regime."""
    a = synth_audio(channels, int(secs * 48000), seed=seed)
    a[:, 2 * 48000:int(3.5 * 48000)] *= 0.01
    return a


def _mids(l):
    s = np.unique(np.sort(np.asarray(l, dtype=np.float64)))
    return np.array([(s[k] + s[k + 1]) / 2 for k in range(len(s) - 1) if s[k + 1] - s[k] > 2e-3])


def thresholds(l, long_run):
    """(min, max_erb, max_df) between LSNR values of l (each at least 1e-3 from every value): max_erb gates runs of 1,
    2-4, more than 8 and more than `long_run` frames of the ERB decoder; max_df gates more of the DF decoder's; min gates
    the quietest 3 %."""
    mids = _mids(l)
    pick = lambda q: float(mids[np.argmin(np.abs(mids - np.quantile(l, q)))])  # noqa: E731
    for q in np.linspace(0.3, 0.95, 66):
        erb = pick(q)
        r = GO.gated_runs(torch.as_tensor(~(np.asarray(l) > erb)))
        if 1 in r and any(2 <= x <= 4 for x in r) and any(x > 8 for x in r) and any(x > long_run for x in r):
            return (pick(0.03), erb, pick(0.35 * q))
    raise AssertionError("no thresholds with the required gated runs")


def check_runs(erb_run, long_run):
    r = GO.gated_runs(erb_run)
    assert 1 in r and any(2 <= x <= 4 for x in r) and any(x > 8 for x in r) and any(x > long_run for x in r), r


def oracle_lsnr(sd, cfg, a, pad):
    _, aux = LO.enhance(sd, cfg.as_dict(), a, pad=pad, return_all=True)
    return aux["lsnr"][0, :, 0].numpy()


# ------------------------------------------------------------------------------------------------ the recurrence alone ----
INST = {256: [(16, 0), (16, 1), (32, 0), (32, 1), (48, 1)], 512: [(16, 0), (16, 1)]}


def ptr(t):
    return None if t is None else t.data_ptr()


def gru(xp, whh, bhh, B, T, H, ns, xg, run=None, h0=None, hT=None, t0=0, Ts=None):
    Ts = T if Ts is None else Ts
    hout = torch.zeros((B, Ts, H), dtype=torch.float32, device="cuda")
    cs = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    if run is None:
        rc = L.dfb_debug_gru_tc(ptr(xp), ptr(whh), ptr(bhh), None, ptr(hout), None, None, 0, ptr(h0), ptr(hT), None, 0, t0, Ts, B, T,
                                H, ns, xg, cs)
    else:
        rc = L.dfb_debug_gru_tc_hold(ptr(xp), ptr(whh), ptr(bhh), None, ptr(hout), None, None, 0, ptr(h0), ptr(hT), None, 0, ptr(run),
                                     t0, Ts, B, T, H, ns, xg, cs)
    assert rc == 0, L.dfb_last_error()
    torch.cuda.synchronize()
    return hout


@pytest.mark.parametrize("H", [256, 512])
def test_hold_equals_compacted_steps(H):
    """For every built instance and random run flags: the outputs at run steps and the final state equal the plain kernel
    run on each row's compacted steps, held steps output the held state, an all-run mask is the plain kernel, and a
    window split with carried h0 / hT equals one window -- all bit for bit."""
    g = torch.Generator().manual_seed(3)
    k = H ** -0.5
    whh = ((torch.rand(3 * H, H, generator=g) * 2 - 1) * k).cuda()
    bhh = ((torch.rand(3 * H, generator=g) * 2 - 1) * k).cuda()
    for ns, xg in INST[H]:
        B, T = ns + 3, 37
        xp = torch.randn(B, T, 3 * H, generator=g).cuda()
        h0 = (torch.rand(B, H, generator=g) * 2 - 1).cuda()
        run = (torch.rand(B, T, generator=g) < 0.6).to(torch.uint8)
        run[0] = 0                     # a row that never runs
        run[1] = 1                     # and one that always does
        run = run.cuda()
        hT = torch.empty(B, H, device="cuda")
        out = gru(xp, whh, bhh, B, T, H, ns, xg, run=run, h0=h0, hT=hT)
        n = run.sum(1).cpu()
        idx = [torch.nonzero(run[b]).view(-1) for b in range(B)]
        xc = torch.zeros_like(xp)
        for b in range(B):
            xc[b, :int(n[b])] = xp[b, idx[b]]
        ref = gru(xc, whh, bhh, B, T, H, ns, xg, h0=h0)
        for b in range(B):
            nb = int(n[b])
            assert torch.equal(out[b, idx[b]], ref[b, :nb]), (H, ns, xg, b)
            last = ref[b, nb - 1] if nb else h0[b]
            assert torch.equal(hT[b], last), (H, ns, xg, b)
            held = torch.nonzero(run[b] == 0).view(-1)
            for t in held.tolist():   # a held step outputs the state of the last run step before it
                prev = idx[b][idx[b] < t]
                want = out[b, prev[-1]] if prev.numel() else h0[b]
                assert torch.equal(out[b, t], want), (H, ns, xg, b, t)
        ones = torch.ones(B, T, dtype=torch.uint8, device="cuda")
        assert torch.equal(gru(xp, whh, bhh, B, T, H, ns, xg, run=ones, h0=h0), gru(xp, whh, bhh, B, T, H, ns, xg, h0=h0))
        for s in (1, 13):
            state = torch.empty(B, H, device="cuda")
            part = torch.zeros(B, T, H, device="cuda")
            cs = torch.cuda.current_stream().cuda_stream
            L = _lib.lib()
            assert L.dfb_debug_gru_tc_hold(ptr(xp), ptr(whh), ptr(bhh), None, ptr(part), None, None, 0, ptr(h0), ptr(state), None, 0,
                                           ptr(run), 0, T, B, s, H, ns, xg, cs) == 0
            assert L.dfb_debug_gru_tc_hold(ptr(xp), ptr(whh), ptr(bhh), None, ptr(part), None, None, 0, ptr(state), ptr(state), None, 0,
                                           ptr(run), s, T, B, T - s, H, ns, xg, cs) == 0
            torch.cuda.synchronize()
            assert torch.equal(part, out) and torch.equal(state, hT), (H, ns, xg, s)


# ---------------------------------------------------------------------------------------------------- ragged batches ----
@pytest.mark.parametrize("kind", KINDS)
def test_batch_equals_oracle(st, kind):
    """A ragged batch (a mono entry, a linked pair, an entry that does not gate) in runtime mode equals the oracle entry by
    entry, through enhance_batch (host path, 4 chunks on two lanes) and enhance_device_ragged at 1, 6 and 8 chunks on one
    or two lanes, which agree within the chunking bound; the mode is far from apply mode.  A 16 kHz entry equals the
    oracle between io.resample's two directions."""
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    audios = [signal(5), signal(6, secs=5.3, channels=2), signal(7, secs=4.1)]
    T_frames = [a.shape[-1] // HOP for a in audios]
    long_run = max(T_frames) // 8 + 1
    ths = []
    for a in audios[:2]:
        ths.append(thresholds(oracle_lsnr(sd, cfg, a[:1], False), long_run))
    ths.append(None)
    want, apply_want = [], []
    for a, th in zip(audios, ths):
        w, aux = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=th, reduce="mean" if a.shape[0] > 1 else None,
                            return_all=True)
        if th is not None:
            check_runs(aux["erb_run"][0], long_run)
        want.append(w)
        apply_want.append(LO.enhance(sd, cfg.as_dict(), a, pad=False, reduce="mean" if a.shape[0] > 1 else None,
                                     stages=None if th is None else dict(zip(("min_db_thresh", "max_db_erb_thresh", "max_db_df_thresh"), th))))
    got = enhance_batch(model, st, audios, False, reduce_mask="mean", lsnr_thresholds=ths, gating_mode="runtime")
    for i in range(3):
        print(kind, i, rms(got[i], want[i]), rms(want[i], apply_want[i]))
        assert rms(got[i], want[i]) <= TOL, (kind, i, rms(got[i], want[i]))
    for i in range(2):
        assert rms(want[i], apply_want[i]) > 20 * TOL, (kind, i)
    assert rms(got[2], apply_want[2]) <= TOL
    assert model.gating_mode == "apply"
    # a 16 kHz entry beside a 48 kHz one: io.resample(oracle(io.resample(x, 16000, 48000)), 48000, 16000)
    a16 = synth_audio(1, 5 * 16000 + 7, seed=9, sr=16000)
    a16[:, 2 * 16000:int(3.5 * 16000)] *= 0.01
    x48 = io.resample(a16, 16000, 48000)
    th16 = thresholds(oracle_lsnr(sd, cfg, x48, False), 8)
    w16, aux = GO.enhance(sd, cfg.as_dict(), x48, pad=False, stages=th16, return_all=True)
    check_runs(aux["erb_run"][0], 8)
    w16 = io.resample(w16, 48000, 16000)
    got = enhance_batch(model, st, [audios[0], a16], False, sr=[48000, 16000], lsnr_thresholds=[ths[0], th16], gating_mode="runtime")
    assert rms(got[0], want[0]) <= TOL
    assert got[1].shape == w16.shape and rms(got[1], w16) <= TOL, (kind, rms(got[1], w16))
    # device path: one row per channel, padded
    rows = [a[c] for a in audios for c in range(a.shape[0])]
    S = max(r.shape[0] for r in rows)
    x = torch.zeros(len(rows), S)
    for b, r in enumerate(rows):
        x[b, :r.shape[0]] = r
    lens = [r.shape[0] for r in rows]
    row_th = [ths[0], ths[1], ths[1], None]
    outs = []
    try:
        for chunks, lanes in ((1, 1), (6, 2), (8, 2), (8, 1)):
            model.set_chunking(chunks, 4, lanes)
            y = enhance_device_ragged(model, st, x.cuda(), lens, False, group_sizes=[1, 2, 1], reduce_mask="mean",
                                      lsnr_thresholds=row_th, gating_mode="runtime").cpu()
            outs.append(y)
    finally:
        model.set_chunking()
    ref_rows = [want[0][0], want[1][0], want[1][1], want[2][0]]
    for y in outs:
        for b in range(4):
            n = ref_rows[b].shape[-1]
            assert rms(y[b, :n], ref_rows[b]) <= TOL, (kind, b)
            assert rms(y[b, :n], outs[0][b, :n]) <= CHUNK_TOL


def test_mixed_batch_entries_equal_uniform_batches(st):
    """Entry i of a runtime-mode batch with mixed settings equals, bit for bit, entry i of the batch with entry i's settings
    given to every entry, and a non-gating entry equals apply mode's bits."""
    kind = "dfn3"
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    audios = [signal(11, secs=3.0), signal(12, secs=2.2), signal(13, secs=2.7)]
    ths = [thresholds(oracle_lsnr(sd, cfg, audios[0], False), 8), None, thresholds(oracle_lsnr(sd, cfg, audios[2], False), 8)]
    mixed = enhance_batch(model, st, audios, False, lsnr_thresholds=ths, atten_lim_db=[0, 6, 12], gating_mode="runtime")
    lims = [0, 6, 12]
    for i in range(3):
        uni = enhance_batch(model, st, audios, False, lsnr_thresholds=[ths[i]] * 3, atten_lim_db=[lims[i]] * 3, gating_mode="runtime")
        assert torch.equal(mixed[i], uni[i]), i
    apply = enhance_batch(model, st, audios, False, lsnr_thresholds=ths, atten_lim_db=lims)
    assert torch.equal(mixed[1], apply[1])


@pytest.mark.parametrize("kind", KINDS)
def test_never_gating_thresholds_give_apply_bits(st, kind):
    """Thresholds that never gate: runtime mode equals apply mode bit for bit on a batch, a streaming handle and a spectral
    handle; with real thresholds the LSNR rows are identical in both modes."""
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    audios = [signal(21, secs=3.1), signal(22, secs=2.0)]
    a = enhance_batch(model, st, audios, False, lsnr_thresholds=NEVER, return_lsnr=True)
    r = enhance_batch(model, st, audios, False, lsnr_thresholds=NEVER, return_lsnr=True, gating_mode="runtime")
    for i in range(2):
        assert torch.equal(a[0][i], r[0][i]) and torch.equal(a[1][i], r[1][i]), i
    th = thresholds(oracle_lsnr(sd, cfg, audios[0], False), 8)
    a = enhance_batch(model, st, audios, False, lsnr_thresholds=th, return_lsnr=True)
    r = enhance_batch(model, st, audios, False, lsnr_thresholds=th, return_lsnr=True, gating_mode="runtime")
    for i in range(2):
        assert torch.equal(a[1][i], r[1][i]), i
        assert not torch.equal(a[0][i], r[0][i]), i
    x = signal(23, secs=2.0, channels=2)
    outs = []
    for mode in ("apply", "runtime"):
        s = DfStream(model, st, batch=2, gating_mode=mode)
        s.set_lsnr_thresholds(*NEVER)
        outs.append(feed(s, x))
    assert torch.equal(outs[0], outs[1])
    spec = st.analysis(np.ascontiguousarray(x.numpy()))
    rows = []
    for mode in ("apply", "runtime"):
        s = DfStream(model, st, batch=2, spectral=True, gating_mode=mode)
        s.set_lsnr_thresholds(*NEVER)
        rows.append(run_spec(s, spec, [5, 17, 40]))
    for k in range(4):   # rows before the latency are NaN / -1 in both
        assert torch.equal(torch.isnan(rows[0][k].float()), torch.isnan(rows[1][k].float())), k
        assert torch.equal(torch.nan_to_num(rows[0][k].float()), torch.nan_to_num(rows[1][k].float())), k


# ------------------------------------------------------------------------------------------------------ streaming ----
SIZES = [1, 3, 16, 33]


def feed(s, x, sizes=SIZES):
    outs, pos, i = [], 0, 0
    n = x.shape[-1] // HOP
    while pos < n:
        k = min(sizes[i % len(sizes)], n - pos)
        outs.append(s.process(x[:, pos * HOP:(pos + k) * HOP]))
        pos += k
        i += 1
    outs.append(s.flush())
    return torch.cat(outs, 1)


def run_spec(s, spec, sizes):
    outs, pos, i = [], 0, 0
    T = spec.shape[1]
    while pos < T:
        k = min(sizes[i % len(sizes)], T - pos)
        outs.append([t.cpu() for t in s.process_spec(torch.from_numpy(np.ascontiguousarray(spec[:, pos:pos + k])))])
        pos += k
        i += 1
    outs.append([t.cpu() for t in s.flush_spec()])
    return [torch.cat([o[k] for o in outs], 1) for k in range(4)]


@pytest.mark.parametrize("kind", KINDS)
def test_stream_equals_oracle(st, kind):
    """A streaming handle in runtime mode (the model's mode, and the handle's own), fed in calls of 1, 3, 16 and 33 hops,
    equals the oracle of the stream alone (pad=False), delayed by the latency."""
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    x = signal(31)
    th = thresholds(oracle_lsnr(sd, cfg, x, False), 33)
    want, aux = GO.enhance(sd, cfg.as_dict(), x, pad=False, stages=th, return_all=True)
    check_runs(aux["erb_run"][0], 33)
    s = DfStream(model, st, batch=1, gating_mode="runtime")
    s.set_lsnr_thresholds(*th)
    y = feed(s, x)[:, s.latency_frames * HOP:]
    assert rms(y, want) <= TOL, (kind, rms(y, want))
    model.set_gating_mode("runtime")
    try:
        s = DfStream(model, st, batch=1)
        s.set_lsnr_thresholds(*th)
        y2 = feed(s, x, [7, 2])[:, s.latency_frames * HOP:]
    finally:
        model.set_gating_mode("apply")
    assert rms(y2, want) <= TOL and rms(y2, y) <= CHUNK_TOL


@pytest.mark.parametrize("kind", KINDS)
def test_mode_switch_on_a_live_handle(st, kind):
    """Apply-mode calls followed by runtime-mode calls equal the oracle whose frames before the switch all ran."""
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    x = signal(41)
    th = thresholds(oracle_lsnr(sd, cfg, x, False), 8)
    s = DfStream(model, st, batch=1, gating_mode="apply")
    s.set_lsnr_thresholds(*th)
    n0 = 150
    outs = [s.process(x[:, :n0 * HOP])]
    switch = n0 - s.latency_frames        # DNN frames already computed in apply mode
    s.set_gating_mode("runtime")
    outs.append(feed(s, x[:, n0 * HOP:]))
    y = torch.cat(outs, 1)[:, s.latency_frames * HOP:]

    def flags(b, l, t):
        e, d = GO.run_flags(l, t)
        e[:switch] = True
        d[:switch] = True
        return e, d
    want = GO.enhance(sd, cfg.as_dict(), x, pad=False, stages=th, flags_of=flags)
    assert rms(y, want) <= TOL, (kind, rms(y, want))
    assert rms(want, GO.enhance(sd, cfg.as_dict(), x, pad=False, stages=th)) > 20 * TOL


@pytest.mark.parametrize("kind", KINDS)
def test_slots_and_groups(st, kind):
    """Slots opened and closed mid-run with their own thresholds, and a slot group (channel 0 decides for the group), in
    runtime mode, 5 hops per call: every session equals the oracle of that session alone."""
    model, sd = model_of(st, kind)
    cfg = cfg_of(kind)
    s = DfStream(model, st, batch=4, reduce_mask="mean", gating_mode="runtime")
    L, n = s.latency_frames, 5
    # slot(s) -> (audio, first call hop); lengths and starts are whole calls
    sessions = {(0,): (signal(51, secs=3.0), 0), (1, 2): (signal(52, secs=2.5, channels=2), 40), (3,): (signal(53, secs=2.0), 90)}
    ths = {k: thresholds(oracle_lsnr(sd, cfg, a[:1], False), 8) for k, (a, _) in sessions.items()}
    got = {k: [] for k in sessions}
    end = max(start + a.shape[-1] // HOP for a, start in sessions.values()) + L + n
    for t in range(0, end, n):
        x = torch.zeros(4, n * HOP)
        for k, (a, start) in sessions.items():
            hops = a.shape[-1] // HOP
            if t == start:
                (s.open_linked if len(k) > 1 else s.open)(list(k))
                s.set_lsnr_thresholds(*ths[k], slots=list(k))
            if t == start + hops:
                s.close(list(k))
            if start <= t < start + hops:
                x[list(k)] = a[:, (t - start) * HOP:(t - start + n) * HOP]
        y = s.process(x)
        for k, (a, start) in sessions.items():
            if start <= t < start + a.shape[-1] // HOP + L:
                got[k].append(y[list(k)])
    for k, (a, _) in sessions.items():
        ys = torch.cat(got[k], 1)[:, L * HOP:L * HOP + a.shape[-1]]
        want = GO.enhance(sd, cfg.as_dict(), a, pad=False, stages=ths[k], reduce="mean" if len(k) > 1 else None)
        assert ys.shape == want.shape, (ys.shape, want.shape)
        assert rms(ys, want) <= TOL, (kind, k, rms(ys, want))


@pytest.mark.parametrize("kind", ["dfn3", "dfn3_ll", "dfn2", "dfn2_ll"])
def test_spectral_handle(st, kind):
    """A spectral handle in runtime mode: the gains of the frames the ERB decoder ran on and the coefficients of those the
    DF decoder ran on equal the oracle's (the decoders run on their frames only); the other frames carry the stage rule's
    constants."""
    cfg = cfg_of(kind)
    sd = random_state_dict(cfg, seed=SEED)
    model = DfNet(cfg, sd, st)
    x = signal(61, secs=4.0)
    th = thresholds(oracle_lsnr(sd, cfg, x, False), 8)
    _, aux = GO.enhance(sd, cfg.as_dict(), x, pad=False, stages=th, return_all=True)
    spec = st.analysis(np.ascontiguousarray(x.numpy()))
    s = DfStream(model, st, batch=1, spectral=True, gating_mode="runtime")
    s.set_lsnr_thresholds(*th)
    L = s.latency_frames
    g, cf, ls, sg = run_spec(s, spec, [1, 3, 16, 33])
    g, cf, sg = g[0, L:], cf[0, L:].reshape(-1, 96, 10), sg[0, L:]
    e, d = aux["erb_run"][0], aux["df_run"][0]
    T = g.shape[0]
    e, d = e[:T], d[:T]
    assert torch.equal(e, (sg == 1) | (sg == 2)) and torch.equal(d, sg == 1)
    m, c = aux["m"][0, 0, :T], aux["coefs"][0, :T]
    assert rms(g[e], m[e]) <= 1e-4 and rms(cf[d], c[d]) <= 1e-4, (kind, rms(g[e], m[e]), rms(cf[d], c[d]))
    s2 = DfStream(model, st, batch=1, spectral=True)
    s2.set_lsnr_thresholds(*th)
    g2, cf2, _, _ = run_spec(s2, spec, [1, 3, 16, 33])
    assert rms(cf2[0, L:].reshape(-1, 96, 10)[d], c[d]) > 1e-4


def test_refusals(st):
    """Bad modes are refused in C (DFB_ERR_INVALID) and change nothing; DeepFilterNet v1 takes the mode and still refuses
    gating."""
    model, _ = model_of(st, "dfn3")
    L = _lib.lib()
    assert L.dfb_model_set_gating_mode(model.handle, 2) == _lib.DFB_ERR_INVALID
    assert L.dfb_model_set_gating_mode(model.handle, -1) == _lib.DFB_ERR_INVALID
    assert L.dfb_model_set_gating_mode(None, 0) == _lib.DFB_ERR_INVALID
    s = DfStream(model, st, batch=1)
    assert L.dfb_stream_set_gating_mode(s._h, 2) == _lib.DFB_ERR_INVALID
    assert L.dfb_stream_set_gating_mode(s._h, -2) == _lib.DFB_ERR_INVALID
    x = signal(71, secs=1.0)
    a = enhance_batch(model, st, [x], False, lsnr_thresholds=NEVER)
    assert torch.equal(a[0], enhance_batch(model, st, [x], False, lsnr_thresholds=NEVER)[0])
    with pytest.raises(ValueError):
        enhance(model, st, x, gating_mode="rt")
    with pytest.raises(ValueError):
        model.set_gating_mode("Runtime")
    assert model.gating_mode == "apply"
    from test_gpu_ragged_ctl import cfg_of as cfg_ctl
    v1 = DfNet(cfg_ctl("v1"), random_state_dict(cfg_ctl("v1"), seed=1), st)
    v1.set_gating_mode("runtime")
    with pytest.raises(Exception):
        enhance_batch(v1, st, [x], False, lsnr_thresholds=(-10.0, 30.0, 20.0))
    y = enhance(v1, st, x)
    v1.set_gating_mode("apply")
    assert torch.equal(y, enhance(v1, st, x))
