"""GPU: streaming slots (DfStream.open / close, dfb_stream_open_slots / close_slots).  A simulated server opens and closes
the slots of one handle on a seeded schedule; every session's output, from the call that opened it to the end of its
tail, must equal a fresh single-stream DfStream fed the same audio in the same call sizes and then flushed, and
enhance(pad=False) of its audio delayed by the latency.  Free slots, and closing slots past their tail, return exact
zeros; only open and closing slots are computed."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.streaming import SLOT_CLOSING, SLOT_FREE, SLOT_OPEN
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TOL = 1e-6          # RMS, as the existing streaming tests
EDGE = 4800         # first / last 100 ms of a session, checked on their own
SIZES = [1, 2, 3, 7, 40]


def cfg_of(kind, **kw):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5, **kw)
    if kind == "dfn3":
        return ModelConfig(model="deepfilternet3", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", **base)
    if kind == "dfn2":
        return ModelConfig(model="deepfilternet2", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=8, enc_lin_groups=8, enc_concat=True, **base)
    return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), emb_hidden_dim=512,
                       df_hidden_dim=512, emb_num_layers=3, df_num_layers=3, lin_groups=16, enc_lin_groups=16,
                       df_gru_skip="groupedlinear", **base)


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean())) if a.size else 0.0


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


def schedule(seed, n_random):
    """[(opens, closes, n hops)] of a server with 8 slots, all open at creation.  The scripted head covers: a close at
    clock 0 before any input, an open in a young handle (clock < 8) on a call of 1 hop, a slot closed after a single hop,
    an open and a close in the same call on different slots, a slot re-opened while it is still closing and an open slot
    re-opened.  Then seeded random traffic with call sizes of 1, 2, 3, 7 and 40 hops, opens late in the stream included."""
    calls = [([], [7], 1),          # clock 0: slot 7 ends before any input
             ([7], [], 1),          # clock 1: young open, call of 1 hop
             ([], [3, 7], 2),       # slot 7 closed after a single hop
             ([6], [], 3),          # clock 4: slot 6 re-opened while open
             ([3], [2], 1),         # open and close in one call on different slots
             ([2], [], 7),          # slot 2 re-opened while closing (1 hop of a >= 2 hop tail out)
             ([5], [0], 40)]
    rng = np.random.default_rng(seed)
    for _ in range(n_random):
        opens, closes = [], []
        for b in range(8):
            u = rng.random()
            if u < 0.12:
                opens.append(b)
            elif u < 0.3:
                closes.append(b)
        calls.append((opens, closes, int(rng.choice(SIZES))))
    return calls


class Session:
    def __init__(self, slot, seed):
        self.slot, self.seed = slot, seed
        self.sizes, self.outs = [], []
        self.closing, self.tail_left, self.done, self.dropped = False, 0, False, False

    def audio(self, total):
        return synth_audio(1, total * HOP, seed=self.seed)[0]


def run_server(model, st, calls, B=8, atten=None, setup=None, seed=0):
    """Runs the schedule on one handle and returns its sessions (finished with their tails, or dropped by a re-open)."""
    s = DfStream(model, st, batch=B, atten_lim_db=atten)
    if setup:
        setup(s)
    lat = s.latency_frames
    total_hops = sum(n for _, _, n in calls) + 1
    sessions, live, next_seed = [], {}, 1000 + 97 * seed
    src = {}

    def new_session(b):
        nonlocal next_seed
        ses = Session(b, next_seed)
        next_seed += 1
        src[id(ses)] = ses.audio(total_hops)
        live[b] = ses
        sessions.append(ses)

    for b in range(B):
        new_session(b)
    noise = torch.Generator().manual_seed(5 + seed)
    for i in range(len(calls) + 1):
        flush = i == len(calls)
        if not flush:
            opens, closes, n = calls[i]
            if closes:
                s.close(closes)
                for b in closes:
                    ses = live.get(b)
                    if ses is not None and not ses.closing:
                        ses.closing, ses.tail_left = True, lat
                        if lat == 0:
                            ses.done = True
                            del live[b]
            if opens:
                s.open(opens)
                for b in opens:
                    if b in live:
                        live[b].dropped = True
                    new_session(b)
            expect = np.array([SLOT_FREE if b not in live else (SLOT_CLOSING if live[b].closing else SLOT_OPEN) for b in range(B)])
            assert np.array_equal(s.slot_states(), expect), (i, s.slot_states(), expect)
            x = torch.randn((B, n * HOP), generator=noise) * 0.3          # rows of free / closing slots are ignored
            for b, ses in live.items():
                if not ses.closing:
                    pos = sum(ses.sizes)
                    x[b] = src[id(ses)][pos * HOP:(pos + n) * HOP]
                    ses.sizes.append(n)
            y = s.process(x.cuda() if i % 2 else x).cpu()
        else:
            for b, ses in list(live.items()):
                if not ses.closing:
                    ses.closing, ses.tail_left = True, lat
                if lat == 0:
                    ses.done = True
                    del live[b]
            y = s.flush()
            n = lat
        rows_used = set()
        for b, ses in list(live.items()):
            row = y[b]
            if not ses.closing:
                ses.outs.append(row)
            elif ses.tail_left > 0:
                k = min(n, ses.tail_left)
                ses.outs.append(row[:k * HOP])
                assert row[k * HOP:].abs().max().item() == 0 if k < n else True, (i, b)
                ses.tail_left -= k
                if ses.tail_left == 0:
                    ses.done = True
                    del live[b]
            rows_used.add(b)
        for b in range(B):
            if b not in rows_used and y.shape[1]:
                assert y[b].abs().max().item() == 0, ("free slot output", i, b)
    assert not live and np.array_equal(s.slot_states(), np.zeros(B))
    for ses in sessions:
        ses.src = src[id(ses)]
    return sessions, lat


def reference(model, st, ses, atten=None, setup=None):
    r = DfStream(model, st, batch=1, atten_lim_db=atten)
    if setup:
        setup(r)
    outs, pos = [], 0
    for n in ses.sizes:
        outs.append(r.process(ses.src[None, pos * HOP:(pos + n) * HOP])[0])
        pos += n
    outs.append(r.flush()[0])
    return torch.cat(outs)


def check_sessions(model, st, sessions, lat, atten=None, setup=None, against_enhance=True):
    checked = 0
    for ses in sessions:
        got = torch.cat(ses.outs) if ses.outs else torch.zeros(0)
        if not ses.sizes:
            assert got.abs().max().item() == 0 if got.numel() else True
            continue
        ref = reference(model, st, ses, atten, setup)
        if ses.dropped:
            assert got.numel() <= ref.numel()
            ref = ref[:got.numel()]
        assert got.shape == ref.shape, (ses.slot, got.shape, ref.shape)
        assert rms(got, ref) < TOL, (ses.slot, ses.sizes, rms(got, ref))
        assert rms(got[:EDGE], ref[:EDGE]) < TOL and rms(got[-EDGE:], ref[-EDGE:]) < TOL, ses.slot
        if against_enhance and not ses.dropped:
            T = sum(ses.sizes) * HOP
            one = enhance(model, st, ses.src[None, :T], pad=False, atten_lim_db=atten)[0]
            assert got[:lat * HOP].abs().max().item() == 0 if lat else True
            assert rms(got[lat * HOP:], one) < TOL, (ses.slot, rms(got[lat * HOP:], one))
        checked += 1
    return checked


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_slots_equal_fresh_streams(st, kind):
    model = DfNet(cfg_of(kind), random_state_dict(cfg_of(kind), seed=91), st)
    sessions, lat = run_server(model, st, schedule(seed=7, n_random=24), seed=1)
    assert lat == {"dfn3": 2, "dfn2": 4, "ll": 0}[kind]
    assert any(s.dropped for s in sessions) and sum(1 for s in sessions if not s.dropped and s.sizes) >= 12
    assert check_sessions(model, st, sessions, lat) >= 12


@pytest.mark.parametrize("variant", ["post_filter", "atten_lim", "lsnr_gating"])
def test_slots_with_options(st, variant):
    cfg = cfg_of("dfn3", mask_pf=variant == "post_filter")
    model = DfNet(cfg, random_state_dict(cfg, seed=92), st)
    atten = 12.0 if variant == "atten_lim" else None
    setup = (lambda s: s.set_lsnr_thresholds()) if variant == "lsnr_gating" else None   # the Rust runtime's defaults
    sessions, lat = run_server(model, st, schedule(seed=8, n_random=12), atten=atten, setup=setup, seed=2)
    assert check_sessions(model, st, sessions, lat, atten=atten, setup=setup, against_enhance=variant != "lsnr_gating") >= 6


def test_only_active_slots_are_computed(st):
    """After all but 2 of 64 slots are closed and their tails are out, a call computes 2 rows: the forward pass's `emb`
    activation holds 2 x window x emb_dim floats."""
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=93), st)
    B = 64
    s = DfStream(model, st, batch=B)
    x = synth_audio(B, 20 * HOP, seed=3)
    s.process(x)
    s.close([b for b in range(B) if b not in (5, 40)])
    s.process(x[:, :HOP * s.latency_frames])        # the tails come out
    assert (s.slot_states() == SLOT_OPEN).sum() == 2 and (s.slot_states() == SLOT_FREE).sum() == B - 2
    n = 3
    y = s.process(x[:, :n * HOP])
    buf = np.zeros(B * 64 * 1024, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, b"emb", buf.ctypes.data, buf.size)
    emb_dim = cfg.nb_erb // 4 * 64
    assert got == 2 * (8 + n) * emb_dim        # kHalo = 8 halo frames + n new frames per stream
    assert y[[b for b in range(B) if b not in (5, 40)]].abs().max() == 0 and y[[5, 40]].abs().max() > 0


def test_slot_errors(st):
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=94), st)
    s = DfStream(model, st, batch=4)
    L = _lib.lib()
    for bad in ([4], [-1], [1, 1]):
        with pytest.raises(ValueError):
            s.open(bad)
        with pytest.raises(ValueError):
            s.close(bad)
        a = (C.c_int64 * len(bad))(*bad)
        for fn in (L.dfb_stream_open_slots, L.dfb_stream_close_slots):
            assert fn(s._h, a, len(bad)) == _lib.DFB_ERR_INVALID
    assert np.array_equal(s.slot_states(), [SLOT_OPEN] * 4)      # a refused call changes nothing
    linked = DfStream(model, st, batch=4, channels=2, reduce_mask="mean")
    for op in (linked.open, linked.close):
        with pytest.raises(_lib.DfbError) as e:
            op([0])
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    # a handle with slot operations cannot be linked afterwards; reset brings back every slot open
    s.close([2])
    with pytest.raises(_lib.DfbError) as e:
        s.set_mask_reduce(2, "mean")
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    s.reset()
    assert np.array_equal(s.slot_states(), [SLOT_OPEN] * 4)
    s.set_mask_reduce(2, "mean")


def test_flush_frees_every_slot_and_slots_reopen(st):
    """flush() = close(all open slots) + latency hops without input; afterwards every slot is free, and a slot opened
    then starts a fresh stream."""
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=95), st)
    s = DfStream(model, st, batch=3)
    x = synth_audio(3, 30 * HOP, seed=9)
    a = torch.cat([s.process(x[:, :11 * HOP]), s.flush()], 1)
    assert np.array_equal(s.slot_states(), [SLOT_FREE] * 3)
    s.open([1])
    b = torch.cat([s.process(x[:, 11 * HOP:]), s.flush()], 1)
    r = DfStream(model, st, batch=1)
    ref = torch.cat([r.process(x[1:2, 11 * HOP:]), r.flush()], 1)[0]
    assert rms(b[1], ref) < TOL and b[[0, 2]].abs().max() == 0
    r.reset()
    assert rms(a[2], torch.cat([r.process(x[2:3, :11 * HOP]), r.flush()], 1)[0]) < TOL
