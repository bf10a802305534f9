"""GPU: held sessions (DfStream.hold / held_slots, dfb_stream_hold_slots).  A held session sits out every call it is held
through, as if the call had not happened: its outputs over the calls it advanced in, followed by its drain or flush, equal
a single-session DfStream fed the same audio in those calls' sizes, bit for bit.  Its neighbours are unaffected; its
input rows are ignored and its output rows are zeros with NaN LSNR; its state rows are not touched; groups, rates,
settings, runtime gating, close / flush / reset / open / export, spectral handles and the row moves behind it."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, libdf
from deepfilternet_b200._lib import DFB_ERR_INVALID, DFB_ERR_UNSUPPORTED, DfbError
from deepfilternet_b200.config import load_config
from deepfilternet_b200.streaming import MODEL_SR, SLOT_FREE, SLOT_OPEN, SLOT_CLOSING
from deepfilternet_b200.weights import random_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "tests", "golden", "models")
SEEDS = {"DeepFilterNet3": 11, "DeepFilterNet3_ll": 14, "DeepFilterNet2": 12, "DeepFilterNet2_ll": 15}   # oracle/synth_models.py
NAMES = list(SEEDS)
SIZES = [1, 2, 3, 5, 7]


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_models = {}


def model_of(name, st):
    if name not in _models:
        cfg = load_config(os.path.join(MODELS, name, "config.ini"), env={})
        _models[name] = DfNet(cfg, random_state_dict(cfg, seed=SEEDS[name]), st)
    return _models[name]


def same(a, b):
    """bit for bit, NaN where the other is NaN"""
    if a.shape != b.shape:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def launches(fn):
    n0 = _lib.lib().dfb_kernel_launches()
    fn()
    return _lib.lib().dfb_kernel_launches() - n0


def rows_moved(s):
    import ctypes as C
    n = C.c_int64()
    assert _lib.lib().dfb_debug_stream_rows_moved(s._h, C.byref(n)) == 0
    return n.value


class Server:
    """A handle whose untracked open slots are fed seeded noise.  Tracked sessions (slot -> its audio at its rate) read
    their own audio only in the calls they advance in and collect those calls' outputs, their sizes and, once closed,
    their drain.  Held rows are fed NaN and must come back as zeros with NaN LSNR.  `lsnr`: the calls request the LSNR
    (and collect it) from now on."""

    def __init__(self, s, seed, lsnr=True):
        self.s, self.g, self.lsnr = s, torch.Generator().manual_seed(seed), lsnr
        self.feed, self.outs, self.lsn, self.sizes, self.drain, self.hooks = {}, {}, {}, {}, {}, {}
        self.held = set()

    def rate(self, b):
        return self.feed[b][2]

    def track(self, slots, audio, sr=MODEL_SR):
        for c, b in enumerate(slots):
            self.feed[b] = [audio[c], 0, sr]
            self.outs[b], self.lsn[b], self.sizes[b] = [], [], []

    def hold(self, slots, held=True):
        self.s.hold(slots, held)
        for b in slots:
            (self.held.add if held else self.held.discard)(b)
        assert sorted(np.flatnonzero(self.s.held_slots()).tolist()) == sorted(self.held)

    def close(self, slots):
        self.s.close(slots)
        for b in slots:
            if b in self.feed:
                f = self.feed[b]
                self.drain[b] = self.latency(f[2])
            if self.s.slot_states()[b] == SLOT_FREE:   # without look-ahead: free at once, no hold left
                self.held.discard(b)

    def latency(self, sr):
        return self.s.rate_latency(sr)[0] if self.s.registered_rates else self.s.latency_frames

    def call(self, n):
        B, w = self.s.batch, self.s.hop
        x = torch.randn((B, n * w), generator=self.g) * 0.1
        for b in self.held:
            x[b] = float("nan")
        for b, f in self.feed.items():
            if b in self.held or b in self.drain:
                continue
            k = n * f[2] // 100
            x[b] = 0
            x[b, :k] = f[0][f[1]:f[1] + k]
            f[1] += k
        out, ls = self.s.process(x, return_lsnr=True) if self.lsnr else (self.s.process(x), None)
        for b in self.held:
            assert out[b].abs().max().item() == 0 and (ls is None or torch.isnan(ls[b]).all()), b
        for b, f in list(self.feed.items()):
            if b in self.held:
                continue
            k = n * f[2] // 100
            if b in self.drain:   # a closed session drains in the calls it advances in
                m = min(n, self.drain[b])
                self.outs[b].append(out[b, :m * f[2] // 100])
                if ls is not None:
                    self.lsn[b].append(ls[b, :m])
                self.drain[b] -= m
                continue
            self.outs[b].append(out[b, :k])
            if ls is not None:
                self.lsn[b].append(ls[b])
            self.sizes[b].append(n)

    def flush(self):
        out, ls = self.s.flush(return_lsnr=True) if self.lsnr else (self.s.flush(), None)
        for b, f in self.feed.items():
            L = self.drain.get(b, self.latency(f[2]))
            self.outs[b].append(out[b, :L * f[2] // 100])
            if ls is not None:
                self.lsn[b].append(ls[b, :L])
        self.held.clear()
        assert not self.s.held_slots().any()

    def result(self, slots):
        return (torch.stack([torch.cat(self.outs[b]) for b in slots]),
                torch.stack([torch.cat(self.lsn[b]) for b in slots]))


def reference(model, st, audio, sizes, sr=MODEL_SR, reduce=None, hooks=None, lsnr_at=0, **kw):
    """the session alone: a single-session handle at its rate fed the same call sizes, then flushed; hooks[i] runs
    before the session's call i; the LSNR is requested from call lsnr_at on"""
    C = audio.shape[0]
    extra = dict(channels=C, reduce_mask=reduce) if C > 1 else {}
    if sr != MODEL_SR:
        extra["sr"] = sr
    srv = Server(DfStream(model, st, batch=C, **extra, **kw), 0)
    srv.track(list(range(C)), audio, sr)
    for i, n in enumerate(sizes):
        if hooks and i in hooks:
            hooks[i](srv.s, list(range(C)))
        srv.lsnr = i >= lsnr_at
        srv.call(n)
    srv.lsnr = True
    srv.flush()
    return srv.result(list(range(C)))


def check_session(model, st, srv, slots, sr=MODEL_SR, reduce=None, hooks=None, lsnr_at=0, **kw):
    got = srv.result(slots)
    audio = torch.stack([srv.feed[b][0] for b in slots])
    ref = reference(model, st, audio, srv.sizes[slots[0]], sr=sr, reduce=reduce, hooks=hooks, lsnr_at=lsnr_at, **kw)
    assert same(got[0], ref[0]), f"audio of slots {slots}"
    assert same(got[1], ref[1]), f"LSNR of slots {slots}"


def audio_of(C, hops, seed, sr=MODEL_SR):
    return synth_audio(C, hops * sr // 100, seed, sr=sr)


@pytest.mark.parametrize("name", NAMES)
def test_held_anywhere(st, name):
    """random call sizes and hold runs of 1, several and more than 8 + look-ahead calls: from the handle's first call
    (an unsettled clock), from a session's open before it ever advanced, right before a close; neighbours on their own
    schedules"""
    model = model_of(name, st)
    rng = np.random.default_rng(SEEDS[name])
    B = 7
    srv = Server(DfStream(model, st, batch=B), 1)
    long_run = 8 + model.cfg.conv_lookahead + 4
    # slot 1: held from the first call; slot 3: opened at call 6 and held from its open; slot 5: held, closed, lifted;
    # slots 0, 2, 4: neighbours held at random; slot 6: a neighbour never held
    for b in range(B):
        if b != 3:
            srv.track([b], audio_of(1, 400, 10 * (b + 1)))
    srv.hold([1])
    schedule = {0: [], 2: [(1, False)], 4: [(1, True)], 5: [(1, False)], 8: [(5, True)], 9: [(1, True)],
                9 + long_run: [(1, False)], 12 + long_run: [(5, "close")], 14 + long_run: [(5, False)]}
    neighbours = [0, 2, 4]
    for i in range(24 + long_run):
        if i == 6:
            srv.s.open([3])
            srv.track([3], audio_of(1, 400, 30))
            srv.hold([3])
        if i == 7 + long_run // 2:
            srv.hold([3], False)
        for b, what in schedule.get(i, []):
            if what == "close":
                srv.close([b])
            elif srv.s.slot_states()[b] != SLOT_FREE:   # (closed without look-ahead: free at once)
                srv.hold([b], what)
        for b in neighbours:   # neighbours toggle their holds at random
            if rng.random() < 0.3:
                srv.hold([b], b not in srv.held)
        srv.call(int(rng.choice(SIZES)))
    states = srv.s.slot_states()
    assert states[1] == SLOT_OPEN and states[5] == SLOT_FREE
    srv.flush()
    for b in range(B):
        check_session(model, st, srv, [b])


@pytest.mark.parametrize("name", NAMES)
def test_held_rows_are_untouched(st, name):
    """snapshots of a held session before and after held calls are byte-identical; its NaN input changes nothing"""
    model = model_of(name, st)
    srv = Server(DfStream(model, st, batch=5), 2)
    srv.track([2], audio_of(1, 100, 40))
    for n in (3, 5, 2, 7):
        srv.call(n)
    srv.hold([2])
    before = srv.s.export([2], device="cpu")
    for n in (1, 7, 3, 5, 2, 2):
        srv.call(n)
    srv.s.hold([0, 4])   # neighbours leave the prefix around it
    srv.held |= {0, 4}
    srv.call(3)
    after = srv.s.export([2], device="cpu")
    assert torch.equal(before, after)
    srv.hold([2, 0, 4], False)
    for n in (2, 3):
        srv.call(n)
    srv.flush()
    check_session(model, st, srv, [2])


def test_linked_groups_and_rates(st):
    """a stereo mean group held and lifted as a unit, a partial list refused; sessions at 8, 16 and 44.1 kHz held on a
    mixed-rate handle and on a handle at one rate"""
    model = model_of("DeepFilterNet3", st)
    srv = Server(DfStream(model, st, batch=6, channels=1, reduce_mask="mean"), 3)
    srv.s.open_linked([1, 2])
    srv.track([1, 2], audio_of(2, 200, 50))
    srv.call(3)
    for bad in ([1], [2], [2, 3]):
        with pytest.raises(DfbError) as e:
            srv.s.hold(bad)
        assert e.value.code == DFB_ERR_INVALID
        assert not srv.s.held_slots().any()
    srv.hold([1, 2])
    for n in (2, 5, 1):
        srv.call(n)
    srv.hold([2, 1], False)
    srv.call(4)
    srv.flush()
    check_session(model, st, srv, [1, 2], reduce="mean")

    rates = (8000, 16000, 44100)
    mixed = Server(DfStream(model, st, batch=6, slot_rates=rates), 4)
    for i, sr in enumerate(rates):
        mixed.s.open([i], sr=sr)
        mixed.track([i], audio_of(1, 200, 60 + i, sr), sr)
    rng = np.random.default_rng(5)
    for k in range(20):
        for i in range(3):
            if rng.random() < 0.35:
                mixed.hold([i], i not in mixed.held)
        mixed.call(int(rng.choice(SIZES)))
    mixed.flush()
    for i, sr in enumerate(rates):
        check_session(model, st, mixed, [i], sr=sr)

    one = Server(DfStream(model, st, batch=4, sr=16000), 6)
    one.track([1], audio_of(1, 200, 70, 16000), 16000)
    for k, n in enumerate((2, 1, 3, 5, 2, 7, 1, 2, 3)):
        if k in (2, 5):
            one.hold([1], k == 2)
        one.call(n)
    one.flush()
    check_session(model, st, one, [1], sr=16000)


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet2"])
def test_settings_made_while_held(st, name):
    """a limit, a beta and LSNR thresholds set while held, twice, act from the session's next advancing call"""
    model = model_of(name, st)
    srv = Server(DfStream(model, st, batch=4), 7)
    srv.track([2], audio_of(1, 200, 80))
    dfn3 = name.startswith("DeepFilterNet3")
    sizes = [3, 2, 5, 1, 4, 2, 3]
    hooks = {}
    for i, n in enumerate(sizes):
        if i in (2, 4):
            srv.hold([2])
            srv.call(2)
            srv.s.set_atten_lim(6.0 if i == 2 else 20.0, slots=[2])
            srv.call(1)
            srv.s.set_atten_lim(12.0 if i == 2 else 3.0, slots=[2])
            if dfn3:
                srv.s.set_post_filter_beta(0.01 if i == 2 else 0.03, slots=[2])
                srv.s.set_lsnr_thresholds(-5.0, 25.0, 10.0 + i, slots=[2])
            srv.call(3)
            srv.hold([2], False)
            lim, beta, i_ = (12.0, 0.01, i) if i == 2 else (3.0, 0.03, i)

            def hook(s, slots, lim=lim, beta=beta, i_=i_):
                s.set_atten_lim(lim, slots=slots)
                if dfn3:
                    s.set_post_filter_beta(beta, slots=slots)
                    s.set_lsnr_thresholds(-5.0, 25.0, 10.0 + i_, slots=slots)
            hooks[len(srv.sizes[2])] = hook
        srv.call(n)
    srv.flush()
    check_session(model, st, srv, [2], hooks=hooks)


def test_runtime_gating(st):
    """runtime gating with gating neighbours; the handle's and the model's gating mode switched while a session is held,
    in both directions; export refuses sessions whose tails disagree"""
    model = model_of("DeepFilterNet3", st)
    th = (-10.0, 0.0, -5.0)
    srv = Server(DfStream(model, st, batch=5, gating_mode="runtime"), 8)
    srv.s.set_lsnr_thresholds(*th)
    srv.track([1], audio_of(1, 300, 90))
    srv.track([3], audio_of(1, 300, 91))
    modes = {}   # session call index -> mode the reference switches to

    def switch(mode):
        srv.s.set_gating_mode(mode)
        modes[len(srv.sizes[1])] = mode

    for n in (3, 5, 2):
        srv.call(n)
    srv.hold([1])
    srv.call(4)
    switch("apply")              # the handle leaves runtime mode while session 1 is held
    srv.call(3)
    srv.call(2)
    switch("runtime")            # ... and comes back as it resumes: 1 continues from its own tails, alone (per-row
    with pytest.raises(DfbError) as e:   # table), while 3 takes its tails from the halo; 3 ran in apply mode since
        srv.s.export([1, 3])
    assert e.value.code == DFB_ERR_INVALID
    srv.hold([1], False)
    for n in (3, 2):
        srv.call(n)
    srv.hold([1])
    switch("apply")
    srv.call(5)
    srv.hold([1], False)         # resumes in apply mode
    srv.call(3)
    srv.hold([1])
    srv.call(2)
    srv.s.set_gating_mode(None)  # the model's default, switched to runtime while held
    model.set_gating_mode("runtime")
    try:
        modes[len(srv.sizes[1])] = "runtime"
        srv.call(3)
        srv.hold([1], False)
        for n in (2, 7, 1):
            srv.call(n)
        srv.flush()
    finally:
        model.set_gating_mode("apply")
    got = srv.result([1])
    ref = reference_gated(model, st, torch.stack([srv.feed[1][0]]), srv.sizes[1], modes, th)
    assert same(got[0], ref[0]) and same(got[1], ref[1])


def reference_gated(model, st, audio, sizes, modes, th):
    """the session alone in runtime gating mode, switched to modes[i] before its call i"""
    srv = Server(DfStream(model, st, batch=1, gating_mode="runtime"), 0)
    srv.s.set_lsnr_thresholds(*th)
    srv.track([0], audio)
    for i, n in enumerate(sizes):
        if i in modes:
            srv.s.set_gating_mode(modes[i])
        srv.call(n)
    srv.flush()
    return srv.result([0])


@pytest.mark.parametrize("name", NAMES)
def test_close_flush_reset_open_export(st, name):
    model = model_of(name, st)
    # a held closing session drains only in calls it advances in; flush ends another held session as its own flush
    srv = Server(DfStream(model, st, batch=4), 9)
    srv.track([0], audio_of(1, 200, 100))
    srv.track([2], audio_of(1, 200, 101))
    for n in (3, 5):
        srv.call(n)
    srv.hold([0, 2])
    srv.call(2)
    srv.close([0])
    drains = srv.s.latency_frames > 0   # without look-ahead a closed slot is free at once
    assert srv.s.slot_states()[0] == (SLOT_CLOSING if drains else SLOT_FREE)
    for n in (7, 1):
        srv.call(n)
    assert srv.s.slot_states()[0] == (SLOT_CLOSING if drains else SLOT_FREE)
    if drains:
        srv.hold([0], False)
    srv.call(1)
    srv.flush()   # 2 is still held
    for b in (0, 2):
        check_session(model, st, srv, [b])
    # open over a held slot and reset clear the hold
    s = DfStream(model, st, batch=3)
    s.process(torch.zeros(3, 2 * s.hop))
    s.hold([1, 2])
    s.open([1])
    assert s.held_slots().tolist() == [False, False, True]
    s.reset()
    assert not s.held_slots().any()
    # a released export of a held session resumed on another handle
    src = Server(DfStream(model, st, batch=4), 10)
    src.track([1], audio_of(1, 200, 102))
    for n in (5, 3, 4, 2):
        src.call(n)
    src.hold([1])
    src.call(3)
    move_and_check(model, st, src, 1)


def move_and_check(model, st, src, b, lsnr_at=0):
    """export(release=True) of src's held session in slot b, resume on another handle that computes LSNR, a few calls and
    a flush there: audio and LSNR equal the session alone (LSNR requested from its call lsnr_at on)"""
    assert src.s.held_slots()[b]
    blob = src.s.export([b], release=True)
    assert not src.s.held_slots().any() and src.s.slot_states()[b] == SLOT_FREE
    dst = Server(DfStream(model, st, batch=3), 11)
    dst.s.close([2])
    dst.call(12)
    dst.s.resume(blob, [2])
    assert not dst.s.held_slots().any()
    dst.feed[2] = [src.feed[b][0], src.feed[b][1], MODEL_SR]
    dst.outs[2], dst.lsn[2], dst.sizes[2] = list(src.outs[b]), list(src.lsn[b]), list(src.sizes[b])
    for n in (2, 5):
        dst.call(n)
    dst.flush()
    check_session(model, st, dst, [2], lsnr_at=lsnr_at)


@pytest.mark.parametrize("name", NAMES)
def test_lsnr_started_after_a_hold(st, name):
    """a session held and resumed before the handle's LSNR head starts: its exported LSNR start is its own, so after a
    resume elsewhere its LSNR (DeepFilterNet2: the tail of frames still to be output included) equals the session alone"""
    model = model_of(name, st)
    src = Server(DfStream(model, st, batch=3), 12, lsnr=False)
    src.track([1], audio_of(1, 200, 110))
    for n in (3, 2):
        src.call(n)
    src.hold([1])
    for n in (7, 5, 7):
        src.call(n)
    src.hold([1], False)
    for n in (2, 3):
        src.call(n)
    lsnr_at = len(src.sizes[1])
    src.lsnr = True   # the handle's first LSNR request
    for n in (1, 4):
        src.call(n)
    src.hold([1])
    src.call(2)
    move_and_check(model, st, src, 1, lsnr_at=lsnr_at)


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet2"])
def test_spectral_handle(st, name):
    """held rows emit NaN / stage -1; the others equal process_spec of a single-session spectral handle"""
    model = model_of(name, st)
    B, F = 4, 481
    g = torch.Generator().manual_seed(12)
    s = DfStream(model, st, batch=B, spectral=True)
    ref = [DfStream(model, st, batch=1, spectral=True) for _ in range(B)]
    held = set()
    rng = np.random.default_rng(3)
    for k in range(16):
        if rng.random() < 0.4:
            b = int(rng.integers(B))
            s.hold([b], b not in held)
            (held.discard if b in held else held.add)(b)
        n = int(rng.choice(SIZES))
        x = torch.randn((B, n, F, 2), generator=g) * 0.05
        out = s.process_spec(torch.view_as_complex(x.contiguous()))
        for b in range(B):
            if b in held:
                assert torch.isnan(out.gains[b]).all() and (out.stage[b] == -1).all()
                continue
            r = ref[b].process_spec(torch.view_as_complex(x[b:b + 1].contiguous()))
            assert same(out.gains[b], r.gains[0]) and same(out.coefs[b], r.coefs[0]), (k, b)
            assert same(out.lsnr[b], r.lsnr[0]) and torch.equal(out.stage[b], r.stage[0]), (k, b)


def test_row_moves(st):
    """a call after hold changes launches k_slot_rows at most twice, a call without none; with 128 sessions, holding one
    in the middle of the prefix moves a bounded number of rows"""
    model = model_of("DeepFilterNet3", st)
    s = DfStream(model, st, batch=256)
    s.close(list(range(128, 256)))
    x = torch.randn(256, 2 * s.hop) * 0.1
    s.process(x)
    s.process(x)
    assert rows_moved(s) == 0

    def changed_then_unchanged():
        c1 = launches(lambda: s.process(x))
        moved = rows_moved(s)
        c2 = launches(lambda: s.process(x))
        assert rows_moved(s) == 0   # no change: no k_slot_rows launch
        assert (c1 - c2 == 0) == (moved == 0) and c1 - c2 <= 2
        return moved

    s.hold([64])
    assert 0 < changed_then_unchanged() <= 2
    s.hold([10, 20, 30, 40, 50])
    s.hold([64], False)
    assert changed_then_unchanged() <= 2 * 6
    s.hold([10, 20, 30, 40, 50], False)
    assert changed_then_unchanged() <= 2 * 5


def test_refusals_change_nothing(st):
    model = model_of("DeepFilterNet3", st)
    s = DfStream(model, st, batch=4)
    s.close([3])
    s.process(torch.zeros(4, 3 * s.hop))
    assert s.slot_states()[3] == SLOT_FREE
    s.hold([1])
    for bad in ([3], [0, 3]):          # a free slot
        with pytest.raises(DfbError) as e:
            s.hold(bad)
        assert e.value.code == DFB_ERR_INVALID
    with pytest.raises(ValueError):
        s.hold([5])
    with pytest.raises(ValueError):
        s.hold([0, 0])
    assert s.held_slots().tolist() == [False, True, False, False]
    fixed = DfStream(model, st, batch=4, channels=2, reduce_mask="mean")
    with pytest.raises(DfbError) as e:
        fixed.hold([0, 1])
    assert e.value.code == DFB_ERR_UNSUPPORTED
    assert not fixed.held_slots().any()
