"""GPU: session export / import (DfStream.export / resume, dfb_stream_export_sessions / import_sessions).  A session is fed
in random call sizes, exported at a call boundary k and resumed elsewhere: the source's outputs before k, then the
destination's from k on and its flush, equal a single-session DfStream fed the same audio in the same call sizes, bit for
bit.  Elsewhere is another slot of the same handle, another handle with other neighbours, batch size and a clock 1000 hops
ahead, a fresh process and a second GPU.  Settings, runtime gating, LSNR rows, linked groups and sample rates travel with
the session; a snapshot disturbs nothing; 128 sessions move in one kernel launch per direction; refused imports change
nothing."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, libdf
from deepfilternet_b200._lib import DFB_ERR_INVALID, DFB_ERR_UNSUPPORTED, DfbError
from deepfilternet_b200.config import load_config
from deepfilternet_b200.streaming import MODEL_SR, SLOT_FREE, session_info
from deepfilternet_b200.weights import random_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "tests", "golden", "models")
SEEDS = {"DeepFilterNet3": 11, "DeepFilterNet3_ll": 14, "DeepFilterNet2": 12, "DeepFilterNet2_ll": 15}   # oracle/synth_models.py
SIZES = [1, 2, 3, 5, 7]


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_models = {}


def model_of(name, st, seed=None):
    key = (name, seed)
    if key not in _models:
        cfg = load_config(os.path.join(MODELS, name, "config.ini"), env={})
        _models[key] = DfNet(cfg, random_state_dict(cfg, seed=SEEDS[name] if seed is None else seed), st)
    return _models[key]


def launches(fn):
    n0 = _lib.lib().dfb_kernel_launches()
    fn()
    return _lib.lib().dfb_kernel_launches() - n0


def same(a, b):
    """bit for bit, NaN where the other is NaN"""
    if a.shape != b.shape:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def sizes_to(total, rng):
    out = []
    while sum(out) < total:
        out.append(min(int(rng.choice(SIZES)), total - sum(out)))
    return out


class Server:
    """A handle with neighbour traffic: every open slot that carries no tracked session is fed seeded noise.  Tracked
    sessions (slot -> [audio at its rate, position, rate]) read their own audio and collect their own outputs."""

    def __init__(self, s, seed, lsnr=False):
        self.s, self.g, self.lsnr = s, torch.Generator().manual_seed(seed), lsnr
        self.feed, self.outs, self.lsn, self.raw = {}, {}, {}, []

    def track(self, slots, audio, sr=MODEL_SR, pos=0):
        for c, b in enumerate(slots):
            self.feed[b] = [audio[c], pos, sr]
            self.outs[b], self.lsn[b] = [], []

    def untrack(self, slots):
        pos = self.feed[slots[0]][1]
        for b in slots:
            del self.feed[b]
        return pos

    def call(self, n):
        B, w = self.s.batch, self.s.hop
        x = torch.randn((B, n * w), generator=self.g) * 0.1
        for b, f in self.feed.items():
            k = n * f[2] // 100
            x[b] = 0
            x[b, :k] = f[0][f[1]:f[1] + k]
            f[1] += k
        r = self.s.process(x, return_lsnr=self.lsnr)
        out, ls = r if self.lsnr else (r, None)
        self.raw.append(out.cpu())
        for b, f in self.feed.items():
            self.outs[b].append(out[b, :n * f[2] // 100])
            if ls is not None:
                self.lsn[b].append(ls[b])

    def flush(self):
        r = self.s.flush(return_lsnr=self.lsnr)
        out, ls = r if self.lsnr else (r, None)
        self.raw.append(out.cpu())
        for b, f in self.feed.items():
            L = self.s.rate_latency(f[2])[0] if self.s.registered_rates else self.s.latency_frames
            self.outs[b].append(out[b, :L * f[2] // 100])
            if ls is not None:
                self.lsn[b].append(ls[b, :L])

    def result(self, slots):
        return (torch.stack([torch.cat(self.outs[b]) for b in slots]),
                torch.stack([torch.cat(self.lsn[b]) for b in slots]) if self.lsnr else None)


def reference(model, st, audio, sizes, sr=MODEL_SR, reduce=None, lsnr=False, hooks=None, **kw):
    """the session alone: a single-session handle at its rate fed the same call sizes, then flushed"""
    C = audio.shape[0]
    extra = dict(channels=C, reduce_mask=reduce) if C > 1 else {}
    if sr != MODEL_SR:
        extra["sr"] = sr
    srv = Server(DfStream(model, st, batch=C, **extra, **kw), 0, lsnr)
    srv.track(list(range(C)), audio, sr)
    for i, n in enumerate(sizes):
        if hooks and i in hooks:
            hooks[i](srv.s, list(range(C)))
        srv.call(n)
    srv.flush()
    return srv.result(list(range(C)))


def make_server(model, st, B, warm, seed, lsnr=False, free=(), setup=None, **kw):
    """B slots fed noise for `warm` hops; the slots in `free` are closed at the start and free by then"""
    srv = Server(DfStream(model, st, batch=B, **kw), seed, lsnr)
    if setup:
        setup(srv.s)
    if free:
        srv.s.close(list(free))
    srv.call(warm)
    assert all(srv.s.slot_states()[list(free)] == SLOT_FREE) if free else True
    return srv


def migrate(model, st, name, k, release, where, H=16, C=1, reduce=None, sr=MODEL_SR, lsnr=False, hooks=None, pending=None,
            src_kw=None, dst_kw=None, dst_setup=None, seed=0):
    """Runs a session of H hops whose export falls at hop k; returns (got, ref) as (audio, lsnr) pairs."""
    rng = np.random.default_rng(seed + 100 * k)
    sizes = sizes_to(k, rng) + sizes_to(H - k, rng)
    nb = len(sizes_to(k, np.random.default_rng(seed + 100 * k)))
    audio = synth_audio(C, H * sr // 100, seed=300 + seed, sr=sr)
    src_kw, dst_kw = dict(src_kw or {}), dict(dst_kw or {})
    ref_hooks = dict(hooks or {})
    if pending:   # a setting made after the last call before the split, which takes effect at the first one after it
        ref_hooks[nb] = pending
    ref = reference(model, st, audio, sizes, sr, reduce, lsnr, ref_hooks, **{k_: v for k_, v in src_kw.items()
                                                                               if k_ == "gating_mode"})
    src = make_server(model, st, 6, 12, seed=1 + seed, lsnr=lsnr, free=(4, 5), reduce_mask=reduce, **src_kw)
    slots = [0, 1][:C]
    open_kw = dict(sr=sr) if src.s.registered_rates else {}
    if C > 1:
        src.s.open_linked(slots, **open_kw)
    else:
        src.s.open(slots, **open_kw)
    src.track(slots, audio, sr)
    for i, n in enumerate(sizes[:nb]):
        if hooks and i in hooks:
            hooks[i](src.s, slots)
        src.call(n)
    if pending:
        pending(src.s, slots)
    blob = src.s.export(slots, release=release)
    pos = src.untrack(slots)
    if where == "slot":          # another slot of the same handle
        dst, dslots = src, [5, 4][:C]
        dst.s.resume(blob, dslots)
    elif where == "handle":      # another batch size, other neighbours, a clock 1000 hops ahead
        dst = make_server(model, st, 7, 1000 + sum(sizes[:nb]), seed=9 + seed, lsnr=lsnr, free=(5, 2), reduce_mask=reduce,
                          setup=dst_setup, **dst_kw)
        dslots = [5, 2][:C]
        dst.s.resume(blob, dslots)
    else:
        raise ValueError(where)
    dst.track(dslots, audio, sr, pos)
    for n in sizes[nb:]:
        dst.call(n)
    dst.flush()
    head = [torch.cat(src.outs[b][:len(sizes[:nb])]) for b in slots]
    tail = [torch.cat(dst.outs[b]) for b in dslots]
    got_a = torch.stack([torch.cat([h, t]) for h, t in zip(head, tail)])
    got_l = None
    if lsnr:
        got_l = torch.stack([torch.cat([torch.cat(src.lsn[b][:nb]), torch.cat(dst.lsn[d])]) for b, d in zip(slots, dslots)])
    return (got_a, got_l), ref, (src, blob, slots, audio, sizes, nb)


def check(got, ref, what=""):
    assert same(got[0], ref[0]), (what, (got[0] - ref[0]).abs().max().item() if got[0].shape == ref[0].shape else got[0].shape)
    if got[1] is not None:
        assert same(got[1], ref[1]), what


# ------------------------------------------------------------------------------------------ split anywhere ----
@pytest.mark.parametrize("name", list(SEEDS))
@pytest.mark.parametrize("where", ["slot", "handle"])
@pytest.mark.parametrize("release", [False, True])
def test_split_anywhere(st, name, where, release):
    model = model_of(name, st)
    H = 16
    for k in (1, 8, H - 1):
        got, ref, _ = migrate(model, st, name, k, release, where, H=H)
        check(got, ref, (name, where, release, k))


def test_snapshot_disturbs_nothing(st):
    """a snapshot mid-stream: the source session and every neighbour give the bits of a run without it"""
    model = model_of("DeepFilterNet3", st)
    outs = []
    for snap in (False, True):
        srv = make_server(model, st, 6, 12, seed=4, lsnr=True, free=(5,))
        srv.s.open([0])
        audio = synth_audio(1, 20 * 480, seed=77)
        srv.track([0], audio)
        res = []
        for i, n in enumerate([3, 1, 5, 2, 7, 2]):
            if snap and i == 3:
                blob = srv.s.export([0])
                assert session_info(blob).sessions[0].age == 9
            srv.g = torch.Generator().manual_seed(50 + i)
            x = torch.randn((6, n * 480), generator=srv.g) * 0.1
            x[0] = audio[0, sum([3, 1, 5, 2, 7, 2][:i]) * 480:][:n * 480]
            res.append(srv.s.process(x, return_lsnr=True))
        res.append(srv.s.flush(return_lsnr=True))
        outs.append(res)
    for (a, la), (b, lb) in zip(*outs):
        assert torch.equal(a, b) and same(la, lb)


# ------------------------------------------------------------------------------------------ state that travels ----
def test_settings_travel(st):
    """per-slot limit, beta and thresholds set before the split, changed in the call just before it and between that call
    and the export"""
    model = model_of("DeepFilterNet3", st)

    def first(s, slots):
        s.set_atten_lim(12.0, slots=slots)
        s.set_post_filter_beta(0.03, slots=slots)

    def last(s, slots):
        s.set_atten_lim(6.0, slots=slots)
        s.set_lsnr_thresholds(-15.0, 35.0, 25.0, slots=slots)

    def pending(s, slots):
        s.set_atten_lim(20.0, slots=slots)
        s.set_post_filter_beta(0.0, slots=slots)

    for where in ("slot", "handle"):
        k = 10
        nb = len(sizes_to(k, np.random.default_rng(100 * k)))
        got, ref, _ = migrate(model, st, "DeepFilterNet3", k, True, where, H=20, lsnr=True, hooks={0: first, nb - 1: last},
                              pending=pending)
        check(got, ref, where)


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet3_ll"])
def test_runtime_gating_travels(st, name):
    model = model_of(name, st)
    probe = reference(model, st, synth_audio(1, 20 * 480, seed=300), [20], lsnr=True)[1]
    q = torch.nanquantile(probe[0], torch.tensor([0.3, 0.8, 0.55])).tolist()

    def gate(s, slots):
        s.set_lsnr_thresholds(q[0], q[1], q[2], slots=slots)

    def gate_all(s):          # the destination's neighbours gate too: their last call kept the decoder tails
        s.set_lsnr_thresholds(q[0], q[1], q[2])

    kw = dict(gating_mode="runtime")
    for where in ("slot", "handle"):
        got, ref, _ = migrate(model, st, name, 9, True, where, H=20, lsnr=True, hooks={0: gate}, src_kw=kw,
                              dst_kw=dict(kw), dst_setup=gate_all, seed=3)
        check(got, ref, where)


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet2"])
def test_lsnr_rows_travel(st, name):
    model = model_of(name, st)
    for k in (1, 9):
        got, ref, _ = migrate(model, st, name, k, True, "handle", H=18, lsnr=True, seed=5)
        check(got, ref, k)


@pytest.mark.parametrize("reduce", ["mean", "max"])
def test_linked_group_travels(st, reduce):
    model = model_of("DeepFilterNet3", st)
    for where in ("slot", "handle"):
        got, ref, (src, blob, *_) = migrate(model, st, "DeepFilterNet3", 7, True, where, H=16, C=2, reduce=reduce, seed=6)
        info = session_info(blob)
        assert [(x.channels, x.reduce_mask) for x in info.sessions] == [(2, reduce)]
        check(got, ref, where)


@pytest.mark.parametrize("sr", [8000, 16000, 44100])
def test_rates_between_mixed_and_single_handles(st, sr):
    """a session at sr moves from a mixed-rate handle to a handle at sr and back"""
    model = model_of("DeepFilterNet3", st)
    mixed = dict(slot_rates=(8000, 16000, 44100))
    single = dict(sr=sr)
    for a, b in ((mixed, single), (single, mixed)):
        got, ref, _ = migrate(model, st, "DeepFilterNet3", 6, True, "handle", H=14, sr=sr, src_kw=a, dst_kw=b, seed=7)
        check(got, ref, (sr, a, b))


def test_48k_session_mixed_to_plain(st):
    model = model_of("DeepFilterNet3", st)
    got, ref, _ = migrate(model, st, "DeepFilterNet3", 6, True, "handle", H=14, src_kw=dict(slot_rates=(16000,)), seed=8)
    check(got, ref)


# ------------------------------------------------------------------------------------------ elsewhere ----
CHILD = r"""
import sys, torch
from deepfilternet_b200 import DfNet, DfStream, libdf
from deepfilternet_b200.config import load_config
from deepfilternet_b200.weights import random_state_dict
cfg_path, seed, blob_path, audio_path, sizes, out_path = sys.argv[1], int(sys.argv[2]), sys.argv[3], sys.argv[4], sys.argv[5], sys.argv[6]
st = libdf.DF(48000, 960, 480, 32, 2)
cfg = load_config(cfg_path, env={})
model = DfNet(cfg, random_state_dict(cfg, seed=seed), st)
s = DfStream(model, st, batch=3)
s.flush()                                   # a new handle has every slot open
s.resume(torch.load(blob_path), [1])
audio = torch.load(audio_path)
outs, pos = [], 0
for n in map(int, sizes.split(",")):
    x = torch.zeros((3, n * 480))
    x[1] = audio[pos:pos + n * 480]
    pos += n * 480
    outs.append(s.process(x)[1])
outs.append(s.flush()[1])
torch.save(torch.cat(outs), out_path)
"""


def test_resume_in_a_fresh_process(st, tmp_path):
    name = "DeepFilterNet3"
    model = model_of(name, st)
    rng = np.random.default_rng(11)
    H, k = 18, 8
    sizes = sizes_to(k, rng) + sizes_to(H - k, rng)
    nb = len(sizes_to(k, np.random.default_rng(11)))
    audio = synth_audio(1, H * 480, seed=91)
    ref = reference(model, st, audio, sizes)[0]
    srv = make_server(model, st, 4, 12, seed=2)
    srv.s.open([2])
    srv.track([2], audio)
    for n in sizes[:nb]:
        srv.call(n)
    blob = srv.s.export([2], release=True, device="cpu")
    torch.save(blob, tmp_path / "blob.pt")
    torch.save(audio[0, k * 480:].clone(), tmp_path / "audio.pt")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(p for p in sys.path if p))
    subprocess.run([sys.executable, "-c", CHILD, os.path.join(MODELS, name, "config.ini"), str(SEEDS[name]),
                    str(tmp_path / "blob.pt"), str(tmp_path / "audio.pt"), ",".join(map(str, sizes[nb:])),
                    str(tmp_path / "out.pt")], check=True, env=env, cwd=ROOT, timeout=600)
    got = torch.cat([torch.cat(srv.outs[2]), torch.load(tmp_path / "out.pt")])
    assert torch.equal(got, ref[0])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one CUDA device: the second-GPU resume needs two")
def test_resume_on_a_second_gpu(st):
    name = "DeepFilterNet3"
    model = model_of(name, st)
    with torch.cuda.device(1):
        st1 = libdf.DF(48000, 960, 480, 32, 2)
        cfg = load_config(os.path.join(MODELS, name, "config.ini"), env={})
        model1 = DfNet(cfg, random_state_dict(cfg, seed=SEEDS[name]), st1)
    rng = np.random.default_rng(12)
    sizes = sizes_to(6, rng) + sizes_to(8, rng)
    nb = len(sizes_to(6, np.random.default_rng(12)))
    audio = synth_audio(1, 14 * 480, seed=92)
    ref = reference(model, st, audio, sizes)[0]
    srv = make_server(model, st, 3, 12, seed=3)
    srv.s.open([0])
    srv.track([0], audio)
    for n in sizes[:nb]:
        srv.call(n)
    blob = srv.s.export([0], release=True)
    pos = srv.untrack([0])
    dst = make_server(model1, st1, 2, 30, seed=4, free=(1,))
    dst.s.resume(blob, [1])
    dst.track([1], audio, pos=pos)
    for n in sizes[nb:]:
        dst.call(n)
    dst.flush()
    assert torch.equal(torch.cat([torch.cat(srv.outs[0]), torch.cat(dst.outs[1])])[None], ref[0])


# ------------------------------------------------------------------------------------------ one launch per direction ----
def test_128_sessions_one_launch_each_way(st):
    """128 sessions move in one pack and one unpack launch, through a device and a host blob; the handles' next call
    follows at once on their own stream (flush takes the host path) and finds every row in place"""
    model = model_of("DeepFilterNet3", st)
    src = make_server(model, st, 128, 12, seed=5)
    slots = list(range(128))
    dst = DfStream(model, st, batch=256)
    dst.flush()
    dst2 = DfStream(model, st, batch=256)
    dst2.flush()
    blob, host = None, None

    def ex(dev):
        nonlocal blob, host
        if dev is None:
            blob = src.s.export(slots)
        else:
            host = src.s.export(slots, device=dev)

    assert launches(lambda: ex(None)) == 1
    assert launches(lambda: dst.resume(blob, list(range(64, 192)))) == 1
    tail = dst.flush()                                   # at once, on the handle's own stream
    assert launches(lambda: ex("cpu")) == 1
    assert launches(lambda: dst2.resume(host, list(range(128, 256)))) == 1
    tail2 = dst2.flush()
    assert session_info(blob).rows == 128 and len(session_info(host).sessions) == 128
    assert torch.equal(blob.cpu(), host)                 # nothing ran between the two exports
    ref = src.s.flush()                                  # the unmoved sessions' tails
    assert torch.equal(tail[64:192], ref) and torch.equal(tail2[128:], ref)
    assert tail[:64].abs().max().item() == 0 and tail2[:128].abs().max().item() == 0


def test_unaligned_blob_view(st):
    """a blob stored at an odd offset of a larger buffer resumes as the blob itself"""
    model = model_of("DeepFilterNet3", st)
    src = make_server(model, st, 2, 12, seed=6)
    blob = src.s.export([0])
    buf = torch.zeros(blob.numel() + 3, dtype=torch.uint8, device=blob.device)
    buf[3:] = blob
    outs = []
    for b in (blob, buf[3:]):
        d = DfStream(model, st, batch=2)
        d.flush()
        d.resume(b, [1])
        outs.append(torch.cat([d.process(torch.ones(2, 3 * 480) * 0.01), d.flush()], 1))
    assert torch.equal(outs[0], outs[1])
    a = np.array([0], np.int32)
    d = DfStream(model, st, batch=1)
    d.flush()
    assert _lib.lib().dfb_stream_import_sessions(d._h, a.ctypes.data_as(_lib.C.POINTER(_lib.C.c_int32)), 1, buf.data_ptr() + 3,
                                                 torch.cuda.current_stream().cuda_stream) == DFB_ERR_INVALID


@pytest.mark.parametrize("name", ["DeepFilterNet3", "DeepFilterNet2"])
def test_unsettled_sources(st, name):
    """sources whose clock has not settled -- a new handle (clock below 8 + look-ahead frames) and one just flushed, whose
    DNN frames still trail the flush -- export sessions that continue exactly in a settled handle and in an idle one"""
    model = model_of(name, st)
    H = 12
    for kind in ("new", "flushed"):
        for k in (1, 3):
            for dst_kind in ("settled", "idle"):
                rng = np.random.default_rng(k)
                sizes = sizes_to(k, rng) + sizes_to(H - k, rng)
                nb = len(sizes_to(k, np.random.default_rng(k)))
                audio = synth_audio(1, H * 480, seed=400 + k)
                ref = reference(model, st, audio, sizes, lsnr=True)
                src = Server(DfStream(model, st, batch=3), seed=k, lsnr=True)
                if kind == "flushed":
                    src.call(15)
                    src.s.flush()
                    src.s.open([1])                      # a neighbour opened with the session
                src.s.open([0])
                src.track([0], audio)
                for n in sizes[:nb]:
                    src.call(n)
                blob = src.s.export([0], release=True)
                pos = src.untrack([0])
                if dst_kind == "settled":
                    dst = make_server(model, st, 4, 30, seed=7, lsnr=True, free=(3,))
                else:
                    dst = Server(DfStream(model, st, batch=2), seed=8, lsnr=True)
                    dst.s.flush()
                dslot = dst.s.batch - 1
                dst.s.resume(blob, [dslot])
                dst.track([dslot], audio, pos=pos)
                for n in sizes[nb:]:
                    dst.call(n)
                dst.flush()
                got = (torch.cat([torch.cat(src.outs[0][:nb]), torch.cat(dst.outs[dslot])])[None],
                       torch.cat([torch.cat(src.lsn[0][:nb]), torch.cat(dst.lsn[dslot])])[None])
                check(got, ref, (kind, k, dst_kind))


# ------------------------------------------------------------------------------------------ refusals ----
def refused(code, fn, text=None):
    with pytest.raises(DfbError) as e:
        fn()
    assert e.value.code == code, e.value
    if text:
        assert text in str(e.value), e.value


def test_refusals_change_nothing(st):
    """each refusal returns its code, and both handles' following outputs equal those of a run without the attempts"""
    name = "DeepFilterNet3"
    model = model_of(name, st)
    other = model_of(name, st, seed=99)
    audio = synth_audio(2, 20 * 480, seed=31)
    runs = []
    for attempt in (False, True):
        src = make_server(model, st, 5, 12, seed=21, free=(4,), reduce_mask="mean")
        dst = make_server(model, st, 4, 40, seed=22, free=(3, 2), reduce_mask="mean")
        src.s.open_linked([0, 1])
        src.track([0, 1], audio)
        src.call(5)
        dst.call(1)
        if attempt:
            good = src.s.export([0, 1])
            refused(DFB_ERR_INVALID, lambda: src.s.export([0]), "list all")           # half a group
            refused(DFB_ERR_INVALID, lambda: src.s.export([1, 0]), "channel 0")      # not in channel order
            refused(DFB_ERR_INVALID, lambda: src.s.export([4]), "free")
            refused(DFB_ERR_INVALID, lambda: dst.s.resume(good, [3, 0]), "not free")  # an occupied slot
            refused(DFB_ERR_INVALID, lambda: DfStream(other, st, batch=2).resume(good, [0, 1]), "fingerprint")
            st1 = libdf.DF(48000, 960, 480, 32, 1)   # the same weights on other ERB bands
            cfg = load_config(os.path.join(MODELS, name, "config.ini"), env={})
            bands = DfNet(cfg, random_state_dict(cfg, seed=SEEDS[name]), st1)
            assert not np.array_equal(st1.erb_widths(), st.erb_widths())
            refused(DFB_ERR_INVALID, lambda: DfStream(bands, st1, batch=2, reduce_mask="mean").resume(good, [0, 1]), "fingerprint")
            bad = good.clone()
            bad[16:20] = torch.from_numpy(np.array([44100], "<i4").view(np.uint8)).to(bad.device)
            refused(DFB_ERR_INVALID, lambda: dst.s.resume(bad, [3, 2]), "DSP state")
            flip = good.clone()
            flip[0] ^= 1
            refused(DFB_ERR_INVALID, lambda: dst.s.resume(flip, [3, 2]), "magic")
            refused(DFB_ERR_INVALID, lambda: dst.s.resume(good[:-4], [3, 2]), "bytes")
            a = np.array([3, 2], np.int32)
            ptr = a.ctypes.data_as(_lib.C.POINTER(_lib.C.c_int32))
            for off, val in ((0, 0x45), (4, 7)):   # the C ABI's own checks of magic and version, without the Python parse
                hb = good.cpu()
                hb[off] = val
                assert _lib.lib().dfb_stream_import_sessions_host(dst.s._h, ptr, 2, hb.data_ptr()) == DFB_ERR_INVALID
            runtime = DfStream(model, st, batch=2, gating_mode="runtime")
            runtime.flush()
            refused(DFB_ERR_INVALID, lambda: runtime.resume(good, [0, 1]), "gating mode")
            plain = DfStream(model, st, batch=2)
            plain.flush()
            refused(DFB_ERR_INVALID, lambda: plain.resume(good, [0, 1]), "reduction")
            closing = make_server(model, st, 3, 20, seed=23, free=(2,), reduce_mask="mean")
            closing.s.close([1])
            refused(DFB_ERR_INVALID, lambda: closing.s.resume(good, [2, 1]), "not free")   # a closing slot
            refused(DFB_ERR_INVALID, lambda: closing.s.export([1]), "closing")
        src.call(3)
        dst.call(3)
        src.flush()
        dst.flush()
        runs.append((src.raw, dst.raw))
    for a, b in zip(runs[0][0] + runs[0][1], runs[1][0] + runs[1][1]):
        assert torch.equal(a, b)


def test_rate_and_handle_refusals(st):
    """an unregistered rate, a spectral handle and v1 are refused, and every handle's next outputs are those of a run
    without the attempts"""
    model = model_of("DeepFilterNet3", st)
    spec_in = torch.randn((2, 4, 481), generator=torch.Generator().manual_seed(3), dtype=torch.complex64) * 0.1
    runs = []
    for attempt in (False, True):
        src = make_server(model, st, 3, 12, seed=1, slot_rates=(16000,))
        src.s.open([0], sr=16000)
        src.call(3)
        plain = make_server(model, st, 2, 12, seed=2, free=(1,))
        other = make_server(model, st, 2, 12, seed=3, free=(1,), sr=8000)
        spec = DfStream(model, st, batch=2, spectral=True)
        spec.process_spec(spec_in)
        if attempt:
            blob = src.s.export([0])
            assert session_info(blob).sessions[0].sr == 16000
            refused(DFB_ERR_INVALID, lambda: plain.s.resume(blob, [1]), "16000 Hz")
            refused(DFB_ERR_INVALID, lambda: other.s.resume(blob, [1]), "16000 Hz")
            refused(DFB_ERR_UNSUPPORTED, lambda: spec.export([0]))
            refused(DFB_ERR_UNSUPPORTED, lambda: spec.resume(blob, [1]))
        for srv in (src, plain, other):
            srv.call(4)
            srv.flush()
        sp = spec.process_spec(spec_in)
        runs.append([t for srv in (src, plain, other) for t in srv.raw] + [t for t in sp if t.is_floating_point()] + [sp.stage])
    for a, b in zip(*runs):
        assert same(a, b)
    cfg = load_config(os.path.join(MODELS, "DeepFilterNet", "config.ini"), env={})
    v1 = DfNet(cfg, random_state_dict(cfg, seed=13), st)
    refused(DFB_ERR_UNSUPPORTED, lambda: DfStream(v1, st, batch=1))   # v1 has no streaming handle, nothing to export
