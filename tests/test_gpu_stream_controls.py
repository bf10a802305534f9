"""GPU: per-slot attenuation limit and post-filter beta (DfStream.set_atten_lim / set_post_filter_beta,
dfb_stream_set_atten_lim / _post_filter_beta) and the LSNR output of process / flush (return_lsnr, dfb_stream_*_lsnr).

* Constant settings: on a seeded 8-slot server every session has its own limit and beta; it must equal a fresh
  single-stream handle with that limit and a model whose post filter is set to that beta, and enhance(pad=False).
* Changes inside a session: the output must equal a float64 restatement that applies each frame's own setting to
  DfNet.forward's spectra, where a setting made between two calls covers every frame whose output starts in the next
  call (hop 0 of that call = the new setting's head of its frame + the previous setting's tail of the frame before).
* LSNR: the value of the frame each output hop carries, NaN where a hop carries none."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dsp_ref64 as R
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.streaming import SLOT_FREE
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TOL = 1e-6          # RMS, as the other streaming tests
EDGE = 4800         # first / last 100 ms of a session, checked on their own
SIZES = [1, 2, 3, 7, 40]
LIMS = [None, 6.0, 12.0, 40.0]
BETAS = [0.0, 0.02, 0.05]
# LSNR in dB against DfNet.forward (whole signal in one window) and between two streaming handles.  The worst |error|
# measured on an H100 80GB HBM3 (400 W power limit) is 0 in every test below: the streaming windows compute the LSNR head
# on the same inputs.  One frame off is 0.12-0.32 dB with these weights, three orders above the tolerance.
LSNR_TOL_FORWARD = 1e-4
LSNR_TOL_STREAM = 1e-4


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


_MODELS = {}


def model_of(st, kind, beta=0.0):
    """The same seeded weights with the post filter off (beta 0) or on with pf_beta = beta."""
    key = (kind, beta)
    if key not in _MODELS:
        cfg = cfg_of(kind, mask_pf=beta > 0, pf_beta=beta if beta > 0 else 0.02)
        _MODELS[key] = DfNet(cfg, random_state_dict(cfg_of(kind), seed=101), st)
    return _MODELS[key]


def single_stream(model, st, audio, sizes, atten=None, lsnr=False):
    """A fresh one-stream handle fed `audio` in calls of `sizes` hops and flushed: (output, lsnr or None)."""
    r = DfStream(model, st, batch=1, atten_lim_db=atten)
    outs, ls, pos = [], [], 0
    for n in sizes:
        y = r.process(audio[None, pos * HOP:(pos + n) * HOP], return_lsnr=lsnr)
        outs.append((y[0] if lsnr else y)[0])
        if lsnr:
            ls.append(y[1][0])
        pos += n
    y = r.flush(return_lsnr=lsnr)
    outs.append((y[0] if lsnr else y)[0])
    if lsnr:
        ls.append(y[1][0])
    return torch.cat(outs), (torch.cat(ls) if lsnr else None)


# ------------------------------------------------------------------------------------------------ constant settings ----
class Session:
    def __init__(self, slot, seed, atten, beta):
        self.slot, self.seed, self.atten, self.beta = slot, seed, atten, beta
        self.sizes, self.outs, self.lsnr = [], [], []
        self.closing, self.tail_left, self.dropped = False, 0, False


def schedule(seed, n_random):
    calls = [([], [7], 1), ([7], [], 1), ([], [3, 7], 2), ([6], [], 3), ([3], [2], 1), ([2], [], 7), ([5], [0], 40)]
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


@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2"])
def test_constant_settings_equal_fresh_streams(st, kind):
    """Each session of a seeded 8-slot server gets its own limit (off, 6, 12, 40 dB) and, for the DeepFilterNet3
    topologies, beta (0, 0.02, 0.05), set before the first call or right after its open.  Its audio equals a fresh
    single-stream handle with that limit on a model whose post filter has that beta, at RMS <= 1e-6 (also over its first
    and last 100 ms), and enhance(pad=False, atten_lim_db=...) delayed by the latency.  Its LSNR equals the fresh
    handle's (LSNR_TOL_STREAM; worst error measured on an H100 80GB HBM3: 0 dB), and is NaN on free slots, before a
    session's first output frame and past a tail."""
    model = model_of(st, kind)
    B = 8
    calls = schedule(seed=11, n_random=24)
    total_hops = sum(n for _, _, n in calls) + 1
    s = DfStream(model, st, batch=B)
    lat = s.latency_frames
    betas = BETAS if kind != "dfn2" else [None]
    sessions, live, count = [], {}, [0]

    def new_session(b):
        i = count[0]
        count[0] += 1
        ses = Session(b, 3000 + i, LIMS[i % len(LIMS)], betas[(i // len(LIMS)) % len(betas)])
        ses.src = synth_audio(1, total_hops * HOP, seed=ses.seed)[0]
        live[b] = ses
        sessions.append(ses)
        s.set_atten_lim(ses.atten, [b])
        if ses.beta is not None:
            s.set_post_filter_beta(ses.beta, [b])

    for b in range(B):
        new_session(b)
    noise = torch.Generator().manual_seed(17)
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
                            del live[b]
            if opens:
                s.open(opens)
                for b in opens:
                    if b in live:
                        live[b].dropped = True
                    new_session(b)
            x = torch.randn((B, n * HOP), generator=noise) * 0.3
            for b, ses in live.items():
                if not ses.closing:
                    pos = sum(ses.sizes)
                    x[b] = ses.src[pos * HOP:(pos + n) * HOP]
                    ses.sizes.append(n)
            y, ls = s.process(x.cuda() if i % 2 else x, return_lsnr=True)
            y, ls = y.cpu(), ls.cpu()
            assert ls.shape == (B, n) and ls.dtype == torch.float32
        else:
            for b, ses in list(live.items()):
                if not ses.closing:
                    ses.closing, ses.tail_left = True, lat
                if lat == 0:
                    del live[b]
            y, ls = s.flush(return_lsnr=True)
            n = lat
        used = set()
        for b, ses in list(live.items()):
            if not ses.closing:
                ses.outs.append(y[b]); ses.lsnr.append(ls[b])
            elif ses.tail_left > 0:
                k = min(n, ses.tail_left)
                ses.outs.append(y[b, :k * HOP]); ses.lsnr.append(ls[b, :k])
                assert torch.isnan(ls[b, k:]).all(), ("LSNR past the tail", i, b)
                ses.tail_left -= k
                if ses.tail_left == 0:
                    del live[b]
            used.add(b)
        for b in range(B):
            if b not in used and n:
                assert torch.isnan(ls[b]).all(), ("free slot LSNR", i, b)
    assert not live
    checked = 0
    for ses in sessions:
        if not ses.sizes:
            continue
        got, gl = torch.cat(ses.outs), torch.cat(ses.lsnr)
        ref, rl = single_stream(model_of(st, kind, ses.beta or 0.0), st, ses.src, ses.sizes, ses.atten, lsnr=True)
        if ses.dropped:
            ref, rl = ref[:got.numel()], rl[:gl.numel()]
        assert got.shape == ref.shape and gl.shape == rl.shape
        assert rms(got, ref) < TOL, (ses.slot, ses.atten, ses.beta, rms(got, ref))
        assert rms(got[:EDGE], ref[:EDGE]) < TOL and rms(got[-EDGE:], ref[-EDGE:]) < TOL
        assert torch.equal(torch.isnan(gl), torch.isnan(rl)) and torch.isnan(gl[:lat]).all()
        ok = ~torch.isnan(rl)
        assert (gl[ok] - rl[ok]).abs().max().item() <= LSNR_TOL_STREAM if ok.any() else True
        if not ses.dropped:
            T = sum(ses.sizes) * HOP
            one = enhance(model_of(st, kind, ses.beta or 0.0), st, ses.src[None, :T], pad=False, atten_lim_db=ses.atten)[0]
            assert rms(got[lat * HOP:], one) < TOL, (ses.slot, rms(got[lat * HOP:], one))
        checked += 1
    assert checked >= 12
    assert len({(x.atten, x.beta) for x in sessions if x.sizes}) >= (4 if kind == "dfn2" else 10)


# -------------------------------------------------------------------------------------------------- mid-session -----
def complex_of(t):
    a = t.detach().cpu().double().numpy()
    return a[..., 0] + 1j * a[..., 1]


def spectra(model, st, audio):
    """DfNet.forward's noisy and enhanced spectra (post filter off) of one session, [T, F] complex."""
    sp, fe, fs = df_features(audio[None], st, model.nb_df)
    return complex_of(sp[:, 0])[0], complex_of(model(sp, fe, fs)[0][:, 0])[0]


def ref64_audio(X, Y, window, lims, betas):
    """float64 audio of one session whose frame t has limit lims[t] (linear, 0 off) and beta betas[t] (0 off): the post
    filter (pf_gain_spec) and the limit (atten_limit) applied per frame to the spectra, then the ISTFT."""
    Z = np.zeros_like(X)
    for t in range(X.shape[0]):
        y = Y[t]
        if betas[t] > 0:
            y, _ = R.pf_gain_spec(y, X[t], np.zeros(y.shape), betas[t])
        if lims[t] > 0:
            y, _ = R.atten_limit(X[t], y, np.zeros(y.shape), lims[t])
        Z[t] = y
    return R.istft(Z[None], window, HOP)[0][0]


def lin(db):
    return 0.0 if db is None or db <= 0 else 10 ** (-db / 20)


@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2"])
def test_mid_session_changes(st, kind):
    """Settings change inside sessions of a 3-slot handle: before the first call, right after an open, in consecutive
    1-hop calls, twice between the same two calls (the last one wins), during a closing tail (models with look-ahead),
    between calls of 1, 2, 3, 7 and 40 hops.  Every session's output equals the float64 restatement (ref64_audio) of its
    frames' settings at RMS <= 1e-6, and every hop whose frame and the frame before it share a setting equals the fresh
    single-stream run with that setting (RMS <= 1e-6).  At each switch hop the error is below 1 % of the gap to the hop
    that takes the new setting for the previous frame's tail too."""
    model = model_of(st, kind)
    pf = kind != "dfn2"
    s = DfStream(model, st, batch=3)
    lat = s.latency_frames
    K = "keep"
    # per call: changes [(slot, atten_db or K, beta or K)], opens, closes, hops
    plan = [
        ([(0, 12.0, 0.05 if pf else K), (1, 6.0, K)], [], [], 3),   # before the first call
        ([], [], [], 1),
        ([(0, 40.0, K)], [], [], 1),                                 # consecutive 1-hop calls
        ([(0, None, 0.02 if pf else K)], [], [], 1),
        ([(0, 6.0, K), (0, 12.0, 0.0 if pf else K)], [], [], 2),     # twice between the same two calls: the last wins
        ([(2, 40.0, K)], [2], [], 7),                                # a new session in slot 2, set right after the open
        ([(1, 12.0, 0.05 if pf else K)], [], [], 40),
        ([(2, None, K)], [], [1], 1),                                # slot 1 closes ...
        ([(1, 40.0, 0.02 if pf else K)] if lat > 1 else [], [], [], 1),   # ... and changes during its tail
        ([(0, 6.0, K), (2, 12.0, 0.02 if pf else K)], [], [], 2),
        ([(0, None, 0.0 if pf else K)], [], [], 1),
        ([(0, 40.0, K)], [], [], 7),
    ]
    total = sum(p[3] for p in plan) + 1
    src = {b: synth_audio(1, total * HOP, seed=700 + b)[0] for b in range(3)}
    fed = {b: 0 for b in range(3)}                 # input hops of the session
    emitted = {b: 0 for b in range(3)}             # output hops of the session (its next hop carries frame emitted - lat)
    cur = {b: (None, 0.0) for b in range(3)}       # (atten_db, beta)
    hist = {b: [] for b in range(3)}               # (first frame it covers, setting) per call
    outs = {b: [] for b in range(3)}
    sizes = {b: [] for b in range(3)}
    closing = {b: False for b in range(3)}
    tail_left = {b: 0 for b in range(3)}
    for changes, opens, closes, n in plan:
        if closes:
            s.close(closes)
            for b in closes:
                closing[b], tail_left[b] = True, lat
        for b in opens:                                  # the slot's old session is dropped; the new one is checked
            s.open([b])
            fed[b] = emitted[b] = 0
            cur[b], hist[b], outs[b], sizes[b] = (None, 0.0), [], [], []
            src[b] = synth_audio(1, total * HOP, seed=900 + b)[0]
        for b, db, beta in changes:
            a, bt = cur[b]
            if db != K:
                s.set_atten_lim(db, [b]); a = db
            if beta != K:
                s.set_post_filter_beta(beta, [b]); bt = beta
            cur[b] = (a, bt)
        x = torch.zeros((3, n * HOP))
        for b in range(3):
            hist[b].append((emitted[b] - lat, cur[b]))
            if not closing[b]:
                x[b] = src[b][fed[b] * HOP:(fed[b] + n) * HOP]
                fed[b] += n
                sizes[b].append(n)
        y = s.process(x.cuda()).cpu()
        for b in range(3):
            k = n if not closing[b] else min(n, tail_left[b])
            outs[b].append(y[b, :k * HOP])
            emitted[b] += k
            if closing[b]:
                tail_left[b] -= k
    y = s.flush()
    for b in range(3):
        hist[b].append((emitted[b] - lat, cur[b]))
        k = lat if not closing[b] else tail_left[b]
        outs[b].append(y[b, :k * HOP])
    window = st.fft_window()
    for b in range(3):
        got = torch.cat(outs[b]).double().numpy()
        T = fed[b]
        assert got.shape[0] == (T + lat) * HOP
        setting = [[sv for f, sv in hist[b] if f <= t][-1] for t in range(T)]
        lims, betas = [lin(a) for a, _ in setting], [bt for _, bt in setting]
        X, Y = spectra(model, st, src[b][:T * HOP])
        ref = ref64_audio(X, Y, window, lims, betas)
        body = got[lat * HOP:]
        assert np.abs(got[:lat * HOP]).max() == 0 if lat else True
        assert rms(body, ref) < TOL, (kind, b, rms(body, ref))
        switches = [t for t in range(1, T) if setting[t] != setting[t - 1]]
        strong = 0
        for t in switches:
            alt = ref64_audio(X, Y, window, [lims[t] if u == t - 1 else lims[u] for u in range(T)],
                              [betas[t] if u == t - 1 else betas[u] for u in range(T)])
            seg = slice(t * HOP, (t + 1) * HOP)
            gap, err = rms(alt[seg], ref[seg]), rms(body[seg], ref[seg])
            if gap > 1e-5:
                assert err < 0.01 * gap, (kind, b, t, err, gap)
                strong += 1
        assert strong >= {0: 5, 1: 1, 2: 2}[b] - (1 if b == 1 and lat <= 1 else 0), (kind, b, strong, switches)
        for sv in set(setting):
            one, _ = single_stream(model_of(st, kind, sv[1]), st, src[b][:T * HOP], sizes[b], sv[0])
            one = one.double().numpy()[lat * HOP:]
            same = [t for t in range(T) if setting[t] == sv and (t == 0 or setting[t - 1] == sv)]
            if not same:                                 # a setting of a single frame: only its switch hop
                continue
            idx = np.concatenate([np.arange(t * HOP, (t + 1) * HOP) for t in same])
            assert rms(body[idx], one[idx]) < TOL, (kind, b, sv, rms(body[idx], one[idx]))


# ------------------------------------------------------------------------------------------------------- LSNR -------
@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2"])
def test_lsnr_of_each_hop(st, kind):
    """A plain handle (no slots) fed in calls of mixed sizes, the LSNR requested on every call and at the flush: hop j
    carries frame j - latency, whose LSNR equals DfNet.forward's lsnr of the whole signal (LSNR_TOL_FORWARD); the first
    `latency` hops are NaN and the flush returns the last `latency` frames'.  Worst error measured on an H100 80GB HBM3:
    0 dB for all three models; the LSNR one frame off differs by 0.25 (dfn3), 0.32 (ll) and 0.12 dB (dfn2)."""
    model = model_of(st, kind)
    B = 2
    s = DfStream(model, st, batch=B)
    lat = s.latency_frames
    sizes = [1, 2, 3, 7, 40, 1, 1, 5]
    T = sum(sizes)
    x = synth_audio(B, T * HOP, seed=41)
    ls, pos = [], 0
    for i, n in enumerate(sizes):
        seg = x[:, pos * HOP:(pos + n) * HOP]
        y, l = s.process(seg.cuda() if i % 2 else seg, return_lsnr=True)
        assert l.device == y.device and l.shape == (B, n)
        ls.append(l.cpu())
        pos += n
    _, l = s.flush(return_lsnr=True)
    assert l.shape == (B, lat)
    ls.append(l)
    got = torch.cat(ls, 1)
    assert got.shape == (B, T + lat)
    assert torch.isnan(got[:, :lat]).all() and not torch.isnan(got[:, lat:]).any()
    sp, fe, fs = df_features(x, st, model.nb_df)
    want = model(sp, fe, fs)[2][..., 0].cpu()
    err = (got[:, lat:] - want).abs().max().item()
    off = (got[:, lat + 1:] - want[:, :-1]).abs().max().item()
    print(f"LSNR {kind}: worst |stream - forward| = {err:.3g} dB, one frame off {off:.3g} dB")
    assert err <= LSNR_TOL_FORWARD, (kind, err)
    assert off > 100 * LSNR_TOL_FORWARD       # one frame off is far outside the tolerance


def test_lsnr_linked_channels_are_per_channel(st):
    """Linked handles return each channel's own LSNR: the same as an unlinked handle fed the same channels, with and
    without stage gating (which reads the group's first channel).  Worst error measured on an H100 80GB HBM3: 0 dB."""
    model = model_of(st, "dfn3")
    x = synth_audio(4, 30 * HOP, seed=43)
    for gating in (False, True):
        res = []
        for linked in (False, True):
            s = DfStream(model, st, batch=4, channels=2 if linked else 1, reduce_mask="mean" if linked else None)
            if gating:
                s.set_lsnr_thresholds()
            a = s.process(x[:, :13 * HOP], return_lsnr=True)[1]
            b = s.process(x[:, 13 * HOP:], return_lsnr=True)[1]
            c = s.flush(return_lsnr=True)[1]
            res.append(torch.cat([a, b, c], 1))
        assert torch.equal(torch.isnan(res[0]), torch.isnan(res[1]))
        ok = ~torch.isnan(res[0])
        assert (res[0][ok] - res[1][ok]).abs().max().item() <= LSNR_TOL_STREAM
        assert (res[1][0, ok[0]] - res[1][1, ok[1]]).abs().max().item() > 0.1   # two channels, two values


def test_lsnr_first_request_later(st):
    """The LSNR head runs from a handle's first request on: a DeepFilterNet3 handle that asks from its third call on
    returns every frame those calls emit; DeepFilterNet2, whose audio trails its DNN by df_lookahead frames, returns NaN
    for the frames whose DNN step ran before the first request."""
    for kind in ("dfn3", "dfn2"):
        model = model_of(st, kind)
        s = DfStream(model, st, batch=1)
        x = synth_audio(1, 30 * HOP, seed=45)
        s.process(x[:, :10 * HOP])
        s.process(x[:, 10 * HOP:15 * HOP])
        _, l = s.process(x[:, 15 * HOP:], return_lsnr=True)
        nan = torch.isnan(l[0])
        df_la = model.cfg.df_lookahead if kind == "dfn2" else 0
        assert nan[:df_la].all() and not nan[df_la:].any(), (kind, nan)


# ----------------------------------------------------------------------------------------------------- errors -------
def test_setting_errors_and_defaults(st):
    """Negative / NaN / infinite beta and NaN limits are DFB_ERR_INVALID, free and out-of-range slots too; beta on
    DeepFilterNet2 and setters on linked handles are DFB_ERR_UNSUPPORTED.  A refused call changes nothing; open() and
    reset() return slots to the handle's settings."""
    model = model_of(st, "dfn3")
    L = _lib.lib()
    s = DfStream(model, st, batch=3, atten_lim_db=12.0)
    one = (C.c_int64 * 1)(0)
    for v in (-0.01, float("nan"), float("inf")):
        assert L.dfb_stream_set_post_filter_beta(s._h, one, 1, v) == _lib.DFB_ERR_INVALID
        with pytest.raises(ValueError):
            s.set_post_filter_beta(v, [0])
    assert L.dfb_stream_set_atten_lim(s._h, one, 1, float("nan")) == _lib.DFB_ERR_INVALID
    for bad in ([3], [-1], [1, 1]):
        a = (C.c_int64 * len(bad))(*bad)
        assert L.dfb_stream_set_atten_lim(s._h, a, len(bad), 6.0) == _lib.DFB_ERR_INVALID
        assert L.dfb_stream_set_post_filter_beta(s._h, a, len(bad), 0.02) == _lib.DFB_ERR_INVALID
        with pytest.raises(ValueError):
            s.set_atten_lim(6.0, bad)
    s.close([2])
    s.process(torch.zeros(3, 10 * HOP))                # slot 2's tail is out: it is free
    assert s.slot_states()[2] == SLOT_FREE
    with pytest.raises(_lib.DfbError) as e:
        s.set_atten_lim(6.0, [0, 2])
    assert e.value.code == _lib.DFB_ERR_INVALID
    dfn2 = DfStream(model_of(st, "dfn2"), st, batch=2)
    with pytest.raises(_lib.DfbError) as e:
        dfn2.set_post_filter_beta(0.02, [0])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    dfn2.set_atten_lim(6.0, [0])
    linked = DfStream(model, st, batch=4, channels=2, reduce_mask="mean")
    for op in (lambda: linked.set_atten_lim(6.0, [0]), lambda: linked.set_post_filter_beta(0.02, [0])):
        with pytest.raises(_lib.DfbError) as e:
            op()
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED

    # a refused call changes nothing, open() and reset() restore the defaults: compare with the handle's own settings
    x = synth_audio(3, 20 * HOP, seed=47)

    def run(h, prep):
        h.reset()
        prep(h)
        return torch.cat([h.process(x[:, :7 * HOP]), h.process(x[:, 7 * HOP:]), h.flush()], 1)

    plain = run(s, lambda h: None)

    def refused(h):
        a = (C.c_int64 * 2)(0, 3)
        assert L.dfb_stream_set_atten_lim(h._h, a, 2, 40.0) == _lib.DFB_ERR_INVALID
        with pytest.raises(ValueError):
            h.set_post_filter_beta(-1.0)
    assert torch.equal(run(s, refused), plain)

    def reopened(h):
        h.set_atten_lim(40.0)
        h.set_post_filter_beta(0.05)
        h.open([0, 1, 2])
    assert rms(run(s, reopened), plain) < TOL
    s.reset()
    s.set_atten_lim(40.0)
    s.set_post_filter_beta(0.05)
    s.reset()
    assert torch.equal(torch.cat([s.process(x[:, :7 * HOP]), s.process(x[:, 7 * HOP:]), s.flush()], 1), plain)
