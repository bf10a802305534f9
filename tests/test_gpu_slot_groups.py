"""GPU: slot groups (DfStream.open_linked / slot_groups, dfb_stream_open_linked / dfb_stream_slot_groups).  A simulated
server opens mono, 2-channel and 3-channel sessions in the slots of one handle on a seeded schedule; every group's output,
from the call that opened it to the end of its tail, must equal a fresh linked handle DfStream(batch=C, channels=C,
reduce_mask=mode) fed the same rows in the same call sizes and then flushed, and enhance_device_ragged(group_sizes=[C],
pad=False) delayed by the latency.  Mono sessions equal fresh single-stream handles, free rows are zero, and
slot_groups() / slot_states() follow the plan after every call."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dsp_ref64 as R
import linked_oracle as LO
from test_gpu_slots import cfg_of, rms
from test_gpu_stream_controls import lin, model_of, ref64_audio
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance_device_ragged, libdf
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.streaming import SLOT_CLOSING, SLOT_FREE, SLOT_OPEN
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TOL = 1e-6          # RMS, as the other streaming tests
EDGE = 4800         # first / last 100 ms of a session, checked on their own
SIZES = [1, 2, 3, 7, 40]
B = 12


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


def schedule(seed, n_random):
    """[(ops, n hops)] of a 12-slot server whose slots are all open (mono) at creation; ops are ("close" | "open" |
    "link", slots) in order.  The scripted head covers a 2-channel group over two open mono slots at clock 0, a young
    3-channel open (clock 1) over closing slots, a 1-hop 3-channel session, a mono re-open, a group closed and re-opened
    while closing in a different layout (3 channels, one of them a mono slot before), an open and a close in one call, and
    a group released from the middle of the prefix with a larger group and a mono session behind it.  Then seeded random
    traffic (see `random_ops`)."""
    head = [([("close", [9, 10, 11]), ("link", [6, 7])], 1),
            ([("link", [9, 11, 10])], 1),
            ([("close", [10, 9, 11]), ("open", [3])], 3),
            ([("close", [6, 7]), ("link", [4, 5])], 1),
            ([("link", [7, 6, 2]), ("close", [0]), ("open", [1])], 1),
            ([("close", [5, 4])], 7),
            ([("link", [11, 5])], 40)]
    return head, np.random.default_rng(seed), n_random


class Group:
    def __init__(self, slots, seed, total):
        self.slots, self.seed = list(slots), seed
        self.src = synth_audio(len(slots), total * HOP, seed=seed)
        self.sizes, self.outs = [], []
        self.closing, self.tail_left, self.dropped = False, 0, False

    def out(self):
        return torch.cat(self.outs, 1) if self.outs else torch.zeros(len(self.slots), 0)


def random_ops(rng, live, n_slots):
    """Closes each open session with probability 0.15, sometimes re-opens a closing one in a new layout, and fills free
    slots with mono, 2- and 3-channel sessions in random slot orders."""
    ops = []
    free = [b for b in range(n_slots) if b not in live]
    rng.shuffle(free)
    for g in {id(g): g for g in live.values()}.values():
        if not g.closing and rng.random() < 0.15:
            ops.append(("close", list(rng.permutation(g.slots))))
        elif g.closing and rng.random() < 0.3:       # re-opened while closing: all of its slots, maybe one more
            slots = list(rng.permutation(g.slots))
            if free and len(slots) < 3 and rng.random() < 0.5:
                slots.insert(int(rng.integers(0, len(slots) + 1)), free.pop())
            ops.append(("link", slots))
    while free and rng.random() < 0.5:
        c = int(rng.choice([1, 2, 3], p=[0.4, 0.35, 0.25]))
        if c > len(free):
            break
        take, free = free[:c], free[c:]
        ops.append(("open", take) if c == 1 else ("link", take))
    return ops


def run_groups(model, st, mode, sched, atten=None, setup=None, seed=0, lsnr=False):
    """Runs the schedule on one 12-slot handle with reduce_mask `mode` and returns its groups (finished with their tails,
    or dropped by a re-open)."""
    head, rng, n_random = sched
    s = DfStream(model, st, batch=B, atten_lim_db=atten, reduce_mask=mode)
    if setup:
        setup(s)
    lat = s.latency_frames
    total = sum(n for _, n in head) + 40 * n_random + 1
    groups, live, count = [], {}, [0]

    def new_group(slots):
        for b in slots:
            if b in live:
                old = live[b]
                old.dropped = True
                for x in old.slots:
                    live.pop(x, None)
        g = Group(slots, 2000 + 37 * seed + count[0], total)
        count[0] += 1
        for b in slots:
            live[b] = g
        groups.append(g)

    for b in range(B):
        new_group([b])
    noise = torch.Generator().manual_seed(5 + seed)
    calls = [c for c in head] + [None] * n_random
    for i in range(len(calls) + 1):
        flush = i == len(calls)
        if not flush:
            if calls[i] is None:
                ops, n = random_ops(rng, live, B), int(rng.choice(SIZES))
            else:
                ops, n = calls[i]
            for op, slots in ops:
                slots = [int(b) for b in slots]
                if op == "close":
                    s.close(slots)
                    for g in {id(live[b]): live[b] for b in slots if b in live}.values():
                        if not g.closing:
                            g.closing, g.tail_left = True, lat
                            if lat == 0:
                                for b in g.slots:
                                    del live[b]
                elif op == "open":
                    s.open(slots)
                    for b in slots:
                        new_group([b])
                else:
                    s.open_linked(slots)
                    new_group(slots)
            want_states = [SLOT_FREE if b not in live else (SLOT_CLOSING if live[b].closing else SLOT_OPEN) for b in range(B)]
            want_groups = [live[b].slots[0] if b in live else -1 for b in range(B)]
            assert s.slot_states().tolist() == want_states, (i, s.slot_states(), want_states)
            assert s.slot_groups().tolist() == want_groups, (i, s.slot_groups(), want_groups)
            x = torch.randn((B, n * HOP), generator=noise) * 0.3          # rows of free / closing slots are ignored
            for g in {id(g): g for g in live.values()}.values():
                if not g.closing:
                    pos = sum(g.sizes)
                    for c, b in enumerate(g.slots):
                        x[b] = g.src[c, pos * HOP:(pos + n) * HOP]
                    g.sizes.append(n)
            res = s.process(x.cuda() if i % 2 else x, return_lsnr=lsnr)
            y, ls = (res[0].cpu(), res[1].cpu()) if lsnr else (res.cpu(), None)
        else:
            for g in {id(g): g for g in live.values()}.values():
                if not g.closing:
                    g.closing, g.tail_left = True, lat
            res = s.flush(return_lsnr=lsnr)
            y, ls = res if lsnr else (res, None)
            n = lat
            if lat == 0:
                live.clear()
        used = set()
        for g in {id(g): g for g in live.values()}.values():
            k = n if not g.closing else min(n, g.tail_left)
            g.outs.append(y[g.slots, :k * HOP])
            if lsnr:
                g.lsnr = getattr(g, "lsnr", []) + [ls[g.slots, :k]]
            if g.closing:
                if k < n:
                    assert y[g.slots, k * HOP:].abs().max().item() == 0, (i, g.slots)
                g.tail_left -= k
                if g.tail_left == 0:
                    for b in g.slots:
                        del live[b]
            used.update(g.slots)
        for b in range(B):
            if b not in used and y.shape[1]:
                assert y[b].abs().max().item() == 0, ("free slot output", i, b)
    assert not live and s.slot_states().tolist() == [SLOT_FREE] * B and s.slot_groups().tolist() == [-1] * B
    return groups, lat


def fresh_linked(model, st, g, mode, atten=None, setup=None, lsnr=False):
    """A fresh handle of the group's channels, linked by `mode`, fed its audio in its call sizes and flushed."""
    C_ = len(g.slots)
    r = DfStream(model, st, batch=C_, atten_lim_db=atten, channels=C_ if mode not in (None, "none") else 1,
                 reduce_mask=mode if C_ > 1 else None)
    if setup:
        setup(r)
    outs, ls, pos = [], [], 0
    for n in g.sizes:
        res = r.process(g.src[:, pos * HOP:(pos + n) * HOP], return_lsnr=lsnr)
        outs.append(res[0] if lsnr else res)
        if lsnr:
            ls.append(res[1])
        pos += n
    res = r.flush(return_lsnr=lsnr)
    outs.append(res[0] if lsnr else res)
    if lsnr:
        ls.append(res[1])
    return torch.cat(outs, 1), (torch.cat(ls, 1) if lsnr else None)


def check_groups(model, st, groups, lat, mode, atten=None, setup=None, against_enhance=True):
    checked = {1: 0, 2: 0, 3: 0}
    for g in groups:
        got = g.out()
        if not g.sizes:
            assert got.numel() == 0 or got.abs().max().item() == 0
            continue
        ref, _ = fresh_linked(model, st, g, mode, atten, setup)
        if g.dropped:
            assert got.shape[1] <= ref.shape[1]
            ref = ref[:, :got.shape[1]]
        assert got.shape == ref.shape, (g.slots, got.shape, ref.shape)
        for c in range(got.shape[0]):
            assert rms(got[c], ref[c]) < TOL, (g.slots, c, g.sizes, rms(got[c], ref[c]))
            assert rms(got[c, :EDGE], ref[c, :EDGE]) < TOL and rms(got[c, -EDGE:], ref[c, -EDGE:]) < TOL, (g.slots, c)
        if against_enhance and not g.dropped:
            T = sum(g.sizes) * HOP
            C_ = len(g.slots)
            link = dict(group_sizes=[C_], reduce_mask=mode) if C_ > 1 else {}
            one = enhance_device_ragged(model, st, g.src[:, :T].cuda().contiguous(), [T] * C_, pad=False, atten_lim_db=atten,
                                        **link).cpu()
            assert got[:, :lat * HOP].abs().max().item() == 0 if lat else True
            for c in range(C_):
                assert rms(got[c, lat * HOP:], one[c]) < TOL, (g.slots, c, rms(got[c, lat * HOP:], one[c]))
        checked[len(g.slots)] += 1
    return checked


@pytest.mark.parametrize("mode", ["max", "mean"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_groups_equal_fresh_linked_handles(st, kind, mode):
    model = DfNet(cfg_of(kind), random_state_dict(cfg_of(kind), seed=191), st)
    groups, lat = run_groups(model, st, mode, schedule(seed=17, n_random=20), seed=1)
    checked = check_groups(model, st, groups, lat, mode)
    assert checked[1] >= 6 and checked[2] >= 3 and checked[3] >= 2, checked
    assert any(g.dropped and len(g.slots) > 1 for g in groups) or lat == 0
    # not vacuous: a linked group differs from its channels run alone
    g = next(g for g in groups if len(g.slots) > 1 and not g.dropped and sum(g.sizes) > 20)
    alone, _ = fresh_linked(model, st, g, None)
    assert rms(g.out()[0], alone[0]) > 1e-4


def test_mode_none_gives_independent_channels(st):
    """Groups on a handle without a reduction are unlinked channels that open and close together: each channel equals a
    fresh single-stream handle."""
    model = DfNet(cfg_of("dfn3"), random_state_dict(cfg_of("dfn3"), seed=192), st)
    groups, lat = run_groups(model, st, None, schedule(seed=18, n_random=12), seed=2)
    n = 0
    for g in groups:
        if not g.sizes or len(g.slots) == 1:
            continue
        got = g.out()
        for c in range(len(g.slots)):
            one = type(g)([g.slots[c]], 0, 1)
            one.src, one.sizes = g.src[c:c + 1], g.sizes
            ref, _ = fresh_linked(model, st, one, None)
            ref = ref[:, :got.shape[1]]
            assert rms(got[c], ref[0]) < TOL, (g.slots, c)
        n += 1
    assert n >= 3


@pytest.mark.parametrize("variant", ["post_filter", "atten_lim", "lsnr_gating"])
def test_groups_with_options(st, variant):
    cfg = cfg_of("dfn3", mask_pf=variant == "post_filter")
    model = DfNet(cfg, random_state_dict(cfg, seed=193), st)
    atten = 12.0 if variant == "atten_lim" else None
    setup = (lambda s: s.set_lsnr_thresholds()) if variant == "lsnr_gating" else None
    groups, lat = run_groups(model, st, "mean", schedule(seed=19, n_random=12), atten=atten, setup=setup, seed=3)
    checked = check_groups(model, st, groups, lat, "mean", atten=atten, setup=setup, against_enhance=variant != "lsnr_gating")
    assert checked[2] + checked[3] >= 4


def test_gating_follows_channel_0(st):
    """LSNR stage gating in a 2-channel group, loud channel 0 and quiet channel 1: the decision of every frame comes from
    channel 0, as on a fixed linked handle (test_gpu_linked.test_streaming_gating_follows_the_first_channel)."""
    cfg = cfg_of("dfn3")
    sd = random_state_dict(cfg, seed=194)
    model = DfNet(cfg, sd, st)
    n = 90
    audio = synth_audio(2, HOP * n, seed=460)
    audio[1] *= 0.03
    _, aux = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean", return_all=True)
    l0 = np.sort(aux["lsnr"][0, :, 0].numpy())
    k = len(l0) // 2
    assert l0[k] - l0[k - 1] > 1e-3
    th = dict(min_db_thresh=-1e9, max_db_erb_thresh=1e9, max_db_df_thresh=float(l0[k - 1] + l0[k]) / 2)
    want = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean", stages=th)
    s = DfStream(model, st, batch=5, reduce_mask="mean")
    s.set_lsnr_thresholds(**th)
    s.close([0, 1, 2, 3, 4])
    s.process(torch.zeros(5, 3 * HOP))
    s.open([0])
    s.open_linked([4, 2])
    x = synth_audio(5, HOP * n, seed=461)
    x[4], x[2] = audio[0], audio[1]
    got = torch.cat([s.process(x[:, :HOP * 33]), s.process(x[:, HOP * 33:]), s.flush()], 1)[:, s.latency_frames * HOP:]
    for c, b in enumerate([4, 2]):
        assert rms(got[b], want[c]) <= 5e-6, (c, rms(got[b], want[c]))
    r = DfStream(model, st, batch=2, channels=2, reduce_mask="mean")
    r.set_lsnr_thresholds(**th)
    ref = torch.cat([r.process(audio[:, :HOP * 33]), r.process(audio[:, HOP * 33:]), r.flush()], 1)[:, r.latency_frames * HOP:]
    assert rms(got[[4, 2]], ref) < TOL
    l1 = aux["lsnr"][1, :, 0].numpy()
    l0f = aux["lsnr"][0, :, 0].numpy()
    assert ((l1 > th["max_db_df_thresh"]) != (l0f > th["max_db_df_thresh"])).any()


def test_lsnr_per_channel_bit_exact(st):
    """process / flush(return_lsnr=True) return each channel's own LSNR: bit for bit, NaN in the same places, those of a
    fresh linked handle of the group."""
    model = model_of(st, "dfn3")
    groups, lat = run_groups(model, st, "max", schedule(seed=20, n_random=10), seed=4, lsnr=True)
    n = 0
    for g in groups:
        if not g.sizes:
            continue
        got = torch.cat(g.lsnr, 1)
        _, ref = fresh_linked(model, st, g, "max", lsnr=True)
        ref = ref[:, :got.shape[1]]
        assert torch.equal(torch.isnan(got), torch.isnan(ref)), g.slots
        assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(ref)), (g.slots, (got - ref).abs().nan_to_num().max())
        n += len(g.slots) > 1
    assert n >= 3


def linked_spectra(model, st, audio, mode):
    """float64 noisy and enhanced spectra [C, T, F] of one group (DeepFilterNet3, no post filter): DfNet.forward's
    outputs, the ERB mask reduced over the channels in fp32 as the apply kernel does, applied by dsp_ref64.apply."""
    sp, fe, fs = df_features(audio, st, model.nb_df)
    _, m, _, coefs = model(sp, fe, fs)
    m_link = LO.reduce_mask(m.cpu(), audio.shape[0], mode)[:, 0].double().numpy()
    cf = coefs.cpu().permute(0, 2, 3, 1, 4).double().numpy()          # [C, T, Fd, O, 2]
    cf = cf[..., 0] + 1j * cf[..., 1]
    X = sp[:, 0].cpu().double().numpy()
    X = X[..., 0] + 1j * X[..., 1]
    c = model.cfg
    Y, _ = R.apply(X, m_link, cf, st.erb_widths(), mode=1, nb_df=c.nb_df, order=c.df_order, lookahead=c.df_lookahead)
    return X, Y


@pytest.mark.parametrize("kind", ["dfn3", "ll"])
def test_group_settings_mid_session(st, kind):
    """Per-group attenuation limit and post-filter beta changed inside the sessions of a 6-slot handle (a 2-channel group,
    a 3-channel group, one mono slot), mode mean.  Every channel equals the float64 restatement of its frames' settings
    with the group's reduced mask at RMS <= 1e-6; at each switch hop the error is below 1 % of the gap to the hop that
    takes the new setting for the previous frame's tail too; away from the switch hops it equals the fresh linked handle
    with that setting."""
    model = model_of(st, kind)
    s = DfStream(model, st, batch=6, reduce_mask="mean")
    lat = s.latency_frames
    A, Bg, M = [4, 1], [2, 5, 3], [0]
    s.open_linked(A)
    s.open_linked(Bg)
    K = "keep"
    plan = [([(A, 12.0, 0.05), (Bg, 6.0, K)], 3),
            ([], 1),
            ([(A, 40.0, K)], 1),
            ([(A, None, 0.02), (M, 6.0, K)], 1),
            ([(Bg, 40.0, 0.02)], 7),
            ([(A, 6.0, K), (A, 12.0, 0.0)], 2),
            ([(Bg, None, 0.0)], 40),
            ([(A, 40.0, 0.05), (Bg, 12.0, K)], 2),
            ([(A, None, K)], 7)]
    total = sum(n for _, n in plan)
    x = synth_audio(6, total * HOP, seed=480)
    cur = {tuple(G): (None, 0.0) for G in (A, Bg, M)}
    hist = {tuple(G): [] for G in (A, Bg, M)}
    outs, pos, sizes = [], 0, []
    for changes, n in plan:
        for G, db, beta in changes:
            a, bt = cur[tuple(G)]
            if db != K:
                s.set_atten_lim(db, G); a = db
            if beta != K:
                s.set_post_filter_beta(beta, G); bt = beta
            cur[tuple(G)] = (a, bt)
        for G in cur:
            hist[G].append((pos - lat, cur[G]))
        outs.append(s.process(x[:, pos * HOP:(pos + n) * HOP].cuda()).cpu())
        pos += n
        sizes.append(n)
    outs.append(s.flush())
    y = torch.cat(outs, 1)
    window = st.fft_window()
    for G in (A, Bg):
        audio = x[list(G)]
        X, Y = linked_spectra(model, st, audio, "mean")
        setting = [[sv for f, sv in hist[tuple(G)] if f <= t][-1] for t in range(total)]
        lims, betas = [lin(a) for a, _ in setting], [bt for _, bt in setting]
        switches = [t for t in range(1, total) if setting[t] != setting[t - 1]]
        assert len(switches) >= 3
        for c, b in enumerate(G):
            body = y[b, lat * HOP:].double().numpy()
            ref = ref64_audio(X[c], Y[c], window, lims, betas)
            assert rms(body, ref) < TOL, (kind, G, c, rms(body, ref))
            strong = 0
            for t in switches:
                alt = ref64_audio(X[c], Y[c], window, [lims[t] if u == t - 1 else lims[u] for u in range(total)],
                                  [betas[t] if u == t - 1 else betas[u] for u in range(total)])
                seg = slice(t * HOP, (t + 1) * HOP)
                gap, err = rms(alt[seg], ref[seg]), rms(body[seg], ref[seg])
                if gap > 1e-5:
                    assert err < 0.01 * gap, (kind, G, c, t, err, gap)
                    strong += 1
            assert strong >= 3, (kind, G, c, strong)
        for sv in set(setting):
            g = Group(G, 0, 1)
            g.src, g.sizes = audio, sizes
            one, _ = fresh_linked(model_of(st, kind, sv[1]), st, g, "mean", atten=sv[0])
            same = [t for t in range(total) if setting[t] == sv and (t == 0 or setting[t - 1] == sv)]
            if not same:
                continue
            idx = np.concatenate([np.arange(t * HOP, (t + 1) * HOP) for t in same])
            for c, b in enumerate(G):
                body = y[b, lat * HOP:].double().numpy()
                assert rms(body[idx], one[c, lat * HOP:].double().numpy()[idx]) < TOL, (kind, G, c, sv)


def test_only_live_rows_are_computed(st):
    """64 slots with two stereo groups and one mono session compute 5 rows: the forward pass's `emb` activation holds
    5 x window x emb_dim floats."""
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=195), st)
    s = DfStream(model, st, batch=64, reduce_mask="max")
    x = synth_audio(64, 40 * HOP, seed=5)
    s.close(list(range(64)))
    s.process(x[:, :HOP * s.latency_frames])
    s.open_linked([40, 3])
    s.open([17])
    s.open_linked([9, 63])
    s.process(x[:, :20 * HOP])                               # the window below: 8 halo frames + the n new ones
    n = 3
    y = s.process(x[:, 20 * HOP:(20 + n) * HOP])
    buf = np.zeros(64 * 64 * 1024, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, b"emb", buf.ctypes.data, buf.size)
    assert got == 5 * (8 + n) * (cfg.nb_erb // 4 * 64)        # kHalo = 8 halo frames + n new frames per stream
    live = [40, 3, 17, 9, 63]
    assert y[[b for b in range(64) if b not in live]].abs().max() == 0 and (y[live].abs().amax(1) > 0).all()


def test_row_moves_take_constant_launches(st):
    """The call after a 2-channel group is released launches as many kernels with 1 row behind it as with 40 (the rows
    close up in one k_slot_rows pass, whatever their number), and the rows that moved keep their streams."""
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=196), st)
    L = _lib.lib()
    x = synth_audio(48, 20 * HOP, seed=6)
    launches = {}
    for behind in (1, 40):
        s = DfStream(model, st, batch=48, reduce_mask="mean")
        lat = s.latency_frames
        s.close(list(range(48)))
        s.process(torch.zeros(48, lat * HOP))
        pool = list(range(2, 48))
        s.open(pool[:40 - behind])
        s.open_linked([0, 1])
        s.open(pool[40 - behind:40])                          # 40 mono sessions, `behind` of them after the group
        outs = [s.process(x[:, :5 * HOP])]
        s.close([1, 0])
        outs.append(s.process(x[:, 5 * HOP:(5 + lat) * HOP]))  # the group's tail: it is free after this call
        assert s.slot_groups()[[0, 1]].tolist() == [-1, -1]
        torch.cuda.synchronize()
        n0 = L.dfb_kernel_launches()
        outs.append(s.process(x[:, (5 + lat) * HOP:(8 + lat) * HOP]))
        torch.cuda.synchronize()
        launches[behind] = int(L.dfb_kernel_launches() - n0)
        y = torch.cat(outs, 1)
        for b in (pool[39], pool[40 - behind]):                 # rows that moved up behind the group
            r = DfStream(model, st, batch=1)
            ref = torch.cat([r.process(x[b:b + 1, :5 * HOP]), r.process(x[b:b + 1, 5 * HOP:(5 + lat) * HOP]),
                             r.process(x[b:b + 1, (5 + lat) * HOP:(8 + lat) * HOP])], 1)[0]
            assert rms(y[b], ref) < TOL, (behind, b)
    assert launches[1] == launches[40], launches


def test_group_errors(st):
    """Partial listings of a live group, duplicate / out-of-range / empty slot lists, open_linked on a fixed-group handle
    and set_mask_reduce after slot operations are refused and change nothing; flush frees every group and reset drops
    them."""
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=197), st)
    L = _lib.lib()
    s = DfStream(model, st, batch=6, reduce_mask="mean")
    s.open_linked([1, 3])
    s.open_linked([5, 0, 2])
    states, groups = s.slot_states().tolist(), s.slot_groups().tolist()
    assert groups == [5, 1, 5, 1, 4, 5] and states == [SLOT_OPEN] * 6

    def unchanged():
        assert s.slot_states().tolist() == states and s.slot_groups().tolist() == groups

    partial = [lambda: s.open([1]), lambda: s.open([3, 4]), lambda: s.open_linked([1, 4]), lambda: s.open_linked([0, 2]),
               lambda: s.close([3]), lambda: s.close([5, 2]), lambda: s.set_atten_lim(6.0, [1]),
               lambda: s.set_post_filter_beta(0.02, [0, 2, 1, 3])]
    for op in partial:
        with pytest.raises(_lib.DfbError) as e:
            op()
        assert e.value.code == _lib.DFB_ERR_INVALID
        unchanged()
    for bad in ([1, 3, 1], [6], [-1], []):
        with pytest.raises(ValueError):
            s.open_linked(bad)
        a = (C.c_int64 * max(1, len(bad)))(*bad)
        assert L.dfb_stream_open_linked(s._h, a, len(bad)) == _lib.DFB_ERR_INVALID
        unchanged()
    with pytest.raises(_lib.DfbError) as e:
        s.set_mask_reduce(2, "mean")
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError) as e:
        s.set_mask_reduce(1, "max")
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    unchanged()
    fixed = DfStream(model, st, batch=4, channels=2, reduce_mask="mean")
    with pytest.raises(_lib.DfbError) as e:
        fixed.open_linked([0, 1])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    # whole groups are accepted in any order, together with mono slots
    s.set_atten_lim(6.0, [3, 1])
    s.set_post_filter_beta(0.02, [2, 4, 0, 5])
    s.process(synth_audio(6, 4 * HOP, seed=7))
    s.flush()
    assert s.slot_states().tolist() == [SLOT_FREE] * 6 and s.slot_groups().tolist() == [-1] * 6
    s.open_linked([2, 4])
    s.process(synth_audio(6, 2 * HOP, seed=8))
    assert s.slot_groups().tolist() == [-1, -1, 2, -1, 2, -1]
    s.reset()
    assert s.slot_states().tolist() == [SLOT_OPEN] * 6 and s.slot_groups().tolist() == list(range(6))
