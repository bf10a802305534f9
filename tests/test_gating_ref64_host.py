"""CPU: tests/gating_ref64.py, the float64 restatement of a runtime-gating window that tests/test_gpu_gating_layers.py
holds the device to.  Its plan agrees with the oracle's stage rule (gating_runtime_oracle.run_flags) at ties with every
threshold; the oracle's fp32 decoders, run on each decoder's own frames only, lie within its bounds; and each check rejects
the mistakes an end-to-end RMS cannot see: `<=` for `<`, an erb_src one frame late, a tail taken from the first K - 1
compacted rows, a fill from frame t - 1, the halo row for the carried one and the reverse, erb_first at the stream's first
frame for a row that has never run."""
import numpy as np
import pytest
import torch

import dfnet_oracle as O
import gating_ref64 as G
import gating_runtime_oracle as GO
import model_ref64 as M
from dsp_ref64 import err_ratio

from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.weights import random_state_dict

F32 = np.float32


def tie_rows(rng, th, T=300):
    """LSNR rows [3][T] in which every threshold value occurs, with neighbours one fp32 ulp either side"""
    vals = [F32(v) for v in th]
    pool = np.concatenate([np.array([v, np.nextafter(v, F32(-np.inf)), np.nextafter(v, F32(np.inf))], F32) for v in vals])
    rows = rng.uniform(-20, 40, size=(3, T)).astype(F32)
    for r in rows:
        pos = rng.choice(T, size=3 * pool.size, replace=False)
        r[pos] = np.tile(pool, 3)
    return rows


THS = [(-10.0, 30.0, 20.0),    # tract's defaults
       (5.5, 12.25, 7.0),
       (25.0, 10.0, 15.0),     # min > max_erb: nothing runs
       (-5.0, 10.0, 30.0)]     # max_df > max_erb: the DF stage is the ERB one


@pytest.mark.parametrize("th", THS)
def test_plan_agrees_with_the_stage_rule_at_ties(th):
    rng = np.random.default_rng(1)
    l = tie_rows(rng, th)
    for v in th:
        assert (l == F32(v)).any()
    pl = G.plan(l, None, 0, 0, [th] * 3, [True] * 3)
    for b in range(3):
        e, d = GO.run_flags(torch.from_numpy(l[b]), tuple(float(F32(v)) for v in th))
        assert np.array_equal(pl["erb_run"][b], e.numpy()) and np.array_equal(pl["df_run"][b], d.numpy()), (th, b)
        assert pl["df_n"][b] == d.sum()
        ie = np.nonzero(e.numpy())[0]
        for t in range(l.shape[1]):
            prev = ie[ie <= t]
            assert pl["erb_src"][b, t] == (prev[-1] if prev.size else -1)
            assert pl["df_pos"][b, t] == d[:t].sum()
    if th[0] > th[1]:
        assert not pl["erb_run"].any()


def test_plan_halo_links_first_and_non_gating_rows():
    rng = np.random.default_rng(2)
    th = THS[1]
    l = tie_rows(rng, th, T=40)
    Rc, w0 = 8, 100
    first = [0, w0 + 20, 0]
    pl = G.plan(l, first, w0, Rc, [th] * 3, [True, True, False], links=[0, 0, 2], has_run_prev=[False, False, True])
    assert pl["erb_run"][:, :Rc].all() and pl["df_run"][:, :Rc].all()
    e0, d0 = GO.run_flags(torch.from_numpy(l[0]), th)
    # row 1 follows row 0's LSNR from its first frame on; before it, nothing runs
    assert not pl["erb_run"][1, Rc:20].any()
    assert np.array_equal(pl["erb_run"][1, 20:], e0.numpy()[20:]) and np.array_equal(pl["df_run"][1, 20:], d0.numpy()[20:])
    assert pl["erb_run"][2].all() and pl["df_run"][2].all()
    s1 = 20 + int(np.nonzero(e0.numpy()[20:])[0][0])
    assert pl["erb_first"][1] == w0 + s1 and pl["erb_first"][2] == 0
    # after an apply-mode window every earlier frame of a started stream ran
    h = G.plan(l, first, w0, Rc, [th] * 3, [True] * 3, from_halo=True)
    assert h["erb_first"][0] == 0 and h["has_run"][0] and h["erb_first"][1] == w0 + s1


def small_cfg(kt, K):
    return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(kt, 3), conv_ch=16,
                       emb_hidden_dim=64, df_hidden_dim=64, emb_num_layers=2, df_num_layers=2, lin_groups=8, enc_lin_groups=8,
                       df_gru_skip="groupedlinear", df_pathway_kernel_size_t=K)


@pytest.mark.parametrize("K", [1, 3, 5])
def test_pathway_of_the_oracle_on_its_run_frames_is_within_the_bound(K):
    """The oracle's fp32 df_convp on the subsequence of DF run frames (tract's decoder alone on its frames) equals
    pathway_q on the compacted rows of two consecutive windows, the second after the first's tail, within the bound."""
    cfg = small_cfg(1, K)
    sd = random_state_dict(cfg, seed=4)
    sd64, ab = M.state64(sd)
    C, Fd = 16, cfg.nb_df
    g = torch.Generator().manual_seed(5)
    T = 60
    c0 = torch.rand(1, C, T, Fd, generator=g)
    run = torch.rand(T, generator=g) < 0.4
    idx = torch.nonzero(run).view(-1)
    want = O.conv_norm_act(c0[:, :, idx], sd, "df_dec.df_convp").permute(0, 2, 3, 1)[0].numpy()   # fp32 oracle
    dev = c0.permute(0, 2, 3, 1).reshape(T, Fd * C).numpy()
    pl = dict(df_run=run.numpy()[None])
    tail = np.zeros((K - 1, Fd * C), F32)
    got, bound = [], []
    for lo, hi in ((0, 25), (25, T)):   # two windows without halo: Rc = 0
        sub = dict(df_run=pl["df_run"][:, lo:hi])
        P = G.compact(dev[lo:hi], tail, sub, 0, 0)
        q, bq = G.pathway_q(sd64, ab, P, Fd, C, cfg.df_order)
        got.append(q[K - 1:]); bound.append(bq[K - 1:])
        tail = G.next_c0_tail(P, K)
    ref, b = np.concatenate(got), np.concatenate(bound)
    assert err_ratio(want, ref, b) <= 1
    # the mutation: each window's tail taken from its first K - 1 compacted rows
    if K > 1:
        P = G.compact(dev[:25], np.zeros((K - 1, Fd * C), F32), dict(df_run=pl["df_run"][:, :25]), 0, 0)
        assert not np.array_equal(P[:K - 1], G.next_c0_tail(P, K))


def test_fill_of_the_oracle_on_its_run_frames_is_within_the_bound():
    """The oracle's fp32 convt3 and mask head on the subsequence of ERB run frames equal convt3 / mask on the filled
    window inputs at those frames, within the bounds: filling forward from the last run frame is running on the run frames."""
    cfg = small_cfg(2, 5)
    sd = random_state_dict(cfg, seed=6)
    sd64, ab = M.state64(sd)
    C, E = 16, cfg.nb_erb
    g = torch.Generator().manual_seed(7)
    T = 50
    run = torch.rand(T, generator=g) < 0.5
    run[0] = True
    idx = torch.nonzero(run).view(-1)
    dec = torch.rand(1, C, T, E // 4, generator=g)
    e3 = torch.rand(1, C, T, E // 4, generator=g)
    e0 = torch.rand(1, C, T, E, generator=g)
    d1 = torch.rand(1, C, T, E, generator=g)
    pl = G.plan(np.zeros((1, T), F32), None, 0, 0, [(0, 0, 0)], [False])
    pl["erb_run"][0] = run.numpy()
    pl["erb_src"][0] = [int(idx[idx <= t][-1]) for t in range(T)]
    flat = lambda x: x[0].permute(1, 2, 0).reshape(T, -1).numpy()   # noqa: E731
    unflat = lambda x, F_: torch.from_numpy(x.reshape(1, T, F_, C)).permute(0, 3, 1, 2).double()   # noqa: E731
    fd, f3, f0, f1 = (unflat(G.filled(flat(x), pl, 0, 0, None, False), x.shape[-1]) for x in (dec, e3, e0, d1))
    d3, bd3 = G.convt3(sd64, ab, fd, f3, 0)
    want = O.conv_norm_act(dec[:, :, idx] + O.conv_norm_act(e3[:, :, idx], sd, "erb_dec.conv3p"), sd, "erb_dec.convt3")
    assert err_ratio(want.numpy(), d3[:, :, idx].numpy(), bd3[:, :, idx].numpy()) <= 1
    m, bm = G.mask(sd64, ab, f0, f1, 0)
    p = O.conv_norm_act(e0[:, :, idx], sd, "erb_dec.conv0p") + d1[:, :, idx]
    want = O.conv_norm_act(p, sd, "erb_dec.conv0_out", act="sigmoid")
    assert err_ratio(want.numpy(), m[:, :, idx].numpy(), bm[:, :, idx].numpy()) <= 1
    # the mutation: a fill from frame t - 1 instead of the last run frame
    x = flat(dec)
    wrong = x.copy()
    for t in range(1, T):
        if not run[t]:
            wrong[t] = x[t - 1]
    assert not np.array_equal(wrong, G.filled(x, pl, 0, 0, None, False))


@pytest.mark.parametrize("which", ["min", "max_erb", "max_df"])
def test_plan_rejects_le_for_lt(which, monkeypatch):
    """`<=` for `<` (or `>=` for `>`) at any one threshold changes the flags of the tie frames."""
    th = THS[1]
    l = tie_rows(np.random.default_rng(3), th)
    good = G.plan(l, None, 0, 0, [th] * 3, [True] * 3)
    k = ["min", "max_erb", "max_df"].index(which)
    bumped = list(th)
    bumped[k] = float(np.nextafter(F32(th[k]), F32(np.inf if k == 0 else -np.inf)))   # x <= v is x < next(v) (x >= v: x > prev(v))
    bad = G.plan(l, None, 0, 0, [bumped] * 3, [True] * 3)
    assert not (np.array_equal(good["erb_run"], bad["erb_run"]) and np.array_equal(good["df_run"], bad["df_run"]))


def test_checks_reject_late_src_swapped_tails_and_early_erb_first():
    rng = np.random.default_rng(4)
    th = THS[1]
    T, Rc, K, W = 40, 8, 5, 6
    l = tie_rows(rng, th, T)
    pl = G.plan(l, [0, 0, 0], 0, Rc, [th] * 3, [True] * 3, has_run_prev=[True] * 3)
    x = rng.standard_normal((T, W)).astype(F32)
    carried = rng.standard_normal(W).astype(F32)
    b = int(np.argmax([(pl["erb_src"][r, Rc:] < 0).any() and (~pl["erb_run"][r, Rc:]).sum() > 2 for r in range(3)]))
    want = G.filled(x, pl, b, Rc, carried, False)
    # erb_src one frame late: the frame after the last run frame
    late = {k: v.copy() for k, v in pl.items()}
    src = pl["erb_src"][b, Rc:]
    late["erb_src"][b, Rc:] = np.where(src >= 0, src + 1, src)
    assert not np.array_equal(want, G.filled(x, late, b, Rc, carried, False))
    # after a runtime window: the halo row Rc - 1 taken where the carried row was meant
    assert not np.array_equal(want, G.filled(x, pl, b, Rc, carried, True))
    # after an apply-mode window: a stale carried row (not the recomputed halo row) taken where the halo row was meant
    stale = x[Rc - 1] + F32(1)
    halo = G.filled(x, pl, b, Rc, None, True)
    assert np.array_equal(halo[0], x[Rc - 1])
    assert not np.array_equal(halo, G.filled(x, pl, b, Rc, stale, False))
    c0 = rng.standard_normal((T, W)).astype(F32)
    carried_tail = rng.standard_normal((K - 1, W)).astype(F32)
    halo_tail = G.halo_tail(c0, Rc, K, 0)
    assert np.array_equal(halo_tail, c0[Rc - (K - 1):Rc])
    # the same two mistakes in the pathway tail: either window's expected rows differ from the other source's
    assert not np.array_equal(G.compact(c0, carried_tail, pl, b, Rc), G.compact(c0, halo_tail, pl, b, Rc))
    # the halo tail at Rc < K - 1 is zero before frame 0, and before the stream's first frame
    h = G.halo_tail(c0, 2, K, 0)
    assert not h[:2].any() and np.array_equal(h[2:], c0[:2])
    assert not G.halo_tail(c0, Rc, K, Rc - 1)[:3].any()
    # erb_first: a row that has never run reads padding before its first run frame, not from its stream's first frame
    fresh = G.plan(l, [0, 0, 0], 0, 0, [th] * 3, [True] * 3, has_run_prev=[False] * 3)
    r = int(np.argmax([not fresh["erb_run"][q, 0] for q in range(3)]))
    assert not fresh["erb_run"][r, 0]
    assert fresh["erb_first"][r] == int(np.argmax(fresh["erb_run"][r])) > 0
