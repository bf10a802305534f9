"""GPU: rated ragged batches (enhance_batch / enhance_device_ragged with sr=, dfb_enhance_ragged with rates).  The offline
resampler alone must be io.resample bit for bit over a ragged batch in any chunking, writing nothing outside its rows;
every entry of a rated batch must equal io.resample(enhance(io.resample(a, r, 48000)), 48000, r) within the ragged
path's bound; and the rated call must keep the batch path's invariants (device vs host, chunking, lanes, stream groups,
48 kHz calls unchanged, workspace)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet_oracle as O
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, enhance, enhance_batch, enhance_device_ragged, io, libdf, ragged
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.weights import random_state_dict

RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 88200, 96000)
SENTINEL = 777.0


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean()))


def cfg_of(kind):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5)
    if kind == "dfn3":
        return ModelConfig(model="deepfilternet3", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", **base)
    if kind == "dfn2":
        return ModelConfig(model="deepfilternet2", conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                           lin_groups=8, enc_lin_groups=8, enc_concat=True, **base)
    if kind == "v1":
        return ModelConfig(model="deepfilternet", conv_lookahead=2, df_lookahead=1, conv_ch=64, conv_kernel=(2, 3),
                           convt_kernel=(2, 3), conv_kernel_inp=(2, 3), conv_k_enc=2, conv_k_dec=2, emb_hidden_dim=512,
                           df_hidden_dim=512, emb_num_layers=3, df_num_layers=2, gru_groups=8, lin_groups=8, enc_lin_groups=8,
                           group_shuffle=True, dfop_method="real_unfold")
    return ModelConfig(model="deepfilternet3", conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), emb_hidden_dim=512,
                       df_hidden_dim=512, emb_num_layers=3, df_num_layers=3, lin_groups=16, enc_lin_groups=16,
                       df_gru_skip="groupedlinear", **base)


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


@pytest.fixture(scope="module")
def dfn3(st):
    cfg = cfg_of("dfn3")
    sd = random_state_dict(cfg, seed=41)
    return DfNet(cfg, sd, st), sd, cfg


# ---------------------------------------------------------------------------------------------- resampler alone ----
def resample_rows(model, up, rates, rows, bounds):
    """dfb_debug_resample_rows over rows (1-D float32 arrays) packed with gaps; returns (output buffer, offsets, lengths)"""
    in_off, pos = [], 3
    for x in rows:
        in_off.append(pos)
        pos += x.size + 5
    xin = np.full(pos, np.nan, np.float32)
    for o, x in zip(in_off, rows):
        xin[o:o + x.size] = x
    olens = [ragged.len_48k(x.size, r) if up else -(-x.size * r // 48000) for x, r in zip(rows, rates)]
    out_off, pos = [], 2
    for n in olens:
        out_off.append(pos)
        pos += n + 3
    d_in = torch.from_numpy(xin).cuda()
    d_out = torch.full((pos,), SENTINEL, device="cuda")
    a = lambda v: np.ascontiguousarray(np.asarray(v, np.int64))   # noqa: E731
    in_off, lens, out_off, bnd = a(in_off), a([x.size for x in rows]), a(out_off), a(bounds)
    r32 = np.ascontiguousarray(np.asarray(rates, np.int32))
    _lib.check(_lib.lib().dfb_debug_resample_rows(int(up), model.handle, d_in.data_ptr(), in_off.ctypes.data, lens.ctypes.data,
                                                  r32.ctypes.data, len(rows), d_out.data_ptr(), out_off.ctypes.data,
                                                  bnd.ctypes.data, bnd.size, torch.cuda.current_stream().cuda_stream))
    return d_out.cpu(), out_off, olens


def chunkings(total):
    """1 chunk; 6 hop-aligned chunks; irregular bounds, not multiples of any nw"""
    def closed(b):   # increasing, > 0, the last past every row's end
        b = sorted({x for x in b if x > 0})
        return b if b[-1] > total else b + [total + 1]
    six = [int(math.ceil(total * k / 6 / 480)) * 480 for k in range(1, 7)]
    odd = [1, 2, 37, 1001, 7919, total // 3 + 13, total // 2 + 1, total - 1, total]
    return [closed([total + 1]), closed(six), closed(odd)]


@pytest.mark.parametrize("rate", RATES)
def test_resample_rows_bit_exact(dfn3, rate):
    model = dfn3[0]
    model.add_rate(rate)
    rng = np.random.default_rng(rate)
    for up in (True, False):
        # from 1 sample to 20 s, some shorter than one tap span
        src = rate if up else 48000
        lens = [1, 3, 17, 40, 1234, src // 3 + 7, 20 * src]
        rows = [(rng.standard_normal(n) * 0.3).astype(np.float32) for n in lens]
        rates = [rate] * len(rows)
        refs = [io.resample(torch.from_numpy(x)[None], rate if up else 48000, 48000 if up else rate)[0] for x in rows]
        total = max(ragged.len_48k(n, rate) for n in lens) if up else max(lens)
        for bounds in chunkings(total):
            got, out_off, olens = resample_rows(model, up, rates, rows, bounds)
            mask = torch.ones(got.numel(), dtype=torch.bool)
            for b, (o, n, ref) in enumerate(zip(out_off, olens, refs)):
                assert n == ref.numel(), (rate, up, b)
                g = got[o:o + n]
                assert torch.equal(g.view(torch.int32), ref.view(torch.int32)), (rate, up, b, len(bounds))
                mask[o:o + n] = False
            assert (got[mask] == SENTINEL).all(), (rate, up, len(bounds))


# ------------------------------------------------------------------------------------------- end to end ----
def composition(model, st, a, r, pad=True, **kw):
    x48 = io.resample(a, r, 48000) if r != 48000 else a
    y48 = enhance(model, st, x48.contiguous(), pad=pad, **kw)
    return io.resample(y48, 48000, r) if r != 48000 else y48


MIX = [(8000, 8000 * 2 + 37), (11025, 11025 + 5), (16000, 16000 * 3 + 11), (44100, 44100 + 901), (48000, 48000 + 240),
       (16000, 1601), (8000, 4000 + 3)]


def entries(mix, seed, channels=1):
    return [(synth_audio(channels, n, seed=seed + i), r) for i, (r, n) in enumerate(mix)]


def assert_composition(model, st, ents, tol=1e-6, pad=True, **kw):
    outs = enhance_batch(model, st, [a for a, _ in ents], pad=pad, sr=[r for _, r in ents], **kw)
    for i, ((a, r), y) in enumerate(zip(ents, outs)):
        ref = composition(model, st, a, r, pad=pad, **kw)
        assert tuple(y.shape) == tuple(ref.shape), (i, r, tuple(y.shape), tuple(ref.shape))
        assert tuple(y.shape) == (a.shape[0], ragged.out_len_at(a.shape[1], r, 480, pad))
        assert int(_lib.lib().dfb_enhance_out_len_at(st.handle, a.shape[1], int(pad), r)) == y.shape[1]
        assert rms(y, ref) < tol, (i, r, rms(y, ref))
    return outs


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_rated_batch_equals_the_composition(st, kind):
    cfg = cfg_of(kind)
    model = DfNet(cfg, random_state_dict(cfg, seed=42), st)
    assert_composition(model, st, entries(MIX, seed=500))


def test_rated_batch_v1(st):
    cfg = cfg_of("v1")
    model = DfNet(cfg, random_state_dict(cfg, seed=43), st)
    assert_composition(model, st, entries([(16000, 8000 + 17), (8000, 8000 + 3), (48000, 24000), (44100, 22050)], seed=520))


@pytest.mark.parametrize("opt", ["nopad", "atten", "mean", "max"])
def test_rated_batch_options(st, dfn3, opt):
    model = dfn3[0]
    if opt == "nopad":
        assert_composition(model, st, entries(MIX, seed=540), pad=False)
    elif opt == "atten":
        assert_composition(model, st, entries(MIX, seed=560), atten_lim_db=6)
    else:
        ents = entries(MIX[:4], seed=580, channels=2) + entries(MIX[4:], seed=590)
        assert_composition(model, st, ents, reduce_mask=opt)


def test_16k_entry_against_the_oracle(st, dfn3):
    model, sd, cfg = dfn3
    a = synth_audio(1, 16000 * 2 + 77, seed=600)
    y = enhance_batch(model, st, [a, synth_audio(1, 30000, seed=601)], sr=[16000, 48000])[0]
    ref = io.resample(torch.as_tensor(O.enhance(sd, cfg.as_dict(), io.resample(a, 16000, 48000), pad=True)), 48000, 16000)
    assert y.shape == ref.shape
    assert rms(y, ref) < 1e-4, rms(y, ref)


# ------------------------------------------------------------------------------------------- invariants ----
def device_rows(ents):
    lens = [a.shape[1] for a, _ in ents]
    x = torch.zeros(len(ents), max(lens))
    for b, (a, _) in enumerate(ents):
        x[b, :lens[b]] = a[0]
    return x.cuda(), lens, [r for _, r in ents]


def test_device_equals_host_and_chunking(st):
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=44), st)
    ents = entries([(16000, 16000 * 9 + 5), (8000, 8000 * 6 + 1), (44100, 44100 * 4 + 7), (48000, 48000 * 5 + 3),
                    (11025, 11025 * 7), (16000, 16000 + 1)], seed=620)
    x, lens, rates = device_rows(ents)
    host = enhance_batch(model, st, [a for a, _ in ents], sr=rates)
    runs = {}
    for ch in [(1, 1, 1), (4, 4, 1), (4, 4, 2), (8, 8, 2), (8, 8, 1)]:
        model.set_chunking(*ch)
        runs[("dev",) + ch] = enhance_device_ragged(model, st, x, lens, sr=rates).cpu()
        hb = enhance_batch(model, st, [a for a, _ in ents], sr=rates)
        runs[("host",) + ch] = torch.zeros_like(runs[("dev",) + ch])
        for b, y in enumerate(hb):
            runs[("host",) + ch][b, :y.shape[1]] = y[0]
    model.set_chunking(0, 4, 2)
    # stream groups: a workspace cap that holds two streams per group
    model.set_max_workspace(model.workspace_bytes() // 3)
    runs["groups_dev"] = enhance_device_ragged(model, st, x, lens, sr=rates).cpu()
    model.set_max_workspace(40 << 30)
    ref = runs[("dev", 1, 1, 1)]
    for b, (y, r) in enumerate(zip(host, rates)):
        n = y.shape[1]
        assert ref.shape[1] >= n
        assert rms(ref[b, :n], y[0]) < 1e-6, b
        assert (ref[b, n:] == 0).all(), b
    for k, v in runs.items():
        assert rms(v, ref) < 1e-6, k


def test_48k_calls_are_unchanged(st, dfn3):
    model = dfn3[0]
    a = [synth_audio(2, 30000, seed=640), synth_audio(1, 4801, seed=641)]
    base = enhance_batch(model, st, a)
    for sr in (None, 48000, [48000, 48000]):
        got = enhance_batch(model, st, a, sr=sr)
        assert all(torch.equal(g, b) for g, b in zip(got, base)), sr
    x, lens, _ = device_rows([(a[1], 48000), (a[0][:1], 48000)])
    d0 = enhance_device_ragged(model, st, x, lens)
    assert torch.equal(enhance_device_ragged(model, st, x, lens, sr=48000), d0)
    assert torch.equal(enhance(model, st, a[0], sr=48000), enhance(model, st, a[0]))
    # one packed batch through dfb_enhance_ragged(_host): rates all 48 kHz are rates null, with or without link groups, and
    # link groups of one are groups null, bit for bit and in as many launches
    L = _lib.lib()
    i64 = lambda v: np.ascontiguousarray(np.asarray(v, np.int64))   # noqa: E731
    lens = i64([30000, 30000, 4801, 12345, 12345, 12345])
    off, n = i64(np.concatenate(([0], np.cumsum(lens)[:-1]))), int(lens.sum())
    ones, groups, r48 = i64([1] * 6), i64([2, 1, 3]), np.full(6, 48000, np.int32)
    x = synth_audio(1, n, seed=642)[0].contiguous()
    stream = torch.cuda.current_stream().cuda_stream

    def run(dev, g=None, n_groups=0, reduce=0, rates=None):
        src, out = (x.cuda(), torch.zeros(n, device="cuda")) if dev else (x, torch.zeros(n))
        n0 = L.dfb_kernel_launches()
        args = (model.handle, st.handle, src.data_ptr(), n, off.ctypes.data, lens.ctypes.data, 6, 1, 0.0, out.data_ptr(), n,
                off.ctypes.data, g, n_groups, reduce, rates, None, 0, None, 0, None)
        _lib.check(L.dfb_enhance_ragged(*args, stream) if dev else L.dfb_enhance_ragged_host(*args))
        return out.cpu(), L.dfb_kernel_launches() - n0

    for dev in (True, False):
        plain = run(dev)
        linked = run(dev, groups.ctypes.data, 3, 2)
        assert not torch.equal(linked[0], plain[0]), dev
        for got, ref in ((run(dev, rates=r48.ctypes.data), plain),
                         (run(dev, ones.ctypes.data, 6, 2), plain),
                         (run(dev, groups.ctypes.data, 3, 2, r48.ctypes.data), linked)):
            assert torch.equal(got[0], ref[0]) and got[1] == ref[1], (dev, got[1], ref[1])


def test_workspace_of_a_rated_call(st):
    cfg = cfg_of("dfn3")
    m16, m48 = DfNet(cfg, random_state_dict(cfg, seed=45), st), DfNet(cfg, random_state_dict(cfg, seed=45), st)
    enhance_batch(m16, st, [torch.randn(1, 16000 * 120) * 0.1 for _ in range(8)], sr=16000)
    enhance_batch(m48, st, [torch.randn(1, 48000 * 120) * 0.1 for _ in range(8)])
    assert 0 < m16.workspace_bytes() <= m48.workspace_bytes()


# ----------------------------------------------------------------------------------------------- errors ----
def test_errors(st, dfn3):
    model = dfn3[0]
    a = synth_audio(1, 16000, seed=660)
    with pytest.raises(ValueError, match="47999"):
        enhance_batch(model, st, [a], sr=47999)
    taps = torch.zeros(16)
    rc = _lib.lib().dfb_model_add_rate(model.handle, 47999, taps.data_ptr(), 47999, 48000, 17, taps.data_ptr(), 48000, 47999, 17)
    assert rc == _lib.DFB_ERR_UNSUPPORTED and b"47999" in _lib.lib().dfb_last_error()
    with pytest.raises(ValueError, match="2 sample rates for 3"):
        enhance_batch(model, st, [a, a, a], sr=[16000, 8000])
    with pytest.raises(RuntimeError, match="shorter than one hop"):
        enhance_batch(model, st, [synth_audio(1, 100, seed=661)], pad=False, sr=16000)
    x, lens, _ = device_rows([(a, 16000), (a, 16000)])
    with pytest.raises(ValueError, match="different sample rates"):
        enhance_device_ragged(model, st, x, lens, group_sizes=[2], reduce_mask="mean", sr=[16000, 8000])
    # the C ABI's own checks: an unregistered rate, and mixed rates in a link group (one 48 kHz length: 48000 samples)
    y = torch.zeros(2, 20000, device="cuda")
    i64 = lambda v: np.ascontiguousarray(np.asarray(v, np.int64))   # noqa: E731
    off, ln, oo, g = i64([0, 16000]), i64([16000, 8000]), i64([0, 20000]), i64([2])
    for rates, groups in (([16000, 12345], None), ([16000, 8000], g)):
        model.add_rate(8000)
        r32 = np.ascontiguousarray(np.asarray(rates, np.int32))
        rc = _lib.lib().dfb_enhance_ragged(model.handle, st.handle, x.data_ptr(), x.numel(), off.ctypes.data, ln.ctypes.data,
                                           2, 1, 0.0, y.data_ptr(), y.numel(), oo.ctypes.data,
                                           groups.ctypes.data if groups is not None else None, 1 if groups is not None else 0,
                                           2 if groups is not None else 0, r32.ctypes.data, None, 0, None, 0, None,
                                           torch.cuda.current_stream().cuda_stream)
        assert rc == _lib.DFB_ERR_INVALID, rates
