"""GPU: ragged batches (streams of different lengths in one call, dfb_enhance_ragged).  Every stream's output must equal the
same stream enhanced alone -- over the whole stream and over its last 100 ms separately, where the look-ahead meets the
stream's end -- whatever the order, layout, time chunking, lanes and stream groups; zero-padding the batch is shown not to
give that."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet_oracle as O
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, enhance, enhance_batch, enhance_device, enhance_device_ragged, init_df, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TAIL = 4800   # the last 100 ms of a stream: its last look-ahead frames and the overlap-add tail


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
def states():
    return libdf.DF(48000, 960, 480, 32, 2)


def out_len(t, pad):
    return t if pad else (t // HOP) * HOP


# about a dozen streams, unsorted: 1 sample, around one hop, 0.1 s (+1), several seconds plus a partial hop, a duplicate
LENGTHS_PAD = [4801, 1, 48000 * 3 + 123, 480, 481, 479, 48000 * 2 + 17, 4801, 9600, 48000 + 240, 24000 + 1, 48000 * 4 + 311]
LENGTHS_NOPAD = [4801, 480, 48000 * 3 + 123, 481, 959, 48000 * 2 + 17, 4801, 9600, 48000 + 240, 24000 + 1, 48000 * 4 + 311, 1440]


def padded(lengths, seed):
    """[B, max] CUDA tensor, row b = lengths[b] samples of a synthetic noisy stream, zeros after."""
    x = synth_audio(len(lengths), max(lengths), seed=seed)
    for b, t in enumerate(lengths):
        x[b, t:] = 0
    return x.cuda()


def alone(model, st, x, lengths, pad, **kw):
    """Every stream through enhance_device on its own."""
    return [enhance_device(model, st, x[b:b + 1, :t].contiguous(), pad=pad, **kw)[0].cpu() for b, t in enumerate(lengths)]


def assert_per_stream(got, refs, lengths, pad, tol=1e-6):
    got = got.cpu()
    for b, (r, t) in enumerate(zip(refs, lengths)):
        n = out_len(t, pad)
        assert r.shape[0] == n, (b, t)
        g = got[b, :n]
        assert rms(g, r) < tol, (b, t, rms(g, r))
        assert rms(g[-TAIL:], r[-TAIL:]) < tol, (b, t, "tail", rms(g[-TAIL:], r[-TAIL:]))
        assert not got[b, n:].any(), (b, t)


@pytest.mark.parametrize("pad", [True, False])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_ragged_equals_each_stream_alone(states, kind, pad):
    st = states
    cfg = cfg_of(kind)
    sd = random_state_dict(cfg, seed=31)
    model = DfNet(cfg, sd, st)
    lengths = LENGTHS_PAD if pad else LENGTHS_NOPAD
    x = padded(lengths, seed=81)
    got = enhance_device_ragged(model, st, x, lengths, pad=pad)
    assert got.shape == (len(lengths), max(out_len(t, pad) for t in lengths))
    refs = alone(model, st, x, lengths, pad)
    assert_per_stream(got, refs, lengths, pad)
    for b in (0, 9):   # 4801 and 48240 samples against the CPU oracle
        t = lengths[b]
        ref = O.enhance(sd, cfg.as_dict(), x[b:b + 1, :t].cpu(), pad=pad)[0]
        assert rms(got[b, :out_len(t, pad)].cpu(), ref) < 1e-4, b


def test_zero_padding_is_not_equivalent(states):
    """Zero-padding to the longest stream and cropping changes the end of every padded stream: its last look-ahead frames
    see the features of padded frames (10 log10(1e-10), normalised) instead of the end of the stream."""
    st = states
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=31), st)
    lengths = [48000 * 2 + 17, 24000 + 1, 9600, 4801, 48000 + 240]
    x = padded(lengths, seed=82)
    ragged = enhance_device_ragged(model, st, x, lengths).cpu()
    zp = enhance_device(model, st, x).cpu()
    diffs = []
    for b, t in enumerate(lengths[1:], 1):
        diffs.append(rms(ragged[b, t - TAIL:t], zp[b, t - TAIL:t]))
        assert rms(ragged[b, :t - TAIL], zp[b, :t - TAIL]) < 1e-6, b   # before the tail both are the same computation
    assert min(diffs) > 1e-5, diffs
    assert rms(ragged[0], zp[0]) < 1e-6                                   # the longest stream is not padded


# 502 frames for the longest stream: 6 chunks of 84 frames; 79680 samples end exactly at the last frame of chunk 2
# ((79680 + 960) / 480 = 168), 40000 one frame into chunk 3, the others in chunks 1, 2, 4 and 5
CHUNK_LENGTHS = [40000, 48000 * 5 + 123, 500, 79680, 120000, 4801, 200000, 79680 + 480]


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_ragged_chunks_lanes_and_groups(states, kind):
    st = states
    cfg = cfg_of(kind)
    sd = random_state_dict(cfg, seed=32)
    model = DfNet(cfg, sd, st)
    lengths = CHUNK_LENGTHS
    x = padded(lengths, seed=83)
    model.set_chunking(1, 1, 1)
    one = enhance_device_ragged(model, st, x, lengths).clone()
    torch.cuda.synchronize()
    per_stream = model.workspace_bytes() / len(lengths)
    runs = {}
    for ch in [(6, 6, 1), (6, 6, 2)]:
        model.set_chunking(*ch)
        runs[ch] = enhance_device_ragged(model, st, x, lengths).clone()
    runs["host"] = torch.zeros_like(one)
    for b, y in enumerate(enhance_batch(model, st, [x[b:b + 1, :t].cpu() for b, t in enumerate(lengths)])):
        runs["host"][b, :y.shape[1]] = y[0].cuda()
    # ~50-frame windows for 3 streams per lane: the 8 streams no longer fit one window and run as stream groups
    model.set_max_workspace(int(per_stream * 3 * 2 * 60 / 512))
    runs["groups"] = enhance_device_ragged(model, st, x, lengths).clone()
    runs["groups_host"] = torch.zeros_like(one)
    for b, y in enumerate(enhance_batch(model, st, [x[b:b + 1, :t].cpu() for b, t in enumerate(lengths)])):
        runs["groups_host"][b, :y.shape[1]] = y[0].cuda()
    torch.cuda.synchronize()
    model.set_max_workspace(64 << 30)
    model.set_chunking(0, 4, 2)
    for name, r in runs.items():
        assert rms(one.cpu(), r.cpu()) < 1e-6, name
    assert_per_stream(one, alone(model, st, x, lengths, True), lengths, True)


def test_layouts_order_and_untouched_output(states):
    st = states
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=33), st)
    lengths = LENGTHS_PAD
    x = padded(lengths, seed=84)
    dev = enhance_device_ragged(model, st, x, lengths).cpu()
    host = enhance_batch(model, st, [x[b:b + 1, :t].cpu() for b, t in enumerate(lengths)])
    for b, t in enumerate(lengths):
        assert host[b].shape == (1, t) and rms(host[b][0], dev[b, :t]) < 1e-6, b
    perm = [5, 2, 11, 0, 7, 3, 9, 1, 10, 4, 8, 6]
    pdev = enhance_device_ragged(model, st, x[perm].contiguous(), [lengths[p] for p in perm]).cpu()
    for i, p in enumerate(perm):
        assert rms(pdev[i], dev[p]) < 1e-6, (i, p)
    # equal lengths through the ragged API == enhance_device
    eq = synth_audio(5, 48000 + 123, seed=85).cuda()
    assert rms(enhance_device_ragged(model, st, eq, [eq.shape[1]] * 5).cpu(), enhance_device(model, st, eq).cpu()) < 1e-6
    # the C entry writes each stream's own output range and nothing else
    L = _lib.lib()
    lens = np.array([4801, 960, 30000], np.int64)
    src = synth_audio(1, int(lens.sum()) + 100, seed=86).cuda()[0].contiguous()
    in_off = np.array([100, 100 + 4801, 100 + 4801 + 960], np.int64)
    out_off = np.array([7, 5000, 7000], np.int64)
    out_d = torch.full((40000,), 7.0, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    no_extras = (None, 0, 0, None, None, 0, None, 0, None)   # no link groups, rates, settings or LSNR rows
    _lib.check(L.dfb_enhance_ragged(model.handle, st.handle, src.data_ptr(), src.numel(), in_off.ctypes.data, lens.ctypes.data, 3, 1,
                                    0.0, out_d.data_ptr(), out_d.numel(), out_off.ctypes.data, *no_extras, stream))
    out = out_d.cpu()
    mask = torch.ones(40000, dtype=torch.bool)
    for o, t, i in zip(out_off, lens, in_off):
        mask[o:o + t] = False
        ref = enhance_device(model, st, src[i:i + t][None].contiguous())[0].cpu()
        assert rms(out[o:o + t], ref) < 1e-6
    assert (out[mask] == 7.0).all()
    # offsets outside the buffers are refused
    for io_, oo_, n_in, n_out in ((in_off, out_off, int(in_off[-1] + lens[-1] - 1), 40000), (in_off, out_off, src.numel(), 36999),
                                  (np.array([-1, 0, 0], np.int64), out_off, src.numel(), 40000)):
        rc = L.dfb_enhance_ragged(model.handle, st.handle, src.data_ptr(), n_in, io_.ctypes.data, lens.ctypes.data, 3, 1, 0.0,
                                  out_d.data_ptr(), n_out, oo_.ctypes.data, *no_extras, stream)
        assert rc == _lib.DFB_ERR_INVALID


@pytest.mark.parametrize("opt", ["atten", "post_filter", "mask_only"])
def test_ragged_options(states, model_dir, opt):
    st = states
    if opt == "atten":
        cfg = cfg_of("dfn3")
        model, kw = DfNet(cfg, random_state_dict(cfg, seed=34), st), dict(atten_lim_db=12.0)
    else:
        model, st, _, _ = init_df(os.path.join(model_dir, "DeepFilterNet3"), log_level="ERROR", **{opt: True})
        kw = {}
    lengths = [24000 + 1, 4801, 48000 * 2 + 17, 481, 9600]
    x = padded(lengths, seed=87)
    got = enhance_device_ragged(model, st, x, lengths, **kw)
    assert_per_stream(got, alone(model, st, x, lengths, True, **kw), lengths, True)


def test_ragged_v1(states):
    """DeepFilterNet v1 runs one window per signal: its stream groups share one frame count.  9600 + 123 and 9600 + 300
    samples have the same frame count (22 with pad, 20 without) but different lengths, so they run in one group."""
    st = states
    cfg = cfg_of("v1")
    model = DfNet(cfg, random_state_dict(cfg, seed=35), st)
    lengths = [24000, 9600 + 123, 24000, 9600 + 300, 9600 + 123, 24000]
    x = padded(lengths, seed=88)
    for pad in (True, False):
        dev = enhance_device_ragged(model, st, x, lengths, pad=pad)
        assert_per_stream(dev, alone(model, st, x, lengths, pad), lengths, pad, tol=1e-7)
        host = enhance_batch(model, st, [x[b:b + 1, :t].cpu() for b, t in enumerate(lengths)], pad=pad)
        for b, t in enumerate(lengths):
            n = out_len(t, pad)
            assert host[b].shape == (1, n) and rms(host[b][0], dev[b, :n].cpu()) < 1e-7, (b, pad)


def test_enhance_batch_api_and_errors(states):
    st = states
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=36), st)
    a = [synth_audio(2, 30000, seed=89), synth_audio(1, 4801, seed=90), synth_audio(3, 12345, seed=91)]
    outs = enhance_batch(model, st, a)
    for x, y in zip(a, outs):
        assert y.shape == x.shape and rms(y, enhance(model, st, x)) < 1e-6
    outs = enhance_batch(model, st, a, pad=False, atten_lim_db=6.0)
    for x, y in zip(a, outs):
        assert rms(y, enhance(model, st, x, pad=False, atten_lim_db=6.0)) < 1e-6
    with pytest.raises(ValueError):
        enhance_batch(model, st, [torch.zeros(480)])
    with pytest.raises(ValueError):
        enhance_batch(model, st, [torch.zeros(1, 480), torch.zeros(1, 0)])
    with pytest.raises(ValueError):
        enhance_batch(model, st, [])
    with pytest.raises(RuntimeError):
        enhance_batch(model, st, [torch.zeros(1, 4800), torch.zeros(1, 100)], pad=False)
    with pytest.raises(RuntimeError):
        enhance(model, st, torch.zeros(1, 100), pad=False)
    x = torch.zeros(2, 960, device="cuda")
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x, [960, 961])
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x, [960, 0])
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x, [960])
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x[0], [960])


def test_cli_batch_size(tmp_path, model_dir):
    from deepfilternet_b200 import io as dio
    from deepfilternet_b200.enhance import run
    src = []
    for i, t in enumerate([48000 + 123, 24000, 96000 + 7]):
        p = str(tmp_path / f"in{i}.wav")
        dio.save_audio(p, synth_audio(1, t, seed=92 + i), 48000)
        src.append(p)
    m = os.path.join(model_dir, "DeepFilterNet3")
    assert run(["-m", m, "-o", str(tmp_path / "b1"), "--log-level", "ERROR"] + src) == 0
    assert run(["-m", m, "-o", str(tmp_path / "b3"), "--log-level", "ERROR", "--batch-size", "3"] + src) == 0
    for i in range(3):
        one, _ = dio.load_audio(str(tmp_path / "b1" / f"in{i}_DeepFilterNet3.wav"))
        three, _ = dio.load_audio(str(tmp_path / "b3" / f"in{i}_DeepFilterNet3.wav"))
        assert one.shape == three.shape and float((one - three).abs().max()) <= 1.0 / 32768.0 + 1e-7, i
