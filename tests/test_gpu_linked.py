"""GPU: linked channels (dfb_enhance_ragged's link groups, dfb_stream_set_mask_reduce).  The channels of a recording share one ERB
mask, the max or mean of theirs; everything else stays per channel.  Checked against the CPU restatement
(tests/linked_oracle.py), against the unlinked path where linking must change nothing, and against each recording
enhanced alone, whatever the batch order, time chunking, lanes and stream groups."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import linked_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, enhance_batch, enhance_device_ragged, init_df, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.streaming import SLOT_FREE, SLOT_OPEN
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TAIL = 4800   # the last 100 ms of a stream


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


def recordings(entries, seed):
    """entries [(channels, length)] -> list of CPU [C, T] recordings with different channels (distinct noise seeds)."""
    return [synth_audio(c, t, seed=seed + 10 * i) for i, (c, t) in enumerate(entries)]


def pack(recs):
    """Recordings -> padded [B, S] CUDA tensor, lengths, group sizes."""
    lengths = [r.shape[1] for r in recs for _ in range(r.shape[0])]
    x = torch.zeros(len(lengths), max(lengths))
    b = 0
    for r in recs:
        x[b:b + r.shape[0], :r.shape[1]] = r
        b += r.shape[0]
    return x.cuda(), lengths, [r.shape[0] for r in recs]


def split(y, recs, pad):
    """[B, max out] result -> per recording [C, out_len] CPU tensors."""
    out, b = [], 0
    y = y.cpu()
    for r in recs:
        out.append(y[b:b + r.shape[0], :out_len(r.shape[1], pad)])
        b += r.shape[0]
    return out


def linked_alone(model, st, recs, pad, reduce):
    out = []
    for r in recs:
        x = r.cuda().contiguous()
        out.append(enhance_device_ragged(model, st, x, [r.shape[1]] * r.shape[0], pad=pad, group_sizes=[r.shape[0]],
                                         reduce_mask=reduce).cpu())
    return out


def assert_close(got, want, tol, what):
    for g, w in zip(got, want):
        assert g.shape == w.shape, what
        for c in range(g.shape[0]):
            assert rms(g[c], w[c]) <= tol, (what, c, rms(g[c], w[c]))
            assert rms(g[c, -TAIL:], w[c, -TAIL:]) <= tol, (what, c, "tail", rms(g[c, -TAIL:], w[c, -TAIL:]))


GROUPS = [(2, 48000 + 123), (3, 24000 + 1), (1, 9600 + 7)]


@pytest.mark.parametrize("reduce", ["max", "mean"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_linked_matches_oracle(states, kind, reduce):
    st = states
    cfg = cfg_of(kind)
    sd = random_state_dict(cfg, seed=61)
    model = DfNet(cfg, sd, st)
    recs = recordings(GROUPS, seed=300)
    x, lengths, groups = pack(recs)
    for pad in (True, False):
        got = split(enhance_device_ragged(model, st, x, lengths, pad=pad, group_sizes=groups, reduce_mask=reduce), recs, pad)
        want = [LO.enhance(sd, cfg.as_dict(), r, pad=pad, reduce=reduce) for r in recs]
        assert_close(got, want, 5e-6, (kind, reduce, pad))
        if pad:   # not vacuous: the linked channels differ from the unlinked ones
            free = split(enhance_device_ragged(model, st, x, lengths, pad=pad), recs, pad)
            assert rms(got[0][0], free[0][0]) > 1e-4


@pytest.mark.parametrize("kind", ["dfn3", "dfn2"])
def test_none_and_singletons_are_unlinked(states, kind):
    st = states
    cfg = cfg_of(kind)
    model = DfNet(cfg, random_state_dict(cfg, seed=62), st)
    recs = recordings(GROUPS, seed=310)
    x, lengths, groups = pack(recs)
    free = enhance_device_ragged(model, st, x, lengths)
    for kw in (dict(group_sizes=groups, reduce_mask=None), dict(group_sizes=groups, reduce_mask="none"),
               dict(group_sizes=[1] * len(lengths), reduce_mask="max"), dict(group_sizes=[1] * len(lengths), reduce_mask="mean")):
        y = enhance_device_ragged(model, st, x, lengths, **kw)
        assert float((y - free).abs().max()) <= 1e-7, kw


# unsorted, mixed lengths and channel counts; entries 0 and 1 (and 4) have one length and sit next to each other
BATCH = [(2, 48000 * 2 + 17), (3, 48000 * 2 + 17), (1, 4801), (2, 24000 + 1), (2, 48000 * 2 + 17), (1, 48000 * 3 + 123),
         (3, 9600)]


@pytest.mark.parametrize("reduce", ["max", "mean"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_linked_batch_equals_each_recording_alone(states, kind, reduce):
    st = states
    cfg = cfg_of(kind)
    model = DfNet(cfg, random_state_dict(cfg, seed=63), st)
    recs = recordings(BATCH, seed=320)
    x, lengths, groups = pack(recs)
    for pad in (True, False):
        got = split(enhance_device_ragged(model, st, x, lengths, pad=pad, group_sizes=groups, reduce_mask=reduce), recs, pad)
        assert_close(got, linked_alone(model, st, recs, pad, reduce), 1e-6, (kind, reduce, pad))


# 418 frames for the longest stream, 6 chunks of 70; sorted: 2 x 200000 | 2 x 120000 | 3 x 79680 | 1 x 40000.  Stream
# groups of 3 would cut the second recording in two.
CHUNK_BATCH = [(3, 79680), (2, 120000), (1, 40000), (2, 200000)]


@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_linked_chunks_lanes_and_groups(states, kind):
    st = states
    cfg = cfg_of(kind)
    model = DfNet(cfg, random_state_dict(cfg, seed=64), st)
    recs = recordings(CHUNK_BATCH, seed=330)
    x, lengths, groups = pack(recs)
    want = linked_alone(model, st, recs, True, "mean")
    model.set_chunking(1, 1, 1)
    one = enhance_device_ragged(model, st, x, lengths, group_sizes=groups, reduce_mask="mean").clone()
    torch.cuda.synchronize()
    per_stream = model.workspace_bytes() / len(lengths)
    runs = {"1,1,1": one}
    for ch in [(6, 6, 1), (6, 6, 2)]:
        model.set_chunking(*ch)
        runs[ch] = enhance_device_ragged(model, st, x, lengths, group_sizes=groups, reduce_mask="mean").clone()
        # the device call is asynchronous and a host call on the same model reuses its stream tables: order them
        torch.cuda.synchronize()
        runs[(ch, "host")] = enhance_batch(model, st, recs, reduce_mask="mean")
    # room for about 3 streams per lane: the natural cut after the third stream falls inside the 2 x 120000 recording
    model.set_max_workspace(int(per_stream * 3 * 2 * 60 / 512))
    runs["groups"] = enhance_device_ragged(model, st, x, lengths, group_sizes=groups, reduce_mask="mean").clone()
    torch.cuda.synchronize()
    runs["groups_host"] = enhance_batch(model, st, recs, reduce_mask="mean")
    # room for about one stream: the 3-channel recording cannot be split, so the call fails instead
    model.set_max_workspace(int(per_stream * 2 * 60 / 512))
    enhance_device_ragged(model, st, x, lengths)   # the unlinked batch still runs, one stream at a time
    with pytest.raises(_lib.DfbError) as e:
        enhance_device_ragged(model, st, x, lengths, group_sizes=groups, reduce_mask="mean")
    assert e.value.code == _lib.DFB_ERR_OOM
    torch.cuda.synchronize()
    with pytest.raises(_lib.DfbError) as e:
        enhance_batch(model, st, recs, reduce_mask="mean")
    assert e.value.code == _lib.DFB_ERR_OOM
    torch.cuda.synchronize()
    model.set_max_workspace(64 << 30)
    model.set_chunking(0, 4, 2)
    for name, r in runs.items():
        got = r if isinstance(r, list) else split(r, recs, True)
        assert_close(got, want, 1e-6, (kind, name))


def test_host_device_and_batch_entry_points(states):
    st = states
    cfg = cfg_of("dfn3")
    model = DfNet(cfg, random_state_dict(cfg, seed=65), st)
    recs = recordings(BATCH, seed=340)
    x, lengths, groups = pack(recs)
    for reduce in ("max", "mean"):
        for pad in (True, False):
            dev = split(enhance_device_ragged(model, st, x, lengths, pad=pad, group_sizes=groups, reduce_mask=reduce), recs, pad)
            batch = enhance_batch(model, st, recs, pad=pad, reduce_mask=reduce)
            one = [enhance(model, st, r, pad=pad, reduce_mask=reduce) for r in recs]
            assert_close(batch, dev, 1e-6, (reduce, pad, "host/device"))
            assert_close(batch, one, 1e-6, (reduce, pad, "batch/enhance"))
    # reduce none through enhance is the unchanged call; errors
    r = recs[0]
    assert torch.equal(enhance(model, st, r, reduce_mask="none"), enhance(model, st, r))
    with pytest.raises(ValueError):
        enhance(model, st, r, reduce_mask="avg")
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x, lengths, reduce_mask="max")                 # no groups
    with pytest.raises(ValueError):
        enhance_device_ragged(model, st, x, lengths, group_sizes=[2, 3], reduce_mask="max")
    with pytest.raises(ValueError):   # 4801 and 24001 samples in one group
        enhance_device_ragged(model, st, x[5:9].contiguous(), lengths[5:9], group_sizes=[1, 3], reduce_mask="max")
    # the C entry point validates on its own
    L = _lib.lib()
    lens = np.array([4801, 4802], np.int64)
    off = np.array([0, 4801], np.int64)
    src = torch.zeros(9603, device="cuda")
    dst = torch.zeros(9603, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for g, red in (([2], 1), ([1, 2], 1), ([1, 1], 3)):
        g = np.array(g, np.int64)
        rc = L.dfb_enhance_ragged(model.handle, st.handle, src.data_ptr(), 9603, off.ctypes.data, lens.ctypes.data, 2, 1, 0.0,
                                  dst.data_ptr(), 9603, off.ctypes.data, g.ctypes.data, g.size, red, None, None, 0, None, 0, None,
                                  stream)
        assert rc == _lib.DFB_ERR_INVALID, (g, red)


@pytest.mark.parametrize("reduce", ["max", "mean"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2", "ll"])
def test_streaming_linked_equals_one_shot(states, kind, reduce):
    st = states
    cfg = cfg_of(kind)
    model = DfNet(cfg, random_state_dict(cfg, seed=66), st)
    n = 157
    recs = recordings([(2, HOP * n), (2, HOP * n)], seed=350)
    audio = torch.cat(recs, 0)
    ref = torch.cat([enhance(model, st, r, pad=False, reduce_mask=reduce) for r in recs], 0)
    s = DfStream(model, st, batch=4, channels=2, reduce_mask=reduce)
    assert s.slot_states().tolist() == [SLOT_OPEN] * 4 and s.slot_groups().tolist() == [0, 0, 2, 2]
    outs, pos = [], 0
    for i, k in enumerate([1, 1, 2, 1, 7, 40, 1, 3, 64, 30, 7]):
        xk = audio[:, pos * HOP:(pos + k) * HOP]
        outs.append(s.process(xk.cuda() if i % 2 else xk).cpu())
        pos += k
    outs.append(s.flush())
    assert s.slot_states().tolist() == [SLOT_FREE] * 4 and s.slot_groups().tolist() == [-1] * 4   # every stream has ended
    lat = s.latency_frames * HOP
    got = torch.cat(outs, 1)
    assert got.shape == (4, n * HOP + lat)
    for c in range(4):
        assert rms(got[c, lat:], ref[c]) <= 1e-6, c
    # the setting cannot change mid-stream; after a reset it can
    with pytest.raises(_lib.DfbError) as e:
        s.set_mask_reduce(2, None)
    assert e.value.code == _lib.DFB_ERR_INVALID
    s.reset()
    assert s.slot_states().tolist() == [SLOT_OPEN] * 4 and s.slot_groups().tolist() == [0, 0, 2, 2]   # the groups survive
    s.set_mask_reduce(1, None)
    assert s.slot_groups().tolist() == [0, 1, 2, 3]
    free = torch.cat([s.process(audio), s.flush()], 1)[:, lat:]
    assert rms(free, enhance(model, st, audio, pad=False)) <= 1e-6
    with pytest.raises(_lib.DfbError):
        DfStream(model, st, batch=3, channels=2, reduce_mask=reduce)


def test_streaming_gating_follows_the_first_channel(states):
    """LSNR stage gating with linked channels: one decision per recording and frame, from its first channel's LSNR.  With
    max_db_df_thresh between two LSNR values around channel 0's median, frames take both stage 2 (gains only) and stage 3
    (gains + deep filter), and channel 1 follows channel 0."""
    st = states
    cfg = cfg_of("dfn3")
    sd = random_state_dict(cfg, seed=67)
    model = DfNet(cfg, sd, st)
    n = 90
    audio = synth_audio(2, HOP * n, seed=360)
    _, aux = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean", return_all=True)
    l0 = np.sort(aux["lsnr"][0, :, 0].numpy())
    k = len(l0) // 2
    assert l0[k] - l0[k - 1] > 1e-3, "no safe threshold between the LSNR values around the median"
    th = dict(min_db_thresh=-1e9, max_db_erb_thresh=1e9, max_db_df_thresh=float(l0[k - 1] + l0[k]) / 2)
    want = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean", stages=th)
    s = DfStream(model, st, batch=2, channels=2, reduce_mask="mean")
    s.set_lsnr_thresholds(**th)
    got = torch.cat([s.process(audio[:, :HOP * 33]), s.process(audio[:, HOP * 33:]), s.flush()], 1)[:, s.latency_frames * HOP:]
    for c in range(2):
        assert rms(got[c], want[c]) <= 5e-6, (c, rms(got[c], want[c]))
    # both stages occur: the gated result differs from the ungated one, and from gains only everywhere
    ungated = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean")
    gains = LO.enhance(sd, cfg.as_dict(), audio, pad=False, reduce="mean", stages=dict(th, max_db_df_thresh=-1e9))
    assert rms(want, ungated) > 1e-5 and rms(want, gains) > 1e-5
    # channel 1 follows channel 0: gating on its own LSNR would give another result
    l1 = aux["lsnr"][1, :, 0].numpy()
    l0f = aux["lsnr"][0, :, 0].numpy()
    assert ((l1 > th["max_db_df_thresh"]) != (l0f > th["max_db_df_thresh"])).any()


def test_v1_linked_is_unsupported(states):
    st = states
    cfg = cfg_of("v1")
    model = DfNet(cfg, random_state_dict(cfg, seed=68), st)
    x = synth_audio(2, 9600, seed=370).cuda()
    with pytest.raises(_lib.DfbError) as e:
        enhance_device_ragged(model, st, x, [9600, 9600], group_sizes=[2], reduce_mask="mean")
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError) as e:
        enhance(model, st, x.cpu(), reduce_mask="max")
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED


def test_cli_reduce_mask(tmp_path, golden_dir, model_dir):
    from deepfilternet_b200 import io as dio
    from deepfilternet_b200.enhance import run
    a, _ = dio.load_audio(os.path.join(golden_dir, "assets", "noisy_snr0.wav"), 48000)
    b, _ = dio.load_audio(os.path.join(golden_dir, "assets", "clean_freesound_33711.wav"), 48000)
    t = min(a.shape[1], b.shape[1], 48000 * 3)
    src = str(tmp_path / "stereo.wav")
    dio.save_audio(src, torch.cat([a[:1, :t], 0.5 * b[:1, :t] + 0.5 * a[:1, :t]], 0), 48000, dtype=torch.float32)
    audio, _ = dio.load_audio(src, 48000)
    assert audio.shape == (2, t)
    m = os.path.join(model_dir, "DeepFilterNet3")
    model, st, _, _ = init_df(m, log_level="ERROR")
    for flag, reduce in ((None, None), ("2", "mean"), ("1", "max")):
        args = ["-m", m, "-o", str(tmp_path / f"o{flag}"), "--log-level", "ERROR", src] + (["--reduce-mask", flag] if flag else [])
        assert run(args) == 0
        written, _ = dio.load_audio(str(tmp_path / f"o{flag}" / "stereo_DeepFilterNet3.wav"))
        ref = (enhance(model, st, audio, reduce_mask=reduce) * (1 << 15)).to(torch.int16).to(torch.float32) / 32768.0
        assert written.shape == ref.shape and float((written - ref).abs().max()) <= 1.0 / 32768.0 + 1e-7, flag
    # --batch-size N links each file's channels too
    assert run(["-m", m, "-o", str(tmp_path / "b2"), "--log-level", "ERROR", "--batch-size", "2", "--reduce-mask", "2", src]) == 0
    one, _ = dio.load_audio(str(tmp_path / "o2" / "stereo_DeepFilterNet3.wav"))
    two, _ = dio.load_audio(str(tmp_path / "b2" / "stereo_DeepFilterNet3.wav"))
    assert float((one - two).abs().max()) <= 1.0 / 32768.0 + 1e-7
