"""GPU: DeepFilterNet2_ll, DeepFilterNet2 at zero look-ahead with a DF pathway conv of 3 time taps, on every enhancement
path: init_df on the seeded model directory against the reference module's outputs and the CPU oracle, the pathway conv
kernel alone for every built time size against float64, chunked and streaming runs at latency 0, streaming slots, ragged
and rated batches, linked channels and the spectral handle; per-slot post-filter beta and LSNR stage gating stay refused,
as for DeepFilterNet2."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import dfn2_ll_model
import dfnet_oracle as O
import golden_io
import linked_oracle as LO
import model_ref64
import ref_harness as rh
from tests_common import synth_audio
from test_gpu_linked import GROUPS, assert_close, pack, recordings, split
from test_gpu_ragged_rates import MIX, assert_composition, entries
from test_gpu_slots import check_sessions, run_server, schedule
from test_gpu_stream_spec import forward_of, maxerr, run_spec

from deepfilternet_b200 import DfStream, _lib, enhance, enhance_device, enhance_device_ragged, init_df
from deepfilternet_b200.model import find_checkpoint, load_state_dict_file
from deepfilternet_b200.weights import umma_sw128_image

HOP = 480
RMS_TOL = 5e-6          # enhance() against the reference module / oracle, as test_gpu_parity.py
TOL = 1e-6              # one code path against another (chunking, streaming, slots), as the streaming tests
LSNR_TOL = 1e-4         # dB


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean())) if a.size else 0.0


@pytest.fixture(scope="module")
def ll(tmp_path_factory):
    d = dfn2_ll_model.make_model_dir(str(tmp_path_factory.mktemp("models")))
    model, st, _, epoch = init_df(d, log_level="ERROR")
    sd = load_state_dict_file(find_checkpoint(os.path.join(d, "checkpoints"))[0])
    return model, st, sd, epoch


def test_end_to_end(ll, golden_dir):
    model, st, sd, epoch = ll
    cfg = model.cfg
    assert epoch == 1 and cfg.model == "deepfilternet2"
    assert (cfg.conv_lookahead, cfg.df_lookahead, cfg.df_pathway_kernel_size_t) == (0, 0, 3)
    g = golden_io.load(os.path.join(golden_dir, "dfnet_DeepFilterNet2_ll.npz"))
    audio = torch.from_numpy(g["audio"])
    out = enhance(model, st, audio)
    assert rms(out, g["enhanced"]) < RMS_TOL
    assert rms(out, O.enhance(sd, cfg.as_dict(), audio, pad=True)) < RMS_TOL
    spec_e, m, lsnr, alpha = model(torch.from_numpy(g["spec"]), torch.from_numpy(g["feat_erb"]), torch.from_numpy(g["feat_spec"]))
    assert rms(spec_e, g["spec_e"]) < 1e-4 and rms(m, g["m"]) < 1e-5 and np.abs(lsnr.numpy() - g["lsnr"]).max() < 1e-3
    assert rms(alpha, g["df_alpha"]) < 1e-5
    # the known answer on the whole 10 s recording: SI-SDR against the clean signal, as the reference module gives it
    noisy = torch.from_numpy(rh.read_wav(os.path.join(golden_dir, "assets", "noisy_snr0.wav")))
    clean = rh.read_wav(os.path.join(golden_dir, "assets", "clean_freesound_33711.wav"))
    s, t = rh.si_sdr(clean, enhance(model, st, noisy, pad=True).numpy()), float(g["si_sdr_target"])
    assert abs(s - t) <= 1e-4 + 1e-4 * abs(t), (s, t)


# ------------------------------------------------------------------------------------------- the pathway conv alone ----
def convp_ref(c0, w1, w2, bn, first):
    """float64 grouped (2) causal temporal conv + 1x1 conv + BN (eval) + ReLU of c0 [B,T,Fd,64]; frames of stream b
    before first[b] read as zeros.  Returns coefs [B,T,Fd,10] and the same chain on absolute values (the error scale)."""
    g, b, mu, var = bn
    kt = w1.shape[2]
    x = c0.double().clone()
    for s, f in enumerate(first):
        x[s, :f] = 0
    x = x.permute(0, 3, 1, 2)                                  # [B,64,T,Fd]
    s = g / torch.sqrt(var + 1e-5)

    def chain(x, w1, w2, bias):   # w2 [out][in]
        y = F.conv2d(F.pad(x, (0, 0, kt - 1, 0)), w1, groups=2)
        return torch.einsum("bitf,oi->botf", y, w2) + bias[None, :, None, None]

    z = chain(x, w1, w2[:, :, 0, 0] * s[:, None], b - mu * s)
    za = chain(x.abs(), w1.abs(), (w2[:, :, 0, 0] * s[:, None]).abs(), (b - mu * s).abs())
    return torch.relu(z).permute(0, 2, 3, 1), za.permute(0, 2, 3, 1)


@pytest.mark.parametrize("kt", [1, 2, 3, 4, 5])
def test_df_convp_kernel(kt):
    """k_df_convp_tc<5, kt> through dfb_debug_df_convp_tc, element by element against float64 (BF16x3 operands: relative
    error ~2^-16 of the absolute-value chain): T at and around the 124-frame output tile and the 128-row box, Fd not a
    multiple of the 8-bin CTA, without and with a slot-start table (one start inside the second tile)."""
    gen = torch.Generator().manual_seed(100 + kt)
    w1 = torch.randn(10, 32, kt, 1, generator=gen, dtype=torch.float64) * 0.2
    w2 = torch.randn(10, 10, 1, 1, generator=gen, dtype=torch.float64) * 0.3
    bn = (1 + 0.1 * torch.randn(10, generator=gen, dtype=torch.float64), 0.1 * torch.randn(10, generator=gen, dtype=torch.float64),
          0.1 * torch.randn(10, generator=gen, dtype=torch.float64), 0.5 + torch.rand(10, generator=gen, dtype=torch.float64))
    s = bn[0] / torch.sqrt(bn[3] + 1e-5)
    img = np.zeros((64, 64), np.float32)
    for g in range(2):
        for dt in range(kt):
            for o in range(5):
                img[g * 32 + dt * 5 + o, g * 32:(g + 1) * 32] = w1[g * 5 + o, :, dt, 0].numpy()
    d_img = torch.from_numpy(umma_sw128_image(img)).cuda()
    d_w2 = torch.from_numpy((w2[:, :, 0, 0] * s[:, None]).T.contiguous().float().numpy()).cuda()
    d_b = (bn[1] - bn[2] * s).float().cuda()
    L = _lib.lib()
    for T in (1, 123, 124, 125, 128, 129, 250):
        for Fd in (13, 96):
            B = 3
            c0 = torch.randn(B, T, Fd, 64, generator=gen)
            for first in (None, [3, 15, 140]):
                w0 = 10
                starts = [0] * B if first is None else [max(f - w0, 0) for f in first]
                ref, absref = convp_ref(c0, w1, w2, bn, starts)
                d_c0 = c0.cuda()
                out = torch.full((B, T, Fd, 10), float("nan"), device="cuda")
                d_first = None if first is None else torch.tensor(first, dtype=torch.int64).cuda()
                _lib.check(L.dfb_debug_df_convp_tc(d_c0.data_ptr(), d_img.data_ptr(), d_w2.data_ptr(), d_b.data_ptr(), out.data_ptr(),
                                                   B, T, Fd, 5, kt, None if d_first is None else d_first.data_ptr(), w0,
                                                   torch.cuda.current_stream().cuda_stream))
                got = out.cpu().double()
                err = (got - ref).abs()
                assert torch.isfinite(got).all(), (kt, T, Fd, first)
                assert (err <= model_ref64.bf16x3_bound(absref)).all(), (kt, T, Fd, first, err.max().item())
    for bad in ((5, 0), (5, 6), (4, 3)):
        rc = L.dfb_debug_df_convp_tc(d_c0.data_ptr(), d_img.data_ptr(), d_w2.data_ptr(), d_b.data_ptr(), out.data_ptr(), 1, 8, 13,
                                     bad[0], bad[1], None, 0, None)
        assert rc == _lib.DFB_ERR_UNSUPPORTED and b"built kernels" in L.dfb_last_error()


# --------------------------------------------------------------------------------------- chunks, streams, slots ----
def test_chunked_equals_one_shot(ll):
    model, st, _, _ = ll
    x = synth_audio(3, 3 * 48000 + 123, seed=71).cuda()
    runs = {}
    for chunks in (1, 6, 40):
        model.set_chunking(chunks, 4, 2)
        runs[chunks] = enhance_device(model, st, x).cpu()
    model.set_chunking(0, 4, 2)
    for chunks in (6, 40):
        assert rms(runs[chunks], runs[1]) < TOL, chunks


def test_streaming_at_latency_zero(ll):
    model, st, _, _ = ll
    n = 157
    x = synth_audio(2, n * HOP, seed=72)
    s = DfStream(model, st, batch=2)
    assert s.latency_frames == 0
    outs, pos = [], 0
    for i, k in enumerate([1, 1, 2, 3, 7, 40, 1, 3, 64, 35]):
        xk = x[:, pos * HOP:(pos + k) * HOP]
        outs.append(s.process(xk.cuda() if i % 2 else xk).cpu())
        pos += k
    assert pos == n
    tail = s.flush()
    assert tail.shape[1] == 0
    got = torch.cat(outs, 1)
    assert got.shape == (2, n * HOP)
    assert rms(got, enhance(model, st, x, pad=False)) < TOL


def test_slots_equal_fresh_streams(ll):
    model, st, _, _ = ll
    sessions, lat = run_server(model, st, schedule(seed=9, n_random=24), seed=3)
    assert lat == 0
    assert any(s.dropped for s in sessions)
    assert check_sessions(model, st, sessions, lat) >= 12


# -------------------------------------------------------------------------------------------------------- batches ----
def test_ragged_and_rated_batches(ll):
    """A ragged batch at 48 kHz and a rated batch of 8 / 16 / 48 kHz entries equal each entry enhanced alone (through
    io.resample to and from 48 kHz for the other rates)."""
    model, st, _, _ = ll
    assert_composition(model, st, entries([(48000, 48000 + 240), (48000, 9600 + 7), (48000, 96000 + 3)], seed=600))
    assert_composition(model, st, entries([(r, n) for r, n in MIX if r in (8000, 16000, 48000)], seed=610))


@pytest.mark.parametrize("reduce", ["max", "mean"])
def test_linked_channels(ll, reduce):
    model, st, sd, _ = ll
    recs = recordings(GROUPS, seed=310)
    x, lengths, groups = pack(recs)
    for pad in (True, False):
        got = split(enhance_device_ragged(model, st, x, lengths, pad=pad, group_sizes=groups, reduce_mask=reduce), recs, pad)
        want = [LO.enhance(sd, model.cfg.as_dict(), r, pad=pad, reduce=reduce) for r in recs]
        assert_close(got, want, 5e-6, (reduce, pad))
    n = 101
    audio = torch.cat(recordings([(2, HOP * n), (2, HOP * n)], seed=360), 0)
    s = DfStream(model, st, batch=4, channels=2, reduce_mask=reduce)
    assert s.latency_frames == 0
    got = torch.cat([s.process(audio[:, :37 * HOP]), s.process(audio[:, 37 * HOP:].cuda()).cpu()], 1)
    ref = torch.cat([enhance(model, st, audio[2 * i:2 * i + 2], pad=False, reduce_mask=reduce) for i in range(2)], 0)
    assert rms(got, ref) < TOL


# ------------------------------------------------------------------------------------------------ spectral handle ----
def test_spectral_handle_at_latency_zero(ll):
    """Rows are DfNet.forward's frames with no shift: gains and coefs to 1e-6, LSNR to 1e-4 dB, for two call schedules."""
    model, st, _, _ = ll
    B = 2
    audio = synth_audio(B, 53 * HOP, seed=73)
    spec = st.analysis(np.ascontiguousarray(audio.numpy()))
    m, c, l = forward_of(model, st, audio)
    for sizes in ([1, 2, 3, 7, 40], [40, 7, 3, 2, 1]):
        s = DfStream(model, st, batch=B, spectral=True)
        assert s.latency_frames == 0 == model.cfg.conv_lookahead
        g, cf, ls, sg = run_spec(s, spec, sizes)
        assert g.shape == (B, 53, 32) and (sg == 1).all()
        assert maxerr(g, m) <= TOL and maxerr(cf, c) <= TOL and maxerr(ls, l) <= LSNR_TOL, (maxerr(g, m), maxerr(cf, c))


def test_refused_settings(ll):
    """As for DeepFilterNet2: per-slot post-filter beta and LSNR stage gating on an audio handle are DFB_ERR_UNSUPPORTED."""
    model, st, _, _ = ll
    s = DfStream(model, st, batch=2)
    with pytest.raises(_lib.DfbError) as e:
        s.set_post_filter_beta(0.02, [0])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError) as e:
        s.set_lsnr_thresholds()
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    s.set_atten_lim(6.0, [0])
