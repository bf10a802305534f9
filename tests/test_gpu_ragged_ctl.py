"""GPU: per-entry settings and LSNR rows of ragged batches (dfb_enhance_ragged, enhance_batch / enhance_device_ragged
with per-entry atten_lim_db / post_filter_beta / lsnr_thresholds and return_lsnr) and per-slot LSNR thresholds
(DfStream.set_lsnr_thresholds(slots=...)).

* Entry i of a batch with mixed settings equals entry i of the same batch with entry i's settings given to every entry
  (bit for bit), and the entry enhanced alone by enhance() with those settings (RMS, as the other ragged tests).
* Gating: forced stages reproduce each stage's definition; mixed stages equal the float restatement of apply_stages on
  DfNet.forward's own outputs (linked_oracle) and a single-stream DfStream with the same thresholds.
* LSNR rows equal DfNet.forward's lsnr of the entry alone under the frame rule of include/dfb200.h."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import linked_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, enhance_batch, enhance_device_ragged, io, libdf, ragged
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

HOP = 480
TOL = 1e-6            # RMS against the entry alone, as tests/test_gpu_ragged.py
LSNR_TOL = 1e-4       # dB against DfNet.forward, as tests/test_gpu_stream_controls.py


def cfg_of(kind, **kw):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5, **kw)
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


def rms(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.sqrt(((a - b) ** 2).mean())) if a.size else 0.0


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_MODELS = {}


def model_of(st, kind, beta=0.0, mask_only=False):
    """Seeded weights (seed 23) with the post filter off (beta 0) or on with pf_beta = beta."""
    key = (kind, beta, mask_only)
    if key not in _MODELS:
        cfg = cfg_of(kind, mask_pf=beta > 0, pf_beta=beta if beta > 0 else 0.02)
        _MODELS[key] = DfNet(cfg, random_state_dict(cfg_of(kind), seed=23), st, run_df=not mask_only)
    return _MODELS[key]


def entries(seed):
    """Ragged entries of 1-20 s at 48 / 16 / 8 kHz, the last one a linked pair: (audios, rates)."""
    secs = [1.0, 20.0, 3.3, 7.7, 2.05]
    rates = [48000, 16000, 8000, 48000, 16000]
    chans = [1, 1, 1, 1, 2]
    out = []
    for i, (s, r, c) in enumerate(zip(secs, rates, chans)):
        out.append(synth_audio(c, int(s * r) + 7 * i, seed=seed + i, sr=r))
    return out, rates


# ------------------------------------------------------------------ per-entry limit and beta ----
@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2"])
def test_per_entry_settings_are_per_entry(st, kind):
    """Mixed limits (and betas, DeepFilterNet3 topologies) over ragged 1-20 s entries at 8 / 16 / 48 kHz with one linked
    pair: entry i equals entry i of the batch with entry i's settings everywhere (bit for bit) and enhance() of the entry
    alone with those settings, the beta as init_df(post_filter=True) with pf_beta = beta_i (RMS <= TOL)."""
    audios, rates = entries(300)
    n = len(audios)
    lims = [None, 6.0, 12.0, 20.0, 3.0]
    betas = [0.0, 0.02, 0.05, 0.1, 0.03] if kind != "dfn2" else None
    model = model_of(st, kind)
    mixed = enhance_batch(model, st, audios, True, lims, "mean", sr=rates, post_filter_beta=betas)
    for i in range(n):
        b_i = betas[i] if betas else None
        uni = enhance_batch(model, st, audios, True, [lims[i]] * n, "mean", sr=rates,
                            post_filter_beta=[b_i] * n if betas else None)
        assert torch.equal(mixed[i], uni[i]), (kind, i)
        alone_model = model_of(st, kind, beta=b_i or 0.0)
        ref = enhance(alone_model, st, audios[i], True, lims[i], reduce_mask="mean", sr=rates[i])
        assert mixed[i].shape == ref.shape
        assert rms(mixed[i], ref) <= TOL, (kind, i, rms(mixed[i], ref))
    # the device path takes the same table per row
    rows = [a[c] for a in audios for c in range(a.shape[0])]
    row_rates = [r for a, r in zip(audios, rates) for _ in range(a.shape[0])]
    row_lims = [l for a, l in zip(audios, lims) for _ in range(a.shape[0])]
    row_betas = [b for a, b in zip(audios, betas) for _ in range(a.shape[0])] if betas else None
    S = max(r.numel() for r in rows)
    x = torch.zeros(len(rows), S)
    for b, r in enumerate(rows):
        x[b, :r.numel()] = r
    y = enhance_device_ragged(model, st, x.cuda(), [r.numel() for r in rows], True, row_lims, group_sizes=[1, 1, 1, 1, 2],
                              reduce_mask="mean", sr=row_rates, post_filter_beta=row_betas).cpu()
    k = 0
    for i, a in enumerate(audios):
        for c in range(a.shape[0]):
            m = mixed[i].shape[1]
            assert rms(y[k, :m], mixed[i][c]) <= TOL, (kind, i, c)
            k += 1


# ------------------------------------------------------------------ gating ----
def test_gating_forced_stages(st):
    """Thresholds that force one stage for every frame of one entry reproduce the stage's definition, as
    tests/test_gpu_parity.py::test_streaming_lsnr_stage_gating does on the streaming path; the other entry does not gate."""
    model = model_of(st, "dfn3")
    audios = [synth_audio(1, 48000 * 2 + 111, seed=81), synth_audio(1, 48000 + 5, seed=82)]
    base = enhance_batch(model, st, audios)

    def run(th, atten=None):
        return enhance_batch(model, st, audios, True, [atten, None], lsnr_thresholds=[th, None])

    out = run((-1e9, 1e9, 1e9))                                      # always stage 3 (gains + DF)
    assert rms(out[0], base[0]) < 1e-7 and rms(out[1], base[1]) < 1e-7
    gains_only = run((-1e9, 1e9, -1e9))[0]                           # always stage 2
    assert rms(gains_only, enhance_batch(model_of(st, "dfn3", mask_only=True), st, audios)[0]) < 1e-7
    assert rms(gains_only, base[0]) > 1e-5
    a = audios[0]
    ident = torch.from_numpy(st.synthesis(st.analysis(F.pad(a, (0, 960)).numpy())))[:, 480:480 + a.shape[1]]
    assert rms(run((-1e9, -1e9, -1e9))[0], ident) < 1e-6             # always stage 1 (unprocessed)
    assert run((1e9, 2e9, 2e9))[0].abs().max() < 1e-7                # always stage 0
    lim = 10 ** (-12 / 20)
    assert rms(run((1e9, 2e9, 2e9), atten=12.0)[0], ident * lim) < 1e-6


def _median_threshold(l):
    s = np.sort(l)
    k = len(s) // 2
    assert s[k] - s[k - 1] > 1e-3, "no safe threshold between the LSNR values around the median"
    return float(s[k - 1] + s[k]) / 2


def test_gating_mixed_stages_per_entry(st):
    """Every entry gates with its own thresholds, set between LSNR values of its own so that two stages occur in it: each
    equals linked_oracle's restatement of apply_stages on DfNet.forward's lsnr / m / coefs for the entry alone, and a
    single-stream DfStream with the same thresholds aligned by its latency (pad=False)."""
    cfg = cfg_of("dfn3")
    sd = random_state_dict(cfg, seed=23)
    model = model_of(st, "dfn3")
    audios = [synth_audio(1, HOP * n, seed=400 + n) for n in (90, 151, 64)]
    ths = []
    for i, a in enumerate(audios):
        _, aux = LO.enhance(sd, cfg.as_dict(), a, pad=False, return_all=True)
        mid = _median_threshold(aux["lsnr"][0, :, 0].numpy())
        # entry 0: stages 2 / 3; entry 1: stages 0 / 3; entry 2: stages 1 / 3
        ths.append([(-1e9, 1e9, mid), (mid, 1e9, 1e9), (-1e9, mid, 1e9)][i])
    got = enhance_batch(model, st, audios, False, lsnr_thresholds=ths)
    for i, (a, th) in enumerate(zip(audios, ths)):
        stages = dict(min_db_thresh=th[0], max_db_erb_thresh=th[1], max_db_df_thresh=th[2])
        want = LO.enhance(sd, cfg.as_dict(), a, pad=False, stages=stages)
        ungated = LO.enhance(sd, cfg.as_dict(), a, pad=False)
        assert rms(got[i], want) <= 5e-6, (i, rms(got[i], want))
        assert rms(want, ungated) > 1e-5
        s = DfStream(model, st, batch=1)
        s.set_lsnr_thresholds(*th)
        y = torch.cat([s.process(a[:, :HOP * 33]), s.process(a[:, HOP * 33:]), s.flush()], 1)[:, s.latency_frames * HOP:]
        assert rms(got[i], y) <= 5e-6, (i, rms(got[i], y))


# ------------------------------------------------------------------ LSNR rows ----
def _forward_lsnr(model, st, a48, pad):
    """DfNet.forward's lsnr of one 48 kHz entry alone [C, T48]: the frames of the (padded) signal, and the frame of value 0."""
    x = F.pad(a48, (0, 960)) if pad else a48
    sp, fe, fs = df_features(x, st, model.nb_df)
    return model(sp, fe, fs)[2][..., 0].cpu(), (1 if pad else 0)


@pytest.mark.parametrize("kind", ["dfn3", "dfn2"])
def test_lsnr_rows(st, kind):
    """LSNR rows at 16, 44.1 and 48 kHz, pad on and off, default / 8 chunks (the 6 s entry has the 512 frames that takes)
    and one / two lanes: value j is
    DfNet.forward's lsnr of frame j + 1 (pad) or j (no pad) of the entry's 48 kHz signal alone; device and host rows are
    the same bits."""
    model = model_of(st, kind)
    rates = [16000, 44100, 48000, 16000]
    audios = [synth_audio(1, int(s * r) + 3, seed=500 + i, sr=r) for i, (s, r) in enumerate(zip((2.5, 1.3, 6.0, 0.7), rates))]
    try:
        for pad in (True, False):
            wants = []
            for a, r in zip(audios, rates):
                a48 = a if r == 48000 else io.resample(a, r, 48000)
                lsnr, f0 = _forward_lsnr(model, st, a48, pad)
                n = int(ragged.lsnr_lens(np.array([a.shape[1]]), r, HOP, pad)[0])
                wants.append(lsnr[0, f0:f0 + n])
                assert wants[-1].numel() == n
            for chunks, lanes in ((0, 2), (8, 1), (8, 2)):
                model.set_chunking(device_chunks=chunks, host_chunks=chunks or 4, lanes=lanes)
                outs, ls = enhance_batch(model, st, audios, pad, sr=rates, return_lsnr=True)
                plain = enhance_batch(model, st, audios, pad, sr=rates)
                for i, w in enumerate(wants):
                    assert torch.equal(outs[i], plain[i])                      # the LSNR output changes no audio bit
                    assert ls[i].shape == w.shape, (i, ls[i].shape, w.shape)
                    err = (ls[i] - w).abs().max().item()
                    assert err <= LSNR_TOL, (kind, pad, chunks, lanes, i, err)
            # device rows equal host rows bit for bit, with the same chunking on both paths (no tapered end chunks: one lane)
            model.set_chunking(device_chunks=4, host_chunks=4, lanes=1)
            _, lh = enhance_batch(model, st, audios, pad, sr=rates, return_lsnr=True)
            S = max(a.shape[1] for a in audios)
            x = torch.zeros(len(audios), S)
            for b, a in enumerate(audios):
                x[b, :a.shape[1]] = a[0]
            _, ld, lens = enhance_device_ragged(model, st, x.cuda(), [a.shape[1] for a in audios], pad, sr=rates, return_lsnr=True)
            ld = ld.cpu()
            for i in range(len(audios)):
                n = int(lens[i])
                assert torch.equal(ld[i, :n], lh[i]) and torch.isnan(ld[i, n:]).all(), i
    finally:
        model.set_chunking()


# ------------------------------------------------------------------ per-slot thresholds ----
def test_per_slot_thresholds(st):
    """Two slots with different thresholds each equal a one-slot handle with that slot's thresholds handle-wide; a slot
    re-opened returns to the handle's setting (no gating)."""
    cfg = cfg_of("dfn3")
    sd = random_state_dict(cfg, seed=23)
    model = model_of(st, "dfn3")
    x = synth_audio(2, HOP * 90, seed=610)
    ths = []
    for b in range(2):
        _, aux = LO.enhance(sd, cfg.as_dict(), x[b:b + 1], pad=False, return_all=True)
        mid = _median_threshold(aux["lsnr"][0, :, 0].numpy())
        ths.append([(-1e9, 1e9, mid), (mid, 1e9, 1e9)][b])

    def feed(s, a):
        return torch.cat([s.process(a[:, :HOP * 33]), s.process(a[:, HOP * 33:]), s.flush()], 1)

    s = DfStream(model, st, batch=2)
    for b in range(2):
        s.set_lsnr_thresholds(*ths[b], slots=[b])
    got = feed(s, x)
    for b in range(2):
        r = DfStream(model, st, batch=1)
        r.set_lsnr_thresholds(*ths[b])
        want = feed(r, x[b:b + 1])[0]
        plain = feed(DfStream(model, st, batch=1), x[b:b + 1])[0]
        assert rms(got[b], want) <= TOL and rms(want, plain) > 1e-5, b
    # reopened: the handle's setting again, which is no gating
    s.open([0, 1])
    got = feed(s, x)
    for b in range(2):
        assert rms(got[b], feed(DfStream(model, st, batch=1), x[b:b + 1])[0]) <= TOL


# ------------------------------------------------------------------ refusals ----
def _table_ptr(tab):
    return tab.ctypes.data if tab is not None else None


def test_refusals(st):
    """The combinations that are not built are refused with DFB_ERR_UNSUPPORTED, in Python and in the library, and a
    malformed table with DFB_ERR_INVALID; a refused call leaves the output untouched."""
    L = _lib.lib()
    a = [synth_audio(1, 9600, seed=700), synth_audio(1, 14400, seed=701)]
    dfn2, dfn3 = model_of(st, "dfn2"), model_of(st, "dfn3")
    for kw in (dict(post_filter_beta=0.02), dict(lsnr_thresholds=(-10, 30, 20))):
        with pytest.raises(_lib.DfbError) as e:
            enhance_batch(dfn2, st, a, **kw)
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    v1 = DfNet(cfg_of("v1"), random_state_dict(cfg_of("v1"), seed=23), st)
    for kw in (dict(atten_lim_db=[3, 6]), dict(return_lsnr=True)):
        with pytest.raises(_lib.DfbError) as e:
            enhance_batch(v1, st, a, **kw)
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError) as e:
        DfStream(dfn2, st, batch=2).set_lsnr_thresholds(slots=[0])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    with pytest.raises(_lib.DfbError) as e:
        DfStream(dfn3, st, batch=2, spectral=True).set_lsnr_thresholds(slots=[0])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED

    # the library itself, on a 2-stream host call
    lens = np.array([9600, 14400], dtype=np.int64)
    in_off = np.array([0, 9600], dtype=np.int64)
    x = torch.cat([t[0] for t in a]).contiguous()
    y = torch.full((24000,), 7.0)
    lz = torch.full((60,), 7.0)
    lo = np.array([0, 30], dtype=np.int64)

    def call(model, tab, n_tab=2, groups=None, red=0, lsnr=False, lsnr_numel=60):
        g = np.asarray(groups, dtype=np.int64) if groups is not None else None
        return L.dfb_enhance_ragged_host(model.handle, st.handle, x.data_ptr(), 24000, in_off.ctypes.data, lens.ctypes.data, 2, 1,
                                         0.0, y.data_ptr(), 24000, in_off.ctypes.data, g.ctypes.data if g is not None else None,
                                         g.size if g is not None else 0, red, None, _table_ptr(tab), n_tab,
                                         lz.data_ptr() if lsnr else None, lsnr_numel, lo.ctypes.data if lsnr else None)

    def tab_of(**kw):
        t = np.zeros(2, dtype=ragged.SETTINGS_DTYPE)
        for k, v in kw.items():
            t[k] = v
        return t

    cases = [(dfn2, tab_of(post_filter_beta=[0.0, 0.02]), {}, _lib.DFB_ERR_UNSUPPORTED),
             (dfn2, tab_of(lsnr_gating=[1, 0]), {}, _lib.DFB_ERR_UNSUPPORTED),
             (v1, tab_of(), {}, _lib.DFB_ERR_UNSUPPORTED),
             (v1, None, dict(lsnr=True), _lib.DFB_ERR_UNSUPPORTED),
             (dfn3, tab_of(), dict(n_tab=1), _lib.DFB_ERR_INVALID),
             (dfn3, tab_of(lsnr_gating=[1, 1], min_db_thresh=[np.nan, 0]), {}, _lib.DFB_ERR_INVALID),
             (dfn3, tab_of(atten_lim_db=[np.nan, 0]), {}, _lib.DFB_ERR_INVALID),
             (dfn3, tab_of(post_filter_beta=[-1.0, 0]), {}, _lib.DFB_ERR_INVALID),
             (dfn3, None, dict(lsnr=True, lsnr_numel=59), _lib.DFB_ERR_INVALID)]
    for i, (model, tab, kw, code) in enumerate(cases):
        assert call(model, tab, **kw) == code, i
        assert (y == 7.0).all() and (lz == 7.0).all(), i
    # a link group takes one setting
    lens[1] = 9600
    assert call(dfn3, tab_of(atten_lim_db=[3.0, 6.0]), groups=[2], red=2) == _lib.DFB_ERR_INVALID
    assert (y == 7.0).all()
    assert call(dfn3, tab_of(atten_lim_db=[3.0, 3.0]), groups=[2], red=2) == 0
