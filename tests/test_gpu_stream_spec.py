"""GPU: the spectral streaming handle (DfStream(spectral=True), dfb_stream_*_spec), the counterpart of the Rust runtime's
df_process_frame_raw: spectrum frames in, ERB gains / deep-filter coefficients / LSNR / stage out, with carried state.

* One-shot equivalence: DF.analysis frames fed in calls of 1, 2, 3, 7 and 40 frames, then flushed, equal DfNet.forward
  on the whole signal with the rows shifted by the latency (conv_lookahead); different call sizes agree.
* Round trip: the rows through dfb_apply and DF.synthesis equal enhance(pad=False).
* CPU oracle, slots and slot groups, stage gating, k_spec_ingest on its own, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dfnet_oracle as O
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance, libdf
from deepfilternet_b200._lib import check
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

HOP, F = 480, 481
SIZES = [1, 2, 3, 7, 40]
TOL = 1e-6               # max |err| of gains / coefs; RMS of sessions and of the round trip
LSNR_TOL = 1e-4          # dB, LSNR_TOL_FORWARD of test_gpu_stream_controls.py
ORACLE_TOL = 1e-4        # RMS against the CPU oracle, as the parity tests
KINDS = ["dfn3", "ll", "dfn2"]


def cfg_of(kind):
    base = dict(conv_ch=64, df_pathway_kernel_size_t=5)
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


def model_of(st, kind, mask_only=False):
    key = (kind, mask_only)
    if key not in _MODELS:
        _MODELS[key] = DfNet(cfg_of(kind), random_state_dict(cfg_of(kind), seed=101), st, run_df=not mask_only)
    return _MODELS[key]


def analysis(st, audio):
    return st.analysis(np.ascontiguousarray(audio.numpy()))   # complex64 [B, T, F]


def run_spec(s, spec, sizes, cuda_every=2):
    """Feed spec [B, T, F] in calls of `sizes` frames (alternately CPU and CUDA), then flush: rows [B, T + latency, ...]."""
    outs, pos = [], 0
    for i, n in enumerate(sizes):
        x = torch.from_numpy(np.ascontiguousarray(spec[:, pos:pos + n]))
        x = x.cuda() if i % cuda_every else x
        r = s.process_spec(x)
        assert all(t.device == x.device for t in r)   # CUDA in, CUDA out; CPU in, CPU out
        outs.append([t.cpu() for t in r])
        pos += n
    outs.append(list(s.flush_spec()))
    return [torch.cat([o[k] for o in outs], 1) for k in range(4)]


def forward_of(model, st, audio):
    """DfNet.forward's m, coefs and lsnr of the whole signal: [B,T,E], [B,T,Fd,O,2], [B,T].  DeepFilterNet2's forward
    returns df_alpha in place of the coefficients: its coefs come from dfb_model_forward on the same features."""
    sp, fe, fs = df_features(audio, st, model.nb_df)
    _, m, lsnr, last = model(sp, fe, fs)
    B, T = m.shape[0], m.shape[2]
    if model.cfg.model == "deepfilternet3":
        coefs = last.permute(0, 2, 3, 1, 4).cpu()
    else:
        d_fe, d_fs = fe[:, 0].contiguous().cuda(), fs[:, 0].contiguous().cuda()
        d_m, d_c = torch.empty((B, T, 32), device="cuda"), torch.empty((B, T, 96, 5, 2), device="cuda")
        check(_lib.lib().dfb_model_forward(model.handle, d_fe.data_ptr(), d_fs.data_ptr(), B, T, d_m.data_ptr(), d_c.data_ptr(),
                                           None, None, torch.cuda.current_stream().cuda_stream))
        coefs = d_c.cpu()
    return m[:, 0].cpu(), coefs, lsnr[..., 0].cpu()


def maxerr(a, b):
    return (a.double() - b.double()).abs().max().item()


# ------------------------------------------------------------------------------------------------ one-shot equivalence ----
@pytest.mark.parametrize("kind", KINDS)
def test_one_shot_equivalence(st, kind):
    """Rows j >= L equal DfNet.forward's frame j - L (gains, coefs max |err| <= 1e-6, LSNR <= 1e-4 dB), the first L rows are
    NaN / -1, for three call schedules that agree with each other to the same bounds; one frame off fails by orders of
    magnitude.  L = conv_lookahead, also for DeepFilterNet2."""
    model = model_of(st, kind)
    B = 2
    sched = [SIZES * 2, SIZES[::-1] * 2, [1] * (2 * sum(SIZES))]
    T = sum(sched[0])
    audio = synth_audio(B, T * HOP, seed=51)
    spec = analysis(st, audio)
    m, c, l = forward_of(model, st, audio)
    runs = []
    for sizes in sched:
        s = DfStream(model, st, batch=B, spectral=True)
        L = s.latency_frames
        assert L == model.cfg.conv_lookahead
        g, cf, ls, sg = run_spec(s, spec, sizes)
        assert g.shape == (B, T + L, 32) and cf.shape == (B, T + L, 96, 5, 2) and ls.shape == (B, T + L) and sg.dtype == torch.int8
        assert torch.isnan(g[:, :L]).all() and torch.isnan(cf[:, :L]).all() and torch.isnan(ls[:, :L]).all()
        assert (sg[:, :L] == -1).all() and (sg[:, L:] == 1).all()
        eg, ec, el = maxerr(g[:, L:], m), maxerr(cf[:, L:], c), maxerr(ls[:, L:], l)
        print(f"{kind} {sizes[:3]}: gains {eg:.3g} coefs {ec:.3g} lsnr {el:.3g} dB")
        assert eg <= TOL and ec <= TOL and el <= LSNR_TOL, (kind, eg, ec, el)
        off = maxerr(g[:, L + 1:], m[:, :-1])
        assert off > 1000 * TOL, (kind, off)   # the alignment is checked to the frame
        runs.append((g, cf, ls))
    for g, cf, ls in runs[1:]:
        assert maxerr(g[:, L:], runs[0][0][:, L:]) <= TOL and maxerr(cf[:, L:], runs[0][1][:, L:]) <= TOL
        assert maxerr(ls[:, L:], runs[0][2][:, L:]) <= LSNR_TOL


# ------------------------------------------------------------------------------------------------------- round trip ----
def apply_rows(model, st, spec, gains, coefs):
    B, T = gains.shape[:2]
    d_spec = torch.from_numpy(np.ascontiguousarray(spec)).cuda()
    d_m, d_c = gains.contiguous().cuda(), coefs.reshape(B, T, 96, 10).contiguous().cuda()
    out = torch.empty_like(d_spec)
    check(_lib.lib().dfb_apply(model.handle, st.handle, d_spec.data_ptr(), d_m.data_ptr(), d_c.data_ptr(), B, T, out.data_ptr(),
                               torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("kind", KINDS)
def test_round_trip(st, kind):
    """The emitted rows, assembled and run through dfb_apply with the same spectrum and DF.synthesis, equal
    enhance(pad=False) at RMS <= 1e-6.  DeepFilterNet3 / 3_ll: the audio handle's LSNR equals the spectral handle's hop
    for hop (both trail the input by conv_lookahead frames)."""
    model = model_of(st, kind)
    B = 3
    T = 2 * sum(SIZES)
    audio = synth_audio(B, T * HOP, seed=53)
    spec = analysis(st, audio)
    s = DfStream(model, st, batch=B, spectral=True)
    L = s.latency_frames
    g, cf, ls, _ = run_spec(s, spec, SIZES * 2)
    y = st.synthesis(apply_rows(model, st, spec, g[:, L:], cf[:, L:]))
    want = enhance(model, st, audio, pad=False)
    assert rms(y, want) < TOL, (kind, rms(y, want))
    if kind != "dfn2":
        a = DfStream(model, st, batch=B)
        assert a.latency_frames == L
        al, pos = [], 0
        for n in SIZES * 2:
            al.append(a.process(audio[:, pos * HOP:(pos + n) * HOP], return_lsnr=True)[1])
            pos += n
        al.append(a.flush(return_lsnr=True)[1])
        al = torch.cat(al, 1)
        assert torch.equal(torch.isnan(al), torch.isnan(ls))
        ok = ~torch.isnan(al)
        assert maxerr(al[ok], ls[ok]) <= LSNR_TOL


# -------------------------------------------------------------------------------------------------------- CPU oracle ----
@pytest.mark.parametrize("kind", KINDS)
def test_cpu_oracle(st, kind):
    """The concatenated gains and coefs equal oracle/dfnet_oracle.dfnet_forward on the oracle's own features (RMS <= 1e-4)."""
    model = model_of(st, kind)
    cfg = cfg_of(kind)
    B, T = 2, 60
    audio = synth_audio(B, T * HOP, seed=55)
    _, aux = O.enhance(random_state_dict(cfg, seed=101), cfg.as_dict(), audio, pad=False, return_all=True)
    spec = torch.view_as_complex(aux["spec"][:, 0].contiguous()).numpy()
    s = DfStream(model, st, batch=B, spectral=True)
    L = s.latency_frames
    g, cf, _, _ = run_spec(s, spec, [7, 40, 13])
    assert rms(g[:, L:], aux["m"][:, 0]) < ORACLE_TOL
    assert rms(cf[:, L:].reshape(B, T, 96, 10), aux["coefs"]) < ORACLE_TOL


# --------------------------------------------------------------------------------------------------- slots and groups ----
def fresh_rows(model, st, spec, sizes, channels=1, reduce=None):
    s = DfStream(model, st, batch=channels, spectral=True, channels=channels, reduce_mask=reduce)
    return run_spec(s, spec, sizes)


@pytest.mark.parametrize("kind", KINDS)
def test_slots_equal_fresh_handles(st, kind):
    """Sessions open and close at staggered calls of an 8-slot spectral handle, including re-opening a live slot and
    closing during the tail: each session equals a fresh one-stream handle fed the same frames (RMS <= 1e-6 and the same
    NaN / -1 pattern), and free rows are NaN / -1."""
    model = model_of(st, kind)
    B = 8
    calls = [([], [7], 1), ([7], [], 1), ([], [3, 7], 2), ([6], [], 3), ([3], [2], 1), ([2], [], 7), ([5], [0], 40),
             ([], [1], 1), ([1], [], 2), ([4], [4], 3), ([0, 6], [], 7), ([], [3], 1), ([3], [], 1)]
    total = sum(n for *_, n in calls) + 1
    s = DfStream(model, st, batch=B, spectral=True)
    L = s.latency_frames
    src = {}
    live, sessions, count = {}, [], [0]

    def new(b):
        ses = dict(slot=b, spec=analysis(st, synth_audio(1, total * HOP, seed=600 + count[0]))[0], sizes=[], rows=[],
                   closing=False, tail=0, dropped=False)
        count[0] += 1
        live[b] = ses
        sessions.append(ses)

    for b in range(B):
        new(b)
    for i in range(len(calls) + 1):
        flush = i == len(calls)
        if not flush:
            closes, opens, n = calls[i]
            if closes:
                s.close(closes)
                for b in closes:
                    ses = live.get(b)
                    if ses and not ses["closing"]:
                        ses["closing"], ses["tail"] = True, L
                        if L == 0:
                            del live[b]
            if opens:
                s.open(opens)
                for b in opens:
                    if b in live:
                        live[b]["dropped"] = True
                    new(b)
            x = np.zeros((B, n, F), np.complex64)
            x[:] = 1e3   # ignored rows: free or closing slots
            for b, ses in live.items():
                if not ses["closing"]:
                    pos = sum(ses["sizes"])
                    x[b] = ses["spec"][pos:pos + n]
                    ses["sizes"].append(n)
            r = s.process_spec(torch.from_numpy(x).cuda() if i % 2 else torch.from_numpy(x))
        else:
            for b, ses in list(live.items()):
                if not ses["closing"]:
                    ses["closing"], ses["tail"] = True, L
                if L == 0:
                    del live[b]
            r = s.flush_spec()
            n = L
        r = [t.cpu() for t in r]
        used = set()
        for b, ses in list(live.items()):
            k = n if not ses["closing"] else min(n, ses["tail"])
            ses["rows"].append([t[b, :k] for t in r])
            if ses["closing"]:
                assert torch.isnan(r[2][b, k:]).all() and (r[3][b, k:] == -1).all(), ("past the tail", i, b)
                ses["tail"] -= k
                if ses["tail"] == 0:
                    del live[b]
            used.add(b)
        for b in range(B):
            if b not in used and n:
                assert torch.isnan(r[0][b]).all() and torch.isnan(r[1][b]).all() and torch.isnan(r[2][b]).all()
                assert (r[3][b] == -1).all(), ("free slot", i, b)
    assert not live
    checked = 0
    for ses in sessions:
        if not ses["sizes"]:
            continue
        got = [torch.cat([row[k] for row in ses["rows"]], 0) for k in range(4)]
        T = sum(ses["sizes"])
        ref = [t[0] for t in fresh_rows(model, st, ses["spec"][None, :T], ses["sizes"])]
        if ses["dropped"]:
            ref = [t[:got[0].shape[0]] for t in ref]
        for a, b_ in zip(got, ref):
            assert a.shape == b_.shape
        assert torch.equal(torch.isnan(got[0]), torch.isnan(ref[0])) and torch.equal(got[3], ref[3])
        ok = ~torch.isnan(ref[2])
        assert rms(got[0][ok], ref[0][ok]) < TOL and rms(got[1][ok], ref[1][ok]) < TOL
        assert maxerr(got[2][ok], ref[2][ok]) <= LSNR_TOL if ok.any() else True
        checked += 1
    assert checked >= 10


@pytest.mark.parametrize("reduce", ["max", "mean"])
def test_slot_groups_reduce_the_gains(st, reduce):
    """A linked slot group (open_linked) next to a one-channel session: the group's gains are the max / mean of its
    members' unlinked gains, bit for bit (mean: fp32 sum in channel order times fl32(1 / C)); coefs and LSNR equal the
    unlinked ones; a linked channels handle (channels=3) gives the same rows."""
    model = model_of(st, "dfn3")
    C3 = 3
    spec = analysis(st, synth_audio(C3 + 1, 60 * HOP, seed=57))
    sizes = [1, 7, 40, 2, 3, 7]
    unl = fresh_rows(model, st, spec[:C3], sizes, channels=C3)
    s = DfStream(model, st, batch=6, spectral=True, reduce_mask=reduce)
    s.open_linked([4, 1, 5])
    s.open([2])
    s.close([0, 3])
    x = np.zeros((6, 60, F), np.complex64)
    x[[4, 1, 5]] = spec[:C3]
    x[2] = spec[C3]
    got = [t for t in run_spec(s, x, sizes)]
    got = [t[[4, 1, 5]] for t in got]
    L = s.latency_frames
    ug = unl[0][:, L:]
    if reduce == "max":
        want = ug.max(0).values
    else:
        want = ug[0].clone()
        for k in range(1, C3):
            want = want + ug[k]
        want = want * torch.tensor(1.0 / C3, dtype=torch.float32)
    for k in range(C3):
        assert torch.equal(got[0][k, L:], want), (reduce, k)
        assert torch.equal(got[1][k, L:], unl[1][k, L:]) and torch.equal(torch.isnan(got[2][k]), torch.isnan(unl[2][k]))
        assert maxerr(got[2][k, L:], unl[2][k, L:]) <= LSNR_TOL
    fixed = fresh_rows(model, st, spec[:C3], sizes, channels=C3, reduce=reduce)
    assert torch.equal(fixed[0][:, L:], got[0][:, L:])


# ---------------------------------------------------------------------------------------------------------- stages ----
def stage_rule(l, th_min, th_erb, th_df):
    return np.where(l < th_min, 0, np.where(l > th_erb, 3, np.where(l > th_df, 2, 1)))


@pytest.mark.parametrize("kind", KINDS)
def test_stages(st, kind):
    """Thresholds at the LSNR's quantiles make all four stages occur: each stage is the rule on the returned LSNR, stages
    0, 2 and 3 carry exactly the table's gains / coefs, stage-1 rows equal the ungated handle's.  On a mask_only model
    stage 1 becomes 2 (zero coefs)."""
    B, T = 2, 2 * sum(SIZES)
    spec = analysis(st, synth_audio(B, T * HOP, seed=59))
    for mask_only in (False, True):
        model = model_of(st, kind, mask_only)
        plain = run_spec(DfStream(model, st, batch=B, spectral=True), spec, SIZES * 2)
        L = model.cfg.conv_lookahead
        lv = plain[2][:, L:].numpy()
        q = np.quantile(lv, [0.2, 0.5, 0.8])
        th = (float(q[0]), float(q[2]), float(q[1]))   # min, max_erb, max_df
        s = DfStream(model, st, batch=B, spectral=True)
        s.set_lsnr_thresholds(*th)
        g, cf, ls, sg = run_spec(s, spec, SIZES * 2)
        assert torch.equal(torch.isnan(ls), torch.isnan(plain[2])) and maxerr(ls[:, L:], plain[2][:, L:]) <= LSNR_TOL
        want = stage_rule(ls[:, L:].numpy(), *th)
        if mask_only:
            want = np.where(want == 1, 2, want)
        got = sg[:, L:].numpy()
        assert (got == want).all() and set(np.unique(got)) == ({0, 2, 3} if mask_only else {0, 1, 2, 3})
        g, cf, sgl = g[:, L:], cf[:, L:], sg[:, L:]
        assert (g[sgl == 0] == 0).all() and (g[sgl == 3] == 1).all() and (cf[sgl != 1] == 0).all()
        for k in (1, 2):
            assert torch.equal(g[sgl == k], plain[0][:, L:][sgl == k])
        assert torch.equal(cf[sgl == 1], plain[1][:, L:][sgl == 1])


# ------------------------------------------------------------------------------------------------ k_spec_ingest alone ----
def db64(spec, widths):
    p = np.abs(spec.astype(np.complex128)) ** 2
    out, o = [], 0
    for w in widths:
        out.append(10 * np.log10(p[..., o:o + w].sum(-1) / w + 1e-10))
        o += w
    return np.stack(out, -1)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 8, 9, 127, 128, 129])
def test_spec_ingest_kernel(st, n):
    """k_spec_ingest (dfb_debug_spec_ingest) on spectra with zero frames and large-magnitude frames: its ERB dB are bit-exact
    against k_analysis's epilogue on the same spectrum and within an explicit bound of float64; its bins are the input's.
    Ragged live rows read their own caller row and zeros from their length on.  Frame counts around the 4-frame tile."""
    L = _lib.lib()
    B = 3
    a = synth_audio(B, n * HOP, seed=61 + n)
    a[0, : (n // 2) * HOP] = 0                # zero frames
    a[1] *= 500.0                             # large-magnitude frames (up to ~|1e5| bins)
    d_a = a.cuda()
    spec = torch.empty((B, n, F, 2), device="cuda")
    erb = torch.empty((B, n, 32), device="cuda")
    check(L.dfb_debug_analysis_erb(st.handle, d_a.data_ptr(), B, n * HOP, spec.data_ptr(), erb.data_ptr(), None))
    widths = st.erb_widths().astype(np.int64)
    rows_src, rows_len = np.array([2, 0, 1, 2], np.int64), np.array([n, n, max(n - 2, 0), 0], np.int64)
    for src, ln in ((None, None), (rows_src, rows_len)):
        nb = B if src is None else len(src)
        e2 = torch.full((nb, n, 32), float("nan"), device="cuda")
        bins = torch.full((nb, n, 96, 2), float("nan"), device="cuda")
        ps = None if src is None else src.ctypes.data_as(C.POINTER(C.c_int64))
        pl = None if src is None else ln.ctypes.data_as(C.POINTER(C.c_int64))
        check(L.dfb_debug_spec_ingest(st.handle, spec.data_ptr(), n, ps, pl, nb, 96, e2.data_ptr(), bins.data_ptr(), None))
        torch.cuda.synchronize()
        sp, e1, e2, bins = spec.cpu(), erb.cpu(), e2.cpu(), bins.cpu()
        for b in range(nb):
            r = b if src is None else int(src[b])
            k = n if src is None else int(ln[b])
            assert torch.equal(e2[b, :k], e1[r, :k]), (n, b)
            assert torch.equal(bins[b, :k], sp[r, :k, :96]), (n, b)
            z = sp[r].numpy().copy()
            z[k:] = 0
            ref = db64(z[..., 0] + 1j * z[..., 1], widths)
            # in-band fp32 sum of w terms: relative error <= (w + 4) 2^-24, i.e. 4.35 (w + 4) 2^-24 dB; log10f and the
            # final product add a few ulps of a result below 128 dB
            bound = 4.35 * (widths + 4) * 2.0 ** -24 + 6e-5
            err = np.abs(e2[b].numpy() - ref)
            assert (err <= bound).all(), (n, b, err.max())
            assert torch.equal(bins[b, k:], torch.zeros_like(bins[b, k:]))
        spec_nan = torch.isnan(e2).any().item()
        assert not spec_nan
    z = e1[0, :n // 2]                       # zero frames: 10 log10(1e-10) = -100 dB in every band
    assert torch.equal(z, torch.full_like(z, e1[0, 0, 0].item())) and ((z + 100).abs() < 1e-4).all() if n // 2 else True


# -------------------------------------------------------------------------------------------------------- refusals ----
def test_refusals(st):
    """create_spec on DeepFilterNet v1 is DFB_ERR_UNSUPPORTED; the audio calls on a spectral handle and the spectral calls
    on an audio handle are DFB_ERR_INVALID; set_atten_lim / set_post_filter_beta on a spectral handle are
    DFB_ERR_UNSUPPORTED.  Each refusal changes nothing: the next call's output is the unrefused handle's."""
    L = _lib.lib()
    v1 = ModelConfig(model="deepfilternet", conv_lookahead=2, df_lookahead=1, conv_ch=64, conv_kernel=(2, 3), convt_kernel=(2, 3),
                     conv_kernel_inp=(2, 3), conv_k_enc=2, conv_k_dec=2, emb_hidden_dim=512, df_hidden_dim=512, emb_num_layers=3,
                     df_num_layers=2, gru_groups=8, lin_groups=8, enc_lin_groups=8, group_shuffle=True, dfop_method="real_unfold")
    m1 = DfNet(v1, random_state_dict(v1, seed=3), st)
    h = C.c_void_p()
    assert L.dfb_stream_create_spec(C.byref(h), m1.handle, st.handle, 1) == _lib.DFB_ERR_UNSUPPORTED and not h.value
    with pytest.raises(_lib.DfbError):
        DfStream(m1, st, spectral=True)

    model = model_of(st, "dfn3")
    B = 2
    audio = synth_audio(B, 20 * HOP, seed=63)
    spec = analysis(st, audio)
    ref = run_spec(DfStream(model, st, batch=B, spectral=True), spec, [3, 17])
    s = DfStream(model, st, batch=B, spectral=True)
    a = DfStream(model, st, batch=B)
    ref_a = torch.cat([a.process(audio[:, :3 * HOP]), a.process(audio[:, 3 * HOP:]), a.flush()], 1)
    a.reset()
    one = (C.c_int64 * 1)(0)
    d_in = torch.zeros((B, 3 * HOP), device="cuda")
    d_out = torch.zeros((B, 3 * HOP), device="cuda")
    d_spec = torch.zeros((B, 3, F, 2), device="cuda")
    d_g = torch.zeros((B, 3, 32), device="cuda")
    cs = torch.cuda.current_stream().cuda_stream
    x = np.zeros((B, 3 * HOP), np.float32)
    xs = np.zeros((B, 3, F, 2), np.float32)
    hg = np.zeros((B, 3, 32), np.float32)
    refusals = [
        (s, lambda: L.dfb_stream_process(s._h, d_in.data_ptr(), 3, d_out.data_ptr(), cs), _lib.DFB_ERR_INVALID),
        (s, lambda: L.dfb_stream_process_lsnr(s._h, d_in.data_ptr(), 3, d_out.data_ptr(), None, cs), _lib.DFB_ERR_INVALID),
        (s, lambda: L.dfb_stream_process_host(s._h, x.ctypes.data, 3, x.ctypes.data), _lib.DFB_ERR_INVALID),
        (s, lambda: L.dfb_stream_flush(s._h, d_out.data_ptr(), cs), _lib.DFB_ERR_INVALID),
        (s, lambda: L.dfb_stream_set_atten_lim(s._h, one, 1, C.c_float(6.0)), _lib.DFB_ERR_UNSUPPORTED),
        (s, lambda: L.dfb_stream_set_post_filter_beta(s._h, one, 1, C.c_float(0.02)), _lib.DFB_ERR_UNSUPPORTED),
        (a, lambda: L.dfb_stream_process_spec(a._h, d_spec.data_ptr(), 3, d_g.data_ptr(), None, None, None, cs), _lib.DFB_ERR_INVALID),
        (a, lambda: L.dfb_stream_process_spec_host(a._h, xs.ctypes.data, 3, hg.ctypes.data, None, None, None), _lib.DFB_ERR_INVALID),
        (a, lambda: L.dfb_stream_flush_spec(a._h, d_g.data_ptr(), None, None, None, cs), _lib.DFB_ERR_INVALID),
    ]
    for h_, call, code in refusals:
        assert call() == code
    with pytest.raises(_lib.DfbError):
        s.process(audio[:, :3 * HOP])
    with pytest.raises(_lib.DfbError):
        a.process_spec(torch.from_numpy(np.ascontiguousarray(spec[:, :3])))
    with pytest.raises(_lib.DfbError) as e:
        s.set_atten_lim(6.0, [0])
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED
    got = run_spec(s, spec, [3, 17])
    for u, v in zip(got, ref):
        assert torch.equal(torch.isnan(u.float()), torch.isnan(v.float()))
        ok = ~torch.isnan(v.float())
        assert torch.equal(u[ok], v[ok])
    got_a = torch.cat([a.process(audio[:, :3 * HOP]), a.process(audio[:, 3 * HOP:]), a.flush()], 1)
    assert torch.equal(got_a, ref_a)
    # DeepFilterNet2 takes LSNR thresholds on a spectral handle, not on an audio one
    m2 = model_of(st, "dfn2")
    DfStream(m2, st, spectral=True).set_lsnr_thresholds()
    with pytest.raises(_lib.DfbError):
        DfStream(m2, st).set_lsnr_thresholds()
