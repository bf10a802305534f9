"""GPU: the apply + synthesis kernel's row-table instances element by element against the float64 row-level reference.

dfb_debug_apply_rows launches what the batch and slot executors launch -- the row-table instance (RG), with link groups
(LINK), with per-row settings (CTL), both, and the generic kernel with rows -- on given spectra and model outputs.  Every
case compares the audio and the enhanced spectrum (spec_out) with tests/dsp_ref64.py's apply_rows at K = 1, and checks that
every element outside the written set keeps its NaN sentinel.  The row geometry puts each edge just before, on and just
after a warp start and a CTA start: a row's end, its first frame (streaming slots), its settings switch (the re-synthesised
frame t0 - 1 of a warp starting on the switch takes the old setting), t_first, Tv < spec_T, a negative and a positive
out_offset, an out_len that cuts a hop and gaps between the output rows.  LSNR inputs sit exactly on each threshold and one
fp32 ulp either side, and the channels of a link group carry different LSNR.  Inputs come from seeds only.

Worst err / bound on an H100 80GB HBM3 at a 700 W power limit: DeepFilterNet3 0.997, DeepFilterNet3_ll 0.994,
DeepFilterNet2 0.997, v1 0.999 (a gain bin's single rounded product against its u |x g| bound); the generic kernel 0.49 at
nb_df = 64 and 0.50 at 24 bands; 16-frame warps 0.996; the production batch 0.38."""
import ctypes as C
import dataclasses
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dsp_ref64 as R
from test_gpu_parity import cfg_of, cfg_v1

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance_device_ragged, libdf
from deepfilternet_b200._lib import DFB_ERR_UNSUPPORTED, DfbError, check
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.weights import random_state_dict

HOP = 480
F = 481
F32 = np.float32
TH = (-10.0, 30.0, 20.0)
KINDS = {   # name: (test_gpu_parity config, nb_df, apply mode, df look-ahead)
    "dfn3": ("dfn3", 96, 1, 2), "ll": ("ll", 96, 1, 0), "dfn2": ("dfn2", 96, 2, 2), "v1": ("v1", 96, 2, 1),
    "dfn3_df64": ("dfn3", 64, 1, 2), "dfn3_e24": ("e24", 96, 1, 2),     # the generic kernel
}
OPTS = {"plain": (False, False), "pf": (True, False), "mask_only": (False, True)}
_libm = C.CDLL("libm.so.6")
_libm.powf.restype, _libm.powf.argtypes = C.c_float, [C.c_float, C.c_float]


def lim_of(db):
    """The library's limit factor of db dB: powf(10, -db / 20) in fp32, from the same libm."""
    return float(_libm.powf(10.0, float(F32(-F32(db) / F32(20)))))


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, HOP, 32, 2)


@pytest.fixture(scope="module")
def models(st):
    out = {}
    for name, (kind, nb_df, _, _) in KINDS.items():
        cfg = dataclasses.replace(cfg_v1() if kind == "v1" else cfg_of(kind), nb_df=nb_df)
        out[name] = DfNet(cfg, random_state_dict(cfg, seed=3), st if cfg.nb_erb == 32 else libdf.DF(48000, 960, HOP, cfg.nb_erb, 2))
    return out


def debug_apply_rows(model, spec, m, c, *, Tf, n_audio, alpha=None, lsnr=None, Tv=0, rows=None, first=None, links=None,
                     reduce="max", ctl=None, th=TH, atten_lim=0.0, w0=0, t_first=0, t_emit=None, out_offset=0, out_len=0,
                     pf=False, mask_only=False):
    """dfb_debug_apply_rows on NaN-filled outputs -> (spec_out [B, Tf, F] complex, audio [n_audio])."""
    L = _lib.lib()
    B, spec_T = spec.shape[:2]
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    d_spec, d_m, d_c = dev(spec.astype(np.complex64).view(np.float32)), dev(m.astype(np.float32)), dev(c.astype(np.complex64).view(np.float32))
    d_a, d_l = dev(None if alpha is None else alpha.astype(np.float32)), dev(None if lsnr is None else lsnr.astype(np.float32))
    audio = torch.full((n_audio,), float("nan"), device="cuda")
    sout = torch.full((B, Tf, F, 2), float("nan"), device="cuda")
    h_rows = None if rows is None else np.ascontiguousarray(rows, np.int64)
    h_first = None if first is None else np.ascontiguousarray(first, np.int64)
    h_links = None if links is None else np.ascontiguousarray(links, np.int32)
    h_ctl = h_sw = h_gate = None
    if ctl is not None:
        h_ctl = np.ascontiguousarray([[x["lim"], x["beta"], x["lim0"], x["beta0"], x["th_min"], x["th_erb"], x["th_df"]]
                                      for x in ctl], np.float32)
        h_sw = np.ascontiguousarray([x["sw"] for x in ctl], np.int64)
        h_gate = np.ascontiguousarray([x["gate"] for x in ctl], np.int32)
    ptr = lambda a: None if a is None else (a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data)   # noqa: E731
    i64p = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int64))   # noqa: E731
    check(L.dfb_model_set_options(model.handle, int(pf), C.c_float(0.02), int(mask_only)))
    try:
        check(L.dfb_debug_apply_rows(model.handle, model.df_state.handle, ptr(d_spec), spec_T, Tv, ptr(d_m), ptr(d_c), ptr(d_a),
                                     ptr(d_l), m.shape[1], B, Tf, t_first, Tf if t_emit is None else t_emit, w0, i64p(h_rows),
                                     i64p(h_first), ptr(h_links), {"max": 1, "mean": 2}[reduce], ptr(h_ctl), i64p(h_sw),
                                     ptr(h_gate), *(C.c_float(x) for x in th), C.c_float(atten_lim), out_offset, out_len,
                                     audio.data_ptr(), sout.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    finally:
        check(L.dfb_model_set_options(model.handle, int(model.post_filter), C.c_float(model.post_filter_beta), int(not model.run_df)))
    return sout.cpu().numpy().view(np.complex64)[..., 0].astype(np.complex128), audio.cpu().numpy().astype(np.float64)


def compare(name, got, ref):
    """got = (spec_out, audio); ref = apply_rows' result: within K = 1 where written, the NaN sentinel elsewhere."""
    worst = 0.0
    for what, g, (r, b, w) in (("spec", got[0], ref[0]), ("audio", got[1], ref[1])):
        assert np.isnan(g[~w]).all(), (name, what, "written outside the row's set")
        assert not np.isnan(g[w]).any(), (name, what, "an element of the row's set not written")
        worst = max(worst, R.err_ratio(g[w], r[w], b[w]))
    print(f"err/bound {name}: {worst:.3g}")
    assert worst <= 1, (name, worst)
    return worst


def inputs(B, spec_T, mc_T, nb_df, E, seed, first_rel=None):
    """Random spectra with exact-zero bins (zero before a slot's first frame, as a slot's spectrum is), masks with exact 0
    and 1 entries, random coefficients, alpha with exact 0 and 1."""
    rng = np.random.default_rng(seed)
    spec = ((rng.standard_normal((B, spec_T, F)) + 1j * rng.standard_normal((B, spec_T, F))) * 0.1).astype(np.complex64)
    spec[rng.random(spec.shape) < 0.1] = 0
    if first_rel is not None:
        for b, f in enumerate(first_rel):
            spec[b, :max(f, 0)] = 0
    m = rng.random((B, mc_T, E)).astype(np.float32)
    m[rng.random(m.shape) < 0.1] = 0
    m[rng.random(m.shape) < 0.1] = 1
    c = ((rng.standard_normal((B, mc_T, nb_df, 5)) + 1j * rng.standard_normal((B, mc_T, nb_df, 5))) * 0.5).astype(np.complex64)
    a = rng.random((B, mc_T)).astype(np.float32)
    a[:, ::5], a[:, 1::5] = 0.0, 1.0
    return spec, m, c, a


def lsnr_rows(B, T, ths, links, seed):
    """LSNR [B, T] over the thresholds ths[b] of each row: exact thresholds, one ulp either side and values inside every
    stage; every channel after a group's first gets other values, so a row gating on its own LSNR sees other stages."""
    rng = np.random.default_rng(seed)
    out = np.empty((B, T), np.float32)
    for b in range(B):
        t = ths[b]
        pick = [x for v in t for x in (np.nextafter(F32(v), F32(-np.inf)), F32(v), np.nextafter(F32(v), F32(np.inf)))]
        pick += [F32(t[0] - 5), F32((t[0] + t[2]) / 2), F32((t[1] + t[2]) / 2), F32(t[1] + 5)]
        out[b] = rng.choice(pick, T)
        if links is not None and links[b][0] != b:
            out[b] = out[b][::-1]
    return out


# Row geometry of the 8-frame-warp window (32-frame CTAs): window frames 0 .. 47 are absolute w0 + t.  Per row: its end
# (window frame; > 48: not ended, synthesises up to t_emit), its first frame and its settings switch, each just before, on
# and just after warp starts 8 / 16 / 40 and CTA start 32.  Every switch lies inside its row's synthesised frames, and rows 9,
# 10, 12, 15 and 16 switch on a warp's first frame t0 with frame t0 - 1 already part of the stream.
W0, TF8 = 5, 48
ENDS = [7, 8, 9, 15, 16, 17, 31, 32, 33, 60, 47, 48, 60, 47, 46, 60, 44, 60]
FIRSTS = [0, 7, 8, 9, -3, 16, 17, 31, 32, 0, 33, 0, 24, 0, 2, 0, 0, 0]
SWITCH = [1, 7, 8, 9, 15, 16, 17, 24, 32, 16, 40, 31, 32, 33, 41, 40, 8, 39]
GROUPS = [(0, 1), (1, 2), (3, 3), (6, 5)]       # link groups (first, n): sizes 1, 2, 3 and 5
GEOMS = [  # t_first, t_emit, spec_T, Tv, out_offset
    dict(t_first=0, t_emit=48, spec_T=48, Tv=48, out_offset=-300),
    dict(t_first=1, t_emit=45, spec_T=52, Tv=50, out_offset=200),
    dict(t_first=8, t_emit=48, spec_T=50, Tv=44, out_offset=480),
]


def geometry(B, geo, Tf=TF8, ends=ENDS, w0=W0, hop_cut=137, gap=333):
    """rows (out_off, out_len, absolute end) with gaps between the output rows and out_len cutting a hop; n_audio."""
    rows, off = [], 0
    for b in range(B):
        Te = ends[b] if ends[b] <= Tf else geo["t_emit"]
        n = max(Te * HOP - geo["out_offset"] - hop_cut * (b % 2), 0)
        rows.append((off, n, ends[b] + w0))
        off += n + gap
    return rows, off


def link_table(B):
    links = [(b, 1) for b in range(B)]
    for f, n in GROUPS:
        for b in range(f, f + n):
            links[b] = (f, n)
    return links


def ctl_table(B, links, gating):
    """Per-row settings: new / old limit and beta with the switch at SWITCH, thresholds per link group (one group does not
    gate, one has other thresholds)."""
    out = []
    for b in range(B):
        f = links[b][0] if links is not None else b
        th = (-12.0, 25.0, 12.0) if f % 3 == 1 else TH
        out.append(dict(lim=lim_of(6 + b % 3 * 6) if b % 4 else 0.0, beta=0.02 * (b % 3), lim0=lim_of(9) if b % 2 else 0.0,
                        beta0=0.03 if b % 3 != 1 else 0.0, sw=SWITCH[b] + W0, th_min=th[0], th_erb=th[1], th_df=th[2],
                        gate=int(gating and f != 3)))
    return out


INSTANCES = ["table_free", "rg", "link_max", "link_mean", "ctl", "link_ctl"]


@pytest.mark.parametrize("lim", [False, True])
@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("inst", INSTANCES)
@pytest.mark.parametrize("kind", ["dfn3", "ll", "dfn2", "v1"])
def test_instances_against_ref64(models, kind, inst, opt, lim):
    """Every specialised instance (table-free, RG, RG + LINK with max / mean, RG + CTL, RG + LINK + CTL) for DeepFilterNet3,
    DeepFilterNet3_ll, DeepFilterNet2 and v1, plain / post filter / mask_only, with and without the limit; LSNR gating
    (handle-wide thresholds, or each row's own with CTL) for the two DeepFilterNet3 models, at the 8-frame warp tiles.  The
    link-mean masks hold frames whose fp32 sum rounds differently in any order but the channel order.  K = 1 (worst err / bound on an H100 80GB HBM3 at 700 W: 0.997 / 0.994 / 0.997 / 0.999 in that order)."""
    _, nb_df, mode, la = KINDS[kind]
    pf, mask_only = OPTS[opt]
    model = models[kind]
    B = len(ENDS)
    geo = GEOMS[(INSTANCES.index(inst) + list(OPTS).index(opt)) % 3]
    table = inst != "table_free"
    first = [f + W0 for f in FIRSTS] if table else None
    spec, m, c, a = inputs(B, geo["spec_T"], TF8, nb_df, 32, seed=zlib.crc32(f"{kind} {inst} {opt} {lim}".encode()) % 1000,
                           first_rel=FIRSTS if table else None)
    links = link_table(B) if inst.startswith("link") else None
    reduce = "mean" if inst == "link_mean" else "max"
    ctl = ctl_table(B, links, mode == 1) if inst.endswith("ctl") else None
    if ctl:
        assert all(0 < SWITCH[b] < (ENDS[b] if ENDS[b] <= TF8 else geo["t_emit"]) for b in range(B))
    if reduce == "mean":
        # frames where channel 0 holds 1 and the others 0.4 ulp(1) each: the fp32 sum in channel order stays 1, in any other
        # order the small terms add up first and round 1 up by one or two ulp, which moves the mean by 2 - 4 u
        for f, n in GROUPS[2:]:
            m[f, 1::4] = 1.0
            m[f + 1:f + n, 1::4] = F32(0.4 * 2.0 ** -23)
    gating = mode == 1
    ths = [(x["th_min"], x["th_erb"], x["th_df"]) for x in ctl] if ctl else [TH] * B
    lsnr = lsnr_rows(B, TF8, ths, links, seed=7) if gating else None
    alpha = a if kind == "v1" else None
    atten = lim_of(12) if lim else 0.0
    if table:
        rows, n_audio = geometry(B, geo)
        out_len = 0
    else:
        rows, out_len = None, TF8 * HOP - geo["out_offset"] - 137
        n_audio = B * out_len
    kw = dict(Tf=TF8, n_audio=n_audio, alpha=alpha, lsnr=lsnr, rows=rows, first=first, links=links, reduce=reduce, ctl=ctl,
              atten_lim=atten, w0=W0 if table else 0, t_first=geo["t_first"], t_emit=geo["t_emit"] if table else TF8,
              out_offset=geo["out_offset"], out_len=out_len)
    got = debug_apply_rows(model, spec, m, c, Tv=geo["Tv"], pf=pf, mask_only=mask_only, **kw)
    ref = R.apply_rows(spec, m, c, model.df_state.erb_widths(), model.df_state.fft_window(), mode=mode, nb_df=nb_df, order=5,
                       lookahead=la, post_filter=pf, mask_only=mask_only, Tv=geo["Tv"], th=TH, **kw)
    if gating:
        seen = set()
        for b in range(B):
            lb = links[b][0] if links else b
            t3 = ths[b]
            seen |= set(R.stage_of(lsnr[lb], *t3).tolist())
        assert seen == {0, 1, 2, 3}
    compare(f"{kind} {inst} {opt} lim={lim}", got, ref)


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("kind", ["dfn3_df64", "dfn3_e24"])
def test_generic_rows_against_ref64(models, kind, opt):
    """k_apply_synthesis_generic with a row table and slot first frames (nb_df = 64, and 24 ERB bands), with the limit.
    K = 1 (worst err / bound on an H100 80GB HBM3 at 700 W: 0.49 at nb_df = 64, 0.50 at 24 bands)."""
    _, nb_df, mode, la = KINDS[kind]
    pf, mask_only = OPTS[opt]
    model = models[kind]
    B, geo = len(ENDS), GEOMS[1]
    first = [f + W0 for f in FIRSTS]
    spec, m, c, _ = inputs(B, geo["spec_T"], TF8, nb_df, model.df_state.nb_erb(), seed=11, first_rel=FIRSTS)
    rows, n_audio = geometry(B, geo)
    kw = dict(Tf=TF8, n_audio=n_audio, rows=rows, first=first, atten_lim=lim_of(9), w0=W0, t_first=geo["t_first"],
              t_emit=geo["t_emit"], out_offset=geo["out_offset"])
    got = debug_apply_rows(model, spec, m, c, Tv=geo["Tv"], pf=pf, mask_only=mask_only, **kw)
    ref = R.apply_rows(spec, m, c, model.df_state.erb_widths(), model.df_state.fft_window(), mode=mode, nb_df=nb_df, order=5,
                       lookahead=la, post_filter=pf, mask_only=mask_only, Tv=geo["Tv"], **kw)
    compare(f"{kind} {opt}", got, ref)


@pytest.mark.parametrize("kind", ["dfn2", "v1", "dfn3_df64", "dfn3_e24"])
def test_refusals(models, kind):
    """LSNR gating is built for DeepFilterNet3's apply kernel only; link groups and per-row settings for the specialised
    kernel only: the launcher refuses the rest with DFB_ERR_UNSUPPORTED."""
    _, nb_df, mode, _ = KINDS[kind]
    model = models[kind]
    B, Tf = 2, 8
    spec, m, c, a = inputs(B, Tf, Tf, nb_df, model.df_state.nb_erb(), seed=1)
    alpha = a if kind == "v1" else None
    rows = [(0, Tf * HOP, Tf), (Tf * HOP, Tf * HOP, Tf)]
    lsnr = np.zeros((B, Tf), np.float32)
    cases = [dict(lsnr=lsnr), dict(lsnr=lsnr, rows=rows)]
    if kind not in ("dfn2", "v1"):
        ctl = [dict(lim=0.0, beta=0.0, lim0=0.0, beta0=0.0, sw=0, th_min=0.0, th_erb=0.0, th_df=0.0, gate=0)] * B
        cases += [dict(rows=rows, links=[(0, 2), (0, 2)]), dict(rows=rows, ctl=ctl)]
    for kw in cases:
        with pytest.raises(DfbError) as e:
            debug_apply_rows(model, spec, m, c, Tf=Tf, n_audio=B * Tf * HOP, out_len=Tf * HOP, alpha=alpha, **kw)
        assert e.value.code == DFB_ERR_UNSUPPORTED, (kw.keys(), e.value)


@pytest.mark.parametrize("inst", ["rg", "link_ctl"])
@pytest.mark.parametrize("kind", ["dfn3", "dfn2"])
def test_16_frame_warps(models, kind, inst):
    """B * Tf / 16 >= 6000 (the shape bench.py runs): 16 frames per warp, 64-frame CTAs.  64 rows of a 1501-frame window;
    rows 0, 1, 36, 37, 62 and 63 are compared in full, with ends at 63, 64, 65, 1472 and 1473, first frames at 15, 16, 47
    and 48, and (link_ctl: the settings of each pair's first row) switches at warp start 48, CTA start 64 and CTA start 1472.
    Every gap between the 64 output rows keeps its NaN sentinel.  K = 1 (worst err / bound on an H100 80GB HBM3 at 700 W:
    0.996)."""
    _, nb_df, mode, la = KINDS[kind]
    model = models[kind]
    B, Tf, w0 = 64, 1501, 2
    ends = [1501] * B
    firsts = [0] * B
    sw = [0] * B
    for b, e, f, s in ((0, 64, 0, 48), (1, 65, 0, 48), (36, 1472, 15, 64), (37, 1473, 16, 64), (62, 1501, 47, 1472), (63, 63, 48, 1472)):
        ends[b], firsts[b], sw[b] = e, f, s
    spec, m, c, _ = inputs(B, Tf, Tf, nb_df, 32, seed=5, first_rel=firsts)
    geo = dict(t_first=1, t_emit=Tf, out_offset=-480)
    rows, n_audio = geometry(B, geo, Tf=Tf, ends=ends, w0=w0)
    links = [(b - b % 2, 2) for b in range(B)] if inst == "link_ctl" else None
    ctl = None
    if inst == "link_ctl":
        ctl = [dict(lim=lim_of(12), beta=0.02 if mode == 1 else 0.0, lim0=0.0, beta0=0.0, sw=sw[b - b % 2] + w0, th_min=TH[0],
                    th_erb=TH[1], th_df=TH[2], gate=int(mode == 1)) for b in range(B)]
    lsnr = lsnr_rows(B, Tf, [TH] * B, links, seed=3) if mode == 1 else None
    first = [f + w0 for f in firsts]
    kw = dict(Tf=Tf, lsnr=lsnr, rows=rows, first=first, links=links, ctl=ctl, w0=w0, t_first=geo["t_first"], t_emit=Tf,
              out_offset=geo["out_offset"], th=TH)
    sout, audio = debug_apply_rows(model, spec, m, c, n_audio=n_audio, **kw)
    inside = np.zeros(n_audio, bool)
    for (o, n, _) in rows:
        inside[o:o + n] = True
    assert np.isnan(audio[~inside]).all(), "written into a gap between output rows"
    sel = [0, 1, 36, 37, 62, 63]
    sub = lambda a: None if a is None else a[sel]   # noqa: E731
    rows_s = [rows[b] for b in sel]
    off0 = [r[0] for r in rows_s]
    rows_s = [(o - off0[0], n, e) for (o, n, e) in rows_s]
    links_s = None if links is None else [(sel.index(links[b][0]), 2) for b in sel]
    ref = R.apply_rows(spec[sel], m[sel], c[sel], model.df_state.erb_widths(), model.df_state.fft_window(), mode=mode,
                       nb_df=nb_df, order=5, lookahead=la, n_audio=n_audio - off0[0], **dict(kw, lsnr=sub(lsnr), rows=rows_s,
                       first=[first[b] for b in sel], links=links_s, ctl=None if ctl is None else [ctl[b] for b in sel]))
    (rY, bY, wY), (ra, ba, wa) = ref
    # the selected rows' audio lies in [off0, ...): keep only their own ranges, as the reference knows nothing of the rest
    a_sel = audio[off0[0]:]
    keep = np.zeros(a_sel.shape, bool)
    for (o, n, _) in rows_s:
        keep[o:o + n] = True
    a_got = np.where(keep, a_sel, np.nan)
    compare(f"{kind} {inst} 16-frame warps", (sout[sel], a_got), ((rY, bY, wY), (ra, ba, wa & keep)))


def model_outputs(model, x, st):
    """df_features' spectrum and dfb_model_forward's m / coefs / lsnr for audio x [B, T] (CPU)."""
    sp, fe, fs = df_features(x, st, model.nb_df)
    B, _, T, E = fe.shape
    d_fe, d_fs = fe.cuda().contiguous(), fs.cuda().contiguous()
    m = torch.empty((B, T, E), device="cuda")
    c = torch.empty((B, T, model.nb_df, 10), device="cuda")
    ls = torch.empty((B, T), device="cuda")
    check(_lib.lib().dfb_model_forward(model.handle, d_fe.data_ptr(), d_fs.data_ptr(), B, T, m.data_ptr(), c.data_ptr(),
                                       ls.data_ptr(), None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    spec = torch.view_as_complex(sp[:, 0].contiguous()).numpy()
    coefs = c.cpu().numpy().view(np.complex64).reshape(B, T, model.nb_df, 5)
    return spec, m.cpu().numpy(), coefs, ls.cpu().numpy()


def test_production_batch_equals_debug_entry(st, models):
    """The debug entry reaches what production reaches: a one-chunk enhance_device_ragged (pad=False, equal lengths, a link
    pair with the mean mask, a settings table with limits, post-filter betas and LSNR gating on two of three entries) equals
    dfb_debug_apply_rows bit for bit, run on df_features' spectrum and dfb_model_forward's m / coefs / lsnr of the same audio;
    and both lie within ref64's row-level bound of those inputs (K = 1; worst err / bound on an H100 80GB HBM3 at 700 W:
    0.38, with the linked pair's 70 frames at stages 0 / 1 / 2 / 3: 11 / 11 / 24 / 24)."""
    model = models["dfn3"]
    B, Tf = 3, 70
    T = Tf * HOP + 123
    g = torch.Generator().manual_seed(4)
    x = (torch.rand(B, T, generator=g) - 0.5) * 0.3
    x[2, 9000:20000] *= 0.01
    spec, m, c, lsnr = model_outputs(model, x, st)
    # thresholds at quantiles of the linked pair's gating LSNR, so that all four stages occur
    q = [float(F32(np.quantile(lsnr[0], f))) for f in (0.15, 0.85, 0.5)]
    lims, betas, ths = [12.0, 12.0, 6.0], [0.02, 0.02, 0.0], [tuple(q), tuple(q), None]
    model.set_chunking(1, 1, 1)
    try:
        out = enhance_device_ragged(model, st, x.cuda().contiguous(), [T] * B, pad=False, group_sizes=[2, 1], reduce_mask="mean",
                                    atten_lim_db=lims, post_filter_beta=betas, lsnr_thresholds=ths)
        torch.cuda.synchronize()
        out = out.cpu().numpy().astype(np.float64)
    finally:
        model.set_chunking()
    Tout = Tf * HOP
    rows = [(b * Tout, Tout, Tf) for b in range(B)]
    links = [(0, 2), (0, 2), (2, 1)]
    ctl = [dict(lim=lim_of(lims[b]), beta=betas[b], lim0=lim_of(lims[b]), beta0=betas[b], sw=0,
                th_min=ths[b][0] if ths[b] else 0.0, th_erb=ths[b][1] if ths[b] else 0.0, th_df=ths[b][2] if ths[b] else 0.0,
                gate=int(ths[b] is not None)) for b in range(B)]
    kw = dict(Tf=Tf, n_audio=B * Tout, lsnr=lsnr, rows=rows, links=links, reduce="mean", ctl=ctl, t_emit=Tf)
    got = debug_apply_rows(model, spec, m, c, **kw)
    stages = R.stage_of(lsnr[0], *q)
    print("stages of the linked pair:", np.bincount(stages, minlength=4))
    assert (np.bincount(stages, minlength=4) > 0).all()
    ref = R.apply_rows(spec, m, c, st.erb_widths(), st.fft_window(), mode=1, nb_df=96, order=5, lookahead=2, **kw)
    compare("debug entry", got, ref)
    compare("production", (got[0], out.reshape(-1)), ref)
    assert np.array_equal(got[1], out.reshape(-1)), np.abs(got[1] - out.reshape(-1)).max()


# ------------------------------------------------------------- the stage rule at equality, through the public API ----
def _equal_cases(ls, pick=None):
    """An LSNR value v of `pick` (default: ls) that occurs once among ls and whose fp32 neighbours do not occur, and for
    each threshold in turn (the other two out of the way) the thresholds at v, one ulp off in the direction that keeps
    every stage, and one ulp off the other way."""
    vals = ls[np.isfinite(ls)].astype(np.float32)
    uniq, cnt = np.unique(vals, return_counts=True)
    own = uniq[cnt == 1]
    if pick is not None:
        own = own[np.isin(own, np.asarray(pick, np.float32))]
    cand = [v for v in own[len(own) // 4:]
            if not np.isin([np.nextafter(v, F32(-np.inf)), np.nextafter(v, F32(np.inf))], vals).any()]
    assert cand
    v = F32(cand[len(cand) // 2])
    lo, hi = np.nextafter(v, F32(-np.inf)), np.nextafter(v, F32(np.inf))
    far = F32(1e4)
    return v, [  # (thresholds at v, kept, changed)
        ((v, far, far), (lo, far, far), (hi, far, far)),            # min: l < th
        ((-far, v, -far), (-far, hi, -far), (-far, lo, -far)),      # max_erb: l > th
        ((-far, far, v), (-far, far, hi), (-far, far, lo)),         # max_df: l > th
    ]


def _check_equal_cases(run, ls, what, pick=None):
    """run(thresholds) -> (audio, lsnr): at v and one ulp kept bit-identical, one ulp moved different."""
    _, cases = _equal_cases(ls, pick)
    for i, (eq, keep, other) in enumerate(cases):
        a_eq, l_eq = run(eq)
        a_keep, _ = run(keep)
        a_oth, _ = run(other)
        assert np.array_equal(a_eq, a_keep), (what, i, "one ulp that keeps every stage changed the output")
        assert not np.array_equal(a_eq, a_oth), (what, i, "one ulp that moves the equal frame's stage changed nothing")
        np.testing.assert_array_equal(l_eq, ls)      # the LSNR depends neither on the thresholds nor on the mode


@pytest.mark.parametrize("mode", ["apply", "runtime"])
def test_stage_rule_at_equal_lsnr(st, models, mode):
    """An LSNR exactly equal to a threshold takes tract's side (tract.rs:658-672: < min, > max_erb, > max_df) in the apply
    kernel and, in runtime mode, in k_gate_plan's choice of the decoders to run.  For each threshold in turn (the other two
    out of the way) it is set to an LSNR value v that occurs once in a ragged batch with a settings table, whose fp32
    neighbours do not occur: moving it one ulp in the direction that keeps every stage gives a bit-identical batch, moving
    it one ulp the other way changes the output."""
    model = models["dfn3"]
    lens = [60 * HOP + 17, 45 * HOP, 52 * HOP + 300]
    g = torch.Generator().manual_seed(9)
    x = ((torch.rand(3, max(lens), generator=g) - 0.5) * 0.3).cuda().contiguous()

    def run(th):
        out = enhance_device_ragged(model, st, x, lens, pad=False, atten_lim_db=[0.0] * len(lens), gating_mode=mode,
                                    return_lsnr=True, lsnr_thresholds=None if th is None else [tuple(float(t) for t in th)] * 3)
        torch.cuda.synchronize()
        return out[0].cpu().numpy(), out[1].cpu().numpy()
    _check_equal_cases(run, run(None)[1], f"batch {mode}")


@pytest.mark.parametrize("mode", ["apply", "runtime"])
def test_stage_rule_at_equal_lsnr_streaming_slot(st, models, mode):
    """The same on a streaming handle: slot 0 of two open slots gates with its own thresholds (the per-slot settings of the
    CTL instance and, in runtime mode, k_gate_plan's), slot 1 does not gate; calls of 5, 16 and 3 hops, then the flush."""
    model = models["dfn3"]
    g = torch.Generator().manual_seed(12)
    x = (torch.rand(2, 70 * HOP, generator=g) - 0.5) * 0.3

    def run(th):
        s = DfStream(model, st, batch=2, gating_mode=mode)
        s.open([0, 1])
        if th is not None:
            s.set_lsnr_thresholds(*(float(t) for t in th), slots=[0])
        outs, lss, pos, i = [], [], 0, 0
        while pos < 70:
            k = min((5, 16, 3)[i % 3], 70 - pos)
            y, l = s.process(x[:, pos * HOP:(pos + k) * HOP], return_lsnr=True)
            outs.append(y.cpu())
            lss.append(l.cpu())
            pos, i = pos + k, i + 1
        y, l = s.flush(return_lsnr=True)
        outs.append(y.cpu())
        lss.append(l.cpu())
        return torch.cat(outs, 1).numpy(), torch.cat(lss, 1).numpy()
    ls = run(None)[1]
    _check_equal_cases(run, ls, f"slot {mode}", pick=ls[0])     # v from the gating slot


SPEC_CODE = np.array([0, 3, 2, 1], np.int8)     # k_spec_emit's codes of stage_of's stages 0 - 3


@pytest.mark.parametrize("mode", ["apply", "runtime"])
def test_spectral_stage_codes_at_equal_lsnr(st, models, mode):
    """A spectral handle's stage codes (k_spec_emit, its own numbering: 0 zeros, 1 gains + DF, 2 gains, 3 unprocessed) equal
    tract's rule applied to its own reported LSNR, with each threshold in turn exactly at an LSNR value v, and one ulp either
    side, in calls of 1, 3, 16 and 33 frames."""
    model = models["dfn3"]
    g = torch.Generator().manual_seed(13)
    x = ((torch.rand(1, 90 * HOP, generator=g) - 0.5) * 0.3).numpy()
    spec = st.analysis(np.ascontiguousarray(x))

    def run(th):
        s = DfStream(model, st, batch=1, spectral=True, gating_mode=mode)
        s.set_lsnr_thresholds(*(float(t) for t in th))
        ls, sg, pos, i = [], [], 0, 0
        T = spec.shape[1]
        while pos < T:
            k = min((1, 3, 16, 33)[i % 4], T - pos)
            o = s.process_spec(torch.from_numpy(np.ascontiguousarray(spec[:, pos:pos + k])))
            ls.append(o.lsnr.cpu())
            sg.append(o.stage.cpu())
            pos, i = pos + k, i + 1
        o = s.flush_spec()
        ls.append(o.lsnr.cpu())
        sg.append(o.stage.cpu())
        return torch.cat(ls, 1).numpy()[0], torch.cat(sg, 1).numpy()[0]
    far = 1e4
    ls, _ = run((-far, far, far))
    v, cases = _equal_cases(ls)
    live = np.isfinite(ls)
    for triple in cases:
        for th in triple:
            l2, sg = run(th)
            np.testing.assert_array_equal(l2, ls)
            assert (sg[~live] == -1).all()
            want = SPEC_CODE[R.stage_of(ls[live], *th)]
            assert np.array_equal(sg[live], want), (th, np.flatnonzero(sg[live] != want))
            assert (sg[live][ls[live] == v] == want[ls[live] == v]).all()
