"""GPU: runtime gating's window kernels (csrc/dfb_model.cu forward_body under `if (gate)`) element by element against
float64 (tests/gating_ref64.py), call by call on streaming handles.  Each streaming call runs one window; after it the
gate plan, the compacted DF pathway rows P and their conv Q, the coefficients, the kt = 2 filled inputs, d3, the mask and
the ERB recurrence's output are fetched (dfb_model_debug_fetch) and checked, with each row's carried tails advanced by the
test from what earlier windows fetched:

  (a) plan: run flags, erb_src, df_pos, df_n and (kt = 2) erb_first exactly, and a spectral handle's emitted stages;
  (b) P rows [0, K - 1 + df_n) bit for bit;  (c) Q on them within the BF16x3 bound;
  (d) coefs = tanh(df_out(dfc)) + Q at DF run frames (+ nothing elsewhere), within model_ref64.coefs' bound;
  (e) kt = 2: dec_emb, e3, d1, e0 filled bit for bit, d3 and m within their bounds with inputs zero before erb_first;
  (f) the ERB recurrence's output at a new frame it did not run on equals the previous frame's, bit for bit.

Thresholds are LSNR values of the stream itself (a first pass records them), so ties decide frames, and one fp32 ulp
either side.  Every edge the scenarios are built to place is asserted to have occurred.

A ragged batch (enhance_device_ragged) in time chunks carries the same tail from one chunk's decoder phase to the next
chunk's gather: its last chunk's P tail rows are checked bit for bit against the c0 of the row's last K - 1 DF run frames.

Departures from the natural model list: the one-tap, nb_df 64 DeepFilterNet3 variant runs on a spectral handle, because
the apply kernel gates nb_df 96 only; DeepFilterNet2's ERB recurrence adds its input to its output (SqueezedGRU's skip),
so its output at a held frame is not the previous one's and (f) does not apply to it.

Worst err / bound over all scenarios on an H100 80GB HBM3 (700 W): Q 0.063, coefs 0.21, d3 0.062, mask 0.0057; the
plan, P, the fills, the held recurrence outputs and the ragged tail are exact.  The file's 14 tests take 50 s there."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import gating_ref64 as G
import model_ref64 as M
from dsp_ref64 import err_ratio
from test_gpu_gating_runtime import HOP, SEED, cfg_of, signal
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, DfStream, _lib, enhance_device_ragged, libdf
from deepfilternet_b200.weights import random_state_dict

C = 64
NEVER = (-1e9, 1e9, 1e9)
F32 = np.float32
MODELS = {
    "dfn3": lambda: cfg_of("dfn3"),
    "dfn3_ll": lambda: cfg_of("dfn3_ll"),
    "dfn3_df64_k1": lambda: dataclasses.replace(cfg_of("dfn3"), nb_df=64, df_pathway_kernel_size_t=1),
    "dfn3_ll_k3": lambda: dataclasses.replace(cfg_of("dfn3_ll"), df_pathway_kernel_size_t=3),
    "dfn2": lambda: cfg_of("dfn2"),
    "dfn2_ll": lambda: cfg_of("dfn2_ll"),
}
# new frames per call: 1, 2 and 3+ frames per k_gate_plan thread, and short calls that mix old and new tail rows
SIZES = [5, 1, 2, 1, 3, 255, 1, 1, 256, 2, 257, 4, 1, 512, 3, 1, 513, 6, 1, 1000, 7, 2, 1, 5, 8, 10, 4, 12, 9, 16, 6, 11] + [10, 9] * 8


@pytest.fixture(scope="module")
def st():
    return libdf.DF(48000, 960, 480, 32, 2)


_BUILT = {}


def built(st, name):
    if name not in _BUILT:
        cfg = MODELS[name]()
        sd = random_state_dict(cfg, seed=SEED)
        _BUILT[name] = (cfg, sd, DfNet(cfg, sd, st)) + M.state64(sd)
    return _BUILT[name]


def fetch(model, name, n, dtype=np.float32):
    words = {np.uint8: (n + 3) // 4, np.int32: n, np.int64: 2 * n, np.uint16: n // 2}.get(dtype, n)
    out = np.empty(words, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), out.ctypes.data, out.size)
    assert got == words, (name, got, words)
    return out.view(dtype)[:n] if dtype is not np.float32 else out


def fetchable(model, name):
    return _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), np.empty(1, np.float32).ctypes.data, 1) == 1


def planes(hi, lo):
    f = lambda u: (u.astype(np.uint32) << 16).view(np.float32).astype(np.float64)   # noqa: E731   (hi / lo bit patterns)
    return f(hi) + f(lo)


class Handle:
    """A streaming handle plus what the test knows of it: the clock, each slot's row, first frame, settings and tails."""

    def __init__(self, name, cfg, sd64, ab, model, st, batch=1, spectral=False, reduce=None):
        self.name, self.cfg, self.sd64, self.ab, self.model = name, cfg, sd64, ab, model
        self.s = DfStream(model, st, batch=batch, spectral=spectral, reduce_mask=reduce, gating_mode="runtime")
        self.spectral, self.batch, self.linked = spectral, batch, reduce is not None
        self.Lmax = cfg.conv_lookahead if spectral else max(cfg.conv_lookahead, cfg.df_lookahead)
        self.lat = self.s.latency_frames
        self.a1 = self.d1 = 0
        self.rows = list(range(batch))               # row -> slot
        self.first = {b: 0 for b in range(batch)}
        self.group = {b: b for b in range(batch)}     # slot -> its group's channel-0 slot
        self.closing = {}                             # slot -> end frame
        self.th = {b: None for b in range(batch)}     # slot -> own (gate, th) or None: the handle's
        self.handle_th = None                         # (gate, th)
        self.kt, self.K = cfg.conv_kernel[0], cfg.df_pathway_kernel_size_t
        E, Fd = cfg.nb_erb, cfg.nb_df
        self.ED = E // 4 * C
        self.widths = (self.ED, self.ED, E * C, E * C)
        self.tails = {b: G.Tails(self.K, Fd * C, self.widths if self.kt > 1 else ()) for b in range(batch)}
        self.last_gru = {}                            # slot -> ERB recurrence output planes at its last frame
        self.gated_last = False                       # the last DNN window ran in runtime mode with gating
        self.mode = "runtime"
        self.ratios = {}
        self.hit = set()

    # ---- settings, mirrored
    def set_th(self, th, enable=True, slots=None):
        th = tuple(float(F32(v)) for v in th)
        self.s.set_lsnr_thresholds(*th, enable=enable, slots=slots)
        if slots is None:
            self.handle_th = (enable, th)
        else:
            for b in slots:
                self.th[b] = (enable, th)

    def set_mode(self, mode):
        self.s.set_gating_mode(mode)
        self.mode = mode

    def open(self, slots, linked=False):
        (self.s.open_linked if linked else self.s.open)(list(slots))
        for b in slots:
            if b in self.rows:
                self.rows.remove(b)
            self.closing.pop(b, None)
        for b in slots:
            self.rows.append(b)
            self.first[b] = self.a1
            self.group[b] = slots[0]
            self.th[b] = None
            self.tails[b] = G.Tails(self.K, self.cfg.nb_df * C, self.widths if self.kt > 1 else ())
            self.last_gru[b] = None
        self.hit.add("opened")

    def close(self, slots):
        self.s.close(list(slots))
        for b in slots:
            self.closing[b] = self.a1
        self.retire()

    def retire(self):
        """closing slots leave once their last frame is out (slots_retire): at once without latency"""
        for b, end in list(self.closing.items()):
            if end <= self.a1 - self.lat:
                self.rows.remove(b)
                del self.closing[b]
                self.hit.add("rows moved")

    def row_settings(self):
        gate, th = [], []
        for b in self.rows:
            own = self.th[b] if self.th[b] is not None else self.handle_th
            gate.append(bool(own and own[0]))
            th.append(own[1] if own else NEVER)
        return gate, th

    # ---- one call
    def call(self, x, n):
        """x: [batch, n hops] audio, or [batch, n, F] spectra"""
        gating = self.mode == "runtime" and any(self.row_settings()[0])
        rows_before = list(self.rows)
        a1n = self.a1 + n
        d1n = max(self.d1, a1n - self.Lmax)
        W0 = max(0, self.d1 - 8)
        Rc, T = self.d1 - W0, d1n - W0
        if self.spectral:
            out = self.s.process_spec(torch.from_numpy(np.ascontiguousarray(x)))
        else:
            out = self.s.process(x)
        torch.cuda.synchronize()
        res = None
        if d1n > self.d1 and rows_before:
            if gating:
                res = self.check(rows_before, W0, Rc, T, out if self.spectral else None)
            self.gated_last = gating
            if not gating:   # the recurrences ran every frame: their last outputs are not the ones the test kept
                self.last_gru = {}
        self.a1, self.d1 = a1n, d1n
        self.retire()
        return res

    def check(self, rows, W0, Rc, T, spec_out):
        cfg, model, K = self.cfg, self.model, self.K
        B, Mf = len(rows), len(rows) * T
        E, Fd, Hd, H = cfg.nb_erb, cfg.nb_df, cfg.df_hidden_dim, cfg.emb_hidden_dim
        Wc, Wq = Fd * C, Fd * 2 * cfg.df_order
        Tp = K - 1 + T - Rc
        from_halo = not self.gated_last
        lsnr = fetch(model, "lsnr", Mf).reshape(B, T)
        gate, th = self.row_settings()
        first = [self.first[b] for b in rows]
        links = [rows.index(self.group[b]) for b in rows] if self.linked else None
        pl = G.plan(lsnr, first, W0, Rc, th, gate, links, from_halo, [self.tails[b].has_run for b in rows])
        pl["Rc"] = Rc
        # (a) the plan
        got = dict(erb_run=fetch(model, "gate_erb_run", Mf, np.uint8).reshape(B, T), df_run=fetch(model, "gate_df_run", Mf, np.uint8).reshape(B, T),
                   erb_src=fetch(model, "gate_erb_src", Mf, np.int32).reshape(B, T), df_pos=fetch(model, "gate_df_pos", Mf, np.int32).reshape(B, T),
                   df_n=fetch(model, "gate_df_n", B, np.int32))
        for k in ("erb_run", "df_run"):
            assert np.array_equal(got[k][:, Rc:] != 0, pl[k][:, Rc:]), (self.name, k, W0)
        for k in ("erb_src", "df_pos"):
            assert np.array_equal(got[k][:, Rc:], pl[k][:, Rc:]), (self.name, k, W0)
        assert np.array_equal(got["df_n"], pl["df_n"]), (self.name, W0)
        if self.kt > 1:
            assert np.array_equal(fetch(model, "gate_erb_first", B, np.int64), pl["erb_first"]), (self.name, W0)
        for r, b in enumerate(rows):
            if gate[r]:
                for k, v in enumerate(th[r]):
                    if (lsnr[links[r] if links else r, max(Rc, first[r] - W0):] == F32(v)).any():
                        self.hit.add(("tie", k))
        if spec_out is not None:
            stage = spec_out[3].cpu().numpy()
            for j in range(stage.shape[1]):
                t = self.a1 - self.lat + j - W0
                if Rc <= t < T:
                    for r, b in enumerate(rows):
                        s = int(stage[b, j])
                        assert (s in (1, 2)) == pl["erb_run"][r, t] and (s == 1) == pl["df_run"][r, t], (self.name, t, s)
                        self.hit.add("stages")
        # (b) compaction, (c) pathway conv
        c0 = fetch(model, "c0", Mf * Wc).reshape(B, T, Wc)
        P = fetch(model, "gate_P", B * Tp * Wc).reshape(B, Tp, Wc)
        Q = fetch(model, "gate_Q", B * Tp * Wq).reshape(B, Tp, Fd, 2 * cfg.df_order)
        if fetchable(model, "dfc"):
            dfc = fetch(model, "dfc", Mf * Hd).reshape(B, T, Hd).astype(np.float64)
        else:
            dfc = planes(*(fetch(model, f"dfc_{p}", Mf * Hd, np.uint16).reshape(B, T, Hd) for p in ("hi", "lo")))
        coefs = fetch(model, "coefs", Mf * Wq).reshape(B, T, Fd, 2 * cfg.df_order)
        for r, b in enumerate(rows):
            tf = max(first[r] - W0, 0)
            tail = G.halo_tail(c0[r], Rc, K, tf) if from_halo else self.tails[b].c0
            want = G.compact(c0[r], tail, pl, r, Rc)
            n = want.shape[0]
            assert np.array_equal(P[r, :n], want), (self.name, "P", r, W0)
            q, bq = G.pathway_q(self.sd64, self.ab, want, Fd, C, cfg.df_order)
            self.ratios["Q"] = max(self.ratios.get("Q", 0), err_ratio(Q[r, K - 1:n], q[K - 1:], bq[K - 1:]))
            # (d) coefficients of the new frames
            ref, bound = G.coefs(self.sd64, self.ab, cfg, dfc[r, Rc:], q, bq, pl["df_run"][r, Rc:], pl["df_pos"][r, Rc:], K)
            self.ratios["coefs"] = max(self.ratios.get("coefs", 0), err_ratio(coefs[r, Rc:], ref, bound))
            self.tails[b].c0 = G.next_c0_tail(want, K)
            dn = int(pl["df_n"][r])
            self.hit.add(("df_n", "many" if dn > K + 1 else dn))
            if gate[r] and not pl["erb_run"][r, Rc:].any() and T - Rc > 0 and first[r] <= W0 + Rc:
                self.hit.add("no ERB run frame")
            if gate[r] and pl["erb_run"][r, Rc] and first[r] <= W0 + Rc:
                self.hit.add("ERB run on first new frame")
            if from_halo:
                self.hit.add(("from_halo Rc", min(Rc, 8)))
        self.hit.add(("new frames", T - Rc))
        if self.kt > 1:
            self.check_fill(rows, pl, W0, Rc, T, from_halo, first)
        if cfg.model != "deepfilternet2":   # DeepFilterNet2 adds the GRU input to its output as a skip: not held
            self.check_gru(rows, pl, W0, Rc, T, gate, first)
        return pl

    def check_fill(self, rows, pl, W0, Rc, T, from_halo, first):
        cfg, model = self.cfg, self.model
        B, Mf, E, ED = len(rows), len(rows) * T, self.cfg.nb_erb, self.ED
        e3w = 2 * ED if cfg.enc_concat else ED
        xs = [fetch(model, "dec_emb", Mf * ED).reshape(B, T, ED), fetch(model, "e3", Mf * e3w).reshape(B, T, e3w)[:, :, :ED],
              fetch(model, "d1", Mf * E * C).reshape(B, T, E * C), fetch(model, "e0", Mf * E * C).reshape(B, T, E * C)]
        d3 = fetch(model, "d3", Mf * ED).reshape(B, T, E // 4, C)
        m = fetch(model, "m", Mf * E).reshape(B, T, E)
        ef = fetch(model, "gate_erb_first", B, np.int64)
        for r, b in enumerate(rows):
            tl = self.tails[b]
            lo = max(Rc - 1, 0)
            for i, x in enumerate(xs):
                # the fetched run rows are the kernels' own; the non-run rows must be the fill of them
                want = G.filled(x[r], pl, r, Rc, tl.run[i], from_halo)
                assert np.array_equal(x[r, lo:], want), (self.name, "fill", i, r, W0)
                tl.run[i] = want[-1].copy()
            tl.has_run = bool(pl["has_run"][r])
            if ef[r] > first[r]:
                self.hit.add("erb_first inside the stream")
            s = int(max(lo, ef[r] - W0))
            if s >= T:
                continue
            t0 = max(Rc, s)
            cl = lambda a, F_: M.channel_last(a[r:r + 1].reshape(1, T, F_, C))   # noqa: E731
            ref, bound = G.convt3(self.sd64, self.ab, cl(xs[0], E // 4), cl(xs[1], E // 4), s)
            got = M.channel_last(d3[r:r + 1])[:, :, t0:]
            self.ratios["d3"] = max(self.ratios.get("d3", 0), err_ratio(got.numpy(), ref[:, :, t0 - s:].numpy(), bound[:, :, t0 - s:].numpy()))
            ref, bound = G.mask(self.sd64, self.ab, cl(xs[3], E), cl(xs[2], E), s)
            got = m[r, t0:][None, None]
            self.ratios["mask"] = max(self.ratios.get("mask", 0), err_ratio(got, ref[:, :, t0 - s:].numpy(), bound[:, :, t0 - s:].numpy()))

    def check_gru(self, rows, pl, W0, Rc, T, gate, first):
        model, H = self.model, self.cfg.emb_hidden_dim
        B, Mf = len(rows), len(rows) * T
        if fetchable(model, "g_b"):
            # (registered with the larger of the two decoders' widths; the ERB recurrence writes it at row pitch H)
            g = fetch(model, "g_b", Mf * max(H, self.cfg.df_hidden_dim))[:Mf * H].reshape(B, T, H)
        else:
            g = np.stack([fetch(model, f"erb_gru_{p}", Mf * H, np.uint16).reshape(B, T, H) for p in ("hi", "lo")], -1)
        for r, b in enumerate(rows):
            tf = max(first[r] - W0, 0)
            for t in range(max(Rc, tf + 1), T):
                if not pl["erb_run"][r, t]:
                    prev = g[r, t - 1] if t > Rc else self.last_gru.get(b)
                    if prev is not None:
                        assert np.array_equal(g[r, t], prev), (self.name, "held", r, W0 + t)
                        self.hit.add("held")
            self.last_gru[b] = g[r, T - 1].copy() if T - 1 >= tf else None

    def report(self):
        print(f"{self.name}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.ratios.items())))
        assert all(v <= 1 for v in self.ratios.values()), (self.name, self.ratios)


def chunks(x, sizes, spectral, st):
    """(call input, hops) of each call over the signal x [B, S]"""
    spec = st.analysis(np.ascontiguousarray(x.numpy())) if spectral else None
    pos = 0
    for n in sizes:
        yield (spec[:, pos:pos + n] if spectral else x[:, pos * HOP:(pos + n) * HOP]), n
        pos += n


def pick(values):
    """fp32 LSNR values at quantiles 0.1, 0.75 and 0.6: (min, max_erb, max_df), each exactly an LSNR of the stream"""
    v = np.sort(np.asarray(values, F32))
    return tuple(float(v[int(q * (v.size - 1))]) for q in (0.1, 0.75, 0.6))


def ulp(th, d):
    return tuple(float(np.nextafter(F32(v), F32(d * np.inf))) for v in th)


# (the apply kernel gates nb_df 96 only: the one-tap, nb_df 64 variant gates on a spectral handle)
SINGLE = [("dfn3", False), ("dfn3_ll", False), ("dfn3_df64_k1", True), ("dfn3_ll_k3", False), ("dfn3", True), ("dfn3_ll", True),
          ("dfn2", True), ("dfn2_ll", True)]


@pytest.mark.parametrize("name,spectral", SINGLE)
def test_single_stream(st, name, spectral):
    """One stream fed in calls of SIZES new frames, with thresholds equal to its own LSNR values and one ulp either side
    (DeepFilterNet3 audio: all three; the others: the exact values)."""
    cfg, sd, model, sd64, ab = built(st, name)
    x = signal(81, secs=sum(SIZES) * HOP / 48000 + 0.2)
    recorded = []
    h = Handle(name, cfg, sd64, ab, model, st, spectral=spectral)
    h.set_th(NEVER)
    for xi, n in chunks(x, SIZES, spectral, st):
        T0 = h.d1
        h.call(xi, n)
        if h.d1 > T0:
            W0 = max(0, T0 - 8)
            recorded.append(fetch(model, "lsnr", h.d1 - W0)[T0 - W0:])
    th = pick(np.concatenate(recorded))
    hits = set()
    for variant in ([th, ulp(th, 1), ulp(th, -1)] if name == "dfn3" and not spectral else [th]):
        h = Handle(name, cfg, sd64, ab, model, st, spectral=spectral)
        h.set_th(variant)
        for xi, n in chunks(x, SIZES, spectral, st):
            h.call(xi, n)
        h.report()
        hits |= h.hit
    for n in (1, 2, 255, 256, 257, 512, 513, 1000):
        assert ("new frames", n) in hits, n
    K = cfg.df_pathway_kernel_size_t
    for d in {0, 1, K - 2, K - 1, K, "many"} - {-1}:
        assert ("df_n", d) in hits, (d, [x for x in hits if x[0] == "df_n"])
    assert {("tie", 0), ("tie", 1), ("tie", 2), "no ERB run frame", "ERB run on first new frame"} <= hits, hits
    if spectral:
        assert "stages" in hits
    if cfg.model != "deepfilternet2":
        assert "held" in hits


@pytest.mark.parametrize("name", ["dfn3", "dfn3_ll"])
def test_mode_switches(st, name):
    """apply -> runtime at d1 = 1, 3 and 20 (the tails come from the halo: Rc < K - 1, and Rc = 8), runtime -> apply ->
    runtime, and a runtime call in which no row gates followed by a gated one."""
    cfg, sd, model, sd64, ab = built(st, name)
    x = signal(82, secs=6.0)
    Lmax = max(cfg.conv_lookahead, cfg.df_lookahead)
    h = Handle(name, cfg, sd64, ab, model, st)
    h.set_th(NEVER)
    h.call(x[:, :200 * HOP], 200)
    th = pick(fetch(model, "lsnr", h.d1))
    hits = set()
    for d1 in (1, 3, 20):
        h = Handle(name, cfg, sd64, ab, model, st)
        h.set_th(th)
        h.set_mode("apply")
        steps = [("apply", d1 + Lmax), ("runtime", 1), ("runtime", 2), ("runtime", 30), ("apply", 4), ("runtime", 3),
                 ("runtime", 40), ("off", 2), ("runtime", 1), ("runtime", 50)]
        pos = 0
        for mode, n in steps:
            if mode == "off":
                h.set_th(th, enable=False)
            else:
                h.set_th(th)
                if mode != h.mode:
                    h.set_mode(mode)
            h.call(x[:, pos * HOP:(pos + n) * HOP], n)
            pos += n
        h.report()
        hits |= h.hit
    for rc in (1, 3, 8):
        assert ("from_halo Rc", rc) in hits, [x for x in hits if x[0] == "from_halo Rc"]


@pytest.mark.parametrize("name", ["dfn3", "dfn3_ll"])
def test_slots(st, name):
    """A 4-slot handle with a linked pair (slots 1, 2; channel 0 decides): per-slot thresholds (an inverted set on slot 3,
    so its first frames are gated, then a normal one; slot 0 not gating for a while), slot 0 closed so that the later rows
    move with their tails, reopened inside a window (zero tails)."""
    cfg, sd, model, sd64, ab = built(st, name)
    h = Handle(name, cfg, sd64, ab, model, st, batch=4, reduce="mean")
    audio = synth_audio(4, 16 * 48000, seed=83)
    audio[:, 3 * 48000:5 * 48000] *= 0.01
    audio[2, 6 * 48000:9 * 48000] *= 0.01    # channel 1 of the pair would gate differently
    h.open([1, 2], linked=True)
    # thresholds from slot 0's LSNR in a first call
    h.set_th(NEVER)
    h.call(audio[:, :40 * HOP], 40)
    W0 = 0
    l = fetch(model, "lsnr", 4 * (h.d1 - W0)).reshape(4, -1)
    th = pick(l[0])
    h.set_th(th)
    h.set_th((th[1] + 5, th[1], th[2]), slots=[3])    # inverted: nothing runs
    pos = 40
    differs = False
    plan = [(3, None), (1, None), (64, "slot3 normal"), (2, "close 0"), (5, None), (1, None), (7, None), (3, "open 0"),
            (1, None), (200, "slot0 off"), (2, None), (300, "slot0 on"), (1, None), (400, None), (5, None)]
    for n, op in plan:
        if op == "slot3 normal":
            h.set_th(th, slots=[3])
        elif op == "close 0":
            h.close([0])
        elif op == "open 0":
            h.open([0])
        elif op == "slot0 off":
            h.set_th(th, enable=False, slots=[0])
        elif op == "slot0 on":
            h.set_th(ulp(th, 1), slots=[0])
        pl = h.call(audio[:, pos * HOP:(pos + n) * HOP], n)
        if pl is not None and 1 in h.rows and 2 in h.rows:
            r1, r2 = h.rows.index(1), h.rows.index(2)
            l = fetch(model, "lsnr", len(h.rows) * (pl["erb_run"].shape[1])).reshape(len(h.rows), -1)
            Rc = pl["Rc"]
            own = ~(l[r2, Rc:] < F32(th[0])) & ~(l[r2, Rc:] > F32(th[1]))
            differs |= bool((own != pl["erb_run"][r2, Rc:]).any())
            assert np.array_equal(pl["erb_run"][r1], pl["erb_run"][r2])
        pos += n
    h.report()
    assert differs
    assert {"opened", "rows moved"} <= h.hit, h.hit
    if cfg.conv_kernel[0] > 1:
        assert "erb_first inside the stream" in h.hit



def fetch_all(model, name, cap):
    """the whole named buffer (at most cap floats)"""
    out = np.empty(cap, np.float32)
    got = _lib.lib().dfb_model_debug_fetch(model.handle, name.encode(), out.ctypes.data, out.size)
    assert 0 < got < cap, (name, got, cap)
    return out[:got]


def ragged_window(model, st, x, th, chunks):
    """enhance_device_ragged of the one row x [1, S] in runtime mode, in at least `chunks` time chunks run back to back on
    one lane -> the last chunk's window: (T, lsnr [T], c0 [T][Wc], df_run [T], P [Tp][Wc])"""
    cfg = model.cfg
    Wc, K = cfg.nb_df * C, cfg.df_pathway_kernel_size_t
    model.set_chunking(chunks, 4, 1)
    try:
        enhance_device_ragged(model, st, x.cuda(), [x.shape[-1]], False, lsnr_thresholds=[th], gating_mode="runtime")
        torch.cuda.synchronize()
    finally:
        model.set_chunking()
    lsnr = fetch_all(model, "lsnr", 1 << 16)
    T = lsnr.size
    P = fetch_all(model, "gate_P", (K + T) * Wc)
    return T, lsnr, fetch(model, "c0", T * Wc).reshape(T, Wc), fetch(model, "gate_df_run", T, np.uint8) != 0, P.reshape(-1, Wc)


@pytest.mark.parametrize("name", ["dfn3", "dfn3_ll_k3"])
def test_ragged_chunk_tail(st, name):
    """A ragged batch in runtime mode, in 4 time chunks of 100 frames on one lane: the last chunk follows a DF-gated
    stretch longer than the halo, so its pathway tail is what the third chunk's decoder phase carried.  Its P rows
    [0, K - 1) equal, bit for bit, the c0 of the row's last K - 1 DF run frames, fetched from the last window of a call on
    the first 300 frames alone, in the same chunks.

    That reference is not a one-chunk call: the features, and so c0 and the LSNR, differ between chunkings in the last
    bits (over the last window of one-chunk and four-chunk calls, c0 rows one to a few ulp apart), as the chunkings'
    outputs do (test_gpu_parity.py's chunking tolerance).  Runs with the same chunk boundaries compute the same frames the
    same way; the truncated call's c0 is checked bit-identical to the full call's where their last windows overlap."""
    cfg, sd, model, sd64, ab = built(st, name)
    K = cfg.df_pathway_kernel_size_t
    x = signal(84, secs=4.0)
    cut = x[:, :300 * HOP]
    Tf, l_one, _, _, _ = ragged_window(model, st, x, NEVER, 1)
    assert Tf == 400
    # DF-gated frames [288, 300): min above their LSNR, or max_df below it, with a margin far above the chunkings' last-bit
    # differences; the flags the device used are asserted below
    gap = l_one[288:300]
    for th in ((float(gap.max()) + 1e-3, 1e9, 1e9), (-1e9, 1e9, float(gap.min()) - 1e-3)):
        runs = np.nonzero(G.plan(l_one[None], None, 0, 0, [th], [True])["df_run"][0])[0]
        if ((runs >= 200) & (runs < 280)).sum() >= K - 1 and (runs >= 300).any():
            break
    else:
        raise AssertionError("no thresholds gate the stretch before the last chunk")
    T, _, c0_last, run_last, P = ragged_window(model, st, x, th, 4)
    Tc, _, c0_cut, run_cut, _ = ragged_window(model, st, cut, th, 3)
    assert T == Tc == 108 and P.shape[0] == K - 1 + 100, (T, Tc, P.shape)   # windows [292, 400) and [192, 300)
    lb = cfg.conv_kernel_inp[0] - 1    # df_conv0's look-back: window row 0 reads zero padding for the frame before it
    assert np.array_equal(c0_last[lb:6], c0_cut[100 + lb:106]), "c0 of frames 292 + lb .. 297 differs"
    assert not run_cut[96:106].any()                        # frames 288 .. 297 gated (298, 299: by the margin)
    runs = 192 + 8 + np.nonzero(run_cut[8:106])[0]          # DF run frames among 200 .. 297 of the truncated call
    assert runs.size >= K - 1 and runs[-1] < 300 - 8, runs   # the carried rows are older than the last chunk's halo
    tail = runs[runs.size - (K - 1):] if K > 1 else runs[:0]
    assert np.array_equal(P[:K - 1], c0_cut[tail - 192]), name
    print(f"{name}: tail frames {tail.tolist()} of the last chunk from frame 300")
