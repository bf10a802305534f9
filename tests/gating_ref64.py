"""Float64 restatement of one runtime-gating window (csrc/dfb_model.cu forward_body under `if (gate)`): the gate plan
(k_gate_plan), the compacted DF pathway rows and their carried tail (k_gate_gather, k_gate_tail), the pathway conv on them
(k_df_convp_tc) and its scatter into the coefficients (k_gate_scatter), and the kt = 2 fill-forward of convt3's and the mask
head's inputs (k_gate_fill).

Conventions: arrays in the device layout, window frames t in [0, T) with the recomputed halo [0, Rc) first and the new
frames [Rc, T) after it; a row's `first` is its stream's absolute first frame (w0 + t is absolute).  Integer outputs and
copies are exact; the float results follow model_ref64's (reference, bound) convention on state64's dicts.
numpy / torch on the CPU only."""
import numpy as np
import torch

import dfnet_oracle as O
import model_ref64 as M
from dsp_ref64 import U


def plan(lsnr, first, w0, Rc, th, gate, links=None, from_halo=False, has_run_prev=None):
    """k_gate_plan of one window.  lsnr [B][T] fp32; first [B] absolute first frames or None (0); th [B][3] fp32 (min,
    max_erb, max_df); gate [B] bool; links [B] the row whose LSNR decides (a link group's channel 0) or None; has_run_prev
    [B]: the carried has_run (ignored when from_halo).  tract.rs:658-672 on the fp32 values: the ERB decoder runs iff
    !(l < min) && !(l > max_erb), the DF decoder iff that and !(l > max_df); frames before a row's first frame run
    neither; halo frames count as run.
    -> dict(erb_run, df_run [B][T] bool, erb_src, df_pos [B][T] int, df_n [B], erb_first [B] absolute, has_run [B] bool)"""
    lsnr = np.asarray(lsnr, np.float32)
    B, T = lsnr.shape
    th = np.asarray(th, np.float32).reshape(B, 3)
    erb_run = np.zeros((B, T), bool)
    df_run = np.zeros((B, T), bool)
    erb_src = np.full((B, T), -1, np.int64)
    df_pos = np.zeros((B, T), np.int64)
    df_n = np.zeros(B, np.int64)
    erb_first = np.zeros(B, np.int64)
    has_run = np.zeros(B, bool)
    for b in range(B):
        f0 = 0 if first is None else int(first[b])
        tf = max(f0 - w0, 0)
        l = lsnr[b if links is None else int(links[b])]
        erb_run[b, :Rc] = df_run[b, :Rc] = True
        erb_src[b, :Rc] = np.arange(Rc)
        for t in range(Rc, T):
            e = t >= tf
            d = e
            if e and gate[b]:
                e = not (l[t] < th[b, 0]) and not (l[t] > th[b, 1])
                d = e and not (l[t] > th[b, 2])
            erb_run[b, t], df_run[b, t] = e, d
        last, n = -1, 0
        for t in range(Rc, T):
            if erb_run[b, t]:
                last = t
            erb_src[b, t] = last
            df_pos[b, t] = n
            n += int(df_run[b, t])
        df_n[b] = n
        runs = np.nonzero(erb_run[b, Rc:])[0]
        s_first = Rc + int(runs[0]) if runs.size else T
        prev = (Rc > 0 and w0 + Rc - 1 >= f0) if from_halo else has_run_prev is not None and bool(has_run_prev[b])
        erb_first[b] = f0 if prev else w0 + s_first
        has_run[b] = prev or s_first < T
    return dict(erb_run=erb_run, df_run=df_run, erb_src=erb_src, df_pos=df_pos, df_n=df_n, erb_first=erb_first, has_run=has_run)


class Tails:
    """What a streaming row carries from window to window in runtime mode, advanced call by call by the test: c0 of the DF
    decoder's last K - 1 run frames and (kt = 2) dec_emb / e3 / d1 / e0 at the ERB decoder's last run frame, with has_run.
    A fresh row (a new stream, a reopened slot) carries zeros; a row moved by slot compaction keeps its object."""

    def __init__(self, K, Wc, run_widths=()):
        self.c0 = np.zeros((K - 1, Wc), np.float32)
        self.run = [np.zeros(w, np.float32) for w in run_widths]
        self.has_run = False


def halo_tail(c0, Rc, K, tf):
    """The pathway tail of a window after an apply-mode or non-gating call, where every earlier frame ran: c0 rows
    Rc - (K - 1) .. Rc - 1 of this window (c0 [T][Wc]), zero before frame 0 or the stream's first window frame tf."""
    out = np.zeros((K - 1, c0.shape[-1]), np.float32)
    for x in range(K - 1):
        t = Rc - (K - 1) + x
        if t >= 0 and t >= tf:
            out[x] = c0[t]
    return out


def compact(c0, tail, pl, b, Rc):
    """Expected rows [0, K - 1 + df_n) of P for row b: the tail [K - 1][Wc], then c0 [T][Wc] of the DF run frames among the
    new ones, in order.  Exact copies."""
    idx = [t for t in range(Rc, c0.shape[0]) if pl["df_run"][b, t]]
    return np.concatenate([tail, c0[idx]], 0) if idx else tail.copy()


def next_c0_tail(P_rows, K):
    """The carried tail after the window: the last K - 1 compacted rows (k_gate_tail)."""
    return P_rows[P_rows.shape[0] - (K - 1):].copy() if K > 1 else P_rows[:0].copy()


def pathway_q(sd64, ab, P, Fd, C, order):
    """relu(df_convp) on the compacted rows P [Tp][Fd * C] (device layout), as k_df_convp_tc computes it on them with
    the carried rows as its look-back -> (Q [Tp][Fd][2 order], bound), valid from row K - 1 on (earlier rows read zero
    padding); BF16x3 as model_ref64.coefs' pathway term."""
    if len(P) == 0:   # a one-tap conv after a window without DF run frames
        return np.zeros((0, Fd, 2 * order)), np.zeros((0, Fd, 2 * order))
    x = M.channel_last(np.asarray(P, np.float32).reshape(1, -1, Fd, C))
    q = O.conv_norm_act(x, sd64, "df_dec.df_convp").permute(0, 2, 3, 1)[0]
    chain = O.conv_norm_act(x.abs(), ab, "df_dec.df_convp", act="none").permute(0, 2, 3, 1)[0]
    return q.numpy(), M.bf16x3_bound(chain).numpy()


def coefs(sd64, ab, cfg, dfc, q, b_q, df_run, df_pos, K):
    """Coefficients of one row's new frames: tanh(df_out(dfc)) (dfc [n][Hd]) plus, at DF run frames, the pathway row
    Q[K - 1 + df_pos] (q / b_q from pathway_q), and nothing elsewhere; model_ref64.coefs' bound."""
    dfc = torch.as_tensor(np.asarray(dfc, np.float64))[None]
    n = dfc.shape[1]
    shape = (n, cfg.nb_df, 2 * cfg.df_order)
    lin = O.grouped_linear(dfc, sd64["df_dec.df_out.0.weight"]).view(shape).numpy()
    lin_chain = O.grouped_linear(dfc.abs(), ab["df_dec.df_out.0.weight"]).view(shape).numpy()
    t = np.tanh(lin)
    p = np.zeros(shape)
    bp = np.zeros(shape)
    for i in range(n):
        if df_run[i]:
            p[i], bp[i] = q[K - 1 + df_pos[i]], b_q[K - 1 + df_pos[i]]
    ref = t + p
    return ref, M.bf16x3_bound(lin_chain) + 2 * U * np.abs(t) + bp + U * np.abs(ref)


def filled(x, pl, b, Rc, carried, from_halo):
    """Expected rows [Rc - 1, T) (from row 0 when Rc = 0) of one kt = 2 input x [T][W] of row b after k_gate_fill: a new
    frame the ERB decoder did not run on takes the row of its last run frame (erb_src), or the carried row before any;
    after an apply-mode call the carried row is the recomputed halo row Rc - 1 (zeros when Rc = 0).  Row Rc - 1 itself
    becomes the carried row, unless from_halo.  Exact copies."""
    x = np.asarray(x)
    out = x.copy()
    if Rc > 0 and not from_halo:
        out[Rc - 1] = carried
    for t in range(Rc, x.shape[0]):
        if pl["erb_run"][b, t]:
            continue
        j = pl["erb_src"][b, t]
        if j >= 0:
            out[t] = x[j]
        elif from_halo:
            out[t] = x[Rc - 1] if Rc > 0 else 0
        else:
            out[t] = carried
    return out[max(Rc - 1, 0):]


def _from(x, s):
    """x [B,C,T,F] from frame s on (frames before s are padding to the causal convs)"""
    return x[:, :, s:]


def convt3(sd64, ab, dec_emb, e3, s):
    """d3 = convt3(dec_emb + relu(conv3p(e3))) (model_ref64.block) on frames [s, T) of the filled inputs, frames before s
    (erb_first, or the window's first needed row) zero -> (ref, bound) over frames [s, T)."""
    return M.block(sd64, ab, "erb_dec.convt3", _from(dec_emb, s), path=("erb_dec.conv3p", _from(e3, s)))


def mask(sd64, ab, e0, d1, s):
    """m = mask head(e0, d1) (model_ref64.mask_head) on frames [s, T), frames before s zero -> (ref, bound) over [s, T)."""
    return M.mask_head(sd64, ab, _from(e0, s), _from(d1, s))
