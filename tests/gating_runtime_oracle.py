"""CPU restatement of the runtime gating mode (include/dfb200.h, dfb_gating_mode DFB_GATING_RUNTIME) on the oracle's
building blocks: the Rust runtime's decoders run only on the frames LSNR stage gating lets through (tract.rs:478-503),
each as tract's pulsed erb_dec / df_dec graphs do, from zero states over the subsequence of its own frames.

* the encoder runs over all frames (so the LSNR is the one of apply mode);
* per stream, the ERB decoder runs on the frames with min <= lsnr <= max_erb, the DF decoder on those that also have
  lsnr <= max_df (tract.rs:658-672 apply_stages), lsnr from the link group's first channel;
* their outputs go back to those frames (zeros elsewhere: no stage applies them), and the stage rule
  (linked_oracle.apply_stages) picks what each frame gets.

With thresholds that never gate this is linked_oracle.enhance; a stream with every frame gated runs no decoder at all.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

import dfnet_oracle as O
import linked_oracle as LO


def run_flags(lsnr: Tensor, th) -> tuple:
    """(erb_run, df_run) bool [T] of one stream from its deciding LSNR [T] and th = (min, max_erb, max_df), with the
    apply kernel's comparisons; th None: every frame runs."""
    if th is None:
        ones = torch.ones(lsnr.shape[0], dtype=torch.bool)
        return ones, ones.clone()
    lo, erb, df = th
    e = ~(lsnr < lo) & ~(lsnr > erb)
    return e, e & ~(lsnr > df)


def decoders(sd, cfg: dict, e0, e1, e2, e3, emb, c0, erb_run: Sequence[Tensor], df_run: Sequence[Tensor]):
    """erb_decoder / df_decoder of each stream b alone on its run frames, scattered back: (m [B,1,T,E], coefs [B,T,Fd,O2])."""
    b, t = emb.shape[0], emb.shape[1]
    m = torch.zeros(b, 1, t, cfg["nb_erb"])
    coefs = torch.zeros(b, t, cfg["nb_df"], 2 * cfg["df_order"])
    for i in range(b):
        ie = torch.nonzero(erb_run[i]).view(-1)
        if ie.numel():
            m[i, :, ie] = O.erb_decoder(sd, cfg, emb[i:i + 1, ie], e3[i:i + 1, :, ie], e2[i:i + 1, :, ie], e1[i:i + 1, :, ie],
                                        e0[i:i + 1, :, ie])[0]
        idf = torch.nonzero(df_run[i]).view(-1)
        if idf.numel():
            coefs[i, idf] = O.df_decoder(sd, cfg, emb[i:i + 1, idf], c0[i:i + 1, :, idf])[0]
    return m, coefs


def dfnet_forward(sd, cfg: dict, erb_widths, spec: Tensor, feat_erb: Tensor, feat_spec: Tensor, ths: Sequence,
                  reduce: Optional[str] = None, channels: int = 1, flags_of=None):
    """linked_oracle.dfnet_forward with the decoders run as above; ths[b]: the thresholds of stream b (its group's) or
    None.  flags_of (optional): (b, lsnr [T], th) -> (erb_run, df_run), in place of run_flags.
    -> (spec_e before the stage rule, m, lsnr, coefs, m_linked, erb_run, df_run)"""
    fs = feat_spec.squeeze(1).permute(0, 3, 1, 2)
    lc = cfg["conv_lookahead"]
    fe = feat_erb
    if lc > 0:
        fe = F.pad(fe, (0, 0, -lc, lc))
        fs = F.pad(fs, (0, 0, -lc, lc))
    e0, e1, e2, e3, emb, c0, lsnr = O.encoder(sd, cfg, fe, fs)
    b = emb.shape[0]
    erb_run, df_run = [], []
    for i in range(b):
        l0 = lsnr[i - i % channels, :, 0]
        e, d = flags_of(i, l0, ths[i]) if flags_of is not None else run_flags(l0, ths[i])
        erb_run.append(e); df_run.append(d)
    m, coefs = decoders(sd, cfg, e0, e1, e2, e3, emb, c0, erb_run, df_run)
    m_link = LO.reduce_mask(m, channels, reduce)
    inv = O.erb_inv_matrix(erb_widths)
    spec_m = O.apply_mask(spec, m_link, inv)
    nb_df, order, la = cfg["nb_df"], cfg["df_order"], cfg["df_lookahead"]
    if cfg["model"] == "deepfilternet2":
        spec_e = spec_m if cfg.get("mask_only", False) else O.deep_filter(spec_m, coefs, nb_df, order, la)
    elif cfg.get("mask_only", False):
        spec_e = spec_m
    else:
        spec_e = O.deep_filter(spec, coefs, nb_df, order, la)
        spec_e[..., nb_df:, :] = spec_m[..., nb_df:, :]
    return spec_e, m, lsnr, coefs, m_link, erb_run, df_run


def features(cfg: dict, audio: Tensor, pad: bool):
    """(libdf state, spec [B,1,T,F,2], erb_feat, spec_feat, erb widths) of dfnet_oracle.enhance."""
    import libdf_oracle as libdf
    n_fft, hop = cfg["fft_size"], cfg["hop_size"]
    st = libdf.DF(cfg["sr"], n_fft, hop, cfg["nb_erb"], cfg.get("min_nb_erb_freqs", 2))
    if pad:
        audio = F.pad(audio, (0, n_fft))
    a = O.norm_alpha(cfg["sr"], hop, cfg.get("norm_tau", 1.0))
    spec = st.analysis(np.ascontiguousarray(audio.numpy()))
    widths = st.erb_widths()
    erb_feat = torch.as_tensor(libdf.erb_norm(libdf.erb(spec, widths), a)).unsqueeze(1)
    spec_feat = torch.view_as_real(torch.as_tensor(libdf.unit_norm(np.ascontiguousarray(spec[..., :cfg["nb_df"]]), a))).unsqueeze(1)
    spec_t = torch.view_as_real(torch.as_tensor(spec)).unsqueeze(1)
    return st, spec_t, erb_feat, spec_feat, widths


@torch.no_grad()
def enhance(sd, cfg: dict, audio: Tensor, pad: bool = True, stages=None, reduce: Optional[str] = None,
            channels: Optional[int] = None, flags_of=None, return_all: bool = False):
    """linked_oracle.enhance in the runtime gating mode: audio [B,T], rows g * channels + c are recording g; stages: one
    (min, max_erb, max_df) for every row, one per row (None: that row does not gate), or None (no gating)."""
    b = audio.shape[0]
    if channels is None:
        channels = b
    ths = list(stages) if stages is not None and not _is_th(stages) else [stages] * b
    st, spec_t, erb_feat, spec_feat, widths = features(cfg, audio, pad)
    spec_e, m, lsnr, coefs, m_link, erb_run, df_run = dfnet_forward(sd, cfg, widths, spec_t.clone(), erb_feat, spec_feat, ths,
                                                                    reduce, channels, flags_of)
    out_spec = spec_e.clone()
    for i in range(b):
        if ths[i] is not None:
            lo, erb, df = ths[i]
            g0 = i - i % channels
            out_spec[i:i + 1] = LO.apply_stages(spec_t[g0:g0 + channels], spec_e[g0:g0 + channels], m_link[g0:g0 + channels],
                                                lsnr[g0:g0 + channels], widths, channels, lo, erb, df)[i - g0:i - g0 + 1]
    enh = torch.view_as_complex(out_spec.squeeze(1).contiguous())
    out = torch.as_tensor(st.synthesis(np.ascontiguousarray(enh.numpy())))
    if pad:
        d = cfg["fft_size"] - cfg["hop_size"]
        out = out[:, d:audio.shape[-1] + d]
    if return_all:
        return out, dict(m=m, m_link=m_link, lsnr=lsnr, coefs=coefs, erb_run=erb_run, df_run=df_run)
    return out


def _is_th(v) -> bool:
    return isinstance(v, (tuple, list)) and len(v) == 3 and all(isinstance(x, (int, float)) for x in v)


def gated_runs(run: Tensor) -> list:
    """Lengths of the maximal runs of frames where `run` is False."""
    out, n = [], 0
    for v in run.tolist():
        if not v:
            n += 1
        elif n:
            out.append(n); n = 0
    if n:
        out.append(n)
    return out
