"""CPU restatement of linked channels (include/dfb200.h, dfb_enhance_ragged's link groups) on top of the oracle's building blocks
(oracle/dfnet_oracle.py, which itself stays the plain reference forward pass).

The channels of one recording run through the network as a batch, each with its own features, states and outputs; the
ERB decoder's mask is then reduced over the channels of each link group (the Rust runtime's ReduceMask,
libDF/src/tract.rs:95-99, 868-902) and every channel applies the shared mask where it applies its own:

  max:  m[t,e] = max_c m_c[t,e]
  mean: m[t,e] = (sum_c m_c[t,e], fp32 in channel order) * fl32(1 / C)

`dfnet_forward` / `enhance` below are dfnet_oracle's with that reduction between erb_decoder and the masked spectrum; with
reduce None / "none" they compute exactly what dfnet_oracle computes.  `apply_stages` restates the streaming runtime's
LSNR stage gating (tract.rs:658-672) with one decision per link group and frame, taken from the group's first channel.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

import dfnet_oracle as O


def reduce_mask(m: Tensor, channels: int, reduce: Optional[str]) -> Tensor:
    """m [B,1,T,E] with B = groups * channels -> every row replaced by its group's max / mean (None / "none": m itself)."""
    if reduce in (None, "none") or channels == 1:
        return m
    b = m.shape[0]
    if b % channels:
        raise ValueError(f"{b} streams are not groups of {channels} channels")
    g = m.reshape(b // channels, channels, *m.shape[1:])
    if reduce == "max":
        r = g[:, 0]
        for c in range(1, channels):
            r = torch.maximum(r, g[:, c])
    elif reduce == "mean":
        r = g[:, 0].clone()
        for c in range(1, channels):   # fp32 sum in channel order, then times fl32(1 / C) (tract.rs:881-898)
            r = r + g[:, c]
        r = r * torch.tensor(np.float32(1.0) / np.float32(channels), dtype=torch.float32)
    else:
        raise ValueError(f"reduce must be None, 'none', 'max' or 'mean', got {reduce!r}")
    return r.repeat_interleave(channels, dim=0)


@torch.no_grad()
def dfnet_forward(sd, cfg: dict, erb_widths, spec: Tensor, feat_erb: Tensor, feat_spec: Tensor,
                  reduce: Optional[str] = None, channels: int = 1):
    """dfnet_oracle.dfnet_forward with linked channels: rows g * channels + c of the batch are recording g.
    -> (spec_e, m (per channel, as the model outputs it), lsnr, coefs, m_linked)"""
    fs = feat_spec.squeeze(1).permute(0, 3, 1, 2)
    lc = cfg["conv_lookahead"]
    fe = feat_erb
    if lc > 0:
        fe = F.pad(fe, (0, 0, -lc, lc))
        fs = F.pad(fs, (0, 0, -lc, lc))
    e0, e1, e2, e3, emb, c0, lsnr = O.encoder(sd, cfg, fe, fs)
    m = O.erb_decoder(sd, cfg, emb, e3, e2, e1, e0)
    m_link = reduce_mask(m, channels, reduce)        # the only step that sees more than one channel
    inv = O.erb_inv_matrix(erb_widths)
    pf, mask_only = bool(cfg.get("mask_pf", False)), bool(cfg.get("mask_only", False))
    m_app = m_link
    if pf and cfg["model"] == "deepfilternet2":   # Mask.pf acts on the shared mask
        beta = 0.02
        m_sin = m_link * torch.sin(math.pi * m_link / 2)
        m_app = (1 + beta) * m_link / (1 + beta * m_link.div(m_sin.clamp_min(1e-12)).pow(2))
    spec_m = O.apply_mask(spec, m_app, inv)
    coefs = O.df_decoder(sd, cfg, emb, c0)
    nb_df, order, la = cfg["nb_df"], cfg["df_order"], cfg["df_lookahead"]
    if cfg["model"] == "deepfilternet2":
        spec_e = spec_m if mask_only else O.deep_filter(spec_m, coefs, nb_df, order, la)
    else:
        if mask_only:
            spec_e = spec_m
        else:
            spec_e = O.deep_filter(spec, coefs, nb_df, order, la)
            spec_e[..., nb_df:, :] = spec_m[..., nb_df:, :]
        if pf:   # per channel: a ratio of the channel's own spectra
            beta, eps = float(cfg.get("pf_beta", 0.02)), 1e-12
            mask = (torch.view_as_complex(spec_e.contiguous()).abs() / torch.view_as_complex(spec.contiguous()).abs().add(eps)).clamp(eps, 1)
            mask_sin = mask * torch.sin(math.pi * mask / 2).clamp_min(eps)
            g = (1 + beta) / (1 + beta * mask.div(mask_sin).pow(2))
            spec_e = spec_e * g.unsqueeze(-1)
    return spec_e, m, lsnr, coefs, m_link


def apply_stages(spec: Tensor, spec_e: Tensor, m_link: Tensor, lsnr: Tensor, erb_widths, channels: int,
                 min_db_thresh: float, max_db_erb_thresh: float, max_db_df_thresh: float) -> Tensor:
    """tract.rs:658-672 per frame, one decision per link group from its FIRST channel's LSNR (DeepFilterNet3, no post
    filter): lsnr < min -> zeros; > max_erb -> the noisy frame; > max_df -> ERB gains on every bin; else spec_e.
    spec / spec_e [B,1,T,F,2], m_link [B,1,T,E], lsnr [B,T,1]."""
    b = spec.shape[0]
    l0 = lsnr[::channels, :, 0].repeat_interleave(channels, dim=0)          # [B,T]
    gains = O.apply_mask(spec, m_link, O.erb_inv_matrix(erb_widths))
    out = spec_e.clone()
    sel = lambda mask: mask.view(b, 1, -1, 1, 1)  # noqa: E731
    out = torch.where(sel(l0 > max_db_df_thresh), gains, out)
    out = torch.where(sel(l0 > max_db_erb_thresh), spec, out)
    out = torch.where(sel(l0 < min_db_thresh), torch.zeros_like(out), out)
    return out


@torch.no_grad()
def enhance(sd, cfg: dict, audio: Tensor, pad: bool = True, atten_lim_db: Optional[float] = None,
            reduce: Optional[str] = None, channels: Optional[int] = None, stages: Optional[dict] = None,
            return_all: bool = False):
    """dfnet_oracle.enhance with linked channels: audio [B,T], rows g * channels + c are recording g (channels defaults to
    all B rows: one recording).  ``stages``: {min_db_thresh, max_db_erb_thresh, max_db_df_thresh} gates every frame as
    `apply_stages` does."""
    import libdf_oracle as libdf
    if channels is None:
        channels = audio.shape[0]
    n_fft, hop = cfg["fft_size"], cfg["hop_size"]
    st = libdf.DF(cfg["sr"], n_fft, hop, cfg["nb_erb"], cfg.get("min_nb_erb_freqs", 2))
    orig_len = audio.shape[-1]
    if pad:
        audio = F.pad(audio, (0, n_fft))
    a = O.norm_alpha(cfg["sr"], hop, cfg.get("norm_tau", 1.0))
    spec = st.analysis(np.ascontiguousarray(audio.numpy()))
    widths = st.erb_widths()
    erb_feat = torch.as_tensor(libdf.erb_norm(libdf.erb(spec, widths), a)).unsqueeze(1)
    spec_feat = torch.view_as_real(
        torch.as_tensor(libdf.unit_norm(np.ascontiguousarray(spec[..., :cfg["nb_df"]]), a))
    ).unsqueeze(1)
    spec_t = torch.view_as_real(torch.as_tensor(spec)).unsqueeze(1)
    spec_e, m, lsnr, coefs, m_link = dfnet_forward(sd, cfg, widths, spec_t.clone(), erb_feat, spec_feat, reduce, channels)
    if stages is not None:
        spec_e = apply_stages(spec_t, spec_e, m_link, lsnr, widths, channels, **stages)
    enh = torch.view_as_complex(spec_e.squeeze(1).contiguous())
    if atten_lim_db is not None and abs(atten_lim_db) > 0:
        lim = 10 ** (-abs(atten_lim_db) / 20)
        enh = torch.as_tensor(spec) * lim + enh * (1 - lim)
    out = torch.as_tensor(st.synthesis(np.ascontiguousarray(enh.numpy())))
    if pad:
        d = n_fft - hop
        out = out[:, d:orig_len + d]
    if return_all:
        return out, dict(m=m, m_link=m_link, lsnr=lsnr, coefs=coefs)
    return out
