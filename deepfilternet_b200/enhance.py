"""Drop-in for ``df.enhance`` (DeepFilterNet/df/enhance.py): ``init_df``, ``df_features``,
``enhance`` with the reference's signatures, argument meaning and return types.  The whole
``enhance()`` path (pad -> STFT -> features -> DNN -> mask + deep filter -> ISTFT -> crop) is ONE
C-ABI call (``dfb_enhance_host``) into the CUDA library; nothing is computed on the CPU.
"""
from __future__ import annotations

import logging
import os
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib, ragged
from ._lib import check
from .io import load_audio, resample, save_audio
from .libdf import DF
from .model import DfNet, load_model

logger = logging.getLogger("deepfilternet_b200")

PRETRAINED_MODELS = ("DeepFilterNet", "DeepFilterNet2", "DeepFilterNet3")
DEFAULT_MODEL = "DeepFilterNet3"
_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model_search_dirs():
    d = []
    if os.environ.get("DFB_MODEL_DIR"):
        d.append(os.environ["DFB_MODEL_DIR"])
    d.append(os.path.join(_REPO, "models", "_ref"))
    return d


def get_model_basedir(m: Optional[str]) -> str:
    """enhance.py:92-98.  The reference downloads the default models; there is no network here, so
    pretrained names resolve to a local directory ($DFB_MODEL_DIR/<name> or models/_ref/<name>)."""
    if m is None:
        m = DEFAULT_MODEL
    if os.path.isdir(m):
        return m
    for base in model_search_dirs():
        cand = os.path.join(base, m)
        if os.path.isdir(cand):
            return cand
    return m


def init_df(
    model_base_dir: Optional[str] = None,
    post_filter: bool = False,
    log_level: str = "INFO",
    log_file: Optional[str] = "enhance.log",
    config_allow_defaults: bool = True,
    epoch: Union[str, int, None] = "best",
    default_model: str = DEFAULT_MODEL,
    mask_only: bool = False,
    device: int = 0,
) -> Tuple[DfNet, DF, str, int]:
    """enhance.py:101-187 -> (model, df_state, suffix, epoch)."""
    model_base_dir = get_model_basedir(model_base_dir or default_model)
    if not os.path.isdir(model_base_dir):
        raise NotADirectoryError("Base directory not found at {}".format(model_base_dir))
    logger.setLevel(getattr(logging, str(log_level).upper(), logging.INFO))
    if epoch is None or (isinstance(epoch, str) and epoch.lower() == "none"):
        raise NotImplementedError("epoch='none' (random weights): use weights.random_state_dict + DfNet")
    model, df_state, ep = load_model(model_base_dir, epoch=epoch, device=device, post_filter=post_filter, mask_only=mask_only)
    suffix = os.path.basename(os.path.abspath(model_base_dir))
    if post_filter:
        suffix += "_pf"   # enhance.py:183-184
    logger.info("Running on device cuda:%d", device)
    logger.info("Model loaded")
    return model, df_state, suffix, ep


def df_features(audio: Tensor, df: DF, nb_df: int, device=None, alpha: Optional[float] = None
                ) -> Tuple[Tensor, Tensor, Tensor]:
    """enhance.py:190-203: audio f32 CPU [C,T] -> (spec [C,1,Tf,F,2], erb_feat [C,1,Tf,E],
    spec_feat [C,1,Tf,nb_df,2]); one fused device pass.  ``alpha`` defaults to the reference's
    ``get_norm_alpha()`` (df/utils.py:108-124) of the config the DF state was loaded with (``init_df`` /
    ``load_model`` stash it on the DF object), else to the value for norm_tau = 1."""
    if alpha is None:
        alpha = getattr(df, "norm_alpha", None)
    if alpha is None:
        from .config import ModelConfig
        alpha = ModelConfig(sr=df.sr(), hop_size=df.hop_size()).norm_alpha
    x = np.ascontiguousarray(audio.detach().cpu().numpy(), dtype=np.float32)
    if x.ndim != 2 or x.size == 0:
        raise RuntimeError("[df] Input array empty or not contiguous.")
    c, t = x.shape
    tf, f, e = t // df.hop_size(), df.fft_size() // 2 + 1, df.nb_erb()
    spec = np.empty((c, 1, tf, f, 2), dtype=np.float32)
    erb_feat = np.empty((c, 1, tf, e), dtype=np.float32)
    spec_feat = np.empty((c, 1, tf, nb_df, 2), dtype=np.float32)
    check(_lib.lib().dfb_features_host(df.handle, x.ctypes.data, c, t, int(nb_df), float(alpha),
                                       spec.ctypes.data, erb_feat.ctypes.data, spec_feat.ctypes.data))
    out = tuple(torch.from_numpy(a) for a in (spec, erb_feat, spec_feat))
    if device is not None:
        out = tuple(a.to(device) for a in out)
    return out


def _rated(model: DfNet, sr, n: int):
    """The batch calls' ``sr``: None when every entry is at 48 kHz, else the rates as int32, each registered on the model."""
    rates = ragged.rates_arg(sr, n)
    if rates is not None:
        for r in sorted(set(rates.tolist())):
            model.add_rate(r)
    return rates


def _settings(model: DfNet, n: int, atten_lim_db, post_filter_beta, lsnr_thresholds, return_lsnr: bool):
    """The batch calls' per-entry settings as a dfb_enhance_settings table (ragged.settings_table), or None when the call
    needs none; the combinations the library refuses are refused here first (DfbError, DFB_ERR_UNSUPPORTED)."""
    c = model.cfg
    default_beta = model.post_filter_beta if (c.model == "deepfilternet3" and model.post_filter) else 0.0
    tab = ragged.settings_table(n, atten_lim_db, post_filter_beta, lsnr_thresholds, default_beta)
    ragged.check_settings_model(c.model, c.nb_erb, c.nb_df, c.df_order, tab, return_lsnr)
    return tab


def _ptr(a):
    """The address of a numpy array or tensor for the library, or None (a null pointer) for None."""
    return None if a is None else a.data_ptr() if isinstance(a, Tensor) else a.ctypes.data


@torch.no_grad()
def enhance(model: DfNet, df_state: DF, audio: Tensor, pad: bool = True,
            atten_lim_db: Optional[float] = None, out: Optional[Tensor] = None, *, reduce_mask: Optional[str] = None,
            sr: Optional[int] = None, post_filter_beta: Optional[float] = None, lsnr_thresholds=None,
            return_lsnr: bool = False, gating_mode: Optional[str] = None):
    """enhance.py:206-250: audio f32 CPU [C,T] @ model sr -> enhanced f32 CPU [C,T]
    (or [C, (T // hop) * hop], delayed by n_fft - hop, when ``pad`` is False).
    ``out`` (extension): optional preallocated (e.g. pinned) CPU tensor for the result.
    ``reduce_mask`` (extension): "max" or "mean" links the C channels as the Rust runtime does (tract.rs:868-902): they
    share one ERB mask, the max or mean of their own (include/dfb200.h, dfb_enhance_ragged); None / "none": every
    channel on its own.
    ``sr`` (extension): the rate of ``audio`` when it is not the model's 48 kHz, as :func:`enhance_batch` takes it.
    ``post_filter_beta`` / ``lsnr_thresholds`` / ``return_lsnr`` (extensions): one value each, as :func:`enhance_batch`
    takes them; with ``return_lsnr`` the result is ``(enhanced, lsnr)``.  ``gating_mode`` as :func:`enhance_batch` takes it."""
    model.eval()
    if gating_mode is not None:
        ragged.gating_mode_code(gating_mode)
    if audio.dim() != 2:
        raise ValueError("audio must have shape [C, T]")
    if isinstance(atten_lim_db, (list, tuple, np.ndarray, Tensor)):
        raise ValueError("enhance() takes one attenuation limit: use enhance_batch for one per entry")
    if (_rated(model, sr, 1) is not None or post_filter_beta is not None or lsnr_thresholds is not None or return_lsnr):
        if post_filter_beta is not None and not ragged._is_number(post_filter_beta):
            raise ValueError("enhance() takes one post-filter beta: use enhance_batch for one per entry")
        if lsnr_thresholds is not None:
            lsnr_thresholds = ragged._thresholds(lsnr_thresholds, "lsnr_thresholds")
        r = enhance_batch(model, df_state, [audio], pad, atten_lim_db, reduce_mask, sr=None if sr is None else [sr],
                          post_filter_beta=post_filter_beta, lsnr_thresholds=lsnr_thresholds, return_lsnr=return_lsnr,
                          gating_mode=gating_mode)
        y = (r[0] if return_lsnr else r)[0]
        if out is not None:
            if out.shape != y.shape or out.dtype != torch.float32 or out.is_cuda or not out.is_contiguous():
                raise ValueError(f"out must be a contiguous float32 CPU tensor of shape {tuple(y.shape)}")
            y = out.copy_(y)
        return (y, r[1][0]) if return_lsnr else y
    x = audio.detach().to("cpu", torch.float32).contiguous()
    c, t = x.shape
    out_len = int(_lib.lib().dfb_enhance_out_len(df_state.handle, t, 1 if pad else 0))
    if out is None:
        out = torch.empty((c, out_len), dtype=torch.float32)
    elif out.shape != (c, out_len) or out.dtype != torch.float32 or out.is_cuda or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float32 CPU tensor of shape {(c, out_len)}")
    lim = abs(float(atten_lim_db)) if atten_lim_db is not None else 0.0
    reduce = ragged.reduce_code(reduce_mask)
    if reduce == 0:
        check(_lib.lib().dfb_enhance_host(model.handle, df_state.handle, x.data_ptr(), c, t, 1 if pad else 0,
                                          lim, out.data_ptr()))
        return out
    lens = np.full(c, t, dtype=np.int64)
    in_off, out_off = np.arange(c, dtype=np.int64) * t, np.arange(c, dtype=np.int64) * out_len
    groups = np.array([c], dtype=np.int64)
    check(_lib.lib().dfb_enhance_ragged_host(model.handle, df_state.handle, x.data_ptr(), c * t, in_off.ctypes.data,
                                             lens.ctypes.data, c, 1 if pad else 0, lim, out.data_ptr(), c * out_len,
                                             out_off.ctypes.data, groups.ctypes.data, 1, reduce, None, None, 0, None, 0, None))
    return out


@torch.no_grad()
def enhance_device(model: DfNet, df_state: DF, audio: Tensor, pad: bool = True,
                   atten_lim_db: Optional[float] = None, out: Optional[Tensor] = None) -> Tensor:
    """Device-resident variant of :func:`enhance`: ``audio`` is a CUDA tensor [B,T] on the model's
    device and the result stays there (asynchronous on the current stream)."""
    if not audio.is_cuda or audio.dtype != torch.float32 or not audio.is_contiguous() or audio.dim() != 2:
        raise ValueError("enhance_device expects a contiguous float32 CUDA tensor of shape [B, T]")
    if audio.device != model.cuda_device:
        raise ValueError(f"audio lives on {audio.device}, the model on {model.cuda_device}")
    b, t = audio.shape
    out_len = int(_lib.lib().dfb_enhance_out_len(df_state.handle, t, 1 if pad else 0))
    if out is None:
        out = torch.empty((b, out_len), dtype=torch.float32, device=audio.device)
    elif (out.shape != (b, out_len) or out.dtype != torch.float32 or not out.is_cuda or out.device != audio.device
          or not out.is_contiguous()):
        raise ValueError(f"out must be a contiguous float32 CUDA tensor of shape {(b, out_len)} on {audio.device}")
    lim = abs(float(atten_lim_db)) if atten_lim_db is not None else 0.0
    with torch.cuda.device(audio.device):
        stream = torch.cuda.current_stream(audio.device).cuda_stream
        check(_lib.lib().dfb_enhance(model.handle, df_state.handle, audio.data_ptr(), b, t, 1 if pad else 0,
                                     lim, out.data_ptr(), stream))
    return out


@torch.no_grad()
def enhance_batch(model: DfNet, df_state: DF, audios: Sequence[Tensor], pad: bool = True,
                  atten_lim_db=None, reduce_mask: Optional[str] = None, *, sr=None, post_filter_beta=None,
                  lsnr_thresholds=None, return_lsnr: bool = False, gating_mode: Optional[str] = None):
    """Several recordings of different lengths in one call: ``audios`` is a sequence of CPU [C_i, T_i] tensors as
    :func:`enhance` takes them, every channel one stream.  Entry i of the result equals
    ``enhance(model, df_state, audios[i], pad, atten_lim_db)``.  The batch is packed into one page-locked buffer and
    enhanced by one ``dfb_enhance_ragged_host`` call, which copies only the streams' own samples and computes only their
    own frames.  The results are views into one page-locked output buffer.  ``reduce_mask`` "max" / "mean": each entry's
    channels are linked, as ``enhance(..., reduce_mask=reduce_mask)`` links them.
    ``sr``: the entries' sample rate, one for all or one per entry (None: 48 kHz).  Entry i at rate r is then
    ``io.resample(enhance(model, df_state, io.resample(audios[i], r, 48000), ...), 48000, r)``, with both resamplers run
    on the device per time chunk so that only rate-r samples cross PCIe (any rate whose
    sinc_fast taps hold at most 2^18 floats, e.g. 8, 11.025, 16, 22.05, 44.1, 96 kHz).
    Per-entry settings: ``atten_lim_db`` one value or one per entry; ``post_filter_beta`` None
    (the model's DeepFilterNet3 post filter), one value or one per entry, 0 = off (DeepFilterNet3 topologies); and
    ``lsnr_thresholds`` None (no gating), one (min_db_thresh, max_db_erb_thresh, max_db_df_thresh) or one per entry (None:
    that entry does not gate) -- the Rust runtime's LSNR stage gating (DeepFilterNet3 topologies).  Entry i then equals
    the batch with entry i's settings given to every entry.  ``return_lsnr``: the result is ``(outputs, lsnrs)``, lsnrs[i]
    float32 [n_i] (a multi-channel entry [C_i, n_i]) with value j the LSNR in dB of the frame 10 ms output hop j carries
    (include/dfb200.h, dfb_enhance_ragged).
    ``gating_mode`` None (the model's, :meth:`DfNet.set_gating_mode`), "apply" or "runtime": with "runtime" a gating
    entry's decoders run only on the frames its stages let through, as the Rust runtime's do (include/dfb200.h,
    dfb_gating_mode); entries that do not gate are computed as in "apply"."""
    model.eval()
    if gating_mode is not None:
        ragged.gating_mode_code(gating_mode)
    xs = list(audios)
    for i, a in enumerate(xs):
        if not isinstance(a, Tensor) or a.dim() != 2:
            raise ValueError(f"entry {i}: audio must be a tensor of shape [C, T]")
    rates = _rated(model, sr, len(xs))
    tab = _settings(model, len(xs), atten_lim_db, post_filter_beta, lsnr_thresholds, return_lsnr)
    shapes = [tuple(a.shape) for a in xs]
    lens, in_off, out_off, n_in, n_out, slices, srates = ragged.packed_layout(shapes, df_state.hop_size(), pad, rates)
    pin = torch.cuda.is_available()
    x = torch.empty(n_in, dtype=torch.float32, pin_memory=pin)
    torch.cat([a.detach().to("cpu", torch.float32).reshape(-1) for a in xs], out=x)
    y = torch.empty(n_out, dtype=torch.float32, pin_memory=pin)
    lim = abs(float(atten_lim_db)) if atten_lim_db is not None and tab is None else 0.0
    reduce = ragged.reduce_code(reduce_mask)
    groups = ragged.packed_groups(shapes) if reduce != 0 else None
    outs = [y[s:s + c * n].view(c, n) for s, c, n in slices]
    chans = np.array([c for c, _ in shapes], dtype=np.int64)
    stab = np.ascontiguousarray(np.repeat(tab, chans)) if tab is not None else None   # every channel takes its entry's
    ln = l_off = lz = None
    if return_lsnr:
        ln = ragged.lsnr_lens(lens, srates, df_state.hop_size(), pad)
        l_off = np.concatenate(([0], np.cumsum(ln)[:-1])).astype(np.int64)
        lz = torch.empty(int(ln.sum()), dtype=torch.float32, pin_memory=pin)
    with model._gating(gating_mode):
        check(_lib.lib().dfb_enhance_ragged_host(model.handle, df_state.handle, x.data_ptr(), n_in, in_off.ctypes.data,
                                                 lens.ctypes.data, lens.size, 1 if pad else 0, lim, y.data_ptr(), n_out,
                                                 out_off.ctypes.data, _ptr(groups), groups.size if groups is not None else 0, reduce,
                                                 srates.ctypes.data, _ptr(stab), lens.size, _ptr(lz), lz.numel() if lz is not None else 0,
                                                 _ptr(l_off)))
    if not return_lsnr:
        return outs
    lsnrs, k = [], 0
    for c, _ in shapes:
        v = lz[int(l_off[k]):int(l_off[k]) + c * int(ln[k])].view(c, int(ln[k]))   # an entry's channels are consecutive
        lsnrs.append(v[0] if c == 1 else v)
        k += c
    return outs, lsnrs


@torch.no_grad()
def enhance_device_ragged(model: DfNet, df_state: DF, audio: Tensor, lengths, pad: bool = True,
                          atten_lim_db=None, out: Optional[Tensor] = None, group_sizes=None,
                          reduce_mask: Optional[str] = None, *, sr=None, post_filter_beta=None, lsnr_thresholds=None,
                          return_lsnr: bool = False, gating_mode: Optional[str] = None):
    """Device-resident ragged batch: ``audio`` is a padded CUDA tensor [B, S] whose row b holds ``lengths[b]`` real
    samples.  Returns [B, max out_len] (asynchronous on the current stream): row b equals :func:`enhance_device` of
    ``audio[b, :lengths[b]]`` alone, and is zero beyond its own output length.  With ``out`` given, only each row's own
    output range is written.
    ``group_sizes`` / ``reduce_mask`` "max" / "mean": linked channels -- group g is the next ``group_sizes[g]`` rows, of
    one length, and they share one ERB mask; each group's rows equal :func:`enhance` of that recording with the same
    ``reduce_mask``.
    ``sr``: the rows' sample rate, one for all or one per row (a link group's rows at one rate), as :func:`enhance_batch`
    takes it; lengths and the result are in each row's own samples (dfb_enhance_ragged).
    ``atten_lim_db`` / ``post_filter_beta`` / ``lsnr_thresholds``: as :func:`enhance_batch` takes them, one per row where
    per entry (a link group's rows take one setting).  ``return_lsnr``: the result is ``(out, lsnr, lsnr_lengths)``, lsnr a
    [B, max n] float32 CUDA tensor whose row b holds lsnr_lengths[b] values (NaN after them), as enhance_batch's.
    ``gating_mode`` as :func:`enhance_batch` takes it."""
    if gating_mode is not None:
        ragged.gating_mode_code(gating_mode)
    if not audio.is_cuda or audio.dtype != torch.float32 or not audio.is_contiguous() or audio.dim() != 2:
        raise ValueError("enhance_device_ragged expects a contiguous float32 CUDA tensor of shape [B, S]")
    if audio.device != model.cuda_device:
        raise ValueError(f"audio lives on {audio.device}, the model on {model.cuda_device}")
    b, s = audio.shape
    lens = lengths.detach().cpu().numpy() if isinstance(lengths, Tensor) else lengths
    lens = np.asarray(lens).reshape(-1)
    if lens.size != b:
        raise ValueError(f"{lens.size} lengths for {b} streams")
    rates = _rated(model, sr, b)
    if rates is None:
        rates = np.full(b, ragged.MODEL_SR, dtype=np.int32)
    tab = _settings(model, b, atten_lim_db, post_filter_beta, lsnr_thresholds, return_lsnr)
    lens, in_off, out_off, ow = ragged.padded_layout(lens, s, df_state.hop_size(), pad, rates)
    reduce = ragged.reduce_code(reduce_mask)
    if group_sizes is None and reduce != 0:
        raise ValueError("reduce_mask needs group_sizes: which rows are the channels of one recording")
    groups = ragged.link_groups(group_sizes, lens) if group_sizes is not None else None
    if groups is not None:
        ragged.check_group_rates(groups, rates)
    if out is None:
        out = torch.zeros((b, ow), dtype=torch.float32, device=audio.device)
    elif (out.shape != (b, ow) or out.dtype != torch.float32 or not out.is_cuda or out.device != audio.device
          or not out.is_contiguous()):
        raise ValueError(f"out must be a contiguous float32 CUDA tensor of shape {(b, ow)} on {audio.device}")
    lim = abs(float(atten_lim_db)) if atten_lim_db is not None and tab is None else 0.0
    ln = l_off = lz = None
    if return_lsnr:
        ln = ragged.lsnr_lens(lens, rates, df_state.hop_size(), pad)
        nl = int(ln.max())
        lz = torch.full((b, nl), float("nan"), dtype=torch.float32, device=audio.device)
        l_off = np.arange(b, dtype=np.int64) * nl
    with torch.cuda.device(audio.device), model._gating(gating_mode):
        stream = torch.cuda.current_stream(audio.device).cuda_stream
        check(_lib.lib().dfb_enhance_ragged(model.handle, df_state.handle, audio.data_ptr(), b * s, in_off.ctypes.data,
                                            lens.ctypes.data, b, 1 if pad else 0, lim, out.data_ptr(), b * ow, out_off.ctypes.data,
                                            _ptr(groups), groups.size if groups is not None else 0, reduce, rates.ctypes.data,
                                            _ptr(tab), b, _ptr(lz), lz.numel() if lz is not None else 0, _ptr(l_off), stream))
    return (out, lz, torch.from_numpy(ln)) if return_lsnr else out


# ------------------------------------------------------------------------------------------ CLI ----
# --reduce-mask N, numbered as the deep-filter binary's flag (libDF/src/bin/enhance_wav.rs:60-62)
REDUCE_MASK_CLI = {0: None, 1: "max", 2: "mean"}


def parse_epoch_type(value: str) -> Union[int, str]:
    """enhance.py:253-261."""
    try:
        return int(value)
    except ValueError:
        assert value in ("best", "latest")
        return value


def setup_df_argument_parser(default_log_level: str = "INFO", parser=None):
    """enhance.py:299-339 (same options)."""
    import argparse
    if parser is None:
        parser = argparse.ArgumentParser()
    parser.add_argument("--model-base-dir", "-m", type=str, default=None,
                        help="Model directory containing checkpoints and config, or a pretrained model name.")
    parser.add_argument("--pf", help="Post-filter that slightly over-attenuates very noisy sections.", action="store_true")
    parser.add_argument("--output-dir", "-o", type=str, default=None, help="Directory in which the enhanced audio files will be stored.")
    parser.add_argument("--log-level", type=str, default=default_log_level, help="Logger verbosity. Can be one of (debug, info, error, none)")
    parser.add_argument("--debug", "-d", action="store_const", const="DEBUG", dest="log_level")
    parser.add_argument("--epoch", "-e", default="best", type=parse_epoch_type,
                        help="Epoch for checkpoint loading. Can be one of ['best', 'latest', <int>].")
    return parser


def main(args) -> int:
    """The `deepFilter` command (enhance.py:47-89): load each file at the model rate, enhance, resample back to the
    file's rate, save next to it (or into --output-dir) with the model suffix."""
    import glob
    import time
    model, df_state, suffix, _ = init_df(args.model_base_dir, post_filter=args.pf, log_level=args.log_level,
                                         config_allow_defaults=True, epoch=args.epoch, mask_only=args.no_df_stage)
    suffix = suffix if args.suffix else None
    if args.output_dir is None:
        args.output_dir = "."
    elif not os.path.isdir(args.output_dir):
        os.mkdir(args.output_dir)
    df_sr = model.cfg.sr
    if args.noisy_dir is not None:
        if len(args.noisy_audio_files) > 0:
            logger.error("Only one of `noisy_audio_files` or `noisy_dir` arguments are supported.")
            return 1
        input_files = sorted(glob.glob(args.noisy_dir + "/*"))
    else:
        assert len(args.noisy_audio_files) > 0, "No audio files provided"
        input_files = args.noisy_audio_files
    n_samples = len(input_files)
    batch_size = max(1, getattr(args, "batch_size", 1))
    for b0 in range(0, n_samples, batch_size):
        # --batch-size N: N files are enhanced by one enhance_batch call; each reports its share of the batch time
        batch = []
        for i in range(b0, min(b0 + batch_size, n_samples)):
            file = input_files[i]
            if not os.path.isfile(file):
                logger.warning("File not found: %s. Skipping...", file)
                continue
            audio, meta = load_audio(file, df_sr, verbose=False)
            batch.append((i, file, audio, meta))
        if not batch:
            continue
        t0 = time.time()
        reduce = REDUCE_MASK_CLI[getattr(args, "reduce_mask", 0)]
        extra = cli_settings(args, model)
        if batch_size == 1:
            outs = [enhance(model, df_state, batch[0][2], pad=args.compensate_delay, atten_lim_db=args.atten_lim, reduce_mask=reduce,
                            **extra)]
        else:
            outs = enhance_batch(model, df_state, [a for _, _, a, _ in batch], pad=args.compensate_delay, atten_lim_db=args.atten_lim,
                                 reduce_mask=reduce, **extra)
        t_batch = time.time() - t0
        total = sum(a.numel() for _, _, a, _ in batch)
        for (i, file, audio_in, meta), audio in zip(batch, outs):
            progress = (i + 1) / n_samples * 100
            t = t_batch * audio_in.numel() / total
            t_audio = audio.shape[-1] / df_sr
            p_str = f"{progress:2.0f}% | " if n_samples > 1 else ""
            logger.info("%sEnhanced noisy audio file '%s' in %.2fs (RT factor: %.3f)", p_str, os.path.basename(file), t, t / t_audio)
            audio = resample(audio.to("cpu"), df_sr, meta.sample_rate)
            save_audio(file, audio, sr=meta.sample_rate, output_dir=args.output_dir, suffix=suffix, log=False)
    return 0


# LSNR stage gating thresholds of the deep-filter binary: its flags and defaults (libDF/src/bin/enhance_wav.rs:41-59)
LSNR_THRESH_CLI = (("min_db_thresh", -15.0), ("max_db_erb_thresh", 35.0), ("max_db_df_thresh", 35.0))


def cli_settings(args, model: DfNet) -> dict:
    """The keyword arguments of enhance / enhance_batch that --pf-beta and the threshold flags ask for: with --pf, a
    DeepFilterNet3 model's post filter takes --pf-beta (where it differs from the model's pf_beta, the plain call runs);
    any threshold flag turns LSNR stage gating on, the flags not given taking the deep-filter binary's defaults, and
    --gating-mode runtime makes the decoders skip the gated frames."""
    kw = {}
    beta = getattr(args, "pf_beta", None)
    if getattr(args, "pf", False) and model.cfg.model == "deepfilternet3" and beta is not None and beta != model.post_filter_beta:
        kw["post_filter_beta"] = args.pf_beta
    th = [getattr(args, name, None) for name, _ in LSNR_THRESH_CLI]
    if any(v is not None for v in th):
        kw["lsnr_thresholds"] = tuple(d if v is None else v for v, (_, d) in zip(th, LSNR_THRESH_CLI))
        if getattr(args, "gating_mode", "apply") != "apply":
            kw["gating_mode"] = args.gating_mode
    return kw


def cli_parser():
    """The `deepFilter` command's arguments (enhance.py:342-379)."""
    parser = setup_df_argument_parser()
    parser.add_argument("--no-delay-compensation", dest="compensate_delay", action="store_false",
                        help="Don't add some padding to compensate the delay introduced by the real-time STFT/ISTFT implementation.")
    parser.add_argument("--atten-lim", "-a", type=int, default=None,
                        help="Attenuation limit in dB by mixing the enhanced signal with the noisy signal.")
    parser.add_argument("noisy_audio_files", type=str, nargs="*", help="List of noisy files to enhance.")
    parser.add_argument("--noisy-dir", "-i", type=str, default=None,
                        help="Input directory containing noisy audio files. Use instead of `noisy_audio_files`.")
    parser.add_argument("--no-suffix", action="store_false", dest="suffix", help="Don't add the model suffix to the enhanced audio files")
    parser.add_argument("--no-df-stage", action="store_true")
    parser.add_argument("--batch-size", type=int, default=1,
                        help="Enhance this many files per call (streams of different lengths in one batch); 1: one file per call.")
    parser.add_argument("--reduce-mask", type=int, default=0, choices=sorted(REDUCE_MASK_CLI),
                        help="Link the channels of a multi-channel file: they share one ERB mask, 1 = the max, 2 = the mean of "
                             "their masks; 0 = every channel on its own (default).")
    # the deep-filter binary's flags (enhance_wav.rs:30-59)
    parser.add_argument("--pf-beta", type=float, default=0.02,
                        help="Post-filter beta (with --pf, DeepFilterNet3). Higher beta results in stronger attenuation.")
    for name, default in LSNR_THRESH_CLI:
        parser.add_argument("--" + name.replace("_", "-"), type=float, default=None,
                            help=f"LSNR stage gating threshold in dB (DeepFilterNet3; default {default:g} when any threshold "
                                 "flag is given). Without any of these flags every frame is processed (no gating).")
    parser.add_argument("--gating-mode", choices=sorted(ragged.GATING_MODES), default="apply",
                        help="With LSNR stage gating: 'apply' runs the network on every frame and applies each frame's stage; "
                             "'runtime' runs each decoder only on the frames its stage lets through, as the deep-filter binary does.")
    return parser


def run(argv=None) -> int:
    """enhance.py:342-379."""
    return main(cli_parser().parse_args(argv))


if __name__ == "__main__":
    raise SystemExit(run())
