"""Host-side layout of a ragged batch (streams of different lengths in one ``dfb_enhance_ragged`` call): lengths, input and
output offsets, and their validation.  Pure functions on shapes, so they are usable and testable without the library."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np


def out_len(length: int, hop: int, pad: bool) -> int:
    """dfb_enhance_out_len: the input length with ``pad``, else the whole hops of it."""
    return int(length) if pad else (int(length) // hop) * hop


def check_lengths(lengths, hop: int, pad: bool, max_len: int = None, rates=None) -> np.ndarray:
    """Lengths as int64, each in its stream's own samples at rates[b] (None: every stream at 48 kHz).  ValueError for a
    length <= 0 or beyond ``max_len``; RuntimeError when ``pad`` is off and a stream is shorter than one hop at 48 kHz (it
    has no frame), as ``enhance()`` does."""
    lens = np.ascontiguousarray(np.asarray(lengths, dtype=np.int64).reshape(-1))
    if lens.size == 0:
        raise ValueError("empty batch")
    if (lens <= 0).any():
        raise ValueError(f"stream lengths must be > 0, got {int(lens.min())}")
    if max_len is not None and (lens > max_len).any():
        raise ValueError(f"stream length {int(lens.max())} exceeds the {max_len} samples per row")
    lens48 = lens if rates is None else -(-lens * MODEL_SR // np.asarray(rates, dtype=np.int64))   # len_48k of every stream
    if not pad and (lens48 < hop).any():
        raise RuntimeError(f"stream of {int(lens48.min())} samples is shorter than one hop ({hop}): no frame to enhance")
    return lens


def padded_layout(lengths, width: int, hop: int, pad: bool, rates=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int]:
    """Rows of a padded [B, width] input and a [B, max out_len] output, row b at rates[b] (None: every row at 48 kHz):
    (lengths, in_offsets, out_offsets, out_width), every count in each row's own samples."""
    lens = check_lengths(lengths, hop, pad, width, rates)
    ow = int(_out_lens(lens, MODEL_SR if rates is None else rates, hop, pad).max())
    rows = np.arange(lens.size, dtype=np.int64)
    return lens, rows * width, rows * ow, ow


def packed_layout(shapes: Sequence[Tuple[int, int]], hop: int, pad: bool, rates=None):
    """Entries [C_i, T_i] packed back to back, every channel one stream, entry i at rates[i] (None: every entry at 48 kHz):
    (lengths, in_offsets, out_offsets, in_numel, out_numel, slices, stream_rates), every count in each stream's own
    samples, where slices[i] = (start, C_i, out_len_i) locates entry i in the packed output and stream_rates are int32, one
    per stream."""
    lens: List[int] = []
    srates: List[int] = []
    for i, shp in enumerate(shapes):
        if len(shp) != 2:
            raise ValueError(f"entry {i}: audio must have shape [C, T], got {tuple(shp)}")
        c, t = int(shp[0]), int(shp[1])
        if c <= 0:
            raise ValueError(f"entry {i}: no channels")
        lens += [t] * c
        srates += [MODEL_SR if rates is None else int(rates[i])] * c
    lens = check_lengths(lens, hop, pad, rates=srates)
    olens = _out_lens(lens, srates, hop, pad)
    in_off = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int64)
    out_off = np.concatenate(([0], np.cumsum(olens)[:-1])).astype(np.int64)
    slices, k = [], 0
    for shp in shapes:
        c = int(shp[0])
        slices.append((int(out_off[k]), c, int(olens[k])))
        k += c
    return lens, in_off, out_off, int(lens.sum()), int(olens.sum()), slices, np.ascontiguousarray(np.array(srates, dtype=np.int32))


# Linked channels (dfb_enhance_ragged's link groups): the channels of one recording share one ERB mask, reduced over them.
# Numbering of dfb_reduce_mask and of the Rust runtime's ReduceMask / --reduce-mask (libDF/src/tract.rs:95-99).
REDUCE_MASK = {"none": 0, "max": 1, "mean": 2}


# include/dfb200.h dfb_gating_mode: what LSNR stage gating does to the network
GATING_MODES = {"apply": 0, "runtime": 1}


def gating_mode_code(mode) -> int:
    """"apply" or "runtime" -> DFB_GATING_APPLY / DFB_GATING_RUNTIME (ValueError otherwise)."""
    if not isinstance(mode, str) or mode not in GATING_MODES:
        raise ValueError(f"gating_mode must be one of {sorted(GATING_MODES)}, not {mode!r}")
    return GATING_MODES[mode]


def reduce_code(reduce_mask) -> int:
    """None, "none", "max" or "mean" -> 0, 0, 1, 2 (ValueError otherwise)."""
    if reduce_mask is None:
        return 0
    if isinstance(reduce_mask, str) and reduce_mask.lower() in REDUCE_MASK:
        return REDUCE_MASK[reduce_mask.lower()]
    raise ValueError(f"reduce_mask must be None, 'none', 'max' or 'mean', got {reduce_mask!r}")


def link_groups(group_sizes, lengths) -> np.ndarray:
    """Link groups as consecutive runs of streams: group g is the next ``group_sizes[g]`` streams of ``lengths``.  Returns
    the sizes as int64; ValueError when a size is < 1, the sizes do not sum to the number of streams, or a group's streams
    differ in length (the channels of one recording have one length)."""
    sizes = np.ascontiguousarray(np.asarray(group_sizes, dtype=np.int64).reshape(-1))
    lens = np.asarray(lengths, dtype=np.int64).reshape(-1)
    if sizes.size == 0:
        raise ValueError("no link groups")
    if (sizes <= 0).any():
        raise ValueError(f"link group sizes must be >= 1, got {int(sizes.min())}")
    if int(sizes.sum()) != lens.size:
        raise ValueError(f"link group sizes sum to {int(sizes.sum())}, the batch has {lens.size} streams")
    b = 0
    for g, n in enumerate(sizes.tolist()):
        if (lens[b:b + n] != lens[b]).any():
            raise ValueError(f"link group {g} has channels of different lengths: {lens[b:b + n].tolist()}")
        b += n
    return sizes


def packed_groups(shapes: Sequence[Tuple[int, int]]) -> np.ndarray:
    """Link groups of a :func:`packed_layout` batch: entry i's C_i channels are one group."""
    return np.ascontiguousarray(np.array([int(shp[0]) for shp in shapes], dtype=np.int64))


# Rated batches (dfb_enhance_ragged's rates): every stream at its own sample rate, resampled to and from the model's 48 kHz
# with io.resample's sinc_fast taps.  A rate is supported when its two gcd-reduced tap tables hold at most MAX_RATE_TAPS
# floats together.
MODEL_SR = 48000
MAX_RATE_TAPS = 1 << 18
SINC_FAST_WIDTH, SINC_FAST_ROLLOFF = 16, 0.99   # io.get_resample_params("sinc_fast"), with resample_kernel's rolloff


def rate_tap_floats(rate: int) -> int:
    """Floats of the sinc_fast tap tables rate -> 48 kHz and 48 kHz -> rate together (io.resample_kernel's shapes)."""
    n = 0
    for orig, new in ((rate, MODEL_SR), (MODEL_SR, rate)):
        g = math.gcd(orig, new)
        og, nw = orig // g, new // g
        width = math.ceil(SINC_FAST_WIDTH * og / (min(og, nw) * SINC_FAST_ROLLOFF))
        n += nw * (2 * width + og)
    return n


def check_rate(rate) -> int:
    """A sample rate as int; ValueError, naming it, for anything but a positive integer whose taps fit MAX_RATE_TAPS."""
    if isinstance(rate, bool) or not isinstance(rate, (int, np.integer)) or int(rate) <= 0:
        raise ValueError(f"sample rate {rate!r}: a positive integer number of Hz")
    rate = int(rate)
    if rate != MODEL_SR and rate_tap_floats(rate) > MAX_RATE_TAPS:
        raise ValueError(f"sample rate {rate} Hz is not supported: its resampler taps would hold {rate_tap_floats(rate)} floats, "
                         f"more than 2^18")
    return rate


def rates_arg(sr, n: int):
    """``sr`` of the batch calls for n entries: None, one rate for all, or one per entry.  Returns the rates as int32, or
    None when every one is 48 kHz (the unrated call).  ValueError for a list of another length or an unsupported rate."""
    if sr is None:
        return None
    if isinstance(sr, (int, np.integer)) and not isinstance(sr, bool):
        rates = [sr] * n
    else:
        rates = list(np.asarray(sr).reshape(-1).tolist()) if not isinstance(sr, (list, tuple)) else list(sr)
        if len(rates) != n:
            raise ValueError(f"{len(rates)} sample rates for {n} entries")
    rates = np.ascontiguousarray(np.array([check_rate(r) for r in rates], dtype=np.int32))
    return None if (rates == MODEL_SR).all() else rates


def len_48k(length: int, rate: int) -> int:
    """io.resample's length of ``length`` samples at ``rate`` resampled to 48 kHz: ceil(length * 48000 / rate)."""
    return -(-int(length) * MODEL_SR // int(rate))


def out_len_at(length: int, rate: int, hop: int, pad: bool) -> int:
    """dfb_enhance_out_len_at: the 48 kHz output length of the resampled stream, resampled back to ``rate``."""
    if int(rate) == MODEL_SR:
        return out_len(length, hop, pad)
    return -(-out_len(len_48k(length, rate), hop, pad) * int(rate) // MODEL_SR)


def _out_lens(lens: np.ndarray, rates, hop: int, pad: bool) -> np.ndarray:
    """:func:`out_len_at` of every stream (int64 lengths, rates one or one per stream) as one int64 array: array arithmetic,
    so that laying out a batch costs no Python call per stream."""
    r = np.asarray(rates, dtype=np.int64)
    o48 = -(-lens * MODEL_SR // r)
    if not pad:
        o48 = o48 // hop * hop
    return -(-o48 * r // MODEL_SR)


def lsnr_lens(lens: np.ndarray, rates, hop: int, pad: bool) -> np.ndarray:
    """dfb_enhance_lsnr_len of every stream (int64 lengths in their own samples, rates one or one per stream): one value per
    10 ms hop of the 48 kHz output, ceil(out48 / hop)."""
    r = np.asarray(rates, dtype=np.int64)
    o48 = -(-np.asarray(lens, dtype=np.int64) * MODEL_SR // r)
    if not pad:
        o48 = o48 // hop * hop
    return -(-o48 // hop)


# Per-entry settings of the batch calls (dfb_enhance_ragged's settings): the layout of dfb_enhance_settings
SETTINGS_DTYPE = np.dtype([("atten_lim_db", "<f4"), ("post_filter_beta", "<f4"), ("lsnr_gating", "<i4"),
                           ("min_db_thresh", "<f4"), ("max_db_erb_thresh", "<f4"), ("max_db_df_thresh", "<f4")])


def _is_number(v) -> bool:
    return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool)


def _per_entry(v, n: int, what: str) -> list:
    """A scalar for every entry or one value per entry (list, tuple, array or tensor of n)."""
    if v is None or _is_number(v):
        return [v] * n
    vals = list(np.asarray(v.detach().cpu() if hasattr(v, "detach") else v, dtype=object).reshape(-1))
    if len(vals) != n:
        raise ValueError(f"{len(vals)} values of {what} for {n} entries")
    return vals


def _thresholds(v, what: str):
    if v is None:
        return None
    t = list(v) if isinstance(v, (list, tuple, np.ndarray)) else None
    if t is None or len(t) != 3 or not all(_is_number(x) for x in t):
        raise ValueError(f"{what}: (min_db_thresh, max_db_erb_thresh, max_db_df_thresh), got {v!r}")
    if any(math.isnan(float(x)) for x in t):
        raise ValueError(f"{what}: a threshold is NaN")
    return tuple(float(x) for x in t)


def settings_table(n: int, atten_lim_db, post_filter_beta, lsnr_thresholds, default_beta: float):
    """The dfb_enhance_settings table of n entries for the batch calls' arguments, or None when they need none: a scalar (or
    None) atten_lim_db with post_filter_beta and lsnr_thresholds None runs the call without a table, as before.
    atten_lim_db: None, a scalar or one per entry (None: off; |db| as enhance() takes it).  post_filter_beta: None (the
    model's, ``default_beta``), a scalar or one per entry, finite and >= 0.  lsnr_thresholds: None (no gating), one
    (min_db_thresh, max_db_erb_thresh, max_db_df_thresh) for all, or one per entry (None: that entry does not gate).
    ValueError for a wrong count, a NaN limit or threshold, or a negative / non-finite beta."""
    if (atten_lim_db is None or _is_number(atten_lim_db)) and post_filter_beta is None and lsnr_thresholds is None:
        return None
    tab = np.zeros(n, dtype=SETTINGS_DTYPE)
    for i, v in enumerate(_per_entry(atten_lim_db, n, "atten_lim_db")):
        if v is not None and not _is_number(v):
            raise ValueError(f"entry {i}: attenuation limit must be a number of dB, got {v!r}")
        if v is not None and math.isnan(float(v)):
            raise ValueError(f"entry {i}: attenuation limit is NaN")
        tab["atten_lim_db"][i] = abs(float(v)) if v is not None else 0.0
    for i, v in enumerate(_per_entry(post_filter_beta, n, "post_filter_beta")):
        if v is None:
            v = default_beta
        if not _is_number(v) or not math.isfinite(float(v)) or float(v) < 0:
            raise ValueError(f"entry {i}: post-filter beta must be finite and >= 0, got {v!r}")
        tab["post_filter_beta"][i] = float(v)
    if lsnr_thresholds is not None:
        if isinstance(lsnr_thresholds, np.ndarray) and lsnr_thresholds.ndim == 1:
            lsnr_thresholds = tuple(lsnr_thresholds.tolist())
        one = isinstance(lsnr_thresholds, (list, tuple)) and len(lsnr_thresholds) == 3 and all(_is_number(x) for x in lsnr_thresholds)
        ths = [lsnr_thresholds] * n if one else list(lsnr_thresholds)
        if len(ths) != n:
            raise ValueError(f"{len(ths)} threshold triples for {n} entries")
        for i, t in enumerate(ths):
            t = _thresholds(t, f"entry {i}: lsnr_thresholds")
            if t is not None:
                tab["lsnr_gating"][i] = 1
                tab["min_db_thresh"][i], tab["max_db_erb_thresh"][i], tab["max_db_df_thresh"][i] = t
    return tab


def check_settings_model(model: str, nb_erb: int, nb_df: int, df_order: int, tab, return_lsnr: bool) -> None:
    """The combinations dfb_enhance_ragged refuses with DFB_ERR_UNSUPPORTED, refused before the library is called
    (DfbError): a settings table needs the specialised apply kernel (df_order 5, nb_df 96, 32 ERB bands) and not DeepFilterNet
    v1; a beta > 0 or gating needs a DeepFilterNet3 topology; DeepFilterNet v1 returns no LSNR rows."""
    from ._lib import DFB_ERR_UNSUPPORTED, DfbError
    if model == "deepfilternet" and (tab is not None or return_lsnr):
        raise DfbError(DFB_ERR_UNSUPPORTED, "per-entry settings and LSNR rows: DeepFilterNet v1 is not supported")
    if tab is None:
        return
    if df_order != 5 or nb_df != 96 or nb_erb != 32:
        raise DfbError(DFB_ERR_UNSUPPORTED, "per-entry settings are built for df_order 5, nb_df 96 and 32 ERB bands")
    if model != "deepfilternet3" and (tab["post_filter_beta"] > 0).any():
        raise DfbError(DFB_ERR_UNSUPPORTED, "per-entry post-filter beta: DeepFilterNet3 topologies only (DeepFilterNet2's beta is fixed)")
    if model != "deepfilternet3" and tab["lsnr_gating"].any():
        raise DfbError(DFB_ERR_UNSUPPORTED, "LSNR stage gating: DeepFilterNet3 topologies only")


def check_group_rates(group_sizes, rates) -> None:
    """ValueError when a link group's streams are at different rates (the channels of one recording have one rate)."""
    b = 0
    for g, n in enumerate(np.asarray(group_sizes, dtype=np.int64).reshape(-1).tolist()):
        if (np.asarray(rates[b:b + n]) != rates[b]).any():
            raise ValueError(f"link group {g} has channels at different sample rates: {np.asarray(rates[b:b + n]).tolist()}")
        b += n
