"""Speech-quality scoring on the device, after ``df.evaluation_utils`` (DeepFilterNet/df/evaluation_utils.py).

Seven metrics, each equal to the reference function applied to one entry alone (include/dfb200.h, DESIGN.md sections
5j, 5m and 5n):

* ``"sisdr"``: ``si_sdr_speechmetrics(clean, degraded)`` at the input rate.
* ``"stoi"``: ``df.stoi.stoi(clean[None], degraded[None], sr)[0]`` (:func:`deepfilternet_b200.stoi.stoi`), NaN for an
  entry with fewer than 512 samples left at 10 kHz after silence removal (the reference leaves garbage there).  This is
  df/stoi.py's STOI, the reference's training-validation STOI, not pystoi's, which its evaluation reports: pystoi removes
  silence and frames the signal differently (DESIGN.md section 5n gives the measured difference).
* ``"ssnr"``: ``df.sepm.SNRseg(c16, d16, 16000)`` after ``io.resample(x, sr, 16000)``, the fifth value of the reference's
  ``CompositeMetric``; NaN for an entry with no frame left.
* ``"llr"`` / ``"wss"``: ``df.sepm.llr(c16, d16, 16000)`` / ``df.sepm.wss(c16, d16, 16000)`` on the same 16 kHz rows;
  NaN for an entry with fewer than 600 samples at 16 kHz (no frame).
* ``"pystoi"`` / ``"estoi"``: ``df.evaluation_utils.stoi(clean, degraded, sr, extended)`` (:func:`stoi`), pystoi's STOI
  and extended STOI after ``io.resample(x, sr, 10000)``, what the reference's ``StoiMetric`` and CI report; NaN for an
  entry of at most 256 samples at 10 kHz (pystoi raises), 1e-5 when fewer than 30 STFT frames remain (pystoi's value).
  ESTOI omits pystoi's eps-scaled random noise.

A batch is scored by one library call (``dfb_metrics_compute(_host)``): resampling, silence removal, STFT, band
envelopes, segment correlations, LPC models, critical-band spectra and every per-entry mean run on the GPU.

``"composite"`` (``df.sepm.composite``: PESQ, CSIG, CBAK, COVL, SSNR) needs PESQ-WB, an external C package this
library does not provide: it is available when the caller passes ``pesq=``, a callable scoring one 16 kHz pair, and
the library computes the rest from the device's LLR, WSS and SSNR.  DNSMOS is not provided.

``python -m deepfilternet_b200.evaluation_utils DATASET_DIR -m MODEL`` scores a VoiceBank-DEMAND style test set as the
reference's ``scripts/test_voicebank_demand.py`` does.
"""
from __future__ import annotations

import csv
import ctypes as C
import logging
import math
import os
from collections import defaultdict
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._lib import check

logger = logging.getLogger("deepfilternet_b200")

# metric name -> (bit of dfb_metrics_compute, name in results and CSV files); the output rows follow the bit order
METRICS = {"sisdr": (1, "SISDR"), "stoi": (2, "STOI"), "ssnr": (4, "SSNR"), "llr": (16, "LLR"), "wss": (32, "WSS"),
           "pystoi": (128, "PYSTOI"), "estoi": (256, "ESTOI")}
# "composite" with a caller's PESQ: its values, in the reference CompositeMetric's order, and the device rows it needs
COMPOSITE_NAMES = ("PESQ", "CSIG", "CBAK", "COVL", "SSNR")
COMPOSITE_BITS = 4 | 16 | 32
COMPOSITE_MIN_LEN16 = 600   # the reference's wss raises below 600 samples at 16 kHz (no frame)
UNSUPPORTED = {
    "composite": "needs PESQ (an external C package)",
    "composite-octave": "needs PESQ and Octave",
    "pesq": "needs PESQ (an external C package)",
    "pesq-nb": "needs PESQ (an external C package)",
    "dnsmos5": "needs DNSMOS's downloaded ONNX models",
}
MAX_TAP_FLOATS = 1 << 18
MAX_ENTRIES = 32767
SINC_FAST_WIDTH, SINC_FAST_ROLLOFF = 16, 0.99


def metric_bits(metrics: Sequence[str]) -> int:
    """The bit mask of ``metrics`` (names as :data:`METRICS`, any case).  ValueError for an empty list, a metric the library
    does not provide (saying what it needs) or an unknown name."""
    if isinstance(metrics, str):
        metrics = [metrics]
    bits = 0
    for m in metrics:
        k = str(m).lower()
        if k in UNSUPPORTED:
            raise ValueError(f"metric {m!r} {UNSUPPORTED[k]}, which deepfilternet_b200 does not provide; "
                             f"available: {sorted(METRICS)}")
        if k not in METRICS:
            raise ValueError(f"unknown metric {m!r}; available: {sorted(METRICS)}")
        bits |= METRICS[k][0]
    if bits == 0:
        raise ValueError("no metric requested")
    return bits


def _split_composite(metrics: Sequence[str], pesq) -> Tuple[List[str], int]:
    """(lower-case names, bits of the device rows they need): "composite" counts as SSNR + LLR + WSS when ``pesq`` is
    given, and raises as :func:`metric_bits` does without it."""
    names = [str(m).lower() for m in ([metrics] if isinstance(metrics, str) else metrics)]
    if pesq is None or "composite" not in names:
        return names, metric_bits(names)
    if not callable(pesq):
        raise ValueError("pesq must be a callable (ref16, deg16) -> float")
    rest = [m for m in names if m != "composite"]
    return names, COMPOSITE_BITS | (metric_bits(rest) if rest else 0)


def composite_values(pesq: Callable[[np.ndarray, np.ndarray], float], ref16: np.ndarray, deg16: np.ndarray, llr: float,
                     wss: float, ssnr: float) -> np.ndarray:
    """df.sepm.composite of one 16 kHz pair from its LLR, WSS and SSNR: float32 (PESQ, CSIG, CBAK, COVL, SSNR), CSIG / CBAK /
    COVL being Hu & Loizou's regressions (IEEE TASLP 16(1), 2008) clipped to [1, 5] in fp64.  NaN for fewer than 600
    samples, where ``pesq`` is not called."""
    if ref16.size < COMPOSITE_MIN_LEN16:
        return np.full(5, np.nan, dtype=np.float32)
    p = float(pesq(ref16, deg16))
    llr, wss, ssnr = float(llr), float(wss), float(ssnr)
    csig = 3.093 - 1.029 * llr + 0.603 * p - 0.009 * wss
    cbak = 1.634 + 0.478 * p - 0.007 * wss + 0.063 * ssnr
    covl = 1.594 + 0.805 * p - 0.512 * llr - 0.007 * wss
    clip = lambda v: min(5.0, max(1.0, v))  # noqa: E731
    return np.asarray([p, clip(csig), clip(cbak), clip(covl), ssnr], dtype=np.float64).astype(np.float32)


def bit_names(bits: int) -> List[str]:
    """The metric names of the rows of a call with ``bits``, in row order."""
    return [k for k, (b, _) in METRICS.items() if bits & b]


def tap_floats(sr: int, to: int) -> int:
    """Floats of io.resample_kernel(sr, to)'s sinc_fast table (0 when sr == to)."""
    if sr == to:
        return 0
    g = math.gcd(sr, to)
    og, nw = sr // g, to // g
    width = math.ceil(SINC_FAST_WIDTH * og / (min(og, nw) * SINC_FAST_ROLLOFF))
    return nw * (2 * width + og)


def check_sr(sr) -> int:
    """A metrics rate as int: ValueError for anything but a positive integer whose sr -> 10 kHz and sr -> 16 kHz tables
    hold at most 2^18 floats together."""
    if isinstance(sr, bool) or not isinstance(sr, (int, np.integer)) or int(sr) <= 0:
        raise ValueError(f"sample rate {sr!r}: a positive integer number of Hz")
    sr = int(sr)
    n = tap_floats(sr, 10000) + tap_floats(sr, 16000)
    if n > MAX_TAP_FLOATS:
        raise ValueError(f"sample rate {sr} Hz is not supported for scoring: its resampler taps would hold {n} floats, more than 2^18")
    return sr


def check_pair_lengths(clean_lengths, degraded_lengths) -> np.ndarray:
    """Entry lengths as contiguous int64: ValueError for an empty batch, more than 32767 entries, a length <= 0 or clean
    and degraded lengths that differ."""
    c = np.ascontiguousarray(np.asarray(clean_lengths, dtype=np.int64).reshape(-1))
    d = np.asarray(degraded_lengths, dtype=np.int64).reshape(-1)
    if c.size == 0:
        raise ValueError("empty batch")
    if c.size > MAX_ENTRIES:
        raise ValueError(f"{c.size} entries: at most {MAX_ENTRIES} per call")
    if d.size != c.size:
        raise ValueError(f"{c.size} clean entries, {d.size} degraded")
    bad = np.nonzero(c != d)[0]
    if bad.size:
        i = int(bad[0])
        raise ValueError(f"entry {i}: clean has {int(c[i])} samples, degraded {int(d[i])}")
    if (c <= 0).any():
        raise ValueError(f"entry lengths must be > 0, got {int(c.min())}")
    return c


def packed_offsets(lengths: np.ndarray) -> Tuple[np.ndarray, int]:
    """Entries back to back: (offsets, total samples)."""
    off = np.concatenate(([0], np.cumsum(lengths)[:-1])).astype(np.int64)
    return np.ascontiguousarray(off), int(lengths.sum())


class _Metrics:
    """A dfb_metrics handle: one device, one input rate."""

    def __init__(self, device: int, sr: int):
        from .io import get_resample_params, resample_kernel

        self.sr = check_sr(sr)
        self.device = int(device)
        taps = []
        for to in (10000, 16000):
            if self.sr == to:
                taps.append((None, 0, 0, 0))
            else:
                k, width, og, nw = resample_kernel(self.sr, to, **get_resample_params("sinc_fast"))
                taps.append((k.contiguous(), og, nw, width))
        self._keep = [t[0] for t in taps]
        h = C.c_void_p()
        (k10, og10, nw10, w10), (k16, og16, nw16, w16) = taps
        check(_lib.lib().dfb_metrics_create(C.byref(h), self.device, self.sr,
                                            k10.data_ptr() if k10 is not None else None, og10, nw10, w10,
                                            k16.data_ptr() if k16 is not None else None, og16, nw16, w16))
        self.handle = h

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None and h.value and _lib is not None:
            try:
                _lib.lib().dfb_metrics_free(h)
            except Exception:  # interpreter shutdown
                pass

    def workspace_bytes(self) -> int:
        return int(_lib.lib().dfb_metrics_workspace_bytes(self.handle))


_HANDLES: Dict[Tuple[int, int], _Metrics] = {}


def metrics_handle(sr: int, device: int = 0) -> _Metrics:
    """The process's metrics handle for (device, sr), created on first use."""
    key = (int(device), check_sr(sr))
    if key not in _HANDLES:
        _HANDLES[key] = _Metrics(*key)
    return _HANDLES[key]


def _rows_to_dict(out: Tensor, bits: int, metrics: Sequence[str]) -> Dict[str, Tensor]:
    rows = {k: out[i] for i, k in enumerate(bit_names(bits))}
    metrics = [metrics] if isinstance(metrics, str) else metrics
    return {str(m).lower(): rows[str(m).lower()] for m in metrics if str(m).lower() != "composite"}


@torch.no_grad()
def evaluate_batch(clean: Sequence[Tensor], degraded: Sequence[Tensor], sr: int,
                   metrics: Sequence[str] = ("sisdr", "stoi", "ssnr"), device: int = 0,
                   pesq: Optional[Callable[[np.ndarray, np.ndarray], float]] = None) -> Dict[str, Tensor]:
    """Scores entries of different lengths in one call: ``clean[i]`` and ``degraded[i]`` are 1-D CPU tensors of one length
    at ``sr`` Hz.  Returns {metric: float32 CPU tensor [B]}, in the order of ``metrics``; entry i equals the reference
    function on entry i alone.  The batch is packed into page-locked buffers and scored by one ``dfb_metrics_compute_host``
    call, which copies only the entries' samples.

    ``"composite"`` needs ``pesq``, a callable ``(ref16, deg16) -> float`` (PESQ-WB of one entry's 16 kHz float32 pair,
    ``io.resample``'s output, which is what the device scores); it is then a float32 tensor [B, 5] of (PESQ, CSIG, CBAK,
    COVL, SSNR) as ``df.sepm.composite``, NaN for entries with fewer than 600 samples at 16 kHz (``pesq`` is not called
    for them).  Without ``pesq`` it raises ValueError; exceptions of ``pesq`` propagate."""
    names, bits = _split_composite(metrics, pesq)
    cs, ds = list(clean), list(degraded)
    for i, t in enumerate(cs + ds):
        if not isinstance(t, Tensor) or t.dim() != 1:
            raise ValueError(f"entry {i % max(len(cs), 1)}: audio must be a 1-D tensor")
    lens = check_pair_lengths([t.numel() for t in cs], [t.numel() for t in ds])
    off, n = packed_offsets(lens)
    h = metrics_handle(sr, device)
    pin = torch.cuda.is_available()
    xc = torch.empty(n, dtype=torch.float32, pin_memory=pin)
    xd = torch.empty(n, dtype=torch.float32, pin_memory=pin)
    torch.cat([t.detach().to("cpu", torch.float32) for t in cs], out=xc)
    torch.cat([t.detach().to("cpu", torch.float32) for t in ds], out=xd)
    out = torch.empty((bin(bits).count("1"), lens.size), dtype=torch.float32)
    check(_lib.lib().dfb_metrics_compute_host(h.handle, xc.data_ptr(), xd.data_ptr(), n, off.ctypes.data, lens.ctypes.data,
                                              lens.ctypes.data, lens.size, bits, out.data_ptr()))
    res = _rows_to_dict(out, bits, names)
    if "composite" in names:
        from .io import resample
        rows = {k: out[i] for i, k in enumerate(bit_names(bits))}
        comp = torch.empty((lens.size, 5), dtype=torch.float32)
        for i, (c, d) in enumerate(zip(cs, ds)):
            c16, d16 = (resample(t.detach().to("cpu", torch.float32).reshape(1, -1), h.sr, 16000, device=device)[0].numpy()
                        for t in (c, d))
            comp[i] = torch.from_numpy(composite_values(pesq, c16, d16, rows["llr"][i], rows["wss"][i], rows["ssnr"][i]))
        res = {m: (comp if m == "composite" else res[m]) for m in names}
    return res


@torch.no_grad()
def evaluate_device_ragged(clean: Tensor, degraded: Tensor, lengths, sr: int,
                           metrics: Sequence[str] = ("sisdr", "stoi", "ssnr")) -> Dict[str, Tensor]:
    """Device-resident scoring: ``clean`` and ``degraded`` are padded float32 CUDA tensors [B, S] whose row b holds
    ``lengths[b]`` samples at ``sr`` Hz.  Returns {metric: CUDA tensor [B]} (asynchronous on the current stream), entry b
    equal to :func:`evaluate_batch` of the rows' first ``lengths[b]`` samples."""
    for name, t in (("clean", clean), ("degraded", degraded)):
        if not isinstance(t, Tensor) or not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 2:
            raise ValueError(f"evaluate_device_ragged expects {name} as a contiguous float32 CUDA tensor of shape [B, S]")
    if clean.shape != degraded.shape or clean.device != degraded.device:
        raise ValueError(f"clean {tuple(clean.shape)} on {clean.device} and degraded {tuple(degraded.shape)} on "
                         f"{degraded.device} differ")
    bits = metric_bits(metrics)
    b, s = clean.shape
    lens = lengths.detach().cpu().numpy() if isinstance(lengths, Tensor) else lengths
    lens = np.asarray(lens).reshape(-1)
    if lens.size != b:
        raise ValueError(f"{lens.size} lengths for {b} rows")
    lens = check_pair_lengths(lens, lens)
    if (lens > s).any():
        raise ValueError(f"entry length {int(lens.max())} exceeds the {s} samples per row")
    off = np.ascontiguousarray(np.arange(b, dtype=np.int64) * s)
    h = metrics_handle(sr, clean.device.index or 0)
    out = torch.empty((bin(bits).count("1"), b), dtype=torch.float32, device=clean.device)
    with torch.cuda.device(clean.device):
        stream = torch.cuda.current_stream(clean.device).cuda_stream
        check(_lib.lib().dfb_metrics_compute(h.handle, clean.data_ptr(), degraded.data_ptr(), b * s, off.ctypes.data,
                                             lens.ctypes.data, lens.ctypes.data, b, bits, out.data_ptr(), stream))
    return _rows_to_dict(out, bits, metrics)


def si_sdr_speechmetrics(reference, estimate) -> float:
    """evaluation_utils.si_sdr_speechmetrics of one pair of equal-length 1-D signals at any rate, on the device."""
    r = torch.as_tensor(np.asarray(reference, dtype=np.float32).reshape(-1))
    e = torch.as_tensor(np.asarray(estimate, dtype=np.float32).reshape(-1))
    # SI-SDR does not resample, so any supported rate serves
    return float(evaluate_batch([r], [e], 48000, ("sisdr",))["sisdr"][0])


def stoi(clean, degraded, sr: int, extended: bool = False) -> float:
    """df.evaluation_utils.stoi: pystoi's STOI (ESTOI with ``extended``) of one pair of equal-length 1-D signals at
    ``sr`` Hz after ``io.resample`` to 10 kHz, on the device."""
    c = np.asarray(clean, dtype=np.float32)
    d = np.asarray(degraded, dtype=np.float32)
    if c.ndim != 1 or d.ndim != 1:
        raise ValueError("stoi expects 1-D signals")
    m = "estoi" if extended else "pystoi"
    return float(evaluate_batch([torch.from_numpy(c)], [torch.from_numpy(d)], sr, (m,))[m][0])


# ----------------------------------------------------------------------------------- evaluation loop ----
def write_csv(path: str, flat_metrics: Dict[str, Dict[str, float]]):
    """evaluation_utils.write_csv: ``filename,metric_a,metric_b,...`` then one row per file."""
    metric_names = list(iter(flat_metrics.values()).__next__().keys())
    with open(path, mode="w", newline="") as csvfile:
        w = csv.writer(csvfile, delimiter=",", quoting=csv.QUOTE_MINIMAL)
        w.writerow(["filename"] + metric_names)
        for fn, m in flat_metrics.items():
            w.writerow([fn] + [str(m[n]) for n in metric_names])


@torch.no_grad()
def evaluation_loop(df_state, model, clean_files: List[str], noisy_files: List[str],
                    metrics: List[str] = ["stoi", "sisdr", "ssnr"],  # noqa: B006 (the reference's signature)
                    save_audio_callback: Optional[Callable[[str, Tensor], None]] = None, batch_size: int = 32,
                    log_percent: int = 25, csv_path_enh: Optional[str] = None, csv_path_noisy: Optional[str] = None,
                    noisy_metric: bool = False,
                    pesq: Optional[Callable[[np.ndarray, np.ndarray], float]] = None) -> Dict[str, float]:
    """evaluation_utils.evaluation_loop: enhance each noisy file and score it against its clean file.

    Per file, as the reference: ``enh = enhance(model, df_state, noisy, pad=False)[0]`` and
    ``clean = df_state.synthesis(df_state.analysis(clean))[0]`` (the same for noisy with ``noisy_metric``), files loaded
    at the model's rate with sinc_fast resampling.  ``batch_size`` files are enhanced by one :func:`enhance_batch` call and
    scored by one metrics call (noisy entries included).  Returns the reference's means, ``"Noisy    STOI"`` (with
    ``noisy_metric``) and ``"Enhanced STOI"`` for each metric in ``metrics`` order; ``csv_path_enh`` / ``csv_path_noisy``
    get the reference's per-file CSV layout.  "composite" needs ``pesq`` (see :func:`evaluate_batch`) and adds PESQ, CSIG,
    CBAK, COVL and SSNR, as the reference's CompositeMetric; other metrics than those of :data:`METRICS` raise ValueError."""
    from .enhance import enhance_batch
    from .io import load_audio

    names, _ = _split_composite(metrics, pesq)
    if len(clean_files) != len(noisy_files):
        raise ValueError(f"{len(clean_files)} clean files, {len(noisy_files)} noisy")
    sr = df_state.sr()
    check_sr(sr)
    # metric -> its (label, column of the metric's values) pairs; "composite" has five
    labels = {m: [(lab, q) for q, lab in enumerate(COMPOSITE_NAMES)] if m == "composite" else [(METRICS[m][1], None)]
              for m in names}
    cols = [lab for m in names for lab, _ in labels[m]]
    enh_vals: Dict[str, List[Tuple[str, float]]] = {c: [] for c in cols}
    noisy_vals: Dict[str, List[Tuple[str, float]]] = {c: [] for c in cols}
    pairs = list(zip(noisy_files, clean_files))
    batch_size = max(1, int(batch_size))
    batches = [pairs[i:i + batch_size] for i in range(0, len(pairs), batch_size)]
    done = 0
    for batch in batches:
        noisy = [load_audio(nf, sr, method="sinc_fast")[0] for nf, _ in batch]
        clean = [load_audio(cf, sr, method="sinc_fast")[0] for _, cf in batch]
        enh = [e[0] for e in enhance_batch(model, df_state, noisy, pad=False)]
        clean = [torch.from_numpy(df_state.synthesis(df_state.analysis(c.numpy()))[0]) for c in clean]
        for (nf, _), c, e in zip(batch, clean, enh):
            if c.shape != e.shape:
                raise RuntimeError(f"{c.shape}, {e.shape}, {os.path.basename(nf)}")
        degraded = list(enh)
        refs = list(clean)
        if noisy_metric:
            degraded += [torch.from_numpy(df_state.synthesis(df_state.analysis(n.numpy()))[0]) for n in noisy]
            refs += clean
        scores = evaluate_batch(refs, degraded, sr, names, device=model.cuda_device.index or 0, pesq=pesq)
        for j, (nf, cf) in enumerate(batch):
            fn = os.path.basename(nf)
            for m in names:
                for lab, q in labels[m]:
                    col = scores[m] if q is None else scores[m][:, q]
                    enh_vals[lab].append((fn, float(col[j])))
                    if noisy_metric:
                        noisy_vals[lab].append((fn, float(col[len(batch) + j])))
            if save_audio_callback is not None:
                save_audio_callback(cf, enh[j].to(torch.float32).view(1, -1))
        prev, done = done, done + len(batch)
        if 0 < log_percent < 100:   # evaluation_utils.log_progress's messages
            for p in range(int(100 * prev / len(pairs)) + 1, int(100 * done / len(pairs)) + 1):
                if p % log_percent == 0:
                    logger.info("Progress: %2d%%", p)

    def flat(vals) -> Dict[str, Dict[str, float]]:
        out: Dict[str, Dict[str, float]] = defaultdict(dict)
        for c in vals:
            for fn, v in vals[c]:
                out[fn][c] = v
        return out

    if csv_path_enh is not None:
        write_csv(csv_path_enh, flat(enh_vals))
    if csv_path_noisy is not None and noisy_metric:
        write_csv(csv_path_noisy, flat(noisy_vals))
    out_dict: Dict[str, float] = {}
    for c in enh_vals:
        if noisy_metric:
            out_dict[f"Noisy    {c}"] = float(np.mean([v for _, v in noisy_vals[c]]))
        out_dict[f"Enhanced {c}"] = float(np.mean([v for _, v in enh_vals[c]]))
    return out_dict


# ---------------------------------------------------------------------------------------------- CLI ----
def cli_parser():
    """scripts/test_voicebank_demand.py's arguments, without --metric-workers and --sleep-ms (no worker pool here)."""
    from .enhance import setup_df_argument_parser

    parser = setup_df_argument_parser()
    parser.add_argument("dataset_dir", type=str,
                        help="Voicebank Demand Test set directory. Must contain 'noisy_testset_wav' and 'clean_testset_wav'.")
    parser.add_argument("--csv-path-enh", type=str, default=None, help="Path to csv score file containing metrics of enhanced audios.")
    parser.add_argument("--csv-path-noisy", type=str, default=None, help="Path to csv score file containing metrics of noisy audios.")
    parser.add_argument("--compute-noisy-metric", action="store_true")
    parser.add_argument("--batch-size", type=int, default=32, help="Files enhanced and scored per call.")
    parser.add_argument("--metrics", type=str, nargs="+", default=["stoi", "sisdr", "ssnr"],
                        help=f"Metrics to compute, of {sorted(METRICS)}, and 'composite' when the pesq package is installed.")
    return parser


def pesq_wb() -> Optional[Callable[[np.ndarray, np.ndarray], float]]:
    """``pesq.pesq(16000, ref, deg, "wb")`` of the ``pesq`` package when it imports, else None."""
    try:
        import pesq as pesq_pkg
    except ImportError:
        return None
    return lambda ref16, deg16: pesq_pkg.pesq(16000, ref16, deg16, "wb")


def main(args) -> Dict[str, float]:
    """scripts/test_voicebank_demand.py main: score the test set, log every mean and print them comma-separated (without
    SSNR, as the reference prints)."""
    import glob

    from .enhance import init_df
    from .io import save_audio

    pesq_fn = pesq_wb() if "composite" in [str(m).lower() for m in args.metrics] else None
    _split_composite(args.metrics, pesq_fn)
    model, df_state, suffix, _ = init_df(args.model_base_dir, post_filter=args.pf, log_level=args.log_level,
                                         config_allow_defaults=True, epoch=args.epoch)
    if not os.path.isdir(args.dataset_dir):
        raise FileNotFoundError(f"{args.dataset_dir} is not a directory")
    sr = df_state.sr()
    noisy_dir = os.path.join(args.dataset_dir, "noisy_testset_wav")
    clean_dir = os.path.join(args.dataset_dir, "clean_testset_wav")
    if not (os.path.isdir(noisy_dir) and os.path.isdir(clean_dir)):
        raise FileNotFoundError(f"{args.dataset_dir} must contain 'noisy_testset_wav' and 'clean_testset_wav'")
    clean_files = sorted(glob.glob(clean_dir + "/*.wav"))
    noisy_files = sorted(glob.glob(noisy_dir + "/*.wav"))
    if args.output_dir is not None:
        os.makedirs(args.output_dir, exist_ok=True)

    def save_audio_callback(cleanfn: str, enh: Tensor):
        save_audio(os.path.basename(cleanfn), enh, sr, output_dir=args.output_dir, suffix=suffix)

    metrics = evaluation_loop(df_state, model, clean_files, noisy_files, metrics=args.metrics,
                              save_audio_callback=save_audio_callback if args.output_dir is not None else None,
                              batch_size=args.batch_size, csv_path_enh=args.csv_path_enh, csv_path_noisy=args.csv_path_noisy,
                              noisy_metric=args.compute_noisy_metric, pesq=pesq_fn)
    for k, v in metrics.items():
        logger.info("%s: %s", k, v)
    print("".join(f"{m}," for k, m in metrics.items() if "SSNR" not in k)[:-1])
    return metrics


if __name__ == "__main__":
    main(cli_parser().parse_args())
