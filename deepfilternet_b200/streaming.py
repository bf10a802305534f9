"""Frame-incremental enhancement with carried state: host-side mirror of the reference's streaming runtime
(``DfTract::process`` libDF/src/tract.rs:509-642; C ABI libDF/src/capi.rs:83-253) for B independent streams at once.

    s = DfStream(model, df_state, batch=4)
    for chunk in chunks:                 # chunk: float32 [4, n * hop], any n >= 1
        out = s.process(chunk)           # [4, n * hop], trailing the input by s.latency_frames hops
    tail = s.flush()                     # [4, latency * hop]

The concatenation of the outputs equals ``enhance(model, df_state, audio, pad=False)`` delayed by
``latency_frames * hop`` samples.  Everything runs in the CUDA library (dfb_stream_* in include/dfb200.h).

``channels`` / ``reduce_mask`` link the channels of each recording as the Rust runtime does: rows g * channels + c are
the channels of recording g and share one ERB mask, the max or mean of theirs (dfb_stream_set_mask_reduce).

Each row is a slot that can start and end its own stream (``open`` / ``close``), so one handle serves calls that come and
go: a call joins whenever a slot is free, and only open and closing slots are computed.  ``open_linked`` opens a call of
several channels in as many slots, linked by the handle's ``reduce_mask`` like a ``channels`` group.  Each slot can change its own
attenuation limit and post-filter beta between two calls (``set_atten_lim`` / ``set_post_filter_beta``), and
``process`` / ``flush`` return the local SNR of every output frame on request (``return_lsnr=True``).

``spectral=True`` makes the handle of the Rust runtime's ``df_process_frame_raw`` (capi.rs:187-212): it takes spectrum
frames from the caller's own filter bank and returns the network's outputs, applying nothing::

    s = DfStream(model, df_state, batch=B, spectral=True)
    out = s.process_spec(spec)           # spec: complex64 [B, n, F], e.g. DF.analysis's
    out.gains, out.coefs, out.lsnr, out.stage
    tail = s.flush_spec()

Row j of a call that starts at input frame k carries frame k + j - ``latency_frames`` (conv_lookahead); rows that carry no
frame are NaN with stage -1 (dfb_stream_create_spec in include/dfb200.h).

``sr`` runs an audio handle at 8, 12, 16, 24, 32 or 44.1 kHz: its hops are ``sr // 100`` samples, and each call is resampled
to 48 kHz on the device (``io.resample``'s sinc_fast taps, with per-slot filter history), enhanced by the unchanged 48 kHz
slot path and resampled back.  ``latency_frames`` grows by one hop and ``latency_samples`` is the resamplers' own delay
(dfb_stream_set_sample_rate in include/dfb200.h)::

    s = DfStream(model, df_state, batch=B, sr=16000)
    out = s.process(chunk)               # chunk: float32 [B, n * 160]

``slot_rates`` makes a mixed-rate handle: a 48 kHz handle whose slots each open at their own rate, so that calls at
different rates share one pass through the slot path.  Rows stay 480 samples per hop; a slot at rate r reads the first
``n * r // 100`` samples of its row and returns as many, followed by zeros.  Each session equals a handle at its own rate
(dfb_stream_add_slot_rate in include/dfb200.h)::

    s = DfStream(model, df_state, batch=256, slot_rates=(8000, 16000))
    s.open([3, 9], sr=16000)
    s.open([7])                          # 48 kHz
    out = s.process(chunk)               # chunk: float32 [256, n * 480]

``export`` takes live sessions out of a handle as one ``uint8`` blob and ``resume`` continues them in free slots of any
compatible handle -- another one, in another process or on another GPU -- with the outputs the source would have given
next (dfb_stream_export_sessions in include/dfb200.h; ``session_info`` reads a blob's header)::

    blob = s.export([3, 9], release=True)        # the sessions leave s
    d.resume(blob, [0, 1])                       # and continue in slots 0 and 1 of d
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple, Optional

import numpy as np
import torch
from torch import Tensor

from . import _lib, io, ragged
from ._lib import DFB_ERR_INVALID, DFB_ERR_UNSUPPORTED, DfbError, check
from .libdf import DF
from .model import DfNet


SLOT_FREE, SLOT_OPEN, SLOT_CLOSING = 0, 1, 2
MODEL_SR = 48000
# rates with a whole number of samples per 10 ms hop that a streaming handle resamples to and from MODEL_SR
STREAM_RATES = (8000, 12000, 16000, 24000, 32000, 44100)


def rate_taps(sr: int):
    """The resamplers of a handle at ``sr``: ((taps, og, nw, width) of sr -> 48 kHz, the same of 48 kHz -> sr), the
    sinc_fast taps of io.resample.  DfbError (DFB_ERR_UNSUPPORTED, as the C ABI) for a rate outside STREAM_RATES."""
    if isinstance(sr, bool) or not isinstance(sr, (int, np.integer)) or int(sr) not in STREAM_RATES:
        raise DfbError(DFB_ERR_UNSUPPORTED, f"sample rate {sr!r}: one of {STREAM_RATES} or {MODEL_SR}")
    p = io.get_resample_params("sinc_fast")
    return io.resample_kernel(int(sr), MODEL_SR, **p), io.resample_kernel(MODEL_SR, int(sr), **p)


def rate_delays(og_up: int, nw_up: int, width_up: int, og_down: int, nw_down: int, width_down: int):
    """(D, E, delay) of a handle whose resamplers have these geometries: the zeros in front of the upsampled session (48 kHz
    samples) and of the downsampled output (rate-r samples), the smallest whole numbers of polyphase groups after which
    every hop's outputs need only input received with that hop, and the delay they add in rate-r samples."""
    D = -(-width_up // og_up) * nw_up
    E = -(-width_down // og_down) * nw_down
    return D, E, D // nw_up * og_up + E


def slot_rate_arg(s, sr, opening: bool = True) -> int:
    """``sr`` of DfStream.open / open_linked (``opening``) or rate_latency as an int, checked against handle ``s`` as the C
    ABI checks it: DfbError DFB_ERR_UNSUPPORTED outside STREAM_RATES and MODEL_SR, DFB_ERR_INVALID for a rate the handle
    does not run.  A mixed-rate handle runs MODEL_SR and its registered rates; any other audio handle runs its own rate,
    but opens no slot at an explicit rate."""
    if isinstance(sr, bool) or not isinstance(sr, (int, np.integer)) or (int(sr) not in STREAM_RATES and int(sr) != MODEL_SR):
        raise DfbError(DFB_ERR_UNSUPPORTED, f"sample rate {sr!r}: one of {STREAM_RATES} or {MODEL_SR}")
    if getattr(s, "spectral", False):
        raise DfbError(DFB_ERR_INVALID, "a spectral handle takes spectra, which have no sample rate")
    reg = tuple(getattr(s, "registered_rates", ()))
    if not reg and opening:
        raise DfbError(DFB_ERR_INVALID, "slots open at their own rates on a handle with slot rates only (slot_rates=...)")
    runs = (MODEL_SR,) + reg if reg else (s.sr,)
    if int(sr) not in runs:
        raise DfbError(DFB_ERR_INVALID, f"sample rate {int(sr)}: this handle runs {runs}")
    return int(sr)


def slot_list(slots, batch: int) -> np.ndarray:
    """``slots`` (an int, or a sequence / array / tensor of ints) as a contiguous int64 array of slot indices of a handle
    with ``batch`` slots.  ValueError when an index is not an integer, lies outside [0, batch) or is listed twice."""
    if isinstance(slots, Tensor):
        slots = slots.detach().cpu().numpy()
    a = np.asarray([slots] if np.isscalar(slots) else slots)
    if a.ndim != 1 and a.size:
        raise ValueError("slots must be a flat list of slot indices")
    if a.size and a.dtype.kind not in "iu":
        raise ValueError("slot indices must be integers")
    a = np.ascontiguousarray(a.reshape(-1), dtype=np.int64)
    bad = a[(a < 0) | (a >= batch)]
    if bad.size:
        raise ValueError(f"slot {int(bad[0])} outside [0, {batch})")
    u, counts = np.unique(a, return_counts=True)
    if (counts > 1).any():
        raise ValueError(f"slot {int(u[counts > 1][0])} listed twice")
    return a


def group_list(slots, batch: int) -> np.ndarray:
    """``slots`` of DfStream.open_linked as slot_list gives them (channel c in the c-th); ValueError also when empty."""
    a = slot_list(slots, batch)
    if not a.size:
        raise ValueError("a slot group needs at least one slot")
    return a


def atten_lim_arg(db: Optional[float]) -> float:
    """``db`` of DfStream.set_atten_lim as the float the C ABI takes: None is 0 (off); NaN and non-numbers are ValueError."""
    if db is None:
        return 0.0
    if isinstance(db, (bool, str)):
        raise ValueError(f"attenuation limit must be a number of dB, got {db!r}")
    v = float(db)
    if math.isnan(v):
        raise ValueError("attenuation limit is NaN")
    return v


def pf_beta_arg(beta: float) -> float:
    """``beta`` of DfStream.set_post_filter_beta as a float: finite and >= 0 (0 turns the post filter off), else
    ValueError."""
    if isinstance(beta, (bool, str)) or beta is None:
        raise ValueError(f"post-filter beta must be a number, got {beta!r}")
    v = float(beta)
    if not math.isfinite(v) or v < 0:
        raise ValueError(f"post-filter beta must be finite and >= 0, got {beta}")
    return v


BLOB_MAGIC, BLOB_VERSION = 0x53424644, 1
_BLOB_HEADER = np.dtype([("magic", "<u4"), ("version", "<u4"), ("fingerprint", "<u8"), ("sr", "<i4"), ("fft_size", "<i4"),
                         ("hop_size", "<i4"), ("nb_erb", "<i4"), ("gating_mode", "<i4"), ("gate_tails", "<i4"),
                         ("n_sessions", "<i4"), ("n_rows", "<i4"), ("total_bytes", "<i8"), ("row_floats", "<i8", (17,))])
_BLOB_SESSION = np.dtype([("age", "<i8"), ("lsnr_start", "<i8"), ("ctl_switch", "<i8"), ("rate", "<i4"), ("channels", "<i4"),
                          ("reduce", "<i4"), ("reserved", "<i4"), ("lim", "<f4"), ("beta", "<f4"), ("gate", "<i4"),
                          ("th", "<f4", (3,)), ("last_lim", "<f4"), ("last_beta", "<f4"), ("prev_lim", "<f4"),
                          ("prev_beta", "<f4"), ("last_gate", "<i4"), ("last_th", "<f4", (3,)), ("up_hist", "<i4"),
                          ("down_hist", "<i4"), ("data_offset", "<i8")])
assert _BLOB_HEADER.itemsize == 192 and _BLOB_SESSION.itemsize == 112
_NO_LSNR = np.iinfo(np.int64).min
_REDUCE_NAMES = {0: None, 1: "max", 2: "mean"}


class SessionInfo(NamedTuple):
    """One session of a blob: its age in hops since it opened, its rate, its channels (a linked group when > 1) and their
    mask reduction, the settings it resumes with (attenuation limit as a linear factor, 0 = off; post-filter beta; LSNR
    gating and its thresholds) and the frame its LSNR output starts at, relative to its frame 0 (None: never asked for)."""
    age: int
    sr: int
    channels: int
    reduce_mask: Optional[str]
    atten_lim: float
    post_filter_beta: float
    lsnr_gating: bool
    thresholds: tuple
    lsnr_start: Optional[int]


class BlobInfo(NamedTuple):
    """The header of a session blob (DfStream.export): the model fingerprint, the DSP state's sr / fft_size / hop_size /
    nb_erb, the gating mode ("apply" / "runtime"), its size in bytes and its sessions in blob order."""
    fingerprint: int
    sr: int
    fft_size: int
    hop_size: int
    nb_erb: int
    gating_mode: str
    nbytes: int
    sessions: tuple

    @property
    def rows(self) -> int:
        """the slots the blob resumes in: one per channel"""
        return sum(x.channels for x in self.sessions)


def blob_arg(blob) -> Tensor:
    """``blob`` of DfStream.resume / session_info: a flat uint8 tensor (CPU or CUDA), else ValueError.  A view that does
    not start on a 16-byte boundary (a slice of blobs stored back to back) is copied: the library reads the rows as
    floats."""
    if not isinstance(blob, Tensor) or blob.dtype != torch.uint8 or blob.dim() != 1:
        raise ValueError(f"a session blob is a flat uint8 tensor, got {getattr(blob, 'dtype', type(blob).__name__)}")
    blob = blob.contiguous()
    return blob.clone() if blob.data_ptr() % 16 else blob


def _blob_error(msg):
    return DfbError(DFB_ERR_INVALID, f"session blob: {msg}")


def blob_header(blob: Tensor):
    """The checked header of a blob_arg: DfbError (DFB_ERR_INVALID) for a bad magic number or version, or a size other
    than the header's."""
    if blob.numel() < _BLOB_HEADER.itemsize:
        raise _blob_error(f"{blob.numel()} bytes, shorter than its header")
    head = blob[:_BLOB_HEADER.itemsize].cpu().numpy().view(_BLOB_HEADER)[0]
    if int(head["magic"]) != BLOB_MAGIC:
        raise _blob_error(f"magic 0x{int(head['magic']):08x}")
    if int(head["version"]) != BLOB_VERSION:
        raise _blob_error(f"version {int(head['version'])} (this library reads {BLOB_VERSION})")
    ns, total = int(head["n_sessions"]), int(head["total_bytes"])
    if ns < 1 or total != blob.numel():
        raise _blob_error(f"{blob.numel()} bytes, its header says {total} in {ns} sessions")
    return head


def session_info(blob) -> BlobInfo:
    """Parses a blob's header on the host (include/dfb200.h, dfb_stream_export_sessions).  DfbError (DFB_ERR_INVALID, as the
    C ABI refuses it) for a blob that is not one: a bad magic number or version, a truncated blob or one whose size is not
    what its header says."""
    blob = blob_arg(blob)
    head = blob_header(blob)
    ns, total = int(head["n_sessions"]), int(head["total_bytes"])
    bad = _blob_error
    end = _BLOB_HEADER.itemsize + ns * _BLOB_SESSION.itemsize
    if end > total:
        raise bad(f"{ns} session records do not fit in {total} bytes")
    recs = blob[_BLOB_HEADER.itemsize:end].cpu().numpy().view(_BLOB_SESSION)
    sessions = []
    for r in recs:
        red = int(r["reduce"])
        if int(r["channels"]) < 1 or red not in _REDUCE_NAMES:
            raise bad("a malformed session record")
        ls = int(r["lsnr_start"])
        sessions.append(SessionInfo(int(r["age"]), int(r["rate"]), int(r["channels"]), _REDUCE_NAMES[red], float(r["lim"]),
                                    float(r["beta"]), bool(r["gate"]), tuple(float(v) for v in r["th"]),
                                    None if ls == _NO_LSNR else ls))
    if sum(x.channels for x in sessions) != int(head["n_rows"]):
        raise bad(f"its sessions hold {sum(x.channels for x in sessions)} channels, its header says {int(head['n_rows'])}")
    return BlobInfo(int(head["fingerprint"]), int(head["sr"]), int(head["fft_size"]), int(head["hop_size"]), int(head["nb_erb"]),
                    "runtime" if int(head["gating_mode"]) == 1 else "apply", total, tuple(sessions))


class SpecFrames(NamedTuple):
    """Outputs of DfStream.process_spec / flush_spec for n rows per stream, on the input's device.  gains float32 [B, n, E]
    (the ERB mask), coefs float32 [B, n, nb_df, order, 2] (``.permute(0, 3, 1, 2, 4)`` gives DfNet.forward's layout),
    lsnr float32 [B, n] (dB), stage int8 [B, n] (0 - 3 as tract.rs:658-672 apply_stages, -1 where the row carries no
    frame; gains, coefs and lsnr are NaN there)."""
    gains: Tensor
    coefs: Tensor
    lsnr: Tensor
    stage: Tensor


def spec_arg(spec, batch: int, freq_bins: int) -> Tensor:
    """``spec`` of DfStream.process_spec, checked: a complex64 tensor (or numpy array) [batch, n >= 1, freq_bins], contiguous.
    ValueError for a wrong rank, batch, frame count or dtype; RuntimeError with the messages of the reference's DF for
    a wrong number of bins or a non-contiguous input."""
    if isinstance(spec, np.ndarray):
        spec = torch.from_numpy(spec)
    if not isinstance(spec, Tensor):
        raise ValueError(f"spec must be a complex64 tensor, got {type(spec).__name__}")
    if spec.dtype != torch.complex64:
        raise ValueError(f"spec must be complex64, got {spec.dtype}")
    if spec.dim() != 3 or spec.shape[0] != batch or spec.shape[1] == 0:
        raise ValueError(f"spec must have shape [{batch}, n, {freq_bins}] with n >= 1, got {list(spec.shape)}")
    if spec.shape[2] != freq_bins:
        raise RuntimeError(f"DF shape error: expected {freq_bins} frequency bins, got {spec.shape[2]}")
    if not spec.is_contiguous():
        raise RuntimeError("[df] Input array empty or not contiguous.")
    return spec


def need_spectral(s) -> None:
    """DfbError (DFB_ERR_INVALID, as the C ABI) unless ``s`` is a spectral handle."""
    if not getattr(s, "spectral", False):
        raise DfbError(DFB_ERR_INVALID, "an audio stream takes audio: create it with spectral=True for process_spec")


class DfStream:
    def __init__(self, model: DfNet, df_state: DF, batch: int = 1, atten_lim_db: Optional[float] = None, channels: int = 1,
                 reduce_mask: Optional[str] = None, spectral: bool = False, sr: Optional[int] = None,
                 slot_rates=None, gating_mode: Optional[str] = None):
        self.model, self.df_state, self.batch = model, df_state, int(batch)
        if gating_mode is not None:
            ragged.gating_mode_code(gating_mode)
        self.registered_rates = ()
        self.spectral = bool(spectral)
        if self.spectral and atten_lim_db is not None:
            raise ValueError("a spectral stream applies nothing: it takes no attenuation limit")
        h = C.c_void_p()
        lim = abs(float(atten_lim_db)) if atten_lim_db is not None else 0.0
        if self.spectral:
            check(_lib.lib().dfb_stream_create_spec(C.byref(h), model.handle, df_state.handle, self.batch))
        else:
            check(_lib.lib().dfb_stream_create(C.byref(h), model.handle, df_state.handle, self.batch, lim))
        self._h = h
        self.freq_bins = int(df_state.fft_size()) // 2 + 1
        self._read_rate()
        try:
            if sr is not None:
                self.set_sample_rate(sr)
            for r in slot_rates or ():
                self.add_slot_rate(r)
            if channels != 1 or ragged.reduce_code(reduce_mask):
                self.set_mask_reduce(channels, reduce_mask)
            if gating_mode is not None:
                self.set_gating_mode(gating_mode)
        except Exception:
            self.__del__()   # a constructor that fails leaves no handle behind
            raise

    def _read_rate(self) -> None:
        L = _lib.lib()
        self.hop = int(L.dfb_stream_frame_length(self._h))
        self.latency_frames = int(L.dfb_stream_latency_frames(self._h))
        self.latency_samples = int(L.dfb_stream_latency_samples(self._h))
        self.sr = self.hop * 100

    def set_sample_rate(self, sr: int) -> None:
        """Run every slot at ``sr`` (STREAM_RATES, or 48000: the model's own rate), resampled on the device; afterwards
        ``hop``, ``latency_frames`` and ``latency_samples`` are the rate's.  Only on a new or reset audio handle before its
        first frame and any slot operation (DfbError otherwise); survives ``reset`` (dfb_stream_set_sample_rate)."""
        if getattr(self, "spectral", False):
            raise DfbError(DFB_ERR_INVALID, "a spectral handle takes spectra, which have no sample rate")
        is_model_sr = isinstance(sr, (int, np.integer)) and not isinstance(sr, bool) and int(sr) == MODEL_SR
        if getattr(self, "registered_rates", ()) and not is_model_sr:
            raise DfbError(DFB_ERR_INVALID, "a handle with slot rates runs at 48000 Hz: its slots open at their rates")
        if is_model_sr:
            check(_lib.lib().dfb_stream_set_sample_rate(self._h, MODEL_SR, None, 0, 0, 0, None, 0, 0, 0))
        else:
            (ku, wu, ou, nu), (kd, wd, od, nd) = rate_taps(sr)
            check(_lib.lib().dfb_stream_set_sample_rate(self._h, int(sr), ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd))
        self._read_rate()

    def add_slot_rate(self, sr: int) -> None:
        """Let slots of this 48 kHz audio handle open at ``sr`` (STREAM_RATES): ``open(..., sr=sr)``.  Only on a new or reset
        handle before its first frame and any slot operation (DfbError otherwise); survives ``reset``.  ``latency_frames``
        becomes L + 1, the longest drain of any slot (dfb_stream_add_slot_rate)."""
        if getattr(self, "spectral", False):
            raise DfbError(DFB_ERR_INVALID, "a spectral handle takes spectra, which have no sample rate")
        if getattr(self, "sr", MODEL_SR) != MODEL_SR:
            raise DfbError(DFB_ERR_INVALID, f"slot rates are registered on a 48 kHz handle: this one runs at {self.sr} Hz")
        (ku, wu, ou, nu), (kd, wd, od, nd) = rate_taps(sr)
        check(_lib.lib().dfb_stream_add_slot_rate(self._h, int(sr), ku.data_ptr(), ou, nu, wu, kd.data_ptr(), od, nd, wd))
        if int(sr) not in self.registered_rates:
            self.registered_rates += (int(sr),)
        self._read_rate()

    def rate_latency(self, sr: int):
        """(frames, samples): the latency of a session at ``sr`` on this handle, as ``latency_frames`` / ``latency_samples``
        of a handle at ``sr``: the hops a closing slot drains for, and the resamplers' delay in samples of ``sr``."""
        sr = slot_rate_arg(self, sr, opening=False)
        L = self.latency_frames - (1 if self.registered_rates or self.sr != MODEL_SR else 0)   # the 48 kHz path's
        if sr == MODEL_SR:
            return L, 0
        (_, wu, ou, nu), (_, wd, od, nd) = rate_taps(sr)
        return L + 1, rate_delays(ou, nu, wu, od, nd, wd)[2]

    def slot_rates(self) -> np.ndarray:
        """int32 [batch]: the rate of each live slot's session, 0 for a free slot (dfb_stream_slot_rates)."""
        out = np.zeros(self.batch, np.int32)
        check(_lib.lib().dfb_stream_slot_rates(self._h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def set_mask_reduce(self, channels: int, reduce_mask: Optional[str]) -> None:
        """Linked channels: rows g * channels + c form recording g; reduce_mask None / "none", "max" or "mean".  Only on a new
        or reset stream."""
        check(_lib.lib().dfb_stream_set_mask_reduce(self._h, int(channels), ragged.reduce_code(reduce_mask)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().dfb_stream_free(h)
            except Exception:
                pass
            self._h = None

    def set_gating_mode(self, mode: Optional[str]) -> None:
        """What LSNR stage gating does to this handle's network from the next call's frames on: "apply", "runtime" (each
        decoder runs only on the frames its stage lets through, as in the Rust runtime; the frames before the switch count
        as run frames) or None, the model's (:meth:`DfNet.set_gating_mode`; the default).  ValueError for any other value
        (dfb_stream_set_gating_mode)."""
        check(_lib.lib().dfb_stream_set_gating_mode(self._h, -1 if mode is None else ragged.gating_mode_code(mode)))

    def set_lsnr_thresholds(self, min_db_thresh: float = -10.0, max_db_erb_thresh: float = 30.0,
                            max_db_df_thresh: float = 20.0, enable: bool = True, slots=None) -> None:
        """Stage gating of the Rust runtime (tract.rs:658-672, defaults tract.rs:180-185); off unless called.
        ``slots`` None: the handle's setting, for every slot without one of its own.  Otherwise the listed slots' own
        setting from the next call on, every frame of it included (the LADSPA plugin's per-instance thresholds; a group
        lists all of its members; ``open`` and ``reset`` return a slot to the handle's; dfb_stream_set_lsnr_thresholds_slots).
        ValueError for a NaN threshold while gating is on."""
        th = (float(min_db_thresh), float(max_db_erb_thresh), float(max_db_df_thresh))
        if slots is None:
            check(_lib.lib().dfb_stream_set_lsnr_thresholds(self._h, int(enable), *th))
            return
        if enable and any(math.isnan(v) for v in th):
            raise ValueError("an LSNR threshold is NaN")
        a = slot_list(slots, self.batch)
        check(_lib.lib().dfb_stream_set_lsnr_thresholds_slots(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size,
                                                              int(enable), *th))

    def reset(self) -> None:
        """Every slot open with a fresh stream, the clock back at 0."""
        check(_lib.lib().dfb_stream_reset(self._h))

    def _slots(self, fn, slots) -> None:
        a = slot_list(slots, self.batch)
        check(fn(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size))

    def open(self, slots, sr: Optional[int] = None) -> None:
        """Start a new stream in each listed slot, from the initial state, as a fresh handle would.  An open or closing
        slot's old stream is dropped without its tail.  Takes effect at the next ``process`` / ``flush``; from then on row
        b of their input and output is that stream, and its output equals ``DfStream(batch=1)`` fed the same audio in the
        same call sizes and flushed at the end.  A live group (``open_linked``) must be listed with all of its members or
        not at all (DfbError otherwise).  ``sr`` on a mixed-rate handle: the sessions run at ``sr`` (48000 or a registered
        rate), each equal to ``DfStream(batch=1, sr=sr)``; None opens at the handle's rate."""
        if sr is None:
            self._slots(_lib.lib().dfb_stream_open_slots, slots)
            return
        sr = slot_rate_arg(self, sr)
        a = slot_list(slots, self.batch)
        check(_lib.lib().dfb_stream_open_slots_at(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size, sr))

    def open_linked(self, slots, sr: Optional[int] = None) -> None:
        """Start one session of ``len(slots)`` channels, channel c in row ``slots[c]``, whose channels share one ERB mask
        reduced by the handle's ``reduce_mask`` (the constructor's, with ``channels=1``; None: unlinked channels that open
        and close together).  Its output equals ``DfStream(batch=C, channels=C, reduce_mask=...)`` fed the same C rows in
        the same call sizes and flushed at the end.  The group moves as a unit: ``open``, ``open_linked``, ``close`` and the
        setters list all of its members or none.  Opening over a live group drops its old session without its tail
        (dfb_stream_open_linked).  ``sr``: the session's rate on a mixed-rate handle, as for ``open``."""
        if sr is not None:
            sr = slot_rate_arg(self, sr)
        a = group_list(slots, self.batch)
        if sr is None:
            check(_lib.lib().dfb_stream_open_linked(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size))
        else:
            check(_lib.lib().dfb_stream_open_linked_at(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size, sr))

    def close(self, slots) -> None:
        """End the stream of each listed open slot after the input it has already been fed.  From the next call on its
        input rows are ignored; over the next ``latency_frames`` hops its output rows carry what ``flush`` would give that
        stream alone, whatever the call sizes, then the slot is free (at once when ``latency_frames`` is 0).  Free slots
        are not computed and return zeros.  Closing a slot that is not open does nothing.  A group closes as a unit: list
        all of its members."""
        self._slots(_lib.lib().dfb_stream_close_slots, slots)

    def _live_or(self, slots) -> np.ndarray:
        if slots is None:
            return np.flatnonzero(self.slot_states() != SLOT_FREE).astype(np.int64)
        return slot_list(slots, self.batch)

    def set_atten_lim(self, db: Optional[float], slots=None) -> None:
        """Attenuation limit of the listed slots (None: every open or closing slot) from the next call on: ``db`` <= 0 or
        None turns it off, else the enhanced spectrum is mixed with 10^(-db / 20) of the noisy one, as ``atten_lim_db`` of
        the constructor.  The slot's first output hop of that call still carries the previous setting's overlap-add tail.
        ``open`` returns a slot to the handle's setting; ``reset`` drops every setting (dfb_stream_set_atten_lim).  A group
        takes one setting: list all of its members."""
        v = atten_lim_arg(db)
        a = self._live_or(slots)
        check(_lib.lib().dfb_stream_set_atten_lim(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size, v))

    def set_post_filter_beta(self, beta: float, slots=None) -> None:
        """DeepFilterNet3 post-filter beta of the listed slots (None: every open or closing slot) from the next call on;
        finite and >= 0, 0 turns the post filter off.  Not available for DeepFilterNet2 (dfb_stream_set_post_filter_beta).
        A group takes one setting: list all of its members."""
        v = pf_beta_arg(beta)
        a = self._live_or(slots)
        check(_lib.lib().dfb_stream_set_post_filter_beta(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size, v))

    def slot_states(self) -> np.ndarray:
        """int32 [batch]: SLOT_FREE (0), SLOT_OPEN (1) or SLOT_CLOSING (2) per slot.  A new or reset handle has every slot
        open; ``flush`` closes them all."""
        out = np.zeros(self.batch, np.int32)
        check(_lib.lib().dfb_stream_slot_states(self._h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def hold(self, slots, held: bool = True) -> None:
        """Hold the listed live slots (``held=False``: lift their hold) from the next call on: a held session sits out every
        call, as if the call had not happened.  Its input rows are ignored, its output rows are zeros and its LSNR NaN; it
        keeps its slot, state, settings and age, and continues bit for bit in the first call after the hold is lifted, so
        that its outputs over the calls it advanced in equal ``DfStream(batch=1)`` fed the same audio in those calls' sizes.
        ``open``, ``reset``, ``export(release=True)`` and ``flush`` lift holds; ``flush`` ends held sessions as their own
        flush would.  A group is held as a unit: list all of its members (dfb_stream_hold_slots).  ValueError for a
        malformed slot list; DfbError for a free slot, part of a group or a handle with fixed channel groups."""
        a = slot_list(slots, self.batch)
        check(_lib.lib().dfb_stream_hold_slots(self._h, a.ctypes.data_as(C.POINTER(C.c_int64)), a.size, int(bool(held))))

    def held_slots(self) -> np.ndarray:
        """bool [batch]: True per held slot (``hold``)."""
        out = np.zeros(self.batch, np.int8)
        check(_lib.lib().dfb_stream_held_slots(self._h, out.ctypes.data_as(C.POINTER(C.c_int8))))
        return out.astype(bool)

    def slot_groups(self) -> np.ndarray:
        """int64 [batch]: per slot, the slot holding channel 0 of its group (the slot itself for a one-channel session),
        -1 for a free slot."""
        out = np.zeros(self.batch, np.int64)
        check(_lib.lib().dfb_stream_slot_groups(self._h, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def export(self, slots, release: bool = False, device=None) -> Tensor:
        """The sessions of the listed open slots as one uint8 blob, on the handle's device (``device`` None or that CUDA
        device) or on the host (``device="cpu"``).  A linked group is listed whole, from its channel 0 in channel order.
        ``release=False``: a snapshot, the sessions and their neighbours continue unchanged.  ``release=True``: the slots
        are free at once, without a look-ahead tail; the sessions live on in the blob, for ``resume`` on this or another
        handle (dfb_stream_export_sessions).  ValueError for a malformed slot list; DfbError for a free or closing slot,
        part of a group, a spectral handle."""
        a = np.ascontiguousarray(group_list(slots, self.batch), dtype=np.int32)
        ptr = a.ctypes.data_as(C.POINTER(C.c_int32))
        nbytes = C.c_int64()
        check(_lib.lib().dfb_stream_session_bytes(self._h, ptr, a.size, C.byref(nbytes)))
        dev = torch.device(device) if device is not None else self.model.cuda_device
        if dev.type == "cpu":   # page-locked: the one device-to-host copy runs at full speed
            out = torch.empty(nbytes.value, dtype=torch.uint8, pin_memory=True)
            self._finish_device_calls()
            check(_lib.lib().dfb_stream_export_sessions_host(self._h, ptr, a.size, int(bool(release)), out.data_ptr()))
            return out
        if dev.type != "cuda" or (dev.index is not None and dev != self.model.cuda_device):
            raise ValueError(f"a blob goes to the handle's device {self.model.cuda_device} or to the cpu, not {dev}")
        out = torch.empty(nbytes.value, dtype=torch.uint8, device=self.model.cuda_device)
        with torch.cuda.device(out.device):
            check(_lib.lib().dfb_stream_export_sessions(self._h, ptr, a.size, int(bool(release)), out.data_ptr(),
                                                        torch.cuda.current_stream(out.device).cuda_stream))
        return out

    def _finish_device_calls(self) -> None:
        """The _host session entry points run on the handle's own stream: let this handle's calls with CUDA tensors, on
        torch's current stream, finish first (the device-pointer entry points run on that stream and synchronise it)."""
        torch.cuda.current_stream(self.model.cuda_device).synchronize()

    def resume(self, blob, slots) -> None:
        """Continue the sessions of ``blob`` (``export``'s, a CPU or CUDA uint8 tensor) in the listed free slots, one per
        channel in blob order; a group lands as a linked group.  The next ``process`` / ``flush`` calls return what the
        source would have returned next, and ``close`` / ``flush`` end them as any session.  Their settings come with them.
        ValueError for a malformed slot list or blob argument; DfbError (DFB_ERR_INVALID) for a blob that is not one, for
        another model, DSP state or gating mode, a rate or group reduction this handle does not run, a slot that is not
        free (dfb_stream_import_sessions)."""
        blob = blob_arg(blob)
        a = np.ascontiguousarray(group_list(slots, self.batch), dtype=np.int32)
        rows = int(blob_header(blob)["n_rows"])   # (the library checks the session records)
        if a.size != rows:
            raise ValueError(f"the blob holds {rows} channels: list {rows} slots, not {a.size}")
        ptr = a.ctypes.data_as(C.POINTER(C.c_int32))
        if not blob.is_cuda:
            self._finish_device_calls()
            check(_lib.lib().dfb_stream_import_sessions_host(self._h, ptr, a.size, blob.data_ptr()))
            return
        blob = blob.to(self.model.cuda_device)
        with torch.cuda.device(blob.device):
            check(_lib.lib().dfb_stream_import_sessions(self._h, ptr, a.size, blob.data_ptr(),
                                                        torch.cuda.current_stream(blob.device).cuda_stream))

    @torch.no_grad()
    def process(self, audio: Tensor, return_lsnr: bool = False):
        """audio float32 [B, n * hop] (CPU or the model's CUDA device) -> enhanced [B, n * hop] on the same device.
        ``return_lsnr``: returns ``(enhanced, lsnr)``, lsnr float32 [B, n] on the same device: the local SNR in dB of the
        frame each output hop carries, NaN where it carries none (a free slot, the first ``latency_frames`` hops of the
        handle or of a session, a closing slot past its tail).  The handle computes the LSNR from its first request on."""
        if audio.dim() != 2 or audio.shape[0] != self.batch or audio.shape[1] == 0 or audio.shape[1] % self.hop:
            raise ValueError(f"audio must have shape [{self.batch}, n * {self.hop}]")
        n = audio.shape[1] // self.hop
        if audio.is_cuda:
            if audio.device != self.model.cuda_device:
                raise ValueError("audio lives on another device than the model")
            x = audio.to(torch.float32).contiguous()
            out = torch.empty_like(x)
            lsnr = torch.empty((self.batch, n), dtype=torch.float32, device=x.device) if return_lsnr else None
            with torch.cuda.device(x.device):
                check(_lib.lib().dfb_stream_process_lsnr(self._h, x.data_ptr(), n, out.data_ptr(),
                                                         lsnr.data_ptr() if return_lsnr else None,
                                                         torch.cuda.current_stream(x.device).cuda_stream))
            return (out, lsnr) if return_lsnr else out
        x = audio.detach().to("cpu", torch.float32).contiguous()
        out = torch.empty_like(x)
        lsnr = torch.empty((self.batch, n), dtype=torch.float32) if return_lsnr else None
        check(_lib.lib().dfb_stream_process_host_lsnr(self._h, x.data_ptr(), n, out.data_ptr(),
                                                      lsnr.data_ptr() if return_lsnr else None))
        return (out, lsnr) if return_lsnr else out

    @torch.no_grad()
    def flush(self, return_lsnr: bool = False):
        """The ``latency_frames`` hops still in flight at the end of every stream (CPU tensor): closes every open slot,
        and their tails come out in this call.  ``return_lsnr``: ``(tail, lsnr)`` with lsnr [B, latency_frames], the
        tail frames' LSNR (CPU)."""
        out = torch.zeros((self.batch, self.latency_frames * self.hop), dtype=torch.float32)
        lsnr = torch.full((self.batch, self.latency_frames), float("nan"), dtype=torch.float32) if return_lsnr else None
        check(_lib.lib().dfb_stream_process_host_lsnr(self._h, None, 0, out.data_ptr(),
                                                      lsnr.data_ptr() if return_lsnr and lsnr.numel() else None))
        return (out, lsnr) if return_lsnr else out

    # ---------------------------------------------------------------------------------------------- spectral mode ----
    def _spec_outputs(self, n: int, device) -> SpecFrames:
        cfg = self.model.cfg
        B, E, Fd, O = self.batch, cfg.nb_erb, cfg.nb_df, cfg.df_order
        return SpecFrames(torch.empty((B, n, E), dtype=torch.float32, device=device),
                          torch.empty((B, n, Fd, O, 2), dtype=torch.float32, device=device),
                          torch.empty((B, n), dtype=torch.float32, device=device),
                          torch.empty((B, n), dtype=torch.int8, device=device))

    @torch.no_grad()
    def process_spec(self, spec) -> SpecFrames:
        """spec complex64 [B, n, F] (CPU or the model's CUDA device, e.g. DF.analysis's frames) -> SpecFrames of n rows per
        stream on the same device: row j carries frame k + j - ``latency_frames`` of a call that starts at input frame k
        (dfb_stream_process_spec)."""
        need_spectral(self)
        spec = spec_arg(spec, self.batch, self.freq_bins)
        n = spec.shape[1]
        if spec.is_cuda:
            if spec.device != self.model.cuda_device:
                raise ValueError("spec lives on another device than the model")
            out = DfStream._spec_outputs(self, n, spec.device)
            with torch.cuda.device(spec.device):
                check(_lib.lib().dfb_stream_process_spec(self._h, spec.data_ptr(), n, *(t.data_ptr() for t in out),
                                                         torch.cuda.current_stream(spec.device).cuda_stream))
            return out
        out = DfStream._spec_outputs(self, n, "cpu")
        check(_lib.lib().dfb_stream_process_spec_host(self._h, spec.data_ptr(), n, *(t.data_ptr() for t in out)))
        return out

    @torch.no_grad()
    def flush_spec(self) -> SpecFrames:
        """The last ``latency_frames`` frames of every stream (CPU), computed with zero look-ahead features; closes every
        open slot, as ``flush``."""
        need_spectral(self)
        out = self._spec_outputs(self.latency_frames, "cpu")
        ptrs = [t.data_ptr() if t.numel() else None for t in out]
        check(_lib.lib().dfb_stream_process_spec_host(self._h, None, 0, *ptrs))
        return out
