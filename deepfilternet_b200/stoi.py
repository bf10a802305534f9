"""Drop-in for ``df.stoi.stoi`` (DeepFilterNet/df/stoi.py), computed on the GPU by the metrics handle of
:mod:`deepfilternet_b200.evaluation_utils`."""
from __future__ import annotations

import torch
from torch import Tensor

from .evaluation_utils import evaluate_batch, evaluate_device_ragged


@torch.no_grad()
def stoi(x: Tensor, y: Tensor, fs_source: int) -> Tensor:
    """df/stoi.py stoi: the STOI of each row of target ``x`` and degraded ``y`` ([B, T] CPU or CUDA tensors at
    ``fs_source`` Hz), float32 [B] on x's device.  Per row, as df/stoi.py computes it:

    1. ``io.resample`` to 10 kHz with sinc_fast taps (none at 10 kHz).
    2. ``remove_silent_frames(x, y, 40, 256, 128)``: both rows padded by ``256 - T % 256`` zeros (a full 256 when T is a
       multiple of 256), ``pad // 2`` in front and the rest at the end; frames of 256 samples at hop 128 times
       ``hann_window(258, periodic=False)[1:-1]``; a frame is kept when its energy
       ``20 log10(|frame| / 16 + eps)`` lies within 40 dB of the row's loudest frame; the kept frames are overlap-added
       and divided by the overlap-added window; the first ``pad // 2`` samples are dropped when the first frame is kept,
       the last ``pad - pad // 2`` when the last frame is kept.
    3. The 512-point STFT of 256-sample frames at hop 128 (the same window, divided by its sum).
    4. The magnitudes of the 15 third-octave bands from 150 Hz (``thirdoct(10000, 512, 15, 150)``).
    5. Segments of 30 frames at every frame offset, or one segment of all L frames when L <= 30.
    6. Per segment and band: y scaled to x's norm, clipped to ``x (1 + 10^(15 / 20))`` (beta = -15 dB), both made
       mean-free and unit-norm; the result is the mean of their correlations over bands and segments.

    A row with fewer than 512 samples after step 2 gets NaN (df/stoi.py skips it and leaves garbage in its slot).
    This is df/stoi.py's STOI, not pystoi's (which the reference uses for reporting, and
    ``evaluation_utils.stoi`` computes): pystoi removes silence and frames the signal differently.  On the reference's
    pretrained outputs for its CI asset the two differ by 3e-4 to 6e-4 (DESIGN.md section 5n)."""
    if x.shape != y.shape:
        raise ValueError("Inputs must have the same shape")
    if x.dim() != 2:
        raise ValueError(f"Expected input shape of [batch_size, samples], but got {tuple(x.shape)}")
    b, t = x.shape
    if x.is_cuda:
        xs = x.detach().to(torch.float32).contiguous()
        ys = y.detach().to(xs.device, torch.float32).contiguous()
        return evaluate_device_ragged(xs, ys, [t] * b, fs_source, ("stoi",))["stoi"]
    return evaluate_batch(list(x.detach().float()), list(y.detach().float()), fs_source, ("stoi",))["stoi"]
