"""Host: session blobs (DfStream.export / resume, include/dfb200.h dfb_stream_export_sessions) without a GPU.
streaming.session_info parses synthetic blobs and refuses malformed ones with DFB_ERR_INVALID, as the C ABI does;
DfStream.resume / export refuse malformed arguments before the library is called."""
import types

import numpy as np
import pytest
import torch

from deepfilternet_b200._lib import DFB_ERR_INVALID, DfbError
from deepfilternet_b200.streaming import (_BLOB_HEADER, _BLOB_SESSION, _NO_LSNR, BLOB_MAGIC, BLOB_VERSION, DfStream,
                                          session_info)

ROW = 1000   # floats per row of arrays 0 .. 14 in these synthetic blobs


def blob(sessions=((12, 48000, 1, 0, 0, 0), (30, 16000, 2, 2, 160, 60)), lsnr=(5, _NO_LSNR)):
    """a well-formed blob: sessions of (age, rate, channels, reduce, up_hist, down_hist)"""
    n = len(sessions)
    head = np.zeros(1, _BLOB_HEADER)
    rec = np.zeros(n, _BLOB_SESSION)
    off = _BLOB_HEADER.itemsize + n * _BLOB_SESSION.itemsize
    rows = 0
    for i, (age, rate, ch, red, up, down) in enumerate(sessions):
        rec[i]["age"], rec[i]["rate"], rec[i]["channels"], rec[i]["reduce"] = age, rate, ch, red
        rec[i]["up_hist"], rec[i]["down_hist"], rec[i]["data_offset"] = up, down, off
        rec[i]["lim"], rec[i]["beta"], rec[i]["gate"], rec[i]["th"] = 0.25, 0.02, 1, (-10, 30, 20)
        rec[i]["lsnr_start"] = lsnr[i]
        off += ch * (ROW + up + down) * 4
        rows += ch
    head["magic"], head["version"], head["fingerprint"] = BLOB_MAGIC, BLOB_VERSION, 0x1234_5678_9ABC_DEF0
    head["sr"], head["fft_size"], head["hop_size"], head["nb_erb"] = 48000, 960, 480, 32
    head["gating_mode"], head["n_sessions"], head["n_rows"], head["total_bytes"] = 1, n, rows, off
    out = np.zeros(off, np.uint8)
    out[:_BLOB_HEADER.itemsize] = head.view(np.uint8)
    out[_BLOB_HEADER.itemsize:_BLOB_HEADER.itemsize + n * _BLOB_SESSION.itemsize] = rec.view(np.uint8)
    return torch.from_numpy(out)


def test_header_parses():
    info = session_info(blob())
    assert (info.fingerprint, info.sr, info.fft_size, info.hop_size, info.nb_erb) == (0x123456789ABCDEF0, 48000, 960, 480, 32)
    assert info.gating_mode == "runtime" and info.rows == 3 and info.nbytes == blob().numel()
    a, b = info.sessions
    assert (a.age, a.sr, a.channels, a.reduce_mask, a.lsnr_start) == (12, 48000, 1, None, 5)
    assert (b.age, b.sr, b.channels, b.reduce_mask, b.lsnr_start) == (30, 16000, 2, "mean", None)
    assert b.atten_lim == 0.25 and abs(b.post_filter_beta - 0.02) < 1e-9 and b.lsnr_gating and b.thresholds == (-10, 30, 20)


@pytest.mark.parametrize("edit, text", [
    (lambda x: x[:100], "shorter than its header"),
    (lambda x: x[:-1], "its header says"),
    (lambda x: torch.cat([x, torch.zeros(4, dtype=torch.uint8)]), "its header says"),
    (lambda x: x.index_put_((torch.tensor([0]),), torch.tensor([0x45], dtype=torch.uint8)), "magic"),
    (lambda x: x.index_put_((torch.tensor([4]),), torch.tensor([2], dtype=torch.uint8)), "version"),
    (lambda x: x.index_put_((torch.tensor([44]),), torch.tensor([4], dtype=torch.uint8)), "channels"),
])
def test_malformed_blobs_are_refused(edit, text):
    with pytest.raises(DfbError) as e:
        session_info(edit(blob().clone()))
    assert e.value.code == DFB_ERR_INVALID and text in str(e.value)


@pytest.mark.parametrize("bad", [np.zeros(300, np.uint8), torch.zeros(300, dtype=torch.float32),
                                 torch.zeros((2, 150), dtype=torch.uint8), b"DFBS"])
def test_blob_argument_must_be_a_flat_uint8_tensor(bad):
    with pytest.raises(ValueError):
        session_info(bad)


def fake_handle(batch=4):
    """what DfStream.resume / export read before they call the library"""
    return types.SimpleNamespace(batch=batch, spectral=False, _h=None)


@pytest.mark.parametrize("slots", [[], [0, 0, 1], [0, 4, 1], [0.5, 1, 2], [[0, 1, 2]]])
def test_resume_refuses_malformed_slots(slots):
    with pytest.raises(ValueError):
        DfStream.resume(fake_handle(), blob(), slots)


def test_resume_refuses_a_slot_count_other_than_the_channels():
    with pytest.raises(ValueError, match="3 channels"):
        DfStream.resume(fake_handle(), blob(), [0, 1])


def test_resume_refuses_a_bad_blob_before_the_library():
    with pytest.raises(DfbError) as e:
        DfStream.resume(fake_handle(), blob()[:-8], [0, 1, 2])
    assert e.value.code == DFB_ERR_INVALID


@pytest.mark.parametrize("slots", [[], [1, 1], [7], [-1]])
def test_export_refuses_malformed_slots(slots):
    with pytest.raises(ValueError):
        DfStream.export(fake_handle(), slots)
