"""CPU: mixed-rate streaming handles (DfStream(slot_rates=...), dfb_stream_add_slot_rate).  The C ABI's declarations and
bindings, and the Python-side refusals, which come before any library call as those of ``sr`` do."""
import os
import re
from types import SimpleNamespace

import pytest

from deepfilternet_b200 import _lib
from deepfilternet_b200.streaming import MODEL_SR, STREAM_RATES, DfStream, rate_delays, rate_taps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {"dfb_stream_add_slot_rate": 10, "dfb_stream_open_slots_at": 4, "dfb_stream_open_linked_at": 4,
       "dfb_stream_slot_rates": 2, "dfb_debug_resample_slots": 9}


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("reached the library")
    monkeypatch.setattr(_lib, "lib", refuse)


def fake(**kw):
    """A handle no library call can succeed on: every refusal below has to come from Python."""
    base = dict(_h=None, spectral=False, registered_rates=(), sr=MODEL_SR, batch=8, latency_frames=2)
    base.update(kw)
    return SimpleNamespace(**base)


def delay(sr):
    (_, wu, ou, nu), (_, wd, od, nd) = rate_taps(sr)
    return rate_delays(ou, nu, wu, od, nd, wd)[2]


def test_new_entry_points_are_declared_and_bound():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dfb200.h")).read(), flags=re.S)
    for name, nargs in NEW.items():
        assert re.search(rf"\b{name}\s*\(", hdr), name
        assert name in _lib.SIGNATURES and len(_lib.SIGNATURES[name][1]) == nargs, name


@pytest.mark.parametrize("sr", [11025, 22050, 96000, 0, 16000.0, "16000", True])
def test_unsupported_rates_are_refused(sr):
    mixed = fake(registered_rates=(8000, 16000), latency_frames=3)
    for call in (lambda: DfStream.open(mixed, [0], sr=sr), lambda: DfStream.open_linked(mixed, [0, 1], sr=sr),
                 lambda: DfStream.rate_latency(mixed, sr)):
        with pytest.raises(_lib.DfbError) as e:
            call()
        assert e.value.code == _lib.DFB_ERR_UNSUPPORTED, sr
    with pytest.raises(_lib.DfbError) as e:
        DfStream.add_slot_rate(fake(), sr)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED


def test_48k_is_not_a_slot_rate_to_register():
    with pytest.raises(_lib.DfbError) as e:
        DfStream.add_slot_rate(fake(), MODEL_SR)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED


@pytest.mark.parametrize("handle", [fake(), fake(sr=16000), fake(registered_rates=(8000,)), fake(spectral=True)])
@pytest.mark.parametrize("sr", [12000, 16000, MODEL_SR])
def test_opening_at_a_rate_the_handle_does_not_run_is_invalid(handle, sr):
    runs = (MODEL_SR,) + handle.registered_rates if handle.registered_rates else ()
    if sr in runs and not handle.spectral:
        return
    for call in (lambda: DfStream.open(handle, [0], sr=sr), lambda: DfStream.open_linked(handle, [0, 1], sr=sr)):
        with pytest.raises(_lib.DfbError) as e:
            call()
        assert e.value.code == _lib.DFB_ERR_INVALID


@pytest.mark.parametrize("handle", [fake(spectral=True), fake(sr=16000), fake(sr=44100)])
def test_slot_rates_register_on_48k_audio_handles_only(handle):
    with pytest.raises(_lib.DfbError) as e:
        DfStream.add_slot_rate(handle, 8000)
    assert e.value.code == _lib.DFB_ERR_INVALID


@pytest.mark.parametrize("sr", [8000, 44100, 22050])
def test_a_mixed_handle_takes_no_other_sample_rate(sr):
    with pytest.raises(_lib.DfbError) as e:
        DfStream.set_sample_rate(fake(registered_rates=(16000,)), sr)
    assert e.value.code == _lib.DFB_ERR_INVALID


@pytest.mark.parametrize("L", [0, 2, 4])
def test_rate_latency(L):
    mixed = fake(registered_rates=(8000, 44100), latency_frames=L + 1)
    assert DfStream.rate_latency(mixed, MODEL_SR) == (L, 0)
    for sr in (8000, 44100):
        assert DfStream.rate_latency(mixed, sr) == (L + 1, delay(sr))
    assert DfStream.rate_latency(fake(latency_frames=L), MODEL_SR) == (L, 0)
    for sr in STREAM_RATES:   # a handle at one rate: its own latency
        assert DfStream.rate_latency(fake(sr=sr, latency_frames=L + 1), sr) == (L + 1, delay(sr))
        with pytest.raises(_lib.DfbError) as e:
            DfStream.rate_latency(fake(sr=sr, latency_frames=L + 1), MODEL_SR)
        assert e.value.code == _lib.DFB_ERR_INVALID
    with pytest.raises(_lib.DfbError) as e:
        DfStream.rate_latency(mixed, 16000)
    assert e.value.code == _lib.DFB_ERR_INVALID
