"""CPU: the generic real FFT of STFT sizes other than 960 / 480 (host emulation of its index algebra), and the refusal of
those sizes on the model path."""
import os
import subprocess

import pytest

from conftest import ROOT

from deepfilternet_b200.config import ModelConfig, load_config
from deepfilternet_b200.model import DfNet


def test_generic_fft_on_host(tmp_path):
    """Host emulation of the Stockham stages, split and merge steps of dfb_fft_generic.cuh in fp32, forward and inverse,
    against a float64 DFT for N = 2..64, every even N up to 1024 and the STFT sizes the GPU tests use: worst err / bound
    (the bound of tests/test_gpu_stft_sizes.py) <= 1, and no plan above 8192."""
    exe = tmp_path / "fft_generic_host_test"
    subprocess.check_call(["nvcc", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-o", str(exe),
                           os.path.join(ROOT, "tests", "host", "fft_generic_host_test.cu")], stderr=subprocess.DEVNULL)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0 and "OK" in out.stdout, out.stdout


@pytest.mark.parametrize("model", ["deepfilternet", "deepfilternet2", "deepfilternet3"])
def test_model_path_refuses_other_stft_sizes(tmp_path, model_dir, model):
    """load_config (the v1 branch and the v2 / v3 branch) and DfNet raise NotImplementedError for a model configured at
    16 kHz with fft 320 / hop 160: the DNN and apply kernels are built for 48 kHz, 960 / 480."""
    name = {"deepfilternet": "DeepFilterNet", "deepfilternet2": "DeepFilterNet2", "deepfilternet3": "DeepFilterNet3"}[model]
    ini = open(os.path.join(model_dir, name, "config.ini")).read()
    p = tmp_path / "config.ini"
    p.write_text(ini)
    assert load_config(str(p), env={}).fft_size == 960
    for env in ({"FFT_SIZE": "320", "HOP_SIZE": "160", "SR": "16000"}, {"FFT_SIZE": "320", "HOP_SIZE": "160"}, {"SR": "16000"}):
        with pytest.raises(NotImplementedError, match="960"):
            load_config(str(p), env=env)
    with pytest.raises(NotImplementedError, match="960"):
        DfNet(ModelConfig(model=model, sr=16000, fft_size=320, hop_size=160), {})
