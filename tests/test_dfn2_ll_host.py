"""DeepFilterNet2_ll on the host: DeepFilterNet2 at zero look-ahead (conv_lookahead = df_lookahead = 0) with a DF pathway
conv of 3 time taps.  Its config parses, the packer emits the kt-3 tensor-core operand image of that conv, the CPU oracle
reproduces the reference module's outputs stored in tests/golden/dfnet_DeepFilterNet2_ll.npz, and the ONNX transplant
of DeepFilterNet2's graphs agrees with its checkpoint (where the unpacked upstream models are present)."""
import glob
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dfn2_ll_model
import dfnet_oracle as O
import golden_io
import ref_harness as rh

from deepfilternet_b200.config import load_config
from deepfilternet_b200.model import find_checkpoint, load_state_dict_file
from deepfilternet_b200.weights import pack_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_MODELS = os.path.join(ROOT, "models", "_ref")
FIXED = {"erb_fb", "erb_comp.c", "erb_comp.mn", "mask.erb_inv_fb"}   # buffers computed from the config, not exported


@pytest.fixture(scope="module")
def ll_dir(tmp_path_factory):
    return dfn2_ll_model.make_model_dir(str(tmp_path_factory.mktemp("models")))


def _cfg_sd(d):
    cfg = load_config(os.path.join(d, "config.ini"), env={})
    return cfg, load_state_dict_file(find_checkpoint(os.path.join(d, "checkpoints"))[0])


def test_config_parses(golden_dir):
    cfg = load_config(os.path.join(golden_dir, "models", "DeepFilterNet2_ll", "config.ini"), env={})
    assert cfg.model == "deepfilternet2"
    assert (cfg.conv_lookahead, cfg.df_lookahead, cfg.df_pathway_kernel_size_t, cfg.df_order) == (0, 0, 3, 5)
    assert (cfg.emb_hidden_dim, cfg.df_hidden_dim, cfg.conv_ch, cfg.enc_concat) == (256, 256, 64, True)
    two = load_config(os.path.join(golden_dir, "models", "DeepFilterNet2", "config.ini"), env={})
    assert (two.conv_lookahead, two.df_lookahead, two.df_pathway_kernel_size_t) == (2, 2, 5)


def decode_sw128(img: np.ndarray, n: int = 64) -> np.ndarray:
    """Inverse of weights.umma_sw128_image: the float64 value hi + lo of each [n][64] entry."""
    words = np.ascontiguousarray(img, dtype=np.float32).view(np.uint32).reshape(2, n, 8, 4)
    rows = np.arange(n)
    out = []
    for pl in words:
        un = np.empty_like(pl)
        for j in range(8):
            un[rows, j] = pl[rows, j ^ (rows & 7)]
        u16 = un.reshape(n, 32).view(np.uint16).reshape(n, 64)   # little endian: element 2i in the low half of word i
        out.append((u16.astype(np.uint32) << 16).view(np.float32).astype(np.float64))
    return out[0] + out[1]


def test_packer_emits_the_kt3_pathway_image(ll_dir):
    cfg, sd = _cfg_sd(ll_dir)
    w, g = pack_state_dict(sd, cfg)
    assert g["df_pathway_kt"] == 3 and g["conv_kt"] == 1 and g["inp_kt"] == 3 and g["emb_hidden"] == 256
    w1 = sd["df_dec.df_convp.1.weight"].double().numpy()   # [10 out][32 in per group][3 t][1]
    assert w1.shape == (10, 32, 3, 1)
    W = decode_sw128(w["df_dec.df_convp.w_sw"])
    # float64 restatement: column n = g*32 + dt*5 + o of the product holds tap dt of output channel g*5 + o
    want = np.zeros((64, 64))
    for grp in range(2):
        for dt in range(3):
            for o in range(5):
                want[grp * 32 + dt * 5 + o, grp * 32:(grp + 1) * 32] = w1[grp * 5 + o, :, dt, 0]
    assert np.abs(W - want).max() <= 2.0 ** -16 * np.abs(want).max()
    # and as a convolution: the shifted sums of the image's product equal the grouped causal conv of torch in float64
    rng = np.random.default_rng(3)
    T = 40
    c0 = rng.standard_normal((T, 64))
    Y = c0 @ W.T                                                 # [T][64]
    z = np.zeros((T, 10))
    for grp in range(2):
        for o in range(5):
            for dt in range(3):
                src = np.arange(T) - 2 + dt
                ok = src >= 0
                z[ok, grp * 5 + o] += Y[src[ok], grp * 32 + dt * 5 + o]
    x = torch.from_numpy(c0.T[None, :, :, None].copy())         # [1, 64, T, 1]
    ref = F.conv2d(F.pad(x, (0, 0, 2, 0)), torch.from_numpy(w1), groups=2)[0, :, :, 0].T.numpy()
    bound = 2.0 ** -15 * (np.abs(c0) @ np.abs(want).T).max()
    assert np.abs(z - ref).max() <= bound
    assert w["df_dec.df_convp.w2"].shape == (10, 10) and w["df_dec.df_convp.b"].shape == (10,)


def test_oracle_matches_reference_module(golden_dir, ll_dir):
    """tests/golden/dfnet_DeepFilterNet2_ll.npz holds the outputs of the reference's deepfilternet2.DfNet built from the _ll
    config with the weights of the model directory."""
    cfg, sd = _cfg_sd(ll_dir)
    g = golden_io.load(os.path.join(golden_dir, "dfnet_DeepFilterNet2_ll.npz"))
    out, aux = O.enhance(sd, cfg.as_dict(), torch.from_numpy(g["audio"]), pad=True, return_all=True)
    assert np.abs(aux["m"].numpy() - g["m"]).max() < 1e-5
    assert np.abs(aux["spec_e"].numpy() - g["spec_e"]).max() < 1e-6
    assert float(np.sqrt(((out.numpy() - g["enhanced"]) ** 2).mean())) < 1e-6
    assert float(g["si_sdr_n_samples"]) == 480000 and np.isfinite(float(g["si_sdr_target"]))


def _ref_dirs():
    ck = glob.glob(os.path.join(REF_MODELS, "DeepFilterNet2", "checkpoints", "*.ckpt*"))
    onnx = os.path.join(REF_MODELS, "DeepFilterNet2_onnx")
    return (ck[0] if ck else None), onnx


@pytest.mark.skipif(not (_ref_dirs()[0] and os.path.isfile(os.path.join(_ref_dirs()[1], "df_dec.onnx"))),
                    reason="needs models/_ref/DeepFilterNet2 and DeepFilterNet2_onnx, which build() unpacks from the reference")
def test_onnx_transplant_of_deepfilternet2_matches_its_checkpoint():
    """DeepFilterNet2's ONNX export maps to the checkpoint's tensor names and shapes (only the fixed buffers are absent),
    and the reference module computes the same outputs from both weight sets."""
    from deepfilternet_b200.onnx_import import state_dict_from_onnx_dir
    ckpt, onnx = _ref_dirs()
    cfg = load_config(os.path.join(onnx, "config.ini"), env={})
    sd_onnx = state_dict_from_onnx_dir(onnx, cfg)
    sd_ck = load_state_dict_file(ckpt)
    assert set(sd_ck) - set(sd_onnx) == FIXED
    assert set(sd_onnx) <= set(sd_ck)
    for k, v in sd_onnx.items():
        assert tuple(v.shape) == tuple(sd_ck[k].shape), k
    if not rh.available():
        pytest.skip("the reference modules are not present")
    rh.import_reference()
    from df.deepfilternet2 import init_model
    from df.config import config as dfc
    from df.enhance import df_features
    import libdf
    dfc.load(os.path.join(onnx, "config.ini"), config_must_exist=True, allow_defaults=True, allow_reload=True)
    st = libdf.DF(sr=48000, fft_size=960, hop_size=480, nb_bands=32, min_nb_erb_freqs=2)
    x = torch.from_numpy(rh.read_wav(os.path.join(ROOT, "tests", "golden", "assets", "noisy_snr0.wav")))[:, 96000:120000]
    spec, ef, sf = df_features(F.pad(x, (0, 960)), st, 96)
    outs = []
    for sd in (sd_ck, sd_onnx):
        net = init_model(st).eval()
        missing, unexpected = net.load_state_dict(sd, strict=False)
        assert set(unexpected) | set(missing) <= FIXED   # the checkpoint's erb_comp.* has no module here
        with torch.no_grad():
            outs.append(net(spec.clone(), ef, sf))
    for a, b in zip(*outs):
        assert (a - b).abs().max().item() <= 1e-5
