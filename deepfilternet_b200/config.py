"""Model hyper-parameters of the enhancement path, read from a model directory's ``config.ini``.

Host-side mirror of the subset of the reference's config system the inference path needs:
``DfParams`` (DeepFilterNet/df/config.py:12-39) and ``ModelParams``
(deepfilternet3.py:25-77, deepfilternet2.py:26-75).  Lookup precedence follows
``Config.__call__`` (config.py:104-141): environment variable named like the upper-cased option,
then ``ini[section]``, then ``ini[settings]``, then the code default.  ``_fix_df``
(config.py:171-186) moves ``df_order`` / ``df_lookahead`` from ``[deepfilternet]`` to ``[df]``.
"""
from __future__ import annotations

import math
import os
from configparser import ConfigParser
from dataclasses import asdict, dataclass, field
from typing import Any, Callable, Optional, Tuple


def _csv_int(v) -> Tuple[int, ...]:
    if isinstance(v, (tuple, list)):
        return tuple(int(x) for x in v)
    return tuple(int(x) for x in str(v).replace(" ", "").split(",") if x != "")


def _bool(v) -> bool:
    s = str(v).lower()
    if s in {"true", "yes", "y", "on", "1"}:
        return True
    if s in {"false", "no", "n", "off", "0"}:
        return False
    raise ValueError("Parse error")


@dataclass
class ModelConfig:
    # [train]
    model: str = "deepfilternet3"
    # [df]  (DfParams)
    sr: int = 48000
    fft_size: int = 960
    hop_size: int = 480
    nb_erb: int = 32
    nb_df: int = 96
    norm_tau: float = 1.0
    lsnr_max: int = 35
    lsnr_min: int = -15
    min_nb_erb_freqs: int = 2
    df_order: int = 5
    df_lookahead: int = 0
    # [deepfilternet]  (ModelParams)
    conv_lookahead: int = 0
    conv_ch: int = 16
    conv_kernel: Tuple[int, ...] = (1, 3)
    convt_kernel: Tuple[int, ...] = (1, 3)
    conv_kernel_inp: Tuple[int, ...] = (3, 3)
    emb_hidden_dim: int = 256
    emb_num_layers: int = 2
    df_hidden_dim: int = 256
    df_num_layers: int = 3
    df_gru_skip: str = "none"
    emb_gru_skip: str = "none"
    emb_gru_skip_enc: str = "none"
    df_pathway_kernel_size_t: int = 1
    enc_concat: bool = False
    lin_groups: int = 1
    enc_lin_groups: int = 16
    gru_type: str = "squeeze"      # DFN2 only
    df_output_layer: str = "groupedlinear"  # DFN2 only
    dfop_method: str = "df"        # DFN2 only
    mask_pf: bool = False
    pf_beta: float = 0.02
    df_n_iter: int = 1
    # DeepFilterNet v1 only (deepfilternet.py:11-53)
    conv_k_enc: int = 2
    conv_k_dec: int = 1
    gru_groups: int = 1
    group_shuffle: bool = True
    path: str = field(default="", compare=False)

    def as_dict(self) -> dict:
        return asdict(self)

    @property
    def freq_bins(self) -> int:
        return self.fft_size // 2 + 1

    @property
    def norm_alpha(self) -> float:
        """df/utils.py:108-124: round(exp(-hop/sr/tau), 3) with growing precision until < 1."""
        a_ = math.exp(-self.hop_size / self.sr / self.norm_tau)
        precision, a = 3, 1.0
        while a >= 1.0:
            a = round(a_, precision)
            precision += 1
        return a


def load_config(path: str, env: Optional[dict] = None) -> ModelConfig:
    """Parse ``config.ini`` like ``config.load`` + ``ModelParams()`` (enhance.py:146-160)."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"No config file found at '{path}'")
    env = os.environ if env is None else env
    parser = ConfigParser()
    with open(path) as f:
        parser.read_file(f)
    # config.py:171-186 (_fix_df)
    if parser.has_section("deepfilternet") and parser.has_section("df"):
        for k in ("df_order", "df_lookahead"):
            if k in parser["deepfilternet"]:
                parser["df"][k] = parser["deepfilternet"][k]
                del parser["deepfilternet"][k]

    def get(option: str, default: Any, cast: Callable, section: str):
        if option.upper() in env:  # config.py:119-122
            return cast(env[option.upper()])
        if parser.has_option(section, option):
            return cast(parser.get(section, option))
        if parser.has_option("settings", option):
            return cast(parser.get("settings", option))
        return cast(default)

    model = get("model", "deepfilternet3", str, "train").lower()
    if model not in ("deepfilternet", "deepfilternet2", "deepfilternet3"):
        raise NotImplementedError(
            f"model '{model}' is outside the H100 hot path (DeepFilterNet/2/3/3_ll/2_ll supported)")
    c = ModelConfig(model=model, path=path)
    S = "df"
    c.sr = get("sr", 48000, int, S)
    c.fft_size = get("fft_size", 960, int, S)
    c.hop_size = get("hop_size", 480, int, S)
    c.nb_erb = get("nb_erb", 32, int, S)
    c.nb_df = get("nb_df", 96, int, S)
    c.norm_tau = get("norm_tau", 1, float, S)
    c.lsnr_max = get("lsnr_max", 35, int, S)
    c.lsnr_min = get("lsnr_min", -15, int, S)
    c.min_nb_erb_freqs = get("min_nb_erb_freqs", 2, int, S)
    c.df_order = get("df_order", 5, int, S)
    c.df_lookahead = get("df_lookahead", 0, int, S)
    S = "deepfilternet"
    c.conv_lookahead = get("conv_lookahead", 0, int, S)
    c.conv_ch = get("conv_ch", 16, int, S)
    if model == "deepfilternet":
        return _load_v1(c, get)
    c.conv_kernel = get("conv_kernel", (1, 3), _csv_int, S)
    c.conv_kernel_inp = get("conv_kernel_inp", (3, 3), _csv_int, S)
    c.emb_hidden_dim = get("emb_hidden_dim", 256, int, S)
    c.df_hidden_dim = get("df_hidden_dim", 256, int, S)
    c.df_pathway_kernel_size_t = get("df_pathway_kernel_size_t", 1, int, S)
    c.df_gru_skip = get("df_gru_skip", "none", str, S).lower()
    c.mask_pf = get("mask_pf", False, _bool, S)
    c.pf_beta = get("pf_beta", 0.02, float, S)
    c.df_n_iter = get("df_n_iter", 1 if model == "deepfilternet3" else 2, int, S)
    if model == "deepfilternet3":
        c.convt_kernel = get("convt_kernel", (1, 3), _csv_int, S)
        c.emb_num_layers = get("emb_num_layers", 2, int, S)
        c.df_num_layers = get("df_num_layers", 3, int, S)
        c.enc_concat = get("enc_concat", False, _bool, S)
        c.lin_groups = get("linear_groups", 1, int, S)
        c.enc_lin_groups = get("enc_linear_groups", 16, int, S)
        c.emb_gru_skip = get("emb_gru_skip", "none", str, S).lower()
        c.emb_gru_skip_enc = get("emb_gru_skip_enc", "none", str, S).lower()
    else:  # deepfilternet2.py:26-75
        c.convt_kernel = c.conv_kernel  # deepfilternet2.py:225-228 uses conv_kernel for convt
        c.emb_num_layers = get("emb_num_layers", 2, int, S)
        c.df_num_layers = get("df_num_layers", 3, int, S)
        c.enc_concat = get("enc_concat", False, _bool, S)
        c.lin_groups = get("linear_groups", 1, int, S)
        c.enc_lin_groups = c.lin_groups
        c.gru_type = get("gru_type", "grouped", str, S)
        c.df_output_layer = get("df_output_layer", "linear", str, S)
        c.dfop_method = get("dfop_method", "real_unfold", str, S)
        if c.gru_type != "squeeze" or c.df_output_layer != "groupedlinear" or c.dfop_method != "df":
            raise NotImplementedError(
                "DeepFilterNet2 variants other than the shipped one (gru_type=squeeze, "
                "df_output_layer=groupedlinear, dfop_method=df) are outside the H100 hot path")
    if c.hop_size * 2 > c.fft_size:
        raise ValueError("hop_size * 2 <= fft_size required (libDF/src/lib.rs:111)")
    if c.df_n_iter != 1:
        raise NotImplementedError("df_n_iter != 1")
    check_supported(c)
    return c


def _load_v1(c: "ModelConfig", get) -> "ModelConfig":
    """ModelParams of DeepFilterNet v1 (deepfilternet.py:11-53).  The kernels build the shipped topology: transposed
    depthwise decoder convs, grouped GRUs / linears with shuffle, `real_unfold` deep filtering with alpha blending."""
    S = "deepfilternet"
    c.conv_k_enc = get("conv_k_enc", 2, int, S)
    c.conv_k_dec = get("conv_k_dec", 1, int, S)
    c.emb_hidden_dim = get("emb_hidden_dim", 256, int, S)
    c.emb_num_layers = get("emb_num_layers", 1, int, S)
    c.df_hidden_dim = get("df_hidden_dim", 256, int, S)
    c.df_num_layers = get("df_num_layers", 3, int, S)
    c.gru_groups = get("gru_groups", 1, int, S)
    c.lin_groups = get("linear_groups", 1, int, S)
    c.enc_lin_groups = c.lin_groups
    c.group_shuffle = get("group_shuffle", True, _bool, S)
    c.dfop_method = get("dfop_method", "real_unfold", str, S)
    c.mask_pf = get("mask_pf", False, _bool, S)
    c.conv_kernel = (c.conv_k_enc, 3)
    c.convt_kernel = (c.conv_k_dec, 3)
    k0 = 1 if c.conv_k_enc == 1 and c.conv_lookahead == 0 else max(2, c.conv_k_enc)   # deepfilternet.py:74
    c.conv_kernel_inp = (k0, 3)
    bad = []
    if get("conv_width_factor", 1, int, S) != 1: bad.append("conv_width_factor != 1")
    if get("conv_dec_mode", "transposed", str, S) != "transposed": bad.append("conv_dec_mode != transposed")
    if not get("conv_depthwise", True, _bool, S) or not get("convt_depthwise", True, _bool, S): bad.append("dense (non-depthwise) convs")
    if c.dfop_method not in ("real_unfold", "real_loop", "real_strided", "complex_strided"): bad.append(f"dfop_method={c.dfop_method}")
    if c.conv_k_enc != 2 or c.conv_k_dec != 2: bad.append("conv_k_enc / conv_k_dec other than 2")
    if c.conv_lookahead != 2: bad.append("conv_lookahead other than 2")
    if c.emb_hidden_dim != c.df_hidden_dim: bad.append("emb_hidden_dim != df_hidden_dim")
    if bad:
        raise NotImplementedError("DeepFilterNet (v1) variants other than the shipped topology are outside the H100 hot path: " + ", ".join(bad))
    if c.hop_size * 2 > c.fft_size:
        raise ValueError("hop_size * 2 <= fft_size required (libDF/src/lib.rs:111)")
    check_stft_size(c)
    return c


def check_stft_size(c: "ModelConfig") -> None:
    """The DNN and apply kernels are built for the shipped models' STFT (48 kHz, fft 960, hop 480); a model configured
    at another rate or size fails loudly.  The DSP state itself (``libdf.DF``, ``df_features``, ``fft_features``)
    runs at every size up to fft 8192."""
    if (c.sr, c.fft_size, c.hop_size) != (48000, 960, 480):
        raise NotImplementedError(
            f"sr={c.sr}, fft_size={c.fft_size}, hop_size={c.hop_size}: the model path is built for sr=48000, "
            "fft_size=960, hop_size=480 only")


MAX_LOOKAHEAD = 3   # kMaxLookahead in csrc/dfb_model.cu
_GROUPED_LINEARS = ("enc.df_fc_emb.0.weight", "enc.emb_gru.linear_in.0.weight", "enc.emb_gru.linear_out.0.weight",
                    "erb_dec.emb_gru.linear_in.0.weight", "erb_dec.emb_gru.linear_out.0.weight",
                    "df_dec.df_gru.linear_in.0.weight", "df_dec.df_skip.weight", "df_dec.df_out.0.weight")


def check_model_shape(c: "ModelConfig", state_dict) -> None:
    """The shapes dfb_model_create refuses (DFB_ERR_UNSUPPORTED), refused before the library is called: a look-ahead
    outside 0..3 (DeepFilterNet v1: a conv look-ahead other than 2), and (DeepFilterNet2 / 3) a grouped linear whose group
    width is not a multiple of 4.  DeepFilterNet v1's grouped linears are packed for the shipped topology only, which the
    library checks on its own (dfb_model_create)."""
    if not (0 <= c.conv_lookahead <= MAX_LOOKAHEAD and 0 <= c.df_lookahead <= MAX_LOOKAHEAD) or (
            c.model == "deepfilternet" and c.conv_lookahead != 2):
        raise NotImplementedError(f"look-ahead (conv {c.conv_lookahead}, df {c.df_lookahead}): the kernels take look-aheads "
                                  f"0..{MAX_LOOKAHEAD} (DeepFilterNet v1: conv 2)")
    if c.model == "deepfilternet":
        return
    for name in _GROUPED_LINEARS:
        if name in state_dict:
            g, ig, hg = state_dict[name].shape
            if ig % 4 or (g > 1 and hg % 4):
                raise NotImplementedError(f"{name}: {g} groups of {ig} x {hg}: the kernels build group widths that are multiples of 4")


def check_supported(c: "ModelConfig") -> None:
    """Options the kernels do not implement must fail loudly instead of being dropped (all shipped
    configs use emb_gru_skip* = none and df_gru_skip in {none, groupedlinear})."""
    check_stft_size(c)
    if c.model == "deepfilternet3":
        if c.emb_gru_skip != "none" or c.emb_gru_skip_enc != "none":
            raise NotImplementedError(
                f"emb_gru_skip={c.emb_gru_skip!r} / emb_gru_skip_enc={c.emb_gru_skip_enc!r}: only 'none' is built "
                "(deepfilternet3.py:125-133, 232-236)")
        if c.df_gru_skip not in ("none", "groupedlinear"):
            raise NotImplementedError(
                f"df_gru_skip={c.df_gru_skip!r}: only 'none' and 'groupedlinear' are built (deepfilternet3.py:296-306)")
