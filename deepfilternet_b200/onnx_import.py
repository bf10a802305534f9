"""Weights of DeepFilterNet3_ll and DeepFilterNet2_ll ship only as ONNX (``enc.onnx`` / ``erb_dec.onnx`` / ``df_dec.onnx``
inside ``models/DeepFilterNet3_ll_onnx.tar.gz`` and ``models/DeepFilterNet2_onnx_ll.tar.gz``; export code:
DeepFilterNet/df/scripts/export.py:133-285).  This
module transplants them into a reference-style ``state_dict`` (SURVEY.md Appendix B) so that the same weight
packer / kernels serve the ONNX-only model.  The ``onnx`` package is not available, so the files are read with
a ~60-line protobuf wire-format reader (only the fields needed: graph.node, graph.initializer, Constant
node tensors).

Mapping (verified against the DeepFilterNet3 checkpoint, whose ONNX export ships next to it; DeepFilterNet2's three
graphs map the same way: the transplant of ``DeepFilterNet2_onnx`` has every tensor name and shape of the
``DeepFilterNet2`` checkpoint except the buffers computed from the config (``erb_fb``, ``erb_comp.*``,
``mask.erb_inv_fb``), and the reference's deepfilternet2 module computes the same outputs from both weight sets to
1e-5, tests/test_dfn2_ll_host.py):
  * Einsum / depthwise-conv / ConvTranspose initialisers keep their torch names (``erb_conv1.1.weight`` ...);
  * a conv that had a BatchNorm behind it appears as an anonymous ``onnx::Conv_<n>`` (weight, bias) pair with
    the BN folded in -> stored as that conv + an identity BatchNorm carrying the bias;
  * GRU weights are ``W[1,3H,in]``, ``R[1,3H,H]``, ``B[1,6H]`` (initialisers or Constant nodes) with gate
    order z,r,h -> reordered to torch's r,z,n and split into ``bias_ih`` / ``bias_hh``;
  * ``lsnr_fc`` / ``df_fc_a`` are MatMul weights ``[in,1]`` plus a named bias.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .config import ModelConfig

_EPS = 1e-5


# ------------------------------------------------------------------ protobuf wire reader ----
def _varint(b: bytes, i: int) -> Tuple[int, int]:
    r = s = 0
    while True:
        c = b[i]
        i += 1
        r |= (c & 0x7F) << s
        s += 7
        if not c & 0x80:
            return r, i


def _fields(b: bytes):
    i, n = 0, len(b)
    while i < n:
        key, i = _varint(b, i)
        f, w = key >> 3, key & 7
        if w == 0:
            v, i = _varint(b, i)
        elif w == 1:
            v = b[i:i + 8]
            i += 8
        elif w == 2:
            ln, i = _varint(b, i)
            v = b[i:i + ln]
            i += ln
        elif w == 5:
            v = b[i:i + 4]
            i += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {w}")
        yield f, w, v


def _tensor(b: bytes) -> Tuple[str, np.ndarray]:
    """TensorProto: dims=1, data_type=2, float_data=4, int64_data=7, name=8, raw_data=9."""
    dims: List[int] = []
    name, dt, raw = "", 1, None
    floats: List[float] = []
    for f, w, v in _fields(b):
        if f == 1:
            if w == 0:
                dims.append(v)
            else:
                j = 0
                while j < len(v):
                    d, j = _varint(v, j)
                    dims.append(d)
        elif f == 2:
            dt = v
        elif f == 8:
            name = v.decode()
        elif f == 9:
            raw = v
        elif f == 4:
            floats.extend(np.frombuffer(v, dtype="<f4").tolist() if w == 2 else [np.frombuffer(v, dtype="<f4")[0]])
    np_dt = {1: "<f4", 7: "<i8", 6: "<i4"}.get(dt)
    if np_dt is None:
        return name, np.zeros(0, dtype=np.float32)
    if raw is not None:
        a = np.frombuffer(raw, dtype=np_dt)
    else:
        a = np.asarray(floats, dtype=np_dt)
    if dims and int(np.prod(dims)) == a.size:
        a = a.reshape(dims)
    return name, a.copy()


def read_onnx(path: str):
    """-> (tensors by name incl. Constant outputs, nodes as (name, op_type, inputs, outputs))."""
    b = open(path, "rb").read()
    graph = next(v for f, w, v in _fields(b) if f == 7)
    tensors: Dict[str, np.ndarray] = {}
    nodes = []
    for f, w, v in _fields(graph):
        if f == 5:
            n, a = _tensor(v)
            tensors[n] = a
        elif f == 1:
            ins, outs, name, op, const = [], [], "", "", None
            for ff, ww, vv in _fields(v):
                if ff == 1:
                    ins.append(vv.decode())
                elif ff == 2:
                    outs.append(vv.decode())
                elif ff == 3:
                    name = vv.decode()
                elif ff == 4:
                    op = vv.decode()
                elif ff == 5:  # AttributeProto: name=1, t=5
                    an, at = None, None
                    for f3, w3, v3 in _fields(vv):
                        if f3 == 1:
                            an = v3.decode()
                        elif f3 == 5:
                            at = v3
                    if an == "value" and at is not None:
                        const = at
            if op == "Constant" and const is not None and outs:
                tensors[outs[0]] = _tensor(const)[1]
            nodes.append((name, op, ins, outs))
    return tensors, nodes


# ------------------------------------------------------------------ ONNX -> state_dict ----
def _gru_reorder(a: np.ndarray, h: int) -> np.ndarray:
    """ONNX gate order z,r,h -> torch r,z,n along the first axis."""
    return np.concatenate([a[h:2 * h], a[0:h], a[2 * h:3 * h]], axis=0)


def _module_of(node_name: str) -> str:
    return node_name.strip("/").split("/")[0]


def _import_graph(path: str, prefix: str, sd: Dict[str, torch.Tensor]) -> None:
    tensors, nodes = read_onnx(path)
    convs: Dict[str, List[Tuple[str, np.ndarray, Optional[np.ndarray]]]] = {}
    grus: Dict[str, int] = {}
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    for name, op, ins, outs in nodes:
        mod = _module_of(name)
        if op in ("Conv", "ConvTranspose"):
            w = tensors[ins[1]]
            b = tensors[ins[2]] if len(ins) > 2 and ins[2] else None
            convs.setdefault(mod, []).append((op, w, b))
        elif op == "GRU":
            W, R, B = tensors[ins[1]][0], tensors[ins[2]][0], tensors[ins[3]][0]
            h = R.shape[1]
            l = grus.get(mod, 0)
            grus[mod] = l + 1
            base = f"{prefix}{mod}.gru"
            sd[f"{base}.weight_ih_l{l}"] = t(_gru_reorder(W, h))
            sd[f"{base}.weight_hh_l{l}"] = t(_gru_reorder(R, h))
            sd[f"{base}.bias_ih_l{l}"] = t(_gru_reorder(B[:3 * h], h))
            sd[f"{base}.bias_hh_l{l}"] = t(_gru_reorder(B[3 * h:], h))
        elif op == "Einsum":
            sd[prefix + ins[1]] = t(tensors[ins[1]])
        elif op == "MatMul" and mod in ("lsnr_fc", "df_fc_a"):
            sd[f"{prefix}{mod}.0.weight"] = t(tensors[ins[1]].reshape(-1, 1).T)
            sd[f"{prefix}{mod}.0.bias"] = t(tensors[f"{mod}.0.bias"])
    for mod, lst in convs.items():
        p = prefix + mod
        first_kt = lst[0][1].shape[2]
        i = 1 if first_kt > 1 else 0  # nn.Sequential index shift of the ConstantPad2d
        for op, w, b in lst:
            sd[f"{p}.{i}.weight"] = t(w)
            i += 1
        bias = lst[-1][2]
        assert bias is not None, f"{p}: expected a BN-folded bias on the last conv"
        n = bias.shape[0]
        # identity BatchNorm carrying the folded bias: scale = 1 / sqrt(var + eps) = 1
        sd[f"{p}.{i}.weight"] = torch.ones(n)
        sd[f"{p}.{i}.bias"] = t(bias)
        sd[f"{p}.{i}.running_mean"] = torch.zeros(n)
        sd[f"{p}.{i}.running_var"] = torch.full((n,), 1.0 - _EPS, dtype=torch.float64).to(torch.float32)
        sd[f"{p}.{i}.num_batches_tracked"] = torch.tensor(0)


def state_dict_from_onnx_dir(model_dir: str, cfg: ModelConfig) -> Optional[Dict[str, torch.Tensor]]:
    files = {"enc.": "enc.onnx", "erb_dec.": "erb_dec.onnx", "df_dec.": "df_dec.onnx"}
    if not all(os.path.isfile(os.path.join(model_dir, f)) for f in files.values()):
        return None
    sd: Dict[str, torch.Tensor] = {}
    for prefix, f in files.items():
        _import_graph(os.path.join(model_dir, f), prefix, sd)
    return sd
