"""The seeded DeepFilterNet2_ll model directory of the DeepFilterNet2_ll tests, in the layout of the shipped models:
<dst>/DeepFilterNet2_ll/config.ini (the shipped configuration, tests/golden/models/DeepFilterNet2_ll) and
checkpoints/model_1.ckpt.best holding weights.random_state_dict(cfg, seed=15).  tests/golden/dfnet_DeepFilterNet2_ll.npz
was produced by the reference's own deepfilternet2 module on exactly these weights (scripts/gen_golden_dfn2_ll.py)."""
from __future__ import annotations

import os
import shutil

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME, EPOCH, SEED = "DeepFilterNet2_ll", 1, 15   # epoch 0 reads as "no checkpoint" upstream


def make_model_dir(dst: str) -> str:
    """Writes the model directory under dst (idempotent) and returns its path."""
    from deepfilternet_b200.config import load_config
    from deepfilternet_b200.weights import random_state_dict
    d = os.path.join(dst, NAME)
    ckpt = os.path.join(d, "checkpoints", f"model_{EPOCH}.ckpt.best")
    if not os.path.isfile(ckpt):
        os.makedirs(os.path.dirname(ckpt), exist_ok=True)
        shutil.copyfile(os.path.join(ROOT, "tests", "golden", "models", NAME, "config.ini"), os.path.join(d, "config.ini"))
        cfg = load_config(os.path.join(d, "config.ini"), env={})
        torch.save(random_state_dict(cfg, seed=SEED), ckpt + ".tmp")
        os.replace(ckpt + ".tmp", ckpt)
    return d
