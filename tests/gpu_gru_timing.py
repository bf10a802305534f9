"""Prints the per-phase clock64 timeline of the GRU kernel (CTA 0) -- run on the GPU box."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from deepfilternet_b200 import DfNet, _lib, enhance_device, libdf
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.weights import random_state_dict
from tests_common import synth_audio
B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
cfg = ModelConfig(model="deepfilternet3", conv_ch=64, conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                  lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", df_pathway_kernel_size_t=5)
if len(sys.argv) > 3 and sys.argv[3] == "ll":   # DeepFilterNet3_ll: H = 512 recurrences (clusters of 16 CTAs)
    cfg = ModelConfig(model="deepfilternet3", conv_ch=64, conv_lookahead=0, df_lookahead=0, conv_kernel=(2, 3), emb_hidden_dim=512,
                      df_hidden_dim=512, emb_num_layers=3, df_num_layers=3, lin_groups=16, enc_lin_groups=16,
                      df_gru_skip="groupedlinear", df_pathway_kernel_size_t=5)
st = libdf.DF(48000, 960, 480, 32, 2)
model = DfNet(cfg, random_state_dict(cfg, 0), st)
model.set_chunking(1, 1, 1)
SEC = int(sys.argv[2]) if len(sys.argv) > 2 else 2
audio = (torch.randn(B, 48000 * SEC, device="cuda") * 0.05).clamp(-1, 1)
enhance_device(model, st, audio); torch.cuda.synchronize()
T = (48000 * SEC + 960) // 480
L = _lib.lib()
L.dfb_debug_gru_timing(model.handle, T, None)
enhance_device(model, st, audio); torch.cuda.synchronize()
buf = np.zeros((T, 8), dtype=np.int64)
L.dfb_debug_gru_timing(model.handle, T, buf.ctypes.data)
d = buf[20:T - 20]
step = np.diff(d[:, 0])
print(f"TC GRU B={B}  cycles/step median {np.median(step):.0f}")
# k_gru_tc stamps: 0 step start, 1 state arrived, 2 MMAs + partial sums done, 3 gates + slice written, 4 slice sent
for a, b_, n in [(0, 1, "wait for h"), (1, 2, "W_hh h (mma.sync)"), (2, 3, "gates + own slice"), (3, 4, "barrier + send")]:
    seg = d[:, b_] - d[:, a]
    print(f"  {n:22s} median {np.median(seg):7.0f}  max {seg.max():7.0f}")
