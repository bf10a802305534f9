"""deepfilternet_b200 -- H100-native (sm_90a) implementation of DeepFilterNet's per-frame
speech-enhancement inference path, behind the reference's own Python API.

    from deepfilternet_b200 import init_df, enhance          # == df.enhance.init_df / enhance
    from deepfilternet_b200 import libdf                      # == pyDF module `libdf`
    deepfilternet_b200.install_dropin()                       # registers `libdf`, `df`, `df.enhance`

The data path is hand-written CUDA in libdfb200.so (built in-tree by __graft_entry__.build()),
reached through the C ABI of include/dfb200.h.  There is no CPU fallback.
"""
from . import libdf  # noqa: F401
from .config import ModelConfig, load_config  # noqa: F401
from .dropin import install_dropin  # noqa: F401
from .enhance import df_features, enhance, enhance_batch, enhance_device, enhance_device_ragged, init_df  # noqa: F401
from .model import DfNet, load_model  # noqa: F401
from .streaming import DfStream  # noqa: F401

__version__ = "0.1.0"
