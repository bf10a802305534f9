"""Generate tests/golden/dfnet_DeepFilterNet2_ll.npz by running the REFERENCE's own Python modules (imported from a
checkout of the reference, see oracle/ref_harness.py) on the seeded weights of tests/dfn2_ll_model.py.
Run:  python scripts/gen_golden_dfn2_ll.py

DeepFilterNet2_ll ships upstream only as ONNX: the fixture holds the outputs of the reference's deepfilternet2.DfNet
built from its config (zero look-ahead, DF pathway kernel 3) with the seeded weights, as oracle/gen_golden.py does for
the other models: a 0.5 s two-channel excerpt of noisy_snr0.wav (audio, enhanced), the forward pass's inputs and outputs
(spec, feat_erb, feat_spec, spec_e, m, lsnr, and df_alpha, the fourth output of DeepFilterNet2's forward), and the
known answer: the SI-SDR against the clean signal of enhance() on the whole 10 s recording (si_sdr_target,
si_sdr_n_samples).  kat.json and the other fixtures are not touched.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import dfn2_ll_model  # noqa: E402
import golden_io  # noqa: E402
import ref_harness as rh  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    d = dfn2_ll_model.make_model_dir(os.path.join(rh.SCRATCH, "synth"))
    rh.import_reference()
    from df.enhance import df_features, enhance, init_df
    import torch.nn.functional as F

    noisy = torch.from_numpy(rh.read_wav(os.path.join(GOLD, "assets", "noisy_snr0.wav")))
    clean = rh.read_wav(os.path.join(GOLD, "assets", "clean_freesound_33711.wav"))
    model, st, _, _ = init_df(d, log_file=None, log_level="ERROR")
    assert type(model).__module__.endswith("deepfilternet2"), type(model)
    target = rh.si_sdr(clean, enhance(model, st, noisy, pad=True).numpy())
    print("DeepFilterNet2_ll", target)
    x = torch.stack([noisy[0, 96000:120000], 0.5 * noisy[0, 130000:154000]])
    y = enhance(model, st, x, pad=True)
    spec, ef, sf = df_features(F.pad(x, (0, st.fft_size())), st, 96)
    with torch.no_grad():
        spec_e, m, lsnr, alpha = model(spec.clone(), ef, sf)
    golden_io.save(os.path.join(GOLD, "dfnet_DeepFilterNet2_ll.npz"), audio=x.numpy(), enhanced=y.numpy(),
                   spec=spec.numpy(), feat_erb=ef.numpy(), feat_spec=sf.numpy(), spec_e=spec_e.numpy(), m=m.numpy(),
                   lsnr=lsnr.numpy(), df_alpha=alpha.numpy(), si_sdr_target=np.float64(target),
                   si_sdr_n_samples=np.int64(noisy.shape[1]))


if __name__ == "__main__":
    main()
