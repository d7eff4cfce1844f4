"""Golden vectors of the whole calibrator on the GPU: the UNMODIFIED reference `HessianQuantCalibrator
.batching_quant_calib()` (utils/quant_calib.py:300-378, with its own utils/net_wrap.py and configs/PTQ4ViT.py) on the
2-block synthetic ViT of tests/test_calibrator_gpu.py (built on the GPU exactly as the test builds it), sequential=False,
mini-batch 4.  Needs a GPU and the reference tree (oracle/ref_harness.reference_path()):

    TQDM_DISABLE=1 python tests/golden/make_calib_gpu_golden.py [out.npz]

Stored: every module's chosen step sizes ("par|<module>|<key>") and, per captured tensor (x / A / B, y, g), its
absolute maximum and a seeded sample of 2048 entries ("cap|<module>|<key>|max|idx|val") -- the full captures are
larger than a golden file may be."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
os.environ.setdefault("TQDM_DISABLE", "1")

from oracle import ref_harness as RH  # noqa: E402
from tests.test_calibrator_gpu import _net, sample_capture  # noqa: E402


def main(path):
    assert RH.available(), "needs the reference tree"
    snap = {}
    ref, _, _ = RH.run_reference_calibrator(_net(), RH.tiny_images(), batch_size=4, sequential=False, snapshot=snap)
    out = {}
    for name, d in ref.items():
        for key, v in d.items():
            out[f"par|{name}|{key}"] = v.numpy()
    for name, d in snap.items():
        for key, t in d.items():
            if t is None:
                continue
            idx = sample_capture(t.numel(), name, key)
            flat = t.detach().reshape(-1).float().cpu()
            out[f"cap|{name}|{key}|max"] = np.array(float(flat.abs().max()), dtype=np.float32)
            out[f"cap|{name}|{key}|val"] = flat[torch.from_numpy(idx)].numpy()
    np.savez_compressed(path, **out)
    print("wrote", len(out), "arrays to", path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "calib_tiny_vit_gpu.npz"))
