"""Golden vectors of the BasePTQ configuration, made by the UNMODIFIED reference on the CPU (dev container):

    TQDM_DISABLE=1 python tests/golden/make_baseptq_golden.py

* conv_easy_small.npz: BatchingEasyQuantConv2d(3 -> 32, 4x4 stride 4, a_bit = 32).calibration_step2()
  (quant_layers/conv.py:279-441) on oracle.ptq_oracle.make_conv_fixture(37, 4, 3, 32, 16, 4), hessian metric,
  eq_alpha 0.5, eq_beta 1.2, eq_n 100, one round: the chosen step size and the score table its argmax was taken of.
* calib_tiny_vit_baseptq.npz: HessianQuantCalibrator.batching_quant_calib() (utils/quant_calib.py:300-378) with the
  reference's utils/net_wrap.py and configs/BasePTQ.py, metric set to hessian as example/test_all.py:53-78 does, on the
  2-block synthetic ViT of make_calib_golden.py (seed 0; 8 images of 32x32, seed 3; mini-batch 4; KL target perturbed by
  oracle/ref_harness.add_target_noise).  Every module's chosen step sizes, for sequential=False and sequential=True."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
os.environ.setdefault("TQDM_DISABLE", "1")

from oracle import ptq_oracle as O  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402
from ptq4vit_b200.utils.models import VisionTransformer  # noqa: E402
from tests import _baseptq_ref as B  # noqa: E402

CONV_FIXTURE = (37, 4, 3, 32, 16, 4)


def main():
    torch.manual_seed(0)
    x, W, b, y, g = O.make_conv_fixture(*CONV_FIXTURE)
    r = B.run_conv_layerwise(x, W, b, y, g, stride=4, search_round=1)
    assert len(r["scores"]) == 1
    np.savez_compressed(os.path.join(HERE, "conv_easy_small.npz"), w_interval=r["w_interval"].numpy().reshape(1, 1, 1, 1),
                        scores_000=r["scores"][0].numpy().reshape(-1))
    out = {}
    for sequential in (False, True):
        torch.manual_seed(0)
        net = VisionTransformer(**RH.TINY_VIT).eval()
        RH.add_target_noise(net, 8, RH.TINY_VIT["num_classes"])
        res, _, _ = B.run_reference_calibrator_baseptq(net, RH.tiny_images(), batch_size=4, sequential=sequential)
        for name, d in res.items():
            for key, v in d.items():
                out[f"{'seq' if sequential else 'par'}|{name}|{key}"] = v.numpy()
    np.savez_compressed(os.path.join(HERE, "calib_tiny_vit_baseptq.npz"), **out)
    print("wrote conv_easy_small.npz and", len(out), "calibrator arrays")


if __name__ == "__main__":
    main()
