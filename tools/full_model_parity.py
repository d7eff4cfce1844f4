"""GPU box: calibrate a whole synthetic ViT (timm names, ptq4vit_b200.utils.models) twice -- with the UNMODIFIED
reference (its own net_wrap / configs/PTQ4ViT.py / HessianQuantCalibrator.batching_quant_calib from oracle/_ref) and with
this package -- and compare every step size of every wrapped module.  BASELINE.json configs[1]: ViT-S/224, 32 images,
reference defaults (n_V = n_H = 1, qkv n_V = 3, 3 rounds, hessian, W8A8).
usage: full_model_parity.py [model] [images] [n_V=n_H] > full_model_parity_<model>.json"""
import importlib
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TQDM_DISABLE", "1")
from oracle import ref_harness as RH  # noqa: E402
from ptq4vit_b200.configs import PTQ4ViT as cfg  # noqa: E402
from ptq4vit_b200.utils import quant_calib as Q  # noqa: E402
from ptq4vit_b200.utils.models import get_net  # noqa: E402
from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net  # noqa: E402


def main():
    model = sys.argv[1] if len(sys.argv) > 1 else "vit_small_patch16_224"
    n_img = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    blocks = int(sys.argv[3]) if len(sys.argv) > 3 else 1       # n_V = n_H of the Linear layers (BASELINE config 3: 24)

    def edit(c):
        c.ptqsl_linear_kwargs.update(n_V=blocks, n_H=blocks)
    size = 384 if "384" in model else 224
    images = torch.randn(n_img, 3, size, size, generator=torch.Generator().manual_seed(3))

    def net():
        n = get_net(model, device="cuda", seed=0)
        RH.add_target_noise(n, n_img, 1000)
        return n

    importlib.reload(cfg)
    edit(cfg)
    ours_net = net()
    wrapped = wrap_modules_in_net(ours_net, cfg)
    cal = Q.HessianQuantCalibrator(ours_net, wrapped, RH.ListLoader(images), sequential=False, batch_size=4)
    torch.cuda.synchronize(); t0 = time.time()
    cal.batching_quant_calib()
    torch.cuda.synchronize(); ours_s = time.time() - t0
    got = RH.collect_intervals(wrapped)
    del ours_net, wrapped, cal
    torch.cuda.empty_cache()

    torch.cuda.synchronize(); t0 = time.time()
    ref, _, _ = RH.run_reference_calibrator(net(), images, batch_size=4, sequential=False, cfg_edit=edit)
    torch.cuda.synchronize(); ref_s = time.time() - t0

    n = bad = 0
    worst = 0.0
    diffs = []
    for name, d in ref.items():
        for key, rv in d.items():
            if key not in got.get(name, {}):
                continue
            gv = got[name][key].reshape(-1)
            rel = ((gv - rv.reshape(-1)).abs() / rv.reshape(-1).abs().clamp_min(1e-30))
            k = int((rel > 2e-6).sum())
            n += rv.numel(); bad += k
            worst = max(worst, float(rel.max()))
            if k:
                diffs.append({"module": name, "key": key, "differing": k, "of": rv.numel(), "max_rel": float(rel.max())})
    out = {"model": model, "images": n_img, "modules": len(ref), "step_sizes": n, "differing": bad, "worst_rel_diff": worst,
           "differing_entries": diffs, "reference_seconds": ref_s, "ours_seconds": ours_s, "speedup_wallclock": ref_s / ours_s,
           "config": f"configs/PTQ4ViT.py: W8A8, n_V=n_H={blocks} (qkv n_V x3, head 1), n_a=1, eq_n=100, 3 rounds, hessian; conv a_bit=32; "
                     "KL target perturbed by a harness hook on the net (oracle/ref_harness.add_target_noise) in both runs"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
