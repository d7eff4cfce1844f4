"""Time the BasePTQ search of a ViT-B/224 on one GPU and print one JSON line.

    python tools/baseptq_search.py [--images 32] [--bit 8] [--runs 3] [--no-reference]

Workload: ptq4vit_b200.configs.BasePTQ with the Hessian metric (as example/test_all.py:53-78 runs it), W{bit}A{bit},
eq_n = 100, one round, 32 synthetic 224x224 images; every module's captured tensors stay resident on the device.  One
warm-up search, then `--runs` timed searches of all modules (CUDA events): the whole search, the time per module type
(patch-embedding conv, qkv, proj, fc1, fc2, head, matmul1, matmul2) and per kernel family (p4v_profile_collect_kinds).

Comparator: the UNMODIFIED reference classes (oracle/_ref, staged by build()) on the same GPU, one seeded layer of each
type at the same sizes (BatchingEasyQuantConv2d, PTQSLBatchingQuantLinear with n_V = 3 for qkv, PTQSLBatchingQuantMatMul),
extrapolated to the model by layer counts as bench.py's `reference_gpu` does.

The card, its power limit and its max SM clock are read by one nvidia-smi query; there is no CPU fallback."""
import argparse
import ctypes
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TQDM_DISABLE", "1")

import torch  # noqa: E402

MODEL = "vit_base_patch16_224"
TYPES = ("conv", "qkv", "proj", "fc1", "fc2", "head", "matmul1", "matmul2")


def module_type(name):
    leaf = name.rsplit(".", 1)[-1]
    return "conv" if leaf == "proj" and "patch_embed" in name else leaf


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, power, sm = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(power), "max_sm_mhz": float(sm)}
    except Exception as exc:          # the numbers stay valid; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "max_sm_mhz": None, "error": repr(exc)[:120]}


def build(images, bit):
    from ptq4vit_b200.configs import BasePTQ as cfg
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import get_net
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    importlib.reload(cfg)
    for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
        d["metric"] = "hessian"
    for d in (cfg.w_bit, cfg.a_bit, cfg.A_bit, cfg.B_bit):
        for k in d:
            d[k] = bit
    dev = torch.device("cuda", 0)
    net = get_net(MODEL, device=dev, seed=0)
    wrapped = wrap_modules_in_net(net, cfg)
    images_t = torch.randn(images, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    cal = Q.HessianQuantCalibrator(net, wrapped, [(images_t, None)], sequential=False, batch_size=4, target_noise=1.0)
    raw = cal._raw_pred_softmax()
    hooks = []
    for m in wrapped.values():
        hooks += cal._hooks_for(m)
    cal._fwd_bwd(raw)
    for h in hooks:
        h.remove()
    net.zero_grad(set_to_none=True)
    work = []
    for name, m in wrapped.items():
        Q._cat_captured(m)
        if isinstance(m.raw_input, list):
            t = dict(A=m.raw_input[0].contiguous(), B=m.raw_input[1].contiguous(), y=m.raw_out.contiguous(), g=m.raw_grad.contiguous())
        else:
            t = dict(x=m.raw_input.contiguous(), y=m.raw_out.contiguous(), g=m.raw_grad.contiguous())
        m.raw_input = m.raw_out = m.raw_grad = None
        work.append((name, m, t))
    torch.cuda.empty_cache()
    return work


def search(work):
    """One search of every module; returns ms per module type (CUDA events, one pair per module)."""
    ev = []
    for name, m, t in work:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if "x" in t:
            m.raw_input, m.raw_out, m.raw_grad = t["x"], t["y"], t["g"]
        else:
            m.raw_input, m.raw_out, m.raw_grad = [t["A"], t["B"]], t["y"], t["g"]
        e0.record()
        with torch.no_grad():
            m.calibration_step2()
        e1.record()
        ev.append((module_type(name), e0, e1))
    torch.cuda.synchronize()
    per = {k: 0.0 for k in TYPES}
    for k, e0, e1 in ev:
        per[k] += e0.elapsed_time(e1)
    return per


def reference(images, bit):
    """Seconds of the reference's calibration_step2() for one layer of every type (same sizes, one round)."""
    from oracle import ptq_oracle as O
    from oracle import ref_harness as RH
    from tests import _baseptq_ref as B
    D, H, tok = 768, 12, 197
    out = {}
    x, W, b, y, g = O.make_conv_fixture(90, images, 3, D, 224, 16)
    out["conv"] = B.run_conv_layerwise(x, W, b, y, g, stride=16, w_bit=bit, search_round=1)["seconds"]
    lin = {"qkv": (D, 3 * D, 3, False, tok), "proj": (D, D, 1, False, tok), "fc1": (D, 4 * D, 1, False, tok),
           "fc2": (4 * D, D, 1, True, tok), "head": (D, 1000, 1, False, 0)}
    for i, (name, (K, Oo, n_V, gelu, t)) in enumerate(lin.items()):
        x, W, b, y, g = O.make_linear_fixture(91 + i, images, t, K, Oo, post_gelu=gelu)
        out[name], _ = RH.time_linear(x, W, b, y, g, False, 100, w_blocks=None, search_round=1, n_V=n_V, n_H=1, n_a=1,
                                      w_bit=bit, a_bit=bit, eq_alpha=0.5)
    for i, (name, (S2, S3, softmax_A)) in enumerate({"matmul1": (D // H, tok, False), "matmul2": (tok, D // H, True)}.items()):
        A, Bm, Y, G = O.make_matmul_fixture(97 + i, images, H, tok, S2, S3, softmax_A=softmax_A)
        out[name], _ = RH.time_matmul(A, Bm, Y, G, False, 100, search_round=1, A_bit=bit, B_bit=bit, eq_alpha=0.5)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/baseptq_search.py needs a CUDA device (no CPU fallback)")
    torch.cuda.set_device(0)
    info = card()
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    work = build(a.images, a.bit)
    counts = {k: sum(module_type(n) == k for n, _, _ in work) for k in TYPES}
    search(work)                                            # warm-up
    runs = []
    for _ in range(a.runs):
        prof = (ctypes.c_double * 12)()
        lib.p4v_profile_collect_kinds(prof, 12)
        lib.p4v_profile_enable(1)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        per = search(work)
        e1.record(); torch.cuda.synchronize()
        lib.p4v_profile_enable(0)
        lib.p4v_profile_collect_kinds(prof, 12)
        runs.append({"total_ms": e0.elapsed_time(e1), "per_type_ms": per,
                     "kernel_ms": {"bf16_sweep": prof[0], "int8_sweep": prof[1], "gram_gemm": prof[2]},
                     "kernel_launches": {"bf16_sweep": int(prof[6]), "int8_sweep": int(prof[7]), "gram_gemm": int(prof[8])}})
    totals = [r["total_ms"] for r in runs]
    med = runs[sorted(range(len(runs)), key=lambda i: totals[i])[len(runs) // 2]]
    out = {"tool": "baseptq_search", "workload": f"{MODEL} {a.images} synthetic imgs, BasePTQ (hessian) W{a.bit}A{a.bit}, "
                                                 "eq_n 100, eq_alpha 0.5, one round, tensors resident",
           "card": info, "modules": counts, "search_s": statistics.median(totals) / 1e3,
           "search_s_spread": [min(totals) / 1e3, max(totals) / 1e3],
           "per_type_ms": {k: round(v, 2) for k, v in med["per_type_ms"].items()},
           "kernel_ms": {k: round(v, 2) for k, v in med["kernel_ms"].items()}, "kernel_launches": med["kernel_launches"],
           "runs": [round(t / 1e3, 4) for t in totals]}
    if not a.no_reference:
        from oracle import ref_harness as RH
        if RH.available():
            t0 = time.time()
            ref = reference(a.images, a.bit)
            job = sum(counts[k] * ref[k] for k in TYPES)
            out["reference_gpu"] = {"per_layer_s": {k: round(v, 3) for k, v in ref.items()},
                                    "extrapolated_search_s": round(job, 2), "speedup": round(job / out["search_s"], 1),
                                    "wall_s": round(time.time() - t0, 1)}
        else:
            out["reference_gpu"] = {"unavailable": "reference not staged under oracle/_ref"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
