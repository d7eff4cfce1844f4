"""Time the frozen patch-embedding convolution against the unfrozen quant_forward on one GPU and print one JSON line.

    python tools/conv_bench.py [--images 8] [--reps 3] [--window 0.5] [--no-model]

Per patch embedding at an evaluation batch of 32 (W8, per-channel min-max step sizes, synthetic weights and images;
CUDA events over enough calls to fill `--window` seconds, after a warm-up, the three variants alternated `--reps` times,
medians reported): ViT-B/224, ViT-B/384, Swin-T/224 and Swin-B/384.  Variants: the unfrozen quant_forward with torch's
default (cuDNN may use TF32), the unfrozen quant_forward in strict FP32 (allow_tf32 off), and the frozen kernel.  For
each, the largest |out - ref| / bound against fp64 (DESIGN.md section 4.9), the bytes the frozen kernel must move
(image read, output written, packed weight read once) with their HBM bound at the H100 SXM data sheet's 3.35 TB/s, and
the bf16 tensor-core operations of the three term products with their bound at the data sheet's 989 TFLOP/s dense.
Then (unless --no-model) the whole quantised ViT-B/224 x 32 forward (calibrated on `--images` images as in
tools/forward_bench.py, PTQ4ViT), Linear and MatMul modules frozen and the attention fused, with the patch embedding
unfrozen and frozen, eager (host clock around a device synchronise) and replayed from one CUDA graph.  The card, its
power limit and max SM clock come from one read-only nvidia-smi query.  Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
os.environ.setdefault("TQDM_DISABLE", "1")

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import attention_bench as AB  # noqa: E402
import forward_bench as FB  # noqa: E402

BF16_DENSE_FLOPS = 989e12      # H100 SXM data sheet
WORKLOADS = {"vit_b224_x32": (768, 16, 224), "vit_b384_x32": (768, 16, 384), "swin_t224_x32": (96, 4, 224),
             "swin_b384_x32": (128, 4, 384)}


def _module(cout, k):
    from ptq4vit_b200.quant_layers.conv import ChannelwiseBatchingQuantConv2d
    g = torch.Generator().manual_seed(k + cout)
    m = ChannelwiseBatchingQuantConv2d(3, cout, k, stride=k, w_bit=8, a_bit=32, mode="quant_forward")
    m.weight.data = torch.randn(m.weight.shape, generator=g) * 0.02
    m.bias.data = torch.randn(cout, generator=g) * 0.05
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    m.w_interval = (m.weight.abs().amax(dim=(1, 2, 3)) / 127.5).reshape(cout, 1, 1, 1)
    m.calibrated = True
    return m


def _ratio(m, x, out):
    w_sim, b = m.quant_weight_bias()
    x64, w64 = x.double(), w_sim.double()
    ref = F.conv2d(x64, w64, b.double(), m.stride)
    mag = F.conv2d(x64.abs(), w64.abs(), None, m.stride)
    bound = (3 * w_sim[0].numel() + 2) * 2.0 ** -23 * mag + 2.0 ** -23 * ref.abs()
    return float(((out.double() - ref).abs() / bound.clamp_min(1e-300)).max())


def workload(name, a):
    cout, k, size = WORKLOADS[name]
    m = _module(cout, k)
    x = torch.randn(32, 3, size, size, generator=torch.Generator().manual_seed(3)).cuda()
    frozen = _module(cout, k).freeze()
    tf32_default = torch.backends.cudnn.allow_tf32

    def tf32():
        torch.backends.cudnn.allow_tf32 = tf32_default
        return m.quant_forward(x)

    def fp32():
        torch.backends.cudnn.allow_tf32 = False
        return m.quant_forward(x)

    variants = {"unfrozen_default": tf32, "unfrozen_fp32": fp32, "frozen": lambda: frozen.quant_forward(x)}
    out = {"workload": name, "out_channels": cout, "kernel": k, "image": size, "K": 3 * k * k}
    with torch.no_grad():
        for v, fn in variants.items():
            out[f"{v}_ratio"] = _ratio(m, x, fn())
            torch.backends.cudnn.allow_tf32 = tf32_default
        for fn in variants.values():          # warm-up
            FB.events_ms(fn, 0.05)
        runs = {v: [] for v in variants}
        for _ in range(a.reps):
            for v, fn in variants.items():
                runs[v].append(FB.events_ms(fn, a.window)[0])
        torch.backends.cudnn.allow_tf32 = tf32_default
    M = 32 * (size // k) ** 2
    nbytes = 4 * x.numel() + 4 * M * cout + frozen._packed.numel()
    flops = 2 * 3 * M * cout * 3 * k * k
    out.update({"bytes": nbytes, "hbm_bound_us": round(nbytes / FB.HBM_BYTES_PER_S * 1e6, 2), "bf16_flops": flops,
                "tensor_bound_us": round(flops / BF16_DENSE_FLOPS * 1e6, 2)})
    for v, r in runs.items():
        out[f"{v}_us"] = round(statistics.median(r) * 1e3, 2)
        out[f"{v}_runs_us"] = [round(t * 1e3, 2) for t in r]
    return out


def whole_model(a):
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d
    from ptq4vit_b200.utils import deploy
    net, wrapped = FB.calibrated_model("PTQ4ViT", a.images, 8)
    deploy.freeze_model(wrapped, matmul=True)
    deploy.fuse_attention(net)
    conv = next(m for m in wrapped.values() if isinstance(m, MinMaxQuantConv2d))
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    whole = {f"model_{s}{g}_ms": [] for s in ("conv_unfrozen", "conv_frozen") for g in ("", "_graph")}
    with torch.no_grad():
        graphs = {}
        for s in ("conv_unfrozen", "conv_frozen"):
            conv.freeze() if s == "conv_frozen" else conv.unfreeze()
            graphs[s] = AB._graph(lambda: net(batch))
        for _ in range(a.reps):
            for s in ("conv_unfrozen", "conv_frozen"):
                conv.freeze() if s == "conv_frozen" else conv.unfreeze()
                whole[f"model_{s}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{s}_graph_ms"].append(FB.wall_ms(graphs[s][0].replay, a.window)[0])
    return {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": 8, "reps": a.reps, "window_s": a.window}
    res["workloads"] = [workload(n, a) for n in WORKLOADS]
    if not a.no_model:
        res["vit_b224_x32_model"] = whole_model(a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
