"""Time the fused frozen MLP against the unfused frozen sequence on one GPU and print one JSON line.

    python tools/mlp_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--configs PTQ4ViT,BasePTQ]

Per MLP block (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps`
times, medians reported), on frozen layers with min-max step sizes and synthetic activations:
  * ViT-B/224 x 32 (6304 rows, 768 -> 3072 -> 768), PTQ4ViT (post-GELU fc2: two int8 planes) and BasePTQ (one plane);
  * Swin-T/224 stage 1 x 32 (100352 rows, 96 -> 384 -> 96; fc2 runs the fused Linear kernel on its own).
unfused = frozen fc1, torch's GELU, frozen fc2 (on its own path); fused = one quant_layers.linear.frozen_mlp call.  Each
block's HBM bound is the bytes each design must move (x read, fc2's image written and read, the output written; the
unfused one also writes and reads the FP32 hidden tensor twice) at the H100 SXM data sheet's 3.35 TB/s.  The GELU pass
alone ([6304, 3072] fp32) is timed too.  Then the whole quantised ViT-B forward of each configuration (calibrated on
`--images` images as in tools/forward_bench.py) with Linear and MatMul modules frozen and the attention fused, with and
without deploy.fuse_mlp, eager (host clock around a device synchronise) and replayed from one CUDA graph.  The card, its
power limit and its max SM clock come from one read-only nvidia-smi query.  Needs a CUDA device."""
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


def _frozen(K, O, n_H, post_gelu, bit, x, seed):
    """A frozen layer with min-max step sizes for the activations x it will see."""
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear, PTQSLBatchingQuantLinear
    g = torch.Generator().manual_seed(seed)
    m = (PostGeluPTQSLBatchingQuantLinear if post_gelu else PTQSLBatchingQuantLinear)(K, O, w_bit=bit, a_bit=bit, n_H=n_H)
    m.weight.data = torch.randn(O, K, generator=g) * K ** -0.5
    m.bias.data = torch.randn(O, generator=g) * 0.1
    m = m.cuda()
    q = 2 ** (bit - 1) - 0.5
    m.w_interval = (m.weight.data.view(1, O, n_H, K // n_H).abs().amax(dim=(1, 3)) / q).view(1, 1, n_H, 1)
    m.a_interval = (x.abs().max() / q).reshape(1, 1)
    m.calibrated = True
    m.mode = "quant_forward"
    for p in m.parameters():
        p.requires_grad_(False)
    return m.freeze()


def block(name, rows, K, H, n_H1, n_H2, post_gelu, a):
    from ptq4vit_b200.quant_layers.linear import frozen_mlp
    x = torch.randn(rows, K, generator=torch.Generator().manual_seed(5)).cuda()
    with torch.no_grad():
        fc1 = _frozen(K, H, n_H1, False, a.bit, x, 1)
        h = F.gelu(fc1(x))
        fc2 = _frozen(H, K, n_H2, post_gelu, a.bit, h, 2)
        del h

        def unfused():
            return fc2(F.gelu(fc1(x)))

        def fused():
            return frozen_mlp(fc1, fc2, x)
        identical = bool(torch.equal(unfused().view(torch.int32), fused().view(torch.int32)))
        runs = AB._time_pair(unfused, fused, a)
    planes = 2 if post_gelu else 1
    img = rows * H * planes                       # fc2's int8 image (segments of these shapes need no padding)
    fused_bytes = 4 * rows * K + 2 * img + 4 * rows * K
    unfused_bytes = 4 * rows * K + 4 * 4 * rows * H + (2 * img if not fc2._frozen_fused else 0) + 4 * rows * K
    out = AB._report(runs, fused_bytes, {"block": name, "rows": rows, "shape": [K, H, K], "fc2_planes": planes,
                                          "fc2_own_path": "fused" if fc2._frozen_fused else "streamed",
                                          "bit_identical": identical})
    out["unfused_bytes"] = unfused_bytes
    out["unfused_hbm_bound_ms"] = round(unfused_bytes / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def gelu_pass(a):
    h = torch.randn(6304, 3072, device="cuda")
    fn = lambda: F.gelu(h)   # noqa: E731
    FB.events_ms(fn, 0.05)
    ms = [FB.events_ms(fn, a.window)[0] for _ in range(a.reps)]
    nbytes = 2 * 4 * h.numel()
    bound = nbytes / FB.HBM_BYTES_PER_S * 1e3
    return {"shape": list(h.shape), "bytes": nbytes, "hbm_bound_ms": round(bound, 4), "ms": round(statistics.median(ms), 4),
            "share_of_hbm_bound": round(bound / statistics.median(ms), 3), "runs_ms": [round(v, 4) for v in ms]}


def whole_model(config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped = FB.calibrated_model(config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True)
    deploy.fuse_attention(net)
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"config": config}
    with torch.no_grad():
        logits = net(batch)
        whole = {"model_unfused_ms": [], "model_fused_ms": [], "model_unfused_graph_ms": [], "model_fused_graph_ms": []}
        graphs = {}
        for mode in ("unfused", "fused"):
            (deploy.fuse_mlp if mode == "fused" else deploy.unfuse_mlp)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        deploy.fuse_mlp(net)
        out["model_bit_identical"] = bool(torch.equal(net(batch).view(torch.int32), logits.view(torch.int32)))
        for _ in range(a.reps):
            for mode in ("unfused", "fused"):
                (deploy.fuse_mlp if mode == "fused" else deploy.unfuse_mlp)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_mlp(net)
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, graphs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--configs", default="PTQ4ViT,BasePTQ")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mlp_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    res["blocks"] = [block("vit_b224_x32_ptq4vit", 6304, 768, 3072, 24, 24, True, a),
                     block("vit_b224_x32_baseptq", 6304, 768, 3072, 1, 1, False, a),
                     block("swin_t_stage1_x32", 32 * 3136, 96, 384, 3, 12, True, a)]
    res["gelu_pass"] = gelu_pass(a)
    res["models"] = [whole_model(c, a) for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
