"""Time the attention operands' quantisation folded into the frozen qkv against the frozen qkv followed by the fused
attention core, on one GPU, and print one JSON line.

    python tools/qkv_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--configs PTQ4ViT] [--models vit,swin]
                              [--no-sites]

Per block (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps` times,
medians reported), on frozen layers and MatMul modules with min-max step sizes and synthetic activations:
  * ViT-B/224 x 32 (6304 rows, 197 tokens, 12 heads): qkv 768 -> 2304, PTQ4ViT-shaped (24 blocks, split-of-softmax
    matmul2) and BasePTQ-shaped (one block, plain matmul2);
  * Swin-T/224 x 32 stage 1 (100352 rows, 49 tokens, 3 heads): the window gather (norm1, roll, partition) folded into
    qkv 96 -> 288, shift 0 and 3 (relative-position bias; the shifted block's mask);
  * Swin-B/384 x 32 stage 1 (294912 rows, 144 tokens, 4 heads): qkv 128 -> 384, the window gather folded, shift 0.
unfused = frozen qkv (FP32 output) then frozen_attention; fused = frozen_qkv_attention (int8 planes).  Each row's HBM
bound is the bytes the folded call must move (x read, the planes written and read once, the attention output written);
`unfused_bytes` has the FP32 qkv output written and read once instead.  Then the whole quantised ViT-B/224 x 32 and
Swin-T/224 x 32 forwards of each configuration (calibrated on `--images` images as in tools/forward_bench.py) with Linear,
MatMul and conv modules frozen and every other fusion on, with and without deploy.fuse_qkv, eager (host clock around a
device synchronise) and replayed from one CUDA graph.  The card, its power limit and its max SM clock come from one
read-only nvidia-smi query.  Needs a CUDA device."""
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

import attention_bench as AB  # noqa: E402
import forward_bench as FB  # noqa: E402
import mlp_bench as MB  # noqa: E402
import residual_bench as RB  # noqa: E402


def _norm(C):
    ln = torch.nn.LayerNorm(C).cuda()
    for p in ln.parameters():
        p.requires_grad_(False)
    return ln


def block(name, images, tokens, C, H, n_H, m2_cls, a, window=None):
    """One attention call; window: (res, ws, shift) of a Swin block whose norm1, roll and partition fold into qkv."""
    from ptq4vit_b200.quant_layers.linear import frozen_gather_linear
    from ptq4vit_b200.quant_layers.matmul import frozen_attention, frozen_qkv_applies, frozen_qkv_attention
    g = torch.Generator().manual_seed(5)
    D = C // H
    scale = D ** -0.5
    with torch.no_grad():
        if window is None:
            x = torch.randn(images, tokens, C, generator=g).cuda()
            norm = gather = bias = mask = None
            qkv = MB._frozen(C, 3 * C, n_H, False, a.bit, x, 1)
            y = qkv(x)
        else:
            res, ws, shift = window
            x = torch.randn(images, res * res, C, generator=g).cuda()
            norm, gather = _norm(C), (images, res, res, ws, shift)
            qkv = MB._frozen(C, 3 * C, n_H, False, a.bit, norm(x), 1)
            y = frozen_gather_linear(norm, qkv, x, ("window", *gather))
            nW = (res // ws) ** 2
            bias = (torch.randn(H, tokens, tokens, generator=g) * 0.5).cuda()
            mask = None
            if shift:
                grp = torch.randint(0, 3, (nW, tokens), generator=g)
                mask = torch.where(grp[:, :, None] == grp[:, None, :], 0.0, -100.0).cuda()
        B = y.numel() // (tokens * 3 * C)
        qkv5 = y.view(B, tokens, 3, H, D)
        m1, m2 = AB._minmax_pair(qkv5 * torch.tensor([scale if window else 1.0, 1.0, 1.0], device="cuda").view(1, 1, 3, 1, 1),
                                 scale, m2_cls, a.bit)
        del y, qkv5
        assert frozen_qkv_applies(qkv, m1, m2, x, tokens, H, D, bias, mask, norm=norm, gather=gather), f"{name}: no fold"
        so = window is not None

        def unfused():
            yy = qkv(x) if window is None else frozen_gather_linear(norm, qkv, x, ("window", *gather))
            return frozen_attention(m1, m2, yy.view(B, tokens, 3, H, D), scale, so, bias=bias, mask=mask)

        def fused():
            return frozen_qkv_attention(qkv, m1, m2, x, tokens, H, D, scale, so, bias=bias, mask=mask, norm=norm, gather=gather)
        identical = RB._bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    rows = B * tokens
    extra = 4 * (0 if bias is None else bias.numel()) + 4 * (0 if mask is None else mask.numel())
    fused_bytes = 4 * rows * C + 2 * 3 * rows * C + 4 * rows * C + extra
    unfused_bytes = 4 * rows * C + 2 * 4 * 3 * rows * C + 4 * rows * C + extra
    out = AB._report(runs, fused_bytes, {"block": name, "rows": rows, "tokens": tokens, "heads": H, "matmul2": m2_cls,
                                          "bit_identical": identical})
    out["unfused_bytes"] = unfused_bytes
    out["unfused_hbm_bound_ms"] = round(unfused_bytes / FB.HBM_BYTES_PER_S * 1e3, 4)
    del x, qkv, m1, m2
    torch.cuda.empty_cache()
    return out


def whole_model(model, config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped = RB._calibrated(model, config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True, conv=True)
    for fuse in (deploy.fuse_attention, deploy.fuse_mlp, deploy.fuse_norm, deploy.fuse_residual, deploy.fuse_gather,
                 deploy.fuse_stem):
        fuse(net)
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"model": model, "config": config}
    with torch.no_grad():
        logits = net(batch)
        out["left_unfolded"] = deploy.fuse_qkv(net)
        out["model_bit_identical"] = RB._bits_equal(net(batch), logits)
        whole = {"model_unfolded_ms": [], "model_folded_ms": [], "model_unfolded_graph_ms": [], "model_folded_graph_ms": []}
        graphs = {}
        for mode in ("unfolded", "folded"):
            (deploy.fuse_qkv if mode == "folded" else deploy.unfuse_qkv)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        for _ in range(a.reps):
            for mode in ("unfolded", "folded"):
                (deploy.fuse_qkv if mode == "folded" else deploy.unfuse_qkv)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_qkv(net)
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
    ap.add_argument("--configs", default="PTQ4ViT")
    ap.add_argument("--models", default="vit,swin")
    ap.add_argument("--no-sites", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qkv_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    if not a.no_sites:
        sos, plain = "SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"
        res["blocks"] = [block("vit_b224_x32_ptq4vit", 32, 197, 768, 12, 24, sos, a),
                         block("vit_b224_x32_baseptq", 32, 197, 768, 12, 1, plain, a),
                         block("swin_t_stage1_x32_shift0", 32, 49, 96, 3, 3, sos, a, window=(56, 7, 0)),
                         block("swin_t_stage1_x32_shift3", 32, 49, 96, 3, 3, sos, a, window=(56, 7, 3)),
                         block("swin_b384_stage1_x32_shift0", 32, 144, 128, 4, 4, sos, a, window=(96, 12, 0))]
    res["models"] = [whole_model(RB.MODELS[m], c, a) for m in a.models.split(",") if m for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
