"""Time a block's residual add folded into the frozen Linear that produces it against the frozen Linear followed by
torch's ops, on one GPU, and print one JSON line.

    python tools/residual_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--configs PTQ4ViT] [--models vit,swin]

Per fold site (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps`
times, medians reported), on frozen layers with min-max step sizes and synthetic activations:
  * ViT-B/224 x 32 (6304 rows): attn.proj (768 -> 768, fused path) and mlp.fc2 (3072 -> 768, streamed path), PTQ4ViT
    (24 x 24 blocks, post-GELU fc2) and BasePTQ (one block); fc2 inside the fused MLP (fc1 -> GELU -> fc2);
  * Swin-T/224 x 32 stage 1 (100352 rows): attn.proj with the window layout at shift 0 and 3 (unfolded: window reverse,
    roll, add) and mlp.fc2 (384 -> 96, fused path).
unfused = the frozen call then torch's ops; fused = the folded call.  Each row's HBM bound is the bytes the folded call
must move (x read, the shortcut read, the output written; on the streamed path also the int8 activation image written
and read) at the H100 SXM data sheet's 3.35 TB/s; `unfused_bytes` adds the Linear's FP32 output written and read by
each torch op.  Then the whole quantised ViT-B/224 x 32 and Swin-T/224 x 32 forwards of each configuration (calibrated
on `--images` images as in tools/forward_bench.py) with Linear, MatMul and conv modules frozen and fuse_attention,
fuse_mlp and fuse_norm on, with and without deploy.fuse_residual, eager (host clock around a device synchronise) and
replayed from one CUDA graph.  The card, its power limit and its max SM clock come from one read-only nvidia-smi query.
Needs a CUDA device."""
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
import mlp_bench as MB  # noqa: E402


def _bits_equal(a, b):
    return bool(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)))


def _unwindow(y, layout):
    from ptq4vit_b200.utils.models import _window_reverse
    images, H, W, ws, shift = layout
    h = _window_reverse(y, ws, H, W)
    if shift:
        h = torch.roll(h, shifts=(shift, shift), dims=(1, 2))
    return h.view(images, H * W, -1)


def site(name, rows, K, O, n_H, post_gelu, a, layout=None, mlp=None):
    """One fold site; layout: Swin's window layout of proj; mlp: (fc1's K, fc1's n_H) of a fused MLP whose fc2 this is."""
    from ptq4vit_b200.quant_layers.linear import frozen_mlp, frozen_residual_applies, frozen_residual_linear
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        if mlp is not None:
            x = torch.randn(rows, mlp[0], generator=g).cuda()
            fc1 = MB._frozen(mlp[0], K, mlp[1], False, a.bit, x, 1)
            lin = MB._frozen(K, O, n_H, post_gelu, a.bit, F.gelu(fc1(x)), 2)
        else:
            x = (torch.randn(rows, K, generator=g) * 2.0).cuda()
            if post_gelu:
                x = F.gelu(x)
            lin = MB._frozen(K, O, n_H, post_gelu, a.bit, x, 2)
        if layout is not None:
            x = x.view(-1, layout[3] ** 2, K)
            res = torch.randn(layout[0], layout[1] * layout[2], O, generator=g).cuda()
        else:
            res = torch.randn(rows, O, generator=g).cuda()
        assert frozen_residual_applies(lin, x, res, layout), f"{name}: the fold does not apply"

        if mlp is not None:
            def unfused():
                return res + frozen_mlp(fc1, lin, x)

            def fused():
                return frozen_mlp(fc1, lin, x, residual=res)
        elif layout is not None:
            def unfused():
                return res + _unwindow(lin(x), layout)

            def fused():
                return frozen_residual_linear(lin, x, res, layout)
        else:
            def unfused():
                return res + lin(x)

            def fused():
                return frozen_residual_linear(lin, x, res)
        identical = _bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    streamed = mlp is not None or not lin._frozen_fused
    planes = 2 if post_gelu else 1
    fused_bytes = 4 * rows * K + 2 * 4 * rows * O + (2 * rows * K * planes if streamed else 0)
    if mlp is not None:           # fc1's input instead of fc2's, and fc2's image written by fc1 and read by fc2
        fused_bytes += 4 * rows * mlp[0] - 4 * rows * K
    passes = 1 + (1 if layout is not None else 0) + (1 if layout is not None and layout[4] else 0)
    unfused_bytes = fused_bytes + passes * 2 * 4 * rows * O
    out = AB._report(runs, fused_bytes, {"site": name, "rows": rows, "shape": [K, O], "path": "streamed" if streamed else "fused",
                                         "bit_identical": identical})
    out["unfused_bytes"] = unfused_bytes
    out["unfused_hbm_bound_ms"] = round(unfused_bytes / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def _calibrated(model, config, images, bit):
    """forward_bench.calibrated_model for another model of the zoo"""
    old = FB.MODEL
    FB.MODEL = model
    try:
        return FB.calibrated_model(config, images, bit)
    finally:
        FB.MODEL = old


def whole_model(model, config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped = _calibrated(model, config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True, conv=True)
    deploy.fuse_attention(net)
    deploy.fuse_mlp(net)
    deploy.fuse_norm(net)
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"model": model, "config": config}
    with torch.no_grad():
        logits = net(batch)
        out["left_unfolded"] = deploy.fuse_residual(net)
        out["model_bit_identical"] = _bits_equal(net(batch), logits)
        whole = {"model_unfolded_ms": [], "model_folded_ms": [], "model_unfolded_graph_ms": [], "model_folded_graph_ms": []}
        graphs = {}
        for mode in ("unfolded", "folded"):
            (deploy.fuse_residual if mode == "folded" else deploy.unfuse_residual)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        for _ in range(a.reps):
            for mode in ("unfolded", "folded"):
                (deploy.fuse_residual if mode == "folded" else deploy.unfuse_residual)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_residual(net)
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, graphs
    torch.cuda.empty_cache()
    return out


MODELS = {"vit": "vit_base_patch16_224", "swin": "swin_tiny_patch4_window7_224"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--configs", default="PTQ4ViT")
    ap.add_argument("--models", default="vit,swin")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("residual_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    swin_rows = 32 * 3136
    res["sites"] = [site("vit_b224_x32_proj_ptq4vit", 6304, 768, 768, 24, False, a),
                    site("vit_b224_x32_proj_baseptq", 6304, 768, 768, 1, False, a),
                    site("vit_b224_x32_fc2_ptq4vit", 6304, 3072, 768, 24, True, a),
                    site("vit_b224_x32_fc2_baseptq", 6304, 3072, 768, 1, False, a),
                    site("vit_b224_x32_fc2_fused_mlp", 6304, 3072, 768, 24, True, a, mlp=(768, 24)),
                    site("swin_t_stage1_x32_proj_shift0", swin_rows, 96, 96, 3, False, a, layout=(32, 56, 56, 7, 0)),
                    site("swin_t_stage1_x32_proj_shift3", swin_rows, 96, 96, 3, False, a, layout=(32, 56, 56, 7, 3)),
                    site("swin_t_stage1_x32_fc2", swin_rows, 384, 96, 12, True, a)]
    res["models"] = [whole_model(MODELS[m], c, a) for m in a.models.split(",") if m for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
