"""Time a LayerNorm folded into its frozen Linear against torch's LayerNorm followed by the frozen Linear, on one GPU, and
print one JSON line.

    python tools/norm_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--configs PTQ4ViT,BasePTQ]

Per fold site (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps`
times, medians reported), on frozen layers with min-max step sizes, an affine LayerNorm and synthetic activations:
  * ViT-B/224 x 32 (6304 rows): norm1 -> qkv (768 -> 2304), norm2 -> fc1 (768 -> 3072), norm2 -> fc1 -> GELU -> fc2 with
    the fused MLP (unfolded: torch's LayerNorm, then frozen_mlp), final norm -> head on the 32 cls rows (unfolded: the
    LayerNorm of all 6304 rows, as the model runs it);
  * Swin-T/224 x 32 stage 1: norm2 -> fc1 (100352 rows, 96 -> 384) and the first PatchMerging, norm -> reduction
    (25088 rows, 384 -> 192; with a bias here).
unfused = F.layer_norm then the frozen Linear (frozen_mlp); fused = the folded call.  Each row's HBM bound is the bytes the
folded call must move (x read, the output written; the MLP also fc2's image written and read) at the H100 SXM data
sheet's 3.35 TB/s; `unfused_bytes` adds the normalised FP32 tensor written and read.  torch's LayerNorm alone is timed
too.  Then the whole quantised ViT-B/224 x 32 forward of each configuration (calibrated on `--images` images as in
tools/forward_bench.py) with Linear, MatMul and conv modules frozen and the attention fused, with and without
deploy.fuse_norm, eager (host clock around a device synchronise) and replayed from one CUDA graph.  The card, its power
limit and its max SM clock come from one read-only nvidia-smi query.  Needs a CUDA device."""
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


def _norm(K, seed):
    g = torch.Generator().manual_seed(seed)
    ln = torch.nn.LayerNorm(K, eps=1e-6)
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.2 * torch.randn(K, generator=g))
        ln.bias.copy_(0.1 * torch.randn(K, generator=g))
    return ln.cuda().requires_grad_(False)


def _bits_equal(a, b):
    return bool(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)))


def site(name, rows, K, O, n_H, a, tokens=None, mlp=None):
    """One fold site; tokens: the head (normalise all rows unfolded, only the cls rows folded); mlp: (hidden n_H, post-GELU)
    of a fused MLP whose fc1 the norm folds into."""
    from ptq4vit_b200.quant_layers.linear import frozen_mlp, frozen_norm_applies, frozen_norm_linear
    x = (torch.randn(rows, K, generator=torch.Generator().manual_seed(5)) * 2.0).cuda()
    ln = _norm(K, 1)
    with torch.no_grad():
        lin = MB._frozen(K, O, n_H, False, a.bit, F.layer_norm(x, (K,), ln.weight, ln.bias, ln.eps), 2)
        fc2 = None
        if mlp is not None:
            fc2 = MB._frozen(O, K, mlp[0], mlp[1], a.bit, F.gelu(lin(ln(x))), 3)
        x3 = x.view(rows // tokens, tokens, K) if tokens else x
        assert frozen_norm_applies(ln, lin, x3), f"{name}: the fold does not apply"

        if fc2 is not None:
            def unfused():
                return frozen_mlp(lin, fc2, ln(x))

            def fused():
                return frozen_mlp(lin, fc2, x, norm=ln)
        elif tokens:
            def unfused():
                return lin(ln(x3)[:, 0])

            def fused():
                return frozen_norm_linear(ln, lin, x3[:, 0])
        else:
            def unfused():
                return lin(ln(x))

            def fused():
                return frozen_norm_linear(ln, lin, x)
        identical = _bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    m = rows // tokens if tokens else rows
    if fc2 is not None:
        planes = 2 if mlp[1] else 1
        fused_bytes = 4 * rows * K + 2 * rows * O * planes + 4 * rows * K
    else:
        fused_bytes = 4 * m * K + 4 * m * O
    unfused_bytes = fused_bytes + 2 * 4 * rows * K + (4 * rows * K if tokens else 0)
    out = AB._report(runs, fused_bytes, {"site": name, "rows": m, "shape": [K, O], "bit_identical": identical})
    out["unfused_bytes"] = unfused_bytes
    out["unfused_hbm_bound_ms"] = round(unfused_bytes / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def layer_norm_alone(rows, K, a):
    x = torch.randn(rows, K, device="cuda")
    ln = _norm(K, 4)
    fn = lambda: F.layer_norm(x, (K,), ln.weight, ln.bias, ln.eps)   # noqa: E731
    with torch.no_grad():
        FB.events_ms(fn, 0.05)
        ms = [FB.events_ms(fn, a.window)[0] for _ in range(a.reps)]
    nbytes = 2 * 4 * x.numel()
    bound = nbytes / FB.HBM_BYTES_PER_S * 1e3
    return {"shape": [rows, K], "bytes": nbytes, "hbm_bound_ms": round(bound, 4), "ms": round(statistics.median(ms), 4),
            "share_of_hbm_bound": round(bound / statistics.median(ms), 3), "runs_ms": [round(v, 4) for v in ms]}


def whole_model(config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped = FB.calibrated_model(config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True, conv=True)
    deploy.fuse_attention(net)
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"config": config}
    with torch.no_grad():
        logits = net(batch)
        out["left_unfolded"] = deploy.fuse_norm(net)
        out["model_bit_identical"] = _bits_equal(net(batch), logits)
        whole = {"model_unfolded_ms": [], "model_folded_ms": [], "model_unfolded_graph_ms": [], "model_folded_graph_ms": []}
        graphs = {}
        for mode in ("unfolded", "folded"):
            (deploy.fuse_norm if mode == "folded" else deploy.unfuse_norm)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        for _ in range(a.reps):
            for mode in ("unfolded", "folded"):
                (deploy.fuse_norm if mode == "folded" else deploy.unfuse_norm)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_norm(net)
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
        raise SystemExit("norm_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    res["sites"] = [site("vit_b224_x32_qkv", 6304, 768, 2304, 24, a),
                    site("vit_b224_x32_fc1", 6304, 768, 3072, 24, a),
                    site("vit_b224_x32_fc1_fused_mlp", 6304, 768, 3072, 24, a, mlp=(24, True)),
                    site("vit_b224_x32_head_cls", 6304, 768, 1000, 24, a, tokens=197),
                    site("swin_t_stage1_x32_fc1", 32 * 3136, 96, 384, 3, a),
                    site("swin_t_merge1_x32_reduction", 32 * 784, 384, 192, 3, a)]
    res["layer_norm_alone"] = [layer_norm_alone(6304, 768, a), layer_norm_alone(32 * 3136, 96, a)]
    res["models"] = [whole_model(c, a) for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
