"""Time Swin's row gathers folded into the frozen Linear that consumes them against torch's ops followed by the frozen
call, on one GPU, and print one JSON line.

    python tools/gather_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--configs PTQ4ViT] [--models swin_t,swin_b384]

Per fold site (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps`
times, medians reported, outputs compared bitwise in the same run), on frozen layers with min-max step sizes and
synthetic activations:
  * the window gather: torch's LayerNorm, roll (shifted blocks), window partition copy and the frozen qkv against the
    folded qkv, at Swin-T/224 x 32 stage 1 (shift 0 and 3), Swin-T/224 x 32 stage 3 (shift 3) and Swin-B/384 x 32
    stage 1 (shift 6);
  * the merge gather: torch's cat of PatchMerging followed by the folded norm -> reduction (fuse_norm's path) against
    the folded merge, at Swin-T/224 x 32's first two PatchMerging layers.
Each site's HBM bound is the bytes the folded call must move (the image read once, the output written) at the H100 SXM
data sheet's 3.35 TB/s; `unfused_bytes` adds what each torch pass writes and the next reads.  Then the whole quantised
forwards (calibrated on `--images` images as in tools/forward_bench.py, at the model's resolution, batch 32) with Linear,
MatMul and conv modules frozen and fuse_attention, fuse_mlp, fuse_norm and fuse_residual on, with and without
deploy.fuse_gather, eager (host clock around a device synchronise) and replayed from one CUDA graph.  The card, its
power limit and its max SM clock come from one read-only nvidia-smi query.  Needs a CUDA device."""
import argparse
import importlib
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


def _bits_equal(a, b):
    return bool(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)))


def _layer_norm(C, seed):
    ln = torch.nn.LayerNorm(C).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.2 * torch.randn(C, generator=g))
        ln.bias.copy_(0.1 * torch.randn(C, generator=g))
    for p in ln.parameters():
        p.requires_grad_(False)
    return ln


def window_site(name, images, C, res, ws, shift, a):
    from ptq4vit_b200.quant_layers.linear import frozen_gather_applies, frozen_gather_linear
    from ptq4vit_b200.utils.models import _window_partition
    g = torch.Generator().manual_seed(5)
    gather = ("window", images, res, res, ws, shift)
    with torch.no_grad():
        x = torch.randn(images, res * res, C, generator=g).cuda()
        norm = _layer_norm(C, 6)
        lin = MB._frozen(C, 3 * C, max(1, C // 32), False, a.bit, norm(x), 2)
        assert frozen_gather_applies(norm, lin, x, gather), f"{name}: the fold does not apply"

        def unfused():
            h = norm(x).view(images, res, res, C)
            if shift:
                h = torch.roll(h, shifts=(-shift, -shift), dims=(1, 2))
            return lin(_window_partition(h, ws))

        def fused():
            return frozen_gather_linear(norm, lin, x, gather)
        identical = _bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    rows = images * res * res
    fused_bytes = 4 * rows * C + 4 * rows * 3 * C
    passes = 2 + (1 if shift else 0)          # LayerNorm, roll, partition: each writes the activations, the next reads
    out = AB._report(runs, fused_bytes, {"site": name, "rows": rows, "shape": [C, 3 * C], "shift": shift,
                                         "bit_identical": identical})
    out["unfused_bytes"] = fused_bytes + passes * 2 * 4 * rows * C
    out["unfused_hbm_bound_ms"] = round(out["unfused_bytes"] / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def merge_site(name, images, C, res, a):
    from ptq4vit_b200.quant_layers.linear import frozen_gather_applies, frozen_gather_linear, frozen_norm_linear
    g = torch.Generator().manual_seed(5)
    gather = ("merge", images, res, res, 0, 0)
    with torch.no_grad():
        x = torch.randn(images, res * res, C, generator=g).cuda()
        norm = _layer_norm(4 * C, 6)

        def cat():
            h = x.view(images, res, res, C)
            return torch.cat([h[:, 0::2, 0::2], h[:, 1::2, 0::2], h[:, 0::2, 1::2], h[:, 1::2, 1::2]], -1).view(images, -1, 4 * C)
        m = MB._frozen(4 * C, 2 * C, 1, False, a.bit, norm(cat()), 2)
        assert frozen_gather_applies(norm, m, x, gather), f"{name}: the fold does not apply"

        def unfused():
            return frozen_norm_linear(norm, m, cat())

        def fused():
            return frozen_gather_linear(norm, m, x, gather)
        identical = _bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    rows = images * res * res // 4
    fused_bytes = 4 * rows * 4 * C + 4 * rows * 2 * C
    out = AB._report(runs, fused_bytes, {"site": name, "rows": rows, "shape": [4 * C, 2 * C], "bit_identical": identical})
    out["unfused_bytes"] = fused_bytes + 2 * 4 * rows * 4 * C
    out["unfused_hbm_bound_ms"] = round(out["unfused_bytes"] / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def _calibrated(model, config, images, bit):
    """forward_bench.calibrated_model for a Swin model of the zoo, calibrated at its own resolution"""
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import _SWIN_ZOO, get_net
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
            d["metric"] = "hessian"
    for d in (cfg.w_bit, cfg.a_bit, cfg.A_bit, cfg.B_bit):
        for k in d:
            d[k] = bit
    size = _SWIN_ZOO[model]["img_size"]
    net = get_net(model, device=torch.device("cuda", 0), seed=0)
    wrapped = wrap_modules_in_net(net, cfg)
    calib = torch.randn(images, 3, size, size, generator=torch.Generator().manual_seed(3))
    Q.HessianQuantCalibrator(net, wrapped, [(calib, None)], sequential=False, batch_size=4, target_noise=1.0).batching_quant_calib()
    torch.cuda.synchronize()
    return net, wrapped, size


def whole_model(model, config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped, size = _calibrated(model, config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True, conv=True)
    deploy.fuse_attention(net)
    deploy.fuse_mlp(net)
    deploy.fuse_norm(net)
    deploy.fuse_residual(net)
    batch = torch.randn(32, 3, size, size, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"model": model, "config": config}
    with torch.no_grad():
        logits = net(batch)
        out["left_unfolded"] = deploy.fuse_gather(net)
        out["model_bit_identical"] = _bits_equal(net(batch), logits)
        whole = {"model_unfolded_ms": [], "model_folded_ms": [], "model_unfolded_graph_ms": [], "model_folded_graph_ms": []}
        graphs = {}
        for mode in ("unfolded", "folded"):
            (deploy.fuse_gather if mode == "folded" else deploy.unfuse_gather)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        out["graph_bit_identical"] = _bits_equal(graphs["unfolded"][1], graphs["folded"][1])
        for _ in range(a.reps):
            for mode in ("unfolded", "folded"):
                (deploy.fuse_gather if mode == "folded" else deploy.unfuse_gather)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_gather(net)
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, graphs
    torch.cuda.empty_cache()
    return out


MODELS = {"swin_t": "swin_tiny_patch4_window7_224", "swin_b384": "swin_base_patch4_window12_384"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--configs", default="PTQ4ViT")
    ap.add_argument("--models", default="swin_t,swin_b384")
    ap.add_argument("--no-sites", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gather_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    if not a.no_sites:
        res["sites"] = [window_site("swin_t224_x32_stage1_qkv_shift0", 32, 96, 56, 7, 0, a),
                        window_site("swin_t224_x32_stage1_qkv_shift3", 32, 96, 56, 7, 3, a),
                        window_site("swin_t224_x32_stage3_qkv_shift3", 32, 384, 14, 7, 3, a),
                        window_site("swin_b384_x32_stage1_qkv_shift6", 32, 128, 96, 12, 6, a),
                        merge_site("swin_t224_x32_merge1", 32, 96, 56, a),
                        merge_site("swin_t224_x32_merge2", 32, 192, 28, a)]
    res["models"] = [whole_model(MODELS[m], c, a) for m in a.models.split(",") if m for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
