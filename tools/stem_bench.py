"""Time the patch embedding's token epilogue folded into the frozen conv against the frozen conv followed by torch's stem
ops, on one GPU, and print one JSON line.

    python tools/stem_bench.py [--images 8] [--bit 8] [--reps 3] [--window 0.5] [--models vit_b,swin_t] [--no-sites]

Per stem (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated `--reps` times,
medians reported, outputs compared bitwise in the same run), on a frozen conv with min-max step sizes and synthetic
images, 32 images each: ViT-B/224 and ViT-B/384 (flatten, transpose, cat with the cls token, + pos_embed) and Swin-T/224
and Swin-B/384 (flatten, transpose, patch_norm).  The bytes model: `conv_out_bytes` is the conv's NCHW output,
`stem_ops_bytes` what torch's stem ops read and write after it (four times that output: the transposing copy reads and
writes it, the add or LayerNorm reads and writes it again), `bytes` what the folded call must move (the image read once,
the token rows written); the bounds are those over the H100 SXM data sheet's 3.35 TB/s.  Then the whole quantised
forwards of ViT-B/224 and Swin-T/224 x 32 (calibrated on `--images` images as in tools/forward_bench.py) with Linear,
MatMul and conv modules frozen and fuse_attention, fuse_mlp, fuse_norm, fuse_residual and fuse_gather on, with and
without deploy.fuse_stem, eager (host clock around a device synchronise) and replayed from one CUDA graph.  The card, its
power limit and its max SM clock come from one read-only nvidia-smi query in the same run.  Needs a CUDA device."""
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


def _bits_equal(a, b):
    return bool(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)))


def _frozen_conv(C, patch, bit, seed=5):
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d
    g = torch.Generator().manual_seed(seed)
    m = MinMaxQuantConv2d(3, C, patch, stride=patch, w_bit=bit, a_bit=32)
    m.weight.data = torch.randn(C, 3, patch, patch, generator=g) * 0.02
    m.bias.data = torch.randn(C, generator=g) * 0.02
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    m.w_interval = (m.weight.data.abs().amax(dim=(1, 2, 3)) / (2 ** (bit - 1) - 0.5)).view(-1, 1, 1, 1)
    m.calibrated = True
    m.freeze()
    m.mode = "quant_forward"
    return m


def stem_site(name, size, patch, C, swin, a, images=32):
    from ptq4vit_b200.quant_layers.conv import frozen_stem, frozen_stem_applies
    g = torch.Generator().manual_seed(6)
    P = (size // patch) ** 2
    with torch.no_grad():
        conv = _frozen_conv(C, patch, a.bit)
        x = torch.randn(images, 3, size, size, generator=g).cuda()
        if swin:
            norm = torch.nn.LayerNorm(C).cuda()
            for p in norm.parameters():
                p.requires_grad_(False)
            assert frozen_stem_applies(conv, x, norm=norm), f"{name}: the fold does not apply"

            def unfused():
                return norm(conv(x).flatten(2).transpose(1, 2))

            def fused():
                return frozen_stem(conv, x, norm=norm)
        else:
            cls = (torch.randn(1, 1, C, generator=g) * 0.02).cuda()
            pos = (torch.randn(1, 1 + P, C, generator=g) * 0.02).cuda()
            assert frozen_stem_applies(conv, x, cls_token=cls, pos_embed=pos), f"{name}: the fold does not apply"

            def unfused():
                y = conv(x).flatten(2).transpose(1, 2)
                return torch.cat([cls.expand(images, -1, -1), y], dim=1) + pos

            def fused():
                return frozen_stem(conv, x, cls_token=cls, pos_embed=pos)
        identical = _bits_equal(unfused(), fused())
        runs = AB._time_pair(unfused, fused, a)
    tokens = P if swin else P + 1
    conv_out = 4 * images * C * P
    image = 4 * x.numel()
    fused_bytes = image + 4 * images * tokens * C
    out = AB._report(runs, fused_bytes, {"site": name, "images": images, "channels": C, "positions": P,
                                         "bit_identical": identical})
    out["conv_out_bytes"] = conv_out
    out["stem_ops_bytes"] = 4 * conv_out
    out["stem_ops_hbm_bound_ms"] = round(out["stem_ops_bytes"] / FB.HBM_BYTES_PER_S * 1e3, 4)
    out["unfused_bytes"] = image + conv_out + out["stem_ops_bytes"]
    out["unfused_hbm_bound_ms"] = round(out["unfused_bytes"] / FB.HBM_BYTES_PER_S * 1e3, 4)
    return out


def _calibrated(model, config, images, bit):
    """forward_bench.calibrated_model for any model of the zoo, calibrated at its own resolution"""
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import _SWIN_ZOO, _ZOO, get_net
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
            d["metric"] = "hessian"
    for d in (cfg.w_bit, cfg.a_bit, cfg.A_bit, cfg.B_bit):
        for k in d:
            d[k] = bit
    size = (_SWIN_ZOO.get(model) or _ZOO[model])["img_size"]
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
    deploy.fuse_gather(net)
    batch = torch.randn(32, 3, size, size, generator=torch.Generator().manual_seed(7)).cuda()
    out = {"model": model, "config": config}
    with torch.no_grad():
        logits = net(batch)
        out["left_unfolded"] = deploy.fuse_stem(net)
        out["model_bit_identical"] = _bits_equal(net(batch), logits)
        whole = {"model_unfolded_ms": [], "model_folded_ms": [], "model_unfolded_graph_ms": [], "model_folded_graph_ms": []}
        graphs = {}
        for mode in ("unfolded", "folded"):
            (deploy.fuse_stem if mode == "folded" else deploy.unfuse_stem)(net)
            graphs[mode] = AB._graph(lambda: net(batch))
        out["graph_bit_identical"] = _bits_equal(graphs["unfolded"][1], graphs["folded"][1])
        for _ in range(a.reps):
            for mode in ("unfolded", "folded"):
                (deploy.fuse_stem if mode == "folded" else deploy.unfuse_stem)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_stem(net)
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, graphs
    torch.cuda.empty_cache()
    return out


MODELS = {"vit_b": "vit_base_patch16_224", "swin_t": "swin_tiny_patch4_window7_224"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--configs", default="PTQ4ViT")
    ap.add_argument("--models", default="vit_b,swin_t")
    ap.add_argument("--no-sites", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    from ptq4vit_b200 import build
    build.build()
    res = {"card": FB.card(), "bit": a.bit, "reps": a.reps, "window_s": a.window}
    if not a.no_sites:
        res["sites"] = [stem_site("vit_b224_x32", 224, 16, 768, False, a), stem_site("vit_b384_x32", 384, 16, 768, False, a),
                        stem_site("swin_t224_x32", 224, 4, 96, True, a), stem_site("swin_b384_x32", 384, 4, 128, True, a)]
    res["models"] = [whole_model(MODELS[m], c, a) for m in a.models.split(",") if m for c in a.configs.split(",") if c]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
