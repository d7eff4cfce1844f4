"""Time the fused frozen attention core against the unfused frozen sequence on one GPU and print one JSON line.

    python tools/attention_bench.py [--images 32] [--bit 8] [--reps 3] [--window 0.5]

Per attention block (CUDA events over enough calls to fill `--window` seconds, after a warm-up, the two alternated
`--reps` times, medians reported):
  * ViT-B/224, batch 32, on the real qkv output of block 0 of a model calibrated as in tools/forward_bench.py (PTQ4ViT:
    split-of-softmax matmul2; BasePTQ: plain): unfused = frozen matmul1, `* scale`, softmax, frozen matmul2 and the
    transpose copy to [B, N, C]; fused = one p4v_attention_frozen_forward call;
  * Swin-T/224 stage 1 (2 x 64 windows of 49 tokens, 3 heads of 32, shifted-window mask and relative-position bias):
    synthetic qkv output and frozen modules with min-max step sizes, the same two sequences.
Each block's HBM bound is the bytes the fused call must move (q, k, v read once, the [B, N, C] output written once;
bias and mask are counted too) at the H100 SXM data sheet's 3.35 TB/s.  Then the whole quantised ViT-B forward of each
configuration with Linear and MatMul modules frozen, unfused against fused (deploy.fuse_attention), eager (host clock
around a device synchronise) and replayed from one CUDA graph.  The card, its power limit and its max SM clock come from
one read-only nvidia-smi query.  Needs a CUDA device; there is no CPU fallback."""
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

import forward_bench as FB  # noqa: E402


def _block_pair(m1, m2, qkv5, scale, scale_on_q, bias=None, mask=None, max_tokens=256):
    """(unfused, fused) callables of one attention core on the frozen modules."""
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    B, N, _, H, D = qkv5.shape

    def unfused():
        q, k, v = qkv5.permute(2, 0, 3, 1, 4).unbind(0)
        if scale_on_q:
            q = q * scale
        attn = m1.quant_forward(q, k.transpose(-2, -1))
        if not scale_on_q:
            attn = attn * scale
        if bias is not None:
            attn = attn + bias.unsqueeze(0)
        if mask is not None:
            nW = mask.shape[0]
            attn = (attn.view(B // nW, nW, H, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, H, N, N)
        return m2.quant_forward(attn.softmax(dim=-1), v).transpose(1, 2).reshape(B, N, H * D)

    def fused():
        return frozen_attention(m1, m2, qkv5, scale, scale_on_q, bias=bias, mask=mask, max_tokens=max_tokens)
    bits = lambda t: t.contiguous().view(torch.int32)
    identical = torch.equal(bits(unfused()), bits(fused()))
    nbytes = 4 * (qkv5.numel() + B * N * H * D + (0 if bias is None else bias.numel()) + (0 if mask is None else mask.numel()))
    return unfused, fused, identical, nbytes


def _time_pair(unfused, fused, a):
    runs = {"unfused_ms": [], "fused_ms": []}
    for fn in (unfused, fused):       # warm-up
        FB.events_ms(fn, 0.05)
    for _ in range(a.reps):
        runs["unfused_ms"].append(FB.events_ms(unfused, a.window)[0])
        runs["fused_ms"].append(FB.events_ms(fused, a.window)[0])
    return runs


def _report(runs, nbytes, extra):
    u, f = statistics.median(runs["unfused_ms"]), statistics.median(runs["fused_ms"])
    bound = nbytes / FB.HBM_BYTES_PER_S * 1e3
    return {**extra, "bytes": nbytes, "hbm_bound_ms": round(bound, 4), "unfused_ms": round(u, 4), "fused_ms": round(f, 4),
            "speedup": round(u / f, 2), "fused_share_of_hbm_bound": round(bound / f, 3),
            "unfused_runs_ms": [round(v, 4) for v in runs["unfused_ms"]], "fused_runs_ms": [round(v, 4) for v in runs["fused_ms"]]}


def vit_config(config, a):
    from ptq4vit_b200.utils import deploy
    net, wrapped = FB.calibrated_model(config, a.images, a.bit)
    deploy.freeze_model(wrapped, matmul=True)
    batch = torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    blk = net.blocks[0].attn
    got = {}
    h = blk.qkv.register_forward_hook(lambda mod, inp, out: got.__setitem__("y", out.detach()))
    with torch.no_grad():
        net(batch)
    h.remove()
    y = got["y"]
    H = blk.num_heads
    qkv5 = y.view(y.shape[0], y.shape[1], 3, H, y.shape[2] // (3 * H))
    out = {"config": config}
    with torch.no_grad():
        unfused, fused, identical, nbytes = _block_pair(blk.matmul1, blk.matmul2, qkv5, blk.scale, False)
        out["block"] = _report(_time_pair(unfused, fused, a), nbytes,
                               {"qkv": list(qkv5.shape), "matmul2": type(blk.matmul2).__name__, "bit_identical": identical})
        logits = net(batch)
        whole = {"model_unfused_ms": [], "model_fused_ms": [], "model_unfused_graph_ms": [], "model_fused_graph_ms": []}
        graphs = {}
        for mode in ("unfused", "fused"):
            (deploy.fuse_attention if mode == "fused" else deploy.unfuse_attention)(net)
            graphs[mode] = _graph(lambda: net(batch))
        deploy.fuse_attention(net)
        out["model_bit_identical"] = bool(torch.equal(net(batch).view(torch.int32), logits.view(torch.int32)))
        for _ in range(a.reps):
            for mode in ("unfused", "fused"):
                (deploy.fuse_attention if mode == "fused" else deploy.unfuse_attention)(net)
                whole[f"model_{mode}_ms"].append(FB.wall_ms(lambda: net(batch), a.window)[0])
                whole[f"model_{mode}_graph_ms"].append(FB.wall_ms(graphs[mode][0].replay, a.window)[0])
        deploy.unfuse_attention(net)
    out["whole"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in whole.items()}
    del net, wrapped, graphs
    torch.cuda.empty_cache()
    return out


def _graph(fn):
    """fn captured in one CUDA graph (warmed up on a side stream first); returns (graph, its output)."""
    fn()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = fn()
    graph.replay()
    return graph, y


def swin_t_stage1(a):
    """2 images x 64 windows of 7 x 7, 3 heads of 32: synthetic qkv output, min-max step sizes, frozen modules."""
    from ptq4vit_b200.quant_layers import matmul as MM
    B_, N, H, D, nW = 128, 49, 3, 32, 64
    g = torch.Generator().manual_seed(3)
    qkv5 = (torch.randn(B_, N, 3 * H * D, generator=g) * 2.0).cuda().view(B_, N, 3, H, D)
    bias = (torch.randn(H, N, N, generator=g) * 0.5).cuda()
    group = torch.randint(0, 3, (nW, N), generator=g)
    mask = torch.where(group[:, :, None] == group[:, None, :], 0.0, -100.0).cuda()
    scale = D ** -0.5
    q, k, v = qkv5.permute(2, 0, 3, 1, 4).unbind(0)

    def minmax(m, A, B):
        amax, bmax = A.abs().amax(dim=(0, 2, 3)), B.abs().amax(dim=(0, 2, 3))
        m.B_interval = (bmax / (m.B_qmax - 0.5)).view(1, H, 1, 1, 1, 1, 1)
        if m.sos:
            m.split = torch.tensor(0.05).cuda()
            m.A_interval = m.split / (m.A_qmax - 1)
        else:
            m.A_interval = (amax / (m.A_qmax - 0.5)).view(1, H, 1, 1, 1, 1, 1)
        m.calibrated, m.mode = True, "quant_forward"
        return m.freeze()
    out = []
    with torch.no_grad():
        m1 = minmax(MM.PTQSLBatchingQuantMatMul(A_bit=a.bit, B_bit=a.bit), q * scale, k.transpose(-2, -1))
        for cls in ("SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"):
            m2 = getattr(MM, cls)(A_bit=a.bit, B_bit=a.bit)
            m2 = minmax(m2, torch.rand(1, H, 1, 1, device="cuda"), v)
            unfused, fused, identical, nbytes = _block_pair(m1, m2, qkv5, scale, True, bias, mask)
            out.append(_report(_time_pair(unfused, fused, a), nbytes,
                               {"qkv": list(qkv5.shape), "matmul2": cls, "bit_identical": identical}))
    return out


def _minmax_pair(qkv5, scale, m2_cls, bit):
    """Frozen matmul1 / matmul2 modules with min-max step sizes of this input (split 0.05 for split-of-softmax)."""
    from ptq4vit_b200.quant_layers import matmul as MM
    H = qkv5.shape[3]
    q, k, v = qkv5.permute(2, 0, 3, 1, 4).unbind(0)

    def minmax(m, A, B):
        amax, bmax = A.abs().amax(dim=(0, 2, 3)), B.abs().amax(dim=(0, 2, 3))
        m.B_interval = (bmax / (m.B_qmax - 0.5)).view(1, H, 1, 1, 1, 1, 1)
        if m.sos:
            m.split = torch.tensor(0.05).cuda()
            m.A_interval = m.split / (m.A_qmax - 1)
        else:
            m.A_interval = (amax / (m.A_qmax - 0.5)).view(1, H, 1, 1, 1, 1, 1)
        m.calibrated, m.mode = True, "quant_forward"
        return m.freeze()
    m1 = minmax(MM.PTQSLBatchingQuantMatMul(A_bit=bit, B_bit=bit), q, k.transpose(-2, -1))
    m2 = minmax(getattr(MM, m2_cls)(A_bit=bit, B_bit=bit), torch.rand(1, H, 1, 1, device="cuda"), v)
    return m1, m2


def _long_kernel(m1, m2, qkv5, scale):
    """A callable running p4v_attention_frozen_forward_long on this call, also where frozen_attention would pick the
    short kernel (N <= 256)."""
    import ctypes

    from ptq4vit_b200 import _lib
    B, N, _, H, D = qkv5.shape
    p1, p2 = m1._frozen_pack(H), m2._frozen_pack(H)
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim, a.scale_on_q, a.n_windows, a.scale = B, N, H, D, 0, 0, scale
    d1, d2 = m1._desc_dims(1, H, 1, 1, 1), m2._desc_dims(1, H, 1, 1, 1)
    strides = (ctypes.c_longlong * 4)(*qkv5.stride()[:4])

    def call():
        out = torch.empty(B, N, H * D, device="cuda")
        _lib.check(_lib.lib().p4v_attention_frozen_forward_long(
            ctypes.byref(a), _lib.ptr(qkv5), strides, ctypes.byref(d1), _lib.ptr(p1), p1.numel(), ctypes.byref(d2),
            _lib.ptr(p2), p2.numel(), None, None, _lib.ptr(out), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "p4v_attention_frozen_forward_long")
        return out
    return call


def long_sequences(a):
    """ViT-B/384 x 32 blocks (577 tokens, 12 heads of 64): unfused frozen core against the long-sequence kernel; and at
    ViT-B/224's 197 tokens the short kernel against the long one.  Synthetic qkv output, min-max step sizes."""
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    out = []
    with torch.no_grad():
        for N in (577, 197):
            g = torch.Generator().manual_seed(N)
            qkv5 = (torch.randn(32, N, 3 * 768, generator=g) * 2.0).cuda().view(32, N, 3, 12, 64)
            for cls in ("SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"):
                m1, m2 = _minmax_pair(qkv5, 64 ** -0.5, cls, a.bit)
                unfused, fused, identical, nbytes = _block_pair(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)
                if N == 577:
                    out.append(_report(_time_pair(unfused, fused, a), nbytes,
                                       {"qkv": list(qkv5.shape), "matmul2": cls, "bit_identical": identical}))
                else:         # the short kernel (fused up to 256 tokens) against the long one, on the same modules
                    long_ = _long_kernel(m1, m2, qkv5, 64 ** -0.5)
                    identical = identical and torch.equal(long_().view(torch.int32), unfused().view(torch.int32))
                    r = _report(_time_pair(fused, long_, a), nbytes, {"qkv": list(qkv5.shape), "matmul2": cls,
                                                                     "bit_identical": identical})
                    out.append({"short_kernel_ms": r.pop("unfused_ms"), "long_kernel_ms": r.pop("fused_ms"), **r})
                del m1, m2
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32, help="calibration images")
    ap.add_argument("--bit", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of calls per timing")
    ap.add_argument("--configs", default="PTQ4ViT,BasePTQ")
    ap.add_argument("--long-only", action="store_true", help="only the long-sequence blocks")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/attention_bench.py needs a CUDA device (no CPU fallback)")
    torch.cuda.set_device(0)
    if a.long_only:
        print(json.dumps({"tool": "attention_bench", "card": FB.card(), "hbm_bytes_per_s_data_sheet": FB.HBM_BYTES_PER_S,
                          "workload": f"synthetic qkv, min-max step sizes, W{a.bit}A{a.bit}", "long_sequences": long_sequences(a)}))
        return
    out = {"tool": "attention_bench", "card": FB.card(),
           "workload": f"{FB.MODEL}, synthetic weights, calibrated on {a.images} synthetic imgs, batch 32, W{a.bit}A{a.bit}; "
                       "Swin-T stage 1 windows, synthetic",
           "hbm_bytes_per_s_data_sheet": FB.HBM_BYTES_PER_S,
           "long_sequences": long_sequences(a),
           "swin_t_stage1": swin_t_stage1(a),
           "vit_b": [vit_config(c, a) for c in a.configs.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
