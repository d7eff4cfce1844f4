"""Swin's row gathers folded into the frozen Linear that consumes them, on the GPU.  Every comparison is of int32 bit
patterns against the unfolded sequence on the same frozen layer: the window gather (norm1, roll(-shift), window
partition, qkv) at Swin-T stages 1-4 and Swin-B/384 stages 1 and 3, shift 0 and window / 2, PTQ4ViT- and BasePTQ-shaped
blocks, W8A8 / W6A6, n_a > 1, batch 1 / 5 / 32, under P4V_SCALAR_DIV=ieee, rows whose mean dwarfs their spread included;
the merge gather (PatchMerging's cat, norm, reduction) at Swin-T's and Swin-B/384's first two merges and at C % 16 != 0,
whose chunks straddle the cat's quarters; the streamed merge runs unfolded.  A folded call allocates only its output,
leaves no LayerNorm, roll, partition copy or cat kernel behind and can be captured in a CUDA graph; calls the rule
refuses run unfolded with the same bits; stale step sizes raise; a whole tiny Swin with every fusion gives the same
logits with and without fuse_gather, eagerly, from one CUDA graph and after a save / load."""
import copy
import importlib
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TINY_SWIN = dict(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} outputs differ, first {bad[:4].tolist()}"


def _layer(K, O, n_V=1, n_H=1, n_a=1, bias=True, bit=8, seed=0):
    """A frozen layer with hand-set step sizes near the min-max ones of a LayerNorm's output (no search needed)."""
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    g = torch.Generator().manual_seed(seed)
    m = PTQSLBatchingQuantLinear(K, O, bias=bias, w_bit=bit, a_bit=bit, n_V=n_V, n_H=n_H, n_a=n_a)
    m.weight.data = torch.randn(O, K, generator=g) * 0.05
    if bias:
        m.bias.data = torch.randn(O, generator=g)
    m = m.cuda()
    q = 2 ** (bit - 1) - 0.5
    wmax = m.weight.data.view(n_V, O // n_V, n_H, K // n_H).abs().amax(dim=(1, 3))
    m.w_interval = (wmax / q * (0.7 + 0.3 * torch.rand(n_V, n_H, generator=g).cuda())).view(n_V, 1, n_H, 1)
    m.a_interval = (3.0 / q * (0.7 + 0.3 * torch.rand(n_a, 1, generator=g))).cuda()
    m.calibrated = True
    m.freeze()
    m.mode = "quant_forward"
    return m


def _norm(C, seed=7):
    ln = torch.nn.LayerNorm(C).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.5 * torch.randn(C, generator=g))
        ln.bias.copy_(0.3 * torch.randn(C, generator=g))
    for p in ln.parameters():
        p.requires_grad_(False)
    return ln


def _x(shape, seed=3, scale=2.0, offset_rows=True):
    """Random rows; with offset_rows every third row gets a mean that dwarfs its spread (LayerNorm's cancellation case)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, generator=g) * scale
    if offset_rows:
        flat = x.view(-1, shape[-1])
        flat[::3] = flat[::3] * 1e-3 + 1000.0 * (1 + torch.rand(flat[::3].shape[0], 1, generator=g))
    return x.cuda()


def _unfolded_window(norm, lin, x, images, H, W, ws, shift):
    from ptq4vit_b200.utils.models import _window_partition
    h = norm(x).view(images, H, W, -1)
    if shift:
        h = torch.roll(h, shifts=(-shift, -shift), dims=(1, 2))
    return lin(_window_partition(h, ws))


def _unfolded_merge(norm, lin, x, images, H, W):
    C = x.shape[-1]
    h = x.view(images, H, W, C)
    h = torch.cat([h[:, 0::2, 0::2], h[:, 1::2, 0::2], h[:, 0::2, 1::2], h[:, 1::2, 1::2]], -1).view(images, -1, 4 * C)
    return lin(norm(h))


def _check(norm, lin, x, gather):
    from ptq4vit_b200.quant_layers.linear import frozen_gather_applies, frozen_gather_linear
    mode, images, H, W, ws, shift = gather
    with torch.no_grad():
        assert frozen_gather_applies(norm, lin, x, gather)
        want = _unfolded_window(norm, lin, x, images, H, W, ws, shift) if mode == "window" else \
            _unfolded_merge(norm, lin, x, images, H, W)
        got = frozen_gather_linear(norm, lin, x, gather)
        torch.cuda.synchronize()
    _same(got, want)


# (C, res, window): Swin-T stages 1-4, Swin-B/384 stages 1 and 3
SWIN_QKV = {"swint_s1": (96, 56, 7), "swint_s2": (192, 28, 7), "swint_s3": (384, 14, 7), "swint_s4": (768, 7, 7),
            "swinb384_s1": (128, 96, 12), "swinb384_s3": (512, 24, 12)}


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("name", list(SWIN_QKV))
def test_window_qkv_bitwise(name, config, bit, monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    C, res, ws = SWIN_QKV[name]
    n = C // 32
    # PTQ4ViT-shaped: q, k and v row blocks, column blocks, activation chunks; BasePTQ-shaped: one block each
    lin = _layer(C, 3 * C, 3 * n if config == "PTQ4ViT" else 1, n if config == "PTQ4ViT" else 1,
                 n if config == "PTQ4ViT" else 1, bit=bit, seed=C + bit)
    assert lin._frozen_fused
    norm = _norm(C, seed=C)
    for B in ((1, 5, 32) if res >= 56 else (1, 5)):
        for shift in (0, ws // 2):
            x = _x((B, res * res, C), seed=B + shift)
            _check(norm, lin, x, ("window", B, res, res, ws, shift))


# (C, res): Swin-T's and Swin-B/384's first two merges; C % 16 != 0 (chunks straddle the quarters)
SWIN_MERGE = {"swint_m1": (96, 56), "swint_m2": (192, 28), "swinb384_m1": (128, 96), "swinb384_m2": (256, 48),
              "c36": (36, 8), "c100": (100, 14)}


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("name", list(SWIN_MERGE))
def test_merge_reduction_bitwise(name, bit, monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    C, res = SWIN_MERGE[name]
    n_a = 4 if C % 16 == 0 else 1
    lin = _layer(4 * C, 2 * C, 1, 1, n_a, bias=False, bit=bit, seed=C + bit)
    assert lin._frozen_fused
    norm = _norm(4 * C, seed=C)
    for B in ((1, 5, 32) if name == "swint_m1" else (1, 5)):
        _check(norm, lin, _x((B, res * res, C), seed=B), ("merge", B, res, res, 0, 0))


def test_streamed_merge_runs_unfolded():
    from ptq4vit_b200.quant_layers.linear import frozen_gather_applies
    from ptq4vit_b200.utils.models import PatchMerging
    pm = PatchMerging(14, 384).cuda().eval()
    pm.reduction = _layer(1536, 768, bias=False, seed=5)
    pm.norm = _norm(1536)
    assert not pm.reduction._frozen_fused
    x = _x((2, 196, 384), seed=6)
    with torch.no_grad():
        want = _unfolded_merge(pm.norm, pm.reduction, x, 2, 14, 14)
        assert not frozen_gather_applies(pm.norm, pm.reduction, x, ("merge", 2, 14, 14, 0, 0))
        pm.fold_gather = True
        _same(pm(x), want)
        pm.fold_norm = True
        _same(pm(x), want)


_PROFILE = """
import sys, torch
sys.path.insert(0, %r)
from tests.test_fold_gather_gpu import _layer, _norm, _unfolded_merge, _unfolded_window, _x
from ptq4vit_b200.quant_layers.linear import frozen_gather_linear
qkv, n1 = _layer(96, 288, 3, 3, 3, seed=21), _norm(96)
red, n2 = _layer(384, 192, bias=False, seed=22), _norm(384)
x = _x((4, 3136, 96), seed=1)
wg, mg = ("window", 4, 56, 56, 7, 3), ("merge", 4, 56, 56, 0, 0)
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.no_grad():
    for tag, fn in (("UNFOLDED_W", lambda: _unfolded_window(n1, qkv, x, 4, 56, 56, 7, 3)),
                    ("FOLDED_W", lambda: frozen_gather_linear(n1, qkv, x, wg)),
                    ("UNFOLDED_M", lambda: _unfolded_merge(n2, red, x, 4, 56, 56)),
                    ("FOLDED_M", lambda: frozen_gather_linear(n2, red, x, mg))):
        fn()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=acts) as prof:
            fn()
            torch.cuda.synchronize()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                print(tag, e.name)
"""


def test_profile_torch_kernels_are_gone():
    """The shifted window gather folded: one kernel, the fused forward, where the unfolded call also ran torch's
    LayerNorm, roll and partition copy; the merge: one kernel where torch's cat and LayerNorm ran.  The profiler runs in a
    child process, so that this process opens no profiler session."""
    r = subprocess.run([sys.executable, "-c", _PROFILE % (ROOT,)], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln.split(" ", 1) for ln in r.stdout.splitlines() if ln.split(" ", 1)[0] in
             ("UNFOLDED_W", "FOLDED_W", "UNFOLDED_M", "FOLDED_M")]
    by = {t: [n for tt, n in lines if tt == t] for t in ("UNFOLDED_W", "FOLDED_W", "UNFOLDED_M", "FOLDED_M")}
    for site in ("W", "M"):
        folded, unfolded = by["FOLDED_" + site], by["UNFOLDED_" + site]
        assert len(folded) == 1 and "forward_tc_kernel" in folded[0], folded
        assert sum("forward_tc_kernel" in n for n in unfolded) == 1, unfolded
        assert any("norm" in n.lower() for n in unfolded), unfolded
    assert len(by["UNFOLDED_W"]) >= 4, by["UNFOLDED_W"]          # LayerNorm, roll, partition copy, qkv
    assert any("cat" in n.lower() for n in by["UNFOLDED_M"]), by["UNFOLDED_M"]


def test_allocations_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import frozen_gather_linear
    qkv, n1 = _layer(96, 288, 3, 3, 3, seed=31), _norm(96)
    red, n2 = _layer(384, 192, bias=False, seed=32), _norm(384)
    x, x2 = _x((4, 3136, 96), seed=1), _x((4, 3136, 96), seed=2)
    wg, mg = ("window", 4, 56, 56, 7, 3), ("merge", 4, 56, 56, 0, 0)
    with torch.no_grad():
        for norm, lin, g in ((n1, qkv, wg), (n2, red, mg)):
            frozen_gather_linear(norm, lin, x, g)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
            frozen_gather_linear(norm, lin, x, g)
            torch.cuda.synchronize()
            assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
            assert _lib.launch_count() - n0 == 1
        want1 = [_unfolded_window(n1, qkv, t, 4, 56, 56, 7, 3) for t in (x, x2)]
        want2 = [_unfolded_merge(n2, red, t, 4, 56, 56) for t in (x, x2)]
        xs = x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_gather_linear(n1, qkv, xs, wg)
            frozen_gather_linear(n2, red, xs, mg)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yw = frozen_gather_linear(n1, qkv, xs, wg)
            ym = frozen_gather_linear(n2, red, xs, mg)
        for i, src in enumerate((x, x2)):
            xs.copy_(src)
            graph.replay()
            torch.cuda.synchronize()
            _same(yw, want1[i])
            _same(ym, want2[i])


def test_refused_calls_run_unfolded_and_stale_steps_raise():
    from ptq4vit_b200.quant_layers.linear import frozen_gather_applies, frozen_gather_linear
    from ptq4vit_b200.utils.models import SwinBlock
    sb = SwinBlock(96, 56, 3, 7, 3).cuda().eval()
    sb.attn.qkv = _layer(96, 288, 3, 3, 3, seed=41)
    sb.norm1 = _norm(96)
    for p in sb.parameters():
        p.requires_grad_(False)
    x = _x((2, 3136, 96), seed=42)
    g = ("window", 2, 56, 56, 7, 3)
    with torch.no_grad():
        want = sb(x)
        sb.fold_gather = True
        _same(sb(x), want)
        # a non-contiguous input runs unfolded, same bits
        xt = x.transpose(0, 1).contiguous().transpose(0, 1)
        assert not frozen_gather_applies(sb.norm1, sb.attn.qkv, xt, g)
        _same(sb(xt), want)
    # grad mode: the input requires grad
    xg = x.clone().requires_grad_(True)
    assert not frozen_gather_applies(sb.norm1, sb.attn.qkv, xg, g)
    y = sb(xg)
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))
    with torch.no_grad():
        # an unfrozen qkv: the unfolded sequence on the unfrozen quant_forward, same bits
        sb.attn.qkv.unfreeze()
        assert not frozen_gather_applies(sb.norm1, sb.attn.qkv, x, g)
        _same(sb(x), want)
        sb.attn.qkv.freeze()
        _same(sb(x), want)
        # stale step sizes
        sb.attn.qkv.a_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_gather_linear(sb.norm1, sb.attn.qkv, x, g)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            sb(x)


def _launches(net, images):
    from ptq4vit_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = net(images)
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
def test_whole_swin_folded_graph_and_save_load(config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import PatchMerging, SwinBlock, SwinTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    from tests import _baseptq_ref as BR
    os.environ.setdefault("TQDM_DISABLE", "1")
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        BR.baseptq_hessian(cfg)

    def fuse_all(net):
        assert deploy.fuse_attention(net) == [] and deploy.fuse_mlp(net) == []
        deploy.fuse_norm(net)
        assert deploy.fuse_residual(net) == []

    with RH.fp32_convolutions():
        net = SwinTransformer(**TINY_SWIN).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True, conv=True)
            fuse_all(net)
            hook_calls = []
            norms = [m.norm1 for m in net.modules() if isinstance(m, SwinBlock)] + \
                    [m.norm for m in net.modules() if isinstance(m, PatchMerging)]
            hooks = [n.register_forward_hook(lambda *_: hook_calls.append(1)) for n in norms]
            want, n_unfolded = _launches(net, images)
            assert len(hook_calls) >= 4, "every block's norm1 ran"
            want2 = net(images2)
            deploy.unfuse_residual(net)
            want_nores = net(images)
            deploy.fuse_residual(net)
            assert deploy.fuse_gather(net) == []
            assert all(m.fold_gather for m in net.modules() if isinstance(m, (SwinBlock, PatchMerging)))
            hook_calls.clear()
            got, n_folded = _launches(net, images)
            assert n_folded == n_unfolded, "the gathers were torch ops; the folded Linears launch as before"
            assert hook_calls == [], "a folded call skips norm1's and PatchMerging.norm's hooks"
            for hk in hooks:
                hk.remove()
            _same(got, want)
            deploy.unfuse_residual(net)
            _same(net(images), want_nores)
            deploy.fuse_residual(net)
            xs = images.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                net(xs)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                ys = net(xs)
            xs.copy_(images2)
            graph.replay()
            torch.cuda.synchronize()
            _same(ys, want2)
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            deploy.load_quantized(wrapped2, path, matmul=True, conv=True)
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert not any(m.fold_gather for m in fresh.modules() if isinstance(m, (SwinBlock, PatchMerging)))
            fuse_all(fresh)
            assert deploy.fuse_gather(fresh) == []
            _same(fresh(images), want)
            deploy.unfuse_gather(net)
            assert not any(m.fold_gather for m in net.modules() if isinstance(m, (SwinBlock, PatchMerging)))
            _same(net(images), want)
