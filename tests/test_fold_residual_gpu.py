"""A block's residual add folded into the frozen Linear that produces it, on the GPU.  Every comparison is of int32 bit
patterns against the unfolded frozen call followed by torch's ops: ViT-B proj (fused path) and fc2 (streamed path),
PTQ4ViT / BasePTQ, W8A8 / W6A6, with and without bias, batch 1 / 5 / 32 under P4V_SCALAR_DIV=ieee; fc2 of a fused MLP
with and without the folded norm2; Swin-T stage-1 / stage-3 and Swin-B/384 stage-1 proj with their window layouts
(shift 0 and > 0) and Swin-T fc2 on both paths.  A folded call adds no launch, allocates only its output, leaves no torch
kernel behind and can be captured in a CUDA graph; calls the rule refuses run unfolded with the same bits; stale step
sizes raise; whole tiny ViT and Swin models with every fusion give the unfolded logits eagerly, from one CUDA graph and
after a save / load."""
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


def _layer(K, O, n_V, n_H, gelu=False, bias=True, bit=8, seed=0):
    """A frozen layer with hand-set step sizes near the min-max ones (no search needed for a forward)."""
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear, PTQSLBatchingQuantLinear
    g = torch.Generator().manual_seed(seed)
    cls = PostGeluPTQSLBatchingQuantLinear if gelu else PTQSLBatchingQuantLinear
    m = cls(K, O, bias=bias, w_bit=bit, a_bit=bit, n_V=n_V, n_H=n_H, n_a=1)
    m.weight.data = torch.randn(O, K, generator=g) * 0.05
    if bias:
        m.bias.data = torch.randn(O, generator=g)
    m = m.cuda()
    q = 2 ** (bit - 1) - 0.5
    wmax = m.weight.data.view(n_V, O // n_V, n_H, K // n_H).abs().amax(dim=(1, 3))
    m.w_interval = (wmax / q * (0.7 + 0.3 * torch.rand(n_V, n_H, generator=g).cuda())).view(n_V, 1, n_H, 1)
    m.a_interval = ((2.5 if gelu else 3.0) / q * (0.7 + 0.3 * torch.rand(1, 1, generator=g))).cuda()
    m.calibrated = True
    m.freeze()
    m.mode = "quant_forward"
    return m


def _x(shape, seed=3, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _same(got, want):
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} outputs differ, first {bad[:4].tolist()}"


def _check(lin, x, res, layout=None):
    from ptq4vit_b200.quant_layers.linear import frozen_residual_applies, frozen_residual_linear
    with torch.no_grad():
        assert frozen_residual_applies(lin, x, res, layout)
        want = res + _unwindow(lin(x), layout, res.shape)
        got = frozen_residual_linear(lin, x, res, layout)
        torch.cuda.synchronize()
    _same(got, want)


def _unwindow(y, layout, shape):
    from ptq4vit_b200.utils.models import _window_reverse
    if layout is None:
        return y
    _images, H, W, ws, shift = layout
    h = _window_reverse(y, ws, H, W)
    if shift:
        h = torch.roll(h, shifts=(shift, shift), dims=(1, 2))
    return h.view(shape)


VIT_TOKENS = 197


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("name", ["proj", "fc2"])
def test_vit_b_bitwise(name, config, bit, monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    K = 768 if name == "proj" else 3072
    n = 24 if config == "PTQ4ViT" else 1
    for bias in (True, False):
        lin = _layer(K, 768, n, n, gelu=name == "fc2" and config == "PTQ4ViT", bias=bias, bit=bit, seed=bit + bias)
        assert lin._frozen_fused == (name == "proj")
        for batch in (1, 5, 32):
            x = _x((batch, VIT_TOKENS, K), seed=batch) * (0.5 if name == "fc2" else 1.0)
            if name == "fc2" and config == "PTQ4ViT":
                x = torch.nn.functional.gelu(x)
            _check(lin, x, _x((batch, VIT_TOKENS, 768), seed=100 + batch))


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
def test_fused_mlp_fc2(config, norm):
    from ptq4vit_b200.quant_layers.linear import (frozen_mlp, frozen_mlp_applies, frozen_mlp_norm_ok, frozen_norm_applies,
                                                  frozen_residual_applies)
    n = 24 if config == "PTQ4ViT" else 1
    fc1 = _layer(768, 3072, n, n, seed=1)
    fc2 = _layer(3072, 768, 1, n, gelu=config == "PTQ4ViT", seed=2)
    ln = None
    if norm:
        ln = torch.nn.LayerNorm(768, eps=1e-6).cuda()
        with torch.no_grad():
            ln.weight.copy_(1.0 + 0.5 * _x((768,), seed=7, scale=1.0))
            ln.bias.copy_(_x((768,), seed=8, scale=0.3))
    for rows in (5, 32 * VIT_TOKENS):
        x, res = _x((rows, 768), seed=rows), _x((rows, 768), seed=rows + 1)
        with torch.no_grad():
            assert frozen_mlp_applies(fc1, fc2, torch.nn.GELU(), x) and frozen_residual_applies(fc2, x, res)
            if norm:
                assert frozen_norm_applies(ln, fc1, x) and frozen_mlp_norm_ok(fc1, fc2)
            want = res + frozen_mlp(fc1, fc2, x, norm=ln)
            got = frozen_mlp(fc1, fc2, x, norm=ln, residual=res)
            torch.cuda.synchronize()
        _same(got, want)


# (C, res, ws): Swin-T stage 1 and 3, Swin-B/384 stage 1
SWIN_PROJ = {"swint_s1": (96, 56, 7), "swint_s3": (384, 14, 7), "swinb384_s1": (128, 96, 12)}


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("name", list(SWIN_PROJ))
def test_swin_proj_window_layout(name, shifted):
    C, res, ws = SWIN_PROJ[name]
    shift = ws // 2 if shifted else 0
    lin = _layer(C, C, C // 32, C // 32, seed=C)
    assert lin._frozen_fused
    for B in ((32, 3) if name == "swint_s1" else (8, 1)):
        layout = (B, res, res, ws, shift)
        _check(lin, _x((B * res * res // (ws * ws), ws * ws, C), seed=B), _x((B, res * res, C), seed=B + 50), layout)


def test_swin_t_fc2_both_paths():
    from ptq4vit_b200.quant_layers.linear import frozen_mlp, frozen_mlp_applies, frozen_residual_applies
    fc1, fc2 = _layer(96, 384, 3, 3, seed=11), _layer(384, 96, 3, 12, gelu=True, seed=12)
    assert fc2._frozen_fused, "Swin-T stage-1 fc2 alone runs the fused kernel"
    x = _x((32, 3136, 96), seed=13)
    res = _x((32, 3136, 96), seed=14)
    with torch.no_grad():
        h = torch.nn.functional.gelu(fc1(x))
    _check(fc2, h, res)
    with torch.no_grad():               # in a fused MLP fc2 streams
        assert frozen_mlp_applies(fc1, fc2, torch.nn.GELU(), x) and frozen_residual_applies(fc2, x, res)
        want = res + frozen_mlp(fc1, fc2, x)
        got = frozen_mlp(fc1, fc2, x, residual=res)
        torch.cuda.synchronize()
    _same(got, want)


_PROFILE = """
import sys, torch
sys.path.insert(0, %r)
from tests.test_fold_residual_gpu import _layer, _unwindow, _x
from ptq4vit_b200.quant_layers.linear import frozen_residual_linear
C, res, ws = 96, 56, 7
layout = (4, res, res, ws, 3)
proj = _layer(C, C, 3, 3, seed=21)
xw, r = _x((4 * res * res // (ws * ws), ws * ws, C), seed=1), _x((4, res * res, C), seed=3)
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.no_grad():
    for tag, fn in (("UNFOLDED", lambda: r + _unwindow(proj(xw), layout, r.shape)),
                    ("FOLDED", lambda: frozen_residual_linear(proj, xw, r, layout))):
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
    """The shifted Swin proj folded: its one kernel is the fused forward, where the unfolded call also ran torch's reverse
    copy, roll and add.  The profiler runs in a child process, so that this process opens no profiler session."""
    r = subprocess.run([sys.executable, "-c", _PROFILE % (ROOT,)], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln.split(" ", 1) for ln in r.stdout.splitlines() if ln.startswith(("UNFOLDED ", "FOLDED "))]
    folded = [n for t, n in lines if t == "FOLDED"]
    unfolded = [n for t, n in lines if t == "UNFOLDED"]
    assert len(folded) == 1 and "forward_tc_kernel" in folded[0], folded
    assert len(unfolded) >= 4 and sum("forward_tc_kernel" in n for n in unfolded) == 1, unfolded


def test_launches_allocations_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import frozen_residual_linear
    from ptq4vit_b200.utils.models import WindowAttention
    C, res, ws = SWIN_PROJ["swint_s1"]
    B, shift = 4, 3
    layout = (B, res, res, ws, shift)
    proj = _layer(C, C, 3, 3, seed=21)
    fc2 = _layer(3072, 768, 24, 24, gelu=True, seed=22)
    wa = WindowAttention(C, ws, 3).cuda()
    wa.proj = proj
    xw, xw2 = _x((B * res * res // (ws * ws), ws * ws, C), seed=1), _x((B * res * res // (ws * ws), ws * ws, C), seed=2)
    r1 = _x((B, res * res, C), seed=3)
    h, r2 = torch.nn.functional.gelu(_x((8 * VIT_TOKENS, 3072), seed=4)), _x((8 * VIT_TOKENS, 768), seed=5)
    with torch.no_grad():
        for lin, x, r, lay in [(proj, xw, r1, layout), (fc2, h, r2, None)]:
            want = r + _unwindow(lin(x), lay, r.shape)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            lin(x)
            torch.cuda.synchronize()
            n_plain = _lib.launch_count() - n0
            frozen_residual_linear(lin, x, r, lay)          # warm: the streamed image exists
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
            y = frozen_residual_linear(lin, x, r, lay)
            torch.cuda.synchronize()
            assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
            assert _lib.launch_count() - n0 == n_plain, "the folded call launches what the plain frozen call does"
            _same(y, want)
        _same(wa._proj(xw, r1, layout), r1 + _unwindow(proj(xw), layout, r1.shape))
        # capture: a host <-> device copy or synchronisation inside the call would fail it
        want1, want2 = r1 + _unwindow(proj(xw), layout, r1.shape), r1 + _unwindow(proj(xw2), layout, r1.shape)
        wantf = r2 + fc2(h)
        xs = xw.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_residual_linear(proj, xs, r1, layout)
            frozen_residual_linear(fc2, h, r2)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ys = frozen_residual_linear(proj, xs, r1, layout)
            yf = frozen_residual_linear(fc2, h, r2)
        graph.replay()
        torch.cuda.synchronize()
        _same(ys, want1)
        _same(yf, wantf)
        xs.copy_(xw2)
        graph.replay()
        torch.cuda.synchronize()
        _same(ys, want2)


def test_refused_calls_run_unfolded_and_stale_steps_raise():
    from ptq4vit_b200.quant_layers.linear import frozen_residual_applies, frozen_residual_linear
    from ptq4vit_b200.utils.models import Attention, Mlp
    proj = _layer(768, 768, 24, 24, seed=31)
    attn = Attention(768, 12).cuda()
    attn.proj = proj
    for p in attn.parameters():
        p.requires_grad_(False)
    x = _x((2, VIT_TOKENS, 768), seed=32)
    r = _x((2, VIT_TOKENS, 768), seed=33)
    with torch.no_grad():
        want = r + attn(x)
        got = attn(x, residual=r)
        _same(got, want)
        # non-contiguous and misaligned shortcuts run unfolded, same bits
        rt = r.transpose(0, 1).contiguous().transpose(0, 1)
        assert not rt.is_contiguous() and not frozen_residual_applies(proj, x, rt)
        _same(attn(x, residual=rt), want)
        r_off = torch.empty(r.numel() + 1, device="cuda")[1:].view(r.shape)
        r_off.copy_(r)
        assert not frozen_residual_applies(proj, x, r_off)
        _same(attn(x, residual=r_off), want)
        # a layout on the streamed path
        fc2 = _layer(3072, 768, 24, 24, seed=34)
        assert not fc2._frozen_fused
        h = _x((2 * 49 * 4, 49, 3072), seed=35, scale=0.5)
        rs = _x((2 * 4, 196, 768), seed=36)
        assert not frozen_residual_applies(fc2, h, rs, (8, 14, 14, 7, 3))
    # grad mode: the shortcut requires grad
    rg = r.clone().requires_grad_(True)
    assert not frozen_residual_applies(proj, x, rg)
    y = attn(x, residual=rg)
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))
    # stale step sizes
    with torch.no_grad():
        frozen_residual_linear(proj, x, r)
        proj.a_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_residual_linear(proj, x, r)
        mlp = Mlp(768, 3072).cuda()
        mlp.fc1, mlp.fc2 = _layer(768, 3072, 24, 24, seed=37), fc2
        mlp.fused = True
        xm = _x((2, VIT_TOKENS, 768), seed=38)
        mlp(xm, residual=r)
        fc2.w_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            mlp(xm, residual=r)


def _launches(net, images):
    from ptq4vit_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = net(images)
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_whole_model_folded_graph_and_save_load(kind, config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import Block, SwinBlock, SwinTransformer, VisionTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    from tests import _baseptq_ref as BR
    os.environ.setdefault("TQDM_DISABLE", "1")
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        BR.baseptq_hessian(cfg)
    with RH.fp32_convolutions():
        net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True, conv=True)
            assert deploy.fuse_attention(net) == [] and deploy.fuse_mlp(net) == []
            deploy.fuse_norm(net)
            hook_calls = []
            hooks = [m.register_forward_hook(lambda *_: hook_calls.append(1)) for m in net.modules()
                     if isinstance(m, (Block, SwinBlock))]
            hooks += [lin.register_forward_hook(lambda *_: hook_calls.append(2)) for m in net.modules()
                      if isinstance(m, (Block, SwinBlock)) for lin in (m.attn.proj, m.mlp.fc2)]
            want, n_unfolded = _launches(net, images)
            proj_calls = hook_calls.count(2)
            want2 = net(images2)
            assert deploy.fuse_residual(net) == []
            assert all(m.fold_residual for m in net.modules() if isinstance(m, (Block, SwinBlock)))
            hook_calls.clear()
            got, n_folded = _launches(net, images)
            assert n_folded == n_unfolded, "the adds were torch ops; the folded Linears launch as before"
            assert hook_calls.count(2) < proj_calls, "a folded call skips proj's / fc2's hooks"
            for hk in hooks:
                hk.remove()
            _same(got, want)
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
            assert deploy.fuse_attention(fresh) == [] and deploy.fuse_mlp(fresh) == []
            deploy.fuse_norm(fresh)
            assert deploy.fuse_residual(fresh) == []
            _same(fresh(images), want)
            deploy.unfuse_residual(net)
            _same(net(images), want)
