"""The patch embedding's token epilogue folded into the frozen conv, on the GPU.  Every comparison is of int32 bit patterns
against the frozen conv followed by torch's ops on the same frozen module: ViT / DeiT's flatten, transpose, cat with the
cls token and pos_embed add, Swin's flatten, transpose and patch_norm.  Every patch geometry of the zoo (ViT-T/S/B-16 at
224, ViT-S/32, ViT-B/384, DeiT-B/384, Swin-T/S/B at 224, Swin-B/384), batch 1 / 5 / 32, W8 and W6, per-channel and
layer-wise step sizes, with and without a conv bias.  The folded stem is one launch that allocates only its output,
leaves no torch cat, add, copy or LayerNorm kernel behind and can be captured in a CUDA graph; refused calls run
unfolded with the same bits; stale step sizes raise; tiny ViT and Swin models with every fusion give the same logits with
and without fuse_stem, eagerly, from one CUDA graph and after a save / load."""
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

# (name, image size, patch, channels, swin) of every patch embedding of the zoo
GEOMETRIES = [
    ("vit_tiny_patch16_224", 224, 16, 192, False), ("vit_small_patch16_224", 224, 16, 384, False),
    ("vit_base_patch16_224", 224, 16, 768, False), ("vit_small_patch32_224", 224, 32, 384, False),
    ("vit_base_patch16_384", 384, 16, 768, False), ("deit_base_patch16_384", 384, 16, 768, False),
    ("swin_tiny_patch4_window7_224", 224, 4, 96, True), ("swin_small_patch4_window7_224", 224, 4, 96, True),
    ("swin_base_patch4_window7_224", 224, 4, 128, True), ("swin_base_patch4_window12_384", 384, 4, 128, True),
]
# (w_bit, layer-wise step size, conv bias): PTQ4ViT's per-channel and BasePTQ's layer-wise patch embedding
CONFIGS = [(8, False, True), (6, True, True), (8, True, False), (6, False, False)]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} outputs differ, first {bad[:4].tolist()}"


def _conv(C, patch, bit=8, layerwise=False, bias=True, seed=0):
    """A frozen patch-embedding conv with hand-set step sizes near the min-max ones (no search needed)."""
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d
    g = torch.Generator().manual_seed(seed)
    m = MinMaxQuantConv2d(3, C, patch, stride=patch, bias=bias, w_bit=bit, a_bit=32)
    m.weight.data = torch.randn(C, 3, patch, patch, generator=g) * 0.05
    if bias:
        m.bias.data = torch.randn(C, generator=g) * 0.5
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    q = 2 ** (bit - 1) - 0.5
    wmax = m.weight.data.abs().amax() if layerwise else m.weight.data.abs().amax(dim=(1, 2, 3))
    jitter = 0.7 + 0.3 * torch.rand(wmax.shape, generator=g).cuda()
    m.w_interval = (wmax / q * jitter).view(-1, 1, 1, 1)
    m.calibrated = True
    m.freeze()
    m.mode = "quant_forward"
    return m


def _stem_params(C, P, seed=5):
    g = torch.Generator().manual_seed(seed)
    cls = (torch.randn(1, 1, C, generator=g) * 0.02).cuda()
    pos = (torch.randn(1, 1 + P, C, generator=g) * 0.02).cuda()
    return cls, pos


def _norm(C, seed=7):
    ln = torch.nn.LayerNorm(C).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        ln.weight.copy_(1.0 + 0.5 * torch.randn(C, generator=g))
        ln.bias.copy_(0.3 * torch.randn(C, generator=g))
    for p in ln.parameters():
        p.requires_grad_(False)
    return ln


def _images(B, size, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 3, size, size, generator=g) * 2.0).cuda()


def _unfolded_vit(conv, x, cls, pos):
    y = conv(x).flatten(2).transpose(1, 2)
    return torch.cat([cls.expand(y.shape[0], -1, -1), y], dim=1) + pos


def _unfolded_swin(conv, x, norm):
    return norm(conv(x).flatten(2).transpose(1, 2))


@pytest.mark.parametrize("config", CONFIGS, ids=lambda c: f"W{c[0]}-{'layerwise' if c[1] else 'channelwise'}-{'bias' if c[2] else 'nobias'}")
@pytest.mark.parametrize("batch", [1, 5, 32])
@pytest.mark.parametrize("name,size,patch,C,swin", GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_stem_bitwise(name, size, patch, C, swin, batch, config):
    from ptq4vit_b200.quant_layers.conv import frozen_stem, frozen_stem_applies
    bit, layerwise, bias = config
    conv = _conv(C, patch, bit, layerwise, bias, seed=sum(map(ord, name)) + 2 * bit + 4 * layerwise + 8 * bias)
    x = _images(batch, size, seed=batch)
    P = (size // patch) ** 2
    with torch.no_grad():
        if swin:
            norm = _norm(C)
            assert frozen_stem_applies(conv, x, norm=norm)
            want = _unfolded_swin(conv, x, norm)
            got = frozen_stem(conv, x, norm=norm)
        else:
            cls, pos = _stem_params(C, P)
            assert frozen_stem_applies(conv, x, cls_token=cls, pos_embed=pos)
            want = _unfolded_vit(conv, x, cls, pos)
            got = frozen_stem(conv, x, cls_token=cls, pos_embed=pos)
    torch.cuda.synchronize()
    assert got.is_contiguous()
    _same(got, want)


def test_swin_rows_with_a_large_mean():
    """Token rows whose mean dwarfs their spread (a large conv bias): LayerNorm's cancellation case."""
    from ptq4vit_b200.quant_layers.conv import frozen_stem
    conv = _conv(96, 4, seed=11)
    with torch.no_grad():
        conv.bias.add_(1000.0)
        norm = _norm(96)
        x = _images(5, 224) * 1e-2
        _same(frozen_stem(conv, x, norm=norm), _unfolded_swin(conv, x, norm))


_PROFILE = """
import sys, torch
sys.path.insert(0, %r)
from tests.test_fold_stem_gpu import _conv, _images, _norm, _stem_params, _unfolded_swin, _unfolded_vit
from ptq4vit_b200.quant_layers.conv import frozen_stem
cv, cs = _conv(768, 16, seed=21), _conv(96, 4, seed=22)
cls, pos = _stem_params(768, 196)
norm = _norm(96)
x = _images(4, 224)
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.no_grad():
    for tag, fn in (("UNFOLDED_V", lambda: _unfolded_vit(cv, x, cls, pos)),
                    ("FOLDED_V", lambda: frozen_stem(cv, x, cls_token=cls, pos_embed=pos)),
                    ("UNFOLDED_S", lambda: _unfolded_swin(cs, x, norm)),
                    ("FOLDED_S", lambda: frozen_stem(cs, x, norm=norm))):
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
    """The folded stem is one kernel, the frozen conv's, where the unfolded one also ran torch's cat and add (ViT) or its
    contiguous copy and LayerNorm (Swin).  The profiler runs in a child process, so that this process opens no profiler
    session."""
    r = subprocess.run([sys.executable, "-c", _PROFILE % (ROOT,)], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    tags = ("UNFOLDED_V", "FOLDED_V", "UNFOLDED_S", "FOLDED_S")
    lines = [ln.split(" ", 1) for ln in r.stdout.splitlines() if ln.split(" ", 1)[0] in tags]
    by = {t: [n for tt, n in lines if tt == t] for t in tags}
    for site in ("V", "S"):
        folded, unfolded = by["FOLDED_" + site], by["UNFOLDED_" + site]
        assert len(folded) == 1 and "forward_conv_kernel" in folded[0], folded
        assert sum("forward_conv_kernel" in n for n in unfolded) == 1 and len(unfolded) >= 2, unfolded
    assert len(by["UNFOLDED_V"]) >= 3, by["UNFOLDED_V"]           # conv, cat (copies), add
    assert any("norm" in n.lower() for n in by["UNFOLDED_S"]), by["UNFOLDED_S"]


def test_one_launch_allocations_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.conv import frozen_stem
    cv, cs = _conv(384, 16, seed=31), _conv(128, 4, bias=False, seed=32)
    cls, pos = _stem_params(384, 196)
    norm = _norm(128)
    x, x2 = _images(4, 224, seed=1), _images(4, 224, seed=2)
    with torch.no_grad():
        for call in (lambda t: frozen_stem(cv, t, cls_token=cls, pos_embed=pos), lambda t: frozen_stem(cs, t, norm=norm)):
            call(x)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
            call(x)
            torch.cuda.synchronize()
            assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
            assert _lib.launch_count() - n0 == 1
        want_v = [_unfolded_vit(cv, t, cls, pos) for t in (x, x2)]
        want_s = [_unfolded_swin(cs, t, norm) for t in (x, x2)]
        xs = x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_stem(cv, xs, cls_token=cls, pos_embed=pos)
            frozen_stem(cs, xs, norm=norm)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yv = frozen_stem(cv, xs, cls_token=cls, pos_embed=pos)
            ys = frozen_stem(cs, xs, norm=norm)
        for i, src in enumerate((x, x2)):
            xs.copy_(src)
            graph.replay()
            torch.cuda.synchronize()
            _same(yv, want_v[i])
            _same(ys, want_s[i])


def _tiny(kind, conv_seed=41):
    """A tiny model whose patch embedding is a frozen conv (everything else in torch)"""
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
    net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
    pe = net.patch_embed.proj
    net.patch_embed.proj = _conv(pe.out_channels, pe.kernel_size[0], seed=conv_seed)
    return net


def test_refused_calls_run_unfolded_and_stale_steps_raise():
    from oracle import ref_harness as RH
    from ptq4vit_b200.quant_layers.conv import frozen_stem, frozen_stem_applies
    from ptq4vit_b200.utils import deploy
    images = RH.tiny_images(n=5, seed=11).cuda()
    for kind in ("vit", "swin"):
        net = _tiny(kind)
        conv = net.patch_embed.proj
        with torch.no_grad():
            want = net(images)
            assert deploy.fuse_stem(net) == [] and net.fold_stem
            _same(net(images), want)
            # a non-contiguous image runs unfolded, same bits
            xt = images.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            assert not xt.is_contiguous()
            args = dict(norm=net.patch_norm) if kind == "swin" else dict(cls_token=net.cls_token, pos_embed=net.pos_embed)
            assert frozen_stem_applies(conv, images, **args) and not frozen_stem_applies(conv, xt, **args)
            _same(net(xt), want)
        # grad wanted: the parameters require grad (nn.Parameter's default) under grad mode
        assert not frozen_stem_applies(conv, images, **args)
        y = net(images)
        assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))
        with torch.no_grad():
            if kind == "vit":
                # a non-FP32 pos_embed: torch's type promotion (FP32 + FP16 -> FP32), unfolded
                pos = net.pos_embed
                net.pos_embed = torch.nn.Parameter(pos.detach().half())
                assert not frozen_stem_applies(conv, images, cls_token=net.cls_token, pos_embed=net.pos_embed)
                net.fold_stem = False
                want64 = net(images)
                net.fold_stem = True
                _same(net(images), want64)
                net.pos_embed = pos
            else:
                # a LayerNorm without affine parameters
                pn = net.patch_norm
                net.patch_norm = torch.nn.LayerNorm(pn.normalized_shape, elementwise_affine=False).cuda()
                assert not frozen_stem_applies(conv, images, norm=net.patch_norm)
                net.fold_stem = False
                want_na = net(images)
                net.fold_stem = True
                _same(net(images), want_na)
                net.patch_norm = pn
            _same(net(images), want)
            # stale step sizes
            conv.w_interval.mul_(1.01)
            with pytest.raises(RuntimeError, match="step sizes changed"):
                frozen_stem(conv, images, **args)
            with pytest.raises(RuntimeError, match="step sizes changed"):
                net(images)


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
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
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
        if kind == "swin":
            assert deploy.fuse_gather(net) == []

    with RH.fp32_convolutions():
        net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True, conv=True)
            fuse_all(net)
            hook_calls = []
            hooks = [net.patch_embed.proj.register_forward_hook(lambda *_: hook_calls.append(1))]
            want, n_unfolded = _launches(net, images)
            assert hook_calls == [1]
            want2 = net(images2)
            assert deploy.fuse_stem(net) == [] and net.fold_stem
            hook_calls.clear()
            got, n_folded = _launches(net, images)
            assert n_folded == n_unfolded, "the stem's ops were torch's; the folded conv launches as before"
            assert hook_calls == [], "a folded call skips the conv's hooks"
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
            assert not fresh.fold_stem, "save_quantized / load_quantized do not record the fold"
            fuse_all(fresh)
            assert deploy.fuse_stem(fresh) == []
            _same(fresh(images), want)
            deploy.unfuse_stem(net)
            assert not net.fold_stem
            _same(net(images), want)
