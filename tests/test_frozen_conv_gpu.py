"""The frozen patch-embedding convolution on the GPU: within its bound against fp64 at every patch geometry of the zoo
(ViT / DeiT at patch 16 and 32, Swin at patch 4, an input whose size is not a multiple of the patch), channel-wise and
layer-wise, W8 and W6, with and without bias, batch 1 and 5 -- and so is the unfrozen quant_forward in strict FP32, which
shows the bound is tight enough to mean something; all three bf16 terms reach the sum; no FP32 weight is read; one
launch and no allocation but the output; stale step sizes raise; grad mode runs the torch path; whole tiny ViT and Swin
models frozen with conv=True, replayed from one CUDA graph, saved and loaded."""
import copy
import importlib
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _module(layerwise, cin, cout, k, w_bit, bias, seed):
    """A calibrated conv module with step sizes near the min-max ones (perturbed per channel, some clamping), no search."""
    from ptq4vit_b200.quant_layers.conv import BatchingEasyQuantConv2d, ChannelwiseBatchingQuantConv2d
    g = torch.Generator().manual_seed(seed)
    cls = BatchingEasyQuantConv2d if layerwise else ChannelwiseBatchingQuantConv2d
    m = cls(cin, cout, k, stride=k, bias=bias, w_bit=w_bit, a_bit=32, mode="quant_forward")
    with torch.no_grad():
        m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.02)
        if bias:
            m.bias.copy_(torch.randn(cout, generator=g) * 0.05)
    m = m.cuda()
    qm = 2 ** (w_bit - 1) - 0.5
    if layerwise:
        wi = (m.weight.detach().abs().max() / qm * 0.9).reshape(1, 1, 1, 1)
    else:
        f = (0.6 + 0.6 * torch.rand(cout, generator=g)).cuda()
        wi = (m.weight.detach().abs().amax(dim=(1, 2, 3)) / qm * f).reshape(cout, 1, 1, 1)
    m.w_interval = wi.contiguous()
    m.a_interval = torch.ones(1, device="cuda")
    m.calibrated = True
    return m


def _bound_ratio(m, x, out):
    """max |out - ref| / bound with ref = fp64(sum x * fl(q*delta) + bias) and
    bound = (3K + 2) 2^-23 sum |x * fl(q*delta)| + 2^-23 |ref|."""
    w_sim, b = m.quant_weight_bias()
    w64, x64 = w_sim.detach().double(), x.double()
    ref = F.conv2d(x64, w64, None if b is None else b.detach().double(), m.stride)
    mag = F.conv2d(x64.abs(), w64.abs(), None, m.stride)
    K = w_sim[0].numel()
    bound = (3 * K + 2) * 2.0 ** -23 * mag + 2.0 ** -23 * ref.abs()
    err = (out.double() - ref).abs()
    assert out.shape == ref.shape and out.is_contiguous()
    return float((err / bound.clamp_min(1e-300)).max())


GEOMETRIES = {            # (in_channels, out_channels, kernel, height, width)
    "vit_b_224": (3, 768, 16, 224, 224),
    "vit_b_384": (3, 768, 16, 384, 384),
    "vit_s_deit_s": (3, 384, 16, 224, 224),
    "deit_ti": (3, 192, 16, 224, 224),
    "patch32": (3, 384, 32, 224, 224),
    "swin_t": (3, 96, 4, 224, 224),
    "swin_b_384": (3, 128, 4, 384, 384),
    "ragged": (3, 768, 16, 230, 221),       # H, W not multiples of the patch (and W not of 4: the scalar gather)
}


@pytest.mark.parametrize("w_bit,bias", [(8, True), (8, False), (6, True), (6, False)])
@pytest.mark.parametrize("layerwise", [False, True], ids=["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("geo", list(GEOMETRIES))
def test_within_bound_of_fp64(geo, layerwise, w_bit, bias):
    from oracle import ref_harness as RH
    cin, cout, k, H, W = GEOMETRIES[geo]
    m = _module(layerwise, cin, cout, k, w_bit, bias, seed=sum(map(ord, geo)) + 10 * layerwise + w_bit + bias)
    batches = (1, 5, 32) if geo == "vit_b_224" else (1, 5)
    worst_f = worst_u = 0.0
    for B in batches:
        x = torch.randn(B, cin, H, W, generator=torch.Generator().manual_seed(B)).cuda()
        with torch.no_grad():
            with RH.fp32_convolutions():
                want = m.quant_forward(x)
            m.freeze()
            got = m.quant_forward(x)
            m.unfreeze()
        rf, ru = _bound_ratio(m, x, got), _bound_ratio(m, x, want)
        assert rf <= 1.0, f"frozen: |err| / bound = {rf}"
        assert ru <= 1.0, f"unfrozen strict FP32: |err| / bound = {ru}"
        worst_f, worst_u = max(worst_f, rf), max(worst_u, ru)
    print(f"\nbound ratio {geo} {'layerwise' if layerwise else 'channelwise'} W{w_bit} bias={bias}: "
          f"frozen {worst_f:.3e} unfrozen-fp32 {worst_u:.3e}")


@pytest.mark.parametrize("layerwise", [False, True])
@pytest.mark.parametrize("geo", ["vit_b_224", "swin_t", "ragged", "patch32"])
def test_all_three_terms_reach_the_sum(geo, layerwise):
    """One power-of-two weight per channel, no bias, pixels with all 24 mantissa bits: S = x * q is exact, so the output
    is fp32(fp64(delta) * fp64(x) * q) bit for bit.  A dropped or mis-split term fails."""
    cin, cout, k, H, W = GEOMETRIES[geo]
    m = _module(layerwise, cin, cout, k, 8, False, seed=5)
    g = torch.Generator().manual_seed(6)
    K = cin * k * k
    wi = m.w_interval.reshape(-1)
    q = torch.zeros(cout, K)
    pos = torch.randint(0, K, (cout,), generator=g)
    e = torch.randint(0, 8, (cout,), generator=g)
    sign = torch.where(torch.rand(cout, generator=g) < 0.5, -1.0, 1.0)
    q[torch.arange(cout), pos] = torch.where(e == 7, -128.0, sign * 2.0 ** e.clamp(max=6).float())
    with torch.no_grad():
        m.weight.copy_((q.cuda() * wi.reshape(-1, 1).expand(cout, K)).reshape(m.weight.shape))
    mant = torch.randint(0, 1 << 23, (2, cin, H, W), generator=g).double()
    x = ((1.0 + mant * 2.0 ** -23) * 2.0 ** torch.randint(-4, 4, (2, cin, H, W), generator=g).double()
         * torch.where(torch.rand(2, cin, H, W, generator=g) < 0.5, -1.0, 1.0).double()).float().cuda()
    with torch.no_grad():
        m.freeze()
        got = m.quant_forward(x)
    # the one nonzero product per channel, exact in fp64 (24 + 24 bits times a power of two), rounded once
    cols = F.unfold(x.double(), k, stride=k)                                    # [images, K, positions], a gather
    coef = (q.double().cuda() * wi.double().reshape(-1, 1))[torch.arange(cout), pos]
    want = (cols[:, pos.cuda(), :] * coef.reshape(1, cout, 1)).float().reshape(got.shape)
    assert torch.equal(_bits(got), _bits(want)), f"{int((_bits(got) != _bits(want)).sum())} of {got.numel()} differ"


def test_no_fp32_weight_is_read():
    from ptq4vit_b200.utils.integer import dequantize_int_weight, quantize_int_weight
    m = _module(False, 3, 768, 16, 8, True, seed=7)
    x = torch.randn(3, 3, 224, 224).cuda()
    with torch.no_grad():
        want = m.freeze().quant_forward(x)
        m2 = copy.deepcopy(m).unfreeze()
        m2.freeze(weight=dequantize_int_weight(m2, quantize_int_weight(m2)))
        assert torch.equal(m2._packed, m._packed)
        m.weight.fill_(float("nan"))
        assert torch.equal(_bits(m.quant_forward(x)), _bits(want))
        assert torch.equal(_bits(m2.quant_forward(x)), _bits(want))


def test_one_launch_no_allocation_repeatable():
    from ptq4vit_b200 import _lib
    m = _module(False, 3, 768, 16, 8, True, seed=8)
    x = torch.randn(32, 3, 224, 224).cuda()
    with torch.no_grad():
        m.freeze()
        want = m.quant_forward(x)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        y = m.quant_forward(x)
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
        assert _lib.launch_count() - n0 == 1
        for _ in range(3):
            assert torch.equal(_bits(m.quant_forward(x)), _bits(want))
    assert torch.equal(_bits(y), _bits(want))


def test_stale_step_sizes_raise_and_grad_mode_runs_torch():
    from oracle import ref_harness as RH
    m = _module(False, 3, 96, 4, 8, True, seed=9)
    x = torch.randn(2, 3, 32, 32).cuda()
    m.freeze()
    with torch.no_grad():
        m.w_interval.mul_(1.0)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            m.quant_forward(x)
        m.unfreeze().freeze()
        m.quant_forward(x)
        m.w_interval = m.w_interval.clone()
        with pytest.raises(RuntimeError, match="step sizes changed"):
            m.quant_forward(x)
    m.unfreeze().freeze()
    xg = x.clone().requires_grad_(True)
    with RH.fp32_convolutions():
        y = m.quant_forward(xg)
        with torch.no_grad():
            m.unfreeze()
            want = m.quant_forward(x)
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))


TINY_SWIN = dict(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_whole_model_conv_frozen_graph_and_save_load(kind, config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d
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
    with RH.fp32_convolutions():
        net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh, fresh2 = copy.deepcopy(net), copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
    images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
    convs = [n for n, m in wrapped.items() if isinstance(m, MinMaxQuantConv2d)]
    assert len(convs) == 1 and "patch_embed" in convs[0]
    conv = wrapped[convs[0]]
    seen = []
    hook = conv.register_forward_hook(lambda mod, inp, out: seen.append((inp[0].detach().clone(), out.detach().clone())))
    with torch.no_grad():
        assert deploy.freeze_model(wrapped, matmul=True, conv=True) == []
        assert all(m.frozen for m in wrapped.values() if hasattr(m, "frozen"))
        want, want2 = net(images), net(images2)
        x_in, y_conv = seen[0]
        assert _bound_ratio(conv, x_in, y_conv) <= 1.0
        hook.remove()
        # the whole forward in one CUDA graph
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
        assert torch.equal(_bits(ys), _bits(want2)), "graph replay of the whole model on new images"
        # saved, and loaded into a fresh copy whose conv weight is NaN: frozen from the file's integers
        path = str(tmp_path / "model_q.pt")
        deploy.save_quantized(wrapped, path)
        state = torch.load(path, weights_only=True)
        assert state["modules"][convs[0]]["w_int"].shape == conv.weight.shape
        wrapped2 = wrap_modules_in_net(fresh, cfg)
        wrapped2[convs[0]].weight.fill_(float("nan"))
        assert deploy.load_quantized(wrapped2, path, matmul=True, conv=True) == []
        for m in wrapped2.values():
            m.mode = "quant_forward"
        assert torch.equal(_bits(fresh(images)), _bits(want))
        # without conv=True the patch embedding alone stays unfrozen
        wrapped3 = wrap_modules_in_net(fresh2, cfg)
        assert deploy.load_quantized(wrapped3, path, matmul=True) == convs
        deploy.unfreeze_model(wrapped)
        assert not any(m.frozen for m in wrapped.values() if hasattr(m, "frozen"))
