"""The long-sequence fused frozen attention core on the GPU: bit-identical (as int32 bit patterns) to matmul1, `* scale`,
torch's softmax, matmul2 and the transpose on the frozen modules for 197 to 1024 tokens, PTQ4ViT (split-of-softmax
matmul2), BasePTQ and the no_softmax ablation (plain matmul2), W8A8 / W6A6, head_dim 64 and 32, n_G = 1 modules, batch 1
and an odd batch, large-amplitude scores; one launch, no copy, no allocation but the output; stale step sizes raise;
grad mode runs unfused; a 577-token block and a whole tiny 577-token ViT fused with max_tokens=1024 give the unfused
bits eagerly, from one CUDA graph and after a save / load."""
import copy
import importlib
import os

import pytest
import torch

from tests.test_fused_attention_gpu import M2, _copies, _frozen_pair, _qkv, _unfused
from tests.test_frozen_matmul_gpu import _bits

pytestmark = pytest.mark.gpu


def _check_long(m1, m2, qkv5, scale):
    from ptq4vit_b200.quant_layers.matmul import frozen_attention, frozen_attention_applies
    B, N, _, H, D = qkv5.shape
    assert frozen_attention_applies(m1, m2, N, D, qkv5, max_tokens=1024)
    with torch.no_grad():
        want = _unfused(m1, m2, qkv5, scale, False)
        got = frozen_attention(m1, m2, qkv5, scale, False, max_tokens=1024)
    assert got.shape == want.shape
    diff = int((_bits(got) != _bits(want)).sum())
    assert diff == 0, f"{diff} of {got.numel()} differ (max abs {float((got - want).abs().max()):.3g})"


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["ptq4vit", "baseptq", "no_softmax"])
@pytest.mark.parametrize("N", [257, 320, 577, 1024])
def test_long_bitwise(N, config, bit):
    _, qkv5 = _qkv(3, N, 12, 64, seed=N + bit)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", M2[config], bit, qkv5, 64 ** -0.5, False)
    _check_long(m1, m2, qkv5, 64 ** -0.5)


@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
@pytest.mark.parametrize("N", [197, 577, 1024])
def test_head_dim_32(N, m2_cls):
    _, qkv5 = _qkv(2, N, 6, 32, seed=N + 3)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, 32 ** -0.5, False)
    _check_long(m1, m2, qkv5, 32 ** -0.5)


@pytest.mark.parametrize("N", [1, 17, 197])
def test_short_sequences_on_the_long_kernel(N):
    """The long kernel's ABI holds N <= 256 too (and rows shorter than a warp): same bits as the unfused sequence."""
    import ctypes

    from ptq4vit_b200 import _lib
    _, qkv5 = _qkv(2, N, 12, 64, seed=N + 50)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul", 8, qkv5, 64 ** -0.5, False)
    B, N, _, H, D = qkv5.shape
    p1, p2 = m1._frozen_pack(H), m2._frozen_pack(H)
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim, a.scale_on_q, a.n_windows, a.scale = B, N, H, D, 0, 0, 64 ** -0.5
    d1, d2 = m1._desc_dims(1, H, 1, 1, 1), m2._desc_dims(1, H, 1, 1, 1)
    with torch.no_grad():
        want = _unfused(m1, m2, qkv5, 64 ** -0.5, False)
        out = torch.empty(B, N, H * D, device="cuda")
        _lib.check(_lib.lib().p4v_attention_frozen_forward_long(
            ctypes.byref(a), _lib.ptr(qkv5), (ctypes.c_longlong * 4)(*qkv5.stride()[:4]), ctypes.byref(d1), _lib.ptr(p1),
            p1.numel(), ctypes.byref(d2), _lib.ptr(p2), p2.numel(), None, None, _lib.ptr(out),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "long")
    assert torch.equal(_bits(out), _bits(want))


@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLQuantMatMul"])
def test_one_group_modules(m2_cls):
    _, qkv5 = _qkv(2, 577, 12, 64, seed=61)
    m1, m2 = _frozen_pair("PTQSLQuantMatMul", m2_cls, 8, qkv5, 64 ** -0.5, False, one_group=True)
    _check_long(m1, m2, qkv5, 64 ** -0.5)


@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
def test_small_and_odd_batches(batch, m2_cls):
    _, qkv5 = _qkv(batch, 577, 12, 64, seed=70 + batch)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, 64 ** -0.5, False)
    _check_long(m1, m2, qkv5, 64 ** -0.5)


@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
def test_large_amplitude_scores(m2_cls):
    """Wide score rows: most probabilities underflow to 0 and a few dominate each row."""
    _, qkv5 = _qkv(2, 577, 12, 64, seed=80, amp=12.0)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, 64 ** -0.5, False)
    _check_long(m1, m2, qkv5, 64 ** -0.5)


def test_one_launch_no_copy_no_allocation():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    _, qkv5 = _qkv(8, 577, 12, 64, seed=91)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul", 8, qkv5, 64 ** -0.5, False)
    call = lambda: frozen_attention(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)  # noqa: E731
    with torch.no_grad():
        want = _unfused(m1, m2, qkv5, 64 ** -0.5, False)
        call()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        copies, y = _copies(call)
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
    assert _lib.launch_count() - n0 == 1
    assert not copies, f"the fused call issued a copy: {copies}"
    assert torch.equal(_bits(y), _bits(want))


def test_stale_step_sizes_raise():
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    _, qkv5 = _qkv(2, 577, 12, 64, seed=92)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul", 8, qkv5, 64 ** -0.5, False)
    with torch.no_grad():
        frozen_attention(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)
        m2.split.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_attention(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)
        m2.unfreeze(); m2.freeze()
        frozen_attention(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)
        m1.B_interval = m1.B_interval * 1.0
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_attention(m1, m2, qkv5, 64 ** -0.5, False, max_tokens=1024)


def _block_577(m2_cls, seed):
    from ptq4vit_b200.utils.models import Attention
    torch.manual_seed(seed)
    blk = Attention(768, 12).cuda().eval()
    x = torch.randn(2, 577, 768, device="cuda")
    with torch.no_grad():
        qkv5 = blk.qkv(x).view(2, 577, 3, 12, 64)
    blk.matmul1, blk.matmul2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, blk.scale, False)
    return blk, x


def _launches(fn):
    from ptq4vit_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    y = fn()
    torch.cuda.synchronize()
    return y, _lib.launch_count() - n0


@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
def test_block_577_tokens(m2_cls):
    from ptq4vit_b200.utils import deploy
    blk, x = _block_577(m2_cls, seed=7)
    with torch.no_grad():
        want = blk(x)
        assert deploy.fuse_attention(blk) == []
        got, n = _launches(lambda: blk(x))
        assert n == 2, "default max_tokens: the two frozen MatMul kernels"
        assert torch.equal(_bits(got), _bits(want))
        assert deploy.fuse_attention(blk, max_tokens=1024) == []
        got, n = _launches(lambda: blk(x))
        assert n == 1, "max_tokens=1024: one fused launch"
        assert torch.equal(_bits(got), _bits(want))
        deploy.unfuse_attention(blk)
        got, n = _launches(lambda: blk(x))
        assert n == 2 and torch.equal(_bits(got), _bits(want))


def test_grad_mode_runs_unfused():
    from ptq4vit_b200.utils import deploy
    blk, x = _block_577("SoSPTQSLBatchingQuantMatMul", seed=8)
    with torch.no_grad():
        want = blk(x)
    deploy.fuse_attention(blk, max_tokens=1024)
    xg = x.clone().requires_grad_(True)
    y, n = _launches(lambda: blk(xg))
    assert n == 2, "grad mode: the two MatMul modules, not the fused kernel"
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))


def test_torch_softmax_is_the_warp_softmax():
    """The kernel restates softmax_warp_forward's sum order: torch must run that kernel for the rows it fuses."""
    acts = [torch.profiler.ProfilerActivity.CUDA]
    for n in (577, 1024):
        x = torch.randn(4, 12, n, n, device="cuda")
        with torch.profiler.profile(activities=acts) as prof:
            x.softmax(dim=-1)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "softmax" in e.name.lower()]
        assert names and all("softmax_warp_forward" in s for s in names), (n, names)


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
def test_tiny_vit_577_fused_graph_and_save_load(config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import Attention, VisionTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    from tests import _baseptq_ref as BR
    os.environ.setdefault("TQDM_DISABLE", "1")
    cfg = importlib.import_module(f"ptq4vit_b200.configs.{config}")
    importlib.reload(cfg)
    if config == "BasePTQ":
        BR.baseptq_hessian(cfg)
    kw = dict(img_size=96, patch=4, dim=64, depth=2, num_heads=2, num_classes=10)      # 24 x 24 patches + cls = 577 tokens
    with RH.fp32_convolutions():
        net = VisionTransformer(**kw).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images(size=96)), sequential=False,
                                 batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=3, size=96, seed=11).cuda(), RH.tiny_images(n=3, size=96, seed=12).cuda()
        n_attn = sum(isinstance(m, Attention) for m in net.modules())
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True)
            want, n_unfused = _launches(lambda: net(images))
            want2 = net(images2)
            assert deploy.fuse_attention(net, max_tokens=1024) == []
            got, n_fused = _launches(lambda: net(images))
            assert n_unfused - n_fused == n_attn, "one fused launch in place of two MatMul launches per attention call"
            assert torch.equal(_bits(got), _bits(want))
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
            assert torch.equal(_bits(ys), _bits(want2)), "graph replay of the fused model on new images"
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            deploy.load_quantized(wrapped2, path, matmul=True)
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert deploy.fuse_attention(fresh, max_tokens=1024) == []
            got2, n_fused2 = _launches(lambda: fresh(images))
            assert n_fused2 == n_fused and torch.equal(_bits(got2), _bits(want))
