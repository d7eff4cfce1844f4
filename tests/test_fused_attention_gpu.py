"""The fused frozen attention core on the GPU: bit-identical (as int32 bit patterns) to matmul1, the scale / bias / mask,
torch's softmax, matmul2 and the transpose on the frozen modules, for ViT-B/224, Swin-T and Swin-B/384 windows, PTQ4ViT
(split-of-softmax matmul2), BasePTQ and the no_softmax ablation (plain matmul2), W8A8 / W6A6, n_G = 1 modules, batch 1
and odd batches; one launch, no copy, no allocation but the output; stale step sizes raise; grad mode and DeiT-B/384's
577 tokens run unfused; whole tiny models fused give the unfused logits eagerly, from one CUDA graph and after a
save / load."""
import copy
import importlib
import os

import pytest
import torch

from tests.test_frozen_matmul_gpu import TINY_SWIN, _bits, _module

pytestmark = pytest.mark.gpu


def _qkv(batch, N, H, D, seed, amp=1.0):
    """The qkv Linear's output [batch, N, 3 * H * D], and its [batch, N, 3, H, D] view."""
    g = torch.Generator().manual_seed(seed)
    y = (torch.randn(batch, N, 3 * H * D, generator=g) * amp).cuda()
    return y, y.view(batch, N, 3, H, D)


def _swin_extras(H, N, nW, seed):
    """A relative-position bias [H, N, N] and a shifted-window mask [nW, N, N] of 0 / -100 entries."""
    g = torch.Generator().manual_seed(seed)
    bias = (torch.randn(H, N, N, generator=g) * 0.5).cuda()
    mask = None
    if nW:
        group = torch.randint(0, 3, (nW, N), generator=g)
        mask = torch.where(group[:, :, None] == group[:, None, :], 0.0, -100.0).cuda()
    return bias, mask


def _unfused(m1, m2, qkv5, scale, scale_on_q, bias=None, mask=None):
    """The attention forward of utils/models.py between qkv and proj, on the modules."""
    B, N, _, H, D = qkv5.shape
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
    attn = attn.softmax(dim=-1)
    return m2.quant_forward(attn, v).transpose(1, 2).reshape(B, N, H * D)


def _frozen_pair(cls1, cls2, bit, qkv5, scale, scale_on_q, bias=None, mask=None, one_group=False, seed=0):
    """matmul1 / matmul2 modules with step sizes near the min-max ones of this input, frozen."""
    q, k, v = qkv5.permute(2, 0, 3, 1, 4).unbind(0)
    H = qkv5.shape[3]
    m1 = _module(cls1, bit, H, q * scale if scale_on_q else q, k.transpose(-2, -1), seed=seed, one_group=one_group)
    m1.mode = "quant_forward"
    probs = _unfused_probs(m1, qkv5, scale, scale_on_q, bias, mask)
    m2 = _module(cls2, bit, H, probs, v, seed=seed + 1, one_group=one_group)
    m2.mode = "quant_forward"
    return m1.freeze(), m2.freeze()


def _unfused_probs(m1, qkv5, scale, scale_on_q, bias, mask):
    B, N, _, H, D = qkv5.shape
    q, k, _ = qkv5.permute(2, 0, 3, 1, 4).unbind(0)
    attn = m1.quant_forward(q * scale if scale_on_q else q, k.transpose(-2, -1))
    attn = attn if scale_on_q else attn * scale
    if bias is not None:
        attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = (attn.view(B // nW, nW, H, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, H, N, N)
    return attn.softmax(dim=-1)


def _check(m1, m2, qkv5, scale, scale_on_q, bias=None, mask=None):
    from ptq4vit_b200.quant_layers.matmul import frozen_attention, frozen_attention_applies
    B, N, _, H, D = qkv5.shape
    assert frozen_attention_applies(m1, m2, N, D, qkv5, bias, mask)
    with torch.no_grad():
        want = _unfused(m1, m2, qkv5, scale, scale_on_q, bias, mask)
        got = frozen_attention(m1, m2, qkv5, scale, scale_on_q, bias=bias, mask=mask)
    assert got.shape == want.shape
    diff = int((_bits(got) != _bits(want)).sum())
    assert diff == 0, f"{diff} of {got.numel()} differ (max abs {float((got - want).abs().max()):.3g})"


VIT_SCALE = 64 ** -0.5
M2 = {"ptq4vit": "SoSPTQSLBatchingQuantMatMul", "baseptq": "PTQSLBatchingQuantMatMul",
      "no_softmax": "PTQSLBatchingQuantMatMul"}      # the no_softmax ablation gives matmul2 the plain class (configs/PTQ4ViT.py)


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["ptq4vit", "baseptq", "no_softmax"])
def test_vit_b_bitwise(config, bit):
    _, qkv5 = _qkv(32, 197, 12, 64, seed=bit)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", M2[config], bit, qkv5, VIT_SCALE, False)
    _check(m1, m2, qkv5, VIT_SCALE, False)


@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLQuantMatMul"])
def test_one_group_modules(m2_cls):
    _, qkv5 = _qkv(4, 197, 12, 64, seed=21)
    m1, m2 = _frozen_pair("PTQSLQuantMatMul", m2_cls, 8, qkv5, VIT_SCALE, False, one_group=True)
    _check(m1, m2, qkv5, VIT_SCALE, False)


@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
def test_small_and_odd_batches(batch, m2_cls):
    _, qkv5 = _qkv(batch, 197, 12, 64, seed=30 + batch)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, VIT_SCALE, False)
    _check(m1, m2, qkv5, VIT_SCALE, False)


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("m2_cls", ["SoSPTQSLBatchingQuantMatMul", "PTQSLBatchingQuantMatMul"])
@pytest.mark.parametrize("shape", [(128, 49, 3, 32, 64),      # Swin-T/224 stage 1: 2 images x 64 windows of 7 x 7
                                   (32, 144, 4, 32, 16)])     # Swin-B/384 stage 1 windows of 12 x 12 (2 images x 16)
def test_swin_windows_bitwise(shape, m2_cls, shifted):
    B_, N, H, D, nW = shape
    _, qkv5 = _qkv(B_, N, H, D, seed=N + shifted, amp=2.0)
    bias, mask = _swin_extras(H, N, nW if shifted else 0, seed=N)
    scale = D ** -0.5
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, scale, True, bias, mask)
    _check(m1, m2, qkv5, scale, True, bias, mask)


def _attention_block(dim, H, N, m2_cls, seed):
    """A models.Attention block with frozen MatMul modules calibrated on its own input x."""
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Attention
    torch.manual_seed(seed)
    blk = Attention(dim, H).cuda().eval()
    x = torch.randn(2, N, dim, device="cuda")
    with torch.no_grad():
        qkv5 = blk.qkv(x).view(2, N, 3, H, dim // H)
    blk.matmul1, blk.matmul2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, 8, qkv5, blk.scale, False)
    return blk, x, deploy


def test_deit_384_runs_unfused():
    from ptq4vit_b200 import _lib
    blk, x, deploy = _attention_block(768, 12, 577, "SoSPTQSLBatchingQuantMatMul", seed=5)
    with torch.no_grad():
        want = blk(x)
        assert deploy.fuse_attention(blk) == []
        n0 = _lib.launch_count()
        got = blk(x)
        torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 2, "577 tokens: the two frozen MatMul kernels, not the fused one"
    assert torch.equal(_bits(got), _bits(want))


def _copies(fn):
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        y = fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "memcpy" in e.name.lower()], y


def test_one_launch_no_copy_no_allocation():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    _, qkv5 = _qkv(8, 197, 12, 64, seed=41)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul", 8, qkv5, VIT_SCALE, False)
    with torch.no_grad():
        want = _unfused(m1, m2, qkv5, VIT_SCALE, False)
        frozen_attention(m1, m2, qkv5, VIT_SCALE, False)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        copies, y = _copies(lambda: frozen_attention(m1, m2, qkv5, VIT_SCALE, False))
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
    assert _lib.launch_count() - n0 == 1
    assert not copies, f"the fused call issued a copy: {copies}"
    assert torch.equal(_bits(y), _bits(want))


def test_stale_step_sizes_raise():
    from ptq4vit_b200.quant_layers.matmul import frozen_attention
    _, qkv5 = _qkv(2, 197, 12, 64, seed=42)
    m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul", 8, qkv5, VIT_SCALE, False)
    with torch.no_grad():
        frozen_attention(m1, m2, qkv5, VIT_SCALE, False)
        m2.split.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_attention(m1, m2, qkv5, VIT_SCALE, False)
        m2.unfreeze(); m2.freeze()
        frozen_attention(m1, m2, qkv5, VIT_SCALE, False)
        m1.B_interval = m1.B_interval * 1.0
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_attention(m1, m2, qkv5, VIT_SCALE, False)


def test_grad_mode_runs_unfused():
    from ptq4vit_b200 import _lib
    blk, x, deploy = _attention_block(768, 12, 197, "SoSPTQSLBatchingQuantMatMul", seed=6)
    deploy.fuse_attention(blk)
    with torch.no_grad():
        want = blk(x)
        deploy.unfuse_attention(blk)
        assert torch.equal(_bits(blk(x)), _bits(want)), "fused and unfused block"
        deploy.fuse_attention(blk)
    xg = x.clone().requires_grad_(True)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    y = blk(xg)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 2, "grad mode: the two MatMul modules, not the fused kernel"
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))


def _attention_launches(net, images, n_attn):
    from ptq4vit_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = net(images)
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_whole_model_fused_graph_and_save_load(kind, config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import Attention, SwinTransformer, VisionTransformer, WindowAttention
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
        attn = [n for n, m in net.named_modules() if isinstance(m, (Attention, WindowAttention))]
        with torch.no_grad():
            assert deploy.fuse_attention(net) == attn, "nothing frozen yet: every attention module is left unfused"
            deploy.unfuse_attention(net)
            deploy.freeze_model(wrapped, matmul=True)
            want, n_unfused = _attention_launches(net, images, len(attn))
            want2 = net(images2)
            assert deploy.fuse_attention(net) == []
            got, n_fused = _attention_launches(net, images, len(attn))
            assert n_unfused - n_fused == len(attn), "one fused launch in place of two MatMul launches per attention call"
            assert torch.equal(_bits(got), _bits(want))
            # the whole fused forward in one CUDA graph
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
            # saved and loaded into a fresh copy, MatMul modules frozen from the file, then fused
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            deploy.load_quantized(wrapped2, path, matmul=True)
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert deploy.fuse_attention(fresh) == []
            got2, n_fused2 = _attention_launches(fresh, images, len(attn))
            assert n_fused2 == n_fused and torch.equal(_bits(got2), _bits(want))
            deploy.unfuse_attention(net)
            assert torch.equal(_bits(net(images)), _bits(want))
