"""The attention operands' quantisation folded into the frozen qkv, on the GPU.  Every comparison is bitwise: the int8
planes against the reference's MatMul quantiser applied to today's frozen qkv output (with and without
P4V_SCALAR_DIV=ieee), and the attention output against frozen qkv followed by frozen_attention -- ViT-B/224 x 32 with
PTQ4ViT (split-of-softmax matmul2) and BasePTQ at W8A8 / W6A6, n_G = 1 modules, DeiT-S, DeiT-Ti and ViT-S/32, Swin-T
stages 1-4 at shift 0 and window / 2 with the gather fold, Swin-B/384 stage 1, ViT with the norm1 fold, batch 1 / 5 / 32.
A folded attention is two launches and allocates only the planes and the output; refused calls run unfolded with the same
bits; stale step sizes raise; whole tiny ViT and Swin models with every fusion give the same logits with and without
fuse_qkv, eagerly, from one CUDA graph and after a save / load."""
import copy
import importlib
import os

import pytest
import torch

from tests.test_fold_gather_gpu import _layer, _norm, _x
from tests.test_frozen_matmul_gpu import TINY_SWIN
from tests.test_fused_attention_gpu import _frozen_pair, _swin_extras

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} outputs differ, first {bad[:4].tolist()}"


def _steps(v, H):
    return torch.as_tensor(v, dtype=torch.float32).reshape(-1).expand(H).reshape(1, H, 1, 1)


def _want_planes(m1, m2, y, B, N, H, D, scale, scale_on_q):
    """MinMaxQuantMatMul.quant_input without the multiply, on today's qkv output y"""
    q, k, v = y.reshape(B, N, 3, H, D).permute(2, 0, 3, 1, 4).unbind(0)
    if scale_on_q:
        q = q * scale
    out = []
    for t, d, qmax in ((q, m1.A_interval, m1.A_qmax), (k, m1.B_interval, m1.B_qmax), (v, m2.B_interval, m2.B_qmax)):
        out.append((t / _steps(d, H).to(t.device)).round_().clamp_(-qmax, qmax - 1))
    return torch.stack(out)


def _case(lin, x, B, N, H, D, scale, scale_on_q, m2_cls, bit, norm=None, gather=None, extras=None, one_group=False):
    """Frozen MatMul modules for this call's qkv output, then the planes and the attention output, both bitwise"""
    from ptq4vit_b200.quant_layers.linear import frozen_gather_linear, frozen_norm_linear
    from ptq4vit_b200.quant_layers.matmul import (frozen_attention, frozen_qkv_applies, frozen_qkv_attention,
                                                  frozen_qkv_planes)
    bias, mask = extras if extras is not None else (None, None)
    with torch.no_grad():
        if gather is not None:
            y = frozen_gather_linear(norm, lin, x, ("window", *gather))
        elif norm is not None:
            y = frozen_norm_linear(norm, lin, x)
        else:
            y = lin(x)
        qkv5 = y.reshape(B, N, 3, H, D)
        m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", m2_cls, bit, qkv5, scale, scale_on_q, bias, mask,
                              one_group=one_group, seed=bit + N)
        assert frozen_qkv_applies(lin, m1, m2, x, N, H, D, bias, mask, norm=norm, gather=gather)
        planes = frozen_qkv_planes(lin, m1, m2, x, N, H, D, scale, scale_on_q, norm=norm, gather=gather)
        want_p = _want_planes(m1, m2, y, B, N, H, D, scale, scale_on_q)
        assert torch.equal(planes.float(), want_p), int((planes.float() != want_p).sum())
        want = frozen_attention(m1, m2, qkv5, scale, scale_on_q, bias=bias, mask=mask)
        got = frozen_qkv_attention(lin, m1, m2, x, N, H, D, scale, scale_on_q, bias=bias, mask=mask, norm=norm, gather=gather)
        torch.cuda.synchronize()
    _same(got, want)
    return lin, m1, m2


M2 = {"ptq4vit": "SoSPTQSLBatchingQuantMatMul", "baseptq": "PTQSLBatchingQuantMatMul"}


def _qkv_layer(C, config, bit, seed):
    n = C // 64
    return _layer(C, 3 * C, 3 * n if config == "ptq4vit" else 1, n if config == "ptq4vit" else 1,
                  n if config == "ptq4vit" else 1, bit=bit, seed=seed)


@pytest.mark.parametrize("ieee", [False, True])
@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["ptq4vit", "baseptq"])
def test_vit_b_bitwise(config, bit, ieee, monkeypatch):
    if ieee:
        monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    lin = _qkv_layer(768, config, bit, seed=bit)
    x = _x((32, 197, 768), seed=bit, scale=1.0, offset_rows=False)
    _case(lin, x, 32, 197, 12, 64, 64 ** -0.5, False, M2[config], bit)


@pytest.mark.parametrize("m2", ["ptq4vit", "baseptq"])
def test_one_group_modules(m2):
    lin = _qkv_layer(384, "baseptq", 8, seed=11)
    _case(lin, _x((5, 197, 384), seed=12, scale=1.0, offset_rows=False), 5, 197, 6, 64, 64 ** -0.5, False, M2[m2], 8,
          one_group=True)


# (C, heads, tokens): DeiT-S, DeiT-Ti, ViT-S/32
SMALL = {"deit_s": (384, 6, 197), "deit_ti": (192, 3, 197), "vit_s32": (384, 6, 50)}


@pytest.mark.parametrize("name", list(SMALL))
def test_small_models_and_batches(name):
    C, H, N = SMALL[name]
    lin = _qkv_layer(C, "ptq4vit", 8, seed=C + N)
    for B in (1, 5, 32):
        _case(lin, _x((B, N, C), seed=B, scale=1.0, offset_rows=False), B, N, H, C // H, (C // H) ** -0.5, False,
              M2["ptq4vit"], 8)


def test_vit_norm1_fold():
    lin = _qkv_layer(768, "ptq4vit", 8, seed=21)
    norm = _norm(768, seed=22)
    for B in (1, 32):
        _case(lin, _x((B, 197, 768), seed=B), B, 197, 12, 64, 64 ** -0.5, False, M2["ptq4vit"], 8, norm=norm)


# (C, heads, res, window): Swin-T stages 1-4, Swin-B/384 stage 1
SWIN = {"swint_s1": (96, 3, 56, 7), "swint_s2": (192, 6, 28, 7), "swint_s3": (384, 12, 14, 7), "swint_s4": (768, 24, 7, 7),
        "swinb384_s1": (128, 4, 96, 12)}


@pytest.mark.parametrize("m2", ["ptq4vit", "baseptq"])
@pytest.mark.parametrize("name", list(SWIN))
def test_swin_gather_bitwise(name, m2):
    C, H, res, ws = SWIN[name]
    n = C // 32
    lin = _layer(C, 3 * C, 3 * n, n, n, seed=C + res)
    norm = _norm(C, seed=C)
    N, nW = ws * ws, (res // ws) ** 2
    for B in ((1, 5) if name != "swint_s1" else (1, 32)):
        for shift in (0, ws // 2) if res > ws else (0,):
            bias, mask = _swin_extras(H, N, nW if shift else 0, seed=C + shift)
            x = _x((B, res * res, C), seed=B + shift)
            _case(lin, x, B * nW, N, H, C // H, (C // H) ** -0.5, True, M2[m2], 8, norm=norm, gather=(B, res, res, ws, shift),
                  extras=(bias, mask))


def test_two_launches_planes_and_output_allocated_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.matmul import frozen_attention, frozen_qkv_attention
    lin = _qkv_layer(768, "ptq4vit", 8, seed=31)
    x, x2 = [_x((8, 197, 768), seed=s, scale=1.0, offset_rows=False) for s in (32, 33)]
    with torch.no_grad():
        y = lin(x)
        m1, m2 = _frozen_pair("PTQSLBatchingQuantMatMul", M2["ptq4vit"], 8, y.view(8, 197, 3, 12, 64), 0.125, False)
        args = (lin, m1, m2)
        frozen_qkv_attention(*args, x, 197, 12, 64, 0.125, False)
        torch.cuda.synchronize()
        n0, a0 = _lib.launch_count(), torch.cuda.memory_stats()["allocation.all.allocated"]
        frozen_qkv_attention(*args, x, 197, 12, 64, 0.125, False)
        torch.cuda.synchronize()
        assert _lib.launch_count() - n0 == 2
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - a0 == 2, "only the planes and the output"
        want = [frozen_attention(m1, m2, lin(t).view(8, 197, 3, 12, 64), 0.125, False) for t in (x, x2)]
        xs = x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_qkv_attention(*args, xs, 197, 12, 64, 0.125, False)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ys = frozen_qkv_attention(*args, xs, 197, 12, 64, 0.125, False)
        for i, src in enumerate((x, x2)):
            xs.copy_(src)
            graph.replay()
            torch.cuda.synchronize()
            _same(ys, want[i])


def _block(dim, heads, seed):
    """An Attention module with frozen qkv, proj, matmul1 and matmul2 (min-max-like step sizes)"""
    from ptq4vit_b200.utils.models import Attention
    att = Attention(dim, heads).cuda().eval()
    att.qkv = _qkv_layer(dim, "baseptq", 8, seed=seed)
    att.proj = _layer(dim, dim, seed=seed + 1)
    return att


def test_refused_calls_run_unfolded_and_stale_steps_raise():
    from ptq4vit_b200.quant_layers.matmul import frozen_qkv_applies, frozen_qkv_attention
    from ptq4vit_b200.utils import deploy
    att = _block(128, 2, seed=41)
    for N in (197, 577):
        x = _x((2, N, 128), seed=N, scale=1.0, offset_rows=False)
        with torch.no_grad():
            y = att.qkv(x)
            att.matmul1, att.matmul2 = _frozen_pair("PTQSLBatchingQuantMatMul", M2["ptq4vit"], 8, y.view(2, N, 3, 2, 64),
                                                    0.125, False)
            deploy.fuse_attention(att, max_tokens=1024)
            want = att(x)
            assert deploy.fuse_qkv(att) == []
            _same(att(x), want)
            assert frozen_qkv_applies(att.qkv, att.matmul1, att.matmul2, x, N, 2, 64) == (N <= 256)
            if N <= 256:
                # an unfrozen qkv runs unfolded, same bits
                att.qkv.unfreeze()
                assert not frozen_qkv_applies(att.qkv, att.matmul1, att.matmul2, x, N, 2, 64)
                _same(att(x), want)
                att.qkv.freeze()
        deploy.unfuse_qkv(att)
    # grad mode: the input requires grad
    xg = x.clone().requires_grad_(True)
    deploy.fuse_qkv(att)
    assert not frozen_qkv_applies(att.qkv, att.matmul1, att.matmul2, xg, 577, 2, 64)
    x = _x((2, 197, 128), seed=197, scale=1.0, offset_rows=False)
    with torch.no_grad():
        y = att.qkv(x)
        att.matmul1, att.matmul2 = _frozen_pair("PTQSLBatchingQuantMatMul", M2["ptq4vit"], 8, y.view(2, 197, 3, 2, 64),
                                                0.125, False)
        deploy.unfuse_qkv(att)
        want = att(x)
        deploy.fuse_qkv(att)
    xg = x.clone().requires_grad_(True)
    assert not frozen_qkv_applies(att.qkv, att.matmul1, att.matmul2, xg, 197, 2, 64)
    out = att(xg)
    assert torch.equal(_bits(out.detach()), _bits(want))
    with torch.no_grad():
        att.matmul1.A_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_qkv_attention(att.qkv, att.matmul1, att.matmul2, x, 197, 2, 64, 0.125, False)
        att.matmul1.A_interval.div_(1.01)
        att.matmul1.unfreeze().freeze()
        att.qkv.a_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            att(x)


def _launches(net, images):
    from ptq4vit_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = net(images)
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_whole_model_folded_graph_and_save_load(kind, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import Attention, SwinTransformer, VisionTransformer, WindowAttention
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    os.environ.setdefault("TQDM_DISABLE", "1")
    cfg = importlib.import_module("ptq4vit_b200.configs.PTQ4ViT")
    importlib.reload(cfg)

    def fuse_all(net):
        assert deploy.fuse_attention(net) == [] and deploy.fuse_mlp(net) == [] and deploy.fuse_residual(net) == []
        deploy.fuse_norm(net)
        deploy.fuse_gather(net)
        deploy.fuse_stem(net)

    with RH.fp32_convolutions():
        net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        attn = [m for m in net.modules() if isinstance(m, (Attention, WindowAttention))]
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True, conv=True)
            fuse_all(net)
            assert not any(m.fold_qkv for m in attn), "fold_qkv defaults to off"
            want, n_unfolded = _launches(net, images)
            want2 = net(images2)
            assert deploy.fuse_qkv(net) == []
            got, n_folded = _launches(net, images)
            assert n_folded == n_unfolded, "qkv and the attention: two launches either way"
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
            fuse_all(fresh)
            assert not any(m.fold_qkv for m in fresh.modules() if isinstance(m, (Attention, WindowAttention)))
            assert deploy.fuse_qkv(fresh) == []
            _same(fresh(images), want)
            deploy.unfuse_qkv(net)
            assert not any(m.fold_qkv for m in attn)
            _same(net(images), want)
