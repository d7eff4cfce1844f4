"""The frozen MatMul forward on the GPU: bit-identical (as int32 bit patterns: the forward's -r makes signed zeros) to the
unfrozen quant_forward for the attention products of ViT-B, DeiT-B/384 and Swin, with the real permuted q / k / v views
and with contiguous copies; equal to an fp64 restatement; one launch, no copy, no allocation but the output; capturable
in a CUDA graph; and whole tiny models frozen with their MatMul modules, replayed from one graph, saved and loaded."""
import copy
import importlib
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _qkv(batch, N, H, hd, seed):
    """q, k, v as the attention blocks make them: permuted views of one qkv output [batch, N, 3, H, hd]."""
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(batch, N, 3, H, hd, generator=g) * 2.0).cuda().permute(2, 0, 3, 1, 4)
    return qkv.unbind(0)


def _module(cls_name, bit, H, A, B, seed=0, one_group=False):
    """A calibrated module with step sizes near the min-max ones (perturbed per head), no search needed."""
    from ptq4vit_b200.quant_layers import matmul as MM
    g = torch.Generator().manual_seed(seed)
    m = getattr(MM, cls_name)(A_bit=bit, B_bit=bit)
    n = 1 if one_group else H
    jitter = lambda: (0.7 + 0.3 * torch.rand(n, generator=g)).cuda()
    if one_group:
        m.n_G_A = m.n_G_B = 1
    amax = A.detach().abs().amax(dim=(0, 2, 3)) if not one_group else A.detach().abs().amax().reshape(1)
    bmax = B.detach().abs().amax(dim=(0, 2, 3)) if not one_group else B.detach().abs().amax().reshape(1)
    m.B_interval = (bmax / (m.B_qmax - 0.5) * jitter()).view(1, n, 1, 1, 1, 1, 1)
    if m.sos:
        m.split = torch.tensor(0.0625 * (0.5 + float(torch.rand(1, generator=g)))).cuda()
        m.A_interval = m.split / (m.A_qmax - 1)
    else:
        m.A_interval = (amax / (m.A_qmax - 0.5) * jitter()).view(1, n, 1, 1, 1, 1, 1)
    m.calibrated = True
    return m


def _attention(batch, N, H, hd, seed=0):
    """(q, k^T) of matmul1 and (softmax probabilities, v) of matmul2, as views."""
    q, k, v = _qkv(batch, N, H, hd, seed)
    probs = (q @ k.transpose(-2, -1) * hd ** -0.5).softmax(dim=-1)
    return (q, k.transpose(-2, -1)), (probs, v)


def _fp64(m, A, B):
    """fq(A) fq(B) restated: integers from fp32 quantisers as the reference's (IEEE quotients: an fp64 quotient of two
    fp32 values rounds to the fp32 one), products summed in fp64 (exact), scaled in fp32."""
    H = A.shape[1]
    dB = torch.as_tensor(m.B_interval, dtype=torch.float32).reshape(-1).expand(H).reshape(1, H, 1, 1)
    Bq = (B.double() / dB.double()).float().round().clamp(-m.B_qmax, m.B_qmax - 1).double()
    if m.sos:
        qm1 = m.A_qmax - 1
        split = torch.as_tensor(m.split, dtype=torch.float32).reshape(1).cpu()
        aux0 = (torch.ones(1, dtype=torch.float64) / qm1).float()
        aux1 = (split.double() / qm1).float()
        hi = (A.clamp(float(split), 1.0) * float(qm1)).round().clamp(0, qm1).double()
        lo = (A.clamp(0, float(split)).double() / float(aux1)).float().round().clamp(0, qm1).double()
        s0, s1 = (dB * aux0.to(dB.device)), (dB * aux1.to(dB.device))
        lo_term = (lo @ Bq).float() * s1
        return (hi @ Bq).float() * s0 + lo_term, lo_term.abs()
    dA = torch.as_tensor(m.A_interval, dtype=torch.float32).reshape(-1).expand(H).reshape(1, H, 1, 1)
    Aq = (A.double() / dA.double()).float().round().clamp(-m.A_qmax, m.A_qmax - 1).double()
    r = -(dA * dB) * (Aq @ Bq).float() + 0.0          # the sweep's fmaf(-scale, acc, 0): a zero product is +0 ...
    return -r, None                                    # ... and the output -r


def _check(m, A, B, fp64=True):
    want = m.quant_forward(A, B)
    m.freeze()
    assert m.frozen
    got = m.quant_forward(A, B)
    assert got.shape == want.shape and torch.equal(_bits(got), _bits(want)), \
        f"{type(m).__name__}: {int((_bits(got) != _bits(want)).sum())} of {got.numel()} differ"
    got_c = m.quant_forward(A.contiguous(), B.contiguous())
    assert torch.equal(_bits(got_c), _bits(want)), "contiguous copies must give the bits of the views"
    if fp64:
        ref, lo_term = _fp64(m, A, B)
        if m.sos:
            # the kernel rounds hi + lo once (fmaf), the restatement rounds the low term first: half an ulp of each result
            # plus half an ulp of the low term (one ulp of the result unless the two terms cancel)
            bound = (got.double().abs() + ref.double().abs() + lo_term.double()) * 2.0 ** -24
            assert bool(((got.double() - ref.double()).abs() <= bound).all()), \
                f"worst {float(((got.double() - ref.double()).abs() / bound).nan_to_num(0.0).max()):.2f} of the fp32 bound"
        else:
            assert torch.equal(_bits(got), _bits(ref)), f"{int((_bits(got) != _bits(ref)).sum())} differ from the fp64 restatement"
    m.unfreeze()
    assert not m.frozen and torch.equal(_bits(m.quant_forward(A, B)), _bits(want))


# ViT-B/224 x 32: matmul1 with PTQ4ViT / BasePTQ (the same class), matmul2 with the split-of-softmax (PTQ4ViT) and
# the plain (BasePTQ) class
@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("which,cls_name", [("matmul1", "PTQSLBatchingQuantMatMul"), ("matmul2", "SoSPTQSLBatchingQuantMatMul"),
                                            ("matmul2", "PTQSLBatchingQuantMatMul"), ("matmul1", "MinMaxQuantMatMul"),
                                            ("matmul2", "MinMaxQuantMatMul")])
def test_vit_b_attention_bitwise(which, cls_name, bit):
    mm1, mm2 = _attention(32, 197, 12, 64)
    A, B = mm1 if which == "matmul1" else mm2
    _check(_module(cls_name, bit, 12, A, B), A, B)


@pytest.mark.parametrize("which", ["matmul1", "matmul2"])
def test_one_group_non_batching_module(which):
    mm1, mm2 = _attention(4, 197, 12, 64, seed=3)
    A, B = mm1 if which == "matmul1" else mm2
    _check(_module("PTQSLQuantMatMul", 8, 12, A, B, one_group=True), A, B)


@pytest.mark.parametrize("shape", [
    (4, 577, 12, 64),      # DeiT-B/384
    (64, 49, 3, 32),       # Swin-T/224 windows: S2 < 64, the unfrozen forward runs bf16
    (16, 144, 4, 32),      # Swin-B/384 windows
    (3, 77, 5, 40),        # odd batch, S1 / S3 not tile multiples, S2 = 40 (not a multiple of 32)
    (2, 130, 2, 72),       # two row tiles with a 2-row tail; matmul2 S3 = 72 > 64: 128-column tiles, two accumulators
])
@pytest.mark.parametrize("cls_name", ["PTQSLBatchingQuantMatMul", "SoSPTQSLBatchingQuantMatMul"])
def test_other_shapes_bitwise(shape, cls_name):
    mm1, mm2 = _attention(*shape, seed=sum(shape))
    if cls_name == "PTQSLBatchingQuantMatMul":
        _check(_module(cls_name, 8, shape[2], *mm1), *mm1)
    _check(_module(cls_name, 8, shape[2], *mm2), *mm2)


@pytest.mark.parametrize("which", ["matmul1", "matmul2"])
def test_ieee_scalar_division(which, monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    mm1, mm2 = _attention(4, 197, 12, 64, seed=5)
    A, B = mm1 if which == "matmul1" else mm2
    _check(_module("SoSPTQSLBatchingQuantMatMul" if which == "matmul2" else "PTQSLBatchingQuantMatMul", 8, 12, A, B), A, B)


def _copies(m, A, B):
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        y = m.quant_forward(A, B)
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "memcpy" in e.name.lower()], y


@pytest.mark.parametrize("which", ["matmul1", "matmul2"])
def test_one_launch_no_copy_no_allocation_and_graph_replay(which):
    from ptq4vit_b200 import _lib
    mm1, mm2 = _attention(8, 197, 12, 64, seed=11)
    mm1b, mm2b = _attention(8, 197, 12, 64, seed=12)
    (A, B), (A2, B2) = (mm1, mm1b) if which == "matmul1" else (mm2, mm2b)
    m = _module("PTQSLBatchingQuantMatMul" if which == "matmul1" else "SoSPTQSLBatchingQuantMatMul", 8, 12, A, B)
    want, want2 = m.quant_forward(A, B), m.quant_forward(A2, B2)
    assert _copies(m, A, B)[0], "the profiler must see the table uploads of the unfrozen forward"
    m.freeze()
    m.quant_forward(A, B)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
    copies, y = _copies(m, A, B)
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
    assert _lib.launch_count() - n0 == 1
    assert not copies, f"the frozen forward issued a copy: {copies}"
    assert torch.equal(_bits(y), _bits(want))
    # capture once, replay on new input (the views' storage is refilled in place)
    As, Bs = A.clone(), B.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m.quant_forward(As, Bs)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ys = m.quant_forward(As, Bs)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(ys), _bits(want))
    As.copy_(A2); Bs.copy_(B2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(ys), _bits(want2)), "graph replay on new input"


def test_stale_step_sizes_raise():
    mm1, mm2 = _attention(2, 197, 12, 64, seed=2)
    m = _module("SoSPTQSLBatchingQuantMatMul", 8, 12, *mm2)
    m.freeze()
    m.quant_forward(*mm2)
    m.split.mul_(1.01)
    with pytest.raises(RuntimeError, match="step sizes changed"):
        m.quant_forward(*mm2)
    m.unfreeze(); m.freeze()
    m.quant_forward(*mm2)
    m.B_interval = m.B_interval * 1.0
    with pytest.raises(RuntimeError, match="step sizes changed"):
        m.quant_forward(*mm2)


def test_grad_mode_call():
    mm1, _ = _attention(2, 197, 12, 64, seed=4)
    A, B = [t.detach().clone().requires_grad_(True) for t in mm1]
    m = _module("PTQSLBatchingQuantMatMul", 8, 12, A, B)
    with torch.no_grad():
        want = m.quant_forward(A, B)
    m.freeze()
    y = m.quant_forward(A, B)
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))
    y.sum().backward()
    assert torch.count_nonzero(A.grad) == 0 and torch.count_nonzero(B.grad) == 0


TINY_SWIN = dict(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_whole_model_frozen_graph_and_save_load(kind, config, tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
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
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        with torch.no_grad():
            want, want2 = net(images), net(images2)
            left = deploy.freeze_model(wrapped, matmul=True)
            matmuls = [n for n, m in wrapped.items() if isinstance(m, MinMaxQuantMatMul)]
            assert matmuls and all(wrapped[n].frozen for n in matmuls)
            assert len(left) == 1 and "patch_embed" in left[0], left
            assert torch.equal(_bits(net(images)), _bits(want))
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
            # saved and loaded into a fresh copy, MatMul modules frozen from the file's step sizes
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            left2 = deploy.load_quantized(wrapped2, path, matmul=True)
            assert sorted(left2) == sorted(left)
            assert all(wrapped2[n].frozen for n in matmuls)
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert torch.equal(_bits(fresh(images)), _bits(want))
            deploy.unfreeze_model(wrapped)
            assert not any(wrapped[n].frozen for n in matmuls)
