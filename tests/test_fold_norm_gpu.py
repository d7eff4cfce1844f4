"""A LayerNorm folded into the frozen Linear that consumes it, on the GPU.  Every comparison is of int32 bit patterns:
the LayerNorm of the fused kernel's prologue (p4v_layer_norm_probe) against torch's F.layer_norm over every width the
zoo normalises, both epsilons and rows that stress the reduction; a profiler guard that torch still runs the kernel the
emulation follows; the folded call against the unfolded frozen lin(norm(x)) for ViT-B qkv, fc1 (plain and composed with
the fused MLP) and head, Swin-T fc1 and a PatchMerging reduction, PTQ4ViT / BasePTQ blocks, W8A8 / W6A6, n_a > 1, row
tails and batch 1 / 5 / 32; one launch, no allocation but the output, CUDA-graph capture and replay; stale step sizes raise,
grad mode and rejected shapes run unfolded; whole tiny ViT and Swin models give the unfolded logits eagerly, from one
CUDA graph and after a save / load."""
import copy
import ctypes
import importlib
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TINY_SWIN = dict(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _layer(K, O, n_V, n_H, n_a=1, gelu=False, bias=True, bit=8, seed=0):
    """A calibrated layer with hand-set step sizes near the min-max ones (no search needed for a forward)."""
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear, PTQSLBatchingQuantLinear
    g = torch.Generator().manual_seed(seed)
    cls = PostGeluPTQSLBatchingQuantLinear if gelu else PTQSLBatchingQuantLinear
    m = cls(K, O, bias=bias, w_bit=bit, a_bit=bit, n_V=n_V, n_H=n_H, n_a=n_a)
    m.weight.data = torch.randn(O, K, generator=g) * 0.05
    if bias:
        m.bias.data = torch.randn(O, generator=g)
    m = m.cuda()
    q = 2 ** (bit - 1) - 0.5
    wmax = m.weight.data.view(n_V, O // n_V, n_H, K // n_H).abs().amax(dim=(1, 3))
    m.w_interval = (wmax / q * (0.7 + 0.3 * torch.rand(n_V, n_H, generator=g).cuda())).view(n_V, 1, n_H, 1)
    m.a_interval = ((2.5 if gelu else 3.0) / q * (0.7 + 0.3 * torch.rand(n_a, 1, generator=g))).cuda()
    m.calibrated = True
    return m

VIT_ROWS = 32 * 197
WIDTHS = [96, 192, 384, 512, 768, 1024, 1536, 2048]


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _probe(x, w, b, eps):
    from ptq4vit_b200 import _lib
    y = torch.empty_like(x)
    _lib.check(_lib.lib().p4v_layer_norm_probe(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), ctypes.c_float(eps), x.shape[0], x.shape[1],
                                               _lib.ptr(y), _stream()), "p4v_layer_norm_probe")
    return y


def _rows(N, seed):
    """Random rows of several scales, rows whose mean dwarfs their spread, constant rows, huge and tiny magnitudes, and
    rows holding inf or NaN."""
    g = torch.Generator().manual_seed(seed)
    parts = [torch.randn(2048, N, generator=g),
             torch.randn(512, N, generator=g) * torch.logspace(-3, 3, 512).unsqueeze(1),
             1000.0 + 1e-3 * torch.randn(256, N, generator=g),
             -3.0e4 + torch.randn(256, N, generator=g),
             torch.full((64, N), 0.37), torch.zeros(16, N), torch.full((16, N), -1.5e6),
             torch.randn(64, N, generator=g) * 1e18, torch.randn(64, N, generator=g) * 1e-20,
             torch.randn(64, N, generator=g) * 1e-38]
    special = torch.randn(32, N, generator=g)
    special[0:8, 3] = float("inf")
    special[8:16, N // 2] = float("-inf")
    special[16:24, 1] = float("nan")
    special[24:32, :2] = torch.tensor([float("inf"), float("-inf")])
    parts.append(special)
    return torch.cat(parts).cuda()


def _affine(N, seed):
    g = torch.Generator().manual_seed(seed)
    return (1.0 + 0.5 * torch.randn(N, generator=g)).cuda(), (0.3 * torch.randn(N, generator=g)).cuda()


def _same_bits(got, want):
    same = (got.view(torch.int32) == want.view(torch.int32)) | (got.isnan() & want.isnan())
    return (~same).nonzero()


@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("N", WIDTHS)
def test_probe_bits_match_torch(N, eps):
    x = _rows(N, seed=N)
    for w, b in [_affine(N, 1), (torch.ones(N, device="cuda"), torch.zeros(N, device="cuda"))]:
        want = F.layer_norm(x, (N,), w, b, eps)
        got = _probe(x, w, b, eps)
        torch.cuda.synchronize()
        bad = _same_bits(got, want)
        assert bad.numel() == 0, f"{bad.shape[0]} elements differ, first (row, col) {bad[:4].tolist()}"


_GUARD = """
import torch, torch.nn.functional as F
widths = %r
inputs = [(torch.randn(64, N, device="cuda"), torch.rand(N, device="cuda") + 0.5, torch.randn(N, device="cuda")) for N in widths]
torch.cuda.synchronize()
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.profiler.profile(activities=acts) as prof:
    for x, w, b in inputs:
        F.layer_norm(x, (x.shape[1],), w, b, 1e-6)
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        block = getattr(e, "block", None) or getattr(e, "kwinputs", {}).get("block")
        print("KERNEL", e.name, "BLOCK", tuple(block)[:2] if block else None)
"""


def test_guard_torch_runs_the_emulated_kernel():
    """torch's LayerNorm at these shapes must still be vectorized_layer_norm_kernel with 128-thread blocks (32 x 4): the
    order p4v_ln_row_stats restates.  A torch that changes it fails here rather than with scattered bit differences.  The
    profiler runs in a child process, so that this process's later profiler sessions start from a clean state."""
    r = subprocess.run([sys.executable, "-c", _GUARD % (WIDTHS,)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    kernels = [ln.split(" BLOCK ") for ln in r.stdout.splitlines() if ln.startswith("KERNEL ")]
    names = [k[0][len("KERNEL "):] for k in kernels]
    assert len(kernels) == len(WIDTHS) and all("vectorized_layer_norm_kernel" in n for n in names), (
        f"torch's LayerNorm at N={WIDTHS} ran {names}, not the vectorised kernel the fold reproduces (DESIGN.md section 4.10)")
    for N, k in zip(WIDTHS, kernels):
        assert k[1] in ("None", "(32, 4)"), f"N={N}: vectorized_layer_norm_kernel block {k[1]}, the emulation assumes (32, 4)"


def _norm(N, eps=1e-6, seed=5):
    ln = torch.nn.LayerNorm(N, eps=eps).cuda()
    w, b = _affine(N, seed)
    with torch.no_grad():
        ln.weight.copy_(w)
        ln.bias.copy_(b)
    return ln


def _frozen(K, O, n_V=1, n_H=1, n_a=1, bit=8, seed=0, bias=True):
    m = _layer(K, O, n_V, n_H, n_a=n_a, bit=bit, seed=seed, bias=bias)
    m.freeze()
    m.mode = "quant_forward"
    return m


def _x(rows, K, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, K, generator=g) * 2.0 + torch.randn(rows, 1, generator=g)).cuda()


def _check_fold(ln, lin, x):
    from ptq4vit_b200.quant_layers.linear import frozen_norm_applies, frozen_norm_linear
    with torch.no_grad():
        assert frozen_norm_applies(ln, lin, x)
        want = lin(ln(x))
        got = frozen_norm_linear(ln, lin, x)
        torch.cuda.synchronize()
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} outputs differ, first {bad[:4].tolist()}"


# name: (K, O, n_V, n_H) -- PTQ4ViT's blocks of the layer, BasePTQ's are 1 x 1
LAYERS = {
    "vitb_qkv": (768, 2304, 24, 24),
    "vitb_fc1": (768, 3072, 24, 24),
    "vitb_head": (768, 1000, 1, 24),
    "swint_fc1": (96, 384, 3, 3),
    "swint_merge1": (384, 192, 1, 3),
}


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
@pytest.mark.parametrize("name", ["vitb_qkv", "vitb_fc1"])
def test_vit_b_folded_bitwise(name, config, bit):
    K, O, n_V, n_H = LAYERS[name]
    if config == "BasePTQ":
        n_V = n_H = 1
    _check_fold(_norm(K), _frozen(K, O, n_V, n_H, bit=bit), _x(VIT_ROWS, K))


@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
def test_vit_b_head_cls_rows(config):
    K, O, n_V, n_H = LAYERS["vitb_head"]
    if config == "BasePTQ":
        n_V = n_H = 1
    ln, head = _norm(K), _frozen(K, O, n_V, n_H, seed=2)
    x = _x(VIT_ROWS, K).view(32, 197, K)
    from ptq4vit_b200.quant_layers.linear import frozen_norm_applies, frozen_norm_linear
    with torch.no_grad():
        want = head(ln(x)[:, 0])
        assert frozen_norm_applies(ln, head, x)
        got = frozen_norm_linear(ln, head, x[:, 0])
    assert torch.equal(_bits(got), _bits(want))


def test_n_a_and_ieee_division(monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    _check_fold(_norm(768, eps=1e-5), _frozen(768, 2304, 24, 24, n_a=4, seed=4), _x(1000, 768, seed=9))


@pytest.mark.parametrize("name", ["swint_fc1", "swint_merge1"])
def test_swin_shapes(name):
    K, O, n_V, n_H = LAYERS[name]
    rows = 32 * 3136 if name == "swint_fc1" else 32 * 784
    lin = _frozen(K, O, n_V, n_H, bias=name != "swint_merge1", seed=6)
    _check_fold(_norm(K, eps=1e-5), lin, _x(rows, K, seed=11))


@pytest.mark.parametrize("rows", [1, 5, 197, 5 * 197, 32 * 197 - 3])
def test_row_tails_and_batches(rows):
    K, O, n_V, n_H = LAYERS["vitb_qkv"]
    _check_fold(_norm(K), _frozen(K, O, n_V, n_H, seed=8), _x(rows, K, seed=rows))


@pytest.mark.parametrize("rows", [5, VIT_ROWS])
@pytest.mark.parametrize("config", ["PTQ4ViT", "BasePTQ"])
def test_composed_with_fused_mlp(config, rows):
    from ptq4vit_b200.quant_layers.linear import frozen_mlp, frozen_mlp_applies, frozen_mlp_norm_ok, frozen_norm_applies
    n = 24 if config == "PTQ4ViT" else 1
    fc1 = _frozen(768, 3072, n, n, seed=1)
    fc2 = _layer(3072, 768, 1, n, gelu=config == "PTQ4ViT", seed=2)
    fc2.freeze()
    fc2.mode = "quant_forward"
    ln, x = _norm(768), _x(rows, 768, seed=12)
    with torch.no_grad():
        assert frozen_norm_applies(ln, fc1, x) and frozen_mlp_applies(fc1, fc2, torch.nn.GELU(), x)
        assert frozen_mlp_norm_ok(fc1, fc2)
        want = fc2(F.gelu(fc1(ln(x))))
        got = frozen_mlp(fc1, fc2, x, norm=ln)
        torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want))


def test_one_launch_no_copy_no_allocation_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import frozen_norm_linear
    K, O, n_V, n_H = LAYERS["vitb_qkv"]
    ln, lin = _norm(K), _frozen(K, O, n_V, n_H, seed=10)
    x, x2 = _x(8 * 197, K, seed=1), _x(8 * 197, K, seed=2)
    with torch.no_grad():
        want, want2 = lin(ln(x)), lin(ln(x2))
        frozen_norm_linear(ln, lin, x)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        y = frozen_norm_linear(ln, lin, x)
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
        assert _lib.launch_count() - n0 == 1
        assert torch.equal(_bits(y), _bits(want))
        # a host <-> device copy or synchronisation inside the call would fail the stream capture below
        xs = x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_norm_linear(ln, lin, xs)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ys = frozen_norm_linear(ln, lin, xs)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys), _bits(want))
        xs.copy_(x2)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys), _bits(want2))


def test_stale_steps_grad_mode_and_rejected_shapes():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import frozen_norm_applies, frozen_norm_linear
    from ptq4vit_b200.utils.models import Attention
    K, O, n_V, n_H = LAYERS["vitb_qkv"]
    ln, lin = _norm(K), _frozen(K, O, n_V, n_H, seed=13)
    x = _x(197, K)
    with torch.no_grad():
        frozen_norm_linear(ln, lin, x)
        lin.a_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_norm_linear(ln, lin, x)
        lin.unfreeze(); lin.freeze()
    attn = Attention(K, 12).cuda()
    attn.qkv = lin
    xb = x.view(1, 197, K)
    with torch.no_grad():
        want = attn(ln(xb))
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        got = attn(xb, norm=ln)
        torch.cuda.synchronize()
        assert _lib.launch_count() - n0 == 1, "no grad: the folded qkv is the one native launch"
        assert torch.equal(_bits(got), _bits(want))
    assert not frozen_norm_applies(ln, lin, xb), "grad mode with LayerNorm parameters that require grad"
    n0 = _lib.launch_count()
    y = attn(xb, norm=ln)
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))
    # rejected shapes run unfolded: an odd width, and a misaligned x
    with torch.no_grad():
        x_off = torch.empty(197 * K + 1, device="cuda")[1:].view(197, K)
        x_off.copy_(x)
        assert not frozen_norm_applies(ln, lin, x_off)
        assert torch.equal(_bits(attn(x_off.view(1, 197, K), norm=ln)), _bits(attn(ln(x_off.view(1, 197, K)))))
        ln_plain = torch.nn.LayerNorm(K, elementwise_affine=False).cuda()
        assert not frozen_norm_applies(ln_plain, lin, x)


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
    with RH.fp32_convolutions():
        net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images, images2 = RH.tiny_images(n=5, seed=11).cuda(), RH.tiny_images(n=5, seed=12).cuda()
        norms = [n for n, m in net.named_modules() if isinstance(m, torch.nn.LayerNorm)]
        with torch.no_grad():
            deploy.freeze_model(wrapped, matmul=True, conv=True)
            assert deploy.fuse_attention(net) == [] and deploy.fuse_mlp(net) == []
            ln_calls = []
            hooks = [m.register_forward_hook(lambda *_: ln_calls.append(1)) for m in net.modules()
                     if isinstance(m, torch.nn.LayerNorm)]
            want, n_unfolded = _launches(net, images)
            calls_unfolded = len(ln_calls)
            want2 = net(images2)
            left = deploy.fuse_norm(net)
            assert len(left) < len(norms)
            ln_calls.clear()
            got, n_folded = _launches(net, images)
            assert n_folded == n_unfolded, "the LayerNorms were torch launches; the folded Linears launch as before"
            assert len(ln_calls) < calls_unfolded, "a folded call skips its LayerNorm module (and its hooks)"
            for h in hooks:
                h.remove()
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
            assert torch.equal(_bits(ys), _bits(want2)), "graph replay of the folded model on new images"
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            deploy.load_quantized(wrapped2, path, matmul=True, conv=True)
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert deploy.fuse_attention(fresh) == [] and deploy.fuse_mlp(fresh) == []
            assert deploy.fuse_norm(fresh) == left
            assert torch.equal(_bits(fresh(images)), _bits(want))
            deploy.unfuse_norm(net)
            assert torch.equal(_bits(net(images)), _bits(want))
