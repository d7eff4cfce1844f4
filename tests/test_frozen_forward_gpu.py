"""The frozen Linear forward on the GPU: bit-identical to the unfrozen quant_forward on both of its paths (fused kernel /
streamed int8 image), within the fp32 bound of an independent fp64 restatement, one launch and no copy per call, capturable
in a CUDA graph, and a whole model frozen, saved and loaded back without its FP32 weights."""
import copy
import importlib
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOK = 197


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


def _x(rows, K, gelu, seed=1):
    x = torch.randn(rows, K, generator=torch.Generator().manual_seed(seed))
    return (F.gelu(x) if gelu else x).cuda()


def _fp64(m, x):
    """fq(x) fq(W)^T + b with the reference's quantisers (fp32 divisions on the device, as quant_weight_bias /
    quant_input run them) and every q * step and the sum in fp64; also sum |terms| for the error bound."""
    O, K = m.weight.shape
    wi = m.w_interval.reshape(m.n_V, 1, m.n_H, 1)
    wq = (m.weight.data.view(m.n_V, O // m.n_V, m.n_H, K // m.n_H) / wi).round().clamp(-m.w_qmax, m.w_qmax - 1)
    w64 = (wq.double() * wi.double()).view(O, K)
    ai = m.a_interval.reshape(m.n_a, 1)
    xv = x.view(-1, m.n_a, K // m.n_a)
    if m.post_gelu:
        neg = 0.16997124254703522 / m.a_qmax
        x64 = (xv / ai).round().clamp(0, m.a_qmax - 1).double() * ai.double() + \
              (xv / neg).round().clamp(-m.a_qmax, 0).double() * float(torch.tensor(neg, dtype=torch.float32))
    else:
        x64 = (xv / ai).round().clamp(-m.a_qmax, m.a_qmax - 1).double() * ai.double()
    x64 = x64.view(-1, K)
    b = torch.zeros(O, dtype=torch.float64, device=x.device) if m.bias is None else m.bias.data.double()
    return x64 @ w64.t() + b, x64.abs() @ w64.abs().t() + b.abs()


CASES = {
    # name: (K, O, n_V, n_H, n_a, gelu, bias, fused)
    "vitb_qkv": (768, 2304, 72, 24, 1, False, True, True),
    "vitb_proj": (768, 768, 24, 24, 1, False, True, True),
    "vitb_fc1": (768, 3072, 24, 24, 1, False, True, True),
    "vitb_fc2": (3072, 768, 24, 24, 1, True, True, False),
    "vitb_head": (768, 1000, 1, 24, 1, False, True, True),
    "n_a3": (768, 768, 24, 24, 3, False, True, True),
    "nobias": (768, 2304, 72, 24, 1, False, False, True),
    "baseptq_qkv": (768, 2304, 3, 1, 1, False, True, True),
    "baseptq_fc2": (3072, 768, 1, 1, 1, True, True, False),
    "swint_fc2": (384, 96, 1, 12, 1, True, True, True),          # post-GELU on the fused path: two planes in shared memory
    "swint_qkv": (96, 288, 3, 3, 1, False, True, True),
    "swinb384_proj": (1024, 1024, 32, 32, 1, False, True, True),
    "odd_segments": (120, 200, 1, 3, 1, False, True, True),      # 40-element segments padded to 64 B, column tail
    "below_boundary": (1440, 256, 1, 1, 1, False, True, True),
    "above_boundary": (1472, 256, 1, 1, 1, False, True, False),
}


def _check(name, bit, rows_list=(32 * TOK,), fp64=True):
    K, O, n_V, n_H, n_a, gelu, bias, fused = CASES[name]
    m = _layer(K, O, n_V, n_H, n_a, gelu, bias, bit)
    xs = [_x(r, K, gelu, seed=r) for r in rows_list]
    want = [m.quant_forward(x) for x in xs]
    m.freeze()
    assert m.frozen and m._frozen_fused == fused
    packed = m._packed
    for x, y0 in zip(xs, want):
        y1 = m.quant_forward(x)
        assert y1.shape == y0.shape and torch.equal(y1, y0), f"{name} W{bit} rows {x.shape[0]}: frozen != unfrozen"
        assert m._packed is packed                       # one packed tensor serves every batch size
        if fp64:
            ref, mag = _fp64(m, x)
            groups = (K // min(K // n_H, K // n_a)) * (2 if gelu else 1)
            bound = (groups + 2) * 2.0 ** -23 * mag
            assert bool(((y1.double() - ref).abs() <= bound).all()), \
                f"{name}: worst ratio {float(((y1.double() - ref).abs() / bound).max()):.2f} of the fp32 bound"
    m.unfreeze()
    assert not m.frozen and torch.equal(m.quant_forward(xs[0]), want[0])


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("name", ["vitb_qkv", "vitb_proj", "vitb_fc1", "vitb_fc2", "vitb_head"])
def test_vit_b_layers_bitwise(name, bit):
    _check(name, bit)


@pytest.mark.parametrize("name", ["n_a3", "nobias", "baseptq_qkv", "baseptq_fc2", "swint_fc2", "swint_qkv", "swinb384_proj",
                                  "odd_segments", "below_boundary", "above_boundary"])
def test_other_shapes_bitwise(name):
    _check(name, 8, rows_list=(3136,) if name.startswith("swin") else (8 * TOK,))


@pytest.mark.parametrize("name", ["vitb_qkv", "vitb_fc2", "swint_fc2"])
def test_row_tails_share_one_packed_tensor(name):
    _check(name, 8, rows_list=(TOK, 3 * TOK, 32 * TOK, 1))


@pytest.mark.parametrize("name", ["vitb_fc2", "swint_fc2", "vitb_proj"])
def test_ieee_scalar_division(name, monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")
    _check(name, 8, rows_list=(4 * TOK,), fp64=False)    # the fp64 restatement divides as torch does on the device


def test_packed_integers_are_the_exported_int8_weight():
    from ptq4vit_b200.utils.integer import quantize_int_weight
    K, O = 768, 2304
    m = _layer(*CASES["vitb_qkv"][:7])
    m.freeze()
    tiles = O // 128                                     # 32-element segments: no padding, K bytes per row
    img = m._packed[:tiles * 128 * K].view(tiles, K // 16, 128, 16).permute(0, 2, 1, 3).reshape(O, K)
    assert torch.equal(img.view(torch.int8), quantize_int_weight(m))


def _copies(m, x):
    """Names of the copy activities one quant_forward issues (torch.profiler), and its output."""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        y = m.quant_forward(x)
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "memcpy" in e.name.lower()], y


def test_one_launch_no_copy_and_graph_replay():
    from ptq4vit_b200 import _lib
    for name, launches in (("vitb_proj", 1), ("vitb_fc2", 2)):
        K, O, n_V, n_H, n_a, gelu, bias, fused = CASES[name]
        m = _layer(K, O, n_V, n_H, n_a, gelu, bias)
        xa, xb = _x(3 * TOK, K, gelu, seed=5), _x(3 * TOK, K, gelu, seed=6)
        want_a, want_b = m.quant_forward(xa), m.quant_forward(xb)
        assert _copies(m, xa)[0], "the profiler must see the table uploads of the unfrozen forward"
        m.freeze()
        m.quant_forward(xa)                               # the streamed path's workspace exists from here on
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        copies, y = _copies(m, xa)
        assert _lib.launch_count() - n0 == launches
        assert torch.equal(y, want_a)
        assert not copies, f"the frozen forward issued a copy: {copies}"
        # capture once, replay on new input
        xs = xa.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m.quant_forward(xs)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ys = m.quant_forward(xs)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ys, want_a)
        xs.copy_(xb)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ys, want_b), f"{name}: graph replay on new input"


def test_frozen_model_save_load_without_fp32_weights(tmp_path):
    from oracle import ref_harness as RH
    from ptq4vit_b200.configs import PTQ4ViT as cfg
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import VisionTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    os.environ.setdefault("TQDM_DISABLE", "1")
    importlib.reload(cfg)
    with RH.fp32_convolutions():
        net = VisionTransformer(**RH.TINY_VIT).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        fresh = copy.deepcopy(net)
        wrapped = wrap_modules_in_net(net, cfg)
        Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4).batching_quant_calib()
        images = RH.tiny_images(n=5, seed=11).cuda()
        with torch.no_grad():
            want = net(images)
            left = deploy.freeze_model(wrapped)
            linear = [n for n, m in wrapped.items() if isinstance(m, MinMaxQuantLinear)]
            assert linear and all(wrapped[n].frozen for n in linear)
            assert sorted(left) == sorted(set(wrapped) - set(linear)) and any("matmul" in n for n in left)
            assert torch.equal(net(images), want)
            path = str(tmp_path / "model_q.pt")
            deploy.save_quantized(wrapped, path)
            # a freshly wrapped copy, its FP32 Linear weights gone: the integers in the file are all it has
            wrapped2 = wrap_modules_in_net(fresh, cfg)
            deploy.load_quantized(wrapped2, path)
            for n in linear:
                wrapped2[n].weight.data.zero_()
            for m in wrapped2.values():
                m.mode = "quant_forward"
            assert torch.equal(fresh(images), want)
            # stale step sizes are refused
            m = wrapped[linear[0]]
            m.w_interval = m.w_interval * 1.01
            with pytest.raises(RuntimeError, match="step sizes changed"):
                net(images)
            m.unfreeze(); m.freeze()
            deploy.unfreeze_model(wrapped)
            assert not any(wrapped[n].frozen for n in linear)
