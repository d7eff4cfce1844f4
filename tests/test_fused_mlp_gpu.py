"""The fused frozen MLP on the GPU.  Every comparison is of int32 bit patterns against the unfused frozen sequence
fc2(F.gelu(fc1(x))): the GELU of the epilogue against torch's over every fp32 bit pattern; fc2's activation image the
fused fc1 writes against the one p4v_quant_image builds from torch's GELU output, byte for byte and padding included;
ViT-B/224, Swin-T stage 1 and Swin-B/384 shapes under PTQ4ViT, BasePTQ and no_postgelu at W8A8 / W6A6; fc2 segments that
straddle fc1's column tiles; row tails and small batches (column tiles split over CTAs); a garbage workspace; two
launches, no copy, no allocation but the output, CUDA-graph replay; stale step sizes raise and grad mode runs unfused;
whole tiny ViT and Swin models fused give the unfused logits eagerly, from one CUDA graph and after a save / load."""
import copy
import ctypes
import importlib
import os

import pytest
import torch
import torch.nn.functional as F

from tests.test_frozen_forward_gpu import _layer
from tests.test_frozen_matmul_gpu import TINY_SWIN, _bits

pytestmark = pytest.mark.gpu

VIT_ROWS = 32 * 197

# name: (dim, hidden, n_V1, n_H1, n_H2, post-GELU fc2)
SHAPES = {
    "vitb_ptq4vit": (768, 3072, 24, 24, 24, True),
    "vitb_baseptq": (768, 3072, 1, 1, 1, False),
    "vitb_no_postgelu": (768, 3072, 24, 24, 24, False),
    "swint_stage1": (96, 384, 3, 3, 12, True),            # fc2 (K = 384) runs the fused kernel on its own
    "swinb384_stage4": (1024, 4096, 32, 32, 32, True),
    "straddle_400": (200, 400, 1, 4, 4, True),            # fc2 segments of 100 columns: chunks across fc1's column tiles
    "straddle_2000": (200, 2000, 1, 4, 8, True),          # 250-column segments, fc2 on the streamed path
}


def _mlp(name, bit=8, seed=0):
    K, H, n_V1, n_H1, n_H2, gelu2 = SHAPES[name]
    fc1 = _layer(K, H, n_V1, n_H1, bit=bit, seed=seed)
    fc2 = _layer(H, K, 1, n_H2, gelu=gelu2, bit=bit, seed=seed + 1)
    for m in (fc1, fc2):
        m.freeze()
        m.mode = "quant_forward"
    return fc1, fc2


def _x(rows, K, seed=3):
    return torch.randn(rows, K, generator=torch.Generator().manual_seed(seed)).cuda()


def _check(fc1, fc2, x):
    """Unfused sequence, then the fused call on a workspace filled with 0xFF: the outputs bitwise, and, where fc2 streams
    (its frozen workspace then holds the image p4v_quant_image built from torch's GELU), every byte of the image."""
    from ptq4vit_b200.quant_layers.linear import frozen_mlp, frozen_mlp_applies
    with torch.no_grad():
        assert frozen_mlp_applies(fc1, fc2, torch.nn.GELU(), x)
        want = fc2(F.gelu(fc1(x)))
        ref_img = None if fc2._frozen_fused else fc2._frozen_ws.clone()
        frozen_mlp(fc1, fc2, x)
        fc2._frozen_ws.fill_(0xFF)
        got = frozen_mlp(fc1, fc2, x)
        torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want))
    if ref_img is not None:
        img = fc2._frozen_ws[:ref_img.numel()]
        bad = (img != ref_img).nonzero()
        assert bad.numel() == 0, f"{bad.shape[0]} image bytes differ, first at {bad[:4].flatten().tolist()}"
    return got


def test_gelu_probe_every_fp32_bit_pattern():
    from ptq4vit_b200 import _lib
    n = 1 << 28
    got = torch.empty(n, dtype=torch.float32, device="cuda")
    for c in range(16):
        bits = torch.arange(-(1 << 31) + c * n, -(1 << 31) + (c + 1) * n, dtype=torch.int32, device="cuda")
        x = bits.view(torch.float32)
        want = F.gelu(x)
        _lib.check(_lib.lib().p4v_gelu_probe(_lib.ptr(x), _lib.ptr(got), n,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "p4v_gelu_probe")
        same = (got.view(torch.int32) == want.view(torch.int32)) | (got.isnan() & want.isnan())
        bad = (~same).nonzero()
        assert bad.numel() == 0, f"{bad.shape[0]} mismatches in chunk {c}, first x bits {bits[bad[:4, 0]].tolist()}"


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("name", ["vitb_ptq4vit", "vitb_baseptq", "vitb_no_postgelu"])
def test_vit_b_bitwise_and_image(name, bit):
    fc1, fc2 = _mlp(name, bit)
    assert not fc2._frozen_fused, "ViT-B's fc2 streams: its image is compared byte for byte"
    _check(fc1, fc2, _x(VIT_ROWS, 768))


@pytest.mark.parametrize("name", ["swint_stage1", "swinb384_stage4", "straddle_400", "straddle_2000"])
def test_other_shapes_bitwise(name):
    fc1, fc2 = _mlp(name)
    _check(fc1, fc2, _x(6304 if name != "swinb384_stage4" else 32 * 144, SHAPES[name][0]))


@pytest.mark.parametrize("rows", [1, 5, 6304])
@pytest.mark.parametrize("name", ["vitb_ptq4vit", "straddle_2000", "swint_stage1"])
def test_row_tails_and_small_batches(name, rows):
    # 1 and 5 rows: one row tile, its column tiles split over CTAs (straddling chunks owned by two CTAs)
    fc1, fc2 = _mlp(name, seed=7)
    _check(fc1, fc2, _x(rows, SHAPES[name][0], seed=rows))


def _copies(fn):
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        y = fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "memcpy" in e.name.lower()], y


def test_two_launches_no_copy_no_allocation_and_graph():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import frozen_mlp
    fc1, fc2 = _mlp("vitb_ptq4vit", seed=11)
    x, x2 = _x(8 * 197, 768, seed=1), _x(8 * 197, 768, seed=2)
    with torch.no_grad():
        want, want2 = fc2(F.gelu(fc1(x))), fc2(F.gelu(fc1(x2)))
        frozen_mlp(fc1, fc2, x)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        allocs0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        copies, y = _copies(lambda: frozen_mlp(fc1, fc2, x))
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - allocs0 == 1, "only the output may be allocated"
        assert _lib.launch_count() - n0 == 2
        assert not copies, f"the fused call issued a copy: {copies}"
        assert torch.equal(_bits(y), _bits(want))
        xs = x.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            frozen_mlp(fc1, fc2, xs)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ys = frozen_mlp(fc1, fc2, xs)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys), _bits(want))
        xs.copy_(x2)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys), _bits(want2))


def test_stale_step_sizes_raise():
    from ptq4vit_b200.quant_layers.linear import frozen_mlp
    fc1, fc2 = _mlp("swint_stage1", seed=12)
    x = _x(64, 96)
    with torch.no_grad():
        frozen_mlp(fc1, fc2, x)
        fc1.a_interval.mul_(1.01)
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_mlp(fc1, fc2, x)
        fc1.unfreeze(); fc1.freeze()
        frozen_mlp(fc1, fc2, x)
        fc2.w_interval = fc2.w_interval * 1.0
        with pytest.raises(RuntimeError, match="step sizes changed"):
            frozen_mlp(fc1, fc2, x)


def test_grad_mode_runs_unfused():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Mlp
    blk = Mlp(768, 3072).cuda()
    blk.fc1, blk.fc2 = _mlp("vitb_ptq4vit", seed=13)
    assert deploy.fuse_mlp(blk) == [] and blk.fused
    x = _x(2 * 197, 768).view(2, 197, 768)
    with torch.no_grad():
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        want = blk(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() - n0 == 2
        deploy.unfuse_mlp(blk)
        assert torch.equal(_bits(blk(x)), _bits(want)), "fused and unfused block"
        deploy.fuse_mlp(blk)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    y = blk(x)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 3, "grad mode: fc1's fused kernel, fc2's image and sweep"
    assert y.grad_fn is not None and torch.equal(_bits(y.detach()), _bits(want))


def _launches(net, images):
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
    from ptq4vit_b200.utils.models import Mlp, SwinTransformer, VisionTransformer
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
        mlps = [n for n, m in net.named_modules() if isinstance(m, Mlp)]
        with torch.no_grad():
            assert deploy.fuse_mlp(net) == mlps, "nothing frozen yet: every Mlp is left unfused"
            deploy.unfuse_mlp(net)
            deploy.freeze_model(wrapped, matmul=True)
            assert deploy.fuse_attention(net) == []
            want, n_unfused = _launches(net, images)
            want2 = net(images2)
            assert deploy.fuse_mlp(net) == []
            got, n_fused = _launches(net, images)
            assert n_fused <= n_unfused      # the tiny models' fc2 (K = 256 / 128) runs the fused Linear kernel on its own
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
            assert deploy.fuse_attention(fresh) == [] and deploy.fuse_mlp(fresh) == []
            got2, n_fused2 = _launches(fresh, images)
            assert n_fused2 == n_fused and torch.equal(_bits(got2), _bits(want))
            deploy.unfuse_mlp(net)
            assert torch.equal(_bits(net(images)), _bits(want))
