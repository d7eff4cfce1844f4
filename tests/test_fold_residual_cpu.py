"""A block's residual add folded into the frozen Linear that produces it, without a GPU: the window layout's arithmetic
against Swin's own partition / reverse / roll, the paths of the fold sites, every rejection of the new entry points
before any launch, the Python rule's early refusals, fuse_residual / unfuse_residual bookkeeping, and a model that was
never folded runs the code it ran before."""
import ctypes

import pytest
import torch


def _window_row(r, images, H, W, ws, shift):
    """The layout of include/ptq4vit_b200.h (p4v_window_row), restated on an index tensor."""
    nH, nW = H // ws, W // ws
    ij, w = r % (ws * ws), r // (ws * ws)
    ww, wh, b = w % nW, (w // nW) % nH, w // (nW * nH)
    i, j = ij // ws, ij % ws
    return b * H * W + ((wh * ws + i + shift) % H) * W + (ww * ws + j + shift) % W


# (res, ws) of each stage: Swin-T/224 (window 7) and Swin-B/384 (window 12)
@pytest.mark.parametrize("res,ws,shift", [(56, 7, 0), (56, 7, 3), (28, 7, 0), (28, 7, 3), (14, 7, 0), (14, 7, 3), (7, 7, 0),
                                          (7, 7, 3), (96, 12, 0), (96, 12, 6), (48, 12, 0), (48, 12, 6), (24, 12, 0),
                                          (24, 12, 6), (12, 12, 0), (12, 12, 6)])
def test_layout_matches_partition_reverse_roll(res, ws, shift):
    from ptq4vit_b200.utils.models import _window_partition, _window_reverse
    B = 2
    rows = B * res * res
    # window row r holds the value computed there; the block sends it through reverse and roll(+shift) to its image row
    win = torch.arange(rows, dtype=torch.int64).view(-1, ws * ws, 1)
    img = _window_reverse(win, ws, res, res)
    if shift:
        img = torch.roll(img, shifts=(shift, shift), dims=(1, 2))
    dst = torch.empty(rows, dtype=torch.int64)
    dst[img.reshape(-1)] = torch.arange(rows)
    got = _window_row(torch.arange(rows), B, res, res, ws, shift)
    assert torch.equal(got, dst)
    # and it is the inverse of the qkv side's gather: partition of the image rolled by -shift
    x = torch.arange(rows, dtype=torch.int64).view(B, res, res, 1)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    assert torch.equal(_window_partition(x, ws).reshape(-1), got)


def _desc(K, O, n_H=1, post_gelu=0, rows=6304, bit=8):
    from ptq4vit_b200 import _lib
    d = _lib.LinearDesc()
    d.rows, d.tokens, d.in_features, d.out_features = rows, 1, K, O
    d.n_V, d.n_H, d.n_a, d.w_bit, d.a_bit = 1, n_H, 1, bit, bit
    d.eq_n, d.search_round, d.post_gelu, d.has_bias = 1, 1, post_gelu, 1
    return d


def _frozen_path(d):
    from ptq4vit_b200 import _lib
    path = ctypes.c_int()
    _lib.check(_lib.lib().p4v_linear_frozen_path(ctypes.byref(d), ctypes.byref(path)), "frozen_path")
    return path.value


@pytest.mark.parametrize("C", [96, 192, 384, 768, 128, 256, 512, 1024])
def test_every_swin_proj_is_on_the_fused_path(C):
    """Swin-T / S (96 .. 768) and Swin-B (128 .. 1024) attention projections take a window layout."""
    for bit in (8, 6):
        assert _frozen_path(_desc(C, C, n_H=max(1, C // 32), bit=bit)) == 1


def test_vit_b_fc2_streams():
    assert _frozen_path(_desc(3072, 768, 24, post_gelu=1)) == 0 and _frozen_path(_desc(3072, 768, 1)) == 0
    assert _frozen_path(_desc(768, 768, 24)) == 1


def _v(a):
    return a and ctypes.c_void_p(a)


def _layout(images, H, W, ws, shift):
    from ptq4vit_b200 import _lib
    return _lib.WindowLayout(images, H, W, ws, shift)


def _call_linear(d, x=4096, bias=16384, packed=1 << 20, ws=3 << 20, ws_bytes=1 << 30, res=8 << 20, layout=None, out=16 << 20):
    """p4v_linear_frozen_forward_res on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_linear_frozen_forward_res(ctypes.byref(d), _v(x), _v(bias), _v(packed), _v(ws), ws_bytes, _v(res),
                                           None if layout is None else ctypes.byref(layout), _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


SWIN_ROWS = 2 * 56 * 56


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(packed=0), "null pointer"), (dict(out=0), "null pointer"), (dict(res=0), "null pointer"),
    (dict(bias=0), "bias is null"), (dict(x=4100), "aligned"), (dict(out=(16 << 20) + 4), "aligned"),
    (dict(res=(8 << 20) + 4), "residual must be 8-byte aligned"),
    (dict(res=(16 << 20) + 1024), "overlaps"), (dict(res=(16 << 20) - 1024), "overlaps"),
    (dict(layout=(2, 56, 56, 7, 7)), "shift"), (dict(layout=(2, 56, 56, 7, -1)), "shift"),
    (dict(layout=(2, 56, 56, 0, 0)), "positive"), (dict(layout=(0, 56, 56, 7, 0)), "positive"),
    (dict(layout=(2, 56, 60, 7, 3)), "multiples of the window"), (dict(layout=(2, 54, 56, 7, 3)), "multiples of the window"),
    (dict(layout=(3, 56, 56, 7, 3)), "rows"), (dict(layout=(1, 56, 56, 7, 3)), "rows"),
])
def test_linear_validation_before_launch(case, match):
    case = dict(case)
    if "layout" in case:
        case["layout"] = _layout(*case["layout"])
    rc, msg = _call_linear(_desc(96, 96, 3, rows=SWIN_ROWS), **case)
    assert rc != 0 and match in msg, msg


def test_streamed_path_rejects_a_layout():
    d = _desc(3072, 768, 24, rows=2 * 3136)
    assert _frozen_path(d) == 0
    rc, msg = _call_linear(d, layout=_layout(2, 56, 56, 7, 0))
    assert rc != 0 and "needs the fused path" in msg, msg
    rc, msg = _call_linear(d, res=(16 << 20) + 8)
    assert rc != 0 and "overlaps" in msg, msg
    rc, msg = _call_linear(d, ws_bytes=1 << 10)
    assert rc != 0 and "workspace too small" in msg, msg


def _pack_bytes(d):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_pack_bytes(ctypes.byref(d), ctypes.byref(n)), "pack_bytes")
    return n.value


def _call_mlp(norm, x=4096, g=8192, b=12288, b1=16384, p1=1 << 20, b2=20480, p2=2 << 20, ws=3 << 20, res=64 << 20,
              out=128 << 20, ws_bytes=1 << 30):
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    d1, d2 = _desc(768, 3072, 24), _desc(3072, 768, 24, post_gelu=1)
    n0 = _lib.launch_count()
    if norm:
        rc = lib.p4v_mlp_frozen_forward_norm_res(ctypes.byref(d1), _v(x), _v(g), _v(b), ctypes.c_float(1e-6), _v(b1), _v(p1),
                                                 _pack_bytes(d1), ctypes.byref(d2), _v(b2), _v(p2), _pack_bytes(d2), _v(ws),
                                                 ws_bytes, _v(res), _v(out), None)
    else:
        rc = lib.p4v_mlp_frozen_forward_res(ctypes.byref(d1), _v(x), _v(b1), _v(p1), _pack_bytes(d1), ctypes.byref(d2), _v(b2),
                                            _v(p2), _pack_bytes(d2), _v(ws), ws_bytes, _v(res), _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(res=0), "null pointer"), (dict(ws=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(b2=0), "bias is null"), (dict(res=(64 << 20) + 4), "residual must be 8-byte aligned"),
    (dict(res=(128 << 20) + 64), "overlaps"), (dict(ws_bytes=1 << 20), "workspace too small"),
])
def test_mlp_validation_before_launch(norm, case, match):
    rc, msg = _call_mlp(norm, **case)
    assert rc != 0 and match in msg, msg


def test_new_symbols_exported():
    from ptq4vit_b200 import _lib
    for name in ("p4v_linear_frozen_forward_res", "p4v_mlp_frozen_forward_res", "p4v_mlp_frozen_forward_norm_res"):
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)


def test_python_rule_refuses_without_frozen_linear():
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear, frozen_residual_applies
    assert not frozen_residual_applies(torch.nn.Linear(64, 32), torch.zeros(3, 64), torch.zeros(3, 32))
    assert not frozen_residual_applies(MinMaxQuantLinear(64, 32), torch.zeros(3, 64), torch.zeros(3, 32)), "not frozen"


def _fake_frozen(lin_cls, K, O):
    q = lin_cls(K, O)
    q._packed = torch.zeros(1, dtype=torch.uint8)          # frozen is faked: the flag is all fuse_residual looks at
    return q


def test_fuse_residual_bookkeeping():
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Block, SwinBlock, get_net
    vit = get_net("vit_tiny_patch16_224", device="cpu", depth=2)
    blocks = [n for n, m in vit.named_modules() if isinstance(m, Block)]
    assert blocks == ["blocks.0", "blocks.1"]
    assert deploy.fuse_residual(vit) == blocks, "no frozen Linear: every block is left unfolded"
    assert not any(getattr(m, "fold_residual", False) for m in vit.modules())
    blk = vit.blocks[1]
    blk.attn.proj = _fake_frozen(MinMaxQuantLinear, 192, 192)
    assert deploy.fuse_residual(vit) == blocks, "fc2 is not frozen"
    blk.mlp.fc2 = _fake_frozen(MinMaxQuantLinear, 768, 192)
    assert deploy.fuse_residual(vit) == ["blocks.0"]
    assert blk.fold_residual and not vit.blocks[0].fold_residual
    deploy.unfuse_residual(vit)
    assert not blk.fold_residual
    swin = get_net("swin_tiny_patch4_window7_224", device="cpu", depths=(2, 2), num_heads=(3, 6))
    sblocks = [n for n, m in swin.named_modules() if isinstance(m, SwinBlock)]
    assert len(sblocks) == 4 and deploy.fuse_residual(swin) == sblocks
    sb = swin.layers[0].blocks[1]
    sb.attn.proj, sb.mlp.fc2 = _fake_frozen(MinMaxQuantLinear, 96, 96), _fake_frozen(MinMaxQuantLinear, 384, 96)
    assert deploy.fuse_residual(swin) == [n for n in sblocks if n != "layers.0.blocks.1"]
    assert sb.fold_residual
    deploy.unfuse_residual(swin)
    assert not any(getattr(m, "fold_residual", False) for m in swin.modules())


def test_default_and_unfoldable_forwards_unchanged():
    """With the flag off the blocks run as before; with it on and nothing frozen, every add runs unfused with the same bits."""
    from ptq4vit_b200.utils.models import Block, SwinBlock
    assert not Block.fold_residual and not SwinBlock.fold_residual
    torch.manual_seed(0)
    blk = Block(64, 2).eval()
    x = torch.randn(2, 5, 64)
    with torch.no_grad():
        want = x + blk.attn(blk.norm1(x))
        want = want + blk.mlp(blk.norm2(want))
        assert torch.equal(blk(x), want)
        blk.fold_residual = True
        assert torch.equal(blk(x).view(torch.int32), want.view(torch.int32))
    for shift in (0, 2):
        sb = SwinBlock(32, 8, 2, 4, shift).eval()
        xs = torch.randn(2, 64, 32)
        with torch.no_grad():
            want = sb(xs)
            sb.fold_residual = True
            assert torch.equal(sb(xs).view(torch.int32), want.view(torch.int32))
