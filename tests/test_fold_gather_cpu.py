"""Swin's row gathers folded into the frozen Linear that consumes them, without a GPU: the window and merge maps restated
on index tensors against Swin's own roll / partition and PatchMerging's cat, the shape rule over every Swin qkv and
reduction, every rejection of the new entry point before any launch, the Python rule's early refusals, fuse_gather /
unfuse_gather bookkeeping, and a model that was never folded runs the code it ran before."""
import ctypes

import pytest
import torch


def _window_src(r, images, H, W, ws, shift):
    """The window gather (p4v_window_row): the image row output row r reads."""
    nH, nW = H // ws, W // ws
    ij, w = r % (ws * ws), r // (ws * ws)
    ww, wh, b = w % nW, (w // nW) % nH, w // (nW * nH)
    i, j = ij // ws, ij % ws
    return b * H * W + ((wh * ws + i + shift) % H) * W + (ww * ws + j + shift) % W


def _merge_src(m, q, H, W):
    """The merge gather (p4v_merge_row + p4v_merge_quarter): the image row quarter q of merged row m reads."""
    j, i, b = m % (W // 2), (m // (W // 2)) % (H // 2), m // ((W // 2) * (H // 2))
    return b * H * W + (2 * i + (q & 1)) * W + 2 * j + (q >> 1)


def _stages():
    """(name, stage, C, res, window) of every stage of every Swin model"""
    from ptq4vit_b200.utils.models import _SWIN_ZOO
    out = []
    for name, cfg in _SWIN_ZOO.items():
        res = cfg["img_size"] // 4
        for s in range(len(cfg["depths"])):
            r = res // 2 ** s
            out.append((name, s, cfg["dim"] * 2 ** s, r, min(cfg["window_size"], r)))
    return out


STAGES = _stages()


@pytest.mark.parametrize("name,stage,C,res,ws", STAGES)
def test_window_map_matches_roll_and_partition(name, stage, C, res, ws):
    from ptq4vit_b200.utils.models import _window_partition
    B = 2
    rows = B * res * res
    for shift in sorted({0, ws // 2 if ws < res else 0}):
        img = torch.arange(rows, dtype=torch.int64).view(B, res, res, 1)
        if shift:
            img = torch.roll(img, shifts=(-shift, -shift), dims=(1, 2))
        want = _window_partition(img, ws).reshape(-1)
        assert torch.equal(_window_src(torch.arange(rows), B, res, res, ws, shift), want)
    # the shifted map also at a stage whose blocks never shift (window == resolution): the kernel takes any shift < window
    if ws == res and ws > 1:
        img = torch.roll(torch.arange(rows, dtype=torch.int64).view(B, res, res, 1), shifts=(-1, -1), dims=(1, 2))
        assert torch.equal(_window_src(torch.arange(rows), B, res, res, ws, 1), _window_partition(img, ws).reshape(-1))


@pytest.mark.parametrize("name,stage,C,res,ws", [s for s in STAGES if s[1] < 3])
def test_merge_map_matches_cat(name, stage, C, res, ws):
    B = 2
    x = torch.arange(B * res * res, dtype=torch.int64).view(B, res, res, 1)
    # PatchMerging.forward's cat, one column per quarter: the image row each quarter of each merged row comes from
    cat = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1).view(-1, 4)
    m = torch.arange(cat.shape[0])
    for q in range(4):
        assert torch.equal(_merge_src(m, q, res, res), cat[:, q])


def _desc(K, O, n_H=1, post_gelu=0, rows=6272, bit=8, bias=1):
    from ptq4vit_b200 import _lib
    d = _lib.LinearDesc()
    d.rows, d.tokens, d.in_features, d.out_features = rows, 1, K, O
    d.n_V, d.n_H, d.n_a, d.w_bit, d.a_bit = 1, n_H, 1, bit, bit
    d.eq_n, d.search_round, d.post_gelu, d.has_bias = 1, 1, post_gelu, bias
    return d


def _gather(mode, images=0, H=0, W=0, ws=0, shift=0):
    from ptq4vit_b200 import _lib
    return _lib.InputGather(_lib.GATHER[mode] if isinstance(mode, str) else mode, _lib.WindowLayout(images, H, W, ws, shift))


def _gather_ok(d, mode):
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    g = _gather(mode)
    _lib.check(_lib.lib().p4v_linear_gather_ok(ctypes.byref(d), ctypes.byref(g), ctypes.byref(ok)), "gather_ok")
    return ok.value


def _norm_ok(d):
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    _lib.check(_lib.lib().p4v_linear_norm_ok(ctypes.byref(d), ctypes.byref(ok)), "norm_ok")
    return ok.value


@pytest.mark.parametrize("bit", [8, 6])
def test_rule_accepts_every_swin_qkv_and_foldable_reduction(bit):
    for _name, stage, C, _res, _ws in STAGES:
        for n_H in (1, C // 32):
            qkv = _desc(C, 3 * C, n_H, bit=bit)
            assert _norm_ok(qkv) == 1 and _gather_ok(qkv, "window") == 1, (C, n_H)
        if stage < 3:
            red = _desc(4 * C, 2 * C, bit=bit, bias=0)
            assert _gather_ok(red, "merge") == _norm_ok(red) == (1 if 4 * C < 1536 else 0), C
    # Swin-T's and Swin-B's first two reductions
    for C in (96, 192, 128, 256):
        assert _gather_ok(_desc(4 * C, 2 * C, bias=0, bit=bit), "merge") == 1


def test_rule_rejections():
    from ptq4vit_b200 import _lib
    assert _gather_ok(_desc(1536, 768, bias=0), "merge") == 0, "streamed path (Swin-T/S's last PatchMerging)"
    assert _gather_ok(_desc(1536, 768, bias=0), "window") == 0
    assert _gather_ok(_desc(3072, 768, 24), "window") == 0, "streamed path (ViT-B fc2)"
    assert _gather_ok(_desc(768, 3072, 24, post_gelu=1), "window") == 0, "post-GELU"
    assert _gather_ok(_desc(768, 3072, 24, post_gelu=1), "merge") == 0, "post-GELU"
    odd = _desc(392, 192)                               # C = 98: in_features % 16 != 0
    assert _norm_ok(odd) == 1 and _gather_ok(odd, "merge") == 0 and _gather_ok(odd, "window") == 1
    assert _gather_ok(_desc(98, 64), "window") == 0, "in_features % 4 != 0"
    ok = ctypes.c_int()
    g = _gather(7)
    assert _lib.lib().p4v_linear_gather_ok(ctypes.byref(_desc(96, 288)), ctypes.byref(g), ctypes.byref(ok)) != 0
    assert "gather mode" in _lib.lib().p4v_last_error().decode()


def test_rule_ignores_rows():
    for rows in (1, 5, 6272, 100000):
        assert _gather_ok(_desc(96, 288, rows=rows), "window") == 1
        assert _gather_ok(_desc(384, 192, rows=rows, bias=0), "merge") == 1


def _v(a):
    return a and ctypes.c_void_p(a)


def _call(d, g, x=1 << 20, gamma=4096, beta=8192, bias=12288, packed=16 << 20, out=64 << 20):
    """p4v_linear_frozen_forward_norm_gather on made-up device addresses: every case here must fail validation, never
    launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_linear_frozen_forward_norm_gather(ctypes.byref(d), _v(x), _v(gamma), _v(beta), ctypes.c_float(1e-5), _v(bias),
                                                  _v(packed), None if g is None else ctypes.byref(g), _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


ROWS = 2 * 56 * 56          # two Swin-T/224 stage-1 images


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(gamma=0), "null pointer"), (dict(packed=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(g=None), "null pointer"), (dict(bias=0), "bias is null"), (dict(x=(1 << 20) + 4), "aligned"),
    (dict(beta=8196), "aligned"), (dict(out=(64 << 20) + 4), "aligned"),
    (dict(out=(1 << 20) + 4096), "x overlaps out"), (dict(x=(64 << 20) + 4096), "x overlaps out"),
    (dict(g=("window", 2, 56, 56, 7, 7)), "shift"), (dict(g=("window", 2, 56, 56, 7, -1)), "shift"),
    (dict(g=("window", 2, 56, 56, 0, 0)), "positive"), (dict(g=("window", 0, 56, 56, 7, 0)), "positive"),
    (dict(g=("window", 2, 56, 60, 7, 3)), "multiples of the window"), (dict(g=("window", 3, 56, 56, 7, 3)), "rows"),
    (dict(g=(0, 2, 56, 56, 7, 3)), "gather mode"),
])
def test_window_validation_before_launch(case, match):
    case = dict(case)
    g = case.pop("g", ("window", 2, 56, 56, 7, 3))
    rc, msg = _call(_desc(96, 288, 3, rows=ROWS), None if g is None else _gather(*g), **case)
    assert rc != 0 and match in msg, msg


@pytest.mark.parametrize("g,match", [
    (("merge", 2, 56, 56, 7, 0), "window and shift must be 0"), (("merge", 2, 56, 56, 0, 1), "window and shift must be 0"),
    (("merge", 2, 55, 56, 0, 0), "even"), (("merge", 2, 56, 57, 0, 0), "even"), (("merge", 0, 56, 56, 0, 0), "positive"),
    (("merge", 4, 56, 56, 0, 0), "the layer has"), (("merge", 2, 56, 28, 0, 0), "the layer has"),
])
def test_merge_validation_before_launch(g, match):
    rc, msg = _call(_desc(384, 192, rows=ROWS // 4, bias=0), _gather(*g), bias=0)
    assert rc != 0 and match in msg, msg


def test_refused_layers_before_launch():
    rc, msg = _call(_desc(1536, 768, rows=2 * 7 * 7, bias=0), _gather("merge", 2, 14, 14), bias=0)
    assert rc != 0 and "p4v_linear_gather_ok" in msg, msg
    rc, msg = _call(_desc(392, 192, rows=ROWS // 4, bias=0), _gather("merge", 2, 56, 56), bias=0)
    assert rc != 0 and "p4v_linear_gather_ok" in msg, msg
    rc, msg = _call(_desc(768, 3072, 24, post_gelu=1, rows=ROWS), _gather("window", 2, 56, 56, 7, 0))
    assert rc != 0 and "p4v_linear_gather_ok" in msg, msg


def test_new_symbols_exported():
    from ptq4vit_b200 import _lib
    for name in ("p4v_linear_gather_ok", "p4v_linear_frozen_forward_norm_gather"):
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)


def test_python_rule_refuses_early():
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear, frozen_gather_applies
    ln = torch.nn.LayerNorm(32)
    x = torch.zeros(2, 16, 32)
    g = ("window", 2, 4, 4, 2, 1)
    assert not frozen_gather_applies(ln, torch.nn.Linear(32, 96), x, g)
    assert not frozen_gather_applies(ln, MinMaxQuantLinear(32, 96), x, g), "not frozen"
    q = _fake_frozen(MinMaxQuantLinear, 32, 96)
    assert not frozen_gather_applies(ln, q, x[:, ::2], ("window", 2, 2, 4, 2, 1)), "not contiguous"
    assert not frozen_gather_applies(ln, q, x, ("window", 2, 4, 4, 3, 1)), "window does not divide the image"
    assert not frozen_gather_applies(ln, q, x, ("window", 3, 4, 4, 2, 1)), "wrong images"
    assert not frozen_gather_applies(ln, q, x, ("window", 2, 4, 4, 2, 2)), "shift >= window"
    assert not frozen_gather_applies(torch.nn.LayerNorm(128), _fake_frozen(MinMaxQuantLinear, 128, 64), x,
                                     ("merge", 2, 4, 4, 1, 0)), "merge with a window"


def _fake_frozen(lin_cls, K, O, bias=True):
    q = lin_cls(K, O, bias=bias)
    q._packed = torch.zeros(1, dtype=torch.uint8)          # frozen is faked: the flag is all fuse_gather reads of it
    q.mode = "quant_forward"
    return q


def test_fuse_gather_bookkeeping():
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import PatchMerging, SwinBlock, get_net
    swin = get_net("swin_tiny_patch4_window7_224", device="cpu", depths=(2, 2, 2, 2), num_heads=(3, 6, 12, 24))
    sites = [n for n, m in swin.named_modules() if isinstance(m, (SwinBlock, PatchMerging))]
    assert len(sites) == 11 and deploy.fuse_gather(swin) == sites, "no frozen Linear: every site is left unfolded"
    assert not any(getattr(m, "fold_gather", False) for m in swin.modules())
    sb, pm = swin.layers[0].blocks[1], swin.layers[0].downsample
    sb.attn.qkv = _fake_frozen(MinMaxQuantLinear, 96, 288)
    pm.reduction = _fake_frozen(MinMaxQuantLinear, 384, 192, bias=False)
    last = swin.layers[2].downsample                     # K = 1536: streamed, never folded
    last.reduction = _fake_frozen(MinMaxQuantLinear, 1536, 768, bias=False)
    left = deploy.fuse_gather(swin)
    assert left == [n for n in sites if n not in ("layers.0.blocks.1", "layers.0.downsample")]
    assert "layers.2.downsample" in left and not last.fold_gather
    assert sb.fold_gather and pm.fold_gather and not swin.layers[0].blocks[0].fold_gather
    # fuse_norm is untouched by it
    assert not pm.fold_norm and not any(getattr(m, "fold_norm2", False) for m in swin.modules())
    deploy.unfuse_gather(swin)
    assert not any(getattr(m, "fold_gather", False) for m in swin.modules())
    vit = get_net("vit_tiny_patch16_224", device="cpu", depth=1)
    assert deploy.fuse_gather(vit) == [], "a ViT has no gather site"


def test_default_and_unfoldable_forwards_unchanged():
    """With the flag off the modules run as before; with it on and nothing frozen, every site runs unfolded, same bits."""
    from ptq4vit_b200.utils.models import PatchMerging, SwinBlock, WindowAttention
    assert not SwinBlock.fold_gather and not PatchMerging.fold_gather
    torch.manual_seed(0)
    for shift in (0, 2):
        sb = SwinBlock(32, 8, 2, 4, shift).eval()
        xs = torch.randn(2, 64, 32)
        with torch.no_grad():
            want = sb(xs)
            for res_flag in (False, True):
                sb.fold_residual = res_flag
                sb.fold_gather = True
                assert torch.equal(sb(xs).view(torch.int32), want.view(torch.int32))
                sb.fold_gather = False
                assert torch.equal(sb(xs).view(torch.int32), want.view(torch.int32))
    pm = PatchMerging(8, 32).eval()
    x = torch.randn(2, 64, 32)
    with torch.no_grad():
        want = pm(x)
        pm.fold_gather = True
        assert torch.equal(pm(x).view(torch.int32), want.view(torch.int32))
    # WindowAttention's new arguments default to today's call
    wa = WindowAttention(32, 4, 2).eval()
    xw = torch.randn(8, 16, 32)
    with torch.no_grad():
        assert torch.equal(wa(xw), wa(xw, None, None, None, None, None))
