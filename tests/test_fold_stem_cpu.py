"""The patch embedding's token epilogue folded into the frozen conv, without a GPU: the shape rules over every patch
embedding of the zoo, every rejection of the new entry points before any launch, the Python rule's refusals,
fuse_stem / unfuse_stem bookkeeping, and a model that was never folded runs the code it ran before."""
import ctypes

import pytest
import torch


def _desc(C, patch=16, images=2, size=224, bias=1, layerwise=0, bit=8, cin=3):
    from ptq4vit_b200 import _lib
    d = _lib.ConvFrozenDesc()
    d.images, d.in_channels, d.height, d.width = images, cin, size, size
    d.out_channels, d.kernel_h, d.kernel_w = C, patch, patch
    d.w_bit, d.layerwise, d.has_bias = bit, layerwise, bias
    return d


def _ok(fn, d):
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    assert getattr(_lib.lib(), fn)(ctypes.byref(d), ctypes.byref(ok)) == 0
    return ok.value


def test_rules_accept_every_zoo_stem():
    from ptq4vit_b200.utils.models import _SWIN_ZOO, _ZOO
    for cfg in _ZOO.values():
        assert _ok("p4v_conv_pos_ok", _desc(cfg["dim"], cfg["patch"])) == 1
    for cfg in _SWIN_ZOO.values():
        assert _ok("p4v_conv_norm_ok", _desc(cfg["dim"], 4)) == 1


def test_rule_rejections():
    assert _ok("p4v_conv_norm_ok", _desc(192, 4)) == 0, "the LayerNorm needs the whole row in one CTA"
    assert _ok("p4v_conv_pos_ok", _desc(192, 4)) == 1
    assert _ok("p4v_conv_pos_ok", _desc(98)) == 0 and _ok("p4v_conv_norm_ok", _desc(98, 4)) == 0, "out_channels % 4"
    assert _ok("p4v_conv_pos_ok", _desc(768, 64, cin=3)) == 0, "K above the frozen conv's rule"
    assert _ok("p4v_conv_pos_ok", _desc(768, bit=9)) == 0
    for size, images in ((1, 1), (224, 0), (100000, 7)):
        assert _ok("p4v_conv_pos_ok", _desc(768, size=size, images=images)) == 1, "the rules ignore the image"


def _v(a):
    return a and ctypes.c_void_p(a)


PACK = 16 << 20
OUT = 64 << 20


def _packed_bytes(d):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    rc = _lib.lib().p4v_conv_pack_bytes(ctypes.byref(d), ctypes.byref(n))
    return n.value if rc == 0 else 1 << 20                # a descriptor outside the rule: the call must refuse it


def _call_pos(d, x=1 << 30, bias=4096, packed=PACK, packed_bytes=None, cls=8192, cls_numel=None, pos=12288,
              pos_numel=None, out=OUT):
    """p4v_conv_frozen_forward_pos on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    P = (d.height // d.kernel_h) * (d.width // d.kernel_w)
    n0 = _lib.launch_count()
    rc = lib.p4v_conv_frozen_forward_pos(ctypes.byref(d), _v(x), _v(bias), _v(packed),
                                         _packed_bytes(d) if packed_bytes is None else packed_bytes, _v(cls),
                                         d.out_channels if cls_numel is None else cls_numel, _v(pos),
                                         (1 + P) * d.out_channels if pos_numel is None else pos_numel, _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


def _call_norm(d, x=1 << 30, bias=4096, packed=PACK, packed_bytes=None, gamma=8192, beta=12288, norm_numel=None, eps=1e-5,
               out=OUT):
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_conv_frozen_forward_norm(ctypes.byref(d), _v(x), _v(bias), _v(packed),
                                          _packed_bytes(d) if packed_bytes is None else packed_bytes, _v(gamma), _v(beta),
                                          d.out_channels if norm_numel is None else norm_numel, ctypes.c_float(eps), _v(out),
                                          None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


VIT_OUT_BYTES = 2 * 197 * 768 * 4


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(packed=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(cls=0), "null pointer"), (dict(pos=0), "null pointer"), (dict(bias=0), "bias is null"),
    (dict(packed_bytes=1024), "packed buffer too small"), (dict(packed=PACK + 4), "aligned"), (dict(x=(1 << 30) + 2), "aligned"),
    (dict(out=OUT + 4), "out must be 16-byte aligned"), (dict(cls=8196), "16-byte aligned"), (dict(pos=12292), "16-byte aligned"),
    (dict(cls_numel=767), "cls has 767 elements"), (dict(pos_numel=196 * 768), "pos_embed has"),
    (dict(x=OUT + 4096), "out overlaps x"), (dict(packed=OUT + VIT_OUT_BYTES - 16), "out overlaps"),
    (dict(bias=OUT - 16), "out overlaps"), (dict(cls=OUT + 1024), "out overlaps cls"),
    (dict(pos=OUT - 4096), "out overlaps cls or pos_embed"),
])
def test_pos_validation_before_launch(case, match):
    rc, msg = _call_pos(_desc(768), **case)
    assert rc != 0 and match in msg, msg


def test_pos_refused_shapes_before_launch():
    rc, msg = _call_pos(_desc(98))
    assert rc != 0 and "p4v_conv_pos_ok" in msg, msg
    rc, msg = _call_pos(_desc(768, size=8))
    assert rc != 0 and "bad geometry" in msg, msg
    rc, msg = _call_pos(_desc(768, bit=9))
    assert rc != 0 and "w_bit" in msg, msg


SWIN_OUT_BYTES = 2 * 56 * 56 * 96 * 4


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(packed=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(gamma=0), "null pointer"), (dict(beta=0), "null pointer"), (dict(bias=0), "bias is null"),
    (dict(gamma=8200), "gamma and beta must be 16-byte aligned"), (dict(beta=12296), "gamma and beta must be 16-byte aligned"),
    (dict(out=OUT + 8), "out must be 16-byte aligned"), (dict(norm_numel=128), "the LayerNorm has 128 features"),
    (dict(eps=-1.0), "eps"), (dict(eps=float("inf")), "eps"), (dict(eps=float("nan")), "eps"),
    (dict(x=OUT + SWIN_OUT_BYTES - 4096), "out overlaps x"), (dict(packed=OUT + 4096), "out overlaps"),
    (dict(gamma=OUT + 16), "out overlaps gamma or beta"), (dict(beta=OUT + SWIN_OUT_BYTES - 16), "out overlaps gamma or beta"),
])
def test_norm_validation_before_launch(case, match):
    rc, msg = _call_norm(_desc(96, 4), **case)
    assert rc != 0 and match in msg, msg


def test_norm_refused_shapes_before_launch():
    rc, msg = _call_norm(_desc(192, 4))
    assert rc != 0 and "out_channels above 128" in msg and "p4v_conv_norm_ok" in msg, msg
    rc, msg = _call_norm(_desc(100 - 2, 4))
    assert rc != 0 and "multiple of 4" in msg, msg


def test_new_symbols_exported():
    from ptq4vit_b200 import _lib
    for name in ("p4v_conv_pos_ok", "p4v_conv_norm_ok", "p4v_conv_frozen_forward_pos", "p4v_conv_frozen_forward_norm"):
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)


def _fake_frozen(C, patch, bias=True):
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d
    q = MinMaxQuantConv2d(3, C, patch, stride=patch, bias=bias, a_bit=32)
    q._packed = torch.zeros(1, dtype=torch.uint8)          # frozen is faked: the flag is all fuse_stem reads of it
    q.w_interval = torch.ones(C, 1, 1, 1)
    q.calibrated = True
    q.mode = "quant_forward"
    return q


def test_python_rule_refuses():
    from ptq4vit_b200.quant_layers.conv import MinMaxQuantConv2d, frozen_stem_applies
    conv = _fake_frozen(64, 8)
    x = torch.zeros(2, 3, 32, 32)
    cls, pos = torch.zeros(1, 1, 64), torch.zeros(1, 17, 64)
    ln = torch.nn.LayerNorm(64)
    with torch.no_grad():
        assert frozen_stem_applies(conv, x, cls_token=cls, pos_embed=pos)
        assert frozen_stem_applies(conv, x, norm=ln)
        assert not frozen_stem_applies(conv, x, cls_token=cls, pos_embed=pos, norm=ln), "one stem at a time"
        assert not frozen_stem_applies(conv, x, cls_token=cls), "cls without pos_embed"
        assert not frozen_stem_applies(conv, x), "neither"
        assert not frozen_stem_applies(MinMaxQuantConv2d(3, 64, 8, stride=8, a_bit=32), x, norm=ln), "not frozen"
        assert not frozen_stem_applies(conv, x.permute(0, 1, 3, 2), norm=ln), "not contiguous"
        assert not frozen_stem_applies(conv, x.double(), norm=ln), "not FP32"
        assert not frozen_stem_applies(conv, x[:, :2].contiguous(), norm=ln), "in_channels"
        assert not frozen_stem_applies(conv, x, cls_token=cls, pos_embed=pos.half()), "pos_embed not FP32"
        assert not frozen_stem_applies(conv, x, cls_token=cls, pos_embed=torch.zeros(1, 16, 64)), "pos_embed rows"
        assert not frozen_stem_applies(conv, x, cls_token=torch.zeros(1, 64), pos_embed=pos), "cls shape"
        assert not frozen_stem_applies(conv, x, cls_token=cls, pos_embed=torch.zeros(17 * 64 + 1)[1:].view(1, 17, 64)), "pos_embed 4 bytes off"
        assert not frozen_stem_applies(conv, x, norm=torch.nn.LayerNorm(64, elementwise_affine=False)), "no affine"
        assert not frozen_stem_applies(conv, x, norm=torch.nn.LayerNorm(32)), "normalized_shape"
        assert not frozen_stem_applies(conv, x, norm=torch.nn.RMSNorm(64)), "not a LayerNorm"
        conv.mode = "raw"
        assert not frozen_stem_applies(conv, x, norm=ln), "not in quant_forward"
        conv.mode = "quant_forward"
        wide = _fake_frozen(192, 4)
        assert not frozen_stem_applies(wide, x, norm=torch.nn.LayerNorm(192)), "p4v_conv_norm_ok: out_channels > 128"
    # grad wanted: the LayerNorm's parameters require grad under grad mode
    assert not frozen_stem_applies(conv, x, norm=ln)
    assert not frozen_stem_applies(conv, x.requires_grad_(), cls_token=cls, pos_embed=pos)


def test_fuse_stem_bookkeeping():
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import get_net
    vit = get_net("vit_tiny_patch16_224", device="cpu", depth=1)
    swin = get_net("swin_tiny_patch4_window7_224", device="cpu", depths=(2, 2, 2, 2), num_heads=(3, 6, 12, 24))
    assert deploy.fuse_stem(vit) == [""] and deploy.fuse_stem(swin) == [""], "no frozen conv: left unfolded"
    assert not vit.fold_stem and not swin.fold_stem
    vit.patch_embed.proj = _fake_frozen(192, 16)
    swin.patch_embed.proj = _fake_frozen(96, 4)
    assert deploy.fuse_stem(vit) == [] and vit.fold_stem
    assert deploy.fuse_stem(swin) == [] and swin.fold_stem
    # the other folds are untouched by it
    assert not vit.fold_norm and not any(getattr(m, "fold_residual", False) or getattr(m, "fold_gather", False)
                                         for net in (vit, swin) for m in net.modules())
    deploy.unfuse_stem(vit)
    deploy.unfuse_stem(swin)
    assert not vit.fold_stem and not swin.fold_stem
    wide = get_net("swin_tiny_patch4_window7_224", device="cpu", dim=192, depths=(2, 2, 2, 2), num_heads=(3, 6, 12, 24))
    wide.patch_embed.proj = _fake_frozen(192, 4)
    assert deploy.fuse_stem(wide) == [""], "p4v_conv_norm_ok refuses out_channels > 128"
    holder = torch.nn.ModuleDict({"a": vit, "b": get_net("vit_tiny_patch16_224", device="cpu", depth=1)})
    assert deploy.fuse_stem(holder) == ["b"] and vit.fold_stem


def test_default_and_unfoldable_forwards_unchanged():
    """With the flag off the models run as before; with it on and no frozen conv, the stem runs unfolded, same bits."""
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
    assert not VisionTransformer.fold_stem and not SwinTransformer.fold_stem
    vit = VisionTransformer(img_size=32, patch=8, dim=64, depth=1, num_heads=2, num_classes=10).eval()
    swin = SwinTransformer(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10).eval()
    x = torch.randn(2, 3, 32, 32)
    with torch.no_grad():
        for net in (vit, swin):
            want = net(x)
            net.fold_stem = True
            assert torch.equal(net(x).view(torch.int32), want.view(torch.int32))
