"""A LayerNorm folded into its frozen Linear, without a GPU: the shape rules, every rejection of the new entry points
before any launch, the Python rule's early refusals, fuse_norm / unfuse_norm bookkeeping, and a model that was never
folded runs the code it ran before."""
import ctypes

import pytest
import torch


def _desc(K, O, n_H=1, post_gelu=0, rows=6304, bit=8):
    from ptq4vit_b200 import _lib
    d = _lib.LinearDesc()
    d.rows, d.tokens, d.in_features, d.out_features = rows, 1, K, O
    d.n_V, d.n_H, d.n_a, d.w_bit, d.a_bit = 1, n_H, 1, bit, bit
    d.eq_n, d.search_round, d.post_gelu, d.has_bias = 1, 1, post_gelu, 1
    return d


def _ok(fn, *descs):
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    _lib.check(getattr(_lib.lib(), fn)(*[ctypes.byref(d) for d in descs], ctypes.byref(ok)), fn)
    return ok.value


def _frozen_path(d):
    from ptq4vit_b200 import _lib
    path = ctypes.c_int()
    _lib.check(_lib.lib().p4v_linear_frozen_path(ctypes.byref(d), ctypes.byref(path)), "frozen_path")
    return path.value


@pytest.mark.parametrize("K,O,n_H", [(768, 2304, 24), (768, 3072, 24), (768, 1000, 24), (96, 384, 3), (384, 192, 3),
                                     (768, 384, 1)])
def test_rule_accepts_vit_and_swin_consumers(K, O, n_H):
    # ViT-B qkv, fc1, head; Swin-T stage-1 fc1; Swin-T's first two PatchMerging reductions
    assert _ok("p4v_linear_norm_ok", _desc(K, O, n_H)) == 1
    assert _ok("p4v_linear_norm_ok", _desc(K, O, n_H, bit=6)) == 1


def test_rule_rejections():
    assert _ok("p4v_linear_norm_ok", _desc(768, 3072, 24, post_gelu=1)) == 0, "post-GELU"
    streamed = _desc(3072, 768, 24)
    assert _frozen_path(streamed) == 0 and _ok("p4v_linear_norm_ok", streamed) == 0, "streamed path (ViT-B fc2)"
    assert _ok("p4v_linear_norm_ok", _desc(1536, 768)) == 0, "streamed path (Swin-T's last PatchMerging)"
    odd = _desc(98, 64)
    assert _frozen_path(odd) == 1 and _ok("p4v_linear_norm_ok", odd) == 0, "in_features % 4 != 0"
    # a fused MLP whose plan has no room left for the LayerNorm's row statistics
    fc1, fc2 = _desc(1152, 3072), _desc(3072, 1152, post_gelu=1)
    assert _ok("p4v_mlp_fused_ok", fc1, fc2) == 1 and _ok("p4v_mlp_norm_ok", fc1, fc2) == 0
    assert _ok("p4v_mlp_norm_ok", _desc(768, 3072, 24), _desc(3072, 768, 24, post_gelu=1)) == 1


def test_rule_ignores_rows():
    for rows in (1, 5, 6304, 100000):
        assert _ok("p4v_linear_norm_ok", _desc(768, 2304, 24, rows=rows)) == 1


def _pack_bytes(d):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_pack_bytes(ctypes.byref(d), ctypes.byref(n)), "pack_bytes")
    return n.value


def _v(a):
    return a and ctypes.c_void_p(a)


def _call_linear(d, x=4096, g=8192, b=12288, eps=1e-6, bias=16384, packed=1 << 20, out=2 << 20):
    """p4v_linear_frozen_forward_norm on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_linear_frozen_forward_norm(ctypes.byref(d), _v(x), _v(g), _v(b), ctypes.c_float(eps), _v(bias), _v(packed),
                                            _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(g=0), "null pointer"), (dict(b=0), "null pointer"), (dict(packed=0), "null pointer"),
    (dict(out=0), "null pointer"), (dict(bias=0), "bias is null"), (dict(x=4100), "aligned"), (dict(g=8194), "aligned"),
    (dict(b=12290), "aligned"), (dict(out=(2 << 20) + 4), "aligned"), (dict(eps=-1e-6), "eps"), (dict(eps=float("inf")), "eps"),
    (dict(eps=float("nan")), "eps"), (dict(gelu=1), "does not fold"), (dict(K=98), "does not fold"),
    (dict(K=3072), "does not fold"),
])
def test_linear_validation_before_launch(case, match):
    case = dict(case)
    d = _desc(case.pop("K", 768), 2304, 1, post_gelu=case.pop("gelu", 0))
    rc, msg = _call_linear(d, **case)
    assert rc != 0 and match in msg, msg


def _call_mlp(d1, d2, x=4096, g=8192, b=12288, eps=1e-6, b1=16384, p1=1 << 20, b2=20480, p2=2 << 20, ws=3 << 20, out=4 << 20,
              ws_bytes=1 << 30):
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_mlp_frozen_forward_norm(ctypes.byref(d1), _v(x), _v(g), _v(b), ctypes.c_float(eps), _v(b1), _v(p1), _pack_bytes(d1),
                                         ctypes.byref(d2), _v(b2), _v(p2), _pack_bytes(d2), _v(ws), ws_bytes, _v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(g=0), "null pointer"), (dict(ws=0), "null pointer"), (dict(b2=0), "bias is null"),
    (dict(x=4104), "aligned"), (dict(ws=(3 << 20) + 8), "aligned"), (dict(eps=float("nan")), "eps"),
    (dict(ws_bytes=1 << 20), "workspace too small"), (dict(wide=1), "do not fuse with the LayerNorm"),
])
def test_mlp_validation_before_launch(case, match):
    case = dict(case)
    if case.pop("wide", 0):
        d1, d2 = _desc(1152, 3072), _desc(3072, 1152, post_gelu=1)
    else:
        d1, d2 = _desc(768, 3072, 24), _desc(3072, 768, 24, post_gelu=1)
    rc, msg = _call_mlp(d1, d2, **case)
    assert rc != 0 and match in msg, msg


def test_python_rule_refuses_without_frozen_linear():
    from ptq4vit_b200.quant_layers.linear import frozen_norm_applies
    ln, lin = torch.nn.LayerNorm(64), torch.nn.Linear(64, 32)
    assert not frozen_norm_applies(ln, lin, torch.zeros(3, 64))
    assert not frozen_norm_applies(torch.nn.LayerNorm(64, elementwise_affine=False), lin, torch.zeros(3, 64))
    assert not frozen_norm_applies(torch.nn.Identity(), lin, torch.zeros(3, 64))


def test_new_symbols_exported():
    from ptq4vit_b200 import _lib
    for name in ("p4v_linear_norm_ok", "p4v_mlp_norm_ok", "p4v_linear_frozen_forward_norm", "p4v_mlp_frozen_forward_norm",
                 "p4v_layer_norm_probe"):
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)


def test_fuse_norm_bookkeeping():
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import get_net
    vit = get_net("vit_tiny_patch16_224", device="cpu", depth=2)
    norms = [n for n, m in vit.named_modules() if isinstance(m, torch.nn.LayerNorm)]
    assert deploy.fuse_norm(vit) == norms, "no frozen Linear: every LayerNorm is left unfolded"
    assert not any(getattr(m, f, False) for m in vit.modules() for f in ("fold_norm", "fold_norm1", "fold_norm2"))
    swin = get_net("swin_tiny_patch4_window7_224", device="cpu", depths=(2, 2), num_heads=(3, 6))
    swin_norms = [n for n, m in swin.named_modules() if isinstance(m, torch.nn.LayerNorm)]
    assert deploy.fuse_norm(swin) == swin_norms
    # a frozen consumer is marked (frozen is faked: the flag is all fuse_norm looks at)
    from ptq4vit_b200.quant_layers.linear import MinMaxQuantLinear
    blk = vit.blocks[0]
    q = MinMaxQuantLinear(192, 576)
    q._packed = torch.zeros(1, dtype=torch.uint8)
    blk.attn.qkv = q
    left = deploy.fuse_norm(vit)
    assert "blocks.0.norm1" not in left and set(left) == set(norms) - {"blocks.0.norm1"}
    assert blk.fold_norm1 and not blk.fold_norm2
    deploy.unfuse_norm(vit)
    assert not blk.fold_norm1


def test_default_forward_unchanged():
    from ptq4vit_b200.utils.models import Block, SwinBlock, get_net
    torch.manual_seed(0)
    blk = Block(64, 2).eval()
    x = torch.randn(2, 5, 64)
    with torch.no_grad():
        want = x + blk.attn(blk.norm1(x))
        want = want + blk.mlp(blk.norm2(want))
        assert torch.equal(blk(x), want)
    assert not Block.fold_norm1 and not Block.fold_norm2 and not SwinBlock.fold_norm2
    vit = get_net("vit_tiny_patch16_224", device="cpu", depth=1, img_size=32)
    with torch.no_grad():
        h = vit.patch_embed(torch.randn(1, 3, 32, 32, generator=torch.Generator().manual_seed(1)))
    assert h.shape[-1] == 192
