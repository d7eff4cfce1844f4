"""The long-sequence fused attention core without a GPU: p4v_attention_frozen_forward_long rejects bad arguments before
any launch, its shape rule, and the max_tokens bookkeeping of fuse_attention / unfuse_attention."""
import ctypes

import pytest

from tests.test_fused_attention_cpu import _descs, _pack_bytes, _tiny_nets


def _call(a, d1, d2, qkv=4096, pack1=8192, pack2=12288, out=16384, bias=None, mask=None, strides=(577 * 2304, 2304, 768, 64),
          bytes1=None, bytes2=None):
    """p4v_attention_frozen_forward_long on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_attention_frozen_forward_long(
        ctypes.byref(a), qkv and ctypes.c_void_p(qkv), (ctypes.c_longlong * 4)(*strides), ctypes.byref(d1),
        pack1 and ctypes.c_void_p(pack1), _pack_bytes(d1) if bytes1 is None else bytes1, ctypes.byref(d2),
        pack2 and ctypes.c_void_p(pack2), _pack_bytes(d2) if bytes2 is None else bytes2, bias and ctypes.c_void_p(bias),
        mask and ctypes.c_void_p(mask), out and ctypes.c_void_p(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(qkv=0), "null pointer"), (dict(pack1=0), "null pointer"), (dict(pack2=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(tokens=0), "empty shape"), (dict(tokens=1025), "1025 tokens"),
    (dict(head_dim=72), "head_dim 72"), (dict(head_dim=24), "head_dim 24"),
    (dict(scale_on_q=1), "scale_on_q"), (dict(bias=8192), "bias and mask"), (dict(mask=8192, n_windows=4), "bias and mask"),
    (dict(qkv=4098), "4-byte aligned"), (dict(out=16388), "8-byte aligned"), (dict(pack2=12296), "16-byte aligned"),
    (dict(pack_heads=11), "packs made for 11 and 11 heads"), (dict(bytes1=16), "pack sizes"), (dict(bytes2=16), "pack sizes"),
    (dict(sos1=1), "matmul1 cannot be split-of-softmax"),
    (dict(strides=(-1, 2304, 768, 64)), "negative stride"), (dict(strides=(577 * 2304, 2304, -768, 64)), "negative stride"),
])
def test_validation_before_launch(case, match):
    case = dict(case)
    a, d1, d2 = _descs(tokens=case.pop("tokens", 577), head_dim=case.pop("head_dim", 64))
    a.scale_on_q = case.pop("scale_on_q", 0)
    a.n_windows = case.pop("n_windows", 0)
    if "pack_heads" in case:
        d1.heads = d2.heads = case.pop("pack_heads")
    if case.pop("sos1", 0):
        d1.sos = 1
    rc, msg = _call(a, d1, d2, **case)
    assert rc != 0 and match in msg, msg
    assert msg.startswith("attention_frozen_forward_long"), msg


def test_long_shape_rule():
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    want = {(1, 64): 1, (197, 64): 1, (257, 64): 1, (577, 64): 1, (577, 32): 1, (577, 16): 1, (1024, 64): 1, (1024, 48): 1,
            (1025, 64): 0, (0, 64): 0, (577, 72): 0, (577, 24): 0, (577, 0): 0, (-1, 64): 0}
    for (n, d), w in want.items():
        _lib.check(_lib.lib().p4v_attention_long_ok(n, d, ctypes.byref(ok)), "long_ok")
        assert ok.value == w, (n, d)
    # the short kernel's rule is unchanged
    _lib.check(_lib.lib().p4v_attention_fused_ok(577, 64, ctypes.byref(ok)), "fused_ok")
    assert ok.value == 0


def _freeze_all(net):
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
    from ptq4vit_b200.utils.models import Attention, WindowAttention
    attn = [m for m in net.modules() if isinstance(m, (Attention, WindowAttention))]
    for m in attn:
        for name in ("matmul1", "matmul2"):
            mm = MinMaxQuantMatMul()
            mm._packed = {1: None}
            setattr(m, name, mm)
    return attn


def test_fuse_max_tokens_bookkeeping():
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Attention, WindowAttention
    vit, swin = _tiny_nets()
    for net in (vit, swin):
        attn = _freeze_all(net)
        assert deploy.fuse_attention(net) == []
        assert all(m.fused for m in attn)
        assert all(m.fused_max_tokens == 256 for m in attn if isinstance(m, Attention))
        assert deploy.fuse_attention(net, max_tokens=1024) == []
        for m in attn:
            if isinstance(m, WindowAttention):
                assert "fused_max_tokens" not in vars(m), "windowed attention keeps the 256-token rule"
            else:
                assert m.fused and m.fused_max_tokens == 1024
        deploy.fuse_attention(net, max_tokens=600)
        assert all(m.fused_max_tokens == 600 for m in attn if isinstance(m, Attention))
        deploy.unfuse_attention(net)
        assert not any(m.fused for m in attn)
        assert all(m.fused_max_tokens == 256 for m in attn if isinstance(m, Attention))


@pytest.mark.parametrize("bad", [255, 0, 1025, 2048, -1, 512.0, "1024", None, True])
def test_fuse_max_tokens_rejects(bad):
    from ptq4vit_b200.utils import deploy
    vit, _ = _tiny_nets()
    attn = _freeze_all(vit)
    with pytest.raises(ValueError, match="max_tokens"):
        deploy.fuse_attention(vit, max_tokens=bad)
    assert not any(m.fused for m in attn), "a rejected call marks nothing"


def test_applies_picks_the_rule_from_n():
    """frozen_attention_applies consults the short rule up to 256 tokens and the long rule only above it, and only up to
    max_tokens; modules that are not frozen never qualify."""
    from ptq4vit_b200.quant_layers import matmul as MM

    class _F(MM.MinMaxQuantMatMul):
        frozen = True
    m1, m2 = _F(), _F()
    m1.mode = m2.mode = "quant_forward"
    assert MM.frozen_attention_applies(m1, m2, 197, 64)
    assert not MM.frozen_attention_applies(m1, m2, 577, 64)
    assert MM.frozen_attention_applies(m1, m2, 577, 64, max_tokens=1024)
    assert MM.frozen_attention_applies(m1, m2, 577, 64, max_tokens=577)
    assert not MM.frozen_attention_applies(m1, m2, 578, 64, max_tokens=577)
    assert not MM.frozen_attention_applies(m1, m2, 577, 72, max_tokens=1024)
    assert not MM.frozen_attention_applies(MM.MinMaxQuantMatMul(), m2, 577, 64, max_tokens=1024)
