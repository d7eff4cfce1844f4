"""The fused frozen attention core without a GPU: the C ABI rejects bad arguments before any launch, the shape rule,
fuse_attention / unfuse_attention bookkeeping, and a model that was never fused runs the plain attention code."""
import ctypes

import pytest
import torch


def _descs(heads=12, tokens=197, head_dim=64, sos2=True):
    from ptq4vit_b200 import _lib
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim, a.scale_on_q, a.n_windows, a.scale = 32, tokens, heads, head_dim, 0, 0, head_dim ** -0.5
    mms = []
    for sos in (0, 1 if sos2 else 0):
        d = _lib.MatMulDesc()
        d.batch, d.heads, d.S1, d.S2, d.S3, d.A_bit, d.B_bit, d.eq_n, d.search_round, d.sos = 1, heads, 1, 1, 1, 8, 8, 1, 1, sos
        mms.append(d)
    return a, mms[0], mms[1]


def _pack_bytes(d):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_matmul_pack_bytes(ctypes.byref(d), ctypes.byref(n)), "pack_bytes")
    return n.value


def _call(a, d1, d2, qkv=4096, pack1=8192, pack2=12288, out=16384, bias=None, mask=None, strides=(197 * 2304, 2304, 768, 64),
          bytes1=None, bytes2=None):
    """p4v_attention_frozen_forward on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    rc = lib.p4v_attention_frozen_forward(
        ctypes.byref(a), qkv and ctypes.c_void_p(qkv), (ctypes.c_longlong * 4)(*strides), ctypes.byref(d1),
        pack1 and ctypes.c_void_p(pack1), _pack_bytes(d1) if bytes1 is None else bytes1, ctypes.byref(d2),
        pack2 and ctypes.c_void_p(pack2), _pack_bytes(d2) if bytes2 is None else bytes2, bias and ctypes.c_void_p(bias),
        mask and ctypes.c_void_p(mask), out and ctypes.c_void_p(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(qkv=0), "null pointer"), (dict(pack1=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(tokens=257), "257 tokens"), (dict(tokens=577), "577 tokens"),
    (dict(head_dim=72), "head_dim 72"), (dict(head_dim=24), "head_dim 24"),
    (dict(qkv=4098), "4-byte aligned"), (dict(out=16388), "8-byte aligned"), (dict(pack2=12296), "16-byte aligned"),
    (dict(bias=4097), "4-byte aligned"),
    (dict(pack_heads=11), "packs made for 11 and 11 heads"), (dict(bytes2=16), "pack sizes"),
    (dict(sos1=1), "matmul1 cannot be split-of-softmax"), (dict(mask=8192), "n_windows"),
    (dict(strides=(-1, 2304, 768, 64)), "negative stride"),
])
def test_validation_before_launch(case, match):
    case = dict(case)
    a, d1, d2 = _descs(tokens=case.pop("tokens", 197), head_dim=case.pop("head_dim", 64))
    if "pack_heads" in case:
        d1.heads = d2.heads = case.pop("pack_heads")
    if case.pop("sos1", 0):
        d1.sos = 1
    rc, msg = _call(a, d1, d2, **case)
    assert rc != 0 and match in msg, msg


def test_shape_rule():
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    want = {(197, 64): 1, (49, 32): 1, (144, 32): 1, (16, 16): 1, (17, 32): 1, (256, 64): 1, (257, 64): 0, (577, 64): 0,
            (197, 72): 0, (197, 40): 0, (0, 64): 0}
    for (n, d), w in want.items():
        _lib.check(_lib.lib().p4v_attention_fused_ok(n, d, ctypes.byref(ok)), "fused_ok")
        assert ok.value == w, (n, d)


class _Frozen(torch.nn.Module):
    """Stands in for a frozen MatMul module (frozen modules need a CUDA device): only the `frozen` flag is read here."""


def _tiny_nets():
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
    vit = VisionTransformer(img_size=32, patch=8, dim=64, depth=2, num_heads=2, num_classes=10)
    swin = SwinTransformer(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)
    return vit, swin


def test_fuse_and_unfuse_bookkeeping():
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Attention, WindowAttention
    for net in _tiny_nets():
        attn = [(n, m) for n, m in net.named_modules() if isinstance(m, (Attention, WindowAttention))]
        assert deploy.fuse_attention(net) == [n for n, _ in attn], "plain MatMul modules are not frozen"
        assert not any(m.fused for _, m in attn)
        # freeze both MatMul modules of the first attention module, only matmul1 of the second
        for i, (_, m) in enumerate(attn[:2]):
            m.matmul1 = MinMaxQuantMatMul()
            m.matmul1._packed = {1: None}
            if i == 0:
                m.matmul2 = MinMaxQuantMatMul()
                m.matmul2._packed = {1: None}
        assert deploy.fuse_attention(net) == [n for n, _ in attn[1:]]
        assert attn[0][1].fused and not any(m.fused for _, m in attn[1:])
        deploy.unfuse_attention(net)
        assert not any(m.fused for _, m in attn)


def test_never_fused_model_runs_the_plain_code(monkeypatch):
    from ptq4vit_b200.utils import models

    def refuse(*a, **k):
        raise AssertionError("the fused path was consulted")
    monkeypatch.setattr(models, "frozen_attention_applies", refuse)
    monkeypatch.setattr(models, "frozen_attention", refuse)
    for net in _tiny_nets():
        with torch.no_grad():
            y = net(torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(0)))
        assert y.shape == (2, 10) and bool(torch.isfinite(y).all())
