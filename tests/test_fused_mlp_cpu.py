"""The fused frozen MLP without a GPU: the C ABI rejects bad arguments before any launch, the shape rule, the Python rule
(exact GELU only), fuse_mlp / unfuse_mlp bookkeeping, and a model that was never fused runs the plain MLP code."""
import ctypes

import pytest
import torch


def _desc(K, O, n_H=24, post_gelu=0, rows=6304, bit=8, n_a=1):
    from ptq4vit_b200 import _lib
    d = _lib.LinearDesc()
    d.rows, d.tokens, d.in_features, d.out_features = rows, 1, K, O
    d.n_V, d.n_H, d.n_a, d.w_bit, d.a_bit = 1, n_H, n_a, bit, bit
    d.eq_n, d.search_round, d.post_gelu, d.has_bias = 1, 1, post_gelu, 1
    return d


def _vitb(**kw1):
    return _desc(768, 3072, **kw1), _desc(3072, 768, post_gelu=1)


def _pack_bytes(d):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_pack_bytes(ctypes.byref(d), ctypes.byref(n)), "pack_bytes")
    return n.value


def _ws_bytes(d1, d2):
    from ptq4vit_b200 import _lib
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_mlp_frozen_workspace_bytes(ctypes.byref(d1), ctypes.byref(d2), ctypes.byref(n)), "ws_bytes")
    return n.value


def _ok(d1, d2):
    from ptq4vit_b200 import _lib
    ok = ctypes.c_int()
    _lib.check(_lib.lib().p4v_mlp_fused_ok(ctypes.byref(d1), ctypes.byref(d2), ctypes.byref(ok)), "fused_ok")
    return ok.value


def _call(d1, d2, x=4096, b1=8192, p1=1 << 20, b2=12288, p2=2 << 20, ws=3 << 20, out=4 << 20, bytes1=None, bytes2=None,
          ws_bytes=None):
    """p4v_mlp_frozen_forward on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    n0 = _lib.launch_count()
    v = lambda a: a and ctypes.c_void_p(a)   # noqa: E731
    rc = lib.p4v_mlp_frozen_forward(
        ctypes.byref(d1), v(x), v(b1), v(p1), _pack_bytes(d1) if bytes1 is None else bytes1,
        ctypes.byref(d2), v(b2), v(p2), _pack_bytes(d2) if bytes2 is None else bytes2,
        v(ws), _ws_bytes(d1, d2) if ws_bytes is None else ws_bytes, v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(p1=0), "null pointer"), (dict(p2=0), "null pointer"), (dict(ws=0), "null pointer"),
    (dict(out=0), "null pointer"), (dict(b1=0), "bias is null"), (dict(b2=0), "bias is null"),
    (dict(rows2=6305, ws_bytes=1 << 30), "same rows"), (dict(fc2_in=1536), "do not fuse"), (dict(fc1_gelu=1), "do not fuse"),
    (dict(bytes1=1024), "packed buffer too small"), (dict(bytes2=1024), "packed buffer too small"),
    (dict(x=4100), "aligned"), (dict(out=(4 << 20) + 4), "aligned"), (dict(ws=(3 << 20) + 8), "aligned"),
    (dict(ws_bytes=1 << 20), "workspace too small"),
])
def test_validation_before_launch(case, match):
    case = dict(case)
    d1, d2 = _vitb(post_gelu=case.pop("fc1_gelu", 0))
    d2.rows = case.pop("rows2", d2.rows)
    if "fc2_in" in case:
        d1.out_features = case.pop("fc2_in")
        d1.n_V = 1
    rc, msg = _call(d1, d2, **case)
    assert rc != 0 and match in msg, msg


def test_workspace_is_fc2s_image():
    # 6304 rows -> 50 row tiles of 128 rows; PTQ4ViT fc2: two planes of 3072 bytes per row, BasePTQ: one
    assert _ws_bytes(*_vitb()) == 50 * 128 * 2 * 3072
    assert _ws_bytes(_desc(768, 3072, n_H=1), _desc(3072, 768, n_H=1)) == 50 * 128 * 3072
    # a 40-column segment is padded to 64 bytes: 200 -> 400 -> 200 with n_H = 4 (segments of 100 -> 128 bytes)
    assert _ws_bytes(_desc(200, 400, n_H=4, rows=5), _desc(400, 200, n_H=4, rows=5)) == 128 * 4 * 128


def test_shape_rule():
    want = [
        (_vitb(), 1),                                                          # ViT-B/224 PTQ4ViT
        ((_desc(768, 3072, n_H=1), _desc(3072, 768, n_H=1)), 1),               # BasePTQ / no_postgelu
        ((_desc(768, 3072, bit=6), _desc(3072, 768, post_gelu=1, bit=6)), 1),  # W6A6
        ((_desc(96, 384, n_H=3), _desc(384, 96, n_H=12, post_gelu=1)), 1),     # Swin-T stage 1 (fc2 fused on its own)
        ((_desc(1024, 4096, n_H=32), _desc(4096, 1024, n_H=32, post_gelu=1)), 1),   # Swin-B/384 stage 4
        ((_desc(200, 400, n_H=4), _desc(400, 200, n_H=4, post_gelu=1)), 1),    # fc2 segments straddle fc1's column tiles
        ((_desc(768, 1536), _desc(3072, 768, post_gelu=1)), 0),                # K mismatch
        (_vitb(post_gelu=1), 0),                                               # post-GELU fc1
        ((_desc(1472, 256, n_H=1), _desc(256, 1472, n_H=1, post_gelu=1)), 0),  # fc1 on the streamed path
    ]
    for (d1, d2), w in want:
        for rows in (1, 6304):              # the rule ignores the rows
            d1.rows = d2.rows = rows
            assert _ok(d1, d2) == w, (d1.in_features, d1.out_features, d2.in_features, d1.post_gelu)


def _frozen_mlp(K=64, H=256):
    """An Mlp whose Linears pass for frozen (frozen modules need a CUDA device: only `frozen` and `mode` are read)."""
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear, PTQSLBatchingQuantLinear
    from ptq4vit_b200.utils.models import Mlp
    m = Mlp(K, H)
    m.fc1 = PTQSLBatchingQuantLinear(K, H, mode="quant_forward", n_H=1)
    m.fc2 = PostGeluPTQSLBatchingQuantLinear(H, K, mode="quant_forward", n_H=1)
    for lin in (m.fc1, m.fc2):
        lin._packed = torch.empty(0, dtype=torch.uint8)
    return m


def test_python_rule():
    from ptq4vit_b200.quant_layers.linear import frozen_mlp_applies
    m = _frozen_mlp()
    x = torch.zeros(4, 64)
    with torch.no_grad():
        assert frozen_mlp_applies(m.fc1, m.fc2, m.act, x)
        assert not frozen_mlp_applies(m.fc1, m.fc2, torch.nn.GELU(approximate="tanh"), x)
        assert not frozen_mlp_applies(m.fc1, m.fc2, torch.nn.ReLU(), x)
        m.fc2.mode = "raw"
        assert not frozen_mlp_applies(m.fc1, m.fc2, m.act, x)
        m.fc2.mode = "quant_forward"
        m.fc1._packed = None
        assert not frozen_mlp_applies(m.fc1, m.fc2, m.act, x)
    m = _frozen_mlp()
    assert not frozen_mlp_applies(m.fc1, m.fc2, m.act, x), "grad mode with parameters that require grad"
    for p in m.parameters():
        p.requires_grad_(False)
    assert frozen_mlp_applies(m.fc1, m.fc2, m.act, x)
    assert not frozen_mlp_applies(m.fc1, m.fc2, m.act, x.requires_grad_())


def _tiny_nets():
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
    vit = VisionTransformer(img_size=32, patch=8, dim=64, depth=2, num_heads=2, num_classes=10)
    swin = SwinTransformer(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)
    return vit, swin


def test_fuse_and_unfuse_bookkeeping():
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Mlp
    for net in _tiny_nets():
        mlps = [(n, m) for n, m in net.named_modules() if isinstance(m, Mlp)]
        assert len(mlps) >= 2
        assert deploy.fuse_mlp(net) == [n for n, _ in mlps], "plain Linears are not frozen"
        assert not any(m.fused for _, m in mlps)
        # freeze both Linears of the first Mlp, only fc1 of the second
        for i, (_, m) in enumerate(mlps[:2]):
            m.fc1 = PTQSLBatchingQuantLinear(m.fc1.in_features, m.fc1.out_features)
            m.fc1._packed = torch.empty(0, dtype=torch.uint8)
            if i == 0:
                m.fc2 = PTQSLBatchingQuantLinear(m.fc2.in_features, m.fc2.out_features)
                m.fc2._packed = torch.empty(0, dtype=torch.uint8)
        assert deploy.fuse_mlp(net) == [n for n, _ in mlps[1:]]
        assert mlps[0][1].fused and not any(m.fused for _, m in mlps[1:])
        assert deploy.fuse_attention(net) != [], "fuse_mlp leaves the attention modules alone"
        deploy.unfuse_mlp(net)
        assert not any(m.fused for _, m in mlps)


def test_never_fused_model_runs_the_plain_code(monkeypatch):
    from ptq4vit_b200.utils import models

    def refuse(*a, **k):
        raise AssertionError("the fused path was consulted")
    monkeypatch.setattr(models, "frozen_mlp_applies", refuse)
    monkeypatch.setattr(models, "frozen_mlp", refuse)
    for net in _tiny_nets():
        with torch.no_grad():
            y = net(torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(0)))
        assert y.shape == (2, 10) and bool(torch.isfinite(y).all())
