"""The qkv fold's host side, without a GPU: the shape rule over every qkv of the zoo and its refusals, the column and row
maps of the planes against torch's reshape, every rejection of the two entry points before anything is launched (null
stream, no device), fuse_qkv / unfuse_qkv bookkeeping, and default forwards that are unchanged."""
import ctypes

import pytest
import torch

from ptq4vit_b200 import _lib
from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear


def _lin(K, O):
    return PTQSLBatchingQuantLinear(K, O, n_V=3, n_H=max(1, K // 64), n_a=max(1, K // 64))


def _attn(tokens, heads, head_dim, batch=1, scale_on_q=0, n_windows=0):
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim, a.scale_on_q, a.n_windows, a.scale = batch, tokens, heads, head_dim, scale_on_q, n_windows, 0.125
    return a


def _ok(lin, tokens, heads, head_dim, gather=0):
    ok = ctypes.c_int(-1)
    _lib.check(_lib.lib().p4v_linear_qkv8_ok(ctypes.byref(lin._desc(1, 1)), ctypes.byref(_attn(tokens, heads, head_dim)), gather,
                                             ctypes.byref(ok)), "p4v_linear_qkv8_ok")
    return ok.value


# (C, heads, tokens, gather): ViT / DeiT Ti/S/B at 224, ViT-S/32; Swin-T/S/B stages 1-4 (window 7), Swin-B/384 (window 12)
ZOO = {"vit_ti": (192, 3, 197, 0), "vit_s": (384, 6, 197, 0), "vit_b": (768, 12, 197, 0), "vit_s32": (384, 6, 50, 0)}
for _name, _C, _H in (("swin_t", 96, 3), ("swin_s", 96, 3), ("swin_b", 128, 4)):
    for _s in range(4):
        ZOO[f"{_name}_s{_s + 1}"] = (_C * 2 ** _s, _H * 2 ** _s, 49, 1)
for _s in range(4):
    ZOO[f"swin_b384_s{_s + 1}"] = (128 * 2 ** _s, 4 * 2 ** _s, 144, 1)


@pytest.mark.parametrize("name", list(ZOO))
def test_rule_holds_over_the_zoo(name):
    C, H, N, gather = ZOO[name]
    assert _ok(_lin(C, 3 * C), N, H, C // H, gather) == 1
    if gather:
        assert _ok(_lin(C, 3 * C), N, H, C // H, 0) == 1


def test_rule_refusals():
    lin = _lin(768, 2304)
    assert _ok(lin, 257, 12, 64) == 0 and _ok(lin, 577, 12, 64) == 0          # the long kernel keeps the FP32 hand-off
    assert _ok(_lin(576, 3 * 576), 197, 8, 72) == 0                             # head_dim 72
    assert _ok(_lin(768, 2304), 197, 6, 64) == 0                                # out_features != 3 C
    assert _ok(_lin(768, 3 * 736), 197, 12, 64) == 0
    streamed = _lin(4096, 3 * 4096)
    path = ctypes.c_int(-1)
    _lib.check(_lib.lib().p4v_linear_frozen_path(ctypes.byref(streamed._desc(1, 1)), ctypes.byref(path)), "path")
    assert path.value == 0
    assert _ok(streamed, 64, 64, 64) == 0                                       # a streamed qkv never folds
    with pytest.raises(_lib.NativeError, match="gather mode"):
        _ok(lin, 197, 12, 64, gather=2)


@pytest.mark.parametrize("B,N,H,D", [(2, 197, 12, 64), (3, 49, 3, 32), (1, 50, 6, 64), (4, 144, 4, 32)])
def test_plane_maps_match_reshape(B, N, H, D):
    """Column c -> (part, h, j) = (c // C, (c % C) // D, c % D) and row r -> (b, n) = (r // N, r % N), the maps of the
    epilogue (forward.cuh FwdQkv8), against reshape(B, N, 3, H, D).permute(2, 0, 3, 1, 4) of index tensors"""
    C = H * D
    rows = torch.arange(B * N).view(B * N, 1).expand(B * N, 3 * C)
    cols = torch.arange(3 * C).view(1, 3 * C).expand(B * N, 3 * C)
    for t, f in ((rows, lambda b, n, p, h, j: b * N + n), (cols, lambda b, n, p, h, j: (p * H + h) * D + j)):
        planes = t.reshape(B, N, 3, H, D).permute(2, 0, 3, 1, 4)
        b, n = torch.meshgrid(torch.arange(B), torch.arange(N), indexing="ij")
        for p in range(3):
            for h in (0, H - 1):
                for j in (0, D - 1):
                    assert torch.equal(planes[p, :, h, :, j], torch.as_tensor(f(b, n, p, h, j)).expand(B, N))
    c = torch.arange(3 * C)
    part, h, j = c // C, (c % C) // D, c % D
    assert torch.equal((part * H + h) * D + j, c)
    # a 16-column group lies in one (part, head)
    g = c.view(-1, 16)
    assert torch.equal((g // C).amin(1), (g // C).amax(1)) and torch.equal((g // D).amin(1), (g // D).amax(1))


def _mm(heads, sos=0, bit=8):
    d = _lib.MatMulDesc()
    d.batch, d.heads, d.S1, d.S2, d.S3, d.A_bit, d.B_bit, d.eq_n, d.search_round, d.sos = 1, heads, 1, 1, 1, bit, bit, 1, 1, sos
    return d


def _pack_bytes(d):
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_matmul_pack_bytes(ctypes.byref(d), ctypes.byref(n)), "pack_bytes")
    return n.value


FAKE = 1 << 36      # 16-byte aligned addresses that are never dereferenced: every rejection comes before a launch


def _qkv8(**kw):
    lin = _lin(768, 2304)
    args = dict(d=lin._desc(2 * 197, 1), x=FAKE, bias=FAKE + (1 << 28), packed=FAKE + (2 << 28), a=_attn(197, 12, 64, batch=2),
                mm1=_mm(12), pack1=FAKE + (3 << 28), b1=None, mm2=_mm(12, sos=1), pack2=FAKE + (4 << 28), b2=None,
                planes=FAKE + (5 << 28), gamma=None, beta=None, eps=0.0, g=None)
    args.update(kw)
    b1 = _pack_bytes(args["mm1"]) if args["b1"] is None else args["b1"]
    b2 = _pack_bytes(args["mm2"]) if args["b2"] is None else args["b2"]
    P = lambda v: None if v is None else ctypes.c_void_p(v)
    rc = _lib.lib().p4v_linear_frozen_forward_qkv8(
        ctypes.byref(args["d"]), P(args["x"]), P(args["bias"]), P(args["packed"]), None if args["a"] is None else ctypes.byref(args["a"]),
        ctypes.byref(args["mm1"]), P(args["pack1"]), b1, ctypes.byref(args["mm2"]), P(args["pack2"]), b2, P(args["planes"]),
        P(args["gamma"]), P(args["beta"]), args["eps"], None if args["g"] is None else ctypes.byref(args["g"]), None)
    return rc, _lib.lib().p4v_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(planes=None), "null pointer"),
    (dict(x=None), "null pointer"),
    (dict(pack1=None), "null pointer"),
    (dict(a=None), "null pointer"),
    (dict(planes=FAKE + 8), "16-byte aligned"),
    (dict(mm1=_mm(6)), "heads"),
    (dict(mm1=_mm(12, sos=1)), "split-of-softmax"),
    (dict(b1=8), "pack sizes"),
    (dict(pack2=FAKE + 4), "16-byte aligned"),
    (dict(a=_attn(197, 12, 48, batch=2)), "do not fold"),
    (dict(a=_attn(197, 6, 128, batch=2), mm1=_mm(6), mm2=_mm(6, sos=1)), "do not fold"),
    (dict(a=_attn(197, 12, 64, batch=3)), "rows"),
    (dict(planes=FAKE + 1024), "overlaps the planes"),
    (dict(gamma=FAKE + (6 << 28), beta=FAKE + (7 << 28), eps=-1.0), "eps"),
    (dict(g=_lib.InputGather(2, _lib.WindowLayout(2, 28, 28, 0, 0))), "gather mode"),
    (dict(g=_lib.InputGather(1, _lib.WindowLayout(2, 14, 14, 7, 0))), "LayerNorm"),
])
def test_forward_rejections_before_launch(kw, msg):
    rc, err = _qkv8(**kw)
    assert rc != 0 and msg in err, err


def _i8(**kw):
    args = dict(a=_attn(197, 12, 64, batch=2), planes=FAKE, mm1=_mm(12), pack1=FAKE + (1 << 28), b1=None, mm2=_mm(12, sos=1),
                pack2=FAKE + (2 << 28), b2=None, bias=None, mask=None, out=FAKE + (3 << 28))
    args.update(kw)
    b1 = _pack_bytes(args["mm1"]) if args["b1"] is None else args["b1"]
    b2 = _pack_bytes(args["mm2"]) if args["b2"] is None else args["b2"]
    P = lambda v: None if v is None else ctypes.c_void_p(v)
    rc = _lib.lib().p4v_attention_frozen_forward_i8(
        ctypes.byref(args["a"]), P(args["planes"]), ctypes.byref(args["mm1"]), P(args["pack1"]), b1, ctypes.byref(args["mm2"]),
        P(args["pack2"]), b2, P(args["bias"]), P(args["mask"]), P(args["out"]), None)
    return rc, _lib.lib().p4v_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(planes=None), "null pointer"),
    (dict(out=None), "null pointer"),
    (dict(planes=FAKE + 4), "planes must be 16-byte aligned"),
    (dict(out=FAKE + (3 << 28) + 4), "8-byte aligned"),
    (dict(a=_attn(577, 12, 64, batch=2)), "tokens"),
    (dict(a=_attn(197, 12, 72, batch=2)), "head_dim"),
    (dict(mm2=_mm(6)), "heads"),
    (dict(mm1=_mm(12, sos=1)), "split-of-softmax"),
    (dict(b2=4), "pack sizes"),
    (dict(mask=FAKE + (4 << 28)), "n_windows"),
    (dict(out=FAKE + 4096), "overlap out"),
])
def test_attention_i8_rejections_before_launch(kw, msg):
    rc, err = _i8(**kw)
    assert rc != 0 and msg in err, err


def test_fuse_qkv_bookkeeping_and_defaults():
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
    from ptq4vit_b200.utils import deploy
    from ptq4vit_b200.utils.models import Attention, SwinTransformer, VisionTransformer, WindowAttention
    for net in (VisionTransformer(img_size=32, patch=8, dim=64, depth=2, num_heads=2, num_classes=10),
                SwinTransformer(img_size=32, patch=4, dim=32, depths=(2, 2), num_heads=(2, 4), window_size=4, num_classes=10)):
        attn = [(n, m) for n, m in net.named_modules() if isinstance(m, (Attention, WindowAttention))]
        assert attn and not any(m.fold_qkv for _, m in attn)
        x = torch.randn(2, 3, 32, 32)
        with torch.no_grad():
            want = net(x)
        # nothing frozen: every attention module is left unfolded
        assert deploy.fuse_qkv(net) == [n for n, _ in attn]
        assert not any(m.fold_qkv for _, m in attn)
        # a frozen qkv with frozen MatMul modules folds; one whose matmul2 is not frozen does not
        for i, (_, m) in enumerate(attn):
            m.qkv = _FrozenStub(m.qkv)
            m.matmul1, m.matmul2 = _FrozenMM(), (_FrozenMM() if i else MinMaxQuantMatMul())
        assert deploy.fuse_qkv(net) == [attn[0][0]]
        assert [m.fold_qkv for _, m in attn] == [False] + [True] * (len(attn) - 1)
        deploy.unfuse_qkv(net)
        assert not any(m.fold_qkv for _, m in attn)
        for _, m in attn:
            m.qkv = m.qkv.inner
            m.matmul1 = m.matmul2 = None
        from ptq4vit_b200.utils.models import MatMul
        for _, m in attn:
            m.matmul1, m.matmul2 = MatMul(), MatMul()
        with torch.no_grad():
            assert torch.equal(net(x), want), "the default forward is unchanged"


class _FrozenStub(PTQSLBatchingQuantLinear):
    """A Linear that reports itself frozen (bookkeeping only: never run)"""

    def __init__(self, inner):
        super().__init__(inner.in_features, inner.out_features)
        self.inner = inner
        self._packed = torch.zeros(1, dtype=torch.uint8)


class _FrozenMM(torch.nn.Module):
    pass


def _frozen_mm():
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul
    m = MinMaxQuantMatMul()
    m._packed = {1: torch.zeros(1, dtype=torch.uint8)}
    return m


_FrozenMM = _frozen_mm
