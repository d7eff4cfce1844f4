"""No-GPU checks of the frozen MatMul forward: the size of the packed buffer, argument validation before any launch, and
freeze() refusing modules it cannot freeze (no kernel is launched here)."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


def _desc(**kw):
    from ptq4vit_b200 import _lib
    d = _lib.MatMulDesc()
    base = dict(batch=32, heads=12, S1=197, S2=64, S3=197, A_bit=8, B_bit=8, eq_n=1, search_round=1, eq_alpha=0.0,
                eq_beta=1.0, sos=0, operand=0, kernel=0, init_layerwise=0, images_per_chunk=0)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _pack_bytes(lib, **kw):
    n = ctypes.c_size_t()
    assert lib.p4v_matmul_pack_bytes(ctypes.byref(_desc(**kw)), ctypes.byref(n)) == 0, lib.p4v_last_error()
    return n.value


def test_pack_bytes_depend_on_heads_and_sos_only(lib):
    n = _pack_bytes(lib)
    assert all(_pack_bytes(lib, batch=b, S1=s, S2=s, S3=s) == n for b in (1, 7, 1024) for s in (1, 49, 197, 577))
    # [dA][dB][split][aux][scale][group meta], each region 256-byte aligned
    assert n == 6 * 256
    assert _pack_bytes(lib, sos=1) == 6 * 256
    assert _pack_bytes(lib, heads=100, sos=1) == 2 * 512 + 3 * 256 + 1024


def _strides(*s):
    return (ctypes.c_longlong * 4)(*s)


# element strides of the ViT-B/224 q view ([32, 197, 3, 12, 64] qkv output permuted) and of k^T, v
Q = (197 * 2304, 64, 2304, 1)
KT = (197 * 2304, 64, 1, 2304)
V = (197 * 2304, 64, 2304, 1)


def _forward(lib, d, A=0x1000, sA=Q, B=0x2000, sB=KT, packed=0x3000, out=0x4000):
    rc = lib.p4v_matmul_frozen_forward(ctypes.byref(d), ctypes.c_void_p(A) if A else None, _strides(*sA) if sA else None,
                                       ctypes.c_void_p(B) if B else None, _strides(*sB) if sB else None,
                                       ctypes.c_void_p(packed) if packed else None, ctypes.c_void_p(out) if out else None, None)
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("bad,msg", [
    (dict(d=dict(A_bit=9)), "bit widths"), (dict(d=dict(B_bit=1)), "bit widths"),
    (dict(d=dict(S2=0)), "empty shape"), (dict(d=dict(batch=0)), "empty shape"),
    (dict(sA=(197 * 2304, 64, 1, 2304)), "A must have unit stride along K"),
    (dict(sB=(197 * 2304, 64, 2304, 3)), "B must have unit stride along K or along N"),
    (dict(sA=(-1, 64, 2304, 1)), "negative stride"),
    (dict(A=0x1002), "4-byte aligned"), (dict(out=0x4001), "4-byte aligned"), (dict(packed=0x3004), "16-byte aligned"),
    (dict(A=0), "null"), (dict(sB=None), "null"), (dict(packed=0), "null"), (dict(out=0), "null"),
])
def test_bad_arguments_are_rejected_before_any_launch(lib, bad, msg):
    from ptq4vit_b200 import _lib
    d = _desc(**bad.pop("d", {}))
    n0 = _lib.launch_count()
    rc, err = _forward(lib, d, **bad)
    assert rc != 0 and msg in err, err
    assert _lib.launch_count() == n0


def test_bad_descriptors_fail_pack_with_the_forward_messages(lib):
    n = ctypes.c_size_t()
    for bad, msg in ((dict(A_bit=9), "bit widths"), (dict(heads=0), "empty shape")):
        assert lib.p4v_matmul_pack_bytes(ctypes.byref(_desc(**bad)), ctypes.byref(n)) != 0
        assert msg in lib.p4v_last_error().decode()
        assert lib.p4v_matmul_quant_forward_workspace_bytes(ctypes.byref(_desc(**bad)), ctypes.byref(n)) != 0
        assert msg in lib.p4v_last_error().decode()
    assert lib.p4v_matmul_pack(ctypes.byref(_desc()), None, None, None, None, 0, None) != 0
    assert "null" in lib.p4v_last_error().decode()
    assert lib.p4v_matmul_pack(ctypes.byref(_desc(sos=1)), ctypes.c_void_p(0x1000), ctypes.c_void_p(0x2000), None,
                               ctypes.c_void_p(0x3000), 4096, None) != 0          # sos needs split
    assert "null" in lib.p4v_last_error().decode()


def test_freeze_needs_a_calibrated_cuda_module():
    from ptq4vit_b200.quant_layers.matmul import MinMaxQuantMatMul, PTQSLBatchingQuantMatMul, SoSPTQSLBatchingQuantMatMul
    for m in (PTQSLBatchingQuantMatMul(), SoSPTQSLBatchingQuantMatMul(), MinMaxQuantMatMul()):
        with pytest.raises(RuntimeError, match="calibrated"):
            m.freeze()
        m.A_interval = m.B_interval = torch.full((1, 3, 1, 1, 1, 1, 1), 0.01)
        m.split = torch.tensor(0.01)
        m.calibrated = True
        with pytest.raises(RuntimeError, match="CUDA"):
            m.freeze()
        assert not m.frozen


def test_freeze_model_leaves_matmul_modules_by_default():
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul
    from ptq4vit_b200.utils import deploy
    m = PTQSLBatchingQuantMatMul()
    m.calibrated = True
    assert deploy.freeze_model({"blocks.0.attn.matmul1": m}) == ["blocks.0.attn.matmul1"] and not m.frozen
