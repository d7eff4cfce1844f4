"""No-GPU checks of the frozen Linear forward: host planning of the packed buffer and of the fused / streamed choice,
argument validation, and the step-size part of save_quantized / load_quantized (no kernel is launched here)."""
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
    d = _lib.LinearDesc()
    base = dict(rows=6304, tokens=1, in_features=768, out_features=2304, n_V=72, n_H=24, n_a=1, w_bit=8, a_bit=8,
                eq_n=1, search_round=1, eq_alpha=0.0, eq_beta=1.0, post_gelu=0, has_bias=1, operand=0, kernel=0)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _pack_bytes(lib, **kw):
    n = ctypes.c_size_t()
    assert lib.p4v_linear_pack_bytes(ctypes.byref(_desc(**kw)), ctypes.byref(n)) == 0, lib.p4v_last_error()
    return n.value


def _path(lib, **kw):
    p = ctypes.c_int(-1)
    assert lib.p4v_linear_frozen_path(ctypes.byref(_desc(**kw)), ctypes.byref(p)) == 0, lib.p4v_last_error()
    return p.value


def _ws(lib, **kw):
    n = ctypes.c_size_t(1)
    assert lib.p4v_linear_frozen_workspace_bytes(ctypes.byref(_desc(**kw)), ctypes.byref(n)) == 0, lib.p4v_last_error()
    return n.value


VIT_B = dict(qkv=dict(), proj=dict(out_features=768, n_V=24), fc1=dict(out_features=3072, n_V=24),
             head=dict(out_features=1000, n_V=1, rows=32),
             fc2=dict(in_features=3072, out_features=768, n_V=24, post_gelu=1))


def test_pack_bytes_do_not_depend_on_rows_and_are_close_to_the_int8_weight(lib):
    n = _pack_bytes(lib)
    assert all(_pack_bytes(lib, rows=r) == n for r in (1, 197, 128, 100000))
    weight, scales = 2304 * 768, 24 * (2304 // 16) * 4
    assert weight + scales <= n <= 1.03 * (weight + scales)
    # the head's 1000 outputs are padded to 8 tiles of 128 rows
    assert 1024 * 768 <= _pack_bytes(lib, **VIT_B["head"]) <= 1.03 * 1024 * 768 + 24 * 64 * 4 + 8192


@pytest.mark.parametrize("bad,msg", [
    (dict(n_H=7), "divide"), (dict(w_bit=9), "bit"), (dict(out_features=120, n_V=5), "multiple of 16"),
    (dict(in_features=4096, n_H=128, n_a=1), "too many K segments for quant_forward"),
])
def test_bad_descriptors_fail_with_the_forward_messages(lib, bad, msg):
    n, p = ctypes.c_size_t(), ctypes.c_int()
    for call, out in ((lib.p4v_linear_pack_bytes, n), (lib.p4v_linear_frozen_path, p), (lib.p4v_linear_frozen_workspace_bytes, n)):
        assert call(ctypes.byref(_desc(**bad)), ctypes.byref(out)) != 0
        assert msg in lib.p4v_last_error().decode()
    # the unfrozen forward rejects the same descriptor with the same message
    assert lib.p4v_linear_quant_forward_workspace_bytes(ctypes.byref(_desc(**bad)), ctypes.byref(n)) != 0
    assert msg in lib.p4v_last_error().decode()


def test_fused_and_streamed_paths(lib):
    for name in ("qkv", "proj", "fc1", "head"):
        assert _path(lib, **VIT_B[name]) == 1, name
        assert _ws(lib, **VIT_B[name]) == 0, name
    # BasePTQ: one block per layer
    assert _path(lib, n_H=1, n_V=3) == 1
    # Swin-T: K = 96 ... 768, post-GELU fc2 of the first stages included
    for K in (96, 192, 384, 768):
        assert _path(lib, in_features=K, out_features=K, n_V=1, n_H=K // 32, rows=3136) == 1
    assert _path(lib, in_features=384, out_features=96, n_V=1, n_H=12, post_gelu=1) == 1
    # ViT-B fc2: 3072 inputs in two parts do not fit shared memory: one int8 activation image of all rows
    fc2 = VIT_B["fc2"]
    assert _path(lib, **fc2) == 0
    assert _ws(lib, **fc2) == 50 * 128 * 2 * 3072
    assert _ws(lib, rows=197, **fc2) == 2 * 128 * 2 * 3072
    # the path is a function of the layer, not of the batch
    assert _path(lib, rows=1) == _path(lib, rows=100000) == 1
    # the boundary: the tile (128 rows x K bytes) beside two 16 KB stages and the control block
    assert _path(lib, in_features=1440, out_features=256, n_V=1, n_H=1) == 1
    assert _path(lib, in_features=1472, out_features=256, n_V=1, n_H=1) == 0


def test_null_pointers_are_rejected_before_any_launch(lib):
    d = _desc()
    assert lib.p4v_linear_pack(ctypes.byref(d), None, None, None, None, 0, None) != 0
    assert "null" in lib.p4v_last_error().decode()
    assert lib.p4v_linear_frozen_forward(ctypes.byref(d), None, None, None, None, 0, None, None) != 0
    assert "null" in lib.p4v_last_error().decode()


def test_freeze_needs_a_calibrated_cuda_module():
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    m = PTQSLBatchingQuantLinear(32, 32, metric="hessian", eq_n=10)
    with pytest.raises(RuntimeError, match="calibrated"):
        m.freeze()
    m.w_interval, m.a_interval, m.calibrated = torch.full((1, 1, 1, 1), 0.01), torch.full((1, 1), 0.02), True
    with pytest.raises(RuntimeError, match="CUDA"):
        m.freeze()
    assert not m.frozen


def test_save_load_round_trips_step_sizes(tmp_path):
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLQuantLinear, PTQSLBatchingQuantLinear
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul
    from ptq4vit_b200.utils import deploy
    g = torch.Generator().manual_seed(1)

    def modules():
        return {"blocks.0.attn.qkv": PTQSLBatchingQuantLinear(64, 96, n_V=3, n_H=2, n_a=1),
                "blocks.0.mlp.fc2": PostGeluPTQSLQuantLinear(128, 64, n_V=1, n_H=4, n_a=1),
                "blocks.0.attn.matmul2": PTQSLBatchingQuantMatMul()}
    src = modules()
    src["blocks.0.attn.qkv"].w_interval = torch.rand(3, 1, 2, 1, generator=g)
    src["blocks.0.attn.qkv"].a_interval = torch.rand(1, 1, generator=g)
    src["blocks.0.mlp.fc2"].w_interval = torch.rand(1, 1, 4, 1, generator=g)
    src["blocks.0.mlp.fc2"].a_interval = [torch.rand(1, 1, generator=g), 0.16997124254703522 / 128]
    src["blocks.0.attn.matmul2"].A_interval = torch.rand(1, 3, 1, 1, 1, 1, 1, generator=g)
    src["blocks.0.attn.matmul2"].B_interval = torch.rand(1, 3, 1, 1, 1, 1, 1, generator=g)
    src["blocks.0.attn.matmul2"].split = torch.tensor(0.0078125)
    path = str(tmp_path / "q.pt")
    deploy.save_quantized(src, path)
    dst = modules()
    left = deploy.load_quantized(dst, path)
    assert sorted(left) == sorted(dst)            # CPU modules: step sizes only, nothing to freeze
    for name, m in src.items():
        assert dst[name].calibrated
        for k in deploy.INTERVALS:
            a, b = getattr(m, k, None), getattr(dst[name], k, None)
            if a is None:
                continue
            if isinstance(a, list):
                assert torch.equal(a[0], b[0]) and a[1] == b[1]
            else:
                assert torch.equal(a, b) and a.shape == b.shape
    with pytest.raises(RuntimeError, match="modules differ"):
        deploy.load_quantized({"other": src["blocks.0.attn.qkv"]}, path)
