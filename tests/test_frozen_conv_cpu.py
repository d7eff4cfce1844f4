"""The frozen patch-embedding convolution without a GPU: the shape rule (C ABI and the module's geometry), every
rejection of p4v_conv_pack / p4v_conv_frozen_forward before any launch, freeze()'s errors, and the deploy bookkeeping of
conv modules (defaults unchanged, a conv entry without integers, step sizes round-tripped)."""
import ctypes
import inspect

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


VIT_B = dict(images=32, in_channels=3, height=224, width=224, out_channels=768, kernel_h=16, kernel_w=16, w_bit=8,
             layerwise=0, has_bias=1)


def _desc(**kw):
    from ptq4vit_b200 import _lib
    d = _lib.ConvFrozenDesc()
    base = dict(VIT_B)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _ok(lib, **kw):
    ok = ctypes.c_int(-1)
    assert lib.p4v_conv_frozen_ok(ctypes.byref(_desc(**kw)), ctypes.byref(ok)) == 0
    return ok.value


def _pack_bytes(lib, **kw):
    n = ctypes.c_size_t()
    assert lib.p4v_conv_pack_bytes(ctypes.byref(_desc(**kw)), ctypes.byref(n)) == 0, lib.p4v_last_error()
    return n.value


@pytest.mark.parametrize("kw,ok", [
    (dict(), 1),
    (dict(in_channels=3, kernel_h=4, kernel_w=4, out_channels=96), 1),              # Swin-T
    (dict(in_channels=3, kernel_h=32, kernel_w=32, out_channels=384), 1),           # ViT-S/32: K = 3072
    (dict(in_channels=16, kernel_h=16, kernel_w=16), 1),                            # K = 4096
    (dict(in_channels=17, kernel_h=16, kernel_w=16), 0),                            # K = 4352
    (dict(out_channels=4096), 1), (dict(out_channels=4097), 0), (dict(out_channels=0), 0),
    (dict(in_channels=0), 0), (dict(kernel_h=0), 0), (dict(kernel_w=0), 0),
    (dict(w_bit=1), 0), (dict(w_bit=2), 1), (dict(w_bit=9), 0),
    (dict(layerwise=2), 0), (dict(has_bias=-1), 0),
    (dict(images=0, height=0, width=0), 1),                                         # not part of the rule
])
def test_shape_rule(lib, kw, ok):
    assert _ok(lib, **kw) == ok


def test_pack_bytes_do_not_depend_on_the_input(lib):
    n = _pack_bytes(lib)
    assert n == 768 * 4 + 6 * 24 * 128 * 32 * 2          # step sizes, then 6 channel tiles x 24 K slabs of bf16
    assert _pack_bytes(lib, images=1, height=384, width=384) == n
    assert _pack_bytes(lib, layerwise=1, has_bias=0, w_bit=6) == n
    assert _pack_bytes(lib, in_channels=3, kernel_h=4, kernel_w=4, out_channels=96) == 512 + 1 * 2 * 8192


def _forward(lib, d=None, x=1 << 20, bias=2 << 20, packed=3 << 20, out=4 << 20, packed_bytes=None):
    """p4v_conv_frozen_forward on made-up device addresses: every case here must fail validation, never launch."""
    from ptq4vit_b200 import _lib
    d = _desc() if d is None else d
    n0 = _lib.launch_count()
    v = lambda a: a and ctypes.c_void_p(a)   # noqa: E731
    if packed_bytes is None:
        n = ctypes.c_size_t(0)
        lib.p4v_conv_pack_bytes(ctypes.byref(d), ctypes.byref(n))
        packed_bytes = n.value
    rc = lib.p4v_conv_frozen_forward(ctypes.byref(d), v(x), v(bias), v(packed), packed_bytes, v(out), None)
    assert _lib.launch_count() == n0
    return rc, lib.p4v_last_error().decode()


@pytest.mark.parametrize("case,match", [
    (dict(x=0), "null pointer"), (dict(packed=0), "null pointer"), (dict(out=0), "null pointer"),
    (dict(bias=0), "bias is null"),
    (dict(d=dict(images=0)), "bad geometry"), (dict(d=dict(height=15)), "bad geometry"), (dict(d=dict(width=8)), "bad geometry"),
    (dict(d=dict(out_channels=0)), "empty"), (dict(d=dict(in_channels=17)), "K = in_channels"),
    (dict(d=dict(out_channels=5000)), "out_channels above 4096"), (dict(d=dict(w_bit=9)), "w_bit"),
    (dict(d=dict(layerwise=3)), "must be 0 or 1"),
    (dict(d=dict(images=1 << 20, height=4096, width=4096)), "too large"),
    (dict(packed_bytes=1000), "packed buffer too small"),
    (dict(packed=(3 << 20) + 8), "aligned"), (dict(x=(1 << 20) + 2), "aligned"), (dict(out=(4 << 20) + 1), "aligned"),
    (dict(bias=(2 << 20) + 2), "aligned"),
])
def test_forward_rejects_before_any_launch(lib, case, match):
    case = dict(case)
    if "d" in case:
        case["d"] = _desc(**case["d"])
        if "packed_bytes" not in case:
            case["packed_bytes"] = 1 << 30
    rc, msg = _forward(lib, **case)
    assert rc != 0 and match in msg and msg.startswith("conv_frozen_forward"), msg


def test_forward_without_bias_needs_no_bias_pointer(lib):
    rc, msg = _forward(lib, d=_desc(has_bias=0, images=0), bias=0)
    assert rc != 0 and "bad geometry" in msg       # validation got past the bias check


@pytest.mark.parametrize("case,match", [
    (dict(weight=0), "null pointer"), (dict(wi=0), "null pointer"), (dict(packed=0), "null pointer"),
    (dict(packed_bytes=8192), "packed buffer too small"), (dict(packed=(3 << 20) + 4), "aligned"),
    (dict(d=dict(kernel_w=0)), "empty"), (dict(d=dict(w_bit=1)), "w_bit"),
])
def test_pack_rejects_before_any_launch(lib, case, match):
    from ptq4vit_b200 import _lib
    d = _desc(**case.get("d", {}))
    v = lambda a: a and ctypes.c_void_p(a)   # noqa: E731
    n0 = _lib.launch_count()
    rc = lib.p4v_conv_pack(ctypes.byref(d), v(case.get("weight", 1 << 20)), v(case.get("wi", 2 << 20)),
                           v(case.get("packed", 3 << 20)), case.get("packed_bytes", 1 << 30), None)
    msg = lib.p4v_last_error().decode()
    assert rc != 0 and match in msg and msg.startswith("conv_pack"), msg
    assert _lib.launch_count() == n0


def test_null_descriptors(lib):
    ok, n = ctypes.c_int(), ctypes.c_size_t()
    assert lib.p4v_conv_frozen_ok(None, ctypes.byref(ok)) != 0
    assert lib.p4v_conv_pack_bytes(None, ctypes.byref(n)) != 0 and "null desc" in lib.p4v_last_error().decode()
    assert lib.p4v_conv_pack_bytes(ctypes.byref(_desc()), None) != 0


def _conv(cls="ChannelwiseBatchingQuantConv2d", cin=3, cout=768, k=16, calibrated=True, **kw):
    from ptq4vit_b200.quant_layers import conv as CV
    args = dict(stride=k, a_bit=32, w_bit=8)
    args.update(kw)
    m = getattr(CV, cls)(cin, cout, k, **args)
    if calibrated:
        layerwise = cls == "BatchingEasyQuantConv2d"
        m.w_interval = torch.full((1 if layerwise else cout, 1, 1, 1), 0.01)
        m.a_interval = torch.full((1,), 0.02)
        m.calibrated = True
    return m


@pytest.mark.parametrize("kw,match", [
    (dict(), None), (dict(cls="BatchingEasyQuantConv2d"), None), (dict(k=4, cout=96), None), (dict(k=32, cout=384), None),
    (dict(stride=8), "stride"), (dict(padding=1), "padding"), (dict(padding="same", stride=1, k=1), "stride|padding"),
    (dict(dilation=2), "dilation"), (dict(groups=3, cout=96), "groups"), (dict(a_bit=8), "a_bit"),
    (dict(cin=17), "shape rule"), (dict(cout=4097), "shape rule"), (dict(w_bit=9), "shape rule"),
])
def test_module_geometry_rule(lib, kw, match):
    import re
    m = _conv(**kw)
    why = m.frozen_unsupported()
    if match is None:
        assert why is None, why
    else:
        assert why is not None and re.search(match, why), why


def test_freeze_errors():
    m = _conv(calibrated=False)
    with pytest.raises(RuntimeError, match="calibrated"):
        m.freeze()
    m = _conv()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.freeze()
    for bad in (dict(a_bit=8), dict(stride=8)):
        with pytest.raises(NotImplementedError):
            _conv(**bad).freeze()
    assert not m.frozen


def test_unfrozen_quant_forward_is_unchanged():
    """A module that was never frozen runs the torch operations of quant_forward."""
    import torch.nn.functional as F
    m = _conv(cin=3, cout=16, k=4).eval()
    x = torch.randn(2, 3, 8, 8)
    with torch.no_grad():
        w_sim, b = m.quant_weight_bias()
        assert torch.equal(m.quant_forward(x), F.conv2d(x, w_sim, b, 4))


def test_deploy_defaults():
    from ptq4vit_b200.utils import deploy
    for fn, name in ((deploy.freeze_model, "conv"), (deploy.freeze_model, "matmul"), (deploy.load_quantized, "conv"),
                     (deploy.load_quantized, "matmul")):
        assert inspect.signature(fn).parameters[name].default is False
    wrapped = {"patch_embed.proj": _conv(cout=32), "uncalibrated": _conv(cout=32, calibrated=False)}
    assert deploy.freeze_model(wrapped) == ["patch_embed.proj", "uncalibrated"]
    assert deploy.freeze_model(wrapped, conv=True) == ["patch_embed.proj", "uncalibrated"]    # CPU modules
    deploy.unfreeze_model(wrapped)
    assert not any(m.frozen for m in wrapped.values())


@pytest.mark.parametrize("conv", [False, True])
def test_save_load_round_trips_conv_step_sizes(tmp_path, conv):
    """CPU modules: the file has step sizes and no integers; conv=True then leaves the conv entries unfrozen."""
    from ptq4vit_b200.utils import deploy
    g = torch.Generator().manual_seed(2)

    def modules():
        return {"patch_embed.proj": _conv(cout=96, k=4, calibrated=False),
                "other.proj": _conv("BatchingEasyQuantConv2d", cout=32, k=8, calibrated=False)}
    src = modules()
    for m in src.values():
        n = 1 if type(m).__name__ == "BatchingEasyQuantConv2d" else m.out_channels
        m.w_interval = torch.rand(n, 1, 1, 1, generator=g)
        m.a_interval = torch.rand(1, generator=g)
        m.calibrated = True
    path = str(tmp_path / "q.pt")
    deploy.save_quantized(src, path)
    state = torch.load(path, weights_only=True)
    assert all("w_int" not in e for e in state["modules"].values())
    dst = modules()
    left = deploy.load_quantized(dst, path, conv=conv)
    assert sorted(left) == sorted(dst)
    for name, m in src.items():
        assert dst[name].calibrated and not dst[name].frozen
        for k in ("w_interval", "a_interval"):
            a, b = getattr(m, k), getattr(dst[name], k)
            assert torch.equal(a, b) and a.shape == b.shape
