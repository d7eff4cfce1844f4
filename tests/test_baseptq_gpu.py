"""BasePTQ on the H100: the layer-wise patch-embedding search and every BasePTQ layer type against the UNMODIFIED
reference on the same GPU (or the oracle on the device where the reference is not staged), the fp64 replay at the
BasePTQ shapes with the kernel path each case takes, the public calibrator under ptq4vit_b200.configs.BasePTQ against
the reference's calibrator with its configs/BasePTQ.py, the integer export, and the default (cosine) metric."""
import importlib
import os

import numpy as np
import pytest
import torch

os.environ.setdefault("TQDM_DISABLE", "1")

from oracle import ptq_oracle as O
from oracle import ref_harness as RH
from tests import _baseptq_ref as B
from tests import _cases as C
from tests import _fp64_ref as R
from tests.test_calibrator_gpu import TINY_SWIN, _as_dict, _count_diff
from tests.test_fp64_parity_gpu import _observed, _profiled, _record
from tests.test_reference_gpu import SCORE_RTOL, TIE_EPS, FLIP_FRAC, _compare_steps

pytestmark = pytest.mark.gpu
IMGS, TOK, D, HEADS = 32, 197, 768, 12
GOLD_CONV = os.path.join(C.GOLD, "conv_easy_small.npz")
GOLD_CALIB = os.path.join(C.GOLD, "calib_tiny_vit_baseptq.npz")


# ---------------------------------------------------------------------------------------- layer-wise patch embedding
def _ours_conv(x, W, b, y, g, stride, w_bit=8, eq_alpha=0.5):
    from ptq4vit_b200.quant_layers.conv import BatchingEasyQuantConv2d
    oc, ic, kh, kwid = W.shape
    m = BatchingEasyQuantConv2d(ic, oc, (kh, kwid), stride=stride, bias=b is not None, a_bit=32, w_bit=w_bit,
                                metric="hessian", eq_alpha=eq_alpha, eq_beta=1.2, eq_n=100, search_round=1)
    m.weight.data = W.clone()
    if b is not None:
        m.bias.data = b.clone()
    m.cuda(); m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x.cuda(), y.cuda(), g.cuda()
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    return m


def _check_conv(m, ref_w, ref_table, x, W, b, stride, w_bit, what):
    got = m.last_scores[0].cpu().numpy().astype(np.float64).reshape(-1)
    ref = np.asarray(ref_table, dtype=np.float64).reshape(-1)
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < SCORE_RTOL, f"{what}: score table differs by {err:.2e} of its maximum"
    assert m.w_interval.shape == (1, 1, 1, 1) and m.a_interval.shape == (1,) and m.calibrated
    assert not hasattr(m, "raw_input") and not hasattr(m, "raw_out") and not hasattr(m, "raw_grad")
    pg, pr = int(got.argmax()), int(ref.argmax())
    rw = torch.as_tensor(ref_w).float().reshape(1, 1, 1, 1)
    if pg == pr:
        assert np.array_equal(m.w_interval.cpu().numpy().view(np.uint32), rw.numpy().view(np.uint32)), what
    else:
        gap = (ref[pr] - ref[pg]) / abs(ref[pr])
        assert gap < TIE_EPS, f"{what}: picked {pg}, reference {pr}, reference gap {gap:.2e}"
    # quantized forward on the reference's step size (conv.py:353-363; fp32 convolution)
    m.w_interval = rw.cuda()
    m.mode = "quant_forward"
    with torch.no_grad(), RH.fp32_convolutions():
        out = m(x[:2].cuda()).cpu()
        w_sim = (W / rw).round_().clamp_(-2 ** (w_bit - 1), 2 ** (w_bit - 1) - 1).mul_(rw)
        ref_out = torch.nn.functional.conv2d(x[:2].cuda(), w_sim.cuda(), None if b is None else b.cuda(), stride=stride).cpu()
    o_err = float((out - ref_out).abs().max() / ref_out.abs().max())
    assert o_err < 1e-5, f"{what}: quantized output differs by {o_err:.2e}"
    return err, pg != pr


def test_layerwise_conv_matches_cpu_golden(monkeypatch):
    monkeypatch.setenv("P4V_SCALAR_DIV", "ieee")     # the golden comes from the reference on the CPU (IEEE division)
    z = np.load(GOLD_CONV)
    x, W, b, y, g = O.make_conv_fixture(37, 4, 3, 32, 16, 4)
    m = _ours_conv(x, W, b, y, g, stride=4)
    _check_conv(m, z["w_interval"], z["scores_000"], x, W, b, 4, 8, "conv_easy_small")


# name: (images, ic, oc, size, kernel = stride, w_bit)
CONV = {"vitb224_w8": (IMGS, 3, 768, 224, 16, 8), "vitb224_w6": (IMGS, 3, 768, 224, 16, 6),
        "swin_patch4_w8": (IMGS, 3, 96, 224, 4, 8)}


@pytest.mark.parametrize("name", list(CONV))
def test_layerwise_patch_embedding_matches_reference_on_gpu(name):
    n, ic, oc, size, k, bit = CONV[name]
    x, W, b, y, g = O.make_conv_fixture(400 + bit + k, n, ic, oc, size, k)
    if RH.available():
        ref = B.run_conv_layerwise(x, W, b, y, g, stride=k, w_bit=bit, search_round=1)
        assert len(ref["scores"]) == 1
        ref_w, ref_table, kind, ref_s = ref["w_interval"], ref["scores"][0].numpy(), "reference", ref["seconds"]
    else:
        with RH.fp32_convolutions():
            wi, sc = B.conv_layerwise_calibrate(W.cuda(), b.cuda(), x.cuda(), y.cuda(), g.cuda(), stride=k, w_bit=bit)
        ref_w, ref_table, kind, ref_s = wi.cpu(), sc.cpu().numpy(), "oracle-on-device", float("nan")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    m = _ours_conv(x, W, b, y, g, stride=k, w_bit=bit)
    e1.record(); torch.cuda.synchronize()
    err, flip = _check_conv(m, ref_w, ref_table, x, W, b, k, bit, name)
    print(f"[baseptq conv] {name} ({kind}): score err {err:.2e}, pick {'near-tie' if flip else 'equal'}; "
          f"reference {ref_s:.2f}s vs ours {e0.elapsed_time(e1):.1f} ms (incl. copies)")


# --------------------------------------------------------------------------------- every BasePTQ layer type, ViT-B
LINEAR = {"qkv": (D, 3 * D, 3, False, TOK), "proj": (D, D, 1, False, TOK), "fc1": (D, 4 * D, 1, False, TOK),
          "fc2": (4 * D, D, 1, True, TOK), "head": (D, 1000, 1, False, 0)}


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("name", list(LINEAR))
def test_baseptq_linear_matches_reference_on_gpu(name, bit):
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    K, Oo, n_V, gelu_input, tok = LINEAR[name]
    x, W, b, y, g = O.make_linear_fixture(500 + bit + len(name), IMGS, tok, K, Oo, post_gelu=gelu_input)
    mod = dict(n_V=n_V, n_H=1, n_a=1, w_bit=bit, a_bit=bit, search_round=1, eq_alpha=0.5)
    if RH.available():
        ref = RH.run_linear(x, W, b, y, g, post_gelu=False, quant_forward=True, **mod)
        ref_tables = [s.numpy() for s in ref["scores"]]
        ref_w, ref_a, ref_out = ref["w_interval"], ref["a_interval"], ref["out"]
    else:
        sp = O.LinearSpec(K, Oo, n_V=n_V, n_H=1, n_a=1, w_bit=bit, a_bit=bit, eq_alpha=0.5, eq_n=100, search_round=1)
        xd, Wd, bd, yd, gd = [t.cuda() for t in (x, W, b, y, g)]
        ref_w, ref_a, log = O.linear_calibrate(sp, Wd, bd, xd, yd, gd, return_scores=True)
        ref_tables = [s.cpu().numpy() for s in log[0][0]] + [s.cpu().numpy() for s in log[0][1]]
        ref_out = O.linear_quant_forward(sp, Wd, bd, xd[:2], ref_w, ref_a).cpu()
        ref_w, ref_a = ref_w.cpu(), ref_a.cpu()
    m = PTQSLBatchingQuantLinear(K, Oo, metric="hessian", eq_beta=1.2, eq_n=100, **mod)
    m.weight.data = W.clone(); m.bias.data = b.clone(); m.cuda(); m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x.cuda(), y.cuda(), g.cuda()
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    flips, worst, compared = _compare_steps(f"{name}/W{bit}A{bit}", [s.cpu().numpy() for s in m.last_scores], ref_tables,
                                            group_independent_until=1)
    w_err = float((m.w_interval.cpu().reshape(-1) - ref_w.reshape(-1)).abs().max() / ref_w.abs().max())
    a_err = float((m.a_interval.cpu().reshape(-1) - ref_a.reshape(-1)).abs().max() / ref_a.abs().max())
    if flips == 0:
        assert w_err < 1e-6 and a_err < 1e-6, f"{name}: step sizes differ without a differing pick ({w_err:.2e}, {a_err:.2e})"
    else:
        assert flips <= max(1, int(FLIP_FRAC * n_V)), f"{name}: {flips} near-tie picks differ"
    m.w_interval, m.a_interval = ref_w.cuda().view(n_V, 1, 1, 1), ref_a.cuda().view(1, 1)
    m.mode = "quant_forward"
    with torch.no_grad():
        out = m(x[:2].cuda()).cpu()
    o_err = float((out - ref_out).abs().max() / ref_out.abs().max())
    assert o_err < 1e-3, f"{name}: quantized layer output differs by {o_err:.3e}"
    print(f"[baseptq parity] {name} W{bit}A{bit}: flips {flips}/{compared}, worst score err {worst:.2e}, out {o_err:.1e}")


@pytest.mark.parametrize("bit", [8, 6])
@pytest.mark.parametrize("name", ["matmul1", "matmul2"])
def test_baseptq_matmul_matches_reference_on_gpu(name, bit):
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul
    softmax_A = name == "matmul2"                        # plain class on the post-softmax operand (no split-of-softmax)
    S2, S3 = (TOK, D // HEADS) if softmax_A else (D // HEADS, TOK)
    A, Bm, Y, G = O.make_matmul_fixture(600 + bit + softmax_A, IMGS, HEADS, TOK, S2, S3, softmax_A=softmax_A)
    mod = dict(A_bit=bit, B_bit=bit, search_round=1, eq_alpha=0.5)
    if RH.available():
        ref = RH.run_matmul(A, Bm, Y, G, sos=False, **mod)
        ref_tables = [s.numpy() for s in ref["scores"]]
        ref_A, ref_B, ref_out = ref["A_interval"], ref["B_interval"], ref["out"]
    else:
        sp = O.MatMulSpec(A_bit=bit, B_bit=bit, eq_alpha=0.5, eq_n=100, search_round=1, sos=False)
        Ad, Bd, Yd, Gd = [t.cuda() for t in (A, Bm, Y, G)]
        ref_A, ref_B, _, log = O.matmul_calibrate(sp, Ad, Bd, Yd, Gd, return_scores=True)
        ref_tables = [log[0][0].cpu().numpy(), log[0][1].cpu().numpy()]
        ref_out = O.matmul_quant_forward(sp, Ad[:2], Bd[:2], ref_A, ref_B).cpu()
        ref_A, ref_B = ref_A.cpu(), ref_B.cpu()
    m = PTQSLBatchingQuantMatMul(metric="hessian", eq_beta=1.2, eq_n=100, **mod)
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = [A.cuda(), Bm.cuda()], Y.cuda(), G.cuda()
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    flips, worst, compared = _compare_steps(f"{name}/W{bit}", [s.cpu().numpy() for s in m.last_scores], ref_tables,
                                            group_independent_until=1)
    a_err = float((m.A_interval.cpu().reshape(-1) - ref_A.reshape(-1)).abs().max() / ref_A.abs().max())
    b_err = float((m.B_interval.cpu().reshape(-1) - ref_B.reshape(-1)).abs().max() / ref_B.abs().max())
    if flips == 0:
        assert a_err < 1e-6 and b_err < 1e-6, f"{name}: step sizes differ without a differing pick ({a_err:.2e}, {b_err:.2e})"
    else:
        assert flips <= 1, f"{name}: {flips} near-tie picks differ"
    m.A_interval = ref_A.cuda().view(1, HEADS, 1, 1, 1, 1, 1)
    m.B_interval = ref_B.cuda().view(1, HEADS, 1, 1, 1, 1, 1)
    with torch.no_grad():
        out = m.quant_forward(A[:2].cuda(), Bm[:2].cuda()).cpu()
    o_err = float((out - ref_out).abs().max() / ref_out.abs().max())
    assert o_err < 1e-3, f"{name}: quantized output differs by {o_err:.3e}"
    print(f"[baseptq parity] {name} W{bit}: flips {flips}/{compared}, worst score err {worst:.2e}, out {o_err:.1e}")


# ------------------------------------------------------------------------------- fp64 replay at the BasePTQ shapes
def test_layerwise_conv_against_fp64():
    x, W, b, y, g = [t.cuda() for t in O.make_conv_fixture(701, 8, 3, 768, 224, 16)]
    from ptq4vit_b200.quant_layers.conv import BatchingEasyQuantConv2d
    m = BatchingEasyQuantConv2d(3, 768, (16, 16), stride=16, bias=True, a_bit=32, metric="hessian", eq_alpha=0.5,
                                eq_beta=1.2, eq_n=100, search_round=1)
    m.weight.data = W.clone(); m.bias.data = b.clone(); m.cuda(); m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    _, launches, rows = _profiled(m.calibration_step2)
    obs = _observed(rows)
    # the conv multiplies the exact 3-term bf16 split of its FP32 im2col: bf16 single-segment sweeps, as channel-wise
    assert launches[0] > 0 and launches[1] == 0 and launches[2] == 0 and obs["modes"] == ["single"], obs
    assert obs["max_stages"] == 4 and not obs["rres"], obs
    rep = B.conv_layerwise_replay(W, b, x, y, g, m.last_scores[0], stride=16)
    R.check_intervals(rep, {"w_interval": m.w_interval}, "conv_layerwise")
    m.mode = "quant_forward"
    with torch.no_grad(), RH.fp32_convolutions():
        out = m(x)
    ref, bound = R.conv_forward(W, b, x, m.w_interval, stride=16)
    fr = R.check_forward(out, ref, bound, "conv_layerwise")
    worst = _record("baseptq/conv_layerwise", rep, obs, fr)
    print(f"[baseptq fp64] conv layer-wise: max err/bound {worst:.3f}, forward {fr:.3f}, paths {obs}")


# name: (K, O, n_V, images, tokens, w_bit, weight tile resident in the activation step)  -- n_H = n_a = 1: every K
# segment is the whole row.  The int8 weight tile stays resident up to K = 800 (768 here); fc2's 3072-byte rows stream,
# and its one candidate group spans 3072 / 128 = 24 stages of the 4-stage ring.
LINEAR64 = {"qkv_nv3": (D, 3 * D, 3, 2, TOK, 8, True), "proj": (D, D, 1, 2, TOK, 8, True),
            "proj_w6a6": (D, D, 1, 2, TOK, 6, True), "fc2_k3072": (4 * D, D, 1, 2, TOK, 8, False),
            "head": (D, 1000, 1, 64, 0, 8, True)}


@pytest.mark.parametrize("name", list(LINEAR64))
def test_baseptq_linear_against_fp64(name, monkeypatch):
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    K, Oo, n_V, n_img, tok, bit, cres = LINEAR64[name]
    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    monkeypatch.setenv("P4V_OPERAND", "auto")
    sp = O.LinearSpec(K, Oo, n_V=n_V, n_H=1, n_a=1, w_bit=bit, a_bit=bit, eq_alpha=0.5, eq_beta=1.2, eq_n=100,
                      search_round=1)
    x, W, b, y, g = [t.cuda() for t in O.make_linear_fixture(800 + len(name), n_img, tok, K, Oo, post_gelu=name.startswith("fc2"))]
    m = PTQSLBatchingQuantLinear(K, Oo, metric="hessian", eq_alpha=0.5, eq_beta=1.2, eq_n=100, search_round=1, n_V=n_V,
                                 n_H=1, n_a=1, w_bit=bit, a_bit=bit)
    m.weight.data = W.clone(); m.bias.data = b.clone(); m.cuda(); m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    _, launches, rows = _profiled(m.calibration_step2)
    obs = _observed(rows)
    # n_H = 1: one K segment of K >= 64 elements, so the layer's operands are int8 and every step sweeps one segment
    assert not R.gram_path(sp) and launches[2] == 0
    assert launches[0] == 0 and launches[1] > 0, f"{name}: expected int8 sweeps only, got {launches} ({obs})"
    assert obs["modes"] == ["single"], f"{name}: consumer modes {obs['modes']} ({obs})"
    assert obs["max_stages"] == 4 and obs["cres"] == cres and not obs["rres"], f"{name}: {obs}"
    rep = R.linear_replay(sp, W, b, x, y, g, m.last_scores, gram=False)
    R.check_intervals(rep, {"w_interval": m.w_interval, "a_interval": m.a_interval}, name)
    m.mode = "quant_forward"
    with torch.no_grad():
        out = m(x)
    ref, bound = R.linear_forward(sp, W, b, x, m.w_interval, m.a_interval)
    fr = R.check_forward(out.reshape(ref.shape), ref, bound, name)
    worst = _record(f"baseptq/linear/{name}", rep, obs, fr)
    print(f"[baseptq fp64] {name}: max err/bound {worst:.3f}, ring stages {obs['max_stages']}, paths {obs}")


# ------------------------------------------------------------------------------------------- the public calibrator
def _net(kind="vit"):
    from ptq4vit_b200.utils.models import SwinTransformer, VisionTransformer
    net = (SwinTransformer(**TINY_SWIN) if kind == "swin" else VisionTransformer(**RH.TINY_VIT)).cuda().eval()
    RH.add_target_noise(net, 8, 10)
    return net


def _ours_calib(kind="vit", keep=None, capture="auto"):
    from ptq4vit_b200.configs import BasePTQ as cfg
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    importlib.reload(cfg)
    B.baseptq_hessian(cfg)
    net = _net(kind)
    wrapped = wrap_modules_in_net(net, cfg)
    cal = Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), sequential=False, batch_size=4,
                                   capture=capture)
    cal.keep_captured = keep
    with RH.fp32_convolutions():
        cal.batching_quant_calib()
    torch.cuda.synchronize()
    importlib.reload(cfg)
    assert all(m.mode == "quant_forward" and m.calibrated for m in wrapped.values())
    return RH.collect_intervals(wrapped), net, wrapped, cal


def _check_int_export(wrapped):
    """utils/integer.get_model_int_weight of the calibrated net, byte for byte against the reference's own function
    (integer.py:8-18) on the same modules.  The reference's `weight / w_interval` only broadcasts for one block; for qkv
    (n_V = 3) its result holds every block's quotient and block v is compared against rows of block v."""
    from ptq4vit_b200.utils import integer as I
    Rf = RH.load()
    ours = I.get_model_int_weight(wrapped)
    ref = Rf.integer.get_model_int_weight(wrapped)
    assert set(ours) == set(ref) and any(k.endswith("patch_embed.proj") for k in ours)
    for name, w in ours.items():
        w, r = w.cpu(), ref[name].cpu()
        assert w.dtype == r.dtype == torch.int8
        if r.shape == w.shape:
            assert torch.equal(w, r), name
        else:
            n_V = wrapped[name].n_V
            rows = w.shape[0] // n_V
            for v in range(n_V):
                assert torch.equal(w[v * rows:(v + 1) * rows], r.reshape(n_V, -1, *w.shape)[v, 0, v * rows:(v + 1) * rows]), name
    return len(ours)


@pytest.mark.parametrize("kind", ["vit", "swin"])
def test_public_calibrator_matches_reference_calibrator(kind):
    snap_ours = {}
    got, net, wrapped, cal = _ours_calib(kind, keep=snap_ours)
    from ptq4vit_b200.quant_layers.conv import BatchingEasyQuantConv2d
    conv = [m for m in wrapped.values() if isinstance(m, BatchingEasyQuantConv2d)]
    assert len(conv) == 1 and conv[0].w_interval.shape == (1, 1, 1, 1)
    if not RH.available():
        if kind == "swin":
            pytest.skip("needs the reference staged by build() (oracle/_ref)")
        ref = _as_dict(np.load(GOLD_CALIB), "par")
        bad, n = _count_diff(got, ref, "BasePTQ vs CPU golden", max_frac=0.15)
        print(f"[baseptq calibrator golden] {bad}/{n} step sizes differ from the CPU reference run")
        return
    snap_ref = {}
    ref, _, _ = B.run_reference_calibrator_baseptq(_net(kind), RH.tiny_images(), batch_size=4, snapshot=snap_ref)
    assert set(ref) == set(got)
    worst = 0.0
    for name, d in snap_ours.items():
        for key, t in d.items():
            if t is None:
                assert snap_ref[name][key] is None, f"{name}.{key}"
                continue
            r = snap_ref[name][key].to(t.device)
            assert t.shape == r.shape, f"captured {name}.{key}: {tuple(t.shape)} vs {tuple(r.shape)}"
            err = float((t - r).abs().max() / (r.abs().max() + 1e-30))
            worst = max(worst, err)
            assert err < 1e-4, f"captured {name}.{key} differs from the reference's capture: {err:.2e}"
    bad, n = _count_diff(got, ref, f"BasePTQ {kind} vs reference on GPU", max_frac=0.05)
    n_int = _check_int_export(wrapped)
    print(f"[baseptq calibrator] {kind}: {len(snap_ours)} modules, captured worst rel diff {worst:.2e}, "
          f"{bad}/{n} step sizes differ (neighbouring-grid near-ties), {n_int} integer weights byte-identical")


# ------------------------------------------------------------------------------------------------ default metric
def test_default_cosine_metric_raises_before_any_launch():
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.configs import BasePTQ as cfg
    importlib.reload(cfg)
    x, W, b, y, g = [t.cuda() for t in O.make_conv_fixture(5, 2, 3, 64, 32, 16)]
    conv = cfg.get_module("qconv", 3, 64, (16, 16), (16, 16), (0, 0), (1, 1), 1, True, "zeros").cuda()
    conv.raw_input, conv.raw_out, conv.raw_grad = x, y, g
    xl, Wl, bl, yl, gl = [t.cuda() for t in O.make_linear_fixture(6, 2, 9, 64, 64)]
    lin = cfg.get_module("qlinear_proj", 64, 64).cuda()
    lin.raw_input, lin.raw_out, lin.raw_grad = xl, yl, gl
    A, Bm, Y, G = [t.cuda() for t in O.make_matmul_fixture(7, 2, 2, 9, 16, 9)]
    mm = cfg.get_module("qmatmul_qk")
    mm.raw_input, mm.raw_out, mm.raw_grad = [A, Bm], Y, G
    for m in (conv, lin, mm):
        before = _lib.launch_count()
        with pytest.raises(NotImplementedError, match="cosine"):
            m.calibration_step2()
        assert _lib.launch_count() == before, type(m).__name__
