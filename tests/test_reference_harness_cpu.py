"""Checks of the test / baseline infrastructure itself on the CPU (dev container): the oracle's restatements of
utils/integer.py against the reference's functions, the reference timing helpers bench.py uses, and bench.py's unit /
extrapolation arithmetic.  The reference checks need the copy build() stages under oracle/_ref."""
import argparse

import pytest
import torch

from oracle import ptq_oracle as O
from oracle import ref_harness as RH

needs_ref = pytest.mark.skipif(not RH.available(), reason="reference tree not staged")


@needs_ref
def test_integer_oracle_matches_reference_functions():
    R = RH.load()
    gen = torch.Generator().manual_seed(2)
    lin = R.linear.PTQSLBatchingQuantLinear(64, 32)
    lin.w_interval = (lin.weight.data.abs().max() / 127.5).view(1, 1, 1, 1)
    assert torch.equal(R.integer.quantize_int_weight(lin).view(32, 64), O.int_plain(lin.weight.data, lin.w_interval.view(1, 1), 128))
    x = torch.randn(4, 9, 64, generator=gen)
    lin.a_interval = (x.abs().max() / 127.5).view(1, 1)
    R.integer.quantize_int_activation(lin, (x,))
    assert torch.equal(lin.int_input[0], O.int_plain(x, lin.a_interval, 128))
    gel = R.linear.PostGeluPTQSLBatchingQuantLinear(64, 32)
    xg = torch.nn.functional.gelu(x * 1.5)
    gel.a_interval = (xg.max() / 127.5).view(1, 1)
    R.integer.quantize_int_activation(gel, (xg,))
    assert torch.equal(gel.int_input[0], O.int_gelu_twin(xg, gel.a_interval, gel.a_neg_interval, 128))
    sos = R.matmul.SoSPTQSLBatchingQuantMatMul()
    S = torch.softmax(torch.randn(2, 3, 10, 10, generator=gen) * 4, -1); V = torch.randn(2, 3, 10, 8, generator=gen)
    sos.split = torch.tensor(2.0 ** -4); sos.A_interval = sos.split / 127
    sos.B_interval = (V.abs().amax((0, 2, 3)) / 127.5).view(1, 3, 1, 1, 1, 1, 1)
    sos._get_padding_parameters(S, V)
    R.integer.quantize_int_activation(sos, (S, V))
    assert torch.equal(sos.int_input[0], O.int_sos_twin(S, sos.split, sos.A_interval, 128))
    assert torch.equal(sos.int_input[1], O.int_plain(V, sos.B_interval.view(1, 3, 1, 1), 128))


@needs_ref
def test_reference_timing_helpers_count_units():
    x, W, b, y, g = O.make_linear_fixture(1, 4, 20, 32, 48)
    s, units = RH.time_linear(x, W, b, y, g, False, eq_n=4, w_blocks=1, n_V=3, n_H=2, n_a=1, search_round=1)
    assert units == 8 and s > 0                      # one column block + one activation step, 4 candidates each
    s, units = RH.time_linear(x, W, b, y, g, False, eq_n=4, w_blocks=None, n_V=3, n_H=2, n_a=1, search_round=2)
    assert units == 2 * (2 + 1) * 4
    A, B, Y, G = O.make_matmul_fixture(2, 2, 3, 12, 8, 12)
    assert RH.time_matmul(A, B, Y, G, False, eq_n=4, search_round=1)[1] == 8
    As, Bs, Ys, Gs = O.make_matmul_fixture(3, 2, 3, 12, 12, 8, softmax_A=True)
    assert RH.time_matmul(As, Bs, Ys, Gs, True, eq_n=4, search_round=1)[1] == 24


def test_bench_unit_accounting_and_extrapolation():
    import bench
    a = argparse.Namespace(model="vit_base_patch16_224", images=32, blocks=24, rounds=3, bit=8)
    types = bench.layer_types(a)
    assert types["qkv"][2]["n_V"] == 72 and types["head"][2]["n_V"] == 1 and types["fc2"][1][2] is True
    total = sum(count * per for (_, _, _, count, per) in types.values())
    assert total == 49 * 7500 + 12 * 600 + 12 * 360        # SURVEY 8d: 367 500 Linear units + MatMul units
    v, job_s, rates = bench.extrapolate(a, {k: (1.0, 10.0) for k in types})
    assert abs(job_s - total / 10.0) < 1e-6 and abs(v - 10.0) < 1e-9
    assert bench.is_default_workload(a) and "n_V=n_H=24" in bench.workload_name(a)


def test_module_cost_uses_probed_shapes():
    from ptq4vit_b200.quant_layers import linear as L, matmul as M
    from ptq4vit_b200.utils import quant_calib as Q
    lin = L.PTQSLBatchingQuantLinear(128, 384, n_V=3, search_round=3)
    c1 = Q.module_cost(lin, 32, {"x": (1, 144, 128)}) - 3 * Q._ROUND_OVERHEAD_S
    c64 = Q.module_cost(lin, 32, {"x": (64, 144, 128)}) - 3 * Q._ROUND_OVERHEAD_S       # Swin: 64 windows per image fold into the leading dim
    assert abs(c64 / c1 - 64.0) < 1e-6
    mm = M.PTQSLBatchingQuantMatMul(search_round=3)
    cm = Q.module_cost(mm, 32, {"A": (64, 4, 144, 32), "B": (64, 4, 32, 144)})
    assert abs(cm - 3 * (Q._ROUND_OVERHEAD_S + 2 * 100 * 2.0 * 32 * 64 * 4 * 144 * 32 * 144 / Q._MATMUL_RATE)) < 1e-9
    # ViT-B/224 x 32 images at n_V = n_H = 24: the model reproduces the per-round times measured on an H100 within 20 %
    qkv = L.PTQSLBatchingQuantLinear(768, 2304, n_V=72, n_H=24, search_round=1)
    qk = M.PTQSLBatchingQuantMatMul(search_round=1)
    assert abs(Q.module_cost(qkv, 32, {"x": (1, 197, 768)}) / 20.9e-3 - 1) < 0.2
    assert abs(Q.module_cost(qk, 32, {"A": (1, 12, 197, 64), "B": (1, 12, 64, 197)}) / 7.7e-3 - 1) < 0.2


@needs_ref
@pytest.mark.parametrize("metric", ["L2_norm", "linear_weighted_L2_norm", "square_weighted_L2_norm"])
def test_weighted_l2_metrics_are_hessian_with_a_surrogate_weight(metric):
    """The product evaluates the reference's squared-error metrics (linear.py:411-416, matmul.py:467-472,
    conv.py:511-516) as the Hessian metric with a surrogate per-element weight (quant_layers/_metric.py).  The
    reference itself must pick the same candidates either way."""
    from ptq4vit_b200.quant_layers._metric import metric_weight
    x, W, b, y, g = O.make_linear_fixture(41, 4, 20, 32, 48)
    mod = dict(n_V=3, n_H=2, n_a=2, search_round=2, eq_n=25)
    direct = RH.run_linear(x, W, b, y, g, quant_forward=False, metric=metric, **mod)
    via = RH.run_linear(x, W, b, y, metric_weight(metric, y, None, "test").clone(), quant_forward=False, metric="hessian", **mod)
    assert torch.equal(direct["w_interval"], via["w_interval"]) and torch.equal(direct["a_interval"], via["a_interval"])
    for sd, sv in zip(direct["scores"], via["scores"]):
        assert float((sd - sv).abs().max() / sd.abs().max()) < 1e-5
    A, B, Y, G = O.make_matmul_fixture(42, 2, 3, 12, 8, 12)
    dm = RH.run_matmul(A, B, Y, G, quant_forward=False, metric=metric, search_round=1, eq_n=25)
    vm = RH.run_matmul(A, B, Y, metric_weight(metric, Y, None, "test").clone(), quant_forward=False, metric="hessian", search_round=1, eq_n=25)
    assert torch.equal(dm["A_interval"], vm["A_interval"]) and torch.equal(dm["B_interval"], vm["B_interval"])
    xc, Wc, bc, yc, gc = O.make_conv_fixture(43, 2, 3, 8, 8, 4)
    dc = RH.run_conv(xc, Wc, bc, yc, gc, stride=4, metric=metric, eq_n=25)
    vc = RH.run_conv(xc, Wc, bc, yc, metric_weight(metric, yc, None, "test").clone(), stride=4, metric="hessian", eq_n=25)
    assert torch.equal(dc["w_interval"], vc["w_interval"])


def test_unsupported_metrics_raise_like_the_reference():
    from ptq4vit_b200.quant_layers._metric import metric_weight
    y = torch.ones(2, 3)
    for metric in ("cosine", "L1_norm", "pearson", "nonsense"):
        with pytest.raises(NotImplementedError):
            metric_weight(metric, y, None, "test")
    with pytest.raises(AssertionError):
        metric_weight("hessian", y, None, "test")
