"""Activation steps of Linear layers whose type is chosen as bf16 (K segments shorter than 64 elements) run on int8
images with the weight tile resident in shared memory.  bf16 with fp32 accumulators and int8 with s32 accumulators form
the same exact integer products and the epilogue runs the same fp32 operations in the same order, so every score table
and step size must be bit-identical to a search with the whole layer forced to bf16 (P4V_OPERAND=bf16)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ptq_oracle as O   # seeded fixtures only

pytestmark = pytest.mark.gpu

# ViT-B/224 x 32 images: (in, out, n_V, n_H, images, tokens); head sees the class token only
SHAPES = {
    "qkv": (768, 2304, 72, 24, 32, 197),
    "proj": (768, 768, 24, 24, 32, 197),
    "fc1": (768, 3072, 24, 24, 32, 197),
    "head": (768, 1000, 1, 24, 32, 1),
    "small": (256, 128, 4, 8, 8, 65),      # 520 rows: not a multiple of 128
}


def _linear(name, rounds=2, seed=21):
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    K, Oo, n_V, n_H, n_img, n_tok = SHAPES[name]
    x, W, b, y, g = O.make_linear_fixture(seed, n_img, n_tok, K, Oo)
    m = PTQSLBatchingQuantLinear(K, Oo, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=rounds,
                                 n_V=n_V, n_H=n_H, n_a=1)
    m.weight.data = W; m.bias.data = b
    return m.cuda(), [t.cuda() for t in (x, y, g)]


def _run(m, x, y, g):
    """Step sizes, every score table, and the int8 sweep launches of one search."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    prof = (ctypes.c_double * 12)()
    lib.p4v_profile_collect_kinds(prof, 12)            # drop anything recorded before
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    lib.p4v_profile_enable(1)
    try:
        with torch.no_grad():
            m.calibration_step2()
        torch.cuda.synchronize()
    finally:
        lib.p4v_profile_enable(0)
    lib.p4v_profile_collect_kinds(prof, 12)
    steps = [m.w_interval.cpu().numpy().copy(), m.a_interval.cpu().numpy().copy()]
    return steps, [s.cpu().numpy().copy() for s in m.last_scores], int(prof[7])


def _int8_vs_bf16(run, monkeypatch, rounds):
    monkeypatch.delenv("P4V_OPERAND", raising=False)
    steps8, logs8, int8_launches = run()
    monkeypatch.setenv("P4V_OPERAND", "bf16")
    steps16, logs16, int8_launches_bf16 = run()
    monkeypatch.delenv("P4V_OPERAND")
    assert int8_launches_bf16 == 0
    assert int8_launches >= rounds, "the activation steps did not run on int8 images"
    assert len(logs8) == len(logs16)
    for i, (a, b) in enumerate(zip(logs8, logs16)):
        assert np.array_equal(a, b), f"score table {i} differs"
    for a, b in zip(steps8, steps16):
        assert np.array_equal(a, b), "step sizes differ"


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_int8_activation_step_matches_bf16(name, monkeypatch):
    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    m, (x, y, g) = _linear(name)
    _int8_vs_bf16(lambda: _run(m, x, y, g), monkeypatch, m.search_round)


@pytest.mark.parametrize("name", ["small", "qkv"])
def test_int8_activation_step_matches_bf16_in_two_chunks(name, monkeypatch):
    from ptq4vit_b200 import _lib
    m, (x, y, g) = _linear(name)
    rows = x.shape[0] * x.shape[1]
    d = m._desc(rows, x.shape[1], m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
    d.rows_per_chunk = -(-rows // 256) * 128            # half the rows, rounded up to whole tiles
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(n.value))

    def run():
        out = _run(m, x, y, g)
        assert m.calib_chunks == 2
        return out

    _int8_vs_bf16(run, monkeypatch, m.search_round)
