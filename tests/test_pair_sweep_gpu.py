"""Pair steps of the tensor-core sweep (post-GELU weight steps, split-of-softmax B steps): one ring stage per candidate
slab shared by the two row parts, evaluated in two 64-column halves.  The pair consumer does the fp32 epilogue of the
multi-segment path in the same order, so every score table and step size must be bit-identical to a search forced onto
the multi-segment path (P4V_NO_PAIR=1)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ptq_oracle as O   # seeded fixtures only

pytestmark = pytest.mark.gpu


def _linear(K, Oo, n_V, n_H, n_img, n_tok, w_bit=8, a_bit=8, seed=11, rounds=2):
    from ptq4vit_b200.quant_layers.linear import PostGeluPTQSLBatchingQuantLinear
    x, W, b, y, g = O.make_linear_fixture(seed, n_img, n_tok, K, Oo, post_gelu=True)
    m = PostGeluPTQSLBatchingQuantLinear(K, Oo, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100,
                                         search_round=rounds, n_V=n_V, n_H=n_H, n_a=1, w_bit=w_bit, a_bit=a_bit)
    m.weight.data = W; m.bias.data = b
    return m.cuda(), [t.cuda() for t in (x, y, g)]


def _run_linear(m, x, y, g):
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    return ([m.w_interval.cpu().numpy().copy(), m.a_interval.cpu().numpy().copy()],
            [s.cpu().numpy().copy() for s in m.last_scores])


def _run_matmul(m, A, B, Y, G):
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = [A, B], Y, G
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    out = [torch.as_tensor(v).cpu().numpy().reshape(-1).copy() for v in (m.A_interval, m.B_interval, m.split)]
    return out, [torch.as_tensor(s).cpu().numpy().copy() for s in m.last_scores]


def _pair_vs_multi(run, monkeypatch):
    monkeypatch.delenv("P4V_NO_PAIR", raising=False)
    steps_pair, logs_pair = run()
    monkeypatch.setenv("P4V_NO_PAIR", "1")
    steps_multi, logs_multi = run()
    monkeypatch.delenv("P4V_NO_PAIR")
    assert len(logs_pair) == len(logs_multi)
    for i, (a, b) in enumerate(zip(logs_pair, logs_multi)):
        assert np.array_equal(a, b), f"score table {i} differs"
    for a, b in zip(steps_pair, steps_multi):
        assert np.array_equal(a, b), "step sizes differ"
    return steps_pair, logs_pair


def test_pair_fc2_vit_b(monkeypatch):
    """ViT-B fc2: 3072 -> 768, n_V = n_H = 24, 8 images of 197 tokens (1576 rows)."""
    m, (x, y, g) = _linear(3072, 768, 24, 24, 8, 197, rounds=1)
    _pair_vs_multi(lambda: _run_linear(m, x, y, g), monkeypatch)


def test_pair_small_ragged_rows_and_simt(monkeypatch):
    """520 rows (not a multiple of 128), 64-wide column blocks; the SIMT kernel picks what the tensor-core kernel picks."""
    m, (x, y, g) = _linear(256, 128, 2, 4, 8, 65)
    steps, logs = _pair_vs_multi(lambda: _run_linear(m, x, y, g), monkeypatch)
    monkeypatch.setenv("P4V_KERNEL", "simt")
    steps_simt, logs_simt = _run_linear(m, x, y, g)
    for i, (a, b) in enumerate(zip(logs, logs_simt)):
        pa, pb = a.reshape(a.shape[0], -1).argmax(0), b.reshape(b.shape[0], -1).argmax(0)
        if not np.array_equal(pa, pb):   # a near-tie may flip; the greedy paths part from there on
            t = np.sort(a.reshape(a.shape[0], -1), axis=0)
            assert np.all(((t[-1] - t[-2]) / np.abs(a).max())[pa != pb] < 1e-5), f"table {i}: picks differ"
            break
    else:
        for a, b in zip(steps, steps_simt):
            assert np.array_equal(a, b)


def test_pair_w6a6(monkeypatch):
    m, (x, y, g) = _linear(512, 256, 4, 4, 6, 65, w_bit=6, a_bit=6, seed=12)
    _pair_vs_multi(lambda: _run_linear(m, x, y, g), monkeypatch)


def test_pair_matmul2_vit_b(monkeypatch):
    """ViT-B matmul2 (attention @ V, split-of-softmax A): 8 images x 12 heads, 197 x 197 @ 197 x 64; K = 197 int8 takes
    two jobs per part (128 + 96 bytes)."""
    from ptq4vit_b200.quant_layers.matmul import SoSPTQSLBatchingQuantMatMul
    A, B, Y, G = [t.cuda() for t in O.make_matmul_fixture(13, 8, 12, 197, 197, 64, softmax_A=True)]
    m = SoSPTQSLBatchingQuantMatMul(metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=2)
    _pair_vs_multi(lambda: _run_matmul(m, A, B, Y, G), monkeypatch)


def test_pair_chunked_linear(monkeypatch):
    """A row-chunked search (3 chunks of at most 256 rows) takes the pair path in every chunk."""
    from ptq4vit_b200 import _lib
    m, (x, y, g) = _linear(256, 128, 1, 4, 8, 65, seed=14)
    d = m._desc(x.shape[0] * x.shape[1], x.shape[1], m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
    d.rows_per_chunk = 256
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(n.value))

    def run():
        out = _run_linear(m, x, y, g)
        assert m.calib_chunks == 3
        return out

    _pair_vs_multi(run, monkeypatch)
