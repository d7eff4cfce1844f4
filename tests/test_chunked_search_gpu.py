"""Memory-bounded search: a layer searched in chunks of rows (Linear) or images (MatMul) chooses what the whole-layer
search chooses.

Chunking is forced through P4V_WORKSPACE_BUDGET, set to the workspace the library plans for the wanted chunk.  Every
score is a sum over rows or images and the per-tile fp32 partials of a chunk are those of the same tiles in one pass, so
only the order of the fp64 score sums changes: slab-path and MatMul step sizes must be bit-identical and their score
tables agree to 1e-12.  The normal-equation weight steps add fp32 sums of H, U and sum (g e)^2 over the chunks: their
tables agree to 1e-6 of their maximum and picks are identical except at near-ties.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ptq_oracle as O   # seeded fixtures only

pytestmark = pytest.mark.gpu


def _cdiv(a, b):
    return -(-a // b)


def _budget_for_linear(m, rows, tokens, k):
    """Budget under which the module's search takes exactly k chunks (k = 1: the whole layer)."""
    from ptq4vit_b200 import _lib
    d = m._desc(rows, tokens, m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
    d.rows_per_chunk = 0 if k == 1 else _cdiv(_cdiv(rows, k), 128) * 128
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    return n.value


def _budget_for_matmul(m, A, B, k):
    from ptq4vit_b200 import _lib
    d = m._desc(A, B, m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
    d.images_per_chunk = 0 if k == 1 else _cdiv(d.batch, k)
    n = ctypes.c_size_t()
    _lib.check(_lib.lib().p4v_matmul_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "workspace")
    return n.value


def _linear(post_gelu, K, Oo, n_V, n_H, n_a, w_bit=8, a_bit=8, n_img=8, n_tok=65, seed=3):
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear, PostGeluPTQSLBatchingQuantLinear
    x, W, b, y, g = O.make_linear_fixture(seed, n_img, n_tok, K, Oo, post_gelu=post_gelu)
    cls = PostGeluPTQSLBatchingQuantLinear if post_gelu else PTQSLBatchingQuantLinear
    m = cls(K, Oo, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=2, n_V=n_V, n_H=n_H, n_a=n_a,
            w_bit=w_bit, a_bit=a_bit)
    m.weight.data = W; m.bias.data = b
    return m.cuda(), [t.cuda() for t in (x, y, g)]


def _run_linear(m, x, y, g, monkeypatch, k):
    monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(_budget_for_linear(m, x.shape[0] * x.shape[1], x.shape[1], k)))
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    assert m.calib_chunks == k
    assert m.calib_need_batching == (k > 1)
    if k > 1:
        rows_per_chunk = _cdiv(_cdiv(x.shape[0] * x.shape[1], k), 128) * 128
        assert m.calib_batch_size == _cdiv(rows_per_chunk, x.shape[1])
    scores = [s.detach().double().cpu().numpy() for s in m.last_scores]
    return m.w_interval.detach().cpu().numpy().reshape(-1), m.a_interval.detach().cpu().numpy().reshape(-1), scores


def _tables_agree(ref, got, rtol, what):
    assert len(ref) == len(got)
    worst = 0.0
    for i, (r, t) in enumerate(zip(ref, got)):
        err = float(np.abs(r - t).max() / np.abs(r).max())
        worst = max(worst, err)
        assert err <= rtol, f"{what}: score table {i} differs by {err:.3e} of its maximum"
    return worst


@pytest.mark.parametrize("n_H,n_a", [(4, 2), (1, 1)])
def test_linear_slab_path_chunks_are_exact(monkeypatch, n_H, n_a):
    """post-GELU (twin-uniform activations): 520 rows in 1, 2 (384 + 136) and 3 (256 + 256 + 8) chunks."""
    m, (x, y, g) = _linear(True, 256, 128, 1, n_H, n_a)
    w1, a1, s1 = _run_linear(m, x, y, g, monkeypatch, 1)
    for k in (2, 3):
        wk, ak, sk = _run_linear(m, x, y, g, monkeypatch, k)
        assert np.array_equal(w1, wk) and np.array_equal(a1, ak), f"{k} chunks: step sizes differ"
        worst = _tables_agree(s1, sk, 1e-12, f"{k} chunks")
        print(f"[chunked linear n_H={n_H} n_a={n_a}] {k} chunks: step sizes identical, tables within {worst:.1e}")


def test_linear_w6a6_slab_path_chunks_are_exact(monkeypatch):
    m, (x, y, g) = _linear(False, 256, 128, 2, 2, 1, w_bit=6, a_bit=6, seed=4)
    w1, a1, s1 = _run_linear(m, x, y, g, monkeypatch, 1)
    w3, a3, s3 = _run_linear(m, x, y, g, monkeypatch, 3)
    assert np.array_equal(w1, w3) and np.array_equal(a1, a3)
    _tables_agree(s1, s3, 1e-12, "W6A6, 3 chunks")


def _gap(table):
    """Per group: the distance of the best score to the runner-up, relative to the table maximum."""
    t = np.sort(table.reshape(table.shape[0], -1), axis=0)
    return (t[-1] - t[-2]) / np.abs(table).max()


@pytest.mark.parametrize("rows", [(8, 65), (8, 256)])
def test_linear_normal_equation_path_chunks(monkeypatch, rows):
    """Narrow column blocks as in ViT qkv (32 columns): whole and chunked, the weight steps take the normal-equation
    form; chunked, H, U and sum (g e)^2 add over the chunks.  Every score table within 1e-6 of its maximum; every pick
    identical unless the whole-layer table's own gap is below 1e-6 (from there on the greedy paths may part).  520 rows
    split 384 + 136 and 256 + 256 + 8; 2048 rows split 1024 + 1024 and 768 + 768 + 512, chunk boundaries on multiples of
    the Gram GEMM's 256-token accumulation splits."""
    n_img, n_tok = rows
    m, (x, y, g) = _linear(False, 256, 192, 3, 8, 1, n_img=n_img, n_tok=n_tok, seed=5)
    w1, a1, s1 = _run_linear(m, x, y, g, monkeypatch, 1)
    for k in (2, 3):
        wk, ak, sk = _run_linear(m, x, y, g, monkeypatch, k)
        worst, compared = 0.0, 0
        for i, (r, t) in enumerate(zip(s1, sk)):
            err = float(np.abs(r - t).max() / np.abs(r).max())
            worst = max(worst, err)
            assert err <= 1e-6, f"{k} chunks: score table {i} differs by {err:.3e} of its maximum"
            compared += 1
            pick_r = np.argmax(r.reshape(r.shape[0], -1), axis=0)
            pick_t = np.argmax(t.reshape(t.shape[0], -1), axis=0)
            if not np.array_equal(pick_r, pick_t):
                ne = pick_r != pick_t
                assert np.all(_gap(r)[ne] < 1e-6), f"{k} chunks: table {i} picks differ where the gap is not a near-tie"
                break
        else:
            assert np.array_equal(w1, wk) and np.array_equal(a1, ak), f"{k} chunks: step sizes differ"
        print(f"[chunked linear, normal-equation form, {x.shape[0] * x.shape[1]} rows] {k} chunks: {compared} tables "
              f"within {worst:.1e} of their maximum")


def _matmul(sos, A_bit, n_img=5, H=3, seed=7):
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul, SoSPTQSLBatchingQuantMatMul
    if sos:
        A, B, Y, G = O.make_matmul_fixture(seed, n_img, H, 65, 65, 32, softmax_A=True)
    else:
        A, B, Y, G = O.make_matmul_fixture(seed, n_img, H, 65, 64, 65)
    cls = SoSPTQSLBatchingQuantMatMul if sos else PTQSLBatchingQuantMatMul
    m = cls(A_bit=A_bit, B_bit=A_bit, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=2)
    return m, [t.cuda() for t in (A, B, Y, G)]


def _run_matmul(m, A, B, Y, G, monkeypatch, k):
    monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(_budget_for_matmul(m, A, B, k)))
    m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = [A, B], Y, G
    with torch.no_grad():
        m.calibration_step2()
    torch.cuda.synchronize()
    assert m.calib_chunks == k and m.calib_need_batching == (k > 1)
    if k > 1:
        assert m.calib_batch_size == _cdiv(A.shape[0], k)
    out = [torch.as_tensor(v).detach().cpu().numpy().reshape(-1) for v in (m.A_interval, m.B_interval)]
    if m.sos:
        out.append(torch.as_tensor(m.split).detach().cpu().numpy().reshape(-1))
    return out, [s.detach().double().cpu().numpy() for s in m.last_scores]


@pytest.mark.parametrize("sos", [False, True])
@pytest.mark.parametrize("bits", [8, 6])
def test_matmul_chunks_are_exact(monkeypatch, sos, bits):
    """5 images in 1, 2 (3 + 2) and 3 (2 + 2 + 1) chunks; plain and split-of-softmax."""
    m, (A, B, Y, G) = _matmul(sos, bits, seed=7 + bits + sos)
    r1, s1 = _run_matmul(m, A, B, Y, G, monkeypatch, 1)
    for k in (2, 3):
        rk, sk = _run_matmul(m, A, B, Y, G, monkeypatch, k)
        for a, b in zip(r1, rk):
            assert np.array_equal(a, b), f"{k} chunks: step sizes differ"
        worst = _tables_agree(s1, sk, 1e-12, f"{k} chunks")
        print(f"[chunked matmul sos={sos} W{bits}A{bits}] {k} chunks: step sizes identical, tables within {worst:.1e}")


def test_deit_b_384_matmul2_under_a_memory_budget(monkeypatch):
    """A synthetic split-of-softmax matmul2 of DeiT-B/384 x 128 images (A [128,12,577,577]): the whole-layer search
    needs a 61 GB workspace.  Under a 20 GB and a 10 GB budget it runs in chunks, chooses the same step sizes, and the
    memory it takes besides the captured tensors stays within the budget."""
    from ptq4vit_b200.quant_layers.matmul import SoSPTQSLBatchingQuantMatMul
    gen = torch.Generator(device="cuda").manual_seed(11)
    A = torch.softmax(torch.randn(128, 12, 577, 577, device="cuda", generator=gen) * 4.0, dim=-1)
    B = torch.randn(128, 12, 577, 64, device="cuda", generator=gen)
    Y = A @ B
    G = torch.randn(Y.shape, device="cuda", generator=gen) * 1e-3
    torch.cuda.synchronize()
    res = []
    for budget in (20 << 30, 10 << 30):
        monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(budget))
        m = SoSPTQSLBatchingQuantMatMul(metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=1)
        m.raw_input, m.raw_out, m.raw_grad = [A, B], Y, G
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            m.calibration_step2()
        torch.cuda.synchronize()
        extra = torch.cuda.max_memory_allocated() - base
        assert m.calib_need_batching and m.calib_chunks > 1
        assert extra <= budget, f"search took {extra} bytes besides the captures, budget {budget}"
        print(f"[384 matmul2] budget {budget >> 30} GB: {m.calib_chunks} chunks of {m.calib_batch_size} images, "
              f"{extra / 2 ** 30:.2f} GB besides the captures")
        res.append([torch.as_tensor(v).detach().cpu().numpy().reshape(-1) for v in (m.A_interval, m.B_interval, m.split)])
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_calibrator_switches_to_per_module_capture_under_a_small_budget(monkeypatch):
    from ptq4vit_b200.configs import PTQ4ViT as cfg
    from ptq4vit_b200.utils import quant_calib as Q
    from ptq4vit_b200.utils.models import VisionTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    from oracle import ref_harness as RH
    import importlib

    def run(capture, capture_budget=None):
        importlib.reload(cfg)
        net = VisionTransformer(**RH.TINY_VIT).cuda().eval()
        RH.add_target_noise(net, 8, 10)
        wrapped = wrap_modules_in_net(net, cfg)
        cal = Q.HessianQuantCalibrator(net, wrapped, RH.ListLoader(RH.tiny_images()), batch_size=4, capture=capture,
                                       capture_budget=capture_budget)
        with RH.fp32_convolutions():
            cal.batching_quant_calib()
        torch.cuda.synchronize()
        return RH.collect_intervals(wrapped), cal

    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    _, cal = run("auto")
    t = cal.timings
    assert t["single_pass"] and t["capture_mode"] == "single_pass"
    assert t["capture_bytes_est"] > 0 and t["min_workspace_bytes"] > 0
    # captures no longer fit next to the smallest workspace, which still fits
    budget = t["capture_bytes_est"] + t["min_workspace_bytes"] - 1
    got_auto, cal = run("auto", budget)
    assert not cal.timings["single_pass"] and cal.timings["capture_mode"] == "per_module"
    assert cal.timings["memory_budget_bytes"] == budget
    got_single, cal = run("single_pass")
    assert cal.timings["single_pass"]
    for name, d in got_single.items():
        for key, v in d.items():
            assert np.array_equal(np.asarray(v), np.asarray(got_auto[name][key])), f"{name}.{key}"
