"""Teacher-forced fp64 restatement of the step-size searches, with an entry-wise error bound (TEST INFRASTRUCTURE).

Given a layer's tensors and the score tables the library logged (``keep_scores=True`` -> ``last_scores``), the
evaluator replays the greedy search step by step:

* quantisation exactly as the reference does it, in fp32 on the tensors' device (min-max step sizes, ``rne(v/Δ)`` then
  clamp, candidate grid ``f_c·Δ⁰``, twin-uniform post-GELU parts with ``Δ₋``, split-of-softmax hi/lo parts and the 20
  split candidates, and DESIGN §5's rule that a NaN quotient (``eq_alpha = 0``) quantises to 0).  On a GPU torch's
  division by a Python scalar is the device's, which the library follows by default; on the CPU it is IEEE, which the
  golden vectors were made with;
* layer outputs ``Σ (q_w·Δ_w)(q_x·Δ_x) + b`` and scores ``-(g·(y-ŷ))²`` (mean over block features, mean over tokens,
  sum over images) in fp64, where every ``q·Δ`` is exact;
* the pick of each group is the FIRST argmax of the logged fp32 table (what ``select_step_kernel`` compares), so every
  table of every round is compared even after a near-tie; the evaluator's final step sizes must then equal the
  library's bitwise.

Error model (u = 2⁻²⁴, γ_n = nu/(1-nu)); every table entry must satisfy ``|got - ref| ≤ bound``.

Slab sweep (``csrc/sweep_tc.cu``, Linear / MatMul / Conv, weight, activation and split steps):
  residual per element  |δe| ≤ γ_{n+4}·(|y| + |b| + P) + κ·P,  P = Σ_k |ŵ_k|·|x̂_k|, n = K segments of the layer.
    The epilogue forms r = y - b and then one ``fmaf(-s, acc, r)`` per segment (sweep_tc.cu "fixed" groups and
    final segment); s = candA·candB is an fp32 product (one u), ``acc_to_float`` may round an s32 (one u) and the
    split-of-softmax hi scale 1/q1 is an fp32 reciprocal (one u).  Integer accumulators (s32, or bf16 integers below
    2²⁴) are exact: κ = 0.  The split search and the conv search multiply an exact 3-term bf16 split of an fp32
    operand; the tensor core adds into fp32 with truncation, so κ = 2u·3K_seg (K_seg products per term).
  score per entry  Σ w·g²(2|e||δe| + δe²) + γ_T·Σ w·(g e)² + u_extra·Σ w·(g e)² + u·|score|,  T = 16: the per-thread
    chain of 4 ``fmaf`` per accumulator, the pair add, the 5-level warp shuffle tree, the quarter add, the g·(…) product
    and the square (sweep_tc.cu epilogue and ``reduce8_over_warp``; conv rows: 4 + 4 + 2 levels).  Tile partials are
    then summed in fp64 (negligible) and the table is logged in fp32 (u·|score|).  The conv search folds Δ⁰ into the
    targets (``(y-b)/Δ⁰`` and ``g·Δ⁰``, DESIGN §4.4): u_extra = 3u and three more u in the residual term.
Normal-equation weight steps (``csrc/gram.cu``, ``gram_gemm.cu``): score = Σ(ge)² - 2d·U + dᵀHd, with e the residual
  of the current step sizes and, over the block's columns, a_m = Σ_k |x̂_k||d_k|, s_m = Σ_k |x̂_k|(|ŵ_c,k| + |ŵ_cur,k|):
    residual  |δe| ≤ slab bound + Σ over the blocks already committed this round of
              γ_{ks+4}·Σ_k |x̂_k||d_k| + 2u·Σ_k |x̂_k|(|ŵ_new,k| + |ŵ_old,k|)  (the rank-ks update of each pick,
              ``gram_update_kernel``: ks fp32 fmas in two chains, d = fq(w) - ŵ_cur from two rounded fp32 products),
              carried through the exact score like the slab residual error;
    Σ(ge)²    γ_M·Σ g²e²  (``e2 = fmaf(ge, ge, e2)`` over the tokens, then ``gram_reduce``);
    2d·U      2·Σ g²|e|(γ_{M+3}·a_m + u·(s_m + a_m))  (U accumulated over M tokens; ``fq_dev`` rounds ŵ_c and ŵ_cur,
              the subtraction rounds d);
    dᵀHd      Σ g²((2⁻¹⁶ + 2u·256 + u·(M/256 + 2ks + 8))·a_m² + 2u·a_m(s_m + a_m))  (``(gs·g)²`` kept as 2 bf16 terms =
              16 mantissa bits, truncating wgmma adds inside each 256-token split, rn adds across splits, the
              ``Hs·dx²`` scaling, the ks² fma evaluation in ``gram_eval_kernel``, and the rounding of d);
    combine   2u·Σ g²(e² + 2|e|a_m + a_m²)  (``e2s - 2·lin + quad`` in fp32).
``quant_forward``: per element ``γ_{n_seg+2}·(|b| + P)`` (one fp32 fma per segment plus the bias add).

Pick check: if the library picks p and the fp64 argmax is q, ``ref[q] - ref[p] ≤ bound[p] + bound[q]``.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ptq_oracle as O

U = 2.0 ** -24
T_SUM = 16                  # fp32 operations a squared residual goes through before the fp64 tile sum (see above)


def gamma(n):
    return n * U / (1.0 - n * U)


def qint(v, delta, lo, hi):
    """clamp(rne(v / delta), lo, hi) as fp32 integers; a NaN quotient (0/0 with eq_alpha = 0) quantises to 0."""
    q = (v / delta).round_()
    q = torch.where(torch.isnan(q), torch.zeros_like(q), q)
    return q.clamp_(lo, hi)


@dataclass
class Step:
    """One logged table: got [n_cand, n_groups] (fp32 from the library), ref / bound fp64, and what the library picked."""
    name: str
    got: np.ndarray
    ref: np.ndarray
    bound: np.ndarray
    pick: np.ndarray


@dataclass
class Replay:
    steps: List[Step] = field(default_factory=list)
    intervals: dict = field(default_factory=dict)        # fp32 tensors, same layout as the library's attributes

    def first_pick(self, name, got, ref, bound):
        got = torch.as_tensor(got).detach().float().cpu().numpy().reshape(ref.shape)
        pick = got.argmax(0)                              # numpy: first maximum, like torch.argmax / select_step
        self.steps.append(Step(name, got, ref, bound, pick))
        return pick


def _score_terms(e, g, w, de):
    """Per-element pieces of a score entry: w·(g e)², and the residual-error term w·g²(2|e|δe + δe²)."""
    g2 = g * g
    sq = w * g2 * e * e
    res = w * g2 * (2.0 * e.abs() * de + de * de)
    return sq, res


def _finish(sq_sum, res_sum, extra_rel=0.0):
    """Score = -Σ w·(g e)² and its bound (see the module docstring)."""
    return -sq_sum, res_sum + (gamma(T_SUM) + extra_rel + U) * sq_sum


# ---------------------------------------------------------------------------------------------------------- Linear
def gram_path(sp: O.LinearSpec, kernel="tcgen05"):
    """Whether the weight steps take the normal-equation form (DESIGN §2 and the planner's rule)."""
    ks = sp.crb_cols
    return kernel == "tcgen05" and not sp.post_gelu and ks <= 64 and ks % 4 == 0 and sp.crb_acts % ks == 0


def segment_lengths(sp):
    """Lengths of the K segments (intersections of a weight column block and an activation chunk)."""
    cuts = sorted(set(range(0, sp.K, sp.crb_cols)) | set(range(0, sp.K, sp.crb_acts)) | {sp.K})
    return [b - a for a, b in zip(cuts, cuts[1:])]


def _segments(sp):
    """Number of K segments, twin-uniform parts counted twice."""
    return len(segment_lengths(sp)) * (2 if sp.post_gelu else 1)


def linear_replay(sp: O.LinearSpec, W, b, x, y, g, tables, *, gram=False, init_layerwise=False, chunk=8):
    """Replay PTQSLBatchingQuantLinear.calibration_step2 (linear.py:536-555; PostGelu :557-642) teacher-forced by the
    logged tables (``last_scores`` order: per round the n_H weight tables [eq_n, n_V], then the n_a activation tables).
    W [O,K], x [..., K], y / g [..., O] (g = the metric's per-element weight); all on one device."""
    dev = W.device
    K, Oo = sp.K, sp.O
    tokens = 1
    for s in x.shape[1:-1]:
        tokens *= int(s)
    X = x.reshape(-1, K).float()
    M = X.shape[0]
    Y, G = y.reshape(M, Oo).double(), g.reshape(M, Oo).double()
    B = torch.zeros(Oo, dtype=torch.float64, device=dev) if b is None else b.double()
    qw, qa = sp.w_qmax, sp.a_qmax
    # min-max initial step sizes (linear.py:380-397, :576-599)
    if init_layerwise:
        w_int = (W.abs().max() / (qw - 0.5)).view(1, 1, 1, 1).repeat(sp.n_V, 1, sp.n_H, 1)
        xm = x.max() if sp.post_gelu else x.abs().max()
        a_int = (xm / (qa - 0.5)).view(1, 1).repeat(sp.n_a, 1)
    else:
        w_int, a_int = O.linear_initial_intervals(sp, W, x)
    f = O.candidate_factors(sp.eq_alpha, sp.eq_beta, sp.eq_n).to(dev)
    w_cands = f.view(-1, 1, 1, 1, 1) * w_int.unsqueeze(0)          # [eq_n+1, n_V, 1, n_H, 1]
    a_cands = f.view(1, 1, -1) * a_int.unsqueeze(-1)               # [n_a, 1, eq_n+1]
    Wv = W.view(sp.n_V, sp.crb_rows, sp.n_H, sp.crb_cols)

    def wq64(wi):                                                  # [O, K] exact q·Δ
        return (qint(Wv, wi, -qw, qw - 1).double() * wi.double()).view(Oo, K)

    neg = sp.a_neg_interval

    def xq64_chunk(xa, ai):                                        # xa [M, crb_acts] fp32, ai 0-d fp32
        if sp.post_gelu:
            pos = qint(xa, ai, 0, qa - 1).double() * ai.double()
            ng = (xa / neg).round_().clamp_(-qa, 0).double() * float(np.float32(neg))
            return pos + ng
        return qint(xa, ai, -qa, qa - 1).double() * ai.double()

    def xq64(ai_all):
        return torch.cat([xq64_chunk(X[:, a * sp.crb_acts:(a + 1) * sp.crb_acts], ai_all[a, 0]) for a in range(sp.n_a)], 1)

    n_seg = _segments(sp)
    g_slab = gamma(n_seg + 4)
    wn = 1.0 / (sp.crb_rows * tokens)                              # mean over the block's features and the tokens
    rep = Replay()
    it = iter(tables)
    for rnd in range(sp.search_round):
        Xq = xq64(a_int)
        Xa = Xq.abs()
        Wq = wq64(w_int)
        upd_err = 0.0            # Gram: error of the rank-ks updates applied to e since the round's residual sweep
        for h in range(sp.n_H):
            c0, c1 = h * sp.crb_cols, (h + 1) * sp.crb_cols
            yb = Xq @ Wq.T + B
            Pb = Xa @ Wq.abs().T
            Xh, Xha = Xq[:, c0:c1], Xa[:, c0:c1]
            Wh = Wq[:, c0:c1]
            yb_h = yb - Xh @ Wh.T
            Pb_h = Pb - Xha @ Wh.abs().T
            ref = np.zeros((sp.eq_n, sp.n_V)); bnd = np.zeros((sp.eq_n, sp.n_V))
            for p0 in range(0, sp.eq_n, chunk):
                p1 = min(sp.eq_n, p0 + chunk)
                cand = w_cands[p0:p1, :, :, h, :]                        # [p, n_V, 1, 1]
                Wc = (qint(Wv[:, :, h, :].unsqueeze(0), cand, -qw, qw - 1).double() * cand.double()).reshape(p1 - p0, Oo, -1)
                yc = yb_h.unsqueeze(0) + torch.matmul(Xh, Wc.transpose(1, 2))
                Pc = Pb_h.unsqueeze(0) + torch.matmul(Xha, Wc.abs().transpose(1, 2))
                e = Y - yc
                de = g_slab * (Y.abs() + B.abs() + Pc)
                if gram:
                    de = de + upd_err
                sq, res = _score_terms(e, G, wn, de)
                grp = lambda t: t.reshape(p1 - p0, M, sp.n_V, sp.crb_rows).sum((1, 3))
                if gram:
                    dW = Wc - Wh.unsqueeze(0)
                    ad = torch.matmul(Xha, dW.abs().transpose(1, 2))                       # Σ|x̂||d|
                    aw = torch.matmul(Xha, (Wc.abs() + Wh.abs().unsqueeze(0)).transpose(1, 2))   # Σ|x̂|(|ŵ_c|+|ŵ_cur|)
                    eb = (Y - yb).abs().unsqueeze(0)
                    g2 = wn * G * G
                    cH = 2.0 ** -16 + 2 * U * 256 + U * (M / 256 + 2 * sp.crb_cols + 8)
                    t_e2 = gamma(M) * g2 * eb * eb
                    t_u = 2.0 * g2 * eb * (gamma(M + 3) * ad + U * (aw + ad))
                    t_h = g2 * (cH * ad * ad + 2 * U * ad * (aw + ad))
                    t_c = 2 * U * g2 * (eb * eb + 2 * eb * ad + ad * ad)
                    extra = grp(t_e2 + t_u + t_h + t_c)
                else:
                    extra = torch.zeros((), dtype=torch.float64, device=dev)
                s, bd = _finish(grp(sq).cpu().numpy(), (grp(res) + extra).cpu().numpy())
                ref[p0:p1], bnd[p0:p1] = s, bd
            pick = rep.first_pick(f"round {rnd} W block {h}", next(it), ref, bnd)
            idx = torch.as_tensor(pick, device=dev).view(1, -1, 1, 1, 1)
            w_int = w_int.clone()
            w_int[:, :, h:h + 1, :] = torch.gather(w_cands[:, :, :, h:h + 1, :], 0, idx).squeeze(0)
            Wn = wq64(w_int)
            if gram:
                Wh_old, Wh_new = Wq[:, c0:c1], Wn[:, c0:c1]
                upd_err = upd_err + gamma(sp.crb_cols + 4) * (Xha @ (Wh_new - Wh_old).abs().T) + \
                    2 * U * (Xha @ (Wh_new.abs() + Wh_old.abs()).T)
            Wq = Wn
        Wa = Wq.abs()
        for a in range(sp.n_a):
            c0, c1 = a * sp.crb_acts, (a + 1) * sp.crb_acts
            Xq = xq64(a_int)
            Xa = Xq.abs()
            yw = Xq @ Wq.T + B
            Pw = Xa @ Wa.T
            y_a = yw - Xq[:, c0:c1] @ Wq[:, c0:c1].T
            P_a = Pw - Xa[:, c0:c1] @ Wa[:, c0:c1].T
            ref = np.zeros((sp.eq_n, 1)); bnd = np.zeros((sp.eq_n, 1))
            xa = X[:, c0:c1]
            for c in range(sp.eq_n):
                xc = xq64_chunk(xa, a_cands[a, 0, c])
                yc = y_a + xc @ Wq[:, c0:c1].T
                Pc = P_a + xc.abs() @ Wa[:, c0:c1].T
                e = Y - yc
                de = g_slab * (Y.abs() + B.abs() + Pc)
                sq, res = _score_terms(e, G, 1.0 / (Oo * tokens), de)
                ref[c], bnd[c] = _finish(np.array([float(sq.sum())]), np.array([float(res.sum())]))
            pick = rep.first_pick(f"round {rnd} X chunk {a}", torch.as_tensor(next(it)).reshape(-1, 1), ref, bnd)
            a_int = a_int.clone()
            a_int[a, 0] = a_cands[a, 0, int(pick[0])]
    rep.intervals = {"w_interval": w_int, "a_interval": a_int}
    return rep


def linear_forward(sp: O.LinearSpec, W, b, x, w_int, a_int):
    """fp64 quant_forward (linear.py:62-67) with the per-element bound γ_{n_seg+2}·(|b| + P)."""
    K, Oo = sp.K, sp.O
    X = x.reshape(-1, K).float()
    qw, qa = sp.w_qmax, sp.a_qmax
    wi = w_int.view(sp.n_V, 1, sp.n_H, 1)
    Wq = (qint(W.view(sp.n_V, sp.crb_rows, sp.n_H, sp.crb_cols), wi, -qw, qw - 1).double() * wi.double()).view(Oo, K)
    xv = X.view(-1, sp.n_a, sp.crb_acts)
    ai = a_int.view(sp.n_a, 1)
    if sp.post_gelu:
        Xq = qint(xv, ai, 0, qa - 1).double() * ai.double() + \
            (xv / sp.a_neg_interval).round_().clamp_(-qa, 0).double() * float(np.float32(sp.a_neg_interval))
    else:
        Xq = qint(xv, ai, -qa, qa - 1).double() * ai.double()
    Xq = Xq.view(-1, K)
    B = torch.zeros(Oo, dtype=torch.float64, device=W.device) if b is None else b.double()
    out = Xq @ Wq.T + B
    bound = gamma(_segments(sp) + 2) * (B.abs() + Xq.abs() @ Wq.abs().T)
    return out, bound


# ---------------------------------------------------------------------------------------------------------- MatMul
def _heads_table(Y, G, out, P, de_coef, kappa, extra_rel=0.0):
    """Per-head score and bound: mean over S3, mean over S1, sum over images (matmul.py:474-480)."""
    w = 1.0 / (Y.shape[2] * Y.shape[3])
    e = Y - out
    de = de_coef * (Y.abs() + P) + kappa * P
    sq, res = _score_terms(e, G, w, de)
    return _finish(sq.sum((0, 2, 3)).cpu().numpy(), res.sum((0, 2, 3)).cpu().numpy(), extra_rel)


def matmul_replay(sp: O.MatMulSpec, A, B, Y, G, tables, *, init_layerwise=False):
    """Replay (SoS)PTQSLBatchingQuantMatMul.calibration_step2 (matmul.py:565-576, :633-644) teacher-forced by the
    logged tables (per round: the A table [eq_n, H] or the split table [20], then the B table [eq_n, H])."""
    dev = A.device
    H, S2 = A.shape[1], A.shape[3]
    Y64, G64 = Y.double(), G.double()
    A64, B64 = A.double(), B.double()
    qA, qB = sp.A_qmax, sp.B_qmax
    if init_layerwise:
        A_int = (A.abs().max() / (qA - 0.5)).view(1).repeat(H).view(1, H, 1, 1, 1, 1, 1)
        B_int = (B.abs().max() / (qB - 0.5)).view(1).repeat(H).view(1, H, 1, 1, 1, 1, 1)
    else:
        A_int, B_int = O.matmul_initial_intervals(sp, A, B)
    f = O.candidate_factors(sp.eq_alpha, sp.eq_beta, sp.eq_n).view(-1, 1, 1, 1, 1, 1, 1, 1).to(dev)
    B_cands = f * B_int.unsqueeze(0)
    hw = lambda t: t.reshape(1, -1, 1, 1)

    def fq64(T, iv, q):
        return qint(T, hw(iv), -q, q - 1).double() * hw(iv).double()

    q1 = qA - 1

    def sos64(split, A_lo_int):
        hi = (A.clamp(split, 1) * q1).round_().clamp_(0, q1).double() / q1
        lo = (A.clamp(0, split) / A_lo_int).round_().clamp_(0, q1).double() * A_lo_int.double()
        return hi + lo

    rep = Replay()
    it = iter(tables)
    g2 = gamma(2 + 4)          # the split-of-softmax steps have two K segments (hi / lo parts); others one
    g1 = gamma(1 + 4)
    if sp.sos:
        split_cands = torch.tensor([2 ** (-i) for i in range(20)], dtype=torch.float32, device=dev)
        split = None
        for rnd in range(sp.search_round):
            ref = np.zeros((20, 1)); bnd = np.zeros((20, 1))
            w = 1.0 / (H * Y.shape[2] * Y.shape[3])
            for i in range(20):
                s = split_cands[i]
                Aq = sos64(s, s / q1)
                out = Aq @ B64
                P = Aq.abs() @ B64.abs()
                de = g2 * (Y64.abs() + P) + 2 * U * 3 * S2 * P
                sq, res = _score_terms(Y64 - out, G64, w, de)
                ref[i], bnd[i] = _finish(np.array([float(sq.sum())]), np.array([float(res.sum())]))
            pick = rep.first_pick(f"round {rnd} split", torch.as_tensor(next(it)).reshape(-1, 1), ref, bnd)
            split = split_cands[int(pick[0])]
            A_int = split / q1
            Aq = sos64(split, A_int)
            ref = np.zeros((sp.eq_n, H)); bnd = np.zeros((sp.eq_n, H))
            for c in range(sp.eq_n):
                Bq = fq64(B, B_cands[c], qB)
                ref[c], bnd[c] = _heads_table(Y64, G64, Aq @ Bq, Aq.abs() @ Bq.abs(), g2, 0.0)
            pick = rep.first_pick(f"round {rnd} B", next(it), ref, bnd)
            B_int = torch.gather(B_cands, 0, torch.as_tensor(pick, device=dev).view(1, 1, -1, 1, 1, 1, 1, 1)).squeeze(0)
        rep.intervals = {"A_interval": A_int, "B_interval": B_int, "split": split}
        return rep
    A_cands = f * A_int.unsqueeze(0)
    for rnd in range(sp.search_round):
        Bq = fq64(B, B_int, qB)
        ref = np.zeros((sp.eq_n, H)); bnd = np.zeros((sp.eq_n, H))
        for c in range(sp.eq_n):
            Aq = fq64(A, A_cands[c], qA)
            ref[c], bnd[c] = _heads_table(Y64, G64, Aq @ Bq, Aq.abs() @ Bq.abs(), g1, 0.0)
        pick = rep.first_pick(f"round {rnd} A", next(it), ref, bnd)
        A_int = torch.gather(A_cands, 0, torch.as_tensor(pick, device=dev).view(1, 1, -1, 1, 1, 1, 1, 1)).squeeze(0)
        Aq = fq64(A, A_int, qA)
        ref = np.zeros((sp.eq_n, H)); bnd = np.zeros((sp.eq_n, H))
        for c in range(sp.eq_n):
            Bq = fq64(B, B_cands[c], qB)
            ref[c], bnd[c] = _heads_table(Y64, G64, Aq @ Bq, Aq.abs() @ Bq.abs(), g1, 0.0)
        pick = rep.first_pick(f"round {rnd} B", next(it), ref, bnd)
        B_int = torch.gather(B_cands, 0, torch.as_tensor(pick, device=dev).view(1, 1, -1, 1, 1, 1, 1, 1)).squeeze(0)
    rep.intervals = {"A_interval": A_int, "B_interval": B_int}
    return rep


def matmul_forward(sp: O.MatMulSpec, A, B, A_int, B_int, split=None):
    """fp64 quant_forward (matmul.py:140-145) with the per-element bound γ_{n_seg+2}·P."""
    q1 = sp.A_qmax - 1
    hw = lambda t: torch.as_tensor(t, device=A.device).reshape(1, -1, 1, 1)
    if sp.sos:
        Aq = (A.clamp(split, 1) * q1).round_().clamp_(0, q1).double() / q1 + \
            (A.clamp(0, split) / A_int).round_().clamp_(0, q1).double() * torch.as_tensor(A_int).double()
        n = 2
    else:
        Aq = qint(A, hw(A_int), -sp.A_qmax, sp.A_qmax - 1).double() * hw(A_int).double()
        n = 1
    Bq = qint(B, hw(B_int), -sp.B_qmax, sp.B_qmax - 1).double() * hw(B_int).double()
    return Aq @ Bq, gamma(n + 2) * (Aq.abs() @ Bq.abs())


# ------------------------------------------------------------------------------------------------------------ Conv
def conv_replay(W, b, x, y, g, table, *, stride, w_bit=8, eq_alpha=0.01, eq_beta=1.2, eq_n=100, chunk=8):
    """Replay ChannelwiseBatchingQuantConv2d.calibration_step2 with a_bit >= 32 (conv.py:591-603): per output channel
    the candidates f_c·Δ⁰[o], im2col by F.unfold, score -Σ_images mean_positions (g·(y - ŷ))²."""
    dev = W.device
    q = 2 ** (w_bit - 1)
    oc = W.shape[0]
    w_int = W.abs().amax([1, 2, 3], keepdim=True) / (q - 0.5)
    f = O.candidate_factors(eq_alpha, eq_beta, eq_n).to(dev)
    cands = f.view(-1, 1, 1, 1, 1) * w_int.unsqueeze(0)
    cols = F.unfold(x.float(), W.shape[2:], stride=stride).double()     # [n, K, L]
    K, L = cols.shape[1], cols.shape[2]
    Y64, G64 = y.reshape(y.shape[0], oc, L).double(), g.reshape(g.shape[0], oc, L).double()
    B = torch.zeros(oc, dtype=torch.float64, device=dev) if b is None else b.double()
    Bb = B.view(1, oc, 1)
    ca = cols.abs()
    ref = np.zeros((eq_n, oc)); bnd = np.zeros((eq_n, oc))
    for p0 in range(0, eq_n, chunk):
        p1 = min(eq_n, p0 + chunk)
        Wq = (qint(W.unsqueeze(0), cands[p0:p1], -q, q - 1).double() * cands[p0:p1].double()).reshape(p1 - p0, 1, oc, K)
        out = torch.matmul(Wq, cols.unsqueeze(0)) + Bb                    # [p, n, oc, L]
        P = torch.matmul(Wq.abs(), ca.unsqueeze(0))
        de = gamma(1 + 4 + 3) * (Y64.abs() + Bb.abs() + P) + 2 * U * 3 * K * P
        sq, res = _score_terms(Y64 - out, G64, 1.0 / L, de)
        ref[p0:p1], bnd[p0:p1] = _finish(sq.sum((1, 3)).cpu().numpy(), res.sum((1, 3)).cpu().numpy(), 3 * U)
    rep = Replay()
    pick = rep.first_pick("conv", table, ref, bnd)
    rep.intervals = {"w_interval": torch.gather(cands, 0, torch.as_tensor(pick, device=dev).view(1, -1, 1, 1, 1)).squeeze(0)}
    return rep


def conv_forward(W, b, x, w_int, *, stride, w_bit=8):
    """fp64 quant_forward of the conv (conv.py:65-70, fp32 activations) with the per-element bound γ_{K+2}·(|b| + P):
    the fp32 input is not integer, so every one of the K products of a dot product may round in the sum."""
    q = 2 ** (w_bit - 1)
    wi = w_int.reshape(-1, 1, 1, 1)
    Wq = (qint(W, wi, -q, q - 1).double() * wi.double()).reshape(W.shape[0], -1)
    cols = F.unfold(x.float(), W.shape[2:], stride=stride).double()            # [n, K, L]
    B = torch.zeros(W.shape[0], dtype=torch.float64, device=W.device) if b is None else b.double()
    out = torch.matmul(Wq, cols) + B.view(1, -1, 1)
    bound = gamma(cols.shape[1] + 2) * (torch.matmul(Wq.abs(), cols.abs()) + B.abs().view(1, -1, 1))
    return out, bound


# ------------------------------------------------------------------------------------------------------ comparison
def check_tables(rep: Replay, what=""):
    """Every entry within its bound, every pick within the bounds of the fp64 argmax.  Returns
    (tables, entries, max |got - ref| / bound, flips) and raises AssertionError naming the first violation."""
    worst, entries, flips = 0.0, 0, 0
    for st in rep.steps:
        err = np.abs(st.got.astype(np.float64) - st.ref)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(st.bound > 0, err / st.bound, np.where(err > 0, np.inf, 0.0))
        r = float(ratio.max())
        worst = max(worst, r)
        entries += st.ref.size
        if r > 1.0:
            c, j = np.unravel_index(int(ratio.argmax()), ratio.shape)
            raise AssertionError(f"{what} {st.name}: entry (cand {c}, group {j}) got {st.got[c, j]:.9e} ref "
                                 f"{st.ref[c, j]:.9e} err/bound {r:.3g}")
        best = st.ref.argmax(0)
        for j, (p, q) in enumerate(zip(st.pick, best)):
            if p != q:
                flips += 1
                gap = st.ref[q, j] - st.ref[p, j]
                if gap > st.bound[p, j] + st.bound[q, j]:
                    raise AssertionError(f"{what} {st.name}: group {j} picked {p}, fp64 argmax {q}, gap {gap:.3e} > "
                                         f"bounds {st.bound[p, j] + st.bound[q, j]:.3e}")
    return len(rep.steps), entries, worst, flips


def check_intervals(rep: Replay, got: dict, what=""):
    """The library's step sizes must equal the replay's bitwise."""
    for k, v in rep.intervals.items():
        a = torch.as_tensor(got[k]).detach().float().cpu().reshape(-1).numpy()
        r = torch.as_tensor(v).detach().float().cpu().reshape(-1).numpy()
        assert a.shape == r.shape and np.array_equal(a.view(np.uint32), r.view(np.uint32)), \
            f"{what} {k}: library {a[:8]} vs fp64 replay {r[:8]}"


def check_forward(got, ref, bound, what=""):
    """Returns max |got - ref| / bound of a quant_forward output."""
    err = (got.double().reshape(ref.shape) - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert ratio <= 1.0, f"{what} quant_forward: err/bound {ratio:.3g}"
    return ratio
