"""BasePTQ test infrastructure (TEST ONLY): the layer-wise EasyQuant conv restated, replayed in fp64, and the UNMODIFIED
reference run through oracle/ref_harness on the same device.

* ``conv_layerwise_calibrate``: plain torch fp32 restatement of ``BatchingEasyQuantConv2d.calibration_step2`` with
  a_bit >= 32 (reference quant_layers/conv.py:279-441), in the style of oracle/ptq_oracle.py's ``conv_calibrate``;
* ``conv_layerwise_replay``: the teacher-forced fp64 replay of the library's layer-wise conv search, with the error model
  of tests/_fp64_ref.py (its ``conv_replay`` summed over the channels);
* ``run_conv_layerwise`` / ``run_reference_calibrator_baseptq``: the reference's class and its calibrator with
  configs/BasePTQ.py (``oracle.ref_harness.load()`` imports it as ``cfg_base``), scores captured by ``capture_argmax``.
"""
from __future__ import annotations

import copy
import importlib
import time

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ptq_oracle as O
from oracle import ref_harness as RH
from tests import _fp64_ref as R

BASE = dict(metric="hessian", eq_alpha=0.5, eq_beta=1.2, eq_n=100)     # configs/BasePTQ.py:13-21 with test_all.py's metric


# ---------------------------------------------------------------------------------------------- oracle restatement
def conv_layerwise_calibrate(W, bias, x, raw_out, raw_grad, stride, padding=0, dilation=1, w_bit=8, eq_alpha=0.5,
                             eq_beta=1.2, eq_n=100):
    """BatchingEasyQuantConv2d.calibration_step2 with a_bit >= 32 (conv.py:429-441): one min-max step size for the whole
    kernel (:313), candidates f_c * delta0 (:432), score = -sum_images mean_positions mean_channels (g*(y - yhat))^2
    (:385-394), the first argmax (:395-396).  The reference passes the input through ``quant_input`` even when
    a_bit = 32 (:383; a_qmax = 2^31, a_interval = max|x| / (2^31 - 0.5), :318), which is restated here: it moves x by
    at most one ulp.  Returns w_interval [1,1,1,1] and the score table [eq_n]."""
    q = 2 ** (w_bit - 1)
    a_qmax = 2 ** 31
    w_int = (W.abs().max() / (q - 0.5)).detach()
    a_int = (x.abs().max() / (a_qmax - 0.5)).detach().view(1)
    x_sim = (x / a_int).round_().clamp_(-a_qmax, a_qmax - 1).mul_(a_int)            # conv.py:64-67 via :383
    cands = O.candidate_factors(eq_alpha, eq_beta, eq_n).to(W.device).view(-1, 1, 1, 1, 1) * w_int
    scores = []
    for c in range(eq_n):
        w_sim = (W / cands[c]).round_().clamp_(-q, q - 1).mul_(cands[c])
        out = F.conv2d(x_sim, w_sim, bias, stride, padding, dilation, 1)
        s = torch.mean(-(raw_grad * (raw_out - out)) ** 2, dim=-3)                   # b, fw, fh   (:344-350)
        scores.append(torch.mean(s, [1, 2]).sum(dim=0))                              # (:388-389)
    scores = torch.stack(scores, 0)
    best = scores.argmax(dim=0).reshape(1, 1, 1, 1, 1)
    return torch.gather(cands, 0, best).squeeze(0), scores


# ---------------------------------------------------------------------------------------------------- fp64 replay
def conv_layerwise_replay(W, b, x, y, g, table, *, stride, w_bit=8, eq_alpha=0.5, eq_beta=1.2, eq_n=100, chunk=8):
    """Replay the library's layer-wise conv search (p4v_conv_desc.layerwise = 1): the channel-wise search of
    tests/_fp64_ref.conv_replay with one Δ⁰ = max|W| / (qmax - 0.5) for every channel, each candidate's per-channel
    sums added in fp64 (negligible) and divided by O·L.  Same per-element error model: Δ⁰ is folded into the targets
    exactly as in the channel-wise search.  ``table`` is [eq_n] or [eq_n, 1]."""
    dev = W.device
    q = 2 ** (w_bit - 1)
    oc = W.shape[0]
    w_int = (W.abs().max() / (q - 0.5)).view(1, 1, 1, 1)
    f = O.candidate_factors(eq_alpha, eq_beta, eq_n).to(dev)
    cands = f.view(-1, 1, 1, 1, 1) * w_int.unsqueeze(0)                                # eq_n+1, 1, 1, 1, 1
    cols = F.unfold(x.float(), W.shape[2:], stride=stride).double()                   # [n, K, L]
    K, L = cols.shape[1], cols.shape[2]
    Y64, G64 = y.reshape(y.shape[0], oc, L).double(), g.reshape(g.shape[0], oc, L).double()
    B = torch.zeros(oc, dtype=torch.float64, device=dev) if b is None else b.double()
    Bb = B.view(1, oc, 1)
    ca = cols.abs()
    ref = np.zeros((eq_n, 1)); bnd = np.zeros((eq_n, 1))
    for p0 in range(0, eq_n, chunk):
        p1 = min(eq_n, p0 + chunk)
        Wq = (R.qint(W.unsqueeze(0), cands[p0:p1], -q, q - 1).double() * cands[p0:p1].double()).reshape(p1 - p0, 1, oc, K)
        out = torch.matmul(Wq, cols.unsqueeze(0)) + Bb                                # [p, n, oc, L]
        P = torch.matmul(Wq.abs(), ca.unsqueeze(0))
        de = R.gamma(1 + 4 + 3) * (Y64.abs() + Bb.abs() + P) + 2 * R.U * 3 * K * P
        sq, res = R._score_terms(Y64 - out, G64, 1.0 / (oc * L), de)
        r, e = R._finish(sq.sum((1, 2, 3)).cpu().numpy(), res.sum((1, 2, 3)).cpu().numpy(), 3 * R.U)
        ref[p0:p1, 0], bnd[p0:p1, 0] = r, e
    rep = R.Replay()
    pick = rep.first_pick("conv_layerwise", np.asarray(torch.as_tensor(table).detach().float().cpu()).reshape(eq_n, 1), ref, bnd)
    rep.intervals = {"w_interval": cands[int(pick[0])].reshape(1, 1, 1, 1)}
    return rep


# -------------------------------------------------------------------------------------------- reference harness
def run_conv_layerwise(x, W, b, y, g, stride, **mod):
    """BatchingEasyQuantConv2d(..., a_bit=32).calibration_step2() of the reference (conv.py:279-441) on the device, its
    score table captured through its one argmax (:395).  Returns dict(w_interval, scores=[table], seconds, module)."""
    Rf = RH.load()
    kw = dict(BASE); kw.update(mod)
    oc, ic, kh, kwid = W.shape
    m = Rf.conv.BatchingEasyQuantConv2d(ic, oc, (kh, kwid), stride=stride, bias=b is not None, a_bit=32, **kw)
    m.weight.data = W.clone()
    if b is not None:
        m.bias.data = b.clone()
    m.to(RH._dev())
    m.raw_input, m.raw_out, m.raw_grad = x.cpu().clone(), y.cpu().clone(), g.cpu().clone()
    scores = []
    RH._sync(); t0 = time.perf_counter()
    with torch.no_grad(), RH.capture_argmax(scores), RH.fp32_convolutions():
        m.calibration_step2()
    RH._sync()
    return dict(w_interval=torch.as_tensor(m.w_interval).detach().float().cpu(), scores=scores,
                seconds=time.perf_counter() - t0, module=m)


def baseptq_hessian(cfg):
    """example/test_all.py:53-78: BasePTQ is run with the Hessian metric."""
    for d in (cfg.ptqsl_conv2d_kwargs, cfg.ptqsl_linear_kwargs, cfg.ptqsl_matmul_kwargs):
        d["metric"] = "hessian"
    return cfg


def run_reference_calibrator_baseptq(net, images, batch_size=4, sequential=False, snapshot=None):
    """HessianQuantCalibrator(...).batching_quant_calib() of the reference with its utils/net_wrap.py and
    configs/BasePTQ.py (metric set to hessian) on a copy of `net`.  Returns (intervals, net copy, wrapped modules)."""
    Rf = RH.load()
    importlib.reload(Rf.cfg_base)
    baseptq_hessian(Rf.cfg_base)
    net_r = copy.deepcopy(net)
    for mod in net_r.modules():
        for leaf in ("matmul1", "matmul2"):
            if hasattr(mod, leaf):
                setattr(mod, leaf, Rf.models.MatMul())
    wrapped = Rf.net_wrap.wrap_modules_in_net(net_r, Rf.cfg_base)
    net_r.to(RH._dev()).eval()
    if snapshot is not None:
        for name, m in wrapped.items():
            orig = m.calibration_step2

            def spy(*a, _orig=orig, _m=m, _name=name, **k):
                d = {}
                if isinstance(_m.raw_input, (list, tuple)):
                    d["A"], d["B"] = _m.raw_input[0].clone(), _m.raw_input[1].clone()
                else:
                    d["x"] = _m.raw_input.clone()
                d["y"] = _m.raw_out.clone()
                d["g"] = _m.raw_grad.clone() if _m.raw_grad is not None else None
                snapshot[_name] = d
                return _orig(*a, **k)
            m.calibration_step2 = spy
    cal = Rf.quant_calib.HessianQuantCalibrator(net_r, wrapped, RH.ListLoader(images), sequential=sequential,
                                                batch_size=batch_size)
    with RH.fp32_convolutions():
        cal.batching_quant_calib()
    importlib.reload(Rf.cfg_base)
    return RH.collect_intervals(wrapped), net_r, wrapped
