"""BasePTQ on the CPU (no GPU): the operator factory against the reference's configs/BasePTQ.py, the layer-wise conv
oracle and fp64 replay pinned to tests/golden/conv_easy_small.npz, the layer-wise conv planning of the C ABI, and the
multi-GPU result rows of a layer-wise conv."""
import ctypes
import importlib
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ptq_oracle as O
from oracle import ref_harness as RH
from ptq4vit_b200.configs import BasePTQ as cfg
from ptq4vit_b200.quant_layers import conv as CV, linear as L, matmul as M
from ptq4vit_b200.utils import quant_calib as Q
from tests import _baseptq_ref as B
from tests import _cases as C
from tests import _fp64_ref as R

needs_ref = pytest.mark.skipif(not RH.available(), reason="reference tree not staged")
GOLD_CONV = os.path.join(C.GOLD, "conv_easy_small.npz")
CONV_FIXTURE = (37, 4, 3, 32, 16, 4)
CONV_ARGS = (3, 768, (16, 16), (16, 16), (0, 0), (1, 1), 1, True, "zeros")       # net_wrap's qconv arguments
TYPES = {"qconv": CONV_ARGS, "qlinear_qkv": (768, 2304), "qlinear_proj": (768, 768), "qlinear_MLP_1": (768, 3072),
         "qlinear_MLP_2": (3072, 768), "qlinear_classifier": (768, 1000), "qlinear_reduction": (1536, 768),
         "qmatmul_qk": (), "qmatmul_scorev": ()}


@pytest.fixture
def fresh_cfg():
    importlib.reload(cfg)
    yield cfg
    importlib.reload(cfg)


# ------------------------------------------------------------------------------------------------- factory contract
@needs_ref
def test_factory_classes_and_kwargs_match_reference(fresh_cfg):
    Rf = RH.load()
    importlib.reload(Rf.cfg_base)
    for name in ("bit", "conv_fc_name_list", "matmul_name_list", "w_bit", "a_bit", "A_bit", "B_bit",
                 "ptqsl_conv2d_kwargs", "ptqsl_linear_kwargs", "ptqsl_matmul_kwargs"):
        assert getattr(fresh_cfg, name) == getattr(Rf.cfg_base, name), name
    for t, args in TYPES.items():
        ours, ref = fresh_cfg.get_module(t, *args), Rf.cfg_base.get_module(t, *args)
        assert type(ours).__name__ == type(ref).__name__, t
        for attr in ("metric", "eq_alpha", "eq_beta", "eq_n", "search_round", "n_V", "n_H", "n_a", "w_bit", "a_bit",
                     "A_bit", "B_bit", "n_G_A", "n_G_B"):
            if hasattr(ref, attr):
                assert getattr(ours, attr) == getattr(ref, attr), f"{t}.{attr}"
    importlib.reload(Rf.cfg_base)


def test_factory_dispatch(fresh_cfg):
    assert fresh_cfg.ptqsl_conv2d_kwargs["metric"] == "cosine" and fresh_cfg.ptqsl_linear_kwargs["eq_alpha"] == 0.5
    conv = fresh_cfg.get_module("qconv", *CONV_ARGS)
    assert type(conv) is CV.BatchingEasyQuantConv2d and conv.a_bit == 32 and (conv.n_V, conv.n_H) == (1, 1)
    assert conv.layerwise and not CV.ChannelwiseBatchingQuantConv2d.layerwise
    for t in ("qlinear_qkv", "qlinear_proj", "qlinear_MLP_1", "qlinear_MLP_2", "qlinear_classifier"):
        assert type(fresh_cfg.get_module(t, *TYPES[t])) is L.PTQSLBatchingQuantLinear, t      # no post-GELU class
    for t in ("qmatmul_qk", "qmatmul_scorev"):
        assert type(fresh_cfg.get_module(t)) is M.PTQSLBatchingQuantMatMul, t                # no split-of-softmax
    assert fresh_cfg.get_module("qlinear_qkv", 768, 2304).n_V == 3
    assert fresh_cfg.get_module("qlinear_classifier", 768, 1000).n_V == 1
    fresh_cfg.ptqsl_linear_kwargs["n_V"] = 2
    assert fresh_cfg.get_module("qlinear_qkv", 768, 2304).n_V == 6
    assert fresh_cfg.get_module("qlinear_classifier", 768, 1000).n_V == 2          # unlike PTQ4ViT, kept as given
    with pytest.raises(NotImplementedError, match="unknown module type"):
        fresh_cfg.get_module("qbogus")


def test_edits_before_get_module_take_effect(fresh_cfg):
    B.baseptq_hessian(fresh_cfg)
    fresh_cfg.ptqsl_conv2d_kwargs["eq_n"] = 7
    fresh_cfg.ptqsl_matmul_kwargs["search_round"] = 2
    fresh_cfg.w_bit["qconv"] = 6
    fresh_cfg.a_bit["qlinear_proj"] = 4
    conv = fresh_cfg.get_module("qconv", *CONV_ARGS)
    assert conv.metric == "hessian" and conv.eq_n == 7 and conv.w_bit == 6
    assert fresh_cfg.get_module("qlinear_proj", 768, 768).a_bit == 4
    assert fresh_cfg.get_module("qmatmul_qk").search_round == 2


def test_wrapped_vit_uses_baseptq_classes(fresh_cfg):
    from ptq4vit_b200.utils.models import VisionTransformer
    from ptq4vit_b200.utils.net_wrap import wrap_modules_in_net
    net = VisionTransformer(**RH.TINY_VIT)
    wrapped = wrap_modules_in_net(net, fresh_cfg)
    assert len(wrapped) == 1 + 2 * 6 + 1
    assert type(net.patch_embed.proj) is CV.BatchingEasyQuantConv2d
    assert type(net.blocks[0].mlp.fc2) is L.PTQSLBatchingQuantLinear
    assert type(net.blocks[0].attn.matmul2) is M.PTQSLBatchingQuantMatMul
    assert net(torch.randn(2, 3, 32, 32)).shape == (2, 10)          # raw mode


def test_restrictions_raise():
    m = CV.BatchingEasyQuantConv2d(3, 8, 4, stride=4, a_bit=8, metric="hessian")
    with pytest.raises(NotImplementedError, match="a_bit >= 32"):
        m.calibration_step2()
    m = CV.BatchingEasyQuantConv2d(4, 8, 4, stride=4, groups=2, a_bit=32, metric="hessian")
    with pytest.raises(NotImplementedError, match="groups"):
        m.calibration_step2()
    m = CV.BatchingEasyQuantConv2d(3, 8, 4, stride=4, a_bit=32, metric="hessian")
    x, W, b, y, g = O.make_conv_fixture(1, 2, 3, 8, 8, 4)
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    with pytest.raises(RuntimeError, match="CUDA"):
        m.calibration_step2()
    m = CV.BatchingEasyQuantConv2d(3, 8, 4, stride=4, a_bit=32, metric="cosine")
    with pytest.raises(NotImplementedError, match="cosine"):
        m.calibration_step2()


# ---------------------------------------------------------------------------------------- oracle and fp64 replay
def test_layerwise_oracle_reproduces_golden():
    z = np.load(GOLD_CONV)
    x, W, b, y, g = O.make_conv_fixture(*CONV_FIXTURE)
    wi, scores = B.conv_layerwise_calibrate(W, b, x, y, g, stride=4)
    C.assert_scores_close(scores.numpy(), z["scores_000"], 2e-4, "conv_easy_small")
    assert int(scores.argmax()) == int(np.argmax(z["scores_000"]))
    assert wi.shape == (1, 1, 1, 1) and float(wi) == float(z["w_interval"].reshape(-1)[0])


@pytest.fixture(scope="module")
def replay():
    z = np.load(GOLD_CONV)
    x, W, b, y, g = O.make_conv_fixture(*CONV_FIXTURE)
    return z, R.Replay, B.conv_layerwise_replay(W, b, x, y, g, z["scores_000"], stride=4)


def test_layerwise_replay_pinned_to_golden(replay):
    z, _, rep = replay
    assert len(rep.steps) == 1
    C.assert_scores_close(rep.steps[0].ref[:, 0], z["scores_000"], 2e-4, "conv_easy_small replay")
    R.check_intervals(rep, {"w_interval": torch.from_numpy(z["w_interval"])}, "conv_easy_small")
    R.check_tables(rep, "conv_easy_small")      # the reference's fp32 table lies within the library's error bound


def test_layerwise_replay_rejects_shifted_entry(replay):
    z, Replay, rep = replay
    st = rep.steps[0]
    c = int(st.ref[:, 0].argmax())
    t = st.ref.astype(np.float32).copy()
    t[c, 0] = np.float32(st.ref[c, 0] - 10 * st.bound[c, 0])
    bad = Replay(intervals=rep.intervals)
    bad.first_pick(st.name, t, st.ref, st.bound)
    with pytest.raises(AssertionError, match="err/bound"):
        R.check_tables(bad)


def test_layerwise_replay_rejects_step_one_grid_point_off(replay):
    z, _, rep = replay
    x, W, b, y, g = O.make_conv_fixture(*CONV_FIXTURE)
    d0 = W.abs().max() / 127.5
    f = O.candidate_factors(0.5, 1.2, 100)
    i = int(np.argmax(z["scores_000"]))
    off = (f[i + 1] * d0).reshape(1, 1, 1, 1)
    with pytest.raises(AssertionError, match="w_interval"):
        R.check_intervals(rep, {"w_interval": off})


# ------------------------------------------------------------------------------------------------------ ABI planning
@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


def _cdesc(**kw):
    from ptq4vit_b200 import _lib
    d = _lib.ConvDesc()
    base = dict(images=32, out_channels=768, K=3 * 16 * 16, positions=14 * 14, w_bit=8, eq_n=100, eq_alpha=0.5,
                eq_beta=1.2, has_bias=1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("shape", [dict(), dict(images=32, out_channels=128, K=48, positions=56 * 56),
                                   dict(images=3, out_channels=7, K=5, positions=3, eq_n=1)])
def test_layerwise_workspace_not_larger_than_channelwise(lib, shape):
    n_c, n_l = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.p4v_conv_workspace_bytes(ctypes.byref(_cdesc(**shape)), ctypes.byref(n_c)) == 0, lib.p4v_last_error()
    assert lib.p4v_conv_workspace_bytes(ctypes.byref(_cdesc(layerwise=1, **shape)), ctypes.byref(n_l)) == 0, lib.p4v_last_error()
    assert 0 < n_l.value <= n_c.value


@pytest.mark.parametrize("bad,msg", [(dict(layerwise=2), "layerwise"), (dict(layerwise=-1), "layerwise"),
                                     (dict(layerwise=1, w_bit=9), "w_bit"), (dict(layerwise=1, eq_n=0), "eq_n"),
                                     (dict(layerwise=1, positions=0), "empty"), (dict(layerwise=1, kernel=1), "tensor-core")])
def test_bad_layerwise_descriptors_fail_loudly(lib, bad, msg):
    n = ctypes.c_size_t()
    assert lib.p4v_conv_workspace_bytes(ctypes.byref(_cdesc(**bad)), ctypes.byref(n)) != 0
    assert msg in lib.p4v_last_error().decode()
    rc = lib.p4v_conv_calibrate(ctypes.byref(_cdesc(**bad)), None, None, None, None, None, None, 0, None, None, None)
    assert rc != 0 and msg in lib.p4v_last_error().decode()


def test_layerwise_null_pointers_are_rejected_before_any_launch(lib):
    before = lib.p4v_launch_count()
    rc = lib.p4v_conv_calibrate(ctypes.byref(_cdesc(layerwise=1)), None, None, None, None, None, None, 0, None, None, None)
    assert rc != 0 and "null" in lib.p4v_last_error().decode()
    assert lib.p4v_launch_count() == before


def test_min_search_workspace_passes_the_layerwise_flag(lib):
    conv_l = CV.BatchingEasyQuantConv2d(3, 768, 16, stride=16, a_bit=32, eq_n=100, eq_alpha=0.5, eq_beta=1.2)
    conv_c = CV.ChannelwiseBatchingQuantConv2d(3, 768, 16, stride=16, a_bit=32, eq_n=100, eq_alpha=0.5, eq_beta=1.2)
    shapes = {"positions": 196, "conv_K": 768}
    n_l = Q.min_search_workspace_bytes(conv_l, 32, shapes)
    n_c = Q.min_search_workspace_bytes(conv_c, 32, shapes)
    n = ctypes.c_size_t()
    assert lib.p4v_conv_workspace_bytes(ctypes.byref(_cdesc(layerwise=1)), ctypes.byref(n)) == 0
    assert n_l == n.value + 4 * 32 * 196 * 768 and n_l < n_c


# ------------------------------------------------------------------------------------------------ multi-GPU rows
def test_pack_unpack_roundtrip_layerwise_conv():
    conv = CV.BatchingEasyQuantConv2d(3, 40, 4, stride=4, a_bit=32)
    conv.w_interval = torch.tensor(0.0123).view(1, 1, 1, 1); conv.a_interval = torch.tensor([7.0])
    assert Q.result_width([conv]) == 2
    row = Q.pack_result(conv, 5)
    conv2 = CV.BatchingEasyQuantConv2d(3, 40, 4, stride=4, a_bit=32)
    Q.unpack_result(conv2, row)
    assert conv2.w_interval.shape == (1, 1, 1, 1) and torch.equal(conv2.w_interval, conv.w_interval)
    assert torch.equal(conv2.a_interval, conv.a_interval) and conv2.calibrated


def _gather_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    net = torch.nn.Linear(2, 2)
    mods = {f"lin{i}": L.PTQSLBatchingQuantLinear(32, 96, n_V=3 if i == 0 else 1, n_H=1, n_a=1) for i in range(4)}
    mods["mm"] = M.PTQSLBatchingQuantMatMul()
    mods["conv"] = CV.BatchingEasyQuantConv2d(3, 40, 4, stride=4, a_bit=32)
    names = list(mods)
    owner = Q.shard_modules(names, [1.0 + i for i in range(len(names))], world)
    for i, n in enumerate(names):
        if owner[n] == rank:
            if n == "conv":
                mods[n].w_interval = torch.tensor(0.25).view(1, 1, 1, 1)
                mods[n].a_interval = torch.tensor([7.0])
            elif n == "mm":
                mods[n].n_G_B = 4
                mods[n].A_interval = torch.full((1, 4, 1, 1, 1, 1, 1), 10.0 + i)
                mods[n].B_interval = torch.full((1, 4, 1, 1, 1, 1, 1), 20.0 + i)
            else:
                m = mods[n]
                m.w_interval = torch.full((m.n_V, 1, 1, 1), float(i)); m.a_interval = torch.full((1, 1), 100.0 + i)
    cal = Q.HessianQuantCalibrator(net, mods, [], distributed=dist)
    cal._gather(owner)
    ok = all(float(mods[f"lin{i}"].w_interval.mean()) == float(i) and float(mods[f"lin{i}"].a_interval) == 100.0 + i
             for i in range(4))
    ok = ok and mods["lin0"].w_interval.shape == (3, 1, 1, 1)
    ok = ok and float(mods["mm"].B_interval.mean()) == 24.0
    c = mods["conv"]
    ok = ok and c.w_interval.shape == (1, 1, 1, 1) and float(c.w_interval) == 0.25 and float(c.a_interval) == 7.0
    ret[rank] = ok
    dist.destroy_process_group()


def test_two_rank_gloo_gather_of_baseptq_step_sizes():
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = 29500 + (os.getpid() + 977) % 2000
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p_ in procs:
        p_.start()
    for p_ in procs:
        p_.join(120)
        assert p_.exitcode == 0
    assert ret[0] and ret[1]
