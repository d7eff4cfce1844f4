"""Every search step against the teacher-forced fp64 evaluator (tests/_fp64_ref.py), at shapes on both sides of the
planner's path choices and at the production shapes the README claims (Swin window attention and patch embedding,
DeiT-B/384 attention).

Each case runs the public class with ``keep_scores=True``, replays the search in fp64 on the same device, and checks
every table entry against the error model, every pick, the final step sizes bitwise and ``quant_forward``.  It also
asserts, from the launch record (``p4v_profile_collect_launches``), the path each case is named for: Gram GEMM or slab
sweeps, int8 or bf16, consumer mode, resident row operand / weight tile and buffers, tail wave; so a planner change
cannot quietly route a case elsewhere.  With ``P4V_PARITY_JSON=<path>`` the per-case ratios max |got - ref| / bound
and the observed launch paths are written there as JSON."""
import ctypes
import json
import os

import pytest
import torch

from oracle import ptq_oracle as O
from oracle import ref_harness as RH
from tests import _fp64_ref as R

pytestmark = pytest.mark.gpu

REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("P4V_PARITY_JSON")
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


LAUNCH_COLS = ("kind", "simt", "mode", "n_stages", "resident_bufs", "rres_bytes", "cres_bytes", "grid", "tiles", "n_cand",
               "cand_groups", "cand_jobs")
MODES = {0: "multi", 1: "single", 2: "pair"}


def _profiled(run):
    """Run ``run()`` with the launch profile on; returns (result, [bf16 sweeps, int8 sweeps, Gram GEMMs], launch rows)
    where every row is what p4v_profile_collect_launches reports for one launch (LAUNCH_COLS)."""
    from ptq4vit_b200 import _lib
    lib = _lib.lib()
    prof = (ctypes.c_double * 12)()
    lib.p4v_profile_collect_kinds(prof, 12)
    lib.p4v_profile_enable(1)
    try:
        with torch.no_grad():
            out = run()
        torch.cuda.synchronize()
    finally:
        lib.p4v_profile_enable(0)
    n = ctypes.c_int()
    _lib.check(lib.p4v_profile_collect_launches(None, 0, ctypes.byref(n)), "p4v_profile_collect_launches")
    buf = (ctypes.c_double * (n.value * len(LAUNCH_COLS)))()
    _lib.check(lib.p4v_profile_collect_launches(buf, n.value, ctypes.byref(n)), "p4v_profile_collect_launches")
    rows = [dict(zip(LAUNCH_COLS, (int(v) for v in buf[i * len(LAUNCH_COLS):(i + 1) * len(LAUNCH_COLS)])))
            for i in range(n.value)]
    lib.p4v_profile_collect_kinds(prof, 12)
    return out, [int(prof[6]), int(prof[7]), int(prof[8])], rows


def _observed(rows):
    """The paths the launches took, from the launch record."""
    sweeps = [r for r in rows if r["kind"] in (0, 1)]
    res = [r for r in sweeps if r["rres_bytes"] > 0]
    cand = [r for r in sweeps if r["n_cand"] > 1]
    return {"modes": sorted({MODES[r["mode"]] for r in sweeps if r["mode"] >= 0 and r["cand_groups"] > 0}),
            "int8_sweeps": sum(r["kind"] == 1 for r in rows), "bf16_sweeps": sum(r["kind"] == 0 for r in rows),
            "gram_gemms": sum(r["kind"] == 2 for r in rows), "simt": any(r["simt"] for r in sweeps),
            "cres": any(r["cres_bytes"] > 0 for r in sweeps), "rres": bool(res),
            "resident_bufs": sorted({r["resident_bufs"] for r in res}),
            "max_stages": max((r["n_stages"] for r in sweeps), default=0),
            "tail": any(r["tiles"] % r["grid"] != 0 for r in cand)}


def _assert_paths(obs, expect, name):
    for k, v in expect.items():
        if k == "mode":
            assert v in obs["modes"], f"{name}: no {v} consumer launch (modes {obs['modes']})"
        elif k == "resident_bufs":
            assert obs["resident_bufs"] == [v], f"{name}: resident buffers {obs['resident_bufs']}, expected {v}"
        else:
            assert obs[k] == v, f"{name}: {k} = {obs[k]}, expected {v}"


def _record(name, rep, obs, fwd_ratio):
    n, entries, worst, flips = R.check_tables(rep, name)
    REPORT[name] = {"launches": obs, "tables": n, "entries": entries, "max_err_over_bound": worst,
                    "pick_flips_within_bound": flips, "steps_bitwise": True, "quant_forward_err_over_bound": fwd_ratio}
    return worst


# ------------------------------------------------------------------------------------------------------------ Linear
# name: (K, O, n_V, n_H, n_a, images, tokens, options)
LINEAR = {
    "gram_ks4": (96, 64, 4, 24, 1, 3, 50, {}),
    "gram_ks60": (240, 96, 2, 4, 1, 2, 130, {}),
    "gram_ks64_int8": (128, 200, 1, 2, 1, 4, 33, {}),
    "slab_ks30": (120, 80, 5, 4, 1, 4, 65, {}),
    "slab_ks68": (272, 128, 2, 4, 1, 4, 65, {}),
    "odd": (75, 37, 1, 3, 1, 3, 41, {"bias": False}),
    "odd_int8": (75, 37, 1, 3, 1, 3, 41, {"bias": False, "operand": "int8"}),
    "misaligned_chunks": (96, 64, 4, 4, 3, 4, 50, {}),
    "gram_na2": (128, 64, 4, 8, 2, 4, 50, {}),
    # post-GELU weight steps, 224 B = 128 + 96 per part: two jobs per candidate group, both parts resident (56 KB, under
    # 60 KB).  With n_H = 1 only the candidate slab streams and the ring has the 2 + 1 stages the pair consumer holds;
    # with n_H = 2 the fixed block streams both operands, the ring gets 2 stages and the step stays multi-segment.
    "postgelu_pair2_w8a8": (224, 128, 2, 1, 1, 4, 65, {"post_gelu": True, "expect": {"mode": "pair", "rres": True}}),
    "postgelu_pair2_w4a4": (224, 128, 2, 1, 1, 4, 65, {"post_gelu": True, "w_bit": 4, "a_bit": 4,
                                                      "expect": {"mode": "pair", "rres": True}}),
    "postgelu_pair2_short_ring": (448, 128, 2, 2, 1, 4, 65, {"post_gelu": True,
                                                            "expect": {"modes": ["multi"], "rres": True}}),
    "postgelu_bf16_a3": (96, 64, 4, 4, 1, 4, 33, {"post_gelu": True, "a_bit": 3, "expect": {"mode": "pair"}}),
    "low_bits_w2a2": (128, 128, 2, 4, 1, 4, 65, {"w_bit": 2, "a_bit": 2}),
    "low_bits_w3a5": (128, 128, 2, 4, 1, 4, 65, {"w_bit": 3, "a_bit": 5}),
    "low_bits_w4a8": (128, 128, 2, 4, 1, 4, 65, {"w_bit": 4, "a_bit": 8}),
    "low_bits_w5a4": (128, 128, 2, 4, 1, 4, 65, {"w_bit": 5, "a_bit": 4}),
    "eq_n1_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_n": 1}),
    "eq_n7_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_n": 7}),
    "eq_n8_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_n": 8}),
    "eq_n9_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_n": 9}),
    "eq_n128_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_n": 128}),
    "eq_n7_slab": (272, 128, 2, 4, 1, 4, 65, {"eq_n": 7}),
    "eq_n128_slab": (272, 128, 2, 4, 1, 4, 65, {"eq_n": 128}),
    "eq_range_half_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_alpha": 0.5, "eq_beta": 1.0}),
    "eq_alpha0_slab": (272, 128, 2, 4, 1, 4, 65, {"eq_alpha": 0.0, "eq_beta": 1.0}),
    "eq_alpha0_gram": (96, 64, 4, 24, 1, 3, 50, {"eq_alpha": 0.0, "eq_beta": 1.0}),
    # int8 weight tile of 800 B x 128 rows = 100 KB stays resident in the activation steps; 832 B does not
    "cres_k800": (800, 128, 1, 1, 1, 2, 65, {"expect": {"cres": True}}),
    "cres_k832": (832, 128, 1, 1, 1, 2, 65, {"expect": {"cres": False}}),
    # weight-step row operand: 480 B x 128 rows = 60 KB stays resident (one buffer: two do not leave 3 ring stages);
    # 512 B streams
    "rres_k960": (960, 128, 1, 2, 1, 2, 65, {"expect": {"rres": True, "resident_bufs": 1, "mode": "single"}}),
    "rres_k1024": (1024, 128, 1, 2, 1, 2, 65, {"expect": {"rres": False, "mode": "single"}}),
    "rows_7": (64, 128, 2, 2, 1, 7, 0, {}),
    "rows_129": (64, 128, 2, 2, 1, 3, 43, {}),
    # 128·SMs rows, O = 128: whole waves; one tile more: a tail wave split at candidate granularity
    "rows_128sms": (64, 128, 2, 2, 1, "sms", 128, {"rounds": 1, "expect": {"tail": False}}),
    "rows_128sms_plus1": (64, 128, 2, 2, 1, "sms+1", 128, {"rounds": 1, "expect": {"tail": True}}),
    # P4V_MAX_GROUPS = 96 segments in the activation step: at the limit
    "many_segments_96": (384, 64, 4, 96, 1, 2, 65, {"rounds": 1}),
    # int8 activation step of a bf16 layer (ks = 32): with one 128-row tile and O = 1024 the int8 candidate planes and
    # the int8 weight copy fit in the bf16 candidate region from eq_n = 9 on (9·96 KB + 8·96 KB <= 9·192 KB), not at 8
    "x8_fit_eq_n8": (768, 1024, 4, 24, 1, 1, 100, {"eq_n": 8, "rounds": 1, "expect": {"int8_sweeps": 0}}),
    "x8_fit_eq_n9": (768, 1024, 4, 24, 1, 1, 100, {"eq_n": 9, "rounds": 1, "x8": True}),
    "init_layerwise": (96, 64, 4, 4, 3, 4, 50, {"init_layerwise": True}),
    "l2_slab": (120, 80, 5, 4, 1, 4, 65, {"metric": "L2_norm"}),
    "linear_weighted_gram": (96, 64, 4, 24, 1, 3, 50, {"metric": "linear_weighted_L2_norm"}),
    "square_weighted_slab": (120, 80, 5, 4, 1, 4, 65, {"metric": "square_weighted_L2_norm"}),
    "chunked2_gram_ks60": (240, 96, 2, 4, 1, 2, 130, {"chunks": 2}),
    "chunked3_gram_ks60": (240, 96, 2, 4, 1, 2, 130, {"chunks": 3}),
    "chunked2_postgelu_pair2": (224, 128, 2, 1, 1, 4, 65, {"post_gelu": True, "chunks": 2, "expect": {"mode": "pair"}}),
    "chunked3_postgelu_pair2": (224, 128, 2, 1, 1, 4, 65, {"post_gelu": True, "chunks": 3, "expect": {"mode": "pair"}}),
}


@pytest.mark.parametrize("name", sorted(LINEAR))
def test_linear_against_fp64(name, monkeypatch):
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers._metric import metric_weight
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear, PostGeluPTQSLBatchingQuantLinear
    K, Oo, n_V, n_H, n_a, n_img, n_tok, o = LINEAR[name]
    n_img = {"sms": _sms(), "sms+1": _sms() + 1}.get(n_img, n_img)
    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    monkeypatch.setenv("P4V_OPERAND", o.get("operand", "auto"))
    post_gelu = o.get("post_gelu", False)
    sp = O.LinearSpec(K, Oo, n_V=n_V, n_H=n_H, n_a=n_a, w_bit=o.get("w_bit", 8), a_bit=o.get("a_bit", 8),
                      eq_alpha=o.get("eq_alpha", 0.01), eq_beta=o.get("eq_beta", 1.2), eq_n=o.get("eq_n", 100),
                      search_round=o.get("rounds", 2), post_gelu=post_gelu)
    x, W, b, y, g = [None if t is None else t.cuda() for t in
                     O.make_linear_fixture(100 + len(name), n_img, n_tok, K, Oo, post_gelu=post_gelu, bias=o.get("bias", True))]
    metric = o.get("metric", "hessian")
    cls = PostGeluPTQSLBatchingQuantLinear if post_gelu else PTQSLBatchingQuantLinear
    m = cls(K, Oo, bias=b is not None, metric=metric, eq_alpha=sp.eq_alpha, eq_beta=sp.eq_beta, eq_n=sp.eq_n,
            search_round=sp.search_round, n_V=n_V, n_H=n_H, n_a=n_a, w_bit=o.get("w_bit", 8), a_bit=o.get("a_bit", 8),
            init_layerwise=o.get("init_layerwise", False))
    m.weight.data = W.clone()
    if b is not None:
        m.bias.data = b.clone()
    m.cuda()
    m.keep_scores = True
    if "chunks" in o:
        rows = x.shape[0] * max(1, n_tok)
        d = m._desc(rows, max(1, n_tok), m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
        d.rows_per_chunk = -(-rows // (128 * o["chunks"])) * 128
        nb = ctypes.c_size_t()
        _lib.check(_lib.lib().p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(nb)), "workspace")
        monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(nb.value))
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    _, launches, rows = _profiled(m.calibration_step2)
    obs = _observed(rows)
    _assert_paths(obs, o.get("expect", {}), name)
    if o.get("x8"):
        assert launches[1] >= sp.search_round, "the activation steps of a bf16 layer run on int8 images"
    if "chunks" in o:
        assert m.calib_chunks == o["chunks"]
    gram = R.gram_path(sp)
    assert (launches[2] > 0) == gram, f"Gram GEMM launches {launches[2]}, expected the {'Gram' if gram else 'slab'} path"
    if o.get("operand") == "int8":
        assert launches[0] == 0 and launches[1] > 0
    if o.get("operand") is None:
        if min(R.segment_lengths(sp)) >= 64:
            assert launches[0] == 0 and launches[1] > 0, "segments of >= 64 elements: every sweep runs int8"
        else:
            assert launches[0] > 0, "a segment under 64 elements: the layer's type is bf16"
            if n_a == 1 and not post_gelu and sp.eq_n >= 100:
                # Segments are padded to 32 bytes: up to 16 elements the int8 candidate planes are as large as the bf16
                # ones, so the weight copy of the int8 activation step does not fit beside them and the step stays bf16.
                if min(R.segment_lengths(sp)) > 16:
                    assert launches[1] >= sp.search_round, "the activation steps of a bf16 layer run on int8 images"
                elif max(R.segment_lengths(sp)) <= 16:
                    assert launches[1] == 0, "int8 activation step planned although it does not fit"
    gw = metric_weight(metric, y, g, "test")
    rep = R.linear_replay(sp, W, b, x, y, gw, m.last_scores, gram=gram, init_layerwise=o.get("init_layerwise", False))
    R.check_intervals(rep, {"w_interval": m.w_interval, "a_interval": m.a_interval}, name)
    m.mode = "quant_forward"
    with torch.no_grad():
        out = m(x)
    ref, bound = R.linear_forward(sp, W, b, x, m.w_interval, m.a_interval)
    fr = R.check_forward(out.reshape(ref.shape), ref, bound, name)
    _record(f"linear/{name}", rep, obs, fr)


def test_linear_too_many_segments_is_refused():
    """97 segments in one activation step exceed P4V_MAX_GROUPS: the library refuses before any launch."""
    from ptq4vit_b200 import _lib
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    x, W, b, y, g = [t.cuda() for t in O.make_linear_fixture(7, 2, 65, 388, 64)]
    m = PTQSLBatchingQuantLinear(388, 64, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=1,
                                 n_V=4, n_H=97, n_a=1)
    m.weight.data = W.clone(); m.bias.data = b.clone(); m.cuda()
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    before = _lib.lib().p4v_launch_count()
    with pytest.raises(_lib.NativeError, match="too many K segments"):
        m.calibration_step2()
    assert _lib.lib().p4v_launch_count() == before


# ------------------------------------------------------------------------------------------------------------ MatMul
# name: (images, heads, S1, S2, S3, split-of-softmax, options)
MATMUL = {
    "swinb384_mm1": (4, 4, 144, 32, 144, False, {}),
    "swinb384_mm2_sos": (4, 4, 144, 144, 32, True, {}),
    "swint224_mm1": (4, 3, 49, 32, 49, False, {}),
    "swint224_mm2_sos": (4, 3, 49, 49, 32, True, {}),
    "deitb384_mm1": (2, 12, 577, 64, 577, False, {"rounds": 1}),
    "deitb384_mm2_sos": (2, 12, 577, 577, 64, True, {"rounds": 1}),
    "deitb384_mm2_sos_bf16": (2, 12, 577, 577, 64, True, {"rounds": 1, "operand": "bf16"}),
    "tiny_s2_1": (3, 2, 1, 1, 1, False, {}),
    "tiny_s2_16": (3, 2, 1, 16, 1, False, {}),
    "bits_a2b2": (4, 3, 49, 32, 49, False, {"A_bit": 2, "B_bit": 2}),
    "bits_a4b4_sos": (4, 3, 49, 49, 32, True, {"A_bit": 4, "B_bit": 4}),
    "eq_n1_sos": (4, 3, 49, 49, 32, True, {"eq_n": 1}),
    "eq_n7_sos": (4, 3, 49, 49, 32, True, {"eq_n": 7}),
    "eq_n128": (4, 3, 49, 32, 49, False, {"eq_n": 128}),
    "init_layerwise_swin": (4, 4, 144, 32, 144, False, {"init_layerwise": True}),
    "chunks2_swint224_mm1": (6, 3, 49, 32, 49, False, {"chunks": 2}),
    "chunks3_swint224_mm1": (6, 3, 49, 32, 49, False, {"chunks": 3}),
    "chunks2_swint224_mm2_sos": (6, 3, 49, 49, 32, True, {"chunks": 2}),
    "chunks3_swint224_mm2_sos": (6, 3, 49, 49, 32, True, {"chunks": 3}),
}


@pytest.mark.parametrize("name", sorted(MATMUL))
def test_matmul_against_fp64(name, monkeypatch):
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul, SoSPTQSLBatchingQuantMatMul
    n_img, H, S1, S2, S3, sos, o = MATMUL[name]
    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    monkeypatch.setenv("P4V_OPERAND", o.get("operand", "auto"))
    sp = O.MatMulSpec(A_bit=o.get("A_bit", 8), B_bit=o.get("B_bit", 8), eq_n=o.get("eq_n", 100),
                      search_round=o.get("rounds", 2), sos=sos)
    A, B, Y, G = [t.cuda() for t in O.make_matmul_fixture(200 + len(name), n_img, H, S1, S2, S3, softmax_A=sos)]
    cls = SoSPTQSLBatchingQuantMatMul if sos else PTQSLBatchingQuantMatMul
    m = cls(A_bit=o.get("A_bit", 8), B_bit=o.get("B_bit", 8), metric="hessian", eq_alpha=sp.eq_alpha,
            eq_beta=sp.eq_beta, eq_n=sp.eq_n, search_round=sp.search_round, init_layerwise=o.get("init_layerwise", False))
    m.keep_scores = True
    if "chunks" in o:
        from ptq4vit_b200 import _lib
        d = m._desc(A, B, m.search_round, (m.eq_alpha, m.eq_beta, m.eq_n))
        d.images_per_chunk = -(-n_img // o["chunks"])
        nb = ctypes.c_size_t()
        _lib.check(_lib.lib().p4v_matmul_workspace_bytes(ctypes.byref(d), ctypes.byref(nb)), "workspace")
        monkeypatch.setenv("P4V_WORKSPACE_BUDGET", str(nb.value))
    m.raw_input, m.raw_out, m.raw_grad = [A, B], Y, G
    _, launches, rows = _profiled(m.calibration_step2)
    obs = _observed(rows)
    if "chunks" in o:
        assert m.calib_chunks == o["chunks"]
    assert launches[2] == 0
    if S2 < 64 or o.get("operand") == "bf16":
        assert launches[1] == 0, "a K segment under 64 elements (or bf16 forced) keeps the MatMul on bf16"
    elif o.get("operand") is None:
        assert launches[1] > 0, "S2 >= 64: the A / B steps run on int8 images"
    if sos:
        assert launches[0] > 0, "the split search multiplies the 3-term bf16 split of B"
        if S2 <= 144:    # both parts of A resident (at most 160 B x 128 rows each): the B steps run as pairs
            assert "pair" in obs["modes"], f"split-of-softmax B steps did not run in pair mode ({obs['modes']})"
    else:
        assert obs["modes"] == ["single"]
    rep = R.matmul_replay(sp, A, B, Y, G, m.last_scores, init_layerwise=o.get("init_layerwise", False))
    got = {"A_interval": m.A_interval, "B_interval": m.B_interval}
    if sos:
        got["split"] = m.split
    R.check_intervals(rep, got, name)
    m.mode = "quant_forward"
    with torch.no_grad():
        out = m(A, B)
    ref, bound = R.matmul_forward(sp, A, B, m.A_interval, m.B_interval, m.split if sos else None)
    fr = R.check_forward(out, ref, bound, name)
    _record(f"matmul/{name}", rep, obs, fr)


# -------------------------------------------------------------------------------------------------------------- Conv
# name: (images, ic, oc, size, kernel = stride, options)
CONV = {
    "swin_patch4": (2, 3, 128, 96, 4, {}),
    "vit_patch16_oc96": (4, 3, 96, 64, 16, {}),
    "swin_patch4_w2": (2, 3, 128, 96, 4, {"w_bit": 2}),
    "swin_patch4_w4": (2, 3, 128, 96, 4, {"w_bit": 4}),
    "vit_patch16_eq_n7": (4, 3, 96, 64, 16, {"eq_n": 7}),
    "vit_patch16_eq_n128": (4, 3, 96, 64, 16, {"eq_n": 128}),
}


@pytest.mark.parametrize("name", sorted(CONV))
def test_conv_against_fp64(name, monkeypatch):
    from ptq4vit_b200.quant_layers.conv import ChannelwiseBatchingQuantConv2d
    n_img, ic, oc, size, k, o = CONV[name]
    monkeypatch.delenv("P4V_OPERAND", raising=False)
    x, W, b, y, g = [t.cuda() for t in O.make_conv_fixture(300 + len(name), n_img, ic, oc, size, k)]
    w_bit, eq_n = o.get("w_bit", 8), o.get("eq_n", 100)
    m = ChannelwiseBatchingQuantConv2d(ic, oc, (k, k), stride=k, bias=True, a_bit=32, w_bit=w_bit, metric="hessian",
                                       eq_alpha=0.01, eq_beta=1.2, eq_n=eq_n, search_round=1)
    m.weight.data = W.clone(); m.bias.data = b.clone()
    m.cuda(); m.keep_scores = True
    m.raw_input, m.raw_out, m.raw_grad = x, y, g
    _, launches, rows = _profiled(m.calibration_step2)
    obs = _observed(rows)
    assert launches[0] > 0 and launches[1] == 0 and launches[2] == 0, "conv runs bf16 sweeps (3-term split of the im2col)"
    assert obs["modes"] == ["single"]
    rep = R.conv_replay(W, b, x, y, g, m.last_scores[0], stride=k, w_bit=w_bit, eq_n=eq_n)
    R.check_intervals(rep, {"w_interval": m.w_interval}, name)
    # quant_forward of the conv is torch's convolution on the fake-quantised weight (conv.py:65-70); fp32 throughout
    m.mode = "quant_forward"
    with torch.no_grad(), RH.fp32_convolutions():
        out = m(x)
    ref, bound = R.conv_forward(W, b, x, m.w_interval, stride=k, w_bit=w_bit)
    fr = R.check_forward(out, ref, bound, name)
    _record(f"conv/{name}", rep, obs, fr)
