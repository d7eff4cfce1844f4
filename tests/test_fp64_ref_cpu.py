"""The fp64 evaluator of tests/_fp64_ref.py pinned to the golden vectors, and shown to be sensitive.

Teacher-forced with the reference's own logged tables (CPU tensors: IEEE division, as the goldens were made), the
evaluator must choose the golden step sizes bitwise, and its fp64 tables must agree with the reference's fp32 tables
within the bar the golden tests use (2·10⁻⁴ of the table maximum).  Its error bound must then reject a table that is
wrong in any of the ways a kernel could be subtly wrong."""
import numpy as np
import pytest
import torch

from oracle import ptq_oracle as O
from tests import _cases as C
from tests import _fp64_ref as R

LINEAR = list(C.CASES["linear"])
MATMUL = list(C.CASES["matmul"])


def _golden_close(rep, gold, what):
    assert len(rep.steps) == len(gold)
    for st, g in zip(rep.steps, gold):
        C.assert_scores_close(st.ref, np.asarray(g).reshape(st.ref.shape), 2e-4, f"{what} {st.name}")


@pytest.mark.parametrize("name", LINEAR)
def test_linear_replay_matches_golden(name):
    sp, (x, W, b, y, g), case = C.linear_case(name)
    z, gold = C.load_golden(name)
    rep = R.linear_replay(sp, W, b, x, y, g, gold)
    _golden_close(rep, gold, name)
    R.check_intervals(rep, {"w_interval": torch.from_numpy(z["w_interval"]), "a_interval": torch.from_numpy(z["a_interval"])}, name)


@pytest.mark.parametrize("name", MATMUL)
def test_matmul_replay_matches_golden(name):
    sp, (A, B, Y, G), case = C.matmul_case(name)
    z, gold = C.load_golden(name)
    rep = R.matmul_replay(sp, A, B, Y, G, gold)
    _golden_close(rep, gold, name)
    got = {"A_interval": torch.from_numpy(np.asarray(z["A_interval"])), "B_interval": torch.from_numpy(z["B_interval"])}
    if sp.sos:
        got["split"] = torch.from_numpy(np.asarray(z["split"]))
    R.check_intervals(rep, got, name)


def test_conv_replay_matches_golden():
    z = np.load(C.GOLD + "/conv_small.npz")
    x, W, b, y, g = O.make_conv_fixture(31, 4, 3, 32, 16, 4)
    rep = R.conv_replay(W, b, x, y, g, z["scores_000"], stride=4)
    _golden_close(rep, [z["scores_000"]], "conv_small")
    R.check_intervals(rep, {"w_interval": torch.from_numpy(z["w_interval"])}, "conv_small")


# ---- sensitivity: a perfect fp32 rounding of the fp64 table passes, each mutation is rejected -----------------------
def _lin_small(**over):
    sp, (x, W, b, y, g), case = C.linear_case("lin_small")
    _, gold = C.load_golden("lin_small")
    args = dict(W=W, b=b, x=x, y=y, g=g)
    args.update(over)
    return sp, args, gold


def _replay(sp, args, tables):
    return R.linear_replay(sp, args["W"], args["b"], args["x"], args["y"], args["g"], tables, gram=True)


@pytest.fixture(scope="module")
def exact():
    """The lin_small replay and its tables rounded to fp32: what a kernel without error would log."""
    sp, args, gold = _lin_small()
    rep = _replay(sp, args, gold)
    return sp, args, gold, rep


def _with_tables(rep, tables):
    out = R.Replay(intervals=rep.intervals)
    for st, t in zip(rep.steps, tables):
        out.first_pick(st.name, t, st.ref, st.bound)
    return out


def test_exact_tables_pass(exact):
    sp, args, gold, rep = exact
    n, entries, worst, _ = R.check_tables(_with_tables(rep, [st.ref.astype(np.float32) for st in rep.steps]))
    assert n == len(gold) and entries == sum(np.asarray(t).size for t in gold) and worst <= 1.0
    # On the entries that decide the picks the bound is ~10⁻³ of the entry (slab ~5·10⁻⁴, Gram ≤ 10⁻³ on this case),
    # while 2·10⁻⁴ of the table maximum is ~0.2 of them: a bound that drifts wide fails here.
    for st in rep.steps:
        best, j = st.ref.argmax(0), range(st.ref.shape[1])
        assert np.all(st.bound[best, j] < 1.5e-3 * np.abs(st.ref[best, j])), st.name


def test_entry_moved_by_ten_bounds_is_rejected(exact):
    sp, args, gold, rep = exact
    tables = [st.ref.astype(np.float32) for st in rep.steps]
    st = rep.steps[1]
    c, j = np.unravel_index(int(st.ref.argmax()), st.ref.shape)
    tables[1] = tables[1].copy()
    tables[1][c, j] = np.float32(st.ref[c, j] - 10 * st.bound[c, j])
    with pytest.raises(AssertionError, match="err/bound"):
        R.check_tables(_with_tables(rep, tables))


def test_rotated_table_is_rejected(exact):
    sp, args, gold, rep = exact
    tables = [st.ref.astype(np.float32) for st in rep.steps]
    tables[2] = np.roll(tables[2], 1, axis=0)
    with pytest.raises(AssertionError):
        R.check_tables(_with_tables(rep, tables))


def test_table_without_one_gradient_group_is_rejected(exact):
    sp, args, gold, rep = exact
    g = args["g"].clone()
    g[..., 16:32] = 0                      # one 16-column group of the epilogue
    bad = _replay(sp, dict(args, g=g), gold)
    tables = [st.ref.astype(np.float32) for st in bad.steps]
    with pytest.raises(AssertionError):
        R.check_tables(_with_tables(rep, tables))


def test_table_without_bias_is_rejected(exact):
    sp, args, gold, rep = exact
    bad = _replay(sp, dict(args, b=None), gold)
    tables = [st.ref.astype(np.float32) for st in bad.steps]
    with pytest.raises(AssertionError):
        R.check_tables(_with_tables(rep, tables))


def test_step_sizes_one_grid_step_off_are_rejected(exact):
    sp, args, gold, rep = exact
    z, _ = C.load_golden("lin_small")
    w = torch.from_numpy(z["w_interval"]).clone()
    w0, _ = O.linear_initial_intervals(sp, args["W"], args["x"])
    f = O.candidate_factors(sp.eq_alpha, sp.eq_beta, sp.eq_n)
    i = int(torch.argmin((f - float(w[0, 0, 0, 0] / w0[0, 0, 0, 0])).abs()))
    w[0, 0, 0, 0] = f[i + 1] * w0[0, 0, 0, 0]
    with pytest.raises(AssertionError, match="w_interval"):
        R.check_intervals(rep, {"w_interval": w, "a_interval": torch.from_numpy(z["a_interval"])})
