"""No-GPU checks of the memory-bounded (chunked) search: workspace planning of the chunk fields of the descriptors,
their validation, and the choice of the chunk count (quant_layers/_chunking.py)."""
import ctypes

import pytest

# Workspace bytes the library planned before the chunk fields existed (W8A8, eq_n = 100, three rounds).  A zero chunk
# field must keep every one of them.
UNCHUNKED_BYTES = {
    "lin_qkv_224x32": 1934457088,
    "lin_fc2_224x32": 2247952640,
    "lin_fc2_384x128": 23425359104,
    "lin_pg_small": 33573376,
    "mm_qk_224x32": 1290555392,
    "mm_sv_224x32": 2863026176,
    "mm_sv_384x128": 60622131968,
}
SHAPES = {
    "lin_qkv_224x32": dict(rows=6304, tokens=197, in_features=768, out_features=2304, n_V=1, n_H=24, n_a=1, post_gelu=0),
    "lin_fc2_224x32": dict(rows=6304, tokens=197, in_features=3072, out_features=768, n_V=1, n_H=24, n_a=1, post_gelu=1),
    "lin_fc2_384x128": dict(rows=73856, tokens=577, in_features=3072, out_features=768, n_V=1, n_H=24, n_a=1, post_gelu=1),
    "lin_pg_small": dict(rows=1040, tokens=65, in_features=256, out_features=128, n_V=1, n_H=4, n_a=2, post_gelu=1),
    "mm_qk_224x32": dict(batch=32, heads=12, S1=197, S2=64, S3=197, sos=0),
    "mm_sv_224x32": dict(batch=32, heads=12, S1=197, S2=197, S3=64, sos=1),
    "mm_sv_384x128": dict(batch=128, heads=12, S1=577, S2=577, S3=64, sos=1),
}


@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


def _desc(name, **kw):
    from ptq4vit_b200 import _lib
    if name.startswith("lin"):
        d = _lib.LinearDesc()
        base = dict(w_bit=8, a_bit=8, eq_n=100, search_round=3, eq_alpha=0.01, eq_beta=1.2, has_bias=1)
    else:
        d = _lib.MatMulDesc()
        base = dict(A_bit=8, B_bit=8, eq_n=100, search_round=3, eq_alpha=0.01, eq_beta=1.2)
    base.update(SHAPES[name])
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _ws(lib, d):
    n = ctypes.c_size_t()
    fn = lib.p4v_linear_workspace_bytes if hasattr(d, "rows_per_chunk") else lib.p4v_matmul_workspace_bytes
    rc = fn(ctypes.byref(d), ctypes.byref(n))
    assert rc == 0, lib.p4v_last_error().decode()
    return n.value


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_zero_chunk_field_keeps_the_whole_layer_plan(lib, name):
    assert _ws(lib, _desc(name)) == UNCHUNKED_BYTES[name]


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_workspace_shrinks_with_the_chunk(lib, name):
    if name.startswith("lin"):
        rows = SHAPES[name]["rows"]
        sizes = sorted({min(rows // 128, c) * 128 for c in (1, 2, 3, 5, 8, 16, 49, 10 ** 6)})
        ws = [_ws(lib, _desc(name, rows_per_chunk=s)) for s in sizes]
    else:
        batch = SHAPES[name]["batch"]
        sizes = sorted({min(batch, c) for c in (1, 2, 3, 7, 16, 64, 10 ** 6)})
        ws = [_ws(lib, _desc(name, images_per_chunk=s)) for s in sizes]
    assert all(a < b for a, b in zip(ws, ws[1:])), list(zip(sizes, ws))
    assert ws[-1] <= UNCHUNKED_BYTES[name]
    assert ws[0] < UNCHUNKED_BYTES[name] / 2      # W candidate planes, H and the residual stay whole-layer


def test_chunked_fc2_and_matmul2_at_384px_fit_a_shared_card(lib):
    """DeiT-B/384 x 128 images: the largest searches need 23 GB and 61 GB whole; chunked they fit in a few GB."""
    assert _ws(lib, _desc("lin_fc2_384x128", rows_per_chunk=128 * 58)) < 3e9
    assert _ws(lib, _desc("mm_sv_384x128", images_per_chunk=16)) < 8e9


@pytest.mark.parametrize("bad,msg", [
    (dict(rows_per_chunk=-128), "rows_per_chunk"), (dict(rows_per_chunk=100), "multiple of 128"),
    (dict(rows_per_chunk=1040 + 128), "rows_per_chunk"),
])
def test_bad_row_chunks_are_rejected(lib, bad, msg):
    n = ctypes.c_size_t()
    assert lib.p4v_linear_workspace_bytes(ctypes.byref(_desc("lin_pg_small", **bad)), ctypes.byref(n)) != 0
    assert msg in lib.p4v_last_error().decode()


@pytest.mark.parametrize("bad", [-1, 33])
def test_bad_image_chunks_are_rejected(lib, bad):
    n = ctypes.c_size_t()
    assert lib.p4v_matmul_workspace_bytes(ctypes.byref(_desc("mm_qk_224x32", images_per_chunk=bad)), ctypes.byref(n)) != 0
    assert "images_per_chunk" in lib.p4v_last_error().decode()


def test_step_wise_surface_takes_whole_layers_only(lib):
    d = _desc("lin_pg_small", rows_per_chunk=256)
    rc = lib.p4v_linear_begin(ctypes.byref(d), 1, 1, None, 1, 1, 1, 1 << 40, None)
    assert rc != 0 and "rows_per_chunk" in lib.p4v_last_error().decode()


def test_choose_chunks_picks_the_fewest_chunks_that_fit():
    from ptq4vit_b200.quant_layers._chunking import choose_chunks
    fixed, per_unit = 1000, 10

    def ws(per):                      # a layer of 1000 units
        return fixed + per_unit * (1000 if per == 0 else per)
    assert choose_chunks(1000, 1, ws, 11000) == (0, 1)
    assert choose_chunks(1000, 1, ws, 10999) == (500, 2)
    assert choose_chunks(1000, 1, ws, 6000) == (500, 2)
    assert choose_chunks(1000, 1, ws, 5999) == (334, 3)
    assert choose_chunks(1000, 1, ws, fixed + per_unit) == (1, 1000)
    with pytest.raises(MemoryError, match="does not fit"):
        choose_chunks(1000, 1, ws, fixed + per_unit - 1)


def test_choose_chunks_respects_the_granule():
    from ptq4vit_b200.quant_layers._chunking import choose_chunks
    seen = []

    def ws(per):
        seen.append(per)
        return 10 * (520 if per == 0 else per)
    # 520 rows in 128-row tiles: 2 chunks of 384 + 136 rows, 3 chunks of 256 + 256 + 8 rows
    assert choose_chunks(520, 128, ws, 3840) == (384, 2)
    assert choose_chunks(520, 128, ws, 2560) == (256, 3)
    assert all(p % 128 == 0 for p in seen)
    with pytest.raises(MemoryError):
        choose_chunks(520, 128, ws, 1279)
    with pytest.raises(MemoryError):
        choose_chunks(100, 128, ws, 999)      # a layer within one tile cannot be split


def test_budget_override(monkeypatch):
    from ptq4vit_b200.quant_layers import _chunking
    monkeypatch.setenv("P4V_WORKSPACE_BUDGET", "12345")
    assert _chunking.workspace_budget(None) == 12345
