"""No-GPU check: running the activation steps of bf16 Linear layers on int8 images reuses the bf16 candidate activation
region, so the workspace the library plans stays byte-for-byte what it was before (W8A8, eq_n = 100, three rounds,
ViT-B/224 x 32 images)."""
import ctypes

import pytest

# (rows, tokens, in, out, n_V, n_H, rows_per_chunk) -> bytes
PLANNED_BYTES = {
    "proj": ((6304, 197, 768, 768, 24, 24, 0), 1531163392),
    "fc1": ((6304, 197, 768, 3072, 24, 24, 0), 2136292864),
    "head": ((32, 1, 768, 1000, 1, 24, 0), 232981504),
    "proj_2chunks": ((6304, 197, 768, 768, 24, 24, 3200), 860495616),
    "fc1_2chunks": ((6304, 197, 768, 3072, 24, 24, 3200), 1435110912),
    "qkv_2chunks": ((6304, 197, 768, 2304, 72, 24, 3200), 1244807936),
}


@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


@pytest.mark.parametrize("name", sorted(PLANNED_BYTES))
def test_workspace_bytes_unchanged(lib, name):
    from ptq4vit_b200 import _lib
    (rows, tokens, K, Oo, n_V, n_H, rpc), want = PLANNED_BYTES[name]
    d = _lib.LinearDesc()
    for k, v in dict(rows=rows, tokens=tokens, in_features=K, out_features=Oo, n_V=n_V, n_H=n_H, n_a=1, post_gelu=0,
                     w_bit=8, a_bit=8, eq_n=100, search_round=3, eq_alpha=0.01, eq_beta=1.2, has_bias=1,
                     rows_per_chunk=rpc).items():
        setattr(d, k, v)
    n = ctypes.c_size_t()
    assert lib.p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)) == 0, lib.p4v_last_error().decode()
    assert n.value == want
