"""No-GPU check: the workspace the library plans for the ViT-B/224 x 32 layers that the other planning tests do not pin
(W8A8, eq_n = 100, three rounds): the patch-embedding conv search, the quantised forwards, and the Linear searches with
the operand type forced."""
import ctypes

import pytest

BASE_LIN = dict(w_bit=8, a_bit=8, eq_n=100, search_round=3, eq_alpha=0.01, eq_beta=1.2, has_bias=1, n_a=1, rows=6304,
                tokens=197)
LIN = {
    "qkv": dict(in_features=768, out_features=2304, n_V=1, n_H=24, post_gelu=0),
    "proj": dict(in_features=768, out_features=768, n_V=24, n_H=24, post_gelu=0),
    "fc1": dict(in_features=768, out_features=3072, n_V=24, n_H=24, post_gelu=0),
    "fc2": dict(in_features=3072, out_features=768, n_V=1, n_H=24, post_gelu=1),
}
BASE_MM = dict(A_bit=8, B_bit=8, eq_n=100, search_round=3, eq_alpha=0.01, eq_beta=1.2, batch=32, heads=12, S1=197)
MM = {"matmul1": dict(S2=64, S3=197, sos=0), "matmul2": dict(S2=197, S3=64, sos=1)}

# (entry point, layer, operand) -> bytes; operand 1 = int8, 2 = bf16
PLANNED_BYTES = {
    ("linear_quant_forward", "qkv", 0): 14500096,
    ("linear_quant_forward", "fc2", 0): 42074624,
    ("matmul_quant_forward", "matmul1", 0): 12604160,
    ("matmul_quant_forward", "matmul2", 0): 55071488,
    ("linear", "proj", 1): 975153664,
    ("linear", "proj", 2): 1531163392,
    ("linear", "fc1", 1): 1401566464,
    ("linear", "fc1", 2): 2136292864,
}
CONV_PATCH_EMBED_BYTES = 234200576


@pytest.fixture(scope="module")
def lib():
    from ptq4vit_b200 import build, _lib
    build.build()
    return _lib.lib()


def _fill(d, kw):
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("key", sorted(PLANNED_BYTES))
def test_layer_workspace_bytes(lib, key):
    from ptq4vit_b200 import _lib
    entry, layer, operand = key
    if entry.startswith("matmul"):
        d = _fill(_lib.MatMulDesc(), {**BASE_MM, **MM[layer], "operand": operand})
    else:
        d = _fill(_lib.LinearDesc(), {**BASE_LIN, **LIN[layer], "operand": operand})
    n = ctypes.c_size_t()
    assert getattr(lib, f"p4v_{entry}_workspace_bytes")(ctypes.byref(d), ctypes.byref(n)) == 0, lib.p4v_last_error().decode()
    assert n.value == PLANNED_BYTES[key]


def test_patch_embedding_conv_workspace_bytes(lib):
    from ptq4vit_b200 import _lib
    d = _fill(_lib.ConvDesc(), dict(images=32, out_channels=768, K=3 * 16 * 16, positions=14 * 14, w_bit=8, eq_n=100,
                                     eq_alpha=0.01, eq_beta=1.2, has_bias=1))
    n = ctypes.c_size_t()
    assert lib.p4v_conv_workspace_bytes(ctypes.byref(d), ctypes.byref(n)) == 0, lib.p4v_last_error().decode()
    assert n.value == CONV_PATCH_EMBED_BYTES
