"""The int8 activation step of a bf16 Linear layer runs on a consumer loop of its own: four K32 candidate groups per ring
stage, the last stage holding the remaining one to four groups with the final one last.  These shapes give last stages
of every size, a step of one stage only, and row and column tiles cut by the layer's edges (the final epilogue's
predicated gradient loads).  Score tables and step sizes must be bit-identical to a search with the whole layer forced
to bf16 (P4V_OPERAND=bf16), which never takes that loop."""
import pytest

from oracle import ptq_oracle as O   # seeded fixtures only
from tests.test_int8_activation_step_gpu import _int8_vs_bf16, _run

pytestmark = pytest.mark.gpu

# (in, out, n_V, n_H, images, tokens): n_H K32 candidate groups (in / n_H = 17 to 32 int8 bytes of K each: with 16 or
# fewer the int8 images are no smaller than the bf16 ones and the step stays on bf16)
SHAPES = {
    "groups2": (64, 96, 2, 2, 3, 43),       # one stage of two groups; 129 rows
    "groups3": (96, 80, 5, 3, 4, 65),       # one stage of three groups; 80 columns
    "groups4_k24": (96, 128, 2, 4, 2, 70),  # one full stage; 24-element segments padded to 32 bytes
    "groups5": (160, 200, 1, 5, 2, 65),     # stages of 4 + 1; 200 columns
    "groups6": (192, 144, 3, 6, 3, 50),     # 4 + 2
    "groups7": (224, 64, 4, 7, 4, 33),      # 4 + 3
    "groups9": (288, 128, 2, 9, 2, 100),    # 4 + 4 + 1
}


def _linear(name, rounds=2, seed=33):
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    K, Oo, n_V, n_H, n_img, n_tok = SHAPES[name]
    x, W, b, y, g = O.make_linear_fixture(seed, n_img, n_tok, K, Oo)
    m = PTQSLBatchingQuantLinear(K, Oo, metric="hessian", eq_alpha=0.01, eq_beta=1.2, eq_n=100, search_round=rounds,
                                 n_V=n_V, n_H=n_H, n_a=1)
    m.weight.data = W; m.bias.data = b
    return m.cuda(), [t.cuda() for t in (x, y, g)]


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_x8_loop_matches_bf16(name, monkeypatch):
    monkeypatch.delenv("P4V_WORKSPACE_BUDGET", raising=False)
    m, (x, y, g) = _linear(name)
    _int8_vs_bf16(lambda: _run(m, x, y, g), monkeypatch, m.search_round)
