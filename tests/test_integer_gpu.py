"""Integer export (SURVEY.md 8f rank 3): ptq4vit_b200.utils.integer against the reference's utils/integer.py functions
running on the same GPU (oracle/_ref) and against the oracle's restatement of their formulas."""
import pytest
import torch

from oracle import ptq_oracle as O
from oracle import ref_harness as RH

pytestmark = pytest.mark.gpu


def _lin(cls, K, Oo, **kw):
    m = cls(K, Oo, **kw)
    gen = torch.Generator().manual_seed(5)
    m.weight.data = torch.randn(Oo, K, generator=gen) * 0.05
    return m.cuda()


def test_int8_weight_and_roundtrip():
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear
    from ptq4vit_b200.utils import integer as I
    m = _lin(PTQSLBatchingQuantLinear, 96, 64, n_V=4, n_H=3)
    wv = m.weight.data.view(4, 16, 3, 32)
    m.w_interval = (wv.abs().amax([1, 3], keepdim=True) / 127.5)
    w_int = I.quantize_int_weight(m)
    ref = O.int_plain(wv, m.w_interval, 128).view(64, 96)
    assert w_int.dtype == torch.int8 and torch.equal(w_int, ref)
    w_sim = I.dequantize_int_weight(m, w_int)
    assert torch.allclose(w_sim, m.quant_weight_bias()[0], rtol=0, atol=0)
    # the reference's own function (valid for one block, integer.py:15)
    if RH.available():
        R = RH.load()
        m1 = _lin(PTQSLBatchingQuantLinear, 96, 64)
        m1.w_interval = (m1.weight.data.abs().max() / 127.5).view(1, 1, 1, 1)
        r = R.linear.PTQSLBatchingQuantLinear(96, 64).cuda()
        r.weight.data = m1.weight.data.clone(); r.w_interval = m1.w_interval.clone()
        assert torch.equal(I.quantize_int_weight(m1).cpu().view(-1), R.integer.quantize_int_weight(r).view(-1))
        assert set(I.get_model_int_weight({"a": m1, "b": torch.nn.Identity()}).keys()) == {"a"}


def test_activation_layouts_match_reference_hooks():
    from ptq4vit_b200.quant_layers.linear import PTQSLBatchingQuantLinear, PostGeluPTQSLBatchingQuantLinear
    from ptq4vit_b200.quant_layers.matmul import PTQSLBatchingQuantMatMul, SoSPTQSLBatchingQuantMatMul
    from ptq4vit_b200.utils import integer as I
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(8, 197, 256, generator=gen).cuda()
    xg = torch.nn.functional.gelu(torch.randn(8, 197, 256, generator=gen) * 1.5).cuda()
    A = torch.randn(8, 6, 197, 64, generator=gen).cuda(); B = torch.randn(8, 6, 64, 197, generator=gen).cuda()
    S = torch.softmax(torch.randn(8, 6, 197, 197, generator=gen) * 4, -1).cuda(); V = torch.randn(8, 6, 197, 64, generator=gen).cuda()

    lin = _lin(PTQSLBatchingQuantLinear, 256, 64); lin.a_interval = (x.abs().max() / 127.5).view(1, 1)
    gel = _lin(PostGeluPTQSLBatchingQuantLinear, 256, 64); gel.a_interval = (xg.max() / 127.5).view(1, 1)
    mm = PTQSLBatchingQuantMatMul()
    mm.A_interval = (A.abs().amax((0, 2, 3)) / 127.5).view(1, 6, 1, 1, 1, 1, 1); mm.B_interval = (B.abs().amax((0, 2, 3)) / 127.5).view(1, 6, 1, 1, 1, 1, 1)
    mm._get_padding_parameters(A, B)
    sos = SoSPTQSLBatchingQuantMatMul()
    sos.split = torch.tensor(2.0 ** -5, device="cuda"); sos.A_interval = sos.split / 127
    sos.B_interval = (V.abs().amax((0, 2, 3)) / 127.5).view(1, 6, 1, 1, 1, 1, 1)
    sos._get_padding_parameters(S, V)

    I.quantize_int_activation(lin, (x,)); I.quantize_int_activation(gel, (xg,))
    I.quantize_int_activation(mm, (A, B)); I.quantize_int_activation(sos, (S, V))
    # oracle restatements (torch ops on the same device)
    assert torch.equal(lin.int_input[0], O.int_plain(x, lin.a_interval, 128))
    assert torch.equal(gel.int_input[0], O.int_gelu_twin(xg, gel.a_interval, gel.a_neg_interval, 128))
    assert torch.equal(mm.int_input[0], O.int_plain(A, mm.A_interval.view(1, 6, 1, 1), 128))
    assert torch.equal(mm.int_input[1], O.int_plain(B, mm.B_interval.view(1, 6, 1, 1), 128))
    assert torch.equal(sos.int_input[0], O.int_sos_twin(S, sos.split, sos.A_interval, 128))
    assert gel.int_input[0].dtype == torch.uint8 and sos.int_input[0].dtype == torch.uint8 and lin.int_input[0].dtype == torch.int8
    if not RH.available():
        return
    # the reference's pre-forward hook on its own classes carrying the same step sizes
    R = RH.load()
    rl = R.linear.PTQSLBatchingQuantLinear(256, 64).cuda(); rl.a_interval = lin.a_interval
    rg = R.linear.PostGeluPTQSLBatchingQuantLinear(256, 64).cuda(); rg.a_interval = gel.a_interval
    rm = R.matmul.PTQSLBatchingQuantMatMul(); rm.A_interval, rm.B_interval = mm.A_interval, mm.B_interval
    rm._get_padding_parameters(A, B)
    rs = R.matmul.SoSPTQSLBatchingQuantMatMul(); rs.split, rs.A_interval, rs.B_interval = sos.split, sos.A_interval, sos.B_interval
    rs._get_padding_parameters(S, V)
    R.integer.quantize_int_activation(rl, (x,)); R.integer.quantize_int_activation(rg, (xg,))
    R.integer.quantize_int_activation(rm, (A, B)); R.integer.quantize_int_activation(rs, (S, V))
    assert torch.equal(lin.int_input[0].cpu(), rl.int_input[0])
    assert torch.equal(gel.int_input[0].cpu(), rg.int_input[0])
    assert torch.equal(mm.int_input[0].cpu(), rm.int_input[0]) and torch.equal(mm.int_input[1].cpu(), rm.int_input[1])
    assert torch.equal(sos.int_input[0].cpu(), rs.int_input[0]) and torch.equal(sos.int_input[1].cpu(), rs.int_input[1])
