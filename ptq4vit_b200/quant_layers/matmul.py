"""MatMul quant operators with the reference's class surface (quant_layers/matmul.py).

Result attributes as in the reference: `A_interval`, `B_interval` of shape
[1, n_G, 1, n_V, 1, n_H, 1] (head-wise: n_G = heads, n_V = n_H = 1); the split-of-softmax
variant keeps a 0-d `split` and a 0-d `A_interval = split / (A_qmax - 1)`.
"""
import ctypes

import torch
from torch import nn

from .. import _lib
from ._chunking import choose_chunks, workspace_budget
from ._metric import metric_weight
from .linear import _flat2d, _frozen_quant_forward, _gather_desc, _norm_call_ok, _wants_no_grad, frozen_gather_applies


class _QuantMatMulFn(torch.autograd.Function):
    """The native quantized product inside autograd: the reference's quant_forward (matmul.py:40-45) rounds both
    operands in place, so no gradient flows to A or B, but the output still has a grad_fn whenever an input requires
    grad -- which the gradient hooks of later modules rely on with sequential=True (utils/quant_calib.py:330-341)."""

    @staticmethod
    def forward(ctx, module, A, B):
        ctx.meta = [(t.shape, t.dtype, t.device) if t.requires_grad else None for t in (A, B)]
        return module._quant_forward_native(A, B)

    @staticmethod
    def backward(ctx, grad_out):
        g = [None if m is None else torch.zeros(m[0], dtype=m[1], device=m[2]) for m in ctx.meta]
        return None, g[0], g[1]


class MinMaxQuantMatMul(nn.Module):
    """reference: quant_layers/matmul.py:8-60"""
    sos = False

    def __init__(self, A_bit=8, B_bit=8, mode="raw"):
        super().__init__()
        self.A_bit = A_bit
        self.B_bit = B_bit
        self.A_interval = None
        self.B_interval = None
        self.A_qmax = 2 ** (self.A_bit - 1)
        self.B_qmax = 2 ** (self.B_bit - 1)
        self.mode = mode
        self.raw_input = None
        self.raw_out = None
        self._packed = None                  # freeze(): {heads: packed step sizes and scale tables (torch.uint8, device)}

    def forward(self, A, B):
        if self.mode == "raw":
            out = A @ B
        elif self.mode == "quant_forward":
            out = self.quant_forward(A, B)
        elif self.mode == "calibration_step1":
            out = self.calibration_step1(A, B)
        elif self.mode == "calibration_step2":
            out = self.calibration_step2(A, B)
        else:
            raise NotImplementedError
        return out

    def quant_input(self, x, interval, qmax):
        x_sim = (x / interval).round_().clamp_(-qmax, qmax - 1)
        x_sim.mul_(interval)
        return x_sim

    def calibration_step1(self, A, B):
        self.raw_input = A.cpu().detach(), B.cpu().detach()
        out = A @ B
        self.raw_out = out.cpu().detach()
        return out

    def calibration_step2(self, A, B):
        """reference: matmul.py:54-60 (layer-wise min-max)"""
        H = A.shape[1]
        self.A_interval = (A.data.abs().max() / (self.A_qmax - 0.5)).detach().view(1, 1, 1, 1, 1, 1, 1).repeat(1, H, 1, 1, 1, 1, 1)
        self.B_interval = (B.data.abs().max() / (self.B_qmax - 0.5)).detach().view(1, 1, 1, 1, 1, 1, 1).repeat(1, H, 1, 1, 1, 1, 1)
        self.calibrated = True
        return self.quant_forward(A, B)

    # ---- native plumbing -------------------------------------------------
    def _desc(self, A, B, search_round=1, eq=(0.0, 1.0, 1)):
        assert A.dim() == 4 and B.dim() == 4 and A.shape[:2] == B.shape[:2] and A.shape[3] == B.shape[2], \
            f"expected A [b,H,S1,S2] and B [b,H,S2,S3], got {tuple(A.shape)} and {tuple(B.shape)}"
        return self._desc_dims(A.shape[0], A.shape[1], A.shape[2], A.shape[3], B.shape[3], search_round, eq)

    def _desc_dims(self, batch, heads, S1, S2, S3, search_round=1, eq=(0.0, 1.0, 1)):
        d = _lib.MatMulDesc()
        d.batch, d.heads, d.S1, d.S2, d.S3 = int(batch), int(heads), int(S1), int(S2), int(S3)
        d.A_bit, d.B_bit = int(self.A_bit), int(self.B_bit)
        d.eq_n, d.search_round = int(eq[2]), int(search_round)
        d.eq_alpha, d.eq_beta = float(eq[0]), float(eq[1])
        d.sos = 1 if self.sos else 0
        d.operand = _lib.default_operand()
        d.kernel = _lib.default_kernel()
        d.init_layerwise = 1 if getattr(self, "init_layerwise", False) else 0
        return d

    @staticmethod
    def _cuda(t):
        if t.device.type != "cuda":
            if not torch.cuda.is_available():
                raise RuntimeError("ptq4vit_b200 MatMul quant layers need a CUDA device (no CPU path)")
            t = t.cuda()
        return t.contiguous().float()

    def quant_forward(self, A, B):
        """reference: matmul.py:40-45 / :140-145 -- fq(A) @ fq(B) on the tensor cores."""
        assert self.calibrated is not None, f"You should run calibrate_forward before run quant_forward for {self}"
        if torch.is_grad_enabled() and (A.requires_grad or B.requires_grad):
            return _QuantMatMulFn.apply(self, A, B)
        return self._quant_forward_native(A, B)

    # ---- frozen module: step sizes packed once (csrc/forward_mm_tc.cu) ----
    def _intervals(self):
        return (self.A_interval, self.B_interval, self.split if self.sos else None)

    def _interval_versions(self):
        return tuple(getattr(t, "_version", None) for t in self._intervals())

    def _n_steps(self):
        """Step-size entries per operand: the heads (head-wise layout) or 1 (n_G = 1: one step size for all heads)."""
        sizes = [torch.as_tensor(self.B_interval).numel()] + ([] if self.sos else [torch.as_tensor(self.A_interval).numel()])
        n = max(sizes)
        if any(k not in (1, n) for k in sizes):
            raise RuntimeError(f"{self}: A_interval and B_interval hold {sizes[1]} and {sizes[0]} step sizes")
        return n

    def _pack(self, heads, dev):
        """The packed tables for `heads` heads (a single step size is expanded to all of them, as the unfrozen forward does)."""
        def flat(v):
            t = torch.as_tensor(v, dtype=torch.float32, device=dev).reshape(-1)
            return (t if t.numel() == heads else t.expand(heads)).contiguous()
        a = None if self.sos else flat(self.A_interval)
        b = flat(self.B_interval)
        split = torch.as_tensor(self.split, dtype=torch.float32, device=dev).reshape(1) if self.sos else None
        d = self._desc_dims(1, heads, 1, 1, 1)
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_matmul_pack_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_matmul_pack_bytes")
        packed = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        _lib.check(lib.p4v_matmul_pack(ctypes.byref(d), _lib.ptr(a), _lib.ptr(b), _lib.ptr(split), _lib.ptr(packed), nbytes.value,
                                       ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "p4v_matmul_pack")
        return packed

    def freeze(self):
        """Pack the module's step sizes and scale tables once; until unfreeze(), quant_forward runs the fused frozen forward
        (one kernel, both operands quantised in shared memory, strided q / k / v views read in place), which is
        bit-identical to the unfrozen one.  With one step size for all heads (n_G = 1) the tables for a given number of
        heads are packed at the first call with that many heads."""
        if not getattr(self, "calibrated", None):
            raise RuntimeError(f"freeze() needs a calibrated module: {self}")
        b = self.B_interval
        if not torch.is_tensor(b) or b.device.type != "cuda":
            raise RuntimeError("ptq4vit_b200 MatMul quant layers freeze step sizes held on a CUDA device (no CPU path)")
        n = self._n_steps()
        self._packed = {n: self._pack(n, b.device)}
        # the step sizes that were packed: the objects (kept, so their identity cannot be reused) and their versions
        self._frozen_intervals = (self._intervals(), self._interval_versions())
        return self

    def unfreeze(self):
        self._packed = self._frozen_intervals = None
        return self

    @property
    def frozen(self):
        return self._packed is not None

    @staticmethod
    def _strides(t, unit_dims):
        """Element strides for the kernel; a dimension of size 1 gets the stride the kernel expects (never used)."""
        return (ctypes.c_longlong * 4)(*[(1 if i in unit_dims else 0) if n == 1 else st
                                         for i, (n, st) in enumerate(zip(t.shape, t.stride()))])

    def _frozen_pack(self, heads):
        """The packed tables of a frozen module for `heads` heads, after checking that its step sizes are the ones
        freeze() packed (with one step size for all heads, the tables for a new head count are packed here)."""
        i0, v0 = self._frozen_intervals
        if any(a is not b for a, b in zip(self._intervals(), i0)) or self._interval_versions() != v0:
            raise RuntimeError(f"{self}: the step sizes changed after freeze(); call unfreeze() (and freeze() again) "
                               "before running the layer")
        packed = self._packed.get(heads)
        if packed is None:
            if self._n_steps() != 1:
                raise RuntimeError(f"{self}: frozen with {self._n_steps()} head-wise step sizes, called with {heads} heads")
            packed = self._packed[heads] = self._pack(heads, next(iter(self._packed.values())).device)
        return packed

    def _frozen_forward(self, A, B):
        assert A.dim() == 4 and B.dim() == 4 and A.shape[:2] == B.shape[:2] and A.shape[3] == B.shape[2], \
            f"expected A [b,H,S1,S2] and B [b,H,S2,S3], got {tuple(A.shape)} and {tuple(B.shape)}"
        packed = self._frozen_pack(A.shape[1])
        dev = packed.device
        A_, B_ = A.to(dev, torch.float32), B.to(dev, torch.float32)
        # read in place: A with unit stride along K, B along K (k^T) or N (v); any other layout is copied once
        if A_.shape[3] > 1 and A_.stride(3) != 1:
            A_ = A_.contiguous()
        if B_.shape[2] > 1 and B_.shape[3] > 1 and 1 not in B_.stride()[2:]:
            B_ = B_.contiguous()
        batch, H, S1, S2 = A_.shape
        S3 = B_.shape[3]
        out = torch.empty(batch, H, S1, S3, dtype=torch.float32, device=dev)
        d = self._desc_dims(batch, H, S1, S2, S3)
        sb = self._strides(B_, (2,) if B_.shape[2] == 1 or B_.stride(2) == 1 else (3,))
        _lib.check(_lib.lib().p4v_matmul_frozen_forward(ctypes.byref(d), _lib.ptr(A_), self._strides(A_, (3,)), _lib.ptr(B_), sb,
                                                        _lib.ptr(packed), _lib.ptr(out),
                                                        ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_matmul_frozen_forward")
        return out

    def _quant_forward_native(self, A, B):
        if self._packed is not None:
            return self._frozen_forward(A, B)
        A_, B_ = self._cuda(A), self._cuda(B)
        dev = A_.device
        d = self._desc(A_, B_)
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_matmul_quant_forward_workspace_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "matmul_quant_forward_workspace")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        out = torch.empty(d.batch, d.heads, d.S1, d.S3, dtype=torch.float32, device=dev)
        H = d.heads
        a_int = torch.as_tensor(self.A_interval, dtype=torch.float32, device=dev).reshape(-1)
        a_int = (a_int if a_int.numel() == H or self.sos else a_int.expand(H)).contiguous()
        b_int = torch.as_tensor(self.B_interval, dtype=torch.float32, device=dev).reshape(-1)
        b_int = (b_int if b_int.numel() == H else b_int.expand(H)).contiguous()
        split = torch.as_tensor(self.split, dtype=torch.float32, device=dev).reshape(1) if self.sos else None
        _lib.check(lib.p4v_matmul_quant_forward(ctypes.byref(d), _lib.ptr(A_), _lib.ptr(B_), _lib.ptr(a_int), _lib.ptr(b_int),
                                                _lib.ptr(split), _lib.ptr(ws), nbytes.value, _lib.ptr(out),
                                                ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_matmul_quant_forward")
        return out


SHORT_ATTENTION_TOKENS = 256      # P4V_ATTN_MAX_TOKENS: the short kernel's limit, and fuse_attention's default
LONG_ATTENTION_TOKENS = 1024      # P4V_ATTN_LONG_MAX_TOKENS: the long-sequence kernel's limit


def frozen_attention_applies(matmul1, matmul2, tokens, head_dim, *inputs, max_tokens=SHORT_ATTENTION_TOKENS):
    """Whether one call of an attention block can run as the fused frozen attention core: both MatMul modules frozen and
    in quant_forward mode, matmul1 not split-of-softmax, no input that requires grad under grad mode, and a shape a
    kernel holds: p4v_attention_fused_ok (at most 256 tokens, head_dim a multiple of 16 up to 64) or, for
    256 < tokens <= max_tokens, p4v_attention_long_ok (at most 1024 tokens, the same head_dim rule)."""
    if not all(isinstance(m, MinMaxQuantMatMul) and m.frozen and m.mode == "quant_forward" for m in (matmul1, matmul2)):
        return False
    if matmul1.sos or (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in inputs)):
        return False
    if tokens > max(max_tokens, SHORT_ATTENTION_TOKENS):
        return False
    ok = ctypes.c_int()
    name = "p4v_attention_fused_ok" if tokens <= SHORT_ATTENTION_TOKENS else "p4v_attention_long_ok"
    _lib.check(getattr(_lib.lib(), name)(int(tokens), int(head_dim), ctypes.byref(ok)), name)
    return bool(ok.value)


def frozen_attention(matmul1, matmul2, qkv, scale, scale_on_q, bias=None, mask=None, max_tokens=SHORT_ATTENTION_TOKENS):
    """The attention core between the qkv and proj Linears in one kernel, for a call where frozen_attention_applies
    holds: csrc/forward_attn_tc.cu up to 256 tokens, csrc/forward_attn_long_tc.cu for 256 < N <= max_tokens (ViT / DeiT
    only: no q-scaling, bias or mask).  `qkv` is the qkv Linear's output viewed as [B, N, 3, heads, head_dim]; returns
    matmul2(softmax(S), v).transpose(1, 2).reshape(B, N, C) with S = matmul1(q, k^T) * scale (scale_on_q=False, ViT) or
    matmul1(q * scale, k^T) + bias [+ mask of window b % nW] (scale_on_q=True, Swin), with the bits of that sequence."""
    B, N, _, H, D = qkv.shape
    if N > max(max_tokens, SHORT_ATTENTION_TOKENS):
        raise ValueError(f"frozen_attention: {N} tokens, more than max_tokens={max_tokens}")
    p1, p2 = matmul1._frozen_pack(H), matmul2._frozen_pack(H)
    dev = p1.device
    qkv = qkv.to(dev, torch.float32)
    if qkv.stride(4) != 1:
        qkv = qkv.contiguous()
    bias = None if bias is None else bias.to(dev, torch.float32).contiguous()
    mask = None if mask is None else mask.to(dev, torch.float32).contiguous()
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim = int(B), int(N), int(H), int(D)
    a.scale_on_q, a.n_windows, a.scale = int(bool(scale_on_q)), 0 if mask is None else int(mask.shape[0]), float(scale)
    d1, d2 = matmul1._desc_dims(1, H, 1, 1, 1), matmul2._desc_dims(1, H, 1, 1, 1)
    out = torch.empty(B, N, H * D, dtype=torch.float32, device=dev)
    name = "p4v_attention_frozen_forward" if N <= SHORT_ATTENTION_TOKENS else "p4v_attention_frozen_forward_long"
    _lib.check(getattr(_lib.lib(), name)(
        ctypes.byref(a), _lib.ptr(qkv), (ctypes.c_longlong * 4)(*qkv.stride()[:4]), ctypes.byref(d1), _lib.ptr(p1), p1.numel(),
        ctypes.byref(d2), _lib.ptr(p2), p2.numel(), _lib.ptr(bias), _lib.ptr(mask), _lib.ptr(out),
        ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), name)
    return out


def _attention_desc(batch, tokens, heads, head_dim, scale, scale_on_q, n_windows=0):
    a = _lib.AttentionDesc()
    a.batch, a.tokens, a.heads, a.head_dim = int(batch), int(tokens), int(heads), int(head_dim)
    a.scale_on_q, a.n_windows, a.scale = int(bool(scale_on_q)), int(n_windows), float(scale)
    return a


def frozen_qkv_ok(qkv, tokens, heads, head_dim, gather=False):
    """The library's shape rule of the qkv fold (p4v_linear_qkv8_ok): out_features == 3 * heads * head_dim, the short
    attention kernel's shape (at most 256 tokens, head_dim a multiple of 16 up to 64), qkv on its fused path, the plan
    with the epilogue's staging (and the LayerNorm's statistics, and with `gather` the window gather's table) fits."""
    ok = ctypes.c_int()
    a = _attention_desc(1, tokens, heads, head_dim, 1.0, False)
    _lib.check(_lib.lib().p4v_linear_qkv8_ok(ctypes.byref(qkv._desc(1, 1)), ctypes.byref(a), _lib.GATHER["window"] if gather else 0,
                                             ctypes.byref(ok)), "p4v_linear_qkv8_ok")
    return bool(ok.value)


def frozen_qkv_applies(qkv, matmul1, matmul2, x, tokens, heads, head_dim, *inputs, norm=None, gather=None):
    """Whether one attention call -- qkv(x) (qkv(norm(x)) with `norm`; with `gather` = (images, height, width, window,
    shift) the windows of roll(norm(x), -shift), as frozen_gather_applies) followed by the attention core -- can run with
    the attention operands' quantisation folded into qkv (frozen_qkv_attention): qkv a frozen Linear layer in
    quant_forward mode, the conditions of frozen_attention_applies on the short kernel (both MatMul modules frozen,
    matmul1 not split-of-softmax, at most 256 tokens, no input -- x and `inputs` -- that requires grad under grad mode),
    those of the LayerNorm or gather fold when one is given, and the library's rule (frozen_qkv_ok).  Decided from the
    shapes before qkv runs, so a refused call runs the unfolded sequence once (DESIGN.md section 4.14)."""
    if tokens > SHORT_ATTENTION_TOKENS or not _frozen_quant_forward(qkv):
        return False
    if not frozen_attention_applies(matmul1, matmul2, tokens, head_dim, x, *inputs):
        return False
    dev = qkv._packed.device
    if not torch.is_tensor(x) or x.dtype != torch.float32 or x.device != dev or x.numel() == 0 or x.shape[-1] != qkv.in_features:
        return False
    if gather is not None:
        if not frozen_gather_applies(norm, qkv, x, ("window", *gather)):
            return False
    elif norm is not None:
        if not _norm_call_ok(norm, qkv, x):
            return False
    elif not _wants_no_grad((x,), (qkv,)):
        return False
    if (x.numel() // x.shape[-1]) % tokens:
        return False
    return frozen_qkv_ok(qkv, tokens, heads, head_dim, gather is not None)


def frozen_qkv_planes(qkv, matmul1, matmul2, x, tokens, heads, head_dim, scale, scale_on_q, norm=None, gather=None):
    """The first launch of frozen_qkv_attention: qkv(x) (with `norm` / `gather` as frozen_qkv_applies) on qkv's fused
    kernel, whose epilogue quantises q (times scale first with scale_on_q), k and v with matmul1's A and B and matmul2's B
    step sizes (csrc/forward_tc.cu).  Returns the int8 planes [3, batch, heads, tokens, head_dim], the bytes the short
    attention kernel would make of qkv's FP32 output; only they are allocated."""
    qkv._check_frozen_intervals()
    p1, p2 = matmul1._frozen_pack(heads), matmul2._frozen_pack(heads)
    dev = qkv._packed.device
    x2 = _flat2d(x.to(dev))
    rows = x2.shape[0]
    planes = torch.empty(3, rows // tokens, heads, tokens, head_dim, dtype=torch.int8, device=dev)
    a = _attention_desc(rows // tokens, tokens, heads, head_dim, scale, scale_on_q)
    d, d1, d2 = qkv._desc(rows, 1), matmul1._desc_dims(1, heads, 1, 1, 1), matmul2._desc_dims(1, heads, 1, 1, 1)
    b = None if qkv.bias is None else qkv.bias.detach().contiguous().float()
    g = None if gather is None else ctypes.byref(_gather_desc(("window", *gather)))
    _lib.check(_lib.lib().p4v_linear_frozen_forward_qkv8(
        ctypes.byref(d), _lib.ptr(x2), _lib.ptr(b), _lib.ptr(qkv._packed), ctypes.byref(a), ctypes.byref(d1), _lib.ptr(p1),
        p1.numel(), ctypes.byref(d2), _lib.ptr(p2), p2.numel(), _lib.ptr(planes), _lib.ptr(None if norm is None else norm.weight),
        _lib.ptr(None if norm is None else norm.bias), 0.0 if norm is None else float(norm.eps), g,
        ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "p4v_linear_frozen_forward_qkv8")
    return planes


def frozen_qkv_attention(qkv, matmul1, matmul2, x, tokens, heads, head_dim, scale, scale_on_q, bias=None, mask=None,
                         norm=None, gather=None):
    """The attention core of frozen_attention on qkv(x) (with `norm` / `gather` as frozen_qkv_applies), for a call where
    frozen_qkv_applies holds, in two launches: qkv's fused kernel writes q, k and v as int8 planes (frozen_qkv_planes),
    and the short attention kernel reads them (csrc/forward_attn_tc.cu).  Bit-identical to frozen qkv followed by
    frozen_attention; qkv's FP32 output never reaches HBM.  Returns [batch, tokens, heads * head_dim]; only the planes and
    it are allocated."""
    planes = frozen_qkv_planes(qkv, matmul1, matmul2, x, tokens, heads, head_dim, scale, scale_on_q, norm=norm, gather=gather)
    p1, p2 = matmul1._frozen_pack(heads), matmul2._frozen_pack(heads)
    dev = planes.device
    batch = planes.shape[1]
    out = torch.empty(batch, tokens, heads * head_dim, dtype=torch.float32, device=dev)
    bias = None if bias is None else bias.to(dev, torch.float32).contiguous()
    mask = None if mask is None else mask.to(dev, torch.float32).contiguous()
    a = _attention_desc(batch, tokens, heads, head_dim, scale, scale_on_q, 0 if mask is None else mask.shape[0])
    d1, d2 = matmul1._desc_dims(1, heads, 1, 1, 1), matmul2._desc_dims(1, heads, 1, 1, 1)
    _lib.check(_lib.lib().p4v_attention_frozen_forward_i8(
        ctypes.byref(a), _lib.ptr(planes), ctypes.byref(d1), _lib.ptr(p1), p1.numel(), ctypes.byref(d2), _lib.ptr(p2), p2.numel(),
        _lib.ptr(bias), _lib.ptr(mask), _lib.ptr(out), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
        "p4v_attention_frozen_forward_i8")
    return out


class PTQSLQuantMatMul(MinMaxQuantMatMul):
    """reference: quant_layers/matmul.py:62-282.  Block structure: only the head-wise layout that
    the Batching classes force (n_G = heads, n_V = n_H = 1) is implemented by the CUDA path."""

    def __init__(self, A_bit=8, B_bit=8, mode="raw", metric="L2_norm", search_round=1, eq_alpha=0.1, eq_beta=2,
                 eq_n=100, parallel_eq_n=10, n_G_A=1, n_V_A=1, n_H_A=1, n_G_B=1, n_V_B=1, n_H_B=1, init_layerwise=False):
        super().__init__(A_bit=A_bit, B_bit=B_bit, mode=mode)
        self.metric = metric
        self.search_round = search_round
        self.eq_alpha = eq_alpha
        self.eq_beta = eq_beta
        self.eq_n = eq_n
        self.parallel_eq_n = parallel_eq_n
        self.n_G_A, self.n_V_A, self.n_H_A = n_G_A, n_V_A, n_H_A
        self.n_G_B, self.n_V_B, self.n_H_B = n_G_B, n_V_B, n_H_B
        self.crb_groups_A = self.crb_groups_B = None
        self.crb_rows_A = self.crb_cols_A = self.crb_rows_B = self.crb_cols_B = None
        self.pad_groups_A = self.pad_groups_B = None
        self.pad_rows_A = self.pad_rows_B = self.pad_cols_A = self.pad_cols_B = None
        self.raw_grad = None
        self.init_layerwise = init_layerwise
        self.split = None
        self.keep_scores = False
        self.last_scores = None

    _force_headwise = False       # the Batching classes set n_G = heads (matmul.py:411-417)

    def _get_padding_parameters(self, A, B):
        """reference: matmul.py:109-122 (groups of consecutive heads, zero padding).  The CUDA path implements the two
        layouts PTQ4ViT meets: one group per head (what the Batching classes force, :411-417) and one group for all
        heads (the constructor default n_G = 1 of the non-batching classes)."""
        H = A.shape[1]
        if self._force_headwise:
            self.n_G_A = self.n_G_B = H
        for n_G in (self.n_G_A, self.n_G_B):
            if n_G not in (1, H):
                raise NotImplementedError(f"ptq4vit_b200 MatMul search: n_G must be 1 or the number of heads ({H}), got {n_G}")
        self.crb_groups_A, self.crb_groups_B = H // self.n_G_A, H // self.n_G_B
        self.crb_rows_A, self.crb_cols_A = A.shape[2], A.shape[3]
        self.crb_rows_B, self.crb_cols_B = B.shape[2], B.shape[3]
        self.pad_groups_A = self.pad_groups_B = 0
        self.pad_rows_A = self.pad_rows_B = self.pad_cols_A = self.pad_cols_B = 0

    def _grad_for_metric(self, y):
        """Per-element weight of the metric (matmul.py:465-479); see _metric.py."""
        return metric_weight(self.metric, y, self.raw_grad, "PTQSLBatchingQuantMatMul")

    def _native_calibrate(self, A, B, Y, G):
        if (self.n_V_A, self.n_H_A, self.n_V_B, self.n_H_B) != (1, 1, 1, 1):
            raise NotImplementedError("ptq4vit_b200 MatMul search implements the head-wise layout only (n_V = n_H = 1)")
        A_, B_, Y_, G_ = self._cuda(A), self._cuda(B), self._cuda(Y), self._cuda(G)
        dev = A_.device
        self._get_padding_parameters(A_, B_)
        n_G = self.n_G_B if self.sos else self.n_G_A
        if not self.sos and self.n_G_A != self.n_G_B:
            raise NotImplementedError("ptq4vit_b200 MatMul search: A and B must use the same group layout")
        if n_G == 1 and A_.shape[1] > 1:      # one group for all heads: the heads become part of the batch
            A_, B_, Y_, G_ = [t.reshape(-1, 1, t.shape[2], t.shape[3]) for t in (A_, B_, Y_, G_)]
        d = self._desc(A_, B_, self.search_round, (self.eq_alpha, self.eq_beta, self.eq_n))
        H = d.heads
        lib = _lib.lib()
        nbytes, nlog = ctypes.c_size_t(), ctypes.c_size_t()

        def ws_bytes(images_per_chunk):
            d.images_per_chunk = images_per_chunk
            _lib.check(lib.p4v_matmul_workspace_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_matmul_workspace_bytes")
            return nbytes.value
        images_per_chunk, n_chunks = choose_chunks(d.batch, 1, ws_bytes, workspace_budget(dev))
        ws_bytes(images_per_chunk)
        if n_chunks > 1:         # the reference's batching attributes (matmul.py:396-409)
            self.calib_need_batching = True
            self.calib_batch_size = max(1, images_per_chunk // (d.batch // int(A.shape[0])))   # heads folded into the batch
        self.calib_chunks = n_chunks
        _lib.check(lib.p4v_matmul_score_log_floats(ctypes.byref(d), ctypes.byref(nlog)), "p4v_matmul_score_log_floats")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        a_int = torch.empty(H, dtype=torch.float32, device=dev)
        b_int = torch.empty(H, dtype=torch.float32, device=dev)
        split = torch.empty(1, dtype=torch.float32, device=dev) if self.sos else None
        log = torch.empty(nlog.value, dtype=torch.float32, device=dev) if self.keep_scores else None
        _lib.check(lib.p4v_matmul_calibrate(ctypes.byref(d), _lib.ptr(A_), _lib.ptr(B_), _lib.ptr(Y_), _lib.ptr(G_), _lib.ptr(ws),
                                            nbytes.value, _lib.ptr(a_int), _lib.ptr(b_int), _lib.ptr(split), _lib.ptr(log),
                                            ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_matmul_calibrate")
        if self.sos:
            self.split = split[0]
            self.A_interval = a_int[0]
        else:
            self.A_interval = a_int.view(1, H, 1, 1, 1, 1, 1)
        self.B_interval = b_int.view(1, H, 1, 1, 1, 1, 1)
        if log is not None:
            out, o = [], 0
            for _ in range(self.search_round):
                n1 = 20 if self.sos else self.eq_n * H
                out.append(log[o:o + n1] if self.sos else log[o:o + n1].view(self.eq_n, H)); o += n1
                out.append(log[o:o + self.eq_n * H].view(self.eq_n, H)); o += self.eq_n * H
            self.last_scores = out

    def calibration_step2(self, A, B):
        """reference: matmul.py:257-282"""
        Y = self.raw_out
        self._native_calibrate(A, B, Y, self._grad_for_metric(Y))
        self.calibrated = True
        del self.raw_input, self.raw_out, self.raw_grad
        return self.quant_forward(A, B)


class SoSPTQSLQuantMatMul(PTQSLQuantMatMul):
    """reference: quant_layers/matmul.py:284-388 (split-of-softmax, twin-uniform A)"""
    sos = True

    def __init__(self, *args, split=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.n_G_A = self.n_V_A = self.n_H_A = 1
        self.A_qmax = 2 ** (self.A_bit - 1)
        self.split = split
        if split is not None:
            self.A_interval = self.split / (self.A_qmax - 1)


class PTQSLBatchingQuantMatMul(PTQSLQuantMatMul):
    """reference: quant_layers/matmul.py:390-576"""
    _force_headwise = True

    def _initialize_calib_parameters(self):
        """reference: matmul.py:396-409.  The search batches only when its workspace does not fit in the free device
        memory; _native_calibrate then sets calib_need_batching and calib_batch_size (images per chunk)."""
        self.calib_size = int(self.raw_input[0].shape[0])
        self.calib_batch_size = int(self.raw_input[0].shape[0])
        self.calib_need_batching = False

    def calibration_step2(self):
        """reference: matmul.py:565-576"""
        self._initialize_calib_parameters()
        Y = self.raw_out
        self._native_calibrate(self.raw_input[0], self.raw_input[1], Y, self._grad_for_metric(Y))
        self.calibrated = True
        del self.raw_input, self.raw_out, self.raw_grad


class SoSPTQSLBatchingQuantMatMul(PTQSLBatchingQuantMatMul):
    """reference: quant_layers/matmul.py:578-644"""
    sos = True

    def __init__(self, *args, split=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.n_G_A = self.n_V_A = self.n_H_A = 1
        self.A_qmax = 2 ** (self.A_bit - 1)
        self.split = split
        if split is not None:
            self.A_interval = self.split / (self.A_qmax - 1)
