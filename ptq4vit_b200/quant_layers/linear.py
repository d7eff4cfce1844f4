"""Linear quant operators with the reference's class surface (quant_layers/linear.py).

Same constructors, attributes (`w_interval [n_V,1,n_H,1]`, `a_interval [n_a,1]`,
`calibrated`, `mode`, `raw_input/raw_out/raw_grad`) and methods; the interval search
and the quantized forward run in the CUDA library (ptq4vit_b200._lib).  There is no
PyTorch fallback for the search: a missing library or a CPU tensor raises.
"""
import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib
from ._chunking import choose_chunks, workspace_budget
from ._metric import metric_weight

GELU_MIN_NEG = 0.16997124254703522  # reference: quant_layers/linear.py:574


def _flat2d(t):
    return t.reshape(-1, t.shape[-1]).contiguous().float()


class _QuantLinearFn(torch.autograd.Function):
    """Keeps the native quantized forward inside autograd.  In the reference `quant_forward` is
    F.linear(x_sim, w_sim, bias) with x_sim / w_sim built by `.round_()` (linear.py:46-67), whose derivative is zero:
    no gradient reaches x or the weight, but the output carries a grad_fn (through the bias / weight Parameters), so
    that with sequential=True the gradient hooks of the modules BEHIND an already-quantized layer still fire
    (utils/quant_calib.py:330-341).  Same here: the output requires grad, every input gradient is zero."""

    @staticmethod
    def forward(ctx, module, x, weight, bias):
        ctx.x_meta = (x.shape, x.dtype, x.device) if x.requires_grad else None
        return module._quant_forward_native(x)

    @staticmethod
    def backward(ctx, grad_out):
        gx = None if ctx.x_meta is None else torch.zeros(ctx.x_meta[0], dtype=ctx.x_meta[1], device=ctx.x_meta[2])
        return None, gx, None, None


class MinMaxQuantLinear(nn.Linear):
    """reference: quant_layers/linear.py:6-92"""

    post_gelu = False

    def __init__(self, in_features: int, out_features: int, bias: bool = True, mode="raw", w_bit=8, a_bit=8,
                 bias_bit=None, bias_correction=False):
        super().__init__(in_features, out_features, bias)
        self.n_calibration_step = 2
        self.mode = mode
        self.w_bit = w_bit
        self.a_bit = a_bit
        self.bias_bit = bias_bit
        assert bias_bit is None, "No support bias bit now"
        self.w_interval = None
        self.a_interval = None
        self.raw_input = None
        self.raw_out = None
        self.metric = None
        self.next_nodes = []
        self.w_qmax = 2 ** (self.w_bit - 1)
        self.a_qmax = 2 ** (self.a_bit - 1)
        self.bias_correction = bias_correction
        # block structure of the base class: one block
        self.n_V = self.n_H = self.n_a = 1
        self._packed = None                  # freeze(): packed integer weights and tables (torch.uint8, device)

    def forward(self, x):
        if self.mode == "raw":
            out = F.linear(x, self.weight, self.bias)
        elif self.mode == "quant_forward":
            out = self.quant_forward(x)
        elif self.mode == "calibration_step1":
            out = self.calibration_step1(x)
        elif self.mode == "calibration_step2":
            out = self.calibration_step2(x)
        else:
            raise NotImplementedError
        return out

    # ---- native plumbing -------------------------------------------------
    def _desc(self, rows, tokens, search_round=1, eq=(0.0, 1.0, 1)):
        d = _lib.LinearDesc()
        d.rows, d.tokens = int(rows), int(tokens)
        d.in_features, d.out_features = self.in_features, self.out_features
        d.n_V, d.n_H, d.n_a = int(self.n_V), int(self.n_H), int(self.n_a)
        d.w_bit, d.a_bit = int(self.w_bit), int(self.a_bit)
        d.eq_n, d.search_round = int(eq[2]), int(search_round)
        d.eq_alpha, d.eq_beta = float(eq[0]), float(eq[1])
        d.post_gelu = 1 if self.post_gelu else 0
        d.has_bias = 0 if self.bias is None else 1
        d.operand = _lib.default_operand()
        d.kernel = _lib.default_kernel()
        d.init_layerwise = 1 if getattr(self, "init_layerwise", False) else 0
        return d

    def _device(self):
        dev = self.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ptq4vit_b200 quant layers need their parameters on a CUDA device "
                               "(no CPU path; the reference semantics live in oracle/ for tests only)")
        return dev

    def _w_flat(self):
        return torch.as_tensor(self.w_interval, dtype=torch.float32, device=self._device()).reshape(-1).contiguous()

    def _a_flat(self):
        a = self.a_interval
        if isinstance(a, (list, tuple)):        # non-batching PostGelu keeps [pos, neg]
            a = a[0]
        return torch.as_tensor(a, dtype=torch.float32, device=self._device()).reshape(-1).contiguous()

    def quant_forward(self, x):
        """reference: linear.py:62-67 -- fq(x) @ fq(W)^T + b on the tensor cores."""
        assert self.calibrated is not None, f"You should run calibrate_forward before run quant_forward for {self}"
        if torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad):
            return _QuantLinearFn.apply(self, x, self.weight, self.bias)
        return self._quant_forward_native(x)

    # ---- frozen layer: integer weights packed once (csrc/forward_tc.cu) ----
    def _interval_versions(self):
        a = self.a_interval[0] if isinstance(self.a_interval, (list, tuple)) else self.a_interval
        return tuple(getattr(t, "_version", None) for t in (self.w_interval, a))

    def freeze(self, weight=None):
        """Pack the layer's int8 weights and scale tables once; until unfreeze(), quant_forward runs the frozen forward,
        which reads no FP32 weight and is bit-identical to the unfrozen one.  `weight`: quantise this [out, in] tensor
        instead of self.weight (utils/deploy.py passes the dequantised integers of a saved model)."""
        if not getattr(self, "calibrated", None):
            raise RuntimeError(f"freeze() needs a calibrated module: {self}")
        dev = self._device()
        d = self._desc(1, 1)
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_linear_pack_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_linear_pack_bytes")
        fused = _rule("p4v_linear_frozen_path", self)
        packed = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        w = (self.weight if weight is None else weight).detach().to(dev).reshape(self.out_features, self.in_features).contiguous().float()
        wi, ai = self._w_flat(), self._a_flat()
        _lib.check(lib.p4v_linear_pack(ctypes.byref(d), _lib.ptr(w), _lib.ptr(wi), _lib.ptr(ai), _lib.ptr(packed), nbytes.value,
                                       ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "p4v_linear_pack")
        self._packed, self._frozen_fused, self._frozen_ws = packed, fused, None
        # the step sizes that were packed: the objects (kept, so their identity cannot be reused) and their versions
        self._frozen_intervals = (self.w_interval, self.a_interval, self._interval_versions())
        return self

    def unfreeze(self):
        self._packed = self._frozen_ws = self._frozen_intervals = None
        return self

    @property
    def frozen(self):
        return self._packed is not None

    def _check_frozen_intervals(self):
        w0, a0, v0 = self._frozen_intervals
        if self.w_interval is not w0 or self.a_interval is not a0 or self._interval_versions() != v0:
            raise RuntimeError(f"{self}: the step sizes changed after freeze(); call unfreeze() (and freeze() again) "
                               "before running the layer")

    def _quant_forward_native(self, x):
        if self._packed is not None:
            return _frozen_call(self, x)
        dev = self._device()
        x2 = _flat2d(x.to(dev))
        d = self._desc(x2.shape[0], 1)
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_linear_quant_forward_workspace_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "quant_forward_workspace")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        out = torch.empty(x2.shape[0], self.out_features, dtype=torch.float32, device=dev)
        w = self.weight.detach().contiguous().float()
        b = None if self.bias is None else self.bias.detach().contiguous().float()
        wi, ai = self._w_flat(), self._a_flat()
        _lib.check(lib.p4v_linear_quant_forward(ctypes.byref(d), _lib.ptr(x2), _lib.ptr(w), _lib.ptr(b), _lib.ptr(wi),
                                                _lib.ptr(ai), _lib.ptr(ws), nbytes.value, _lib.ptr(out),
                                                ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_linear_quant_forward")
        return out.reshape(*x.shape[:-1], self.out_features)

    def quant_weight_bias(self):
        """reference: linear.py:46-55 / :152-162 (fake-quantized weight as a float tensor)."""
        wi = torch.as_tensor(self.w_interval, dtype=torch.float32, device=self.weight.device).reshape(self.n_V, 1, self.n_H, 1)
        w = self.weight.view(self.n_V, self.out_features // self.n_V, self.n_H, self.in_features // self.n_H)
        w_sim = (w / wi).round_().clamp_(-self.w_qmax, self.w_qmax - 1).mul_(wi).view(self.out_features, self.in_features)
        return w_sim, self.bias

    def quant_input(self, x):
        """reference: linear.py:57-60 / :164-169 / :601-607."""
        ai = self._a_flat().to(x.device).reshape(self.n_a, 1)
        xv = x.reshape(*x.shape[:-1], self.n_a, self.in_features // self.n_a)
        if self.post_gelu:
            neg = GELU_MIN_NEG / self.a_qmax
            x_pos = (xv / ai).round_().clamp_(0, self.a_qmax - 1).mul_(ai)
            x_neg = (xv / neg).round_().clamp_(-self.a_qmax, 0).mul_(neg)
            return (x_pos + x_neg).reshape_as(x)
        return (xv / ai).round_().clamp_(-self.a_qmax, self.a_qmax - 1).mul_(ai).reshape_as(x)

    def _bias_correction_quant_forward(self, x):
        """reference: linear.py:69-77"""
        if self.bias_correction and self.bias is not None:
            w_sim = self.quant_weight_bias()[0]
            x_sim = self.quant_input(x)
            eps = F.linear(x_sim, w_sim - self.weight.data, None)
            eps = torch.mean(eps, dim=(list(range(len(eps.shape) - 1))), keepdim=False)
            self.bias -= eps
            self.bias_correction = False
        return self.quant_forward(x)

    def calibration_step1(self, x):
        """reference: linear.py:79-84"""
        out = F.linear(x, self.weight, self.bias)
        self.raw_input = x.cpu().detach()
        self.raw_out = out.cpu().detach()
        return out

    def calibration_step2(self, x):
        """reference: linear.py:86-92 (layer-wise min-max)"""
        self.w_interval = (self.weight.data.abs().max() / (self.w_qmax - 0.5)).detach()
        self.a_interval = (x.abs().max() / (self.a_qmax - 0.5)).detach()
        self.calibrated = True
        out = self._bias_correction_quant_forward(x)
        return out


def _rule(fn, *layers, extra=()):
    """A shape rule of the library (an int written through its last argument) over the layers' descriptors and the
    ctypes structures `extra`, all by reference; the rules ignore the rows."""
    ok = ctypes.c_int()
    args = [ctypes.byref(m._desc(1, 1)) for m in layers] + [ctypes.byref(a) for a in extra]
    _lib.check(getattr(_lib.lib(), fn)(*args, ctypes.byref(ok)), fn)
    return bool(ok.value)


def _frozen_quant_forward(m):
    """m is a frozen Linear layer in quant_forward mode"""
    return isinstance(m, MinMaxQuantLinear) and m.frozen and m.mode == "quant_forward"


def _wants_no_grad(tensors, modules):
    """Under grad mode no tensor and no parameter of the modules requires grad (else the unfused call has a grad_fn)"""
    return not (torch.is_grad_enabled() and (any(t.requires_grad for t in tensors) or
                                             any(p.requires_grad for m in modules for p in m.parameters())))


def _window_layout_ok(height, width, window, shift):
    """Swin's window rule: windows tile the image and the shift lies inside one"""
    return window > 0 and height % window == 0 and width % window == 0 and 0 <= shift < window


def _streamed_image(lin, dev, fn, *descs):
    """lin's int8 activation image of a streamed call (fn: the library call that sizes it), kept in lin between calls
    and allocated again when it is too small or on another device."""
    nbytes = ctypes.c_size_t()
    _lib.check(getattr(_lib.lib(), fn)(*[ctypes.byref(d) for d in descs], ctypes.byref(nbytes)), fn)
    if lin._frozen_ws is None or lin._frozen_ws.numel() < nbytes.value or lin._frozen_ws.device != dev:
        lin._frozen_ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    return lin._frozen_ws


def _frozen_call(lin, x, norm=None, fc2=None, residual=None, layout=None, gather=None):
    """One library call of frozen layers: lin(x), on lin's fused kernel or its streamed path; with `norm`, lin(norm(x))
    with the LayerNorm folded into lin's fused kernel; with `fc2`, fc2(gelu(lin(...))) as the fused MLP; with
    `residual`, residual + that output, the add folded into the last layer's store (with `layout`, an (images, height,
    width, window, shift) window layout of lin's output rows: Swin's window reverse and reverse shift before the add);
    with `gather` (and `norm`), lin(norm(rows of the image x)), the rows gathered by lin's fused kernel (see
    frozen_gather_applies).  The callers' rules say which applies; the library validates the call.  Only the output (and a
    missing streamed image) is allocated."""
    for m in (lin, fc2):
        if m is not None:
            m._check_frozen_intervals()
    dev = lin._packed.device
    x2 = _flat2d(x.to(dev))
    b1, b2 = (None if m is None or m.bias is None else m.bias.detach().contiguous().float() for m in (lin, fc2))
    rows = x2.shape[0] if gather is None else _gather_rows(gather)
    d1 = lin._desc(rows, 1)
    args = [ctypes.byref(d1), _lib.ptr(x2)]
    if norm is not None:
        args += [_lib.ptr(norm.weight), _lib.ptr(norm.bias), float(norm.eps)]
    args += [_lib.ptr(b1), _lib.ptr(lin._packed)]
    ws = None
    if fc2 is not None:                  # fc1's epilogue writes fc2's image, kept in fc2
        d2 = fc2._desc(x2.shape[0], 1)
        args += [lin._packed.numel(), ctypes.byref(d2), _lib.ptr(b2), _lib.ptr(fc2._packed), fc2._packed.numel()]
        ws = _streamed_image(fc2, dev, "p4v_mlp_frozen_workspace_bytes", d1, d2)
    elif norm is None and not lin._frozen_fused:
        ws = _streamed_image(lin, dev, "p4v_linear_frozen_workspace_bytes", d1)
    if fc2 is not None or norm is None:
        args += [_lib.ptr(ws), 0 if ws is None else ws.numel()]
    last = lin if fc2 is None else fc2
    out = torch.empty(rows, last.out_features, dtype=torch.float32, device=dev)
    fn = ("p4v_linear_frozen_forward" if fc2 is None else "p4v_mlp_frozen_forward") + ("" if norm is None else "_norm")
    if gather is not None:
        fn += "_gather"
        args.append(ctypes.byref(_gather_desc(gather)))
    if residual is not None:
        fn += "_res"
        args.append(_lib.ptr(residual))
        if fc2 is None:
            args.append(None if layout is None else ctypes.byref(_lib.WindowLayout(*[int(v) for v in layout])))
    _lib.check(getattr(_lib.lib(), fn)(*args, _lib.ptr(out), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), fn)
    if residual is not None:
        return out.view(residual.shape)
    if gather is not None:
        mode, images, _height, _width, window, _shift = gather
        return out.view(-1, window * window, lin.out_features) if mode == "window" else out.view(images, -1, lin.out_features)
    return out.reshape(*x.shape[:-1], last.out_features)


def _gather_desc(gather):
    mode, *layout = gather
    return _lib.InputGather(_lib.GATHER[mode], _lib.WindowLayout(*[int(v) for v in layout]))


def _gather_rows(gather):
    """The output rows of a gathered call: the image's rows (window), a quarter of them (merge)"""
    mode, images, height, width, _window, _shift = gather
    return images * height * width if mode == "window" else images * (height // 2) * (width // 2)


def frozen_mlp_applies(fc1, fc2, act, x):
    """Whether one call of an MLP block fc2(act(fc1(x))) can run as the fused frozen MLP (frozen_mlp): fc1 and fc2 frozen
    Linear layers in quant_forward mode, act exactly torch's exact GELU (nn.GELU(approximate='none')), under grad mode
    no input and no parameter of the layers that requires grad (the unfused call then carries a grad_fn), and a shape the
    kernel holds (p4v_mlp_fused_ok: fc1.out_features == fc2.in_features, fc1 not post-GELU and on its fused kernel, the
    shared-memory plan fits)."""
    if not (_frozen_quant_forward(fc1) and _frozen_quant_forward(fc2)):
        return False
    if type(act) is not nn.GELU or act.approximate != "none":
        return False
    return _wants_no_grad((x,), (fc1, fc2)) and _rule("p4v_mlp_fused_ok", fc1, fc2)


def frozen_mlp(fc1, fc2, x, norm=None, residual=None):
    """fc2(gelu(fc1(x))) of two frozen layers in two launches (csrc/forward_tc.cu: fc1 with a GELU-and-quantise
    epilogue writing fc2's int8 activation image; fc2's sweep forward), for a call where frozen_mlp_applies holds.  The
    bits are those of the unfused sequence.  fc2's image is kept between calls in fc2's frozen workspace.
    With `norm` (an nn.LayerNorm for which frozen_norm_applies(norm, fc1, x) and frozen_mlp_norm_ok(fc1, fc2) hold):
    fc2(gelu(fc1(norm(x)))), the LayerNorm folded into fc1's activation quantiser, still two launches.
    With `residual` (frozen_residual_applies(fc2, x, residual) holds): residual + that, added in fc2's store."""
    return _frozen_call(fc1, x, norm=norm, fc2=fc2, residual=residual)


def frozen_residual_applies(lin, x, residual, layout=None):
    """Whether residual + lin(x) -- with `layout` (images, height, width, window, shift), residual + Swin's window reverse
    and reverse roll of lin(x) -- can run as one folded call (frozen_residual_linear), or as the same add folded into a
    fused MLP whose fc2 is `lin` (frozen_mlp(..., residual=)): lin a frozen Linear layer in quant_forward mode, residual an
    FP32 tensor on lin's device, contiguous, 8-byte aligned, with the output's shape (with a layout: its number of rows
    and lin's out_features per row), under grad mode nothing that requires grad, and a layout only for a layer on its
    fused path (the streamed path adds in identity rows only).  x is the input of the call: lin's, or fc1's of the MLP."""
    if not _frozen_quant_forward(lin):
        return False
    dev = lin._packed.device
    if not torch.is_tensor(residual) or residual.dtype != torch.float32 or residual.device != dev:
        return False
    if not residual.is_contiguous() or residual.data_ptr() % 8 or x.numel() == 0:
        return False
    rows = x.numel() // x.shape[-1]
    if layout is None:
        if tuple(residual.shape) != (*x.shape[:-1], lin.out_features):
            return False
    else:
        images, height, width, window, shift = (int(v) for v in layout)
        if not lin._frozen_fused or residual.shape[-1] != lin.out_features or residual.numel() != rows * lin.out_features:
            return False
        if not (_window_layout_ok(height, width, window, shift) and images * height * width == rows):
            return False
    return _wants_no_grad((x, residual), (lin,))


def frozen_residual_linear(lin, x, residual, layout=None):
    """residual + lin(x) in the launches of lin(x), for a call where frozen_residual_applies holds: lin's fused kernel or
    its streamed sweep adds the shortcut as it stores each output value (csrc/forward_tc.cu, csrc/sweep_tc.cu), with
    `layout` at the row Swin's window reverse and reverse roll send it to; bit-identical to the unfolded sequence and lin's
    FP32 output never reaches HBM.  Returns a new tensor of residual's shape; only it is allocated."""
    return _frozen_call(lin, x, residual=residual, layout=layout)


def frozen_norm_applies(norm, lin, x):
    """Whether lin(norm(x)) can run as one folded call (frozen_norm_linear): `norm` exactly an nn.LayerNorm with weight and
    bias over lin.in_features, `lin` a frozen Linear layer in quant_forward mode whose shape holds the fold
    (p4v_linear_norm_ok: on the fused kernel, not post-GELU, in_features % 4 == 0, the shared-memory plan fits), x FP32 on
    lin's device, under grad mode no input and no parameter of norm or lin that requires grad, and the case in which torch
    itself runs its vectorised LayerNorm kernel (FP32 weight and bias, 16-byte aligned data) -- the kernel whose bits the
    fold reproduces (DESIGN.md section 4.10)."""
    return _norm_call_ok(norm, lin, x) and _rule("p4v_linear_norm_ok", lin)


def _layer_norm_ok(norm, features, dev):
    """The LayerNorm conditions of every fold that reproduces it: exactly an nn.LayerNorm with weight and bias over
    `features` (a multiple of 4), both FP32, contiguous and 16-byte aligned on dev -- torch's vectorised case"""
    if type(norm) is not nn.LayerNorm or norm.weight is None or norm.bias is None:
        return False
    if tuple(norm.normalized_shape) != (features,) or features % 4 != 0:
        return False
    return not any(p.dtype != torch.float32 or p.device != dev or not p.is_contiguous() or p.data_ptr() % 16
                   for p in (norm.weight, norm.bias))


def _norm_call_ok(norm, lin, x):
    """frozen_norm_applies without the library's shape rule"""
    if not _frozen_quant_forward(lin):
        return False
    dev = lin._packed.device
    if not _layer_norm_ok(norm, lin.in_features, dev):
        return False
    if x.dtype != torch.float32 or x.device != dev or x.numel() == 0:
        return False
    if x.is_contiguous() and x.data_ptr() % 16:       # torch normalises a non-contiguous x from an aligned copy
        return False
    return _wants_no_grad((x,), (norm, lin))


def frozen_mlp_norm_ok(fc1, fc2):
    """The shape rule of frozen_mlp(..., norm=): fc1 and fc2 fuse (p4v_mlp_fused_ok) and the plan with the LayerNorm's
    row statistics still fits (p4v_mlp_norm_ok)."""
    return _rule("p4v_mlp_norm_ok", fc1, fc2)


def frozen_norm_linear(norm, lin, x):
    """lin(norm(x)) in one launch, for a call where frozen_norm_applies(norm, lin, x) holds: torch's exact LayerNorm
    computed in the activation quantiser of lin's fused kernel (csrc/forward_tc.cu), bit-identical to the unfolded call;
    the normalised activations never reach HBM.  Only the output is allocated."""
    return _frozen_call(lin, x, norm=norm)


def frozen_gather_ok(lin, mode):
    """The library's shape rule of a row gather (p4v_linear_gather_ok) for lin, mode "window" or "merge":
    p4v_linear_norm_ok, in_features % 16 == 0 for the merge, the shared-memory plan with the table of source rows fits."""
    return _rule("p4v_linear_gather_ok", lin, extra=(_gather_desc((mode, 0, 0, 0, 0, 0)),))


def frozen_gather_applies(norm, lin, x, gather):
    """Whether lin(norm(rows gathered from x)) can run as one folded call (frozen_gather_linear).  gather is
    ("window", images, height, width, window, shift): x is Swin's [images, height * width, C] block input and the rows
    are those of window_partition(roll(x, (-shift, -shift))), C = lin.in_features; or ("merge", images, height, width, 0,
    0): x is PatchMerging's [images, height * width, C] input and the rows are its cat of the 2x2 neighbourhoods,
    C = lin.in_features / 4.  The conditions of frozen_norm_applies, x contiguous with the image's shape, a valid layout
    and the library's rule (frozen_gather_ok) -- DESIGN.md section 4.12."""
    mode, images, height, width, window, shift = gather
    if mode not in _lib.GATHER or not torch.is_tensor(x) or not x.is_contiguous():
        return False
    C = lin.in_features if mode == "window" else lin.in_features // 4
    if x.dim() < 2 or x.shape[-1] != C or x.numel() != images * height * width * C or images <= 0:
        return False
    if mode == "window":
        if not _window_layout_ok(height, width, window, shift):
            return False
    elif not (window == 0 and shift == 0 and height % 2 == 0 and width % 2 == 0 and lin.in_features == 4 * C):
        return False
    return _norm_call_ok(norm, lin, x) and frozen_gather_ok(lin, mode)


def frozen_gather_linear(norm, lin, x, gather):
    """lin(norm(rows gathered from x)) in one launch, for a call where frozen_gather_applies(norm, lin, x, gather) holds:
    lin's fused kernel reads each row from the image x, computes torch's exact LayerNorm of it and quantises it
    (csrc/forward_tc.cu), bit-identical to torch's LayerNorm, roll and window partition (or cat) followed by lin.  Returns
    the window rows [images * windows, window^2, out_features] or the merged rows [images, height * width / 4,
    out_features]; only the output is allocated."""
    return _frozen_call(lin, x, norm=norm, gather=gather)


class PTQSLQuantLinear(MinMaxQuantLinear):
    """reference: quant_layers/linear.py:94-260"""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, mode="raw", w_bit=8, a_bit=8,
                 bias_bit=None, bias_correction=False, metric="L2_norm", search_round=1, eq_alpha=0, eq_beta=1,
                 eq_n=100, parallel_eq_n=10, n_H=1, n_V=1, n_a=1, init_layerwise=False):
        super().__init__(in_features, out_features, bias=bias, mode=mode, w_bit=w_bit, a_bit=a_bit, bias_bit=bias_bit,
                         bias_correction=bias_correction)
        self.metric = metric
        self.search_round = search_round
        self.eq_alpha = eq_alpha
        self.eq_beta = eq_beta
        self.eq_n = eq_n
        self.n_H = n_H
        self.n_V = n_V
        self.n_a = n_a
        self.crb_rows = out_features // n_V
        self.crb_cols = in_features // n_H  # ignore remnent != 0 situations
        self.crb_acts = in_features // n_a
        self.parallel_eq_n = parallel_eq_n   # kept for signature parity; the CUDA path sizes its chunks by device memory
        self.init_layerwise = init_layerwise
        self.raw_grad = None
        self.last_scores = None              # optional per-step score tables (set P4V_SCORE_LOG=1 or keep_scores=True)
        self.keep_scores = False

    # ---- native search ---------------------------------------------------
    def _grad_for_metric(self, y):
        """Per-element weight of the metric (linear.py:406-422); see _metric.py."""
        return metric_weight(self.metric, y, self.raw_grad, "_get_similarity")

    def _native_calibrate(self, x, y, g):
        dev = self._device()
        tokens = 1
        if x.dim() > 2:
            for s in x.shape[1:-1]:
                tokens *= int(s)
        x2, y2, g2 = _flat2d(x.to(dev)), _flat2d(y.to(dev)), _flat2d(g.to(dev))
        d = self._desc(x2.shape[0], tokens, self.search_round, (self.eq_alpha, self.eq_beta, self.eq_n))
        lib = _lib.lib()
        nbytes, nlog = ctypes.c_size_t(), ctypes.c_size_t()

        def ws_bytes(rows_per_chunk):
            d.rows_per_chunk = rows_per_chunk
            _lib.check(lib.p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_linear_workspace_bytes")
            return nbytes.value
        # rows per chunk: a multiple of the 128-row tile; 0 (the whole layer) whenever it fits
        rows_per_chunk, n_chunks = choose_chunks(d.rows, 128, ws_bytes, workspace_budget(dev))
        ws_bytes(rows_per_chunk)
        if n_chunks > 1:         # the reference's batching attributes: images per chunk (a chunk may end inside an image)
            self.calib_need_batching = True
            self.calib_batch_size = -(-rows_per_chunk // tokens)
        self.calib_chunks = n_chunks
        _lib.check(lib.p4v_linear_score_log_floats(ctypes.byref(d), ctypes.byref(nlog)), "p4v_linear_score_log_floats")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        w = self.weight.detach().contiguous().float()
        b = None if self.bias is None else self.bias.detach().contiguous().float()
        w_int = torch.empty(self.n_V * self.n_H, dtype=torch.float32, device=dev)
        a_int = torch.empty(self.n_a, dtype=torch.float32, device=dev)
        log = torch.empty(nlog.value, dtype=torch.float32, device=dev) if self.keep_scores else None
        _lib.check(lib.p4v_linear_calibrate(ctypes.byref(d), _lib.ptr(x2), _lib.ptr(w), _lib.ptr(b), _lib.ptr(y2),
                                            _lib.ptr(g2), _lib.ptr(ws), nbytes.value, _lib.ptr(w_int), _lib.ptr(a_int),
                                            _lib.ptr(log), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_linear_calibrate")
        self.w_interval = w_int.view(self.n_V, 1, self.n_H, 1)
        self.a_interval = a_int.view(self.n_a, 1)
        self.last_scores = self._split_log(log) if log is not None else None

    def _split_log(self, log):
        out, o = [], 0
        for _ in range(self.search_round):
            for _h in range(self.n_H):
                out.append(log[o:o + self.eq_n * self.n_V].view(self.eq_n, self.n_V)); o += self.eq_n * self.n_V
            for _a in range(self.n_a):
                out.append(log[o:o + self.eq_n]); o += self.eq_n
        return out

    def calibration_step2(self, x):
        """reference: linear.py:235-260 (x already on the device; raw_out/raw_grad attributes)"""
        y = self.raw_out
        self._native_calibrate(x, y, self._grad_for_metric(y))
        if self.post_gelu:   # the non-batching PostGelu class stores [pos, neg] (linear.py:316-320)
            self.a_interval = [self.a_interval, GELU_MIN_NEG / self.a_qmax]
        self.calibrated = True
        with torch.no_grad():
            out = self._bias_correction_quant_forward(x)
        del self.raw_input, self.raw_out, self.raw_grad
        return out


class PostGeluPTQSLQuantLinear(PTQSLQuantLinear):
    """reference: quant_layers/linear.py:262-347 (twin-uniform post-GELU activations)"""
    post_gelu = True


class PTQSLBatchingQuantLinear(PTQSLQuantLinear):
    """reference: quant_layers/linear.py:349-555"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.calib_size = None
        self.calib_batch_size = None
        self.calib_need_batching = False

    def _initialize_calib_parameters(self):
        """reference: linear.py:365-378.  The search batches only when its workspace does not fit in the free device
        memory; _native_calibrate then sets calib_need_batching and calib_batch_size (images per chunk of rows)."""
        self.calib_size = int(self.raw_input.shape[0])
        self.calib_batch_size = int(self.raw_input.shape[0])
        self.calib_need_batching = False

    def calibration_step2(self):
        """reference: linear.py:536-555 -- only uses the cached raw inputs / outs / grads."""
        self._initialize_calib_parameters()
        y = self.raw_out
        self._native_calibrate(self.raw_input, y, self._grad_for_metric(y))
        self.calibrated = True
        del self.raw_input, self.raw_out, self.raw_grad
        return None


class PostGeluPTQSLBatchingQuantLinear(PTQSLBatchingQuantLinear):
    """reference: quant_layers/linear.py:557-642"""
    post_gelu = True

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.a_neg_interval = GELU_MIN_NEG / self.a_qmax
