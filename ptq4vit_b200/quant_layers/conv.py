"""Conv2d quant operators with the reference's class surface (quant_layers/conv.py).

PTQ4ViT wraps exactly one convolution per network, the patch embedding, with
`ChannelwiseBatchingQuantConv2d(..., a_bit=32)` (configs/PTQ4ViT.py:52-54): per-output-channel weight
step sizes, activations left in FP32.  The search runs in the CUDA library as a batched product over
the images: rows = output channels (candidate planes of the quantised kernel), columns = output
positions (im2col of the FP32 input, split exactly into three bf16 terms), one score per channel.

BasePTQ wraps it with `BatchingEasyQuantConv2d(..., a_bit=32)` (configs/BasePTQ.py:48-50): one weight
step size for the whole kernel.  The library runs the same search with every channel given that step
size and sums the per-channel scores of a candidate into one (`p4v_conv_desc.layerwise`).

After calibration a module can be frozen (`freeze()`): its integer weights are packed once as a bf16 image, and every
quant_forward call that wants no gradient runs one kernel that gathers the patches from the image, splits the FP32
pixels exactly into three bf16 terms and multiplies them with the integers on the tensor cores
(csrc/forward_conv_tc.cu).  It reads no FP32 weight and does not depend on torch's TF32 setting.  Not bit-identical to
cuDNN's F.conv2d: the contract is a bound against fp64 (DESIGN.md section 4.9).

frozen_stem folds the model's stem after the patch embedding into that kernel's store (DESIGN.md section 4.13): ViT's cls
token and pos_embed, Swin's patch_norm.  It returns the bits of the frozen conv followed by torch's ops.
"""
import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib
from ._metric import check_metric, metric_weight
from .linear import _layer_norm_ok


class MinMaxQuantConv2d(nn.Conv2d):
    """reference: quant_layers/conv.py:9-89"""

    def __init__(self, in_channels: int, out_channels: int, kernel_size, stride=1, padding=0, dilation=1, groups: int = 1,
                 bias: bool = True, padding_mode: str = "zeros", mode="raw", w_bit=8, a_bit=8, bias_bit=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, padding_mode)
        self.n_calibration_steps = 2
        self.mode = mode
        self.w_bit = w_bit
        self.a_bit = a_bit
        self.bias_bit = bias_bit
        assert bias_bit is None, "No support bias bit now"
        self.w_interval = None
        self.a_interval = None
        self.bias_interval = None
        self.raw_input = None
        self.raw_out = None
        self.metric = None
        self.next_nodes = []
        self.w_qmax = 2 ** (self.w_bit - 1)
        self.a_qmax = 2 ** (self.a_bit - 1)
        self._packed = None                  # freeze(): packed bf16 integer weights and step sizes (torch.uint8, device)

    def forward(self, x):
        if self.mode == "raw":
            out = F.conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)
        elif self.mode == "quant_forward":
            out = self.quant_forward(x)
        elif self.mode == "calibration_step1":
            out = self.calibration_step1(x)
        elif self.mode == "calibration_step2":
            out = self.calibration_step2(x)
        else:
            raise NotImplementedError
        return out

    def quant_weight_bias(self):
        """reference: conv.py:53-62"""
        wi = torch.as_tensor(self.w_interval, dtype=torch.float32, device=self.weight.device)
        w_sim = (self.weight / wi).round_().clamp_(-self.w_qmax, self.w_qmax - 1).mul_(wi)
        return w_sim, self.bias

    def quant_input(self, x):
        """reference: conv.py:64-67"""
        ai = torch.as_tensor(self.a_interval, dtype=torch.float32, device=x.device)
        return (x / ai).round_().clamp_(-self.a_qmax, self.a_qmax - 1).mul_(ai)

    def quant_forward(self, x):
        """reference: conv.py:69-74.  A frozen module runs the packed forward for calls that want no gradient (under grad
        mode no input and no parameter requires grad); every other call runs the torch operations below."""
        assert self.calibrated is not None, f"You should run calibrate_forward before run quant_forward for {self}"
        if self._packed is not None and not (torch.is_grad_enabled() and
                                             (x.requires_grad or any(p.requires_grad for p in self.parameters()))):
            return self._frozen_forward(x)
        w_sim, bias_sim = self.quant_weight_bias()
        x_sim = self.quant_input(x) if self.a_bit < 32 else x
        return F.conv2d(x_sim, w_sim, bias_sim, self.stride, self.padding, self.dilation, self.groups)

    # ---- frozen module: integer weights packed once (csrc/forward_conv_tc.cu) ----
    def _frozen_desc(self, x=None):
        d = _lib.ConvFrozenDesc()
        if x is not None:
            d.images, d.in_channels, d.height, d.width = (int(s) for s in x.shape)
        else:
            d.in_channels = self.in_channels
        d.out_channels = self.out_channels
        d.kernel_h, d.kernel_w = (int(k) for k in self.kernel_size)
        d.w_bit = int(self.w_bit)
        d.layerwise = 1 if self.w_interval is not None and torch.as_tensor(self.w_interval).numel() == 1 else 0
        d.has_bias = 0 if self.bias is None else 1
        return d

    def frozen_unsupported(self):
        """Why freeze() cannot pack this module (None when it can): the frozen forward implements a_bit >= 32 and the
        patch-embedding geometry -- kernel == stride, no padding, dilation 1, groups 1 -- within the library's shape rule
        (p4v_conv_frozen_ok: K = in_channels * kh * kw and out_channels at most 4096, w_bit in [2, 8])."""
        if self.a_bit < 32:
            return f"a_bit = {self.a_bit}: the frozen convolution keeps the activations in FP32 (a_bit >= 32)"
        if tuple(self.stride) != tuple(self.kernel_size):
            return f"stride {tuple(self.stride)} != kernel_size {tuple(self.kernel_size)}"
        if isinstance(self.padding, str) or any(p != 0 for p in self.padding):
            return f"padding {self.padding!r}: only padding 0"
        if any(dl != 1 for dl in self.dilation):
            return f"dilation {tuple(self.dilation)}: only dilation 1"
        if self.groups != 1:
            return f"groups = {self.groups}: only groups 1"
        if self.w_interval is not None and torch.as_tensor(self.w_interval).numel() not in (1, self.out_channels):
            return f"w_interval has {torch.as_tensor(self.w_interval).numel()} entries: one per output channel or one"
        ok = ctypes.c_int()
        d = self._frozen_desc()
        _lib.check(_lib.lib().p4v_conv_frozen_ok(ctypes.byref(d), ctypes.byref(ok)), "p4v_conv_frozen_ok")
        if not ok.value:
            return (f"K = {d.in_channels * d.kernel_h * d.kernel_w}, out_channels = {d.out_channels}, w_bit = {d.w_bit}: "
                    "outside the shape rule of p4v_conv_frozen_ok")
        return None

    def freeze(self, weight=None):
        """Pack the module's integers (the export quantiser's, utils.integer) as bf16 and its step sizes once; until
        unfreeze(), quant_forward calls that want no gradient run the frozen forward, which reads no FP32 weight.
        `weight`: quantise this [out, in, kh, kw] tensor instead of self.weight (utils/deploy.py passes the dequantised
        integers of a saved model)."""
        if not getattr(self, "calibrated", None):
            raise RuntimeError(f"freeze() needs a calibrated module: {self}")
        why = self.frozen_unsupported()
        if why is not None:
            raise NotImplementedError(f"{type(self).__name__}.freeze(): {why}")
        dev = self.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ptq4vit_b200 quant layers need their parameters on a CUDA device (no CPU path)")
        d = self._frozen_desc()
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_conv_pack_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_conv_pack_bytes")
        packed = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        w = (self.weight if weight is None else weight).detach().to(dev).reshape(self.out_channels, -1).contiguous().float()
        wi = torch.as_tensor(self.w_interval, dtype=torch.float32, device=dev).reshape(-1).contiguous()
        _lib.check(lib.p4v_conv_pack(ctypes.byref(d), _lib.ptr(w), _lib.ptr(wi), _lib.ptr(packed), nbytes.value,
                                     ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "p4v_conv_pack")
        self._packed = packed
        # the step sizes that were packed: the object (kept, so its identity cannot be reused) and its version
        self._frozen_interval = (self.w_interval, getattr(self.w_interval, "_version", None))
        return self

    def unfreeze(self):
        self._packed = self._frozen_interval = None
        return self

    @property
    def frozen(self):
        return self._packed is not None

    def _check_frozen_interval(self):
        w0, v0 = self._frozen_interval
        if self.w_interval is not w0 or getattr(self.w_interval, "_version", None) != v0:
            raise RuntimeError(f"{self}: the step sizes changed after freeze(); call unfreeze() (and freeze() again) "
                               "before running the layer")

    def _frozen_forward(self, x):
        self._check_frozen_interval()
        dev = self._packed.device
        x4 = x.to(dev).contiguous().float()
        if x4.dim() != 4 or x4.shape[1] != self.in_channels:
            raise ValueError(f"{self}: expected input [images, {self.in_channels}, height, width], got {tuple(x.shape)}")
        d = self._frozen_desc(x4)
        out = torch.empty(d.images, self.out_channels, d.height // d.kernel_h, d.width // d.kernel_w, dtype=torch.float32,
                          device=dev)
        b = None if self.bias is None else self.bias.detach().contiguous().float()
        _lib.check(_lib.lib().p4v_conv_frozen_forward(ctypes.byref(d), _lib.ptr(x4), _lib.ptr(b), _lib.ptr(self._packed),
                                                      self._packed.numel(), _lib.ptr(out),
                                                      ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_conv_frozen_forward")
        return out

    def calibration_step1(self, x):
        """reference: conv.py:76-81"""
        out = F.conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)
        self.raw_input = x.cpu().detach()
        self.raw_out = out.cpu().detach()
        return out

    def calibration_step2(self, x):
        """reference: conv.py:83-89 (layer-wise min-max)"""
        self.w_interval = (self.weight.data.abs().max() / (self.w_qmax - 0.5)).detach()
        self.a_interval = (x.abs().max() / (self.a_qmax - 0.5)).detach()
        self.calibrated = True
        return self.quant_forward(x)


def frozen_stem_ok(conv, norm):
    """The library's shape rule of the stem fold for a conv module: p4v_conv_pos_ok (norm False: ViT's cls token and
    pos_embed) or p4v_conv_norm_ok (norm True: Swin's patch_norm, out_channels <= 128).  Both need out_channels % 4 == 0."""
    ok = ctypes.c_int()
    fn = "p4v_conv_norm_ok" if norm else "p4v_conv_pos_ok"
    _lib.check(getattr(_lib.lib(), fn)(ctypes.byref(conv._frozen_desc()), ctypes.byref(ok)), fn)
    return bool(ok.value)


def frozen_stem_applies(conv, x, cls_token=None, pos_embed=None, norm=None):
    """Whether a model's stem can run as one folded call (frozen_stem): with cls_token and pos_embed (ViT / DeiT)
    torch.cat((cls_token.expand(B, -1, -1), conv(x).flatten(2).transpose(1, 2)), 1) + pos_embed, with norm (Swin)
    norm(conv(x).flatten(2).transpose(1, 2)).  conv a frozen conv module in quant_forward mode; x an FP32, contiguous
    [images, in_channels, height, width] image on its device; cls_token [1, 1, C] and pos_embed [1, 1 + positions, C] FP32,
    contiguous and 16-byte aligned there (C = out_channels); norm with the conditions of the LayerNorm folds (an affine
    nn.LayerNorm over C, torch's vectorised case); under grad mode nothing that requires grad; and the library's rule
    (frozen_stem_ok)."""
    if (norm is None) == (cls_token is None) or (cls_token is None) != (pos_embed is None):
        return False
    if not (isinstance(conv, MinMaxQuantConv2d) and conv.frozen and conv.mode == "quant_forward"):
        return False
    dev = conv._packed.device
    if not torch.is_tensor(x) or x.dtype != torch.float32 or x.device != dev or not x.is_contiguous() or x.dim() != 4:
        return False
    (kh, kw), C = conv.kernel_size, conv.out_channels
    if x.shape[0] < 1 or x.shape[1] != conv.in_channels or x.shape[2] < kh or x.shape[3] < kw:
        return False
    params = list(conv.parameters())
    if norm is None:
        shapes = ((1, 1, C), (1, 1 + (x.shape[2] // kh) * (x.shape[3] // kw), C))
        for t, shape in zip((cls_token, pos_embed), shapes):
            if not torch.is_tensor(t) or t.dtype != torch.float32 or t.device != dev or not t.is_contiguous() or \
                    t.data_ptr() % 16 or tuple(t.shape) != shape:
                return False
        params += [cls_token, pos_embed]
    else:
        if not _layer_norm_ok(norm, C, dev):
            return False
        params += list(norm.parameters())
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
        return False
    return frozen_stem_ok(conv, norm is not None)


def frozen_stem(conv, x, cls_token=None, pos_embed=None, norm=None):
    """The model's stem in one launch, for a call where frozen_stem_applies holds: the frozen conv's kernel stores the
    token rows instead of its NCHW output (csrc/forward_conv_tc.cu) -- with cls_token and pos_embed the [images,
    1 + positions, C] rows of ViT's cat and pos_embed add, with norm the [images, positions, C] rows normalised with
    torch's exact LayerNorm -- bit-identical to the frozen conv followed by torch's ops.  Only the output is allocated."""
    conv._check_frozen_interval()
    dev = conv._packed.device
    d = conv._frozen_desc(x)
    P, C = (d.height // d.kernel_h) * (d.width // d.kernel_w), conv.out_channels
    b = None if conv.bias is None else conv.bias.detach().contiguous().float()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    lib = _lib.lib()
    if norm is None:
        out = torch.empty(d.images, 1 + P, C, dtype=torch.float32, device=dev)
        _lib.check(lib.p4v_conv_frozen_forward_pos(ctypes.byref(d), _lib.ptr(x), _lib.ptr(b), _lib.ptr(conv._packed),
                                                   conv._packed.numel(), _lib.ptr(cls_token), cls_token.numel(),
                                                   _lib.ptr(pos_embed), pos_embed.numel(), _lib.ptr(out), stream),
                   "p4v_conv_frozen_forward_pos")
    else:
        out = torch.empty(d.images, P, C, dtype=torch.float32, device=dev)
        _lib.check(lib.p4v_conv_frozen_forward_norm(ctypes.byref(d), _lib.ptr(x), _lib.ptr(b), _lib.ptr(conv._packed),
                                                    conv._packed.numel(), _lib.ptr(norm.weight), _lib.ptr(norm.bias), C,
                                                    float(norm.eps), _lib.ptr(out), stream),
                   "p4v_conv_frozen_forward_norm")
    return out


class PTQSLQuantConv2d(MinMaxQuantConv2d):
    """reference: quant_layers/conv.py:126-277 -- constructor surface (the sub-layerwise search of the non-batching
    class is not part of PTQ4ViT's configuration; only the channel-wise batching class below searches natively)."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size, stride=1, padding=0, dilation=1, groups: int = 1,
                 bias: bool = True, padding_mode: str = "zeros", mode="raw", w_bit=8, a_bit=8, bias_bit=None,
                 metric="L2_norm", search_round=1, eq_alpha=0.1, eq_beta=2, eq_n=100, parallel_eq_n=10, n_V=1, n_H=1,
                 init_layerwise=False):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, bias=bias, padding_mode=padding_mode, mode=mode, w_bit=w_bit, a_bit=a_bit,
                         bias_bit=bias_bit)
        self.metric = metric
        self.search_round = search_round
        self.eq_alpha = eq_alpha
        self.eq_beta = eq_beta
        self.eq_n = int(eq_n)
        self.n_H = n_H
        self.n_V = n_V
        self.parallel_eq_n = parallel_eq_n
        self.crb_rows = out_channels // n_V
        self.crb_cols = in_channels // n_H
        self.init_layerwise = init_layerwise
        self.raw_grad = None
        self.keep_scores = False
        self.last_scores = None


class _BatchingConvSearch(PTQSLQuantConv2d):
    """The weight search of the Batching conv classes with a_bit >= 32, run by the library (csrc/conv_api.cu): per output
    channel, or one step size for the whole kernel when `layerwise` is set."""
    batching = True
    layerwise = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.calib_size = None
        self.calib_batch_size = None
        self.calib_need_batching = False

    def _initialize_calib_parameters(self):
        """reference: conv.py:297-310, :467-480; a whole layer fits in HBM, no batching."""
        self.calib_size = int(self.raw_input.shape[0])
        self.calib_batch_size = int(self.raw_input.shape[0])

    def _grad_for_metric(self, y):
        """Per-element weight of the metric (conv.py:336-349, :509-522); see _metric.py."""
        return metric_weight(self.metric, y, self.raw_grad, "_get_similarity")

    def _check_supported(self):
        name = type(self).__name__
        check_metric(self.metric)
        if self.a_bit < 32:
            raise NotImplementedError(f"{name}: the CUDA path implements a_bit >= 32 (activation quantizer off), as "
                                      "configs/PTQ4ViT.py:54 and configs/BasePTQ.py:50 use it")
        if self.groups != 1 or self.init_layerwise:
            raise NotImplementedError(f"{name}: groups == 1 and init_layerwise=False only")

    def _native_weight_search(self):
        self._initialize_calib_parameters()
        dev = self.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ptq4vit_b200 quant layers need their parameters on a CUDA device (no CPU path)")
        x = self.raw_input.to(dev).float()
        y = self.raw_out.to(dev).float().contiguous()
        g = self._grad_for_metric(y).to(dev).float().contiguous()
        n, oc = y.shape[0], y.shape[1]
        L = y.shape[2] * y.shape[3]
        nw = 1 if self.layerwise else oc
        # im2col of the FP32 input: [n, L, K] (row l = one output position), K = ic*kh*kw in the kernel's own order
        cols = F.unfold(x, self.kernel_size, self.dilation, self.padding, self.stride).transpose(1, 2).contiguous()
        K = cols.shape[2]
        w2 = self.weight.detach().reshape(oc, K).contiguous().float()
        b = None if self.bias is None else self.bias.detach().contiguous().float()
        d = _lib.ConvDesc()
        d.images, d.out_channels, d.K, d.positions = n, oc, K, L
        d.w_bit, d.eq_n = int(self.w_bit), int(self.eq_n)
        d.eq_alpha, d.eq_beta = float(self.eq_alpha), float(self.eq_beta)
        d.has_bias = 0 if b is None else 1
        d.kernel = _lib.default_kernel()
        d.layerwise = 1 if self.layerwise else 0
        lib = _lib.lib()
        nbytes = ctypes.c_size_t()
        _lib.check(lib.p4v_conv_workspace_bytes(ctypes.byref(d), ctypes.byref(nbytes)), "p4v_conv_workspace_bytes")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        w_int = torch.empty(nw, dtype=torch.float32, device=dev)
        log = torch.empty(self.eq_n * nw, dtype=torch.float32, device=dev) if self.keep_scores else None
        _lib.check(lib.p4v_conv_calibrate(ctypes.byref(d), _lib.ptr(cols), _lib.ptr(w2), _lib.ptr(b), _lib.ptr(y.view(n, oc, L)),
                                          _lib.ptr(g.view(n, oc, L)), _lib.ptr(ws), nbytes.value, _lib.ptr(w_int), _lib.ptr(log),
                                          ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "p4v_conv_calibrate")
        self.w_interval = w_int.view(nw, 1, 1, 1)
        # conv.py:312-320, :490-496: max over the calibration batches of max|x| / (a_qmax - 0.5) (unused when a_bit >= 32)
        self.a_interval = (x.abs().max() / (self.a_qmax - 0.5)).detach().view(1)
        self.last_scores = [log.view(self.eq_n, nw)] * int(self.search_round) if log is not None else None
        self.calibrated = True
        del self.raw_input, self.raw_out, self.raw_grad

    def calibration_step2(self):
        """The weight search does not depend on anything the rounds change when the activations are not quantized, so
        its result is the same in every round: it is run once."""
        self._check_supported()
        self._native_weight_search()
        return None


class BatchingEasyQuantConv2d(_BatchingConvSearch):
    """reference: quant_layers/conv.py:279-441 (layer-wise EasyQuant).  `a_bit >= 32` turns the activation quantizer off
    (the only way BasePTQ uses this class); ONE weight step size for the whole kernel, searched over
    fl(f_c * max|W| / (w_qmax - 0.5)) (:313, :432) by the first maximum of
    -sum_images mean_positions mean_channels (g * (y - yhat_c))^2 (:387-396).  w_interval has shape [1,1,1,1].
    quant_weight_bias / quant_forward are MinMaxQuantConv2d's (a scalar step size broadcasts)."""
    layerwise = True

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.n_V = 1
        self.n_H = 1


class ChannelwiseBatchingQuantConv2d(_BatchingConvSearch):
    """reference: quant_layers/conv.py:444-613.  `a_bit >= 32` turns the activation quantizer off (the only way
    PTQ4ViT uses this class); the weight step size is searched per output channel."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.n_V = self.out_channels
        self.n_H = 1
