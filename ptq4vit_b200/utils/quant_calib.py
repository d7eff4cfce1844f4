"""Calibration drivers with the reference's surface (utils/quant_calib.py:9-378).

`HessianQuantCalibrator(net, wrapped_modules, calib_loader, sequential=False, batch_size=1)
.batching_quant_calib()` is the entry point the reference's experiments time
(example/test_all.py:31-34).  GPU-first changes, results unchanged:

* capture: with sequential=False every module stays in "raw" mode while the others calibrate
  (quant_calib.py:369-372), so the captured (input, output, grad) tensors do not depend on the
  order -- ONE forward+backward sweep over the calibration images with hooks on all modules
  replaces the reference's one-sweep-per-module loop (quant_calib.py:317-356), and the tensors
  stay in HBM instead of bouncing through host memory (quant_calib.py:173-201).  With
  capture="auto" the captures of this rank are estimated from the shapes seen in the first batch of
  the target pass: when they cannot fit in free device memory (or `capture_budget` bytes) next to the
  largest of the smallest search workspaces, or with `capture="per_module"` or sequential=True, the
  reference's loop is used.
* search: `module.calibration_step2()` runs the CUDA search.
* multi-GPU: modules are independent => static LPT sharding over ranks, every rank captures,
  searches its share, and one all_gather of the chosen step sizes ends the job.
"""
import ctypes
import time

import torch
import torch.nn.functional as F

from .. import _lib
from ..quant_layers._chunking import device_free_bytes
from ..quant_layers.conv import BatchingEasyQuantConv2d, MinMaxQuantConv2d
from ..quant_layers.linear import MinMaxQuantLinear, PTQSLBatchingQuantLinear, PTQSLQuantLinear
from ..quant_layers.matmul import MinMaxQuantMatMul, PTQSLBatchingQuantMatMul, PTQSLQuantMatMul


# ---------------------------------------------------------------- hooks (device resident)
def _keep_grad(module, output):
    """The gradient of the loss w.r.t. the module output (what the reference's `register_backward_hook(grad_hook)`
    receives as grad_output[0], quant_calib.py:173-176, :330), taken with a tensor hook: it fires whenever a
    gradient reaches the output, independent of which inputs require grad."""
    if not (torch.is_grad_enabled() and output.requires_grad):
        return

    def _hook(grad):
        if module.raw_grad is None:
            module.raw_grad = []
        module.raw_grad.append(grad.detach())
    output.register_hook(_hook)


def grad_hook(module, grad_input, grad_output):
    """reference: quant_calib.py:173-176 (kept for API parity; the calibrators below use tensor hooks)."""
    if module.raw_grad is None:
        module.raw_grad = []
    module.raw_grad.append(grad_output[0].detach())


def linear_forward_hook(module, input, output):
    """reference: quant_calib.py:178-183 (tensors stay on the device)."""
    if module.raw_input is None:
        module.raw_input = []
    if module.raw_out is None:
        module.raw_out = []
    module.raw_input.append(input[0].detach())
    module.raw_out.append(output.detach())


conv2d_forward_hook = linear_forward_hook          # reference: quant_calib.py:185-190


def matmul_forward_hook(module, input, output):
    """reference: quant_calib.py:192-199"""
    if module.raw_input is None:
        module.raw_input = [[], []]
    if module.raw_out is None:
        module.raw_out = []
    module.raw_input[0].append(input[0].detach())
    module.raw_input[1].append(input[1].detach())
    module.raw_out.append(output.detach())


def _cat_captured(module):
    if isinstance(module, (MinMaxQuantLinear, MinMaxQuantConv2d)):
        module.raw_input = torch.cat(module.raw_input, dim=0)
        module.raw_out = torch.cat(module.raw_out, dim=0)
    if isinstance(module, MinMaxQuantMatMul):
        module.raw_input = [torch.cat(_, dim=0) for _ in module.raw_input]
        module.raw_out = torch.cat(module.raw_out, dim=0)
    if getattr(module, "raw_grad", None) is not None and isinstance(module.raw_grad, list):
        module.raw_grad = torch.cat(module.raw_grad, dim=0)


# ---------------------------------------------------------------- work model + sharding
# Measured on an H100 80GB HBM3 at a 400 W power limit (ViT-B/224 x 32 images, W8A8, one search round): qkv 20.9 ms,
# proj 10.3 ms, fc1 27.1 ms, head 3.1 ms, matmul1 7.7 ms.  A fixed part per module and round (operand images, per-step
# launches) plus executed work at the rate each kernel family sustains.  The conv rate is not measured on the H100; it only
# places the single patch-embedding module.
_ROUND_OVERHEAD_S = 4.7e-3
_LINEAR_RATE = 2.66e14     # "units" below per second: eq_n * 2*M*K*O * (1 + n_a)
_MATMUL_RATE = 1.29e14     # 2 * eq_n * 2*b*H*S1*S2*S3 per second (197-token tiles are 59 % full)
_CONV_RATE = 1.5e13        # eq_n * 2 * MACs per second (three bf16 term products per MAC)


def module_cost(module, n_img, shapes=None, tokens_hint=197):
    """Estimated seconds of one module's search on an H100 (only ratios matter for the sharding).
    Linear  : rounds * (overhead + eq_n * 2*M*K*O * (1 [all weight steps together multiply each K slab once] + n_a) / rate)
    MatMul  : rounds * (overhead + 2 * eq_n * 2*b*H*S1*S2*S3 / rate)
    `shapes` = per-image input shapes recorded by a probe forward ({"x": (lead, tokens.., K)} / {"A": (lead, H, S1, S2), ...});
    `lead` folds windows into the batch (Swin)."""
    rounds = getattr(module, "search_round", 1)
    eq_n = getattr(module, "eq_n", 1)
    if isinstance(module, MinMaxQuantLinear):
        rows = tokens_hint
        if shapes is not None and "x" in shapes:
            rows = 1
            for s in shapes["x"][:-1]:
                rows *= int(s)
        gemm = 2.0 * n_img * rows * module.in_features * module.out_features
        return rounds * (_ROUND_OVERHEAD_S + eq_n * gemm * (1.0 + getattr(module, "n_a", 1)) / _LINEAR_RATE)
    if isinstance(module, MinMaxQuantConv2d):
        macs = 0.0 if shapes is None else shapes.get("conv_macs", 0.0)
        return _ROUND_OVERHEAD_S + eq_n * 2.0 * n_img * macs / _CONV_RATE          # searched once (see quant_layers/conv.py)
    if isinstance(module, MinMaxQuantMatMul):
        if shapes is not None and "A" in shapes:
            H, S1, S2 = [int(s) for s in shapes["A"][-3:]]
            S3 = int(shapes["B"][-1])
            lead = 1
            for s in shapes["A"][:-3]:
                lead *= int(s)
        else:
            lead, H, S1, S2, S3 = 1, 12, tokens_hint, 64, tokens_hint
        return rounds * (_ROUND_OVERHEAD_S + 2 * eq_n * 2.0 * n_img * lead * H * S1 * S2 * S3 / _MATMUL_RATE)
    return 0.0


def _prod(shape):
    n = 1
    for s in shape:
        n *= int(s)
    return n


def capture_bytes(module, n_img, shapes):
    """Bytes of the tensors the single-pass capture keeps for one module until its search: fp32 input(s), output and
    output gradient, from the per-image shapes seen in the target pass (see HessianQuantCalibrator._record_shapes)."""
    if shapes is None:
        return 0
    if "x" in shapes:
        rows = n_img * _prod(shapes["x"][:-1])
        return 4 * rows * (int(shapes["x"][-1]) + 2 * module.out_features)
    if "A" in shapes:
        lead, H, S1, S2 = _prod(shapes["A"][:-3]), *[int(s) for s in shapes["A"][-3:]]
        S3 = int(shapes["B"][-1])
        return 4 * n_img * lead * H * (S1 * S2 + S2 * S3 + 2 * S1 * S3)
    return 4 * n_img * (shapes.get("x_elems", 0) + 2 * shapes.get("y_elems", 0))


def min_search_workspace_bytes(module, n_img, shapes):
    """Device memory the module's search needs at least: its workspace split into the smallest chunks the library takes
    (128 rows of a Linear, one image of a MatMul); the conv search (not chunked) with its im2col matrix; 0 for modules
    without a native search."""
    if shapes is None:
        return 0
    lib = _lib.lib()
    n = ctypes.c_size_t()
    eq = (module.eq_alpha, module.eq_beta, module.eq_n) if hasattr(module, "eq_n") else None
    if isinstance(module, PTQSLQuantLinear) and "x" in shapes:
        rows = n_img * _prod(shapes["x"][:-1])
        d = module._desc(rows, _prod(shapes["x"][1:-1]), module.search_round, eq)
        d.rows_per_chunk = 128 if rows > 128 else 0
        _lib.check(lib.p4v_linear_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "p4v_linear_workspace_bytes")
        return n.value
    if isinstance(module, PTQSLQuantMatMul) and "A" in shapes:
        batch = n_img * _prod(shapes["A"][:-3])
        A = torch.empty((batch,) + tuple(shapes["A"][-3:]), device="meta")
        B = torch.empty((batch,) + tuple(shapes["B"][-3:]), device="meta")
        d = module._desc(A, B, module.search_round, eq)
        d.images_per_chunk = 1
        _lib.check(lib.p4v_matmul_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "p4v_matmul_workspace_bytes")
        return n.value
    if isinstance(module, MinMaxQuantConv2d) and hasattr(module, "eq_n") and "positions" in shapes:
        d = _lib.ConvDesc()
        d.images, d.out_channels, d.K, d.positions = n_img, module.out_channels, shapes["conv_K"], shapes["positions"]
        d.w_bit, d.eq_n, d.eq_alpha, d.eq_beta = int(module.w_bit), int(module.eq_n), float(module.eq_alpha), float(module.eq_beta)
        d.has_bias = 0 if module.bias is None else 1
        d.layerwise = 1 if isinstance(module, BatchingEasyQuantConv2d) else 0
        _lib.check(lib.p4v_conv_workspace_bytes(ctypes.byref(d), ctypes.byref(n)), "p4v_conv_workspace_bytes")
        return n.value + 4 * n_img * shapes["positions"] * shapes["conv_K"]
    return 0


def shard_modules(names, costs, world_size):
    """Static longest-processing-time assignment: returns owner[name] = rank.  Deterministic."""
    order = sorted(range(len(names)), key=lambda i: (-costs[i], i))
    load = [0.0] * world_size
    owner = {}
    for i in order:
        r = min(range(world_size), key=lambda k: (load[k], k))
        owner[names[i]] = r
        load[r] += costs[i]
    return owner


def _flat_results(module):
    if isinstance(module, (MinMaxQuantLinear, MinMaxQuantConv2d)):
        vals = [module.w_interval]
        if module.a_interval is not None:
            vals.append(module.a_interval)
    else:
        vals = [module.A_interval, module.B_interval]
        if getattr(module, "sos", False):
            vals.append(module.split)
    dev = None
    for v in vals:
        if torch.is_tensor(v) and v.device.type == "cuda":
            dev = v.device
    return [torch.as_tensor(v, dtype=torch.float32, device=dev).reshape(-1) for v in vals]


def pack_result(module, width):
    """Flatten a calibrated module's step sizes into a fixed-width fp32 row for the all_gather."""
    flat = torch.cat(_flat_results(module))
    assert flat.numel() <= width, f"result of {type(module).__name__} does not fit the gather row ({flat.numel()} > {width})"
    row = torch.zeros(width, dtype=torch.float32, device=flat.device)
    row[:flat.numel()] = flat
    return row


def _conv_weight_steps(module):
    """Weight step sizes of a searched conv: one (layer-wise EasyQuant) or one per output channel."""
    return 1 if isinstance(module, BatchingEasyQuantConv2d) else module.out_channels


def unpack_result(module, row, heads=None):
    """Inverse of pack_result (the module's static block structure gives the split points)."""
    if isinstance(module, MinMaxQuantConv2d):
        nw = _conv_weight_steps(module)
        module.w_interval = row[:nw].clone().view(nw, 1, 1, 1)
        module.a_interval = row[nw:nw + 1].clone()
    elif isinstance(module, MinMaxQuantLinear):
        nw = module.n_V * module.n_H
        module.w_interval = row[:nw].clone().view(module.n_V, 1, module.n_H, 1)
        module.a_interval = row[nw:nw + module.n_a].clone().view(module.n_a, 1)
    else:
        H = heads if heads is not None else module.n_G_B
        if getattr(module, "sos", False):
            module.A_interval = row[0].clone()
            module.B_interval = row[1:1 + H].clone().view(1, H, 1, 1, 1, 1, 1)
            module.split = row[1 + H].clone()
        else:
            module.A_interval = row[:H].clone().view(1, H, 1, 1, 1, 1, 1)
            module.B_interval = row[H:2 * H].clone().view(1, H, 1, 1, 1, 1, 1)
        module.n_G_A = module.n_G_B = H
    module.calibrated = True


def result_width(modules):
    w = 1
    for m in modules:
        if isinstance(m, MinMaxQuantConv2d):
            w = max(w, _conv_weight_steps(m) + 1)      # weight step sizes + the (unused) activation step size
        elif isinstance(m, MinMaxQuantLinear):
            w = max(w, m.n_V * m.n_H + m.n_a)
        else:
            w = max(w, 2 * 64 + 1)        # up to 64 heads + split
    return w


# ---------------------------------------------------------------- host-resident captures
def search_from_host(items, device, out_host=None):
    """Search a list of modules whose captured tensors live in (pinned) HOST memory, as the reference's calibrators
    keep them (`.cpu()` in its hooks, `.cuda()` per module before the search; quant_calib.py:173-201, :317-356).

    items: [(module, {"x"|"A","B", "y", "g": pinned cpu tensors})].  The host->device copies of module i+1 run on a
    side stream while module i searches; the chosen step sizes are copied back asynchronously into pinned buffers and
    one synchronisation ends the call.  Returns (h2d_bytes, d2h_bytes)."""
    copy_stream = torch.cuda.Stream(device=device)
    main = torch.cuda.current_stream(device)
    h2d = d2h = 0

    def stage(i):
        with torch.cuda.stream(copy_stream):
            dev = {k: v.to(device, non_blocking=True) for k, v in items[i][1].items()}
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return dev, ev

    results = []
    nxt = stage(0) if items else None
    for i, (m, hb) in enumerate(items):
        dev, ev = nxt
        nxt = stage(i + 1) if i + 1 < len(items) else None
        main.wait_event(ev)
        for v in dev.values():
            v.record_stream(main)
        h2d += sum(v.numel() * v.element_size() for v in dev.values())
        if "x" in dev:
            m.raw_input, m.raw_out, m.raw_grad = dev["x"], dev["y"], dev["g"]
        else:
            m.raw_input, m.raw_out, m.raw_grad = [dev["A"], dev["B"]], dev["y"], dev["g"]
        with torch.no_grad():
            m.calibration_step2()
        m.raw_input = m.raw_out = m.raw_grad = None
        for j, o in enumerate(_flat_results(m)):
            buf = torch.empty(o.numel(), dtype=torch.float32, pin_memory=True) if out_host is None else out_host[i][j]
            buf.copy_(o.detach(), non_blocking=True)
            results.append(buf)
            d2h += o.numel() * 4
    main.synchronize()
    return h2d, d2h


# ---------------------------------------------------------------- calibrators
class QuantCalibrator():
    """reference: utils/quant_calib.py:9-171"""

    def __init__(self, net, wrapped_modules, calib_loader, sequential=True):
        self.net = net
        self.wrapped_modules = wrapped_modules
        self.calib_loader = calib_loader
        self.sequential = sequential
        self.calibrated = False
        self.batch_size = getattr(calib_loader, "batch_size", None) or 1   # the reference forgets this attribute (quant_calib.py:131)

    def _device(self):
        return next(self.net.parameters()).device

    def _loader_batches(self):
        for item in self.calib_loader:
            inp = item[0] if isinstance(item, (tuple, list)) else item
            yield inp

    def _run_net_no_grad(self):
        dev = self._device()
        with torch.no_grad():
            for inp in self._loader_batches():
                self.net(inp.to(dev))

    def sequential_quant_calib(self):
        """reference: quant_calib.py:28-55 -- two sweeps over the calibration data; in the second one every module
        searches its step sizes on the (already quantized) activations that reach it and forwards its quantized output."""
        n_calibration_steps = 2
        for step in range(n_calibration_steps):
            for name, module in self.wrapped_modules.items():
                if hasattr(module, "calibrated"):
                    if step == 1:
                        module.mode = "raw"
                    elif step == 2:        # unreachable, as in the reference (:39-42)
                        module.mode = "quant_forward"
                else:
                    module.mode = f"calibration_step{step + 1}"
            self._run_net_no_grad()
        for name, module in self.wrapped_modules.items():
            module.mode = "quant_forward"
        torch.cuda.empty_cache()

    def parallel_quant_calib(self):
        """reference: quant_calib.py:57-93 -- step 1 collects every module's raw input/output in one sweep,
        step 2 searches each module on its own FP32 tensors."""
        for name, module in self.wrapped_modules.items():
            module.mode = "raw" if hasattr(module, "calibrated") else "calibration_step1"
        self._run_net_no_grad()
        dev = self._device()
        for name, module in self.wrapped_modules.items():
            if hasattr(module, "calibrated"):
                continue
            module.mode = "calibration_step2"
            with torch.no_grad():
                if isinstance(module, (MinMaxQuantLinear, MinMaxQuantConv2d)):
                    module.forward(module.raw_input.to(dev))
                elif isinstance(module, MinMaxQuantMatMul):
                    module.forward(module.raw_input[0].to(dev), module.raw_input[1].to(dev))
        for name, module in self.wrapped_modules.items():
            module.mode = "quant_forward"
        torch.cuda.empty_cache()

    def quant_calib(self):
        """reference: quant_calib.py:95-104"""
        if self.sequential:
            self.sequential_quant_calib()
        else:
            self.parallel_quant_calib()
        self.calibrated = True

    # -- shared by the batching drivers
    def _forward_hooks_for(self, module, want_grad):
        hooks = []
        if isinstance(module, MinMaxQuantLinear):
            hooks.append(module.register_forward_hook(linear_forward_hook))
        if isinstance(module, MinMaxQuantConv2d):
            hooks.append(module.register_forward_hook(conv2d_forward_hook))
        if isinstance(module, MinMaxQuantMatMul):
            hooks.append(module.register_forward_hook(matmul_forward_hook))
        if want_grad:
            hooks.append(module.register_forward_hook(lambda mod, inp, out: _keep_grad(mod, out)))
        return hooks

    def _mini_batches(self):
        """(offset of the mini-batch inside the calibration set, images) in the reference's order
        (quant_calib.py:130-134 / :332-335)."""
        off = 0
        for inp in self._loader_batches():
            n = inp.shape[0]
            for batch_st in range(0, n, self.batch_size):
                yield off + batch_st, inp[batch_st:batch_st + self.batch_size]
            off += n

    def batching_quant_calib(self):
        """reference: quant_calib.py:106-171 -- forward-only capture per module, then calibration_step2() on the
        cached tensors (metrics that need no gradient)."""
        dev = self._device()
        for name, module in self.wrapped_modules.items():
            hooks = self._forward_hooks_for(module, want_grad=False)
            with torch.no_grad():
                for _, inp_ in self._mini_batches():
                    self.net(inp_.to(dev))
            _cat_captured(module)
            for hook in hooks:
                hook.remove()
            with torch.no_grad():
                module.calibration_step2()
            module.mode = "quant_forward" if self.sequential else "raw"
        for name, module in self.wrapped_modules.items():
            module.mode = "quant_forward"
        self.calibrated = True


class HessianQuantCalibrator(QuantCalibrator):
    """reference: utils/quant_calib.py:203-378"""

    def __init__(self, net, wrapped_modules, calib_loader, sequential=False, batch_size=1, capture="auto",
                 distributed=None, target_noise=0.0, capture_budget=None):
        super().__init__(net, wrapped_modules, calib_loader, sequential=sequential)
        self.batch_size = batch_size
        self.capture = capture
        self.distributed = distributed
        self.target_noise = target_noise     # synthetic benches: perturb the KL target so that gradients are not ~0
        self.timings = {}
        self.keep_captured = None            # tests: a dict to receive {name: captured tensors} before they are consumed
        self.capture_budget = capture_budget  # capture="auto": bytes for captures + search (None: the free device memory)

    # -- target distribution (quant_calib.py:228-232 / :308-313)
    def _raw_pred_softmax(self, shapes=None):
        """The net's softmax over every calibration image; with a dict `shapes`, also the per-image input shapes of every
        wrapped module (see _record_shapes), taken from the first batch."""
        dev = self._device()
        preds = []
        hooks = self._record_shapes(shapes) if shapes is not None else []
        with torch.no_grad():
            for inp in self._loader_batches():
                self._batch_images = int(inp.shape[0])
                preds.append(F.softmax(self.net(inp.to(dev)), dim=-1).detach())
                for h in hooks:
                    h.remove()
                hooks = []
        raw = torch.cat(preds, dim=0)
        if self.target_noise > 0:
            gen = torch.Generator(device=raw.device).manual_seed(1234)
            logits = raw.clamp_min(1e-30).log()
            logits = logits + self.target_noise * torch.randn(logits.shape, generator=gen, device=logits.device)
            raw = F.softmax(logits, dim=-1)
        return raw

    def _fwd_bwd(self, raw_pred_softmax):
        """quant_calib.py:333-341: KL(self) backward in mini-batches of self.batch_size."""
        dev = self._device()
        for off, inp_ in self._mini_batches():
            self.net.zero_grad()
            inp_ = inp_.to(dev)
            pred = self.net(inp_)
            tgt = raw_pred_softmax[off:off + inp_.shape[0]]
            loss = F.kl_div(F.log_softmax(pred, dim=-1), tgt, reduction="batchmean")
            loss.backward()

    def _hooks_for(self, module, hessian_only=False):
        want = hasattr(module, "metric") and (module.metric == "hessian" or not hessian_only)
        return self._forward_hooks_for(module, want_grad=want)

    # -- layer-wise sharding (only meaningful when sequential=False) and the capture plan
    def _record_shapes(self, shapes):
        """Forward hooks filling `shapes` with the per-image input shapes of every wrapped module, as the first forward
        they see (of self._batch_images images) has them; window attention folds windows into the batch dimension:
        lead = windows per image.  Returns the hooks."""
        def rec(name):
            def f(mod, inp, out):
                if name in shapes:
                    return
                lead = max(1, int(inp[0].shape[0]) // self._batch_images)
                if isinstance(mod, MinMaxQuantMatMul):
                    shapes[name] = {"A": (lead,) + tuple(inp[0].shape[1:]), "B": tuple(inp[1].shape[1:])}
                elif isinstance(mod, MinMaxQuantConv2d):
                    k = mod.kernel_size
                    shapes[name] = {"conv_macs": float(out.shape[1] * out.shape[2] * out.shape[3] * mod.in_channels * k[0] * k[1]),
                                    "x_elems": inp[0][0].numel(), "y_elems": out[0].numel(),
                                    "positions": int(out.shape[2] * out.shape[3]), "conv_K": int(mod.in_channels * k[0] * k[1])}
                else:
                    shapes[name] = {"x": (lead,) + tuple(inp[0].shape[1:])}
            return f
        return [m.register_forward_hook(rec(n)) for n, m in self.wrapped_modules.items()]

    def _probe_shapes(self):
        """Per-image input shapes of every wrapped module from one forward of one image (no grad)."""
        shapes = {}
        hooks = self._record_shapes(shapes)
        first = next(iter(self._loader_batches()))
        self._batch_images = 1
        with torch.no_grad():
            self.net(first[:1].to(self._device()))
        for h in hooks:
            h.remove()
        return shapes

    def _my_modules(self, shapes=None):
        """This rank's modules and the owner of every module (None on one rank).  `shapes`: as _record_shapes fills
        them; probed with one forward when not given."""
        names = list(self.wrapped_modules.keys())
        dist = self.distributed
        if dist is None or not dist.is_initialized() or dist.get_world_size() == 1 or self.sequential:
            return names, None
        n_img = sum(inp.shape[0] for inp in self._loader_batches())
        shapes = shapes if shapes is not None else self._probe_shapes()
        costs = [module_cost(self.wrapped_modules[n], n_img, shapes.get(n)) for n in names]
        owner = shard_modules(names, costs, dist.get_world_size())
        return [n for n in names if owner[n] == dist.get_rank()], owner

    def _capture_plan(self, my_names, shapes):
        """capture="auto": one capture pass for all of this rank's modules when their captured tensors fit in the free
        device memory (or `capture_budget`) next to the largest memory one of their searches needs at least, else the
        per-module loop.  Returns (single_pass, estimated capture bytes, that search memory, budget)."""
        n_img = sum(inp.shape[0] for inp in self._loader_batches())
        mods = [(self.wrapped_modules[n], shapes.get(n)) for n in my_names]
        est = sum(capture_bytes(m, n_img, s) for m, s in mods)
        ws = max([min_search_workspace_bytes(m, n_img, s) for m, s in mods] + [0])
        budget = self.capture_budget if self.capture_budget is not None else device_free_bytes(self._device())
        return est + ws <= budget, est, ws, budget

    def _gather(self, owner):
        dist = self.distributed
        names = list(self.wrapped_modules.keys())
        mods = [self.wrapped_modules[n] for n in names]
        width = result_width(mods) + 1          # last column: head count of MatMul modules (only their owner knows it)
        dev = self._device()
        mine = torch.zeros(len(names), width, dtype=torch.float32, device=dev)
        for i, n in enumerate(names):
            if owner[n] == dist.get_rank():
                mine[i, :width - 1] = pack_result(mods[i], width - 1).to(dev)
                if isinstance(mods[i], MinMaxQuantMatMul):
                    mine[i, width - 1] = float(mods[i].n_G_B)
        gathered = [torch.zeros_like(mine) for _ in range(dist.get_world_size())]
        dist.all_gather(gathered, mine)           # the one collective of the job
        for i, n in enumerate(names):
            r = owner[n]
            if r != dist.get_rank():
                h = int(gathered[r][i, width - 1].item()) if isinstance(mods[i], MinMaxQuantMatMul) else None
                unpack_result(mods[i], gathered[r][i, :width - 1], heads=h)

    def _snapshot(self, name, module):
        if self.keep_captured is None:
            return
        if isinstance(module.raw_input, (list, tuple)):
            d = {"A": module.raw_input[0], "B": module.raw_input[1]}
        else:
            d = {"x": module.raw_input}
        d["y"] = module.raw_out
        d["g"] = module.raw_grad
        self.keep_captured[name] = {k: (v.detach().clone() if v is not None else None) for k, v in d.items()}

    def _clock(self):
        torch.cuda.synchronize(self._device()) if self._device().type == "cuda" else None
        return time.perf_counter()

    def batching_quant_calib(self):
        """reference: quant_calib.py:300-378"""
        t0 = self._clock()
        auto = (not self.sequential) and self.capture == "auto"
        shapes = {}
        raw_pred_softmax = self._raw_pred_softmax(shapes)
        my_names, owner = self._my_modules(shapes)
        plan = {}
        if auto:
            fits, est, ws, budget = self._capture_plan(my_names, shapes)
            single_pass = fits
            plan = {"capture_bytes_est": est, "min_workspace_bytes": ws, "memory_budget_bytes": budget}
        else:
            single_pass = (not self.sequential) and self.capture == "single_pass"
        t_capture = t_search = 0.0
        if single_pass:
            hooks = []
            for name in my_names:
                hooks += self._hooks_for(self.wrapped_modules[name])
            self._fwd_bwd(raw_pred_softmax)
            for h in hooks:
                h.remove()
            self.net.zero_grad(set_to_none=True)
            t1 = self._clock(); t_capture = t1 - t0
            for name in my_names:
                module = self.wrapped_modules[name]
                _cat_captured(module)
                self._snapshot(name, module)
                with torch.no_grad():
                    module.calibration_step2()
                module.mode = "raw"
            t2 = self._clock(); t_search = t2 - t1
        else:
            t_capture = self._clock() - t0
            for name in my_names:
                ta = self._clock()
                module = self.wrapped_modules[name]
                hooks = self._hooks_for(module)
                self._fwd_bwd(raw_pred_softmax)
                _cat_captured(module)
                for h in hooks:
                    h.remove()
                self._snapshot(name, module)
                tb = self._clock(); t_capture += tb - ta
                with torch.no_grad():
                    module.calibration_step2()
                module.mode = "quant_forward" if self.sequential else "raw"
                t_search += self._clock() - tb
            t2 = self._clock()
        if owner is not None:
            self._gather(owner)
        for name, module in self.wrapped_modules.items():
            module.mode = "quant_forward"
        self.calibrated = True
        t3 = self._clock()
        self.timings = {"capture_s": t_capture, "search_s": t_search, "gather_s": t3 - t2, "total_s": t3 - t0,
                        "modules_searched": len(my_names), "single_pass": bool(single_pass),
                        "capture_mode": "single_pass" if single_pass else "per_module", **plan}

    def quant_calib(self):
        """reference: quant_calib.py:216-298 -- the non-batching driver: per module one forward+backward sweep, then
        `calibration_step2(x)` / `(A, B)` with the captured input as argument (the Batching classes take none)."""
        raw_pred_softmax = self._raw_pred_softmax()
        dev = self._device()
        for name, module in self.wrapped_modules.items():
            hooks = self._hooks_for(module, hessian_only=True)
            self._fwd_bwd(raw_pred_softmax)
            _cat_captured(module)
            for h in hooks:
                h.remove()
            self._snapshot(name, module)
            with torch.no_grad():
                if isinstance(module, (PTQSLBatchingQuantLinear, PTQSLBatchingQuantMatMul)) or getattr(module, "batching", False):
                    module.calibration_step2()
                elif isinstance(module, (MinMaxQuantLinear, MinMaxQuantConv2d)):
                    module.calibration_step2(module.raw_input.to(dev))
                elif isinstance(module, MinMaxQuantMatMul):
                    module.calibration_step2(module.raw_input[0].to(dev), module.raw_input[1].to(dev))
            module.mode = "quant_forward" if self.sequential else "raw"
        for name, module in self.wrapped_modules.items():
            module.mode = "quant_forward"
        self.calibrated = True
