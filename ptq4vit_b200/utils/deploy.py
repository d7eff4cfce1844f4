"""After calibration: freeze a wrapped model's Linear layers into packed integer weights (and, on request, its MatMul
modules into packed step sizes and its patch-embedding convolution into packed integer weights), save the quantised
model and load it back.  What the reference does right after calibrating (example/test_all.py:31-36 evaluates with quant_forward,
example/get_int.py exports the integer weights) as one deployable state.

File format (`torch.save`): {"format": 1, "modules": {name: entry}} with, per wrapped module, its step sizes
(`w_interval`, `a_interval`, `A_interval`, `B_interval`, `split` -- whichever it has, stored as they are) and, for Linear
layers and conv modules on a CUDA device, `w_int`: the int8 weight as `utils.integer.quantize_int_weight` exports it
(through the same export quantiser at any w_bit; conv: [out, in, kh, kw]), and `w_bit`.  At W8 the `w_int` entries alone
are what the reference's get_model_int_weight returns.

Loading freezes every Linear from the integers in the file: the pack kernel is fed with `w_int * step_W` (the block's
step size) and quantises it again.  That returns the same integers exactly: fl(q * s) = q s (1 + e) with |e| <= 2^-24,
and the IEEE quotient by s is within |q| * 2^-23 <= 2^-16 of q, far from a rounding tie, so rne gives q.  No FP32
weight of the module is read, and the frozen forward reads none either.  The argument holds per step size, so it holds
for the per-channel step sizes of a conv module as well.

With `matmul=True` the MatMul modules are frozen as well: their step sizes and scale tables are packed once and every
call runs one fused kernel that quantises both activation operands in shared memory (csrc/forward_mm_tc.cu), with the
same bits.  A model frozen that way runs its whole quantised forward without host work between kernels, so it can be
captured in one CUDA graph.  The default leaves the MatMul modules as they are.

With `conv=True` the patch-embedding convolution is frozen too (a_bit >= 32, kernel == stride, no padding, dilation 1,
groups 1: every model here): its integers are packed once as bf16 and each call runs one kernel that gathers the patches
from the image and multiplies the exact three-term bf16 split of the FP32 pixels with them (csrc/forward_conv_tc.cu).
Unlike the other frozen modules it is not bit-identical to the unfrozen quant_forward, which is cuDNN's F.conv2d (and,
under torch's default allow_tf32, rounds its operands to TF32): its contract is a bound against fp64 (DESIGN.md section
4.9).  Loading with `conv=True` freezes the conv from the file's integers; the default leaves it as it is.

`fuse_attention(net)` goes one step further for attention blocks whose two MatMul modules are frozen: the whole core
between the qkv and proj Linears -- matmul1, the scale, bias and mask, the softmax, matmul2 and the transpose to
[B, N, C] -- runs as one kernel (csrc/forward_attn_tc.cu) with the bits of the unfused sequence, and the score matrix
never reaches HBM.  It is opt-in; `unfuse_attention(net)` undoes it.  `fuse_attention(net, max_tokens=1024)` also fuses
the ViT / DeiT attention calls of 257 to 1024 tokens (384-pixel models: 577), with a kernel that quantises the keys and
values of a head once and recomputes the scores instead of storing them (csrc/forward_attn_long_tc.cu).

`fuse_mlp(net)` does the same for the MLP blocks whose fc1 and fc2 are frozen: fc1's kernel applies the GELU and fc2's
activation quantiser in its epilogue and writes fc2's int8 activation image, which fc2's sweep forward reads -- two
launches instead of four, bit-identical, and the FP32 hidden activations never reach HBM.  Opt-in as well;
`unfuse_mlp(net)` undoes it.

`fuse_norm(net)` folds a LayerNorm into the frozen Linear that consumes it (a pre-norm block's norm1 -> attn.qkv and
norm2 -> mlp.fc1, Swin's norm2 -> fc1, PatchMerging's norm -> reduction, a ViT's final norm -> head, of which only the cls
rows are normalised): torch's exact LayerNorm runs in the Linear's activation quantiser, one launch instead of two and
no normalised tensor in HBM, bit-identical.  It composes with fuse_attention and fuse_mlp (norm2, fc1, GELU and fc2's
quantiser in one kernel).  A folded call skips the LayerNorm's forward hooks, so it is opt-in; `unfuse_norm(net)` undoes
it.

`fuse_residual(net)` folds each block's residual adds into the frozen Linear whose output they add: `x + attn(...)`
into attn.proj (in a Swin block also the window reverse and the reverse roll before the add, through a window layout of
proj's output rows) and `x + mlp(...)` into mlp.fc2, fused MLP included.  The Linear's store adds the shortcut, so its
FP32 output never reaches HBM and the torch add (reverse, roll) kernels are gone, bit-identical.  It composes with the
other fusions.  A folded call skips proj's and fc2's forward hooks, so it is opt-in; `unfuse_residual(net)` undoes it.

`fuse_gather(net)` folds the row gathers in front of Swin's LayerNorm folds: a Swin block's norm1, roll(-shift) and
window partition into attn.qkv, and PatchMerging's cat of the 2x2 neighbourhoods (and its norm) into reduction.  The
Linear's fused kernel reads each row from the block's input image, normalises it with torch's exact LayerNorm and
quantises it, so the normalised, rolled, partitioned or concatenated copies never reach HBM, bit-identical.  It composes
with the other fusions.  A folded call skips the LayerNorm's forward hooks, so it is opt-in; `unfuse_gather(net)` undoes
it.
`fuse_stem(net)` folds the model's stem after a frozen patch-embedding conv into the conv kernel's store: ViT / DeiT's
flatten, transpose, cat with the cls token and pos_embed add, Swin's flatten, transpose and patch_norm.  The kernel
stores the token rows the first block reads, bit-identical to the frozen conv followed by torch's ops, so the NCHW output
and its copies never reach HBM.  It composes with the other fusions.  A folded call skips the conv's and patch_norm's
forward hooks, so it is opt-in; `unfuse_stem(net)` undoes it.
`fuse_qkv(net)` folds the attention operands' quantisation into the frozen qkv of every attention block whose qkv,
matmul1 and matmul2 are frozen and which runs fused (fuse_attention): qkv's kernel quantises its output with matmul1's and
matmul2's step sizes and writes int8 q, k and v, which the short attention kernel reads instead of quantising the FP32
qkv output, bit-identical.  Calls above 256 tokens keep the FP32 hand-off.  It composes with the other fusions (norm1 and
Swin's gather into qkv, the residual into proj).  A folded call skips qkv's forward hooks, so it is opt-in;
`unfuse_qkv(net)` undoes it.
None of the fusions is recorded by save_quantized: apply them again after load_quantized.
"""
import torch

from ..quant_layers.conv import MinMaxQuantConv2d, frozen_stem_ok
from ..quant_layers.linear import MinMaxQuantLinear, frozen_gather_ok
from ..quant_layers.matmul import LONG_ATTENTION_TOKENS, SHORT_ATTENTION_TOKENS, MinMaxQuantMatMul
from . import integer
from .models import Attention, Block, Mlp, PatchMerging, SwinBlock, SwinTransformer, VisionTransformer, WindowAttention

INTERVALS = ("w_interval", "a_interval", "A_interval", "B_interval", "split")


def _freezes(m, matmul, conv=False):
    if isinstance(m, MinMaxQuantConv2d):
        return conv and m.weight.device.type == "cuda" and m.frozen_unsupported() is None
    return isinstance(m, MinMaxQuantLinear) or (matmul and isinstance(m, MinMaxQuantMatMul))


def freeze_model(wrapped_modules, matmul=False, conv=False):
    """Freeze every calibrated Linear, with matmul=True every calibrated MatMul and with conv=True every calibrated conv
    module the frozen convolution implements (MinMaxQuantConv2d.frozen_unsupported() is None, on a CUDA device); returns
    the names of the modules left as they are.  By default (matmul=False, conv=False) the MatMul and conv modules keep
    their quant_forward and are among the names returned, as before they could be frozen."""
    left = []
    for name, m in wrapped_modules.items():
        if getattr(m, "calibrated", None) and _freezes(m, matmul, conv):
            m.freeze()
        else:
            left.append(name)
    return left


def unfreeze_model(wrapped_modules):
    for m in wrapped_modules.values():
        if isinstance(m, (MinMaxQuantLinear, MinMaxQuantMatMul, MinMaxQuantConv2d)):
            m.unfreeze()


def fuse_attention(net, max_tokens=SHORT_ATTENTION_TOKENS):
    """Mark every attention module of `net` whose matmul1 and matmul2 are frozen MatMul modules as fused: each call that
    qualifies (no input requiring grad under grad mode, at most 256 tokens, head_dim a multiple of 16 up to 64) runs the
    fused attention core; any other call runs the modules as before.  With max_tokens in (256, 1024], ViT / DeiT
    `Attention` calls of 256 < N <= max_tokens run fused as well, on the long-sequence kernel (the kernel is chosen from N;
    Swin's `WindowAttention` keeps the 256-token rule).  Returns the names of the attention modules left unfused because
    a MatMul module is not frozen."""
    if isinstance(max_tokens, bool) or not isinstance(max_tokens, int) or \
            not SHORT_ATTENTION_TOKENS <= max_tokens <= LONG_ATTENTION_TOKENS:
        raise ValueError(f"fuse_attention: max_tokens must be an int in [{SHORT_ATTENTION_TOKENS}, {LONG_ATTENTION_TOKENS}], "
                         f"got {max_tokens!r}")
    left = []
    for name, m in net.named_modules():
        if isinstance(m, (Attention, WindowAttention)):
            m.fused = all(isinstance(mm, MinMaxQuantMatMul) and mm.frozen for mm in (m.matmul1, m.matmul2))
            if isinstance(m, Attention):
                m.fused_max_tokens = max_tokens
            if not m.fused:
                left.append(name)
    return left


def unfuse_attention(net):
    for m in net.modules():
        if isinstance(m, (Attention, WindowAttention)):
            m.fused = False
        if isinstance(m, Attention):
            m.fused_max_tokens = SHORT_ATTENTION_TOKENS


def fuse_mlp(net):
    """Mark every `Mlp` module of `net` whose fc1 and fc2 are frozen Linear layers as fused: each call that qualifies
    (quant_layers.linear.frozen_mlp_applies: exact GELU, no gradient wanted, a shape the kernel holds) runs fc1, the
    GELU and fc2's activation quantiser as one kernel that writes fc2's int8 activation image, then fc2's sweep forward,
    with the bits of the unfused sequence; the FP32 hidden activations never reach HBM.  A fused call skips the forward
    hooks of fc1, act and fc2, so the fusion is opt-in; any other call runs the modules as before.  Returns the names of
    the Mlp modules left unfused because a Linear is not frozen."""
    left = []
    for name, m in net.named_modules():
        if isinstance(m, Mlp):
            m.fused = all(isinstance(l, MinMaxQuantLinear) and l.frozen for l in (m.fc1, m.fc2))
            if not m.fused:
                left.append(name)
    return left


def unfuse_mlp(net):
    for m in net.modules():
        if isinstance(m, Mlp):
            m.fused = False


def _norm_sites(m):
    """The (flag, LayerNorm, consuming Linear) fold sites of module m"""
    if isinstance(m, Block):
        return [("fold_norm1", m.norm1, m.attn.qkv), ("fold_norm2", m.norm2, m.mlp.fc1)]
    if isinstance(m, SwinBlock):
        return [("fold_norm2", m.norm2, m.mlp.fc1)]
    if isinstance(m, PatchMerging):
        return [("fold_norm", m.norm, m.reduction)]
    if isinstance(m, VisionTransformer):
        return [("fold_norm", m.norm, m.head)]
    return []


def fuse_norm(net):
    """Mark every LayerNorm fold site of `net` whose consumer is a frozen Linear layer: Block.norm1 -> attn.qkv,
    Block.norm2 -> mlp.fc1, SwinBlock.norm2 -> mlp.fc1, PatchMerging.norm -> reduction and VisionTransformer.norm -> head.
    Each call that qualifies (quant_layers.linear.frozen_norm_applies: an affine nn.LayerNorm over in_features, torch's
    vectorised case, no gradient wanted, a shape the fused kernel holds) normalises its input inside the Linear's
    activation quantiser, with the bits of the unfolded call; any other call runs the LayerNorm and the Linear as before.
    A folded call skips the LayerNorm's forward hooks, which is why the fold is opt-in.  It composes with fuse_attention
    and fuse_mlp; save_quantized / load_quantized do not record it.  Returns the names of the LayerNorm modules left
    unfolded (Swin's norm1, final norm and patch_norm always are)."""
    folded = set()
    for m in net.modules():
        for flag, norm, lin in _norm_sites(m):
            on = isinstance(lin, MinMaxQuantLinear) and lin.frozen
            setattr(m, flag, on)
            if on:
                folded.add(id(norm))
    return [name for name, m in net.named_modules() if isinstance(m, torch.nn.LayerNorm) and id(m) not in folded]


def unfuse_norm(net):
    for m in net.modules():
        for flag, _norm, _lin in _norm_sites(m):
            setattr(m, flag, False)


def fuse_residual(net):
    """Mark every `Block` and `SwinBlock` of `net` whose attn.proj and mlp.fc2 are frozen Linear layers: each residual add
    that qualifies (quant_layers.linear.frozen_residual_applies: an FP32 contiguous shortcut of the output's shape, no
    gradient wanted, a window layout only on proj's fused path) is done by the store of the Linear that produces it --
    Swin's window reverse and reverse roll included -- with the bits of the unfolded sequence; any other call runs the
    modules and torch's ops as before.  A folded call skips the forward hooks of proj and fc2, which is why the fold is
    opt-in.  It composes with fuse_attention, fuse_mlp and fuse_norm; save_quantized / load_quantized do not record it.
    Returns the names of the blocks left unfolded."""
    left = []
    for name, m in net.named_modules():
        if isinstance(m, (Block, SwinBlock)):
            m.fold_residual = all(isinstance(l, MinMaxQuantLinear) and l.frozen for l in (m.attn.proj, m.mlp.fc2))
            if not m.fold_residual:
                left.append(name)
    return left


def unfuse_residual(net):
    for m in net.modules():
        if isinstance(m, (Block, SwinBlock)):
            m.fold_residual = False


def _gather_site(m):
    """The (consuming Linear, gather mode) of a row-gather fold site, or None"""
    if isinstance(m, SwinBlock):
        return m.attn.qkv, "window"
    if isinstance(m, PatchMerging):
        return m.reduction, "merge"
    return None


def fuse_gather(net):
    """Mark every row-gather fold site of `net` whose Linear is frozen and takes the gather (quant_layers.linear.
    frozen_gather_ok): a SwinBlock's norm1 -> roll(-shift) -> window partition -> attn.qkv, and a PatchMerging's 2x2 cat
    -> norm -> reduction.  Each call that qualifies (quant_layers.linear.frozen_gather_applies: the conditions of the
    LayerNorm fold, a contiguous input of the image's shape) reads its rows from the block's input inside the Linear's
    activation quantiser, with the bits of the unfolded sequence; any other call runs the modules and torch's ops as
    before (PatchMerging's fold_norm path included).  A folded call skips the LayerNorm's forward hooks, which is why the
    fold is opt-in.  It composes with fuse_attention, fuse_mlp, fuse_norm and fuse_residual; save_quantized /
    load_quantized do not record it.  Returns the names of the sites left unfolded (a reduction on the streamed path, such
    as Swin-T's last one, always is)."""
    left = []
    for name, m in net.named_modules():
        site = _gather_site(m)
        if site is not None:
            lin, mode = site
            m.fold_gather = isinstance(lin, MinMaxQuantLinear) and lin.frozen and frozen_gather_ok(lin, mode)
            if not m.fold_gather:
                left.append(name)
    return left


def unfuse_gather(net):
    for m in net.modules():
        if _gather_site(m) is not None:
            m.fold_gather = False


def _stem_site(m):
    """The (patch-embedding conv, whether the fold normalises) of a model whose stem folds, or None"""
    if isinstance(m, VisionTransformer):
        return m.patch_embed.proj, False
    if isinstance(m, SwinTransformer):
        return m.patch_embed.proj, True
    return None


def fuse_stem(net):
    """Mark every VisionTransformer and SwinTransformer in `net` (net itself included) whose patch_embed.proj is a frozen
    conv module that takes the fold (quant_layers.conv.frozen_stem_ok: out_channels % 4 == 0, Swin also <= 128).  Each
    call that qualifies (quant_layers.conv.frozen_stem_applies: an FP32 contiguous image, FP32 aligned cls_token and
    pos_embed of the expected shapes or patch_norm with the conditions of the LayerNorm folds, no gradient wanted) runs
    the stem as one launch of the conv kernel that stores the token rows -- ViT's cls rows and pos_embed added, Swin's
    rows normalised by patch_norm -- with the bits of the frozen conv followed by torch's ops; any other call runs the
    modules and torch's ops as before.  A folded call skips the forward hooks of the conv, of patch_embed and of
    patch_norm, which is why the fold is opt-in.  It composes with every other fusion; save_quantized / load_quantized do
    not record it.  Returns the names of the models left unfolded ("" for net itself)."""
    left = []
    for name, m in net.named_modules():
        site = _stem_site(m)
        if site is not None:
            conv, norm = site
            m.fold_stem = isinstance(conv, MinMaxQuantConv2d) and conv.frozen and frozen_stem_ok(conv, norm)
            if not m.fold_stem:
                left.append(name)
    return left


def unfuse_stem(net):
    for m in net.modules():
        if _stem_site(m) is not None:
            m.fold_stem = False


def fuse_qkv(net):
    """Mark every `Attention` and `WindowAttention` of `net` whose qkv is a frozen Linear layer and whose matmul1 and
    matmul2 are frozen MatMul modules: each call that also runs fused (fuse_attention) and qualifies
    (quant_layers.matmul.frozen_qkv_applies: the short attention kernel, no gradient wanted, the conditions of the norm1
    or gather fold it carries, a shape the fused kernel holds) has qkv's kernel quantise q, k and v with the attention's
    step sizes and write them as int8 planes, which the attention kernel reads -- with the bits of the unfolded call, and
    qkv's FP32 output never reaches HBM; any other call runs the modules as before.  A folded call skips qkv's forward
    hooks, which is why the fold is opt-in.  It composes with every other fusion; save_quantized / load_quantized do not
    record it.  Returns the names of the attention modules left unfolded."""
    left = []
    for name, m in net.named_modules():
        if isinstance(m, (Attention, WindowAttention)):
            m.fold_qkv = isinstance(m.qkv, MinMaxQuantLinear) and m.qkv.frozen and \
                all(isinstance(mm, MinMaxQuantMatMul) and mm.frozen for mm in (m.matmul1, m.matmul2))
            if not m.fold_qkv:
                left.append(name)
    return left


def unfuse_qkv(net):
    for m in net.modules():
        if isinstance(m, (Attention, WindowAttention)):
            m.fold_qkv = False


def _to(v, device):
    """A step size as stored / restored: tensors cloned onto `device`, lists element-wise, Python numbers as they are."""
    if torch.is_tensor(v):
        return v.detach().to(device).clone()
    if isinstance(v, (list, tuple)):
        return [_to(e, device) for e in v]
    return v


def save_quantized(wrapped_modules, path):
    modules = {}
    for name, m in wrapped_modules.items():
        entry = {k: _to(getattr(m, k), "cpu") for k in INTERVALS if getattr(m, k, None) is not None}
        if isinstance(m, MinMaxQuantLinear) and getattr(m, "calibrated", None) and m.weight.device.type == "cuda":
            O, K = m.out_features, m.in_features
            entry["w_int"] = integer._export(m.weight.detach().reshape(O, K), m.w_interval, O // m.n_V, m.n_V, K // m.n_H,
                                             m.n_H, integer.MODE_INT8, m.w_bit).cpu()
            entry["w_bit"] = int(m.w_bit)
        elif isinstance(m, MinMaxQuantConv2d) and getattr(m, "calibrated", None) and m.weight.device.type == "cuda":
            O = m.out_channels
            n_d = torch.as_tensor(m.w_interval).numel()          # one step size per output channel, or one
            entry["w_int"] = integer._export(m.weight.detach().reshape(O, -1), m.w_interval, O // n_d, n_d, m.weight[0].numel(),
                                             1, integer.MODE_INT8, m.w_bit).view(m.weight.shape).cpu()
            entry["w_bit"] = int(m.w_bit)
        modules[name] = entry
    torch.save({"format": 1, "modules": modules}, path)


def load_quantized(wrapped_modules, path, matmul=False, conv=False):
    """Restore the step sizes of every module in the file, mark the modules calibrated and freeze the Linear layers from
    the file's int8 weights (with matmul=True also the MatMul modules from their step sizes, with conv=True also the conv
    modules from their int8 weights; a conv entry without them stays unfrozen).  Returns the names of the modules that
    were not frozen."""
    state = torch.load(path, map_location="cpu", weights_only=True)
    if state.get("format") != 1:
        raise RuntimeError(f"{path}: not a ptq4vit_b200 quantised-model file")
    missing = sorted(set(state["modules"]) ^ set(wrapped_modules))
    if missing:
        raise RuntimeError(f"{path}: modules differ from the wrapped model: {missing[:8]}")
    params = [p for m in wrapped_modules.values() for p in m.parameters()]
    device = params[0].device if params else torch.device("cpu")      # MatMul modules have no parameters of their own
    left = []
    for name, m in wrapped_modules.items():
        entry = state["modules"][name]
        for k in INTERVALS:
            if k in entry:
                setattr(m, k, _to(entry[k], device))
        m.calibrated = True
        int_weights = isinstance(m, MinMaxQuantLinear) or \
            (conv and isinstance(m, MinMaxQuantConv2d) and m.frozen_unsupported() is None)
        if int_weights and "w_int" in entry and m.weight.device.type == "cuda":
            if entry["w_bit"] != m.w_bit:
                raise RuntimeError(f"{path}: {name} was saved with w_bit {entry['w_bit']}, the module has {m.w_bit}")
            m.freeze(weight=integer.dequantize_int_weight(m, entry["w_int"].to(device)))
        elif matmul and isinstance(m, MinMaxQuantMatMul) and device.type == "cuda":
            m.freeze()
        else:
            left.append(name)
    return left
