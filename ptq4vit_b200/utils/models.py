"""Minimal ViT / DeiT definitions with timm's submodule names (patch_embed.proj, blocks.N.attn.{qkv,proj},
blocks.N.mlp.{fc1,fc2}, head) and the reference's attention rewrite that routes q@k^T and attn@v through
`matmul1` / `matmul2` modules (utils/models.py:10-26, :58-60).  timm and pretrained weights are not
available offline, so weights are synthetic (trunc-normal 0.02) -- this is harness code, not the hot path."""
import torch
import torch.nn as nn

from ..quant_layers.conv import frozen_stem, frozen_stem_applies
from ..quant_layers.linear import (frozen_gather_applies, frozen_gather_linear, frozen_mlp, frozen_mlp_applies,
                                   frozen_mlp_norm_ok, frozen_norm_applies, frozen_norm_linear, frozen_residual_applies,
                                   frozen_residual_linear)
from ..quant_layers.matmul import frozen_attention, frozen_attention_applies, frozen_qkv_applies, frozen_qkv_attention


def _norm_linear(norm, lin, x):
    """lin(norm(x)): folded into one call when frozen_norm_applies holds, else the two modules as they are."""
    if frozen_norm_applies(norm, lin, x):
        return frozen_norm_linear(norm, lin, x)
    return lin(norm(x))


def _linear_res(lin, x, residual):
    """residual + lin(x) (lin(x) without a residual): the add folded into lin's store when frozen_residual_applies holds,
    else the module and torch's add as they are."""
    if residual is None:
        return lin(x)
    if frozen_residual_applies(lin, x, residual):
        return frozen_residual_linear(lin, x, residual)
    return residual + lin(x)


class MatMul(nn.Module):
    def forward(self, A, B):
        return A @ B


class Attention(nn.Module):
    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3)
        self.proj = nn.Linear(dim, dim)
        self.matmul1 = MatMul()
        self.matmul2 = MatMul()

    fused = False      # set by utils.deploy.fuse_attention: run the frozen attention core as one kernel when it applies
    fused_max_tokens = 256   # set by utils.deploy.fuse_attention: sequences up to this length run fused (the long
                             # kernel above 256 tokens)
    fold_qkv = False   # set by utils.deploy.fuse_qkv: with `fused`, qkv writes int8 q, k and v for the short attention
                       # kernel when it applies

    def forward(self, x, norm=None, residual=None):
        """norm: a LayerNorm to apply to x first (Block with fold_norm1), folded into qkv when it applies.  residual: a
        tensor to add to the output (Block with fold_residual), folded into proj when it applies."""
        B, N, C = x.shape
        H, D = self.num_heads, C // self.num_heads
        if self.fold_qkv and self.fused and frozen_qkv_applies(self.qkv, self.matmul1, self.matmul2, x, N, H, D, norm=norm):
            return _linear_res(self.proj, frozen_qkv_attention(self.qkv, self.matmul1, self.matmul2, x, N, H, D, self.scale,
                                                               scale_on_q=False, norm=norm), residual)
        y = self.qkv(x) if norm is None else _norm_linear(norm, self.qkv, x)
        if self.fused and frozen_attention_applies(self.matmul1, self.matmul2, N, C // self.num_heads, y,
                                                   max_tokens=self.fused_max_tokens):
            qkv5 = y.reshape(B, N, 3, self.num_heads, C // self.num_heads)
            return _linear_res(self.proj, frozen_attention(self.matmul1, self.matmul2, qkv5, self.scale, scale_on_q=False,
                                                           max_tokens=self.fused_max_tokens), residual)
        qkv = y.reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        attn = self.matmul1(q, k.transpose(-2, -1)) * self.scale
        attn = attn.softmax(dim=-1)
        x = self.matmul2(attn, v).transpose(1, 2).reshape(B, N, C)
        return _linear_res(self.proj, x, residual)


class Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)

    fused = False      # set by utils.deploy.fuse_mlp: run fc1, GELU and fc2 as the fused frozen MLP when it applies

    def forward(self, x, norm=None, residual=None):
        """norm: a LayerNorm to apply to x first (Block / SwinBlock with fold_norm2), folded into fc1 when it applies.
        residual: a tensor to add to the output (Block / SwinBlock with fold_residual), folded into fc2 when it applies."""
        if norm is not None:
            if frozen_norm_applies(norm, self.fc1, x):
                if not (self.fused and frozen_mlp_applies(self.fc1, self.fc2, self.act, x)):
                    return _linear_res(self.fc2, self.act(frozen_norm_linear(norm, self.fc1, x)), residual)
                if frozen_mlp_norm_ok(self.fc1, self.fc2):
                    return self._fused(x, norm, residual)
            x = norm(x)
        if self.fused and frozen_mlp_applies(self.fc1, self.fc2, self.act, x):
            return self._fused(x, None, residual)
        return _linear_res(self.fc2, self.act(self.fc1(x)), residual)

    def _fused(self, x, norm, residual):
        if residual is None:
            return frozen_mlp(self.fc1, self.fc2, x, norm=norm)
        if frozen_residual_applies(self.fc2, x, residual):
            return frozen_mlp(self.fc1, self.fc2, x, norm=norm, residual=residual)
        return residual + frozen_mlp(self.fc1, self.fc2, x, norm=norm)


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4.0):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = Attention(dim, num_heads)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))

    fold_norm1 = False     # set by utils.deploy.fuse_norm: hand norm1 to attn, which folds it into qkv when it applies
    fold_norm2 = False     # set by utils.deploy.fuse_norm: hand norm2 to mlp, which folds it into fc1 when it applies
    fold_residual = False  # set by utils.deploy.fuse_residual: hand the shortcut to attn and mlp, which fold the adds
                           # into proj and fc2 when they apply

    def forward(self, x):
        if self.fold_residual:
            return self._forward_res(x)
        if not (self.fold_norm1 or self.fold_norm2):
            x = x + self.attn(self.norm1(x))
            return x + self.mlp(self.norm2(x))
        x = x + (self.attn(x, norm=self.norm1) if self.fold_norm1 else self.attn(self.norm1(x)))
        return x + (self.mlp(x, norm=self.norm2) if self.fold_norm2 else self.mlp(self.norm2(x)))

    def _forward_res(self, x):
        x = self.attn(x, norm=self.norm1, residual=x) if self.fold_norm1 else self.attn(self.norm1(x), residual=x)
        return self.mlp(x, norm=self.norm2, residual=x) if self.fold_norm2 else self.mlp(self.norm2(x), residual=x)


class PatchEmbed(nn.Module):
    def __init__(self, img_size, patch, dim):
        super().__init__()
        self.num_patches = (img_size // patch) ** 2
        self.proj = nn.Conv2d(3, dim, kernel_size=patch, stride=patch)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class VisionTransformer(nn.Module):
    def __init__(self, img_size=224, patch=16, dim=768, depth=12, num_heads=12, num_classes=1000, seed=0):
        super().__init__()
        self.patch_embed = PatchEmbed(img_size, patch, dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + 1, dim))
        self.blocks = nn.Sequential(*[Block(dim, num_heads) for _ in range(depth)])
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.head = nn.Linear(dim, num_classes)
        gen = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name_, p_ in self.named_parameters():
                if p_.dim() > 1:
                    p_.copy_(torch.nn.init.trunc_normal_(torch.empty_like(p_), std=0.02, generator=gen))
                elif name_.endswith("bias") and "norm" not in name_:
                    # nn.Linear / nn.Conv2d draw their biases from the global RNG: make the whole net a function of `seed`
                    p_.copy_(torch.empty_like(p_).uniform_(-0.02, 0.02, generator=gen))
            # synthetic nets have no trained structure: widen activations so that the blocks differ
            for blk in self.blocks:
                blk.attn.qkv.weight.mul_(4.0)
                blk.mlp.fc1.weight.mul_(4.0)
            self.head.weight.mul_(8.0)
            self.pos_embed.copy_(torch.nn.init.trunc_normal_(torch.empty_like(self.pos_embed), std=0.02, generator=gen))

    fold_norm = False      # set by utils.deploy.fuse_norm: fold norm into head, normalising only the cls rows
    fold_stem = False      # set by utils.deploy.fuse_stem: the frozen patch-embedding conv stores the token rows, the cls
                           # rows and pos_embed added, when it applies

    def forward(self, x):
        if self.fold_stem and frozen_stem_applies(self.patch_embed.proj, x, cls_token=self.cls_token, pos_embed=self.pos_embed):
            x = frozen_stem(self.patch_embed.proj, x, cls_token=self.cls_token, pos_embed=self.pos_embed)
        else:
            x = self.patch_embed(x)
            x = torch.cat([self.cls_token.expand(x.shape[0], -1, -1), x], dim=1) + self.pos_embed
        x = self.blocks(x)
        # LayerNorm is per row: the cls rows normalised alone have the bits of the whole tensor's cls rows
        if self.fold_norm and frozen_norm_applies(self.norm, self.head, x):
            return frozen_norm_linear(self.norm, self.head, x[:, 0])
        x = self.norm(x)
        return self.head(x[:, 0])


# ---------------------------------------------------------------- Swin (timm names: layers.N.blocks.M.attn / .mlp, layers.N.downsample.reduction)
def _window_partition(x, ws):
    B, H, W, C = x.shape
    x = x.view(B, H // ws, ws, W // ws, ws, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, ws * ws, C)


def _window_reverse(win, ws, H, W):
    B = win.shape[0] // ((H // ws) * (W // ws))
    x = win.view(B, H // ws, W // ws, ws, ws, -1)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, H, W, -1)


def _window_qkv(norm, qkv, x, layout):
    """qkv(window_partition(roll(norm(x), (-shift, -shift)))) of a Swin block input x [images, height * width, C] with
    layout = (images, height, width, window, shift): one folded call when frozen_gather_applies holds (the LayerNorm, the
    roll and the partition in qkv's activation quantiser), else the modules and torch's ops as they are."""
    images, H, W, ws, shift = layout
    gather = ("window", images, H, W, ws, shift)
    if frozen_gather_applies(norm, qkv, x, gather):
        return frozen_gather_linear(norm, qkv, x, gather)
    h = norm(x).view(images, H, W, -1)
    if shift > 0:
        h = torch.roll(h, shifts=(-shift, -shift), dims=(1, 2))
    return qkv(_window_partition(h, ws))


class WindowAttention(nn.Module):
    """reference: utils/models.py:28-56 (window_attention_forward) -- q is scaled BEFORE matmul1; relative position
    bias and the shifted-window mask are added outside the MatMul modules."""

    def __init__(self, dim, window_size, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.window_size = (window_size, window_size)
        self.scale = (dim // num_heads) ** -0.5
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, num_heads))
        coords = torch.stack(torch.meshgrid(torch.arange(window_size), torch.arange(window_size), indexing="ij")).flatten(1)
        rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += window_size - 1
        rel[:, :, 1] += window_size - 1
        rel[:, :, 0] *= 2 * window_size - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3)
        self.proj = nn.Linear(dim, dim)
        self.softmax = nn.Softmax(dim=-1)
        self.matmul1 = MatMul()
        self.matmul2 = MatMul()

    fused = False      # set by utils.deploy.fuse_attention, as Attention.fused
    fold_qkv = False   # set by utils.deploy.fuse_qkv, as Attention.fold_qkv

    def forward(self, x, mask=None, residual=None, layout=None, norm=None, gather=None):
        """residual, layout: (SwinBlock with fold_residual) return residual + the image of the output windows under
        layout = (images, height, width, window, shift) -- window reverse, then roll by (shift, shift) -- with the
        reverse, roll and add folded into proj's store when it applies.  norm, gather: (SwinBlock with fold_gather) x is
        the block's input [images, height * width, C] and the windows are those of roll(norm(x), (-shift, -shift)) under
        gather = (images, height, width, window, shift), with the LayerNorm, roll and partition folded into qkv when it
        applies."""
        if self.fold_qkv and self.fused:
            N = x.shape[1] if gather is None else gather[3] * gather[3]
            H, D = self.num_heads, x.shape[-1] // self.num_heads
            if frozen_qkv_applies(self.qkv, self.matmul1, self.matmul2, x, N, H, D, self.relative_position_bias_table, mask,
                                  norm=norm, gather=gather):
                bias = self.relative_position_bias_table[self.relative_position_index.view(-1)].view(N, N, -1).permute(2, 0, 1).contiguous()
                return self._proj(frozen_qkv_attention(self.qkv, self.matmul1, self.matmul2, x, N, H, D, self.scale,
                                                       scale_on_q=True, bias=bias, mask=mask, norm=norm, gather=gather),
                                  residual, layout)
        if gather is None:
            B_, N, C = x.shape
            y = self.qkv(x)
        else:
            y = _window_qkv(norm, self.qkv, x, gather)
            B_, N, C = y.shape[0], y.shape[1], x.shape[-1]
        if self.fused:
            bias = self.relative_position_bias_table[self.relative_position_index.view(-1)].view(N, N, -1).permute(2, 0, 1).contiguous()
            if frozen_attention_applies(self.matmul1, self.matmul2, N, C // self.num_heads, y, bias, mask):
                qkv5 = y.reshape(B_, N, 3, self.num_heads, C // self.num_heads)
                return self._proj(frozen_attention(self.matmul1, self.matmul2, qkv5, self.scale, scale_on_q=True, bias=bias,
                                                   mask=mask), residual, layout)
        qkv = y.reshape(B_, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        q = q * self.scale
        attn = self.matmul1(q, k.transpose(-2, -1))
        bias = self.relative_position_bias_table[self.relative_position_index.view(-1)].view(N, N, -1).permute(2, 0, 1).contiguous()
        attn = attn + bias.unsqueeze(0)
        if mask is not None:
            nW = mask.shape[0]
            attn = attn.view(B_ // nW, nW, self.num_heads, N, N) + mask.unsqueeze(1).unsqueeze(0)
            attn = attn.view(-1, self.num_heads, N, N)
        attn = self.softmax(attn)
        x = self.matmul2(attn, v).transpose(1, 2).reshape(B_, N, C)
        return self._proj(x, residual, layout)

    def _proj(self, x, residual, layout):
        if residual is None:
            return self.proj(x)
        if frozen_residual_applies(self.proj, x, residual, layout):
            return frozen_residual_linear(self.proj, x, residual, layout)
        _images, H, W, ws, shift = layout
        h = _window_reverse(self.proj(x), ws, H, W)
        if shift > 0:
            h = torch.roll(h, shifts=(shift, shift), dims=(1, 2))
        return residual + h.view(residual.shape)


class SwinBlock(nn.Module):
    def __init__(self, dim, res, num_heads, window_size, shift):
        super().__init__()
        self.res, self.ws, self.shift = res, window_size, shift
        self.norm1 = nn.LayerNorm(dim)
        self.attn = WindowAttention(dim, window_size, num_heads)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, dim * 4)
        mask = None
        if shift > 0:
            img = torch.zeros(1, res, res, 1)
            cnt = 0
            for h in (slice(0, -window_size), slice(-window_size, -shift), slice(-shift, None)):
                for w in (slice(0, -window_size), slice(-window_size, -shift), slice(-shift, None)):
                    img[:, h, w, :] = cnt
                    cnt += 1
            mw = _window_partition(img, window_size).view(-1, window_size * window_size)
            mask = mw.unsqueeze(1) - mw.unsqueeze(2)
            mask = mask.masked_fill(mask != 0, -100.0).masked_fill(mask == 0, 0.0)
        self.register_buffer("attn_mask", mask)

    fold_norm2 = False     # set by utils.deploy.fuse_norm, as Block.fold_norm2
    fold_residual = False  # set by utils.deploy.fuse_residual, as Block.fold_residual (proj's add with the window layout)
    fold_gather = False    # set by utils.deploy.fuse_gather: hand x and norm1 to attn, which folds norm1, the roll and the
                           # window partition into qkv when it applies

    def forward(self, x):
        if self.fold_residual:
            return self._forward_res(x)
        B, L, C = x.shape
        H = W = self.res
        if self.fold_gather:
            win = self.attn(x, mask=self.attn_mask, norm=self.norm1, gather=(B, H, W, self.ws, self.shift))
        else:
            h = self.norm1(x).view(B, H, W, C)
            if self.shift > 0:
                h = torch.roll(h, shifts=(-self.shift, -self.shift), dims=(1, 2))
            win = self.attn(_window_partition(h, self.ws), mask=self.attn_mask)
        h = _window_reverse(win, self.ws, H, W)
        if self.shift > 0:
            h = torch.roll(h, shifts=(self.shift, self.shift), dims=(1, 2))
        x = x + h.view(B, L, C)
        if self.fold_norm2:
            return x + self.mlp(x, norm=self.norm2)
        return x + self.mlp(self.norm2(x))

    def _forward_res(self, x):
        B, L, C = x.shape
        H = W = self.res
        layout = (B, H, W, self.ws, self.shift)
        if self.fold_gather:
            x = self.attn(x, mask=self.attn_mask, residual=x, layout=layout, norm=self.norm1, gather=layout)
        else:
            h = self.norm1(x).view(B, H, W, C)
            if self.shift > 0:
                h = torch.roll(h, shifts=(-self.shift, -self.shift), dims=(1, 2))
            x = self.attn(_window_partition(h, self.ws), mask=self.attn_mask, residual=x, layout=layout)
        return self.mlp(x, norm=self.norm2, residual=x) if self.fold_norm2 else self.mlp(self.norm2(x), residual=x)


class PatchMerging(nn.Module):
    def __init__(self, res, dim):
        super().__init__()
        self.res = res
        self.norm = nn.LayerNorm(4 * dim)
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)

    fold_norm = False      # set by utils.deploy.fuse_norm: fold norm into reduction when it applies
    fold_gather = False    # set by utils.deploy.fuse_gather: fold the 2x2 cat and norm into reduction when it applies

    def forward(self, x):
        B, L, C = x.shape
        if self.fold_gather:
            gather = ("merge", B, self.res, self.res, 0, 0)
            if frozen_gather_applies(self.norm, self.reduction, x, gather):
                return frozen_gather_linear(self.norm, self.reduction, x, gather)
        x = x.view(B, self.res, self.res, C)
        x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1).view(B, -1, 4 * C)
        if self.fold_norm:
            return _norm_linear(self.norm, self.reduction, x)
        return self.reduction(self.norm(x))


class SwinStage(nn.Module):
    def __init__(self, dim, res, depth, num_heads, window_size, downsample):
        super().__init__()
        ws = min(window_size, res)
        self.blocks = nn.Sequential(*[SwinBlock(dim, res, num_heads, ws, 0 if (i % 2 == 0 or ws >= res) else ws // 2) for i in range(depth)])
        self.downsample = PatchMerging(res, dim) if downsample else None

    def forward(self, x):
        x = self.blocks(x)
        return self.downsample(x) if self.downsample is not None else x


class SwinTransformer(nn.Module):
    def __init__(self, img_size=384, patch=4, dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=12,
                 num_classes=1000, seed=0):
        super().__init__()
        self.patch_embed = PatchEmbed(img_size, patch, dim)
        self.patch_norm = nn.LayerNorm(dim)
        res = img_size // patch
        self.layers = nn.Sequential(*[SwinStage(dim * 2 ** i, res // 2 ** i, depths[i], num_heads[i], window_size, i + 1 < len(depths))
                                      for i in range(len(depths))])
        self.norm = nn.LayerNorm(dim * 2 ** (len(depths) - 1))
        self.head = nn.Linear(dim * 2 ** (len(depths) - 1), num_classes)
        gen = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name_, p_ in self.named_parameters():
                if p_.dim() > 1:
                    p_.copy_(torch.nn.init.trunc_normal_(torch.empty_like(p_), std=0.02, generator=gen))
                elif name_.endswith("bias") and "norm" not in name_:
                    p_.copy_(torch.empty_like(p_).uniform_(-0.02, 0.02, generator=gen))
            for m in self.modules():
                if isinstance(m, WindowAttention):
                    m.qkv.weight.mul_(4.0)
                if isinstance(m, Mlp):
                    m.fc1.weight.mul_(4.0)
            self.head.weight.mul_(8.0)

    fold_stem = False      # set by utils.deploy.fuse_stem: the frozen patch-embedding conv stores the token rows
                           # normalised by patch_norm, when it applies

    def forward(self, x):
        if self.fold_stem and frozen_stem_applies(self.patch_embed.proj, x, norm=self.patch_norm):
            x = frozen_stem(self.patch_embed.proj, x, norm=self.patch_norm)
        else:
            x = self.patch_norm(self.patch_embed(x))
        x = self.norm(self.layers(x))
        return self.head(x.mean(dim=1))


_SWIN_ZOO = {
    "swin_tiny_patch4_window7_224": dict(img_size=224, dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=7),
    "swin_small_patch4_window7_224": dict(img_size=224, dim=96, depths=(2, 2, 18, 2), num_heads=(3, 6, 12, 24), window_size=7),
    "swin_base_patch4_window7_224": dict(img_size=224, dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=7),
    "swin_base_patch4_window12_384": dict(img_size=384, dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=12),
}


_ZOO = {
    "vit_tiny_patch16_224": dict(img_size=224, patch=16, dim=192, depth=12, num_heads=3),
    "vit_small_patch32_224": dict(img_size=224, patch=32, dim=384, depth=12, num_heads=6),
    "vit_small_patch16_224": dict(img_size=224, patch=16, dim=384, depth=12, num_heads=6),
    "vit_base_patch16_224": dict(img_size=224, patch=16, dim=768, depth=12, num_heads=12),
    "vit_base_patch16_384": dict(img_size=384, patch=16, dim=768, depth=12, num_heads=12),
    "deit_tiny_patch16_224": dict(img_size=224, patch=16, dim=192, depth=12, num_heads=3),
    "deit_small_patch16_224": dict(img_size=224, patch=16, dim=384, depth=12, num_heads=6),
    "deit_base_patch16_224": dict(img_size=224, patch=16, dim=768, depth=12, num_heads=12),
    "deit_base_patch16_384": dict(img_size=384, patch=16, dim=768, depth=12, num_heads=12),
}


def get_net(name, device="cuda", seed=0, **override):
    """reference: utils/models.py:62-91 (timm.create_model + attention rewrite); here: synthetic weights."""
    if name in _SWIN_ZOO:
        cfg = dict(_SWIN_ZOO[name]); cfg.update(override)
        return SwinTransformer(seed=seed, **cfg).to(device).eval()
    cfg = dict(_ZOO[name]); cfg.update(override)
    net = VisionTransformer(seed=seed, **cfg)
    return net.to(device).eval()


