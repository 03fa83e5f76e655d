"""Per-object ("group") convolution blocks around the hot path -- cuDNN via PyTorch, unchanged in role.

Tensors named g carry an object axis: [B, K, C, H, W]; x tensors are shared across objects [B, C, H, W].
State-dict names mirror the reference (cutie/model/group_modules.py:39-126, cutie/model/channel_attn.py:7-39,
cutie/model/modules.py:8-85) so checkpoints load; the code is a fresh restatement.
"""
import math
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from cutie_b200 import kernels as K_
from cutie_b200.model.fuse import conv_add, conv_plain, conv_relu


def fold(g: torch.Tensor) -> torch.Tensor:
    return g.reshape(g.shape[0] * g.shape[1], *g.shape[2:])


def unfold(t: torch.Tensor, B: int) -> torch.Tensor:
    return t.reshape(B, t.shape[0] // B, *t.shape[1:])


def resize_objects(g: torch.Tensor, ratio: float, mode: str) -> torch.Tensor:
    B = g.shape[0]
    kw = dict(align_corners=False) if mode == 'bilinear' else {}
    return unfold(F.interpolate(fold(g), scale_factor=ratio, mode=mode, **kw), B)


def area_resize(owner: nn.Module, x: torch.Tensor, size) -> torch.Tensor:
    """F.interpolate(x, size=size, mode='area') for [..., H, W]; an integer-factor reduction goes through
    cutie_area_pool where `owner.glue_dispatch` (attached by CUTIE.optimize_for_inference) found it faster."""
    H, W = x.shape[-2:]
    h, w = int(size[0]), int(size[1])
    lead = x.shape[:-2]

    def aten():
        return F.interpolate(x.reshape(-1, 1, H, W), size=(h, w), mode='area').reshape(*lead, h, w)
    t = getattr(owner, 'glue_dispatch', None)
    if t is None or h == 0 or w == 0 or H % h or W % w or H // h != W // w or H // h < 2 or H // h > 64:
        return aten()
    f = H // h
    return t('area_pool', (tuple(x.shape), f), aten, lambda trial: K_.area_pool(x, f), x)


class ObjConv2d(nn.Conv2d):
    """nn.Conv2d applied independently to every object (group_modules.py:39-43)."""

    def forward(self, g: torch.Tensor) -> torch.Tensor:
        return unfold(super().forward(fold(g)), g.shape[0])


class ChannelAttnResBlock(nn.Module):
    """relu-conv3x3-relu-conv3x3, ECA channel gate, residual (channel_attn.py:7-39)."""

    def __init__(self, c_in: int, c_out: int):
        super().__init__()
        self.conv1 = nn.Conv2d(c_in, c_out, 3, padding=1)
        self.conv2 = nn.Conv2d(c_out, c_out, 3, padding=1)
        t = int((abs(math.log2(c_out)) + 1) // 2)
        k = t if t % 2 else t + 1
        self.conv = nn.Conv1d(1, 1, k, padding=(k - 1) // 2, bias=False)
        self.downsample = nn.Identity() if c_in == c_out else nn.Conv2d(c_in, c_out, 1)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        t = getattr(self, 'glue_dispatch', None)
        twins = getattr(self, 'cl_twins', None)
        if (t is None or twins is None or x.dim() != 4 or not x.is_contiguous() or x.shape[1] % 4
                or twins[0].weight.device != x.device):
            return self._forward(x, self.conv1, self.conv2)
        # NCHW input (our transformer kernels emit channel-major pixels): cuDNN then re-lays-out input, weight AND output
        # around each 3x3 convolution (6 + 7 + 6 us around a 19 us kernel at 480p).  Alternative, A/B-ed on the device: one
        # copy to channels-last on entry, channels-last weight twins, everything in between channels-last.
        tol = 2e-2 if torch.backends.cudnn.allow_tf32 else 2e-4
        return t('caresblock_channels_last', (tuple(x.shape),), lambda: self._forward(x, self.conv1, self.conv2),
                 lambda trial: self._forward(x.contiguous(memory_format=torch.channels_last), *twins).contiguous(), x,
                 rtol=tol)                         # .contiguous(): the copy back to NCHW is part of what is timed

    def make_channels_last_twins(self):
        """conv1 / conv2 copies with channels-last weights (sharing the bias Parameters), for the channels-last variant of
        forward(); plain attributes, so state_dict is unchanged.  Needs c_in == c_out (no projection shortcut)."""
        if not isinstance(self.downsample, nn.Identity):
            return None
        twins = []
        for conv in (self.conv1, self.conv2):
            tw = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding)
            tw.weight = nn.Parameter(conv.weight.detach().clone().contiguous(memory_format=torch.channels_last),
                                     requires_grad=False)
            tw.bias = conv.bias
            twins.append(tw.eval())
        object.__setattr__(self, 'cl_twins', tuple(twins))
        return self.cl_twins

    def _forward(self, x: torch.Tensor, conv1: nn.Conv2d, conv2: nn.Conv2d) -> torch.Tensor:
        y = conv2(conv_relu(conv1, x, relu_in=True))
        skip = self.downsample(x)

        def aten():
            gate = self.conv(y.mean(dim=(2, 3)).unsqueeze(1)).sigmoid().transpose(1, 2).unsqueeze(-1)
            return y * gate + skip
        t = getattr(self, 'glue_dispatch', None)
        if t is None:
            return aten()
        # conv1d + sigmoid + mul + add as cutie_eca_scale_add (in place into the fresh convolution output)
        return t('eca_scale_add', (tuple(y.shape), tuple(y.stride()), tuple(skip.stride())), aten,
                 lambda trial: K_.eca_scale_add_(y.clone(memory_format=torch.preserve_format) if trial else y, skip,
                                                 self.conv.weight), y)


class ObjResBlock(nn.Module):
    """group_modules.py:46-64."""

    def __init__(self, c_in: int, c_out: int):
        super().__init__()
        self.downsample = nn.Identity() if c_in == c_out else ObjConv2d(c_in, c_out, 1)
        self.conv1 = ObjConv2d(c_in, c_out, 3, padding=1)
        self.conv2 = ObjConv2d(c_out, c_out, 3, padding=1)

    def forward(self, g):
        t = getattr(self, 'glue_dispatch', None)
        twins = getattr(self, 'cl_twins', None)
        if (t is None or twins is None or g.dim() != 5 or not g.is_contiguous() or g.shape[2] % 4
                or twins[0].weight.device != g.device):
            return self._forward(g, self.conv1, self.conv2, self.downsample)
        # The decoder feeds this block NCHW tensors (cutie_upsample2x_add), so cuDNN transposes input and weight around
        # each 3x3 convolution and falls back to legacy NCHW-output engines (82 / 49 / 2 x 70 us at 480p, 3 objects).
        # Alternative, A/B-ed on the device: one copy to channels-last on entry, channels-last weight twins throughout.
        tol = 2e-2 if torch.backends.cudnn.allow_tf32 else 2e-4

        def channels_last(trial):
            B, K = g.shape[:2]
            x = fold(g).contiguous(memory_format=torch.channels_last)
            return unfold(self._forward4(x, *twins).contiguous(), B)      # back to NCHW inside the timed variant
        return t('objresblock_channels_last', (tuple(g.shape),),
                 lambda: self._forward(g, self.conv1, self.conv2, self.downsample), channels_last, g, rtol=tol)

    def make_channels_last_twins(self):
        """Plain nn.Conv2d copies of conv1 / conv2 / the 1x1 projection shortcut with channels-last weights (sharing the
        bias Parameters), for the channels-last variant of forward(); plain attributes, state_dict unchanged."""
        def twin(conv):
            tw = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding)
            tw.weight = nn.Parameter(conv.weight.detach().clone().contiguous(memory_format=torch.channels_last),
                                     requires_grad=False)
            tw.bias = conv.bias
            return tw.eval()
        ds = None if isinstance(self.downsample, nn.Identity) else twin(self.downsample)
        object.__setattr__(self, 'cl_twins', (twin(self.conv1), twin(self.conv2), ds))
        return tuple(tw for tw in self.cl_twins if tw is not None)

    def _forward(self, g, conv1, conv2, downsample):
        ds = None if isinstance(downsample, nn.Identity) else downsample
        return unfold(self._forward4(fold(g), conv1, conv2, ds), g.shape[0])

    @staticmethod
    def _forward4(x, conv1, conv2, downsample):
        """The block on a folded [B*K, C, H, W] tensor: relu - conv1 - relu - conv2, plus the (projected) input; the
        residual add rides in conv2's epilogue where the model's fuser chose a form that can carry it."""
        skip = x if downsample is None else conv_plain(downsample, x)
        return conv_add(conv2, conv_relu(conv1, x, relu_in=True), skip)


class _AddDistributor(nn.Module):
    """x_transform(x) broadcast over objects + g_transform(g) (group_modules.py:67-104, method='add')."""

    def __init__(self, x_dim: int, g_dim: int, out_dim: int):
        super().__init__()
        self.x_transform = nn.Conv2d(x_dim, out_dim, 1)
        self.g_transform = ObjConv2d(g_dim, out_dim, 1)

    def forward(self, x, g):
        return self.x_transform(x).unsqueeze(1) + self.g_transform(g)


class FeatureFusion(nn.Module):
    """group_modules.py:107-126: fuse a shared feature map into per-object features."""

    def __init__(self, x_dim: int, g_dim: int, out_dim: int):
        super().__init__()
        self.distributor = _AddDistributor(x_dim, g_dim, out_dim)
        self.block1 = ChannelAttnResBlock(out_dim, out_dim)
        self.block2 = ChannelAttnResBlock(out_dim, out_dim)

    def forward(self, x, g):
        B = g.shape[0]
        return unfold(self.block2(self.block1(fold(self.distributor(x, g)))), B)


class UpsampleBlock(nn.Module):
    """modules.py:8-20: x2 bilinear upsample of g, add skip feature, ObjResBlock."""

    def __init__(self, c_in: int, c_out: int):
        super().__init__()
        self.out_conv = ObjResBlock(c_in, c_out)

    def forward(self, g, skip):
        if g.is_cuda:
            # fused sm_90a kernel (raises if the library is missing): ATen's bilinear kernel runs one thread per
            # output PIXEL and loops over objects x channels inside it -- 7 CTAs at 480p
            return self.out_conv(K_.upsample2x_add(g, skip))
        # CPU tensors only reach this block when the oracle harness (oracle/cpu_core.py, tests) borrows the
        # convolutional modules; InferenceCore itself cannot run on CPU (its kernels reject CPU tensors)
        return self.out_conv(resize_objects(g, 2, 'bilinear') + skip.unsqueeze(1))


def gated_update(h: torch.Tensor, v: torch.Tensor, owner: nn.Module = None) -> torch.Tensor:
    """modules.py:37-45: GRU-like update; v carries [forget | update | candidate] along channels.  With
    `owner.glue_dispatch` attached the eight ATen launches may run as cutie_gated_update."""
    d = v.shape[2] // 3

    def aten():
        f = torch.sigmoid(v[:, :, :d])
        u = torch.sigmoid(v[:, :, d:2 * d])
        n = torch.tanh(v[:, :, 2 * d:])
        return f * h * (1 - u) + u * n
    t = getattr(owner, 'glue_dispatch', None) if owner is not None else None
    if t is None or h.dim() != 5 or v.shape[2] != 3 * h.shape[2]:
        return aten()
    return t('gated_update', (tuple(h.shape), tuple(h.stride()), tuple(v.stride())), aten,
             lambda trial: K_.gated_update(h, v), h)


class MultiScaleSensoryUpdater(nn.Module):
    """modules.py:46-68 (decoder side): fuse stride-16/8/4 object features into the sensory memory."""

    def __init__(self, g_dims: List[int], mid_dim: int, sensory_dim: int):
        super().__init__()
        self.g16_conv = ObjConv2d(g_dims[0], mid_dim, 1)
        self.g8_conv = ObjConv2d(g_dims[1], mid_dim, 1)
        self.g4_conv = ObjConv2d(g_dims[2], mid_dim, 1)
        self.transform = ObjConv2d(mid_dim + sensory_dim, sensory_dim * 3, 3, padding=1)
        self.transform.amp_fp32 = True      # fp32 under autocast too, as modules.py:62-64 (a plain attribute: no state_dict key)

    def forward(self, g16, g8, g4, h):
        if isinstance(g4, (tuple, list)):
            # channel groups handed over separately (decoder features | logits): area pooling is per channel, so pooling
            # the pieces and concatenating at 1/16 of the size equals pooling their concatenation -- without the
            # full-resolution torch.cat (a 40 MB copy per frame at 480p)
            g4s = torch.cat([area_resize(self, t, (t.shape[-2] // 4, t.shape[-1] // 4)) for t in g4], 2)
        else:
            g4s = area_resize(self, g4, (g4.shape[-2] // 4, g4.shape[-1] // 4))
        g = self.g16_conv(g16) + self.g8_conv(area_resize(self, g8, (g8.shape[-2] // 2, g8.shape[-1] // 2))) + \
            self.g4_conv(g4s)
        return gated_update(h.float(), self.transform(torch.cat([g.float(), h.float()], 2)), self)


class DeepSensoryUpdater(nn.Module):
    """modules.py:71-85 (mask-encoder side)."""

    def __init__(self, f_dim: int, sensory_dim: int):
        super().__init__()
        self.transform = ObjConv2d(f_dim + sensory_dim, sensory_dim * 3, 3, padding=1)
        self.transform.amp_fp32 = True      # fp32 under autocast too, as modules.py:79-81

    def forward(self, g, h):
        return gated_update(h.float(), self.transform(torch.cat([g.float(), h.float()], 2)), self)
