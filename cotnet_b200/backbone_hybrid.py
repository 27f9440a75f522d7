"""SE-CoTNetD trunks (BASELINE.json configs[3], [4]): the second caller of the hot path (SURVEY.md section 8f rank 2).

A plain-PyTorch mirror of ``models/cotnet_hybrid.py`` -- ``CoTHybridNet`` (:338-452), ``CoTBottleneck`` (:118-204),
``downsample_avg`` (:222-236) -- and of ``models/layers/split_attn.py:31-88`` (``SplitAttnConv2d``), with the reference's
module names so that its checkpoints load with ``strict=True``:

    conv1.{0,1,3,4,6}  bn1  layer{1..4}.{i}.{conv1,bn1,conv2.<...>,conv3,bn3,downsample.{1,2}}  fc

``conv2`` is the CoT layer (``cot_layer.CoTLayer``: libcotb200 kernels) where the reference uses it -- every block of
layer4 and the even blocks of layer3 -- and ``SplitAttnConv2d`` (radix 1, swish) elsewhere (:138-156).  The BatchNorm /
ReLU / residual glue of the bottleneck and the 3x3/s2 ``avd`` pooling reuse the fused kernels of the CoTNet trunk
(``backbone.Bottleneck``); the split-attention block runs its bn0 -> SiLU -> pool -> MLP -> gate chain on the CoT tail kernels
(``fused.split_attn_tail``), only its 3x3 convolution stays cuDNN.
Only what ``se_cotnetd_{50,101,152}`` (:458-483) configure is implemented: deep stem, no stem max-pool, stride 2 in every
stage, avg-pool down-sampling, optional BlurPool anti-aliasing (152).
"""
import functools
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import dropblock, fused
from .backbone import StochasticDepth
from .cot_layer import CoTLayer


class BlurPool2d(nn.Module):
    """models/layers/blur_pool.py:19-58 with filt_size 3: reflect-pad 1, depthwise [1,2,1]x[1,2,1]/16, stride 2."""

    def __init__(self, channels, filt_size=3, stride=2):
        super().__init__()
        assert filt_size == 3
        self.channels, self.stride = channels, stride
        c = torch.tensor([0.25, 0.5, 0.25])
        self.register_buffer("_filt", (c[:, None] * c[None, :])[None, None].repeat(channels, 1, 1, 1), persistent=False)

    def forward(self, x):
        return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), self._filt.to(x.dtype), stride=self.stride, groups=x.shape[1])


class SplitAttnConv2d(nn.Module):
    """models/layers/split_attn.py:31-88.  conv -> bn0 -> act -> GAP -> fc1 -> bn1 -> act -> fc2 -> sigmoid (radix 1) /
    radix-softmax -> rescale."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 radix=1, reduction_factor=4):
        super().__init__()
        self.radix, self.cardinality = radix, groups
        mid_chs = out_channels * radix
        attn_chs = max(in_channels * radix // reduction_factor, 32)
        self.conv = nn.Conv2d(in_channels, mid_chs, kernel_size, stride, padding, dilation, groups=groups * radix, bias=bias)
        self.bn0 = nn.BatchNorm2d(mid_chs)
        self.act0 = nn.SiLU(inplace=True)
        self.fc1 = nn.Conv2d(out_channels, attn_chs, 1, groups=groups)
        self.bn1 = nn.BatchNorm2d(attn_chs)
        self.act1 = nn.SiLU(inplace=True)
        self.fc2 = nn.Conv2d(attn_chs, mid_chs, 1, groups=groups)

    def forward(self, x, drop_block=None):
        """drop_block: None or a function applied after bn0 (models/layers/split_attn.py:66-67).  With it, a channels_last CUDA
        input runs bn0 on the fused BatchNorm kernels and the rest of the chain in plain PyTorch."""
        if self.radix == 1 and self.cardinality == 1 and fused.supported(x) and drop_block is None:
            # channels_last CUDA tensors: everything after the convolution on the fused tail kernels (fused.split_attn_tail)
            u = self.conv(x).contiguous(memory_format=torch.channels_last)
            return fused.split_attn_tail(u, self.bn0, self.fc1, self.bn1, self.fc2)
        if drop_block is not None and fused.supported(x):
            x = fused.bn_act(self.conv(x).contiguous(memory_format=torch.channels_last), self.bn0)
        else:
            x = self.bn0(self.conv(x))
        if drop_block is not None:
            x = drop_block(x)
        x = self.act0(x)
        B, RC, H, W = x.shape
        if self.radix > 1:
            xr = x.reshape(B, self.radix, RC // self.radix, H, W)
            gap = xr.sum(dim=1)
        else:
            gap = x
        gap = F.adaptive_avg_pool2d(gap, 1)
        attn = self.fc2(self.act1(self.bn1(self.fc1(gap))))
        if self.radix > 1:
            attn = attn.view(B, self.cardinality, self.radix, -1).transpose(1, 2)
            attn = F.softmax(attn, dim=1).reshape(B, -1)
            out = (xr * attn.reshape(B, self.radix, RC // self.radix, 1, 1)).sum(dim=1)
        else:
            out = x * torch.sigmoid(attn).view(B, -1, 1, 1)
        return out.contiguous(memory_format=torch.channels_last) if fused._is_cl(x) and not x.is_contiguous() else out.contiguous()


class CoTBottleneck(nn.Module):
    """models/cotnet_hybrid.py:118-204 (cardinality 1, base_width 64; drop path through forward's drop_scale, DropBlock through its
    drop_block_key)."""
    expansion = 4

    def __init__(self, block_idx, inplanes, planes, stride=1, downsample=None, aa_layer=None, radix=1, avd=False,
                 avd_first=True, conv_dim=(), c4_dim=-1, c4_idx=()):
        super().__init__()
        width = planes
        outplanes = planes * self.expansion
        self.avd_first = avd_first
        self.avd = None
        self.conv1 = nn.Conv2d(inplanes, width, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.act1 = nn.ReLU(inplace=True)

        def pool(s):
            return nn.AvgPool2d(3, s, padding=1) if aa_layer is None else aa_layer(channels=width, stride=s)

        if (width in conv_dim) or (width == c4_dim and block_idx not in c4_idx):      # :138
            if stride > 1 and avd:
                self.avd = pool(stride)
                stride = 1
            self.conv2 = SplitAttnConv2d(width, width, kernel_size=3, stride=stride, padding=1, reduction_factor=4,
                                         dilation=1, groups=1, radix=radix)
        else:
            self.conv2 = CoTLayer(width, kernel_size=3)
            if stride > 1:
                self.avd = pool(stride)
        self.conv3 = nn.Conv2d(width, outplanes, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(outplanes)
        self.act3 = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride
        self.drop_block = None          # the stage's dropblock.DropBlock (set by the trunk)
        self.drop_block_sites = ()

    def zero_init_last_bn(self):
        nn.init.zeros_(self.bn3.weight)

    def drop_block_site_names(self):
        """bn1, bn0 of a split-attention conv2 (models/cotnet_hybrid.py:146), bn3."""
        return ("bn1", "conv2.bn0", "bn3") if isinstance(self.conv2, SplitAttnConv2d) else ("bn1", "bn3")

    def set_drop_block(self, spec, site):
        """Give the block its stage's DropBlock (or None) and its site numbers from `site` on; returns the next free site."""
        self.drop_block = spec
        n = 0 if spec is None else len(self.drop_block_site_names())
        self.drop_block_sites = tuple(range(site, site + n))
        return site + n

    def _site(self, key, i):
        """drop_block(., key, site i) of this block, or None without DropBlock."""
        if key is None:
            return None
        return functools.partial(dropblock.drop_block, key=key, site=self.drop_block_sites[i], spec=self.drop_block)

    def _pool(self, y):
        if isinstance(self.avd, nn.AvgPool2d) and self.avd.kernel_size == 3 and self.avd.stride == 2 and fused.supported(y):
            return fused.avg_pool3x3s2(y)
        return self.avd(y)

    def _conv2(self, y, key):
        if key is not None and isinstance(self.conv2, SplitAttnConv2d):
            return self.conv2(y, drop_block=self._site(key, 1))
        return self.conv2(y)

    def forward(self, x, drop_scale=None, drop_block_key=None):
        cl = torch.channels_last
        key = drop_block_key if self.drop_block is not None else None
        if fused.supported(x):      # channels_last CUDA tensors: fused BatchNorm(+ReLU,+residual) glue like backbone.Bottleneck
            y = fused.conv1x1_bn(x, self.conv1, self.bn1, relu=True)
            if key is not None:     # on the ReLU output: relu(a)*M*s == relu(a*M*s), s > 0
                y = self._site(key, 0)(y)
            if self.avd is not None and self.avd_first:
                y = self._pool(y)
            y = self._conv2(y.contiguous(memory_format=cl), key)
            if self.avd is not None and not self.avd_first:
                y = self._pool(y.contiguous(memory_format=cl))
            residual = x
            if self.downsample is not None:
                d = self.downsample
                residual = fused.conv1x1_bn(d[0](x).contiguous(memory_format=cl), d[1], d[2], relu=False)
            if key is not None:
                z = fused.conv1x1_bn(y.contiguous(memory_format=cl), self.conv3, self.bn3, relu=False)
                return dropblock.drop_block_res_relu(z, residual.contiguous(memory_format=cl), key, self.drop_block_sites[-1],
                                                     self.drop_block, drop_scale)
            return fused.conv1x1_bn(y.contiguous(memory_format=cl), self.conv3, self.bn3, relu=True,
                                    res=residual.contiguous(memory_format=cl), drop_scale=drop_scale)
        residual = x
        y = self.bn1(self.conv1(x))
        if key is not None:                                                          # :177-178
            y = self._site(key, 0)(y)
        y = self.act1(y)
        if self.avd is not None and self.avd_first:
            y = self.avd(y)
        y = self._conv2(y, key)
        if self.avd is not None and not self.avd_first:
            y = self.avd(y)
        y = self.bn3(self.conv3(y))
        if key is not None:                                                          # :191-192
            y = self._site(key, -1)(y)
        if drop_scale is not None:                                                   # :194-195
            y = y * drop_scale.to(y.dtype).view(-1, 1, 1, 1)
        if self.downsample is not None:
            residual = self.downsample(residual)
        y = y + residual
        return self.act3(y)


def _downsample_avg(in_channels, out_channels, stride):
    """models/cotnet_hybrid.py:222-236 (dilation 1)."""
    pool = nn.Identity() if stride == 1 else nn.AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False)
    return nn.Sequential(pool, nn.Conv2d(in_channels, out_channels, 1, stride=1, padding=0, bias=False), nn.BatchNorm2d(out_channels))


class CoTHybridNet(StochasticDepth, nn.Module):
    """models/cotnet_hybrid.py:338-452 for stem_type='deep', avg_down=True, output_stride=32."""

    def __init__(self, layers, num_classes=1000, in_chans=3, stem_width=64, aa_layer=None, zero_init_last_bn=True,
                 block_args=None, drop_rate=0., drop_path_rate=0., drop_block_rate=0.):
        super().__init__()
        block_args = dict(block_args or {})
        inplanes = stem_width * 2
        self.conv1 = nn.Sequential(
            nn.Conv2d(in_chans, stem_width, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(stem_width), nn.ReLU(inplace=True),
            nn.Conv2d(stem_width, stem_width, 3, stride=1, padding=1, bias=False), nn.BatchNorm2d(stem_width), nn.ReLU(inplace=True),
            nn.Conv2d(stem_width, inplanes, 3, stride=1, padding=1, bias=False))
        self.bn1 = nn.BatchNorm2d(inplanes)
        self.act1 = nn.ReLU(inplace=True)
        for i, (planes, n) in enumerate(zip([64, 128, 256, 512], layers)):          # make_blocks (:244-283): stride 2 in every stage
            blocks = []
            for b in range(n):
                stride = 2 if b == 0 else 1
                down = _downsample_avg(inplanes, planes * 4, stride) if (b == 0) else None
                blocks.append(CoTBottleneck(b, inplanes, planes, stride, down, aa_layer=aa_layer, **block_args))
                inplanes = planes * 4
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*blocks))
        self.num_features = 2048
        self.global_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(self.num_features, num_classes)
        self._init_regularisers(drop_rate, drop_path_rate, drop_block_rate)
        for m in self.modules():                                                     # :415-424
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0.0)
        if zero_init_last_bn:
            for m in self.modules():
                if hasattr(m, "zero_init_last_bn"):
                    m.zero_init_last_bn()

    def forward_features(self, x):
        if fused.supported(x):
            c = self.conv1
            cl = torch.channels_last
            x = fused.bn_act(c[0](x).contiguous(memory_format=cl), c[1], relu=True)
            x = fused.bn_act(c[3](x).contiguous(memory_format=cl), c[4], relu=True)
            x = fused.bn_act(c[6](x).contiguous(memory_format=cl), self.bn1, relu=True)
        else:
            x = self.act1(self.bn1(self.conv1(x)))
        return self._run_blocks(x)

    def forward(self, x):
        return self._classifier(self.global_pool(self.forward_features(x)).flatten(1))

    def cot_layers(self):
        return [m for m in self.modules() if isinstance(m, CoTLayer)]


def _args(n_l3, **kw):
    return dict(radix=1, conv_dim={64, 128}, c4_dim=256, c4_idx=set(range(0, n_l3, 2)), **kw)


def se_cotnetd_50(**kw):                                                             # :458-464
    return CoTHybridNet([3, 4, 6, 3], stem_width=32, block_args=_args(6, avd=False, avd_first=True), **kw)


def se_cotnetd_101(**kw):                                                            # :466-472
    return CoTHybridNet([3, 4, 23, 3], stem_width=64, block_args=_args(23, avd=False, avd_first=True), **kw)


def se_cotnetd_152(**kw):                                                            # :474-480
    return CoTHybridNet([3, 8, 36, 3], stem_width=64, aa_layer=BlurPool2d, block_args=_args(36, avd=True, avd_first=False), **kw)


def se_cotnetd_152_L(**kw):                                                          # :476-482
    """The SE-CoTNetD-152 trunk under the name the reference registers for its 320 x 320 data config (cot_l, crop_pct 0.909).
    MODELS lists each distinct trunk once, so this second name of se_cotnetd_152 is not in it."""
    return se_cotnetd_152(**kw)


MODELS = {"se_cotnetd_50": se_cotnetd_50, "se_cotnetd_101": se_cotnetd_101, "se_cotnetd_152": se_cotnetd_152}
