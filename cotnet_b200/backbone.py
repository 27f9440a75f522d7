"""The caller of the hot path: a timm-style ResNet trunk whose bottleneck ``conv2`` is the CoT block.

Host code stays PyTorch (BASELINE.json north_star); this file exists so the bench / tests can run
CoTNet-50 / CoTNeXt-50 end to end on the GPU box, where /root/reference is absent.  Module names follow
the reference (``models/resnet.py:448-611`` ResNet, ``models/cotnet.py:181-264`` Bottleneck) so its
checkpoints load unchanged:  conv1, bn1, layer{1..4}.{i}.{conv1,bn1,conv2.<CotLayer keys>,conv3,bn3,
downsample.{0,1}}, fc.

Only what the four ``cotnet*`` entry points (models/cotnet.py:266-288) use is implemented: 7x7 stem,
max-pool, [3,4,6,3]/[3,4,23,3] stages, 1x1 conv down-sample, 3x3/2 avg-pool in front of the CoT layer
of stride-2 blocks (``avd``, :199-202,:237-238), global average pool + fc.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import dropblock, fused
from .cot_layer import CotLayer, CoXtLayer


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, cardinality=1, base_width=64):
        super().__init__()
        width = int(math.floor(planes * (base_width / 64)) * cardinality)
        outplanes = planes * self.expansion
        self.conv1 = nn.Conv2d(inplanes, width, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.act1 = nn.ReLU(inplace=True)
        self.avd = nn.AvgPool2d(3, 2, padding=1) if stride > 1 else None
        self.conv2 = CotLayer(width, kernel_size=3) if cardinality == 1 else CoXtLayer(width, kernel_size=3)
        self.conv3 = nn.Conv2d(width, outplanes, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(outplanes)
        self.act3 = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride
        self.drop_block = None          # the stage's dropblock.DropBlock (set by the trunk), applied after bn1 and bn3
        self.drop_block_sites = ()

    def zero_init_last_bn(self):
        nn.init.zeros_(self.bn3.weight)

    def drop_block_site_names(self):
        return ("bn1", "bn3")

    def set_drop_block(self, spec, site):
        """Give the block its stage's DropBlock (or None) and its site numbers from `site` on; returns the next free site."""
        self.drop_block = spec
        self.drop_block_sites = () if spec is None else (site, site + 1)
        return site + len(self.drop_block_sites)

    def forward(self, x, drop_scale=None, drop_block_key=None):
        """drop_scale: None or [B] per-sample stochastic-depth scales applied to bn3's output before the residual add
        (models/cotnet.py:256-257); drop_block_key: None or the trunk's [2] int64 DropBlock key of this forward (both drawn by
        the trunk, StochasticDepth)."""
        key = drop_block_key if self.drop_block is not None else None
        if fused.supported(x):
            return self._forward_fused(x, drop_scale, key)
        residual = x
        x = self.bn1(self.conv1(x))
        if key is not None:                                                     # models/cotnet.py:233-234
            x = dropblock.drop_block(x, key, self.drop_block_sites[0], self.drop_block)
        x = self.act1(x)
        if self.avd is not None:
            x = self.avd(x)
        x = self.conv2(x)
        x = self.bn3(self.conv3(x))
        if key is not None:                                                     # :250-251
            x = dropblock.drop_block(x, key, self.drop_block_sites[1], self.drop_block)
        if drop_scale is not None:
            x = x * drop_scale.to(x.dtype).view(-1, 1, 1, 1)
        if self.downsample is not None:
            residual = self.downsample(residual)
        x += residual
        return self.act3(x)

    def _forward_fused(self, x, drop_scale=None, key=None):
        """channels_last path: bn1+ReLU and bn3+residual+ReLU (SURVEY section 8f rank 1) run on the fused BatchNorm
        kernels (2 passes each way) instead of ATen's channels_last batch-norm kernels.  With DropBlock the bn1 mask is applied
        to the ReLU output (relu(a)*M*s == relu(a*M*s), s > 0) and bn3 runs without residual and ReLU, which the DropBlock
        tail kernel adds."""
        cl = torch.channels_last
        residual = x
        y = fused.conv1x1_bn(x, self.conv1, self.bn1, relu=True)
        if key is not None:
            y = dropblock.drop_block(y, key, self.drop_block_sites[0], self.drop_block)
        if self.avd is not None:
            y = fused.avg_pool3x3s2(y)              # nn.AvgPool2d(3, 2, padding=1) on the fused NHWC kernel
        y = self.conv2(y.contiguous(memory_format=cl))
        if self.downsample is not None:
            residual = fused.conv1x1_bn(residual, self.downsample[0], self.downsample[1], relu=False)
        if key is not None:
            z = fused.conv1x1_bn(y.contiguous(memory_format=cl), self.conv3, self.bn3, relu=False)
            return dropblock.drop_block_res_relu(z, residual.contiguous(memory_format=cl), key, self.drop_block_sites[1],
                                                 self.drop_block, drop_scale)
        return fused.conv1x1_bn(y.contiguous(memory_format=cl), self.conv3, self.bn3, relu=True,
                                res=residual.contiguous(memory_format=cl), drop_scale=drop_scale)


class StochasticDepth:
    """Stochastic depth and classifier dropout of the reference trunks (``drop_path_rate`` / ``drop_rate`` of create_model;
    models/resnet.py:409-440,608-609, models/cotnet_hybrid.py:275,442-443), shared by CoTResNet and CoTHybridNet.

    Block i of the n bottlenecks drops its residual branch with probability ``drop_path_rate * i / (n - 1)``.  In training the
    trunk draws every block's per-sample scales with ONE ``torch.rand(n, B)`` (fp32) per forward, s = floor(keep + u) / keep,
    so a captured CUDA graph draws new masks at every replay (torch's Philox offsets); the scales reach the fused BatchNorm
    kernels of bn3 (``fused.conv1x1_bn(drop_scale=)``).  No parameter or buffer is added: state dicts do not change.

    While stochastic depth is active (training mode, drop_path_rate > 0) the trunk calls the bottlenecks one by one to hand each
    its scales, so the ``layer1`` .. ``layer4`` Sequential containers are not called: hooks registered on those four modules do
    not fire then (hooks on the blocks and everything inside them do).  In eval mode, or with drop_path_rate 0, the stages run
    as before.

    DropBlock (``drop_block_rate``, models/resnet.py:397-401): stages 3 and 4 share one dropblock.DropBlock each; the trunk draws
    ONE [2] int64 key per training forward (``torch.randint`` on the input's device, so a captured graph draws a new key at every
    replay) and hands it to the blocks, whose sites are numbered in forward order (dropblock.py).  While it is active the trunk
    calls its blocks one by one, as for stochastic depth."""

    #: test hook: a [n_blocks, B] tensor of per-sample scales used instead of the random draw (training mode only)
    fixed_drop_path_scales = None
    #: test hook: a [2] int64 DropBlock key used instead of the random draw (training mode only)
    fixed_drop_block_key = None

    def _init_regularisers(self, drop_rate, drop_path_rate, drop_block_rate=0.):
        self.drop_rate = float(drop_rate)
        self.drop_path_rate = float(drop_path_rate)
        self.drop_block_rate = float(drop_block_rate)
        blocks = self.blocks()
        n = len(blocks)
        for i, blk in enumerate(blocks):
            blk.drop_path_rate = self.drop_path_rate * i / (n - 1)
        self._dp_keep = {}
        site = 0
        for name, spec in zip(("layer1", "layer2", "layer3", "layer4"), dropblock.stage_drop_blocks(self.drop_block_rate)):
            for blk in getattr(self, name):
                site = blk.set_drop_block(spec, site)
        self.n_drop_block_sites = site

    def drop_block_table(self):
        """[(block name, site name, site number, DropBlock)] of every DropBlock site, in forward order."""
        out = []
        for name in ("layer1", "layer2", "layer3", "layer4"):
            for i, blk in enumerate(getattr(self, name)):
                for where, s in zip(blk.drop_block_site_names(), blk.drop_block_sites):
                    out.append(("%s.%d" % (name, i), where, s, blk.drop_block))
        return out

    def blocks(self):
        return [b for name in ("layer1", "layer2", "layer3", "layer4") for b in getattr(self, name)]

    def drop_path_rates(self):
        return [b.drop_path_rate for b in self.blocks()]

    def _drop_path_scales(self, x):
        if not (self.training and self.drop_path_rate > 0.):
            return None
        B = x.shape[0]
        if self.fixed_drop_path_scales is not None:
            s = self.fixed_drop_path_scales.to(device=x.device, dtype=torch.float32)
            assert s.shape == (len(self.blocks()), B), "fixed_drop_path_scales must be [n_blocks, B]"
            return s.contiguous()
        keep = self._dp_keep.get(x.device)
        if keep is None:
            keep = torch.tensor([1. - r for r in self.drop_path_rates()], dtype=torch.float32, device=x.device).view(-1, 1)
            self._dp_keep[x.device] = keep
        return torch.floor(keep + torch.rand(keep.shape[0], B, dtype=torch.float32, device=x.device)) / keep

    def _drop_block_key(self, x):
        if not (self.training and self.drop_block_rate > 0.):
            return None
        if self.fixed_drop_block_key is not None:
            k = self.fixed_drop_block_key.to(device=x.device, dtype=torch.int64)
            assert k.shape == (2,), "fixed_drop_block_key must be [2] int64"
            return k
        return torch.randint(0, 2 ** 32, (2,), dtype=torch.int64, device=x.device)

    def _run_blocks(self, x):
        s = self._drop_path_scales(x)
        key = self._drop_block_key(x)
        if s is None and key is None:
            return self.layer4(self.layer3(self.layer2(self.layer1(x))))
        for i, blk in enumerate(self.blocks()):
            x = blk(x, drop_scale=s[i] if (s is not None and blk.drop_path_rate > 0.) else None, drop_block_key=key)
        return x

    def _classifier(self, x):
        if self.drop_rate:
            x = F.dropout(x, p=self.drop_rate, training=self.training)
        return self.fc(x)


class CoTResNet(StochasticDepth, nn.Module):
    def __init__(self, layers, num_classes=1000, in_chans=3, cardinality=1, base_width=64, zero_init_last_bn=True,
                 drop_rate=0., drop_path_rate=0., drop_block_rate=0.):
        super().__init__()
        self.num_classes = num_classes
        inplanes = 64
        self.conv1 = nn.Conv2d(in_chans, inplanes, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(inplanes)
        self.act1 = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        for i, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
            stride = 1 if i == 0 else 2
            blocks = []
            for b in range(n):
                s = stride if b == 0 else 1
                down = None
                if b == 0 and (s != 1 or inplanes != planes * Bottleneck.expansion):
                    down = nn.Sequential(
                        nn.Conv2d(inplanes, planes * Bottleneck.expansion, 1, stride=s, bias=False),
                        nn.BatchNorm2d(planes * Bottleneck.expansion))
                blocks.append(Bottleneck(inplanes, planes, s, down, cardinality, base_width))
                inplanes = planes * Bottleneck.expansion
            self.add_module("layer%d" % (i + 1), nn.Sequential(*blocks))
        self.num_features = inplanes
        self.global_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(self.num_features, num_classes)
        self._init_regularisers(drop_rate, drop_path_rate, drop_block_rate)
        # models/resnet.py:575-584
        for m in self.modules():
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
            if x.dtype == torch.bfloat16:
                # conv1 + bn1 + ReLU: 7x7/s2 stem on the 4-tap wgmma implicit GEMM, BatchNorm statistics from its epilogue
                # (fused.stem_conv_bn falls back to cuDNN + the fused BatchNorm kernels for geometries it does not take)
                x = fused.max_pool3x3s2(fused.stem_conv_bn(x, self.conv1, self.bn1, relu=True))
            else:
                x = fused.max_pool3x3s2(fused.bn_act(self.conv1(x).contiguous(memory_format=torch.channels_last), self.bn1, relu=True))
        else:
            x = self.maxpool(self.act1(self.bn1(self.conv1(x))))
        return self._run_blocks(x)

    def forward(self, x):
        x = self.global_pool(self.forward_features(x)).flatten(1)
        return self._classifier(x)

    def cot_layers(self):
        return [m for m in self.modules() if isinstance(m, (CotLayer, CoXtLayer))]


def cotnet50(**kw):
    return CoTResNet([3, 4, 6, 3], **kw)                                   # models/cotnet.py:270-273


def cotnext50_2x48d(**kw):
    return CoTResNet([3, 4, 6, 3], cardinality=2, base_width=48, **kw)     # :275-278


def cotnet101(**kw):
    return CoTResNet([3, 4, 23, 3], **kw)                                  # :280-283


def cotnext101_2x48d(**kw):
    return CoTResNet([3, 4, 23, 3], cardinality=2, base_width=48, **kw)    # :285-288


MODELS = {"cotnet50": cotnet50, "cotnext50_2x48d": cotnext50_2x48d, "cotnet101": cotnet101,
          "cotnext101_2x48d": cotnext101_2x48d}
