"""A plain-torch stand-in for the part of `timm` that the reference's MiDaS code uses: `create_model("vit_base_resnet50_384")`, the
ViT-B/16 hybrid whose patch embedding is a ResNetV2-50 trunk (preact=False, stem_type "same", StdConv2dSame with eps 1e-8,
GroupNorm(32) + ReLU, stages of 3, 4, 9 bottlenecks), under timm's attribute names.  Injected as sys.modules["timm"] it lets the
reference's own condition.midas.depth import and run on the CPU (tests/golden/make_midas_golden.py).  The names, the padding rule
and the standardisation eps restate timm's published source; they were not checked against a timm install."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def _pad_same(x, k, s):
    ih, iw = x.shape[-2:]
    ph = max((math.ceil(ih / s) - 1) * s + k - ih, 0)
    pw = max((math.ceil(iw / s) - 1) * s + k - iw, 0)
    return F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))


class StdConv2dSame(nn.Conv2d):
    """Weight-standardised convolution with TF "SAME" padding (static where stride 1, as timm resolves it)."""

    def __init__(self, cin, cout, k, stride=1, eps=1e-8):
        super().__init__(cin, cout, k, stride=stride, padding=(k - 1) // 2 if stride == 1 else 0, bias=False)
        self.same_pad = stride != 1
        self.eps = eps

    def forward(self, x):
        if self.same_pad:
            x = _pad_same(x, self.kernel_size[0], self.stride[0])
        w = F.batch_norm(self.weight.reshape(1, self.out_channels, -1), None, None, training=True, momentum=0., eps=self.eps).reshape_as(self.weight)
        return F.conv2d(x, w, None, self.stride, self.padding)


class GroupNormAct(nn.GroupNorm):
    def __init__(self, c, apply_act=True):
        super().__init__(32, c, eps=1e-5)
        self.apply_act = apply_act

    def forward(self, x):
        x = F.group_norm(x, self.num_groups, self.weight, self.bias, self.eps)
        return F.relu(x) if self.apply_act else x


class MaxPool2dSame(nn.MaxPool2d):
    def forward(self, x):
        ih, iw = x.shape[-2:]
        ph = max((math.ceil(ih / 2) - 1) * 2 + 3 - ih, 0)
        pw = max((math.ceil(iw / 2) - 1) * 2 + 3 - iw, 0)
        x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=-float("inf"))
        return F.max_pool2d(x, 3, 2)


class DownsampleConv(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv = StdConv2dSame(cin, cout, 1, stride)
        self.norm = GroupNormAct(cout, apply_act=False)

    def forward(self, x):
        return self.norm(self.conv(x))


class Bottleneck(nn.Module):
    def __init__(self, cin, cout, stride, proj):
        super().__init__()
        mid = cout // 4
        self.downsample = DownsampleConv(cin, cout, stride) if proj else None
        self.conv1, self.norm1 = StdConv2dSame(cin, mid, 1), GroupNormAct(mid)
        self.conv2, self.norm2 = StdConv2dSame(mid, mid, 3, stride), GroupNormAct(mid)
        self.conv3, self.norm3 = StdConv2dSame(mid, cout, 1), GroupNormAct(cout, apply_act=False)

    def forward(self, x):
        shortcut = self.downsample(x) if self.downsample is not None else x
        x = self.norm1(self.conv1(x))
        x = self.norm2(self.conv2(x))
        x = self.norm3(self.conv3(x))
        return F.relu(x + shortcut)


class ResNetStage(nn.Module):
    def __init__(self, cin, cout, stride, depth):
        super().__init__()
        self.blocks = nn.Sequential(*[Bottleneck(cin if i == 0 else cout, cout, stride if i == 0 else 1, i == 0) for i in range(depth)])

    def forward(self, x):
        return self.blocks(x)


class ResNetV2(nn.Module):
    def __init__(self, layers=(3, 4, 9)):
        super().__init__()
        self.stem = nn.Sequential()
        self.stem.add_module("conv", StdConv2dSame(3, 64, 7, 2))
        self.stem.add_module("norm", GroupNormAct(64))
        self.stem.add_module("pool", MaxPool2dSame(3, 2))
        cin, stages = 64, []
        for i, (d, c) in enumerate(zip(layers, (256, 512, 1024))):
            stages.append(ResNetStage(cin, c, 1 if i == 0 else 2, d))
            cin = c
        self.stages = nn.Sequential(*stages)

    def forward(self, x):
        return self.stages(self.stem(x))


class HybridEmbed(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone = ResNetV2()
        self.proj = nn.Conv2d(1024, 768, 1)


class Mlp(nn.Module):
    def __init__(self, c, h):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(c, h), nn.Linear(h, c)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x)))


class Attention(nn.Module):
    def __init__(self, c, heads):
        super().__init__()
        self.heads, self.scale = heads, (c // heads) ** -0.5
        self.qkv, self.proj = nn.Linear(c, 3 * c), nn.Linear(c, c)

    def forward(self, x):
        B, N, C = x.shape
        q, k, v = self.qkv(x).reshape(B, N, 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4)
        attn = ((q @ k.transpose(-2, -1)) * self.scale).softmax(-1)
        return self.proj((attn @ v).transpose(1, 2).reshape(B, N, C))


class Block(nn.Module):
    def __init__(self, c, heads):
        super().__init__()
        self.norm1 = nn.LayerNorm(c, eps=1e-6)
        self.attn = Attention(c, heads)
        self.norm2 = nn.LayerNorm(c, eps=1e-6)
        self.mlp = Mlp(c, 4 * c)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class VisionTransformer(nn.Module):
    def __init__(self):
        super().__init__()
        self.patch_embed = HybridEmbed()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, 768))
        self.pos_embed = nn.Parameter(torch.zeros(1, 1 + 24 * 24, 768))
        self.pos_drop = nn.Identity()
        self.blocks = nn.Sequential(*[Block(768, 12) for _ in range(12)])
        self.norm = nn.LayerNorm(768, eps=1e-6)
        self.head = nn.Linear(768, 1000)


def create_model(name, pretrained=False, **kwargs):
    if name != "vit_base_resnet50_384" or pretrained:
        raise NotImplementedError(f"timm stand-in: only create_model('vit_base_resnet50_384', pretrained=False), not {name!r}")
    return VisionTransformer()
