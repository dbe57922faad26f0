"""HRNet encoder variant of the hot path (BASELINE config 5, `MODEL.ENCODER_TYPE: hrnet48`).

Drop-in for the reference's `HRnet_encoder` / `hrnet_mid` (models/encoder.py:176-352) and the `HighResolutionNet` trunk
they wrap (models/model_zoo/hrnet.py:235-527, head_type 'none').  The torch.nn modules below are PARAMETER CONTAINERS
laid out so that `state_dict()` reproduces the reference's keys in the reference's order (released checkpoints load,
deterministic seeded initialisation matches); their `forward` methods launch the sm_90a kernels of librih_b200.so through
`renderih_b200.ops` on NHWC row matrices [N*H*W, C].  Nothing here calls a torch convolution / normalisation kernel.

Width table = `get_config` (hrnet.py:584-636): stage1 is one branch of 4 bottlenecks (64 -> 256), stages 2..4 have
2 / 3 / 4 branches of 4 BasicBlocks with (C, 2C, 4C, 8C) channels and 1 / 4 / 3 modules ('w18_small_*' differ).
"""
import os

import torch
import torch.nn as nn

from . import ops

BN_MOMENTUM = 0.1   # model_zoo/hrnet.py:18

# name -> (stage1 (blocks, planes), [(modules, blocks per branch, channels)] for stages 2..4)      hrnet.py:584-636
WIDTHS = {
    'w18_small_v1': ((1, 32), [(1, 2, (16, 32)), (1, 2, (16, 32, 64)), (1, 2, (16, 32, 64, 128))]),
    'w18_small_v2': ((2, 64), [(1, 2, (18, 36)), (3, 2, (18, 36, 72)), (2, 2, (18, 36, 72, 144))]),
}
for _c in (18, 30, 32, 40, 44, 48, 64):
    WIDTHS['w%d' % _c] = ((4, 64), [(1, 4, (_c, 2 * _c)), (4, 4, (_c, 2 * _c, 4 * _c)), (3, 4, (_c, 2 * _c, 4 * _c, 8 * _c))])


def _cl(conv):
    conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
    return conv


def _conv(cin, cout, k, stride=1, bias=False):
    return _cl(nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2, bias=bias))


def _bn(c):
    return nn.BatchNorm2d(c, momentum=BN_MOMENTUM)


def _cbr_seq(cin, cout, k, stride=1, relu=True, bias=False):
    """nn.Sequential(conv, bn[, relu]) with the reference's child indices 0 / 1 / 2"""
    layers = [_conv(cin, cout, k, stride, bias), _bn(cout)]
    if relu:
        layers.append(nn.ReLU(inplace=True))
    return nn.Sequential(*layers)


# ----------------------------------------------------------------------------- kernel-side helpers
def conv_bn(x, conv, bn, N, H, training, relu=True, res=None, alias_input=False):
    """Conv2d(+bias) -> BatchNorm2d -> (+res) -> (ReLU) on a square NHWC map; returns (y, Ho) -- or (y, Ho, x_alias) with alias_input:
    route the residual use of x through x_alias and its gradient is accumulated by this convolution's dgrad kernel (ops.conv2d).
    Training-mode batch statistics come out of the convolution's epilogue when it runs on the tensor-core path."""
    k, st, pd = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    fold = None if (training or alias_input or torch.is_grad_enabled() or conv.bias is not None) else bn.__dict__.get('_rih_fold')
    if fold is not None:       # inference: BatchNorm (+ residual + ReLU) in the convolution's epilogue (ops.conv2d_bn_eval)
        return ops.conv2d_bn_eval(x, conv.weight, N, H, H, st, pd, fold, order=0, relu=relu, res=res), (H + 2 * pd - k) // st + 1
    stats = torch.empty(2 * conv.out_channels, device=x.device, dtype=torch.float64) if training else None
    y = ops.conv2d(x, conv.weight, conv.bias, N, H, H, stride=st, pad=pd, stats=stats, alias_input=alias_input)
    xa = None
    if alias_input:
        y, xa = y
    y = ops.batchnorm(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, res=res, training=training,
                      momentum=bn.momentum, eps=bn.eps, relu=relu, stats=stats)
    Ho = (H + 2 * pd - k) // st + 1
    return (y, Ho, xa) if alias_input else (y, Ho)


def _first_conv_with_alias(x, conv, bn, N, H, training):
    """(out, x_for_the_residual_path): the alias form when gradients will flow (training), the plain form otherwise"""
    if training and x.requires_grad:
        out, _, xa = conv_bn(x, conv, bn, N, H, training, alias_input=True)
        return out, xa
    return conv_bn(x, conv, bn, N, H, training)[0], x


def stem_conv_bn(x, conv, bn, N, H, training, image_needs_grad):
    """First convolution on the 3-channel image (+BN+ReLU).  With Cin = 3 neither vector loads nor TMA apply to an implicit
    GEMM, so when the image needs no gradient the input is im2col'ed once (K padded to a multiple of 32) and the convolution
    becomes one dense GEMM [N*Ho*Wo, Kpad] x [Cout, Kpad]^T."""
    if image_needs_grad:
        return conv_bn(x, conv, bn, N, H, training)
    Cout, Cin, R, S = conv.weight.shape
    st, pd = conv.stride[0], conv.padding[0]
    K = R * S * Cin
    Kpad = (K + 31) // 32 * 32
    A = ops.im2col(x, N, H, H, R, S, st, pd, Kpad)
    w2d = torch.nn.functional.pad(conv.weight.permute(0, 2, 3, 1).reshape(Cout, K), (0, Kpad - K))   # tiny
    stats = torch.empty(2 * Cout, device=x.device, dtype=torch.float64) if training else None
    y = ops.linear(A, w2d, conv.bias, stats=stats, as_conv=True)
    y = ops.batchnorm(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, training=training, momentum=bn.momentum,
                      eps=bn.eps, relu=True, stats=stats)
    return y, (H + 2 * pd - R) // st + 1


class BasicBlock(nn.Module):
    """model_zoo/hrnet.py:28-58"""
    expansion = 1

    def __init__(self, inplanes, planes):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 3)
        self.bn1 = _bn(planes)
        self.conv2 = _conv(planes, planes, 3)
        self.bn2 = _bn(planes)

    def forward(self, x, N, H):
        tr = self.training
        out, xa = _first_conv_with_alias(x, self.conv1, self.bn1, N, H, tr)
        out, _ = conv_bn(out, self.conv2, self.bn2, N, H, tr, relu=True, res=xa)
        return out


class Bottleneck(nn.Module):
    """model_zoo/hrnet.py:61-100 (stride always 1 on this path)"""
    expansion = 4

    def __init__(self, inplanes, planes):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 1)
        self.bn1 = _bn(planes)
        self.conv2 = _conv(planes, planes, 3)
        self.bn2 = _bn(planes)
        self.conv3 = _conv(planes, planes * 4, 1)
        self.bn3 = _bn(planes * 4)
        self.downsample = None
        if inplanes != planes * 4:
            self.downsample = nn.Sequential(_conv(inplanes, planes * 4, 1), _bn(planes * 4))

    def forward(self, x, N, H):
        tr = self.training
        out, xa = _first_conv_with_alias(x, self.conv1, self.bn1, N, H, tr)
        out, _ = conv_bn(out, self.conv2, self.bn2, N, H, tr)
        idt = xa
        if self.downsample is not None:
            idt, _ = conv_bn(xa, self.downsample[0], self.downsample[1], N, H, tr, relu=False)
        out, _ = conv_bn(out, self.conv3, self.bn3, N, H, tr, relu=True, res=idt)
        return out


class HighResolutionModule(nn.Module):
    """model_zoo/hrnet.py:103-232: parallel branches of BasicBlocks + all-to-all fusion"""

    def __init__(self, channels, num_blocks):
        super().__init__()
        nb = len(channels)
        self.branches = nn.ModuleList([nn.Sequential(*[BasicBlock(c, c) for _ in range(num_blocks)]) for c in channels])
        self.fuse_layers = None
        if nb > 1:
            rows = []
            for i in range(nb):
                row = []
                for j in range(nb):
                    if j > i:        # 1x1 conv + BN (+ nearest x 2^(j-i), folded into the fuse-sum kernel)
                        row.append(nn.Sequential(_conv(channels[j], channels[i], 1), _bn(channels[i]),
                                                 nn.Upsample(scale_factor=2 ** (j - i), mode='nearest')))
                    elif j == i:
                        row.append(None)
                    else:            # i-j stride-2 3x3 convs; only the last one changes the channel count and has no ReLU
                        row.append(nn.Sequential(*[_cbr_seq(channels[j], channels[i] if k == i - j - 1 else channels[j], 3, 2,
                                                            relu=(k != i - j - 1)) for k in range(i - j)]))
                rows.append(nn.ModuleList(row))
            self.fuse_layers = nn.ModuleList(rows)

    def forward(self, xs, N, Hs):
        tr = self.training
        nb = len(xs)
        xs = list(xs)
        for i in range(nb):
            for blk in self.branches[i]:
                xs[i] = blk(xs[i], N, Hs[i])
        if nb == 1:
            return xs
        outs = []
        for i in range(nb):
            terms, factors = [], []
            for j in range(nb):
                fl = self.fuse_layers[i][j]
                if j == i:
                    terms.append(xs[j]); factors.append(1)
                elif j > i:
                    t, _ = conv_bn(xs[j], fl[0], fl[1], N, Hs[j], tr, relu=False)
                    terms.append(t); factors.append(2 ** (j - i))
                else:
                    t, h = xs[j], Hs[j]
                    for k, seq in enumerate(fl):
                        t, h = conv_bn(t, seq[0], seq[1], N, h, tr, relu=(k != len(fl) - 1))
                    terms.append(t); factors.append(1)
            outs.append(ops.fuse_sum(terms, factors, N, Hs[i], relu=True))
        return outs


class HighResolutionNet(nn.Module):
    """model_zoo/hrnet.py:235-527 with head_type 'none': returns the 4 branch maps [(x, H)] fine -> coarse"""

    def __init__(self, name, in_channels=3):
        super().__init__()
        (s1_blocks, s1_planes), stages = WIDTHS[name]
        self.conv1 = _conv(in_channels, 64, 3, 2)
        self.bn1 = _bn(64)
        self.conv2 = _conv(64, 64, 3, 2)
        self.bn2 = _bn(64)
        layer1 = [Bottleneck(64, s1_planes)] + [Bottleneck(4 * s1_planes, s1_planes) for _ in range(s1_blocks - 1)]
        self.layer1 = nn.Sequential(*layer1)
        pre = [4 * s1_planes]
        self.stage_channels = []
        for si, (modules, blocks, channels) in enumerate(stages):
            channels = list(channels)
            setattr(self, 'transition%d' % (si + 1), self._transition(pre, channels))
            setattr(self, 'stage%d' % (si + 2), nn.Sequential(*[HighResolutionModule(channels, blocks) for _ in range(modules)]))
            pre = channels
            self.stage_channels.append(channels)

    @staticmethod
    def _transition(pre, cur):
        """hrnet.py:410-444: same-resolution 3x3 conv when the width changes, stride-2 3x3 conv chains for new branches"""
        layers = []
        for i, c in enumerate(cur):
            if i < len(pre):
                layers.append(_cbr_seq(pre[i], c, 3) if c != pre[i] else None)
            else:
                n = i + 1 - len(pre)
                layers.append(nn.Sequential(*[_cbr_seq(pre[-1], c if j == n - 1 else pre[-1], 3, 2) for j in range(n)]))
        return nn.ModuleList(layers)

    def forward(self, x, N, H, image_needs_grad):
        tr = self.training
        x, H = stem_conv_bn(x, self.conv1, self.bn1, N, H, tr, image_needs_grad)
        x, H = conv_bn(x, self.conv2, self.bn2, N, H, tr)
        for blk in self.layer1:
            x = blk(x, N, H)
        ys, Hs = [x], [H]
        for si in range(3):
            trans = getattr(self, 'transition%d' % (si + 1))
            xs, hs = [], []
            for i, t in enumerate(trans):
                if i < len(ys):
                    if t is None:
                        xs.append(ys[i]); hs.append(Hs[i])
                    else:
                        y, h = conv_bn(ys[i], t[0], t[1], N, Hs[i], tr)
                        xs.append(y); hs.append(h)
                else:
                    y, h = ys[-1], Hs[-1]
                    for seq in t:
                        y, h = conv_bn(y, seq[0], seq[1], N, h, tr)
                    xs.append(y); hs.append(h)
            for mod in getattr(self, 'stage%d' % (si + 2)):
                xs = mod(xs, N, hs)
            ys, Hs = xs, hs
        return list(zip(ys, Hs))


def _hr_name(model_type):
    name = 'w' + model_type[model_type.find('hrnet') + 5:]
    if name not in WIDTHS:
        raise ValueError('no such HRnet: %r' % model_type)
    return name


class HRnet_encoder(nn.Module):
    """models/encoder.py:176-240"""

    def __init__(self, model_type, pretrained='', handNum=2, heatmapDim=21):
        super().__init__()
        self.hrnet = HighResolutionNet(_hr_name(model_type), in_channels=3)
        if pretrained and os.path.isfile(pretrained):      # encoder.py:187-194
            have = self.hrnet.state_dict()
            sd = {k: v for k, v in torch.load(pretrained, map_location='cpu').items() if k in have and 'classifier' not in k}
            self.hrnet.load_state_dict(sd, strict=False)
        self.fmaps_dim = list(self.hrnet.stage_channels[-1])[::-1]
        self.handNum = handNum
        tot = sum(self.fmaps_dim)
        self.hms_decoder = self._mask_decoder(tot, heatmapDim * handNum)
        self.dp_decoder = self._mask_decoder(tot, 1 + 3 * handNum)

    @staticmethod
    def _mask_decoder(c, out_dim):
        return nn.Sequential(_conv(c, c, 1, bias=True), nn.BatchNorm2d(c), nn.ReLU(inplace=True), _conv(c, out_dim, 1, bias=True))

    def forward(self, img):
        N, C, H, W = img.shape
        assert H == W
        if not self.training:
            ops.bn_fold_refresh(self)       # inference: fold every BatchNorm of the encoder for the convolution epilogues (one launch)
        x = ops.nchw_to_nhwc(img)
        ys = self.hrnet(x, N, H, img.requires_grad)
        H0 = ys[0][1]
        cat = ops.hr_concat([y for y, _ in ys], N, H0)
        outs = []
        for dec in (self.hms_decoder, self.dp_decoder):
            h, _ = conv_bn(cat, dec[0], dec[1], N, H0, self.training)
            outs.append(ops.conv2d(h, dec[3].weight, dec[3].bias, N, H0, H0))
        hms = ops.nhwc_to_nchw(outs[0], N, H0, H0)
        mask = ops.nhwc_to_nchw(outs[1], N, H0, H0, 0, 1).view(N, H0, H0)           # out[:, 0]   (encoder.py:235)
        dp = ops.nhwc_to_nchw(outs[1], N, H0, H0, 1, outs[1].shape[1] - 1)           # out[:, 1:]
        return hms, mask, dp, ys[::-1], None, None


class hrnet_mid(nn.Module):
    """models/encoder.py:243-352: per-level 1x1 (Conv -> ReLU -> BN) to the decoder width + the classification-style head
    (incre bottlenecks, stride-2 downsamp convs, 1x1 to 2048, global average) that produces the global feature."""

    def __init__(self, model_type, in_fmapDim, out_fmapDim):
        super().__init__()
        _hr_name(model_type)
        in_fmapDim = list(in_fmapDim)           # coarse -> fine (the reference reverses its argument in place, encoder.py:260)
        self.convs = nn.ModuleList([nn.Sequential(_conv(in_fmapDim[i], out_fmapDim[i], 1), nn.ReLU(inplace=True), nn.BatchNorm2d(out_fmapDim[i]))
                                    for i in range(len(out_fmapDim))])
        self.global_feature_dim = 2048
        self.fmaps_dim = list(out_fmapDim)
        fine_first = in_fmapDim[::-1]
        head = [32, 64, 128, 256]
        self.incre_modules = nn.ModuleList([nn.Sequential(Bottleneck(c, head[i])) for i, c in enumerate(fine_first)])
        self.downsamp_modules = nn.ModuleList([_cbr_seq(head[i] * 4, head[i + 1] * 4, 3, 2, bias=True) for i in range(len(fine_first) - 1)])
        self.final_layer = _cbr_seq(head[3] * 4, 2048, 1, bias=True)

    def get_info(self):
        return {'global_feature_dim': self.global_feature_dim, 'fmaps_dim': self.fmaps_dim}

    def forward(self, img_fmaps, hms_fmaps=None, dp_fmaps=None, N=None):
        tr = self.training
        from .model import _conv_relu_bn
        if not tr:
            ops.bn_fold_refresh(self)
        fmaps = [(_conv_relu_bn(x, seq[0], seq[2], N, H, H, tr), H) for (x, H), seq in zip(img_fmaps, self.convs)]
        rev = img_fmaps[::-1]
        y = self.incre_modules[0][0](rev[0][0], N, rev[0][1])
        for i, ds in enumerate(self.downsamp_modules):
            a = self.incre_modules[i + 1][0](rev[i + 1][0], N, rev[i + 1][1])
            b, h = conv_bn(y, ds[0], ds[1], N, rev[i][1], tr)
            y = ops.fuse_sum([a, b], [1, 1], N, h, relu=False)
        y, h = conv_bn(y, self.final_layer[0], self.final_layer[1], N, rev[-1][1], tr)
        return ops.global_avgpool(y, N, h * h), fmaps
