"""H100-native drop-in for the reference's `models.model.HandNET_GCN` (models/model.py:18-60).

Same constructor contract (`load_model(cfg)`), same forward signature and 4-tuple result structure, same
1093 state_dict keys (so released checkpoints load) -- but `forward` runs hand-written sm_90a kernels from
librih_b200.so through `renderih_b200.ops`.  torch.nn modules are used ONLY as parameter containers (their
own forward is never called); feature maps are NHWC row matrices [N*H*W, C], tokens are [B*V, F].
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .assets import load_model_assets
from .config import load_cfg

IMG_SIZE = 256  # dataset/dataset_utils.py:4


class GraphCSR:
    """Sparse rescaled Laplacian L (and L^T) on the device.  The reference densifies it (gcn.py:79-86) and calls
    torch.mm (gcn.py:54); here it stays CSR (<= 11 nnz per row) and feeds a fused SpMM + [x, Lx] interleave."""

    def __init__(self, L):
        import scipy.sparse as sp
        if isinstance(L, np.ndarray):
            L = sp.csr_matrix(L)
        L = sp.csr_matrix(L).astype(np.float32)
        L.sort_indices()
        LT = sp.csr_matrix(L.T)
        LT.sort_indices()
        self.V = L.shape[0]
        self._host = [np.asarray(L.indptr, np.int32), np.asarray(L.indices, np.int32), np.asarray(L.data, np.float32),
                      np.asarray(LT.indptr, np.int32), np.asarray(LT.indices, np.int32), np.asarray(LT.data, np.float32)]
        self.device = None

    def to(self, device):
        if self.device != device:
            t = [torch.from_numpy(a).to(device) for a in self._host]
            self.rowptr, self.col, self.val, self.rowptr_t, self.col_t, self.val_t = t
            self.device = device
        return self

    def dense(self):
        import scipy.sparse as sp
        return torch.from_numpy(sp.csr_matrix((self._host[2], self._host[1], self._host[0]), shape=(self.V, self.V)).toarray())


def _cl(conv):
    """Store a Conv2d weight channels_last so its memory is [Cout, R, S, Cin] (what the kernels read)."""
    conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
    return conv


# ============================================================================ encoder (models/encoder.py:21-173)
def _conv_bn(x, conv, bn, N, H, W, training, relu=True, res=None, alias_input=False):
    """torchvision order Conv -> BN -> (+res) -> ReLU.  alias_input: returns (y, Ho, x_alias) -- see ops.conv2d."""
    k = conv.kernel_size[0]
    fold = None if (training or alias_input or torch.is_grad_enabled() or conv.bias is not None) else bn.__dict__.get('_rih_fold')
    if fold is not None:     # inference: the BatchNorm (+ residual + ReLU) rides in the convolution's epilogue
        y = ops.conv2d_bn_eval(x, conv.weight, N, H, W, conv.stride[0], conv.padding[0], fold, order=0, relu=relu, res=res)
        return y, (H + 2 * conv.padding[0] - k) // conv.stride[0] + 1
    stats = torch.empty(2 * conv.out_channels, device=x.device, dtype=torch.float64) if training else None
    y = ops.conv2d(x, conv.weight, None, N, H, W, stride=conv.stride[0], pad=conv.padding[0], stats=stats, alias_input=alias_input)
    xa = None
    if alias_input:
        y, xa = y
    Ho = (H + 2 * conv.padding[0] - k) // conv.stride[0] + 1
    y = ops.batchnorm(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, res=res, training=training,
                      momentum=bn.momentum, eps=bn.eps, relu=relu, stats=stats)
    return (y, Ho, xa) if alias_input else (y, Ho)


def _conv_relu_bn(x, conv, bn, N, H, W, training):
    """repo order Conv -> ReLU -> BN (models/model_zoo/__init__.py:56-82, models/encoder.py:52-54)"""
    fold = None if (training or torch.is_grad_enabled() or conv.bias is not None) else bn.__dict__.get('_rih_fold')
    if fold is not None:
        return ops.conv2d_bn_eval(x, conv.weight, N, H, W, conv.stride[0], conv.padding[0], fold, order=1, relu=True)
    stats = torch.empty(2 * conv.out_channels, device=x.device, dtype=torch.float64) if training else None
    y = ops.conv2d(x, conv.weight, None, N, H, W, stride=conv.stride[0], pad=conv.padding[0], relu=True,
                   relu_masked_by_consumer=True, stats=stats)
    return ops.batchnorm(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, training=training,
                         momentum=bn.momentum, eps=bn.eps, relu=False, mask_input=True, stats=stats)


class ResNetSimple_decoder(nn.Module):
    """models/encoder.py:21-64"""

    def __init__(self, expansion=4, fDim=(256, 256, 256, 256), direction=('flat', 'up', 'up', 'up'), out_dim=3):
        super().__init__()
        self.models = nn.ModuleList()
        fDim = [512 * expansion] + list(fDim)
        self.direction = list(direction)
        for i, d in enumerate(direction):
            k = 1 if d == 'flat' else 3
            layers = []
            if d == 'up':
                layers.append(nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True))
            layers.append(_cl(nn.Conv2d(fDim[i], fDim[i + 1], kernel_size=k, stride=1, padding=k // 2, bias=False)))
            layers.append(nn.ReLU(inplace=True))
            layers.append(nn.BatchNorm2d(fDim[i + 1]))
            self.models.append(nn.Sequential(*layers))
        self.final_layer = _cl(nn.Conv2d(fDim[-1], out_dim, kernel_size=1, stride=1, padding=0))

    def stage(self, i, x, N, H):
        """Stage i of the reference's Sequential list (encoder.py:33-47): [bilinear x2] -> conv -> ReLU -> BN.  -> (x, H)"""
        seq = self.models[i]
        if self.direction[i] == 'up':
            x = ops.bilinear2x(x, N, H, H)
            H = 2 * H
            conv, bn = seq[1], seq[3]
        else:
            conv, bn = seq[0], seq[2]
        return _conv_relu_bn(x, conv, bn, N, H, H, self.training), H

    def head(self, x, N, H):
        return ops.conv2d(x, self.final_layer.weight, self.final_layer.bias, N, H, H)

    def forward(self, x, N, H):
        fmaps = []
        for i in range(len(self.models)):
            x, H = self.stage(i, x, N, H)
            fmaps.append((x, H))
        return self.head(x, N, H), fmaps, H


class ResNetSimple(nn.Module):
    """models/encoder.py:67-126 (torchvision trunk used as a parameter container only)"""

    def __init__(self, model_type='resnet50', fmapDim=(128, 128, 128, 128), handNum=2, heatmapDim=21, aux_heads=True):
        super().__init__()
        import torchvision.models as tvm
        assert model_type in ('resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152')       # models/encoder.py:74
        self.resnet = getattr(tvm, model_type)(weights=None)
        self.expansion = 1 if model_type in ('resnet18', 'resnet34') else 4                         # basic blocks vs bottlenecks
        for m in self.resnet.modules():
            if isinstance(m, nn.Conv2d):
                _cl(m)
        self.aux_heads = aux_heads      # False: common/myhand/encoder_lijun.py:62-104 (trunk only, returns the 4 feature maps)
        if aux_heads:
            self.hms_decoder = ResNetSimple_decoder(self.expansion, fmapDim, ('flat', 'up', 'up', 'up'), heatmapDim * handNum)
            self.dp_decoder = ResNetSimple_decoder(self.expansion, fmapDim, ('flat', 'up', 'up', 'up'), handNum + 3 * handNum)
        self.handNum = handNum

    def _stem(self, x, N, H, needs_input_grad):
        """conv1 7x7/2 (3 -> 64) + bn1 + ReLU.  With 3 input channels an implicit GEMM cannot be vectorised or fed by TMA, so
        (when the image needs no gradient) the input is im2col'ed once to 160-wide rows and the conv runs as a dense GEMM."""
        r = self.resnet
        conv, bn = r.conv1, r.bn1
        if needs_input_grad or not self.training:
            return _conv_bn(x, conv, bn, N, H, H, self.training)
        Cout, Cin, R, S = conv.weight.shape
        K, Kpad = R * S * Cin, (R * S * Cin + 31) // 32 * 32
        A = ops.im2col(x, N, H, H, R, S, conv.stride[0], conv.padding[0], Kpad)
        w2d = torch.nn.functional.pad(conv.weight.permute(0, 2, 3, 1).reshape(Cout, K), (0, Kpad - K))   # tiny (64 x 160)
        stats = torch.empty(2 * Cout, device=x.device, dtype=torch.float64)
        y = ops.linear(A, w2d, None, stats=stats, as_conv=True)
        y = ops.batchnorm(y, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, training=True, momentum=bn.momentum, eps=bn.eps,
                          relu=True, stats=stats)
        return y, (H + 2 * conv.padding[0] - R) // conv.stride[0] + 1

    def _bottleneck(self, blk, x, N, H):
        tr = self.training
        # the block input feeds conv1 AND the residual path: the residual path hangs off conv1's alias output, so its gradient is
        # accumulated by conv1's dgrad kernel instead of a separate add over the largest activations of the network
        fuse = tr and x.requires_grad
        if fuse:
            out, _, xa = _conv_bn(x, blk.conv1, blk.bn1, N, H, H, tr, alias_input=True)
        else:
            (out, _), xa = _conv_bn(x, blk.conv1, blk.bn1, N, H, H, tr), x
        out, Ho = _conv_bn(out, blk.conv2, blk.bn2, N, H, H, tr)
        if blk.downsample is not None:
            identity, _ = _conv_bn(xa, blk.downsample[0], blk.downsample[1], N, H, H, tr, relu=False)
        else:
            identity = xa
        out, _ = _conv_bn(out, blk.conv3, blk.bn3, N, Ho, Ho, tr, relu=True, res=identity)
        return out, Ho

    def _basic(self, blk, x, N, H):
        """torchvision BasicBlock (resnet18 / resnet34, models/encoder.py:75-80): conv3x3 -> BN -> ReLU -> conv3x3 -> BN, + identity
        (1x1 stride-2 conv + BN when the block down-samples), ReLU.  Same residual-gradient routing as the bottleneck."""
        tr = self.training
        fuse = tr and x.requires_grad
        if fuse:
            out, Ho, xa = _conv_bn(x, blk.conv1, blk.bn1, N, H, H, tr, alias_input=True)
        else:
            (out, Ho), xa = _conv_bn(x, blk.conv1, blk.bn1, N, H, H, tr), x
        if blk.downsample is not None:
            identity, _ = _conv_bn(xa, blk.downsample[0], blk.downsample[1], N, H, H, tr, relu=False)
        else:
            identity = xa
        out, _ = _conv_bn(out, blk.conv2, blk.bn2, N, Ho, Ho, tr, relu=True, res=identity)
        return out, Ho

    def trunk(self, img, fold_done=False):
        """stem + layer1..4 (encoder.py:107-118) -> [x1 (8x8), x2, x3, x4 (64x64)] as (NHWC rows, H) pairs."""
        N = img.shape[0]
        r = self.resnet
        if not self.training and not fold_done:
            ops.bn_fold_refresh(self)        # inference: one launch folds every BatchNorm of the encoder for the conv epilogues
        x, H = self.stem(img)
        feats = []
        for layer in (r.layer1, r.layer2, r.layer3, r.layer4):
            for blk in layer:
                x, H = self._bottleneck(blk, x, N, H) if self.expansion == 4 else self._basic(blk, x, N, H)
            # this layer's output gradient is complete exactly when every later layer / head has been back-propagated (train.TrainStep
            # starts the gradient all-reduce of those parameters then)
            ops.backward_marker(x, 'encoder.resnet.layer%d' % (len(feats) + 1))
            feats.append((x, H))
        x4, x3, x2, x1 = feats
        return [x1, x2, x3, x4]

    def stem(self, img):
        """conv1 + bn1 + ReLU + max-pool (encoder.py:107-110) in one of three forms: the implicit-GEMM stem_conv (tensor-core modes, 256 x 256
        images, no image gradient), _stem's im2col GEMM (no image gradient) or _conv_bn (the image needs a gradient).  -> (NHWC rows, H)"""
        N, C, H, W = img.shape
        assert H == W
        r = self.resnet
        if not img.requires_grad and ops.stem_supported(H, W):
            # conv1 straight from the NCHW image: zero-bordered NHWC4 copy + wgmma implicit GEMM (no im2col buffer), train and eval mode
            conv, bn = r.conv1, r.bn1
            fold = None if (self.training or torch.is_grad_enabled()) else bn.__dict__.get('_rih_fold')
            stats = torch.empty(2 * 64, device=img.device, dtype=torch.float64) if self.training else None
            x = ops.stem_conv(img, conv.weight, stats, fold)
            if fold is None:
                x = ops.batchnorm(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, tracked=bn.num_batches_tracked, training=self.training,
                                  momentum=bn.momentum, eps=bn.eps, relu=True, stats=stats)
            H = H // 2
        else:
            x = ops.nchw_to_nhwc(img)
            x, H = self._stem(x, N, H, img.requires_grad)
        x = ops.maxpool3x3s2(x, N, H, H)
        return x, (H - 1) // 2 + 1

    def aux_outputs(self, hms, out, N, Hh):
        """NHWC head outputs -> the NCHW hms / mask / dense maps of encoder.py:121-125."""
        return (ops.nhwc_to_nchw(hms, N, Hh, Hh), ops.nhwc_to_nchw(out, N, Hh, Hh, 0, self.handNum),
                ops.nhwc_to_nchw(out, N, Hh, Hh, self.handNum, out.shape[1] - self.handNum))

    def forward(self, img):
        N = img.shape[0]
        img_fmaps = self.trunk(img)
        if not self.aux_heads:
            return img_fmaps
        x1 = img_fmaps[0]
        hms, hms_fmaps, Hh = self.hms_decoder(x1[0], N, x1[1])
        out, dp_fmaps, _ = self.dp_decoder(x1[0], N, x1[1])
        hms, mask, dp = self.aux_outputs(hms, out, N, Hh)
        return hms, mask, dp, img_fmaps, hms_fmaps, dp_fmaps


class resnet_mid(nn.Module):
    """models/encoder.py:129-173"""

    def __init__(self, model_type='resnet50', in_fmapDim=(128, 128, 128, 128), out_fmapDim=(256, 256, 256, 256)):
        super().__init__()
        self.expansion = 1 if model_type in ('resnet18', 'resnet34') else 4                         # models/encoder.py:135-138
        self.img_fmaps_dim = [512 * self.expansion, 256 * self.expansion, 128 * self.expansion, 64 * self.expansion]
        self.convs = nn.ModuleList()
        for i in range(len(out_fmapDim)):
            inDim = 2 * in_fmapDim[i] + (self.img_fmaps_dim[i] if i > 0 else 0)
            self.convs.append(nn.Sequential(_cl(nn.Conv2d(inDim, out_fmapDim[i], kernel_size=1, bias=False)),
                                            nn.ReLU(inplace=True), nn.BatchNorm2d(out_fmapDim[i])))
        self.global_feature_dim = 512 * self.expansion
        self.fmaps_dim = list(out_fmapDim)

    def get_info(self):
        return {'global_feature_dim': self.global_feature_dim, 'fmaps_dim': self.fmaps_dim}

    def level(self, i, img_fmaps, hms_fmap, dp_fmap, N):
        """Level i of encoder.py:168-172: cat(hms fmap, dp fmap[, trunk feature]) -> conv1x1 -> ReLU -> BN.  -> (x, H)"""
        seq = self.convs[i]
        parts = [hms_fmap[0], dp_fmap[0]]
        if i > 0:
            parts.append(img_fmaps[i][0])
        H = hms_fmap[1]
        x = ops.concat_channels(parts)
        return _conv_relu_bn(x, seq[0], seq[2], N, H, H, self.training), H

    def forward(self, img_fmaps, hms_fmaps, dp_fmaps, N, fold_done=False):
        if not self.training and not fold_done:
            ops.bn_fold_refresh(self)
        x1, H1 = img_fmaps[0]
        global_feature = ops.global_avgpool(x1, N, H1 * H1)
        return global_feature, [self.level(i, img_fmaps, hms_fmaps[i], dp_fmaps[i], N) for i in range(len(self.convs))]


# ============================================================================ two-hand concurrency
# The forward pass overlaps independent work on five side streams per device; under CUDA-graph capture each fork / join becomes a pair
# of parallel graph branches, and autograd replays every backward node on its forward stream, so the backward pass overlaps the same way.
#   left, right   the two hands' sub-graphs of a DualGraph level, independent until `inter_attn` mixes them.  Each of their kernels
#                 (4032 ... 16128 token rows) fills well under half of the H100's 132 SMs.  High priority: the latency-bound hand
#                 branches are scheduled ahead of concurrent convolution work.
#   grid0, grid1  the image-grid encoders of a DualGraph level, which depend only on the image feature map.
#   aux           the convolution side of HandNET_GCN behind the trunk (heat-map / dense-pose stages, mid levels, aux heads).
_SIDE_STREAMS = {}


def _side_stream(device, role):
    key = (device.type, device.index, role)
    st = _SIDE_STREAMS.get(key)
    if st is None:
        st = _SIDE_STREAMS[key] = torch.cuda.Stream(device=device, priority=-1 if role in ('left', 'right') else 0)
        if role == 'aux':
            # cap the persistent grid of the tensor-core GEMMs / convolutions launched on it, leaving the other SMs to the token decoder
            # while the convolution pipeline runs.  72 was chosen on a 148-SM GPU and has not been tuned on the H100 (132 SMs).
            from ._lib import call
            call('rih_set_stream_cta_limit', st.cuda_stream, 72)
        elif role == 'left':
            try:      # parameters shared by both hands accumulate gradients from two streams by design; silence torch's advisory
                torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)
            except Exception:
                pass
    return st


def fork(device, role, fn):
    """Run fn() on side stream `role`, forked off the current stream, without joining.  -> handle for `join`."""
    s = _side_stream(device, role)
    s.wait_stream(torch.cuda.current_stream(device))
    ops.note_stream(s)
    with torch.cuda.stream(s):
        out = fn()
        ev = torch.cuda.Event()
        ev.record(s)
    return out, ev


def join(handle):
    """Make the current stream wait for a `fork` branch and hand over its result.  Every tensor in it is registered with the caching
    allocator as used by the joining stream (it was allocated on the side stream's pool)."""
    out, ev = handle
    cur = torch.cuda.current_stream()
    cur.wait_event(ev)
    _record_stream_tree(out, cur)
    return out


def run_hands(device, fn_left, fn_right):
    """(fn_left(), fn_right()) run concurrently on the two hand streams."""
    left = fork(device, 'left', fn_left)
    right = fork(device, 'right', fn_right)
    return join(left), join(right)


# ============================================================================ decoder blocks (models/model_attn/*.py)
class GCN_ResBlock(nn.Module):
    """models/model_attn/gcn.py:72-110 -- note norm1 is computed-and-discarded by the reference (103-104): it is a
    dead parameter here too (kept for state_dict parity, receives no gradient)."""

    def __init__(self, in_dim, out_dim, mid_dim, graph, graph_k, drop_out):
        super().__init__()
        assert graph_k == 2, 'Chebyshev order K=2 only (reference default utils/defaults.yaml:20)'
        self.graph = graph
        self.in_dim = in_dim
        self.norm1 = nn.LayerNorm(in_dim, eps=1e-6)
        self.fc1 = nn.Linear(in_dim * graph_k, mid_dim)
        self.norm2 = nn.LayerNorm(out_dim, eps=1e-6)
        self.fc2 = nn.Linear(mid_dim * graph_k, out_dim)
        self.shortcut = nn.Linear(in_dim, out_dim)
        self.norm3 = nn.LayerNorm(out_dim, eps=1e-6)
        self.p = drop_out

    def forward(self, x, B, V, relu_out):
        g = self.graph.to(x.device)
        p = self.p if self.training else 0.0
        if x.requires_grad and ops.FUSED['alias']:        # x feeds the graph convolution AND the shortcut: the shortcut hangs off the alias output (no autograd add)
            c, x = ops.cheb(x, g, B, V, alias_input=True)
        else:
            c = ops.cheb(x, g, B, V)
        x1 = ops.linear(c, self.fc1.weight, self.fc1.bias)
        x1 = ops.layernorm(x1, self.norm2.weight, self.norm2.bias, relu=True)
        c = ops.cheb(x1, g, B, V)
        x1 = ops.linear(c, self.fc2.weight, self.fc2.bias, p_drop=p)
        x2 = ops.linear(x, self.shortcut.weight, self.shortcut.bias)
        return ops.layernorm(x1, self.norm3.weight, self.norm3.bias, b=x2, relu=relu_out)


class MLP_GraphBlock(nn.Module):
    """`GCN_ResBlock` of the common/myhand default variant (common/myhand/model_attn/DualGraph_lijun.py:28-58): same parameter names,
    but no Laplacian -- relu(norm1(x)) -> fc1 -> relu(norm2) -> fc2 -> dropout, + shortcut(x), norm3."""

    def __init__(self, in_dim, out_dim, mid_dim, graph, graph_k, drop_out):
        super().__init__()
        self.in_dim = in_dim
        self.norm1 = nn.LayerNorm(in_dim, eps=1e-6)
        self.fc1 = nn.Linear(in_dim, mid_dim)
        self.norm2 = nn.LayerNorm(out_dim, eps=1e-6)
        self.fc2 = nn.Linear(mid_dim, out_dim)
        self.shortcut = nn.Linear(in_dim, out_dim)
        self.norm3 = nn.LayerNorm(out_dim, eps=1e-6)
        self.p = drop_out

    def forward(self, x, B, V, relu_out):
        p = self.p if self.training else 0.0
        if x.requires_grad and ops.FUSED['alias']:
            x1, x = ops.layernorm(x, self.norm1.weight, self.norm1.bias, relu=True, alias_input=True)
        else:
            x1 = ops.layernorm(x, self.norm1.weight, self.norm1.bias, relu=True)
        x1 = ops.linear(x1, self.fc1.weight, self.fc1.bias)
        x1 = ops.layernorm(x1, self.norm2.weight, self.norm2.bias, relu=True)
        x1 = ops.linear(x1, self.fc2.weight, self.fc2.bias, p_drop=p)
        x2 = ops.linear(x, self.shortcut.weight, self.shortcut.bias)
        return ops.layernorm(x1, self.norm3.weight, self.norm3.bias, b=x2, relu=relu_out)


class GraphLayer(nn.Module):
    """models/model_attn/gcn.py:113-138"""

    def __init__(self, in_dim, out_dim, graph, graph_k, graph_layer_num, drop_out, block_cls=None):
        super().__init__()
        block_cls = block_cls or GCN_ResBlock
        self.GCN_blocks = nn.ModuleList([block_cls(in_dim, out_dim, out_dim, graph, graph_k, drop_out)])
        for _ in range(graph_layer_num - 1):
            self.GCN_blocks.append(block_cls(out_dim, out_dim, out_dim, graph, graph_k, drop_out))

    def forward(self, x, B, V):
        n = len(self.GCN_blocks)
        for i, blk in enumerate(self.GCN_blocks):
            x = blk(x, B, V, relu_out=(i != n - 1))
        return x


def _ln_res(x, ln):
    """(LayerNorm(x), x') for a pre-LN residual block: x' is x routed through the LayerNorm node's alias output when gradients flow, so the
    residual branch's gradient is summed by the LN-backward kernel."""
    if x.requires_grad and ops.FUSED['alias']:
        return ops.layernorm(x, ln.weight, ln.bias, alias_input=True)
    return ops.layernorm(x, ln.weight, ln.bias), x


class MLP_res_block(nn.Module):
    """models/model_attn/self_attn.py:17-33"""

    def __init__(self, in_dim, hid_dim, dropout):
        super().__init__()
        self.layer_norm = nn.LayerNorm(in_dim, eps=1e-6)
        self.fc1 = nn.Linear(in_dim, hid_dim)
        self.fc2 = nn.Linear(hid_dim, in_dim)
        self.p = dropout

    def forward(self, x):
        p = self.p if self.training else 0.0
        h, x = _ln_res(x, self.layer_norm)
        h = ops.linear(h, self.fc1.weight, self.fc1.bias, relu=True, p_drop=p)
        return ops.linear(h, self.fc2.weight, self.fc2.bias, res=x, p_drop=p)


class SelfAttn(nn.Module):
    """models/model_attn/self_attn.py:36-85"""

    def __init__(self, f_dim, hid_dim=None, n_heads=4, dropout=0.1):
        super().__init__()
        d = f_dim // n_heads
        hid_dim = hid_dim or f_dim
        self.n_heads, self.f_dim = n_heads, f_dim
        self.w_qs = nn.Linear(f_dim, n_heads * d)
        self.w_ks = nn.Linear(f_dim, n_heads * d)
        self.w_vs = nn.Linear(f_dim, n_heads * d)
        self.layer_norm = nn.LayerNorm(f_dim, eps=1e-6)
        self.fc = nn.Linear(n_heads * d, f_dim)
        self.ff = MLP_res_block(f_dim, hid_dim, dropout)
        self.p = dropout

    def fused_param_groups(self):
        """Parameters the fused projections read as one stacked matrix / vector (train.FlatParams keeps them back to back)."""
        return [(self.w_qs.weight, self.w_ks.weight, self.w_vs.weight), (self.w_qs.bias, self.w_ks.bias, self.w_vs.bias)]

    def forward(self, x, B, S):
        p = self.p if self.training else 0.0
        xn, x = _ln_res(x, self.layer_norm)
        o = ops.attention_proj(xn, None, self.w_qs, self.w_ks, self.w_vs, B, self.n_heads, S, S, p_drop=p)     # ONE GEMM for q | k | v
        x = ops.linear(o, self.fc.weight, self.fc.bias, res=x, p_drop=p)
        return self.ff(x)

    def forward_query_subset(self, verts_f, extra_f, B, V, E):
        """SelfAttn over cat([verts (V), extra (E)]) keeping only the V vertex rows (img_attn.py:86-90):
        rows >= V are only ever used as keys/values, so Q / fc / MLP run on the vertex rows alone -- exact."""
        p = self.p if self.training else 0.0
        vn, verts_f = _ln_res(verts_f, self.layer_norm)
        en = ops.layernorm(extra_f, self.layer_norm.weight, self.layer_norm.bias)
        xn = ops.concat_rows(vn, en, B, V, E)
        o = ops.attention_proj(vn, xn, self.w_qs, self.w_ks, self.w_vs, B, self.n_heads, V, V + E, p_drop=p)   # q from the vertex rows, [k | v] as one GEMM
        x = ops.linear(o, self.fc.weight, self.fc.bias, res=verts_f, p_drop=p)
        return self.ff(x)


class img_feat_to_grid(nn.Module):
    """models/model_attn/img_attn.py:37-67"""

    def __init__(self, img_size, img_f_dim, grid_size, grid_f_dim, n_heads, dropout):
        super().__init__()
        self.img_size, self.grid_size, self.grid_f_dim = img_size, grid_size, grid_f_dim
        self.position_embeddings = nn.Embedding(grid_size * grid_size, grid_f_dim)
        patch = img_size // grid_size
        self.proj = _cl(nn.Conv2d(img_f_dim, grid_f_dim, kernel_size=patch, stride=patch))
        self.self_attn = SelfAttn(grid_f_dim, n_heads=n_heads, hid_dim=grid_f_dim, dropout=dropout)

    def patches(self, img, B):
        """The patch matrix both hands' grid encoders of a level read (kernel == stride: patches are disjoint, im2col is a pure re-ordering),
        or None when the convolution path is taken."""
        x, H = img
        p = self.proj.stride[0]
        if p > 1 and x.shape[1] % 4 == 0:
            return ops.patchify(x, B, H, H, p)
        return None

    def forward(self, img, B, patches=None):
        x, H = img
        assert H == self.img_size
        G = self.grid_size * self.grid_size
        p = self.proj.stride[0]
        if p > 1 and x.shape[1] % 4 == 0:
            # kernel == stride: patches are disjoint, so im2col is a pure re-ordering and the conv is ONE dense GEMM
            w2d = self.proj.weight.permute(0, 2, 3, 1).reshape(self.proj.weight.shape[0], -1)   # view of the channels_last weight
            P = patches if patches is not None else ops.patchify(x, B, H, H, p)
            g = ops.linear(P, w2d, self.proj.bias, relu=True)
        else:
            g = ops.conv2d(x, self.proj.weight, self.proj.bias, B, H, H, stride=p, pad=0, relu=True)
        g = ops.posemb(g, self.position_embeddings.weight, B, G, 1)
        return self.self_attn(g, B, G)


class img_attn(nn.Module):
    """models/model_attn/img_attn.py:70-92"""

    def __init__(self, verts_f_dim, img_f_dim, n_heads, dropout):
        super().__init__()
        self.fc = nn.Linear(img_f_dim, verts_f_dim)
        self.Attn = SelfAttn(verts_f_dim, n_heads=n_heads, hid_dim=verts_f_dim, dropout=dropout)

    def forward(self, verts_f, img_f, B, V, G):
        img_f = ops.linear(img_f, self.fc.weight, self.fc.bias)
        return self.Attn.forward_query_subset(verts_f, img_f, B, V, G)


class img_ex(nn.Module):
    """models/model_attn/img_attn.py:95-115"""

    def __init__(self, img_size, img_f_dim, grid_size, grid_f_dim, verts_f_dim, n_heads, dropout):
        super().__init__()
        self.encoder = img_feat_to_grid(img_size, img_f_dim, grid_size, grid_f_dim, n_heads, dropout)
        self.attn = img_attn(verts_f_dim, grid_f_dim, n_heads, dropout)
        self.G = grid_size * grid_size

    def forward(self, img, verts_f, B, V, grid=None):
        """grid: the image-grid tokens when they were already produced on another stream (`fork`)."""
        if grid is None:
            grid = self.encoder(img, B)
        return self.attn(verts_f, grid, B, V, self.G)


class inter_attn(nn.Module):
    """models/model_attn/inter_attn.py:36-123 (w_qs/w_ks/w_vs/fc are shared between the two hands)"""

    def __init__(self, f_dim, n_heads=4, dropout=0.1, variant='cross'):
        super().__init__()
        # 'cross': models/model_attn/inter_attn.py (each hand queries the OTHER hand's keys);
        # 'lijun': common/myhand/model_attn/inter_attn_lijun.py:79-91 (LayerNorm of Lf + Rf, own keys, the other hand's values)
        assert variant in ('cross', 'lijun')
        self.variant = variant
        self.L_self_attn_layer = SelfAttn(f_dim, n_heads=n_heads, hid_dim=f_dim, dropout=dropout)
        self.R_self_attn_layer = SelfAttn(f_dim, n_heads=n_heads, hid_dim=f_dim, dropout=dropout)
        d = f_dim // n_heads
        self.n_heads = n_heads
        self.w_qs = nn.Linear(f_dim, n_heads * d)
        self.w_ks = nn.Linear(f_dim, n_heads * d)
        self.w_vs = nn.Linear(f_dim, n_heads * d)
        self.fc = nn.Linear(n_heads * d, f_dim)
        self.layer_norm1 = nn.LayerNorm(f_dim, eps=1e-6)
        self.layer_norm2 = nn.LayerNorm(f_dim, eps=1e-6)
        self.ffL = MLP_res_block(f_dim, f_dim, dropout)
        self.ffR = MLP_res_block(f_dim, f_dim, dropout)
        self.p = dropout

    def fused_param_groups(self):
        return [(self.w_ks.weight, self.w_vs.weight), (self.w_ks.bias, self.w_vs.bias)]

    def forward(self, Lf, Rf, B, V):
        p = self.p if self.training else 0.0
        Lf, Rf = run_hands(Lf.device, lambda: self.L_self_attn_layer(Lf, B, V), lambda: self.R_self_attn_layer(Rf, B, V))
        lij = self.variant == 'lijun'
        H = self.n_heads
        if not lij:
            L2, Lf = _ln_res(Lf, self.layer_norm1)
            R2, Rf = _ln_res(Rf, self.layer_norm2)
            # each hand's queries against the OTHER hand's keys / values (shared weights): q and [k | v] projections as one GEMM each;
            # reference order of the two dropout1 draws: attn_R2L then attn_L2R (inter_attn.py:101-102)
            feat_R2L = ops.attention_proj(L2, R2, self.w_qs, self.w_ks, self.w_vs, B, H, V, V, p_drop=p)
            feat_L2R = ops.attention_proj(R2, L2, self.w_qs, self.w_ks, self.w_vs, B, H, V, V, p_drop=p)
            xR = ops.linear(feat_L2R, self.fc.weight, self.fc.bias, res=Rf, p_drop=p)
            xL = ops.linear(feat_R2L, self.fc.weight, self.fc.bias, res=Lf, p_drop=p)
            return run_hands(xL.device, lambda: self.ffL(xL), lambda: self.ffR(xR))
        L2 = ops.layernorm(Lf, self.layer_norm1.weight, self.layer_norm1.bias, b=Rf if lij else None)
        R2 = ops.layernorm(Rf, self.layer_norm2.weight, self.layer_norm2.bias, b=Lf if lij else None)
        Lq = ops.linear(L2, self.w_qs.weight, self.w_qs.bias)
        Lk = ops.linear(L2, self.w_ks.weight, self.w_ks.bias)
        Lv = ops.linear(L2, self.w_vs.weight, self.w_vs.bias)
        Rq = ops.linear(R2, self.w_qs.weight, self.w_qs.bias)
        Rk = ops.linear(R2, self.w_ks.weight, self.w_ks.bias)
        Rv = ops.linear(R2, self.w_vs.weight, self.w_vs.bias)
        # reference order of the two dropout1 draws: attn_R2L then attn_L2R (inter_attn.py:101-102)
        feat_R2L = ops.attention(Lq, Lk if lij else Rk, Rv, B, H, V, V, p_drop=p)
        feat_L2R = ops.attention(Rq, Rk if lij else Lk, Lv, B, H, V, V, p_drop=p)
        xR = ops.linear(feat_L2R, self.fc.weight, self.fc.bias, res=Rf, p_drop=p)
        xL = ops.linear(feat_R2L, self.fc.weight, self.fc.bias, res=Lf, p_drop=p)
        return run_hands(xL.device, lambda: self.ffL(xL), lambda: self.ffR(xR))


class DualGraphLayer(nn.Module):
    """models/model_attn/DualGraph.py:21-91 (the position-embedding add is fused into the caller's entry kernel)"""

    def __init__(self, verts_in_dim, verts_out_dim, graph_L, graph_R, graph_k, graph_layer_num, img_size, img_f_dim,
                 grid_size, grid_f_dim, n_heads, dropout, block_cls=None, attn_variant='cross'):
        super().__init__()
        self.verts_num = graph_L.V
        self.verts_in_dim = verts_in_dim
        self.position_embeddings = nn.Embedding(self.verts_num, verts_in_dim)
        self.graph_left = GraphLayer(verts_in_dim, verts_out_dim, graph_L, graph_k, graph_layer_num, dropout, block_cls)
        self.graph_right = GraphLayer(verts_in_dim, verts_out_dim, graph_R, graph_k, graph_layer_num, dropout, block_cls)
        self.img_ex_left = img_ex(img_size, img_f_dim, grid_size, grid_f_dim, verts_out_dim, n_heads, dropout)
        self.img_ex_right = img_ex(img_size, img_f_dim, grid_size, grid_f_dim, verts_out_dim, n_heads, dropout)
        self.attn = inter_attn(verts_out_dim, n_heads=n_heads, dropout=dropout, variant=attn_variant)

    def forward(self, Lf, Rf, img_f, B):
        """Lf/Rf already carry `+ position_embeddings` (added by the entry / upsample kernels)."""
        V = self.verts_num
        # the image-grid tokens (patch GEMM + position embedding + a 64-token SelfAttn, ~14 launches per hand) depend only on the feature map:
        # they start on their own streams now and run beside the 28-launch graph-convolution chains of the two hands
        gp = fork(Lf.device, 'grid0', lambda: self.img_ex_left.encoder.patches(img_f, B))      # one patch matrix per level, shared by both hands
        gl = fork(Lf.device, 'grid0', lambda: self.img_ex_left.encoder(img_f, B, patches=join(gp)))
        gr = fork(Lf.device, 'grid1', lambda: self.img_ex_right.encoder(img_f, B, patches=join(gp)))
        Lf, Rf = run_hands(Lf.device, lambda: self.img_ex_left(img_f, self.graph_left(Lf, B, V), B, V, grid=join(gl)),
                           lambda: self.img_ex_right(img_f, self.graph_right(Rf, B, V), B, V, grid=join(gr)))
        return self.attn(Lf, Rf, B, V)


class DualGraph(nn.Module):
    """models/model_attn/DualGraph.py:94-139"""

    def __init__(self, verts_in_dim, verts_out_dim, graphs_L, graphs_R, graph_k, graph_layer_num, img_size, img_f_dim,
                 grid_size, grid_f_dim, n_heads, dropout, block_cls=None, attn_variant='cross'):
        super().__init__()
        self.layers = nn.ModuleList()
        for i in range(len(verts_in_dim)):
            self.layers.append(DualGraphLayer(verts_in_dim[i], verts_out_dim[i], graphs_L[i], graphs_R[i], graph_k[i],
                                              graph_layer_num[i], img_size[i], img_f_dim[i], grid_size[i], grid_f_dim[i],
                                              n_heads, dropout, block_cls, attn_variant))

    def forward(self, Lf, Rf, img_f_list, B):
        for i, layer in enumerate(self.layers):
            if i > 0:  # graph_upsample(x, 2) of the previous level + this level's position embeddings
                emb = layer.position_embeddings.weight
                Lf = ops.posemb(Lf, emb, B, layer.verts_num, 2)
                Rf = ops.posemb(Rf, emb, B, layer.verts_num, 2)
            Lf, Rf = layer(Lf, Rf, img_f_list[i], B)
        return Lf, Rf


class GCN_vert_convert:
    """models/model_zoo/__init__.py:85-96 (index tensors are cached per device so the gathers are CUDA-graph capturable)"""

    def __init__(self, vertex_num, graph_perm_reverse, graph_perm):
        self.graph_perm_reverse = np.asarray(graph_perm_reverse)[:vertex_num]
        self.graph_perm = list(graph_perm)
        self._cache = {}

    def _idx(self, which, device):
        k = (which, str(device))
        if k not in self._cache:
            src = self.graph_perm if which == 'perm' else self.graph_perm_reverse
            self._cache[k] = torch.as_tensor(np.asarray(src, dtype=np.int64)).to(device)
        return self._cache[k]

    def vert_to_GCN(self, x):
        return x[:, self._idx('perm', x.device)]

    def GCN_to_vert(self, x):
        return x[:, self._idx('rev', x.device)]


class decoder(nn.Module):
    """models/decoder.py:29-174"""

    def __init__(self, global_feature_dim, f_in_Dim, f_out_Dim, gcn_in_dim, gcn_out_dim, graph_k, graph_layer_num,
                 left_graph_dict, right_graph_dict, vertex_num=778, dense_coor=None, num_attn_heads=4,
                 upsample_weight=None, dropout=0.05, block_cls=None, attn_variant='cross', mano_lists=True):
        super().__init__()
        self.mano_lists = mano_lists     # False: common/myhand/decoder_lijun_graph.py:316-320 returns empty MANO lists
        f_in_Dim = list(f_in_Dim)[:-1]
        gd = {'left': left_graph_dict, 'right': right_graph_dict}
        graph_L = {}
        for side in ('left', 'right'):
            Ls = list(gd[side]['coarsen_graphs_L'])
            Ls.reverse()                      # decoder.py:53-54 (we reverse a copy; the reference mutates the dict)
            graph_L[side] = Ls
        self.vNum_in = graph_L['left'][0].shape[0]
        self.vNum_out = graph_L['left'][2].shape[0]
        self.vNum_all = graph_L['left'][-1].shape[0]
        self.vNum_mano = vertex_num
        self.gf_dim = global_feature_dim
        self.gcn_in_dim, self.gcn_out_dim = list(gcn_in_dim), list(gcn_out_dim)
        self.register_buffer('dense_coor', torch.from_numpy(np.asarray(dense_coor)).float())
        self.converter = {s: GCN_vert_convert(self.vNum_mano, gd[s]['graph_perm_reverse'], gd[s]['graph_perm'])
                          for s in ('left', 'right')}
        graphs = {s: [GraphCSR(L) for L in graph_L[s][:3]] for s in ('left', 'right')}
        self.dual_gcn = DualGraph(self.gcn_in_dim, self.gcn_out_dim, graphs['left'], graphs['right'],
                                  [graph_k] * 3, [graph_layer_num] * 3, [8, 16, 32], f_in_Dim, [8, 8, 8], list(f_out_Dim),
                                  num_attn_heads, dropout, block_cls, attn_variant)
        self.gf_layer_left = nn.Sequential(nn.Linear(self.gf_dim, self.gcn_in_dim[0] - 3),
                                           nn.LayerNorm(self.gcn_in_dim[0] - 3, eps=1e-6))
        self.gf_layer_right = nn.Sequential(nn.Linear(self.gf_dim, self.gcn_in_dim[0] - 3),
                                            nn.LayerNorm(self.gcn_in_dim[0] - 3, eps=1e-6))
        self.unsample_layer = nn.Linear(self.vNum_out, self.vNum_mano, bias=False)
        self.coord_head = nn.Linear(self.gcn_out_dim[-1], 3)
        self.avg_head = nn.Linear(self.vNum_out, 1)
        self.params_head = nn.Linear(self.gcn_out_dim[-1], 3)
        if upsample_weight is not None:
            self.unsample_layer.weight.data.copy_(torch.as_tensor(upsample_weight).float())
        self._pe_cache = None
        self._idx_cache = {}

    def get_upsample_weight(self):
        return self.unsample_layer.weight.data

    def get_converter(self):
        return self.converter

    def _hand_pe(self):
        """decoder.get_hand_pe (decoder.py:118-126): input independent -> computed once per dense_coor version."""
        dc = self.dense_coor
        key = (dc._version, dc.device, dc.data_ptr())
        if self._pe_cache is None or self._pe_cache[0] != key:
            host = dc.detach().float().cpu() * 2 - 1
            pes = []
            for side in ('left', 'right'):
                pe = host[self.converter[side].graph_perm]                       # vert_to_GCN
                p = pe.shape[0] // self.vNum_in
                pe = pe.view(self.vNum_in, p, 3).mean(dim=1)                     # graph_avg_pool(p)
                pes.append(pe.contiguous().to(dc.device))
            self._pe_cache = (key, pes)
        return self._pe_cache[1]

    def _rev_idx(self, side, device):
        k = (side, device)
        if k not in self._idx_cache:
            self._idx_cache[k] = torch.from_numpy(np.asarray(self.converter[side].graph_perm_reverse, np.int32)).to(device)
        return self._idx_cache[k]

    def forward(self, x, fmaps):
        assert x.shape[1] == self.gf_dim
        fmaps = fmaps[:-1]
        B = x.shape[0]
        pel, per = self._hand_pe()
        emb0 = self.dual_gcn.layers[0].position_embeddings.weight
        feats = []
        for seq, pe in ((self.gf_layer_left, pel), (self.gf_layer_right, per)):
            g = ops.linear(x, seq[0].weight, seq[0].bias)
            g = ops.layernorm(g, seq[1].weight, seq[1].bias)
            feats.append(ops.gf_broadcast(g, pe, emb0, B, self.vNum_in))
        Lf, Rf = self.dual_gcn(feats[0], feats[1], fmaps, B)

        scale, trans2d, verts3d, verts2d = {}, {}, {}, {}
        result = {'verts3d': {}, 'verts2d': {}}
        def tail(f):
            return ops.decoder_tail(f, self.avg_head.weight.view(-1), self.avg_head.bias, self.params_head.weight, self.params_head.bias,
                                    self.coord_head.weight, self.coord_head.bias, self.unsample_layer.weight, B, self.vNum_out, float(IMG_SIZE))
        tails = run_hands(Lf.device, lambda: tail(Lf), lambda: tail(Rf))
        for side, (s, t, v3c, v2c, v3, v2) in zip(('left', 'right'), tails):
            scale[side], trans2d[side] = s, t
            verts3d[side], verts2d[side] = v3c, v2c
            result['verts3d'][side], result['verts2d'][side] = v3, v2
        paramsDict = {'scale': scale, 'trans2d': trans2d}
        handDictList = [{'verts3d': verts3d, 'verts2d': verts2d}]
        otherInfo = {'verts3d_MANO_list': {'left': [], 'right': []}, 'verts2d_MANO_list': {'left': [], 'right': []}}
        div = self.vNum_all // self.vNum_out
        for side in (('left', 'right') if self.mano_lists else ()):
            idx = self._rev_idx(side, x.device)
            otherInfo['verts3d_MANO_list'][side].append(ops.gather_rows(verts3d[side], idx, div))
            otherInfo['verts2d_MANO_list'][side].append(ops.gather_rows(verts2d[side], idx, div))
        return result, paramsDict, handDictList, otherInfo


# ============================================================================ model (models/model.py:18-60)
class HandNET_GCN(nn.Module):
    def __init__(self, encoder, mid_model, decoder):
        super().__init__()
        self.encoder = encoder
        self.mid_model = mid_model
        self.decoder = decoder

    def forward(self, img):
        if not (isinstance(img, torch.Tensor) and img.is_cuda):
            raise RuntimeError('renderih_b200.HandNET_GCN runs only on CUDA (sm_90a) tensors; there is no CPU fallback')
        if img.dtype != torch.float32:
            raise RuntimeError('renderih_b200.HandNET_GCN expects float32 images')
        ops.seed_state.begin_forward()
        if self.training:
            ops.seed_state.advance(img.device)
        N = img.shape[0]
        # inference: ONE launch folds every BatchNorm of the network into (scale, shift) vectors for the convolution epilogues
        fold_done = (not (self.encoder.training and self.mid_model.training)) and ops.bn_fold_refresh(self)
        if type(self.encoder) is ResNetSimple and self.encoder.aux_heads and type(self.mid_model) is resnet_mid:
            result, paramsDict, handDictList, otherInfo, hms, mask, dp = self._forward_pipelined(img, N, fold_done)
        else:
            hms, mask, dp, img_fmaps, hms_fmaps, dp_fmaps = self.encoder(img)
            global_feature, fmaps = self.mid_model(img_fmaps, hms_fmaps, dp_fmaps, N)
            result, paramsDict, handDictList, otherInfo = self.decoder(global_feature, fmaps)
        if hms is not None:
            otherInfo['hms'] = hms
        if mask is not None:
            otherInfo['mask'] = mask
        if dp is not None:
            otherInfo['dense'] = dp
        return result, paramsDict, handDictList, otherInfo


    def _forward_pipelined(self, img, N, fold_done=False):
        """Same arithmetic as encoder -> mid_model -> decoder, issued as two concurrent pipelines: everything behind the trunk on the
        convolution side (heat-map / dense-pose decoder stages at 8, 16, 32, 64 px, the mid 1x1 convs, the aux heads) runs on the aux stream
        and publishes each mid level with an event; the token decoder (main + hand streams) waits for level i only when DualGraph layer i
        starts.  DualGraph layer 1 overlaps the 16 px stage, layer 2 the 32 px stage, layer 3 the 64 px stage + heads, which nothing in the
        decoder reads.  autograd replays every node on its forward stream, so the backward pass is pipelined the same way."""
        enc, mid = self.encoder, self.mid_model
        img_fmaps = enc.trunk(img, fold_done)
        x1, H1 = img_fmaps[0]
        global_feature = ops.global_avgpool(x1, N, H1 * H1)
        fmaps = _StreamedFmaps()

        def conv_side():
            xh, xd, H = x1, x1, H1
            for i in range(len(mid.convs)):
                xh, Hn = enc.hms_decoder.stage(i, xh, N, H)
                xd, _ = enc.dp_decoder.stage(i, xd, N, H)
                H = Hn
                fmaps.publish(mid.level(i, img_fmaps, (xh, H), (xd, H), N))
            hms, mask, dp = enc.aux_outputs(enc.hms_decoder.head(xh, N, H), enc.dp_decoder.head(xd, N, H), N, H)
            return hms, mask, dp, list(fmaps)
        side = fork(img.device, 'aux', conv_side)
        out = self.decoder(global_feature, fmaps)
        hms, mask, dp, _ = join(side)
        return out + (hms, mask, dp)


def _record_stream_tree(obj, stream):
    if torch.is_tensor(obj):
        if obj.is_cuda:
            obj.record_stream(stream)
    elif isinstance(obj, dict):
        for v in obj.values():
            _record_stream_tree(v, stream)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _record_stream_tree(v, stream)


class _StreamedFmaps(list):
    """List of (feature map, H) pairs produced on another stream: the consuming stream waits for a level's event when that level is read."""

    def __init__(self, fmaps=(), events=()):
        super().__init__(fmaps)
        self.events = list(events)

    def publish(self, level):
        """Append a (feature map, H) level and record an event on the current (producing) stream."""
        ev = torch.cuda.Event()
        ev.record()
        self.append(level)
        self.events.append(ev)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return _StreamedFmaps(list.__getitem__(self, i), self.events[i])
        torch.cuda.current_stream().wait_event(self.events[i])
        return list.__getitem__(self, i)


def load_encoder(cfg):
    et = cfg.MODEL.ENCODER_TYPE
    if 'resnet' in et:
        enc = ResNetSimple(model_type=et, fmapDim=[128, 128, 128, 128], handNum=2, heatmapDim=21)
        mid = resnet_mid(model_type=et, in_fmapDim=[128, 128, 128, 128], out_fmapDim=cfg.MODEL.DECONV_DIMS)
        return enc, mid
    if 'hrnet' in et:                  # models/encoder.py:365-372
        from .hrnet import HRnet_encoder, hrnet_mid
        enc = HRnet_encoder(model_type=et, pretrained=getattr(cfg.MODEL, 'ENCODER_PRETRAIN_PATH', ''), handNum=2, heatmapDim=21)
        mid = hrnet_mid(model_type=et, in_fmapDim=enc.fmaps_dim, out_fmapDim=cfg.MODEL.DECONV_DIMS)
        return enc, mid
    raise NotImplementedError('encoder %r: only resnet18/34/50/101/152 and hrnet* encoders exist in the reference (models/encoder.py:355-374)' % et)


def load_decoder(cfg, encoder_info, assets=None, asset_root=None):
    a = assets if assets is not None else load_model_assets(cfg, asset_root)
    return decoder(global_feature_dim=encoder_info['global_feature_dim'], f_in_Dim=encoder_info['fmaps_dim'],
                   f_out_Dim=cfg.MODEL.IMG_DIMS, gcn_in_dim=cfg.MODEL.GCN_IN_DIM, gcn_out_dim=cfg.MODEL.GCN_OUT_DIM,
                   graph_k=cfg.MODEL.graph_k, graph_layer_num=cfg.MODEL.graph_layer_num, vertex_num=778,
                   dense_coor=a['dense_coor'], left_graph_dict=a['left_graph'], right_graph_dict=a['right_graph'],
                   num_attn_heads=4, upsample_weight=a['upsample'], dropout=cfg.TRAIN.dropout)


def load_model(cfg=None, assets=None, asset_root=None):
    """`models.model.load_model(cfg)` (models/model.py:40-60).  cfg: path | CfgNode-like | None (defaults)."""
    if cfg is None or isinstance(cfg, str):
        cfg = load_cfg(cfg)
    encoder, mid_model = load_encoder(cfg)
    dec = load_decoder(cfg, mid_model.get_info(), assets=assets, asset_root=asset_root)
    return HandNET_GCN(encoder, mid_model, dec)
