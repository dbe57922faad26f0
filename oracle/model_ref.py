"""CPU oracle: functional restatement of `models.model.HandNET_GCN.forward` (reference models/model.py:25-37).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Plain torch fp32 ops on a reference-layout state_dict, NCHW.
Pinned against the UNMODIFIED reference imported in the authoring container (oracle/make_golden.py writes
tests/golden/*.pt; tests/test_oracle_golden.py re-checks them on every run).  The reference's own tests hold no
golden vectors for this path (SURVEY.md section 4), so these self-generated fixtures are the only pin.

Every function cites the reference lines it follows.
"""
import numpy as np
import torch
import torch.nn.functional as F

IMG_SIZE = 256  # dataset/dataset_utils.py:4


def _bn(x, sd, pre, training, momentum=0.1, eps=1e-5):
    """nn.BatchNorm2d; in training mode batch statistics are used and running stats in `sd` are updated in place."""
    return F.batch_norm(x, sd[pre + '.running_mean'], sd[pre + '.running_var'], sd[pre + '.weight'], sd[pre + '.bias'],
                        training, momentum, eps)


def _ln(x, sd, pre):
    return F.layer_norm(x, (x.shape[-1],), sd[pre + '.weight'], sd[pre + '.bias'], 1e-6)


def _lin(x, sd, pre):
    return F.linear(x, sd[pre + '.weight'], sd.get(pre + '.bias'))


def _drop(x, p, training):
    return F.dropout(x, p, training) if (training and p > 0) else x


# ---------------------------------------------------------------- encoder: models/encoder.py:107-126 + torchvision Bottleneck
# `conv` (default F.conv2d, same signature) replaces every convolution of the encoder functions below, so that a test can run the
# same graph with convolutions in another arithmetic (e.g. fp64 products of TF32-rounded operands).
def _bottleneck(x, sd, pre, stride, has_ds, tr, conv=F.conv2d):
    out = F.relu(_bn(conv(x, sd[pre + '.conv1.weight']), sd, pre + '.bn1', tr))
    out = F.relu(_bn(conv(out, sd[pre + '.conv2.weight'], stride=stride, padding=1), sd, pre + '.bn2', tr))
    out = _bn(conv(out, sd[pre + '.conv3.weight']), sd, pre + '.bn3', tr)
    idt = x
    if has_ds:
        idt = _bn(conv(x, sd[pre + '.downsample.0.weight'], stride=stride), sd, pre + '.downsample.1', tr)
    return F.relu(out + idt)


def _simple_decoder(x, sd, pre, tr, conv=F.conv2d):
    """ResNetSimple_decoder.forward, models/encoder.py:58-64: flat 1x1 then 3x (bilinear x2, 3x3 conv, ReLU, BN)."""
    fmaps = []
    x = _bn(F.relu(conv(x, sd[pre + '.models.0.0.weight'])), sd, pre + '.models.0.2', tr)
    fmaps.append(x)
    for i in (1, 2, 3):
        x = F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True)
        x = _bn(F.relu(conv(x, sd['%s.models.%d.1.weight' % (pre, i)], padding=1)), sd, '%s.models.%d.3' % (pre, i), tr)
        fmaps.append(x)
    out = conv(x, sd[pre + '.final_layer.weight'], sd[pre + '.final_layer.bias'])
    return out, fmaps


def resnet_trunk(sd, img, tr, blocks=(3, 4, 6, 3), conv=F.conv2d):
    """torchvision ResNet-50 trunk as driven by ResNetSimple.forward (models/encoder.py:107-118 == common/myhand/encoder_lijun.py:91-104)"""
    p = 'encoder.resnet'
    x = F.relu(_bn(conv(img, sd[p + '.conv1.weight'], stride=2, padding=3), sd, p + '.bn1', tr))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    for li, nb in enumerate(blocks):
        for bi in range(nb):
            stride = 2 if (bi == 0 and li > 0) else 1
            x = _bottleneck(x, sd, '%s.layer%d.%d' % (p, li + 1, bi), stride, bi == 0, tr, conv=conv)
        feats.append(x)
    return feats[::-1]          # [x1 (8x8), x2, x3, x4 (64x64)]


def graph_mid_forward(sd, img_f, tr):
    """resnet_mid.forward of the myhand variant, common/myhand/encoder_lijun.py:140-146"""
    gf = F.adaptive_avg_pool2d(img_f[0], 1).flatten(1)
    return gf, [_bn(F.relu(F.conv2d(img_f[i], sd['mid_model.convs.%d.0.weight' % i])), sd, 'mid_model.convs.%d.2' % i, tr) for i in range(4)]


def encoder_forward(sd, img, tr, blocks=(3, 4, 6, 3), conv=F.conv2d):
    p = 'encoder.resnet'
    x = F.relu(_bn(conv(img, sd[p + '.conv1.weight'], stride=2, padding=3), sd, p + '.bn1', tr))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    for li, nb in enumerate(blocks):
        for bi in range(nb):
            stride = 2 if (bi == 0 and li > 0) else 1
            x = _bottleneck(x, sd, '%s.layer%d.%d' % (p, li + 1, bi), stride, bi == 0, tr, conv=conv)
        feats.append(x)
    x4, x3, x2, x1 = feats
    hms, hms_f = _simple_decoder(x1, sd, 'encoder.hms_decoder', tr, conv=conv)
    out, dp_f = _simple_decoder(x1, sd, 'encoder.dp_decoder', tr, conv=conv)
    return hms, out[:, :2], out[:, 2:], [x1, x2, x3, x4], hms_f, dp_f


def mid_forward(sd, img_f, hms_f, dp_f, tr, conv=F.conv2d):
    """resnet_mid.forward, models/encoder.py:165-173 (conv1x1 helper = Conv -> ReLU -> BN, model_zoo/__init__.py:56-62)"""
    gf = F.adaptive_avg_pool2d(img_f[0], 1).flatten(1)
    fmaps = []
    for i in range(4):
        x = torch.cat((hms_f[i], dp_f[i]), 1)
        if i > 0:
            x = torch.cat((x, img_f[i]), 1)
        fmaps.append(_bn(F.relu(conv(x, sd['mid_model.convs.%d.0.weight' % i])), sd, 'mid_model.convs.%d.2' % i, tr))
    return gf, fmaps


# ---------------------------------------------------------------- HRNet encoder: models/model_zoo/hrnet.py + models/encoder.py:176-352
def _count(sd, pre):
    """number of consecutive integer children `pre.0`, `pre.1`, ... present in the state dict"""
    n = 0
    while any(k.startswith('%s.%d.' % (pre, n)) for k in sd):
        n += 1
    return n


def _basic_block(x, sd, pre, tr, conv=F.conv2d):
    """BasicBlock.forward, model_zoo/hrnet.py:41-58 (branch blocks never carry a downsample: in == out channels)"""
    out = F.relu(_bn(conv(x, sd[pre + '.conv1.weight'], padding=1), sd, pre + '.bn1', tr))
    out = _bn(conv(out, sd[pre + '.conv2.weight'], padding=1), sd, pre + '.bn2', tr)
    return F.relu(out + x)


def _conv_bn_seq(x, sd, pre, tr, stride=1, relu=True):
    """nn.Sequential(Conv2d 3x3 (pre.0), BatchNorm2d (pre.1)[, ReLU]) as used by transitions / fuse layers / downsamp modules"""
    w = sd[pre + '.0.weight']
    y = _bn(F.conv2d(x, w, sd.get(pre + '.0.bias'), stride=stride, padding=w.shape[-1] // 2), sd, pre + '.1', tr)
    return F.relu(y) if relu else y


def _hr_module(xs, sd, pre, tr):
    """HighResolutionModule.forward, model_zoo/hrnet.py:215-232 (fuse layers built at :167-210)"""
    nb = len(xs)
    xs = list(xs)
    for i in range(nb):
        for b in range(_count(sd, '%s.branches.%d' % (pre, i))):
            xs[i] = _basic_block(xs[i], sd, '%s.branches.%d.%d' % (pre, i, b), tr)
    if nb == 1:
        return xs
    out = []
    for i in range(nb):
        y = None
        for j in range(nb):
            fp = '%s.fuse_layers.%d.%d' % (pre, i, j)
            if j == i:
                t = xs[j]
            elif j > i:      # 1x1 conv -> BN -> nearest upsample 2^(j-i)
                t = _bn(F.conv2d(xs[j], sd[fp + '.0.weight']), sd, fp + '.1', tr)
                t = F.interpolate(t, scale_factor=2 ** (j - i), mode='nearest')
            else:            # (i-j) stride-2 3x3 convs, ReLU on all but the last
                t = xs[j]
                for k in range(i - j):
                    t = _conv_bn_seq(t, sd, '%s.%d' % (fp, k), tr, stride=2, relu=(k != i - j - 1))
            y = t if y is None else y + t
        out.append(F.relu(y))
    return out


def hrnet_forward(sd, img, tr, p='encoder.hrnet'):
    """HighResolutionNet.forward (head_type 'none'), model_zoo/hrnet.py:493-527"""
    x = F.relu(_bn(F.conv2d(img, sd[p + '.conv1.weight'], stride=2, padding=1), sd, p + '.bn1', tr))
    x = F.relu(_bn(F.conv2d(x, sd[p + '.conv2.weight'], stride=2, padding=1), sd, p + '.bn2', tr))
    for b in range(_count(sd, p + '.layer1')):
        x = _bottleneck(x, sd, '%s.layer1.%d' % (p, b), 1, (p + '.layer1.%d.downsample.0.weight' % b) in sd, tr)
    ys = [x]
    for stage, trans in (('stage2', 'transition1'), ('stage3', 'transition2'), ('stage4', 'transition3')):
        nb = _count(sd, '%s.%s.0.branches' % (p, stage))
        xs = []
        for i in range(nb):
            tp = '%s.%s.%d' % (p, trans, i)
            if i < len(ys):
                # same-resolution transition: conv3x3+BN+ReLU when the channel count changes (transition1.0), else identity
                src = ys[i] if stage != 'stage2' else x
                xs.append(_conv_bn_seq(src, sd, tp, tr) if (tp + '.0.weight') in sd else src)
            else:
                t = ys[-1] if stage != 'stage2' else x
                for j in range(_count(sd, tp)):
                    t = _conv_bn_seq(t, sd, '%s.%d' % (tp, j), tr, stride=2)
                xs.append(t)
        for m in range(_count(sd, '%s.%s' % (p, stage))):
            xs = _hr_module(xs, sd, '%s.%s.%d' % (p, stage, m), tr)
        ys = xs
    return ys


def _mask_decoder(x, sd, pre, tr):
    """HRnet_encoder.mask_decoder, models/encoder.py:207-221: 1x1 conv (bias) -> BN -> ReLU -> 1x1 conv (bias)"""
    x = F.relu(_bn(F.conv2d(x, sd[pre + '.0.weight'], sd[pre + '.0.bias']), sd, pre + '.1', tr))
    return F.conv2d(x, sd[pre + '.3.weight'], sd[pre + '.3.bias'])


def hrnet_encoder_forward(sd, img, tr):
    """HRnet_encoder.forward, models/encoder.py:223-240"""
    ys = hrnet_forward(sd, img, tr)
    size = ys[0].shape[2:]
    x = torch.cat([ys[0]] + [F.interpolate(y, size=size, mode='bilinear', align_corners=True) for y in ys[1:]], 1)
    hms = _mask_decoder(x, sd, 'encoder.hms_decoder', tr)
    out = _mask_decoder(x, sd, 'encoder.dp_decoder', tr)
    return hms, out[:, 0], out[:, 1:], ys[::-1], None, None


def hrnet_mid_forward(sd, img_f, tr):
    """hrnet_mid.forward, models/encoder.py:333-352 (img_f is coarse -> fine; the head walks fine -> coarse)"""
    fmaps = [_bn(F.relu(F.conv2d(img_f[i], sd['mid_model.convs.%d.0.weight' % i])), sd, 'mid_model.convs.%d.2' % i, tr)
             for i in range(len(img_f))]
    rev = img_f[::-1]
    y = _bottleneck(rev[0], sd, 'mid_model.incre_modules.0.0', 1, True, tr)
    for i in range(len(rev) - 1):
        y = _bottleneck(rev[i + 1], sd, 'mid_model.incre_modules.%d.0' % (i + 1), 1, True, tr) + \
            _conv_bn_seq(y, sd, 'mid_model.downsamp_modules.%d' % i, tr, stride=2)
    y = F.relu(_bn(F.conv2d(y, sd['mid_model.final_layer.0.weight'], sd['mid_model.final_layer.0.bias']), sd, 'mid_model.final_layer.1', tr))
    return F.avg_pool2d(y, kernel_size=y.shape[2:]).view(y.shape[0], -1), fmaps


# ---------------------------------------------------------------- decoder blocks
def graph_conv_cheby(x, sd, pre, L, K=2):
    """models/model_attn/gcn.py:34-69 (dense Laplacian product, Fin x K interleave)"""
    B, V, Fin = x.shape
    x0 = x.permute(1, 2, 0).contiguous().view(V, Fin * B)
    xs = [x0]
    if K > 1:
        x1 = torch.mm(L, x0)
        xs.append(x1)
    for _ in range(2, K):
        x2 = 2 * torch.mm(L, x1) - x0
        xs.append(x2)
        x0, x1 = x1, x2
    xx = torch.stack(xs, 0).view(K, V, Fin, B).permute(3, 1, 2, 0).contiguous().view(B * V, Fin * K)
    return _lin(xx, sd, pre).view(B, V, -1)


def gcn_resblock(x, sd, pre, L, p, tr):
    """GCN_ResBlock.forward, gcn.py:99-110 -- relu(norm1(x)) is discarded by the reference (103-104)."""
    x1 = graph_conv_cheby(x, sd, pre + '.fc1', L)
    x1 = F.relu(_ln(x1, sd, pre + '.norm2'))
    x1 = graph_conv_cheby(x1, sd, pre + '.fc2', L)
    x1 = _drop(x1, p, tr)
    x2 = _lin(x, sd, pre + '.shortcut')
    return _ln(x1 + x2, sd, pre + '.norm3')


def mlp_graph_block(x, sd, pre, p, tr):
    """GCN_ResBlock.forward of the myhand variant (no Laplacian), common/myhand/model_attn/DualGraph_lijun.py:46-58"""
    x1 = _lin(F.relu(_ln(x, sd, pre + '.norm1')), sd, pre + '.fc1')
    x1 = _lin(F.relu(_ln(x1, sd, pre + '.norm2')), sd, pre + '.fc2')
    x1 = _drop(x1, p, tr)
    return _ln(x1 + _lin(x, sd, pre + '.shortcut'), sd, pre + '.norm3')


def graph_layer(x, sd, pre, L, p, tr, n=4, variant='intaghand'):
    """GraphLayer.forward, gcn.py:132-138 (== DualGraph_lijun.py:82-88)"""
    for i in range(n):
        if variant == 'graph':
            x = mlp_graph_block(x, sd, '%s.GCN_blocks.%d' % (pre, i), p, tr)
        else:
            x = gcn_resblock(x, sd, '%s.GCN_blocks.%d' % (pre, i), L, p, tr)
        if i != n - 1:
            x = F.relu(x)
    return x


def mlp_res(x, sd, pre, p, tr):
    """MLP_res_block.forward, self_attn.py:27-33"""
    h = _ln(x, sd, pre + '.layer_norm')
    h = _drop(F.relu(_lin(h, sd, pre + '.fc1')), p, tr)
    return x + _drop(_lin(h, sd, pre + '.fc2'), p, tr)


def _heads(t, B, H):
    return t.view(B, -1, H, t.shape[-1] // H).transpose(1, 2)


def self_attn(x, sd, pre, p, tr, H=4):
    """SelfAttn.forward, self_attn.py:63-85"""
    B, V, f = x.shape
    xn = _ln(x, sd, pre + '.layer_norm')
    q, k, v = (_heads(_lin(xn, sd, pre + n), B, H) for n in ('.w_qs', '.w_ks', '.w_vs'))
    attn = torch.matmul(q, k.transpose(-1, -2)) / (f // H) ** 0.5
    attn = _drop(F.softmax(attn, -1), p, tr)
    out = torch.matmul(attn, v).transpose(1, 2).contiguous().view(B, V, -1)
    x = x + _drop(_lin(out, sd, pre + '.fc'), p, tr)
    return mlp_res(x, sd, pre + '.ff', p, tr)


def img_ex(img, verts_f, sd, pre, p, tr):
    """img_ex.forward, img_attn.py:111-115 -> img_feat_to_grid (51-67) + img_attn (79-92)"""
    B = img.shape[0]
    w = sd[pre + '.encoder.proj.weight']
    g = F.relu(F.conv2d(img, w, sd[pre + '.encoder.proj.bias'], stride=w.shape[-1]))
    g = g.view(B, g.shape[1], -1).transpose(-1, -2) + sd[pre + '.encoder.position_embeddings.weight'][None]
    g = self_attn(g, sd, pre + '.encoder.self_attn', p, tr)
    V = verts_f.shape[1]
    x = torch.cat([verts_f, _lin(g, sd, pre + '.attn.fc')], 1)
    return self_attn(x, sd, pre + '.attn.Attn', p, tr)[:, :V]


def inter_attn(Lf, Rf, sd, pre, p, tr, H=4, variant='intaghand'):
    """inter_attn.forward, inter_attn.py:73-123; variant 'graph' = common/myhand/model_attn/inter_attn_lijun.py:73-123 (lines 79-80, 90-91 differ)"""
    Lf = self_attn(Lf, sd, pre + '.L_self_attn_layer', p, tr)
    Rf = self_attn(Rf, sd, pre + '.R_self_attn_layer', p, tr)
    B, V, f = Lf.shape
    if variant == 'graph':
        L2, R2 = _ln(Lf + Rf, sd, pre + '.layer_norm1'), _ln(Rf + Lf, sd, pre + '.layer_norm2')
    else:
        L2, R2 = _ln(Lf, sd, pre + '.layer_norm1'), _ln(Rf, sd, pre + '.layer_norm2')
    Lq, Lk, Lv = (_heads(_lin(L2, sd, pre + n), B, H) for n in ('.w_qs', '.w_ks', '.w_vs'))
    Rq, Rk, Rv = (_heads(_lin(R2, sd, pre + n), B, H) for n in ('.w_qs', '.w_ks', '.w_vs'))
    nrm = (f // H) ** 0.5
    kL, kR = (Lk, Rk) if variant == 'graph' else (Rk, Lk)      # keys paired with Lq / Rq
    a_R2L = _drop(F.softmax(torch.matmul(Lq, kL.transpose(-1, -2)) / nrm, -1), p, tr)
    a_L2R = _drop(F.softmax(torch.matmul(Rq, kR.transpose(-1, -2)) / nrm, -1), p, tr)
    f_L2R = torch.matmul(a_L2R, Lv).transpose(1, 2).contiguous().view(B, V, -1)
    f_R2L = torch.matmul(a_R2L, Rv).transpose(1, 2).contiguous().view(B, V, -1)
    f_L2R = _drop(_lin(f_L2R, sd, pre + '.fc'), p, tr)
    f_R2L = _drop(_lin(f_R2L, sd, pre + '.fc'), p, tr)
    return mlp_res(Lf + f_R2L, sd, pre + '.ffL', p, tr), mlp_res(Rf + f_L2R, sd, pre + '.ffR', p, tr)


def graph_upsample(x, p):
    """DualGraph.py:11-18 (nearest xp on the vertex axis)"""
    return x.repeat_interleave(p, dim=1) if p > 1 else x


def projection_batch(scale, trans2d, label3d, img_size=IMG_SIZE):
    """utils/manoutils.py:26-44"""
    scale = (scale * img_size)[:, None, None]
    trans2d = (trans2d * img_size / 2 + img_size / 2)[:, None]
    return scale * label3d[..., :2] + trans2d


def prepare_assets(assets):
    """Dense Laplacians of the 3 decoder levels (gcn.py:79-86) + permutations, from the raw asset dicts."""
    out = {}
    for side in ('left', 'right'):
        g = assets[side + '_graph']
        Ls = list(g['coarsen_graphs_L'])[::-1]           # decoder.py:53-54
        out[side] = {
            'L': [torch.from_numpy(np.asarray(L.todense() if hasattr(L, 'todense') else L, dtype=np.float32)) for L in Ls[:3]],
            'perm': [int(v) for v in g['graph_perm']],
            'perm_rev': np.asarray(g['graph_perm_reverse'])[:778],
            'vNum_all': Ls[-1].shape[0],
        }
    return out


def decoder_forward(sd, A, gf, fmaps, p, tr, variant='intaghand'):
    """decoder.forward, models/decoder.py:128-174; variant 'graph' = common/myhand/decoder_lijun_graph.py:279-320"""
    fmaps = fmaps[:-1]
    B = gf.shape[0]
    dc = sd['decoder.dense_coor'][None].repeat(B, 1, 1) * 2 - 1
    feats = {}
    for side, name in (('left', 'decoder.gf_layer_left'), ('right', 'decoder.gf_layer_right')):
        pe = dc[:, A[side]['perm']]                                        # vert_to_GCN
        pe = F.avg_pool1d(pe.permute(0, 2, 1), pe.shape[1] // 63).permute(0, 2, 1)   # graph_avg_pool
        g = _ln(_lin(gf, sd, name + '.0'), sd, name + '.1')
        feats[side] = torch.cat([g[:, None].repeat(1, 63, 1), pe], -1)
    Lf, Rf = feats['left'], feats['right']
    for i in range(3):
        pre = 'decoder.dual_gcn.layers.%d' % i
        emb = sd[pre + '.position_embeddings.weight'][None]
        Lf, Rf = Lf + emb, Rf + emb
        Lf = graph_layer(Lf, sd, pre + '.graph_left', A['left']['L'][i], p, tr, variant=variant)
        Rf = graph_layer(Rf, sd, pre + '.graph_right', A['right']['L'][i], p, tr, variant=variant)
        Lf = img_ex(fmaps[i], Lf, sd, pre + '.img_ex_left', p, tr)
        Rf = img_ex(fmaps[i], Rf, sd, pre + '.img_ex_right', p, tr)
        Lf, Rf = inter_attn(Lf, Rf, sd, pre + '.attn', p, tr, variant=variant)
        if i != 2:
            Lf, Rf = graph_upsample(Lf, 2), graph_upsample(Rf, 2)
    scale, trans2d, v3, v2 = {}, {}, {}, {}
    result = {'verts3d': {}, 'verts2d': {}}
    for side, f in (('left', Lf), ('right', Rf)):
        t = _lin(f.transpose(-1, -2), sd, 'decoder.avg_head')[..., 0]
        t = _lin(t, sd, 'decoder.params_head')
        scale[side], trans2d[side] = t[:, 0], t[:, 1:]
        v3[side] = _lin(f, sd, 'decoder.coord_head')
        v2[side] = projection_batch(scale[side], trans2d[side], v3[side])
        up = F.linear(v3[side].transpose(1, 2), sd['decoder.unsample_layer.weight']).transpose(1, 2)
        result['verts3d'][side] = up
        result['verts2d'][side] = projection_batch(scale[side], trans2d[side], up)
    other = {'verts3d_MANO_list': {'left': [], 'right': []}, 'verts2d_MANO_list': {'left': [], 'right': []}}
    for side in (('left', 'right') if variant != 'graph' else ()):
        pr, va = A[side]['perm_rev'], A[side]['vNum_all']
        other['verts3d_MANO_list'][side].append(graph_upsample(v3[side], va // v3[side].shape[1])[:, pr])
        other['verts2d_MANO_list'][side].append(graph_upsample(v2[side], va // v2[side].shape[1])[:, pr])
    return result, {'scale': scale, 'trans2d': trans2d}, [{'verts3d': v3, 'verts2d': v2}], other


# ---------------------------------------------------------------- 'newgraph' MANO tail: common/myhand/decoder_lijun_mano.py:26-58, 238-305
def _mlp_hardswish(x, sd, pre, n_lin, act_final):
    """make_linear_layers (decoder_lijun_mano.py:70-81): Linear (+ Hardswish except, optionally, after the last)"""
    idx = 0
    for i in range(n_lin):
        x = _lin(x, sd, '%s.%d' % (pre, idx))
        idx += 1
        if i < n_lin - 1 or act_final:
            x = F.hardswish(x)
            idx += 1
    return x


def rot6d_to_rotmat(x):
    """ParamRegressor.rot6d_to_rotmat, decoder_lijun_mano.py:36-43"""
    x = x.view(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    b1 = F.normalize(a1)
    b2 = F.normalize(a2 - torch.einsum('bi,bi->b', b1, a2).unsqueeze(-1) * b1)
    return torch.stack((b1, b2, torch.linalg.cross(b1, b2, dim=-1)), dim=-1)


def rotation_matrix_to_angle_axis(R):
    """common/myhand/utils/comm.py:176-200 (3x3 input path) = rotation_matrix_to_quaternion (:250-324) then quaternion_to_angle_axis (:203-247)"""
    rt = R.transpose(1, 2)
    m22 = rt[:, 2, 2] < 1e-6
    m01 = rt[:, 0, 0] > rt[:, 1, 1]
    m0n1 = rt[:, 0, 0] < -rt[:, 1, 1]
    t = [1 + rt[:, 0, 0] - rt[:, 1, 1] - rt[:, 2, 2], 1 - rt[:, 0, 0] + rt[:, 1, 1] - rt[:, 2, 2],
         1 - rt[:, 0, 0] - rt[:, 1, 1] + rt[:, 2, 2], 1 + rt[:, 0, 0] + rt[:, 1, 1] + rt[:, 2, 2]]
    q = [torch.stack([rt[:, 1, 2] - rt[:, 2, 1], t[0], rt[:, 0, 1] + rt[:, 1, 0], rt[:, 2, 0] + rt[:, 0, 2]], -1),
         torch.stack([rt[:, 2, 0] - rt[:, 0, 2], rt[:, 0, 1] + rt[:, 1, 0], t[1], rt[:, 1, 2] + rt[:, 2, 1]], -1),
         torch.stack([rt[:, 0, 1] - rt[:, 1, 0], rt[:, 2, 0] + rt[:, 0, 2], rt[:, 1, 2] + rt[:, 2, 1], t[2]], -1),
         torch.stack([t[3], rt[:, 1, 2] - rt[:, 2, 1], rt[:, 2, 0] - rt[:, 0, 2], rt[:, 0, 1] - rt[:, 1, 0]], -1)]
    masks = [m22 & m01, m22 & ~m01, ~m22 & m0n1, ~m22 & ~m0n1]
    masks = [mk.view(-1, 1).type_as(q[0]) for mk in masks]
    quat = sum(qi * mk for qi, mk in zip(q, masks))
    quat = quat / torch.sqrt(sum(ti.view(-1, 1) * mk for ti, mk in zip(t, masks))) * 0.5
    v = quat[:, 1:]
    sin2 = (v * v).sum(-1)
    sin_t, cos_t = torch.sqrt(sin2), quat[:, 0]
    two_theta = 2.0 * torch.where(cos_t < 0.0, torch.atan2(-sin_t, -cos_t), torch.atan2(sin_t, cos_t))
    k = torch.where(sin2 > 0.0, two_theta / sin_t, 2.0 * torch.ones_like(sin_t))
    aa = v * k.unsqueeze(-1)
    return torch.where(torch.isnan(aa), torch.zeros_like(aa), aa)


def _rodrigues_t(axis):
    """rodrigues_batch, common/utils/manolayer.py:32-48"""
    angle = torch.norm(axis, p=2, dim=1, keepdim=True) + 1e-8
    u = axis / angle
    L = torch.zeros((axis.shape[0], 3, 3), dtype=axis.dtype)
    L[:, 2, 1] = u[:, 0]; L[:, 1, 2] = -u[:, 0]
    L[:, 0, 2] = u[:, 1]; L[:, 2, 0] = -u[:, 1]
    L[:, 1, 0] = u[:, 2]; L[:, 0, 1] = -u[:, 2]
    return torch.eye(3, dtype=axis.dtype)[None] + torch.sin(angle)[..., None] * L + (1 - torch.cos(angle))[..., None] * L.bmm(L)


def newgraph_tail(sd, A, base_out, img_size=IMG_SIZE):
    """decoder.forward of the 'newgraph' variant after the shared graph part, decoder_lijun_mano.py:238-305.  A['mano'][side]: MANO dict
    (left shapedirs already flipped as in :171-173); A['mano_jr21'][side]: MANO.joint_regressor_torch (common/utils/mano.py:48-79)."""
    from . import mano_ref
    res0, params, hlist, _ = base_out
    scale, trans2d = params['scale'], params['trans2d']
    up = res0['verts3d']
    result = {'verts3d': {}, 'verts2d': {}, 'v3d_left': up['left'], 'v3d_right': up['right']}
    j3d = {s: torch.einsum('bik,ji->bjk', up[s], A['mano_jr21'][s]) for s in ('left', 'right')}
    root_rel = j3d['right'][:, 0] - j3d['left'][:, 0]
    pred, sl = {}, {}
    for s in ('left', 'right'):
        B = up[s].shape[0]
        feat = _mlp_hardswish(up[s].reshape(B, -1), sd, 'decoder.param_regressor.fc', 2, True)
        rotmat = rot6d_to_rotmat(_mlp_hardswish(feat, sd, 'decoder.param_regressor.fc_pose', 2, False))
        pose = rotation_matrix_to_angle_axis(rotmat).reshape(B, -1)
        shape = torch.tanh(_mlp_hardswish(feat, sd, 'decoder.param_regressor.fc_shape', 2, False)) * 3
        v, j = mano_ref.mano_forward_torch(A['mano'][s], _rodrigues_t(pose[:, :3]), pose[:, 3:], shape, use_pca=True, center_idx=None)
        v, j = v * 1000 / 1000, j * 1000 / 1000                                  # common/utils/manolayer.py:323-325 then :255-256
        v = v - j[:, 0:1]
        sl[s] = (0.095 / torch.linalg.norm(j[:, 9:10] - j[:, 0:1], dim=-1)).reshape(-1, 1, 1)
        v = v * sl[s]
        pred[s] = {'verts3d': v, 'joints3d': j, 'mano_pose': pose, 'mano_shape': shape}
        result['verts2d'][s] = projection_batch(scale[s], trans2d[s], v, img_size)
    result['verts3d']['left'] = pred['left']['verts3d']
    result['verts3d']['right'] = pred['right']['verts3d'] + root_rel.reshape(-1, 1, 3)
    other = {'length': (sl['left'] + sl['right']) / 2, 'root_rel': root_rel, 'verts3d_MANO_list': pred, 'verts2d_MANO_list': {'left': [], 'right': []}}
    params = {'scale': scale, 'trans2d': trans2d, 'scalelength_left': sl['left'], 'scalelength_right': sl['right'], 'root_rel': root_rel}
    return result, params, hlist, other


def model_forward(sd, assets_prepared, img, training=False, dropout=0.0):
    """HandNET_GCN.forward, models/model.py:25-37.  `sd` maps reference state_dict keys to tensors (BN running
    statistics are updated in place when training=True, exactly like nn.BatchNorm2d)."""
    if 'encoder.resnet.conv1.weight' in sd and 'encoder.hms_decoder.final_layer.weight' not in sd:
        # the common/myhand "graph" model (lijun_model_graph.py:27-34): trunk -> mid -> decoder, no auxiliary maps
        gf, fmaps = graph_mid_forward(sd, resnet_trunk(sd, img, training), training)
        out = decoder_forward(sd, assets_prepared, gf, fmaps, dropout, training, variant='graph')
        if 'decoder.param_regressor.fc.0.weight' in sd:      # 'newgraph': lijun_model_newgraph.py + decoder_lijun_mano.py
            out = newgraph_tail(sd, assets_prepared, out)
        return out
    if 'encoder.hrnet.conv1.weight' in sd:      # ENCODER_TYPE: hrnet* (models/encoder.py:365-372)
        hms, mask, dp, img_f, _, _ = hrnet_encoder_forward(sd, img, training)
        gf, fmaps = hrnet_mid_forward(sd, img_f, training)
    else:
        hms, mask, dp, img_f, hms_f, dp_f = encoder_forward(sd, img, training)
        gf, fmaps = mid_forward(sd, img_f, hms_f, dp_f, training)
    result, params, hlist, other = decoder_forward(sd, assets_prepared, gf, fmaps, dropout, training)
    other['hms'], other['mask'], other['dense'] = hms, mask, dp
    return result, params, hlist, other


# ---------------------------------------------------------------- loss: core/Loss.py:20-277 (calc_loss_GCN), epoch < NORM_EPOCH
def make_joint_regressor(J_regressor16):
    """GraphLoss.process_J_regressor, core/Loss.py:38-53"""
    J = J_regressor16.clone().float()
    tips = torch.zeros(5, J.shape[1])
    for i, v in enumerate((745, 317, 444, 556, 673)):
        tips[i, v] = 1.0
    J = torch.cat([J, tips], 0)
    order = [0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20]
    return J[order].contiguous()


def _edges(v, faces):
    e = v[:, faces]
    return torch.stack([e[:, :, 0] - e[:, :, 1], e[:, :, 1] - e[:, :, 2], e[:, :, 2] - e[:, :, 0]], 2)


def graph_loss_side(J21, faces, perm, v3d_gt, v2d_gt, v3d_pred, v2d_pred, v3dList, v2dList, img_size=IMG_SIZE, level=5):
    """GraphLoss.calc_loss, core/Loss.py:128-162 + calc_mano_loss 103-115"""
    sl1, mse = F.smooth_l1_loss, F.mse_loss
    d = {}
    d['vert2d_loss'] = mse(v2d_pred / img_size * 2 - 1, v2d_gt / img_size * 2 - 1)
    d['vert3d_loss'] = sl1(v3d_pred, v3d_gt)
    d['joint_loss'] = sl1(torch.matmul(J21, v3d_pred), torch.matmul(J21, v3d_gt))
    eg, ep = _edges(v3d_gt, faces), _edges(v3d_pred, faces)
    n_gt = F.normalize(torch.cross(eg[:, :, 0], eg[:, :, 1], dim=-1), dim=-1).unsqueeze(2)
    t = torch.sum(F.normalize(ep, dim=-1) * n_gt, -1)
    d['norm_loss'] = sl1(t, torch.zeros_like(t))
    d['edge_loss'] = sl1(torch.linalg.norm(ep, dim=-1), torch.linalg.norm(eg, dim=-1))
    v3g, v2g = v3d_gt[:, perm], v2d_gt[:, perm]
    gts3, gts2 = [], []
    for _ in range(level):
        gts3.append(v3g); gts2.append(v2g)
        v3g = F.avg_pool1d(v3g.permute(0, 2, 1), 2).permute(0, 2, 1)
        v2g = F.avg_pool1d(v2g.permute(0, 2, 1), 2).permute(0, 2, 1)
    c3, c2 = [], []
    for a3, a2 in zip(v3dList, v2dList):
        j = [g.shape[1] for g in gts3].index(a3.shape[1])
        c3.append(sl1(a3, gts3[j]))
        c2.append(mse(a2 / img_size * 2 - 1, gts2[j] / img_size * 2 - 1))
    return d, {'v3d_loss': c3, 'v2d_loss': c2}


def calc_loss_GCN(out, labels, loss_assets, epoch=0, w3d=100., w2d=50., w_norm=10., w_edge=2000., norm_epoch=50):
    """calc_loss_GCN, core/Loss.py:201-277 (aux loss disabled at :213, upsample_weight=None path)."""
    result, params, hlist, other = out
    v3d_r = labels['v3d_r'] + labels['root_rel'][:, None]
    sides = {}
    for side, v3g, v2g in (('left', labels['v3d_l'], labels['v2d_l']), ('right', v3d_r, labels['v2d_r'])):
        la = loss_assets[side]
        sides[side] = graph_loss_side(la['J21'], la['faces'], la['perm'], v3g, v2g, result['verts3d'][side], result['verts2d'][side],
                                      [h['verts3d'][side] for h in hlist], [h['verts2d'][side] for h in hlist])
    m = {k: (sides['left'][0][k] + sides['right'][0][k]) / 2 for k in sides['left'][0]}
    alpha = 0 if epoch < norm_epoch else 1
    total = w3d * m['vert3d_loss'] + w2d * m['vert2d_loss'] + w3d * m['joint_loss'] + w_norm * m['norm_loss'] + alpha * w_edge * m['edge_loss']
    for i in range(len(sides['left'][1]['v3d_loss'])):
        total = total + w3d * (sides['left'][1]['v3d_loss'][i] + sides['right'][1]['v3d_loss'][i]) / 2 \
                      + w2d * (sides['left'][1]['v2d_loss'][i] + sides['right'][1]['v2d_loss'][i]) / 2
    return total
