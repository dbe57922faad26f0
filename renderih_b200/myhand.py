"""The `common/myhand` "graph" model variant -- what the reference's `apps/train.py` and `apps/eval_interhand.py` build by default
(`core/lijun_trainer.py:102-113` -> `common/myhand/lijun_model_graph.load_graph_model`), SURVEY.md 8(f) row 1.

Deltas against `models.model.HandNET_GCN`, all served by the same sm_90a kernels:
  * encoder: torchvision ResNet-50 trunk only, no heat-map / dense-pose heads (common/myhand/encoder_lijun.py:62-104);
  * mid: one 1x1 Conv -> ReLU -> BN per trunk level (2048 / 1024 / 512 / 256 -> 256) + global average pool (encoder_lijun.py:107-146);
  * DualGraph blocks without a Laplacian: LN -> ReLU -> Linear -> LN -> ReLU -> Linear + shortcut (model_attn/DualGraph_lijun.py:28-58);
  * inter-hand attention normalises Lf + Rf and attends with each hand's OWN keys over the other hand's values
    (model_attn/inter_attn_lijun.py:79-91);
  * the decoder returns empty MANO lists and no auxiliary maps (decoder_lijun_graph.py:316-320); it owns MANO layers (used by the
    reference's loss / renderer code, not by forward) whose persistent buffers are part of the 1051-key state_dict.
Same `forward(img) -> (result, paramsDict, handDictList, otherInfo)` contract and the same state_dict keys in the same order.
"""
import os

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .assets import default_asset_root, load_mano_dict, load_model_assets
from .config import load_cfg
from .manolayer import ManoLayer
from .model import MLP_GraphBlock, ResNetSimple, _StreamedFmaps, _cl, _conv_relu_bn, decoder as _decoder_base, fork, join


class resnet_mid(nn.Module):
    """common/myhand/encoder_lijun.py:107-146"""

    def __init__(self, model_type='resnet50', in_fmapDim=(2048, 1024, 512, 256), out_fmapDim=(256, 256, 256, 256)):
        super().__init__()
        self.convs = nn.ModuleList([nn.Sequential(_cl(nn.Conv2d(in_fmapDim[i], out_fmapDim[i], kernel_size=1, bias=False)),
                                                  nn.ReLU(inplace=True), nn.BatchNorm2d(out_fmapDim[i])) for i in range(len(out_fmapDim))])
        self.global_feature_dim = 512 * 4
        self.fmaps_dim = list(out_fmapDim)

    def get_info(self):
        return {'global_feature_dim': self.global_feature_dim, 'fmaps_dim': self.fmaps_dim}

    def level(self, i, img_fmaps, N):
        x, H = img_fmaps[i]
        seq = self.convs[i]
        return _conv_relu_bn(x, seq[0], seq[2], N, H, H, self.training), H

    def forward(self, img_fmaps, N):
        x1, H1 = img_fmaps[0]
        gf = ops.global_avgpool(x1, N, H1 * H1)
        return gf, [self.level(i, img_fmaps, N) for i in range(len(self.convs))]


class MANO(nn.Module):
    """common/utils/mano.py:39-79: holder of a ManoLayer plus the 21-joint regressor (tips 745/317/445/556/673, reordered)."""

    def __init__(self, mano_dict):
        super().__init__()
        self.layer = ManoLayer(mano_dict, center_idx=None, out_scale=1000.0)     # common/utils/manolayer.py: millimetres
        self.vertex_num, self.joint_num = 778, 21
        self.face = self.layer.faces
        jr = self.layer.J_regressor.numpy()
        tips = np.zeros((5, jr.shape[1]), np.float32)
        for i, v in enumerate((745, 317, 445, 556, 673)):
            tips[i, v] = 1.0
        jr = np.concatenate((jr, tips))[[0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20], :]
        self.joint_regressor = jr
        self.register_buffer('joint_regressor_torch', torch.from_numpy(jr).float())

    def get_3d_joints(self, vertices):
        return torch.einsum('bik,ji->bjk', [vertices, self.joint_regressor_torch])


class decoder(_decoder_base):
    """common/myhand/decoder_lijun_graph.py:150-320"""

    def __init__(self, cfg, mano_left, mano_right, **kw):
        super().__init__(block_cls=MLP_GraphBlock, attn_variant='lijun', mano_lists=False, **kw)
        self.cfg = cfg
        self.mano = bool(getattr(cfg, 'mano_flag', False))
        if self.mano:
            raise NotImplementedError('decoder_lijun_graph with mano_flag=True only adds an unused ParamRegressor (decoder_lijun_graph.py:226); '
                                      'use load_new_model for the MANO tail')
        self._init_mano(mano_left, mano_right)

    def _init_mano(self, mano_left, mano_right):
        self.mano_left = MANO(mano_left)
        self.mano_left_layer = self.mano_left.layer
        self.mano_right = MANO(mano_right)
        self.mano_right_layer = self.mano_right.layer
        self.left_face = torch.as_tensor(np.asarray(self.mano_left_layer.faces).astype(np.int64))
        self.right_face = torch.as_tensor(np.asarray(self.mano_right_layer.faces).astype(np.int64))
        # decoder_lijun_graph.py:234-236: the released MANO_LEFT has a mirrored first shape direction
        if torch.sum(torch.abs(self.mano_left_layer.shapedirs[:, 0, :] - self.mano_right_layer.shapedirs[:, 0, :])) < 1:
            self.mano_left_layer.shapedirs[:, 0, :] *= -1


def rot6d_to_rotmat(x):
    """6-D rotation representation -> rotation matrices (Gram-Schmidt on the two 3-vectors interleaved in x), the construction used by
    `ParamRegressor.rot6d_to_rotmat` (common/myhand/decoder_lijun_mano.py:36-43).  x: [N, 6] -> [N, 3, 3] with columns b1, b2, b3."""
    x = x.reshape(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    b1 = torch.nn.functional.normalize(a1, dim=1)
    b2 = torch.nn.functional.normalize(a2 - (b1 * a2).sum(dim=1, keepdim=True) * b1, dim=1)
    b3 = torch.linalg.cross(b1, b2, dim=1)
    return torch.stack((b1, b2, b3), dim=-1)


def rotmat_to_axis_angle(R):
    """Rotation matrices [N,3,3] -> axis-angle [N,3] through a unit quaternion, with the branch structure of the conversion the
    reference calls (common/myhand/utils/comm.py:176-200 -> :250-324 matrix -> quaternion, :203-247 quaternion -> axis-angle):
    the quaternion component with the largest magnitude is chosen by the signs / order of the diagonal, the angle is taken with atan2
    on the half-angle sine / cosine (folded to the cos >= 0 half), NaNs (zero rotation) become 0."""
    m = R.transpose(1, 2)               # the reference works on the transpose
    d0, d1, d2 = m[:, 0, 0], m[:, 1, 1], m[:, 2, 2]
    low = d2 < 1e-6
    c0 = low & (d0 > d1)
    c1 = low & ~(d0 > d1)
    c2 = ~low & (d0 < -d1)
    t = torch.where(c0, 1 + d0 - d1 - d2, torch.where(c1, 1 - d0 + d1 - d2, torch.where(c2, 1 - d0 - d1 + d2, 1 + d0 + d1 + d2)))
    s01, s02, s12 = m[:, 0, 1] + m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2], m[:, 1, 2] + m[:, 2, 1]
    a01, a20, a12 = m[:, 0, 1] - m[:, 1, 0], m[:, 2, 0] - m[:, 0, 2], m[:, 1, 2] - m[:, 2, 1]
    qa = torch.stack([a12, t, s01, s02], -1)       # x largest
    qb = torch.stack([a20, s01, t, s12], -1)       # y largest
    qc = torch.stack([a01, s02, s12, t], -1)       # z largest
    qd = torch.stack([t, a12, a20, a01], -1)       # w largest
    sel = lambda c: c[:, None]
    q = torch.where(sel(c0), qa, torch.where(sel(c1), qb, torch.where(sel(c2), qc, qd)))
    q = q / torch.sqrt(t)[:, None] * 0.5
    w, v = q[:, 0], q[:, 1:]
    sin2 = (v * v).sum(-1)
    sin_h = torch.sqrt(sin2)
    two_theta = 2.0 * torch.where(w < 0.0, torch.atan2(-sin_h, -w), torch.atan2(sin_h, w))
    k = torch.where(sin2 > 0.0, two_theta / sin_h, torch.full_like(sin_h, 2.0))
    aa = v * k[:, None]
    return torch.where(torch.isnan(aa), torch.zeros_like(aa), aa)


class ParamRegressor(nn.Module):
    """common/myhand/decoder_lijun_mano.py:26-58: 2334 -> 1024 -> 512 trunk, two 512 -> 128 -> {96, 10} heads (Hardswish), 6-D rotations
    of the 16 joints -> axis-angle.  The Linear layers run on the GEMM kernels; the activations and the rotation conversions are a few
    torch elementwise ops on [B, <= 1024] tensors."""

    def __init__(self, joint_num=778):
        super().__init__()
        self.joint_num = joint_num

        def mlp(dims, act_final):
            layers = []
            for i in range(len(dims) - 1):
                layers.append(nn.Linear(dims[i], dims[i + 1]))
                if i < len(dims) - 2 or act_final:
                    layers.append(nn.Hardswish(inplace=True))
            return nn.Sequential(*layers)
        self.fc = mlp([joint_num * 3, 1024, 512], True)
        self.fc_pose = mlp([512, 128, 16 * 6], False)
        self.fc_shape = mlp([512, 128, 10], False)

    @staticmethod
    def _run(seq, x):
        for m in seq:
            x = ops.linear(x, m.weight, m.bias) if isinstance(m, nn.Linear) else torch.nn.functional.hardswish(x)
        return x

    def forward(self, verts):
        B = verts.shape[0]
        feat = self._run(self.fc, verts.reshape(B, self.joint_num * 3))
        rotmat = rot6d_to_rotmat(self._run(self.fc_pose, feat))
        pose = rotmat_to_axis_angle(rotmat).reshape(B, -1)
        return pose, self._run(self.fc_shape, feat), rotmat


class decoder_mano(decoder):
    """common/myhand/decoder_lijun_mano.py:81-305 ('newgraph'): the graph decoder followed by the MANO tail -- ParamRegressor on the
    up-sampled 778-vertex mesh -> (pose, shape) -> ManoLayer (one fused kernel each way) -> root-centred, bone-length-normalised mesh."""

    def __init__(self, cfg, mano_left, mano_right, **kw):
        nn.Module.__init__(self)
        _decoder_base.__init__(self, block_cls=MLP_GraphBlock, attn_variant='lijun', mano_lists=False, **kw)
        self.cfg = cfg
        self.mano = True
        self.param_regressor = ParamRegressor(joint_num=778)
        self._init_mano(mano_left, mano_right)

    def forward(self, x, fmaps):
        from .manolayer import rodrigues_batch
        from .model import IMG_SIZE
        res, paramsDict, handDictList, _ = _decoder_base.forward(self, x, fmaps)
        scale, trans2d = paramsDict['scale'], paramsDict['trans2d']
        up = {s: res['verts3d'][s] for s in ('left', 'right')}          # unsample_layer output (decoder_lijun_mano.py:243)
        result = {'verts3d': {}, 'verts2d': {}, 'v3d_left': up['left'], 'v3d_right': up['right']}
        j0 = {s: torch.einsum('bik,i->bk', up[s], getattr(self, 'mano_' + s).joint_regressor_torch[0]) for s in ('left', 'right')}
        root_rel = j0['right'] - j0['left']                              # joint 0 of get_3d_joints (:244-246)
        pred, sl = {}, {}
        for s in ('left', 'right'):
            pose, shape, _ = self.param_regressor(up[s])
            shape = torch.tanh(shape) * 3
            v, j = getattr(self, 'mano_%s_layer' % s)(rodrigues_batch(pose[:, :3]), pose[:, 3:], shape)     # millimetres
            v, j = v / 1000, j / 1000
            v = v - j[:, 0:1]
            sl[s] = (0.095 / torch.linalg.norm(j[:, 9:10] - j[:, 0:1], dim=-1)).reshape(-1, 1, 1)           # bone-length rescale (:265-268)
            v = v * sl[s]
            pred[s] = {'verts3d': v, 'joints3d': j, 'mano_pose': pose, 'mano_shape': shape}
            sc = (scale[s] * IMG_SIZE)[:, None, None]
            result['verts2d'][s] = sc * v[..., :2] + (trans2d[s] * IMG_SIZE / 2 + IMG_SIZE / 2)[:, None]      # projection_batch
        result['verts3d']['left'] = pred['left']['verts3d']
        result['verts3d']['right'] = pred['right']['verts3d'] + root_rel.reshape(-1, 1, 3)
        otherInfo = {'length': (sl['left'] + sl['right']) / 2, 'root_rel': root_rel,
                     'verts3d_MANO_list': {'left': pred['left'], 'right': pred['right']}, 'verts2d_MANO_list': {'left': [], 'right': []}}
        paramsDict = {'scale': scale, 'trans2d': trans2d, 'scalelength_left': sl['left'], 'scalelength_right': sl['right'], 'root_rel': root_rel}
        return result, paramsDict, handDictList, otherInfo


class HandNET_GCN(nn.Module):
    """common/myhand/lijun_model_graph.py:19-34"""

    def __init__(self, encoder, mid_model, decoder, cliff=False):
        super().__init__()
        self.encoder = encoder
        self.mid_model = mid_model
        self.decoder = decoder
        self.cliff = cliff

    def forward(self, img):
        if not (isinstance(img, torch.Tensor) and img.is_cuda):
            raise RuntimeError('renderih_b200.myhand.HandNET_GCN runs only on CUDA (sm_90a) tensors; there is no CPU fallback')
        if img.dtype != torch.float32:
            raise RuntimeError('renderih_b200.myhand.HandNET_GCN expects float32 images')
        ops.seed_state.begin_forward()
        if self.training:
            ops.seed_state.advance(img.device)
        N = img.shape[0]
        img_fmaps = self.encoder(img)
        if type(self.mid_model) is not resnet_mid:
            global_feature, fmaps = self.mid_model(img_fmaps, N)
            return self.decoder(global_feature, fmaps)
        # same pipelining as models.model.HandNET_GCN._forward_pipelined: the four mid 1x1 conv + BN levels run on the aux stream, each level's
        # event gates the DualGraph layer that reads it (the 64 px level feeds nothing in the decoder and overlaps all of it)
        x1, H1 = img_fmaps[0]
        global_feature = ops.global_avgpool(x1, N, H1 * H1)
        fmaps = _StreamedFmaps()

        def mid_levels():
            for i in range(len(self.mid_model.convs)):
                fmaps.publish(self.mid_model.level(i, img_fmaps, N))
            return list(fmaps)
        side = fork(img.device, 'aux', mid_levels)
        out = self.decoder(global_feature, fmaps)
        join(side)
        return out


def load_new_model(cfg=None, cliff=False, assets=None, mano_assets=None, asset_root=None):
    """`load_new_model(cfg)` of common/myhand/lijun_model_newgraph.py:34-71: the graph model with the MANO tail (decoder_lijun_mano)."""
    return load_graph_model(cfg, cliff, assets, mano_assets, asset_root, decoder_cls=decoder_mano)


def load_graph_model(cfg=None, cliff=False, assets=None, mano_assets=None, asset_root=None, decoder_cls=None):
    """`load_graph_model(cfg)` of common/myhand/lijun_model_graph.py:37-70.  cfg: path | CfgNode-like | None (defaults).
    assets / mano_assets: pre-loaded graph / MANO dictionaries (tests use synthetic ones); default = the reference's misc/ files."""
    if cfg is None or isinstance(cfg, str):
        cfg = load_cfg(cfg)
    et = cfg.MODEL.ENCODER_TYPE
    if 'resnet' not in et:
        raise NotImplementedError('myhand graph variant: only the ResNet encoders are built (common/myhand/encoder_lijun.py:328-337)')
    encoder = ResNetSimple(model_type=et, fmapDim=[128, 128, 128, 128], handNum=2, heatmapDim=21, aux_heads=False)
    mid = resnet_mid(model_type=et, in_fmapDim=[2048, 1024, 512, 256], out_fmapDim=cfg.MODEL.DECONV_DIMS)
    a = assets if assets is not None else load_model_assets(cfg, asset_root)
    if mano_assets is None:
        root = asset_root or default_asset_root()
        mano_assets = {s: load_mano_dict(os.path.join(root, 'mano', 'MANO_%s.pkl' % s.upper())) for s in ('left', 'right')}
    info = mid.get_info()
    dec = (decoder_cls or decoder)(cfg, mano_assets['left'], mano_assets['right'],
                  global_feature_dim=info['global_feature_dim'], f_in_Dim=info['fmaps_dim'], f_out_Dim=cfg.MODEL.IMG_DIMS,
                  gcn_in_dim=cfg.MODEL.GCN_IN_DIM, gcn_out_dim=cfg.MODEL.GCN_OUT_DIM, graph_k=cfg.MODEL.graph_k,
                  graph_layer_num=cfg.MODEL.graph_layer_num, vertex_num=778, dense_coor=a['dense_coor'],
                  left_graph_dict=a['left_graph'], right_graph_dict=a['right_graph'], num_attn_heads=4,
                  upsample_weight=a['upsample'], dropout=cfg.TRAIN.dropout)
    return HandNET_GCN(encoder, mid, dec, cliff)
