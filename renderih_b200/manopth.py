"""The pose optimiser's hand model on the GPU: a drop-in for the extended hassony2 `manopth` ManoLayer
(pose_data_optimize/manopth/manopth/manolayer.py) in the mode every caller builds it with, root_rot_mode = joint_rot_mode = 'quat',
use_pca=False (hocontact/postprocess/geo_optimizer_both_batch.py:54-77, collision/CollisionFilter.py:52-71, collision/CollisionCheck.py:31-50,
scripts/HandPoseArguer.py:13-21, helpful_py/export_mano_obj.py:24-32).  Forward and backward are one kernel each (csrc/manopth.cu);
there is no CPU path.  MANO is read with `assets.load_mano_dict`, so chumpy is not needed.

Conventions reproduced (line numbers of manolayer.py unless stated):

* Rotations: th_pose_coeffs [B,64] or [B,16,4] are quaternions (w,x,y,z), root first.  Each rotation-matrix entry is divided by |q|^2
  rather than built from a normalised q (quatutils.py:188-221).  Left hands negate q.y and q.z first (:243-245); the gradient carries
  that sign.
* Kinematic chain: the hard-coded three-level chain (:276-312), not kintree_table.  `transf` [B,16,4,4] is in native MANO joint order.
* Shape: with th_betas None or of one element, the zero `th_betas` buffer is used for every hand (:259-264); with share_betas, the batch
  mean of th_betas (:266-267).  Left hands have th_shapedirs[:, 0, :] negated at construction (:169-170).
* Joints: the 16 global joint positions; with root_palm, joint 0 is replaced by the mean of vertices 95 and 22 (:339-341); finger tips
  are vertices 745, 317, 444, 556, 673 (right) or 745, 317, 445, 556, 673 (left) (:335-338); then reordered with the :345 list.  Metres.
* Centring (:347-366), decided over the WHOLE th_trans tensor: if th_trans is None or its norm is 0, joint center_idx is subtracted
  (nothing when center_idx is None); otherwise th_trans is added and nothing is subtracted.  transf's translation is the global
  translation - centre + th_trans.  The decision is taken on the device (no host synchronisation; the reference's
  `bool(torch.norm(th_trans) == 0)` synchronises).  A negative center_idx indexes from the end, as Python indexing does.
* Returns (verts [B,778,3], joints [B,21,3]) + (transf,) if return_transf + (th_pose_coeffs,) if return_full_pose (:371-380); the full
  pose is the input tensor itself.

Not supported: the 'axisang' / 'rotmat' modes and PCA (NotImplementedError), float64 inputs.
"""
import ctypes
import os

import numpy as np
import torch
from torch.nn import Module

from ._lib import call
from .assets import load_mano_dict

_MODES = ('axisang', 'rotmat', 'quat')


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


class ManoLayer(Module):
    """manopth.manolayer.ManoLayer with the reference's constructor; only root_rot_mode = joint_rot_mode = 'quat', use_pca=False runs.
    mano_root: a directory holding MANO_RIGHT.pkl / MANO_LEFT.pkl, or a MANO dict of this side (e.g. assets.synthetic_mano)."""

    def __init__(self, center_idx=None, flat_hand_mean=True, ncomps=6, side='right', mano_root='mano/models', use_pca=True,
                 root_rot_mode='axisang', joint_rot_mode='axisang', robust_rot=False, return_transf=False, return_full_pose=False):
        super().__init__()
        # the reference's argument checks, in its order and with its exception types (:68-118)
        if root_rot_mode not in _MODES:
            raise KeyError("root_rot_mode must be one of 'axisang', 'rotmat' or 'quat', got {}".format(root_rot_mode))
        if use_pca and joint_rot_mode != 'axisang':
            raise TypeError("with use_pca, joint_rot_mode must be 'axisang', got {}".format(joint_rot_mode))
        if joint_rot_mode == 'axisang':
            if root_rot_mode not in ('axisang', 'rotmat'):
                raise KeyError("rot_mode not compatible: with joint_rot_mode 'axisang', root_rot_mode must be 'axisang' or 'rotmat', "
                               "got {}".format(root_rot_mode))
        elif root_rot_mode != joint_rot_mode:
            raise KeyError('rot_mode not compatible: root and joint rot modes must be equal, got {} for root and {} for joint'.format(
                root_rot_mode, joint_rot_mode))
        if use_pca or joint_rot_mode != 'quat':
            raise NotImplementedError('renderih_b200.manopth.ManoLayer runs root_rot_mode = joint_rot_mode = quat without PCA only; got '
                                      'root_rot_mode={}, joint_rot_mode={}, use_pca={}'.format(root_rot_mode, joint_rot_mode, use_pca))
        if side not in ('right', 'left'):
            raise ValueError("side must be 'right' or 'left', got {}".format(side))
        self.center_idx = center_idx
        self.flat_hand_mean = flat_hand_mean
        self.robust_rot = robust_rot
        self.return_transf = return_transf
        self.return_full_pose = return_full_pose
        self.use_pca = use_pca
        self.ncomps = 45
        self.rot = 4
        self.root_rot_mode = root_rot_mode
        self.joint_rot_mode = joint_rot_mode
        self.side = side
        if isinstance(mano_root, dict):
            self.mano_path, d = None, mano_root
        else:
            self.mano_path = os.path.join(mano_root, 'MANO_RIGHT.pkl' if side == 'right' else 'MANO_LEFT.pkl')
            d = load_mano_dict(self.mano_path)
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32)))
        jr = d['J_regressor']
        jr = jr.toarray() if hasattr(jr, 'toarray') else np.asarray(jr)
        sd = np.asarray(d['shapedirs'])
        self.register_buffer('th_betas', torch.zeros(1, sd.shape[-1]))
        self.register_buffer('th_shapedirs', f32(sd))
        self.register_buffer('th_posedirs', f32(d['posedirs']))
        self.register_buffer('th_v_template', f32(d['v_template']).unsqueeze(0))
        self.register_buffer('th_J_regressor', f32(jr))
        self.register_buffer('th_weights', f32(d['weights']))
        self.register_buffer('th_faces', torch.from_numpy(np.asarray(d['f']).astype(np.int64)))
        self.register_buffer('th_hands_mean_quat', None)
        self.kintree_table = np.asarray(d['kintree_table'])
        self.kintree_parents = list(self.kintree_table[0].tolist())
        if side == 'left':
            self.th_shapedirs[:, 0, :] *= -1
        self._derived = None

    def _tables(self, device):
        """Device tables in the kernel's layout, rebuilt when a buffer is replaced or changed in place."""
        bufs = (self.th_shapedirs, self.th_posedirs, self.th_v_template, self.th_J_regressor, self.th_weights)
        key = (device,) + tuple((b._version, b.data_ptr()) for b in bufs)
        if self._derived is None or self._derived[0] != key:
            if tuple(self.th_shapedirs.shape) != (778, 3, 10) or tuple(self.th_posedirs.shape) != (778, 3, 135):
                raise ValueError('MANO tables of unexpected shape: shapedirs %s, posedirs %s' % (tuple(self.th_shapedirs.shape),
                                                                                                  tuple(self.th_posedirs.shape)))
            t = [self.th_shapedirs.to(device).reshape(2334, 10).t().contiguous(),
                 self.th_posedirs.to(device).reshape(2334, 135).t().contiguous(),
                 self.th_v_template.to(device).reshape(2334).contiguous(),
                 self.th_J_regressor.to(device).reshape(16, 778).contiguous(),
                 self.th_weights.to(device).reshape(778, 16).contiguous()]
            arr = (ctypes.c_void_p * 5)(*[x.data_ptr() for x in t])
            self._derived = (key, t, arr)
        return self._derived[2]

    def forward(self, th_pose_coeffs, th_betas=None, th_trans=None, root_palm=None, share_betas=None):
        q = th_pose_coeffs
        for name, t in (('th_pose_coeffs', q), ('th_betas', th_betas), ('th_trans', th_trans)):
            if t is not None and not (isinstance(t, torch.Tensor) and t.is_cuda):
                raise RuntimeError('renderih_b200.manopth.ManoLayer: %s must be a CUDA tensor (there is no CPU path)' % name)
            if t is not None and t.dtype != torch.float32:
                raise TypeError('renderih_b200.manopth.ManoLayer: %s must be float32, got %s' % (name, t.dtype))
        B = q.shape[0] if q.dim() > 0 else 0
        if not ((q.dim() == 2 and q.shape[1] == 64) or (q.dim() == 3 and tuple(q.shape[1:]) == (16, 4))):
            raise ValueError('th_pose_coeffs must be [B,64] or [B,16,4] quaternions, got %s' % (tuple(q.shape),))
        if self.center_idx is not None and not -21 <= int(self.center_idx) < 21:
            raise IndexError('center_idx %d out of range for 21 joints' % int(self.center_idx))
        center = -1 if self.center_idx is None else int(self.center_idx) % 21
        dev = q.device
        betas, shared = None, 1
        if th_betas is not None and th_betas.numel() != 1:
            if tuple(th_betas.shape) != (B, 10):
                raise ValueError('th_betas must be [B,10] = [%d,10], got %s' % (B, tuple(th_betas.shape)))
            if th_betas.device != dev:
                raise RuntimeError('th_betas is on %s, th_pose_coeffs on %s' % (th_betas.device, dev))
            if share_betas is not None and bool(share_betas):
                betas = th_betas.mean(0, keepdim=True)
            else:
                betas, shared = th_betas, 0
        trans = None
        if th_trans is not None:
            if th_trans.device != dev:
                raise RuntimeError('th_trans is on %s, th_pose_coeffs on %s' % (th_trans.device, dev))
            try:
                trans = th_trans.expand(B, 3)
            except RuntimeError:
                raise ValueError('th_trans must broadcast to [B,3] = [%d,3], got %s' % (B, tuple(th_trans.shape)))
        palm = root_palm is not None and bool(root_palm)
        verts, joints, transf = _ManopthFn.apply(self, q.reshape(B, 16, 4), betas, shared, trans, center, int(palm), bool(self.return_transf))
        results = [verts, joints]
        if self.return_transf:
            results.append(transf)
        if self.return_full_pose:
            results.append(th_pose_coeffs)
        return tuple(results)


class _ManopthFn(torch.autograd.Function):
    """rih_manopth_fwd / rih_manopth_bwd: outputs (verts, joints, transf or None) and their gradient."""

    @staticmethod
    def forward(ctx, layer, quat, betas, shared, trans, center, palm, want_transf):
        dev, B = quat.device, quat.shape[0]
        quat = quat.contiguous()
        betas = None if betas is None else betas.contiguous()
        trans = None if trans is None else trans.contiguous()
        side = 1 if layer.side == 'left' else 0
        verts = torch.empty(B, 778, 3, device=dev)
        joints = torch.empty(B, 21, 3, device=dev)
        transf = torch.empty(B, 16, 4, 4, device=dev) if want_transf else None
        flag = None
        with torch.cuda.device(dev):
            tables = layer._tables(dev)
            st = _stream(quat)
            if trans is not None:
                flag = torch.empty(1, dtype=torch.int32, device=dev)
                call('rih_manopth_translate_flag', trans.data_ptr(), trans.numel(), flag.data_ptr(), st)
            call('rih_manopth_fwd', tables, quat.data_ptr(), _ptr(betas), shared, _ptr(trans), _ptr(flag), center, palm, side,
                 verts.data_ptr(), joints.data_ptr(), _ptr(transf), B, st)
        ctx.layer, ctx.args = layer, (shared, center, palm, side)
        ctx.save_for_backward(quat, betas, trans, flag)
        ctx.set_materialize_grads(False)
        return verts, joints, transf

    @staticmethod
    def backward(ctx, g_verts, g_joints, g_transf):
        quat, betas, trans, flag = ctx.saved_tensors
        shared, center, palm, side = ctx.args
        dev, B = quat.device, quat.shape[0]
        c = lambda g: None if g is None else g.float().contiguous()
        g_verts, g_joints, g_transf = c(g_verts), c(g_joints), c(g_transf)
        need = ctx.needs_input_grad      # (layer, quat, betas, shared, trans, center, palm, want_transf)
        d_quat = torch.empty_like(quat) if need[1] else None
        d_betas = torch.empty_like(betas) if (betas is not None and need[2]) else None
        d_trans = torch.empty_like(trans) if (trans is not None and need[4]) else None
        work = torch.empty(B, 10, device=dev) if (d_betas is not None and shared) else None
        with torch.cuda.device(dev):
            call('rih_manopth_bwd', ctx.layer._tables(dev), quat.data_ptr(), _ptr(betas), shared, _ptr(trans), _ptr(flag), center, palm, side,
                 _ptr(g_verts), _ptr(g_joints), _ptr(g_transf), _ptr(d_quat), _ptr(d_betas), _ptr(d_trans), _ptr(work), B, _stream(quat))
        return None, d_quat, d_betas, None, d_trans, None, None, None
