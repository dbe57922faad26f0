"""The pose data pipeline's joint-limit validity rate on the GPU: a drop-in for pose_data_optimize/Ver2Code/ValidJudge/ValidJudger.py and
GetValidRate.py, both hands of every frame judged in one launch (csrc/valid_judge.cu).

    judger = ValidJudger(mano_root, device='cuda:0')
    rate = judger.ComputeValidation(left_pose, right_pose)      # [B,16,4] float32 MANO quaternions each -> 0-dim float32 CUDA tensor
    get_valid_rate(root_path, mano_root, device)                # GetValidRate.py over every mocap file in root_path

The "valid rate" the reference prints is in fact the INVALID fraction: the share of frames in which either hand breaks a joint limit by
more than 0.1 degree.  The number is kept as the reference computes it.

Conventions reproduced (ValidJudger.py, HandPoseConverter.py):
* joint matrices (mano_quat_2_mat_tensor, :214-231): the quaternions as given, with NO normalisation first (unlike the optimiser's
  ergonomics prior), the left hand's y and z negated, quaternion_to_rotation_matrix, then invM_U_n_0^T R invU_M_n_1^T with the
  converter matrices of geo_loss.converter_matrices; M = zero_mat^T ja for joints 1..15, zero_mat being ja at identity quaternions;
* ValidationJudge (:41-111): splank atan2(-x.z, x.x) and bend atan2(x.y, x.x) in degrees, x the first column of M, against the
  reference's two range tables; the score is max(max splank excess, max bend excess), each excess in radians.  Steps 1 and 2 are
  computed and discarded by the reference and are not computed here;
* ComputeValidation (:113-123): ((right > th) + left > th) > 0 with th = 0.1 / 180 * pi rounded to float32, i.e. either hand over the
  limit; the count is taken on the device and divided by B in float32.  The rate is printed, as the reference prints it.

The scores differ from the reference's float32 ones by float32 rounding: the converter products are folded into one matrix per joint.
Not supported: CPU tensors (RuntimeError), quaternions other than float32 (TypeError).
"""
import os

import numpy as np
import torch

from ._lib import call
from .geo_loss import _conv_table, _rest_pose, converter_matrices
from .manopth import ManoLayer


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


class ValidJudger:
    """ValidJudger(mano_root, device): mano_root is a directory with MANO_RIGHT.pkl / MANO_LEFT.pkl, or {'right': mano dict, 'left':
    mano dict}.  The converter matrices come from each side's rest pose (HandPoseConverter.py:29-69)."""

    def __init__(self, mano_root, device='cuda:0'):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('ValidJudger: a CUDA device is required (there is no CPU path)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        roots = mano_root if isinstance(mano_root, dict) else {'right': mano_root, 'left': mano_root}
        self.converter, conv = {}, []
        with torch.no_grad():
            for side in ('left', 'right'):
                layer = ManoLayer(mano_root=roots[side], side=side, use_pca=False, flat_hand_mean=True, center_idx=0, root_rot_mode='quat',
                                  joint_rot_mode='quat').to(self.device)
                self.converter[side] = converter_matrices(side, *_rest_pose(layer, self.device)[1:])
                conv.append(_conv_table(*self.converter[side]))
        self._conv = torch.from_numpy(np.stack(conv)).to(self.device)          # [2,15,18]: left, right

    def scores(self, left_pose, right_pose):
        """ValidationJudge of both hands -> (scores [2,B] float32 in radians, left row then right row; invalid-frame count [1] int64),
        on the device, without synchronising."""
        for name, q in (('left_pose', left_pose), ('right_pose', right_pose)):
            if not (isinstance(q, torch.Tensor) and q.is_cuda):
                raise RuntimeError('ValidJudger: %s must be a CUDA tensor (there is no CPU path)' % name)
            if q.dtype != torch.float32:
                raise TypeError('ValidJudger: %s must be float32, got %s' % (name, q.dtype))
            if q.dim() != 3 or q.shape[0] < 1 or tuple(q.shape[1:]) != (16, 4):
                raise ValueError('ValidJudger: %s must be [B,16,4] with B >= 1, got %s' % (name, tuple(q.shape)))
            if q.device != self.device:
                raise RuntimeError('ValidJudger: %s is on %s, the judger on %s' % (name, q.device, self.device))
        if left_pose.shape != right_pose.shape:
            raise ValueError('ValidJudger: left_pose %s and right_pose %s differ' % (tuple(left_pose.shape), tuple(right_pose.shape)))
        B = left_pose.shape[0]
        ql, qr = left_pose.contiguous(), right_pose.contiguous()
        score = torch.empty(2, B, device=self.device)
        invalid = torch.empty(1, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            call('rih_valid_judge', ql.data_ptr(), qr.data_ptr(), self._conv.data_ptr(), B, score.data_ptr(), invalid.data_ptr(), _stream(ql))
        return score, invalid

    def ComputeValidation(self, left_pose, right_pose):
        """The fraction of frames where either hand breaks a joint limit (the reference's "valid rate", which counts the INVALID ones):
        a 0-dim float32 CUDA tensor, also printed."""
        _, invalid = self.scores(left_pose, right_pose)
        rate = invalid[0] / left_pose.shape[0]
        print(rate)
        return rate


def get_valid_rate(root_path, mano_root, device='cuda:0'):
    """GetValidRate.py: every mocap file in root_path (os.listdir order) loaded in mode 0, euler angles converted to MANO quaternions,
    ComputeValidation per file, the per-file rates weighted by frame count.  Prints "valid rate: ..." and returns that 0-dim tensor
    (the invalid fraction, as in the reference)."""
    from .mocap_optimize import euler_to_mano_quat
    V = ValidJudger(mano_root, device)
    total_poses, valid_poses = 0, 0
    for data_name in os.listdir(root_path):
        raw = np.load(os.path.join(root_path, data_name), allow_pickle=True).item()
        left = torch.from_numpy(euler_to_mano_quat(raw['left']['rot'], 'left', *V.converter['left'])).to(V.device)
        right = torch.from_numpy(euler_to_mano_quat(raw['right']['rot'], 'right', *V.converter['right'])).to(V.device)
        r = V.ComputeValidation(left, right)
        total_poses += left.shape[0]
        valid_poses += r * left.shape[0]
    rate = valid_poses / total_poses
    print('valid rate: {}'.format(rate))
    return rate
