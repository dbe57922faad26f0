"""numpy / scipy statement of the pose data pipeline's conversion and augmentation stages (pose_data_optimize/scripts/HandPoseConverter.py
:159-212, 272-332, HandPoseArguer.py:33-173, Ver2Code/NatureJudge/PoseArgue.py:34-174), vectorised over frames and with the uniforms
passed in.  It makes the reference's scipy calls on the same arrays, so its results equal the reference's bit for bit; it is the GPU
tests' large-batch oracle and the host baseline of tests/baselines/bench_pose_data.py.

TEST INFRASTRUCTURE -- never imported by the product package.
"""
import numpy as np
from scipy.spatial.transform import Rotation

FLIP = np.asarray(([1, 0, 0], [0, -1, 0], [0, 0, -1]))
BEND_LISTS = (((2, 5, 11, 8), (-8, 110)), ((13,), (-20, 40)), ((14,), (-8, 50)), ((3, 6, 12, 9, 15), None), ((1, 4, 10, 7), (-25, 70)))
BEND_JOINTS = tuple(j for js, _ in BEND_LISTS for j in js)
SPLANK_JOINTS = (1, 4, 10, 7, 13)
# (normal bend range, splank ranges, bend maximum, splank maximum) per arguer; PoseArguer's maxima are scaled by random_level
ARGUERS = {'HandPoseArguer': ((-8, 90), ((-6, 20), (-10, 10), (-15, 6), (-35, 6), (-9, 80)), 120, 30),
           'PoseArguer': ((-8, 95), ((-25, 15), (-15, 15), (-25, 15), (-20, 30), (-30, 30)), 120, 45)}


def ranges(arguer):
    """[20,2] (lo, hi) of the 20 draws of a frame copy in the reference's draw order."""
    normal, splank = ARGUERS[arguer][:2]
    rows = []
    for js, r in BEND_LISTS:
        rows += [r if r is not None else normal] * len(js)
    return np.asarray(rows + list(splank), dtype=np.float64)


def draw_uniforms(B, A):
    """numpy's global RandomState in the reference's order: all bend draws (frame-major, BEND_JOINTS, A each), then all splank draws ->
    [B,20,A]."""
    ub = np.random.rand(B * len(BEND_JOINTS) * A).reshape(B, len(BEND_JOINTS), A)
    us = np.random.rand(B * len(SPLANK_JOINTS) * A).reshape(B, len(SPLANK_JOINTS), A)
    return np.concatenate([ub, us], 1)


def adjustments(euler, u, rng, max_bend, max_splank):
    """angle_random_adjust for every draw: euler [B,16,3], u [B,20,A] -> [B,20,A] degrees."""
    out = np.empty_like(u)
    for k, j in enumerate(BEND_JOINTS + SPLANK_JOINTS):
        M = max_bend if k < len(BEND_JOINTS) else max_splank
        a = euler[:, j, 2 if k < len(BEND_JOINTS) else 1]
        pos = np.maximum(np.minimum(M, rng[k, 1] - a), 0)
        neg = np.minimum(np.maximum(-M, rng[k, 0] - a), 0)
        out[:, k] = (pos - neg)[:, None] * u[:, k] + neg[:, None]
    return out


def _apply(vec_pose, adj, axis):
    """apply_adjustment with get_rotation_around_dyaxis's matrices: vec_pose [R,16,3], adj [R,16]."""
    e = np.zeros(adj.shape + (3,))
    e[..., axis] = adj
    m = Rotation.from_euler('xyz', e.reshape(-1, 3), True).as_matrix().reshape(-1, 16, 3, 3)
    rot = Rotation.from_euler('xyz', vec_pose.reshape(-1, 3), True).as_matrix().reshape(-1, 16, 3, 3) @ m
    rot = rot.reshape(-1, 3, 3)
    return Rotation.from_matrix(rot).as_euler('xyz', degrees=True).reshape(-1, 16, 3), rot


def argue_pose(euler, u, arguer='HandPoseArguer', random_level=1.0, stages=False):
    """argue_pose(pose_type='euler') with explicit uniforms: euler [B,16,3], u [B,20,A] -> [B*A,16,3] (row i*A + a).  With stages, also
    (first-pass euler, the two passes' matrices) for branch-margin checks."""
    euler = np.asarray(euler, dtype=np.float64)
    B, A = euler.shape[0], u.shape[2]
    _, _, mb, ms = ARGUERS[arguer]
    adj = adjustments(euler, u, ranges(arguer), mb * random_level, ms * random_level)
    bend, splank = np.zeros((B, A, 16)), np.zeros((B, A, 16))
    bend[:, :, list(BEND_JOINTS)] = adj[:, :len(BEND_JOINTS)].transpose(0, 2, 1)
    splank[:, :, list(SPLANK_JOINTS)] = adj[:, len(BEND_JOINTS):].transpose(0, 2, 1)
    first, m1 = _apply(np.repeat(euler, A, axis=0), bend.reshape(B * A, 16), 2)
    out, m2 = _apply(first, splank.reshape(B * A, 16), 1)
    return (out, first, np.concatenate([m1, m2])) if stages else out


def euler_2_mano_quat(euler, side, inv_m0, inv_u1, stages=False):
    """euler [N,16,3] or [16,3] -> [N,16,4] float32 (w,x,y,z)."""
    e = np.asarray(euler)
    e = e[np.newaxis] if e.ndim == 2 else e
    mat = Rotation.from_euler('xyz', e.reshape(-1, 3), degrees=True).as_matrix().reshape(e.shape[0], 16, 3, 3)
    mat = inv_m0 @ mat @ inv_u1
    if side == 'left':
        mat[:, 0] = np.tile(FLIP[np.newaxis], (len(mat), 1, 1)) @ mat[:, 0]
    mat = mat.reshape(-1, 3, 3)
    q = Rotation.from_matrix(mat).as_quat()[:, [3, 0, 1, 2]].reshape(-1, 16, 4)
    if side == 'left':
        q[:, :, 2:] = -q[:, :, 2:]
    return (q.astype(np.float32), mat) if stages else q.astype(np.float32)


def mano_quat_2_euler(quat, side, inv_m0, inv_u1, stages=False):
    """[N,16,4] or [16,4] (w,x,y,z) -> [N,16,3] float64 degrees; the input is not modified."""
    q = np.array(quat)
    q = q[np.newaxis] if q.ndim <= 2 else q
    if side == 'left':
        q[:, :, 2:] = -q[:, :, 2:]
    mat = Rotation.from_quat(q.reshape(-1, 4)[:, [1, 2, 3, 0]]).as_matrix().reshape(-1, 16, 3, 3)
    if side == 'left':
        mat[:, 0] = np.tile(FLIP[np.newaxis], (len(mat), 1, 1)) @ mat[:, 0]
    mat = (inv_m0.swapaxes(1, 2) @ mat @ inv_u1.swapaxes(1, 2)).reshape(-1, 3, 3)
    e = Rotation.from_matrix(mat).as_euler('xyz', degrees=True).reshape(-1, 16, 3)
    return (e, mat) if stages else e


def axis_angle_2_mano_quat(aa, side, hands_mean, flat_hand=False):
    """(N,16,3), (16,3), (N,48) or (48) -> [N,16,4] float32 (w,x,y,z); hands_mean [1,15,3] float32 added unless flat_hand."""
    a = np.asarray(aa, dtype=np.float32).reshape((-1, 16, 3))
    if not flat_hand:
        a = np.hstack([a[:, 0:1], a[:, 1:] + hands_mean.reshape(1, 15, 3)])
    q = Rotation.from_rotvec(a.reshape(-1, 3)).as_quat().reshape(a.shape[0], 16, 4)
    q = np.asarray(q, dtype=np.float32)[..., [3, 0, 1, 2]]
    if side == 'left':
        q[:, :, 2:] = -q[:, :, 2:]
    return q


def mano_quat_flat_2_normal(quat, side, hands_mean, return_type='quat'):
    """MANO quaternions reshaped to (-1,16,4) float32 -> axis-angle with hands_mean subtracted (float64 [N,16,3]) or, for 'quat', that
    through axis_angle_2_mano_quat(flat_hand=True)."""
    q = np.array(quat, dtype=np.float32).reshape((-1, 16, 4))
    if side == 'left':
        q[:, :, 2:] = -q[:, :, 2:]
    aa = Rotation.from_quat(q[..., [1, 2, 3, 0]].reshape(-1, 4)).as_rotvec().reshape(q.shape[0], 16, 3)
    aa = np.hstack([aa[:, 0:1], aa[:, 1:] - hands_mean.reshape(1, 15, 3)])
    return axis_angle_2_mano_quat(aa, side, hands_mean, flat_hand=True) if return_type == 'quat' else aa


def euler_margin(e):
    """Smallest distance in degrees of euler angles [..., 3] from the points where as_euler branches: the gimbal test (second angle at
    +-90) and the +-180 wrap of the first and third angles."""
    e = np.asarray(e)
    return float(min(np.abs(np.abs(e[..., 1]) - 90).min(), (180 - np.abs(e[..., 0])).min(), (180 - np.abs(e[..., 2])).min()))


def branch_margin(mat):
    """Smallest gap between the largest and second-largest of (M00, M11, M22, trace) over matrices [..., 3, 3]: from_matrix's branch."""
    m = np.asarray(mat)
    d = np.stack([m[..., 0, 0], m[..., 1, 1], m[..., 2, 2], m[..., 0, 0] + m[..., 1, 1] + m[..., 2, 2]], -1)
    d = np.sort(d, -1)
    return float((d[..., 3] - d[..., 2]).min())
