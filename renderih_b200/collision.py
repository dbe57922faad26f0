"""The pose data pipeline's collision filter on the GPU: a drop-in for pose_data_optimize/collision/CollisionFilter.py (and the count
CollisionCheck.py thresholds), with the per-frame contact count computed by csrc/collision.cu for every frame of a batch in one launch.

    count = hand_collision_count(verts_a, verts_b, faces, trans_a=None, trans_b=None)     # int64 [B] on the device
    kept_fraction = filter_collision_data(target_data_path, out_put_path, mano_root='../assets/mano')

Stated deviation.  The reference counts the contacts trimesh / python-fcl report between the two meshes of a frame
(CollisionManager.in_collision_internal(return_data=True), :107-124).  FCL's own triangle test and its multiplicity of contact points
cannot be reproduced or checked here: neither library is part of this project or of the reference tree.  The count here is defined as
the number of (face of hand A, face of hand B) pairs whose closed triangles intersect, decided by Guigue and Devillers' orientation
predicates in float64 (a zero-area face intersects nothing).  `max_contacts` keeps the reference's default of 75 (CollisionCheck.py
uses 100: `hand_collision_count(...) <= 100`), so a threshold tuned on FCL's contact count may need retuning against this one.

Conventions reproduced (CollisionFilter.py):
* data_loader in mode 0 (:27-39): loc * 1.0 / 100, euler angles -> MANO quaternions (HandPoseConverter.euler_2_mano_quat, here
  mocap_optimize.euler_to_mano_quat), both hands through the quaternion ManoLayer with flat_hand_mean=True, center_idx=0;
* float32 vertices plus the float64 loc, so the coordinates are float64 by torch promotion (:96-99);
* the LEFT layer's faces for both meshes (:84);
* a frame is kept when its count is <= max_contacts (:121);
* the saved dict is what copy_dict_struct / dict_add (:9-25) build, quirks included: the first kept frame appears twice, every 1-D
  leaf (e.g. capture_frame_id) becomes [K+1,1], and with no kept frame every leaf stays np.asarray([]) (float64, shape (0,)).

Not supported: CPU tensors (RuntimeError), vertices other than float32 / float64 (TypeError), more than 1024 vertices or 2048 faces
(ValueError).
"""
import os

import numpy as np
import torch

from ._lib import call

MAX_VERTS, MAX_FACES = 1024, 2048


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _checked_faces(faces, V, dev):
    if not (isinstance(faces, torch.Tensor) and faces.is_cuda):
        raise RuntimeError('hand_collision_count: faces must be a CUDA tensor (there is no CPU path)')
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError('hand_collision_count: faces must be int32 or int64, got %s' % faces.dtype)
    if faces.dim() != 2 or faces.shape[1] != 3 or not 1 <= faces.shape[0] <= MAX_FACES:
        raise ValueError('hand_collision_count: faces must be [F,3] with 1 <= F <= %d, got %s' % (MAX_FACES, tuple(faces.shape)))
    if faces.device != dev:
        raise RuntimeError('hand_collision_count: faces are on %s, the vertices on %s' % (faces.device, dev))
    if not torch.cuda.is_current_stream_capturing():
        lo, hi = torch.stack([faces.min(), faces.max()]).tolist()
        if lo < 0 or hi >= V:
            raise ValueError('hand_collision_count: face indices must lie in [0, %d), got [%d, %d]' % (V, lo, hi))
    return faces.to(torch.int32).contiguous()


def hand_collision_count(verts_a, verts_b, faces, trans_a=None, trans_b=None, stats=None):
    """Per frame, the number of (face of hand A, face of hand B) pairs whose closed triangles intersect.

    verts_a, verts_b: [B,V,3] CUDA float32 or float64 (both the same), V <= 1024.  trans_a, trans_b: None or [B,3] float64 (other float
    dtypes are converted to float64), added to every vertex in float64.  faces: [F,3] integer indices into the vertices, the table of
    both meshes, F <= 2048.  -> int64 [B] on the device.  stats: None or an int64 [B,2] CUDA tensor that receives each frame's number of
    box tests and exact triangle tests.  The face indices are checked on the host (one synchronisation) outside CUDA-graph capture; under
    capture an out-of-range face table makes the kernel report -1 for every frame instead of reading out of bounds."""
    for name, v in (('verts_a', verts_a), ('verts_b', verts_b)):
        if not (isinstance(v, torch.Tensor) and v.is_cuda):
            raise RuntimeError('hand_collision_count: %s must be a CUDA tensor (there is no CPU path)' % name)
        if v.dtype not in (torch.float32, torch.float64):
            raise TypeError('hand_collision_count: %s must be float32 or float64, got %s' % (name, v.dtype))
    if verts_a.dtype != verts_b.dtype:
        raise TypeError('hand_collision_count: verts_a is %s, verts_b %s' % (verts_a.dtype, verts_b.dtype))
    if verts_a.dim() != 3 or verts_a.shape[0] < 1 or verts_a.shape[2] != 3 or not 3 <= verts_a.shape[1] <= MAX_VERTS:
        raise ValueError('hand_collision_count: verts_a must be [B,V,3] with B >= 1, 3 <= V <= %d, got %s' % (MAX_VERTS, tuple(verts_a.shape)))
    if verts_b.shape != verts_a.shape:
        raise ValueError('hand_collision_count: verts_b must be %s like verts_a, got %s' % (tuple(verts_a.shape), tuple(verts_b.shape)))
    dev = verts_a.device
    if verts_b.device != dev:
        raise RuntimeError('hand_collision_count: verts_a is on %s, verts_b on %s' % (dev, verts_b.device))
    B, V = verts_a.shape[0], verts_a.shape[1]
    f = _checked_faces(faces, V, dev)
    ts = []
    for name, t in (('trans_a', trans_a), ('trans_b', trans_b)):
        if t is not None:
            if not (isinstance(t, torch.Tensor) and t.is_cuda):
                raise RuntimeError('hand_collision_count: %s must be a CUDA tensor (there is no CPU path)' % name)
            if not t.dtype.is_floating_point:
                raise TypeError('hand_collision_count: %s must be a floating-point tensor, got %s' % (name, t.dtype))
            if tuple(t.shape) != (B, 3):
                raise ValueError('hand_collision_count: %s must be [%d,3], got %s' % (name, B, tuple(t.shape)))
            if t.device != dev:
                raise RuntimeError('hand_collision_count: %s is on %s, the vertices on %s' % (name, t.device, dev))
            t = t.to(torch.float64).contiguous()
        ts.append(t)
    if stats is not None and not (isinstance(stats, torch.Tensor) and stats.device == dev and stats.dtype == torch.int64
                                  and tuple(stats.shape) == (B, 2) and stats.is_contiguous()):
        raise ValueError('hand_collision_count: stats must be a contiguous int64 [%d,2] tensor on %s' % (B, dev))
    va, vb = verts_a.contiguous(), verts_b.contiguous()
    count = torch.empty(B, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        call('rih_hand_collision_count', va.data_ptr(), vb.data_ptr(), int(va.dtype == torch.float64),
             None if ts[0] is None else ts[0].data_ptr(), None if ts[1] is None else ts[1].data_ptr(), f.data_ptr(), V, f.shape[0], B,
             count.data_ptr(), None if stats is None else stats.data_ptr(), _stream(va))
    return count


# ---------------------------------------------------------------------------------------------------------------- the filter
def filtered_records(raw_data, keep):
    """copy_dict_struct + dict_add over the kept frames (CollisionFilter.py:9-25, :121-123), vectorised: raw_data a nested dict whose
    leaves are indexed by frame, keep [N] bool -> the dict the reference saves."""
    kept = np.nonzero(np.asarray(keep, bool))[0]

    def build(d):
        out = {}
        for k, v in d.items():
            if isinstance(v, dict):
                out[k] = build(v)
            elif len(kept) == 0:
                out[k] = np.asarray([])
            else:
                a = np.asarray(v)[np.concatenate([kept[:1], kept])]     # np.row_stack of [i:i+1] slices, the first one twice
                out[k] = a.reshape(-1, 1) if a.ndim == 1 else a
        return out
    return build(raw_data)


def filter_collision_data(target_data_path, out_put_path, mano_root='../assets/mano', max_contacts=75, batch_size=4096, device='cuda'):
    """filter_collision_data (CollisionFilter.py:41-127): loads the optimised mocap dict at target_data_path, counts each frame's
    intersecting face pairs on the GPU, saves the frames with at most max_contacts of them with np.save(out_put_path, ...) in the
    reference's layout, prints the kept fraction and returns it.  mano_root: a directory with MANO_RIGHT.pkl / MANO_LEFT.pkl, or
    {'right': mano dict, 'left': mano dict}."""
    from .geo_loss import _rest_pose, converter_matrices
    from .manopth import ManoLayer
    from .mocap_optimize import euler_to_mano_quat
    dev = torch.device(device)
    if dev.type != 'cuda':
        raise RuntimeError('filter_collision_data: a CUDA device is required (there is no CPU path)')
    raw = np.load(target_data_path, allow_pickle=True).item()
    roots = mano_root if isinstance(mano_root, dict) else {'right': mano_root, 'left': mano_root}
    layer = {s: ManoLayer(mano_root=roots[s], side=s, use_pca=False, ncomps=6, flat_hand_mean=True, center_idx=0, root_rot_mode='quat',
                          joint_rot_mode='quat').to(dev) for s in ('right', 'left')}
    faces = layer['left'].th_faces.to(dev)
    n = len(raw['right']['loc'])
    counts = []
    with torch.no_grad():
        conv = {s: converter_matrices(s, *_rest_pose(layer[s], dev)[1:]) for s in ('right', 'left')}
        hand = {}
        for s in ('right', 'left'):
            hand[s] = (torch.from_numpy(euler_to_mano_quat(raw[s]['rot'], s, *conv[s])), torch.from_numpy(np.asarray(raw[s]['loc']) * 1.0 / 100),
                       torch.from_numpy(np.asarray(raw[s]['shape']).astype(np.float32)))
        for s0 in range(0, n, batch_size):
            v = {}
            for s in ('right', 'left'):
                q, loc, shape = (t[s0:s0 + batch_size].to(dev) for t in hand[s])
                v[s] = (layer[s](q, shape.reshape(len(q), -1))[0], loc)
            counts.append(hand_collision_count(v['right'][0], v['left'][0], faces, v['right'][1], v['left'][1]))
    keep = (torch.cat(counts) <= max_contacts).cpu().numpy()
    np.save(out_put_path, filtered_records(raw, keep))
    frac = int(keep.sum()) / n
    print(frac)
    return frac
