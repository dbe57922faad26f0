"""The mocap pose optimiser's driver on the GPU: a drop-in for pose_data_optimize/batch_optimize_mocap_origin.py (step 3 of the pipeline in
pose_data_optimize/README.md), the only caller of GeOptimizer, on its discrete path (discrete_optimize = True, :340).

    scene = Scene(mano_root='assets/mano', anchor_root='assets/anchor')          # both hand models and the anchor tables, read once
    info = scene.update_scene(hand_pose, sub_hand_pose, hand_tsl, sub_hand_tsl, hand_shape, anchor_id=None)   # [B] frames, one launch
    out_dict = run_sample(device, hoptim, info)                                    # set_opt_val + optimize
    optimized = optimize_mocap(raw_data, hoptim, scene, batch_size, optimize_interval, mocap_scale)      # main's four attempts
    main(args)                                                                     # the reference's argparse namespace (:743-786)

Scene.update_scene is the reference's update_scene (:227-317) and search_anchors (:62-130) for a whole batch of frames: both hands through
renderih_b200.manopth.ManoLayer (quat, flat_hand_mean=True, center_idx as main builds them, :429-450), then csrc/scene.cu
(rih_mocap_search_anchors), one CTA per frame.  It returns the frames stacked as combine_frame_inf (:320-335) stacks them, as CUDA tensors
in the dtypes run_sample converts them to (:706-734):

* vertex_contact [B,108], hand_region [B,108] (zeros), anchor_id / anchor_padding_mask [B,108,4]: int64;
* anchor_elasti [B,108,4], obj_anchors / obj_normals [B,108,3], hand_pose / obj_pose [B,16,4], hand_tsl / obj_tsl [B,3], hand_shape
  [B,20]: float32;  optimize_it [B,1]: bool (:533-538).

Conventions reproduced:

* Geometry (:256-270): vertices + translation in float32; anchors (recover_anchor, anchorutils.py:51-62) in float64, because the anchor
  weights come from np.loadtxt as float64; the face normals at the anchor faces in float32 in numpy's order (cross, norm, divide), the
  sub-hand normal negated.  Distances, the 0.015 / 0.02 thresholds and 0.5 cos(pi d / t) + 0.5 in float64; elasticities stored as float32.
* Fresh branch (anchor_id=None, :116-127): a main anchor is a candidate for sub anchor i unless sub_normal_i . main_normal_j > -0.6
  (float32); other distances become 1000.0.  contact_able = d < 0.015; the 4 smallest distances give anchor_id, with their elasticities;
  anchor_padding_mask = elasticity > 0; vertex_contact = any(contact_able).
* Previous-id branch (:75-91): distances at the given ids only, no normal mask, threshold 0.02.
* Both branches (:129): elasticities are scaled by 0.3 unless the sub anchor's or the main anchor's merged_vertex_assignment class is 4
  (the shipped table has no class 4, so the factor applies everywhere).
* optimize_mocap, main's discrete path (:373-593): frame subsampling by optimize_interval; euler -> MANO quaternions once on the host in
  float64 with scipy, as HandPoseConverter.euler_2_mano_quat / mano_quat_2_euler (HandPoseConverter.py:164-212) with the converter
  matrices of renderih_b200.geo_loss; four attempts scaling the initial coef_val (lambda_repulsion_loss x1, x0.1, x30, x1;
  lambda_contact_loss x1, x15, x0.1, x5) with n_iter 50, 40, 75, 50 (:460-479); anchor ids recomputed over all frames at attempts 0 and 3
  and reused at attempts 1 and 2 (:484-501); batches of batch_size, the last one partial (:513-560); the consistency masks are zeros,
  since discrete_optimize multiplies get_joint_change by 0 (:509-511).  Pose and translation state stays on the device across attempts;
  GeOptimizer.optimize() returns CPU tensors, which are copied back.
* The reference's quirks: hand_shape is taken from the un-subsampled shape arrays (:391-398; frame k of the subsampled sequence uses the
  shape row k); the returned dict's 'rot' has the subsampled length and 'loc' is scaled by 100; 'shape' becomes [N,10] float32 for each
  side (:397-398, :582-585).

Deviations:

* Ties: np.argsort's default sort is not stable, and masked candidates tie at exactly 1000.0.  Here ties go to the lowest index.  The
  choice matters: attempts 1 and 2 re-evaluate those ids without the normal mask.
* Translations are float32 throughout.  The reference holds them in float64; its first anchor pass adds the float64 mocap translations to
  the float32 vertices, every later pass sees float32 values (the optimiser's outputs).
* The normals' dot product is summed left to right in float32; the reference's BLAS may order or fuse it differently (rounding level).
* get_anchor_similarity and filter_anchor_id / filter_quat_loc are not computed: discrete_optimize discards them (:503-504, :575-577).
* update_scene does not return the keys only visualisation reads (hand_verts_3d, hand_joints_3d, obj_verts_3d, hand_face, :662-703), nor
  those run_sample never reads; vis=True raises NotImplementedError (there is no open3d viewer).  The anchor tables are read once at
  construction, as geo_loss.AnchorLayer reads them; the reference's per-frame anchor_load_driver also opens anchor_mapping_path.pkl, which
  the tree does not ship.

CPU tensors raise RuntimeError, non-float32 poses / translations / shapes TypeError, wrong shapes or anchor ids outside [0, 108)
ValueError.
"""
import os

import numpy as np
import torch
from scipy.spatial.transform import Rotation

from ._lib import call
from .assets import default_asset_root
from .geo_loss import ANCHOR_DIR, _rest_pose, anchor_tables, converter_matrices
from .manopth import ManoLayer

SHAPE_DIM = 10
DIM = 4                                                   # search_anchors' `dim`
# main's four attempts (:460-479): (lambda_repulsion_loss factor, lambda_contact_loss factor, n_iter)
ATTEMPTS = ((1.0, 1.0, 50), (0.1, 15.0, 40), (30.0, 0.1, 75), (1.0, 5.0, 50))
ANCHOR_ATTEMPTS = (0, 3)                                  # attempts that recompute the anchor ids (:484)
_FLIP = np.asarray(([1, 0, 0], [0, -1, 0], [0, 0, -1]))   # HandPoseConverter.py:175-176, :199-200


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _check(name, t, shape, device=None):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError('mocap_optimize: %s must be a CUDA tensor (there is no CPU path)' % name)
    if t.dtype != torch.float32:
        raise TypeError('mocap_optimize: %s must be float32, got %s' % (name, t.dtype))
    if tuple(t.shape) != tuple(shape):
        raise ValueError('mocap_optimize: %s must be %s, got %s' % (name, list(shape), tuple(t.shape)))
    if device is not None and t.device != device:
        raise RuntimeError('mocap_optimize: %s is on %s, expected %s' % (name, t.device, device))
    return t.contiguous()


# ---------------------------------------------------------------------------------------------------------------- host conversions
def euler_to_mano_quat(euler, side, inv_m0, inv_u1):
    """HandPoseConverter.euler_2_mano_quat (HandPoseConverter.py:164-188): euler [N,16,3] or [16,3] ('xyz', degrees) -> [N,16,4] float32
    MANO quaternions (w,x,y,z), in float64 with scipy.  inv_m0 / inv_u1: the converter matrices of this side (geo_loss.converter_matrices)."""
    e = np.asarray(euler)
    if e.ndim == 2:
        e = e[np.newaxis]
    n, J = e.shape[0], e.shape[1]
    mat = np.zeros([n, J, 3, 3])
    for j in range(J):
        mat[:, j] = Rotation.from_euler('xyz', e[:, j, :], degrees=True).as_matrix()
    mat = inv_m0 @ mat @ inv_u1
    if side == 'left':
        mat[:, 0] = np.tile(_FLIP[np.newaxis], (len(mat), 1, 1)) @ mat[:, 0]
    q = Rotation.from_matrix(mat.reshape(-1, 3, 3)).as_quat()
    if q.ndim <= 1:
        q = q[np.newaxis]
    q = q[:, [3, 0, 1, 2]].reshape(-1, J, 4)
    if side == 'left':
        q[:, :, 2] = -q[:, :, 2]
        q[:, :, 3] = -q[:, :, 3]
    return q.astype(np.float32)


def mano_quat_to_euler(quat, side, inv_m0, inv_u1):
    """HandPoseConverter.mano_quat_2_euler (HandPoseConverter.py:190-212): [N,16,4] or [16,4] MANO quaternions -> [N,16,3] float64 euler
    angles ('xyz', degrees).  Unlike the reference, the input array is not modified."""
    q = np.array(quat)
    if q.ndim <= 2:
        q = q[np.newaxis]
    n, J = q.shape[0], q.shape[1]
    if side == 'left':
        q[:, :, 2] = -q[:, :, 2]
        q[:, :, 3] = -q[:, :, 3]
    q = q.reshape(-1, 4)
    mat = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix().reshape(-1, J, 3, 3)
    if side == 'left':
        mat[:, 0] = np.tile(_FLIP[np.newaxis], (len(mat), 1, 1)) @ mat[:, 0]
    mat = inv_m0.swapaxes(1, 2) @ mat @ inv_u1.swapaxes(1, 2)
    out = np.zeros([n, J, 3])
    for j in range(J):
        out[:, j] = Rotation.from_matrix(mat[:, j]).as_euler('xyz', degrees=True)
    return out


# ---------------------------------------------------------------------------------------------------------------- scene
class Scene:
    """Both hand models and the anchor tables of the mocap driver (main, :429-450, and anchor_load_driver, :245).  mano_root: a directory
    with MANO_RIGHT.pkl / MANO_LEFT.pkl, or {'right': mano dict, 'left': mano dict}.  The anchor tables come from anchor_root's
    face_vertex_idx.txt, anchor_weight.txt and merged_vertex_assignment.txt, or from the arrays given (geo_loss.anchor_tables)."""

    def __init__(self, mano_root='assets/mano', anchor_root=None, face_vert_idx=None, anchor_weight=None, class_types=None, center_idx=0,
                 device='cuda'):
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('Scene: a CUDA device is required (there is no CPU path)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        roots = mano_root if isinstance(mano_root, dict) else {'right': mano_root, 'left': mano_root}
        quat = dict(joint_rot_mode='quat', root_rot_mode='quat', use_pca=False, ncomps=6, flat_hand_mean=True, center_idx=center_idx,
                    return_transf=True)
        self.main_hand = ManoLayer(mano_root=roots['right'], side='right', **quat).to(self.device)
        self.sub_hand = ManoLayer(mano_root=roots['left'], side='left', **quat).to(self.device)
        fvi, aw = anchor_tables(anchor_root, face_vert_idx, anchor_weight)
        if class_types is None:
            root = anchor_root if anchor_root is not None else os.path.join(default_asset_root(), ANCHOR_DIR)
            class_types = np.loadtxt(os.path.join(root, 'merged_vertex_assignment.txt'), dtype=np.int64)
        cls = np.asarray(class_types).reshape(-1)
        if cls.shape[0] != fvi.shape[0] or not np.issubdtype(cls.dtype, np.integer):
            raise ValueError('class_types must be %d integers, got %s %s' % (fvi.shape[0], cls.dtype, cls.shape))
        if fvi.shape[0] < DIM:
            raise ValueError('search_anchors needs at least %d anchors, got %d' % (DIM, fvi.shape[0]))
        self.n_anchors = fvi.shape[0]
        self._fvi = torch.from_numpy(fvi.astype(np.int32)).to(self.device)
        self._aw = torch.from_numpy(aw).to(self.device)
        self._cls = torch.from_numpy(cls.astype(np.int32)).to(self.device)
        self.converter = {}
        with torch.no_grad():
            for side, layer in (('right', self.main_hand), ('left', self.sub_hand)):
                _, joints, transf = _rest_pose(layer, self.device)
                self.converter[side] = converter_matrices(side, joints, transf)

    def update_scene(self, hand_pose, sub_hand_pose, hand_tsl, sub_hand_tsl, hand_shape, anchor_id=None):
        """update_scene (:227-317) for B frames: poses [B,16,4], translations [B,3], shapes [B,20] (right betas, then left), anchor_id
        None or [B,A,4] integer ids in [0,A) -> the stacked frame-info dict (module docstring).  Validating anchor_id synchronises once."""
        dev = self.device
        B = hand_pose.shape[0] if isinstance(hand_pose, torch.Tensor) and hand_pose.dim() == 3 else -1
        hand_pose = _check('hand_pose', hand_pose, (B, 16, 4), dev)
        sub_hand_pose = _check('sub_hand_pose', sub_hand_pose, (B, 16, 4), dev)
        hand_tsl = _check('hand_tsl', hand_tsl, (B, 3), dev)
        sub_hand_tsl = _check('sub_hand_tsl', sub_hand_tsl, (B, 3), dev)
        hand_shape = _check('hand_shape', hand_shape, (B, 2 * SHAPE_DIM), dev)
        if B < 1:
            raise ValueError('mocap_optimize: update_scene needs at least one frame')
        A = self.n_anchors
        prev = None
        if anchor_id is not None:
            if not (isinstance(anchor_id, torch.Tensor) and anchor_id.is_cuda):
                raise RuntimeError('mocap_optimize: anchor_id must be a CUDA tensor (there is no CPU path)')
            if anchor_id.dtype.is_floating_point or anchor_id.dtype.is_complex or anchor_id.dtype == torch.bool:
                raise TypeError('mocap_optimize: anchor_id must be an integer tensor, got %s' % anchor_id.dtype)
            if tuple(anchor_id.shape) != (B, A, DIM):
                raise ValueError('mocap_optimize: anchor_id must be [%d,%d,%d], got %s' % (B, A, DIM, tuple(anchor_id.shape)))
            if anchor_id.device != dev:
                raise RuntimeError('mocap_optimize: anchor_id is on %s, expected %s' % (anchor_id.device, dev))
            lo, hi = torch.stack([anchor_id.min(), anchor_id.max()]).tolist()
            if lo < 0 or hi >= A:
                raise ValueError('mocap_optimize: anchor_id must lie in [0, %d), got [%d, %d]' % (A, lo, hi))
            prev = anchor_id.to(torch.int64).contiguous()
        with torch.no_grad():
            v_main = self.main_hand(hand_pose, hand_shape[:, :SHAPE_DIM])[0]
            v_sub = self.sub_hand(sub_hand_pose, hand_shape[:, SHAPE_DIM:])[0]
        ids = torch.empty(B, A, DIM, dtype=torch.int64, device=dev)
        elasti = torch.empty(B, A, DIM, device=dev)
        pad = torch.empty(B, A, DIM, dtype=torch.int64, device=dev)
        contact = torch.empty(B, A, dtype=torch.int64, device=dev)
        opt_it = torch.empty(B, 1, dtype=torch.bool, device=dev)
        anchors = torch.empty(B, A, 3, device=dev)
        normals = torch.empty(B, A, 3, device=dev)
        with torch.cuda.device(dev):
            call('rih_mocap_search_anchors', v_main.data_ptr(), v_sub.data_ptr(), hand_tsl.data_ptr(), sub_hand_tsl.data_ptr(),
                 self._fvi.data_ptr(), self._aw.data_ptr(), self._cls.data_ptr(), A, None if prev is None else prev.data_ptr(), B,
                 ids.data_ptr(), elasti.data_ptr(), pad.data_ptr(), contact.data_ptr(), opt_it.data_ptr(), anchors.data_ptr(),
                 normals.data_ptr(), _stream(v_main))
        return {'vertex_contact': contact, 'hand_region': torch.zeros(B, A, dtype=torch.int64, device=dev), 'anchor_id': ids,
                'anchor_elasti': elasti, 'anchor_padding_mask': pad, 'hand_pose': hand_pose, 'hand_shape': hand_shape, 'hand_tsl': hand_tsl,
                'obj_tsl': sub_hand_tsl, 'obj_pose': sub_hand_pose, 'obj_anchors': anchors, 'obj_normals': normals, 'optimize_it': opt_it}


# ---------------------------------------------------------------------------------------------------------------- driver
def run_sample(device, hoptim, info, hand_closed_path=None, vis=False):
    """run_sample (:654-738): set_opt_val's keyword arguments from an update_scene dict (plus info['batch_size']), with no host round
    trip, then hoptim.optimize().  The consistency masks are zeros (discrete_optimize, :509-511)."""
    if vis:
        raise NotImplementedError('run_sample: vis is not supported (there is no open3d viewer)')
    B = int(info['batch_size'])
    hand_pose, obj_pose = info['hand_pose'], info['obj_pose']
    zeros = torch.zeros(B, 16, device=hand_pose.device)
    hoptim.set_opt_val(vertex_contact=info['vertex_contact'], contact_region=info['hand_region'], anchor_id=info['anchor_id'],
                       anchor_elasti=info['anchor_elasti'], anchor_padding_mask=info['anchor_padding_mask'], hand_shape_init=info['hand_shape'],
                       hand_tsl_init=info['hand_tsl'], hand_pose_gt=([0], hand_pose[:, 0:1, :]),
                       hand_pose_init=(list(range(1, 16)), hand_pose[:, 1:, :]), runtime_vis=9527, obj_tsl_init=info['obj_tsl'],
                       obj_pose_gt=([0], obj_pose[:, 0:1, :]), obj_pose_init=(list(range(1, 16)), obj_pose[:, 1:, :]),
                       obj_anchors=info['obj_anchors'], obj_normals=info['obj_normals'], optimize_it=info['optimize_it'], batch_size=B,
                       consistent_mask=[zeros, zeros])
    return hoptim.optimize(progress=False)


def attempt_table(lambda_repulsion, lambda_contact):
    """[(lambda_repulsion_loss, lambda_contact_loss, n_iter, recompute anchor ids)] of main's four attempts (:460-501)."""
    return [(lambda_repulsion * fr, lambda_contact * fc, n, k in ANCHOR_ATTEMPTS) for k, (fr, fc, n) in enumerate(ATTEMPTS)]


def optimize_mocap(raw_data, hoptim, scene, batch_size, optimize_interval=1, mocap_scale=1.0):
    """main's discrete path (:373-593) on a loaded mocap dict {'right': {'rot' [N,16,3], 'loc' [N,3], 'shape' [N,1,10]}, 'left': ...}
    -> the dict main saves: raw_data's structure with each side's 'rot' (euler, subsampled), 'loc' (x100, subsampled) and 'shape'
    ([N,10] float32) replaced.  raw_data itself is not modified."""
    if batch_size < 1 or optimize_interval < 1:
        raise ValueError('optimize_mocap: batch_size and optimize_interval must be >= 1')
    dev = scene.device
    frames = np.arange(0, len(raw_data['right']['rot']), optimize_interval)                    # :374-383
    quat, tsl = {}, {}
    for side in ('right', 'left'):
        quat[side] = torch.from_numpy(euler_to_mano_quat(np.asarray(raw_data[side]['rot'])[frames], side, *scene.converter[side])).to(dev)
        loc = np.asarray(raw_data[side]['loc'])[frames] / 100 * mocap_scale                       # load_mocap_data, :387-388
        tsl[side] = torch.from_numpy(np.ascontiguousarray(loc, dtype=np.float32)).to(dev)
    shape = torch.cat([torch.from_numpy(np.asarray(raw_data[s]['shape']).astype(np.float32)).squeeze(1) for s in ('right', 'left')], 1)
    n = len(frames)
    if shape.shape[0] < n:
        raise ValueError('optimize_mocap: %d shape rows for %d frames' % (shape.shape[0], n))
    shape_dev = shape[:n].to(dev)                                # frame k uses shape row k of the un-subsampled arrays (:391-398, :493)
    base = (hoptim.coef_val['lambda_repulsion_loss'], hoptim.coef_val['lambda_contact_loss'])
    ids = torch.empty(n, scene.n_anchors, DIM, dtype=torch.int64, device=dev)
    for rep, con, n_iter, recompute in attempt_table(*base):
        hoptim.coef_val['lambda_repulsion_loss'] = rep
        hoptim.coef_val['lambda_contact_loss'] = con
        hoptim.n_iter = n_iter
        for s in range(0, n, batch_size):
            e = min(s + batch_size, n)
            if recompute:                                        # the anchor pass over all frames precedes the batches (:484-501)
                ids[s:e] = scene.update_scene(quat['right'][s:e], quat['left'][s:e], tsl['right'][s:e], tsl['left'][s:e],
                                              shape_dev[s:e])['anchor_id']
        for s in range(0, n, batch_size):
            e = min(s + batch_size, n)
            info = scene.update_scene(quat['right'][s:e], quat['left'][s:e], tsl['right'][s:e], tsl['left'][s:e], shape_dev[s:e],
                                      anchor_id=ids[s:e])
            info['batch_size'] = e - s
            res = run_sample(dev, hoptim, info)
            quat['right'][s:e].copy_(res['optimized_hand_pose'])
            tsl['right'][s:e].copy_(res['optimized_hand_tsl'])
            quat['left'][s:e].copy_(res['optimized_sub_hand_pose'])
            tsl['left'][s:e].copy_(res['optimized_sub_hand_tsl'])
    out = {k: (dict(v) if isinstance(v, dict) else v) for k, v in raw_data.items()}
    for side, cols in (('right', slice(0, SHAPE_DIM)), ('left', slice(SHAPE_DIM, None))):
        out[side]['rot'] = mano_quat_to_euler(quat[side].cpu().numpy(), side, *scene.converter[side])
        out[side]['loc'] = tsl[side].cpu().numpy().astype(np.float64) * 100
        out[side]['shape'] = shape.numpy()[:, cols]
    return out


def main(args):
    """main (:338-593) with the reference's argparse namespace (:743-786): builds the optimiser and the scene, loads args.mocap_path, runs
    optimize_mocap and saves args.optimized_mocap_path with np.save.  With args.reoptimize_raw it converts that file's quaternions to
    euler angles and saves them instead (:350-371)."""
    from .ge_optimizer import GeOptimizer
    if getattr(args, 'vis', False):
        raise NotImplementedError('main: --vis is not supported (there is no open3d viewer)')
    device = 'cuda:%s' % args.gpu
    scene = Scene(mano_root=args.mano_root, anchor_root=args.anchor_root, center_idx=args.center_idx, device=device)
    if args.reoptimize_raw != '':
        raw = np.load(args.reoptimize_raw, allow_pickle=True).item()
        out = {side: {'rot': mano_quat_to_euler(raw[side]['rot'], side, *scene.converter[side]), 'loc': raw[side]['loc'] * 100}
               for side in ('right', 'left')}
        np.save(args.optimized_mocap_path, {'right': out['right'], 'left': out['left']})
        return
    raw_data = np.load(args.mocap_path, allow_pickle=True).item()
    torch.manual_seed(args.manual_seed)                          # set_all_seeds (:25-29)
    np.random.seed(args.manual_seed)
    hoptim = GeOptimizer(device, lr=1e-2, n_iter=100, verbose=False, mano_root=args.mano_root, anchor_path=args.anchor_root,
                         lambda_contact_loss=args.lambda_contact_loss, lambda_repulsion_loss=args.lambda_repulsion_loss,
                         repulsion_query=args.repulsion_query, repulsion_threshold=args.repulsion_threshold, mode='both')
    out = optimize_mocap(raw_data, hoptim, scene, args.batch_size, args.optimize_interval, args.mocap_scale)
    np.save(args.optimized_mocap_path, out)
