"""The pose data pipeline's conversion and augmentation stages on the GPU (steps 1, 2 and 4 of pose_data_optimize/README.md): drop-ins for
scripts/HandPoseConverter.py, scripts/HandPoseArguer.py, Ver2Code/NatureJudge/PoseArgue.py and the scripts that drive them
(data/template_0_pose_convert.py, template_1_pose_argue.py, template_3_pose_reconvert.py, Ver2Code/NatureJudge/data_birth.py).

    hpc = HandPoseConverter(side='left', root='assets/mano')      # root: a MANO directory or a MANO dict of this side
    quat = hpc.euler_2_mano_quat(euler)                           # [N,16,3] degrees -> [N,16,4] float32, one launch (csrc/pose_data.cu)
    poses = HandPoseArguer(side='right').argue_pose(euler, argue_size=5, pose_type='euler')      # [N*5,16,3], one launch
    poses = PoseArguer(side='right').argue_pose(euler, 15, 'euler', random_level=0.7, generator=seed)   # device Philox draws
    convert_annotations(annots) / argue_data(data, ...) / reconvert_optimized(paths, template, ...) / birth_data(data, ...)

Every rotation is a float64 device statement of the scipy Rotation calls the reference makes (from_euler / as_matrix / from_matrix /
as_euler 'xyz' in degrees, from_rotvec / as_rotvec, from_quat); csrc/pose_data.cu lists their branch rules.  numpy input, which is what
every reference caller passes, is staged through the GPU and returned as numpy; CUDA tensors stay on the device (float64 for euler
angles and HandPoseConverter.mano_quat_2_euler's quaternions, float32 or float64 where the reference casts to float32 itself).  CPU
torch tensors raise RuntimeError, other dtypes TypeError, wrong shapes ValueError.  No call synchronises with the host except the copy
back of numpy results.

Augmentation (HandPoseArguer.py:33-173, PoseArgue.py:34-174): for each frame i, copy a and joint, the adjustment (pos - neg) u + neg of
angle_random_adjust with the bounds from the frame's original angle (z: bend, y: splank), then euler(R(e) Rz(bend)) and from that
euler(R(.) Ry(splank)).  The uniforms come either from numpy's global RandomState in the reference's order (all bend draws frame-major,
joints 2,5,11,8, 13, 14, 3,6,12,9,15, 1,4,10,7, argue_size each; then all splank draws, joints 1,4,10,7,13), so np.random.seed(s)
gives the reference's poses, or, with generator= (an int seed or a CUDA torch.Generator), from Philox-4x32-10 on the device.

Reproduced quirks:
* argue_pose round-trips every joint through both adjustments, the unadjusted ones too: joint 0 and, in the splank pass, every joint
  but the five bases (HandPoseArguer.py:51-52, 82-96);
* birth_data converts both hands with the right-hand converter (data_birth.py:24, 43);
* with add_origin, birth_data appends the raw euler rows to the axis-angle output (data_birth.py:49-52), and its confidence is 1.0
  for them.

Deviations:
* inputs are never modified; the reference's mano_quat_2_euler and mano_quat_flat_2_normal negate a left hand's array in place
  (HandPoseConverter.py:195-197, 311-313);
* no scipy gimbal-lock UserWarning; a matrix with non-positive determinant gives NaN instead of scipy's ValueError;
* axis_angle_2_mano_quat and mano_quat_flat_2_normal take order='wxyz' only, the order every pipeline script uses;
* euler input to argue_pose is taken as float64 (the reference keeps a float32 array's dtype for its adjustments);
* vis=True raises NotImplementedError (there is no open3d viewer).
"""
import copy
import os

import numpy as np
import torch

from ._lib import call
from .assets import load_mano_dict
from .geo_loss import CONVERTER_BETAS, _rest_pose, converter_matrices
from .manopth import ManoLayer

# bend_argue's (HandPoseArguer.py:117-127) and splank_argue's (:145-146) joint ranges in draw order; PoseArguer differs in the normal
# bend range and the splank ranges (PoseArgue.py:118-147)
_BEND_LISTS = (((2, 5, 11, 8), (-8, 110)), ((13,), (-20, 40)), ((14,), (-8, 50)), ((3, 6, 12, 9, 15), None), ((1, 4, 10, 7), (-25, 70)))
SPLANK_JOINTS = (1, 4, 10, 7, 13)
BEND_JOINTS = tuple(j for js, _ in _BEND_LISTS for j in js)
N_DRAWS = len(BEND_JOINTS) + len(SPLANK_JOINTS)


def _ranges(normal_bend, splank):
    rows = []
    for js, r in _BEND_LISTS:
        rows += [r if r is not None else normal_bend] * len(js)
    return np.asarray(rows + list(splank), dtype=np.float64)


_NP = {torch.float32: np.float32, torch.float64: np.float64}


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _stage(who, x, dtypes, device):
    """-> (CUDA tensor, came_from_numpy).  numpy / lists go to the device in dtypes[0]; CUDA tensors of a dtype in dtypes are taken as they
    are (the first dtype is what the kernel reads: a float32 tensor is widened, a float64 one rounded as numpy would)."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise RuntimeError('%s: a CUDA tensor or a numpy array is required, got a CPU tensor (there is no CPU path)' % who)
        if x.dtype not in dtypes:
            raise TypeError('%s: expected %s, got %s' % (who, ' or '.join(str(d) for d in dtypes), x.dtype))
        return x.to(dtypes[0]).contiguous(), False
    a = np.asarray(x)
    if not (np.issubdtype(a.dtype, np.floating) or np.issubdtype(a.dtype, np.integer)):
        raise TypeError('%s: expected a numeric array, got %s' % (who, a.dtype))
    return torch.from_numpy(np.ascontiguousarray(a, dtype=_NP[dtypes[0]])).to(device), True


def _shape(who, t, shape):
    if tuple(t.shape) != tuple(shape) or t.shape[0] < 1:
        raise ValueError('%s: expected shape %s with N >= 1, got %s' % (who, list(shape), tuple(t.shape)))


def _out(t, numpy):
    return t.cpu().numpy() if numpy else t


class HandPoseConverter:
    """HandPoseConverter(shape=None, side='right', root='../assets/mano', data_type='np', device='cuda:0') (HandPoseConverter.py:29-79).
    root: a MANO directory, a MANO dict of this side or {'right': dict, 'left': dict}.  The converter matrices come from the rest pose through renderih_b200.manopth.ManoLayer (geo_loss.converter_matrices), float32 as the
    reference stores them; hands_mean from the MANO dict."""

    def __init__(self, shape=None, side='right', root='../assets/mano', data_type='np', device='cuda:0'):
        if side not in ('right', 'left'):
            raise ValueError("side must be 'right' or 'left', got %r" % (side,))
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('HandPoseConverter: a CUDA device is required (there is no CPU path)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.side = side
        if isinstance(root, dict):       # the layer negates the left hand's shapedirs in place: give it a copy, not the caller's array
            mano = dict(root[side] if side in root else root)
            mano['shapedirs'] = np.array(mano['shapedirs'], dtype=np.float32)
        else:
            mano = load_mano_dict(os.path.join(root, 'MANO_%s.pkl' % side.upper()))
        self.mano_layer = ManoLayer(mano_root=mano, use_pca=False, ncomps=6, flat_hand_mean=True, center_idx=9, return_transf=True, side=side,
                                    root_rot_mode='quat', joint_rot_mode='quat').to(self.device)
        self.shape = torch.tensor([CONVERTER_BETAS]) if shape is None else shape
        self.faces = np.asarray(mano['f']).astype(np.int64)
        self.joint_idx = np.asarray([[0, 1, 2, 3, 4], [0, 5, 6, 7, 8], [0, 9, 10, 11, 12], [0, 13, 14, 15, 16], [0, 17, 18, 19, 20]])
        self.axis_idx = np.asarray([[0, 13, 14, 15], [0, 1, 2, 3], [0, 4, 5, 6], [0, 10, 11, 12], [0, 7, 8, 9]])
        with torch.no_grad():
            self.invM_U_n_0, self.invU_M_n_1 = converter_matrices(side, *_rest_pose(self.mano_layer, self.device)[1:])
        self._conv_src = None
        self.data_type = data_type
        if data_type == 'tensor':
            self.invU_M_n_1 = torch.from_numpy(self.invU_M_n_1).to(self.device)
            self.invM_U_n_0 = torch.from_numpy(self.invM_U_n_0).to(self.device)
        self.th_hands_mean = np.asarray(mano['hands_mean'], dtype=np.float32).reshape(1, 15, 3)
        self._hands_mean = torch.from_numpy(self.th_hands_mean.reshape(45)).to(self.device)
        self._left = 1 if side == 'left' else 0

    def _tables(self):
        """[16,18] float32 on the device: invM_U_n_0 then invU_M_n_1 per joint, rebuilt whenever either attribute has been reassigned."""
        src = (self.invM_U_n_0, self.invU_M_n_1)
        if self._conv_src is None or any(a is not b for a, b in zip(src, self._conv_src)):
            m = [np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float32).reshape(16, 9) for x in src]
            self._conv = torch.from_numpy(np.concatenate(m, 1)).to(self.device)
            self._conv_src = src
        return self._conv

    def euler_2_mano_quat(self, euler_list):
        """(N,16,3) or (16,3) euler angles ('xyz', degrees) -> (N,16,4) float32 MANO quaternions (w,x,y,z) (:159-188)."""
        e, np_in = _stage('euler_2_mano_quat', euler_list, (torch.float64,), self.device)
        e = e[None] if e.dim() == 2 else e
        _shape('euler_2_mano_quat', e, (e.shape[0], 16, 3))
        q = torch.empty(e.shape[0], 16, 4, device=self.device)
        with torch.cuda.device(self.device):
            call('rih_pose_euler_to_mano_quat', e.data_ptr(), e.shape[0], self._left, self._tables().data_ptr(), q.data_ptr(), _stream(e))
        return _out(q, np_in)

    def mano_quat_2_euler(self, batch_quat):
        """(N,16,4) or (16,4) MANO quaternions -> (N,16,3) float64 euler angles ('xyz', degrees) (:190-212)."""
        q, np_in = _stage('mano_quat_2_euler', batch_quat, (torch.float64, torch.float32), self.device)
        q = q[None] if q.dim() <= 2 else q
        _shape('mano_quat_2_euler', q, (q.shape[0], 16, 4))
        e = torch.empty(q.shape[0], 16, 3, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            call('rih_pose_mano_quat_to_euler', q.data_ptr(), q.shape[0], self._left, self._tables().data_ptr(), e.data_ptr(), _stream(q))
        return _out(e, np_in)

    def axis_angle_2_mano_quat(self, baa_list, flat_hand=False, order='wxyz'):
        """(N,16,3), (16,3), (N,48) or (48) axis-angle, cast to float32 -> (N,16,4) float32 MANO quaternions; hands_mean is added to joints
        1..15 unless flat_hand (:272-301)."""
        if order != 'wxyz':
            raise ValueError("axis_angle_2_mano_quat: only order='wxyz' is supported, got %r" % (order,))
        a, np_in = _stage('axis_angle_2_mano_quat', baa_list, (torch.float32, torch.float64), self.device)
        if a.numel() % 48 or a.numel() == 0:
            raise ValueError('axis_angle_2_mano_quat: %s does not reshape to (-1,16,3)' % (tuple(a.shape),))
        a = a.reshape(-1, 16, 3)
        q = torch.empty(a.shape[0], 16, 4, device=self.device)
        with torch.cuda.device(self.device):
            call('rih_pose_axis_angle_to_mano_quat', a.data_ptr(), a.shape[0], self._left, 1 if flat_hand else 0, self._tables().data_ptr(),
                 self._hands_mean.data_ptr(), q.data_ptr(), _stream(a))
        return _out(q, np_in)

    def mano_quat_flat_2_normal(self, batch_quat, order='wxyz', return_type='quat'):
        """MANO quaternions reshaped to (-1,16,4), cast to float32 -> axis-angle with hands_mean subtracted from joints 1..15: (N,16,3)
        float64 for return_type 'aa' (any value but 'quat'), or those through axis_angle_2_mano_quat(flat_hand=True) for 'quat'
        (:303-332)."""
        if order != 'wxyz':
            raise ValueError("mano_quat_flat_2_normal: only order='wxyz' is supported, got %r" % (order,))
        q, np_in = _stage('mano_quat_flat_2_normal', batch_quat, (torch.float32, torch.float64), self.device)
        if q.numel() % 64 or q.numel() == 0:
            raise ValueError('mano_quat_flat_2_normal: %s does not reshape to (-1,16,4)' % (tuple(q.shape),))
        q = q.reshape(-1, 16, 4)
        rq = return_type == 'quat'
        out = torch.empty(q.shape[0], 16, 4 if rq else 3, dtype=torch.float32 if rq else torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            call('rih_pose_mano_quat_flat_to_normal', q.data_ptr(), q.shape[0], self._left, 1 if rq else 0, self._tables().data_ptr(),
                 self._hands_mean.data_ptr(), out.data_ptr(), _stream(q))
        return _out(out, np_in)

    def _joints(self, who, vec, shape):
        v, np_v = _stage(who, vec, (torch.float32, torch.float64), self.device)
        s, _ = _stage(who, shape, (torch.float32, torch.float64), self.device)
        center = self.mano_layer.center_idx
        self.mano_layer.center_idx = None
        try:
            with torch.no_grad():
                j = self.mano_layer(v, s)[1]
        finally:
            self.mano_layer.center_idx = center
        return j, np_v

    def trans_2_loc(self, vec, shape, trans, loc_center_idx):
        """(:334-344) joint loc_center_idx of the uncentred hand plus trans."""
        j, np_in = self._joints('trans_2_loc', vec, shape)
        if np_in:
            return j[:, loc_center_idx].cpu().numpy() + np.asarray(trans)
        return j[:, loc_center_idx] + trans

    def loc_2_trans(self, vec_, shape_, loc, loc_center_idx):
        """(:346-354) loc minus joint loc_center_idx of the uncentred hand."""
        j, np_in = self._joints('loc_2_trans', vec_, shape_)
        if np_in:
            return np.asarray(loc) - j[:, loc_center_idx].cpu().numpy()
        return loc - j[:, loc_center_idx]


class _Arguer:
    NORMAL_BEND, SPLANK, MAX_BEND, MAX_SPLANK = None, None, None, None

    def __init__(self, shape=None, side='right', root='assets/mano', device='cuda:0'):
        self.hpc = HandPoseConverter(side=side, root=root, device=device)
        self.hand_model = self.hpc.mano_layer
        self.device = self.hpc.device
        self.splank_mask = []
        self.shape = torch.tensor([CONVERTER_BETAS]) if shape is None else shape
        self.faces = self.hpc.faces
        self.ranges = _ranges(self.NORMAL_BEND, self.SPLANK)
        self._ranges = torch.from_numpy(self.ranges).to(self.device)

    def _argue(self, origin_vec_pose, argue_size, pose_type, vis, level, generator, return_adjust):
        if vis:
            raise NotImplementedError('argue_pose: vis=True needs open3d, which is not supported')
        A = int(argue_size)
        if A < 1:
            raise ValueError('argue_pose: argue_size must be >= 1, got %d' % A)
        if pose_type == 'quat':
            q, np_in = _stage('argue_pose', origin_vec_pose, (torch.float64, torch.float32), self.device)
            e = self.hpc.mano_quat_2_euler(q)
        else:
            e, np_in = _stage('argue_pose', origin_vec_pose, (torch.float64,), self.device)
        e = e[None] if e.dim() <= 2 else e
        _shape('argue_pose', e, (e.shape[0], 16, 3))
        B = e.shape[0]
        out = torch.empty(B * A, 16, 3, dtype=torch.float64, device=self.device)
        adj = torch.empty(B, N_DRAWS, A, dtype=torch.float64, device=self.device) if return_adjust else None
        u, seed, offset = None, 0, 0
        if generator is None:           # numpy's global stream, in bend_argue's then splank_argue's order
            ub = np.random.rand(B * len(BEND_JOINTS) * A).reshape(B, len(BEND_JOINTS), A)
            us = np.random.rand(B * len(SPLANK_JOINTS) * A).reshape(B, len(SPLANK_JOINTS), A)
            u = torch.from_numpy(np.concatenate([ub, us], 1)).to(self.device)
        elif isinstance(generator, torch.Generator):
            if generator.device.type != 'cuda':
                raise TypeError('argue_pose: generator must be an int seed or a CUDA torch.Generator')
            seed, offset = generator.initial_seed(), generator.get_offset()
            generator.set_offset(offset + -(-B * N_DRAWS * A // 4) * 4)
        else:
            seed = int(generator)
        seed &= (1 << 64) - 1
        with torch.cuda.device(self.device):
            call('rih_pose_argue', e.data_ptr(), B, A, self._ranges.data_ptr(), float(self.MAX_BEND * level), float(self.MAX_SPLANK * level),
                 None if u is None else u.data_ptr(), seed, offset, out.data_ptr(), None if adj is None else adj.data_ptr(), _stream(e))
        if return_adjust:
            return _out(out, np_in), _out(adj, np_in)
        return _out(out, np_in)


class HandPoseArguer(_Arguer):
    """HandPoseArguer(shape=None, side='right', root='assets/mano') (scripts/HandPoseArguer.py:11-173): bend maxima 120, splank 30."""
    NORMAL_BEND, SPLANK = (-8, 90), ((-6, 20), (-10, 10), (-15, 6), (-35, 6), (-9, 80))
    MAX_BEND, MAX_SPLANK = 120, 30

    def argue_pose(self, origin_vec_pose, argue_size=10, pose_type='quat', vis=False, generator=None, return_adjust=False):
        """(N,16,3) euler or, for pose_type 'quat', (N,16,4) MANO quaternions -> (N*argue_size,16,3) float64 euler, row i*argue_size + a.
        generator: None (numpy's global RandomState, the reference's stream), an int seed or a CUDA torch.Generator (device Philox).
        return_adjust: also return the applied adjustments in degrees, (N,20,argue_size) in draw order."""
        return self._argue(origin_vec_pose, argue_size, pose_type, vis, 1.0, generator, return_adjust)


class PoseArguer(_Arguer):
    """PoseArguer(shape=None, side='right', root='../../assets/mano') (Ver2Code/NatureJudge/PoseArgue.py:12-174): bend maxima
    120 * random_level, splank 45 * random_level."""
    NORMAL_BEND, SPLANK = (-8, 95), ((-25, 15), (-15, 15), (-25, 15), (-20, 30), (-30, 30))
    MAX_BEND, MAX_SPLANK = 120, 45

    def __init__(self, shape=None, side='right', root='../../assets/mano', device='cuda:0'):
        super().__init__(shape, side, root, device)

    def argue_pose(self, origin_vec_pose, argue_size=10, pose_type='quat', vis=False, random_level=1.0, generator=None, return_adjust=False):
        """As HandPoseArguer.argue_pose, with the maxima scaled by random_level."""
        return self._argue(origin_vec_pose, argue_size, pose_type, vis, random_level, generator, return_adjust)


def _generator(generator):
    """Drivers draw several times: an int seed becomes a CUDA torch.Generator so that each draw gets its own Philox offset."""
    if generator is None or isinstance(generator, torch.Generator):
        return generator
    return torch.Generator(device='cuda').manual_seed(int(generator))


# ---------------------------------------------------------------------------------------------------------------------------- drivers
def convert_annotations(annots, root='assets/mano', convert_data_path=None, device='cuda:0'):
    """data/template_0_pose_convert.py: RenderIH annotations (each with mano_params[side]['oripose' [48], 'trans' [1,3], 'shape' [1,10]])
    -> {'right', 'left': {'rot' [N,16,3] euler, 'loc' [N,3] root joint + trans in cm, 'shape' [N,1,10]}, 'capture_frame_id' [N]}, the
    frames numbered 0..N-1; saved to convert_data_path when given."""
    hpc = {s: HandPoseConverter(side=s, root=root, device=device) for s in ('left', 'right')}
    out = {}
    for side in ('right', 'left'):
        aa = [a['mano_params'][side]['oripose'] for a in annots]
        shape = [a['mano_params'][side]['shape'] for a in annots]
        trans = [a['mano_params'][side]['trans'][0] for a in annots]
        quat = hpc[side].axis_angle_2_mano_quat(aa, flat_hand=False)
        rot = hpc[side].mano_quat_2_euler(quat)
        loc = hpc[side].trans_2_loc(quat, np.asarray(shape).squeeze(1), np.asarray(trans), 0)
        out[side] = dict(rot=rot, loc=loc * 100, shape=np.asarray(shape))
    out = dict(right=out['right'], left=out['left'], capture_frame_id=np.asarray(list(range(len(annots)))))
    if convert_data_path is not None:
        np.save(convert_data_path, out)
    return out


def argue_data(data, argue_size=5, add_origin=False, splice_data_length=5000, out_dir='data', root='assets/mano', start_id=0, end_id=-1,
               generator=None, device='cuda:0'):
    """data/template_1_pose_argue.py on a converted dict: each hand's rot augmented by HandPoseArguer in the dict's key order, loc / shape /
    capture_frame_id repeated argue_size times (the originals appended with add_origin), then saved in splices of splice_data_length as
    out_dir/template_argued_data{k}.npy.  -> the saved paths.  The input dict is not modified."""
    gen = _generator(generator)
    data = copy.deepcopy(data)
    raw = copy.deepcopy(data) if add_origin else None
    hpa = {s: HandPoseArguer(side=s, root=root, device=device) for s in ('right', 'left')}
    end_id = len(data['capture_frame_id']) if end_id == -1 else end_id
    for side_id in list(data.keys()):
        if side_id in ('left', 'right'):
            rot = data[side_id]['rot'][start_id:end_id]
            data[side_id]['loc'] = np.repeat(data[side_id]['loc'][start_id:end_id], argue_size, axis=0)
            data[side_id]['shape'] = np.repeat(data[side_id]['shape'][start_id:end_id], argue_size, axis=0)
            data[side_id]['rot'] = hpa[side_id].argue_pose(np.asarray(rot), pose_type='euler', argue_size=argue_size, generator=gen)
            if add_origin:
                for key_id in data[side_id]:
                    data[side_id][key_id] = np.vstack([data[side_id][key_id], raw[side_id][key_id][start_id:end_id]])
        elif side_id == 'capture_frame_id':
            data[side_id] = np.repeat(data[side_id][start_id:end_id], argue_size)
            if add_origin:
                data[side_id] = np.append(data[side_id], raw[side_id][start_id:end_id])
    paths, total = [], len(data['capture_frame_id'])
    for k, left_idx in enumerate(range(0, total, splice_data_length)):
        right_idx = min(total, left_idx + splice_data_length)
        sub = {}
        for key, v in data.items():
            if key in ('left', 'right'):
                sub[key] = dict(v)
                for leaf in ('loc', 'rot', 'shape'):
                    sub[key][leaf] = v[leaf][left_idx:right_idx]
            elif key == 'capture_frame_id':
                sub[key] = v[left_idx:right_idx]
            else:
                sub[key] = copy.deepcopy(v)
        paths.append(os.path.join(out_dir, 'template_argued_data' + str(k) + '.npy'))
        np.save(paths[-1], sub)
    return paths


def _empty_struct(d):
    """copy_dict_struct (template_3_pose_reconvert.py:7-13): the dict tree with every leaf an empty array."""
    if type(d) is not dict:
        return np.asarray([])
    return {k: _empty_struct(v) for k, v in d.items()}


def reconvert_optimized(paths, template, out_dir='data/optimezed_argued_data', root='assets/mano', device='cuda:0'):
    """data/template_3_pose_reconvert.py: each optimised mocap file (mode 0, scale 1.0: loc / 100) converted back to one RenderIH-style
    annotation per frame -- the template's structure with mano_params[side] = {pose [48] axis-angle, trans [1,3], shape [1,10]} --
    saved as out_dir/{capture_id}_{save_id}_.npy, save_id bumped past existing files.  template: the annotation dict or its path.
    -> the saved paths."""
    os.makedirs(out_dir, exist_ok=True)
    if isinstance(template, str):
        template = np.load(template, allow_pickle=True)
    struct = _empty_struct(template)
    hpc = {s: HandPoseConverter(side=s, root=root, device=device) for s in ('left', 'right')}
    saved = []
    for data_name in paths:
        raw = np.load(data_name, allow_pickle=True).item()
        res = {}
        for side in ('right', 'left'):
            rot, loc, shape = raw[side]['rot'], raw[side]['loc'] * 1.0 / 100, raw[side]['shape']
            quat = hpc[side].euler_2_mano_quat(rot)
            res[side] = (hpc[side].mano_quat_flat_2_normal(quat, return_type='aa'), hpc[side].loc_2_trans(quat, shape, loc, 0), shape)
        for data_id, capture_id in enumerate(raw['capture_frame_id']):
            capture_id = capture_id if type(capture_id) is str else str(capture_id)
            d = copy.deepcopy(struct)
            for side in ('left', 'right'):
                aa, trans, shape = res[side]
                d['mano_params'][side]['pose'] = aa[data_id]
                d['mano_params'][side]['trans'] = trans[data_id:data_id + 1]
                d['mano_params'][side]['shape'] = shape[data_id:data_id + 1]
            save_id = 0
            path = os.path.join(out_dir, capture_id + '_{}_'.format(save_id) + '.npy')
            while os.path.exists(path):
                save_id += 1
                path = os.path.join(out_dir, capture_id + '_{}_'.format(save_id) + '.npy')
            np.save(path, d)
            saved.append(path)
    return saved


def birth_data(data, argue_size=15, add_origin=True, splice_data_length=100000000, out_dir='./data', root='../../assets/mano', start_id=0,
               end_id=-1, generator=None, device='cuda:0'):
    """Ver2Code/NatureJudge/data_birth.py's loop on a converted dict: for random_level 1.0, 0.9, ..., 0.1 (rr in np.arange(0, 1, 0.1)) and
    each hand in the dict's key order, PoseArguer.argue_pose then, with the RIGHT converter for both hands, euler -> MANO quaternion ->
    flat axis-angle; confidence rr per row.  With add_origin the raw euler rows of the left then the right hand follow, confidence 1.0.
    Everything stays on the device until the splices out_dir/argued_hand_pose_{k}.npy = {'rot', 'confidence' (a list)} are written.
    -> the saved paths."""
    gen = _generator(generator)
    hpa = {s: PoseArguer(side=s, root=root, device=device) for s in ('right', 'left')}
    rhpc = hpa['right'].hpc
    dev = rhpc.device
    end_id = len(data['capture_frame_id']) if end_id == -1 else end_id
    rots = {s: torch.from_numpy(np.ascontiguousarray(data[s]['rot'][start_id:end_id], dtype=np.float64)).to(dev)
            for s in data if s in ('left', 'right')}
    parts, rates = [], []
    for rr in np.arange(0.0, 1.0, 0.1):
        for side_id in list(data.keys()):
            if side_id in ('left', 'right'):
                argued = hpa[side_id].argue_pose(rots[side_id], pose_type='euler', argue_size=argue_size, random_level=1.0 - rr, generator=gen)
                parts.append(rhpc.mano_quat_flat_2_normal(rhpc.euler_2_mano_quat(argued), return_type='aa'))
                rates.append(np.full(argued.shape[0], rr))
    if add_origin:
        for side_id in ('left', 'right'):
            parts.append(torch.from_numpy(np.asarray(data[side_id]['rot'][start_id:end_id], dtype=np.float64)).to(dev))
            rates.append(np.full(end_id - start_id, 1.0))
    rot = torch.cat(parts).cpu().numpy()
    conf = np.concatenate(rates)
    paths = []
    for k, left_idx in enumerate(range(0, len(conf), splice_data_length)):
        right_idx = min(len(conf), left_idx + splice_data_length)
        paths.append(os.path.join(out_dir, 'argued_hand_pose_' + str(k) + '.npy'))
        np.save(paths[-1], dict(rot=rot[left_idx:right_idx], confidence=conf[left_idx:right_idx].tolist()))
    return paths
