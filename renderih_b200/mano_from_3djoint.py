"""Fitting MANO to 3-D hand joints on the GPU: a drop-in for the reference's offline tool utils/mano_from_3djoint (convert2mano.py,
AIK.py, utils.py), batched over frames and both hands.

    fitter = JointFitter('mano', 'cuda')                       # MANO_LEFT.pkl / MANO_RIGHT.pkl, as convert2mano.py:134-141 loads them
    csv_data = read_worldpos_csv('take_worldpos.csv')          # or a pandas DataFrame: any mapping column -> sequence
    left, right = get_3djoints_batch(csv_data, range(F))       # [F,21,3] each
    out = fitter.fit(left, right)                              # out['left'] / out['right']: pose_R, beta, verts, joints, ori_pose, finite
    convert('take_worldpos.csv', frames=range(F))              # the script for every frame: the .obj files and the parameters

One frame of one hand is what the reference script computes for `frame_idx` (convert2mano.py:133-245):
  1. the joints of `left` / `right` from the CSV row (get_3djoints, :22-37);
  2. the template: the layer's joints at pose_R = I, beta = 0 (ManoLayer(center_idx=9, use_pca=True); the left layer's
     shapedirs[:, 0, :] negated, :134-136);
  3. adaptive_IK (AIK.py:16-104) on the joints scaled to the template's |j9 - j0| and moved to its wrist (:164-169), cast to float32;
  4. 200 iterations of torch.optim.Adam(lr=0.1) over the free matrices pose_R [16,3,3] and beta [10]: the layer with root pose_R[0] and
     PCA coefficients mat2aa(pose_R[1:]), the loss mean |(j - j[0]) - (joints - joints[0]) / 100|, and lr = 0.1 (200 - i) / 200 after
     step i (:175-200);
  5. the outputs (:203-245): the wrist-relative vertices * 100 + joints[0] (cur_frame{idx}_{hand}.obj), ori_pose = [mat2aa(pose_R[0]),
     pca2axis(mat2aa(pose_R[1:])) - hands_mean], and the manopth mesh of ori_pose (ori_frame{idx}_{hand}.obj).

On the device: rih_mfit_aik runs step 3 for every frame (float64, one thread per frame); one optimiser iteration for all frames of a hand
is rih_mfit_rotmat_to_aa_fwd, rih_mano_fwd, rih_mfit_joint_l1, rih_mano_bwd, rih_mfit_rotmat_to_aa_bwd, rih_ge_adam_step and
rih_mfit_lr_step, captured in one CUDA graph and replayed `iterations` times.  The batched loss is the sum of the per-frame means, so
each frame's gradient, and with the elementwise Adam its whole trajectory, is that of fitting the frame alone; no kernel reduces across
frames, so a frame's result is bitwise the same in any batch.

Reproduced quirks:
* pose_R is a free matrix: Adam moves it off the rotations and mat2aa reads whatever it holds, with mat2quat's branch choice.
* mat2aa's gradient is NaN at an exactly zero rotation (the 0 / 0 of two_theta / sin_theta and of sqrt's backward), and AIK gives NaN
  where a target bone is exactly parallel to its template bone (axangle2mat normalises a zero axis).  Such a hand's frame comes out NaN,
  as in the reference; `finite` [B] marks the frames whose pose_R and beta are finite.
* A reflection from the Kabsch fit is kept unless some singular value is below 1e-4 (AIK.py:59-66).

Deviations:
* The ori_frame mesh comes from renderih_b200.manopth.ManoLayer, which runs quaternions only: [root_aa, pca2axis(aa)] (what the
  reference's axis-angle layer builds from ori_pose with flat_hand_mean=False) is converted to quaternions on the device the way that
  layer's batch_rodrigues does (|aa + 1e-8|, half angle).  Against the reference's axis-angle layer the vertices agree to float32
  rounding (about 1e-6 of the mesh size).
* get_3djoints raises ValueError when a hand does not get exactly 21 joints (the reference reshapes whatever it found).

Out of scope: the matplotlib plot and tmp1.jpg (:153-157); get_all_3djoint and the BVH input, which the script never calls (:39-96);
the commented-out beta regulariser (:193-195).  The package does not import pandas: read_worldpos_csv uses the csv module.
"""
import csv
import os

import numpy as np
import torch

from ._lib import call
from .ge_optimizer import ADAM_EPS, BETAS, beta_powers
from .manolayer import ManoLayer
from .manopth import ManoLayer as ManopthLayer

LEFT = ['Wrist_L', 'ThumbFinger1_L', 'ThumbFinger2_L', 'ThumbFinger3_L', 'ThumbFinger4_L', 'IndexFinger1_L', 'IndexFinger2_L',
        'IndexFinger3_L', 'IndexFinger4_L', 'MiddleFinger1_L', 'MiddleFinger2_L', 'MiddleFinger3_L', 'MiddleFinger4_L', 'RingFinger1_L',
        'RingFinger2_L', 'RingFinger3_L', 'RingFinger4_L', 'PinkyFinger1_L', 'PinkyFinger2_L', 'PinkyFinger3_L', 'PinkyFinger4_L']
RIGHT = [n[:-1] + 'R' for n in LEFT]
SIDES = ('left', 'right')
ITERATIONS, LR = 200, 0.1
_NP = 154                     # variables per frame: root 9 | 15 joint matrices 135 | beta 10


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _cuda(name, t, dtype=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError('mano_from_3djoint: %s must be a tensor, got %s' % (name, type(t).__name__))
    if not t.is_cuda:
        raise RuntimeError('mano_from_3djoint: %s must be a CUDA tensor (there is no CPU path)' % name)
    if not t.is_floating_point() or (dtype is not None and t.dtype != dtype):
        raise TypeError('mano_from_3djoint: %s must be %s, got %s' % (name, dtype or 'a float tensor', t.dtype))
    return t


# ------------------------------------------------------------------------------------------------------------------ joints
def _columns(keys, names):
    """The reference's column rule (convert2mano.py:22-37): for each name in order, every column containing it, in column order, except
    columns containing 'End'."""
    return [k for n in names for k in keys if n in k and 'End' not in k]


def _check21(cols, side):
    if len(cols) != 63:
        raise ValueError('get_3djoints: the %s hand has %d values, not 21 joints x 3 (columns: %s)' % (side, len(cols), cols))


def get_3djoints(csv_data, frame_idx=0):
    """(left [21,3], right [21,3]) float64 of row frame_idx; csv_data is any mapping column name -> sequence (a DataFrame works)."""
    keys = list(csv_data.keys())
    out = []
    for side, names in zip(SIDES, (LEFT, RIGHT)):
        cols = _columns(keys, names)
        _check21(cols, side)
        out.append(np.array([csv_data[c][frame_idx] for c in cols], dtype=np.float64).reshape(-1, 3))
    return tuple(out)


def get_3djoints_batch(csv_data, frames):
    """(left [F,21,3], right [F,21,3]) float64 for the rows in frames."""
    keys = list(csv_data.keys())
    frames = list(frames)
    out = []
    for side, names in zip(SIDES, (LEFT, RIGHT)):
        cols = _columns(keys, names)
        _check21(cols, side)
        a = np.empty((len(frames), 63), np.float64)
        for i, c in enumerate(cols):
            col = csv_data[c]
            a[:, i] = [col[f] for f in frames]
        out.append(a.reshape(-1, 21, 3))
    return tuple(out)


def read_worldpos_csv(path):
    """A world-position CSV -> {column: float64 array} (columns that do not parse as numbers stay lists of strings), as pandas.read_csv
    gives them to get_3djoints."""
    with open(path, newline='') as f:
        rows = list(csv.reader(f))
    header, body = rows[0], [r for r in rows[1:] if r]
    data = {}
    for i, name in enumerate(header):
        vals = [r[i] if i < len(r) else '' for r in body]
        try:
            data[name] = np.array([float(v) if v != '' else np.nan for v in vals], dtype=np.float64)
        except ValueError:
            data[name] = vals
    return data


# ------------------------------------------------------------------------------------------------------------------ AIK, mat2aa
def adaptive_IK(T, P):
    """AIK.adaptive_IK: numpy T, P [21,3] -> numpy [1,16,3,3] float64; or float64 CUDA tensors T [21,3] | [B,21,3], P [B,21,3] ->
    [B,16,3,3].  The arithmetic runs on the GPU (rih_mfit_aik) in float64."""
    if isinstance(T, torch.Tensor) or isinstance(P, torch.Tensor):
        T, P = _cuda('T', T, torch.float64), _cuda('P', P, torch.float64)
        if P.dim() != 3 or tuple(P.shape[1:]) != (21, 3) or tuple(T.shape[-2:]) != (21, 3) or T.dim() not in (2, 3) or \
                (T.dim() == 3 and T.shape[0] != P.shape[0]):
            raise ValueError('adaptive_IK: T must be [21,3] or [B,21,3] and P [B,21,3], got %s and %s' % (tuple(T.shape), tuple(P.shape)))
        T, P = T.contiguous(), P.contiguous()
        out = torch.empty(P.shape[0], 16, 3, 3, dtype=torch.float64, device=P.device)
        with torch.cuda.device(P.device):
            call('rih_mfit_aik', T.data_ptr(), int(T.dim() == 3), 0.0, 0, P.data_ptr(), P.shape[0], out.data_ptr(), _stream(P))
        return out
    T, P = np.asarray(T, np.float64), np.asarray(P, np.float64)
    if T.shape != (21, 3) or P.shape != (21, 3):
        raise ValueError('adaptive_IK: T and P must be [21,3], got %s and %s' % (T.shape, P.shape))
    dev = torch.device('cuda', torch.cuda.current_device())
    return adaptive_IK(torch.from_numpy(T).to(dev), torch.from_numpy(P).to(dev)[None]).cpu().numpy()


class _Mat2aaFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, R):
        R = R.contiguous()
        aa = torch.empty(R.shape[0], 3, device=R.device)
        with torch.cuda.device(R.device):
            call('rih_mfit_rotmat_to_aa_fwd', R.data_ptr(), R.shape[0], aa.data_ptr(), _stream(R))
        ctx.save_for_backward(R)
        return aa

    @staticmethod
    def backward(ctx, g):
        (R,) = ctx.saved_tensors
        dR = torch.empty_like(R)
        with torch.cuda.device(R.device):
            call('rih_mfit_rotmat_to_aa_bwd', R.data_ptr(), g.float().contiguous().data_ptr(), R.shape[0], dR.data_ptr(), _stream(R))
        return dR


def mat2aa(R):
    """utils.mat2aa: rotation matrices [N,3,3] float32 CUDA -> axis-angle [N,3], differentiable (the reference's gradient, NaN at an
    exactly zero rotation included)."""
    _cuda('R', R, torch.float32)
    if R.dim() != 3 or tuple(R.shape[1:]) != (3, 3):
        raise ValueError('mat2aa: R must be [N,3,3], got %s' % (tuple(R.shape),))
    return _Mat2aaFn.apply(R)


def aa_to_quat(aa):
    """[..., 3] axis-angle -> [..., 4] quaternions (w, x, y, z) as manopth's batch_rodrigues forms them: angle |aa + 1e-8|."""
    n = torch.linalg.vector_norm(aa + 1e-8, dim=-1, keepdim=True)
    half = n * 0.5
    return torch.cat([torch.cos(half), torch.sin(half) * (aa / n)], -1)


# ------------------------------------------------------------------------------------------------------------------ the fit
class _Side:
    """Buffers and the captured iteration of one hand for batch B, `iterations` and lr."""

    def __init__(self, layer, B, n, lr0, dev):
        self.layer, self.B, self.n, self.lr0 = layer, B, n, lr0
        f = lambda *s: torch.zeros(*s, device=dev)
        self.flat, self.grad, self.m, self.v = f(B * _NP), f(B * _NP), f(B * _NP), f(B * _NP)
        self.aa, self.d_aa = f(B, 45), f(B, 45)
        self.verts, self.joints, self.g_j, self.target, self.loss = f(B, 778, 3), f(B, 21, 3), f(B, 21, 3), f(B, 21, 3), f(B)
        self.hist = f(n, B)
        self.pose64 = torch.zeros(B, 16, 3, 3, dtype=torch.float64, device=dev)
        self.lr = torch.zeros(1, dtype=torch.float64, device=dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.pow = torch.stack([beta_powers(b, n) for b in BETAS]).to(dev)
        self.graph = None

    def _ptr(self, t, off=0):
        return t.data_ptr() + 4 * off

    def forward(self, st):
        """aa = mat2aa(pose_R[:, 1:]); verts, joints = layer(pose_R[:, 0], aa, beta)."""
        B, L = self.B, self.layer
        call('rih_mfit_rotmat_to_aa_fwd', self._ptr(self.flat, 9 * B), 15 * B, self.aa.data_ptr(), st)
        call('rih_mano_fwd', L._tables(self.flat.device), L._parent_arr, self.flat.data_ptr(), self.aa.data_ptr(), 1, 45,
             self._ptr(self.flat, 144 * B), None, None, L.center_idx, 0, self.verts.data_ptr(), self.joints.data_ptr(), B, st)

    def iteration(self, st):
        B, L = self.B, self.layer
        self.forward(st)
        call('rih_mfit_joint_l1', self.joints.data_ptr(), self.target.data_ptr(), B, self.loss.data_ptr(), self.g_j.data_ptr(),
             self.hist.data_ptr(), self.step.data_ptr(), self.n, st)
        call('rih_mano_bwd', L._tables(self.flat.device), L._parent_arr, self.flat.data_ptr(), self.aa.data_ptr(), 1, 45,
             self._ptr(self.flat, 144 * B), None, None, L.center_idx, 0, None, self.g_j.data_ptr(), self.grad.data_ptr(),
             self.d_aa.data_ptr(), self._ptr(self.grad, 144 * B), None, None, B, st)
        call('rih_mfit_rotmat_to_aa_bwd', self._ptr(self.flat, 9 * B), self.d_aa.data_ptr(), 15 * B, self._ptr(self.grad, 9 * B), st)
        n = B * _NP
        call('rih_ge_adam_step', self.flat.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), n, n, n, n, 1,
             self.lr.data_ptr(), self.step.data_ptr(), self.pow[0].data_ptr(), self.pow[1].data_ptr(), self.n, BETAS[0], BETAS[1], ADAM_EPS,
             st)
        call('rih_mfit_lr_step', self.lr.data_ptr(), self.step.data_ptr(), self.lr0, self.n, st)

    def capture(self):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.iteration(torch.cuda.current_stream().cuda_stream)
        self.graph = g


class JointFitter:
    """The reference script's two layers and templates (convert2mano.py:134-141, :162-165) and its fit, batched over frames.
    mano_root: a directory holding MANO_LEFT.pkl / MANO_RIGHT.pkl, or {'left': mano dict, 'right': mano dict}."""

    def __init__(self, mano_root='mano', device='cuda'):
        dev = torch.device(device)
        if dev.type != 'cuda':
            raise RuntimeError('JointFitter: a CUDA device is required (there is no CPU path)')
        self.device = torch.device('cuda', torch.cuda.current_device() if dev.index is None else dev.index)
        src = {s: mano_root[s] if isinstance(mano_root, dict) else os.path.join(mano_root, 'MANO_%s.pkl' % s.upper()) for s in SIDES}
        self.mano_layer = {s: ManoLayer(src[s]).to(self.device) for s in SIDES}
        with torch.no_grad():
            self.mano_layer['left'].shapedirs[:, 0, :] *= -1
        self._mano_root = mano_root
        self._ori = None
        self.template, self.t_norm = {}, {}
        with torch.cuda.device(self.device):
            eye = torch.eye(3, device=self.device)
            for s in SIDES:
                with torch.no_grad():
                    _, j = self.mano_layer[s](eye[None], mat2aa(eye.repeat(15, 1, 1)).reshape(1, 45), torch.zeros(1, 10, device=self.device))
                t = j[0].cpu().numpy()                                  # float32, as the reference's template
                self.template[s] = torch.from_numpy(t.astype(np.float64)).to(self.device)
                self.t_norm[s] = float(np.linalg.norm(t[9] - t[0]))
        self._sides = {}

    def ori_layer(self, side):
        """renderih_b200.manopth.ManoLayer for the ori_frame mesh: the reference builds manopth's layer (use_pca=False,
        flat_hand_mean=False) and negates the left layer's th_shapedirs[:, 0, :] once more (convert2mano.py:137-140)."""
        if self._ori is None:
            r = self._mano_root
            self._ori = {}
            for s in SIDES:
                root = r[s] if isinstance(r, dict) else r
                layer = ManopthLayer(mano_root=root, side=s, use_pca=False, root_rot_mode='quat', joint_rot_mode='quat',
                                     flat_hand_mean=True).to(self.device)
                if s == 'left':
                    with torch.no_grad():
                        layer.th_shapedirs[:, 0, :] *= -1
                self._ori[s] = layer
        return self._ori[side]

    def _side(self, s, B, n, lr):
        key = (s, B, n, lr)
        if key not in self._sides:
            self._sides = {k: v for k, v in self._sides.items() if k[0] != s}         # one shape per hand stays captured
            self._sides[key] = _Side(self.mano_layer[s], B, n, lr, self.device)
        return self._sides[key]

    def fit(self, left_joints, right_joints, iterations=ITERATIONS, lr=LR, return_history=False):
        """Fit both hands.  *_joints: [B,21,3] float CUDA tensors in the CSV's units (either may be None to skip that hand).  Returns
        {'left': ..., 'right': ...}, each {'pose_R' [B,16,3,3], 'beta' [B,10], 'verts' [B,778,3] and 'joints' [B,21,3] of the final
        parameters relative to joint 0 (convert2mano.py:216-217), 'ori_pose' [B,48], 'finite' [B] bool, 'loss' [iterations,B] if
        return_history}, CUDA tensors; nothing synchronises with the host."""
        n = int(iterations)
        if n < 1:
            raise ValueError('JointFitter.fit: iterations must be >= 1, got %d' % n)
        out = {}
        with torch.cuda.device(self.device):
            for s, J in zip(SIDES, (left_joints, right_joints)):
                if J is None:
                    continue
                _cuda('%s_joints' % s, J)
                if J.dim() != 3 or tuple(J.shape[1:]) != (21, 3) or J.shape[0] < 1:
                    raise ValueError('JointFitter.fit: %s_joints must be [B,21,3], got %s' % (s, tuple(J.shape)))
                if J.device != self.device:
                    raise RuntimeError('JointFitter.fit: %s_joints is on %s, the fitter on %s' % (s, J.device, self.device))
                out[s] = self._fit_side(s, J.double().contiguous(), n, float(lr), return_history)
        return out

    def _fit_side(self, s, J, n, lr, history):
        B = J.shape[0]
        sd = self._side(s, B, n, lr)
        st = _stream(J)
        call('rih_mfit_aik', self.template[s].data_ptr(), 0, self.t_norm[s], 1, J.data_ptr(), B, sd.pose64.data_ptr(), st)
        with torch.no_grad():
            p = sd.pose64.reshape(B, 16, 9)
            sd.flat[:9 * B].copy_(p[:, 0].reshape(-1))
            sd.flat[9 * B:144 * B].copy_(p[:, 1:].reshape(-1))
            sd.flat[144 * B:].zero_()
            sd.target.copy_((J - J[:, 0:1]) / 100)
            sd.m.zero_()
            sd.v.zero_()
            sd.step.zero_()
            sd.lr.fill_(lr)
        if sd.graph is None:
            sd.capture()
        for _ in range(n):
            sd.graph.replay()
        sd.forward(st)                                  # the final parameters' mesh (convert2mano.py:204-210)
        pose_R = torch.cat([sd.flat[:9 * B].view(B, 1, 9), sd.flat[9 * B:144 * B].view(B, 15, 9)], 1).view(B, 16, 3, 3)
        beta = sd.flat[144 * B:].view(B, 10).clone()
        j0 = sd.joints[:, 0:1]
        layer = self.mano_layer[s]
        aa = mat2aa(pose_R.reshape(-1, 3, 3)).reshape(B, 48)
        ori_pose = torch.cat([aa[:, :3], layer.pca2axis(aa[:, 3:]) - layer.hands_mean], 1)
        res = {'pose_R': pose_R.clone(), 'beta': beta, 'verts': sd.verts - j0, 'joints': sd.joints - j0, 'ori_pose': ori_pose,
               'finite': torch.isfinite(pose_R.reshape(B, -1)).all(1) & torch.isfinite(beta).all(1)}
        if history:
            res['loss'] = sd.hist.clone()
        return res

    def ori_mesh(self, side, res):
        """The reference's ori_frame vertices before the / 1000 (convert2mano.py:226-236): manopth's mesh of ori_pose and beta, [B,778,3],
        and its joints [B,21,3]."""
        layer = self.mano_layer[side]
        aa = mat2aa(res['pose_R'].reshape(-1, 3, 3)).reshape(-1, 48)
        full = torch.cat([aa[:, :3], layer.pca2axis(aa[:, 3:])], 1).reshape(-1, 16, 3)
        q = aa_to_quat(full)
        if side == 'left':                              # the quaternion layer mirrors y and z of a left hand; axis-angle input does not
            q = q * torch.tensor([1.0, 1.0, -1.0, -1.0], device=q.device)
        return self.ori_layer(side)(q.contiguous(), res['beta'])[:2]


def save_obj(path, verts, faces):
    """utils.save_obj (utils.py:47-56) without colours."""
    with open(path, 'w') as f:
        f.write(''.join('v {} {} {}\n'.format(v[0], v[1], v[2]) for v in verts))
        f.write(''.join('f {} {} {}\n'.format(a + 1, b + 1, c + 1) for a, b, c in np.asarray(faces).astype(np.int64)))


def convert(csv_path, frames=None, out_dir='.', write_obj=True, mano_root='mano', device='cuda', fitter=None):
    """convert2mano.py for every frame in frames (default: every row of the CSV), both hands batched.  Writes cur_frame{idx}_{hand}.obj
    and ori_frame{idx}_{hand}.obj under out_dir when write_obj, and returns {'frames': [...], 'left': {...}, 'right': {...}} with the
    per-frame pose_R [F,16,3,3], beta [F,10], ori_pose [F,48] and finite [F] as numpy arrays."""
    data = read_worldpos_csv(csv_path) if isinstance(csv_path, (str, os.PathLike)) else csv_path
    if frames is None:
        frames = range(len(next(iter(data.values()))))
    frames = [int(f) for f in frames]
    fitter = fitter or JointFitter(mano_root, device)
    dev = fitter.device
    joints = dict(zip(SIDES, get_3djoints_batch(data, frames)))
    J = {s: torch.from_numpy(joints[s]).to(dev) for s in SIDES}
    res = fitter.fit(J['left'], J['right'])
    ret = {'frames': frames}
    for s in SIDES:
        r = res[s]
        ret[s] = {k: r[k].cpu().numpy() for k in ('pose_R', 'beta', 'ori_pose', 'finite')}
        if not write_obj:
            continue
        j0 = J[s][:, 0:1]
        cur = ((r['verts'] * 100).double() + j0).cpu().numpy()
        with torch.no_grad():
            ov, oj = fitter.ori_mesh(s, r)
        ov, oj = ov / 1000, oj / 1000
        ori = (((ov - oj[:, 0:1]) * 100).double() + j0).cpu().numpy()
        faces = fitter.mano_layer[s].faces
        os.makedirs(out_dir, exist_ok=True)
        for i, f in enumerate(frames):
            save_obj(os.path.join(out_dir, 'cur_frame{}_{}.obj'.format(f, s)), cur[i], faces)
            save_obj(os.path.join(out_dir, 'ori_frame{}_{}.obj'.format(f, s)), ori[i], faces)
    return ret
