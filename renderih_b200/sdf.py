"""Two-hand anti-penetration SDF loss: drop-ins for the pose optimiser's `NewLoss` (pose_data_optimize/code_sdf/sdf_template.py:19-157,
built at hocontact/postprocess/geo_optimizer_both_batch.py:46 and weighted 0.02 * lambda_repulsion_loss at :816) and for the dense grid of
its hand-built extension `sdf.SDF` (pose_data_optimize/lib/sdf/sdf/sdf.py, kernel sdf_cuda_kernel.cu:243-304).  The kernels are in
csrc/sdf.cu; there is no CPU path: every tensor input must be a CUDA tensor.

Conventions reproduced:

* Grid (`SDF`, sdf_cuda_kernel.cu:252-263,299): phi [B,G,G,G] with phi[b,k,j,i], i (x) fastest.  Voxel (i,j,k) has its centre at
  c = -1 + (idx + 0.5) * d per axis with d = 2 / (G - 1).  Reference quirk, kept because the optimiser was tuned with it: these centres
  sit half a voxel off the nodes -1 + idx * d that grid_sample(align_corners=True) samples later.
* phi = Euclidean distance from c to the nearest face (the closed triangle point set) when c is inside, else 0 (:291-293).  c is inside
  when the ray from c towards (-1,-1,-1) hits an odd number of faces (:284-289): Moller-Trumbore with the unnormalised direction
  (-1,-1,-1) - c, |det| < 1e-6 rejected, u in [0,1], v >= 0, u + v <= 1 inclusive, hits counted for t >= 0 (:96-138).  A zero-area face
  is never hit; its distance is the distance to its segments.  Distance and parity do not depend on the winding.
* Every voxel is written.  The reference launches B*G^3/512 blocks of 512 threads (:316-317) and leaves a remainder of voxels at 0;
  at G = 32 there is none.  That dropped tail is not reproduced.
* NewLoss (sdf_template.py:57-157): vertices [B,2,V,3], hand 0 the right hand and hand 1 the left (:62-63).  Per sample and hand, the
  frame c_h = (min + max) / 2 and s_h = (1 + scale_factor) * 0.5 * max_xyz(max - min) of its vertices (:84-87), constants without
  gradient (computed under no_grad there).  Phi_h = SDF of (v - c_h) / s_h with the closed hand faces -- the same face file for both
  hands (:31-32).  Each vertex v of hand h is mapped into the other hand's frame, x = (v - c_o) / s_o, and p is the trilinear sample of
  Phi_o at x as grid_sample(align_corners=True, padding_mode='zeros') takes it (:120-134): ix = (x + 1) / 2 * (G - 1), x indexes W,
  y H and z D, a corner outside the grid counts 0.  m_v = the number of the 16 parts of part_vert that contain v.
  L_h[v] = m_v * p / 4, O_h[v] = m_v * p * s_o, loss[b] = sum_v (L_left + L_right) (:136-148).
* Returns (:151-157): loss [B]; with return_per_vert_loss (loss, L_left, L_right); with return_origin_scale_loss as well
  (loss, cat([L_left, L_right], 1), [O_left, O_right]).  Every returned tensor is differentiable with respect to the vertices, through x
  only: dp/dx is the trilinear gradient of the cell torch's grid_sampler_3d backward picks (floor of ix), scaled by (G - 1) / 2, then
  by 1 / s_o.  The reference's asserts (:108-109,114-115) synchronise with the device; nothing here does.
* Defaults, under the asset root (`assets.default_asset_root()`): faces = pose_data_optimize/assets/closed_hand/hand_mesh_close.obj,
  the watertight right MANO hand the reference ships (1552 faces: the 1538 MANO faces and 14 closing the wrist); part_vert =
  part_vert.npy.  UNVERIFIED: NewLoss itself loads code_sdf/right.npy, which is not in the reference tree; the closed obj stands in for it.
  Both can be passed instead (`faces=`, `part_vert=`).

The fused loss computes only the voxels the other hand's vertices touch (at most 8 V of G^3 per grid); its values equal sampling the
dense grid.  Face and part indices are validated once, at construction.
"""
import os

import numpy as np
import torch

from ._lib import call
from .assets import default_asset_root

CLOSED_HAND_OBJ = os.path.join('pose_data_optimize', 'assets', 'closed_hand', 'hand_mesh_close.obj')
PART_VERT = 'part_vert.npy'
_CHECKED = set()          # (pointer, version, shape, device, V) of CUDA face tensors sdf() has validated


def _require_cuda(name, *tensors):
    for t in tensors:
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError('renderih_b200.sdf.%s: CUDA tensors required (there is no CPU path)' % name)


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _grid_size(G):
    G = int(G)
    if not 2 <= G <= 64:
        raise ValueError('grid_size %d outside 2..64' % G)
    return G


def load_obj_faces(path):
    """[F,3] int64 zero-based face indices of a triangle .obj file."""
    faces = []
    with open(path) as f:
        for line in f:
            if line.startswith('f '):
                faces.append([int(tok.split('/')[0]) - 1 for tok in line.split()[1:4]])
    return np.asarray(faces, dtype=np.int64)


def load_part_vert(path):
    d = np.load(path, allow_pickle=True)[()]
    return [d[k] for k in sorted(d)]


def _check_faces(faces):
    f = np.asarray(faces.detach().cpu() if isinstance(faces, torch.Tensor) else faces)
    if f.ndim != 2 or f.shape[1] != 3 or f.shape[0] < 1 or not np.issubdtype(f.dtype, np.integer):
        raise ValueError('faces must be a non-empty integer [F,3] array, got %s %s' % (f.dtype, f.shape))
    if f.min() < 0:
        raise ValueError('faces contain negative vertex indices')
    return f.astype(np.int32)


def sdf(faces, vertices, grid_size=32):
    """Dense grid phi [B,G,G,G] of the closed mesh faces [F,3] over vertices [B,V,3] (CUDA, already in [-1,1]^3).  Not differentiable,
    like the reference's SDFFunction.  faces may be a host array or a CUDA tensor; its indices are checked against V (a CUDA tensor is
    copied to the host for that, once: an unchanged int32 CUDA tensor that passed is used as it is)."""
    _require_cuda('sdf', vertices)
    G = _grid_size(grid_size)
    if vertices.dim() != 3 or vertices.shape[2] != 3:
        raise ValueError('vertices must be [B,V,3], got %s' % (tuple(vertices.shape),))
    B, V = vertices.shape[:2]
    v = vertices.detach().float().contiguous()
    key = (faces.data_ptr(), faces._version, tuple(faces.shape), faces.device, V) if isinstance(faces, torch.Tensor) else None
    if key is not None and faces.dtype == torch.int32 and faces.device == v.device and faces.is_contiguous() and key in _CHECKED:
        fd = faces              # validated before (no host copy: safe inside CUDA-graph capture)
    else:
        f = _check_faces(faces)
        if f.max() >= V:
            raise ValueError('faces index vertex %d of %d' % (f.max(), V))
        fd = torch.from_numpy(f).to(v.device)
        if key is not None:
            _CHECKED.add(key)
    phi = torch.empty(B, G, G, G, device=v.device)
    call('rih_sdf_grid', fd.data_ptr(), fd.shape[0], v.data_ptr(), B, V, G, phi.data_ptr(), _stream(v))
    return phi


class SDF(torch.nn.Module):
    """lib/sdf/sdf/sdf.py SDF: forward(faces, vertices, grid_size=32) -> phi [B,G,G,G]."""

    def forward(self, faces, vertices, grid_size=32):
        return sdf(faces, vertices, grid_size)


def penetration(vertices, faces, mult, grid_size=32, scale_factor=0.1):
    """The fused forward: vertices [B,2,V,3] fp32 contiguous CUDA, faces [F,3] / mult [V] int32 CUDA (validated by the caller).
    -> loss [B], L [B,2,V], O [B,2,V], dL/dv [B,2,V,3], center [B,2,3], scale [B,2]; hand order as in `vertices`."""
    B, _, V, _ = vertices.shape
    dev = vertices.device
    loss = torch.empty(B, device=dev)
    L, O = torch.empty(B, 2, V, device=dev), torch.empty(B, 2, V, device=dev)
    dLdv = torch.empty(B, 2, V, 3, device=dev)
    center, scale = torch.empty(B, 2, 3, device=dev), torch.empty(B, 2, device=dev)
    call('rih_sdf_penetration', vertices.data_ptr(), B, V, faces.data_ptr(), faces.shape[0], mult.data_ptr(), _grid_size(grid_size),
         (1 + scale_factor) * 0.5, loss.data_ptr(), L.data_ptr(), O.data_ptr(), dLdv.data_ptr(), center.data_ptr(), scale.data_ptr(),
         _stream(vertices))
    return loss, L, O, dLdv, center, scale


class _PenetrationFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, faces, mult, grid_size, scale_factor):
        loss, L, O, dLdv, _, scale = penetration(vertices, faces, mult, grid_size, scale_factor)
        ctx.save_for_backward(dLdv, scale)
        ctx.set_materialize_grads(False)
        return loss, L, O

    @staticmethod
    def backward(ctx, g_loss, g_L, g_O):
        dLdv, scale = ctx.saved_tensors
        B, _, V, _ = dLdv.shape
        g = [None if t is None else t.float().contiguous() for t in (g_loss, g_L, g_O)]
        dv = torch.empty_like(dLdv)
        call('rih_sdf_penetration_bwd', dLdv.data_ptr(), scale.data_ptr(), B, V, *[None if t is None else t.data_ptr() for t in g], dv.data_ptr(),
             _stream(dLdv))
        return dv, None, None, None, None


class NewLoss(torch.nn.Module):
    """sdf_template.py NewLoss on the GPU: NewLoss(grid_size=32) then forward(vertices [B,2,V,3], scale_factor=0.1,
    return_per_vert_loss=False, return_origin_scale_loss=False).  faces: [F,3] closed-hand faces, part_vert: the 16 parts (a dict or a
    list of vertex-index collections); both default to the reference's files under the asset root (see the module docstring)."""

    def __init__(self, grid_size=32, robustifier=None, faces=None, part_vert=None, device='cuda'):
        super().__init__()
        self.grid_size = _grid_size(grid_size)
        self.robustifier = robustifier          # stored and unused, as in the reference
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('NewLoss: a CUDA device is required (there is no CPU path)')
        root = default_asset_root()
        if faces is None:
            faces = load_obj_faces(os.path.join(root, CLOSED_HAND_OBJ))
        if part_vert is None:
            part_vert = load_part_vert(os.path.join(root, PART_VERT))
        f = _check_faces(faces)
        parts = list(part_vert.values()) if isinstance(part_vert, dict) else list(part_vert)
        idx = [np.unique(np.asarray(sorted(p) if isinstance(p, (set, frozenset)) else p, dtype=np.int64).reshape(-1)) for p in parts]
        allp = np.concatenate(idx) if idx else np.zeros(0, np.int64)
        if allp.size and allp.min() < 0:
            raise ValueError('part_vert contains negative vertex indices')
        self._max_index = int(max(f.max(), allp.max() if allp.size else -1))
        self._counts = np.bincount(allp, minlength=self._max_index + 1).astype(np.int32)     # m_v: parts containing v (no duplicates within a part)
        self.faces = torch.from_numpy(f).to(self.device)
        self._mult = {}

    def _mult_for(self, V):
        if V not in self._mult:
            m = np.zeros(V, np.int32)
            m[:len(self._counts)] = self._counts
            self._mult[V] = torch.from_numpy(m).to(self.device)
        return self._mult[V]

    def forward(self, vertices, scale_factor=0.1, return_per_vert_loss=False, return_origin_scale_loss=False):
        _require_cuda('NewLoss', vertices)
        if vertices.dim() != 4 or vertices.shape[1] != 2 or vertices.shape[3] != 3:
            raise ValueError('vertices must be [B,2,V,3], got %s' % (tuple(vertices.shape),))
        V = vertices.shape[2]
        if V <= self._max_index:
            raise ValueError('faces / part_vert index vertex %d but the hands have %d vertices' % (self._max_index, V))
        if vertices.device != self.faces.device:
            raise RuntimeError('NewLoss: vertices on %s, loss built for %s' % (vertices.device, self.faces.device))
        loss, L, O = _PenetrationFn.apply(vertices.float().contiguous(), self.faces, self._mult_for(V), self.grid_size, float(scale_factor))
        if not return_per_vert_loss:
            return loss
        if not return_origin_scale_loss:
            return loss, L[:, 1], L[:, 0]
        return loss, torch.cat([L[:, 1], L[:, 0]], 1), [O[:, 1], O[:, 0]]
