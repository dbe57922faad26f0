"""The pose optimiser's hand-prior and contact terms on the GPU: a drop-in for what `GeOptimizer.loss_fn`
(pose_data_optimize/hocontact/postprocess/geo_optimizer_both_batch.py:498-859, two-hand mode) adds to its loss besides the hand models
and the anti-penetration term -- the anchor layer (manopth/manopth/anchorlayer.py), the contact energy, the quaternion-norm term, the
edge-length term and the ergonomics prior (hocontact/postprocess/geo_loss.py).  Kernels in csrc/geo_loss.cu; there is no CPU path.

    anchor = AnchorLayer()                                   # forward(vertices [B,778,3]) -> anchors [B,108,3], differentiable
    prior = HandPriorLoss(mano_right, mano_left)             # the optimiser's two renderih_b200.manopth.ManoLayer instances
    prior.set_contacts(anchor_id, anchor_elastic, anchor_padding_mask)      # [B,108,D] each; validated here, once
    quat_norm_loss, edge_loss, contact_loss, ergonic_loss = prior(quat_right, quat_left, verts_right, verts_left)

quat_* are the assembled, unnormalised [B,16,4] (or [B,64]) poses (:501-513); verts_* the rebuilt vertices after the translation add
(:539-565).  Each term is a 0-dim tensor summed over both hands, as the reference's `+=` does, and differentiable with respect to the
quaternions and the vertices.  Forward and backward never synchronise with the host and can be captured in a CUDA graph; the upstream
gradients are read on the device.

Conventions reproduced (geo_loss.py unless stated):

* Anchors (anchorutils.py:51-65): anchor a = v0 + w1 (v1 - v0) + w2 (v2 - v0) of face_vertex_idx[a] = (v0, v1, v2) with
  anchor_weight[a] = (w1, w2).  The tables are pose_data_optimize/assets/anchor/{face_vertex_idx,anchor_weight}.txt under
  `assets.default_asset_root()`, or arrays passed in; anchor_mapping_path.pkl, which the reference opens and only stores, is not read.
* quat-norm (:197-202): mean((|q|^2 - 1)^2) over B x 16 per hand, on the unnormalised quaternions.
* Joint matrices (HandPoseConverter.py:214-231, quatutils.py:7-30,168-221): q is normalised with F.normalize(eps=1e-12) (its gradient
  included), the left hand negates q.y and q.z, R has each entry divided by |q|^2 again, and ja = invM_U_n_0^T R invU_M_n_1^T.  The
  left root's sign flip (:227) touches joint 0 only, which the ergonomics prior does not read.
* Converter matrices (HandPoseConverter.py:29-130): the rest joints and transforms of each side's layer at identity quaternions and
  the converter's hard-coded betas (:43-44), computed with the layer's own forward, then axis_convert / init_convert_matrix in float64
  (the left hand's x axis and up_axis_base, :88-93, and root flip, :108-109), stored as float32 like the reference.  zero_ja is ja at
  identity quaternions (geo_optimizer_both_batch.py:98-104).
* Ergonomics, hand_pose_ergonomics_loss (:360-444) on M = zero_ja^T ja for joints 1..15, x/y/z the columns of M: step 1 the
  (x.z)^2 + (y.z)^2 + (z.z - 1)^2 means over the ten non-base joints; step 2 the twist (M21 - M12) / 2 of the four finger bases, and of
  the thumb base above 0.5; step 3 splank atan2(-x.z, x.x) and bend atan2(x.y, x.x) in degrees against the reference's ranges, the
  excess in radians squared; step 4 min(b10 - 3/4 b7, 0)^2 in radians after negative bend angles are zeroed in place, so the gradient
  through a negative angle is 0.  At every other kink (relu, torch.max, clamp(max=0)) the squared term has value and derivative 0,
  so torch's tie rules change nothing.  target_second_bend_angle (:438) is dead code and is not computed.
* Edge (:162-183, 241-244): mean((|v_i - v_j| - L0)^2) over B x E per hand.  The edge list is HandLoss.get_edge_idx of the RIGHT layer's
  faces in first-seen order, for both hands -- a reference quirk (geo_optimizer_both_batch.py:229 passes hand_faces).  L0 are the
  edge lengths of each side's own identity-pose, zero-beta vertices (:457-470).  torch.norm's gradient is 0 at a zero length.
* Contact (:20-27, geo_optimizer_both_batch.py:603-612): main (right) anchor anchor_id[b,i,k] is paired with sub (left) anchor i;
  the term is sum e |A_main - A_sub|^2 over every (b, i, k) -- e in the numerator whatever the mask -- divided by the sum of
  anchor_padding_mask over the batch, and 0 when that sum is <= 0.  The decision is taken on the device (the reference's
  `mask.sum() <= 0` synchronises).  The reference returns a shape-[1] zero in that case; this returns a 0-dim zero.

Not supported: float64 inputs (TypeError), CPU tensors (RuntimeError), more than 128 anchors.
"""
import ctypes
import os

import numpy as np
import torch
from torch.nn import Module

from ._lib import call
from .assets import default_asset_root

ANCHOR_DIR = os.path.join('pose_data_optimize', 'assets', 'anchor')
N_VERTS = 778
MAX_ANCHORS = 128
# HandPoseConverter.py:43-44: the betas its rest pose is built with
CONVERTER_BETAS = (0.5082395, -0.39488167, -1.7484332, 1.6630946, 0.34428665, -1.37387, 0.38293332, 1.196094, 0.6538949, -0.94331187)
# HandPoseConverter.py:53-57, 82
_AXIS_IDX = ((0, 13, 14, 15), (0, 1, 2, 3), (0, 4, 5, 6), (0, 10, 11, 12), (0, 7, 8, 9))
_JOINTS_MAPPING = (5, 6, 7, 9, 10, 11, 17, 18, 19, 13, 14, 15, 1, 2, 3)


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _check_tensor(who, name, t):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError('renderih_b200.geo_loss.%s: %s must be a CUDA tensor (there is no CPU path)' % (who, name))
    if t.dtype != torch.float32:
        raise TypeError('renderih_b200.geo_loss.%s: %s must be float32, got %s' % (who, name, t.dtype))


def anchor_tables(anchor_root=None, face_vert_idx=None, anchor_weight=None):
    """-> (face_vert_idx [A,3] int64, anchor_weight [A,2] float64), from the arrays given or from face_vertex_idx.txt /
    anchor_weight.txt under anchor_root (default: pose_data_optimize/assets/anchor under the asset root)."""
    root = anchor_root if anchor_root is not None else os.path.join(default_asset_root(), ANCHOR_DIR)
    if face_vert_idx is None:
        face_vert_idx = np.loadtxt(os.path.join(root, 'face_vertex_idx.txt'), dtype=np.int64)
    if anchor_weight is None:
        anchor_weight = np.loadtxt(os.path.join(root, 'anchor_weight.txt'))
    f = np.asarray(face_vert_idx)
    w = np.asarray(anchor_weight, dtype=np.float64)
    if f.ndim != 2 or f.shape[1] != 3 or not np.issubdtype(f.dtype, np.integer) or not 1 <= f.shape[0] <= MAX_ANCHORS:
        raise ValueError('face_vert_idx must be an integer [A,3] array with 1 <= A <= %d, got %s %s' % (MAX_ANCHORS, f.dtype, f.shape))
    if w.shape != (f.shape[0], 2):
        raise ValueError('anchor_weight must be [%d,2], got %s' % (f.shape[0], w.shape))
    if f.min() < 0 or f.max() >= N_VERTS:
        raise ValueError('face_vert_idx indexes vertices outside 0..%d' % (N_VERTS - 1))
    return f.astype(np.int64), w


def edge_index(faces):
    """HandLoss.get_edge_idx (geo_loss.py:162-177): the undirected edges of faces [F,3] in first-seen order, edges (0,1), (1,2), (0,2) of
    each face, each pair in the order Python lists the set {i, j}.  -> [E,2] int64."""
    seen = {}
    for a, b, c in np.asarray(faces).astype(np.int64).tolist():
        for i, j in ((a, b), (b, c), (a, c)):
            if i == j:
                raise ValueError('face (%d, %d, %d) repeats a vertex' % (a, b, c))
            key = (min(i, j), max(i, j))
            if key not in seen:
                seen[key] = list({i, j})
    return np.asarray(list(seen.values()), dtype=np.int64).reshape(-1, 2)


def converter_matrices(side, joints, transf):
    """HandPoseConverter.axis_convert + init_convert_matrix (HandPoseConverter.py:81-130) in float64 from the rest pose's joints [21,3]
    and transforms [16,4,4] -> (invM_U_n_0, invU_M_n_1), each [16,3,3] float32 as the reference stores them."""
    j = np.asarray(joints, dtype=np.float64)
    T = np.asarray(transf, dtype=np.float64)[:, :3, :3]
    jm = np.asarray(_JOINTS_MAPPING)
    x = j[jm] - j[jm + 1]
    if side == 'right':
        up = np.array([[0, 1, 0]] * 12 + [[1, 1, 1]] * 3, dtype=np.float64)
    else:
        x = -x
        up = np.array([[0, -1, 0]] * 12 + [[1, -1, -1]] * 3, dtype=np.float64)     # the second assignment of :90-93
    x = np.einsum('kji,kj->ki', T[1:], x)              # R_k^T x_k
    z = np.cross(x, up)
    y = np.cross(z, x)
    x, y, z = [a / np.linalg.norm(a, axis=-1, keepdims=True) for a in (x, y, z)]
    u = np.tile(np.eye(3), (16, 1, 1))
    u[1:] = np.stack([x, y, z], -1)                     # columns x, y, z
    if side == 'left':
        u[0] = np.diag([1.0, -1.0, -1.0])
    u = T @ u
    inv_m0 = np.tile(np.eye(3), (16, 1, 1)).astype(np.float32)
    inv_u1 = np.tile(np.eye(3), (16, 1, 1)).astype(np.float32)
    for finger in _AXIS_IDX:
        for k, a in enumerate(finger):
            prev, a = (0, 0) if k == 0 else (finger[k - 1], a)
            inv_u1[a] = u[a].T @ T[a]
            inv_m0[a] = T[prev].T @ u[prev]
    return inv_m0, inv_u1


def _conv_table(inv_m0, inv_u1):
    """[15,18] float32 per joint 1..15: P = zero_ja^T invM_U_n_0^T then C = invU_M_n_1^T, so that M = zero_ja^T ja = P R C."""
    out = np.zeros((15, 18), dtype=np.float64)
    for t in range(15):
        A = inv_m0[t + 1].astype(np.float64).T
        C = inv_u1[t + 1].astype(np.float64).T
        out[t, :9] = ((A @ C).T @ A).reshape(9)
        out[t, 9:] = C.reshape(9)
    return out.astype(np.float32)


def _csr(rows, n, *cols):
    """Entries grouped by row, in their given order within a row -> (ptr [n+1], *cols permuted alike)."""
    rows = np.asarray(rows)
    order = np.argsort(rows, kind='stable')
    ptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(ptr, rows + 1, 1)
    return (np.cumsum(ptr),) + tuple(np.asarray(c)[order] for c in cols)


def _anchor_csr(fvi, w):
    """vertex -> (anchor, coefficient of the vertex in the anchor) with coefficients 1 - w1 - w2, w1, w2."""
    A = fvi.shape[0]
    coef = np.stack([1.0 - w[:, 0] - w[:, 1], w[:, 0], w[:, 1]], 1)
    return _csr(fvi.reshape(-1), N_VERTS, np.repeat(np.arange(A), 3), coef.reshape(-1))


class _Tables(Module):
    def _put(self, name, array, dtype):
        self.register_buffer(name, torch.as_tensor(np.ascontiguousarray(array)).to(dtype), persistent=False)


class AnchorLayer(_Tables):
    """manopth.anchorlayer.AnchorLayer: forward(vertices [B,778,3]) -> anchors [B,A,3] (A = 108 for the reference's tables).
    Buffers face_vert_idx [1,A,3] and anchor_weight [1,A,2] as the reference registers them."""

    def __init__(self, anchor_root=None, face_vert_idx=None, anchor_weight=None):
        super().__init__()
        fvi, w = anchor_tables(anchor_root, face_vert_idx, anchor_weight)
        self.register_buffer('face_vert_idx', torch.from_numpy(fvi).long().unsqueeze(0))
        self.register_buffer('anchor_weight', torch.from_numpy(w).float().unsqueeze(0))
        self.fvi = torch.from_numpy(fvi).long()
        self.n_anchors = fvi.shape[0]
        ptr, ent, coef = _anchor_csr(fvi, self.anchor_weight[0].double().numpy())
        self._put('_fvi', fvi, torch.int32)
        self._put('_ptr', ptr, torch.int32)
        self._put('_ent', ent, torch.int32)
        self._put('_coef', coef, torch.float32)

    def forward(self, vertices):
        _check_tensor('AnchorLayer', 'vertices', vertices)
        if vertices.dim() != 3 or tuple(vertices.shape[1:]) != (N_VERTS, 3):
            raise ValueError('vertices must be [B,%d,3], got %s' % (N_VERTS, tuple(vertices.shape)))
        if vertices.device != self._fvi.device:
            raise RuntimeError('AnchorLayer: vertices on %s, layer on %s' % (vertices.device, self._fvi.device))
        return _AnchorFn.apply(self, vertices.contiguous())


class _AnchorFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, verts):
        B = verts.shape[0]
        out = torch.empty(B, layer.n_anchors, 3, device=verts.device)
        with torch.cuda.device(verts.device):
            call('rih_geo_anchor_fwd', layer._fvi.data_ptr(), layer.anchor_weight.data_ptr(), layer.n_anchors, verts.data_ptr(), N_VERTS, B,
                 out.data_ptr(), _stream(verts))
        ctx.layer, ctx.B = layer, B
        return out

    @staticmethod
    def backward(ctx, g):
        layer, B = ctx.layer, ctx.B
        g = g.float().contiguous()
        dv = torch.empty(B, N_VERTS, 3, device=g.device)
        with torch.cuda.device(g.device):
            call('rih_geo_anchor_bwd', layer._ptr.data_ptr(), layer._ent.data_ptr(), layer._coef.data_ptr(), layer.n_anchors, g.data_ptr(),
                 N_VERTS, B, dv.data_ptr(), _stream(g))
        return None, dv


def check_contacts(anchor_id, anchor_elastic, anchor_padding_mask, n_anchors):
    """Validate the optimiser's contact tensors ([B,A,D] each: integer anchor ids in [0,A), float32 elasticities, an integer or bool
    padding mask) -> (anchor_id, anchor_elastic, anchor_padding_mask) as int32 / float32 / int32 tensors on their device.  Synchronises
    with the device when they are CUDA tensors."""
    ids, el, mk = (torch.as_tensor(t) for t in (anchor_id, anchor_elastic, anchor_padding_mask))
    if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
        raise TypeError('anchor_id must be an integer tensor, got %s' % ids.dtype)
    if el.dtype != torch.float32:
        raise TypeError('anchor_elastic must be float32, got %s' % el.dtype)
    if mk.dtype.is_floating_point or mk.dtype.is_complex:
        raise TypeError('anchor_padding_mask must be an integer or bool tensor, got %s' % mk.dtype)
    if ids.dim() != 3 or ids.shape[0] < 1 or ids.shape[1] != n_anchors or ids.shape[2] < 1:
        raise ValueError('anchor_id must be [B,%d,D] with B, D >= 1, got %s' % (n_anchors, tuple(ids.shape)))
    for name, t in (('anchor_elastic', el), ('anchor_padding_mask', mk)):
        if t.shape != ids.shape:
            raise ValueError('%s must have the shape of anchor_id %s, got %s' % (name, tuple(ids.shape), tuple(t.shape)))
    if not (ids.device == el.device == mk.device):
        raise RuntimeError('the contact tensors are on different devices')
    lo, hi = int(ids.min()), int(ids.max())
    if lo < 0 or hi >= n_anchors:
        raise ValueError('anchor_id must lie in [0, %d), got [%d, %d]' % (n_anchors, lo, hi))
    m = mk.long()
    if int(m.min()) < -2 ** 31 or int(m.max()) >= 2 ** 31:
        raise ValueError('anchor_padding_mask values do not fit in int32')
    return ids.to(torch.int32), el, m.to(torch.int32)


class HandPriorLoss(_Tables):
    """The optimiser's quat-norm, edge, contact and ergonomics terms for both hands (see the module docstring).  mano_right / mano_left:
    the optimiser's renderih_b200.manopth.ManoLayer instances of each side, on the CUDA device the loss runs on; they are used at
    construction only.  The anchor tables as for AnchorLayer."""

    def __init__(self, mano_right, mano_left, anchor_root=None, face_vert_idx=None, anchor_weight=None):
        super().__init__()
        from .manopth import ManoLayer
        for want, layer in (('right', mano_right), ('left', mano_left)):
            if not isinstance(layer, ManoLayer):
                raise TypeError('mano_%s must be a renderih_b200.manopth.ManoLayer, got %s' % (want, type(layer).__name__))
            if layer.side != want:
                raise ValueError('mano_%s is a %s-hand layer' % (want, layer.side))
        dev = mano_right.th_v_template.device
        if dev.type != 'cuda':
            raise RuntimeError('HandPriorLoss: the MANO layers must be on a CUDA device (there is no CPU path)')
        if mano_left.th_v_template.device != dev:
            raise RuntimeError('HandPriorLoss: the MANO layers are on %s and %s' % (dev, mano_left.th_v_template.device))
        self.anchor_layer = AnchorLayer(anchor_root, face_vert_idx, anchor_weight).to(dev)
        self.n_anchors = self.anchor_layer.n_anchors
        edges = edge_index(mano_right.th_faces.cpu().numpy())
        if edges.size == 0 or edges.max() >= N_VERTS:
            raise ValueError('the right layer faces index vertices outside 0..%d' % (N_VERTS - 1))
        self.register_buffer('hand_edges', torch.from_numpy(edges).to(dev))
        self.n_edges = edges.shape[0]
        rest, conv, self.converter = [], [], {}
        with torch.no_grad():
            for side, layer in (('right', mano_right), ('left', mano_left)):
                v, joints, transf = _rest_pose(layer, dev)
                rest.append(torch.norm(v[self.hand_edges[:, 0]] - v[self.hand_edges[:, 1]], p=2, dim=-1))    # geo_loss.py:180-183
                inv_m0, inv_u1 = converter_matrices(side, joints, transf)
                self.converter[side] = (inv_m0, inv_u1)
                conv.append(_conv_table(inv_m0, inv_u1))
        self.register_buffer('static_edge_len', torch.stack(rest).contiguous())         # [2,E]: right, left
        n = self.n_edges
        # vertex -> (other vertex, edge): both ends of every edge, in edge order within a vertex
        ptr, other, eid = _csr(edges.reshape(-1), N_VERTS, edges[:, ::-1].reshape(-1), np.repeat(np.arange(n), 2))
        self._put('_edges', edges, torch.int32)
        self._put('_e_ptr', ptr, torch.int32)
        self._put('_e_other', other, torch.int32)
        self._put('_e_id', eid, torch.int32)
        self._put('_conv', np.stack(conv), torch.float32)
        self.to(dev)
        self._contacts = None

    def _table_ptrs(self):
        a = self.anchor_layer
        return [t.data_ptr() for t in (a._fvi, a.anchor_weight, a._ptr, a._ent, a._coef, self._edges, self.static_edge_len, self._e_ptr,
                                       self._e_other, self._e_id, self._conv)]

    def set_contacts(self, anchor_id, anchor_elastic, anchor_padding_mask):
        """The optimiser's contact correspondences (set_opt_val, geo_optimizer_both_batch.py:133-208): [B,A,D] each.  Validated here
        (this may synchronise) and copied into buffers this module owns: a CUDA graph captured over forward / backward replays with the
        contacts set last, as long as B and D do not change."""
        ids, el, mk = check_contacts(anchor_id, anchor_elastic, anchor_padding_mask, self.n_anchors)
        dev = self._conv.device
        cur = self._contacts
        if cur is not None and cur[0].shape == ids.shape:
            for dst, src in zip(cur, (ids, el, mk)):
                dst.copy_(src)
        else:
            self._contacts = tuple(t.to(dev, copy=True).contiguous() for t in (ids, el, mk))

    def forward(self, quat_right, quat_left, verts_right, verts_left):
        for name, t in (('quat_right', quat_right), ('quat_left', quat_left), ('verts_right', verts_right), ('verts_left', verts_left)):
            _check_tensor('HandPriorLoss', name, t)
            if t.device != self._conv.device:
                raise RuntimeError('HandPriorLoss: %s is on %s, the loss on %s' % (name, t.device, self._conv.device))
        B = quat_right.shape[0] if quat_right.dim() else 0
        for name, q in (('quat_right', quat_right), ('quat_left', quat_left)):
            if not ((q.dim() == 3 and tuple(q.shape) == (B, 16, 4)) or (q.dim() == 2 and tuple(q.shape) == (B, 64))):
                raise ValueError('%s must be [B,16,4] or [B,64] with B = %d, got %s' % (name, B, tuple(q.shape)))
        for name, v in (('verts_right', verts_right), ('verts_left', verts_left)):
            if tuple(v.shape) != (B, N_VERTS, 3):
                raise ValueError('%s must be [%d,%d,3], got %s' % (name, B, N_VERTS, tuple(v.shape)))
        if self._contacts is None:
            raise RuntimeError('HandPriorLoss: call set_contacts() before the forward')
        if self._contacts[0].shape[0] != B:
            raise ValueError('HandPriorLoss: the contacts were set for batch %d, the inputs have batch %d' % (self._contacts[0].shape[0], B))
        terms = _PriorFn.apply(self, quat_right.reshape(B, 16, 4).contiguous(), quat_left.reshape(B, 16, 4).contiguous(),
                               verts_right.contiguous(), verts_left.contiguous())
        return tuple(terms.unbind(0))


def _rest_pose(layer, dev):
    """Through the layer's own forward: the identity-pose, zero-beta vertices the optimiser's static edge lengths come from
    (geo_optimizer_both_batch.py:457-470), and the converter's rest joints and transforms (HandPoseConverter.py:58-62: identity
    quaternions, the hard-coded betas, centre joint 9) as float64 arrays."""
    from .manopth import _ManopthFn
    ident = torch.zeros(1, 16, 4, device=dev)
    ident[..., 0] = 1.0
    v = layer(ident.reshape(1, 64), torch.zeros(1, 10, device=dev))[0][0]
    betas = torch.tensor([CONVERTER_BETAS], dtype=torch.float32, device=dev)
    _, joints, transf = _ManopthFn.apply(layer, ident, betas, 0, None, 9, 0, True)
    return v, joints[0].cpu().double().numpy(), transf[0].cpu().double().numpy()


class _PriorFn(torch.autograd.Function):
    """rih_geo_prior_fwd / rih_geo_prior_bwd: terms [4] = quat-norm, edge, contact, ergonomics."""

    @staticmethod
    def forward(ctx, loss, q_r, q_l, v_r, v_l):
        ids, el, mk = loss._contacts
        B, D = q_r.shape[0], ids.shape[2]
        dev = q_r.device
        part = torch.empty(B, 8, device=dev)
        count = torch.empty(B, dtype=torch.int64, device=dev)
        terms = torch.empty(4, device=dev)
        den = torch.empty(1, device=dev)
        tables = loss._table_ptrs()
        with torch.cuda.device(dev):
            call('rih_geo_prior_fwd', _ptr_array(tables), loss.n_anchors, loss.n_edges, q_r.data_ptr(), q_l.data_ptr(), v_r.data_ptr(),
                 v_l.data_ptr(), ids.data_ptr(), el.data_ptr(), mk.data_ptr(), D, B, part.data_ptr(), count.data_ptr(), terms.data_ptr(),
                 den.data_ptr(), _stream(q_r))
        ctx.loss = loss
        ctx.save_for_backward(q_r, q_l, v_r, v_l, ids, el, den)
        return terms

    @staticmethod
    def backward(ctx, g):
        q_r, q_l, v_r, v_l, ids, el, den = ctx.saved_tensors
        loss = ctx.loss
        g = g.float().contiguous()
        need = ctx.needs_input_grad          # (loss, q_r, q_l, v_r, v_l)
        d = [torch.empty_like(t) if need[i + 1] else None for i, t in enumerate((q_r, q_l, v_r, v_l))]
        ptr = lambda t: None if t is None else t.data_ptr()
        with torch.cuda.device(g.device):
            call('rih_geo_prior_bwd', _ptr_array(loss._table_ptrs()), loss.n_anchors, loss.n_edges, q_r.data_ptr(), q_l.data_ptr(),
                 v_r.data_ptr(), v_l.data_ptr(), ids.data_ptr(), el.data_ptr(), ids.shape[2], q_r.shape[0], g.data_ptr(), den.data_ptr(),
                 *[ptr(t) for t in d], _stream(g))
        return (None, *d)


def _ptr_array(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)
