"""H100-native drop-in for the reference's `models/manolayer.py` ManoLayer (FK + LBS), lines 100-322.

Same constructor / forward contract; forward is ONE fused CUDA kernel (csrc/mano.cu).  Inputs on the CPU
(the reference's dataset code calls the layer with CPU tensors, dataset/interhand.py:102-109) are staged to
the GPU and the outputs are returned on the input's device -- the arithmetic always runs on the GPU.
"""
import ctypes

import numpy as np
import torch
from torch.nn import Module

from . import ops
from .assets import load_mano_dict
from ._lib import call
from .rotations import build_mano_frame, rodrigues_batch, rotmat_to_axis, se3_apply, se3_from, vec2mat   # noqa: F401  (re-exported API surface)


class ManoLayer(Module):
    def __init__(self, manoPath, center_idx=9, use_pca=True, new_skel=False, device=None, out_scale=None):
        super().__init__()
        # out_scale = 1000: the `common/utils/manolayer.py` copy of this layer converts its outputs to millimetres (lines 323-325)
        self.out_scale = out_scale
        self.center_idx = center_idx
        self.use_pca = use_pca
        self.new_skel = new_skel
        manoData = manoPath if isinstance(manoPath, dict) else load_mano_dict(manoPath)
        self.new_order = [0, 13, 14, 15, 16, 1, 2, 3, 17, 4, 5, 6, 18, 10, 11, 12, 19, 7, 8, 9, 20]
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32)))
        self.register_buffer('hands_components', f32(manoData['hands_components']))
        self.register_buffer('hands_components_inv', torch.inverse(self.hands_components))
        jr = manoData['J_regressor']
        jr = np.asarray(jr.todense()) if hasattr(jr, 'todense') else np.asarray(jr)
        self.register_buffer('J_regressor', f32(jr), persistent=False)
        self.register_buffer('J_zero', f32(manoData['J']), persistent=False)
        self.register_buffer('weights', f32(manoData['weights']), persistent=False)
        self.register_buffer('posedirs', f32(manoData['posedirs']), persistent=False)
        self.register_buffer('v_template', f32(manoData['v_template']), persistent=False)
        self.register_buffer('shapedirs', f32(manoData['shapedirs']), persistent=False)
        self.register_buffer('hands_mean', f32(manoData['hands_mean']), persistent=False)
        self.faces = manoData['f']
        self.parent = [-1] + [int(manoData['kintree_table'][0, i]) for i in range(1, 16)]
        self._parent_arr = (ctypes.c_int * 16)(*[max(p, 0) for p in self.parent])
        self._derived = None
        self._run_device = device

    def get_faces(self):
        return self.faces

    def train(self, mode=True):   # the reference overrides these without recursing (manolayer.py:157-161)
        self.is_train = mode

    def eval(self):
        self.train(False)

    # ---- parameter conversions between the PCA / axis-angle / rotation-matrix pose representations (API of models/manolayer.py:163-248;
    #      formulations in renderih_b200/rotations.py).  Light host-side helpers, not on the hot path.
    def pca2axis(self, pca):
        """[bs, n<=45] PCA coefficients -> [bs,45] axis-angle (first n principal components + mean pose)."""
        return torch.addmm(self.hands_mean, pca, self.hands_components[:pca.shape[1]])

    def axis2pca(self, axis):
        return torch.mm(axis - self.hands_mean, self.hands_components_inv)

    def axis2Rmat(self, axis):
        return rodrigues_batch(axis.reshape(-1, 3)).reshape(-1, 15, 3, 3)

    def Rmat2axis(self, R):
        return rotmat_to_axis(R).reshape(-1, 45)

    def pca2Rmat(self, pca):
        return self.axis2Rmat(self.pca2axis(pca))

    def Rmat2pca(self, R):
        return self.axis2pca(self.Rmat2axis(R))

    def get_local_frame(self, shape):
        """Zero-pose local joint frames [bs,15,3,3] for shape coefficients [bs,10] (models/manolayer.py:217-227).  The finger tips of this
        helper are vertices 744/320/444/555/672 -- NOT the 745/317/444/556/673 of forward() -- exactly as in the reference."""
        with torch.no_grad():
            v = self.v_template + torch.einsum('vck,bk->bvc', self.shapedirs, shape)
            j21 = torch.cat([torch.einsum('jv,bvc->bjc', self.J_regressor, v), v[:, [744, 320, 444, 555, 672]]], dim=1)
            return build_mano_frame(j21[:, self.new_order])

    buildSE3_batch = staticmethod(se3_from)
    SE3_apply = staticmethod(se3_apply)

    # ---- device-side constant tables (transposed for coalesced reads); rebuilt if a buffer is mutated in place
    def _tables(self, device):
        bufs = (self.hands_components, self.hands_mean, self.shapedirs, self.posedirs, self.v_template, self.J_regressor, self.weights)
        key = (device,) + tuple((b._version, b.data_ptr()) for b in bufs)
        if self._derived is None or self._derived[0] != key:
            t = [self.hands_components.to(device).contiguous(), self.hands_mean.to(device).contiguous(),
                 self.shapedirs.to(device).reshape(2334, 10).t().contiguous(),     # [10][2334]
                 self.posedirs.to(device).reshape(2334, 135).t().contiguous(),     # [135][2334]
                 self.v_template.to(device).reshape(2334).contiguous(),
                 self.J_regressor.to(device).contiguous(), self.weights.to(device).contiguous()]
            arr = (ctypes.c_void_p * 7)(*[x.data_ptr() for x in t])
            self._derived = (key, t, arr)
        return self._derived[2]

    def forward(self, root_rotation, pose, shape, trans=None, scale=None):
        """-> (verts [B,778,3], joints [B,21,3]); differentiable w.r.t. every tensor argument (one fused backward kernel)."""
        in_dev = root_rotation.device
        if in_dev.type == 'cuda':
            dev = in_dev
        else:
            if not torch.cuda.is_available():
                raise RuntimeError('renderih_b200.ManoLayer needs a CUDA device (sm_90a); there is no CPU fallback')
            dev = torch.device(self._run_device or 'cuda')
        f = lambda t: None if t is None else t.to(device=dev, dtype=torch.float32)     # keeps the autograd graph
        R, P, S, T, C = f(root_rotation), f(pose), f(shape), f(trans), f(scale)
        bs = R.shape[0]
        if self.use_pca:
            assert P.dim() == 2 and P.shape[1] <= 45
        else:
            assert tuple(P.shape[1:]) == (15, 3, 3)
        assert S.shape == (bs, 10)
        v, j = _ManoFn.apply(self, R, P, S, T, C)
        if self.out_scale is not None:
            v, j = v * self.out_scale, j * self.out_scale
        if in_dev != dev:
            v, j = v.to(in_dev), j.to(in_dev)
        return v, j


class _ManoFn(torch.autograd.Function):
    """rih_mano_fwd / rih_mano_bwd (csrc/mano.cu): ManoLayer.forward, models/manolayer.py:250-322, and its gradient."""

    @staticmethod
    def forward(ctx, layer, R, P, S, T, C):
        dev = R.device
        R, P, S = R.contiguous(), P.contiguous(), S.contiguous()
        T = None if T is None else T.contiguous()
        C = None if C is None else C.contiguous()
        bs = R.shape[0]
        ncomps = P.shape[1] if layer.use_pca else 0
        v = torch.empty((bs, 778, 3), device=dev, dtype=torch.float32)
        j = torch.empty((bs, 21, 3), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            tables = layer._tables(dev)
            call('rih_mano_fwd', tables, layer._parent_arr, R.data_ptr(), P.data_ptr(), int(layer.use_pca), ncomps, S.data_ptr(),
                 ops._p(T), ops._p(C), -1 if layer.center_idx is None else int(layer.center_idx), int(layer.new_skel),
                 v.data_ptr(), j.data_ptr(), bs, torch.cuda.current_stream(dev).cuda_stream)
        ctx.layer = layer
        ctx.ncomps = ncomps
        ctx.save_for_backward(R, P, S, T, C)
        return v, j

    @staticmethod
    def backward(ctx, gv, gj):
        R, P, S, T, C = ctx.saved_tensors
        layer, dev, bs = ctx.layer, R.device, R.shape[0]
        c = lambda g: None if g is None else g.contiguous().float()
        gv, gj = c(gv), c(gj)
        need = ctx.needs_input_grad      # (layer, R, P, S, T, C)
        dR = torch.empty_like(R) if need[1] else None
        dP = torch.empty_like(P) if need[2] else None
        dS = torch.empty_like(S) if need[3] else None
        dT = torch.empty_like(T) if (T is not None and need[4]) else None
        dC = torch.empty_like(C) if (C is not None and need[5]) else None
        with torch.cuda.device(dev):
            tables = layer._tables(dev)
            call('rih_mano_bwd', tables, layer._parent_arr, R.data_ptr(), P.data_ptr(), int(layer.use_pca), ctx.ncomps, S.data_ptr(),
                 ops._p(T), ops._p(C), -1 if layer.center_idx is None else int(layer.center_idx), int(layer.new_skel),
                 ops._p(gv), ops._p(gj), ops._p(dR), ops._p(dP), ops._p(dS), ops._p(dT), ops._p(dC), bs,
                 torch.cuda.current_stream(dev).cuda_stream)
        return None, dR, dP, dS, dT, dC
