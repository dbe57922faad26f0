"""Two-hand mesh renderer: a drop-in for the reference's `mano_two_hands_renderer` (utils/vis_utils.py:39-100,153-289), which is built on
pytorch3d, plus the per-sample hand mask IoU of utils/compute_maskiou.py:59-64,250-263.  Rasterisation and shading are the CUDA kernels of
csrc/render.cu; there is no CPU path: every tensor input must be a CUDA tensor.  Outputs never require grad (the reference's one
differentiable use, the render loss of common/myhand/decoder.py:411-438, cannot be reached: its import is commented out).

Conventions reproduced (pytorch3d's, as the reference configures them):

* Orthographic camera (`build_camera`, vis_utils.py:62-71: R = diag(-1,-1,1), T = (0,0,10), focal = 2*scale, principal point = -trans2d,
  NDC): a vertex (x,y,z) lands at column u = S*scale*x + S/2*(tx+1), row v = S*scale*y + S/2*(ty+1), where pixel (row r, col c) has
  its centre at (c+0.5, r+0.5).  At S = 256 this is `projection_batch` (utils/manoutils.py:26-44), the model's own verts2d.  Depth z+10.
* Perspective camera (vis_utils.py:72-79, intrinsics K [B,3,3] turned into NDC focal / principal point): u = fx*x/z + cx,
  v = fy*y/z + cy in the same frame, depth z.  A face with any vertex at z <= 0 is not drawn.  Barycentrics are perspective-correct
  (pytorch3d's MeshRasterizer default for a perspective camera).
* Coverage (RasterizationSettings(blur_radius=0, faces_per_pixel=1), vis_utils.py:45-49): a pixel is covered when its centre lies
  strictly inside a face (a centre exactly on an edge is outside); zero-area faces are not drawn; no back-face culling; only the nearest
  face counts, and on equal (fp32) depth the lower face index.
* Faces: cat(right_faces[:, [1,0,2]], right_faces + 778) -- the left hand reuses the right hand's faces with the winding swapped
  (vis_utils.py:166-170); the single-hand methods use the first 1538 rows (:259).
* `render_rgb_orth` maps the right hand into the left hand's camera: s = scale_r/scale_l, d = -(t_l - t_r)/2/scale_l, v_r <- s*v_r,
  v_r.xy += d (vis_utils.py:206-228), in fp32 like the reference, without modifying the caller's tensor.  Both hands share one z-buffer.
* Colours: default vertex colours left (204,153,0), right (102,102,255) (:184-191); masks left (0,0,255), right (0,255,0) with ambient
  light (:230-239); the single-hand mask 255 with ambient light (:267-274); dense pose dense_coor*255 for both hands with ambient light
  (:276-289).
* Shading, HardPhongShader: colour = (ambient + diffuse)*texel + specular with PointLights(location=(0,0,-1)) and pytorch3d's default
  light colours (ambient 0.5, diffuse 0.3, specular 0.2) and Materials (all colours 1, shininess 64); the viewer is the camera centre
  in world coordinates, (0,0,-10) for the orthographic camera and the origin for the perspective one.  Vertex normals are pytorch3d's
  `Meshes.verts_normals` (sum of the corner cross products of a vertex's faces, normalised).  AmbientLights: ambient 1 only.
  UNVERIFIED: these pytorch3d defaults are taken from its documentation; pytorch3d is not a dependency of this package, so they are
  not cross-checked against it here.
* Blend: hard, on a white background (1,1,1); `Renderer.render` divides the colour by 255 (:98-99), so background `img` pixels are
  1/255 -- which the `== 1` mask test of compute_maskiou relies on.  alpha is 1 on covered pixels, 0 elsewhere.
* Mask IoU (`bm0`, compute_maskiou.py:59-64): |L n R| / (|L| + |R| - |L n R|) of the two hands' single-hand coverage masks, NaN when
  both are empty (numpy's 0/0).

Not supported (NotImplementedError): UV textures (`uv_verts` / `uv_faces` / `texture`, which no reference caller passes), custom
`lights`, and a tuple `img_size` (the non-square 480x640 `render_tzionas` path, compute_maskiou.py:281).
Fragments: `pix_to_face` holds the face index within each image (pytorch3d packs it across the batch), -1 for background.
"""
import collections
import os

import numpy as np
import torch

from ._lib import call
from .assets import default_asset_root, load_mano_dict, load_pickle
from .config import get_cfg_defaults

HAND_V = 778
Fragments = collections.namedtuple('Fragments', 'pix_to_face zbuf bary_coords')   # [B,S,S,1], [B,S,S,1], [B,S,S,1,3] (faces_per_pixel = 1)


def _require_cuda(name, *tensors):
    for t in tensors:
        if t is not None and not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError('renderih_b200.render.%s: CUDA tensors required (there is no CPU path)' % name)


def _square(img_size):
    if isinstance(img_size, (tuple, list)):
        raise NotImplementedError('non-square images (the 480x640 render_tzionas path, utils/compute_maskiou.py:281) are not supported')
    return int(img_size)


def _camera(B, cameras=None, scale=None, trans2d=None):
    """-> (cam [B,4] fp32 contiguous, perspective flag).  Orthographic (scale [B], trans2d [B,2]) wins when given, as in build_camera."""
    if scale is not None and trans2d is not None:
        _require_cuda('camera', scale, trans2d)
        cam = torch.cat([scale.detach().float().reshape(-1, 1), trans2d.detach().float().reshape(-1, 2), torch.zeros_like(scale, dtype=torch.float32).reshape(-1, 1)], 1)
        return cam.expand(B, 4).contiguous(), 0
    if cameras is not None:
        _require_cuda('camera', cameras)
        K = cameras.detach().float()
        cam = torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], 1)
        return cam.expand(B, 4).contiguous(), 1
    raise ValueError('a camera is required: cameras [B,3,3] (perspective) or scale [B] with trans2d [B,2] (orthographic)')


def _verts(name, v):
    _require_cuda(name, v)
    if v.dim() != 3 or v.shape[2] != 3:
        raise ValueError('renderih_b200.render.%s: vertices must be [B,V,3], got %s' % (name, tuple(v.shape)))
    return v.detach().float().contiguous()


def _faces(faces, device):
    f = faces if isinstance(faces, torch.Tensor) else torch.from_numpy(np.asarray(faces, dtype=np.int64))
    f = f.to(device=device, dtype=torch.int32).contiguous()
    if f.dim() != 2 or f.shape[1] != 3:
        raise ValueError('faces must be [F,3]')
    return f


def _raster_keys(verts, faces, cam, persp, S):
    B, V = verts.shape[:2]
    keys = torch.empty(B, S, S, dtype=torch.int64, device=verts.device)     # uint64 keys, see csrc/render.cu
    call('rih_render_raster', verts.data_ptr(), B, V, faces.data_ptr(), faces.shape[0], cam.data_ptr(), persp, S, keys.data_ptr(),
         torch.cuda.current_stream(verts.device).cuda_stream)
    return keys


def rasterize(verts, faces, camera, img_size):
    """Fragments of the nearest face per pixel.  verts [B,V,3] CUDA; faces [F,3] (any integer array, shared by the batch; a face naming a
    vertex outside [0,V) is not drawn); camera: intrinsics [B,3,3] (perspective) or a (scale [B], trans2d [B,2]) pair (orthographic).
    -> Fragments(pix_to_face int32 [B,S,S,1] (-1 background), zbuf [B,S,S,1] (-1), bary_coords [B,S,S,1,3] (-1))."""
    S = _square(img_size)
    verts = _verts('rasterize', verts)
    B, V = verts.shape[:2]
    if isinstance(camera, (tuple, list)):
        cam, persp = _camera(B, scale=camera[0], trans2d=camera[1])
    else:
        cam, persp = _camera(B, cameras=camera)
    f = _faces(faces, verts.device)
    keys = _raster_keys(verts, f, cam, persp, S)
    p2f = torch.empty(B, S, S, dtype=torch.int32, device=verts.device)
    zbuf = torch.empty(B, S, S, device=verts.device)
    bary = torch.empty(B, S, S, 3, device=verts.device)
    call('rih_render_shade', keys.data_ptr(), verts.data_ptr(), None, B, V, f.data_ptr(), f.shape[0], cam.data_ptr(), persp, S, None, None, None,
         p2f.data_ptr(), zbuf.data_ptr(), bary.data_ptr(), torch.cuda.current_stream(verts.device).cuda_stream)
    return Fragments(p2f.unsqueeze(-1), zbuf.unsqueeze(-1), bary.unsqueeze(-2))


def hand_mask_iou(v3d_left, v3d_right, faces, img_size, cameras=None, scale=None, trans2d=None):
    """Per-sample IoU [B] (fp32, NaN when both masks are empty) of the two hands' coverage masks, each hand rasterised alone with faces
    [F,3] through the same camera (intrinsics [B,3,3], or scale [B] + trans2d [B,2]) -- utils/compute_maskiou.py:250-263.  Feeds the
    occlusion buckets of `EvalMetrics.summary(mask)` (apps/eval_interhand.py:230-234)."""
    S = _square(img_size)
    vl, vr = _verts('hand_mask_iou', v3d_left), _verts('hand_mask_iou', v3d_right)
    if vl.shape != vr.shape:
        raise ValueError('hand_mask_iou: both hands need the same [B,V,3] shape')
    B, V = vl.shape[:2]
    cam, persp = _camera(B, cameras, scale, trans2d)
    f = _faces(faces, vl.device)
    bits = torch.empty(2 * B * S * ((S + 31) // 32), dtype=torch.int32, device=vl.device)
    iou = torch.empty(B, device=vl.device)
    call('rih_render_mask_iou', vl.data_ptr(), vr.data_ptr(), B, V, f.data_ptr(), f.shape[0], cam.data_ptr(), persp, S, bits.data_ptr(),
         iou.data_ptr(), torch.cuda.current_stream(vl.device).cuda_stream)
    return iou


def _vertex_face_csr(faces, V):
    """vertex -> (3 * face + corner) in ascending face order: the fixed summation order of the vertex normals."""
    flat = faces.reshape(-1)
    order = np.argsort(flat, kind='stable').astype(np.int32)
    ptr = np.zeros(V + 1, np.int32)
    ptr[1:] = np.cumsum(np.bincount(flat, minlength=V))
    return ptr, order


class _Mesh:
    """Device-side faces and the vertex -> face CSR of one face set."""

    def __init__(self, faces, V, device):
        self.V = V
        self.faces = torch.from_numpy(np.ascontiguousarray(faces, dtype=np.int32)).to(device)
        ptr, corner = _vertex_face_csr(faces, V)
        self.vf_ptr, self.vf_corner = torch.from_numpy(ptr).to(device), torch.from_numpy(corner).to(device)


class mano_two_hands_renderer:
    """utils/vis_utils.py:153-289 on the GPU.  mano_path: {'left','right'} of MANO pickle paths or loaded MANO dicts (as ManoLayer takes);
    dense_path: the v_color.pkl path or a [778,3] array.  Defaults resolve under the asset root ($RIH_ASSET_ROOT), as load_model does.
    Only the right hand's faces are used (the left hand's are the same with the winding swapped, vis_utils.py:166-170)."""

    def __init__(self, mano_path=None, dense_path=None, img_size=224, device='cuda'):
        self.img_size = _square(img_size)
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('mano_two_hands_renderer: a CUDA device is required (there is no CPU path)')
        cfg, root = get_cfg_defaults(), default_asset_root()
        if mano_path is None:
            mano_path = {s: os.path.join(root, cfg.MISC.MANO_PATH, 'MANO_%s.pkl' % s.upper()) for s in ('left', 'right')}
        right = mano_path['right'] if isinstance(mano_path['right'], dict) else load_mano_dict(mano_path['right'])
        rf = np.asarray(right['f'], dtype=np.int64)
        if rf.ndim != 2 or rf.shape[1] != 3 or rf.min() < 0 or rf.max() >= HAND_V:
            raise ValueError('MANO faces must be [F,3] indices into %d vertices' % HAND_V)
        self.faces_np = np.concatenate([rf[:, [1, 0, 2]], rf + HAND_V])
        self.faces = torch.from_numpy(self.faces_np).to(self.device).unsqueeze(0)         # [1,2F,3] int64, as the reference's self.faces
        self._two = _Mesh(self.faces_np, 2 * HAND_V, self.device)
        self._one = _Mesh(self.faces_np[:len(rf)], HAND_V, self.device)
        if dense_path is None:
            dense_path = os.path.join(root, cfg.MISC.DENSE_COLOR)
        dense = load_pickle(dense_path) if isinstance(dense_path, (str, os.PathLike)) else dense_path
        self.dense_coor = torch.as_tensor(np.asarray(dense, dtype=np.float32)).to(self.device) * 255
        if tuple(self.dense_coor.shape) != (HAND_V, 3):
            raise ValueError('dense colours must be [%d,3]' % HAND_V)
        col = torch.zeros(2 * HAND_V, 3, device=self.device)
        col[:HAND_V] = torch.tensor([204., 153., 0.]); col[HAND_V:] = torch.tensor([102., 102., 255.])
        self._rgb_colors = col
        col = torch.zeros(2 * HAND_V, 3, device=self.device)
        col[:HAND_V, 2] = 255; col[HAND_V:, 1] = 255
        self._mask_colors = col
        self._dense_colors = torch.cat([self.dense_coor, self.dense_coor]).contiguous()
        self._single_colors = torch.ones(HAND_V, 3, device=self.device)
        self._single_mask_colors = torch.full((HAND_V, 3), 255., device=self.device)

    # ---- core: raster -> (normals) -> shade
    def _render(self, mesh, verts, colors, cameras, scale, trans2d, amblights):
        verts = _verts('mano_two_hands_renderer', verts)
        B, V = verts.shape[:2]
        if V != mesh.V:
            raise ValueError('expected [B,%d,3] vertices, got %s' % (mesh.V, tuple(verts.shape)))
        colors = torch.as_tensor(colors).to(device=verts.device, dtype=torch.float32).expand(V, 3).contiguous()
        cam, persp = _camera(B, cameras, scale, trans2d)
        S, st = self.img_size, torch.cuda.current_stream(verts.device).cuda_stream
        keys = _raster_keys(verts, mesh.faces, cam, persp, S)
        normals = None
        if not amblights:
            normals = torch.empty(B, V, 3, device=verts.device)
            call('rih_render_vertex_normals', verts.data_ptr(), B, V, mesh.faces.data_ptr(), mesh.vf_ptr.data_ptr(), mesh.vf_corner.data_ptr(),
                 normals.data_ptr(), st)
        img = torch.empty(B, S, S, 3, device=verts.device)
        alpha = torch.empty(B, S, S, device=verts.device)
        call('rih_render_shade', keys.data_ptr(), verts.data_ptr(), None if normals is None else normals.data_ptr(), B, V, mesh.faces.data_ptr(),
             mesh.faces.shape[0], cam.data_ptr(), persp, S, colors.data_ptr(), img.data_ptr(), alpha.data_ptr(), None, None, None, st)
        return img, alpha

    @staticmethod
    def _unsupported(uv_verts=None, uv_faces=None, texture=None, lights=None):
        if uv_verts is not None or uv_faces is not None or texture is not None:
            raise NotImplementedError('UV textures are not supported (no reference caller passes uv_verts / uv_faces / texture)')
        if lights is not None:
            raise NotImplementedError('custom lights are not supported: amblights selects AmbientLights, otherwise PointLights at (0,0,-1)')

    def _two_hands(self, v3d_left, v3d_right):
        _require_cuda('mano_two_hands_renderer', v3d_left, v3d_right)
        return torch.cat((v3d_left.detach(), v3d_right.detach()), dim=1)

    # ---- the reference's methods
    def render_rgb(self, cameras=None, scale=None, trans2d=None, v3d_left=None, v3d_right=None, uv_verts=None, uv_faces=None, texture=None,
                   v_color=None, amblights=False, lights=None):
        """vis_utils.py:176-204 -> (img [B,S,S,3], alpha [B,S,S])."""
        self._unsupported(uv_verts, uv_faces, texture, lights)
        colors = self._rgb_colors if v_color is None else v_color
        return self._render(self._two, self._two_hands(v3d_left, v3d_right), colors, cameras, scale, trans2d, amblights)

    def render_rgb_orth(self, scale_left=None, trans2d_left=None, scale_right=None, trans2d_right=None, v3d_left=None, v3d_right=None,
                        uv_verts=None, uv_faces=None, texture=None, v_color=None, amblights=False):
        """vis_utils.py:206-228: both hands through the left hand's orthographic camera -> (img, alpha)."""
        self._unsupported(uv_verts, uv_faces, texture)
        _require_cuda('render_rgb_orth', scale_left, trans2d_left, scale_right, trans2d_right, v3d_right)
        scale_left, trans2d_left = scale_left.detach(), trans2d_left.detach()
        s = (scale_right.detach() / scale_left).unsqueeze(-1).unsqueeze(-1)
        d = (-(trans2d_left - trans2d_right.detach()) / 2 / scale_left.unsqueeze(-1)).unsqueeze(1)
        vr = s * v3d_right.detach()                 # a new tensor: the caller's v3d_right is not modified
        vr[..., :2] = vr[..., :2] + d
        return self.render_rgb(scale=scale_left, trans2d=trans2d_left, v3d_left=v3d_left, v3d_right=vr, v_color=v_color, amblights=amblights)

    def render_mask(self, cameras=None, scale=None, trans2d=None, v3d_left=None, v3d_right=None):
        """vis_utils.py:230-239 -> img [B,S,S,3]: left (0,0,1), right (0,1,0), background 1/255."""
        return self.render_rgb(cameras, scale, trans2d, v3d_left, v3d_right, v_color=self._mask_colors, amblights=True)[0]

    def render_single_rgb(self, cameras=None, scale=None, trans2d=None, v3d_left=None, v3d_right=None, uv_verts=None, uv_faces=None, texture=None,
                          v_color=None, amblights=False, lights=None):
        """vis_utils.py:241-263: v3d_left alone with the first 1538 faces -> (img, alpha).  v3d_right is ignored, as in the reference."""
        self._unsupported(uv_verts, uv_faces, texture, lights)
        colors = self._single_colors if v_color is None else v_color
        return self._render(self._one, v3d_left, colors, cameras, scale, trans2d, amblights)

    def render_single_mask(self, cameras=None, scale=None, trans2d=None, v3d=None):
        """vis_utils.py:267-274 -> img [B,S,S,3]: 1 on the hand, 1/255 elsewhere."""
        return self.render_single_rgb(cameras, scale, trans2d, v3d, v_color=self._single_mask_colors, amblights=True)[0]

    def render_densepose(self, cameras=None, scale=None, trans2d=None, v3d_left=None, v3d_right=None):
        """vis_utils.py:276-289 -> (img, alpha) with the dense-pose colours of both hands, ambient light."""
        return self._render(self._two, self._two_hands(v3d_left, v3d_right), self._dense_colors, cameras, scale, trans2d, True)

    def mask_iou(self, cameras=None, scale=None, trans2d=None, v3d_left=None, v3d_right=None):
        """`hand_mask_iou` with this renderer's single-hand faces and image size (compute_maskiou.py:250-263) -> [B]."""
        return hand_mask_iou(v3d_left, v3d_right, self._one.faces, self.img_size, cameras, scale, trans2d)
