"""Dataset preparation on the GPU: drop-ins for the reference's utils/dataset_gen/interhand.py (`--gen_anno 1`: crops and annotations of
InterHand2.6M's interacting frames; `--gen_anno 0`: the ori_handdict labels), rendering_code/step7_gen_annotations.py (heatmaps, masks and
dense maps of RenderIH's frames, and their ori_handdict labels), dataset/heatmap.py's HeatmapGenerator and dataset/dataset_utils.py's cut_img.

    select_data(data_path, save_path, 'train')                      # img/{idx}.jpg, anno/{idx}.pkl
    InterHand_dataset(save_path, 'train', 0).run()                   # ori_handdict/{idx}.npy
    render_data(save_path, 'train', start_idx)                       # color_hms / color_mask / color_dense
    step7.InterHand_dataset(data_path, 'train', start).run()        # ori_handdict/{idx}.npy of the RenderIH layout
    main(['--gen_anno', '1', '--data_path', ..., '--save_path', ...]);  step7.main([...])

Frames go through in batches (512 by default, the reference's DataLoader batch): both hands through ManoLayer (csrc/mano.cu), then the
camera geometry and crop box (rih_dsgen_geometry), the crop and frame mean (rih_dsgen_crop_u8), the heatmaps (rih_dsgen_heatmaps) and
the renderer's mask and dense map with per-frame cameras (csrc/render.cu); csrc/dataset_gen.cu lists the dtype of every step.  JSON,
pickle, cv.imread / cv.imwrite and np.save stay on the host, overlapped by a thread pool; file names, the idx numbering and every dict
key and dtype are the reference's.  numpy input to HeatmapGenerator and cut_img is staged through the GPU and returned as numpy; CUDA
tensors stay on the device.  CPU tensors raise RuntimeError, unsupported dtypes TypeError, wrong shapes ValueError.

Reproduced quirks:
* load_mano's bare `except` turns any failure of a hand's parameters (missing entry, wrong length) into None (interhand.py:155-174), and
  cut_inter_img skips such a frame (:197);
* idx advances only for kept frames (:188, 227);
* the `dist < 9999999` test (:200-201) fails only for NaN: the minimum over vertex index of |left_i - right_i| propagates NaN;
* a frame whose mean is below 10 is skipped after its dist test (:202-204);
* heatmaps are written as {idx}_{k}_{hand}.jpg for k = 0..6 (joints 3k..3k+2 as the three channels), left hand first
  (step7_gen_annotations.py:258-278);
* hand_dict['R'] = R @ params['R'][0], the camera rotation times the root rotation (interhand.py:285, step7_gen_annotations.py:343);
* fix_shape flips the left hand's shapedirs[:, 0, :] when the two hands' are near-identical (interhand.py:21-24).

Deviations:
* vis=1 and plot_2d_hand raise NotImplementedError (there is no matplotlib);
* step 7's render_data loop runs to start_idx + 100000 and raises FileNotFoundError at the first missing annotation
  (step7_gen_annotations.py:249-251); the drop-in stops there instead;
* the mask and dense map come from this package's renderer (renderih_b200.render), not pytorch3d;
* there is no tqdm bar; the scripts' main() has no default data paths (the reference's are its authors' directories);
* a missing frame image raises FileNotFoundError before its batch is written (the reference fails on `img.mean()` of None after writing the
  frames before it); a camera that cannot be loaded raises for the first kept frame that needs it, as in the reference;
* the camera transform (v @ cam_R.T + cam_t) requires float32 cam_R / cam_t, which is what load_camera produces;
* cut_img takes uint8 HxWx3 images only, the frames every caller passes.
"""
import argparse
import concurrent.futures
import glob
import json
import os
import os.path as osp
import pickle

import numpy as np
import torch

from ._lib import call
from .assets import default_asset_root
from .config import get_cfg_defaults
from .manolayer import ManoLayer
from .rotations import rodrigues_batch

IMG_SIZE, HAND_BBOX_RATIO, HEATMAP_SIZE, HEATMAP_SIGMA = 256, 0.8, 64, 2      # dataset/dataset_utils.py:4-7
BATCH = 512
HAND_V, HAND_J = 778, 21
SIDES = ('left', 'right')
_IO_THREADS = 8


def _cv():
    import cv2
    return cv2


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _stage(who, x, dtypes):
    """-> (tensor in dtypes[0], came_from_numpy): a CUDA tensor of a dtype in dtypes converted as numpy would, or a numpy array's host copy
    (the caller checks its shape, then moves it to the device)."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise RuntimeError('%s: a CUDA tensor or a numpy array is required, got a CPU tensor (there is no CPU path)' % who)
        if x.dtype not in dtypes:
            raise TypeError('%s: expected %s, got %s' % (who, ' or '.join(str(d) for d in dtypes), x.dtype))
        return x.to(dtypes[0]).contiguous(), False
    a = np.asarray(x)
    want = {torch.float64: np.float64, torch.float32: np.float32, torch.uint8: np.uint8}
    if a.dtype not in [np.dtype(want[d]) for d in dtypes]:
        raise TypeError('%s: expected %s, got %s' % (who, ' or '.join(str(d) for d in dtypes), a.dtype))
    return torch.from_numpy(np.ascontiguousarray(a, dtype=want[dtypes[0]])), True


def get_mano_path():
    """utils/manoutils.py:68-74: the MANO pickles under the asset root ($RIH_ASSET_ROOT)."""
    path = os.path.join(default_asset_root(), get_cfg_defaults().MISC.MANO_PATH)
    return {'left': os.path.join(path, 'MANO_LEFT.pkl'), 'right': os.path.join(path, 'MANO_RIGHT.pkl')}


def fix_shape(mano_layer):
    """interhand.py:21-24: flip the left hand's first shape direction when it equals the right hand's (the MANO release's bug)."""
    if torch.sum(torch.abs(mano_layer['left'].shapedirs[:, 0, :] - mano_layer['right'].shapedirs[:, 0, :])) < 1:
        print('Fix shapedirs bug of MANO')
        mano_layer['left'].shapedirs[:, 0, :] *= -1


def _mano_layers(mano_path):
    layers = {'right': ManoLayer(mano_path['right'], center_idx=None), 'left': ManoLayer(mano_path['left'], center_idx=None)}
    fix_shape(layers)
    return layers


def plot_2d_hand(*args, **kwargs):
    raise NotImplementedError('plot_2d_hand needs matplotlib, which this package does not use')


# ------------------------------------------------------------------------------------------------------------------------ kernels
class HeatmapGenerator:
    """dataset/heatmap.py:11-39 on the GPU.  joints [N,2|3] or [B,N,2|3] float32 / float64 (the third column is visibility)
    -> hms [B,N,res,res] float32 (rih_dsgen_heatmaps).  planes=True also returns the uint8 [B,N/3,res,res,3] images cv.imwrite makes of
    hms[k].transpose(1, 2, 0) * 255."""

    def __init__(self, output_res=128, sigma=-1):
        self.output_res = output_res
        if sigma < 0:
            sigma = self.output_res / 32
        self.sigma = sigma

    def __call__(self, joints, scale=1, planes=False):
        j, as_np = _stage('HeatmapGenerator', joints, (torch.float64, torch.float32))
        if j.dim() == 2:
            j = j[None]
        if j.dim() != 3 or j.shape[-1] not in (2, 3):
            raise ValueError('HeatmapGenerator: joints must be [N,2|3] or [B,N,2|3], got %s' % (tuple(j.shape),))
        if j.shape[-1] == 2:
            j = torch.cat([j, torch.ones_like(j[..., :1])], -1)
        j = j.to('cuda').contiguous()
        B, N, res = j.shape[0], j.shape[1], int(self.output_res)
        if planes and N % 3:
            raise ValueError('HeatmapGenerator: planes need a multiple of 3 joints, got %d' % N)
        sigma = self.sigma * scale
        hms = torch.empty(B, N, res, res, device=j.device)
        pl = torch.empty(B, N // 3, res, res, 3, dtype=torch.uint8, device=j.device) if planes else None
        with torch.cuda.device(j.device):
            call('rih_dsgen_heatmaps', j.data_ptr(), B, N, res, float(2 * sigma ** 2), hms.data_ptr(), None if pl is None else pl.data_ptr(), _stream(j))
        out = (hms, pl) if planes else (hms,)
        out = tuple(t.cpu().numpy() for t in out) if as_np else out
        return out if planes else out[0]


def heatmap_planes(joints, res=HEATMAP_SIZE, sigma=HEATMAP_SIGMA):
    """Only the uint8 planes of HeatmapGenerator(res, sigma)(joints): joints [B,N,3] CUDA float64 -> [B,N/3,res,res,3] uint8."""
    B, N = joints.shape[:2]
    pl = torch.empty(B, N // 3, res, res, 3, dtype=torch.uint8, device=joints.device)
    call('rih_dsgen_heatmaps', joints.data_ptr(), B, N, res, float(2 * sigma ** 2), None, pl.data_ptr(), _stream(joints))
    return pl


def crop_u8(frames, M, size=IMG_SIZE, sums=False):
    """cv.warpAffine(frames[b], M[b], (size, size)) for frames [B,H,W,3] CUDA uint8 and M [B,2,3] CUDA float64 forward matrices
    -> crops [B,size,size,3] uint8 (and with sums=True the exact int64 byte sum of each source frame)."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and isinstance(M, torch.Tensor) and M.is_cuda):
        raise RuntimeError('crop_u8: CUDA tensors required (there is no CPU path)')
    if frames.dtype != torch.uint8 or M.dtype != torch.float64:
        raise TypeError('crop_u8: frames must be uint8 and M float64, got %s / %s' % (frames.dtype, M.dtype))
    if frames.dim() != 4 or frames.shape[3] != 3 or tuple(M.shape) != (frames.shape[0], 2, 3):
        raise ValueError('crop_u8: expected frames [B,H,W,3] and M [B,2,3], got %s / %s' % (tuple(frames.shape), tuple(M.shape)))
    frames, M = frames.contiguous(), M.contiguous()
    B, H, W = frames.shape[:3]
    out = torch.empty(B, size, size, 3, dtype=torch.uint8, device=frames.device)
    s = torch.empty(B, dtype=torch.int64, device=frames.device) if sums else None
    with torch.cuda.device(frames.device):
        call('rih_dsgen_crop_u8', frames.data_ptr(), B, H, W, M.data_ptr(), int(size), out.data_ptr(), None if s is None else s.data_ptr(), _stream(frames))
    return (out, s) if sums else out


def geometry(verts, joints, R, t, K, crop=False, radio=HAND_BBOX_RATIO, img_size=IMG_SIZE):
    """rih_dsgen_geometry for B frames: verts / joints {'left','right'} of CUDA float32 [B,778,3] / [B,21,3] (joints may be None), R [B,3,3]
    and t [B,3] CUDA float32, K [B,3,3] CUDA float64.  -> dict of CUDA tensors: v3d, j3d, v2d, j2d (left hand first), valid (the dist
    test), K (updated by cut_img when crop) and, when crop, M [B,2,3] and cut2d (the 2-D verts mapped by M)."""
    B, dev = verts['left'].shape[0], verts['left'].device
    for who, x, dt in (('verts', verts['left'], torch.float32), ('verts', verts['right'], torch.float32), ('R', R, torch.float32),
                       ('t', t, torch.float32), ('K', K, torch.float64)):
        if not x.is_cuda:
            raise RuntimeError('geometry: CUDA tensors required (there is no CPU path)')
        if x.dtype != dt:
            raise TypeError('geometry: %s must be %s, got %s' % (who, dt, x.dtype))
    if tuple(verts['right'].shape) != (B, HAND_V, 3) or tuple(verts['left'].shape) != (B, HAND_V, 3) or tuple(R.shape) != (B, 3, 3) \
            or tuple(t.shape) != (B, 3) or tuple(K.shape) != (B, 3, 3):
        raise ValueError('geometry: expected verts [B,778,3], R [B,3,3], t [B,3], K [B,3,3]')
    c = lambda x: None if x is None else x.contiguous()
    vl, vr, R, t, K = c(verts['left']), c(verts['right']), c(R), c(t), c(K)
    jl = jr = None
    if joints is not None:
        jl, jr = c(joints['left']), c(joints['right'])
        if tuple(jl.shape) != (B, HAND_J, 3) or tuple(jr.shape) != (B, HAND_J, 3) or jl.dtype != torch.float32 or jr.dtype != torch.float32:
            raise ValueError('geometry: joints must be float32 [B,21,3]')
    e = lambda *s, dt=torch.float64: torch.empty(*s, dtype=dt, device=dev)
    out = {'v3d': e(B, 2, HAND_V, 3, dt=torch.float32), 'v2d': e(B, 2, HAND_V, 2), 'valid': e(B, dt=torch.int32), 'K': e(B, 3, 3)}
    if joints is not None:
        out.update(j3d=e(B, 2, HAND_J, 3, dt=torch.float32), j2d=e(B, 2, HAND_J, 2))
    if crop:
        out.update(M=e(B, 2, 3), cut2d=e(B, 2, HAND_V, 2))
    p = lambda k: out[k].data_ptr() if k in out else None
    with torch.cuda.device(dev):
        call('rih_dsgen_geometry', vl.data_ptr(), vr.data_ptr(), None if jl is None else jl.data_ptr(), None if jr is None else jr.data_ptr(),
             R.data_ptr(), t.data_ptr(), K.data_ptr(), B, int(crop), float(radio), int(img_size), p('v3d'), p('j3d'), p('v2d'), p('j2d'),
             p('valid'), p('M'), p('K'), p('cut2d'), _stream(vl))
    return out


def cut_img(img_list, label2d_list, camera=None, radio=0.7, img_size=256):
    """dataset/dataset_utils.py:12-42: crop every image of img_list around the box of all labels (rih_dsgen_cut, rih_dsgen_crop_u8).
    -> (images [img_size,img_size,3] uint8, labels [n,2] float64 mapped by M, camera).  camera (3x3, numpy or CUDA tensor) is
    updated in place and returned, like the reference."""
    labels, as_np = [], True
    for lab in label2d_list:
        x, from_np = _stage('cut_img', lab, (torch.float64, torch.float32))
        if x.dim() != 2 or x.shape[1] != 2:
            raise ValueError('cut_img: labels must be [n,2], got %s' % (tuple(x.shape),))
        labels.append(x.to('cuda'))
        as_np = as_np and from_np
    pts = torch.cat(labels).contiguous()
    dev = pts.device
    M = torch.empty(1, 2, 3, dtype=torch.float64, device=dev)
    cut = torch.empty_like(pts)
    K = None
    if camera is not None:
        K, _ = _stage('cut_img', camera, (torch.float64, torch.float32))
        if tuple(K.shape) != (3, 3):
            raise ValueError('cut_img: camera must be 3x3')
        K = K.to('cuda').contiguous().clone()
    with torch.cuda.device(dev):
        call('rih_dsgen_cut', pts.data_ptr(), 1, pts.shape[0], float(radio), int(img_size), M.data_ptr(), cut.data_ptr(),
             None if K is None else K.data_ptr(), _stream(pts))
    imgs = []
    for img in img_list:
        f, from_np = _stage('cut_img', img, (torch.uint8,))
        if f.dim() != 3 or f.shape[2] != 3:
            raise ValueError('cut_img: images must be HxWx3 uint8, got %s' % (tuple(f.shape),))
        out = crop_u8(f.to(dev)[None], M, img_size)[0]
        imgs.append(out.cpu().numpy() if from_np else out)
    outs = list(torch.split(cut, [x.shape[0] for x in labels]))
    if as_np:
        outs = [o.cpu().numpy() for o in outs]
    if camera is not None:
        if isinstance(camera, torch.Tensor):
            camera.copy_(K)
        else:
            camera[...] = K.cpu().numpy()
    return imgs, outs, camera


# ------------------------------------------------------------------------------------------------------------------------ MANO
def _parse_hand(param):
    """The parameter handling of load_mano (interhand.py:157-169) -> (root axis [3], pose [45], shape [10], trans [3]) float32 tensors,
    raising on anything the reference's try block would fail on."""
    pose = torch.FloatTensor(param['pose']).view(-1, 3)
    shape = torch.FloatTensor(param['shape']).view(1, -1)
    trans = torch.FloatTensor(param['trans']).view(1, 3)
    if pose.shape[0] != 16 or shape.shape[1] != 10:
        raise ValueError('MANO parameters of the wrong size')
    return pose[0], pose[1:].reshape(45), shape[0], trans[0]


class _Mano:
    """Both hands' ManoLayer on the device; the PCA pose and root rotation conversions run on the host, one frame at a time, as in
    the reference, so their results do not depend on the batch size."""

    def __init__(self, mano_path, device):
        self.layer = _mano_layers(mano_path if mano_path is not None else get_mano_path())
        self.device = torch.device(device)

    def from_axis(self, hand, root, pose, shape, trans):
        """root [n,3], pose [n,45] axis-angle -> (mano params {'R','pose','shape','trans'} as float32 numpy [n,...], verts, joints)."""
        layer = self.layer[hand]
        with torch.no_grad():
            R = rodrigues_batch(root)
            pca = torch.cat([layer.axis2pca(pose[k:k + 1] + layer.hands_mean) for k in range(pose.shape[0])])
        return {'R': R, 'pose': pca, 'shape': shape, 'trans': trans}, *self.forward(hand, R, pca, shape, trans)

    def forward(self, hand, R, pca, shape, trans):
        d = lambda x: torch.as_tensor(x, dtype=torch.float32).to(self.device)
        with torch.no_grad():
            return self.layer[hand](d(R), d(pca), d(shape), trans=d(trans))


def _hand_dicts(mano, datas):
    """InterHand_dataset.__getitem__'s label dicts (interhand.py:259-289, step7_gen_annotations.py:317-347) for the loaded annotations
    -> (list of hand_dict, geometry output)."""
    verts, joints = {}, {}
    for hand in SIDES:      # params: R [1,3,3], pose [1,45], shape [1,10], trans [1,3], as load_mano stores them
        ps = [d['mano_params'][hand] for d in datas]
        verts[hand], joints[hand] = mano.forward(hand, *(np.concatenate([np.asarray(p[k], np.float32) for p in ps]) for k in ('R', 'pose', 'shape', 'trans')))
    cams = [d['camera'] for d in datas]
    for c in cams:
        if np.asarray(c['R']).dtype != np.float32 or np.asarray(c['t']).dtype != np.float32:
            raise TypeError('camera R and t must be float32, as load_camera writes them')
    dev = mano.device
    R = torch.from_numpy(np.stack([np.asarray(c['R']).reshape(3, 3) for c in cams])).to(dev)
    t = torch.from_numpy(np.stack([np.asarray(c['t']).reshape(3) for c in cams])).to(dev)
    K = torch.from_numpy(np.stack([np.asarray(c['camera'], np.float64) for c in cams])).to(dev)
    g = geometry(verts, joints, R, t, K)
    h = {k: g[k].cpu().numpy() for k in ('v3d', 'j3d', 'v2d', 'j2d')}
    out = []
    for b, d in enumerate(datas):
        hd = {}
        for k, hand in enumerate(SIDES):
            params = d['mano_params'][hand]
            hd[hand] = {'hms': [], 'verts3d': h['v3d'][b, k].copy(), 'joints3d': h['j3d'][b, k].copy(), 'verts2d': h['v2d'][b, k].copy(),
                        'joints2d': h['j2d'][b, k].copy(), 'R': d['camera']['R'] @ params['R'][0], 'pose': params['pose'][0],
                        'shape': params['shape'][0], 'camera': d['camera']['camera']}
        out.append(hd)
    return out, g


def _batches(n, batch_size):
    for lo in range(0, n, batch_size):
        yield range(lo, min(n, lo + batch_size))


def _wait(futures):
    for f in futures:
        f.result()


# ------------------------------------------------------------------------------------------------------------------------ interhand.py
class InterHandLoader:
    """interhand.py:88-181.  mano_path: {'left','right'} MANO pickle paths or dicts (default: get_mano_path())."""

    def __init__(self, data_path, split='train', mano_path=None, device='cuda'):
        assert split in ['train', 'test', 'val']
        self.root_path = data_path
        self.img_root_path = os.path.join(self.root_path, 'images')
        self.annot_root_path = os.path.join(self.root_path, 'annotations')
        self.mano = _Mano(mano_path, device)
        self.mano_layer = self.mano.layer
        self.split = split
        base = osp.join(self.annot_root_path, self.split, 'InterHand2.6M_' + self.split)
        with open(base + '_data.json') as f:
            self.data_info = json.load(f)
        with open(base + '_camera.json') as f:
            self.cam_params = json.load(f)
        with open(base + '_joint_3d.json') as f:
            self.joints = json.load(f)
        with open(base + '_MANO_NeuralAnnot.json') as f:
            self.mano_params = json.load(f)
        self.data_size = len(self.data_info['images'])

    def __len__(self):
        return self.data_size

    def show_data(self, idx):
        for k in self.data_info['images'][idx].keys():
            print(k, self.data_info['images'][idx][k])
        for k in self.data_info['annotations'][idx].keys():
            print(k, self.data_info['annotations'][idx][k])

    def load_camera(self, idx):
        """interhand.py:126-144 (host numpy): cam_R [3,3] and cam_t [3] float32, cameraIn [3,3] float64."""
        img_info = self.data_info['images'][idx]
        cam_param = self.cam_params[str(img_info['capture'])]
        cam_idx = str(img_info['camera'])
        cam_t = np.array(cam_param['campos'][cam_idx], dtype=np.float32).reshape(3)
        cam_R = np.array(cam_param['camrot'][cam_idx], dtype=np.float32).reshape(3, 3)
        cam_t = -np.dot(cam_R, cam_t.reshape(3, 1)).reshape(3) / 1000
        focal = np.array(cam_param['focal'][cam_idx], dtype=np.float32).reshape(2)
        princpt = np.array(cam_param['princpt'][cam_idx], dtype=np.float32).reshape(2)
        cameraIn = np.array([[focal[0], 0, princpt[0]],
                             [0, focal[1], princpt[1]],
                             [0, 0, 1]])
        return cam_R, cam_t, cameraIn

    def load_mano_batch(self, idxs):
        """load_mano for every frame of idxs, both hands batched through ManoLayer.
        -> (mano_dicts: list of {'left','right'} -> {'R','pose','shape','trans'} float32 numpy or None,
            verts {'left','right'} CUDA [n,778,3], joints [n,21,3] (NaN rows where a hand failed), ok [n,2] bool numpy (left, right))."""
        n = len(idxs)
        dicts = [{} for _ in range(n)]
        ok = np.zeros((n, 2), bool)
        verts, joints = {}, {}
        for k, hand in enumerate(SIDES):
            rows, parsed = [], []
            for r, i in enumerate(idxs):
                info = self.data_info['images'][i]
                try:
                    parsed.append(_parse_hand(self.mano_params[str(info['capture'])][str(info['frame_idx'])][hand]))
                    rows.append(r)
                except Exception:      # the reference's bare except (interhand.py:172-174)
                    dicts[r][hand] = None
            v = torch.full((n, HAND_V, 3), float('nan'), device=self.mano.device)
            j = torch.full((n, HAND_J, 3), float('nan'), device=self.mano.device)
            if rows:
                root, pose, shape, trans = (torch.stack([p[c] for p in parsed]) for c in range(4))
                params, hv, hj = self.mano.from_axis(hand, root, pose, shape, trans)
                sel = torch.tensor(rows, device=self.mano.device)
                v[sel], j[sel] = hv, hj
                for q, r in enumerate(rows):
                    dicts[r][hand] = {key: params[key][q:q + 1].numpy().copy() for key in ('R', 'pose', 'shape', 'trans')}
                    ok[r, k] = True
            verts[hand], joints[hand] = v, j
        return dicts, verts, joints, ok

    def load_mano(self, idx):
        """interhand.py:146-176 -> (mano_dict, coord_dict); coord_dict[hand] = {'verts' [1,778,3], 'joints' [1,21,3]} CPU tensors or None."""
        dicts, verts, joints, ok = self.load_mano_batch([idx])
        coord = {h: ({'verts': verts[h].cpu(), 'joints': joints[h].cpu()} if ok[0, k] else None) for k, h in enumerate(SIDES)}
        return dicts[0], coord

    def load_img(self, idx):
        img_info = self.data_info['images'][idx]
        return _cv().imread(osp.join(self.img_root_path, self.split, img_info['file_name']))


def cut_inter_img(loader, save_path, split, batch_size=BATCH):
    """interhand.py:184-227 in batches: img/{idx}.jpg and anno/{idx}.pkl of every kept interacting frame."""
    cv = _cv()
    os.makedirs(osp.join(save_path, split, 'img'), exist_ok=True)
    os.makedirs(osp.join(save_path, split, 'anno'), exist_ok=True)
    dev = loader.mano.device
    idx = 0
    with concurrent.futures.ThreadPoolExecutor(_IO_THREADS) as pool:
        for chunk in _batches(len(loader), batch_size):
            cand = [i for i in chunk if loader.data_info['annotations'][i]['hand_type'] == 'interacting'
                    and loader.data_info['annotations'][i]['hand_type_valid']]
            if not cand:
                continue
            dicts, verts, _, ok = loader.load_mano_batch(cand)
            cams, cam_err = [], {}
            for r, i in enumerate(cand):
                try:
                    cams.append(loader.load_camera(i))
                except Exception as e:     # raised only if the frame gets as far as load_camera (interhand.py:206)
                    cam_err[r] = e
                    cams.append((np.eye(3, dtype=np.float32), np.zeros(3, np.float32), np.eye(3)))
            R = torch.from_numpy(np.stack([c[0] for c in cams])).to(dev)
            t = torch.from_numpy(np.stack([c[1] for c in cams])).to(dev)
            K = torch.from_numpy(np.stack([c[2] for c in cams])).to(dev)
            g = geometry(verts, None, R, t, K, crop=True)
            valid = g['valid'].cpu().numpy().astype(bool) & ok.all(1)
            rows = [r for r in range(len(cand)) if valid[r]]
            if not rows:
                continue
            imgs = list(pool.map(loader.load_img, [cand[r] for r in rows]))
            for r, im in zip(rows, imgs):
                if im is None:
                    raise FileNotFoundError('cannot read the image of frame %d: %s' % (cand[r], loader.data_info['images'][cand[r]]['file_name']))
            crops, means = [None] * len(rows), [None] * len(rows)
            for shape in sorted({im.shape for im in imgs}):
                ks = [k for k, im in enumerate(imgs) if im.shape == shape]
                if len(shape) != 3 or shape[2] != 3 or imgs[ks[0]].dtype != np.uint8:
                    raise ValueError('frames must be HxWx3 uint8 images, got %s %s' % (shape, imgs[ks[0]].dtype))
                src = torch.from_numpy(np.stack([imgs[k] for k in ks])).to(dev)
                c, s = crop_u8(src, g['M'][[rows[k] for k in ks]], IMG_SIZE, sums=True)
                c, s = c.cpu().numpy(), s.cpu().numpy()
                for q, k in enumerate(ks):
                    crops[k], means[k] = c[q], np.float64(s[q]) / np.float64(imgs[k].size)
            Kc = g['K'].cpu().numpy()
            futures = []
            for k, r in enumerate(rows):
                if means[k] < 10:
                    continue
                if r in cam_err:
                    raise cam_err[r]
                i = cand[r]
                data_info = {'inter_idx': idx, 'image': loader.data_info['images'][i], 'annotation': loader.data_info['annotations'][i],
                             'mano_params': dicts[r], 'camera': {'R': cams[r][0], 't': cams[r][1], 'camera': Kc[r].copy()}}
                futures.append(pool.submit(cv.imwrite, osp.join(save_path, split, 'img', '{}.jpg'.format(idx)), crops[k]))
                futures.append(pool.submit(_dump_pickle, osp.join(save_path, split, 'anno', '{}.pkl'.format(idx)), data_info))
                idx = idx + 1
            _wait(futures)
    return idx


def _dump_pickle(path, obj):
    with open(path, 'wb') as file:
        pickle.dump(obj, file)


def _load_pickle(path):
    with open(path, 'rb') as file:
        return pickle.load(file)


def select_data(DATA_PATH, save_path, split, mano_path=None, batch_size=BATCH):
    """interhand.py:230-232."""
    loader = InterHandLoader(DATA_PATH, split=split, mano_path=mano_path)
    return cut_inter_img(loader, save_path, split, batch_size)


class _OriHandDict:
    """The ori_handdict pass shared by both scripts' InterHand_dataset: frame idx + start reads img/{.}.jpg and anno/{.}.pkl and writes
    ori_handdict/{.}.npy."""
    img_dir = ann_dir = out_dir = None

    def __len__(self):
        return self.size

    def __getitem__(self, idx):
        return self.get_batch([idx])[0]

    def get_batch(self, idxs):
        """-> [(img, hand_dict)] for the frames idx + start of idxs; writes their ori_handdict files."""
        cv = _cv()
        ids = [i + self.start_idx for i in idxs]
        with concurrent.futures.ThreadPoolExecutor(_IO_THREADS) as pool:
            imgs = pool.map(lambda i: cv.imread(osp.join(self.img_dir, '{}.jpg'.format(i))), ids)
            datas = list(pool.map(lambda i: _load_pickle(os.path.join(self.ann_dir, '{}.pkl'.format(i))), ids))
            dicts, _ = _hand_dicts(self.mano, datas)
            _wait([pool.submit(np.save, os.path.join(self.out_dir, '{}'.format(i)), d) for i, d in zip(ids, dicts)])
            return list(zip(imgs, dicts))

    def run(self, batch_size=BATCH):
        """The script's DataLoader loop over the whole dataset (interhand.py:309-317, step7_gen_annotations.py:380-387)."""
        for chunk in _batches(len(self), batch_size):
            self.get_batch(list(chunk))


class InterHand_dataset(_OriHandDict):
    """interhand.py:234-291: data_path/split/{img,anno} -> data_path/split/ori_handdict."""

    def __init__(self, data_path, split, start, mano_path=None, device='cuda'):
        assert split in ['train', 'test', 'val']
        self.split = split
        self.mano = _Mano(mano_path, device)
        self.mano_layer = self.mano.layer
        os.makedirs(os.path.join(data_path, self.split, 'ori_handdict'), exist_ok=True)
        self.data_path = data_path
        self.size = len(glob.glob(osp.join(data_path, split, 'anno', '*.pkl')))
        self.start_idx = start
        self.img_dir, self.ann_dir = osp.join(data_path, split, 'img'), osp.join(data_path, split, 'anno')
        self.out_dir = os.path.join(data_path, split, 'ori_handdict')


def main(argv=None):
    """interhand.py:294-317: --gen_anno 1 writes the crops and annotations of train and test, --gen_anno 0 their ori_handdict labels
    (--data_path is then the processed directory, as in the reference)."""
    parser = argparse.ArgumentParser()
    parser.add_argument('--gen_anno', type=int, default=0)
    parser.add_argument('--data_path', type=str, required=True)
    parser.add_argument('--save_path', type=str, default=None)
    parser.add_argument('--start', type=int, default=0)
    parser.add_argument('--batch_size', type=int, default=BATCH)
    opt = parser.parse_args(argv)
    if opt.gen_anno:
        if opt.save_path is None:
            parser.error('--save_path is required with --gen_anno 1')
        for split in ['train', 'test']:
            select_data(opt.data_path, opt.save_path, split, batch_size=opt.batch_size)
    else:
        for split in ['train', 'test']:
            dataset = InterHand_dataset(data_path=opt.data_path, split=split, start=opt.start)
            print('len dataset ', len(dataset), flush=True)
            dataset.run(opt.batch_size)


# ------------------------------------------------------------------------------------------------------------------------ step 7
def render_data(save_path, split, start_idx, mano_path=None, dense_path=None, batch_size=BATCH, device='cuda'):
    """step7_gen_annotations.py:235-288 in batches: color_hms/{idx}_{k}_{hand}.jpg, color_mask/{idx}.jpg and color_dense/{idx}.jpg for
    color_annot/{idx}.pkl, idx = start_idx, start_idx + 1, ... up to the first missing annotation (at most 100000).  -> frames done."""
    from .render import mano_two_hands_renderer
    cv = _cv()
    for d in ('color_mask', 'color_dense', 'color_hms'):
        os.makedirs(osp.join(save_path, split, d), exist_ok=True)
    mano_path = mano_path if mano_path is not None else get_mano_path()
    mano = _Mano(mano_path, device)
    renderer = mano_two_hands_renderer(mano_path=mano_path, dense_path=dense_path, img_size=IMG_SIZE, device=device)
    print(' start idx ', start_idx, flush=True)
    ann = lambda i: osp.join(save_path, split, 'color_annot', '{}.pkl'.format(i))
    idx, stop = start_idx, start_idx + 100000
    with concurrent.futures.ThreadPoolExecutor(_IO_THREADS) as pool:
        while idx < stop:
            ids = []
            while len(ids) < batch_size and idx + len(ids) < stop and osp.exists(ann(idx + len(ids))):
                ids.append(idx + len(ids))
            if not ids:
                break
            idx += len(ids)
            datas = list(pool.map(lambda i: _load_pickle(ann(i)), ids))
            _, g = _hand_dicts(mano, datas)
            B = len(ids)
            j = g['j2d'] * HEATMAP_SIZE / IMG_SIZE                                    # [B,2,21,2]
            j = torch.cat([j, torch.ones_like(j[..., :1])], -1).reshape(B * 2, HAND_J, 3).contiguous()
            planes = heatmap_planes(j).reshape(B, 2, HAND_J // 3, HEATMAP_SIZE, HEATMAP_SIZE, 3)
            cams = torch.from_numpy(np.stack([np.asarray(d['camera']['camera'], np.float64) for d in datas])).to(mano.device).float()
            vl, vr = g['v3d'][:, 0], g['v3d'][:, 1]
            mask = renderer.render_mask(cameras=cams, v3d_left=vl, v3d_right=vr)
            dense, _ = renderer.render_densepose(cameras=cams, v3d_left=vl, v3d_right=vr)
            mask, dense = _to_u8(mask, 255.0).cpu().numpy(), _to_u8(dense, 255.0).cpu().numpy()
            planes = planes.cpu().numpy()
            futures = []
            for b, i in enumerate(ids):
                for h, hand in enumerate(SIDES):
                    for k in range(HAND_J // 3):
                        futures.append(pool.submit(cv.imwrite, os.path.join(save_path, split, 'color_hms', '{}_{}_{}.jpg'.format(i, k, hand)), planes[b, h, k]))
                futures.append(pool.submit(cv.imwrite, osp.join(save_path, split, 'color_mask', '{}.jpg'.format(i)), mask[b]))
                futures.append(pool.submit(cv.imwrite, osp.join(save_path, split, 'color_dense', '{}.jpg'.format(i)), dense[b]))
            _wait(futures)
    return idx - start_idx


def _to_u8(x, scale):
    """cv.imwrite's conversion of the float32 image x * scale (rih_dsgen_scale_u8)."""
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    call('rih_dsgen_scale_u8', x.data_ptr(), x.numel(), float(scale), out.data_ptr(), _stream(x))
    return out


class Step7Dataset(_OriHandDict):
    """step7_gen_annotations.py:291-359 (its InterHand_dataset): data_path/{color_img,color_annot} -> data_path/ori_handdict."""

    def __init__(self, data_path, split, start, vis=0, mano_path=None, device='cuda'):
        assert split in ['train', 'test', 'val']
        if vis:
            raise NotImplementedError('vis=1 plots with matplotlib, which this package does not use')
        self.split = split
        self.mano = _Mano(mano_path, device)
        self.mano_layer = self.mano.layer
        self.data_path = data_path
        self.size = len(glob.glob(osp.join(data_path, 'color_annot', '*.pkl')))
        os.makedirs(os.path.join(self.data_path, 'ori_handdict'), exist_ok=True)
        self.start_idx = start
        self.vis = vis
        self.img_dir, self.ann_dir = osp.join(data_path, 'color_img'), osp.join(data_path, 'color_annot')
        self.out_dir = os.path.join(data_path, 'ori_handdict')


def step7_main(argv=None):
    """step7_gen_annotations.py:363-387: --gen_anno 1 renders the labels of the train split from --start, --gen_anno 0 writes its
    ori_handdict labels."""
    parser = argparse.ArgumentParser()
    parser.add_argument('--gen_anno', type=int, default=0)
    parser.add_argument('--data_path', type=str, default=None)
    parser.add_argument('--save_path', type=str, default=None)
    parser.add_argument('--vis', type=int, default=0)
    parser.add_argument('--start', type=int, default=366358)
    parser.add_argument('--batch_size', type=int, default=BATCH)
    opt = parser.parse_args(argv)
    if opt.gen_anno:
        if opt.save_path is None:
            parser.error('--save_path is required with --gen_anno 1')
        for split in ['train']:
            render_data(opt.save_path, split, opt.start, batch_size=opt.batch_size)
    else:
        if opt.data_path is None:
            parser.error('--data_path is required with --gen_anno 0')
        for split in ['train']:
            dataset = Step7Dataset(data_path=opt.data_path, split=split, start=opt.start, vis=opt.vis)
            print('len dataset ', len(dataset), flush=True)
            dataset.run(opt.batch_size)


class step7:
    """The names of rendering_code/step7_gen_annotations.py, which reuses interhand.py's names for its own dataset class."""
    render_data = staticmethod(render_data)
    InterHand_dataset = Step7Dataset
    InterHandLoader = InterHandLoader
    select_data = staticmethod(select_data)
    fix_shape = staticmethod(fix_shape)
    main = staticmethod(step7_main)
