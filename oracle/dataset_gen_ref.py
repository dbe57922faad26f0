"""numpy restatement of the dataset preparation arithmetic (csrc/dataset_gen.cu): the camera geometry of both hands, cut_img's box,
crop matrix and camera update (dataset/dataset_utils.py:12-42), the crop (cv2.warpAffine's fixed-point 8-bit path with any source and
destination size), and HeatmapGenerator (dataset/heatmap.py) with cv.imwrite's uint8 conversion.

The float32 steps are float32 numpy element-wise operations and the float64 steps float64 ones, in the order the kernels use, so the
kernels agree with this module bit for bit where the reference's own `@` (a BLAS call with its own summation order) may differ in the
last bit.  TEST INFRASTRUCTURE -- never imported by the product package.
"""
import numpy as np

from oracle.augment_ref import invert_affine


def cam_xform(p, R, t):
    """p [n,3] float32 @ R.T + t: ((p0*R[r,0] + p1*R[r,1]) + p2*R[r,2]) + t[r] in float32."""
    p, R, t = np.asarray(p, np.float32), np.asarray(R, np.float32), np.asarray(t, np.float32).reshape(3)
    return np.stack([((p[:, 0] * R[r, 0] + p[:, 1] * R[r, 1]) + p[:, 2] * R[r, 2]) + t[r] for r in range(3)], 1)


def project(p, K):
    """(p @ K.T)[:, :2] / (p @ K.T)[:, 2:] in float64 for p [n,3] float32."""
    p, K = np.asarray(p, np.float32).astype(np.float64), np.asarray(K, np.float64)
    h = np.stack([(p[:, 0] * K[r, 0] + p[:, 1] * K[r, 1]) + p[:, 2] * K[r, 2] for r in range(3)], 1)
    return h[:, :2] / h[:, 2:]


def dist_ok(left, right):
    """interhand.py:200-201: min |left_i - right_i| (float32, NaN-propagating) < 9999999."""
    d = np.asarray(left, np.float32) - np.asarray(right, np.float32)
    n = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return bool(n.min() < 9999999)


def cut(pts, radio, img_size, K=None):
    """cut_img without the image for the labels pts [n,2] float64 -> (M [2,3], pts mapped by M [n,2], updated copy of K or None)."""
    pts = np.asarray(pts, np.float64)
    mn, mx = pts.min(0), pts.max(0)
    mid = (mn + mx) / 2
    L = np.max(mx - mn) / 2 / radio
    s = img_size / 2 / L
    M = np.array([[s * 1.0, s * 0.0, s * (L - mid[0])], [s * 0.0, s * 1.0, s * (L - mid[1])]])
    out = np.stack([(pts[:, 0] * M[r, 0] + pts[:, 1] * M[r, 1]) + M[r, 2] for r in range(2)], 1)
    if K is not None:
        K = np.array(K, np.float64)
        K[0, 0] = K[0, 0] * M[0, 0]
        K[1, 1] = K[1, 1] * M[1, 1]
        K[0, 2] = K[0, 2] * M[0, 0] + M[0, 2]
        K[1, 2] = K[1, 2] * M[1, 1] + M[1, 2]
    return M, out, K


def geometry(verts, joints, R, t, K, crop=False, radio=0.8, img_size=256):
    """One frame, both hands: verts / joints {'left','right'} float32 [778,3] / [21,3] (joints may be None).  -> dict like
    renderih_b200.dataset_gen.geometry for one frame (left hand first)."""
    hands = ('left', 'right')
    v3d = np.stack([cam_xform(verts[h], R, t) for h in hands])
    out = {'v3d': v3d, 'v2d': np.stack([project(v, K) for v in v3d]), 'valid': dist_ok(verts['left'], verts['right']),
           'K': np.array(K, np.float64)}
    if joints is not None:
        out['j3d'] = np.stack([cam_xform(joints[h], R, t) for h in hands])
        out['j2d'] = np.stack([project(j, K) for j in out['j3d']])
    if crop:
        M, c, Kc = cut(out['v2d'].reshape(-1, 2), radio, img_size, K)
        out.update(M=M, cut2d=c.reshape(2, -1, 2), K=Kc)
    return out


def warp_u8(img, M, S):
    """cv2.warpAffine(img, M, (S, S)) for uint8 HxWx3 img, INTER_LINEAR, BORDER_CONSTANT 0 (the rule of oracle/augment_ref.warp_affine_u8
    with a destination size of its own)."""
    H, W = img.shape[:2]
    Mi = invert_affine(M)
    x = np.arange(S, dtype=np.float64)
    rnd = lambda v: np.clip(np.rint(v), -2147483648, 2147483647).astype(np.int64)
    adelta, bdelta = rnd(Mi[0, 0] * x * 1024), rnd(Mi[1, 0] * x * 1024)
    X0, Y0 = rnd((Mi[0, 1] * x + Mi[0, 2]) * 1024) + 16, rnd((Mi[1, 1] * x + Mi[1, 2]) * 1024) + 16
    X, Y = (X0[:, None] + adelta[None, :]) >> 5, (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    src = img.astype(np.int64)
    acc = np.zeros((S, S, img.shape[2]), np.int64)
    for dy, dx, w in ((0, 0, (32 - fy) * (32 - fx)), (0, 1, (32 - fy) * fx), (1, 0, fy * (32 - fx)), (1, 1, fy * fx)):
        yy, xx = sy + dy, sx + dx
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        acc += np.where(ok[..., None], src[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0) * w[..., None]
    return ((acc + 512) >> 10).astype(np.uint8)


def heatmaps(joints, res, sigma, scale=1):
    """HeatmapGenerator(res, sigma)(joints, scale) for joints [B,N,2|3] -> [B,N,res,res] float32 (dataset/heatmap.py:4-39)."""
    joints = np.asarray(joints)
    if joints.ndim == 2:
        joints = joints[None]
    if joints.shape[-1] == 2:
        joints = np.concatenate([joints, np.ones_like(joints[..., :1])], -1)
    s = sigma * scale
    xl, yl = np.arange(res, dtype=np.float64)[None, :], np.arange(res, dtype=np.float64)[:, None]
    out = np.zeros(joints.shape[:2] + (res, res), np.float32)
    for b in range(joints.shape[0]):
        for n, pt in enumerate(joints[b]):
            x, y = pt[0], pt[1]
            if pt[2] > 0 and not (x < 0 or y < 0 or x >= res or y >= res):
                out[b, n] = np.exp(-((xl - x) ** 2 + (yl - y) ** 2) / (2 * s ** 2))
    return out


def planes_u8(hms):
    """cv.imwrite's uint8 of hms[k].transpose(1, 2, 0) * 255 for hms [N,res,res] float32 (N = 3K) -> [K,res,res,3] (NaN -> 0)."""
    v = np.asarray(hms, np.float32) * np.float32(255)
    v = np.where(np.isnan(v), 0, np.clip(np.rint(v), 0, 255)).astype(np.uint8)
    return v.reshape(-1, 3, *v.shape[1:]).transpose(0, 2, 3, 1)
