"""Float64 numpy oracle of the two-hand renderer (renderih_b200/render.py, csrc/render.cu), written from the conventions stated in
render.py's docstring -- pytorch3d's rasteriser and HardPhongShader as utils/vis_utils.py:39-289 configures them -- not from the
CUDA code: projection for both cameras, the strict-interior edge test at pixel centres, the depth test with ties to the lower face
index, perspective-correct barycentrics, vertex normals, Phong / ambient shading, the hard blend, the division by 255, and the mask IoU.

Besides its answer, the oracle flags each pixel whose answer an implementation may legitimately get otherwise ("ambiguous"):
  * EDGE: the centre is within TOL_PX pixels of an edge line of the winning face, or of any face that covers or nearly covers it at a
    depth not behind the winner (such a face could be counted as covering and win).  The CUDA kernels evaluate the projection and the
    edge functions in fp64 from the same fp32 inputs, in a different operation order; at the image sizes used (S <= 8192) that moves a
    centre relative to an edge by < 1e-11 px, so TOL_PX = 1e-6 px flags every centre whose side could differ, and no more than a
    1e-6 px band around each edge.  Comparisons against inputs that went through fp32 arithmetic (the model's verts2d) pass a larger
    tol_px.
  * DEPTH: the winner and another covering face have depths within TOL_DEPTH relative of each other.  The kernels order faces by the
    fp32 rounding of the depth (ties to the lower face index), which cannot reverse an order but can merge two depths less than
    2 ulp apart: TOL_DEPTH = 2^-22.
In coverage mode (masks, IoU, 2-D rasterisation) depth plays no part: a pixel is ambiguous when no face covers it away from an edge
and some face covers or nearly covers it.
"""
import numpy as np

TOL_PX = 1e-6
TOL_DEPTH = 2.0 ** -22
HAND_V = 778
AMBIENT, DIFFUSE, SPECULAR, SHININESS = 0.5, 0.3, 0.2, 64.0
LIGHT = np.array([0.0, 0.0, -1.0])


# ----------------------------------------------------------------------------- cameras
def ortho_cam(scale, trans2d):
    """[B] scale, [B,2] trans2d -> [B,4] camera rows (scale, tx, ty, 0)."""
    scale, trans2d = np.asarray(scale, np.float64).reshape(-1), np.asarray(trans2d, np.float64).reshape(-1, 2)
    return np.stack([scale, trans2d[:, 0], trans2d[:, 1], np.zeros_like(scale)], 1)


def persp_cam(K):
    """[B,3,3] intrinsics -> [B,4] camera rows (fx, fy, cx, cy)."""
    K = np.asarray(K, np.float64)
    return np.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], 1)


def project(verts, cam, persp, S):
    """verts [V,3] -> (u, v, depth) [V] each.  Orthographic (vis_utils.py:62-71 in pytorch3d's NDC): u = S*scale*x + S/2*(tx+1), depth z+10;
    perspective (:72-79): u = fx*x/z + cx, depth z.  Pixel (r,c) has its centre at (c+0.5, r+0.5)."""
    X = np.asarray(verts, np.float64)
    c = np.asarray(cam, np.float64)
    if persp:
        z = X[:, 2]
        return c[0] * X[:, 0] / z + c[2], c[1] * X[:, 1] / z + c[3], z
    return S * c[0] * X[:, 0] + S / 2 * (c[1] + 1), S * c[0] * X[:, 1] + S / 2 * (c[2] + 1), X[:, 2] + 10.0


def orth_right_into_left(scale_l, trans2d_l, scale_r, trans2d_r, v_right):
    """render_rgb_orth's map of the right hand into the left camera (vis_utils.py:214-220), in float32 with the reference's operation order."""
    f = np.float32
    sl, sr = np.asarray(scale_l, f), np.asarray(scale_r, f)
    tl, tr = np.asarray(trans2d_l, f), np.asarray(trans2d_r, f)
    s = (sr / sl)[:, None, None]
    d = (-(tl - tr) / f(2) / sl[:, None])[:, None, :]
    v = s * np.asarray(v_right, f)
    v[..., :2] = v[..., :2] + d
    return v


# ----------------------------------------------------------------------------- rasterisation of one image
def _pairs(u, v, d, faces, S, persp, tol_px):
    """Every (pixel, face) pair whose centre the face covers or nearly covers -> dict of flat arrays."""
    faces = np.asarray(faces, np.int64)
    U, Vv, D = u[faces], v[faces], d[faces]
    ok = np.isfinite(U).all(1) & np.isfinite(Vv).all(1) & np.isfinite(D).all(1)
    if persp:
        ok &= (D > 0).all(1)
    area = (U[:, 1] - U[:, 0]) * (Vv[:, 2] - Vv[:, 0]) - (Vv[:, 1] - Vv[:, 0]) * (U[:, 2] - U[:, 0])
    ok &= area != 0
    fid = np.nonzero(ok)[0]
    pad = 2 * tol_px
    with np.errstate(invalid='ignore'):
        c0 = np.clip(np.ceil(U[fid].min(1) - 0.5 - pad), 0, S).astype(np.int64)
        c1 = np.clip(np.floor(U[fid].max(1) - 0.5 + pad), -1, S - 1).astype(np.int64)
        r0 = np.clip(np.ceil(Vv[fid].min(1) - 0.5 - pad), 0, S).astype(np.int64)
        r1 = np.clip(np.floor(Vv[fid].max(1) - 0.5 + pad), -1, S - 1).astype(np.int64)
    w_, h_ = np.maximum(c1 - c0 + 1, 0), np.maximum(r1 - r0 + 1, 0)
    keep = (w_ > 0) & (h_ > 0)
    fid, c0, r0, w_, h_ = fid[keep], c0[keep], r0[keep], w_[keep], h_[keep]
    n = w_ * h_
    out = {k: [] for k in ('pix', 'face', 'inside', 'near', 'w')}
    start, chunk = 0, 1 << 22
    while start < len(fid):          # chunks of at most ~4M pairs
        stop = start + 1
        tot = n[start]
        while stop < len(fid) and tot + n[stop] <= chunk:
            tot += n[stop]; stop += 1
        sel = slice(start, stop)
        f = np.repeat(fid[sel], n[sel])
        loc = np.arange(tot) - np.repeat(np.cumsum(n[sel]) - n[sel], n[sel])
        ww = np.repeat(w_[sel], n[sel])
        r = np.repeat(r0[sel], n[sel]) + loc // ww
        c = np.repeat(c0[sel], n[sel]) + loc % ww
        px, py = c + 0.5, r + 0.5
        sgn = np.sign(area[f])
        W, near_k, cand = [], [], np.ones(tot, bool)
        for k in range(3):
            a, b = (k + 1) % 3, (k + 2) % 3
            du, dv = U[f, b] - U[f, a], Vv[f, b] - Vv[f, a]
            wk = du * (py - Vv[f, a]) - dv * (px - U[f, a])
            tol = tol_px * (np.abs(du) + np.abs(dv))        # |w| / edge length is the distance to the edge line
            cand &= sgn * wk > -tol
            near_k.append(np.abs(wk) <= tol)
            W.append(wk)
        W = np.stack(W, 1)
        inside = ((W > 0).all(1) | (W < 0).all(1))
        near = cand & np.logical_or.reduce(near_k)
        m = cand
        for k, x in (('pix', r * S + c), ('face', f), ('inside', inside), ('near', near), ('w', W)):
            out[k].append(x[m])
        start = stop
    if not out['pix']:
        return {'pix': np.zeros(0, np.int64), 'face': np.zeros(0, np.int64), 'inside': np.zeros(0, bool), 'near': np.zeros(0, bool),
                'w': np.zeros((0, 3))}
    return {k: np.concatenate(x) for k, x in out.items()}


def _bary_depth(pr, u, v, d, faces, persp):
    """Screen barycentrics w/sum(w), perspective-corrected under the perspective camera, and the depth at the centre."""
    w = pr['w']
    b = w / w.sum(1, keepdims=True)
    D = d[np.asarray(faces, np.int64)[pr['face']]]
    if persp:
        q = b / D
        qs = q.sum(1, keepdims=True)
        return q / qs, 1.0 / qs[:, 0]
    return b, (b * D).sum(1)


def raster_image(verts, faces, cam, persp, S, tol_px=TOL_PX, tol_depth=TOL_DEPTH):
    """One image -> dict(pix_to_face [S,S] int64 (-1 background), zbuf [S,S] (-1), bary [S,S,3] (-1), ambiguous [S,S] bool)."""
    u, v, d = project(verts, cam, persp, S)
    pr = _pairs(u, v, d, faces, S, persp, tol_px)
    bary, depth = _bary_depth(pr, u, v, d, faces, persp)
    P = S * S
    ins = np.nonzero(pr['inside'])[0]
    order = ins[np.lexsort((pr['face'][ins], depth[ins], pr['pix'][ins]))]        # by pixel, then depth, then face index
    first = order[np.unique(pr['pix'][order], return_index=True)[1]]
    win_d = np.full(P, np.inf); win_f = np.full(P, -1, np.int64)
    win_d[pr['pix'][first]] = depth[first]; win_f[pr['pix'][first]] = pr['face'][first]
    dw = win_d[pr['pix']]
    with np.errstate(invalid='ignore'):
        tol = tol_depth * np.maximum(np.abs(depth), np.where(np.isfinite(dw), np.abs(dw), 0))
        flag = (pr['near'] & (depth <= dw + tol)) | (pr['inside'] & (pr['face'] != win_f[pr['pix']]) & (np.abs(depth - dw) <= tol))
    amb = np.zeros(P, bool); amb[pr['pix'][flag]] = True
    zbuf = np.full(P, -1.0); zbuf[pr['pix'][first]] = depth[first]
    B3 = np.full((P, 3), -1.0); B3[pr['pix'][first]] = bary[first]
    return {'pix_to_face': win_f.reshape(S, S), 'zbuf': zbuf.reshape(S, S), 'bary': B3.reshape(S, S, 3), 'ambiguous': amb.reshape(S, S)}


def coverage_2d(uv, faces, S, tol_px=TOL_PX):
    """Coverage of 2-D pixel-space points uv [V,2] (no camera, no depth) -> (covered [S,S] bool, ambiguous [S,S] bool)."""
    uv = np.asarray(uv, np.float64)
    pr = _pairs(uv[:, 0], uv[:, 1], np.ones(len(uv)), faces, S, False, tol_px)
    P = S * S
    cov = np.zeros(P, bool); cov[pr['pix'][pr['inside']]] = True
    robust = np.zeros(P, bool); robust[pr['pix'][pr['inside'] & ~pr['near']]] = True
    anynear = np.zeros(P, bool); anynear[pr['pix'][pr['near']]] = True
    return cov.reshape(S, S), (anynear & ~robust).reshape(S, S)


def coverage(verts, faces, cam, persp, S, tol_px=TOL_PX):
    """Coverage mask of one hand through a camera -> (covered, ambiguous) [S,S] bool."""
    u, v, d = project(verts, cam, persp, S)
    if persp:            # a face with a vertex at z <= 0 is not drawn: push it out of the image
        bad = ~(d > 0)
        u, v = u.copy(), v.copy(); u[bad] = np.nan; v[bad] = np.nan
    return coverage_2d(np.stack([u, v], 1), faces, S, tol_px)


# ----------------------------------------------------------------------------- shading
def vertex_normals(verts, faces):
    """pytorch3d Meshes.verts_normals: per vertex, the sum of cross(x[k+1] - x[k], x[k+2] - x[k]) over its face corners, normalised (eps 1e-6)."""
    X = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64)
    n = np.zeros_like(X)
    for k in range(3):
        p0, p1, p2 = X[faces[:, k]], X[faces[:, (k + 1) % 3]], X[faces[:, (k + 2) % 3]]
        np.add.at(n, faces[:, k], np.cross(p1 - p0, p2 - p0))
    return _normalize(n)


def _normalize(x):
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), 1e-6)


def shade(frag, verts, faces, colors, persp, phong):
    """HardPhongShader (phong=True: PointLights at (0,0,-1), ambient 0.5 / diffuse 0.3 / specular 0.2, shininess 64) or AmbientLights
    (ambient 1) + hard blend on white + / 255 -> (img [S,S,3], alpha [S,S])."""
    X = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64)
    col = np.broadcast_to(np.asarray(colors, np.float64), (len(X), 3))
    p2f = frag['pix_to_face'].reshape(-1)
    cov = p2f >= 0
    idx = faces[p2f[cov]]                                # [n,3]
    b = frag['bary'].reshape(-1, 3)[cov][:, :, None]     # [n,3,1]
    tex = (b * col[idx]).sum(1)
    if phong:
        N = vertex_normals(X, faces)
        p = (b * X[idx]).sum(1)
        n = _normalize((b * N[idx]).sum(1))
        l = _normalize(LIGHT - p)
        cam_c = np.array([0.0, 0.0, 0.0 if persp else -10.0])
        view = _normalize(cam_c - p)
        cosl = (n * l).sum(1)
        refl = -l + 2 * cosl[:, None] * n
        alpha_s = np.maximum((view * refl).sum(1), 0) * (cosl > 0)
        rgb = (AMBIENT + DIFFUSE * np.maximum(cosl, 0))[:, None] * tex + (SPECULAR * alpha_s ** SHININESS)[:, None]
    else:
        rgb = tex
    S = frag['pix_to_face'].shape[0]
    img = np.ones((S * S, 3)); img[cov] = rgb
    alpha = cov.astype(np.float64)
    return (img / 255.0).reshape(S, S, 3), alpha.reshape(S, S)


def render(verts, faces, cams, persp, S, colors, phong):
    """Batch: verts [B,V,3], cams [B,4] -> dict of [B,...] arrays: img, alpha, pix_to_face, zbuf, bary, ambiguous."""
    out = {k: [] for k in ('img', 'alpha', 'pix_to_face', 'zbuf', 'bary', 'ambiguous')}
    for i in range(len(verts)):
        fr = raster_image(verts[i], faces, cams[i], persp, S)
        img, alpha = shade(fr, verts[i], faces, colors, persp, phong)
        for k in ('pix_to_face', 'zbuf', 'bary', 'ambiguous'):
            out[k].append(fr[k])
        out['img'].append(img); out['alpha'].append(alpha)
    return {k: np.stack(x) for k, x in out.items()}


# ----------------------------------------------------------------------------- the two-hand mesh and the mask IoU
def two_hand_faces(right_faces):
    """vis_utils.py:166-170: cat(right_faces[:, [1,0,2]], right_faces + 778)."""
    rf = np.asarray(right_faces, np.int64)
    return np.concatenate([rf[:, [1, 0, 2]], rf + HAND_V])


def bm0(mask1, mask2):
    """utils/compute_maskiou.py:59-64 with NaN for an empty union (numpy's 0/0)."""
    a, b = np.count_nonzero(mask1 == 1), np.count_nonzero(mask2 == 1)
    inter = np.count_nonzero(np.logical_and(mask1, mask2))
    with np.errstate(invalid='ignore'):
        return np.float64(inter) / np.float64(a + b - inter)


def mask_iou(v_left, v_right, faces, cams, persp, S):
    """-> (iou [B], ambiguous pixel count [B] (either mask), union [B])."""
    iou, amb, uni = [], [], []
    for i in range(len(v_left)):
        cl, al = coverage(v_left[i], faces, cams[i], persp, S)
        cr, ar = coverage(v_right[i], faces, cams[i], persp, S)
        iou.append(bm0(cl.astype(np.float64), cr.astype(np.float64)))
        amb.append(int((al | ar).sum())); uni.append(int((cl | cr).sum()))
    return np.array(iou), np.array(amb), np.array(uni)
