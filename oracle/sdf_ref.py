"""Float64 numpy oracle of the two-hand anti-penetration SDF loss (renderih_b200/sdf.py, csrc/sdf.cu): the dense grid of the reference's
lib/sdf extension and the NewLoss of pose_data_optimize/code_sdf/sdf_template.py, written from the conventions in renderih_b200/sdf.py.

TEST INFRASTRUCTURE -- never imported by the product package.

`voxel_phi` also flags voxels whose inside/outside answer depends on rounding: for a face the ray could hit (its barycentrics and t
within the tolerance of the accepted ranges), the ray passes within `rel` (relative, in barycentric units) of one of its edges or vertices,
|det| lies within `rel` (relative to |e1| |d| |e2|) of the 1e-6 threshold, or t is within `rel` of 0.  Such a voxel's phi is not compared.
"""
import numpy as np

EPS_DET = 1e-6


# ---- closed test meshes
BOX_FACES = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4],
                      [2, 3, 7], [2, 7, 6], [1, 2, 6], [1, 6, 5], [0, 4, 7], [0, 7, 3]])


def box(lo, hi):
    (x0, y0, z0), (x1, y1, z1) = lo, hi
    v = np.array([[x0, y0, z0], [x1, y0, z0], [x1, y1, z0], [x0, y1, z0], [x0, y0, z1], [x1, y0, z1], [x1, y1, z1], [x0, y1, z1]])
    return v, BOX_FACES.copy()


def icosphere(r=0.7, level=2):
    t = (1 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t], [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
         [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.array(v) * r, np.array(f)


def centers(G):
    """[G^3,3] voxel centres in the order of phi[k,j,i] flattened (i, the x index, fastest): -1 + (idx + 0.5) * 2 / (G - 1)."""
    d = 2.0 / (G - 1)
    c = -1.0 + (np.arange(G) + 0.5) * d
    k, j, i = np.meshgrid(c, c, c, indexing='ij')
    return np.stack([i.ravel(), j.ravel(), k.ravel()], 1)


def _seg_dist2(p, a, b):
    e = b - a
    w = p[:, None, :] - a[None]
    ee = (e * e).sum(-1)
    t = np.where(ee > 0, (w * e[None]).sum(-1) / np.where(ee > 0, ee, 1.0), 0.0)
    t = np.clip(t, 0.0, 1.0)
    r = w - t[..., None] * e[None]
    return (r * r).sum(-1)


def _tri_dist2(p, tri):
    """[P,F] squared distances from points p [P,3] to the closed triangles tri [F,3,3]."""
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(-1)
    ins = np.broadcast_to(nn[None] > 0, (len(p), len(nn))).copy()
    for u, w in ((a, b), (b, c), (c, a)):
        side = (np.cross((w - u)[None], p[:, None, :] - u[None]) * n[None]).sum(-1)
        ins &= side >= 0
    h = ((p[:, None, :] - a[None]) * n[None]).sum(-1)
    plane = h * h / np.where(nn > 0, nn, 1.0)[None]
    edges = np.minimum(_seg_dist2(p, a, b), np.minimum(_seg_dist2(p, b, c), _seg_dist2(p, c, a)))
    return np.where(ins, plane, edges)


def _ray(p, tri, rel):
    """-> (hits [P,F] bool, ambiguous [P] bool) of the rays from p towards (-1,-1,-1) against tri [F,3,3]."""
    d = -1.0 - p                                        # [P,3]
    v0 = tri[:, 0]
    e1, e2 = tri[:, 1] - v0, tri[:, 2] - v0             # [F,3]
    pv = np.cross(d[:, None, :], e2[None])              # [P,F,3]
    det = (e1[None] * pv).sum(-1)
    mag = np.linalg.norm(d, axis=-1)[:, None] * np.linalg.norm(e1, axis=-1)[None] * np.linalg.norm(e2, axis=-1)[None]
    with np.errstate(divide='ignore', invalid='ignore'):
        inv = 1.0 / det
        tv = p[:, None, :] - v0[None]
        u = (tv * pv).sum(-1) * inv
        qv = np.cross(tv, e1[None])
        v = (d[:, None, :] * qv).sum(-1) * inv
        t = (e2[None] * qv).sum(-1) * inv
    w = 1.0 - u - v
    ok_det = np.abs(det) >= EPS_DET
    hits = ok_det & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t >= 0)
    near = (u >= -rel) & (v >= -rel) & (w >= -rel) & (t >= -rel) & np.isfinite(t)        # a hit up to the tolerance
    amb = near & ((np.minimum(np.minimum(np.abs(u), np.abs(v)), np.abs(w)) <= rel) | (np.abs(t) <= rel))
    amb |= near & (np.abs(np.abs(det) - EPS_DET) <= rel * mag)
    return hits, amb.any(1)


def voxel_phi(faces, verts, pts, rel=1e-9, chunk=2048):
    """phi and the ambiguity flag at points pts [P,3] (voxel centres) of the closed mesh faces [F,3] over verts [V,3]: the distance to the
    nearest face when the ray towards (-1,-1,-1) hits an odd number of faces, else 0."""
    tri = np.asarray(verts, np.float64)[np.asarray(faces)]
    pts = np.asarray(pts, np.float64)
    phi, amb = np.zeros(len(pts)), np.zeros(len(pts), bool)
    for s in range(0, len(pts), chunk):
        p = pts[s:s + chunk]
        hits, a = _ray(p, tri, rel)
        inside = hits.sum(1) % 2 == 1
        amb[s:s + chunk] = a
        if inside.any():
            phi[s:s + chunk][inside] = np.sqrt(_tri_dist2(p[inside], tri).min(1))
    return phi, amb


def grid(faces, verts, G, rel=1e-9):
    """Dense grid [G,G,G] (phi[k,j,i]) and its ambiguity flags for one mesh."""
    phi, amb = voxel_phi(faces, verts, centers(G), rel)
    return phi.reshape(G, G, G), amb.reshape(G, G, G)


def trilinear(phi, x):
    """grid_sample(align_corners=True, padding_mode='zeros') of phi [D,H,W] at x [N,3] (x -> W, y -> H, z -> D), and d/dx [N,3]: the
    gradient of the cell floor(ix) picks, including the (G - 1) / 2 scaling."""
    phi = np.asarray(phi, np.float64)
    x = np.asarray(x, np.float64)
    size = np.array([phi.shape[2], phi.shape[1], phi.shape[0]])
    g = (x + 1.0) / 2.0 * (size - 1)
    g0 = np.floor(g)
    f = g - g0
    g0 = g0.astype(np.int64)
    p = np.zeros(len(x))
    dp = np.zeros((len(x), 3))
    for n in range(8):
        o = np.array([n & 1, (n >> 1) & 1, n >> 2])
        idx = g0 + o
        inb = np.all((idx >= 0) & (idx < size), 1)
        val = np.zeros(len(x))
        val[inb] = phi[idx[inb, 2], idx[inb, 1], idx[inb, 0]]
        w = np.where(o == 1, f, 1.0 - f)                 # [N,3]
        sgn = np.where(o == 1, 1.0, -1.0)
        p += val * w.prod(1)
        for a in range(3):
            b, c = [k for k in range(3) if k != a]
            dp[:, a] += val * sgn[a] * w[:, b] * w[:, c]
    return p, dp * (size - 1) / 2.0


def frame(verts, scale_factor=0.1):
    """Centre (min + max) / 2 and scale (1 + scale_factor) * 0.5 * longest side of one hand's bounding box, in fp32 as torch computes
    them in the reference (the frame is a constant of the loss, so the kernel and the oracle share it exactly)."""
    v = np.asarray(verts, np.float32)
    lo, hi = v.min(0), v.max(0)
    return (lo + hi) / np.float32(2), np.float32((1 + scale_factor) * 0.5) * (hi - lo).max()


def part_counts(part_vert, V):
    """m_v: the number of parts containing vertex v (each part counted once per vertex)."""
    m = np.zeros(V, np.int64)
    for p in part_vert:
        m[np.unique(np.asarray(list(p), np.int64))] += 1
    return m


def newloss(verts, faces, mult, G=32, scale_factor=0.1, rel=1e-9):
    """NewLoss of one sample: verts [2,V,3] (hand 0 right, 1 left), faces [F,3], mult [V].  Only the voxels the loss reads are evaluated.
    -> dict loss, L [2,V], O [2,V], dLdv [2,V,3] (dL/dv with the frames constant), ambiguous [2,V] (a corner's phi is ambiguous)."""
    verts = np.asarray(verts, np.float32)
    V = verts.shape[1]
    out = {'L': np.zeros((2, V)), 'O': np.zeros((2, V)), 'dLdv': np.zeros((2, V, 3)), 'ambiguous': np.zeros((2, V), bool)}
    mult = np.asarray(mult, np.float64)
    for h in (0, 1):
        q = 1 - h
        c, s = frame(verts[h], scale_factor)
        own = (verts[h] - c) / s                         # fp32, as the grid's vertices are normalised
        x = ((verts[q] - c) / s).astype(np.float64)
        gi = np.floor((x + 1.0) / 2.0 * (G - 1)).astype(np.int64)
        need = set()
        for n in range(8):
            idx = gi + np.array([n & 1, (n >> 1) & 1, n >> 2])
            ok = np.all((idx >= 0) & (idx < G), 1)
            need.update(((idx[ok, 2] * G + idx[ok, 1]) * G + idx[ok, 0]).tolist())
        need = np.array(sorted(need), np.int64)
        phi, amb = np.zeros(G ** 3), np.zeros(G ** 3, bool)
        if len(need):
            phi[need], amb[need] = voxel_phi(faces, own.astype(np.float64), centers(G)[need], rel)
        p, dp = trilinear(phi.reshape(G, G, G), x)
        out['L'][q] = mult * p / 4
        out['O'][q] = mult * p * np.float64(s)
        out['dLdv'][q] = (mult / 4)[:, None] * dp / np.float64(s)
        flag = np.zeros(V, bool)
        for n in range(8):
            idx = gi + np.array([n & 1, (n >> 1) & 1, n >> 2])
            ok = np.all((idx >= 0) & (idx < G), 1)
            flag[ok] |= amb[(idx[ok, 2] * G + idx[ok, 1]) * G + idx[ok, 0]]
        out['ambiguous'][q] = flag
    out['loss'] = out['L'].sum()
    return out
