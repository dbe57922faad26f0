"""numpy float64 restatement of renderih_b200/csrc/collision.cu (the two-hand collision count) and of ValidJudger.ValidationJudge.

Collision: per frame, the number of (face of hand A, face of hand B) pairs whose closed triangles intersect, decided by Guigue and
Devillers' orientation predicates with their coplanar 2-D branch.  Every determinant is spelled out as the kernel evaluates it --
differences, then products, then sums, left to right, each one IEEE float64 operation (numpy elementwise ops and Python floats never
fuse a multiply-add) -- so the kernel's counts and these agree exactly.  The exactly coplanar pairs (rare outside coincident meshes)
run through a scalar restatement of the 2-D branch on Python floats.

Each pair is also classified as fragile when some determinant that decided it lies within its floating-point error bound of zero, so
that the exact sign could differ: 16 eps times the determinant's permanent for a 3x3 determinant of differences, 8 eps for the 2-D
ones (eps = 2**-53).  A fragile pair may get a different answer in exact arithmetic; any other pair gets the exact answer.
"""
import numpy as np

EPS = 2.0 ** -53
EB3, EB2 = 16 * EPS, 8 * EPS


# ------------------------------------------------------------------------------------------------------------------------ decisions
def order(sp, sq, sr):
    """The permutation rule of both levels of the 3-D test -> (rotation putting the lone vertex first: 0 pqr, 1 qrp, 2 rpq, whether the
    other triangle's last two vertices swap), or None when all three signs are zero."""
    if sp > 0:
        if sq > 0:
            return 2, True
        if sr > 0:
            return 1, True
        return 0, False
    if sp < 0:
        if sq < 0:
            return 2, False
        if sr < 0:
            return 1, False
        return 0, True
    if sq < 0:
        return (1, True) if sr >= 0 else (0, False)
    if sq > 0:
        return (0, True) if sr > 0 else (1, False)
    if sr > 0:
        return 2, False
    if sr < 0:
        return 2, True
    return None


# sign triple (each -1, 0, 1; index 9 (sp+1) + 3 (sq+1) + (sr+1)) -> rotation, swap, coplanar
_LUT = np.zeros((27, 3), np.int64)
for _i in range(27):
    _o = order(_i // 9 - 1, _i // 3 % 3 - 1, _i % 3 - 1)
    _LUT[_i] = (0, 0, 1) if _o is None else (_o[0], int(_o[1]), 0)


# ------------------------------------------------------------------------------------------------------------------------ 3-D, vectorised
def _sub(a, b):
    return a - b


def _cross(a, b):
    """[..., 3] x [..., 3], each component one difference of two rounded products."""
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _perm_cross(a, b):
    """The absolute values of the products behind each cross component, summed: the permanent's inner factor."""
    a, b = np.abs(a), np.abs(b)
    return np.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)


def _det(a, b, c):
    """dot(a, b x c) -> (value, fragile)."""
    d = _dot(a, _cross(b, c))
    return d, np.abs(d) <= EB3 * _dot(np.abs(a), _perm_cross(b, c))


def _rot(t, r):
    """t [P,3,3] triangles, r [P] rotations -> vertices (k + r) % 3."""
    idx = (np.arange(3)[None, :] + r[:, None]) % 3
    return np.take_along_axis(t, idx[:, :, None], 1)


def tri_tri(t1, t2):
    """Closed triangles t1, t2 [P,3,3] float64 (vertices p, q, r) -> (intersect [P] bool, fragile [P] bool)."""
    t1 = np.asarray(t1, np.float64)
    t2 = np.asarray(t2, np.float64)
    P = t1.shape[0]
    hit = np.zeros(P, bool)
    frag = np.zeros(P, bool)
    e1, f1 = _sub(t1[:, 0], t1[:, 2]), _sub(t1[:, 1], t1[:, 2])
    e2, f2 = _sub(t2[:, 0], t2[:, 2]), _sub(t2[:, 1], t2[:, 2])
    n1, n2 = _cross(e1, f1), _cross(e2, f2)
    pc1, pc2 = _perm_cross(e1, f1), _perm_cross(e2, f2)
    # zero area: the computed normal is exactly (0, 0, 0); fragile when every component is within its bound
    frag |= (np.abs(n1) <= 2 * EB2 * pc1).all(-1) | (np.abs(n2) <= 2 * EB2 * pc2).all(-1)
    live = ~((n1 == 0).all(-1) | (n2 == 0).all(-1))
    d1 = np.stack([_dot(_sub(t1[:, k], t2[:, 2]), n2) for k in range(3)], -1)
    d1f = np.stack([np.abs(d1[:, k]) <= EB3 * _dot(np.abs(_sub(t1[:, k], t2[:, 2])), pc2) for k in range(3)], -1)
    s1 = np.sign(d1).astype(np.int64)
    frag |= live & d1f.any(-1)
    live &= ~((s1[:, 0] == s1[:, 1]) & (s1[:, 0] == s1[:, 2]) & (s1[:, 0] != 0))
    d2 = np.stack([_dot(_sub(t2[:, k], t1[:, 2]), n1) for k in range(3)], -1)
    d2f = np.stack([np.abs(d2[:, k]) <= EB3 * _dot(np.abs(_sub(t2[:, k], t1[:, 2])), pc1) for k in range(3)], -1)
    s2 = np.sign(d2).astype(np.int64)
    frag |= live & d2f.any(-1)
    live &= ~((s2[:, 0] == s2[:, 1]) & (s2[:, 0] == s2[:, 2]) & (s2[:, 0] != 0))
    L = _LUT[9 * (s1[:, 0] + 1) + 3 * (s1[:, 1] + 1) + (s1[:, 2] + 1)]
    a = _rot(t1, L[:, 0])
    i2 = np.tile(np.arange(3), (P, 1))
    i2[L[:, 1] == 1] = (0, 2, 1)
    s2p = np.take_along_axis(s2, i2, 1)
    M = _LUT[9 * (s2p[:, 0] + 1) + 3 * (s2p[:, 1] + 1) + (s2p[:, 2] + 1)]
    cop = live & ((L[:, 2] == 1) | (M[:, 2] == 1))
    gen = live & ~cop
    i2 = np.take_along_axis(i2, (np.arange(3)[None, :] + M[:, 0:1]) % 3, 1)
    b = np.take_along_axis(t2, i2[:, :, None], 1)
    a[M[:, 1] == 1] = a[M[:, 1] == 1][:, [0, 2, 1]]
    # CHECK_MIN_MAX(p1, q1, r1, p2, q2, r2)
    da, fa = _det(_sub(b[:, 1], a[:, 1]), _sub(b[:, 0], a[:, 1]), _sub(a[:, 0], a[:, 1]))
    db, fb = _det(_sub(b[:, 2], a[:, 0]), _sub(b[:, 0], a[:, 0]), _sub(a[:, 2], a[:, 0]))
    frag |= gen & (fa | ((da <= 0) & fb))
    hit |= gen & ~(da > 0) & ~(db > 0)
    for k in np.nonzero(cop)[0]:
        h, fr = coplanar(t1[k].tolist(), t2[k].tolist(), n1[k].tolist(), pc1[k].tolist())
        hit[k] = h
        frag[k] = True      # entered on exactly zero determinants, each within its bound unless the permanents vanish
        frag[k] |= fr
    return hit, frag


# ------------------------------------------------------------------------------------------------------------------------ 2-D, scalar
class _Orient:
    """orient2d on Python floats, recording whether any evaluated value lay within its bound."""

    def __init__(self):
        self.fragile = False

    def __call__(self, a, b, c):
        l = (a[0] - c[0]) * (b[1] - c[1])
        r = (a[1] - c[1]) * (b[0] - c[0])
        d = l - r
        if abs(d) <= EB2 * (abs(l) + abs(r)):
            self.fragile = True
        return d


def _test_vertex(o, P1, Q1, R1, P2, Q2, R2):
    if o(R2, P2, Q1) >= 0.0:
        if o(R2, Q2, Q1) <= 0.0:
            if o(P1, P2, Q1) > 0.0:
                return o(P1, Q2, Q1) <= 0.0
            return o(P1, P2, R1) >= 0.0 and o(Q1, R1, P2) >= 0.0
        return o(P1, Q2, Q1) <= 0.0 and o(R2, Q2, R1) <= 0.0 and o(Q1, R1, Q2) >= 0.0
    if o(R2, P2, R1) >= 0.0:
        if o(Q1, R1, R2) >= 0.0:
            return o(P1, P2, R1) >= 0.0
        return o(Q1, R1, Q2) >= 0.0 and o(R2, R1, Q2) >= 0.0
    return False


def _test_edge(o, P1, Q1, R1, P2, Q2, R2):
    if o(R2, P2, Q1) >= 0.0:
        if o(P1, P2, Q1) >= 0.0:
            return o(P1, Q1, R2) >= 0.0
        return o(Q1, R1, P2) >= 0.0 and o(R1, P1, P2) >= 0.0
    if o(R2, P2, R1) >= 0.0:
        if o(P1, P2, R1) < 0.0:
            return False
        return o(P1, R1, R2) >= 0.0 or o(Q1, R1, R2) >= 0.0
    return False


def _ccw_2d(o, p1, q1, r1, p2, q2, r2):
    if o(p2, q2, p1) >= 0.0:
        if o(q2, r2, p1) >= 0.0:
            if o(r2, p2, p1) >= 0.0:
                return True
            return _test_edge(o, p1, q1, r1, p2, q2, r2)
        if o(r2, p2, p1) >= 0.0:
            return _test_edge(o, p1, q1, r1, r2, p2, q2)
        return _test_vertex(o, p1, q1, r1, p2, q2, r2)
    if o(q2, r2, p1) >= 0.0:
        if o(r2, p2, p1) >= 0.0:
            return _test_edge(o, p1, q1, r1, q2, r2, p2)
        return _test_vertex(o, p1, q1, r1, q2, r2, p2)
    return _test_vertex(o, p1, q1, r1, r2, p2, q2)


def coplanar(t1, t2, n, pc):
    """coplanar_tri_tri3d on Python floats: t1, t2 [3][3], n the first triangle's computed normal, pc its permanents -> (hit, fragile)."""
    nx, ny, nz = abs(n[0]), abs(n[1]), abs(n[2])
    pts = list(t1) + list(t2)
    if nx > nz and nx >= ny:
        ax, pq, k = (2, 1), True, 0
    elif ny > nz and ny >= nx:
        ax, pq, k = (0, 2), True, 1
    else:
        ax, pq, k = (0, 1), False, 2
    src = [1, 0, 2, 4, 3, 5] if pq else list(range(6))
    p1, q1, r1, p2, q2, r2 = [(pts[s][ax[0]], pts[s][ax[1]]) for s in src]
    o = _Orient()
    o.fragile = abs(n[k]) <= 2 * EB2 * pc[k]          # the dropped component could be zero in exact arithmetic
    if o(p1, q1, r1) < 0.0:
        q1, r1 = r1, q1
    if o(p2, q2, r2) < 0.0:
        q2, r2 = r2, q2
    return _ccw_2d(o, p1, q1, r1, p2, q2, r2), o.fragile


# ------------------------------------------------------------------------------------------------------------------------ per frame
def _boxes(X, faces):
    t = X[faces]                                   # [F,3,3]
    return t, t.min(1), t.max(1)


def frame_count(xa, xb, faces):
    """One frame: xa, xb [V,3] float64 coordinates, faces [F,3] -> (count, fragile pairs).  The float64 box culling is exact and closed,
    so it never drops an intersecting pair."""
    faces = np.asarray(faces, np.int64)
    ta, la, ha = _boxes(np.asarray(xa, np.float64), faces)
    tb, lb, hb = _boxes(np.asarray(xb, np.float64), faces)
    ia = np.nonzero(((la <= hb.max(0)) & (lb.min(0) <= ha)).all(1))[0]
    ib = np.nonzero(((lb <= ha.max(0)) & (la.min(0) <= hb)).all(1))[0]
    count = fragile = 0
    for s in range(0, len(ia), 256):
        i = ia[s:s + 256]
        ov = ((la[i, None] <= hb[None, ib]) & (lb[None, ib] <= ha[i, None])).all(-1)
        pi, pj = np.nonzero(ov)
        if len(pi):
            h, f = tri_tri(ta[i[pi]], tb[ib[pj]])
            count += int(h.sum())
            fragile += int(f.sum())
    return count, fragile


def counts(xa, xb, faces):
    """xa, xb [B,V,3] float64 -> (count [B], fragile [B]) int64."""
    out = np.array([frame_count(a, b, faces) for a, b in zip(xa, xb)], np.int64).reshape(-1, 2)
    return out[:, 0], out[:, 1]


# ------------------------------------------------------------------------------------------------------------------------ test meshes
def ellipsoid_mesh(rings=24, segments=32, axes=(0.045, 0.02, 0.012)):
    """A closed UV ellipsoid of hand size: rings * segments + 2 vertices, 2 * rings * segments faces (770 / 1536 by default) ->
    (vertices [V,3] float64, faces [F,3] int32)."""
    th = np.pi * (np.arange(rings) + 1) / (rings + 1)
    ph = 2 * np.pi * np.arange(segments) / segments
    T, Pp = np.meshgrid(th, ph, indexing='ij')
    v = np.stack([np.cos(T), np.sin(T) * np.cos(Pp), np.sin(T) * np.sin(Pp)], -1).reshape(-1, 3)
    v = np.concatenate([[[1.0, 0, 0]], v, [[-1.0, 0, 0]]]) * np.asarray(axes)
    f = []
    ring = lambda r, s: 1 + r * segments + s % segments
    for s in range(segments):
        f.append((0, ring(0, s), ring(0, s + 1)))
        f.append((len(v) - 1, ring(rings - 1, s + 1), ring(rings - 1, s)))
    for r in range(rings - 1):
        for s in range(segments):
            f.append((ring(r, s), ring(r + 1, s), ring(r + 1, s + 1)))
            f.append((ring(r, s), ring(r + 1, s + 1), ring(r, s + 1)))
    return v, np.asarray(f, np.int32)


def two_hand_frames(B, regime, seed, f64=False):
    """B frames of two ellipsoid 'hands' with a smooth random deformation each: regime 'apart' (no box overlap), 'touching' (surfaces
    meeting over a few faces), 'deep' (heavily interpenetrating) or 'coincident' (hand B is hand A).  -> (va, vb [B,V,3] float32 or
    float64 centred vertices, ta, tb [B,3] float64 translations, faces [F,3] int32)."""
    v0, faces = ellipsoid_mesh()
    rng = np.random.default_rng(seed)

    def hand():
        A = np.eye(3) + rng.normal(size=(B, 3, 3)) * 0.08
        w = rng.normal(size=(B, 1, 3)) * 0.004
        v = np.einsum('bij,vj->bvi', A, v0) + w * np.sin(40 * v0[None, :, :1])
        return v
    va, vb = hand(), hand()
    ta = rng.normal(size=(B, 3)) * 0.01
    gap = {'apart': 0.2, 'touching': 0.038, 'deep': 0.01, 'coincident': 0.0}[regime]
    d = rng.normal(size=(B, 3)) * np.asarray([1, 0.2, 0.2])
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    tb = ta + d * gap * (1 + 0.05 * rng.normal(size=(B, 1)))
    if regime == 'coincident':
        vb, tb = va.copy(), ta.copy()
    dt = np.float64 if f64 else np.float32
    return va.astype(dt), vb.astype(dt), ta, tb, faces


# ------------------------------------------------------------------------------------------------------------------------ validity
BEND = ((-25, 70), (-4, 110), (-8, 90), (-25, 80), (-7, 100), (-8, 90), (-22, 70), (-8, 90), (-8, 90), (-25, 70), (-10, 100), (-8, 90),
        (-20, 40), (-35, 50), (-10, 100))
SPLANK = {0: (-25, 15), 3: (-15, 15), 9: (-25, 15), 6: (-20, 30), 12: (-30, 30)}


def quat_to_R(q):
    """quatutils.quaternion_to_rotation_matrix on [..., 4] (w, x, y, z), no normalisation first."""
    w, x, y, z = (q[..., i] for i in range(4))
    n = w * w + x * x + y * y + z * z
    R = np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (w * y + x * z), 2 * (w * z + x * y), w * w - x * x + y * y - z * z,
                  2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (w * x + y * z), w * w - x * x - y * y + z * z], -1) / n[..., None]
    return R.reshape(q.shape[:-1] + (3, 3))


def valid_scores(quat, side, inv_m0, inv_u1):
    """ValidationJudge (ValidJudger.py:41-111) in float64 on quat [B,16,4] MANO quaternions of one side, with the converter matrices
    of that side -> scores [B] in radians."""
    q = np.asarray(quat, np.float64).copy()
    if side == 'left':
        q[..., 2:] = -q[..., 2:]
    R = quat_to_R(q)[:, 1:]
    A = np.asarray(inv_m0, np.float64)[1:].transpose(0, 2, 1)
    C = np.asarray(inv_u1, np.float64)[1:].transpose(0, 2, 1)
    zero = A @ C
    M = zero.transpose(0, 2, 1)[None] @ (A[None] @ R @ C[None])
    bend = np.degrees(np.arctan2(M[..., 1, 0], M[..., 0, 0]))
    spl = np.degrees(np.arctan2(-M[..., 2, 0], M[..., 0, 0]))
    ex = lambda a, lo, hi: np.maximum(np.maximum(a - hi, 0), np.maximum(lo - a, 0)) / 180 * np.pi
    s = np.zeros(len(q))
    for t, (lo, hi) in SPLANK.items():
        s = np.maximum(s, ex(spl[:, t], lo, hi))
    b = np.zeros(len(q))
    for t, (lo, hi) in enumerate(BEND):
        b = np.maximum(b, ex(bend[:, t], lo, hi))
    return np.maximum(s, b)


def invalid_rate(left_scores, right_scores):
    """ComputeValidation's rate: the fraction of frames where either hand's score exceeds 0.1 degree (in radians, as float32)."""
    th = np.float32(0.1 / 180 * np.pi)
    return float(((np.asarray(right_scores) > th) | (np.asarray(left_scores) > th)).mean())
