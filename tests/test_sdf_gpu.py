"""The CUDA anti-penetration SDF loss (renderih_b200/sdf.py, csrc/sdf.cu) against the float64 oracle (oracle/sdf_ref.py) and a float64
torch composition of the reference's NewLoss, on synthetic meshes only.

Meshes: an axis-aligned box, an icosphere, and posed hands -- ManoLayer on the synthetic MANO tensors, triangulated with the convex hull of
a perturbed ellipsoid's 778 points (a closed genus-0 mesh with 2V - 4 = 1552 faces: the closed MANO hand's size).  Grid voxels are
compared where the oracle does not flag their parity as rounding-dependent; the flag tolerance is 1e-6, the fp32 rounding of the kernel.
"""
import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

from oracle import sdf_ref as S
from oracle.sdf_ref import box, icosphere
from renderih_b200 import assets as A
from renderih_b200.manolayer import ManoLayer, rodrigues_batch
from renderih_b200.sdf import SDF, NewLoss, penetration, sdf

pytestmark = pytest.mark.gpu
PHI_TOL, REL = 2e-5, 1e-6


def _hull_faces(seed=0):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(778, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    p *= np.array([1.0, 0.6, 0.35])                     # random points on an ellipsoid: all on its hull
    f = ConvexHull(p).simplices.astype(np.int64)
    assert f.shape == (1552, 3)
    return f


def _parts(seed=0):
    rng = np.random.default_rng(seed + 1)
    owner = rng.integers(0, 16, 778)
    parts = [set(np.nonzero(owner == k)[0].tolist()) for k in range(16)]
    for k in range(16):                                   # overlapping parts, as in part_vert.npy (934 entries over 778 vertices)
        parts[k] |= set(rng.choice(778, 10, replace=False).tolist())
    return parts


@pytest.fixture(scope='module')
def env():
    faces = _hull_faces()
    parts = _parts()
    layers = {s: ManoLayer(A.synthetic_mano(0, s), center_idx=9, use_pca=True) for s in ('left', 'right')}
    return faces, parts, layers


def _hands(env, B, seed, gap=0.0):
    """[B,2,778,3] posed hands (hand 0 right, 1 left); gap shifts them apart along x."""
    _, _, layers = env
    g = torch.Generator().manual_seed(seed)
    out = []
    for side, dx in (('right', gap), ('left', -gap)):
        rot = rodrigues_batch((torch.rand(B, 3, generator=g) - 0.5) * 2.0).cuda()
        pose, shape = torch.randn(B, 45, generator=g) * 0.6, torch.randn(B, 10, generator=g) * 0.5
        v, _ = layers[side](rot, pose.cuda(), shape.cuda())
        out.append(v + torch.tensor([dx, 0.0, 0.0], device='cuda'))
    return torch.stack(out, 1).contiguous()


def _normalise(v):
    lo, hi = v.min(dim=1)[0], v.max(dim=1)[0]
    c = ((lo + hi) / 2)[:, None]
    s = (1.1 * 0.5 * (hi - lo).max(dim=-1)[0])[:, None, None]
    return (v - c) / s


def _check_grid(phi, meshes, faces, G):
    """meshes [B,V,3] (numpy, normalised) -> flagged fraction; asserts agreement on unflagged voxels."""
    flagged = 0
    for b in range(len(meshes)):
        ref, amb = S.grid(faces, meshes[b], G, rel=REL)
        got = phi[b].cpu().numpy().astype(np.float64)
        ok = ~amb
        assert np.array_equal(got[ok] > 0, ref[ok] > 0), ((got[ok] > 0) != (ref[ok] > 0)).sum()
        err = np.abs(got[ok] - ref[ok]).max()
        assert err <= PHI_TOL, err
        assert (ref > 0).sum() > 0
        flagged += amb.sum()
    return flagged / (len(meshes) * G ** 3)


@pytest.mark.parametrize('G', [8, 17, 32])
@pytest.mark.parametrize('mesh', ['box', 'icosphere', 'hands'])
def test_dense_grid_matches_oracle(env, mesh, G):
    B = 3
    if mesh == 'box':
        rng = np.random.default_rng(G)
        ms = []
        for _ in range(B):
            lo = rng.uniform(-0.8, -0.2, 3)
            v, f = box(lo, lo + rng.uniform(0.5, 1.0, 3))
            ms.append(v)
        verts = np.stack(ms)
    elif mesh == 'icosphere':
        v, f = icosphere(0.75)
        rng = np.random.default_rng(G + 1)
        verts = np.stack([v * (0.8 + 0.2 * rng.random()) + rng.uniform(-0.1, 0.1, 3) for _ in range(B)])
    else:
        f = env[0]
        verts = _normalise(_hands(env, B, seed=G)[:, 0]).cpu().numpy()
    vt = torch.from_numpy(verts.astype(np.float32)).cuda()
    phi = sdf(f, vt, G)
    assert torch.equal(phi, SDF()(torch.from_numpy(f).int().cuda(), vt, G))
    frac = _check_grid(phi, vt.double().cpu().numpy(), f, G)
    print('%s G=%d: flagged fraction %.2e' % (mesh, G, frac))
    assert frac < 0.01


def _composition(v, faces, parts, G=32, sf=0.1):
    """The reference's NewLoss in float64 torch over the kernel's own dense grids: -> loss, L [B,2,V], O [B,2,V] (hand order of v).
    The normalised coordinates are taken in fp32 as the kernel takes them; their gradient is 1 / s (the frame is a constant)."""
    B, _, V, _ = v.shape
    v64 = v.detach().double().requires_grad_(True)
    vd = v.detach()
    lo, hi = vd.min(dim=2)[0], vd.max(dim=2)[0]
    c = ((lo + hi) / 2)[:, :, None]                              # [B,2,1,3]
    s = ((1 + sf) * 0.5 * (hi - lo).max(dim=-1)[0])[:, :, None, None]
    own = (vd - c) / s
    grids = [sdf(faces, own[:, h].contiguous(), G) for h in (0, 1)]
    L, O = [None, None], [None, None]
    for h in (0, 1):
        q = 1 - h
        x32 = (vd[:, q] - c[:, h]) / s[:, h]
        x = x32.double() + (v64[:, q] - v64[:, q].detach()) / s[:, h].double()
        acc = torch.zeros(B, V, dtype=torch.float64, device=v.device)
        accO = torch.zeros(B, V, dtype=torch.float64, device=v.device)
        for p in parts:
            idx = torch.tensor(sorted(p), device=v.device)
            val = torch.nn.functional.grid_sample(grids[h].double()[:, None], x[:, idx].view(B, -1, 1, 1, 3), align_corners=True).view(B, -1)
            acc = acc.index_add(1, idx, val)
            accO = accO.index_add(1, idx, val * s[:, h, 0].double())
        L[q], O[q] = acc / 4, accO
    L, O = torch.stack(L, 1), torch.stack(O, 1)
    return L.sum((1, 2)), L, O, v64


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_newloss_matches_composition_all_return_modes(env):
    faces, parts, _ = env
    B = 6
    v = _hands(env, B, seed=3)
    crit = NewLoss(faces=faces, part_vert=parts)
    loss_r, L_r, O_r, v64 = _composition(v, faces, parts)
    assert float(loss_r.min()) > 0
    vv = v.clone().requires_grad_(True)
    loss = crit(vv)
    assert _rel(loss, loss_r) <= 1e-5
    (g,) = torch.autograd.grad(loss.sum(), vv)
    (gr,) = torch.autograd.grad(loss_r.sum(), v64, retain_graph=True)
    assert _rel(g, gr) <= 1e-5, _rel(g, gr)
    loss, Ll, Lr = crit(vv, return_per_vert_loss=True)
    assert _rel(Ll, L_r[:, 1]) <= 1e-5 and _rel(Lr, L_r[:, 0]) <= 1e-5
    w = torch.randn(B, 778, device='cuda', dtype=torch.float64)
    (g,) = torch.autograd.grad((Ll * w).sum() + 0.5 * loss.sum(), vv)
    (gr,) = torch.autograd.grad((L_r[:, 1] * w).sum() + 0.5 * loss_r.sum(), v64, retain_graph=True)
    assert _rel(g, gr) <= 1e-5
    loss, Lcat, (Ol, Or) = crit(vv, return_per_vert_loss=True, return_origin_scale_loss=True)
    assert _rel(Lcat, torch.cat([L_r[:, 1], L_r[:, 0]], 1)) <= 1e-5
    assert _rel(Ol, O_r[:, 1]) <= 1e-5 and _rel(Or, O_r[:, 0]) <= 1e-5
    w2 = torch.randn(B, 1556, device='cuda', dtype=torch.float64)
    (g,) = torch.autograd.grad((Lcat * w2).sum() + (Ol * w[:, :778]).sum() - Or.sum(), vv)
    (gr,) = torch.autograd.grad((torch.cat([L_r[:, 1], L_r[:, 0]], 1) * w2).sum() + (O_r[:, 1] * w[:, :778]).sum() - O_r[:, 0].sum(), v64)
    assert _rel(g, gr) <= 1e-5


def test_finite_difference_of_per_vertex_loss(env):
    faces, parts, _ = env
    v = _hands(env, 2, seed=5)
    mult = torch.from_numpy(S.part_counts(parts, 778).astype(np.int32)).cuda()
    ft = torch.from_numpy(faces.astype(np.int32)).cuda()
    _, L, _, dLdv, center, scale = penetration(v, ft, mult)
    G = 32
    checked = 0
    for b in range(2):
        for q in (0, 1):
            h = 1 - q
            x = (v[b, q] - center[b, h]) / scale[b, h]
            ix = (x + 1) / 2 * (G - 1)
            frac = ix - ix.floor()
            lo, hi = v[b, q].min(0)[0], v[b, q].max(0)[0]
            inner = ((v[b, q] > lo) & (v[b, q] < hi)).all(1)
            cand = torch.nonzero(((frac > 0.3) & (frac < 0.7)).all(1) & inner & (L[b, q] > 0) & (ix > 0).all(1) & (ix < G - 1).all(1))[:, 0]
            for vi in cand[:4].tolist():
                for a in range(3):
                    hstep = 0.2 * float(scale[b, h]) * 2 / (G - 1)       # 0.2 of a cell: stays in the cell from frac in (0.3, 0.7)
                    Ls = []
                    for sgn in (1, -1):
                        vp = v.clone()
                        vp[b, q, vi, a] += sgn * hstep
                        Ls.append(float(penetration(vp, ft, mult)[1][b, q, vi]))
                    fd = (Ls[0] - Ls[1]) / (2 * hstep)
                    an = float(dLdv[b, q, vi, a])
                    assert abs(fd - an) <= 1e-4 * max(abs(an), float(dLdv.abs().max()) * 1e-2), (fd, an)
                    checked += 1
    assert checked >= 12


def test_sanity_separated_penetrating_and_descent(env):
    faces, parts, _ = env
    crit = NewLoss(faces=faces, part_vert=parts)
    far = _hands(env, 4, seed=7, gap=1.0).requires_grad_(True)
    loss = crit(far)
    (g,) = torch.autograd.grad(loss.sum(), far)
    assert (loss == 0).all() and (g == 0).all()
    v = _hands(env, 4, seed=7).requires_grad_(True)
    loss = crit(v)
    assert (loss > 0).all()
    (g,) = torch.autograd.grad(loss.sum(), v)
    step = 1e-3 / float(g.abs().max())
    with torch.no_grad():
        after = crit(v - step * g)
    assert float(after.sum()) < float(loss.sum())


def test_deterministic_and_cuda_graph(env):
    faces, parts, _ = env
    v = _hands(env, 16, seed=9)
    mult = torch.from_numpy(S.part_counts(parts, 778).astype(np.int32)).cuda()
    ft = torch.from_numpy(faces.astype(np.int32)).cuda()
    a, b = penetration(v, ft, mult), penetration(v, ft, mult)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    vn = _normalise(v[:, 0]).contiguous()
    grid_e = sdf(faces, vn, 32)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        penetration(v, ft, mult)
        sdf(ft, vn, 32)                                      # validates ft once; the captured call then needs no host copy
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = penetration(v, ft, mult) + (sdf(ft, vn, 32),)
    for o in out:
        o.zero_()
    g.replay()
    torch.cuda.synchronize()
    for o, e in zip(out, a + (grid_e,)):
        assert torch.equal(o, e)


def test_fused_equals_sampling_the_dense_grid(env):
    """The fused kernel computes only the touched corners; sampled the same way, the dense grid gives the same per-vertex loss."""
    faces, parts, _ = env
    v = _hands(env, 4, seed=11)
    mult = torch.from_numpy(S.part_counts(parts, 778).astype(np.int32)).cuda()
    _, L, _, _, center, scale = penetration(v, torch.from_numpy(faces.astype(np.int32)).cuda(), mult)
    for h in (0, 1):
        own = (v[:, h] - center[:, h, None]) / scale[:, h, None, None]
        grid = sdf(faces, own.contiguous(), 32)
        x = (v[:, 1 - h] - center[:, h, None]) / scale[:, h, None, None]
        p = torch.nn.functional.grid_sample(grid[:, None], x.view(4, -1, 1, 1, 3), align_corners=True).view(4, -1)
        assert _rel(L[:, 1 - h], mult * p / 4) <= 1e-6


def test_batch_6144(env):
    faces, parts, _ = env
    B = 6144
    v = _hands(env, B, seed=13)
    crit = NewLoss(faces=faces, part_vert=parts)
    vv = v.clone().requires_grad_(True)
    loss = crit(vv)
    (g,) = torch.autograd.grad(loss.sum(), vv)
    assert torch.isfinite(loss).all() and (loss > 0).float().mean() > 0.5
    idx = torch.tensor([0, 1, 777, 3000, 4097, 6143], device='cuda')
    loss_r, _, _, v64 = _composition(v[idx], faces, parts)
    (gr,) = torch.autograd.grad(loss_r.sum(), v64)
    assert _rel(loss[idx], loss_r) <= 1e-5
    assert _rel(g[idx], gr) <= 1e-5


def test_matches_oracle_newloss(env):
    faces, parts, _ = env
    v = _hands(env, 2, seed=17)
    crit = NewLoss(faces=faces, part_vert=parts)
    loss, Lcat, (Ol, Or) = crit(v, return_per_vert_loss=True, return_origin_scale_loss=True)
    mult = S.part_counts(parts, 778)
    for b in range(2):
        ref = S.newloss(v[b].cpu().numpy(), faces, mult, rel=REL)
        ok = ~ref['ambiguous']
        assert ok.mean() > 0.95
        L = torch.stack([Lcat[b, 778:], Lcat[b, :778]]).cpu().numpy()
        assert np.abs(L - ref['L'])[ok].max() <= 1e-5 * np.abs(ref['L']).max()
        assert abs(float(loss[b]) - ref['loss']) <= 1e-5 * ref['loss'] or not ok.all()


def test_rejected_inputs(env):
    faces, parts, _ = env
    crit = NewLoss(faces=faces, part_vert=parts)
    v = _hands(env, 1, seed=1)
    with pytest.raises(RuntimeError):
        crit(v.cpu())
    with pytest.raises(RuntimeError):
        sdf(faces, v[:, 0].cpu(), 32)
    with pytest.raises(RuntimeError):
        NewLoss(faces=faces, part_vert=parts, device='cpu')
    with pytest.raises(ValueError):
        crit(v[:, 0])                                        # [B,V,3]: not two hands
    with pytest.raises(ValueError):
        crit(torch.zeros(1, 3, 778, 3, device='cuda'))
    with pytest.raises(ValueError):
        sdf(faces, v[0, 0], 32)
    bad = faces.copy(); bad[5, 1] = 778
    with pytest.raises(ValueError):
        NewLoss(faces=bad, part_vert=parts)(v)
    bad[5, 1] = -1
    with pytest.raises(ValueError):
        NewLoss(faces=bad, part_vert=parts)
    with pytest.raises(ValueError):
        sdf(bad, v[:, 0], 32)
    with pytest.raises(ValueError):
        NewLoss(faces=faces, part_vert=parts[:-1] + [{3, 800}])(v)
    with pytest.raises(ValueError):
        NewLoss(faces=faces, part_vert=parts[:-1] + [{-2, 3}])
    with pytest.raises(ValueError):
        NewLoss(faces=faces[:, :2], part_vert=parts)
    for G in (1, 65):
        with pytest.raises(ValueError):
            NewLoss(grid_size=G, faces=faces, part_vert=parts)
        with pytest.raises(ValueError):
            sdf(faces, v[:, 0], G)
    for G in (2, 64):
        assert torch.isfinite(NewLoss(grid_size=G, faces=faces, part_vert=parts)(v)).all()
