"""The CUDA two-hand renderer (renderih_b200/render.py, csrc/render.cu) against the float64 oracle (oracle/render_ref.py), on synthetic
assets only.

Meshes: the main cases pose two hands with ManoLayer (synthetic MANO tensors, random poses) and triangulate them with the convex hull of
the template -- a closed surface of well-shaped triangles like the real MANO mesh; the synthetic MANO's own faces (random vertex
triples: long, overlapping slivers) are a stress case.  A pixel is compared where the oracle does not flag it as ambiguous (its
centre within 1e-6 px of a deciding edge, or two candidate depths within fp32 rounding; see oracle/render_ref.py).
Tolerances: zbuf / bary to fp32 rounding of the fp64 values the kernels compute; images 2e-6 absolute for ambient shading, 1e-5 for Phong.
"""
import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

from oracle import fixtures
from oracle import render_ref as R
from renderih_b200 import assets as A
from renderih_b200.manolayer import ManoLayer, rodrigues_batch
from renderih_b200.render import hand_mask_iou, mano_two_hands_renderer, rasterize

pytestmark = pytest.mark.gpu
AMB_TOL, PHONG_TOL = 2e-6, 1e-5


def _hull_mano(side):
    m = dict(A.synthetic_mano(0, side))
    m['f'] = ConvexHull(m['v_template']).simplices.astype(np.int64)
    return m


@pytest.fixture(scope='module')
def env():
    manos = {s: _hull_mano(s) for s in ('left', 'right')}
    layers = {s: ManoLayer(manos[s], center_idx=9, use_pca=True) for s in ('left', 'right')}
    dense = A.synthetic_assets(0)['dense_coor']
    return manos, layers, dense


def _renderer(env, S, mano=None):
    manos, _, dense = env
    return mano_two_hands_renderer(mano_path=mano or manos, dense_path=dense, img_size=S, device='cuda')


def _hands(env, B, seed, gap=0.05):
    _, layers, _ = env
    g = torch.Generator().manual_seed(seed)
    out = []
    for side, dx in (('left', -gap), ('right', gap)):
        rot = rodrigues_batch((torch.rand(B, 3, generator=g) - 0.5) * 2.0).cuda()
        pose, shape = torch.randn(B, 45, generator=g) * 0.6, torch.randn(B, 10, generator=g) * 0.5
        v, _ = layers[side](rot, pose.cuda(), shape.cuda())
        out.append(v + torch.tensor([dx, 0.0, 0.0], device='cuda'))
    return out


def _camera(B, S, persp, seed):
    g = torch.Generator().manual_seed(seed + 7)
    if persp:
        K = torch.zeros(B, 3, 3)
        K[:, 0, 0] = S * (1.0 + 0.3 * torch.rand(B, generator=g)); K[:, 1, 1] = K[:, 0, 0] * (0.9 + 0.2 * torch.rand(B, generator=g))
        K[:, :2, 2] = S / 2 + (torch.rand(B, 2, generator=g) - 0.5) * S * 0.2; K[:, 2, 2] = 1
        return {'cameras': K.cuda()}, R.persp_cam(K.numpy())
    scale, t = 1.5 + torch.rand(B, generator=g), (torch.rand(B, 2, generator=g) - 0.5) * 0.3
    return {'scale': scale.cuda(), 'trans2d': t.cuda()}, R.ortho_cam(scale.numpy(), t.numpy())


def _place(v, persp):
    return v + torch.tensor([0.0, 0.0, 0.6], device='cuda') if persp else v


def _cam_arg(cam):
    return cam['cameras'] if 'cameras' in cam else (cam['scale'], cam['trans2d'])


def _check_fragments(frag, ref, max_amb=1e-3):
    p2f = frag.pix_to_face[..., 0].cpu().numpy()
    amb = ref['ambiguous']
    assert amb.mean() <= max_amb, amb.mean()
    ok = ~amb
    bad = (p2f != ref['pix_to_face']) & ok
    assert not bad.any(), '%d non-ambiguous pixels differ' % bad.sum()
    cov = ok & (ref['pix_to_face'] >= 0)
    z, b = frag.zbuf[..., 0].cpu().numpy().astype(np.float64), frag.bary_coords[..., 0, :].cpu().numpy().astype(np.float64)
    assert np.all(np.abs(z[cov] - ref['zbuf'][cov]) <= 2.0 ** -23 * np.abs(ref['zbuf'][cov]))
    assert np.abs(b[cov] - ref['bary'][cov]).max(initial=0) <= 3e-7
    bg = ok & (ref['pix_to_face'] < 0)
    assert (z[bg] == -1).all() and (b[bg] == -1).all()
    return p2f


@pytest.mark.parametrize('persp', [0, 1])
@pytest.mark.parametrize('S', [64, 256])
@pytest.mark.parametrize('B', [1, 5, 64])
def test_fragments_match_oracle(env, B, S, persp):
    r = _renderer(env, S)
    vl, vr = _hands(env, B, seed=10 * B + S + persp)
    v = _place(torch.cat([vl, vr], 1), persp)
    cam, cams = _camera(B, S, persp, B + S)
    frag = rasterize(v, r.faces_np, _cam_arg(cam), S)
    ref = R.render(v.cpu().numpy(), r.faces_np, cams, persp, S, np.ones(3), False)
    p2f = _check_fragments(frag, ref)
    assert (p2f >= 0).mean() > 0.02          # the hands are on screen


def _img_check(img, alpha, ref, p2f, tol):
    ok = ~ref['ambiguous'] & (p2f == ref['pix_to_face'])
    img, alpha = img.cpu().numpy().astype(np.float64), alpha.cpu().numpy()
    err = np.abs(img - ref['img'])[ok].max()
    assert err <= tol, err
    assert np.array_equal(alpha[ok], ref['alpha'][ok])
    assert np.allclose(img[ok & (ref['pix_to_face'] < 0)], 1 / 255, rtol=0, atol=1e-9)


@pytest.mark.parametrize('persp', [0, 1])
def test_images_match_oracle_for_every_method(env, persp):
    B, S = 5, 128
    r = _renderer(env, S)
    vl, vr = (_place(x, persp) for x in _hands(env, B, seed=3 + persp))
    cam, cams = _camera(B, S, persp, 5)
    F1 = len(r.faces_np) // 2
    two, one = r.faces_np, r.faces_np[:F1]
    vboth = torch.cat([vl, vr], 1)
    p2f_two = rasterize(vboth, two, _cam_arg(cam), S).pix_to_face[..., 0].cpu().numpy()
    p2f_one = rasterize(vl, one, _cam_arg(cam), S).pix_to_face[..., 0].cpu().numpy()
    nb = vboth.cpu().numpy()
    default = np.concatenate([np.tile([204., 153., 0.], (778, 1)), np.tile([102., 102., 255.], (778, 1))])
    mask = np.concatenate([np.tile([0., 0., 255.], (778, 1)), np.tile([0., 255., 0.], (778, 1))])
    dense = np.concatenate([env[2], env[2]]).astype(np.float32).astype(np.float64) * np.float32(255)
    cases = [
        (lambda: r.render_rgb(v3d_left=vl, v3d_right=vr, **cam), nb, two, default, True, p2f_two),
        (lambda: r.render_rgb(v3d_left=vl, v3d_right=vr, amblights=True, v_color=(10., 200., 30.), **cam), nb, two, [10., 200., 30.], False, p2f_two),
        (lambda: (r.render_mask(v3d_left=vl, v3d_right=vr, **cam), None), nb, two, mask, False, p2f_two),
        (lambda: r.render_densepose(v3d_left=vl, v3d_right=vr, **cam), nb, two, dense, False, p2f_two),
        (lambda: r.render_single_rgb(v3d_left=vl, **cam), vl.cpu().numpy(), one, np.ones(3), True, p2f_one),
        (lambda: (r.render_single_mask(v3d=vl, **cam), None), vl.cpu().numpy(), one, np.full(3, 255.), False, p2f_one),
    ]
    for fn, verts, faces, colors, phong, p2f in cases:
        img, alpha = fn()
        ref = R.render(verts, faces, cams, persp, S, colors, phong)
        if alpha is None:
            alpha = torch.from_numpy(ref['alpha'])
        _img_check(img, alpha, ref, p2f, PHONG_TOL if phong else AMB_TOL)


def test_render_rgb_orth_matches_oracle(env):
    B, S = 5, 128
    r = _renderer(env, S)
    vl, vr = _hands(env, B, seed=21, gap=0.0)
    g = torch.Generator().manual_seed(4)
    sl, sr = (1.5 + torch.rand(B, generator=g)).cuda(), (1.5 + torch.rand(B, generator=g)).cuda()
    tl, tr = ((torch.rand(B, 2, generator=g) - 0.5) * 0.4).cuda(), ((torch.rand(B, 2, generator=g) - 0.5) * 0.4).cuda()
    vr_before = vr.clone()
    img, alpha = r.render_rgb_orth(sl, tl, sr, tr, vl, vr)
    assert torch.equal(vr, vr_before)
    vr_m = R.orth_right_into_left(sl.cpu().numpy(), tl.cpu().numpy(), sr.cpu().numpy(), tr.cpu().numpy(), vr.cpu().numpy())
    nb = np.concatenate([vl.cpu().numpy(), vr_m], 1)
    cams = R.ortho_cam(sl.cpu().numpy(), tl.cpu().numpy())
    p2f = rasterize(torch.from_numpy(nb).cuda(), r.faces_np, (sl, tl), S).pix_to_face[..., 0].cpu().numpy()
    default = np.concatenate([np.tile([204., 153., 0.], (778, 1)), np.tile([102., 102., 255.], (778, 1))])
    ref = R.render(nb, r.faces_np, cams, False, S, default, True)
    assert ref['ambiguous'].mean() <= 1e-3
    _img_check(img, alpha, ref, p2f, PHONG_TOL)


def test_stress_random_sliver_faces(env):
    B, S = 2, 64
    synth = {s: A.synthetic_mano(0, s) for s in ('left', 'right')}
    r = _renderer(env, S, mano=synth)
    vl, vr = _hands(env, B, seed=5, gap=0.02)
    for persp in (0, 1):
        cam, cams = _camera(B, S, persp, 9)
        v = _place(torch.cat([vl, vr], 1), persp)
        frag = rasterize(v, r.faces_np, _cam_arg(cam), S)
        ref = R.render(v.cpu().numpy(), r.faces_np, cams, persp, S, np.ones(3), False)
        _check_fragments(frag, ref, max_amb=1e-2)
        img = r.render_mask(v3d_left=_place(vl, persp), v3d_right=_place(vr, persp), **cam)
        refm = R.render(v.cpu().numpy(), r.faces_np, cams, persp, S, np.concatenate([np.tile([0., 0., 255.], (778, 1)), np.tile([0., 255., 0.], (778, 1))]), False)
        _img_check(img, torch.from_numpy(refm['alpha']), refm, frag.pix_to_face[..., 0].cpu().numpy(), AMB_TOL)


def test_stress_offscreen_fullscreen_and_degenerate_faces():
    S = 64
    verts = torch.tensor([[
        [-5.0, -5.0, 0.1], [5.0, -5.0, 0.2], [0.0, 8.0, 0.3],          # 0: covers the whole image
        [0.5, 0.5, -0.2], [3.0, 0.6, -0.2], [0.7, 3.0, -0.2],          # 1: partly off-screen (in front)
        [4.0, 4.0, -0.5], [6.0, 4.0, -0.5], [4.0, 6.0, -0.5],          # 2: fully off-screen
        [0.1, 0.1, -0.9], [0.3, 0.3, -0.9], [0.5, 0.5, -0.9],          # 3: collinear (zero area), in front of everything
        [-0.3, 0.2, -0.9],                                             # 4: repeated vertex (zero area)
    ]], device='cuda')
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11], [12, 12, 10]])
    scale, t = torch.tensor([0.4], device='cuda'), torch.tensor([[0.0, 0.0]], device='cuda')
    frag = rasterize(verts, faces, (scale, t), S)
    ref = R.render(verts.cpu().numpy(), faces, R.ortho_cam([0.4], [[0.0, 0.0]]), False, S, np.ones(3), False)
    p2f = _check_fragments(frag, ref, max_amb=2e-2)
    assert (p2f >= 0).all()                                             # the big face covers every pixel
    assert set(np.unique(p2f)) == {0, 1}
    assert (p2f == 1).sum() > 100


def test_consistent_with_model_projection(env):
    from renderih_b200.model import load_model
    a = A.synthetic_assets(0)
    model = load_model(assets=a)
    model.load_state_dict(fixtures.init_state_dict(model.state_dict()))
    model = model.cuda().eval()
    with torch.no_grad():
        result, params = model(fixtures.make_image(2).cuda())[:2]
    S = 256
    r = _renderer(env, S)
    v3, v2 = result['verts3d'], result['verts2d']
    _, alpha = r.render_rgb_orth(params['scale']['left'], params['trans2d']['left'], params['scale']['right'], params['trans2d']['right'],
                                 v3['left'], v3['right'])
    F1 = len(r.faces_np) // 2
    hand = r.faces_np[:F1]
    for b in range(2):
        cl, al = R.coverage_2d(v2['left'][b].cpu().numpy(), hand, S, tol_px=1e-3)
        cr, ar = R.coverage_2d(v2['right'][b].cpu().numpy(), hand, S, tol_px=1e-3)
        ok = ~(al | ar)
        cov = alpha[b].cpu().numpy() > 0
        assert (cl | cr).sum() > 0
        assert np.array_equal(cov[ok], (cl | cr)[ok]), (cov[ok] != (cl | cr)[ok]).sum()
        assert (al | ar).mean() < 1e-3


@pytest.mark.parametrize('persp', [0, 1])
def test_hand_mask_iou(env, persp):
    B, S = 5, 128
    r = _renderer(env, S)
    vl, vr = (_place(x, persp) for x in _hands(env, B, seed=31, gap=0.03))
    cam, cams = _camera(B, S, persp, 13)
    one = r.faces_np[:len(r.faces_np) // 2]
    iou = hand_mask_iou(vl, vr, one, S, **cam).cpu().numpy().astype(np.float64)
    ref, amb, uni = R.mask_iou(vl.cpu().numpy(), vr.cpu().numpy(), one, cams, persp, S)
    assert (uni > 0).all() and (ref > 0).any()
    assert np.all(np.abs(iou - ref) <= amb / uni + 1e-6), (iou, ref)
    assert np.array_equal(r.mask_iou(v3d_left=vl, v3d_right=vr, **cam).cpu().numpy(), iou.astype(np.float32))
    same = hand_mask_iou(vl, vl, one, S, **cam).cpu().numpy()
    assert (same == 1).all()
    far = vr + torch.tensor([0.0, 50.0, 0.0], device='cuda')      # off-screen
    assert (hand_mask_iou(vl, far, one, S, **cam).cpu().numpy() == 0).all()
    assert np.isnan(hand_mask_iou(far, far, one, S, **cam).cpu().numpy()).all()


def test_deterministic_and_cuda_graph(env):
    B, S = 8, 128
    r = _renderer(env, S)
    vl, vr = _hands(env, B, seed=41)
    cam, _ = _camera(B, S, 0, 17)
    a = r.render_rgb(v3d_left=vl, v3d_right=vr, **cam)
    b = r.render_rgb(v3d_left=vl, v3d_right=vr, **cam)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    eager = (a[0], r.render_densepose(v3d_left=vl, v3d_right=vr, **cam)[0], r.mask_iou(v3d_left=vl, v3d_right=vr, **cam))
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        r.render_rgb(v3d_left=vl, v3d_right=vr, **cam)
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = (r.render_rgb(v3d_left=vl, v3d_right=vr, **cam)[0], r.render_densepose(v3d_left=vl, v3d_right=vr, **cam)[0],
               r.mask_iou(v3d_left=vl, v3d_right=vr, **cam))
    for o in out:
        o.zero_()
    g.replay()
    torch.cuda.synchronize()
    for o, e in zip(out, eager):
        assert torch.equal(o, e) or (torch.isnan(e).any() and torch.equal(torch.nan_to_num(o), torch.nan_to_num(e)))


def test_rejected_inputs(env):
    r = _renderer(env, 64)
    vl, vr = _hands(env, 1, seed=1)
    cam, _ = _camera(1, 64, 0, 1)
    with pytest.raises(RuntimeError):
        r.render_rgb(v3d_left=vl.cpu(), v3d_right=vr.cpu(), **cam)
    with pytest.raises(RuntimeError):
        hand_mask_iou(vl.cpu(), vr.cpu(), r.faces_np[:10], 64, **cam)
    with pytest.raises(NotImplementedError):
        mano_two_hands_renderer(mano_path=env[0], dense_path=env[2], img_size=(480, 640))
    with pytest.raises(NotImplementedError):
        r.render_rgb(v3d_left=vl, v3d_right=vr, uv_verts=torch.zeros(1, 10, 2, device='cuda'), **cam)
    with pytest.raises(NotImplementedError):
        r.render_rgb(v3d_left=vl, v3d_right=vr, lights=object(), **cam)
    vg = vl.clone().requires_grad_(True)
    img, alpha = r.render_rgb(v3d_left=vg, v3d_right=vr, **cam)
    assert not img.requires_grad and not alpha.requires_grad
