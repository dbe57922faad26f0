"""End-to-end parity of the CUDA path: HandNET_GCN (forward, forward+backward through calc_loss_GCN) and ManoLayer
against the CPU oracle on the same seeded inputs, and against the golden vectors the unmodified reference produced.

Stated tolerances (float32 arithmetic, different summation orders through ~60 layers):
  eval-mode forward  : 2e-5 relative to each tensor's max magnitude (the fp32 CPU oracle itself is ~1e-6 from fp64)
  train-mode forward : 5e-3 relative at batch 2 -- BatchNorm batch statistics over as few as 128 samples make the
                       net ill-conditioned: the fp32 CPU oracle is already 1e-4..8e-4 away from its own fp64 evaluation
                       (measured, DESIGN.md "Numerics"), so that is the floor any fp32 implementation can be held to
  loss               : 1e-3 relative (train mode)
  gradients          : 2e-2 relative per-tensor norm (train mode, same conditioning argument)
  ManoLayer vertices : 2e-6 m absolute (north_star 1e-6 m scale)
"""
import os

import numpy as np
import pytest
import torch

from oracle import fixtures, mano_ref, model_ref
from renderih_b200 import assets as rih_assets

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FWD_TOL, TRAIN_FWD_TOL, GRAD_TOL = 2e-5, 5e-3, 2e-2
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def flat(out):
    result, params, hlist, other = out
    d = {}
    for side in ('left', 'right'):
        d['verts3d_' + side] = result['verts3d'][side]; d['verts2d_' + side] = result['verts2d'][side]
        d['scale_' + side] = params['scale'][side]; d['trans2d_' + side] = params['trans2d'][side]
        d['v3c_' + side] = hlist[0]['verts3d'][side]; d['v2c_' + side] = hlist[0]['verts2d'][side]
        d['v3list_' + side] = other['verts3d_MANO_list'][side][0]; d['v2list_' + side] = other['verts2d_MANO_list'][side][0]
    for k in ('hms', 'mask', 'dense'):
        d[k + '_sub'] = other[k][:, :, ::8, ::8]; d[k + '_mean'] = other[k].mean(dim=(2, 3))
        d[k] = other[k]
    return d


@pytest.fixture(scope='module')
def gold():
    return torch.load(os.path.join(GOLD, 'model_synth_b2.pt'), weights_only=False)


@pytest.fixture(scope='module')
def setup(gold):
    from renderih_b200.model import load_model
    a = rih_assets.synthetic_assets(0)
    model = load_model(assets=a)
    sd = fixtures.init_state_dict(model.state_dict())
    assert fixtures.checksum(sd) == gold['weights_sha256']
    model.load_state_dict(sd)
    return a, sd, model.cuda()


def test_forward_eval_matches_oracle_and_reference_golden(gold, setup):
    a, sd, model = setup
    model.eval()
    img = fixtures.make_image(gold['batch'])
    with torch.no_grad():
        out = flat(model(img.cuda()))
        ora = flat(model_ref.model_forward({k: v.clone() for k, v in sd.items()}, model_ref.prepare_assets(a), img, training=False))
    worst = {}
    for k, v in ora.items():
        assert out[k].shape == v.shape, k
        worst[k] = rel_err(out[k], v)
    print('eval fwd rel errs vs oracle:', {k: '%.2e' % e for k, e in worst.items()})
    for k, e in worst.items():
        assert e < FWD_TOL, (k, e)
    for k, v in gold['eval'].items():
        assert rel_err(out[k], v) < FWD_TOL, ('golden', k, rel_err(out[k], v))
    # MPJPE-style number (SURVEY 8d): joints = J21 @ verts3d, root-relative, mean L2, in the model's units x1000
    la = fixtures.make_loss_assets(a, rih_assets.synthetic_mano(0, 'left'), rih_assets.synthetic_mano(0, 'right'))
    for side in ('left', 'right'):
        J = la[side]['J21']
        jo = torch.matmul(J, out['verts3d_' + side].cpu()); jr = torch.matmul(J, ora['verts3d_' + side])
        jo, jr = jo - jo[:, :1], jr - jr[:, :1]
        mpjpe = float((jo - jr).norm(dim=-1).mean()) * 1000
        scale = float(jr.norm(dim=-1).mean()) * 1000
        print('MPJPE(ours vs oracle) %s: %.3e (joint scale %.3e) -> relative %.2e' % (side, mpjpe, scale, mpjpe / scale))
        assert mpjpe / scale < FWD_TOL


def test_forward_eval_tensor_core_tf32_mode(gold, setup):
    """wgmma path: TF32 multiplicands (10-bit mantissa, truncated by the hardware) with fp32 accumulation for the 1x1
    convolutions and nn.Linear GEMMs -- the arithmetic the reference's own cuDNN convolutions use on this GPU by default.
    Stated tolerance: 5e-2 relative to each tensor's max magnitude (single-pass, TRUNCATING TF32 through ~60 layers: the
    truncation bias accumulates coherently; measured 5e-4 ... 2e-2).  This mode is a speed option, not the parity mode."""
    from renderih_b200 import ops
    a, sd, model = setup
    model.load_state_dict(sd)
    model.eval()
    img = fixtures.make_image(gold['batch'])
    ops.set_gemm_mode('tf32', 'tf32')
    try:
        with torch.no_grad():
            out = flat(model(img.cuda()))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    errs = {k: rel_err(out[k], v) for k, v in gold['eval'].items()}
    print('tf32-mode eval rel errs vs reference golden:', {k: '%.2e' % e for k, e in errs.items()})
    for k, e in errs.items():
        assert e < 5e-2, (k, e)


def test_forward_eval_reference_numerics_class_mode(gold, setup):
    """bench.py's default arithmetic: TF32 (round-to-nearest) convolutions -- what the reference's cuDNN convolutions do on
    this GPU by default -- and fp32-faithful 3xTF32 nn.Linear GEMMs.  Stated tolerance: 1e-2 relative to each tensor's max."""
    from renderih_b200 import ops
    a, sd, model = setup
    model.load_state_dict(sd)
    model.eval()
    img = fixtures.make_image(gold['batch'])
    ops.set_gemm_mode('tf32rn', 'tf32x3')
    try:
        with torch.no_grad():
            out = flat(model(img.cuda()))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    errs = {k: rel_err(out[k], v) for k, v in gold['eval'].items()}
    print('ref-class (tf32rn conv + 3xTF32 linear) eval rel errs vs reference golden:', {k: '%.2e' % e for k, e in errs.items()})
    for k, e in errs.items():
        assert e < 1e-2, (k, e)


def test_forward_eval_mean_compensated_truncating_tf32(gold, setup):
    """'tf32c' convolutions (truncating TF32 + 7.05e-4 mean compensation in the epilogue) + 3xTF32 Linears: must be as accurate as
    the round-to-nearest variant (stated tolerance 1e-2, same as the reference-numerics-class mode)."""
    from renderih_b200 import ops
    a, sd, model = setup
    model.load_state_dict(sd)
    model.eval()
    img = fixtures.make_image(gold['batch'])
    ops.set_gemm_mode('tf32c', 'tf32x3')
    try:
        with torch.no_grad():
            out = flat(model(img.cuda()))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    errs = {k: rel_err(out[k], v) for k, v in gold['eval'].items()}
    print('tf32c conv + 3xTF32 linear eval rel errs vs reference golden:', {k: '%.2e' % e for k, e in errs.items()})
    for k, e in errs.items():
        assert e < 1e-2, (k, e)


def test_forward_eval_tensor_core_3xtf32_mode(gold, setup):
    """wgmma with the in-kernel hi/lo split (3 MMAs per step): fp32-faithful tensor-core arithmetic.
    Stated tolerance: 1e-3 relative to each tensor's max magnitude (measured 3e-5 ... 4.5e-4: limited by the tensor core's
    truncating internal accumulation, two orders of magnitude tighter than single-pass TF32)."""
    from renderih_b200 import ops
    a, sd, model = setup
    model.load_state_dict(sd)
    model.eval()
    img = fixtures.make_image(gold['batch'])
    ops.set_gemm_mode('tf32x3', 'tf32x3')
    try:
        with torch.no_grad():
            out = flat(model(img.cuda()))
    finally:
        ops.set_gemm_mode('simt', 'simt')
    errs = {k: rel_err(out[k], v) for k, v in gold['eval'].items()}
    print('tf32x3-mode eval rel errs vs reference golden:', {k: '%.2e' % e for k, e in errs.items()})
    for k, e in errs.items():
        assert e < 1e-3, (k, e)


def test_forward_backward_train_matches_oracle_and_reference_golden(gold, setup):
    a, sd, model = setup
    model.load_state_dict(sd)
    model.train()
    for m in model.modules():
        if hasattr(m, 'p'):
            m.p = 0.0       # dropout RNG streams cannot match torch's: parity runs use TRAIN.dropout = 0 (SURVEY 7)
    model.decoder.unsample_layer.weight.requires_grad_(False)
    img = fixtures.make_image(gold['batch'])
    la = fixtures.make_loss_assets(a, rih_assets.synthetic_mano(0, 'left'), rih_assets.synthetic_mano(0, 'right'))
    la_cuda = {s: {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()} for s, d in la.items()}
    labels = fixtures.make_labels(gold['batch'])
    model.zero_grad()
    out = model(img.cuda())
    loss = model_ref.calc_loss_GCN(out, {k: v.cuda() for k, v in labels.items()}, la_cuda)   # loss graph in torch (caller side)
    loss.backward()
    fo = flat(out)
    for k, v in gold['train']['out'].items():
        assert rel_err(fo[k], v) < TRAIN_FWD_TOL, ('train fwd', k, rel_err(fo[k], v))
    print('loss ours %.6f reference %.6f' % (float(loss), gold['train']['loss']))
    assert abs(float(loss) - gold['train']['loss']) / gold['train']['loss'] < 1e-3
    assert rel_err(model.encoder.resnet.bn1.running_mean, gold['train']['bn1_running_mean']) < 1e-4
    assert rel_err(model.encoder.resnet.bn1.running_var, gold['train']['bn1_running_var']) < 1e-4
    params = dict(model.named_parameters())
    for k in gold['train']['no_grad_keys']:
        g = params[k].grad
        assert g is None or float(g.abs().max()) == 0.0, k
    worst = (0.0, None)
    for k, g in gold['train']['grads'].items():
        mine = params[k].grad
        assert mine is not None, k
        if k.endswith('w_ks.bias'):
            continue   # mathematically zero gradient (softmax shift invariance): round-off only
        e = abs(float(mine.norm()) - g['norm']) / max(g['norm'], 1e-6)
        if e > worst[0]:
            worst = (e, k)
        assert e < GRAD_TOL, (k, e, float(mine.norm()), g['norm'])
        if 'full' in g and g['norm'] > 1e-3:
            cos = float(torch.nn.functional.cosine_similarity(mine.detach().cpu().flatten().double(), g['full'].flatten().double(), dim=0))
            assert cos > 0.995, (k, cos)   # direction of small gradient tensors (element-wise equality is ill-conditioned at batch 2)
    print('worst grad-norm rel err %.2e at %s' % worst)


def test_train_mode_with_dropout_runs_and_is_finite(setup):
    a, sd, model = setup
    model.load_state_dict(sd)
    model.train()
    for m in model.modules():
        if hasattr(m, 'p'):
            m.p = 0.05
    out = model(fixtures.make_image(2).cuda())
    s = sum(v.float().sum() for v in (out[0]['verts3d']['left'], out[0]['verts3d']['right'], out[0]['verts2d']['left']))
    s.backward()
    assert torch.isfinite(s)
    n = sum(1 for p in model.parameters() if p.grad is not None and torch.isfinite(p.grad).all())
    assert n > 700


def test_mano_layer_matches_reference_golden_and_oracle():
    from renderih_b200.manolayer import ManoLayer, rodrigues_batch
    mg = torch.load(os.path.join(GOLD, 'mano_synth.pt'), weights_only=False)
    inp = fixtures.make_mano_inputs(5)
    root = rodrigues_batch(inp['axis'])
    for case in mg['cases']:
        c = case['cfg']
        layer = ManoLayer(rih_assets.synthetic_mano(0, case['side']), center_idx=c['center_idx'], use_pca=c['use_pca'], new_skel=c['new_skel'])
        pose = inp['pose_pca'][:, :c['ncomps']] if c['use_pca'] else layer.axis2Rmat(inp['pose_axis'])
        tr, sc = (inp['trans'], inp['scale']) if c['ts'] else (None, None)
        v, j = layer(root.cuda(), pose.cuda(), inp['shape'].cuda(), None if tr is None else tr.cuda(), None if sc is None else sc.cuda())
        ev, ej = float((v.cpu() - case['v']).abs().max()), float((j.cpu() - case['j']).abs().max())
        print('mano %s %s: max |dv| %.2e  max |dj| %.2e' % (case['side'], c, ev, ej))
        assert ev < 2e-6 and ej < 2e-6
        v2, j2 = layer(root, pose, inp['shape'], tr, sc)       # CPU inputs -> staged through the GPU, returned on CPU
        assert v2.device.type == 'cpu' and float((v2 - case['v']).abs().max()) < 2e-6


def test_mano_layer_batch_sizes_and_edge_cases():
    from renderih_b200.manolayer import ManoLayer
    m = rih_assets.synthetic_mano(0, 'right')
    md = dict(m); md['J_regressor'] = np.asarray(m['J_regressor'].todense())
    layer = ManoLayer(m, center_idx=9, use_pca=True)
    for bs in (1, 64, 257):
        g = torch.Generator().manual_seed(bs)
        root = torch.linalg.qr(torch.randn(bs, 3, 3, generator=g))[0]
        pose, shape = torch.randn(bs, 45, generator=g) * 0.5, torch.randn(bs, 10, generator=g)
        v, j = layer(root.cuda(), pose.cuda(), shape.cuda())
        vr, jr = mano_ref.mano_forward(md, root.numpy(), pose.numpy(), shape.numpy())
        assert np.abs(v.cpu().numpy() - vr).max() < 2e-6 and np.abs(j.cpu().numpy() - jr).max() < 2e-6
    v, j = layer(torch.zeros(0, 3, 3).cuda(), torch.zeros(0, 45).cuda(), torch.zeros(0, 10).cuda())   # empty batch
    assert v.shape == (0, 778, 3) and j.shape == (0, 21, 3)
    z = torch.zeros(1, 45).cuda()   # zero pose: Rodrigues at the 1e-8 guard (manolayer.py:37)
    v, j = layer(torch.eye(3)[None].cuda(), z, torch.zeros(1, 10).cuda())
    vr, jr = mano_ref.mano_forward(md, np.eye(3)[None], np.zeros((1, 45)), np.zeros((1, 10)))
    assert np.abs(v.cpu().numpy() - vr).max() < 2e-6


def test_mano_layer_backward_matches_reference_golden_and_oracle():
    """Fused backward kernel (rih_mano_bwd) against the unmodified reference's autograd gradients (tests/golden/mano_grad_synth.pt)
    and, at other batch sizes / option combinations, against autograd through the float64 torch restatement.
    Stated tolerance: 2e-5 relative to each gradient tensor's max magnitude (fp32 reductions over 2334 terms)."""
    from renderih_b200.manolayer import ManoLayer, rodrigues_batch
    gg = torch.load(os.path.join(GOLD, 'mano_grad_synth.pt'), weights_only=False)
    inp = fixtures.make_mano_inputs(5)
    wv, wj = fixtures.make_mano_loss_weights(5)
    for case in gg['cases']:
        c = case['cfg']
        layer = ManoLayer(rih_assets.synthetic_mano(0, case['side']), center_idx=c['center_idx'], use_pca=c['use_pca'], new_skel=c['new_skel'])
        root = rodrigues_batch(inp['axis']).cuda().requires_grad_(True)
        pose = (inp['pose_pca'][:, :c['ncomps']] if c['use_pca'] else layer.axis2Rmat(inp['pose_axis'])).clone().cuda().requires_grad_(True)
        shape = inp['shape'].clone().cuda().requires_grad_(True)
        tr = inp['trans'].clone().cuda().requires_grad_(True) if c['ts'] else None
        sc = inp['scale'].clone().cuda().requires_grad_(True) if c['ts'] else None
        v, j = layer(root, pose, shape, tr, sc)
        ((v * wv.cuda()).sum() + (j * wj.cuda()).sum()).backward()
        errs = {}
        for name, t in (('d_root', root), ('d_pose', pose), ('d_shape', shape), ('d_trans', tr), ('d_scale', sc)):
            if t is not None:
                errs[name] = rel_err(t.grad, case[name])
        print('mano bwd %s %s:' % (case['side'], c), {k: '%.1e' % e for k, e in errs.items()})
        for k, e in errs.items():
            assert e < 2e-5, (case['side'], c, k, e)
    # other batch sizes, only one of the two outputs used, zero pose (Rodrigues at the 1e-8 guard), vs the fp64 restatement
    m = rih_assets.synthetic_mano(0, 'right')
    for bs, use_pca, center, new_skel, only in ((1, True, 9, False, 'v'), (64, True, None, True, 'j'), (130, False, 4, False, 'both'), (3, True, 9, False, 'zero')):
        g = torch.Generator().manual_seed(100 + bs)
        layer = ManoLayer(m, center_idx=center, use_pca=use_pca, new_skel=new_skel)
        root = torch.linalg.qr(torch.randn(bs, 3, 3, generator=g))[0]
        pose = torch.randn(bs, 45, generator=g) * 0.5 if use_pca else layer.axis2Rmat(torch.randn(bs, 45, generator=g) * 0.5)
        if only == 'zero':
            pose = -layer.hands_mean[None].repeat(bs, 1).mm(layer.hands_components_inv)      # axis-angle == 0 for every joint
        shape, trans, scale = torch.randn(bs, 10, generator=g), torch.randn(bs, 3, generator=g), torch.rand(bs, generator=g) + 0.5
        cv, cj = torch.randn(bs, 778, 3, generator=g), torch.randn(bs, 21, 3, generator=g)
        ours = [t.clone().cuda().requires_grad_(True) for t in (root, pose, shape, trans, scale)]
        ref = [t.clone().double().requires_grad_(True) for t in (root, pose, shape, trans, scale)]
        v, j = layer(*ours)
        vr, jr = mano_ref.mano_forward_torch(m, *ref, use_pca=use_pca, center_idx=center, new_skel=new_skel)
        lo = (v * cv.cuda()).sum() * (only != 'j') + (j * cj.cuda()).sum() * (only != 'v')
        lr = (vr * cv.double()).sum() * (only != 'j') + (jr * cj.double()).sum() * (only != 'v')
        lo.backward(); lr.backward()
        for name, a, b in zip(('root', 'pose', 'shape', 'trans', 'scale'), ours, ref):
            if only == 'zero' and name == 'pose':
                continue      # d/d(axis) at |axis| = 0: the reference's norm subgradient (0) times 1/eps factors -- not a meaningful number
            e = rel_err(a.grad, b.grad)
            assert e < 2e-5, (bs, use_pca, center, new_skel, only, name, e)
        assert torch.isfinite(ours[1].grad).all()
    # empty batch
    layer = ManoLayer(m, center_idx=9, use_pca=True)
    z = [torch.zeros(0, 3, 3).cuda().requires_grad_(True), torch.zeros(0, 45).cuda().requires_grad_(True), torch.zeros(0, 10).cuda().requires_grad_(True)]
    v, j = layer(*z)
    (v.sum() + j.sum()).backward()
    assert z[1].grad.shape == (0, 45)


@pytest.mark.parametrize('variant', ['resnet50', 'graph'])
def test_train_step_launches_only_on_registered_side_streams(variant):
    """Every kernel of a train-mode forward + backward is launched on the caller's stream or on a side stream registered in
    ops.STEP_STREAMS: train.TrainStep's overlapped gradient all-reduce waits on exactly those streams.  The forward forks onto the
    five side streams (left / right hand, two image-grid encoders, the convolution-side aux stream), none of them serialised."""
    from renderih_b200 import _lib, ops
    from renderih_b200.model import load_model
    from renderih_b200.myhand import load_graph_model
    a = rih_assets.synthetic_assets(0)
    if variant == 'graph':
        model = load_graph_model(None, assets=a, mano_assets={s: rih_assets.synthetic_mano(0, s) for s in ('left', 'right')})
    else:
        model = load_model(assets=a)
    model.load_state_dict(fixtures.init_state_dict(model.state_dict()))
    model = model.cuda().train()
    img = fixtures.make_image(2).cuda()
    caller = torch.cuda.current_stream().cuda_stream or 0
    _lib.TRACE = []
    try:
        result, _, _, other = model(img)
        fwd = {args[-1] or 0 for _, args, _, _ in _lib.TRACE}
        loss = sum(result['verts3d'][s].sum() + result['verts2d'][s].sum() for s in ('left', 'right'))
        loss = loss + sum(other[k].sum() for k in ('hms', 'mask', 'dense') if k in other)
        loss.backward()
        launched = {args[-1] or 0 for _, args, _, _ in _lib.TRACE}
    finally:
        _lib.TRACE = None
    registered = set(ops.STEP_STREAMS)
    assert launched <= registered | {caller}, (variant, launched - registered - {caller})
    wgrad = {st.cuda_stream for st in ops._WG['streams'].values()}
    side = fwd - {caller} - wgrad
    assert len(side) == 5 and side <= registered, (variant, side)
