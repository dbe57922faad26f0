"""The two-hand pose optimiser (renderih_b200/ge_optimizer.py, csrc/ge_optim.cu) against the unmodified reference loop
(tests/golden/ge_optimizer_synth.pt), against an eager loop of the same CUDA loss modules with torch.optim.Adam and ReduceLROnPlateau
(oracle/ge_optimizer_ref.eager_optimize), and its kernels against torch's optimiser and scheduler.

Tolerances: every iteration's total within LOSS_TOL = 1e-4 relative; the learning-rate sequences exactly equal; the final poses within
POSE_TOL * lr and the translations within POSE_TOL * 0.01 lr (each group's own lr), i.e. the trajectories differ by less than a quarter
of one Adam step (an Adam step moves a variable by about lr), except where a gradient is at rounding level: against the eager loop
(50 iterations, up to B = 1024) fewer than EAGER_FRAC of the entries may drift further, each by at most 2 n_iter steps; in the golden
'min_lr' case the translations' gradient is pure rounding noise and gets the same 2 n_iter bound.  The differences come from fp32 summation order (CPU against GPU, or
torch's lerp against the kernel's b1 m + (1 - b1) g)."""
import math

import pytest
import torch

from oracle import ge_optimizer_ref as G
from oracle import make_golden_ge_optimizer as M
from renderih_b200 import ge_optimizer as GO
from renderih_b200._lib import call

pytestmark = pytest.mark.gpu
LOSS_TOL, POSE_TOL = 1e-4, 0.25
EAGER_FRAC = 5e-2         # share of entries allowed beyond POSE_TOL * lr against the eager loop (test_against_eager_driver)


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


def _check_out(out, ref, lr, what, tsl_tol=None):
    tsl_tol = POSE_TOL * 0.01 * lr if tsl_tol is None else tsl_tol
    for k, tol in (('optimized_hand_pose', POSE_TOL * lr), ('optimized_sub_hand_pose', POSE_TOL * lr), ('optimized_hand_tsl', tsl_tol),
                   ('optimized_sub_hand_tsl', tsl_tol)):
        err = float((out[k] - ref[k]).abs().max())
        print('%s %s max err %.2e (tolerance %.2e)' % (what, k, err, tol))
        assert out[k].shape == ref[k].shape and out[k].device.type == 'cpu'
        assert err <= tol, (what, k, err)


def test_matches_reference_golden():
    gold = M.load()
    for case in gold['cases']:
        opt = G.build(case['weights'], lr=case['lr'], n_iter=case['n_iter'], lambda_contact_loss=case['lambda_contact_loss'],
                      lambda_repulsion_loss=0.0)                  # the golden loop's penetration term is a zero
        opt.set_opt_val(**G.to_device(case['kwargs'], 'cuda'))
        out = opt.optimize()
        loss, lrs = opt.loss_history(), opt.lr_history()
        err = max(_rel(a, b) for a, b in zip(loss, case['loss']))
        print('%-15s total max rel err %.2e over %d iterations' % (case['name'], err, case['n_iter']))
        assert err < LOSS_TOL, case['name']
        assert torch.equal(lrs, case['lrs']), case['name']
        # 'min_lr' has no contact or penetration term, so the translations' gradient is rounding noise of the edge term (translation
        # invariant); Adam normalises it, and each step may go either way on either side: the bound is 2 n_iter steps of that group
        tsl_tol = 2 * case['n_iter'] * 0.01 * case['lr'] if case['name'] == 'min_lr' else None
        _check_out(out, case['out'], case['lr'], case['name'], tsl_tol)


def _eager_case(B, seed, n_iter=50):
    # every nature row masked, one logit clear of the threshold at the start and with pred scale 1: no row's mask flips in 50
    # iterations, a hard decision fp32 rounding could otherwise take differently in the two loops
    weights = G.nature_weights(B, seed, 1000 + seed, scale=1.0, rule='all')
    kw = G.inputs(B, seed, device='cuda')
    opt = G.build(weights, n_iter=n_iter)
    return opt, kw


@pytest.mark.parametrize('B', [1, 64, 257, 1024])
def test_against_eager_driver(B):
    opt, kw = _eager_case(B, 700 + B)
    opt.set_opt_val(**kw)
    hist = []
    ref = G.eager_optimize(opt, kw, opt.n_iter, history=hist)
    out = opt.optimize()
    loss, lrs = opt.loss_history(), opt.lr_history()
    err = max(_rel(a, h[0]) for a, h in zip(loss, hist))
    print('B=%d total max rel err %.2e, final %.5g' % (B, err, float(loss[-1])))
    assert err < LOSS_TOL
    assert lrs.tolist() == [h[1] for h in hist]
    # Over 50 iterations a few pose coordinates whose gradient is near rounding level (Adam normalises it, so the step's direction is
    # decided by rounding) drift apart by whole steps; the bulk must agree to a quarter step, every coordinate to 2 n_iter steps.
    for k, lr in (('optimized_hand_pose', opt.lr), ('optimized_sub_hand_pose', opt.lr), ('optimized_hand_tsl', 0.01 * opt.lr),
                  ('optimized_sub_hand_tsl', 0.01 * opt.lr)):
        d = (out[k] - ref[k]).abs()
        frac = float((d > POSE_TOL * lr).double().mean())
        print('B=%d %s max err %.2e, %.2e of the entries beyond %.2e' % (B, k, float(d.max()), frac, POSE_TOL * lr))
        assert frac < EAGER_FRAC and float(d.max()) <= 2 * opt.n_iter * lr, (B, k, frac, float(d.max()))


def test_graph_replay_equals_eager_replay_bitwise():
    opt, kw = _eager_case(16, 31, n_iter=12)
    outs = []
    for use_graph in (True, False):
        opt.use_graph = use_graph
        opt.set_opt_val(**kw)
        outs.append((opt.optimize(), opt.loss_history(), opt.lr_history(), opt.adam_state()))
    (o1, l1, r1, s1), (o2, l2, r2, s2) = outs
    assert all(torch.equal(o1[k], o2[k]) for k in o1)
    assert torch.equal(l1, l2) and torch.equal(r1, r2)
    assert all(torch.equal(a, b) for a, b in zip(s1[:3], s2[:3])) and s1[3] == s2[3] == 12


def test_no_host_synchronisation_during_replays():
    opt, kw = _eager_case(8, 41, n_iter=3)
    opt.set_opt_val(**kw)
    opt.optimize()                                    # captures
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        opt.launch(10)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(opt.loss_history()) == 10


def test_state_persists_and_recaptures_only_when_needed():
    opt, kw = _eager_case(8, 51, n_iter=10)
    opt.set_opt_val(**kw)
    hist = []
    ref = G.eager_optimize(opt, kw, 25, history=hist)   # one eager run of 25 iterations = our 10 + 15 with the state carried over
    opt.optimize()
    graph = opt._graph
    opt.n_iter = 15
    out = opt.optimize()
    assert opt._graph is graph                          # n_iter change: no recapture
    assert opt.adam_state()[3] == 25
    loss = opt.loss_history()
    assert len(loss) == 15 and max(_rel(a, h[0]) for a, h in zip(loss, hist[10:])) < LOSS_TOL
    _check_out(out, ref, opt.lr, 'second call')
    # coef_val change: takes effect without recapture
    opt.set_opt_val(**kw)
    opt.coef_val['lambda_contact_loss'] = 150.0
    opt.coef_val['lambda_repulsion_loss'] = 0.05
    hist = []
    ref = G.eager_optimize(opt, kw, 15, history=hist)
    out = opt.optimize()
    assert opt._graph is graph
    assert max(_rel(a, h[0]) for a, h in zip(opt.loss_history(), hist)) < LOSS_TOL
    _check_out(out, ref, opt.lr, 'new coef_val')
    # new data at the same B and split: replays the same graph
    kw2 = G.inputs(8, 52, device='cuda')
    opt.set_opt_val(**kw2)
    hist = []
    ref = G.eager_optimize(opt, kw2, 15, history=hist)
    out = opt.optimize()
    assert opt._graph is graph
    _check_out(out, ref, opt.lr, 'new data')
    # a new split and a new B recapture
    split = (([3, 0], [1, 2] + list(range(4, 16))), G.CALLER_SPLIT)
    for kw3 in (G.inputs(8, 53, split, device='cuda'), G.inputs(5, 54, device='cuda')):
        opt.set_opt_val(**kw3)
        hist = []
        ref = G.eager_optimize(opt, kw3, 15, history=hist)
        out = opt.optimize()
        assert opt._graph is not graph
        graph = opt._graph
        _check_out(out, ref, opt.lr, 'recaptured')


def test_pose_lags_one_adam_step():
    opt, kw = _eager_case(4, 61, n_iter=6)
    opt.set_opt_val(**kw)
    out = opt.optimize()
    flat = opt.adam_state()[0].cpu()
    B, n = 4, 15
    var_r = flat[6 * B:6 * B + 4 * B * n].reshape(B, n, 4)
    assert not torch.equal(out['optimized_hand_pose'][:, 1:], var_r)           # the leaves moved after the pose was stored
    opt.set_opt_val(**kw)
    opt.n_iter = 5
    out5 = opt.optimize()
    flat5 = opt.adam_state()[0].cpu()
    assert torch.equal(out['optimized_hand_pose'][:, 1:], flat5[6 * B:6 * B + 4 * B * n].reshape(B, n, 4))   # = the leaves after 5 steps
    assert torch.equal(out['optimized_hand_pose'][:, 0], kw['hand_pose_gt'][1][:, 0].cpu())
    assert torch.equal(out['optimized_hand_tsl'], flat[:3 * B].reshape(B, 3))                                  # translations: after step 6
    assert not torch.equal(out5['optimized_hand_tsl'], out['optimized_hand_tsl'])


def test_assembly_of_unsorted_split():
    split = (([9, 2, 14], [5, 0, 1, 3, 4, 6, 7, 8, 10, 11, 12, 13, 15]), ([15], list(range(15))[::-1]))
    opt, _ = _eager_case(3, 71, n_iter=1)
    kw = G.inputs(3, 71, split, device='cuda')
    opt.set_opt_val(**kw)
    out = opt.optimize()
    for key, pose in (('hand_pose', 'optimized_hand_pose'), ('obj_pose', 'optimized_sub_hand_pose')):
        ref = G.assemble(kw[key + '_gt'][0], kw[key + '_gt'][1], kw[key + '_init'][0], kw[key + '_init'][1]).cpu()
        assert torch.equal(out[pose], ref)


def test_adam_kernel_matches_torch_adam():
    g = torch.Generator().manual_seed(0)
    sizes = (30, 30, 600, 600)
    lrs = [1e-4, 1e-4, 1e-2, 1e-2]
    x0 = [torch.randn(n, generator=g) for n in sizes]
    ref = [x.clone().cuda().requires_grad_(True) for x in x0]
    opt = torch.optim.Adam([{'params': [p], 'lr': lr} for p, lr in zip(ref, lrs)])
    flat = torch.cat(x0).cuda()
    m, v = torch.zeros_like(flat), torch.zeros_like(flat)
    lr_dev = torch.tensor(lrs, dtype=torch.float64, device='cuda')
    step = torch.zeros(1, dtype=torch.int32, device='cuda')
    pw = torch.stack([GO.beta_powers(b, 256) for b in GO.BETAS]).cuda()
    ends = [sum(sizes[:k + 1]) for k in range(4)]
    for t in range(200):
        grads = [torch.randn(n, generator=g).cuda() * (0.1 + t % 7) for n in sizes]
        if t == 100:                                    # lr changed mid-way through device memory
            lr_dev.mul_(0.5)
            for grp in opt.param_groups:
                grp['lr'] *= 0.5
        for p, gr in zip(ref, grads):
            p.grad = gr.clone()
        opt.step()
        gflat = torch.cat(grads)
        call('rih_ge_adam_step', flat.data_ptr(), gflat.data_ptr(), m.data_ptr(), v.data_ptr(), *ends, 4, lr_dev.data_ptr(), step.data_ptr(),
             pw[0].data_ptr(), pw[1].data_ptr(), 256, 0.9, 0.999, 1e-8, torch.cuda.current_stream().cuda_stream)
    errs = []
    for p, a, b in zip(ref, [0] + ends[:3], ends):      # per group, relative to its largest magnitude: the measure rih_adamw_step's test uses
        errs.append(float((flat[a:b] - p.detach()).abs().max() / p.detach().abs().max()))
    err = max(errs)
    print('Adam kernel vs torch.optim.Adam after 200 steps: max rel err %.2e' % err)
    assert err < 1e-6 and int(step) == 200


def _kernel_lrs(seq, lrs):
    dev = 'cuda'
    d = torch.tensor([math.inf] + list(lrs), dtype=torch.float64, device=dev)
    ist = torch.zeros(3, dtype=torch.int32, device=dev)
    n = len(seq)
    losses = torch.tensor(seq, dtype=torch.float32, device=dev)
    hist = torch.zeros(n, device=dev)
    lr_hist = torch.zeros(n, len(lrs), dtype=torch.float64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    for k in range(n):
        call('rih_ge_plateau_step', losses[k].data_ptr(), d[1:].data_ptr(), len(lrs), d.data_ptr(), ist[1:].data_ptr(), hist.data_ptr(),
             lr_hist.data_ptr(), ist[2:].data_ptr(), n, 0.5, 20, 1e-5, 1e-4, 1e-8, st)
    assert torch.equal(hist.isnan(), losses.isnan()) and torch.equal(hist.nan_to_num(), losses.nan_to_num())
    return lr_hist.cpu().tolist()


def test_plateau_kernel_matches_torch_scheduler_bitwise():
    seqs = G.crafted_sequences()
    g = torch.Generator().manual_seed(1)
    for k in range(4):
        seqs['random_%d' % k] = (torch.rand(400, generator=g) * (1 + k) + torch.linspace(2, 0, 400)).tolist()
    for name, seq in seqs.items():
        lrs = [1e-5 + 5e-9, 1e-4, 1e-2, 2e-5] if name == 'eps_rule' else G.LRS
        assert _kernel_lrs(seq, lrs) == G.torch_lrs(seq, lrs), name


def test_rejected_inputs():
    opt, kw = _eager_case(3, 81, n_iter=1)
    with pytest.raises(RuntimeError, match='CUDA'):
        opt.set_opt_val(**dict(kw, hand_tsl_init=kw['hand_tsl_init'].cpu()))
    with pytest.raises(RuntimeError, match='CUDA'):
        opt.set_opt_val(**dict(kw, anchor_id=kw['anchor_id'].cpu()))
    with pytest.raises(TypeError, match='float32'):
        opt.set_opt_val(**dict(kw, obj_tsl_init=kw['obj_tsl_init'].double()))
    with pytest.raises(TypeError, match='float32'):
        opt.set_opt_val(**dict(kw, hand_pose_init=(kw['hand_pose_init'][0], kw['hand_pose_init'][1].double())))
    for bad in (dict(hand_tsl_init=kw['hand_tsl_init'][:2]), dict(hand_shape_init=kw['hand_shape_init'][:, :10]),
                dict(obj_pose_init=(kw['obj_pose_init'][0], kw['obj_pose_init'][1][:, :14])), dict(batch_size=0)):
        with pytest.raises(ValueError):
            opt.set_opt_val(**dict(kw, **bad))
    with pytest.raises(RuntimeError, match='set_opt_val'):
        opt.optimize()
