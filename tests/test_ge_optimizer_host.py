"""Checks of the two-hand pose optimiser (renderih_b200/ge_optimizer.py) that need no GPU: the golden file's consistency, the scheduler
rules of csrc/ge_optim.cu restated in Python against torch's ReduceLROnPlateau, the bias-correction table, and set_opt_val's rejections."""
import math
import os

import pytest
import torch

from oracle import ge_optimizer_ref as G
from oracle.ge_optimizer_ref import LRS, crafted_sequences, torch_lrs
from renderih_b200 import ge_optimizer as GO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ge_optimizer_synth.pt')


def test_golden_file_is_self_consistent():
    from oracle import make_golden_ge_optimizer as M
    gold = M.load(GOLD)
    assert [c['name'] for c in gold['cases']] == [c[0] for c in M.CASES]
    assert os.path.getsize(GOLD) < 300_000
    for case in gold['cases']:
        B, n, lr = case['batch'], case['n_iter'], case['lr']
        assert case['loss'].shape == (n,) and case['lrs'].shape == (n, 4)
        assert torch.isfinite(case['loss']).all()
        out = case['out']
        assert out['optimized_hand_pose'].shape == (B, 16, 4) and out['optimized_sub_hand_pose'].shape == (B, 16, 4)
        assert out['optimized_hand_tsl'].shape == (B, 3) and out['optimized_sub_hand_tsl'].shape == (B, 3)
        kw = case['kwargs']
        for key, pose in (('hand_pose', 'optimized_hand_pose'), ('obj_pose', 'optimized_sub_hand_pose')):
            gi, gv = kw[key + '_gt']
            assert torch.equal(out[pose][:, gi], gv)                       # the gt rows are never moved
        # the stored lr sequence is what the scheduler rules give on the stored loss sequence
        state = {'best': math.inf, 'num_bad': 0, 'lr': [0.01 * lr, 0.01 * lr, lr, lr]}
        for k in range(n):
            GO.plateau_step(state, case['loss'][k])
            assert state['lr'] == case['lrs'][k].tolist(), (case['name'], k)
    low = gold['cases'][[c['name'] for c in gold['cases']].index('min_lr')]
    assert (low['lrs'][:, :2] == 1e-5).all()


def _rules_lrs(losses, lrs):
    state = {'best': math.inf, 'num_bad': 0, 'lr': list(lrs)}
    out = []
    for a in losses:
        GO.plateau_step(state, torch.tensor(a, dtype=torch.float32))
        out.append(list(state['lr']))
    return out


@pytest.mark.parametrize('name', ['nan', 'exact_tie', 'min_lr_floor', 'eps_rule', 'random'])
def test_scheduler_rules_match_torch(name):
    seq = crafted_sequences()[name]
    lrs = [1e-5 + 5e-9, 1e-4, 1e-2, 2e-5] if name == 'eps_rule' else LRS
    ours, ref = _rules_lrs(seq, lrs), torch_lrs(seq, lrs)
    assert ours == ref
    if name == 'min_lr_floor':
        assert ref[-1] == [1e-5] * 4
    if name == 'eps_rule':
        assert ref[-1][0] == 1e-5 + 5e-9                # old - new = 5e-9 <= eps: never changed
    if name == 'exact_tie':
        assert ref[21] != ref[20]                       # the tie is not an improvement: 21 bad epochs, then a reduction


def test_bias_correction_table_is_python_pow():
    for beta in GO.BETAS:
        tab = GO.beta_powers(beta, 3000)
        assert tab.dtype == torch.float64 and tab.shape == (3001,)
        assert all(float(tab[t]) == beta ** t for t in range(3001))
        assert all(1 - float(tab[t]) == 1 - beta ** float(t) for t in (1, 2, 50, 2999))


def _bare():
    return object.__new__(GO.GeOptimizer)


def test_set_opt_val_rejects_bad_partitions_without_cuda():
    kw = G.inputs(2, 0)
    cases = [
        (dict(hand_pose_gt=([0, 1], kw['hand_pose_gt'][1]), hand_pose_init=kw['hand_pose_init']), RuntimeError, 'repeat hand_pose'),
        (dict(hand_pose_init=(list(range(2, 16)), kw['hand_pose_init'][1][:, 1:])), RuntimeError, 'hand_pose: not enough'),
        (dict(obj_pose_gt=([0, 5], kw['obj_pose_gt'][1]), obj_pose_init=kw['obj_pose_init']), RuntimeError, 'repeat obj_pose'),
        (dict(obj_pose_init=(list(range(1, 15)), kw['obj_pose_init'][1][:, :14])), RuntimeError, 'obj_pose: not enough'),
        (dict(hand_shape_gt=kw['hand_shape_init']), RuntimeError, 'both hand_shape'),
        (dict(hand_tsl_gt=kw['hand_tsl_init']), RuntimeError, 'both hand_tsl'),
        (dict(hand_shape_init=None), NotImplementedError, 'shape'),
        (dict(hand_tsl_init=None, hand_tsl_gt=kw['hand_tsl_init']), NotImplementedError, 'vec_sub_tsl'),
        (dict(hand_tsl_init=None), NotImplementedError, 'hand_tsl_init'),
        (dict(obj_tsl_init=None), NotImplementedError, 'obj_tsl_init'),
        (dict(hand_pose_gt=None), NotImplementedError, 'hand_pose_gt'),
        (dict(obj_pose_init=None), NotImplementedError, 'obj_pose_gt'),
        (dict(runtime_vis=object()), NotImplementedError, 'open3d'),
    ]
    for change, exc, match in cases:
        with pytest.raises(exc, match=match):
            GO.GeOptimizer.set_opt_val(_bare(), **dict(kw, **change))
    with pytest.raises(NotImplementedError):
        GO.GeOptimizer.optimize(_bare(), progress=True)
    with pytest.raises(NotImplementedError):
        GO.GeOptimizer('cuda', mode='hand')
