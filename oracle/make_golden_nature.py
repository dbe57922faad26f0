"""Generate tests/golden/nature_synth.pt by running the UNMODIFIED reference discriminator nature loss: Pos2dDiscriminator of
Ver2Code/Discriminator/discrim.py and the unbound GeOptimizer.NatureLoss of hocontact/postprocess/geo_optimizer_both_batch.py, called on
a SimpleNamespace(disc=..., device='cpu'), both imported in place from /root/reference/pose_data_optimize.

Run in the authoring container only:   python -m oracle.make_golden_nature
What is substituted to import them: the stand-ins of make_golden_geo_loss (open3d, trimesh, termcolor, the numpy aliases, the chumpy-free
MANO loader), `termcolor.colored`, and an empty `sdf` module for code_sdf/sdf_template.py.  discrim.pth is not in the reference tree, so
each case's weights are torch.nn.Linear's default initialisation drawn from a numpy generator (oracle/nature_ref.init_state_dict) with a
chosen scale and offset of layer_pred; they and the inputs are rebuilt from the stored seeds by load().  The leaves are the normalised
[B,16,4] poses, so the optimiser's [:, 1:] views are exercised and the root rows' gradient is 0.  The file stores the state_dict keys,
each case's probabilities, masks, loss and both pose gradients.  Nothing derived from MANO is written.
"""
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import nature_ref as R  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
THRESH = -math.log(1.5)           # the mask p1 < 1.5 p0 is l0 - l1 > -ln 1.5
# name, batch, input seed, weight seed, layer_pred scale, how layer_pred's bias is set
CASES = (('mixed', 32, 11, 101, 40.0, 'median'),
         ('one_empty', 16, 12, 102, 40.0, 'one_empty'),
         ('both_empty', 8, 13, 103, 1.0, 'p1_to_1'),
         ('saturated', 16, 14, 104, 1e5, 'median'),
         ('batch_1', 1, 15, 105, 1.0, 'none'))


def poses(B, seed):
    """Normalised [B,16,4] float32 poses of both hands: F.normalize of a perturbed identity, as the optimiser normalises (:708, :736)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(2):
        q = rng.normal(size=(B, 16, 4)) * 0.5
        q[..., 0] += 1.0
        out.append(F.normalize(torch.from_numpy(q).float(), dim=-1))
    return out


def _diffs(sd, right16, left16):
    """l0 - l1 per row [2,B] in float64."""
    return torch.stack([(lambda z: z[:, 0] - z[:, 1])(R.logits(sd, R.features(q[:, 1:].double())[0])) for q in (right16, left16)])


def weights(case):
    """-> (seed, pred_scale, pred_bias) of a case, the bias chosen from the case's rule."""
    name, B, iseed, wseed, scale, rule = case
    sd = R.init_state_dict(wseed, scale)
    d = _diffs(sd, *poses(B, iseed))
    if rule == 'median':
        v = d.flatten().sort().values
        k = v.numel() // 2                  # the threshold half-way between the two middle rows, away from a tie
        bias = (THRESH - float(v[k - 1] + v[k]) / 2, 0.0)
    elif rule == 'one_empty':
        lo, hi = sorted(float(d[h].max()) for h in range(2))
        assert hi - lo > 1.0, (lo, hi)
        bias = (THRESH - (lo + hi) / 2, 0.0)
    elif rule == 'p1_to_1':
        bias = (0.0, 50.0)
    else:
        bias = (0.0, 0.0)
    return wseed, scale, bias


def load(path):
    """The golden file with each case's state_dict and [B,16,4] poses rebuilt from the stored seeds."""
    gold = torch.load(path, weights_only=False)
    for case in gold['cases']:
        seed, scale, bias = case['weights']
        case['state_dict'] = R.init_state_dict(seed, scale, bias)
        case['right'], case['left'] = poses(case['batch'], case['input_seed'])
    return gold


def import_reference():
    from oracle import make_golden_geo_loss
    make_golden_geo_loss.import_reference()
    sys.modules['termcolor'].colored = lambda s, *a, **k: s
    sdf = types.ModuleType('sdf')
    sdf.SDF = object
    sys.modules.setdefault('sdf', sdf)
    from hocontact.postprocess.geo_optimizer_both_batch import GeOptimizer
    from Ver2Code.Discriminator.discrim import Pos2dDiscriminator
    return Pos2dDiscriminator, GeOptimizer.NatureLoss


def main():
    Pos2dDiscriminator, nature_loss = import_reference()
    gold = {'meta': {'source': 'Ver2Code/Discriminator/discrim.py Pos2dDiscriminator and GeOptimizer.NatureLoss '
                               '(hocontact/postprocess/geo_optimizer_both_batch.py:110-132) executed in place on CPU',
                     'torch': torch.__version__,
                     'stored': 'probs [2,B,2] (right, left), mask [2,B], loss, d_right / d_left [B,16,4]; weights and poses rebuilt by load()'},
            'keys': None, 'cases': []}
    for case in CASES:
        name, B, iseed = case[:3]
        wseed, scale, bias = weights(case)
        sd = R.init_state_dict(wseed, scale, bias)
        disc = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).eval()
        gold['keys'] = list(disc.state_dict().keys())
        disc.load_state_dict(sd, strict=True)
        right, left = (t.clone().requires_grad_(True) for t in poses(B, iseed))
        loss = nature_loss(types.SimpleNamespace(disc=disc, device='cpu'), right[:, 1:], left[:, 1:])       # the call of :802
        if loss.requires_grad:
            loss.backward()
        with torch.no_grad():
            probs = torch.stack([disc(right[:, 1:].reshape(B, -1)), disc(left[:, 1:].reshape(B, -1))])
        mask = probs[..., 1] < 1.5 * probs[..., 0]
        grads = [t.grad.clone() if t.grad is not None else torch.zeros_like(t) for t in (right, left)]
        assert float(grads[0][:, 0].abs().max()) == 0.0 and float(grads[1][:, 0].abs().max()) == 0.0
        _, _, _, info = R.weighted_case(sd, right, left)
        flags = R.row_flags(info)
        n = mask.sum(1).tolist()
        if name == 'mixed':
            assert all(0 < k < B for k in n), n
        elif name == 'one_empty':
            assert sorted(k == 0 for k in n) == [False, True], n
        elif name == 'both_empty':
            assert n == [0, 0] and float(loss) == 0.0 and not loss.requires_grad
        elif name == 'saturated':
            p = probs[mask]
            assert bool((p[:, 1] == 0).any()) and bool((p[:, 0] == 1).any()), 'no row reaches the -100 clamp and the 1e-12 floor'
            assert all(0 < k < B for k in n), n
        assert not flags.any(), (name, {k: v.nonzero().tolist() for k, v in info['flags'].items()})
        gold['cases'].append({'name': name, 'batch': B, 'input_seed': iseed, 'weights': (wseed, scale, bias), 'probs': probs.clone(),
                              'mask': mask, 'loss': loss.detach().clone(), 'd_right': grads[0], 'd_left': grads[1]})
        print('%-10s B=%-3d masked %s loss %.6g max|d| %.3g' % (name, B, n, float(loss), max(float(g.abs().max()) for g in grads)))
    torch.save(gold, os.path.join(GOLD, 'nature_synth.pt'))
    print('nature golden: %d cases, %d bytes' % (len(gold['cases']), os.path.getsize(os.path.join(GOLD, 'nature_synth.pt'))))


if __name__ == '__main__':
    main()
