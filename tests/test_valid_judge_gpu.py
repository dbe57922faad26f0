"""rih_valid_judge (csrc/valid_judge.cu) through renderih_b200.valid_judge against the golden file of the unmodified reference
ValidJudger (tests/golden/valid_judge_synth.pt)."""
import os

import numpy as np
import pytest
import torch

from renderih_b200 import assets
from renderih_b200.valid_judge import ValidJudger, get_valid_rate

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'valid_judge_synth.pt')
# radians: float32 rounding of atan2 and of the folded converter products, with angles of up to a few radians
SCORE_TOL = 2e-5


def mano():
    # a fresh dict per judger: manopth.ManoLayer negates the left hand's shapedirs of the dict it is given in place
    return {s: assets.synthetic_mano(0, s) for s in ('right', 'left')}


def test_scores_and_rate_match_golden(capsys):
    g = torch.load(GOLD, weights_only=False)
    judger = ValidJudger(mano(), device='cuda')
    ql, qr = g['quat']['left'].cuda(), g['quat']['right'].cuda()
    score, invalid = judger.scores(ql, qr)
    assert (score[0].cpu() - g['scores']['left']).abs().max() < SCORE_TOL
    assert (score[1].cpu() - g['scores']['right']).abs().max() < SCORE_TOL
    n = g['split']
    for (lo, hi), want in zip(((0, n), (n, ql.shape[0])), g['file_rates']):
        rate = judger.ComputeValidation(ql[lo:hi], qr[lo:hi])
        assert rate.is_cuda and rate.dim() == 0 and rate.dtype == torch.float32
        assert float(rate) == want
    printed = capsys.readouterr().out
    assert printed.count('tensor(') == 2
    assert 0 < int(invalid) < ql.shape[0]


def test_get_valid_rate_golden(tmp_path, capsys):
    g = torch.load(GOLD, weights_only=False)
    n = g['split']
    for name, sl in (('a.npy', slice(0, n)), ('b.npy', slice(n, None))):
        raw = {s: {k: v[sl] for k, v in g['raw'][s].items()} for s in ('right', 'left')}
        np.save(tmp_path / name, raw)
    rate = get_valid_rate(str(tmp_path), mano(), 'cuda')
    assert float(rate) == pytest.approx(float(g['rate']), abs=1e-7)
    assert 'valid rate: ' in capsys.readouterr().out


def test_rejected_inputs():
    judger = ValidJudger(mano(), device='cuda')
    q = torch.zeros(3, 16, 4, device='cuda')
    q[..., 0] = 1
    with pytest.raises(RuntimeError):
        judger.ComputeValidation(q.cpu(), q)
    with pytest.raises(TypeError):
        judger.ComputeValidation(q.double(), q)
    with pytest.raises(ValueError):
        judger.ComputeValidation(q[:, :15], q[:, :15])
    with pytest.raises(ValueError):
        judger.ComputeValidation(q, q[:2])
    with pytest.raises(RuntimeError):
        ValidJudger(mano(), device='cpu')
    assert float(judger.ComputeValidation(q, q)) == 0.0
