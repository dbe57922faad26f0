"""rih_hand_collision_count (csrc/collision.cu) against the numpy oracle (oracle/collision_ref.py): counts must be EQUAL on the same
float64 coordinates.  Also filter_collision_data against the golden file of the unmodified reference, graph capture and rejected inputs."""
import os

import numpy as np
import pytest
import torch

from oracle import collision_ref as C
from renderih_b200 import assets
from renderih_b200.collision import filter_collision_data, hand_collision_count

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'collision_synth.pt')


def _coords(v, t):
    return np.asarray(v, np.float64) + t[:, None]


def _run(va, vb, ta, tb, faces, stats=None):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return hand_collision_count(d(va), d(vb), d(faces), d(ta), d(tb), stats=stats).cpu().numpy()


@pytest.mark.parametrize('regime', ['apart', 'touching', 'deep'])
@pytest.mark.parametrize('B,f64', [(1, False), (37, True), (37, False)])
def test_counts_equal_oracle(regime, B, f64):
    va, vb, ta, tb, faces = C.two_hand_frames(B, regime, seed=B + len(regime), f64=f64)
    want, _ = C.counts(_coords(va, ta), _coords(vb, tb), faces)
    got = _run(va, vb, ta, tb, faces)
    assert got.tolist() == want.tolist()
    if regime == 'apart':
        assert (want == 0).all()
    else:
        assert (want > 0).any()


@pytest.mark.parametrize('f64', [False, True])
def test_counts_equal_oracle_4096(f64):
    """4096 frames: 96 distinct frames of the three regimes, each repeated, in shuffled order; every repeat must give the same count."""
    parts = [C.two_hand_frames(32, r, seed=7 + i, f64=f64) for i, r in enumerate(('apart', 'touching', 'deep'))]
    va, vb, ta, tb = (np.concatenate([p[k] for p in parts]) for k in range(4))
    faces = parts[0][4]
    want, _ = C.counts(_coords(va, ta), _coords(vb, tb), faces)
    idx = np.random.default_rng(0).integers(0, 96, 4096)
    stats = torch.empty(4096, 2, dtype=torch.int64, device='cuda')
    got = _run(va[idx], vb[idx], ta[idx], tb[idx], faces, stats)
    assert got.tolist() == want[idx].tolist()
    s = stats.cpu().numpy()
    assert (s[:, 1] <= s[:, 0]).all() and (s[:, 1] >= got).all()


def test_coincident_hands():
    """The worst case for the broad phase: hand B is hand A, so every face meets itself and its neighbours, coplanar pairs included."""
    va, vb, ta, tb, faces = C.two_hand_frames(3, 'coincident', seed=3)
    want, frag = C.counts(_coords(va, ta), _coords(vb, tb), faces)
    stats = torch.empty(3, 2, dtype=torch.int64, device='cuda')
    got = _run(va, vb, ta, tb, faces, stats)
    assert got.tolist() == want.tolist()
    assert (want >= faces.shape[0]).all()
    assert (stats[:, 0].cpu().numpy() == faces.shape[0] ** 2).all()


def test_golden_vertices():
    """On the reference's own vertices (float32 plus the float64 loc) the kernel reproduces the golden counts."""
    g = torch.load(GOLD, weights_only=False)
    got = hand_collision_count(g['rv'].cuda(), g['lv'].cuda(), g['faces'].cuda(), g['right_loc'].cuda(), g['left_loc'].cuda())
    assert got.cpu().tolist() == g['counts'].tolist()


def _same(a, b):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b)
        for k in a:
            _same(a[k], b[k])
    else:
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize('batch_size', [4096, 5])
def test_filter_collision_data_golden(tmp_path, batch_size, capsys):
    g = torch.load(GOLD, weights_only=False)
    src, dst = tmp_path / 'in.npy', tmp_path / 'out.npy'
    np.save(src, g['raw'])
    mano = {s: assets.synthetic_mano(0, s) for s in ('right', 'left')}
    frac = filter_collision_data(str(src), str(dst), mano_root=mano, batch_size=batch_size)
    assert frac == g['kept_fraction']
    assert capsys.readouterr().out.strip() == str(g['kept_fraction'])
    _same(np.load(dst, allow_pickle=True).item(), g['saved'])


def test_cuda_graph_capture():
    va, vb, ta, tb, faces = C.two_hand_frames(16, 'deep', seed=5)
    want, _ = C.counts(_coords(va, ta), _coords(vb, tb), faces)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    args = [d(va), d(vb), d(faces), d(ta), d(tb)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        hand_collision_count(*args)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = hand_collision_count(*args)
    args[0].copy_(d(vb))                      # the graph reads the buffers at replay: hand A now coincides with hand B
    args[3].copy_(d(tb))
    g.replay()
    torch.cuda.synchronize()
    coinc, _ = C.counts(_coords(vb, tb), _coords(vb, tb), faces)
    assert out.cpu().tolist() == coinc.tolist() and coinc.tolist() != want.tolist()


def test_rejected_inputs():
    va, vb, ta, tb, faces = C.two_hand_frames(2, 'deep', seed=1)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    A, Bv, F, TA = d(va), d(vb), d(faces), d(ta)
    with pytest.raises(RuntimeError):
        hand_collision_count(A.cpu(), Bv, F)
    with pytest.raises(RuntimeError):
        hand_collision_count(A, Bv, F.cpu())
    with pytest.raises(RuntimeError):
        hand_collision_count(A, Bv, F, TA.cpu())
    with pytest.raises(TypeError):
        hand_collision_count(A.half(), Bv.half(), F)
    with pytest.raises(TypeError):
        hand_collision_count(A, Bv.double(), F)
    with pytest.raises(TypeError):
        hand_collision_count(A, Bv, F.float())
    with pytest.raises(TypeError):
        hand_collision_count(A, Bv, F, TA.long())
    with pytest.raises(ValueError):
        hand_collision_count(A, Bv[:1], F)
    with pytest.raises(ValueError):
        hand_collision_count(A[:, :, :2], Bv[:, :, :2], F)
    with pytest.raises(ValueError):
        hand_collision_count(A, Bv, F, TA[:1])
    with pytest.raises(ValueError):
        hand_collision_count(A, Bv, F[:, :2])
    with pytest.raises(ValueError):
        hand_collision_count(A, Bv, torch.cat([F, F]))            # 3072 faces: more than 2048
    big = torch.zeros(2, 1025, 3, device='cuda')
    with pytest.raises(ValueError):
        hand_collision_count(big, big, F)
    for bad in (-1, va.shape[1]):
        f = F.clone()
        f[7, 1] = bad
        with pytest.raises(ValueError):
            hand_collision_count(A, Bv, f)
    with pytest.raises(ValueError):
        hand_collision_count(A, Bv, F, stats=torch.empty(2, 2, device='cuda'))
