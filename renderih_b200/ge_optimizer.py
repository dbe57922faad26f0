"""The two-hand pose optimiser on the GPU: a drop-in for `GeOptimizer` (pose_data_optimize/hocontact/postprocess/
geo_optimizer_both_batch.py:22-930) in the mode its caller runs, mode='both' (batch_optimize_mocap_origin.py:403-416, 706-737).

    hoptim = GeOptimizer('cuda', lr=1e-2, n_iter=100, mano_root=..., anchor_path=..., lambda_contact_loss=..., mode='both')
    hoptim.set_opt_val(**opt_val_kwargs)            # the caller's keyword arguments, unchanged
    out_dict = hoptim.optimize()                    # optimized_hand_pose / _hand_tsl / _sub_hand_pose / _sub_hand_tsl, CPU tensors

One iteration is the reference's loss_fn + backward + Adam step + scheduler step (:872-880): the pose assembly (csrc/ge_optim.cu), both
renderih_b200.manopth.ManoLayer hands, the translation adds, renderih_b200.geo_loss.HandPriorLoss, renderih_b200.sdf.NewLoss,
F.normalize and renderih_b200.nature.NatureLoss, then torch.optim.Adam and ReduceLROnPlateau as kernels whose learning rates, step count
and scheduler state live in device memory.  optimize() captures that iteration in one CUDA graph and replays it n_iter times without
synchronising with the host, then synchronises once to build out_dict.  The graph is captured on the first call after the batch size or
the gt / variable joint split changes; at most one graph is alive.  Everything else set_opt_val changes is copied into buffers this object
owns, and the loss weights are refreshed from coef_val on every call, so the caller's passes (new data, new coef_val / n_iter) replay
the same graph.

Conventions reproduced:

* Variables (set_opt_val, :255-354, :406-432): hand_tsl_init [B,3], obj_tsl_init [B,3] and the init rows of hand_pose / obj_pose
  ([B,n,4] each, at their joint indices) are optimised; the gt rows and the shape ([B,20], given as gt or init: constant either way,
  :239-248, :530) are not.  Adam param groups in the reference's order: hand_tsl and obj_tsl at 0.01 lr, the right and left variable
  joints at lr; torch.optim.Adam's defaults betas (0.9, 0.999), eps 1e-8, no weight decay.  ReduceLROnPlateau(mode='min', factor=0.5,
  patience=20, min_lr=1e-5) with threshold 1e-4 'rel', cooldown 0, eps 1e-8, stepped on each iteration's pre-step total.  The bias
  corrections beta ** t come from a host table of Python doubles, as torch forms them.
* Both optimiser and scheduler are rebuilt by set_opt_val (:428-432) and persist across optimize() calls until the next one.
* Assembly (assemble_batch_pose_vec, :480-485): joint j takes the gt or variable row whose index is j; any partition of range(16) works.
  The index lists must not overlap and must cover range(16) (the reference's RuntimeErrors, :283-286, :346-349).
* Total (:805-825): quat_norm + edge + lambda_contact_loss * contact + 0.02 * lambda_repulsion_loss * pen + ergonomics + nature, with
  pen = NewLoss(cat(right, left verts)).mean() and the nature loss of the normalised assembled poses [:, 1:] (:802).  The vertices are the
  centred MANO outputs plus each hand's translation (:539-565).
* out_dict (:922-930): optimized_hand_pose / optimized_sub_hand_pose are the poses assembled at the START of the last iteration -- one
  Adam step behind, since loss_fn stores them (:516-517) before optimizer.step() moves the leaves (:879); optimized_hand_tsl /
  optimized_sub_hand_tsl are the translations after the last step (:923, :929).

Deviations:

* Terms whose weight is commented out or 0 are not computed: pose_reg, pose_consistent, the angle-limit and joint-axis terms (and the
  AxisLayer / angle-axis work feeding them, :713-726), shape_reg (the shape is not optimised) and 0.0 * hand_tsl_loss.  Their gradient
  contribution is an exact +-0 for finite inputs.
* There is no per-iteration print (:803) and no loss dict (:846-858); loss_history() and lr_history() return the totals and learning
  rates of the last optimize() call instead.
* Terms are 0-dim where the reference returns shape [1].

Not supported, each NotImplementedError: mode other than 'both'; optimising the shape (neither hand_shape_gt nor hand_shape_init: the left
hand slices an empty [1,10] tensor, :527, :543); hand_tsl_gt or neither hand_tsl argument (vec_sub_tsl is left undefined, :536, :544, or
a [3] translation is broadcast as [3,1] against [B,21,3], :267, :556); a hand or obj pose without both gt and init (a 2-D init is
concatenated with a 3-D gt, or the normalised pose stays undefined, :293-340, :802); runtime_vis other than None / 9527 (there is no open3d
viewer); progress=True.  CPU tensors raise RuntimeError, non-float32 poses / translations / shapes TypeError, wrong shapes ValueError.
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

from ._lib import call
from .geo_loss import HandPriorLoss
from .manopth import ManoLayer
from .nature import NatureLoss, Pos2dDiscriminator
from .sdf import NewLoss

BETAS = (0.9, 0.999)
ADAM_EPS = 1e-8
# ReduceLROnPlateau(min_lr=1e-5, mode="min", factor=0.5, patience=20) with torch's defaults threshold=1e-4 ('rel'), cooldown=0, eps=1e-8
PLATEAU = {'factor': 0.5, 'patience': 20, 'min_lr': 1e-5, 'threshold': 1e-4, 'eps': 1e-8}
N_GROUPS = 4                  # hand_tsl, obj_tsl, hand pose, obj pose (:414-423)
DISCRIM_PATH = os.path.join('Ver2Code', 'Discriminator', 'discrim.pth')
_MIN_CAPACITY = 1024          # initial length of the loss history and of the beta-power table


def beta_powers(beta, n):
    """[n + 1] float64: beta ** t for t = 0..n, each a Python double as torch.optim.Adam forms it (`beta1 ** step`, step a float)."""
    return torch.tensor([beta ** float(t) for t in range(n + 1)], dtype=torch.float64)


def plateau_step(state, loss):
    """The rules rih_ge_plateau_step applies, on the host: state = {'best', 'num_bad', 'lr': [..]} (floats) is updated in place for one
    scheduler step on `loss` (a float32 value widened to double)."""
    a = float(loss)
    if a < state['best'] * (1.0 - PLATEAU['threshold']):
        state['best'], state['num_bad'] = a, 0
    else:
        state['num_bad'] += 1
    if state['num_bad'] > PLATEAU['patience']:
        for i, old in enumerate(state['lr']):
            new = max(old * PLATEAU['factor'], PLATEAU['min_lr'])
            if old - new > PLATEAU['eps']:
                state['lr'][i] = new
        state['num_bad'] = 0
    return state


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _tensor(name, t, shape, device):
    """Validate a float32 CUDA tensor of the given shape (None entries: any size)."""
    if not isinstance(t, torch.Tensor):
        raise TypeError('GeOptimizer: %s must be a tensor, got %s' % (name, type(t).__name__))
    if not t.is_cuda:
        raise RuntimeError('GeOptimizer: %s must be a CUDA tensor (there is no CPU path)' % name)
    if t.dtype != torch.float32:
        raise TypeError('GeOptimizer: %s must be float32, got %s' % (name, t.dtype))
    if t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)):
        raise ValueError('GeOptimizer: %s must be %s, got %s' % (name, list(shape), tuple(t.shape)))
    if t.device != device:
        raise RuntimeError('GeOptimizer: %s is on %s, the optimiser on %s' % (name, t.device, device))
    return t


def _split(name, gt, init):
    """The (idx, val) pairs of a hand's gt and init joints -> (gt_idx, gt_val, var_idx, var_val) with the reference's checks."""
    if gt is None or init is None:
        raise NotImplementedError('GeOptimizer: %s_gt and %s_init must both be given: without one of them the reference concatenates a 2-D '
                                  'init with a 3-D gt or leaves the normalised pose undefined (geo_optimizer_both_batch.py:293-340, :802)'
                                  % (name, name))
    (gi, gv), (vi, vv) = gt, init
    gi, vi = [int(i) for i in gi], [int(i) for i in vi]
    if len(set(gi).intersection(set(vi))) > 0:
        raise RuntimeError('repeat %s gt & init provided' % name)
    if set(gi).union(set(vi)) != set(range(16)):
        raise RuntimeError('%s: not enough gt & init' % name)
    if len(gi) + len(vi) != 16:
        raise ValueError('GeOptimizer: %s gt and init indices repeat a joint: %s, %s' % (name, gi, vi))
    return gi, gv, vi, vv


class _AssembleFn(torch.autograd.Function):
    """rih_ge_assemble_fwd / _bwd: flat variables -> (right pose, left pose [B,16,4], hand_tsl, obj_tsl [B,3])."""

    @staticmethod
    def forward(ctx, opt, flat):
        B, dev = opt._B, flat.device
        out = [torch.empty(B, 16, 4, device=dev), torch.empty(B, 16, 4, device=dev), torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev)]
        call('rih_ge_assemble_fwd', flat.data_ptr(), opt._gt[0].data_ptr(), opt._gt[1].data_ptr(), opt._tables.data_ptr(), B, opt._n_var[0],
             opt._n_var[1], *[t.data_ptr() for t in out], _stream(flat))
        ctx.opt = opt
        ctx.set_materialize_grads(False)
        return tuple(out)

    @staticmethod
    def backward(ctx, d_pr, d_pl, d_tr, d_tl):
        opt = ctx.opt
        g = [None if t is None else t.float().contiguous() for t in (d_pr, d_pl, d_tr, d_tl)]
        d_flat = torch.empty_like(opt._flat)
        call('rih_ge_assemble_bwd', *[_ptr(t) for t in g], opt._tables[32:].data_ptr(), opt._B, opt._n_var[0], opt._n_var[1], d_flat.data_ptr(),
             _stream(d_flat))
        return None, d_flat


class GeOptimizer:
    """geo_optimizer_both_batch.GeOptimizer with the reference's constructor (see the module docstring).  Besides the reference's
    arguments: discrim, the discriminator weights (a path, default the reference's relative Ver2Code/Discriminator/discrim.pth, or a
    state_dict); sdf_faces / sdf_part_vert, passed to NewLoss; anchor_face_vert_idx / anchor_weight, the anchor tables instead of
    anchor_path's files.  mano_root may also be {'right': mano dict, 'left': mano dict}."""

    def __init__(self, device, lr=1e-2, n_iter=2500, verbose=False, mano_root='assets/mano', anchor_path='assets/anchor', fhb=False,
                 load_fhb_path='assets/mano/fhb_skel_centeridx9.pkl', compensate_tsl=False, lambda_contact_loss=10.0, lambda_repulsion_loss=0.5,
                 repulsion_query=0.030, repulsion_threshold=0.080, mode='both', discrim=None, sdf_faces=None, sdf_part_vert=None,
                 anchor_face_vert_idx=None, anchor_weight=None):
        if mode != 'both':
            raise NotImplementedError("GeOptimizer runs mode='both' only: the single-hand branch of loss_fn reads an undefined anchor_pos "
                                      '(geo_optimizer_both_batch.py:640-645)')
        self.mode = mode
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError('GeOptimizer: a CUDA device is required (there is no CPU path)')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.lr = lr
        self.n_iter = n_iter
        self.verbose = verbose
        self.compensate_tsl = compensate_tsl
        self.runtime_vis = None
        self.coef_val = {'lambda_contact_loss': lambda_contact_loss, 'lambda_repulsion_loss': lambda_repulsion_loss,
                         'repulsion_query': repulsion_query, 'repulsion_threshold': repulsion_threshold}
        quat = dict(joint_rot_mode='quat', root_rot_mode='quat', use_pca=False, center_idx=0, flat_hand_mean=True, return_transf=True,
                    return_full_pose=True)
        roots = mano_root if isinstance(mano_root, dict) else {'right': mano_root, 'left': mano_root}
        self.mano_layer = ManoLayer(mano_root=roots['right'], side='right', **quat).to(self.device)
        self.sub_mano_layer = ManoLayer(mano_root=roots['left'], side='left', **quat).to(self.device)
        with torch.cuda.device(self.device):
            self.prior = HandPriorLoss(self.mano_layer, self.sub_mano_layer, anchor_root=anchor_path, face_vert_idx=anchor_face_vert_idx,
                                       anchor_weight=anchor_weight)
        self.anti_penetration_loss_fun = NewLoss(faces=sdf_faces, part_vert=sdf_part_vert, device=self.device)
        self.disc = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).to(self.device).eval()
        sd = torch.load(DISCRIM_PATH if discrim is None else discrim, map_location=self.device) if not isinstance(discrim, dict) else discrim
        self.disc.load_state_dict(sd, strict=True)
        self.nature = NatureLoss(self.disc)
        self.use_graph = True          # False: run the same iteration eagerly (the captured graph's reference)
        self.optimizing = False
        self._key = None               # (B, split, contact shape) the buffers are allocated for
        self._graph = self._graph_out = None
        self._last = None
        self._steps = 0                # Adam steps taken since set_opt_val (known on the host: every call runs n_iter of them)
        self._n_last = 0
        self._cap_pow = self._cap_hist = 0

    # ------------------------------------------------------------------------------------------------------------------ set_opt_val
    def set_opt_val(self, vertex_contact, contact_region, anchor_id, anchor_elasti, anchor_padding_mask, hand_region_assignment=None,
                    hand_palm_vertex_mask=None, hand_shape_gt=None, hand_tsl_gt=None, hand_pose_gt=None, hand_shape_init=None, hand_tsl_init=None,
                    hand_pose_init=None, hand_compensate_root=None, runtime_vis=None, obj_anchors=None, obj_normals=None, obj_tsl_gt=None,
                    obj_pose_gt=None, obj_tsl_init=None, obj_pose_init=None, optimize_it=None, batch_size=None, consistent_mask=None):
        """The reference's set_opt_val (:133-447): validates the arguments, copies them into buffers this object owns and resets the Adam
        moments, the step count and the scheduler.  vertex_contact, contact_region, obj_anchors, obj_normals, optimize_it and
        consistent_mask feed nothing the total uses and are only kept (const_val)."""
        if runtime_vis not in (None, 9527):
            raise NotImplementedError('GeOptimizer: runtime_vis must be None or 9527 (there is no open3d viewer)')
        if hand_shape_gt is not None and hand_shape_init is not None:
            raise RuntimeError('both hand_shape gt and init are provided')
        if hand_shape_gt is None and hand_shape_init is None:
            raise NotImplementedError('GeOptimizer: optimising the shape is not supported: the reference slices an empty [1,10] tensor for '
                                      'the left hand (geo_optimizer_both_batch.py:527, :543)')
        if hand_tsl_gt is not None and hand_tsl_init is not None:
            raise RuntimeError('both hand_tsl gt and init are provided')
        if hand_tsl_init is None:
            raise NotImplementedError('GeOptimizer: hand_tsl_init is required: with hand_tsl_gt the reference leaves vec_sub_tsl undefined '
                                      '(:536, :544), without either it broadcasts a [3] translation as [3,1] (:267, :556)')
        if obj_tsl_init is None:
            raise NotImplementedError('GeOptimizer: obj_tsl_init is required in two-hand mode (:273)')
        splits = [_split('hand_pose', hand_pose_gt, hand_pose_init), _split('obj_pose', obj_pose_gt, obj_pose_init)]
        if not isinstance(batch_size, (int, np.integer)) or isinstance(batch_size, bool) or batch_size < 1:
            raise ValueError('GeOptimizer: batch_size must be an int >= 1, got %r' % (batch_size,))
        B, dev = int(batch_size), self.device
        shape = _tensor('hand_shape_gt' if hand_shape_gt is not None else 'hand_shape_init',
                        hand_shape_gt if hand_shape_gt is not None else hand_shape_init, (B, 20), dev)
        tsl = [_tensor('hand_tsl_init', hand_tsl_init, (B, 3), dev), _tensor('obj_tsl_init', obj_tsl_init, (B, 3), dev)]
        vals = []
        for name, (gi, gv, vi, vv) in zip(('hand_pose', 'obj_pose'), splits):
            vals.append((_tensor(name + '_gt values', gv, (B, len(gi), 4), dev), _tensor(name + '_init values', vv, (B, len(vi), 4), dev)))
        anchor_id, anchor_elasti, anchor_padding_mask = (torch.as_tensor(t) for t in (anchor_id, anchor_elasti, anchor_padding_mask))
        for name, t in (('anchor_id', anchor_id), ('anchor_elasti', anchor_elasti), ('anchor_padding_mask', anchor_padding_mask)):
            if not t.is_cuda:
                raise RuntimeError('GeOptimizer: %s must be a CUDA tensor (there is no CPU path)' % name)
        if anchor_id.dim() != 3 or anchor_id.shape[0] != B:
            raise ValueError('GeOptimizer: anchor_id must be [B=%d,A,D], got %s' % (B, tuple(anchor_id.shape)))

        split = tuple((tuple(gi), tuple(vi)) for gi, _, vi, _ in splits)
        key = (B, split, tuple(anchor_id.shape))
        if key != self._key:
            self._allocate(B, split, splits)
            self._key = key
        contacts_before = self.prior._contacts
        self.prior.set_contacts(anchor_id, anchor_elasti, anchor_padding_mask)
        if contacts_before is not None and self.prior._contacts is not contacts_before:
            self._graph = self._graph_out = None          # new contact buffers: the graph read the old ones
        with torch.no_grad():
            self._shape.copy_(shape)
            parts = [tsl[0].reshape(-1), tsl[1].reshape(-1), vals[0][1].reshape(-1), vals[1][1].reshape(-1)]
            off = 0
            for p in parts:
                self._flat[off:off + p.numel()].copy_(p)
                off += p.numel()
            for h in range(2):
                self._gt[h].copy_(vals[h][0])
            self._m.zero_()
            self._v.zero_()
            lr = [0.01 * self.lr, 0.01 * self.lr, 1 * self.lr, 1 * self.lr]
            self._dstate.copy_(torch.tensor([float('inf')] + lr, dtype=torch.float64))
            self._istate.zero_()
        self._steps = 0
        self._last = None
        self._n_last = 0
        self.optimizing = True
        self.runtime_vis = runtime_vis
        self.const_val = {'batch_size': B, 'optimize_it': optimize_it, 'consistent_mask': consistent_mask, 'vertex_contact': vertex_contact,
                          'contact_region': contact_region, 'full_obj_verts_3d': obj_anchors, 'full_obj_normals': obj_normals,
                          'hand_pose_gt_idx': list(split[0][0]), 'hand_pose_var_idx': list(split[0][1]),
                          'obj_pose_gt_idx': list(split[1][0]), 'obj_pose_var_idx': list(split[1][1])}

    def _allocate(self, B, split, splits):
        """Buffers for batch B and this gt / variable split; drops the captured graph."""
        self._graph = self._graph_out = None
        dev = self.device
        self._B = B
        self._n_var = (len(split[0][1]), len(split[1][1]))
        n = 6 * B + 4 * B * sum(self._n_var)
        self._seg = (3 * B, 6 * B, 6 * B + 4 * B * self._n_var[0], n)
        self._flat = torch.zeros(n, device=dev, requires_grad=True)
        self._m, self._v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        self._gt = [torch.zeros(B, 16 - self._n_var[h], 4, device=dev) for h in range(2)]
        self._shape = torch.zeros(B, 20, device=dev)
        tab = np.zeros(64, np.int32)
        for h, (gi, _, vi, _) in enumerate(splits):
            for k, j in enumerate(gi):
                tab[h * 16 + j] = -k - 1
            for k, j in enumerate(vi):
                tab[h * 16 + j] = k
                tab[32 + h * 16 + k] = j
        self._tables = torch.from_numpy(tab).to(dev)
        self._dstate = torch.zeros(1 + N_GROUPS, dtype=torch.float64, device=dev)     # best, lr[4]
        self._istate = torch.zeros(3, dtype=torch.int32, device=dev)                 # step, num_bad, it
        self._w = torch.zeros(2, device=dev)                                          # lambda_contact, 0.02 * lambda_repulsion
        self._cap_pow = self._cap_hist = 0
        self._ensure_capacity(1, 1)

    def _ensure_capacity(self, n_pow, n_hist):
        """Grow the beta-power table / the loss history (doubling) so that they cover n_pow steps and n_hist iterations; growing drops
        the captured graph, which holds their addresses and lengths."""
        if n_pow > self._cap_pow:
            self._cap_pow = max(_MIN_CAPACITY, 1 << (int(n_pow) - 1).bit_length())
            self._pow = torch.stack([beta_powers(b, self._cap_pow) for b in BETAS]).to(self.device)
            self._graph = self._graph_out = None
        if n_hist > self._cap_hist:
            self._cap_hist = max(_MIN_CAPACITY, 1 << (int(n_hist) - 1).bit_length())
            self._hist = torch.zeros(self._cap_hist, device=self.device)
            self._lr_hist = torch.zeros(self._cap_hist, N_GROUPS, dtype=torch.float64, device=self.device)
            self._graph = self._graph_out = None

    # ------------------------------------------------------------------------------------------------------------------ iteration
    def _loss(self):
        """loss_fn's total (:501-825) -> (total, right pose, left pose), differentiable with respect to self._flat."""
        pr, pl, tr, tl = _AssembleFn.apply(self, self._flat)
        vr = self.mano_layer(pr, self._shape[:, :10])[0] + tr.unsqueeze(1)
        vl = self.sub_mano_layer(pl, self._shape[:, 10:])[0] + tl.unsqueeze(1)
        qn, edge, contact, ergo = self.prior(pr, pl, vr, vl)
        pen = self.anti_penetration_loss_fun(torch.cat((vr.unsqueeze(1), vl.unsqueeze(1)), 1)).mean()
        nat = self.nature(F.normalize(pr, dim=-1)[:, 1:], F.normalize(pl, dim=-1)[:, 1:])
        loss = qn + edge + self._w[0] * contact + self._w[1] * pen + ergo + nat
        return loss, pr, pl

    def _iteration(self):
        """One optimiser iteration (:874-880) on the current stream: forward, backward, Adam with the current lrs, then the scheduler on
        this iteration's total."""
        loss, pr, pl = self._loss()
        (grad,) = torch.autograd.grad(loss, [self._flat])
        st = _stream(grad)
        e = self._seg
        d = self._dstate
        call('rih_ge_adam_step', self._flat.data_ptr(), grad.data_ptr(), self._m.data_ptr(), self._v.data_ptr(), e[0], e[1], e[2], e[3], N_GROUPS,
             d[1:].data_ptr(), self._istate.data_ptr(), self._pow[0].data_ptr(), self._pow[1].data_ptr(), self._cap_pow, BETAS[0], BETAS[1],
             ADAM_EPS, st)
        call('rih_ge_plateau_step', loss.data_ptr(), d[1:].data_ptr(), N_GROUPS, d.data_ptr(), self._istate[1:].data_ptr(), self._hist.data_ptr(),
             self._lr_hist.data_ptr(), self._istate[2:].data_ptr(), self._cap_hist, PLATEAU['factor'], PLATEAU['patience'], PLATEAU['min_lr'],
             PLATEAU['threshold'], PLATEAU['eps'], st)
        return loss.detach(), pr.detach(), pl.detach()

    def _capture(self):
        self._graph = self._graph_out = None
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):                      # warm-up without the optimiser step: the state is not touched
                loss = self._loss()[0]
                torch.autograd.grad(loss, [self._flat])
        torch.cuda.current_stream(self.device).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self._iteration()
        self._graph, self._graph_out = graph, out

    def launch(self, n_iter=None):
        """Queue n_iter (default self.n_iter) iterations on the current stream without synchronising with the host (after the first
        capture); optimize() is launch() followed by one synchronisation."""
        if not self.optimizing:
            raise RuntimeError('GeOptimizer: call set_opt_val() before optimize()')
        n = int(self.n_iter if n_iter is None else n_iter)
        if n < 0:
            raise ValueError('GeOptimizer: n_iter must be >= 0, got %d' % n)
        with torch.cuda.device(self.device):
            self._ensure_capacity(self._steps + n, n)
            w = torch.tensor([1 * self.coef_val['lambda_contact_loss'], 0.02 * self.coef_val['lambda_repulsion_loss']],
                             dtype=torch.float32).pin_memory()
            self._w_host = w                               # kept alive until the copy has run (optimize() synchronises)
            self._w.copy_(w, non_blocking=True)
            self._istate[2:].zero_()                       # the loss history restarts
            if n and self.use_graph and self._graph is None:
                self._capture()
            for _ in range(n):
                if self.use_graph:
                    self._graph.replay()
                else:
                    self._last = self._iteration()
            if n and self.use_graph:
                self._last = self._graph_out
        self._steps += n
        self._n_last = n

    def optimize(self, progress=False):
        """Run n_iter iterations and return the reference's out_dict of CPU tensors (:922-930)."""
        if progress:
            raise NotImplementedError('GeOptimizer.optimize: progress bars are not supported')
        self.launch()
        if self._last is None:
            raise RuntimeError('GeOptimizer: no iteration has run since set_opt_val (n_iter = 0)')
        _, pr, pl = self._last
        B = self._B
        flat = self._flat.detach()
        return dict(optimized_hand_pose=pr.cpu(), optimized_hand_tsl=flat[:3 * B].reshape(B, 3).cpu(),
                    optimized_sub_hand_pose=pl.cpu(), optimized_sub_hand_tsl=flat[3 * B:6 * B].reshape(B, 3).cpu())

    def loss_history(self):
        """[n] float32 CPU: the total of every iteration of the last optimize() call (synchronises)."""
        return self._hist[:self._n_last].cpu()

    def lr_history(self):
        """[n,4] float64 CPU: the learning rates of the four param groups after every scheduler step of the last optimize() call."""
        return self._lr_hist[:self._n_last].cpu()

    def adam_state(self):
        """(flat variables, exp_avg, exp_avg_sq, step, lrs) copies, for inspection."""
        return (self._flat.detach().clone(), self._m.clone(), self._v.clone(), int(self._istate[0]), self._dstate[1:].cpu())
