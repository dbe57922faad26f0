"""Training step plumbing for the hot path: flat parameter / gradient buffers, fused AdamW, one NCCL all-reduce,
whole-step CUDA-graph capture.

Mirrors what the reference's trainer does around `network(imgTensors)` (core/lijun_trainer.py:262-313: forward,
calc_loss_GCN, zero_grad / backward / AdamW step, DDP gradient all-reduce) with H100-first mechanics:
  * every trainable tensor is a view of ONE flat fp32 buffer, gradients likewise -> zero_grad is one memset,
    the data-parallel exchange is ONE all-reduce of the flat gradient (155 MB) over NVLink, AdamW is one kernel;
  * BatchNorm statistics stay per rank (the reference uses no SyncBN, SURVEY.md 2.1);
  * the whole step (forward, loss, backward, optimizer) is captured into a CUDA graph and replayed.
"""
import torch
import torch.distributed as dist

from ._lib import call
from . import ops


def lr_at_epoch(epoch, base_lr, init_lr=None, warm_up_epoch=3, gamma=0.1, step_size=80, min_thres=0.05):
    """Learning rate of the reference's `StepLR_withWarmUp` (utils/lr_sc.py:159-175) at `epoch` (= the scheduler's `last_epoch`):
    linear warm-up from init_lr (the trainer passes 1e-2 * LR, core/lijun_trainer.py:147-153) over `warm_up_epoch` epochs, then
    base_lr * max(gamma ** ((epoch - warm_up) // step_size), min_thres)."""
    if init_lr is None:
        init_lr = 1e-2 * base_lr
    if epoch < warm_up_epoch:
        return init_lr + (base_lr - init_lr) * (epoch / warm_up_epoch)
    return base_lr * max(gamma ** ((epoch - warm_up_epoch) // step_size), min_thres)


class FlatParams:
    """Re-home the given parameters (and their .grad) into flat contiguous buffers, preserving each tensor's strides
    (conv weights stay channels_last)."""

    def __init__(self, params, groups=()):
        """groups: tuples of parameters that must lie back to back in the flat buffers (same for their gradients), in the given order --
        e.g. (w_qs.weight, w_ks.weight, w_vs.weight), which the fused Q/K/V projection reads as ONE [3d, d] matrix (ops.AttnProjFn)."""
        params = [p for p in params if p.requires_grad]
        assert params, 'no trainable parameters'
        present = {id(p) for p in params}
        member = {}
        for g in groups:
            if all(id(p) in present for p in g) and all(p.numel() % 4 == 0 for p in g):
                for p in g:
                    member[id(p)] = g
        ordered, placed = [], set()
        for p in params:
            if id(p) in placed:
                continue
            for q in member.get(id(p), (p,)):
                ordered.append(q); placed.add(id(q))
        params = ordered
        dev = params[0].device
        self.params = params
        total = 0
        offs = []
        for p in params:
            offs.append(total)
            total += (p.numel() + 3) // 4 * 4        # keep every tensor 16-byte aligned
        self.numel = total
        self.offsets = offs
        self.flat = torch.zeros(total, device=dev, dtype=torch.float32)
        self.grad = torch.zeros(total, device=dev, dtype=torch.float32)
        self.exp_avg = torch.zeros(total, device=dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(total, device=dev, dtype=torch.float32)
        self.step_count = 0
        for p, off in zip(params, offs):
            n = p.numel()
            assert p.is_contiguous() or (p.dim() == 4 and p.permute(0, 2, 3, 1).is_contiguous()), 'dense tensors only'
            view = torch.as_strided(self.flat, p.shape, p.stride(), off)
            view.copy_(p.data)
            p.data = view
            p.grad = torch.as_strided(self.grad, p.shape, p.stride(), off)
            if p.is_cuda:
                ops.register_grad_target(p, p.grad)   # backward kernels accumulate straight into the flat gradient

    def zero_grad(self):
        self.grad.zero_()

    def all_reduce(self, group=None):
        """The single gradient exchange of a data-parallel step (sum; the mean is folded into adamw_step)."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.grad, op=dist.ReduceOp.SUM, group=group)
            return dist.get_world_size(group)
        return 1

    # -- optimizer state in torch.optim.AdamW's own layout, so the reference's optimizer resume (MODEL_PARAM.OPTIM_PATH,
    #    core/lijun_trainer.py:131-144) round-trips: state[i] = {'step', 'exp_avg', 'exp_avg_sq'} per parameter in `self.params` order
    def _views(self, flat):
        return [torch.as_strided(flat, p.shape, p.stride(), off) for p, off in zip(self.params, self.offsets)]

    def state_dict(self, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, index=None, n_params=None):
        """index: {id(parameter): position in the optimizer's parameter list} (default: position in this buffer).  TrainStep passes the
        position among the model's trainable parameters, i.e. the numbering `torch.optim.AdamW(network.parameters())` uses in the
        reference trainer; parameters that never receive a gradient have no state there either."""
        index = index or {id(p): i for i, p in enumerate(self.params)}
        state = {}
        for p, m, v in zip(self.params, self._views(self.exp_avg), self._views(self.exp_avg_sq)):
            state[index[id(p)]] = {'step': torch.tensor(float(self.step_count)), 'exp_avg': m.detach().clone().contiguous(),
                                   'exp_avg_sq': v.detach().clone().contiguous()}
        group = {'lr': lr, 'betas': tuple(betas), 'eps': eps, 'weight_decay': weight_decay, 'amsgrad': False, 'maximize': False,
                 'foreach': None, 'capturable': False, 'differentiable': False, 'fused': None,
                 'params': list(range(n_params if n_params is not None else len(self.params)))}
        return {'state': state, 'param_groups': [group]}

    def load_state_dict(self, sd, index=None):
        state = sd['state']
        index = index or {id(p): i for i, p in enumerate(self.params)}
        steps = set()
        for p, m, v in zip(self.params, self._views(self.exp_avg), self._views(self.exp_avg_sq)):
            i = index[id(p)]
            st = state.get(i, state.get(str(i)))
            if st is None:
                continue
            m.copy_(st['exp_avg']); v.copy_(st['exp_avg_sq'])
            steps.add(int(float(st['step'])))
        assert len(steps) <= 1, 'per-parameter step counts differ (%s): the fused AdamW kernel keeps one' % sorted(steps)
        self.step_count = steps.pop() if steps else 0

    def snapshot(self):
        """Copy of everything an optimizer step mutates (used to undo the warm-up / dry-run steps of TrainStep)."""
        return (self.flat.clone(), self.exp_avg.clone(), self.exp_avg_sq.clone(), self.step_count)

    def restore(self, snap):
        self.flat.copy_(snap[0]); self.exp_avg.copy_(snap[1]); self.exp_avg_sq.copy_(snap[2]); self.step_count = snap[3]
        self.grad.zero_()

    def adamw_step(self, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, grad_scale=1.0, step=None):
        """torch.optim.AdamW semantics (decoupled weight decay) as one kernel over the flat buffer."""
        if step is None:
            self.step_count += 1
            step = self.step_count
        call('rih_adamw_step', self.flat.data_ptr(), self.grad.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
             self.numel, float(lr), float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step), float(grad_scale),
             torch.cuda.current_stream().cuda_stream)


def _mutable_state(model, device):
    """Everything besides parameters that a training-mode forward mutates: module buffers (BatchNorm running statistics,
    num_batches_tracked) and the device-resident dropout seed."""
    bufs = [b for b in model.buffers()]
    ops.seed_state.ptr(device)
    key = device.index if device.index is not None else torch.cuda.current_device()
    return bufs, ops.seed_state.tensors[key]


class _Preserve:
    """Context manager: snapshot the model's buffers + the dropout seed (+ optionally the flat optimizer state) on entry, restore on exit,
    so dry runs / warm-up steps leave a loaded checkpoint bit-identical."""

    def __init__(self, model, device, flatp=None):
        self.bufs, self.seed = _mutable_state(model, device)
        self.flatp = flatp

    def __enter__(self):
        self.saved = [b.detach().clone() for b in self.bufs]
        self.saved_seed = self.seed.clone()
        self.snap = self.flatp.snapshot() if self.flatp is not None else None
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        with torch.no_grad():
            for b, s in zip(self.bufs, self.saved):
                b.copy_(s)
            self.seed.copy_(self.saved_seed)
        if self.snap is not None:
            self.flatp.restore(self.snap)
        return False


def trainable_used_params(model, loss_fn, img):
    """Parameters that actually receive a gradient (the reference needs find_unused_parameters=True because 63 tensors
    never do, SURVEY.md 2.1): found with one dry-run backward.  The dry run leaves no trace: BatchNorm running statistics and the
    dropout seed are restored afterwards."""
    for p in model.parameters():
        p.grad = None
    with _Preserve(model, img.device):
        out = model(img)
        loss_fn(out).backward()
    used = [p for p in model.parameters() if p.requires_grad and p.grad is not None]
    for p in model.parameters():
        p.grad = None
    return used


class TrainStep:
    """One data-parallel training step: forward -> loss -> backward -> (all-reduce) -> AdamW, optionally CUDA-graphed."""

    def __init__(self, model, loss_fn, example_img, lr=3e-4, weight_decay=1e-2, use_graph=True, group=None, labels=None):
        """labels: optional dict of DEVICE tensors that `loss_fn` reads (the batch's ground truth).  They are the step's static label
        buffers: `__call__(img, labels)` / `prefetch(img, labels)` copy each new batch's labels into them, like the image."""
        self.model, self.loss_fn, self.group = model, loss_fn, group
        self.labels = labels or {}
        self.lr, self.wd = lr, weight_decay
        self.base_lr = lr
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        groups = [g for m in model.modules() if hasattr(m, 'fused_param_groups') for g in m.fused_param_groups()]
        self.flatp = FlatParams(trainable_used_params(model, loss_fn, example_img), groups=groups)
        if self.world > 1:
            # DDP broadcasts rank 0's parameters and buffers at construction (core/lijun_trainer.py:122-127); without it any per-rank
            # difference at init (seed, a checkpoint loaded on one rank) would persist under identical averaged gradients
            dist.broadcast(self.flatp.flat, 0, group=group)
            for t in list(model.buffers()) + [p.data for p in model.parameters() if not any(p is q for q in self.flatp.params)]:
                if t.is_cuda and t.numel() > 0:
                    dist.broadcast(t, 0, group=group)
        try:      # the two decoder streams make some AccumulateGrad nodes run on a side stream; torch's advisory warning is expected here
            torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)
        except Exception:
            pass
        self._setup_overlap()
        self.static_img = example_img.clone()
        self.graph = None
        self.loss = None
        self.use_graph = use_graph

    # ---- gradient all-reduce overlapped with backward (SURVEY 5 / 8e; DDP's bucketed reducer does this in the reference, core/lijun_trainer.py:122-127)
    def _setup_overlap(self):
        """Split the flat gradient into segments that finish one after the other during backward and all-reduce each on a communication
        stream as soon as it is complete, instead of one exposed 155 MB all-reduce after backward.  Segments follow the model's backward
        markers (ops.backward_marker): [everything after the ResNet trunk: aux decoders, mid, token decoder] -> layer4 -> layer3 -> the rest.
        Models without markers (HRNet, ...) fall back to one all-reduce at the end of backward (still inside the captured step).
        `RIH_OVERLAP_ALLREDUCE=0` restores the single all-reduce issued after the graph replay."""
        import os
        self.overlap = self.world > 1 and os.environ.get('RIH_OVERLAP_ALLREDUCE', '1') != '0'
        self._segments, self._comm = {}, None
        if not self.overlap:
            return
        self._comm = torch.cuda.Stream(device=self.flatp.flat.device)
        names = {id(p): k for k, p in self.model.named_parameters()}
        first = {}                      # prefix -> first offset of a parameter with that prefix in the flat buffer
        for p, off in zip(self.flatp.params, self.flatp.offsets):
            k = names.get(id(p), '')
            for pre in ('encoder.resnet.layer3.', 'encoder.resnet.layer4.'):
                if k.startswith(pre):
                    first[pre] = min(first.get(pre, off), off)
            if not k.startswith('encoder.resnet.'):
                first['rest'] = min(first.get('rest', off), off)
        n = self.flatp.numel
        if all(k in first for k in ('encoder.resnet.layer3.', 'encoder.resnet.layer4.', 'rest')) and \
                first['encoder.resnet.layer3.'] < first['encoder.resnet.layer4.'] < first['rest']:
            l3, l4, rest = first['encoder.resnet.layer3.'], first['encoder.resnet.layer4.'], first['rest']
            # marker name -> (lo, hi): the gradient of layer k's OUTPUT is complete when everything after layer k has been back-propagated
            self._segments = {'encoder.resnet.layer4': (rest, n), 'encoder.resnet.layer3': (l4, rest), 'encoder.resnet.layer2': (l3, l4)}
        self._pending = None

    def _reduce_range(self, lo, hi):
        """All-reduce grad[lo:hi] on the communication stream, ordered after every stream of the step that may still be writing into it."""
        if hi <= lo:
            return
        dev = self.flatp.flat.device
        self._comm.wait_stream(torch.cuda.current_stream(dev))
        for st in list(ops.STEP_STREAMS.values()):
            self._comm.wait_stream(st)
        with torch.cuda.stream(self._comm):
            dist.all_reduce(self.flatp.grad[lo:hi], op=dist.ReduceOp.SUM, group=self.group)

    def _on_marker(self, name):
        seg = self._segments.get(name)
        if seg is None or self._pending is None or name in self._pending['done']:
            return
        self._pending['done'].add(name)
        self._pending['ranges'].append(seg)
        self._reduce_range(*seg)

    def _finish_reduce(self):
        """After backward: all-reduce whatever no marker covered (layer1-2 + stem, or everything), then join the communication stream."""
        done = sorted(self._pending['ranges'])
        lo = 0
        for a, b in done + [(self.flatp.numel, self.flatp.numel)]:
            self._reduce_range(lo, a)
            lo = max(lo, b)
        torch.cuda.current_stream(self.flatp.flat.device).wait_stream(self._comm)
        self._pending = None

    def _optim_index(self):
        train = [p for p in self.model.parameters() if p.requires_grad]
        return {id(p): i for i, p in enumerate(train)}, len(train)

    def optimizer_state_dict(self):
        """AdamW state in torch.optim.AdamW's layout, numbered like `torch.optim.AdamW(network.parameters())` numbers the model's trainable
        parameters (the reference trainer's optimizer, core/lijun_trainer.py:131-144), so MODEL_PARAM.OPTIM_PATH checkpoints round-trip."""
        index, n = self._optim_index()
        return self.flatp.state_dict(lr=self.lr, weight_decay=self.wd, index=index, n_params=n)

    def load_optimizer_state_dict(self, sd):
        self.flatp.load_state_dict(sd, index=self._optim_index()[0])

    def set_epoch(self, epoch, cfg=None, **kw):
        """Learning-rate schedule of the reference trainer (SURVEY 8 f3): the fused AdamW kernel takes the rate as a launch argument
        (it runs outside the captured graph), so the schedule costs nothing per step."""
        if cfg is not None:
            kw = dict(warm_up_epoch=cfg.TRAIN.warm_up, gamma=cfg.TRAIN.lr_decay_gamma, step_size=cfg.TRAIN.lr_decay_step, **kw)
            self.base_lr = cfg.TRAIN.LR
        self.lr = lr_at_epoch(epoch, getattr(self, 'base_lr', self.lr), **kw)
        return self.lr

    def _step_body(self, reduce=True):
        self.flatp.zero_grad()
        do_overlap = self.overlap and reduce and not getattr(self, 'skip_all_reduce', False)
        if do_overlap:
            self._pending = {'done': set(), 'ranges': []}
            ops.MARKER_CALLBACK[0] = self._on_marker
        try:
            out = self.model(self.static_img)
            loss = self.loss_fn(out)
            loss.backward()
            if do_overlap:
                self._finish_reduce()
        finally:
            ops.MARKER_CALLBACK[0] = None
        return loss.detach()

    def _eager_no_opt(self):
        """Forward + loss + backward, eager, no collective and no optimizer step (measurement passes: parameters stay where they are)."""
        return self._step_body(reduce=False)

    def _eager(self):
        loss = self._step_body()
        if not self.overlap:
            self.flatp.all_reduce(self.group)
        self.flatp.adamw_step(self.lr, weight_decay=self.wd, grad_scale=1.0 / self.world)
        return loss

    def capture(self, warmup=3, reduce=True):
        """Warm up forward+backward on a side stream, then capture them into one CUDA graph; the NCCL all-reduce and the fused AdamW
        kernel run after each replay on the same stream.  Neither the warm-up passes nor the capture pass (which executes nothing, but
        the warm-up does) leave a trace: parameters, Adam moments, step count, BatchNorm running statistics and the dropout seed are
        snapshotted before and restored after, so resuming from a checkpoint through TrainStep does not perturb the loaded model."""
        with _Preserve(self.model, self.static_img.device, self.flatp):
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(warmup):
                    self._step_body(reduce)    # forward + backward (+ the overlapped gradient all-reduce when world > 1): no optimizer step
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.loss = self._step_body(reduce)
        return self

    def prefetch(self, img_host, labels_host=None):
        """Start the host -> device copy of the NEXT step's batch (pinned host tensors: the image and, optionally, its labels) on a copy
        stream, overlapping the current step; the next `__call__()` (without arguments) moves it into the graph's static inputs with
        device-to-device copies.  This is the input double-buffering a DataLoader with `pin_memory` + `non_blocking` gives the reference
        trainer (core/lijun_trainer.py:246-262: imgTensors and every label tensor go `.to(rank)` each iteration)."""
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.static_img.device)
            self._stage = torch.empty_like(self.static_img)
            self._stage_labels = {k: torch.empty_like(v) for k, v in self.labels.items()}
            self._stage_free = None
        if self._stage_free is not None:
            self._copy_stream.wait_event(self._stage_free)      # the previous stage -> static copy must have consumed the buffers
        with torch.cuda.stream(self._copy_stream):
            self._stage.copy_(img_host, non_blocking=True)
            for k, v in (labels_host or {}).items():
                self._stage_labels[k].copy_(v, non_blocking=True)
        self._staged = True
        self._staged_keys = tuple((labels_host or {}).keys())

    def __call__(self, img=None, labels=None):
        if img is not None:
            self.static_img.copy_(img, non_blocking=True)
            for k, v in (labels or {}).items():
                self.labels[k].copy_(v, non_blocking=True)
        elif getattr(self, '_staged', False):
            cur = torch.cuda.current_stream()
            cur.wait_stream(self._copy_stream)
            self.static_img.copy_(self._stage, non_blocking=True)
            for k in self._staged_keys:
                self.labels[k].copy_(self._stage_labels[k], non_blocking=True)
            self._stage_free = torch.cuda.Event()
            self._stage_free.record(cur)
            self._staged = False
        if self.graph is None:
            return self._eager()
        self.graph.replay()
        if not self.overlap and not getattr(self, 'skip_all_reduce', False):   # overlapped mode: the all-reduce segments are inside the captured step
            self.flatp.all_reduce(self.group)
        self.flatp.adamw_step(self.lr, weight_decay=self.wd, grad_scale=1.0 / self.world)
        return self.loss
