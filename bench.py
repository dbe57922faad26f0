#!/usr/bin/env python
"""Benchmark of the RenderIH hot path on H100.

    python bench.py --gpus N --steps K --warmup W            # ours: BASELINE.json configs[2] (the headline metric)
    python bench.py --impl reference ...                     # the UNMODIFIED reference's own CPU path on the host cores
    python bench.py --config forward|mano                    # BASELINE.json configs[1] / configs[0] as extra lines (1 GPU)
    python bench.py --encoder hrnet48 --gpus N               # BASELINE.json configs[4]

Default = images/sec of one training step (forward + calc_loss_GCN + backward + gradient all-reduce + AdamW) at batch 64 per
GPU, 256x256 synthetic images.  Prints ONE JSON line on rank 0 (contract in the task statement):
  value               device-timed images/s with inputs resident in HBM
  e2e                 the same step through the public TrainStep API from pinned HOST buffers (image + labels H2D every step, loss D2H)
  roofline            the kernel CLASS with the largest share of the step (all wgmma GEMM / implicit-GEMM launches), each launch
                      bracketed by CUDA events on its own stream during one eager step; + `step`: whole-step achieved / peak
  roofline_top_kernel the single most expensive launch timed alone (+ DRAM traffic from the committed ncu capture)
  gpu_eager_baseline  the UNMODIFIED reference graph `.cuda()` in eager PyTorch on the same GPU (north_star's comparator) and the
                      resulting `speedup_vs_gpu_eager`
  parity              arithmetic mode of the run, the tolerance the tests assert for it, and the measured MPJPE (mm) of this build
                      against the CPU oracle on a fixed batch
  cpu_baseline        the reference's own CPU path on a bounded sample (kind "reference"; "port" only if the staged reference is absent)
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# SURVEY.md 8(d): FlopCounterMode on the reference (algorithmic 2*MAC FLOPs per image, forward+backward / forward)
FLOPS = {'resnet50': (50.450e9, 17.721e9), 'hrnet48': (168.090e9, 56.201e9),
         'graph': (38.422e9, 13.268e9),     # common/myhand graph variant (ResNet-50 trunk), FlopCounterMode on the reference built on CPU
         'newgraph': (38.464e9, 13.283e9)}  # + ParamRegressor / MANO tail (matmul FLOPs only; the ManoLayer is ~1.2 MFLOP per hand)
# tolerance tests/test_model_gpu.py asserts per arithmetic mode (relative to each output tensor's max magnitude, eval forward)
PARITY_TOL = {'simt': 2e-5, 'ref': 1e-2, 'refrn': 1e-2, 'tf32c': 1e-2, 'tf32rn': 1e-2, 'tf32': 5e-2, 'tf32x3': 1e-3}


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--config', default='train', choices=['train', 'forward', 'mano'],
                    help='train = BASELINE.json configs[2]/[3]/[4] (headline), forward = configs[1] (batch-64 eval forward), mano = configs[0] (ManoLayer only)')
    ap.add_argument('--batch', type=int, default=None, help='images per GPU (default 64; 32 for --encoder hrnet48 = BASELINE.json configs[4])')
    ap.add_argument('--encoder', default='resnet50', choices=['resnet50', 'hrnet48', 'graph', 'newgraph'],
                    help='resnet50 = BASELINE.json configs[2] (the headline metric), hrnet48 = configs[4] (MODEL.ENCODER_TYPE), '
                         'graph = the common/myhand default model variant (SURVEY 8 f1; ResNet-50 trunk, batch 64), '
                         'newgraph = the same with the ParamRegressor + MANO tail, trained with mano_loss_GCN')
    ap.add_argument('--no-graph', action='store_true')
    ap.add_argument('--gemm-mode', default='ref', choices=['ref', 'refrn', 'simt', 'tf32', 'tf32rn', 'tf32c', 'tf32x3'],
                    help="arithmetic of the conv / Linear GEMMs; 'ref' = the reference's own GPU numerics class: TF32 convolutions (as "
                         "cuDNN runs them by default; here truncating TF32 with the 7.05e-4 mean shrinkage compensated in the epilogue, "
                         "measured as accurate as round-to-nearest) + fp32-faithful (3xTF32) nn.Linear GEMMs; 'refrn' = same with "
                         "round-to-nearest TF32 convolutions")
    ap.add_argument('--cpu-batch', type=int, default=4, help='bounded CPU sample size for cpu_baseline / --impl reference')
    ap.add_argument('--skip-cpu-baseline', action='store_true')
    ap.add_argument('--skip-gpu-eager', action='store_true', help='do not time the reference graph in eager PyTorch on this GPU')
    ap.add_argument('--gpu-eager-iters', type=int, default=100, help='timed iterations of the GPU eager baseline (SURVEY 8d: 20 warm-up + 100)')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write what the last step computed as DIR/<name>.npy (float32 / float64, at most 64 MB in all; '
                         'large outputs as a fixed seeded sample) so that two builds can be compared output for output')
    a = ap.parse_args()
    if a.batch is None:
        a.batch = 32 if a.encoder == 'hrnet48' else 64
    return a


DUMP_LIMIT = 64 << 20       # bytes written by --dump-outputs in all


def dump_outputs(path, arrays):
    """arrays: {name: tensor or ndarray}.  Writes DIR/<name>.npy in float32 (float64 stays float64).  An array larger than its share of
    DUMP_LIMIT is replaced by a fixed sample of its flattened elements (the same sorted indices in every run) and named <name>_sample."""
    import numpy as np
    os.makedirs(path, exist_ok=True)
    share = DUMP_LIMIT // max(1, len(arrays))
    for name, a in arrays.items():
        a = a.detach().cpu().numpy() if hasattr(a, 'detach') else np.asarray(a)
        a = a.astype(np.float64 if a.dtype == np.float64 else np.float32)
        if a.nbytes > share:
            idx = np.sort(np.random.default_rng(0).choice(a.size, share // a.itemsize, replace=False))
            a, name = a.reshape(-1)[idx], name + '_sample'
        np.save(os.path.join(path, name + '.npy'), a)


def peaks():
    try:
        with open(os.path.join(ROOT, 'MEASURED_PEAKS.json')) as f:
            p = json.load(f)
        return {'hbm_gbs': p['hbm_gbs'], 'tflops': p['bf16_tflops'], 'tflops_sustained': p.get('bf16_tflops_sustained', p['bf16_tflops']),
                'src': 'measured (MEASURED_PEAKS.json)'}
    except Exception:
        return {'hbm_gbs': 3350.0, 'tflops': 989.0, 'tflops_sustained': 989.0, 'src': 'H100 SXM data sheet (dense BF16, 700 W card), not measured'}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = 'clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,' \
        'clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap'

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.index), '--query-gpu=' + self.Q, '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if not self.proc:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        for r in self.rows:
            f = [x.strip() for x in r.split(',')]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = float(f[1])
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith('active'):
                    reasons.add(n)
        sm.sort()
        return {'sm_mhz': sm[len(sm) // 2] if sm else None, 'sm_max_mhz': mx, 'samples': len(sm), 'reasons': sorted(reasons)}


def metric_name(args):
    """ONE name per configuration for every N (the gradient all-reduce is part of the step; with one rank it has nothing to exchange)."""
    if args.config == 'forward':
        return 'images/sec forward (eval) @batch%d 256x256' % args.batch
    if args.config == 'mano':
        return 'hands/sec ManoLayer forward (FK + LBS)'
    return 'images/sec fwd+bwd @batch%d 256x256 (training step: fwd + %s + bwd + grad all-reduce + AdamW)' % (
        args.batch, 'mano_loss_GCN' if args.encoder == 'newgraph' else 'calc_loss_GCN')


def workload_name(encoder, batch, config='train'):
    enc = {'graph': 'common/myhand graph variant (ResNet50 trunk)',
           'newgraph': 'common/myhand newgraph variant (graph + ParamRegressor + MANO tail, mano_loss_GCN)'}.get(encoder, encoder)
    if config == 'forward':
        return 'BASELINE.json configs[1]: HandNET_GCN %s cfg, batch %d, 256x256, eval mode, random-init weights, synthetic graph/MANO assets' % (enc, batch)
    return 'BASELINE.json configs[%d]: HandNET_GCN %s cfg, batch %d/GPU, 256x256, train mode (batch-stat BN, dropout 0.05), random-init weights, ' \
           'synthetic graph/MANO assets' % (4 if encoder == 'hrnet48' else 2, enc, batch)


def host_cores():
    """CPU threads this process can actually run on: the scheduler affinity mask, capped by the cgroup CPU quota (a container on
    a 128-thread host may own far fewer; oversubscribing torch's intra-op pool there makes the CPU baseline tens of times slower
    than it really is).  This IS the fixed thread policy of both CPU legs: all usable threads, no auto-tuning."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    try:
        with open('/sys/fs/cgroup/cpu.max') as f:
            q, per = f.read().split()[:2]
        if q != 'max':
            n = max(1, min(n, int(float(q) / float(per) + 0.999)))
    except Exception:
        pass
    return n


# ============================================================================ CPU legs (the only places that execute oracle/)
def cpu_reference_time(batch, steps, warmup, encoder='resnet50', forward_only=False, budget_s=150.0):
    """The reference's own CPU path: the UNMODIFIED reference (oracle/_ref/src or /root/reference through oracle/ref_driver.py) --
    models.model.load_model + core.Loss.calc_loss_GCN + torch.optim.AdamW -- on all usable host threads, one warm-up step.
    Falls back to the oracle port (oracle/model_ref.py) only when the reference is not staged or the variant cannot be built on a CPU
    (the common/myhand variants hard-code .cuda()).  -> (seconds per step, cores, steps timed, kind)"""
    cores = host_cores()
    from oracle import ref_driver
    if ref_driver.available() and encoder in ('resnet50', 'hrnet48'):
        r = ref_driver.time_reference('cpu', batch, steps, warmup, encoder_type=encoder, forward_only=forward_only, threads=cores, budget_s=budget_s)
        return r['ms_per_step'] * 1e-3, cores, r['steps'], 'reference'
    t, n = cpu_port_step_time(batch, steps, warmup, budget_s, encoder, cores, forward_only)
    return t, cores, n, 'port'


def cpu_port_step_time(batch, steps, warmup, budget_s, encoder, cores, forward_only=False):
    """The reference algorithm's CPU port (oracle/model_ref.py): forward + calc_loss_GCN + backward + AdamW, fp32."""
    import torch
    from oracle import fixtures, model_ref
    from renderih_b200 import assets as A
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    a = A.synthetic_assets(0)
    cfg = load_cfg()
    if encoder in ('graph', 'newgraph'):
        from renderih_b200 import myhand
        build = myhand.load_graph_model if encoder == 'graph' else myhand.load_new_model
        sd = fixtures.init_state_dict(build(cfg, assets=a, mano_assets={s: A.synthetic_mano(0, s) for s in ('left', 'right')}).state_dict())
    else:
        cfg.MODEL.ENCODER_TYPE = encoder
        sd = fixtures.init_state_dict(load_model(cfg, assets=a).state_dict())
    torch.set_num_threads(cores)
    for k, v in sd.items():
        if v.is_floating_point() and 'running_' not in k and '.mano_' not in k and k not in ('decoder.dense_coor', 'decoder.unsample_layer.weight'):
            v.requires_grad_(True)
    Ap = model_ref.prepare_assets(a)
    if encoder == 'newgraph':
        Ap = fixtures.add_mano_assets(Ap, A.synthetic_mano(0, 'left'), A.synthetic_mano(0, 'right'))
    la = fixtures.make_loss_assets(a, A.synthetic_mano(0, 'left'), A.synthetic_mano(0, 'right'))
    img, labels = fixtures.make_image(batch), fixtures.make_labels(batch)
    opt = torch.optim.AdamW([v for v in sd.values() if v.requires_grad], lr=cfg.TRAIN.LR, weight_decay=cfg.TRAIN.weight_decay)
    times = []
    t_begin = time.perf_counter()
    for i in range(warmup + steps):
        if times and time.perf_counter() - t_begin > budget_s:
            break
        for v in sd.values():
            v.grad = None
        t0 = time.perf_counter()
        if forward_only:
            with torch.no_grad():
                model_ref.model_forward(sd, Ap, img, training=False)
        else:
            out = model_ref.model_forward(sd, Ap, img, training=True, dropout=0.05)
            if encoder == 'newgraph':      # mesh terms on the MANO vertices + pose / shape terms (the loss graph is a few hundred small ops either way)
                loss = model_ref.calc_loss_GCN((out[0], out[1], [], out[3]), labels, la) + sum((d['mano_pose'] ** 2).mean() + (d['mano_shape'] ** 2).mean()
                                                                                                  for d in out[3]['verts3d_MANO_list'].values())
            else:
                loss = model_ref.calc_loss_GCN(out, labels, la)
            loss.backward()
            opt.step()
        t1 = time.perf_counter()
        if i >= warmup:
            times.append(t1 - t0)
    return sum(times) / len(times), len(times)


def cpu_sample_text(args, kind, cores, fwd=False):
    what = 'eval forward' if fwd else 'fwd + calc_loss_GCN + bwd + AdamW'
    src = {'reference': 'the UNMODIFIED reference (models.model.load_model, core.Loss.calc_loss_GCN, torch.optim.AdamW) run from its own sources',
           'port': 'oracle/model_ref.py (torch CPU port of the reference graph)'}[kind]
    return 'batch %d %s, %s, torch CPU fp32, %d of %d usable threads, 1 warm-up step' % (args.cpu_batch, what, src, cores, host_cores())


def run_reference(args):
    """`--impl reference`: the reference's own CPU implementation of the path on the box's host cores.  Under torchrun only rank 0 works."""
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    fwd = args.config == 'forward'
    if args.config == 'mano':
        return run_mano(args, reference_only=True)
    t, cores, nsteps, kind = cpu_reference_time(args.cpu_batch, steps=max(1, min(args.steps, 5)), warmup=1, encoder=args.encoder, forward_only=fwd)
    v = args.cpu_batch / t
    line = {'impl': 'reference', 'metric': metric_name(args), 'value': v, 'unit': 'images/s',
            'n_gpus': args.gpus, 'steps': nsteps, 'warmup': 1, 'ms_per_step': t * 1e3,
            'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
            'config': {'workload': workload_name(args.encoder, args.batch, args.config), 'global_batch': args.batch * args.gpus, 'parallelism': 'dp%d' % args.gpus,
                       'reference_arm': 'the reference\'s own CPU path on the host cores (one process whatever N: a CPU baseline does not scale with the GPU count), '
                                        'each step a bounded sample of batch %d images of the batch-%d workload' % (args.cpu_batch, args.batch)},
            'cpu_baseline': {'value': v, 'unit': 'images/s', 'cores': cores, 'kind': kind, 'sample': cpu_sample_text(args, kind, cores, fwd)},
            'e2e': {'value': v, 'unit': 'images/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}
    print(json.dumps(line))


# ============================================================================ GPU measurement helpers
def gpu_eager_baseline(args, forward_only=False):
    """north_star's comparator: `reference.cuda()` in eager PyTorch on THIS GPU -- the unmodified reference model + loss + AdamW driven by
    oracle/ref_driver.py (20 warm-up + `--gpu-eager-iters` timed iterations, CUDA events, cudnn.benchmark on; SURVEY 8d).  cuDNN TF32
    convolutions on (torch's default, what a user of the reference gets) and, shorter, off."""
    try:
        from oracle import ref_driver
        if not ref_driver.available():
            return {'unavailable': 'reference sources not staged (python -m oracle.build_ref)'}
        if args.encoder not in ('resnet50', 'hrnet48'):
            return {'unavailable': 'the common/myhand variants are compared through the resnet50 line'}
        import torch
        n = args.gpu_eager_iters
        a = ref_driver.time_reference('cuda', args.batch, n, 20, encoder_type=args.encoder, forward_only=forward_only, cudnn_tf32=True)
        torch.cuda.empty_cache()
        b = ref_driver.time_reference('cuda', args.batch, max(5, n // 5), 5, encoder_type=args.encoder, forward_only=forward_only, cudnn_tf32=False)
        torch.cuda.empty_cache()
        return {'what': 'the UNMODIFIED reference (models.model.load_model%s) .cuda(), eager PyTorch %s, cudnn.benchmark=True, batch %d, same GPU, CUDA events'
                        % ('' if forward_only else ' + core.Loss.calc_loss_GCN + torch.optim.AdamW', torch.__version__, args.batch),
                'value': a['images_per_s'], 'unit': 'images/s', 'ms_per_step': a['ms_per_step'], 'warmup': 20, 'steps': a['steps'],
                'cudnn_tf32': True, 'matmul_tf32': False,
                'fp32_only': {'value': b['images_per_s'], 'ms_per_step': b['ms_per_step'], 'steps': b['steps'], 'cudnn_tf32': False}}
    except Exception as e:      # a baseline that cannot run must not take the bench line down with it
        return {'unavailable': '%s: %s' % (type(e).__name__, str(e)[:200])}


def top_kernel_roofline(torch, batch, pk, conv_mode):
    """Time the single most expensive kernel of the step alone: the 3x3 128->128 conv at 64x64 (2.42 GF/img fwd, SURVEY 8a1),
    in the arithmetic mode the step runs its convolutions in.  `traffic` = DRAM bytes per launch of that kernel from the
    committed `ncu --set full` capture (profiles/*roofline_kernel.json; NOT measured in this run), when present."""
    from renderih_b200 import ops
    N, H, C = batch, 64, 128
    x = torch.randn(N * H * H, C, device='cuda')
    w = (torch.randn(C, C, 3, 3, device='cuda') * 0.03).contiguous(memory_format=torch.channels_last)
    for _ in range(3):
        ops.conv2d(x, w, None, N, H, H, stride=1, pad=1)
    torch.cuda.synchronize()
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ops.conv2d(x, w, None, N, H, H, stride=1, pad=1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    flops = 2.0 * N * H * H * C * 9 * C
    ach = flops / (ms * 1e-3) / 1e12
    traffic, src = None, None
    for name in ('r02_roofline_kernel.json', 'r01_roofline_kernel.json'):
        try:
            with open(os.path.join(ROOT, 'profiles', name)) as f:
                traffic = json.load(f).get(conv_mode, {}).get('dram_bytes_per_launch')
            src = 'profiles/' + name
            if traffic:
                break
        except Exception:
            pass
    return {'bound': 'tensor', 'kernel': 'conv3x3 128->128 @64x64 batch %d fwd (gemm_tc_persistent_kernel<..ConvFwdProducer..>, %s)' % (batch, conv_mode),
            'achieved': ach, 'peak': pk['tflops'], 'unit': 'TFLOP/s', 'frac': ach / pk['tflops'], 'frac_of_tf32_peak': ach / (0.5 * pk['tflops']),
            'traffic': traffic, 'traffic_source': (src + ' (ncu --set full capture, not measured in this run)') if traffic else None,
            'ms_per_launch': ms, 'algorithmic_flops_per_launch': flops, 'algorithmic_bytes_per_launch': 4.0 * (2 * N * H * H * C + 9 * C * C),
            'peak_source': pk['src'] + ' bf16 dense burst (kernel timed alone); the TF32 tensor peak is half of it'}


def _gemm_flops(name, a):
    """Algorithmic 2*MAC flops of one GEMM-class C-ABI call from its arguments (include/rih_b200.h), or None for other entry points."""
    if name in ('rih_linear_fwd',):
        return 2.0 * a[7] * a[8] * a[9]
    if name in ('rih_linear_dgrad', 'rih_linear_wgrad'):
        return 2.0 * a[6] * a[7] * a[8]
    if name in ('rih_conv2d_fwd', 'rih_conv2d_dgrad', 'rih_conv2d_wgrad'):
        g = a[4] if name == 'rih_conv2d_fwd' else a[3]
        N, H, W, Cin, Ho, Wo, Cout, R, S = [int(g[i]) for i in range(9)]
        return 2.0 * N * Ho * Wo * Cout * R * S * Cin
    if name == 'rih_attn_tc_fwd':
        B, H, Sq, Sk, d = a[11:16]
        return 4.0 * B * H * Sq * Sk * d
    if name == 'rih_attn_tc_bwd':
        B, H, Sq, Sk, d = a[18:23]
        return 10.0 * B * H * Sq * Sk * d      # dP, dV, dQ, dK + the P recompute-free path (DESIGN 4)
    if name in ('rih_linear_group_fwd', 'rih_linear_group_dgrad', 'rih_linear_group_wgrad'):
        return None     # accounted by the caller through TRACE_FLOPS (grouped launches carry their own flop count)
    return None


def class_roofline(torch, step, pk, flops_step, ms_step):
    """The dominant kernel CLASS of the step, measured live: during ONE eager (un-captured) step every C-ABI launch is bracketed by CUDA
    events on the stream it is launched on (`_lib.TRACE`); the launches that run on the wgmma GEMM / implicit-GEMM kernels
    (nn.Linear, Conv2d and attention contractions: forward, dgrad, wgrad) form the class.  achieved = sum of their algorithmic flops /
    sum of their event-timed durations.  Event pairs around a short kernel include a few microseconds of launch gap, so this
    under-states the class a little; the share of the step is computed against the sum over ALL traced launches (serialised time)."""
    from renderih_b200 import _lib
    from renderih_b200.ops import GROUP_FLOPS
    import ctypes
    _lib.TRACE = []
    counts = (ctypes.c_longlong * 3)()
    try:
        _lib.call('rih_gemm_launch_counts', None, 1)
        step._eager_no_opt()
        torch.cuda.synchronize()
        trace = _lib.TRACE
        _lib.call('rih_gemm_launch_counts', counts, 0)
    finally:
        _lib.TRACE = None
    per = {}
    total_ms = 0.0
    for name, a, e0, e1 in trace:
        ms = e0.elapsed_time(e1)
        total_ms += ms
        fl = _gemm_flops(name, a)
        if fl is None and name in GROUP_FLOPS:
            fl = GROUP_FLOPS[name](a)
        ent = per.setdefault(name, [0, 0.0, 0.0])
        ent[0] += 1; ent[1] += ms; ent[2] += fl or 0.0
    cls = {k: v for k, v in per.items() if v[2] > 0}
    cms = sum(v[1] for v in cls.values())
    cfl = sum(v[2] for v in cls.values())
    n = sum(v[0] for v in cls.values())
    ach = cfl / (cms * 1e-3) / 1e12 if cms > 0 else 0.0
    peak = pk['tflops_sustained']
    top = sorted(per.items(), key=lambda kv: -kv[1][1])[:12]

    def small_ints(a):       # the shape / flag arguments of a call (pointers and stream handles are large)
        out = []
        for v in a:
            v = getattr(v, 'value', v)
            if isinstance(v, int) and 0 <= v < (1 << 24):
                out.append(v)
        return out
    slow = sorted(((e0.elapsed_time(e1), name, a) for name, a, e0, e1 in trace), key=lambda t: -t[0])[:16]
    return {'bound': 'tensor', 'kernel': 'class: every wgmma GEMM / implicit-GEMM launch of the step (gemm_tc_persistent_kernel<...>: Conv2d, nn.Linear and attention '
                                         'contractions, fwd + dgrad + wgrad), %d launches' % n,
            'achieved': ach, 'peak': peak, 'unit': 'TFLOP/s', 'frac': ach / peak, 'frac_of_tf32_peak': ach / (0.5 * peak), 'traffic': None,
            'share_of_step_kernel_time': cms / total_ms if total_ms else None, 'class_ms_per_step': cms, 'all_kernels_ms_per_step_serialised': total_ms,
            'algorithmic_flops_per_step_class': cfl, 'launches_traced': len(trace),
            'how': 'one eager step, CUDA events around every C-ABI launch on its own stream (cold launch gaps included); ncu launch list of the same step: profiles/',
            'peak_source': pk['src'] + ' bf16 dense SUSTAINED (kernels timed inside a long step); operands are TF32, whose tensor peak is half of it',
            'by_entry_point_ms': {k: round(v[1], 3) for k, v in top},
            'gemm_launches_by_path': {'wgmma_tma_store_epilogue': counts[0], 'wgmma_thread_store_epilogue': counts[1], 'exact_fp32_simt': counts[2]},
            'slowest_calls': [{'ms': round(ms, 3), 'entry': name, 'int_args': small_ints(a)} for ms, name, a in slow],
            'step': {'achieved': flops_step / (ms_step * 1e-3) / 1e12, 'peak': peak, 'unit': 'TFLOP/s',
                     'frac': flops_step / (ms_step * 1e-3) / 1e12 / peak, 'frac_of_tf32_peak': flops_step / (ms_step * 1e-3) / 1e12 / (0.5 * peak),
                     'what': 'whole-step algorithmic flops (SURVEY 8d) / device-timed step'}}


def measured_parity(torch, args, conv_mode, lin_mode):
    """MPJPE (mm) and max relative error of THIS build's eval forward in the run's arithmetic against the fp32 CPU oracle (oracle/model_ref.py,
    pinned to the reference's goldens) on the fixed seeded batch the tests use (batch 4, seeded weights).  Root-relative joints through the
    21x778 regressor (SURVEY 8d); the model's unit is metres."""
    from oracle import fixtures, model_ref
    from renderih_b200 import assets as A, ops
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    if args.encoder not in ('resnet50', 'hrnet48'):
        return None
    a = A.synthetic_assets(0)
    cfg = load_cfg()
    cfg.MODEL.ENCODER_TYPE = args.encoder
    model = load_model(cfg, assets=a)
    sd = fixtures.init_state_dict(model.state_dict())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    img = fixtures.make_image(4)
    with torch.no_grad():
        out = model(img.cuda())
        ora = model_ref.model_forward({k: v.clone() for k, v in sd.items()}, model_ref.prepare_assets(a), img, training=False)
    la = fixtures.make_loss_assets(a, A.synthetic_mano(0, 'left'), A.synthetic_mano(0, 'right'))
    mp, rel = [], []
    for side in ('left', 'right'):
        J = la[side]['J21']
        o, r = out[0]['verts3d'][side].cpu(), ora[0]['verts3d'][side]
        jo, jr = torch.matmul(J, o), torch.matmul(J, r)
        jo, jr = jo - jo[:, :1], jr - jr[:, :1]
        mp.append(float((jo - jr).norm(dim=-1).mean()) * 1000)
        rel.append(float((o - r).abs().max() / r.abs().max()))
    del model
    return {'arithmetic': 'conv=%s, linear/attention=%s' % (conv_mode, lin_mode),
            'tolerance_asserted': PARITY_TOL.get(args.gemm_mode), 'tolerance_where': 'tests/test_model_gpu.py (relative to each output tensor\'s max magnitude, eval forward)',
            'mpjpe_vs_oracle_mm': max(mp), 'verts3d_max_rel_err_vs_oracle': max(rel),
            'north_star_target_mm': 1e-3, 'note': 'the exact-fp32 mode (--gemm-mode simt) meets 1e-3 mm; TF32 convolutions are the reference\'s own GPU default '
                                                   '(its cuDNN path is 3.8e-4..5.9e-3 relative from its CPU result, DESIGN 5)',
            'sample': 'batch 4, seeded weights/inputs (oracle/fixtures.py), eval mode'}


# ============================================================================ configs[0]: ManoLayer
def run_mano(args, reference_only=False):
    """BASELINE.json configs[0]: ManoLayer-only forward.  Ours: one fused kernel per call on the GPU, batch 1 (latency) and batch 64
    (+ a large batch for bandwidth); reference: models/manolayer.ManoLayer on the CPU (its own sources), batch 1 and 64."""
    import numpy as np
    import torch
    from oracle import fixtures, mano_ref
    from renderih_b200 import assets as A
    m = A.synthetic_mano(0, 'right')
    cores = host_cores()
    torch.set_num_threads(cores)
    ref_ms, kind = {}, 'port'
    try:
        from oracle import ref_driver, ref_bridge as rb
        if ref_driver.available():
            import pickle
            import tempfile
            with tempfile.TemporaryDirectory() as tmp:
                p = os.path.join(tmp, 'MANO_RIGHT.pkl')
                with open(p, 'wb') as f:
                    pickle.dump(m, f)
                layer = rb.import_reference().mano.ManoLayer(p, center_idx=9, use_pca=True)
            kind = 'reference'
            for bs in (1, 64):
                inp = fixtures.make_mano_inputs(bs)
                root = torch.from_numpy(mano_ref.rodrigues(inp['axis'].numpy()))
                for _ in range(3):
                    layer(root, inp['pose_pca'], inp['shape'])
                n = 30
                t0 = time.perf_counter()
                for _ in range(n):
                    layer(root, inp['pose_pca'], inp['shape'])
                ref_ms[bs] = (time.perf_counter() - t0) / n * 1e3
    except Exception as e:
        ref_ms = {'error': str(e)[:200]}
    if not ref_ms or 'error' in ref_ms:
        md = dict(m); md['J_regressor'] = np.asarray(m['J_regressor'].todense())
        for bs in (1, 64):
            inp = fixtures.make_mano_inputs(bs)
            root = mano_ref.rodrigues(inp['axis'].numpy())
            t0 = time.perf_counter()
            for _ in range(5):
                mano_ref.mano_forward(md, root, inp['pose_pca'].numpy(), inp['shape'].numpy())
            ref_ms[bs] = (time.perf_counter() - t0) / 5 * 1e3
    cpu = {'value': 64 / (ref_ms[64] * 1e-3), 'unit': 'hands/s', 'cores': cores, 'kind': kind, 'latency_ms_bs1': ref_ms[1], 'latency_ms_bs64': ref_ms[64],
           'sample': 'models/manolayer.ManoLayer.forward (PCA pose, 45 comps) on CPU tensors, batch 1 and 64, mean of 30 calls after 3 warm-up'}
    if reference_only:
        print(json.dumps({'impl': 'reference', 'metric': metric_name(args), 'value': cpu['value'], 'unit': 'hands/s', 'n_gpus': args.gpus, 'steps': 30, 'warmup': 3,
                          'ms_per_step': ref_ms[64], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
                          'config': {'workload': 'BASELINE.json configs[0]: ManoLayer-only forward, batch 64 (and batch 1 latency)'}, 'cpu_baseline': cpu,
                          'e2e': {'value': cpu['value'], 'unit': 'hands/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}}))
        return
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device: there is no CPU fallback for the product path'
    from renderih_b200 import _lib
    from renderih_b200.manolayer import ManoLayer
    _lib.load()
    layer = ManoLayer(m, center_idx=9, use_pca=True)
    pk = peaks()
    res = {}
    for bs in (1, 64, 16384):
        inp = fixtures.make_mano_inputs(bs)
        root = torch.from_numpy(mano_ref.rodrigues(inp['axis'].numpy())).cuda()
        pose, shape = inp['pose_pca'].cuda(), inp['shape'].cuda()
        for _ in range(5):
            layer(root, pose, shape)
        torch.cuda.synchronize()
        n = max(args.steps, 50)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            v, j = layer(root, pose, shape)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        hroot, hpose, hshape = root.cpu().pin_memory(), pose.cpu().pin_memory(), shape.cpu().pin_memory()
        hv = torch.empty(v.shape).pin_memory()
        t0 = time.perf_counter()
        for _ in range(n):
            vv, jj = layer(hroot.cuda(non_blocking=True), hpose.cuda(non_blocking=True), hshape.cuda(non_blocking=True))
            hv.copy_(vv, non_blocking=True)
            torch.cuda.synchronize()
        ms_e2e = (time.perf_counter() - t0) / n * 1e3
        io = bs * ((9 + 45 + 10) * 4 + (778 + 21) * 3 * 4)
        res[bs] = {'ms': ms, 'hands_per_s': bs / ms * 1e3, 'io_bytes': io, 'gbs': io / (ms * 1e-3) / 1e9, 'e2e_ms': ms_e2e, 'e2e_hands_per_s': bs / ms_e2e * 1e3}
    big = res[16384]
    line = {'metric': metric_name(args), 'value': res[64]['hands_per_s'], 'unit': 'hands/s', 'n_gpus': 1, 'steps': max(args.steps, 50), 'warmup': 5,
            'ms_per_step': res[64]['ms'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
            'config': {'workload': 'BASELINE.json configs[0]: ManoLayer-only forward (PCA pose 45 comps, centre joint 9), batch 64; batch 1 latency and a 16384-hand batch alongside',
                       'l2': 'the 1.5 MB of MANO tables stay L2 resident; per-hand I/O is 9.8 KB'},
            'latency_ms': {'bs1': res[1]['ms'], 'bs64': res[64]['ms'], 'bs16384': big['ms']},
            'hands_per_s': {'bs1': res[1]['hands_per_s'], 'bs64': res[64]['hands_per_s'], 'bs16384': big['hands_per_s']},
            'e2e': {'value': res[64]['e2e_hands_per_s'], 'unit': 'hands/s', 'ms_per_step': res[64]['e2e_ms'], 'h2d_bytes_per_step': 64 * 64 * 4, 'd2h_bytes_per_step': 64 * 778 * 3 * 4,
                    'bs1_latency_ms': res[1]['e2e_ms'], 'note': 'ManoLayer.forward from pinned host tensors, vertices copied back, wall clock incl. synchronize'},
            'gpu_launches': 1 * max(args.steps, 50), 'launches_per_step': 1,
            'roofline': {'bound': 'hbm', 'kernel': 'mano_fwd_kernel (one CTA per hand), batch 16384', 'achieved': big['gbs'], 'peak': pk['hbm_gbs'], 'unit': 'GB/s',
                         'frac': big['gbs'] / pk['hbm_gbs'], 'traffic': None, 'algorithmic_bytes_per_launch': big['io_bytes'],
                         'note': 'latency / L2-bound by design: 1.17 MFLOP and 9.8 KB of HBM I/O per hand against 1.26 MB of L2-resident pose blend shapes',
                         'peak_source': pk['src']},
            'cpu_baseline': cpu, 'speedup_vs_cpu_reference': {'bs1_latency': ref_ms[1] / res[1]['ms'], 'bs64_throughput': res[64]['hands_per_s'] / cpu['value']}}
    print(json.dumps(line))


# ============================================================================ ours: training step / forward
def build_ours(args, torch, rank, train):
    from renderih_b200 import assets as A
    from renderih_b200.config import load_cfg
    from renderih_b200.model import load_model
    cfg = load_cfg()
    a = A.synthetic_assets(0)
    torch.manual_seed(cfg.SEED)
    if args.encoder in ('graph', 'newgraph'):
        from renderih_b200 import myhand
        build = myhand.load_graph_model if args.encoder == 'graph' else myhand.load_new_model
        model = build(cfg, assets=a, mano_assets={s: A.synthetic_mano(0, s) for s in ('left', 'right')}).cuda()
    else:
        cfg.MODEL.ENCODER_TYPE = args.encoder
        model = load_model(cfg, assets=a).cuda()
    model.train() if train else model.eval()          # train mode: batch-stat BN, dropout 0.05 (reference defaults)
    model.decoder.unsample_layer.weight.requires_grad_(False)   # MODEL.freeze_upsample
    return cfg, a, model


def run_forward(args):
    """BASELINE.json configs[1]: batch-64 eval-mode forward on one GPU, device-timed over a captured CUDA graph + e2e from pinned host batches
    with the result vertices read back; the reference graph in eager PyTorch on the same GPU beside it."""
    import torch
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device: there is no CPU fallback for the product path'
    torch.cuda.set_device(0)
    from renderih_b200 import _lib, ops
    _lib.load()
    conv_mode, lin_mode = {'ref': ('tf32c', 'tf32x3'), 'refrn': ('tf32rn', 'tf32x3')}.get(args.gemm_mode, (args.gemm_mode, args.gemm_mode))
    eager = None if args.skip_gpu_eager else gpu_eager_baseline(args, forward_only=True)
    ops.set_gemm_mode(conv_mode, lin_mode)
    cfg, a, model = build_ours(args, torch, 0, train=False)
    B = args.batch
    g = torch.Generator().manual_seed(cfg.SEED)
    host = [torch.randn(B, 3, 256, 256, generator=g).pin_memory() for _ in range(2)]
    static_in = host[0].cuda()
    c0 = _lib.CALLS[0]
    with torch.no_grad():
        out = model(static_in)
    launches = _lib.CALLS[0] - c0
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            model(static_in)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        out = model(static_in)
    res = out[0]['verts3d']
    host_out = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in res.items()}

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for _ in range(max(3, args.warmup)):
        graph.replay()
    sampler = ClockSampler(0)
    sampler.start()
    steps = args.steps
    ms_dev = timed(lambda i: graph.replay(), steps)

    def e2e(i):
        static_in.copy_(host[i % 2], non_blocking=True)
        graph.replay()
        for k in res:
            host_out[k].copy_(res[k], non_blocking=True)
        torch.cuda.current_stream().synchronize()
    for i in range(2):
        e2e(i)
    ms_e2e = timed(e2e, steps)
    clocks = sampler.stop()
    if args.dump_outputs:                     # the last timed forward: what a caller reads back
        dump_outputs(args.dump_outputs, {'verts3d_%s' % k: v for k, v in host_out.items()})
    pk = peaks()
    gf = FLOPS[args.encoder][1]
    value = B / (ms_dev * 1e-3)
    line = {'metric': metric_name(args), 'value': value, 'unit': 'images/s', 'n_gpus': 1, 'steps': steps, 'warmup': max(3, args.warmup),
            'ms_per_step': ms_dev, 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
            'dtype': 'f32 storage; wgmma TF32 convolutions + 3xTF32 Linear / attention GEMMs (--gemm-mode %s), fp32 accumulate' % args.gemm_mode, 'data': 'synthetic',
            'config': {'workload': workload_name(args.encoder, B, 'forward'), 'cuda_graph': True, 'algorithmic_gflop_per_image_fwd': gf / 1e9,
                       'l2': 'per-step working set (activations, > 1 GB) >> 50 MB L2; no explicit flush needed'},
            'achieved_tflops': value * gf / 1e12,
            'roofline': {'bound': 'tensor', 'kernel': 'whole forward (encoder + attention/GCN decoder + heads): north_star\'s 70 %% target is stated on this',
                         'achieved': value * gf / 1e12, 'peak': pk['tflops_sustained'], 'unit': 'TFLOP/s', 'frac': value * gf / 1e12 / pk['tflops_sustained'],
                         'frac_of_tf32_peak': value * gf / 1e12 / (0.5 * pk['tflops_sustained']), 'traffic': None,
                         'peak_source': pk['src'] + ' bf16 dense sustained; TF32 operands: tensor peak is half of it'},
            'e2e': {'value': B / (ms_e2e * 1e-3), 'unit': 'images/s', 'ms_per_step': ms_e2e, 'h2d_bytes_per_step': B * 3 * 256 * 256 * 4,
                    'd2h_bytes_per_step': sum(v.numel() * 4 for v in res.values())},
            'gpu_launches': launches * steps, 'launches_per_step': launches, 'clocks': clocks,
            'gpu_eager_baseline': eager, 'speedup_vs_gpu_eager': (value / eager['value']) if eager and 'value' in eager else None}
    if not args.skip_cpu_baseline:
        t, cores, n, kind = cpu_reference_time(args.cpu_batch, steps=2, warmup=1, encoder=args.encoder, forward_only=True, budget_s=60)
        line['cpu_baseline'] = {'value': args.cpu_batch / t, 'unit': 'images/s', 'cores': cores, 'kind': kind, 'sample': cpu_sample_text(args, kind, cores, True)}
    print(json.dumps(line))


def run_ours(args):
    import torch
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device: there is no CPU fallback for the product path'
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    from renderih_b200 import _lib, assets as A
    from renderih_b200.loss import GraphLoss, calc_loss_GCN
    from renderih_b200.train import TrainStep
    _lib.load()
    from renderih_b200 import ops as _ops
    conv_mode, lin_mode = {'ref': ('tf32c', 'tf32x3'), 'refrn': ('tf32rn', 'tf32x3')}.get(args.gemm_mode, (args.gemm_mode, args.gemm_mode))
    # north_star's comparator first (rank 0, before our model takes memory / clocks warm either way): the reference graph in eager PyTorch
    eager = None
    if rank == 0 and world == 1 and not args.skip_gpu_eager:
        eager = gpu_eager_baseline(args)
    _ops.set_gemm_mode(conv_mode, lin_mode)
    flops_fb = FLOPS[args.encoder][0]
    cfg, a, model = build_ours(args, torch, rank, train=True)
    B = args.batch
    g = torch.Generator().manual_seed(cfg.SEED + rank)
    host_imgs = [torch.randn(B, 3, 256, 256, generator=g).pin_memory() for _ in range(2)]

    def make_labels():
        d = {k: (torch.randn(*s, generator=g) * 0.05) for k, s in (('v3d_l', (B, 778, 3)), ('v3d_r', (B, 778, 3)), ('root_rel', (B, 3)))}
        d.update({k: (torch.rand(B, 778, 2, generator=g) * 256) for k in ('v2d_l', 'v2d_r')})
        if args.encoder == 'newgraph':
            d.update({k: (torch.randn(B, n, generator=g) * 0.3) for k, n in (('lp_gt', 48), ('rp_gt', 48), ('ls_gt', 10), ('rs_gt', 10))})
        return {k: v.pin_memory() for k, v in d.items()}
    host_labels = [make_labels() for _ in range(2)]
    lab = {k: v.cuda() for k, v in host_labels[0].items()}          # the step's static label buffers (refreshed from the host every e2e step)
    ml, mr = A.synthetic_mano(0, 'left'), A.synthetic_mano(0, 'right')
    jl = torch.from_numpy(__import__('numpy').asarray(ml['J_regressor'].todense(), dtype='float32'))
    jr = torch.from_numpy(__import__('numpy').asarray(mr['J_regressor'].todense(), dtype='float32'))
    gl, gr = GraphLoss(jl, ml['f'], 4, 'cuda'), GraphLoss(jr, mr['f'], 4, 'cuda')
    conv = model.decoder.converter
    z = torch.zeros(B, 21, 3, device='cuda')
    if args.encoder == 'newgraph':
        from renderih_b200.loss import ManoLoss, mano_loss_GCN
        gl, gr = ManoLoss(jl, ml['f'], 4, 'cuda'), ManoLoss(jr, mr['f'], 4, 'cuda')

    def loss_fn(out):
        if args.encoder == 'newgraph':
            return mano_loss_GCN(cfg, 0, gl, gr, conv['left'], conv['right'], out[0], out[1], out[2], out[3], None, None, None,
                                 lab['v2d_l'], z[..., :2], lab['v2d_r'], z[..., :2], lab['v3d_l'], z, lab['v3d_r'], z, lab['root_rel'], 256,
                                 lab['lp_gt'], lab['ls_gt'], lab['rp_gt'], lab['rs_gt'])[0]
        return calc_loss_GCN(cfg, 0, gl, gr, conv['left'], conv['right'], out[0], out[1], out[2], out[3], None, None, None,
                             lab['v2d_l'], z[..., :2], lab['v2d_r'], z[..., :2], lab['v3d_l'], z, lab['v3d_r'], z, lab['root_rel'], 256)[0]

    step = TrainStep(model, loss_fn, host_imgs[0].cuda(), lr=cfg.TRAIN.LR, weight_decay=cfg.TRAIN.weight_decay, use_graph=not args.no_graph, labels=lab)
    c0 = _lib.CALLS[0]
    step._eager()
    torch.cuda.synchronize()
    calls_per_step = _lib.CALLS[0] - c0
    if not args.no_graph:
        step.capture(warmup=2)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            fn(i)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device='cuda')
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps

    for i in range(max(3, args.warmup)):
        step()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms_dev = timed(lambda i: step(), args.steps)                       # inputs already resident in HBM
    losses = []

    step.prefetch(host_imgs[0], host_labels[0])

    def e2e_step(i):
        loss = step()                                                    # consumes the batch whose H2D copy was started one step ahead ...
        step.prefetch(host_imgs[(i + 1) % 2], host_labels[(i + 1) % 2])   # ... and starts the next one (pinned memory, copy stream): image + labels every step
        losses.append(float(loss))                                       # D2H read of the step's result (synchronises every step)

    for i in range(2):
        e2e_step(i)
    ms_e2e = timed(e2e_step, args.steps)
    clocks = sampler.stop() if rank == 0 else None
    if rank == 0 and args.dump_outputs:       # the last timed step: its loss and the parameters it updated
        dump_outputs(args.dump_outputs, {'loss': [losses[-1]], 'params': step.flatp.flat})
    exposed = None
    if world > 1:        # exposed communication = step time with the gradient exchange - step time without it (one extra timed pass on every rank)
        if getattr(step, 'overlap', False) and not args.no_graph:
            step.capture(warmup=1, reduce=False)       # the overlapped all-reduce segments live inside the captured step: capture a variant without them
        step.skip_all_reduce = True
        ms_nocomm = timed(lambda i: step(), args.steps)
        step.skip_all_reduce = False
        exposed = ms_dev - ms_nocomm
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    pk = peaks()
    total_imgs = B * world
    value = total_imgs / (ms_dev * 1e-3)
    e2e = total_imgs / (ms_e2e * 1e-3)
    h2d = B * 3 * 256 * 256 * 4 + sum(v.numel() * 4 for v in host_labels[0].values())
    roof = class_roofline(torch, step, pk, B * flops_fb, ms_dev)
    roof_top = top_kernel_roofline(torch, B, pk, conv_mode)
    line = {'metric': metric_name(args),
            'value': value, 'unit': 'images/s', 'n_gpus': world, 'steps': args.steps, 'warmup': max(3, args.warmup), 'ms_per_step': ms_dev,
            'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': {'simt': 'f32', 'refrn': 'f32 storage; wgmma TF32(rn) convolutions (cuDNN-default class of the reference) + 3xTF32 fp32-faithful Linear GEMMs, fp32 accumulate',
                      'tf32': 'tf32 (truncating) conv+Linear, fp32 accumulate/storage', 'tf32c': 'tf32 (truncating, mean-compensated) conv+Linear, fp32 accumulate/storage',
                      'ref': 'f32 storage; wgmma TF32 convolutions (truncating + mean-compensated: the accuracy class of the reference\'s cuDNN-TF32 default, measured) + 3xTF32 fp32-faithful Linear GEMMs, fp32 accumulate', 'tf32rn': 'tf32 (rn) conv+Linear, fp32 accumulate/storage',
                      'tf32x3': '3xTF32 (fp32-faithful) conv+Linear, fp32 accumulate/storage'}[args.gemm_mode], 'data': 'synthetic',
            'config': {'workload': workload_name(args.encoder, B),
                       'global_batch': total_imgs, 'parallelism': 'dp%d' % world, 'cuda_graph': not args.no_graph,
                       'l2': 'per-step working set (activations, several GB) >> 50 MB L2; no explicit flush needed',
                       'algorithmic_gflop_per_image': flops_fb / 1e9},
            'achieved_tflops': value * flops_fb / 1e12 / world,
            'e2e': {'value': e2e, 'unit': 'images/s', 'ms_per_step': ms_e2e, 'h2d_bytes_per_step': h2d, 'd2h_bytes_per_step': 4,
                    'note': 'TrainStep public API from pinned float32 host batches: image AND labels of step i+1 are copied on a copy stream while step i runs (input double buffering), loss read back every step'},
            'gpu_launches': calls_per_step * args.steps, 'launches_per_step': calls_per_step,
            'clocks': clocks, 'roofline': roof, 'roofline_top_kernel': roof_top, 'last_loss': losses[-1] if losses else None}
    if exposed is not None:
        line['all_reduce'] = {'exposed_ms': exposed, 'bytes': step.flatp.numel * 4,
                              'mode': ('overlapped with backward: %d segments all-reduced on a communication stream inside the captured step as their gradients complete'
                                       % (len(step._segments) + 1)) if getattr(step, 'overlap', False) else 'one all-reduce of the flat gradient after backward'}
    if eager is not None:
        line['gpu_eager_baseline'] = eager
        line['speedup_vs_gpu_eager'] = (value / eager['value']) if 'value' in eager else None
    if world == 1 and not args.skip_cpu_baseline:
        try:
            line['parity'] = measured_parity(torch, args, conv_mode, lin_mode)
        except Exception as e:
            line['parity'] = {'error': str(e)[:200]}
        t, cores, _, kind = cpu_reference_time(args.cpu_batch, steps=2, warmup=1, encoder=args.encoder, budget_s=90)
        line['cpu_baseline'] = {'value': args.cpu_batch / t, 'unit': 'images/s', 'cores': cores, 'kind': kind, 'sample': cpu_sample_text(args, kind, cores)}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    a = parse()
    if a.impl == 'reference':
        run_reference(a)
    elif a.config == 'mano':
        run_mano(a)
    elif a.config == 'forward':
        run_forward(a)
    else:
        run_ours(a)
