"""The pose optimiser's discriminator nature loss on the GPU: a drop-in for `Pos2dDiscriminator` (pose_data_optimize/Ver2Code/
Discriminator/discrim.py:66-105) and `GeOptimizer.NatureLoss` (hocontact/postprocess/geo_optimizer_both_batch.py:110-132, built at
:106-108 and called at :802).  Kernels in csrc/nature.cu; there is no CPU path.

    disc = Pos2dDiscriminator(num_joints=15, hid_dim=512, dropout=0.05).cuda().eval()
    disc.load_state_dict(torch.load('Ver2Code/Discriminator/discrim.pth'))          # the reference's keys and shapes, strictly
    nature = NatureLoss(disc)
    nature_loss = nature(var_hand_pose_normalized[:, 1:], var_sub_hand_pose_normalized[:, 1:])      # 0-dim, differentiable

The poses are [B,15,4] (or [B,60]) quaternions, real part first; a [:, 1:] view of a contiguous [B,16,4] tensor is read in place.
Forward and backward never synchronise with the host and can be captured in a CUDA graph; the upstream gradient is read on the device.

Conventions reproduced:

* Features (utlize.py:41-69, 208-289): quaternion_to_matrix with two_s = 2 / |q|^2 (so the gradient flows through |q|^2), then
  matrix_to_euler_angles(R, 'XYZ') = (atan2(-R12, R22), asin(R02), atan2(-R01, R00)); feature 3 j + c for joint j + 1.  The left hand
  is passed as it is, without the y/z sign flip of HandPoseConverter (the optimiser passes the normalised poses, :802).
* MLP (discrim.py:89-105): d1 = lrelu(L1 x), d2 = lrelu(L2 d1), d3 = lrelu(L3 d2 + d1), d4 = L4 d3 (no activation),
  d5 = lrelu(L_last d4), p = softmax(L_pred d5); LeakyReLU slope 0.01, whose backward uses the slope at an input of exactly 0.  The
  `dropout` argument creates no layer.  Both hands go through the same discriminator.
* Loss (geo_optimizer_both_batch.py:110-132): per hand mask = p1 < 1.5 p0 (strict, fp32); over the masked rows
  binary_cross_entropy(p[mask], (0, 1)), the mean over 2 n elements of torch's -max(log1p(-p0), -100) - max(log(p1), -100); a hand with
  an empty mask contributes 0; the result is the sum of both hands.  The backward is torch's: (p - y) / max(p (1 - p), 1e-12) / (2 n)
  (torch/_decomp/decompositions.py binary_cross_entropy_backward), then the softmax backward p * (g - sum g p).  The empty-mask rule is
  decided on the device; the reference's `nature_mask.sum() > 0` synchronises twice.
* NaN: at |R02| >= 1 (asin) and at atan2(0, 0) the features and their derivatives follow the reference's formulas, without clamping.
  A row whose probabilities are NaN fails the mask and so takes no part in the loss.

Deviations:

* Parameters have requires_grad=False and no gradient is computed for them; the reference accumulates gradients into the frozen
  weights, which nothing reads.
* When both masks are empty the result is a 0-dim zero with a zero gradient; the reference returns the constant torch.tensor(0.0).
* A row whose d(probs) is zero (every row outside the masks) gets a zero pose gradient, where the reference's 0 * NaN gives NaN for a
  row whose features are NaN.
* The arithmetic is exact fp32 on CUDA cores in a fixed order; it does not follow the library's GEMM precision mode
  (ops.set_gemm_mode), so the hard mask decision does not change with it.

Not supported: num_joints != 15 or hid_dim != 512 (NotImplementedError), float64 inputs (TypeError), CPU tensors (RuntimeError).
"""
import ctypes

import torch
from torch import nn

from ._lib import call

NUM_JOINTS, HID_DIM = 15, 512
SIGN_WORDS = 4 * HID_DIM // 32        # per row: the sign bits of the four activated hidden layers (csrc/nature.cu)
LAYERS = ('pose_layer_1', 'pose_layer_2', 'pose_layer_3', 'pose_layer_4', 'layer_last', 'layer_pred')


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _check_tensor(who, name, t):
    if not isinstance(t, torch.Tensor):
        raise TypeError('renderih_b200.nature.%s: %s must be a tensor, got %s' % (who, name, type(t).__name__))
    if not t.is_cuda:
        raise RuntimeError('renderih_b200.nature.%s: %s must be a CUDA tensor (there is no CPU path)' % (who, name))
    if t.dtype != torch.float32:
        raise TypeError('renderih_b200.nature.%s: %s must be float32, got %s' % (who, name, t.dtype))


def _pose_rows(who, name, x):
    """[B,60] or [B,15,4] -> ([B,15,4] view with joint stride 4 and component stride 1, row stride in floats)."""
    _check_tensor(who, name, x)
    if x.dim() == 2 and x.shape[1] == NUM_JOINTS * 4:
        x = x.unflatten(1, (NUM_JOINTS, 4))
    if x.dim() != 3 or tuple(x.shape[1:]) != (NUM_JOINTS, 4):
        raise ValueError('%s must be [B,%d] or [B,%d,4], got %s' % (name, NUM_JOINTS * 4, NUM_JOINTS, tuple(x.shape)))
    if x.stride(2) != 1 or x.stride(1) != 4 or (x.shape[0] > 1 and x.stride(0) < NUM_JOINTS * 4):
        x = x.contiguous()
    return x, (x.stride(0) if x.shape[0] > 1 else NUM_JOINTS * 4)


class Pos2dDiscriminator(nn.Module):
    """Ver2Code/Discriminator/discrim.py Pos2dDiscriminator for num_joints=15, hid_dim=512: forward(x [B,60] | [B,15,4] quaternions)
    -> softmax [B,2], differentiable with respect to x.  Parameters pose_layer_{1..4}, layer_last and layer_pred have the reference's
    names, shapes and default initialisation, and requires_grad=False (see the module docstring)."""

    def __init__(self, num_joints=15, hid_dim=512, dropout=0.05):
        super().__init__()
        if num_joints != NUM_JOINTS or hid_dim != HID_DIM:
            raise NotImplementedError('Pos2dDiscriminator runs num_joints=%d, hid_dim=%d only (the pose optimiser\'s), got %s, %s'
                                      % (NUM_JOINTS, HID_DIM, num_joints, hid_dim))
        self.pose_layer_1 = nn.Linear(num_joints * 3, hid_dim)
        self.pose_layer_2 = nn.Linear(hid_dim, hid_dim)
        self.pose_layer_3 = nn.Linear(hid_dim, hid_dim)
        self.pose_layer_4 = nn.Linear(hid_dim, hid_dim)
        self.layer_last = nn.Linear(hid_dim, hid_dim)
        self.layer_pred = nn.Linear(hid_dim, 2)
        self.hid_dim = hid_dim
        self.requires_grad_(False)

    def _param_ptrs(self, device):
        ptrs = []
        for name in LAYERS:
            layer = getattr(self, name)
            for kind, t in (('weight', layer.weight), ('bias', layer.bias)):
                if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError('Pos2dDiscriminator: %s.%s must be a contiguous float32 tensor on %s, got %s %s'
                                       % (name, kind, device, t.dtype, t.device))
                ptrs.append(t.data_ptr())
        return (ctypes.c_void_p * len(ptrs))(*ptrs)

    def forward(self, x):
        rows, ld = _pose_rows('Pos2dDiscriminator', 'x', x)
        return _DiscFn.apply(self, rows, ld, None, 0)


class _DiscFn(torch.autograd.Function):
    """rih_nature_disc_fwd / rih_nature_disc_bwd on the rows of a, then of b when it is given -> probs [n,2]."""

    @staticmethod
    def forward(ctx, disc, a, lda, b, ldb):
        B, dev = a.shape[0], a.device
        n = 2 * B if b is not None else B
        probs = torch.empty(n, 2, device=dev)
        need = any(ctx.needs_input_grad)
        signs = torch.empty(n, SIGN_WORDS, dtype=torch.int32, device=dev) if need else None
        params = disc._param_ptrs(dev)
        with torch.cuda.device(dev):
            call('rih_nature_disc_fwd', params, a.data_ptr(), lda, None if b is None else b.data_ptr(), ldb, B, probs.data_ptr(),
                 None if signs is None else signs.data_ptr(), _stream(a))
        if need:
            ctx.disc, ctx.ld = disc, (lda, ldb)
            ctx.has_b = b is not None
            ctx.save_for_backward(a, b if b is not None else a, probs, signs)
        return probs

    @staticmethod
    def backward(ctx, g):
        a, b, probs, signs = ctx.saved_tensors
        g = g.float().contiguous()
        B, dev = a.shape[0], a.device
        da = torch.empty(B, NUM_JOINTS, 4, device=dev)
        db = torch.empty(B, NUM_JOINTS, 4, device=dev) if ctx.has_b else None
        with torch.cuda.device(dev):
            call('rih_nature_disc_bwd', ctx.disc._param_ptrs(dev), a.data_ptr(), ctx.ld[0], b.data_ptr() if ctx.has_b else None, ctx.ld[1],
                 B, probs.data_ptr(), signs.data_ptr(), g.data_ptr(), da.data_ptr(), None if db is None else db.data_ptr(), _stream(g))
        return None, da, None, db, None


class _LossFn(torch.autograd.Function):
    """rih_nature_loss_fwd / rih_nature_loss_bwd: probs [2B,2] (right rows first) -> 0-dim loss."""

    @staticmethod
    def forward(ctx, probs, B):
        dev = probs.device
        loss = torch.empty((), device=dev)
        count = torch.empty(2, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            call('rih_nature_loss_fwd', probs.data_ptr(), B, loss.data_ptr(), count.data_ptr(), _stream(probs))
        ctx.B = B
        ctx.save_for_backward(probs, count)
        return loss

    @staticmethod
    def backward(ctx, g):
        probs, count = ctx.saved_tensors
        g = g.float().contiguous()
        gp = torch.empty_like(probs)
        with torch.cuda.device(g.device):
            call('rih_nature_loss_bwd', probs.data_ptr(), count.data_ptr(), ctx.B, g.data_ptr(), gp.data_ptr(), _stream(g))
        return gp, None


class NatureLoss(nn.Module):
    """GeOptimizer.NatureLoss: forward(right_pose, left_pose) -> 0-dim loss, differentiable with respect to both poses ([B,15,4] or
    [B,60] each, B >= 1; the optimiser passes the [:, 1:] views of its normalised [B,16,4] poses).  disc: a Pos2dDiscriminator on the
    poses' CUDA device."""

    def __init__(self, disc):
        super().__init__()
        if not isinstance(disc, Pos2dDiscriminator):
            raise TypeError('NatureLoss: disc must be a renderih_b200.nature.Pos2dDiscriminator, got %s' % type(disc).__name__)
        self.disc = disc

    def forward(self, right_pose, left_pose):
        r, ldr = _pose_rows('NatureLoss', 'right_pose', right_pose)
        l, ldl = _pose_rows('NatureLoss', 'left_pose', left_pose)
        B = r.shape[0]
        if l.shape[0] != B or B < 1:
            raise ValueError('right_pose and left_pose must have the same batch B >= 1, got %d and %d' % (B, l.shape[0]))
        if r.device != l.device:
            raise RuntimeError('NatureLoss: right_pose is on %s, left_pose on %s' % (r.device, l.device))
        probs = _DiscFn.apply(self.disc, r, ldr, l, ldl)
        return _LossFn.apply(probs, B)
