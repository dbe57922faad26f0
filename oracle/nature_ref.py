"""Independent float64 torch statement of the pose optimiser's discriminator nature loss (GeOptimizer.NatureLoss,
pose_data_optimize/hocontact/postprocess/geo_optimizer_both_batch.py:110-132, with Pos2dDiscriminator of Ver2Code/Discriminator/
discrim.py:66-105 and the quaternion / Euler conversions of utlize.py:41-69, 208-289), written from the math, with its gradient.

The probabilities are rounded to float32 before the mask and the binary cross-entropy, as the reference computes them, so the hard
decisions and torch's clamps (-100 on the logs, 1e-12 on p (1 - p)) act on the values the reference sees; the cross-entropy backward is
torch's formula, (p - y) / max(p (1 - p), 1e-12) / numel, not the autograd of the clamped forward.  `flags` marks rows ([2, B]: right,
left) whose float32 result is not determined by this float64 one:
  * 'tie':       |p1 - 1.5 p0| within rounding of the mask's threshold;
  * 'asin':      |R02| within rounding of 1, where asin and its derivative are ill-conditioned (or NaN);
  * 'saturated': a masked row with min(p) between 1e-30 and 1e-5, where float32's p0 or p1 rounds to 1 and the softmax backward cancels.

TEST INFRASTRUCTURE -- never imported by the product package.
"""
import math

import numpy as np
import torch

LAYERS = ('pose_layer_1', 'pose_layer_2', 'pose_layer_3', 'pose_layer_4', 'layer_last', 'layer_pred')
SHAPES = {'pose_layer_1': (512, 45), 'pose_layer_2': (512, 512), 'pose_layer_3': (512, 512), 'pose_layer_4': (512, 512),
          'layer_last': (512, 512), 'layer_pred': (2, 512)}
SLOPE = 0.01
TIE_TOL, ASIN_TOL, SAT_LO, SAT_HI = 1e-5, 1e-5, 1e-30, 1e-5


def state_dict_keys():
    return [n + s for n in LAYERS for s in ('.weight', '.bias')]


def init_state_dict(seed, pred_scale=1.0, pred_bias=(0.0, 0.0)):
    """torch.nn.Linear's default initialisation drawn from a numpy generator (weight and bias uniform in +-1/sqrt(fan_in)), then
    layer_pred.weight * pred_scale and pred_bias added to layer_pred.bias -> {key: float32 tensor}."""
    rng = np.random.default_rng(seed)
    sd = {}
    for n in LAYERS:
        out, inp = SHAPES[n]
        k = 1.0 / math.sqrt(inp)
        sd[n + '.weight'] = torch.from_numpy(rng.uniform(-k, k, size=(out, inp))).float()
        sd[n + '.bias'] = torch.from_numpy(rng.uniform(-k, k, size=(out,))).float()
    sd['layer_pred.weight'] = (sd['layer_pred.weight'].double() * pred_scale).float()
    sd['layer_pred.bias'] = (sd['layer_pred.bias'].double() + torch.tensor(pred_bias, dtype=torch.float64)).float()
    return sd


def features(q):
    """[N,15,4] quaternions (real part first) -> (features [N,45], R02 [N,15])."""
    r, i, j, k = q.unbind(-1)
    s = 2.0 / (q * q).sum(-1)
    r00, r01, r02 = 1 - s * (j * j + k * k), s * (i * j - k * r), s * (i * k + j * r)
    r12, r22 = s * (j * k - i * r), 1 - s * (i * i + j * j)
    e = torch.stack([torch.atan2(-r12, r22), torch.asin(r02), torch.atan2(-r01, r00)], -1)
    return e.reshape(q.shape[0], 45), r02


def _lrelu(z):
    return torch.where(z > 0, z, SLOPE * z)        # slope 0.01 at z == 0, as torch's LeakyReLU backward takes it


def logits(sd, x):
    """features [N,45] -> logits [N,2] through the discriminator's MLP in float64."""
    W = {n: (sd[n + '.weight'].to(x), sd[n + '.bias'].to(x)) for n in LAYERS}
    lin = lambda n, h: h @ W[n][0].T + W[n][1]
    d1 = _lrelu(lin('pose_layer_1', x))
    d2 = _lrelu(lin('pose_layer_2', d1))
    d3 = _lrelu(lin('pose_layer_3', d2) + d1)
    d4 = lin('pose_layer_4', d3)
    d5 = _lrelu(lin('layer_last', d4))
    return lin('layer_pred', d5)


def discriminator(sd, q):
    """[N,15,4] -> (probs [N,2], R02 [N,15])."""
    x, r02 = features(q)
    return torch.softmax(logits(sd, x), dim=1), r02


class _BCE(torch.autograd.Function):
    """binary_cross_entropy(p, y, reduction='mean') with torch's forward clamps and its backward formula."""

    @staticmethod
    def forward(ctx, p, y):
        ctx.save_for_backward(p, y)
        hundred = p.new_tensor(-100.0)
        return ((y - 1) * torch.maximum(torch.log1p(-p), hundred) - y * torch.maximum(torch.log(p), hundred)).mean()

    @staticmethod
    def backward(ctx, g):
        p, y = ctx.saved_tensors
        return g * (p - y) / torch.clamp(p * (1 - p), min=1e-12) / p.numel(), None


def bce(p, y):
    return _BCE.apply(p, y)


def _round32(p):
    """p with the value rounded to float32 and the gradient passed straight through."""
    return p + (p.detach().float().double() - p.detach())


def nature_loss(sd, right, left):
    """right, left [B,15,4] -> (0-dim loss, {'probs': [2,B,2] (float32 values), 'mask': [2,B], 'flags': {kind: [2,B]}})."""
    B = right.shape[0]
    loss = right.new_zeros(())
    probs, masks, flags = [], [], {'tie': [], 'asin': [], 'saturated': []}
    for q in (right, left):
        p64, r02 = discriminator(sd, q)
        p = _round32(p64)
        m = p[:, 1] < 1.5 * p[:, 0]
        if bool(m.any()):
            y = torch.cat([torch.zeros(B, 1), torch.ones(B, 1)], 1).to(p)
            loss = loss + bce(p[m], y[m])
        pd = p.detach()
        probs.append(pd)
        masks.append(m)
        flags['tie'].append((pd[:, 1] - 1.5 * pd[:, 0]).abs() < TIE_TOL)
        flags['asin'].append(((1 - r02.detach().abs()) < ASIN_TOL).any(1) | torch.isnan(r02.detach()).any(1))
        mn = pd.min(1).values
        flags['saturated'].append(m & (mn > SAT_LO) & (mn < SAT_HI))
    return loss, {'probs': torch.stack(probs), 'mask': torch.stack(masks), 'flags': {k: torch.stack(v) for k, v in flags.items()}}


def weighted_case(sd, right16, left16):
    """The optimiser's call on normalised [B,16,4] poses: loss = NatureLoss(right16[:, 1:], left16[:, 1:]) -> (loss, d_right16,
    d_left16, info); the gradients are with respect to the [B,16,4] leaves, so the root rows' gradient is 0."""
    leaves = [t.detach().double().clone().requires_grad_(True) for t in (right16, left16)]
    loss, info = nature_loss(sd, leaves[0][:, 1:], leaves[1][:, 1:])
    if loss.requires_grad:
        loss.backward()
    grads = [l.grad if l.grad is not None else torch.zeros_like(l) for l in leaves]
    return loss.detach(), grads[0], grads[1], info


def row_flags(info):
    """[2,B] True where a row's float32 result is not determined by the float64 one (any kind)."""
    f = info['flags']
    return f['tie'] | f['asin'] | f['saturated']
