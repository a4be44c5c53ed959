"""Float64 restatement of FSP (finite_scalar_perturbation.py of the reference, "fsp") for the tests (TEST INFRASTRUCTURE ONLY).

- `row_chain`: the per-element chain of fsp:323-351 in float64 (numpy), given the draws.
- `moments`, `norm_loss`: the batch moments of fsp:93-99 and VectorNorm's loss (fsp:126-133).
- `stats_grad`: the closed-form gradient of the moments (DESIGN 4.11); `stats_grad_autograd` the same by float64 autograd of
  the batch-moment formula, to check it.
- `eager_forward`: the reference's forward written as eager torch on any device (draws made with torch.rand_like in the
  reference's order), for the GPU tests and tools/bench_fsp.py.
"""
from __future__ import annotations

import math

import numpy as np
import torch
from scipy import special

ACTS = ("tanh", "sigmoid", "normal", "laplace", "cauchy")
UNIT_STD = 0.28867513459481287

PRESETS = {
    "none": (0., 0., 1., 0., 0., 0., 0., 0.),
    "var": (0., 0.1, 1., 0.07, 0., 0., 0., 0.),
    "kurt": (0., 0.1, 1., 0.07, 0., 0.06, 0., 0.05),
    "var_tanh": (0., 0.1, 0.8225, 0.07, 0., 0., 0., 0.),
    "var_sigmoid": (0., 0.1, 3.29, 0.07, 0., 0., 0., 0.),
    "var_laplace": (0., 0.1, 2., 0.07, 0., 0., 0., 0.),
}   # (l1_target, l1_weight, ..., l4_target, l4_weight)


def act_f64(name, z):
    z = np.asarray(z, np.float64)
    if name == "tanh":
        return (np.tanh(z) + 1.) / 2.
    if name == "sigmoid":
        return special.expit(z)
    if name == "normal":
        return (1. + special.erf(z / math.sqrt(2.))) / 2.
    if name == "laplace":
        return 0.5 * (1. + np.sign(z) * (1. - np.exp(-np.abs(z))))
    return np.arctan(z) / np.pi + 0.5


def inv_act_f64(name, p):
    p = np.asarray(p, np.float64)
    with np.errstate(divide="ignore"):
        if name == "tanh":
            return np.arctanh(2. * p - 1.)
        if name == "sigmoid":
            return special.logit(p)
        if name == "normal":
            return special.erfinv(2. * p - 1.) * math.sqrt(2.)
        if name == "laplace":
            return -np.sign(p - 0.5) * np.log(1. - 2. * np.abs(p - 0.5))
        return np.tan((p - 0.5) * np.pi)


def act_grad_f64(name, z):
    z = np.asarray(z, np.float64)
    if name == "tanh":
        return 0.5 * (1. - np.tanh(z) ** 2)
    if name == "sigmoid":
        s = special.expit(z)
        return s * (1. - s)
    if name == "normal":
        return np.exp(-z * z / 2.) / math.sqrt(2. * np.pi)
    if name == "laplace":
        return 0.5 * np.exp(-np.abs(z)) * np.sign(z) ** 2
    return 1. / (np.pi * (1. + z * z))


def basis(levels):
    return np.cumprod([1] + list(levels[:-1])).astype(np.int64)


def row_chain(z, levels, act, inv=False, eps=1.1920928955078125e-07, u1=None, u2=None, qrate=0.):
    """float64 fp:323-351 on z (N, d): (q_z, indices int64, level_indices, accept mask or None).  act values are computed in
    float64, so only elements away from a bin edge (see `pre_floor`) are comparable with an fp32 run."""
    L = np.asarray(levels, np.float64)
    a = act_f64(act, z)
    lev = np.floor(np.minimum(a, 1. - eps) * L)
    q = (lev + 0.5) / L
    accept = None
    if u1 is not None:
        pmax = (np.float32(1.) / (2 * np.asarray(levels)).astype(np.float32)).astype(np.float64)   # fp32 in torch (fsp:333)
        prop = a + pmax * (np.asarray(u1, np.float64) * 2. - 1.)
        accept = (prop > 0.) & (prop < 1.)
        pa = np.where(accept, prop, a)
        q = np.where(np.asarray(u2, np.float64) > qrate, pa, q)
    if inv:
        qz = inv_act_f64(act, np.clip(q, eps, 1. - eps))
    else:
        qz = (q - 0.5) / UNIT_STD
    idx = (lev.astype(np.int64) * basis(levels)).sum(-1)
    return qz, idx, lev, accept


def pre_floor(z, levels, act, eps=1.1920928955078125e-07):
    """act(z) * L in float64 (the value floored into the level index)."""
    return np.minimum(act_f64(act, z), 1. - eps) * np.asarray(levels, np.float64)


def near_integer(v, rel=2. ** -19):
    """Elements within `rel` (relative) of an integer: fp32 and float64 may floor them differently."""
    return np.abs(v - np.round(v)) <= rel * np.maximum(np.abs(v), 1.)


def moments(z):
    """float64 (mean, unbiased variance, skewness, kurtosis - 3) of z (N, d) over the rows, std clamped at 1e-8."""
    z = np.asarray(z, np.float64)
    n = z.shape[0]
    m = z.mean(0)
    u = z - m
    var = (u * u).sum(0) / (n - 1)
    sd = np.maximum(np.sqrt(var), 1e-8)
    t = u / sd
    return m, var, (t ** 3).mean(0), (t ** 4).mean(0) - 3.


def norm_loss(stats, norm):
    return sum(((np.asarray(s, np.float64) - norm[2 * k]) ** 2).mean() * norm[2 * k + 1] for k, s in enumerate(stats))


def stats_grad(z, G):
    """The closed-form d/dz of sum_k G[k] . stat_k (G (4, d)): a cubic in t = (z - m) / std per column."""
    z = np.asarray(z, np.float64)
    n = z.shape[0]
    m = z.mean(0)
    u = z - m
    var = (u * u).sum(0) / (n - 1)
    sdr = np.sqrt(var)
    sd = np.maximum(sdr, 1e-8)
    c = (sdr >= 1e-8).astype(np.float64)
    t = u / sd
    s, k3 = (t ** 3).mean(0), (t ** 4).mean(0)
    a2 = (t * t).mean(0)
    Gm, Gv, Gs, Gk = (np.asarray(g, np.float64) for g in G)
    return (Gm / n + Gv * 2. * u / (n - 1)
            + Gs * (3. * (t * t - a2) / (n * sd) - c * 3. * s * t / (sd * (n - 1)))
            + Gk * (4. * (t ** 3 - s) / (n * sd) - c * 4. * k3 * t / (sd * (n - 1))))


def norm_loss_grad_weights(stats, norm, d):
    """d norm_loss / d stat_k, (4, d)."""
    return np.stack([2. * norm[2 * k + 1] * (np.asarray(s, np.float64) - norm[2 * k]) / d for k, s in enumerate(stats)])


def _stats_torch(z):
    variance, mean = torch.var_mean(z, dim=0, unbiased=True)
    std = variance.sqrt().clamp_min(1e-8)
    t = (z - mean) / std
    return mean, variance, t.pow(3).mean(0), t.pow(4).mean(0) - 3.


def stats_grad_autograd(z, G):
    z = torch.as_tensor(np.asarray(z, np.float64)).requires_grad_(True)
    stats = _stats_torch(z)
    sum((s * torch.as_tensor(np.asarray(g, np.float64))).sum() for s, g in zip(stats, G)).backward()
    return z.grad.numpy()


_TORCH_ACT = {
    "tanh": lambda z: (torch.tanh(z) + 1.0) / 2.0,
    "sigmoid": torch.sigmoid,
    "normal": lambda z: (1.0 + torch.erf(z / math.sqrt(2.0))) / 2.0,
    "laplace": lambda z: 0.5 * (1.0 + torch.sign(z) * (1.0 - torch.exp(-torch.abs(z)))),
    "cauchy": lambda z: torch.arctan(z) / torch.pi + 0.5,
}
_TORCH_INV = {
    "tanh": lambda p: torch.arctanh(p * 2.0 - 1.0),
    "sigmoid": torch.logit,
    "normal": lambda p: torch.erfinv(2.0 * p - 1.0) * math.sqrt(2.0),
    "laplace": lambda p: -torch.sign(p - 0.5) * torch.log(1.0 - 2.0 * torch.abs(p - 0.5)),
    "cauchy": lambda p: torch.tan((p - 0.5) * torch.pi),
}


def eager_forward(z, levels, act="tanh", inv=False, quantize_rate=1.0, norm=PRESETS["var_tanh"], eps=None):
    """The reference's step on z (N, d) (after project_in) as eager torch: (q_z, level_indices, norm_loss, stats, p_accept or
    None).  With quantize_rate < 1 it draws torch.rand_like twice, in the reference's order."""
    eps = eps or torch.finfo(z.dtype).eps
    L = torch.as_tensor(levels, dtype=torch.int32, device=z.device)
    stats = _stats_torch(z)
    loss = sum(((s - norm[2 * k]) ** 2).mean() * norm[2 * k + 1] for k, s in enumerate(stats))
    a = _TORCH_ACT[act](z)
    lev = (a.clamp_max(1.0 - eps) * L).floor()
    q = (lev + 0.5) / L
    q = a + (q - a).detach()
    p_accept = None
    if quantize_rate < 1.0:
        prop = a + (1.0 / (L * 2)) * (torch.rand_like(a) * 2.0 - 1.0)
        ok = (prop > 0.0) & (prop < 1.0)
        p_accept = ok.float().mean()
        q = torch.where(torch.rand_like(q) > quantize_rate, torch.where(ok, prop, a), q)
    if inv:
        qz = _TORCH_INV[act](q.clamp(eps, 1.0 - eps))
        qz = z + (qz - z).detach()
    else:
        qz = (q - 0.5) / UNIT_STD
    return qz, lev.detach(), loss, stats, p_accept
