"""`FSP` (finite_scalar_perturbation.py of the reference, "fsp"): finite scalar perturbation on the vqb_fsp_* kernels.

Everything per element runs in csrc/vq_fsp.cu: the CDF activation, the quantization and the perturbation inside the bins
(fsp:323-351), the batch moments and VectorNorm's loss (fsp:93-140) and one backward for both.  The two uniform draws of the
perturbation are made here with torch, in the reference's order and dtype, so a seeded run consumes the generator exactly as
the reference does on the same device; the kernel reads them as two input planes.  project_in / project_out stay nn.Linear
(torch), as in FSQ.  One deliberate deviation: the index is the exact mixed-radix integer, where the reference sums
level_indices * basis in z's dtype (lossy in bf16, DESIGN 4.11).
"""
from __future__ import annotations

import math

import torch
from torch import nn

from . import ops
from .codebook import _unsupported

_ACTS = {"tanh": 0, "sigmoid": 1, "normal": 2, "laplace": 3, "cauchy": 4}
_MAX_D = 16

_PRESETS = {   # fsp:144-193
    "none": dict(l1_weight=0.0, l2_weight=0.0, l3_weight=0.0, l4_weight=0.0),
    "var": dict(l1_target=0.0, l1_weight=0.1, l2_target=1.0, l2_weight=0.07, l3_weight=0.0, l4_weight=0.0),
    "kurt": dict(l1_target=0.0, l1_weight=0.1, l2_target=1.0, l2_weight=0.07, l3_target=0.0, l3_weight=0.06, l4_target=0.0,
                 l4_weight=0.05),
    "var_tanh": dict(l1_target=0.0, l1_weight=0.1, l2_target=0.8225, l2_weight=0.07, l3_weight=0.0, l4_weight=0.0),
    "var_sigmoid": dict(l1_target=0.0, l1_weight=0.1, l2_target=3.29, l2_weight=0.07, l3_weight=0.0, l4_weight=0.0),
    "var_laplace": dict(l1_target=0.0, l1_weight=0.1, l2_target=2.0, l2_weight=0.07, l3_weight=0.0, l4_weight=0.0),
}


def _cast(v: float, dtype: torch.dtype) -> float:
    """A Python scalar as torch casts it to `dtype` for a comparison or a clamp."""
    return torch.tensor(v, dtype=torch.float64).to(dtype).item()


def _rand(z: torch.Tensor) -> torch.Tensor:
    """One perturbation draw, torch.rand_like of the reference's act_z / q_act_z (fsp:334, :340)."""
    return torch.rand_like(z)


class _FSPFunction(torch.autograd.Function):
    """z (N, d) -> (q (N, d), norm_loss, stats (4, d), indices, level indices, accept count).  One vqb_fsp_forward and one
    vqb_fsp_stats; the backward (vqb_fsp_backward) keeps z and the (d,) statistics, not the draws."""

    @staticmethod
    def forward(ctx, z, u1, u2, levels, act, inv, norm, clamp_hi, qrate, inv_lo, inv_hi, quantize):
        ctx.set_materialize_grads(False)
        stats, loss, aux = ops.fsp_stats(z, norm)
        if quantize:
            out, idx, lev, acc = ops.fsp_forward(z, act, inv, levels, clamp_hi, u1, u2, qrate, inv_lo, inv_hi)
        else:   # VectorNorm alone
            out = idx = lev = acc = None
        ctx.save_for_backward(z, aux)
        ctx.cfg = (act, inv, norm)
        ctx.mark_non_differentiable(*(t for t in (idx, lev, acc) if t is not None))
        return out, loss, stats, idx, lev, acc

    @staticmethod
    def backward(ctx, g_out, g_loss, g_stats, *_):
        z, aux = ctx.saved_tensors
        act, inv, norm = ctx.cfg
        gz = None
        if ctx.needs_input_grad[0]:
            gz = ops.fsp_backward(z, act, inv, g_out, aux, g_stats, g_loss, norm)
        return (gz,) + (None,) * 11


def fsp_stats_apply(z: torch.Tensor, norm):
    """VectorNorm on z (N, d): (norm_loss, stats (4, d)), differentiable w.r.t. z."""
    z = ops.float_input(z, "FSP")
    _, loss, stats, *_ = _FSPFunction.apply(z, None, None, None, 0, False, norm, 0., 0., 0., 0., False)
    return loss, stats


class VectorNorm(nn.Module):
    """The reference's VectorNorm (fsp:105-198): the targets and weights of the batch-moment loss as plain attributes."""

    def __init__(self, l1_target=0.0, l1_weight=0.1, l2_target=1.0, l2_weight=0.07, l3_target=0.0, l3_weight=0.06, l4_target=0.0,
                 l4_weight=0.05, eps=1e-8):
        super().__init__()
        self.l1_target, self.l1_weight = l1_target, l1_weight
        self.l2_target, self.l2_weight = l2_target, l2_weight
        self.l3_target, self.l3_weight = l3_target, l3_weight
        self.l4_target, self.l4_weight = l4_target, l4_weight
        self.eps = eps

    def norm_args(self):
        if self.eps != 1e-8:
            _unsupported("VectorNorm eps other than 1e-8 (the std clamp of batch_stats)")
        return (self.l1_target, self.l1_weight, self.l2_target, self.l2_weight, self.l3_target, self.l3_weight, self.l4_target,
                self.l4_weight)

    def forward(self, z):
        loss, stats = fsp_stats_apply(z, self.norm_args())
        mean, variance, skewness, kurtosis = stats.unbind(0)
        return loss, {"mean": mean, "variance": variance, "skewness": skewness, "kurtosis": kurtosis}

    @classmethod
    def build(cls, name):
        assert name in _PRESETS, f"unknown vector_norm preset: {name}, available: {list(_PRESETS.keys())}"
        return cls(**_PRESETS[name])


class FSP(nn.Module):
    """Drop-in for the reference's FSP (fsp:204-363): same constructor, non-persistent buffers (`_levels`, `_basis`),
    projections built in the same order (a seeded construction gives the same weights), same outputs and dtypes and the same
    generator use.  len(levels) > 16 and prod(levels) >= 2^31 are refused."""

    def __init__(self, levels, dim=None, channel_first=False, projection_has_bias=True, act_name="tanh", quantize_rate=0.0,
                 need_inv_act=False, vector_norm="var_tanh"):
        super().__init__()
        assert 0.0 <= quantize_rate <= 1.0, f"quantize_rate must be in [0.0, 1.0], got {quantize_rate}"
        levels = list(levels)
        if len(levels) > _MAX_D:
            _unsupported(f"FSP with more than {_MAX_D} levels")
        if math.prod(levels) >= 2 ** 31:
            _unsupported("FSP with prod(levels) >= 2^31 (the int32 basis would overflow)")
        codebook_dim = len(levels)
        self.codebook_dim = codebook_dim
        self.dim = codebook_dim if dim is None else dim
        self.channel_first = channel_first
        _levels = torch.tensor(levels, dtype=torch.int32)
        self.register_buffer("_levels", _levels, persistent=False)
        _basis = torch.cumprod(torch.tensor([1] + levels[:-1]), dim=0, dtype=torch.int32)
        self.register_buffer("_basis", _basis, persistent=False)
        self.codebook_size = _levels.prod().item()
        self.has_projections = self.dim != self.codebook_dim
        if self.has_projections:
            self.project_in = nn.Linear(self.dim, self.codebook_dim, bias=projection_has_bias)
            self.project_out = nn.Linear(self.codebook_dim, self.dim, bias=projection_has_bias)
        else:
            self.project_in = nn.Identity()
            self.project_out = nn.Identity()
        assert act_name in _ACTS, f"CDF activation {act_name} not available: {list(_ACTS.keys())}"
        self.act_name = act_name
        self.need_inv_act = need_inv_act
        self.quantize_rate = quantize_rate
        self.vector_norm = VectorNorm.build(vector_norm)

    def __repr__(self):
        return (
            f"FSP(\n"
            f"  levels={self._levels.tolist()},\n"
            f"  codebook_size={self.codebook_size},\n"
            f"  codebook_dim={self.codebook_dim},\n"
            f"  dim={self.dim},\n"
            f"  act_name='{self.act_name}',\n"
            f"  need_inv_act={self.need_inv_act},\n"
            f"  quantize_rate={self.quantize_rate}\n"
            f")"
        )

    # ---- index helpers (fsp:283-307) ----

    def level_indices_to_indices(self, level_indices):
        """The exact mixed-radix index (the reference sums level_indices * basis in their dtype)."""
        return (level_indices.to(torch.int64) * self._basis).sum(dim=-1).to(torch.int32)

    def indices_to_level_indices(self, indices):
        return (indices[..., None] // self._basis) % self._levels

    def _decode(self, indices, want_act, eps=1e-6):
        return ops.fsp_decode(indices, self.codebook_dim, _ACTS[self.act_name], self.need_inv_act, self._levels,
                              _cast(eps, torch.float32), _cast(1.0 - eps, torch.float32), want_act, not want_act)

    def indices_to_act_value(self, indices):
        return self._decode(indices, True)[0]

    def indices_to_codes(self, indices, eps: float = 1e-6):
        codes = self.project_out(self._decode(indices, False, eps)[1])
        if self.channel_first:
            codes = codes.movedim(-1, 1)
        return codes

    def forward(self, z, eps: float | None = None):
        eps = eps or torch.finfo(z.dtype).eps
        if self.channel_first:
            z = z.movedim(1, -1)
        z_shape = z.shape
        assert z_shape[-1] == self.dim, f"expected dimension of {self.dim} but found dimension of {z_shape[-1]}"
        z = z.reshape(-1, self.dim)
        z = self.project_in(z)
        z = ops.float_input(z, "FSP")
        quantize_rate = self.quantize_rate if self.training else 1.0
        perturb = quantize_rate < 1.0
        u1 = u2 = None
        if perturb:
            u1 = _rand(z)
            u2 = _rand(z)
        out_dtype = torch.float32 if perturb else z.dtype   # the fp32 p_max_norm promotes the output chain (fsp:333-341)
        q_z, norm_loss, stats, indices, level_indices, accepted = _FSPFunction.apply(
            z, u1, u2, self._levels, _ACTS[self.act_name], self.need_inv_act, self.vector_norm.norm_args(),
            _cast(1.0 - eps, z.dtype), _cast(quantize_rate, z.dtype), _cast(eps, out_dtype), _cast(1.0 - eps, out_dtype), True)
        mean, variance, skewness, kurtosis = stats.unbind(0)
        other_info = {}
        if perturb:
            other_info["p_accept_prob"] = accepted.float() / z.numel()
        q_z = self.project_out(q_z)
        level_indices = level_indices.reshape(z_shape[:-1] + (-1,))
        indices = indices.reshape(z_shape[:-1])
        q_z = q_z.reshape(z_shape)
        if self.channel_first:
            q_z = q_z.movedim(-1, 1)
        norm_info = {"mean": mean, "variance": variance, "skewness": skewness, "kurtosis": kurtosis}
        return q_z, indices, norm_loss, {"level_indices": level_indices, "norm_info": norm_info, **other_info}
