"""`LFQ` (lookup_free_quantization.py of the reference, "lfq"): lookup-free quantization on the vqb_lfq_* kernels.

The row chain — the soft clamp, the spherical l2norm, the sign, the index bits, the straight-through value and, for a
ResidualLFQ, every stage's residual and running sum — is one vqb_lfq_forward launch over z (N, G, d), and its backward one
vqb_lfq_backward launch that recomputes the stages from z.  The entropy loss (lfq:347-403) never builds the (rows, K)
probabilities: vqb_lfq_entropy streams the codes once for the sum of h(p) and the column sums of p, and
vqb_lfq_entropy_backward streams them once more for the gradient (DESIGN §4.10).  What is left is on (c, K)-sized and scalar
tensors and stays torch: the entropy of the averages, the distributed mean, the softplus and the loss assembly, so autograd
carries their gradients into the two kernels.  project_in / project_out and the orthogonal rotation stay torch matmuls.
"""
from __future__ import annotations

from collections import namedtuple
from functools import partial
from math import ceil, log2

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn
from torch.distributed import nn as dist_nn

from . import ops
from .codebook import _unsupported

Return = namedtuple('Return', ['quantized', 'indices', 'entropy_aux_loss'])
LossBreakdown = namedtuple('LossBreakdown', ['per_sample_entropy', 'batch_entropy', 'commitment'])

MAX_CODEBOOK_DIM = 20


def is_distributed():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def maybe_distributed_mean(t):
    """The mean over the ranks of the per-rank (c, K) means: the autograd-aware all-reduce, divided by the world size.

    `dist_nn.all_reduce` is out of place (it reduces a copy and returns it).  lfq:41 discards that return value, so the
    reference divides its local mean by the world size; here the reduced mean is used, the cross-rank average the batch
    entropy is defined on (DESIGN §4.10).  Its backward all-reduces the gradient of the mean, which every rank holds equally."""
    if not is_distributed():
        return t
    return dist_nn.all_reduce(t) / dist.get_world_size()


def entropy(prob):
    """lfq:70-74 on a (c, K) tensor."""
    return (-prob * prob.clamp(min=1e-5).log()).sum(dim=-1)


def code_magnitude(scale: float, d: int, spherical: bool) -> float:
    """The fp32 magnitude of every code element: the scale, or l2norm(+-scale) * scale as the reference computes it."""
    if not spherical:
        return float(torch.tensor(scale, dtype=torch.float32))
    return float((F.normalize(torch.full((1, d), float(scale)), dim=-1) * scale)[0, 0])


class CosineSimLinear(nn.Module):
    """lfq:78-92."""

    def __init__(self, dim_in, dim_out, scale=1.):
        super().__init__()
        self.scale = scale
        self.weight = nn.Parameter(torch.randn(dim_in, dim_out))

    def forward(self, x):
        x = F.normalize(x, dim=-1)
        w = F.normalize(self.weight, dim=0)
        return (x @ w) * self.scale


class _LFQChain(torch.autograd.Function):
    """z (N, G, d) -> (out (N, G, d), entropy input (n_active, N, G, d) fp32 or None, commitment sums (n_active,) or None)."""

    @staticmethod
    def forward(ctx, z, Q, n_active, residual, training, spherical, params, indices, want_ent, rowmask, want_commit):
        ctx.set_materialize_grads(False)
        out, ent, commit = ops.lfq_forward(z, Q, n_active, residual, training, spherical, params, indices, want_ent, rowmask,
                                           want_commit)
        ctx.save_for_backward(z, params, rowmask)
        ctx.cfg = (Q, n_active, residual, training, spherical)
        return out, ent, commit

    @staticmethod
    def backward(ctx, g_out, g_ent, g_commit):
        z, params, rowmask = ctx.saved_tensors
        Q, n_active, residual, training, spherical = ctx.cfg
        if g_out is None:
            g_out = torch.zeros_like(z)
        cc = (2 * g_commit).float() if g_commit is not None else None
        gz = ops.lfq_backward(z, g_out, Q, n_active, residual, training, spherical, params, g_ent, cc, rowmask)
        return (gz,) + (None,) * 10


class _LFQEntropy(torch.autograd.Function):
    """Entropy inputs x (S, N, G, d) -> (sum over the rows of sum_k h(p) per (s, g) (S * G,) fp64, column sums of p (S * G, K)
    or None)."""

    @staticmethod
    def forward(ctx, x, rows, R, m, tau, want_col):
        ctx.set_materialize_grads(False)
        pse, col = ops.lfq_entropy(x, rows, R, m, tau, want_col)
        ctx.save_for_backward(x, rows, m)
        ctx.cfg = (R, tau)
        return pse, col

    @staticmethod
    def backward(ctx, g_pse, g_col):
        x, rows, m = ctx.saved_tensors
        R, tau = ctx.cfg
        S, _, G, _ = x.shape
        cp = g_pse.float() if g_pse is not None else torch.zeros(S * G, device=x.device)
        gx = ops.lfq_entropy_backward(x, rows, R, m, tau, cp, g_col)
        return gx, None, None, None, None, None


def lfq_chain(z, Q, n_active, residual, training, spherical, params, indices, want_ent, rowmask, want_commit):
    """Runs the row chain on z (N, G, d) (made contiguous and aligned); differentiable w.r.t. z."""
    z = ops.float_input(z, "LFQ")
    return _LFQChain.apply(z, Q, n_active, residual, training, spherical, params, indices, want_ent, rowmask, want_commit)


def sample_rows(num_tokens: int, frac: float):
    """lfq:365-370: the same CPU draw as the reference; -> the sampled positions (increasing), int64 on the CPU."""
    num_sampled = int(num_tokens * frac)
    rand_mask = torch.randn(num_tokens).argsort(dim=-1) < num_sampled
    return rand_mask.nonzero().flatten()


def entropy_losses(ent, mask, frac, tau, m, independent):
    """Per-sample and batch entropy (lfq:356-398) of every stage and group.  ent (S, N, G, d) fp32 stage inputs; mask (N,) bool
    or None; m (S,) code magnitudes.  independent: each (stage, group) is its own LFQ with one codebook (ResidualLFQ layers,
    GroupedResidualLFQ groups: one frac draw each, group-major); otherwise the G groups are the codebooks of one LFQ (S = 1).
    -> (PSE, CBE), each (S, G) fp32 and differentiable w.r.t. ent: the mean over the rows of sum_k h(p), and the entropy of the
    average p (with a mask, the reference's reduce leaves every row its own average: CBE = PSE)."""
    S, N, G, d = ent.shape
    dev = ent.device
    if mask is not None and is_distributed():
        raise NotImplementedError("vqb200 LFQ: mask= together with multi-GPU training (the reference all-reduces a per-row "
                                  "(M * c, K) tensor)")
    x = ent
    base = mask.nonzero().flatten() if mask is not None else None
    if mask is not None and not independent and G > 1:   # the (M * c) items of one LFQ's codebooks, as rows of one group
        base = (base[:, None] * G + torch.arange(G, device=dev)).flatten()
        x = ent.reshape(S, N * G, 1, d)
    num_tokens = base.numel() if base is not None else N
    rows, R = base, num_tokens
    if frac < 1.:
        draws = x.shape[2] * S if independent else 1
        order = [s * x.shape[2] + g for g in range(x.shape[2]) for s in range(S)] if independent else [0]
        picks = [None] * draws
        for sg in order:
            picks[sg] = sample_rows(num_tokens, frac)
        picks = torch.stack(picks).to(dev)
        rows = base[picks] if base is not None else picks
        R = picks.shape[1]
        if draws == 1:
            rows = rows[0]
    if rows is not None:
        rows = rows.int().contiguous()
    if R == 0:   # the reference's mean over no rows is NaN; an empty row list is an argument error of the kernels
        raise ValueError("vqb200 LFQ: the entropy loss has no rows (an all-false mask, or frac_per_sample_entropy * tokens < 1)")
    per_row = mask is not None
    pse, col = _LFQEntropy.apply(x, rows, R, m, tau, not per_row)
    if per_row:
        pse = (pse.view(S, -1).sum(1, keepdim=True) / (R * x.shape[2])).float().expand(S, G) if not independent else \
            (pse / R).float().view(S, G)
        return pse, pse
    pse = (pse / R).float().view(S, G)
    avg = maybe_distributed_mean((col / R).view(S, G, -1))
    return pse, entropy(avg)


class LFQ(nn.Module):
    """Drop-in for the reference's LFQ (lfq:96-468): same constructor, buffers (`mask`, `zero`, `codebook`, and `orthogonal_rot`
    when rotating), projections built in the same order, same outputs, dtypes and RNG consumption.  A straight-through
    activation other than nn.Identity, force_quantization_f32 = False and codebooks above 2^20 codes are refused."""

    def __init__(self, *, dim=None, codebook_size=None, entropy_loss_weight=0.1, commitment_loss_weight=0., diversity_gamma=1.,
                 straight_through_activation=nn.Identity(), num_codebooks=1, keep_num_codebooks_dim=None, codebook_scale=1.,
                 frac_per_sample_entropy=1., has_projections=None, projection_has_bias=True, soft_clamp_input_value=None,
                 cosine_sim_project_in=False, cosine_sim_project_in_scale=None, channel_first=None,
                 experimental_softplus_entropy_loss=False, entropy_loss_offset=5., spherical=False, force_quantization_f32=True,
                 orthogonal_rotation=False):
        super().__init__()
        assert dim is not None or codebook_size is not None, 'either dim or codebook_size must be specified for LFQ'
        assert codebook_size is None or log2(codebook_size).is_integer(), \
            f'your codebook size must be a power of 2 for lookup free quantization (suggested {2 ** ceil(log2(codebook_size))})'
        if type(straight_through_activation) is not nn.Identity:
            _unsupported("LFQ straight_through_activation other than nn.Identity")
        if not force_quantization_f32:
            _unsupported("LFQ force_quantization_f32=False (quantizing in the input dtype)")
        codebook_size = codebook_size if codebook_size is not None else 2 ** dim
        self.codebook_size = codebook_size
        codebook_dim = int(log2(codebook_size))
        if codebook_dim > MAX_CODEBOOK_DIM:
            _unsupported(f"LFQ codebook_size above 2^{MAX_CODEBOOK_DIM}")
        codebook_dims = codebook_dim * num_codebooks
        dim = dim if dim is not None else codebook_dims
        has_projections = has_projections if has_projections is not None else dim != codebook_dims
        if cosine_sim_project_in:
            cosine_sim_project_in = cosine_sim_project_in_scale if cosine_sim_project_in_scale is not None else codebook_scale
            project_in_klass = partial(CosineSimLinear, scale=cosine_sim_project_in)
        else:
            project_in_klass = partial(nn.Linear, bias=projection_has_bias)
        self.project_in = project_in_klass(dim, codebook_dims) if has_projections else nn.Identity()
        self.project_out = nn.Linear(codebook_dims, dim, bias=projection_has_bias) if has_projections else nn.Identity()
        self.has_projections = has_projections
        self.dim = dim
        self.codebook_dim = codebook_dim
        self.num_codebooks = num_codebooks
        keep_num_codebooks_dim = keep_num_codebooks_dim if keep_num_codebooks_dim is not None else num_codebooks > 1
        assert not (num_codebooks > 1 and not keep_num_codebooks_dim)
        self.keep_num_codebooks_dim = keep_num_codebooks_dim
        self.channel_first = channel_first
        self.activation = straight_through_activation
        self.spherical = spherical
        self.orthogonal_rotation = orthogonal_rotation
        if orthogonal_rotation:
            orthogonal_rot = torch.empty(codebook_dim, codebook_dim)
            nn.init.orthogonal_(orthogonal_rot)
            self.register_buffer('orthogonal_rot', orthogonal_rot)
        assert 0 < frac_per_sample_entropy <= 1.
        self.frac_per_sample_entropy = frac_per_sample_entropy
        self.diversity_gamma = diversity_gamma
        self.entropy_loss_weight = entropy_loss_weight
        self.codebook_scale = codebook_scale
        self.commitment_loss_weight = commitment_loss_weight
        self.soft_clamp_input_value = soft_clamp_input_value
        assert soft_clamp_input_value is None or soft_clamp_input_value >= codebook_scale
        self.entropy_loss_offset = entropy_loss_offset
        self.experimental_softplus_entropy_loss = experimental_softplus_entropy_loss
        self.register_buffer('mask', 2 ** torch.arange(codebook_dim - 1, -1, -1))
        self.register_buffer('zero', torch.tensor(0.), persistent=False)
        self.force_quantization_f32 = force_quantization_f32
        all_codes = torch.arange(codebook_size)
        bits = ((all_codes[..., None].int() & self.mask) != 0).float()
        self.register_buffer('codebook', self.bits_to_codes(bits).float(), persistent=False)
        self._magnitude = code_magnitude(codebook_scale, codebook_dim, spherical)
        self._params = ops.DeviceTables(self._make_params)

    def bits_to_codes(self, bits):
        return bits * self.codebook_scale * 2 - self.codebook_scale

    @property
    def dtype(self):
        return self.codebook.dtype

    def maybe_l2norm(self, t):
        return F.normalize(t, dim=-1) * self.codebook_scale if self.spherical else t

    def _make_params(self):
        """(3, 1) fp32: scale, code magnitude, soft-clamp value (0 when it is off, or runs in torch before the rotation)."""
        in_kernel_clamp = self.soft_clamp_input_value is not None and not self.orthogonal_rotation
        c = self.soft_clamp_input_value if in_kernel_clamp else 0.
        return (torch.tensor([[self.codebook_scale], [self._magnitude], [c]], dtype=torch.float32),)

    def _decode(self, indices):
        """vqb_lfq_decode of (..., c) indices -> fp32 codes (..., c, d), +-magnitude."""
        idx = indices.contiguous()
        lead = idx.shape
        vals = self._params.get(idx.device)[0][1]
        _, codes = ops.lfq_decode(idx.view(-1, 1, 1), self.codebook_dim, vals, False, True)
        return codes.reshape(*lead, self.codebook_dim)

    def indices_to_codes(self, indices, project_out=True):
        """lfq:228-263."""
        is_img_or_video = indices.ndim >= (3 + int(self.keep_num_codebooks_dim))
        should_transpose = self.channel_first if self.channel_first is not None else is_img_or_video
        if not self.keep_num_codebooks_dim:
            indices = indices[..., None]
        codes = self._decode(indices).to(self.dtype)
        if self.orthogonal_rotation:
            codes = codes @ self.orthogonal_rot.t()
        codes = codes.reshape(*codes.shape[:-2], -1)
        if project_out:
            codes = self.project_out(codes)
        if should_transpose:
            codes = codes.movedim(-1, 1)
        return codes

    def forward(self, x, inv_temperature=100., return_loss_breakdown=False, mask=None):
        is_img_or_video = x.ndim >= 4
        should_transpose = self.channel_first if self.channel_first is not None else is_img_or_video
        if should_transpose:   # 'b d ... -> b ... d', pack 'b * d'
            x = x.movedim(1, -1)
            spatial = x.shape[1:-1]
            x = x.reshape(x.shape[0], -1, x.shape[-1])
        assert x.shape[-1] == self.dim, f'expected dimension of {self.dim} but received {x.shape[-1]}'
        x = self.project_in(x)
        rot = self.orthogonal_rotation
        if rot and self.soft_clamp_input_value is not None:   # the clamp precedes the rotation: torch
            cv = self.soft_clamp_input_value
            x = (x / cv).tanh() * cv
        b, n = x.shape[0], x.shape[1]
        c, d = self.num_codebooks, self.codebook_dim
        z = x.reshape(b * n, c, d)
        if rot:
            z = z @ self.orthogonal_rot
        N = b * n
        train = self.training
        indices = torch.empty((N, c), dtype=torch.int64, device=z.device)
        flat_mask = mask.reshape(N) if mask is not None else None
        want_commit = train and self.commitment_loss_weight > 0.
        rowmask = flat_mask.to(torch.uint8) if (want_commit and flat_mask is not None) else None
        params, = self._params.get(z.device)
        out, ent, commit = lfq_chain(z, 1, 1, False, train, self.spherical, params, indices.view(N, c, 1), train, rowmask,
                                     want_commit)
        if train:
            m = params[1]
            pse, cbe = entropy_losses(ent, flat_mask, self.frac_per_sample_entropy, inv_temperature, m, False)
            per_sample_entropy, codebook_entropy = pse[0].mean(), cbe[0].mean()
            entropy_aux_loss = per_sample_entropy - self.diversity_gamma * codebook_entropy
        else:
            entropy_aux_loss = per_sample_entropy = codebook_entropy = self.zero
        if train and self.experimental_softplus_entropy_loss:
            entropy_aux_loss = F.softplus(entropy_aux_loss + self.entropy_loss_offset)
        if want_commit:
            count = (int(flat_mask.sum()) if flat_mask is not None else N) * c * d
            commit_loss = (commit[0] / count).float()
        else:
            commit_loss = self.zero
        if rot:
            out = out @ self.orthogonal_rot.t()
        out = self.project_out(out.reshape(b, n, c * d))
        indices = indices.reshape(b, n, c)
        if should_transpose:
            out = out.reshape(b, *spatial, out.shape[-1]).movedim(-1, 1)
            indices = indices.reshape(b, *spatial, c)
        if not self.keep_num_codebooks_dim:
            indices = indices.squeeze(-1)
        aux_loss = entropy_aux_loss * self.entropy_loss_weight + commit_loss * self.commitment_loss_weight
        ret = Return(out, indices, aux_loss)
        if not return_loss_breakdown:
            return ret
        return ret, LossBreakdown(per_sample_entropy, codebook_entropy, commit_loss)
