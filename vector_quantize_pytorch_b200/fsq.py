"""`FSQ` (finite_scalar_quantization.py of the reference, "fsq"): finite scalar quantization on the vqb_fsq_* kernels.

Everything per element runs in csrc/vq_fsq.cu: the bound (fsq:147-169), codes_to_indices (fsq:220-224), the straight-through
backward and indices -> codes (fsq:209-218).  The per-dimension constants the kernels take are computed here, once per device,
with the reference's own torch expressions on the CPU (`fsq_tables`), so the kernels only repeat the reference's per-element
operations.  project_in / project_out stay nn.Linear (torch), as VectorQuantize's projections do.  `num_codebooks` maps onto the
kernels' group axis: z (N, c, d) is one launch.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .codebook import _unsupported

def fsq_tables(levels: torch.Tensor, basis: torch.Tensor, sym: bool, hard: bool):
    """The fp32 constant table (7, d) and the int32 (levels, basis) table (2, d) of vqb_fsq_* (include/vqb200.h), from the FSQ
    buffers `_levels` / `_basis` on the CPU, with the expressions of fsq:152-156, :165-166, :197-207."""
    levels = levels.cpu()
    basis = basis.cpu()
    hw = (levels // 2).float()
    if sym:
        a = (levels - 1).float()
        b = 2. / (levels - 1)
        shift = torch.zeros_like(b)
        rb = 1 / b
    else:
        eps = 1e-3
        a = (levels - 1) * (1 + eps) / 2
        b = torch.where(levels % 2 == 0, 0.5, 0.0)
        shift = b / a if hard else torch.atanh(b / a)
        rb = torch.ones_like(a)
    consts = torch.stack([a, b, shift, hw, basis.float(), rb, 1 / hw]).float().contiguous()
    ints = torch.stack([levels.int(), basis.int()]).contiguous()
    return consts, ints


class _FSQFunction(torch.autograd.Function):
    """z (N, G, d) -> (out (N, G, d) in the chain's dtype, indices).  One vqb_fsq_forward; the backward recomputes the stages
    from z (vqb_fsq_backward), nothing but z is kept."""

    @staticmethod
    def forward(ctx, z, work_dtype, Q, n_active, sym, hard, consts, scales, clampv, indices):
        out = ops.fsq_forward(z, work_dtype, Q, n_active, sym, hard, consts, scales, clampv, indices)
        ctx.save_for_backward(z, consts, scales, clampv)
        ctx.cfg = (Q, n_active, sym, hard)
        return out

    @staticmethod
    def backward(ctx, g):
        z, consts, scales, clampv = ctx.saved_tensors
        Q, n_active, sym, hard = ctx.cfg
        gz = ops.fsq_backward(z, g, Q, n_active, sym, hard, consts, scales, clampv) if ctx.needs_input_grad[0] else None
        return (gz,) + (None,) * 9


def fsq_apply(z, work_dtype, Q, n_active, sym, hard, consts, scales, clampv, indices):
    """Runs the kernel pair on z (N, G, d) (made contiguous), indices written through their (N, G, Q) view `indices`;
    differentiable w.r.t. z."""
    z = ops.float_input(z, "FSQ", work_dtype=work_dtype)
    return _FSQFunction.apply(z, work_dtype, Q, n_active, sym, hard, consts, scales, clampv, indices)


class FSQ(nn.Module):
    """Drop-in for the reference's FSQ (fsq:64-320): same constructor, buffers (`_levels`, `_basis`, `implicit_codebook`,
    non-persistent), projections built in the same order (a seeded construction gives the same weights), same outputs and
    dtypes.  noise_dropout > 0, orthogonal_rotation and force_quantization_f32 = False are refused."""

    def __init__(self, levels, dim=None, num_codebooks=1, keep_num_codebooks_dim=None, scale=None,
                 allowed_dtypes=(torch.float32, torch.float64), channel_first=False, projection_has_bias=True, return_indices=True,
                 force_quantization_f32=True, preserve_symmetry=False, noise_dropout=0., bound_hard_clamp=False,
                 orthogonal_rotation=False):
        super().__init__()
        assert not (any([l == 2 for l in levels]) and not preserve_symmetry), \
            'turn on `preserve_symmetry` for using any levels == 2, or use a greater level'
        assert not (noise_dropout > 0 and not preserve_symmetry)
        if noise_dropout > 0:
            _unsupported("FSQ noise_dropout (per-element Bernoulli and uniform draws in training, fsq:179-193)")
        if orthogonal_rotation:
            _unsupported("FSQ orthogonal_rotation")
        if not force_quantization_f32:
            _unsupported("FSQ force_quantization_f32=False (quantizing in the input dtype)")
        if any(d not in (torch.float32, torch.float64) for d in allowed_dtypes):
            _unsupported("FSQ allowed_dtypes beyond float32 / float64 (quantizing in a low-precision dtype)")
        levels = list(levels)
        _levels = torch.tensor(levels, dtype=torch.int32)
        self.register_buffer('_levels', _levels, persistent=False)
        _basis = torch.cumprod(torch.tensor([1] + levels[:-1]), dim=0, dtype=torch.int32)
        self.register_buffer('_basis', _basis, persistent=False)
        self.scale = scale
        self.preserve_symmetry = preserve_symmetry
        self.noise_dropout = noise_dropout
        codebook_dim = len(levels)
        self.codebook_dim = codebook_dim
        effective_codebook_dim = codebook_dim * num_codebooks
        self.num_codebooks = num_codebooks
        self.effective_codebook_dim = effective_codebook_dim
        keep_num_codebooks_dim = num_codebooks > 1 if keep_num_codebooks_dim is None else keep_num_codebooks_dim
        assert not (num_codebooks > 1 and not keep_num_codebooks_dim)
        self.keep_num_codebooks_dim = keep_num_codebooks_dim
        self.dim = len(_levels) * num_codebooks if dim is None else dim
        self.channel_first = channel_first
        has_projections = self.dim != effective_codebook_dim
        self.project_in = nn.Linear(self.dim, effective_codebook_dim, bias=projection_has_bias) if has_projections else nn.Identity()
        self.project_out = nn.Linear(effective_codebook_dim, self.dim, bias=projection_has_bias) if has_projections else nn.Identity()
        self.has_projections = has_projections
        self.return_indices = return_indices
        if return_indices:
            self.codebook_size = self._levels.prod().item()
            implicit_codebook = self._indices_to_codes(torch.arange(self.codebook_size))
            self.register_buffer('implicit_codebook', implicit_codebook, persistent=False)
        self.allowed_dtypes = allowed_dtypes
        self.force_quantization_f32 = force_quantization_f32
        self.bound_hard_clamp = bound_hard_clamp
        self.orthogonal_rotation = orthogonal_rotation
        self._tables = ops.DeviceTables(self._make_tables)

    def _make_tables(self):
        return fsq_tables(self._levels, self._basis, self.preserve_symmetry, self.bound_hard_clamp)

    # ---- index helpers (fsq:195-245): small integer / elementwise torch expressions of the reference ----

    def _scale_and_shift(self, zhat_normalized):
        if self.preserve_symmetry:
            return (zhat_normalized + 1.) / (2. / (self._levels - 1))
        half_width = self._levels // 2
        return (zhat_normalized * half_width) + half_width

    def _scale_and_shift_inverse(self, zhat):
        if self.preserve_symmetry:
            return zhat * (2. / (self._levels - 1)) - 1.
        half_width = self._levels // 2
        return (zhat - half_width) / half_width

    def _indices_to_codes(self, indices):
        return self._scale_and_shift_inverse(self.indices_to_level_indices(indices))

    def indices_to_level_indices(self, indices):
        """Converts indices to indices at each level, perhaps needed for a transformer with factorized embeddings."""
        return (indices[..., None] // self._basis) % self._levels

    def codes_to_indices(self, zhat):
        """Converts a `code` to an index in the codebook."""
        assert zhat.shape[-1] == self.codebook_dim
        zhat = self._scale_and_shift(zhat)
        return (zhat * self._basis).sum(dim=-1).round().to(torch.int32)

    def _decode(self, indices):
        """vqb_fsq_decode of (..., c) or (...) indices -> fp32 codes (..., c, d)."""
        consts, ints = self._tables.get(indices.device)
        idx = indices.contiguous()
        lead = idx.shape
        codes, _ = ops.fsq_decode(idx.view(-1, 1, 1), self.codebook_dim, torch.float32, self.preserve_symmetry, consts, ints, None,
                                  True, False)
        return codes.reshape(*lead, self.codebook_dim)

    def indices_to_codes(self, indices):
        """Inverse of `codes_to_indices` (fsq:226-245)."""
        assert indices is not None
        is_img_or_video = indices.ndim >= (3 + int(self.keep_num_codebooks_dim))
        codes = self._decode(indices)
        if self.keep_num_codebooks_dim:
            codes = codes.reshape(*codes.shape[:-2], -1)
        codes = self.project_out(codes)
        if is_img_or_video or self.channel_first:
            codes = codes.movedim(-1, 1)
        return codes

    def forward(self, z):
        is_img_or_video = z.ndim >= 4
        need_move_channel_last = is_img_or_video or self.channel_first
        if need_move_channel_last:   # fsq:261-263
            z = z.movedim(1, -1)
            spatial = z.shape[1:-1]
            z = z.reshape(z.shape[0], -1, z.shape[-1])
        assert z.shape[-1] == self.dim, f'expected dimension of {self.dim} but found dimension of {z.shape[-1]}'
        z = self.project_in(z)
        lead = z.shape[:-1]
        c, d = self.num_codebooks, self.codebook_dim
        zf = z.reshape(-1, c, d)
        N = zf.shape[0]
        consts, _ = self._tables.get(z.device)
        indices = torch.empty((N, c), dtype=torch.int32, device=z.device)
        codes = fsq_apply(zf, z.dtype, 1, 1, self.preserve_symmetry, self.bound_hard_clamp, consts, None, None, indices.view(N, c, 1))
        out = self.project_out(codes.reshape(*lead, c * d))
        indices = indices.reshape(*lead, c)
        if need_move_channel_last:   # fsq:309-313
            out = out.reshape(out.shape[0], *spatial, out.shape[-1]).movedim(-1, 1)
            indices = indices.reshape(indices.shape[0], *spatial, c)
        if not self.return_indices:
            return out, None
        if not self.keep_num_codebooks_dim:
            indices = indices.squeeze(-1)
        return out, indices
