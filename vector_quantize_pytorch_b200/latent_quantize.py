"""`LatentQuantize` (latent_quantization.py of the reference, "lq"): latent quantization on the vqb_lq_* kernels.

The per-latent value search, the straight-through codes z + (q - z) and the packed int32 index run in one kernel
(vqb_lq_quantize), from tables packed out of the *current* `values_per_latent`, so values loaded or edited after construction
are used by the next forward.  The two-sided mse loss and its gradient are vqb_lq_loss / vqb_lq_loss_backward; the loss makes
no host sync (which terms exist is decided from the weights given at construction).  project_in / project_out stay nn.Linear,
as in FSQ and VectorQuantize.  indices -> codes is the reference's torch expression (lq:194-209), bit for bit.  The values
never receive a gradient, as in the reference (lq:174).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import _C, ops
from .codebook import _unsupported


class _LQQuantize(torch.autograd.Function):
    """z (N, C * D) -> (codes (N, C * D) fp32, indices (N, C) int32); the straight-through gradient: d z = d codes in z's dtype."""

    @staticmethod
    def forward(ctx, z, C, vals, meta):
        codes, idx = ops.lq_quantize(z, C, vals, meta)
        ctx.z_dtype = z.dtype
        ctx.mark_non_differentiable(idx)
        return codes, idx

    @staticmethod
    def backward(ctx, g, _g_idx):
        gz = None if g is None or not ctx.needs_input_grad[0] else g.to(ctx.z_dtype)
        return gz, None, None, None


class _LQLoss(torch.autograd.Function):
    """w_c mse(x, out) + w_q mse(out, x) of the packed rows x (fp32 / bf16) and out (fp32): the quantization term's gradient
    goes to x, the commitment term's to out (lq:140-146, :293-308)."""

    @staticmethod
    def forward(ctx, x, out, wc, wq, use_c, use_q):
        x, out = x.contiguous(), out.contiguous()
        ctx.save_for_backward(x, out, wc, wq)
        ctx.use = (use_c, use_q)
        return ops.lq_loss(x, out, wc, wq, use_c, use_q)

    @staticmethod
    def backward(ctx, g):
        x, out, wc, wq = ctx.saved_tensors
        use_c, use_q = ctx.use
        want_x, want_out = ctx.needs_input_grad[0] and use_q, ctx.needs_input_grad[1] and use_c
        if not (want_x or want_out):
            return (None,) * 6
        gx, gout = ops.lq_loss_backward(x, out, g, wc, wq, use_c, use_q, want_x, want_out)
        return gx, gout, None, None, None, None


class LatentQuantize(nn.Module):
    """Drop-in for the reference's LatentQuantize (lq:28-310): same constructor, buffers, parameters (a seeded construction gives
    the reference's state_dict), outputs and dtypes.  The input is channel-first (b, dim, ...); returns (out (b, dim, ...),
    indices int32 (b, ..., c) or (b, ...), loss).  Refused (NotImplementedError): `in_place_codebook_optimizer` (the
    reference's branch reads an attribute it never sets, lq:264), prod(levels) >= 2^31 (the indices are int32), tables over
    the kernel's shared-memory cap, and inputs or tables that are not fp32 / bf16 (tables fp32)."""

    def __init__(self, levels, dim, commitment_loss_weight=0.1, quantization_loss_weight=0.1, num_codebooks=1,
                 codebook_dim=-1, keep_num_codebooks_dim=None, optimize_values=True, in_place_codebook_optimizer=None):
        super().__init__()
        if in_place_codebook_optimizer is not None:
            _unsupported("LatentQuantize in_place_codebook_optimizer (the reference's branch reads `self.optimize_values`, which "
                         "it never sets, lq:264)")
        self.dim = dim
        self.in_place_codebook_optimizer = in_place_codebook_optimizer
        _levels = torch.tensor(levels, dtype=torch.int32)
        if isinstance(levels, int):
            _levels = _levels.repeat(codebook_dim)   # RuntimeError for codebook_dim = -1, as in the reference
        if int(_levels.prod()) >= 2 ** 31:
            _unsupported(f"LatentQuantize with prod(levels) = {int(_levels.prod())} >= 2^31 (its indices are int32)")
        if len(_levels) > _C.VQB_LQ_MAX_DIM or int(_levels.sum()) > _C.VQB_LQ_MAX_VALUES:
            _unsupported(f"LatentQuantize value tables over the kernel's shared-memory cap ({len(_levels)} latents, "
                         f"{int(_levels.sum())} values; at most {_C.VQB_LQ_MAX_DIM} and {_C.VQB_LQ_MAX_VALUES})")
        self.register_buffer("commitment_loss_weight", torch.tensor(commitment_loss_weight, dtype=torch.float32),
                             persistent=False)
        self.register_buffer("quantization_loss_weight", torch.tensor(quantization_loss_weight, dtype=torch.float32),
                             persistent=False)
        self.register_buffer("_levels", _levels, persistent=False)
        _basis = torch.cumprod(torch.concat([torch.tensor([1], dtype=torch.int32), _levels[:-1]], dim=0), dim=0)
        self.register_buffer("_basis", _basis, persistent=False)
        self.codebook_dim = codebook_dim if codebook_dim > 0 else len(_levels)
        effective_codebook_dim = self.codebook_dim * num_codebooks
        self.num_codebooks = num_codebooks
        self.effective_codebook_dim = effective_codebook_dim
        keep_num_codebooks_dim = keep_num_codebooks_dim if keep_num_codebooks_dim else num_codebooks > 1   # lq:94-96
        assert not (num_codebooks > 1 and not keep_num_codebooks_dim)
        self.keep_num_codebooks_dim = keep_num_codebooks_dim
        has_projections = self.dim != effective_codebook_dim
        self.project_in = nn.Linear(self.dim, effective_codebook_dim) if has_projections else nn.Identity()
        self.project_out = nn.Linear(effective_codebook_dim, self.dim) if has_projections else nn.Identity()
        self.has_projections = has_projections
        self.codebook_size = self._levels.prod().item()
        all_indices = torch.arange(self.codebook_size)[:, None]
        implicit_codebook = self._scale_and_shift_inverse((all_indices // self._basis) % self._levels)
        self.register_buffer("implicit_codebook", implicit_codebook, persistent=False)
        values_per_latent = [torch.linspace(-0.5, 0.5, level) if level % 2 == 1 else torch.arange(level) / level - 0.5
                             for level in _levels]
        if optimize_values:
            self.values_per_latent = nn.ParameterList([nn.Parameter(values) for values in values_per_latent])
        else:
            self.values_per_latent = values_per_latent   # plain CPU tensors, not in the state_dict (lq:138)
        self.optimize_values = optimize_values
        self._weights_on = (float(commitment_loss_weight) != 0, float(quantization_loss_weight) != 0)
        self._hw_basis = ((_levels // 2).tolist(), _basis.tolist())   # host copies: building meta reads no device buffer
        self._meta = ops.DeviceTables(self._make_meta)
        self._host_tables = {}   # device -> (CPU snapshot, device copy) of CPU-held tables

    # ---- the reference's helpers (lq:140-209), as torch expressions ----

    def quantization_loss(self, z, zhat, reduce="mean"):
        return F.mse_loss(zhat.detach(), z, reduction=reduce)

    def commitment_loss(self, z, zhat, reduce="mean"):
        return F.mse_loss(z.detach(), zhat, reduction=reduce)

    def _scale_and_shift(self, zhat_normalized):
        half_width = self._levels // 2
        return (zhat_normalized * 2 * half_width) + half_width

    def _scale_and_shift_inverse(self, zhat):
        half_width = self._levels // 2
        return (zhat - half_width) / half_width / 2

    def codes_to_indices(self, zhat):
        """Converts a `code` which contains the number per latent to an index in the codebook."""
        assert zhat.shape[-1] == self.codebook_dim
        zhat = self._scale_and_shift(zhat)
        return (zhat * self._basis).sum(dim=-1).to(torch.int32)

    def indices_to_codes(self, indices, project_out=True):
        """Inverse of `codes_to_indices` (lq:194-209): the fixed lattice, not `values_per_latent`."""
        codes = self._scale_and_shift_inverse((indices[..., None] // self._basis) % self._levels)
        if self.keep_num_codebooks_dim:
            codes = codes.reshape(*codes.shape[:-2], -1)
        if project_out:
            codes = self.project_out(codes)
        return codes.movedim(-1, 1)

    # ---- the kernel path ----

    def _make_meta(self):
        """meta (3, D) int32 of vqb_lq_quantize: the current table lengths, half widths, basis (from host copies)."""
        return (torch.tensor([[v.numel() for v in self.values_per_latent], *self._hw_basis], dtype=torch.int32),)

    def _check_tables(self, values):
        """The reference's exceptions for tables that do not match codebook_dim: quantize indexes past the tables
        (IndexError, lq:160) and codes_to_indices broadcasts codes against more levels (RuntimeError, lq:181)."""
        if len(values) < self.codebook_dim:
            raise IndexError(f"LatentQuantize has {len(values)} value tables for codebook_dim {self.codebook_dim}")
        if len(values) > self.codebook_dim:
            raise RuntimeError(f"LatentQuantize codes of width {self.codebook_dim} do not broadcast against "
                               f"{len(values)} levels")
        if any(v.dtype != torch.float32 for v in values):
            _unsupported("LatentQuantize value tables that are not float32")
        lens = [v.numel() for v in values]
        if min(lens) < 1 or sum(lens) > _C.VQB_LQ_MAX_VALUES:
            _unsupported(f"LatentQuantize value tables of {sum(lens)} values (1 to {_C.VQB_LQ_MAX_VALUES} in all, none empty)")
        return tuple(lens)

    def _kernel_tables(self, device):
        """(vals, meta) of vqb_lq_quantize from the values as they are now, however they were changed (`.data` edits move no
        version counter).  Tables on the device are concatenated on every call, one small device copy and no host sync, as
        the reference reads them on every call; CPU-held tables (optimize_values=False) are compared by content with the
        snapshot last copied to this device, on the host, and copied again when they differ."""
        values = list(self.values_per_latent)
        lens = self._check_tables(values)
        meta = self._meta.get(device, key=lens)[0]
        if all(v.device == device for v in values):
            return torch.cat([v.detach().reshape(-1) for v in values]), meta
        snap = torch.cat([v.detach().reshape(-1).cpu() for v in values])
        held = self._host_tables.get(device)
        if held is None or held[0].shape != snap.shape or not torch.equal(held[0].view(torch.int32), snap.view(torch.int32)):
            held = self._host_tables[device] = (snap, snap.to(device))
        return held[1], meta

    def _loss_weights(self):
        """The two weights as fp32 device scalars for the kernels (a module cast to another dtype casts these buffers too),
        and the dtype of the reference's loss, w * mse: the weights' dtype promoted with fp32."""
        wc, wq = self.commitment_loss_weight, self.quantization_loss_weight
        dtype = torch.promote_types(torch.promote_types(wc.dtype, wq.dtype), torch.float32)
        return wc.float(), wq.float(), dtype

    def quantize(self, z):
        """Quantizes z (..., codebook_dim): the straight-through codes z + (q - z) in fp32 (lq:148-176)."""
        return self._quantize(z)[0]

    def _quantize(self, z):
        """(codes (..., D) fp32, indices (...) int32) of z (..., D) through the kernel, the codes straight-through to z."""
        lead = z.shape[:-1]
        vals, meta = self._kernel_tables(z.device)
        codes, idx = _LQQuantize.apply(z.reshape(-1, self.codebook_dim), 1, vals, meta)
        return codes.reshape(*lead, self.codebook_dim), idx.reshape(lead)

    def quantize_and_project(self, z, is_img_or_video, ps):
        """lq:211-225: z (b, n, c, d) -> (codes (b, n, c d), out (b, dim, *ps[0]), indices (b, *ps[0], c), the c axis dropped
        without keep_num_codebooks_dim).  ps: einops' packed shapes of the n axis, [spatial shape]."""
        codes, indices = self._quantize(z)
        b = z.shape[0]
        spatial = tuple(ps[0])
        codes = codes.reshape(*codes.shape[:2], -1)
        out = self.project_out(codes)
        out = out.reshape(b, *spatial, out.shape[-1]).movedim(-1, 1)
        indices = indices.reshape(b, *spatial, indices.shape[-1])
        if not self.keep_num_codebooks_dim:
            indices = indices.squeeze(-1)
        return codes, out, indices

    def forward(self, z):
        if z.dtype not in ops.FLOAT_DTYPES:
            _unsupported(f"LatentQuantize inputs of dtype {z.dtype} (float32 and bfloat16 only)")
        original_input = z
        b, spatial = z.shape[0], z.shape[2:]
        # 'b d ... -> b ... d', packed to (b, n, d): one contiguous copy, shared by the kernel and the loss
        z = z.movedim(1, -1).reshape(b, -1, z.shape[1]).contiguous()
        assert z.shape[-1] == self.dim, f"expected dimension of {self.dim} but found dimension of {z.shape[-1]}"
        x_rows = z
        z = self.project_in(z)
        n, c = z.shape[1], self.num_codebooks
        vals, meta = self._kernel_tables(z.device)
        codes, indices = _LQQuantize.apply(z.reshape(b * n, c * self.codebook_dim), c, vals, meta)
        out_rows = self.project_out(codes.view(b, n, c * self.codebook_dim))
        indices = indices.view(b, *spatial, c)
        if not self.keep_num_codebooks_dim:
            indices = indices.squeeze(-1)
        use_c, use_q = self._weights_on
        wc, wq, loss_dtype = self._loss_weights()
        if self.training and (use_c or use_q):
            loss = _LQLoss.apply(x_rows, out_rows, wc, wq, use_c, use_q).to(loss_dtype)
        else:
            loss = torch.zeros((), dtype=loss_dtype, device=original_input.device)
        out = out_rows.reshape(b, *spatial, out_rows.shape[-1]).movedim(-1, 1)
        return out, indices, loss
