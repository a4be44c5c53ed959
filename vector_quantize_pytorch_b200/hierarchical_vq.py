"""`HierarchicalVQ` — drop-in for the reference's multi-scale residual VQ over image feature maps (hierarchical_vq.py, "hvq").

At every scale the running residual is pooled to (s, s), searched by ONE shared `VectorQuantize` (search, EMA update, k-means
init, dead-code expiry and the rotation trick are that module's kernels), upsampled back to (H, W), passed through phi and
added to the reconstruction / subtracted from the residual (hvq:133-147).  The pool, the upsample and the residual update are
the sm_90a kernels of csrc/vq_hvq.cu: the pool writes the channel-last rows the search reads (the (B, D, s, s) map handed to
`vq` is a view of them), the upsample reads the rows the search wrote and, for the identity phi, also writes recon + q and
residual - q; the blended phi's (1 - r) q + r conv(q) and both updates are one more pass.  phi's 3x3 conv stays nn.Conv2d.
fp32 only.
"""
from __future__ import annotations

from typing import Sequence

import torch
from torch import nn

from . import ops
from .codebook import _unsupported
from .vector_quantize import VectorQuantize

_MAX_DIM = 1024   # the search's widest rows (DESIGN §4.1); it also needs dim % 8 == 0


class _Pool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, s):
        ctx.hw = x.shape[-2:]
        return ops.hvq_pool(x, s)

    @staticmethod
    def backward(ctx, g):
        return ops.hvq_pool_backward(g, *ctx.hw), None


class _Upsample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, H, W):
        ctx.s = q.shape[-1]
        return ops.hvq_upsample(q, H, W)[0]

    @staticmethod
    def backward(ctx, g):
        return ops.hvq_upsample_backward(g, None, ctx.s), None, None


class _UpsampleUpdate(torch.autograd.Function):
    """(recon + u, resid - u) with u = upsample(q) (the identity phi); recon None: 0 + u; resid None: recon + u alone."""

    @staticmethod
    def forward(ctx, q, recon, resid, H, W):
        ctx.set_materialize_grads(False)
        ctx.s = q.shape[-1]
        ctx.two = resid is not None
        _, recon_out, resid_out = ops.hvq_upsample(q, H, W, recon, resid, want_q=False, want_recon=True, want_resid=ctx.two)
        return (recon_out, resid_out) if ctx.two else recon_out

    @staticmethod
    def backward(ctx, g_recon, g_resid=None):
        if g_recon is None and g_resid is None:
            return None, None, None, None, None
        need = ctx.needs_input_grad
        g_q = ops.hvq_upsample_backward(g_recon, g_resid, ctx.s) if need[0] else None
        return g_q, g_recon if need[1] else None, g_resid if need[2] else None, None, None


class _BlendUpdate(torch.autograd.Function):
    """(recon + q, resid - q) with q = (1 - r) up + r conv (hvq:25); recon None: 0 + q; resid None: recon + q alone."""

    @staticmethod
    def forward(ctx, up, conv, recon, resid, r):
        ctx.set_materialize_grads(False)
        ctx.r = r
        ctx.two = resid is not None
        recon_out, resid_out = ops.hvq_blend_update(up, conv, r, recon, resid, want_resid=ctx.two)
        return (recon_out, resid_out) if ctx.two else recon_out

    @staticmethod
    def backward(ctx, g_recon, g_resid=None):
        if g_recon is None and g_resid is None:
            return None, None, None, None, None
        need = ctx.needs_input_grad
        g_up, g_conv = ops.hvq_blend_backward(g_recon, g_resid, ctx.r) if need[0] or need[1] else (None, None)
        return g_up, g_conv, g_recon if need[2] else None, g_resid if need[3] else None, None


class _Phi2D(nn.Module):
    """hvq:16-25.  The conv is built even when the ratio makes phi the identity, so construction draws from the RNG like the
    reference's; `HierarchicalVQ` applies the blend itself, fused with the residual update."""

    def __init__(self, dim: int, resi_ratio: float):
        super().__init__()
        self.resi_ratio = float(abs(resi_ratio))
        self.conv = nn.Conv2d(dim, dim, 3, padding=1)

    @property
    def is_identity(self) -> bool:
        return self.resi_ratio <= 1e-8


class HierarchicalVQ(nn.Module):
    def __init__(
        self,
        *,
        dim: int,
        codebook_size: int,
        scales: Sequence[int],
        decay: float = 0.99,
        commitment_weight: float = 1.,
        rotation_trick: bool = False,
        kmeans_init: bool = True,
        kmeans_iters: int = 10,
        threshold_ema_dead_code: int = 2,
        stochastic_sample_codes: bool = False,
        sample_codebook_temp: float = 0.1,
        orthogonal_reg_weight: float = 0.,
        orthogonal_reg_max_codes: int = 128,
        orthogonal_reg_active_codes_only: bool = False,
        quant_resi: float = 0.5,
        share_quant_resi: int = 1,
        accept_image_fmap: bool = False
    ):
        super().__init__()
        assert accept_image_fmap, 'HierarchicalVQ currently expects accept_image_fmap = True'

        scales = [int(scale) for scale in scales]
        assert len(scales) > 0
        assert scales == sorted(scales)
        assert all(scale > 0 for scale in scales)

        if dim % 8 != 0 or dim > _MAX_DIM:
            _unsupported(f"HierarchicalVQ with dim = {dim} (the search needs a multiple of 8 up to {_MAX_DIM})")

        self.dim = dim
        self.scales = tuple(scales)
        self.accept_image_fmap = True

        self.vq = VectorQuantize(
            dim=dim,
            codebook_size=codebook_size,
            decay=decay,
            commitment_weight=commitment_weight,
            rotation_trick=rotation_trick,
            kmeans_init=kmeans_init,
            kmeans_iters=kmeans_iters,
            threshold_ema_dead_code=threshold_ema_dead_code,
            stochastic_sample_codes=stochastic_sample_codes,
            sample_codebook_temp=sample_codebook_temp,
            orthogonal_reg_weight=orthogonal_reg_weight,
            orthogonal_reg_max_codes=orthogonal_reg_max_codes,
            orthogonal_reg_active_codes_only=orthogonal_reg_active_codes_only,
            accept_image_fmap=True
        )

        if share_quant_resi == 1:
            self.phi_shared = _Phi2D(dim, quant_resi)
            self.phi_levels = None
        else:
            num_phi_levels = len(self.scales) if share_quant_resi <= 0 else min(len(self.scales), int(share_quant_resi))
            self.phi_shared = None
            self.phi_levels = nn.ModuleList([_Phi2D(dim, quant_resi) for _ in range(num_phi_levels)])

    def _choose_phi(self, scale_index: int):  # hvq:87-102 (Python's round: ties to even)
        if self.phi_shared is not None:
            return self.phi_shared

        assert self.phi_levels is not None

        if len(self.phi_levels) == len(self.scales):
            return self.phi_levels[scale_index]

        if len(self.scales) == 1:
            return self.phi_levels[0]

        position = scale_index / float(len(self.scales) - 1)
        phi_index = round(position * (len(self.phi_levels) - 1))
        phi_index = max(0, min(len(self.phi_levels) - 1, phi_index))
        return self.phi_levels[phi_index]

    def _add_scale(self, q, recon, resid, full_hw, scale_index: int):
        """hvq:104-112, :143-144: upsample q to full_hw, apply phi, return (recon + q, resid - q), or recon + q alone when
        resid is None.  recon None counts as zeros."""
        H, W = full_hw
        phi = self._choose_phi(scale_index)
        if phi.is_identity:
            return _UpsampleUpdate.apply(q, recon, resid, H, W)
        up = _Upsample.apply(q, H, W)
        return _BlendUpdate.apply(up, phi.conv(up), recon, resid, phi.resi_ratio)

    def forward(self, x, indices=None, sample_codebook_temp=None, **kwargs):
        assert indices is None, 'reconstruction-from-indices path not implemented in forward'
        del kwargs

        assert x.ndim == 4, 'expected image fmap of shape (batch, channels, height, width)'
        batch, dim, height, width = x.shape
        assert dim == self.dim
        if x.dtype != torch.float32:
            raise TypeError(f"vqb200 HierarchicalVQ supports float32 inputs, got {x.dtype}")
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")

        vq_kwargs = {} if sample_codebook_temp is None else dict(sample_codebook_temp=sample_codebook_temp)
        residual = x.contiguous()
        reconstruction = None
        all_indices = []
        all_commit_losses = []
        last = len(self.scales) - 1

        for scale_index, scale in enumerate(self.scales):
            residual_down = _Pool.apply(residual, scale)
            quantized, scale_indices, commit_loss = self.vq(residual_down, **vq_kwargs)
            # the residual after the last scale is never read: only the reconstruction is written then
            out = self._add_scale(quantized, reconstruction, residual if scale_index < last else None, (height, width),
                                  scale_index)
            reconstruction, residual = out if scale_index < last else (out, None)
            all_indices.append(scale_indices)
            all_commit_losses.append(commit_loss)

        if self.training:
            mean_commit_loss = torch.stack(all_commit_losses).mean()
        else:   # VectorQuantize's eval loss is its constant zero at every scale: their mean is that zero
            mean_commit_loss = all_commit_losses[0]
        return reconstruction, tuple(all_indices), mean_commit_loss

    def get_output_from_indices(self, indices):  # hvq:152-170: always rebuilt at (scales[-1], scales[-1])
        assert isinstance(indices, (tuple, list))
        assert len(indices) == len(self.scales)

        first = indices[0]
        assert first.ndim == 3
        full_hw = (self.scales[-1], self.scales[-1])

        reconstructed = None
        for scale_index, scale_indices in enumerate(indices):
            q = self.vq.get_output_from_indices(scale_indices)
            reconstructed = self._add_scale(q, reconstructed, None, full_hw, scale_index)

        return reconstructed
