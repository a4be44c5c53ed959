"""`ResidualLFQ` and `GroupedResidualLFQ` (residual_lfq.py of the reference, "rlfq") on the vqb_lfq_* kernels.

Every stage of rlfq:179-193 — layer q's soft clamp, l2norm, sign, straight-through value, the residual and the running sum —
is one vqb_lfq_forward launch with the stages in registers; a GroupedResidualLFQ runs all its groups in that launch (z (N, G, d)),
and the entropy statistics of every (stage, group) in one vqb_lfq_entropy launch.  The backward is one vqb_lfq_entropy_backward
and one vqb_lfq_backward.  The layers are real `LFQ` modules (their buffers and configuration), built as the reference builds
them: codebook_scale 2^-q, the soft-clamp value halved per layer.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .lfq import LFQ, entropy_losses, lfq_chain
from .codebook import _unsupported
from .residual_common import GroupedResidual, get_maybe_sync_seed
from .residual_fsq import ResidualFSQ
import torch.nn.functional as F

MAX_QUANTIZERS = 64   # the stages the row kernels hold (vqb_lfq_forward)


class ResidualLFQ(nn.Module):
    """Drop-in for the reference's ResidualLFQ (rlfq:44-214): same constructor, `layers`, projections, outputs, dtypes and RNG
    consumption.  orthogonal_rotation in the layers is refused (it would put a matmul between the stages)."""

    def __init__(self, *, dim, num_quantizers, codebook_size, quantize_dropout=False, quantize_dropout_cutoff_index=0,
                 quantize_dropout_multiple_of=1, soft_clamp_input_value=None, **kwargs):
        super().__init__()
        if kwargs.get('orthogonal_rotation', False):
            _unsupported("ResidualLFQ with orthogonal_rotation")
        if num_quantizers > MAX_QUANTIZERS:
            _unsupported(f"ResidualLFQ with more than {MAX_QUANTIZERS} quantizers")
        codebook_dim = int(torch.tensor(codebook_size).log2().item())
        requires_projection = codebook_dim != dim
        self.project_in = nn.Linear(dim, codebook_dim) if requires_projection else nn.Identity()
        self.project_out = nn.Linear(codebook_dim, dim) if requires_projection else nn.Identity()
        self.has_projections = requires_projection
        self.num_quantizers = num_quantizers
        self.layers = nn.ModuleList([])
        for ind in range(num_quantizers):
            self.layers.append(LFQ(dim=codebook_dim, codebook_scale=2 ** -ind, soft_clamp_input_value=soft_clamp_input_value,
                                   **kwargs))
            if soft_clamp_input_value is not None:
                soft_clamp_input_value *= 0.5
        assert all([not lfq.has_projections for lfq in self.layers])
        self.quantize_dropout = quantize_dropout and num_quantizers > 1
        assert quantize_dropout_cutoff_index >= 0
        self.quantize_dropout_cutoff_index = quantize_dropout_cutoff_index
        self.quantize_dropout_multiple_of = quantize_dropout_multiple_of
        self.codebook_dim = codebook_dim
        self._params = ops.DeviceTables(self._make_params)

    _n_active = ResidualFSQ._n_active
    _decode = ResidualFSQ._decode
    get_codes_from_indices = ResidualFSQ.get_codes_from_indices
    get_output_from_indices = ResidualFSQ.get_output_from_indices

    @property
    def codebooks(self):
        return torch.stack([layer.codebook for layer in self.layers], dim=0)

    def _make_params(self):
        """(3, Q) fp32: per layer scale, code magnitude, soft-clamp value (0: none); and (Q,) the non-spherical code values."""
        rows = [[float(l.codebook_scale) for l in self.layers], [l._magnitude for l in self.layers],
                [float(l.soft_clamp_input_value or 0.) for l in self.layers]]
        t = torch.tensor(rows, dtype=torch.float32)
        return t, t[0].contiguous()

    def _launch(self, z, mask, n_active, grouped):
        """z (N, G, d) -> (out (N, G, d), indices (N, Q) or (G, N, Q) when `grouped`, losses (G, Q) fp32)."""
        N, G, d = z.shape
        Q = self.num_quantizers
        lay = self.layers[0]
        train = self.training
        params, _ = self._params.get(z.device)
        if grouped:
            indices = torch.empty((G, N, Q), dtype=torch.int64, device=z.device)
            view = indices.permute(1, 0, 2)
        else:
            indices = torch.empty((N, Q), dtype=torch.int64, device=z.device)
            view = indices.view(N, 1, Q)
        flat_mask = mask.reshape(N) if mask is not None else None
        want_commit = train and lay.commitment_loss_weight > 0.
        rowmask = flat_mask.to(torch.uint8) if (want_commit and flat_mask is not None) else None
        out, ent, commit = lfq_chain(z, Q, n_active, True, train, lay.spherical, params, view, train, rowmask, want_commit)
        if not train:
            return out, indices, torch.zeros((G, Q), device=z.device)
        pse, cbe = entropy_losses(ent, flat_mask, lay.frac_per_sample_entropy, 100., params[1, :n_active].contiguous(), True)
        aux = pse - lay.diversity_gamma * cbe                                   # (n_active, G)
        if lay.experimental_softplus_entropy_loss:
            aux = F.softplus(aux + lay.entropy_loss_offset)
        loss = aux * lay.entropy_loss_weight
        if want_commit:
            count = (int(flat_mask.sum()) if flat_mask is not None else N) * d
            loss = loss + (commit.view(n_active, 1) / count).float() * lay.commitment_loss_weight
        else:
            loss = loss + lay.zero * lay.commitment_loss_weight
        losses = torch.cat([loss.t(), torch.zeros((G, Q - n_active), device=z.device)], dim=1)
        return out, indices, losses

    def forward(self, x, mask=None, return_all_codes=False, rand_quantize_dropout_fixed_seed=None):
        n_active, _ = self._n_active(rand_quantize_dropout_fixed_seed, x.device)
        z = self.project_in(x)
        lead = z.shape[:-1]
        d = z.shape[-1]
        out, indices, losses = self._launch(z.reshape(-1, 1, d), mask, n_active, False)
        quantized_out = self.project_out(out.reshape(*lead, d))
        all_indices = indices.reshape(*lead, self.num_quantizers)
        ret = (quantized_out, all_indices, losses[0])
        if not return_all_codes:
            return ret
        return (*ret, self.get_codes_from_indices(all_indices))

    def _decode_rows(self, idx, want_sum, want_codes):
        """vqb_lfq_decode of (N, 1, Q) indices (rlfq:101-136): the layers' (non-spherical) `codebook` rows, zeros for dropped
        stages."""
        _, vals = self._params.get(idx.device)
        return ops.lfq_decode(idx, self.codebook_dim, vals, want_sum, want_codes)


class GroupedResidualLFQ(GroupedResidual):
    """Drop-in for the reference's GroupedResidualLFQ (rlfq:218-292): `groups` ResidualLFQs over column blocks of the features,
    all groups in one forward launch, one entropy launch and one backward chain."""

    def __init__(self, *, dim, groups=1, accept_image_fmap=False, **kwargs):
        if accept_image_fmap:
            _unsupported("GroupedResidualLFQ accept_image_fmap=True")
        super().__init__(ResidualLFQ, dim=dim, groups=groups, accept_image_fmap=accept_image_fmap, **kwargs)

    def forward(self, x, mask=None, return_all_codes=False):
        shape, split_dim, device = x.shape, self.split_dim, x.device
        assert shape[split_dim] == self.dim
        chunks = x.chunk(self.groups, dim=split_dim)
        seed = get_maybe_sync_seed(device) if self.training else None   # rlfq:275, shared by the groups
        n_act = [rvq._n_active(seed, device)[0] for rvq in self.rvqs]
        zs = [rvq.project_in(chunk) for rvq, chunk in zip(self.rvqs, chunks)]
        lead, d = zs[0].shape[:-1], zs[0].shape[-1]
        z = torch.stack([zz.reshape(-1, d) for zz in zs], dim=1)   # (N, G, d): one launch for every group
        first = self.rvqs[0]
        out, indices, losses = first._launch(z, mask, n_act[0], True)
        quantized = torch.cat([rvq.project_out(out[:, g].reshape(*lead, d)) for g, rvq in enumerate(self.rvqs)], dim=split_dim)
        all_indices = indices.reshape(self.groups, *lead, first.num_quantizers)
        ret = (quantized, all_indices, losses)
        if not return_all_codes:
            return ret
        return (*ret, tuple(rvq.get_codes_from_indices(i) for rvq, i in zip(self.rvqs, all_indices)))
