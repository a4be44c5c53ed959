"""`ResidualFSQ` and `GroupedResidualFSQ` (residual_fsq.py of the reference, "rfsq") on the vqb_fsq_* kernels.

The whole stage loop of rfsq:193-241 — the soft clamp, every stage's bound, indices, scaling, residual and running sum — is one
vqb_fsq_forward launch over the (N, d) rows with the Q stages in registers; a GroupedResidualFSQ runs all its groups in that one
launch (the groups are column blocks, z (N, G, d)).  The backward is one vqb_fsq_backward launch that recomputes the stages from
z.  Indices -> codes (get_codes_from_indices, get_output_from_indices) is vqb_fsq_decode.  The projections stay nn.Linear.

The chain's dtype follows torch's promotion exactly as the reference's expressions do: the soft-clamp value and the stage scales
are dimensioned fp32 buffers, so a bf16 input of an fp32 module is quantized, scaled and summed in fp32 (and quantized_out is
fp32); a module moved to bf16 runs the outer chain in bf16, rounding after every op, and each stage in fp32 (fsq:279-301).
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .fsq import FSQ, fsq_apply
from .residual_common import GroupedResidual, dropout_cut, get_maybe_sync_seed, pad_dropped


def _work_dtype(z_dtype, clampv, scales):
    """The dtype rfsq:195 and :234-239 compute in: torch's promotion of the input with the soft-clamp value, then the scales."""
    dt = z_dtype
    if clampv is not None:
        dt = torch.result_type(torch.empty(0, dtype=z_dtype), clampv)
    return torch.promote_types(dt, scales.dtype)


class ResidualFSQ(nn.Module):
    """Drop-in for the reference's ResidualFSQ (rfsq:49-273): same constructor and buffers (`scales`, `soft_clamp_input_value`),
    projections and `layers` built in the same order, same outputs, dtypes and RNG consumption (quantize dropout)."""

    def __init__(self, *, levels, num_quantizers, dim=None, is_channel_first=False, quantize_dropout=False,
                 quantize_dropout_cutoff_index=0, quantize_dropout_multiple_of=1, soft_clamp_input_value=None, bound_hard_clamp=True,
                 **kwargs):
        super().__init__()
        codebook_dim = len(levels)
        dim = codebook_dim if dim is None else dim
        requires_projection = codebook_dim != dim
        self.project_in = nn.Linear(dim, codebook_dim) if requires_projection else nn.Identity()
        self.project_out = nn.Linear(codebook_dim, dim) if requires_projection else nn.Identity()
        self.has_projections = requires_projection
        self.is_channel_first = is_channel_first
        self.num_quantizers = num_quantizers
        self.levels = levels
        self.layers = nn.ModuleList([])
        levels_tensor = torch.tensor(levels)
        assert (levels_tensor > 1).all()
        scales = []
        for ind in range(num_quantizers):
            scales.append(levels_tensor.float() ** -ind)
            self.layers.append(FSQ(levels=levels, dim=codebook_dim, preserve_symmetry=True, bound_hard_clamp=bound_hard_clamp,
                                   **kwargs))
        assert all([not fsq.has_projections for fsq in self.layers])
        self.codebook_size = self.layers[0].codebook_size
        self.register_buffer('scales', torch.stack(scales), persistent=False)
        self.quantize_dropout = quantize_dropout and num_quantizers > 1
        assert quantize_dropout_cutoff_index >= 0
        self.quantize_dropout_cutoff_index = quantize_dropout_cutoff_index
        self.quantize_dropout_multiple_of = quantize_dropout_multiple_of
        if bound_hard_clamp:
            assert soft_clamp_input_value is None
            soft_clamp_input_value = 1 + (1 / (levels_tensor - 1))
        if isinstance(soft_clamp_input_value, (list, float)):
            soft_clamp_input_value = torch.tensor(soft_clamp_input_value)
        self.register_buffer('soft_clamp_input_value', soft_clamp_input_value, persistent=False)
        self._scale_tables = ops.DeviceTables(self._make_scale_tables)

    def _make_scale_tables(self):
        """(2, Q, d) stage scales and their reciprocals, (2, d) soft-clamp value and reciprocal (None without a soft clamp): the
        values the reference's ops use (the buffers as stored; a 0-dim clamp value is broadcast), reciprocals in fp32."""
        d = len(self.levels)
        s = self.scales.detach().cpu().float()
        scales = torch.stack([s, 1 / s]).contiguous()
        c = self.soft_clamp_input_value
        if c is None:
            return scales, None
        c = c.detach().cpu().float().expand(d)
        return scales, torch.stack([c, 1 / c]).contiguous()

    @property
    def codebooks(self):
        return torch.stack([layer.implicit_codebook for layer in self.layers], dim=0)

    def _chain_dtype(self, z_dtype):
        return _work_dtype(z_dtype, self.soft_clamp_input_value, self.scales)

    def _codes_dtype(self):
        """dtype of get_codes_from_indices (rfsq:151-160): the implicit codebooks times the scales."""
        return torch.promote_types(self.layers[0].implicit_codebook.dtype, self.scales.dtype)

    def _n_active(self, seed, device):
        """Leading stages that quantize (rfsq:204-223): all, or with quantize dropout in training the sampled cut."""
        if not (self.training and self.quantize_dropout and torch.is_grad_enabled()):
            return self.num_quantizers, False
        return dropout_cut(self, seed, device), True

    def _pre(self, x):
        """Channel-first packing and project_in (rfsq:183-189): -> rows (N, d), and what _post needs to restore the layout."""
        spatial = None
        if self.is_channel_first:
            x = x.movedim(1, -1)
            spatial = x.shape[1:-1]
            x = x.reshape(x.shape[0], -1, x.shape[-1])
        z = self.project_in(x)
        return z.reshape(-1, z.shape[-1]), (z.shape[:-1], spatial)

    def _post(self, out, indices, layout):
        """project_out, then the channel-first layout back (rfsq:245-258)."""
        lead, spatial = layout
        out = self.project_out(out.reshape(*lead, out.shape[-1]))
        indices = indices.reshape(*lead, indices.shape[-1])
        if self.is_channel_first:
            out = out.reshape(out.shape[0], *spatial, out.shape[-1]).movedim(-1, 1)
            indices = indices.reshape(indices.shape[0], *spatial, indices.shape[-1]).movedim(-1, 1)
        return out, indices

    def _tables(self, device):
        c = self.soft_clamp_input_value
        consts, ints = self.layers[0]._tables.get(device)
        scales, clampv = self._scale_tables.get(device, (self.scales.dtype, None if c is None else c.dtype))
        return consts, ints, scales, clampv

    def _launch(self, z, n_active, dropped, grouped):
        """One vqb_fsq_forward over z (N, G, d) -> (out (N, G, d), indices (N, Q), or (G, N, Q) when `grouped`)."""
        N, G, _ = z.shape
        Q = self.num_quantizers
        work = self._chain_dtype(z.dtype)
        consts, _, scales, clampv = self._tables(z.device)
        # torch.stack of the int32 stage indices with the int64 null indices of the dropped stages (rfsq:223, :249) is int64
        idx_dtype = torch.int64 if dropped and n_active < Q else torch.int32
        if grouped:
            indices = torch.empty((G, N, Q), dtype=idx_dtype, device=z.device)
            view = indices.permute(1, 0, 2)
        else:
            indices = torch.empty((N, Q), dtype=idx_dtype, device=z.device)
            view = indices.view(N, 1, Q)
        out = fsq_apply(z, work, Q, n_active, True, self.layers[0].bound_hard_clamp, consts, scales, clampv, view)
        return out, indices

    def forward(self, x, return_all_codes=False, rand_quantize_dropout_fixed_seed=None):
        n_active, dropped = self._n_active(rand_quantize_dropout_fixed_seed, x.device)
        z, layout = self._pre(x)
        N, d = z.shape
        out, indices = self._launch(z.reshape(N, 1, d), n_active, dropped, False)
        quantized_out, all_indices = self._post(out.reshape(N, d), indices, layout)
        ret = (quantized_out, all_indices)
        if not return_all_codes:
            return ret
        return (*ret, self.get_codes_from_indices(all_indices))

    def _decode(self, indices, want_sum, want_codes):
        """'b ... q' indices (rfsq:131-171, rlfq:101-136) through `_decode_rows`: -> (sum (b, ..., d) or None, codes
        (Q, b, ..., d) or None)."""
        Q = self.num_quantizers
        indices = pad_dropped(indices, Q, self.quantize_dropout,
                              'quantize dropout must be greater than 0 if you wish to reconstruct from a signal with less fine '
                              'quantizations')
        lead = indices.shape[:-1]
        flat = indices.reshape(-1, indices.shape[-1]).contiguous()
        s, codes = self._decode_rows(flat.view(flat.shape[0], 1, Q), want_sum, want_codes)
        s = s.reshape(*lead, s.shape[-1]) if s is not None else None
        codes = codes.reshape(Q, *lead, codes.shape[-1]) if codes is not None else None
        return s, codes

    def _decode_rows(self, idx, want_sum, want_codes):
        """vqb_fsq_decode of (N, 1, Q) indices."""
        consts, ints, scales, _ = self._tables(idx.device)
        return ops.fsq_decode(idx, len(self.levels), self._codes_dtype(), True, consts, ints, scales, want_sum, want_codes)

    def get_codes_from_indices(self, indices):
        return self._decode(indices, False, True)[1]

    def get_output_from_indices(self, indices):
        return self.project_out(self._decode(indices, True, False)[0])


class GroupedResidualFSQ(GroupedResidual):
    """Drop-in for the reference's GroupedResidualFSQ (rfsq:277-350): `groups` ResidualFSQs over column blocks of the features.
    The forward is ONE vqb_fsq_forward launch for all groups (and one backward launch); the indices come out as
    torch.stack of the groups' (G, b, ..., Q)."""

    def __init__(self, *, dim, groups=1, accept_image_fmap=False, **kwargs):
        super().__init__(ResidualFSQ, dim=dim, groups=groups, accept_image_fmap=accept_image_fmap, **kwargs)
        self.codebook_size = self.rvqs[0].codebook_size

    def forward(self, x, return_all_codes=False):
        shape, split_dim, device = x.shape, self.split_dim, x.device
        assert shape[split_dim] == self.dim
        chunks = x.chunk(self.groups, dim=split_dim)
        seed = get_maybe_sync_seed(device) if self.training else None   # rfsq:334, shared by the groups
        pre = [rvq._pre(chunk) for rvq, chunk in zip(self.rvqs, chunks)]
        n_act = [rvq._n_active(seed, device) for rvq in self.rvqs]
        z = torch.stack([p[0] for p in pre], dim=1)   # (N, G, d): one launch for every group
        first = self.rvqs[0]
        if any(n != n_act[0] for n in n_act) or any(r.layers[0].bound_hard_clamp != first.layers[0].bound_hard_clamp or
                                                    r._chain_dtype(z.dtype) != first._chain_dtype(z.dtype) for r in self.rvqs):
            raise ValueError("GroupedResidualFSQ: the groups must share their configuration")
        n_active, dropped = n_act[0]
        out, indices = first._launch(z, n_active, dropped, True)
        outs, idxs = [], []
        for g, (rvq, (_, layout)) in enumerate(zip(self.rvqs, pre)):
            o, i = rvq._post(out[:, g], indices[g], layout)
            outs.append(o)
            idxs.append(i)
        quantized = torch.cat(outs, dim=split_dim)
        all_indices = torch.stack(idxs)
        if not return_all_codes:
            return quantized, all_indices
        # rfsq:340-349: the third output is the tuple of the groups' all_codes, as zip(*out) leaves it
        return quantized, all_indices, tuple(rvq.get_codes_from_indices(i) for rvq, i in zip(self.rvqs, idxs))
