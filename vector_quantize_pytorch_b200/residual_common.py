"""What the residual quantizer stacks (ResidualVQ, ResidualSimVQ, ResidualFSQ, ResidualLFQ) share with the reference's
residual modules: the quantize-dropout seed and cut, the -1 padding of dropped stages' indices, and the grouped wrapper."""
from __future__ import annotations

import math
import random

import torch
import torch.distributed as distributed
import torch.nn.functional as F
from torch import nn


def sync_seed(device) -> torch.Tensor:
    """The reference's seed draw (rvq:96-103, rfsq:39-45): one torch.randint on the device, all-reduced over the ranks.
    Returned as the device tensor: `.item()` synchronises with the device, so callers take the value only when they need it."""
    seed = torch.randint(0, 10_000, (), device=device)
    if distributed.is_available() and distributed.is_initialized() and distributed.get_world_size() > 1:
        distributed.all_reduce(seed)
    return seed


def get_maybe_sync_seed(device) -> int:
    """`sync_seed`'s value, as the reference's get_maybe_sync_seed returns it."""
    return sync_seed(device).item()


def dropout_cut(rvq, seed, device) -> int:
    """The number of leading layers a quantize-dropout forward of `rvq` runs (rvq:423-439, rfsq:204-223): python's
    random.Random(seed).randrange(cutoff, Q) is the last active layer, rounded up to a multiple of quantize_dropout_multiple_of
    (rvq:39-40); without a seed one is drawn by `get_maybe_sync_seed`."""
    Q = rvq.num_quantizers
    if seed is None:
        seed = get_maybe_sync_seed(device)
    index = random.Random(seed).randrange(rvq.quantize_dropout_cutoff_index, Q)
    mult = rvq.quantize_dropout_multiple_of
    if mult != 1:
        index = math.ceil((index + 1) / mult) * mult - 1
    return min(index + 1, Q)


def pad_dropped(indices, Q, quantize_dropout, message):
    """Coarse indices (fewer than Q columns) padded with -1 = "layer dropped"; only a quantize-dropout module takes them (the
    assertion `message` is the reference's wording)."""
    missing = Q - indices.shape[-1]
    if missing > 0:
        assert quantize_dropout, message
        indices = F.pad(indices, (0, missing), value=-1)
    return indices


class GroupedResidual(nn.Module):
    """The reference's grouped wrappers (rvq:634-724, rfsq:277-350, rlfq:218-292): `groups` residual quantizers of class
    `rvq_cls` over column blocks of the features, built in group order as `rvqs`."""

    def __init__(self, rvq_cls, *, dim, groups, accept_image_fmap, **kwargs):
        super().__init__()
        self.dim = dim
        self.groups = groups
        assert (dim % groups) == 0
        self.accept_image_fmap = accept_image_fmap
        self.rvqs = nn.ModuleList([rvq_cls(dim=dim // groups, **kwargs) for _ in range(groups)])

    @property
    def codebooks(self):
        return torch.stack(tuple(rvq.codebooks for rvq in self.rvqs))

    @property
    def split_dim(self):
        return 1 if self.accept_image_fmap else -1

    def get_codes_from_indices(self, indices):
        return torch.stack(tuple(rvq.get_codes_from_indices(i) for rvq, i in zip(self.rvqs, indices)))

    def get_output_from_indices(self, indices):
        return torch.cat(tuple(rvq.get_output_from_indices(i) for rvq, i in zip(self.rvqs, indices)), dim=self.split_dim)
