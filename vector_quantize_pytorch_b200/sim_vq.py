"""SimVQ (sim_vq.py of the reference, SURVEY §8f): a frozen random codebook seen through a learned linear map.  The search
— `torch.cdist` + `argmin` over the implicit codebook (sim_vq.py:111-113) — runs on the same tensor-core kernel with the same
exact re-score as VectorQuantize; everything that carries gradient (the gather from the implicit codebook, the two commitment
terms, the rotation trick / straight-through estimator, sim_vq.py:117-132) stays autograd glue around it."""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .vector_quantize import rotate_to


class SimVQ(nn.Module):
    def __init__(self, dim, codebook_size, codebook_transform: nn.Module | None = None, init_fn=lambda t: t, channel_first=False,
                 rotation_trick=True, input_to_quantize_commit_loss_weight=0.25, commitment_weight=1., frozen_codebook_dim=None):
        super().__init__()
        self.codebook_size = codebook_size
        self.channel_first = channel_first
        frozen_codebook_dim = dim if frozen_codebook_dim is None else frozen_codebook_dim
        codebook = torch.randn(codebook_size, frozen_codebook_dim) * (frozen_codebook_dim ** -0.5)   # sim_vq.py:57
        codebook = init_fn(codebook)
        if codebook_transform is None:
            codebook_transform = nn.Linear(frozen_codebook_dim, dim, bias=False)
        self.code_transform = codebook_transform
        self.register_buffer("frozen_codebook", codebook)
        self.rotation_trick = rotation_trick
        self.input_to_quantize_commit_loss_weight = input_to_quantize_commit_loss_weight
        self.commitment_weight = commitment_weight

    @property
    def codebook(self):  # sim_vq.py:81-83
        return self.code_transform(self.frozen_codebook)

    def indices_to_codes(self, indices):  # sim_vq.py:85-97
        quantized = self.code_transform(self.frozen_codebook[indices])
        if self.channel_first:
            quantized = quantized.movedim(-1, 1)
        return quantized

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        if self.channel_first:
            x = x.movedim(1, -1)
        shape = x.shape
        x = x.reshape(shape[0], -1, shape[-1])                     # pack 'b * d'
        implicit_codebook = self.codebook
        with torch.no_grad():                                       # sim_vq.py:111-113: argmin of cdist == our arg-max search
            flat = x.detach().reshape(-1, shape[-1])
            if flat.dtype not in (torch.float32, torch.bfloat16):
                flat = flat.float()
            flat = flat.contiguous()
            embed = implicit_codebook.detach().float().contiguous()
            cb = ops.prepare_codebook(embed, False)
            indices = ops.search(flat, cb, embed).idx.long().reshape(x.shape[:-1])
        quantized = implicit_codebook[indices]                      # sim_vq.py:117
        commit_loss = (F.mse_loss(x.detach(), quantized) +
                       F.mse_loss(x, quantized.detach()) * self.input_to_quantize_commit_loss_weight)   # sim_vq.py:121-124
        if self.rotation_trick:
            quantized = rotate_to(x, quantized)                     # sim_vq.py:126-128
        else:
            quantized = (quantized - x).detach() + x
        quantized = quantized.reshape(shape)
        indices = indices.reshape(shape[:-1])
        if self.channel_first:
            quantized = quantized.movedim(-1, 1)
        return quantized, indices, commit_loss * self.commitment_weight
