"""`RandomProjectionQuantizer` — drop-in for the reference's BEST-RQ target generator (random_projection_quantizer.py, "rpq";
arXiv:2202.01855): a frozen layer norm and random projection per codebook, then a cosine nearest code per codebook.

The layer norm and the projection are one sm_90a kernel (csrc/vq_rpq.cu, `ops.rpq_norm_project`) that writes the fp32 rows
the reference hands to its `VectorQuantize`; the normalised input is never written.  With more than one codebook the rows
then pass through `vq.project_in` (torch's nn.Linear, following torch's precision settings) and are searched head by head by
`VectorQuantize.eval_indices`, which writes neither the quantized rows nor runs `project_out`: the reference discards both.
fp32, (batch, seq, dim) inputs only, indices only.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .codebook import _unsupported
from .vector_quantize import VectorQuantize

_MAX_WIDTH = 1024   # the search's widest rows (DESIGN §4.1); it also needs a multiple of 8


class RandomProjectionQuantizer(nn.Module):
    """BEST-RQ targets (Chiu et al. 2022, arXiv:2202.01855): each of `num_codebooks` frozen random projections of the
    layer-normed frames picks its cosine-nearest code in its own codebook of `codebook_size` codes.  `kwargs` go to the
    inner `VectorQuantize`."""

    def __init__(
        self,
        *,
        dim,
        codebook_size,
        codebook_dim,
        num_codebooks=1,
        norm=True,
        **kwargs
    ):
        super().__init__()
        # the reference's VectorQuantize gets dim = codebook_dim * num_codebooks and no codebook_dim, so every head searches
        # rows of that width (rpq:37-44)
        width = codebook_dim * num_codebooks
        if width % 8 != 0 or width > _MAX_WIDTH:
            _unsupported(f"RandomProjectionQuantizer with a per-head width codebook_dim * num_codebooks = {width} (the search "
                         f"needs a multiple of 8 up to {_MAX_WIDTH})")
        self.num_codebooks = num_codebooks

        rand_projs = torch.empty(num_codebooks, dim, codebook_dim)
        nn.init.xavier_normal_(rand_projs)
        self.register_buffer('rand_projs', rand_projs)

        # nn.LayerNorm's eps (1e-5) is the one the kernel applies
        self.norm = nn.LayerNorm(dim, elementwise_affine=False) if norm else nn.Identity()

        self.vq = VectorQuantize(
            dim=width,
            heads=num_codebooks,
            codebook_size=codebook_size,
            use_cosine_sim=True,
            separate_codebook_per_head=True,
            **kwargs
        )

    @torch.no_grad()
    def forward(self, x, indices=None):
        """int64 indices of x (batch, seq, dim): (batch, seq) for one codebook, (batch, seq, num_codebooks) otherwise."""
        if indices is not None:
            _unsupported("RandomProjectionQuantizer.forward(indices=...) cross-entropy loss")
        if x.ndim != 3:
            raise TypeError(f"vqb200 RandomProjectionQuantizer expects (batch, seq, dim) inputs, got shape {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise TypeError(f"vqb200 RandomProjectionQuantizer supports float32 inputs, got {x.dtype}")
        b, n, _ = x.shape
        rows = ops.rpq_norm_project(x, self.rand_projs, isinstance(self.norm, nn.LayerNorm)).view(b, n, -1)
        self.vq.eval()   # rpq:56, on every call
        return self.vq.eval_indices(rows)
