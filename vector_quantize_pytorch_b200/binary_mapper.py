"""`BinaryMapper` (binary_mapper.py of the reference, "bm"): `bits` logits per row -> a one-hot over 2^bits codes, trained
by a straight-through estimator (Fleuret, arXiv 2510.17558).

The O(rows * bits) work stays in torch in the reference's op order: the tempered probabilities, the Bernoulli draw (through
`_bernoulli`, so a seeded run consumes the generator exactly as the reference does on the same device), the index, the aux
loss and `log_prob`.  The O(rows * 2^bits) work runs in csrc/vq_binmap.cu: the output is a memset plus one row kernel that
writes the hot element, and the backward streams the upstream gradient once without building the (rows, 2^bits) soft codes
the reference's straight-through keeps (bm:173-180).  Only the logits are saved for the backward (DESIGN 4.12).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd.function import once_differentiable

from . import ops
from .codebook import _unsupported

_MAX_BITS = 20
NAT = math.log(2)


def binary_entropy(logits: torch.Tensor) -> torch.Tensor:
    """Sum over the last dim of the Bernoulli entropy of sigmoid(logits), in nats (bm:28-31)."""
    p = logits.sigmoid()
    return -(p * F.logsigmoid(logits) + (1. - p) * F.logsigmoid(-logits)).sum(dim=-1)


def _bernoulli(prob: torch.Tensor) -> torch.Tensor:
    """The sampled bits, prob.bernoulli() as the reference draws them (bm:153)."""
    return prob.bernoulli()


class _BinaryMapperST(torch.autograd.Function):
    """logits (rows, bits) fp32 contiguous, indices (rows,) int64 -> the straight-through one-hot (rows, 2^bits) fp32.  The
    backward (vqb_binmap_backward) keeps the logits alone."""

    @staticmethod
    def forward(ctx, logits, indices, num_codes):
        out = torch.zeros((logits.shape[0], num_codes), dtype=torch.float32, device=logits.device)
        ops.binmap_hot(out, logits, indices)
        ctx.save_for_backward(logits)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        logits, = ctx.saved_tensors
        return ops.binmap_backward(logits, g), None, None


class BinaryMapper(nn.Module):
    """Drop-in for the reference's BinaryMapper (bm:45-194): same constructor, non-persistent buffers (`power_two`, `codes`,
    `zero`), `num_codes`, methods and return shapes and dtypes.  Logits are fp32 or bf16 on a CUDA device; the straight-through
    path needs fp32 logits (the reference cannot run it on others either).  1 <= bits <= 20."""

    def __init__(self, bits=1, kl_loss_threshold=NAT, deterministic_on_eval=False):
        super().__init__()
        if not 1 <= bits <= _MAX_BITS:
            _unsupported(f"BinaryMapper with bits = {bits}: 1 to {_MAX_BITS} bits (at most 2^{_MAX_BITS} codes) are supported")
        self.bits = bits
        self.num_codes = 2 ** bits
        power_two = 2 ** torch.arange(bits)
        codes = (torch.arange(self.num_codes)[:, None] & power_two) != 0   # codes[k, j]: bit j of k, least significant first
        self.register_buffer("power_two", power_two, persistent=False)
        self.register_buffer("codes", codes, persistent=False)
        self.kl_loss_threshold = kl_loss_threshold
        self.register_buffer("zero", torch.tensor(0.), persistent=False)
        self.deterministic_on_eval = deterministic_on_eval

    def binary_entropy(self, logits):
        return binary_entropy(logits)

    def calc_aux_loss(self, logits, reduce_aux_kl_loss=True):
        """relu(bits ln 2 - H(logits) - threshold) per row (bm:75-87): its mean, or per row with the leading dims."""
        lead = logits.shape[:-1]
        kl = self.bits * NAT - self.binary_entropy(logits.reshape(-1, logits.shape[-1]))
        aux = F.relu(kl - self.kl_loss_threshold)
        return aux.mean() if reduce_aux_kl_loss else aux.reshape(lead)

    def log_prob(self, logits, *, indices=None, one_hot=None, sum_bits=True):
        """log P(code) under independent sigmoid(logits) bits (bm:89-122), per bit or summed; the code from `indices` or the
        argmax of `one_hot`."""
        assert (indices is None) != (one_hot is None), "either indices or one_hot must be provided"
        if one_hot is not None:
            indices = one_hot.argmax(dim=-1)
        lead = logits.shape[:-1]
        flat = logits.reshape(-1, logits.shape[-1])
        chosen = self.codes[indices.reshape(-1)]
        per_bit = torch.where(chosen, F.logsigmoid(flat), F.logsigmoid(-flat))
        if not sum_bits:
            return per_bit.reshape(logits.shape)
        return per_bit.sum(dim=-1).reshape(lead)

    def forward(self, logits, temperature=1., straight_through=None, calc_aux_loss=None, deterministic=None,
                return_indices=False, reduce_aux_kl_loss=True):
        if deterministic is None:
            deterministic = self.deterministic_on_eval and not self.training
        if straight_through is None:
            straight_through = self.training
        if calc_aux_loss is None:
            calc_aux_loss = self.training
        logits = ops.float_input(logits, "BinaryMapper", what="logits")
        if straight_through and logits.dtype != torch.float32:
            raise TypeError(f"BinaryMapper's straight-through needs float32 logits, got {logits.dtype}: the reference's einsum "
                            f"of {logits.dtype} log-sigmoids against the float code table cannot run either")
        assert logits.shape[-1] == self.bits, f"logits must have a last dimension of {self.bits}"
        lead = logits.shape[:-1]
        flat = logits.reshape(-1, self.bits)
        prob = (flat / temperature).sigmoid()
        sampled = (prob > 0.5).long() if deterministic else _bernoulli(prob).long()
        indices = (self.power_two * sampled).sum(dim=-1)
        aux = self.zero
        if calc_aux_loss:
            aux = self.calc_aux_loss(logits, reduce_aux_kl_loss=reduce_aux_kl_loss)
        if straight_through:
            one_hot = _BinaryMapperST.apply(flat, indices, self.num_codes)
        else:
            one_hot = ops.binmap_hot(torch.zeros((flat.shape[0], self.num_codes), dtype=torch.float32, device=flat.device),
                                     None, indices)
        one_hot = one_hot.reshape(*lead, self.num_codes)
        indices = indices.reshape(lead)
        if not return_indices:
            return one_hot, aux
        return one_hot, indices, aux
