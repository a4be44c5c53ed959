"""`ResidualSimVQ` (residual_sim_vq.py of the reference, rsv): a stack of `SimVQ` layers quantizing the residual in turn.

The forward is one vqb_rvq_forward program (one FFI call, one cached CUDA graph): per stage, the search of the residual against
the stage's implicit codebook (the VQB_RVQ_STAGE op; with `update = 1` when the codebooks need a gradient, so that the stage's
per-code statistics [count | sum of residual rows] come out of it) and the stage tail (vqb_rsimvq_tail: gradient-estimator value,
next residual, running sum, commitment loss).  The backward is one row kernel over all stages (vqb_rsimvq_backward) that
recomputes the residuals from x; the codebook gradients are K x D elementwise ops on the forward's statistics, and autograd
carries them into each layer's `code_transform`.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .residual_common import pad_dropped
from .residual_vq import ResidualVQ, _PlanCache
from .sim_vq import SimVQ


class _Plan:
    """The cached program of one forward configuration on one device.  It owns every buffer its ops keep pointing into — codebook
    operands, the residual ping-pong, loss scratch and, through its program, the search's scratch (index and workspace) — so
    they are freed together with the plan; the per-call pointers (input, codebooks, outputs, statistics) are patched by `run`
    before every launch."""

    def __init__(self, mod, N, D, K, n_active, want_stats, device):
        Q = mod.num_quantizers
        self.N, self.D, self.K, self.Q, self.n_active = N, D, K, Q, n_active
        self.operands = [ops.CodebookOperands.allocate(K, D, False, device) for _ in range(n_active)]
        self.bufs = [torch.empty((N, D), dtype=torch.float32, device=device) for _ in range(min(2, n_active - 1))]
        self.loss_sum = torch.zeros((n_active,), dtype=torch.float64, device=device)
        self.stat_floats = ops.stats_floats(K, D) if want_stats else 0
        # placeholders, dropped after the build: `run` patches every pointer into them before each launch
        x0 = torch.empty((N, D), dtype=torch.float32, device=device)
        codes0 = torch.empty((n_active, K, D), dtype=torch.float32, device=device)
        idx0 = torch.empty((N, Q), dtype=torch.int64, device=device)
        out0 = torch.empty((N, D), dtype=torch.float32, device=device)
        losses0 = torch.empty((Q,), dtype=torch.float32, device=device)
        stats0 = torch.empty((max(1, n_active * self.stat_floats),), dtype=torch.float32, device=device)
        prog = ops.RvqProgram(device)
        r = x0
        for q in range(n_active):
            layer = mod.layers[q]
            nxt = self.bufs[q & 1] if q + 1 < n_active else None
            F_ = self.stat_floats
            idx32, _ = prog.stage(0, r, self.operands[q], (None, None, codes0[q]), update=1 if want_stats else 0,
                                  do_normalise=False, decay=0.0, eps=0.0,
                                  stats=stats0[q * F_:(q + 1) * F_] if want_stats else None)
            prog.simvq_tail(0, r, codes0[q], idx32, rotation=layer.rotation_trick, r_next=nxt, qsum=out0, first=q == 0,
                            idx64_out=idx0[:, q], idx_stride=Q, loss_sum=self.loss_sum[q:q + 1], loss_out=losses0[q:q + 1],
                            input_weight=layer.input_to_quantize_commit_loss_weight, weight=layer.commitment_weight)
            r = nxt
        self.prog = prog.freeze()

    def run(self, flat, codes, indices, out, losses, stats):
        arr = self.prog.arr
        row_bytes = self.K * self.D * 4
        for q in range(self.n_active):
            st, tl = arr[2 * q].stage, arr[2 * q + 1].simvq
            st.embed = tl.codes = codes.data_ptr() + q * row_bytes
            tl.qsum = out.data_ptr()
            tl.idx64_out = indices.data_ptr() + 8 * q
            tl.loss_out = losses.data_ptr() + 4 * q
            if stats is not None:
                st.stats = stats.data_ptr() + 4 * q * self.stat_floats
        arr[0].stage.x = arr[1].simvq.r = flat.data_ptr()
        for q in range(self.n_active):   # the implicit codebooks change with the transform: fresh operands every forward
            ops.prepare_codebook(codes[q], False, out=self.operands[q])
        self.prog.run()


class _ResidualSimVQFunction(torch.autograd.Function):
    """(x (N, D), C_0 .. C_{n_active-1}) -> (quantized_out, indices (N, Q), losses (Q,)) of rsv:182-203."""

    @staticmethod
    def forward(ctx, mod, n_active, want_stats, x, *codebooks):
        N, D = x.shape
        Q = mod.num_quantizers
        codes = torch.stack([c.detach() for c in codebooks])   # the codebooks the stages search, kept for the backward
        K = codes.shape[1]
        dev = x.device
        rotation = bool(mod.layers[0].rotation_trick)
        if any(bool(layer.rotation_trick) != rotation for layer in mod.layers[:n_active]):
            raise ValueError("ResidualSimVQ: every layer must use the same gradient estimator (rotation_trick)")
        key = (dev, N, D, K, n_active, want_stats,
               tuple((bool(layer.rotation_trick), float(layer.input_to_quantize_commit_loss_weight), float(layer.commitment_weight))
                     for layer in mod.layers[:n_active]))
        plan = _PlanCache.get_or_build(mod, key, lambda: _Plan(mod, N, D, K, n_active, want_stats, dev))
        out = torch.empty_like(x)
        if n_active < Q:   # rsv:153-187: the dropped stages report index -1 and a zero loss
            indices = torch.full((N, Q), -1, dtype=torch.int64, device=dev)
        else:
            indices = torch.empty((N, Q), dtype=torch.int64, device=dev)
        losses = torch.zeros((Q,), dtype=torch.float32, device=dev)
        stats = torch.empty((n_active * plan.stat_floats,), dtype=torch.float32, device=dev) if want_stats else None
        plan.run(x, codes, indices, out, losses, stats)
        ctx.mark_non_differentiable(indices)
        ctx.save_for_backward(x, codes, indices, stats)
        ctx.stat_floats = plan.stat_floats
        ctx.rotation = rotation
        ctx.weights = [(float(layer.input_to_quantize_commit_loss_weight), float(layer.commitment_weight))
                       for layer in mod.layers[:n_active]]
        return out, indices, losses

    @staticmethod
    def backward(ctx, g_out, g_indices, g_losses):
        x, codes, indices, stats = ctx.saved_tensors
        n_active, K, D = codes.shape
        numel = x.numel()
        grads = [None, None, None, None] + [None] * n_active
        gl = g_losses[:n_active].float()
        if ctx.needs_input_grad[3]:
            # d loss_q / d r_q = dL/dloss_q * weight * input_weight * 2 (r_q - c_q) / numel (sim_vq.py:123)
            scales = [2.0 * iw * w / numel for iw, w in ctx.weights]
            if len(set(scales)) == 1:
                gls = gl * scales[0]
            else:
                gls = torch.stack([gl[q] * s for q, s in enumerate(scales)])
            grads[3] = ops.rsimvq_backward(x, codes, indices, ctx.rotation, g_out.float().contiguous(), gls.contiguous())
        off = ops.stats_offset(K)
        for q in range(n_active):
            if not ctx.needs_input_grad[4 + q]:
                continue
            # d loss_q / d C_q = dL/dloss_q * weight * 2 (count * c - sum of the rows that chose c) / numel (sim_vq.py:122): the
            # first commitment term is the only one that reaches the codebook (rotate_to carries none to its target)
            base = q * ctx.stat_floats
            count = stats[base:base + K]
            rows = stats[base + off:base + off + K * D].view(K, D)
            grads[4 + q] = (count[:, None] * codes[q] - rows) * (gl[q] * (2.0 * ctx.weights[q][1] / numel))
        return tuple(grads)


class ResidualSimVQ(nn.Module):
    """Drop-in for the reference's ResidualSimVQ (rsv:51-83): `num_quantizers` SimVQ layers built in order (so a reference
    state_dict loads key for key), fp32 inputs `b * d` or channel-first."""

    def __init__(self, *, dim, num_quantizers, codebook_size, heads=1, quantize_dropout=False, quantize_dropout_cutoff_index=0,
                 quantize_dropout_multiple_of=1, channel_first=False, rotation_trick=True, **sim_vq_kwargs):
        super().__init__()
        assert heads == 1, "residual vq is not compatible with multi-headed codes"
        self.channel_first = channel_first
        self.num_quantizers = num_quantizers
        self.layers = nn.ModuleList([SimVQ(dim=dim, codebook_size=codebook_size, rotation_trick=rotation_trick,
                                           channel_first=channel_first, **sim_vq_kwargs) for _ in range(num_quantizers)])
        self.quantize_dropout = quantize_dropout and num_quantizers > 1
        assert quantize_dropout_cutoff_index >= 0
        self.quantize_dropout_cutoff_index = quantize_dropout_cutoff_index
        self.quantize_dropout_multiple_of = quantize_dropout_multiple_of

    # rsv:153-171: the last active layer of a training forward with quantize dropout (seed as get_maybe_sync_seed draws it)
    _active_layers = ResidualVQ._active_layers

    @property
    def codebook_size(self):
        return self.layers[0].codebook_size

    @property
    def codebooks(self):  # rsv:93-97
        return torch.stack([layer.codebook for layer in self.layers])

    def get_codes_from_indices(self, indices):  # rsv:99-135
        Q = self.num_quantizers
        indices = pad_dropped(indices, Q, self.quantize_dropout,
                              "quantize dropout must be greater than 0 if you wish to reconstruct from a signal with less fine "
                              "quantizations")
        lead = indices.shape[:-1]
        flat = indices.reshape(-1, Q)
        mask = flat == -1
        books = self.codebooks
        codes = books[torch.arange(Q, device=flat.device)[:, None], flat.masked_fill(mask, 0).t()]   # (Q, rows, D)
        codes = codes.masked_fill(mask.t()[..., None], 0.)
        codes = codes.reshape(Q, *lead, codes.shape[-1])
        if self.channel_first:
            codes = codes.movedim(-1, 2)   # 'q b ... d -> q b d ...'
        return codes

    def get_output_from_indices(self, indices):  # rsv:137-140
        return self.get_codes_from_indices(indices).sum(dim=0)

    def forward(self, x, return_all_codes=False, rand_quantize_dropout_fixed_seed=None):
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        # the reference searches with torch.cdist, which needs x and the (fp32) codebook in one dtype and has no bf16 / fp16 CPU
        # kernel: fp32 is the dtype it runs
        if x.dtype != torch.float32:
            raise TypeError(f"ResidualSimVQ supports float32 inputs, got {x.dtype}")
        Q = self.num_quantizers
        n_active = self._active_layers(rand_quantize_dropout_fixed_seed, x.device)
        xin = x.movedim(1, -1) if self.channel_first else x
        shape = xin.shape
        flat = xin.reshape(-1, shape[-1]).contiguous()
        codebooks = [layer.codebook for layer in self.layers[:n_active]]   # rsv:177-180: dropped layers are never run
        for c in codebooks:
            if c.dtype != torch.float32:
                raise TypeError(f"ResidualSimVQ supports float32 codebooks, got {c.dtype}")
        want_stats = torch.is_grad_enabled() and any(c.requires_grad for c in codebooks)
        quantized, indices, losses = _ResidualSimVQFunction.apply(self, n_active, want_stats, flat, *codebooks)
        quantized = quantized.reshape(shape)
        if self.channel_first:
            quantized = quantized.movedim(-1, 1)
        indices = indices.reshape(*shape[:-1], Q)
        ret = (quantized, indices, losses)
        if return_all_codes:
            ret = (*ret, self.get_codes_from_indices(indices))
        return ret
