"""`ResidualVQ` / `GroupedResidualVQ` — drop-ins for residual_vq.py:166-630 and :634-724 of the reference
(no beam search, no implicit neural codebook; quantize dropout and masks run on the stage-wise path).

Every stage's search writes the next residual (residual -= q, rvq:524) from its fused tail and its indices
straight into the (..., Q) int64 result; quantized_out += q (rvq:525) is rebuilt from those indices in one
pass after the last stage (rounded to the input dtype exactly where the reference rounds).  The EMA
statistics of ALL stages (and, for the grouped module, all groups) are packed into one buffer so that
multi-GPU training needs ONE all-reduce per forward instead of the reference's 2 per codebook per stage.
"""
from __future__ import annotations

import math
import os
import random

import torch
import torch.distributed as distributed
from torch import nn

from . import ops
from .codebook import _unsupported
from .dist import allreduce_packed, PeerReducer
from .vector_quantize import VectorQuantize, directional_reparam


class _PlanCache(dict):
    """Cached op lists of a module (raw device pointers inside): never copied or pickled along with the module."""

    def __deepcopy__(self, memo):
        return _PlanCache()

    def __reduce__(self):
        return (_PlanCache, ())


class _PlanPart:
    """One ResidualVQ forward inside an ops.RvqProgram: stage ops (rvq:469-568), the running sum (rvq:525), the deferred EMA
    ops (rvq:593-597 / vqp:616-617, :576-584).  Built once per configuration; `bind` patches the per-call pointers."""

    def __init__(self, rvq, prog, lane, flat, books, do_update, persistent_io=False):
        # persistent_io (GroupedResidualVQ: its cat / stack copy the results anyway): input, indices and output live in
        # buffers owned by the plan, so every pointer of the graph is stable and a forward is a pure replay
        self.io = None
        if persistent_io:
            flat = flat.clone(memory_format=torch.contiguous_format)
        N, D = flat.shape
        Q = rvq.num_quantizers
        dev, dtype = flat.device, flat.dtype
        training = rvq.training
        self.rvq, self.N, self.D, self.Q, self.dtype, self.dev = rvq, N, D, Q, dtype, dev
        self.bufs = [torch.empty_like(flat) for _ in range(min(2, Q - 1))]          # persistent: the residual ping-pong
        stat_sizes = [ops.stats_floats(b.codebook_size, D) if u else 0 for b, u in zip(books, do_update)]
        offs = [sum(stat_sizes[:i]) for i in range(Q)]
        self.peer = rvq._peer if (sum(stat_sizes) and any(b.use_ddp and u for b, u in zip(books, do_update))) else None
        if self.peer is not None:   # this plan is bound to ONE of the two alternating symmetric buffers (the key holds the parity)
            par = self.peer.step & 1
            self.packed, peer_ptrs = self.peer.bufs[par][:sum(stat_sizes)], self.peer.stats_ptrs[par]
        else:
            self.packed = torch.empty((sum(stat_sizes),), dtype=torch.float32, device=dev) if sum(stat_sizes) else None
        self.losses = rvq._loss_buf
        self.books = books
        all_idx = torch.empty((N, Q), dtype=torch.int64, device=dev)               # placeholders: `bind` patches the pointers
        out0 = torch.empty((N, D), dtype=dtype, device=dev)
        if persistent_io:
            self.io = (flat, all_idx, out0)
        # fp32 rows (Euclidean): a stage's tail also writes the bf16 hi / lo split of its residual — the next stage's MMA operand —
        # so that only stage 0 runs the split kernel over its input (536 MB of HBM traffic per stage at config 3)
        split = dtype == torch.float32 and not books[0].use_cosine_sim and Q > 1
        self.planes = [torch.empty((2, N, D), dtype=torch.bfloat16, device=dev) for _ in range(min(2, Q - 1))] if split else None
        self.first = len(prog.ops)
        residual = flat
        for q, book in enumerate(books):
            nxt = self.bufs[q & 1] if q + 1 < Q else None
            want_loss = training and rvq.layers[q].has_commitment_loss
            prog.stage(lane, residual, book.operands(), book._state2d(), update=1 if do_update[q] else 0, do_normalise=False,
                       decay=book.decay, eps=book.eps, idx64_out=all_idx[:, q], idx_stride=Q,
                       loss_out=self.losses[q:q + 1] if want_loss else None, loss_weight=rvq.layers[q].commitment_weight,
                       resid_out=nxt, stats=self.packed[offs[q]:offs[q] + stat_sizes[q]] if stat_sizes[q] else None,
                       ws_key=id(book),
                       a_planes_in=self.planes[(q - 1) & 1] if (split and q > 0) else None,
                       planes_out=self.planes[q & 1] if (split and nxt is not None) else None)
            residual = nxt
        # the running sum reads the codebooks the stages searched: before the EMA ops
        self.stack = None if rvq.shared_codebook else torch.stack([b.embed[0] for b in books])
        embeds = books[0].embed[0] if rvq.shared_codebook else self.stack
        self.acc = len(prog.ops)
        prog.accumulate(lane, embeds, all_idx, out0)
        self.refreshed = []
        if self.peer is not None:
            prog.barrier(lane, self.peer)      # every rank's statistics of this forward are in place (vqp:603, :607)
        final_ema = training and rvq.shared_codebook and rvq.vq_is_ema_updating and any(do_update)   # rvq:593-597
        if rvq.shared_codebook and all(stat_sizes) and Q > 1 and books[0].manual_ema_update:
            # one codebook, Q stages: every stage lerps the same buffers in turn (rvq:302-306) and update_ema follows once
            # (rvq:593-597) — ONE launch pair applies the Q statistics slices in order and normalises
            shared = books[0]
            cs, ea, emb = shared._state2d()
            if self.peer is not None:
                prog.ema_peers(lane, cs, ea, emb, self.peer, peer_ptrs, 0, shared.operands(), decay=shared.decay, eps=shared.eps,
                               do_normalise=final_ema, n_lerp=Q, slice_stride=stat_sizes[0])
            else:
                prog.ema(lane, cs, ea, emb, self.packed, shared.operands(), decay=shared.decay, eps=shared.eps, do_lerp=True,
                         do_normalise=final_ema, n_lerp=Q, slice_stride=stat_sizes[0])
            if final_ema:
                self.refreshed.append(shared)
            return
        for q, book in enumerate(books):
            if not stat_sizes[q]:
                continue
            normalise = book.ema_update and not book.manual_ema_update
            cs, ea, emb = book._state2d()
            if self.peer is not None:
                prog.ema_peers(lane, cs, ea, emb, self.peer, peer_ptrs, offs[q], book.operands(), decay=book.decay, eps=book.eps,
                               do_normalise=normalise)
            else:
                prog.ema(lane, cs, ea, emb, self.packed[offs[q]:offs[q] + stat_sizes[q]], book.operands(), decay=book.decay,
                         eps=book.eps, do_lerp=True, do_normalise=normalise)
            if normalise:
                self.refreshed.append(book)
        if final_ema:
            shared = books[0]
            cs, ea, emb = shared._state2d()
            prog.ema(lane, cs, ea, emb, None, shared.operands(), decay=shared.decay, eps=shared.eps, do_lerp=False,
                     do_normalise=True)
            self.refreshed.append(shared)

    def bind(self, arr, flat):
        """Fresh outputs for this call + the pointers of the cached ops that change from call to call."""
        if self.stack is not None:
            torch.stack([b.embed[0] for b in self.books], out=self.stack)
        if not self.rvq.training:
            self.losses.zero_()
        if self.peer is not None:
            self.peer.step += 1          # the next forward uses the other symmetric buffer (and the plan cached for it)
        if self.io is not None:
            if flat is not self.io[0]:
                self.io[0].copy_(flat.reshape(self.N, self.D))
            return self.io[1], self.io[2], None
        all_idx = torch.empty((self.N, self.Q), dtype=torch.int64, device=self.dev)
        out = torch.empty((self.N, self.D), dtype=self.dtype, device=self.dev)
        ip = all_idx.data_ptr()
        arr[self.first].stage.x = flat.data_ptr()
        for q in range(self.Q):
            arr[self.first + q].stage.idx64_out = ip + 8 * q
        arr[self.acc].acc.idx = ip
        arr[self.acc].acc.out = out.data_ptr()
        return all_idx, out, flat

    def finish(self, bound, shape, return_all_codes, project=True):
        all_idx, out, _ = bound
        rvq = self.rvq
        for b in self.refreshed:
            b._mark_operands_fresh()
        out = out.reshape(shape)
        if project:
            out = rvq.project_out(out)  # rvq:610
        ret = (out, all_idx.reshape(*shape[:-1], self.Q), self.losses.clone())
        if return_all_codes:
            ret = (*ret, rvq.get_codes_from_indices(ret[1]))
        return ret


class ResidualVQ(nn.Module):
    def __init__(
        self,
        *,
        dim,
        num_quantizers=None,
        codebook_size,
        codebook_dim=None,
        shared_codebook=False,
        diveq=False,
        heads=1,
        quantize_dropout=False,
        quantize_dropout_cutoff_index=0,
        quantize_dropout_multiple_of=1,
        accept_image_fmap=False,
        implicit_neural_codebook=False,
        mlp_kwargs: dict = dict(),
        beam_size=None,
        eval_beam_size=None,
        beam_score_quantizer_weights=None,
        quant_grad_frac=0.,
        **vq_kwargs,
    ):
        super().__init__()
        assert heads == 1, "residual vq is not compatible with multi-headed codes"  # rvq:191
        assert num_quantizers is not None or isinstance(codebook_size, tuple)  # rvq:192
        if implicit_neural_codebook:
            _unsupported("implicit_neural_codebook")
        if (beam_size is not None and beam_size > 1) or (eval_beam_size is not None and eval_beam_size > 1):
            _unsupported("beam search")
        if accept_image_fmap:
            _unsupported("ResidualVQ(accept_image_fmap=True)")
        if quant_grad_frac != 0.:
            _unsupported("quant_grad_frac != 0")

        codebook_dim = dim if codebook_dim is None else codebook_dim
        self.codebook_dim = codebook_dim
        requires_projection = codebook_dim != dim
        self.project_in = nn.Linear(dim, codebook_dim) if requires_projection else nn.Identity()
        self.project_out = nn.Linear(codebook_dim, dim) if requires_projection else nn.Identity()
        self.has_projections = requires_projection
        self.accept_image_fmap = accept_image_fmap

        if shared_codebook:  # rvq:213-217
            vq_kwargs.update(manual_ema_update=True)
        self.diveq = diveq
        if diveq:  # rvq:222-232: the codebooks learn from the DiVeQ gradient of quantized_out alone
            vq_kwargs.update(ema_update=False, learnable_codebook=True, route_gradients_to_input=False, commitment_weight=0.)

        codebook_sizes = codebook_size if isinstance(codebook_size, tuple) else (codebook_size,) * num_quantizers
        num_quantizers = len(codebook_sizes) if num_quantizers is None else num_quantizers
        assert len(codebook_sizes) == num_quantizers
        self.num_quantizers = num_quantizers
        self.codebook_sizes = codebook_sizes
        self.uniform_codebook_size = len(set(codebook_sizes)) == 1

        self.layers = nn.ModuleList([
            VectorQuantize(dim=codebook_dim, codebook_size=k, codebook_dim=codebook_dim, **vq_kwargs) for k in codebook_sizes
        ])  # rvq:249
        self.quantize_dropout = bool(quantize_dropout) and num_quantizers > 1  # rvq:253
        assert quantize_dropout_cutoff_index >= 0  # rvq:255
        self.quantize_dropout_cutoff_index = quantize_dropout_cutoff_index
        self.quantize_dropout_multiple_of = quantize_dropout_multiple_of  # rvq:258
        self.vq_is_ema_updating = self.layers[0].ema_update
        # rvq:268: 1 under DiVeQ; the residual then only feeds the searches, so no gradient flows through it either way
        self.quant_grad_frac = 1. if diveq else 0.
        self.shared_codebook = shared_codebook
        if shared_codebook:  # rvq:295-306: every layer aliases ONE Codebook
            assert self.uniform_codebook_size
            codebook = self.layers[0]._codebook
            for vq in self.layers[1:]:
                vq._codebook = codebook

    # ------------------------------------------------------------------ reference surface
    @property
    def codebook_size(self):
        return self.layers[0].codebook_size

    @property
    def codebooks(self):  # rvq:312-322
        books = tuple(layer._codebook.embed[0] for layer in self.layers)
        return torch.stack(books) if self.uniform_codebook_size else books

    def _pad_dropped(self, indices):
        """rvq:333-339: coarse indices (fewer than num_quantizers columns) are padded with -1 = "layer dropped"."""
        missing = self.num_quantizers - indices.shape[-1]
        if missing > 0:
            assert self.quantize_dropout, "quantize dropout must be on to reconstruct from fewer than num_quantizers indices"  # rvq:338
            indices = torch.nn.functional.pad(indices, (0, missing), value=-1)
        return indices

    def get_codes_from_indices(self, indices):  # rvq:324-376
        indices = self._pad_dropped(indices)
        q_idx = indices.reshape(-1, self.num_quantizers)
        codes = [self.layers[q]._codebook.decode(q_idx[:, q]) for q in range(self.num_quantizers)]
        return torch.stack(codes).reshape(self.num_quantizers, *indices.shape[:-1], self.codebook_dim)

    def get_output_from_indices(self, indices):  # rvq:378-382: sum over quantizers in ONE gather kernel
        indices = self._pad_dropped(indices)
        if self.uniform_codebook_size and not (torch.is_grad_enabled() and self._codebooks_need_grad()):
            out = ops.decode(self.codebooks.detach().contiguous(), indices)
        else:
            out = self.get_codes_from_indices(indices).sum(dim=0)
        return self.project_out(out)

    # ------------------------------------------------------------------ forward
    def _stage_plan(self):
        return [vq._codebook for vq in self.layers]

    def _peer_reducer(self, numel, device):
        """One symmetric-memory buffer for the statistics of ALL stages (dist.PeerReducer); None -> NCCL all-reduce."""
        if not getattr(self, "_peer_tried", False) or (self._peer is not None and self._peer.numel < numel):
            self._peer_tried = True
            self._peer = PeerReducer.create(numel, device)
        return self._peer

    def forward(self, x, mask=None, indices=None, return_all_codes=False, sample_codebook_temp=None,
                freeze_codebook=False, beam_size=None, rand_quantize_dropout_fixed_seed=None,
                _stats_sink=None, _projected=False):
        if indices is not None:
            _unsupported("ResidualVQ.forward(indices=)")
        if beam_size is not None and beam_size > 1:
            _unsupported("beam search")
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        if mask is not None:
            return self._forward_masked(x, mask, return_all_codes, freeze_codebook, rand_quantize_dropout_fixed_seed)
        if not _projected:   # _projected: the masked path hands in compacted rows that went through project_in already
            x = self.project_in(x)
        if torch.is_grad_enabled() and (x.requires_grad or self._codebooks_need_grad()):
            # gradients (to the input or to project_in, rvq:406, or to learnable codebooks) need the per-stage
            # straight-through / rotation / codebook-gradient glue of VectorQuantize: take the layered path
            return self._forward_layered(x, freeze_codebook, return_all_codes,
                                         self._active_layers(rand_quantize_dropout_fixed_seed, x.device))
        shape, dtype = x.shape, x.dtype
        if dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"vqb200 supports float32 and bfloat16 inputs, got {dtype}")
        flat = x.detach().reshape(-1, shape[-1]).contiguous()
        N, D = flat.shape
        Q = self.num_quantizers
        dev = flat.device
        training = self.training
        books = self._stage_plan()

        losses = self._ensure_loss_buf(dev)
        n_run = self._active_layers(rand_quantize_dropout_fixed_seed, dev)   # < Q: quantize dropout skips the layers after it
        do_update = [q < n_run and b.updates(training, freeze_codebook) for q, b in enumerate(books)]
        if not _projected and n_run == Q and self._program_ok(books, do_update):
            # the whole forward — stages, running sum, deferred EMA updates — as ONE vqb_rvq_forward call / one CUDA graph,
            # from a cached op list in which only the per-call pointers (input, indices, output) are patched
            key = self._part_key(flat, books, do_update)
            plans = self.__dict__.setdefault("_plans", _PlanCache())
            plan = plans.get(key)
            if plan is None:
                if len(plans) >= 8:
                    plans.clear()
                prog = ops.RvqProgram(dev)
                part = self._plan_part(prog, 0, flat, books, do_update)
                plan = plans[key] = (prog.freeze(), part)
            prog, part = plan
            bound = part.bind(prog.arr, flat)
            prog.run()
            if not self.diveq:
                return part.finish(bound, shape, return_all_codes)
            out, *rest = part.finish(bound, shape, return_all_codes, project=False)
            return (self.project_out(directional_reparam(x, out)), *rest)   # rvq:603-606, in every mode

        if n_run < Q:   # rvq:473-476: the skipped layers report index -1 and loss 0
            all_idx = torch.full((N, Q), -1, dtype=torch.int64, device=dev)
            losses.zero_()
        else:
            all_idx = torch.empty((N, Q), dtype=torch.int64, device=dev)
        if not training:
            losses.zero_()
        # dead-code expiry samples from the stage inputs after the (deferred) EMA update: keep them all then
        keep_inputs = training and not freeze_codebook and any(b.has_dead_code_replacement for b in books)
        bufs = [torch.empty_like(flat) for _ in range(Q - 1 if keep_inputs else min(2, Q - 1))]
        residual = flat  # rvq:411 (never written: stage 0 reads the caller's tensor)
        stage_inputs = []
        # A shared codebook that replaces dead codes is modified BETWEEN stages by the reference (every layer's
        # update_codebook ends with expire_codes_, vqp:641, on the one aliased Codebook): such stages cannot be deferred.
        inline = [u and self.shared_codebook and b.has_dead_code_replacement for b, u in zip(books, do_update)]
        stat_sizes = [ops.stats_floats(b.codebook_size, D) if (u and not i) else 0 for b, u, i in zip(books, do_update, inline)]
        packed, peer_ptrs = None, None
        if sum(stat_sizes):
            peer = self._peer_reducer(sum(stat_sizes), dev) if any(b.use_ddp for b in books) else None
            if peer is not None:   # statistics straight into symmetric memory: summed over the ranks inside the EMA kernels
                buf, peer_ptrs = peer.next_buffer()
                packed = buf[:sum(stat_sizes)]
            else:
                packed = torch.empty((sum(stat_sizes),), dtype=torch.float32, device=dev)
        offs = [sum(stat_sizes[:i]) for i in range(Q)]

        inline_embeds = []   # the shared codebook as each inline stage searched it
        for q, book in enumerate(books[:n_run]):  # rvq:469
            nxt = (bufs[q] if keep_inputs else bufs[q & 1]) if q + 1 < n_run else None
            if keep_inputs:
                stage_inputs.append(residual)
            if inline[q]:
                if not book._initted_host:   # k-means init precedes the search (quantize_rows would run it next)
                    book.init_embed_(book.transform_input(residual).float())
                inline_embeds.append(book.embed[0].clone())
            want_loss = training and self.layers[q].has_commitment_loss
            book.quantize_rows(
                residual, update=do_update[q], idx64_out=all_idx[:, q], idx_stride=Q,
                loss_out=losses[q:q + 1] if want_loss else None, loss_weight=self.layers[q].commitment_weight,
                resid_out=nxt, stats_out=packed[offs[q]:offs[q] + stat_sizes[q]] if stat_sizes[q] else None,
                defer_ema=not inline[q])
            residual = nxt

        # quantized_out (rvq:410, :525): rebuilt from the indices of the stages that ran, in one pass over the codebooks they
        # searched, instead of a read-modify-write of (N x D) in every stage.  Only inline stages change a codebook between
        # stages; every other update is deferred to _finish_update below.  Codebooks of different sizes are zero-padded to
        # the largest: every index of a stage is below its own size.
        if inline_embeds:
            searched = torch.stack(inline_embeds)
        elif self.shared_codebook:
            searched = books[0].embed[0]
        else:
            searched = torch.nn.utils.rnn.pad_sequence([b.embed[0] for b in books[:n_run]], batch_first=True)
        quantized_out = ops.rvq_accumulate(searched, all_idx[:, :n_run].contiguous(), dtype)

        if packed is not None or any(inline):
            if _stats_sink is not None:  # GroupedResidualVQ gathers every group's statistics into one collective
                _stats_sink.append((self, packed, offs, stat_sizes, do_update, (stage_inputs, shape, peer_ptrs)))
            else:
                self._finish_update(packed, offs, stat_sizes, do_update, (stage_inputs, shape, peer_ptrs), synced=False)

        quantized_out = quantized_out.reshape(shape)
        if self.diveq:   # rvq:603-606, in every mode
            quantized_out = directional_reparam(x, quantized_out)
        if not _projected:
            quantized_out = self.project_out(quantized_out)  # rvq:610
        ret = (quantized_out, all_idx.reshape(*shape[:-1], Q), losses.clone())
        if return_all_codes:
            ret = (*ret, self.get_codes_from_indices(ret[1]))
        return ret

    def _active_layers(self, fixed_seed, device) -> int:
        """Number of leading layers that quantize in this forward.  Training with quantize_dropout (rvq:423-439): python's
        random.Random(seed).randrange(cutoff, Q) is the last active layer, rounded up to a multiple if asked; without an explicit
        seed one is drawn like the reference's get_maybe_sync_seed (rvq:96-103: torch.randint on the device, all-reduced, .item())."""
        Q = self.num_quantizers
        if not (self.training and self.quantize_dropout):
            return Q
        if fixed_seed is None:
            seed = torch.randint(0, 10_000, (), device=device)
            if distributed.is_available() and distributed.is_initialized() and distributed.get_world_size() > 1:
                distributed.all_reduce(seed)
            fixed_seed = seed.item()
        index = random.Random(fixed_seed).randrange(self.quantize_dropout_cutoff_index, Q)
        mult = self.quantize_dropout_multiple_of
        if mult != 1:
            index = math.ceil((index + 1) / mult) * mult - 1  # rvq:39-40, :439
        return min(index + 1, Q)

    def _forward_masked(self, x, mask, return_all_codes, freeze_codebook, dropout_seed=None):
        """mask (B, N) bool.  The reference hands the mask to every layer (rvq:495): a layer searches every row, but masked rows
        take no part in its statistics or loss (vqp:599-600, :1317-1325) and come back as zeros / index -1 (vqp:1378-1396), so their
        residual is never reduced and their running sum stays zero.  That is exactly the forward over the COMPACTED unmasked rows
        with zeros / -1 scattered around it — which is what runs here (stage-wise path: the compacted row count changes from call
        to call, a cached program per count would not pay).  project_in / project_out see every row (rvq:406, :610)."""
        books = self._stage_plan()
        if any(b.learnable_codebook for b in books):
            _unsupported("ResidualVQ.forward(mask=) with learnable codebooks")
        if any(b.use_cosine_sim for b in books):
            _unsupported("ResidualVQ.forward(mask=) with use_cosine_sim (the masked loss is taken against the un-normalised input, vqp:1319)")
        if any(not vq.return_zeros_for_masked_padding for vq in self.layers):
            _unsupported("ResidualVQ.forward(mask=) with return_zeros_for_masked_padding=False")
        if self.training and any(b.has_dead_code_replacement for b in books):
            _unsupported("ResidualVQ.forward(mask=) with dead-code replacement")
        xp = self.project_in(x)  # rvq:406
        if xp.requires_grad and torch.is_grad_enabled():
            _unsupported("ResidualVQ.forward(mask=) on inputs / projections that require grad")
        assert xp.ndim == 3 and mask.shape == xp.shape[:2]
        B, N, D = xp.shape
        Q = self.num_quantizers
        rows = mask.reshape(-1).nonzero(as_tuple=True)[0]  # host sync (the reference's masked path syncs as well)
        quantized = torch.zeros((B * N, D), dtype=xp.dtype, device=xp.device)
        all_idx = torch.full((B * N, Q), -1, dtype=torch.int64, device=xp.device)
        if rows.numel() > 0:
            xc = xp.detach().reshape(-1, D)[rows].unsqueeze(0)
            qc, ic, losses = self.forward(xc, freeze_codebook=freeze_codebook, _projected=True,
                                          rand_quantize_dropout_fixed_seed=dropout_seed)
            quantized[rows] = qc[0]
            all_idx[rows] = ic[0]
        else:
            losses = torch.zeros((Q,), dtype=torch.float32, device=xp.device)
        ret = (self.project_out(quantized.reshape(B, N, D)), all_idx.reshape(B, N, Q), losses)  # rvq:610
        if return_all_codes:
            ret = (*ret, self.get_codes_from_indices(ret[1]))
        return ret

    def _codebooks_need_grad(self):
        return any(vq._codebook.embed.requires_grad for vq in self.layers)

    def _program_ok(self, books, do_update):
        """One-call path (ops.RvqProgram): every stage deferred, no collective, no dead-code expiry, nothing parked on `.grad`
        (accum_ema_update), codebooks initialised and stackable."""
        if os.environ.get("VQB_RVQ_PROGRAM", "1") == "0":
            return False
        if ops.PROFILE_EVENTS is not None or not self.uniform_codebook_size:
            return False
        n_ops = len(books) + 1 + sum(do_update) + 2
        if n_ops > ops.RvqProgram.MAX_OPS:
            return False
        for b, u in zip(books, do_update):
            if not b._initted_host:
                return False
            if u and (b.has_dead_code_replacement or b.cluster_size.grad is not None or b.embed_avg.grad is not None):
                return False
        ddp = [b.use_ddp for b, u in zip(books, do_update) if u]
        if any(ddp):
            # multi-GPU: the statistics go to symmetric memory and the EMA ops sum over the ranks (barrier + peer loads inside
            # the program); without peer memory the stage-wise path does ONE NCCL all-reduce instead
            if not all(ddp):
                return False
            dev, D = books[0].embed.device, books[0].embed.shape[-1]
            numel = sum(ops.stats_floats(b.codebook_size, D) for b, u in zip(books, do_update) if u)
            if self._peer_reducer(numel, dev) is None:
                return False
        return True

    def _ensure_loss_buf(self, dev):
        """Per-stage losses land in a persistent buffer (stable pointers for the graph cache); callers get a clone."""
        loss_buf = getattr(self, "_loss_buf", None)
        if loss_buf is None or loss_buf.device != dev or loss_buf.numel() != self.num_quantizers:
            loss_buf = torch.zeros((self.num_quantizers,), dtype=torch.float32, device=dev)
            self._loss_buf = loss_buf
        return loss_buf

    def _part_key(self, flat, books, do_update):
        """Everything a cached op list depends on, except the per-call pointers `_PlanPart.bind` patches.  `book.operands()`
        refreshes the tensor-core operands if `embed` was changed from outside since the last forward."""
        peer = getattr(self, "_peer", None) if any(b.use_ddp and u for b, u in zip(books, do_update)) else None
        return (tuple(flat.shape), flat.dtype, flat.device, self.training, tuple(do_update), None if peer is None else peer.step & 1,
                tuple((id(b), id(b.operands()), b.embed.data_ptr(), b.cluster_size.data_ptr(), b.embed_avg.data_ptr()) for b in books))

    def _plan_part(self, prog, lane, flat, books, do_update, persistent_io=False):
        return _PlanPart(self, prog, lane, flat, books, do_update, persistent_io)

    def _finish_update(self, packed, offs, stat_sizes, do_update, stage_inputs, synced):
        """ONE all-reduce for all stages (reference: 2 per stage, vqp:603/:607), then the per-stage lerps in
        order (vqp:616-617) and update_ema — once at the end for a shared codebook (rvq:593-597) — and the dead-code
        expiry: per stage from that stage's input (vqp:641), for a shared codebook once over all residuals (rvq:599-601).
        stage_inputs: (the Q stage inputs (N, D) — kept only when some codebook replaces dead codes —, input shape)."""
        stage_inputs, shape, peer_ptrs = stage_inputs
        books = self._stage_plan()
        peer = self._peer if peer_ptrs is not None else None
        if peer is not None:
            peer.barrier()       # every rank's statistics of this forward are in place
        elif not synced and packed is not None and any(b.use_ddp for b in books):
            allreduce_packed(packed)
        for q, book in enumerate(books):
            if not do_update[q] or not stat_sizes[q]:   # nothing to do, or already applied inline
                continue
            normalise = book.ema_update and not book.manual_ema_update
            if peer is not None:
                book.lerp_stats_peers(peer, peer_ptrs, offs[q], normalise)
            else:
                book.lerp_stats(packed[offs[q]:offs[q] + stat_sizes[q]], normalise=normalise)
            if not self.shared_codebook and book.has_dead_code_replacement:
                book.expire_codes_(book.transform_input(stage_inputs[q]).float())  # vqp:641 on the fp32 `flatten`
        if self.training and self.shared_codebook:
            shared = books[0]
            if self.vq_is_ema_updating and any(do_update):
                shared.update_ema()
            if shared.has_dead_code_replacement and any(do_update):
                # rvq:599-601 -> vqp:1051-1054 -> :573-574: the reference hands '(b) (n l) d' to Codebook.expire_codes_, whose
                # 'h ... d -> h (...) d' reads the batch axis as the codebook axis, and `replace` zips it with the (1, K)
                # mask: only batch element 0's rows (n-major, stage-minor) are sampled from.  Reproduced as is.
                n0 = stage_inputs[0].shape[0] // shape[0] if len(shape) > 2 else stage_inputs[0].shape[0]
                rows = torch.stack([r[:n0] for r in stage_inputs], dim=1).reshape(-1, stage_inputs[0].shape[-1])
                shared.expire_codes_(shared.transform_input(rows))

    def _forward_layered(self, x, freeze_codebook, return_all_codes, n_run=None):
        """Differentiable path: the reference's Python loop (rvq:469-568) over our VectorQuantize layers.
        `x` is already projected (rvq:406).  n_run < Q: quantize dropout (rvq:473-476)."""
        quantized_out = torch.zeros_like(x)
        residual = x
        all_idx, all_losses = [], []
        for q, vq in enumerate(self.layers):
            if n_run is not None and q >= n_run:
                all_idx.append(torch.full(x.shape[:-1], -1, dtype=torch.int64, device=x.device))
                all_losses.append(torch.zeros((), dtype=torch.float32, device=x.device))
                continue
            quantized, ind, loss = vq(residual, freeze_codebook=freeze_codebook)
            residual = residual - quantized.detach()
            quantized_out = quantized_out + quantized
            all_idx.append(ind)
            all_losses.append(loss)
        if self.training and self.shared_codebook and self.vq_is_ema_updating and not freeze_codebook:
            self.layers[0]._codebook.update_ema()
        if self.diveq:   # rvq:603-606: every stage's codebook gets the DiVeQ gradient of quantized_out
            quantized_out = directional_reparam(x, quantized_out)
        ret = (self.project_out(quantized_out), torch.stack(all_idx, dim=-1), torch.stack(all_losses))
        if return_all_codes:
            ret = (*ret, self.get_codes_from_indices(ret[1]))
        return ret


class GroupedResidualVQ(nn.Module):
    def __init__(self, *, dim, groups=1, accept_image_fmap=False, **kwargs):
        super().__init__()
        self.dim = dim
        self.groups = groups
        assert (dim % groups) == 0  # rvq:646
        if accept_image_fmap:
            _unsupported("GroupedResidualVQ(accept_image_fmap=True)")
        self.accept_image_fmap = accept_image_fmap
        self.rvqs = nn.ModuleList([ResidualVQ(dim=dim // groups, **kwargs) for _ in range(groups)])  # rvq:651-658

    @property
    def codebooks(self):
        return torch.stack(tuple(rvq.codebooks for rvq in self.rvqs))

    @property
    def split_dim(self):
        return -1

    def get_codes_from_indices(self, indices):
        return torch.stack(tuple(rvq.get_codes_from_indices(i) for rvq, i in zip(self.rvqs, indices)))

    def get_output_from_indices(self, indices):
        return torch.cat(tuple(rvq.get_output_from_indices(i) for rvq, i in zip(self.rvqs, indices)), dim=-1)

    def _program_ok(self, chunks, freeze_codebook):
        """All groups in one ops.RvqProgram: every group qualifies (ResidualVQ._program_ok), no gradient path, and the op list fits."""
        if torch.is_grad_enabled() and (any(c.requires_grad for c in chunks) or any(r._codebooks_need_grad() for r in self.rvqs)):
            return False
        if any(rvq.diveq for rvq in self.rvqs):
            return False
        total = 0
        for rvq, c in zip(self.rvqs, chunks):
            if not c.is_cuda or c.dtype not in (torch.float32, torch.bfloat16):
                return False
            if torch.is_grad_enabled() and any(p.requires_grad for p in rvq.project_in.parameters()):
                return False
            books = rvq._stage_plan()
            upd = [b.updates(rvq.training, freeze_codebook) for b in books]
            if not rvq._program_ok(books, upd):
                return False
            total += len(books) + 1 + sum(upd) + 2
        return total <= ops.RvqProgram.MAX_OPS

    def forward(self, x, indices=None, return_all_codes=False, sample_codebook_temp=None, freeze_codebook=False, mask=None):
        if indices is not None:
            _unsupported("GroupedResidualVQ.forward(indices=)")
        assert x.shape[-1] == self.dim
        chunks = x.chunk(self.groups, dim=-1)  # rvq:690
        if self.training:
            # the reference draws one torch.randint here even without quantize-dropout (rvq:701 -> :96-103);
            # consume it too so that seeded runs stay aligned with the reference's RNG stream.
            seed = torch.randint(0, 10_000, (), device=x.device)
            if distributed.is_available() and distributed.is_initialized() and distributed.get_world_size() > 1:
                distributed.all_reduce(seed)
        dropout_seed = None
        if self.training and any(rvq.quantize_dropout for rvq in self.rvqs):
            dropout_seed = int(seed.item())   # rvq:701: the SAME dropout index in every group
        if mask is not None:   # rvq:698: every group receives the mask (ResidualVQ._forward_masked)
            outs = [rvq(c, mask=mask, freeze_codebook=freeze_codebook, return_all_codes=return_all_codes,
                        rand_quantize_dropout_fixed_seed=dropout_seed) for rvq, c in zip(self.rvqs, chunks)]
            sink = []
        elif dropout_seed is None and self._program_ok(chunks, freeze_codebook):
            # every group's stages in ONE vqb_rvq_forward call: the groups are independent chains on parallel lanes; the op
            # list is cached, only the per-call pointers are patched
            flats, keys = [], []
            for rvq, c in zip(self.rvqs, chunks):
                xin = rvq.project_in(c).detach()
                flat = xin.reshape(-1, xin.shape[-1])     # a strided view of the group's columns: copied into the plan's buffer
                books = rvq._stage_plan()
                upd = [b.updates(rvq.training, freeze_codebook) for b in books]
                rvq._ensure_loss_buf(flat.device)
                flats.append((flat, xin.shape, books, upd))
                keys.append(rvq._part_key(flat, books, upd))
            key = tuple(keys)
            plans = self.__dict__.setdefault("_plans", _PlanCache())
            plan = plans.get(key)
            if plan is None:
                if len(plans) >= 8:
                    plans.clear()
                prog = ops.RvqProgram(x.device)
                parts = [rvq._plan_part(prog, g % 4, f[0], f[2], f[3], persistent_io=True)
                         for g, (rvq, f) in enumerate(zip(self.rvqs, flats))]
                plan = plans[key] = (prog.freeze(), parts)
            prog, parts = plan
            bound = [part.bind(prog.arr, f[0]) for part, f in zip(parts, flats)]
            prog.run()
            outs = [part.finish(b, f[1], return_all_codes) for part, b, f in zip(parts, bound, flats)]
            sink = []
        else:
            sink = []
            outs = [rvq(c, freeze_codebook=freeze_codebook, return_all_codes=return_all_codes, _stats_sink=sink,
                        rand_quantize_dropout_fixed_seed=dropout_seed) for rvq, c in zip(self.rvqs, chunks)]  # rvq:706
        if sink:
            need_sync = any(b.use_ddp for rvq, *_ in sink for b in rvq._stage_plan()) and all(e[5][2] is None for e in sink)
            if need_sync:  # no peer memory: ONE NCCL collective for every codebook of every group
                flat_all = torch.cat([p for _, p, *_ in sink])
                allreduce_packed(flat_all)
                pos = 0
                for rvq, packed, offs, sizes, upd, inputs in sink:
                    n = packed.numel()
                    rvq._finish_update(flat_all[pos:pos + n], offs, sizes, upd, inputs, synced=True)
                    pos += n
            else:
                for rvq, packed, offs, sizes, upd, inputs in sink:
                    rvq._finish_update(packed, offs, sizes, upd, inputs, synced=True)
        quantized = torch.cat([o[0] for o in outs], dim=-1)  # rvq:719-721
        all_indices = torch.stack([o[1] for o in outs])
        commit_losses = torch.stack([o[2] for o in outs])
        ret = (quantized, all_indices, commit_losses)
        if return_all_codes:
            ret = (*ret, torch.stack([o[3] for o in outs]))
        return ret
