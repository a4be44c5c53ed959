"""`ResidualVQ` / `GroupedResidualVQ` — drop-ins for residual_vq.py:166-630 and :634-724 of the reference
(no beam search, no implicit neural codebook; quantize dropout and masks run on the stage-wise path).

`ResidualVQ.forward` is one row pipeline: rows in, compaction of a masked batch, ONE row quantizer — layered (gradients), the
cached one-call program or stage-wise — and one tail.  Every stage's search writes the next residual (residual -= q, rvq:524)
from its fused tail and its indices straight into the (..., Q) int64 result; quantized_out += q (rvq:525) is rebuilt from those
indices in one pass after the last stage (rounded to the input dtype exactly where the reference rounds).  The codebook updates
after the searches are described once (`_CodebookUpdates`), recorded into the program or applied eagerly.  The EMA statistics
of ALL stages (and, for the grouped module, all groups) are packed into one buffer so that multi-GPU training needs ONE
all-reduce per forward instead of the reference's 2 per codebook per stage.
"""
from __future__ import annotations

import os

import torch
from torch import nn

from . import ops
from .codebook import _unsupported
from .dist import allreduce_packed, PeerReducer
from .residual_common import GroupedResidual, dropout_cut, pad_dropped, sync_seed
from .vector_quantize import VectorQuantize, directional_reparam

_DTYPES = (torch.float32, torch.bfloat16)


class _PlanCache(dict):
    """Cached op lists of a module (raw device pointers inside): never copied or pickled along with the module."""

    def __deepcopy__(self, memo):
        return _PlanCache()

    def __reduce__(self):
        return (_PlanCache, ())

    @staticmethod
    def get_or_build(module, key, build):
        """The module's cached plan for `key`, made by `build()` when missing.  At most 8 are kept: a full cache is emptied."""
        plans = module.__dict__.setdefault("_plans", _PlanCache())
        plan = plans.get(key)
        if plan is None:
            if len(plans) >= 8:
                plans.clear()
            plan = plans[key] = build()
        return plan


class _CodebookUpdates:
    """The codebook updates that follow the searches of one ResidualVQ forward: the lerps of the packed statistics in stage
    order (vqp:616-617), update_ema — for a shared codebook once, at the end (rvq:593-597) — and dead-code expiry (vqp:641;
    rvq:599-601).  `record` appends them to a program, `apply` runs them eagerly.  The statistics go to one packed buffer
    (`stats(q)`: stage q's slice), local or the peer-memory buffer `begin` takes.  A shared codebook that replaces dead codes
    is changed BETWEEN stages by the reference (every layer's update_codebook ends with expire_codes_, vqp:641, on the one
    aliased Codebook): such "inline" stages update inside their own search and have no slice."""

    def __init__(self, rvq, books, do_update, D, device):
        self.books, self.do_update = books, do_update
        self.shared = rvq.shared_codebook
        self.inline = [u and self.shared and b.has_dead_code_replacement for b, u in zip(books, do_update)]
        self.sizes = [ops.stats_floats(b.codebook_size, D) if (u and not i) else 0
                      for b, u, i in zip(books, do_update, self.inline)]
        self.offs = [sum(self.sizes[:q]) for q in range(len(books))]
        total = sum(self.sizes)
        self.use_ddp = any(b.use_ddp for b in books)
        self.peer = self.peer_ptrs = self.packed = None
        if total and self.use_ddp:
            self.peer = rvq._peer_reducer(total, device)
        if self.peer is not None:   # the buffer `begin` takes: statistics summed over the ranks inside the EMA kernels
            parity = self.peer.step & 1
            self.packed, self.peer_ptrs = self.peer.bufs[parity][:total], self.peer.stats_ptrs[parity]
        elif total:
            self.packed = torch.empty((total,), dtype=torch.float32, device=device)
        # (stage, codebook, update_ema after the lerp): a shared codebook is manual (rvq:213-217) and normalised once, at the end
        self.steps = [(q, b, b.ema_update and not b.manual_ema_update) for q, b in enumerate(books) if self.sizes[q]]
        self.final_ema = rvq.training and self.shared and rvq.vq_is_ema_updating and any(do_update)   # rvq:593-597
        self.stage_inputs = []      # the stage inputs (N, D), kept by the stage-wise path when codes can expire
        self.rows0 = 0              # rows of batch element 0: the shared codebook's expiry samples only those (see `apply`)

    def stats(self, q):
        return self.packed[self.offs[q]:self.offs[q] + self.sizes[q]] if self.sizes[q] else None

    def begin(self):
        """Once per forward, before its statistics are written: the peer reducer moves on to the other parity buffer."""
        if self.peer is not None:
            self.peer.next_buffer()

    def record(self, prog, lane):
        """Append the updates to `prog` (no inline stages: the program path has no dead-code expiry).  Returns the codebooks
        whose search operands the program refreshes."""
        books, peer = self.books, self.peer
        if peer is not None:
            prog.barrier(lane, peer)      # every rank's statistics of this forward are in place (vqp:603, :607)

        def ema(book, q, normalise, **kw):
            cs, ea, emb = book._state2d()
            if peer is not None:
                prog.ema_peers(lane, cs, ea, emb, peer, self.peer_ptrs, self.offs[q], book.operands(), decay=book.decay,
                               eps=book.eps, do_normalise=normalise, **kw)
            else:
                prog.ema(lane, cs, ea, emb, self.stats(q), book.operands(), decay=book.decay, eps=book.eps, do_lerp=True,
                         do_normalise=normalise, **kw)

        if self.shared and len(self.steps) == len(books) > 1:
            # one codebook, Q stages: ONE op applies the Q statistics slices in stage order, then normalises once
            ema(books[0], 0, self.final_ema, n_lerp=len(books), slice_stride=self.sizes[0])
            return [books[0]] if self.final_ema else []
        for q, book, normalise in self.steps:
            ema(book, q, normalise)
        refreshed = [book for _, book, normalise in self.steps if normalise]
        if self.final_ema:
            cs, ea, emb = books[0]._state2d()
            prog.ema(lane, cs, ea, emb, None, books[0].operands(), decay=books[0].decay, eps=books[0].eps, do_lerp=False,
                     do_normalise=True)
            refreshed.append(books[0])
        return refreshed

    @staticmethod
    def apply_all(pending):
        """Run the updates of one or more forwards (the groups of a GroupedResidualVQ) eagerly: without peer memory ONE
        all-reduce covers every codebook of all of them (reference: 2 per codebook per stage, vqp:603/:607)."""
        local = [u for u in pending if u.packed is not None]
        if local and any(u.use_ddp for u in pending) and all(u.peer is None for u in pending):
            flat = allreduce_packed(local[0].packed if len(local) == 1 else torch.cat([u.packed for u in local]))
            pos = 0
            for u in local:   # every forward's slice of the summed statistics
                n = u.packed.numel()
                u.packed = flat[pos:pos + n]
                pos += n
        for u in pending:
            u.apply()

    def apply(self):
        """The lerps, update_ema and expiry, after the statistics are summed over the ranks (`apply_all`)."""
        peer = self.peer
        if peer is not None:
            peer.barrier()       # every rank's statistics of this forward are in place
        for q, book, normalise in self.steps:
            if peer is not None:
                book.lerp_stats_peers(peer, self.peer_ptrs, self.offs[q], normalise)
            else:
                book.lerp_stats(self.stats(q), normalise=normalise)
            if not self.shared and book.has_dead_code_replacement:
                book.expire_codes_(book.transform_input(self.stage_inputs[q]).float())  # vqp:641 on the fp32 `flatten`
        shared = self.books[0]
        if self.final_ema:
            shared.update_ema()
        if self.shared and shared.has_dead_code_replacement and any(self.do_update):
            # rvq:599-601 -> vqp:1051-1054 -> :573-574: the reference hands '(b) (n l) d' to Codebook.expire_codes_, whose
            # 'h ... d -> h (...) d' reads the batch axis as the codebook axis, and `replace` zips it with the (1, K)
            # mask: only batch element 0's rows (n-major, stage-minor) are sampled from.  Reproduced as is.
            rows = torch.stack([r[:self.rows0] for r in self.stage_inputs], dim=1).reshape(-1, self.stage_inputs[0].shape[-1])
            shared.expire_codes_(shared.transform_input(rows))


def _run_program(owner, rvqs, flats, plan, persistent_io=False):
    """ResidualVQ forwards — stages, running sum, codebook updates — as ONE vqb_rvq_forward call / one CUDA graph, the forwards
    (the groups of a GroupedResidualVQ) as independent chains on parallel lanes.  The op list is cached on `owner`; only the
    per-call pointers (input, indices, output) are patched.  plan: each forward's (codebooks, stages that update).
    Returns each forward's (quantized rows, indices (N, Q), losses (Q,))."""
    for rvq, flat in zip(rvqs, flats):
        rvq._ensure_loss_buf(flat.device)
    key = tuple(rvq._part_key(flat, books, upd) for rvq, flat, (books, upd) in zip(rvqs, flats, plan))

    def build():
        prog = ops.RvqProgram(flats[0].device)
        parts = [_PlanPart(rvq, prog, g % 4, flat, books, upd, persistent_io)
                 for g, (rvq, flat, (books, upd)) in enumerate(zip(rvqs, flats, plan))]
        return prog.freeze(), parts
    prog, parts = _PlanCache.get_or_build(owner, key, build)
    bound = [part.bind(prog.arr, flat) for part, flat in zip(parts, flats)]
    prog.run()
    return [part.finish(b) for part, b in zip(parts, bound)]


class _PlanPart:
    """One ResidualVQ forward inside an ops.RvqProgram: stage ops (rvq:469-568), the running sum (rvq:525), the recorded
    codebook updates (`_CodebookUpdates.record`).  Built once per configuration; `bind` patches the per-call pointers."""

    def __init__(self, rvq, prog, lane, flat, books, do_update, persistent_io=False):
        # persistent_io (GroupedResidualVQ: its cat / stack copy the results anyway): input, indices and output live in
        # buffers owned by the plan, so every pointer of the graph is stable and a forward is a pure replay
        self.io = None
        if persistent_io:
            flat = flat.clone(memory_format=torch.contiguous_format)
        N, D = flat.shape
        Q = rvq.num_quantizers
        dev, dtype = flat.device, flat.dtype
        self.rvq, self.N, self.D, self.Q, self.dtype, self.dev = rvq, N, D, Q, dtype, dev
        self.bufs = [torch.empty_like(flat) for _ in range(min(2, Q - 1))]          # persistent: the residual ping-pong
        self.updates = _CodebookUpdates(rvq, books, do_update, D, dev)
        self.losses = rvq._loss_buf
        all_idx = torch.empty((N, Q), dtype=torch.int64, device=dev)               # placeholders: `bind` patches the pointers
        out0 = torch.empty((N, D), dtype=dtype, device=dev)
        if persistent_io:
            self.io = (flat, all_idx, out0)
        # fp32 rows (Euclidean): a stage's tail also writes the bf16 hi / lo split of its residual — the next stage's MMA operand —
        # so that only stage 0 runs the split kernel over its input (536 MB of HBM traffic per stage at config 3)
        split = dtype == torch.float32 and not books[0].use_cosine_sim and Q > 1
        self.planes = [torch.empty((2, N, D), dtype=torch.bfloat16, device=dev) for _ in range(min(2, Q - 1))] if split else None
        # the operands the ops point into, held so that the id() of each in `ResidualVQ._part_key` names them for this plan's life
        self.operands = [book.operands() for book in books]
        self.first = len(prog.ops)
        residual = flat
        for q, book in enumerate(books):
            nxt = self.bufs[q & 1] if q + 1 < Q else None
            want_loss = rvq.training and rvq.layers[q].has_commitment_loss
            prog.stage(lane, residual, self.operands[q], book._state2d(), update=1 if do_update[q] else 0, do_normalise=False,
                       decay=book.decay, eps=book.eps, idx64_out=all_idx[:, q], idx_stride=Q,
                       loss_out=self.losses[q:q + 1] if want_loss else None, loss_weight=rvq.layers[q].commitment_weight,
                       resid_out=nxt, stats=self.updates.stats(q),
                       a_planes_in=self.planes[(q - 1) & 1] if (split and q > 0) else None,
                       planes_out=self.planes[q & 1] if (split and nxt is not None) else None)
            residual = nxt
        # the running sum reads the codebooks the stages searched: before the EMA ops
        self.stack = None if rvq.shared_codebook else torch.stack([b.embed[0] for b in books])
        embeds = books[0].embed[0] if rvq.shared_codebook else self.stack
        self.acc = len(prog.ops)
        prog.accumulate(lane, embeds, all_idx, out0)
        self.refreshed = self.updates.record(prog, lane)

    def bind(self, arr, flat):
        """Fresh outputs for this call + the pointers of the cached ops that change from call to call."""
        if self.stack is not None:
            torch.stack([b.embed[0] for b in self.updates.books], out=self.stack)
        if not self.rvq.training:
            self.losses.zero_()
        self.updates.begin()          # with peer memory the next forward uses the other buffer (and the plan cached for it)
        if self.io is not None:
            if flat is not self.io[0]:
                self.io[0].copy_(flat.reshape(self.N, self.D))
            return self.io[1], self.io[2]
        all_idx = torch.empty((self.N, self.Q), dtype=torch.int64, device=self.dev)
        out = torch.empty((self.N, self.D), dtype=self.dtype, device=self.dev)
        ip = all_idx.data_ptr()
        arr[self.first].stage.x = flat.data_ptr()
        for q in range(self.Q):
            arr[self.first + q].stage.idx64_out = ip + 8 * q
        arr[self.acc].acc.idx = ip
        arr[self.acc].acc.out = out.data_ptr()
        return all_idx, out

    def finish(self, bound):
        """(quantized rows, indices (N, Q), losses (Q,)) of the call `bound` came from, after the program ran."""
        for b in self.refreshed:
            b._mark_operands_fresh()
        all_idx, out = bound
        return out, all_idx, self.losses.clone()


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
        return pad_dropped(indices, self.num_quantizers, self.quantize_dropout,
                           "quantize dropout must be on to reconstruct from fewer than num_quantizers indices")  # rvq:338

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

    def _do_update(self, books, freeze_codebook, n_run):
        """Which stages change their codebook in this forward: the active ones (quantize dropout, rvq:473-476) that update."""
        return [q < n_run and b.updates(self.training, freeze_codebook) for q, b in enumerate(books)]

    def _peer_reducer(self, numel, device):
        """One symmetric-memory buffer for the statistics of ALL stages (dist.PeerReducer); None -> NCCL all-reduce."""
        if not getattr(self, "_peer_tried", False) or (self._peer is not None and self._peer.numel < numel):
            self._peer_tried = True
            self._peer = PeerReducer.create(numel, device)
        return self._peer

    def _takes_layered(self, x):
        """Gradients (to the input or to project_in, rvq:406, or to learnable codebooks) need the per-stage straight-through /
        rotation / codebook-gradient glue of VectorQuantize: the layered path."""
        return torch.is_grad_enabled() and (x.requires_grad or self._codebooks_need_grad())

    def forward(self, x, mask=None, indices=None, return_all_codes=False, sample_codebook_temp=None,
                freeze_codebook=False, beam_size=None, rand_quantize_dropout_fixed_seed=None):
        if indices is not None:
            _unsupported("ResidualVQ.forward(indices=)")
        if beam_size is not None and beam_size > 1:
            _unsupported("beam search")
        return self._forward_projected(self.project_in(x), mask, return_all_codes, freeze_codebook,  # rvq:406
                                       rand_quantize_dropout_fixed_seed)

    def _forward_projected(self, x, mask, return_all_codes, freeze_codebook, dropout_seed, pending=None):
        """The row pipeline after project_in.  `pending` (GroupedResidualVQ): a list the stage-wise path appends its
        `_CodebookUpdates` to instead of applying them, so that all groups share one all-reduce."""
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        shape, D, Q = x.shape, x.shape[-1], self.num_quantizers
        books = self._stage_plan()
        rows = masked = None
        if mask is not None:
            if any(b.learnable_codebook for b in books):
                _unsupported("ResidualVQ.forward(mask=) with learnable codebooks")
            if any(b.use_cosine_sim for b in books):
                _unsupported("ResidualVQ.forward(mask=) with use_cosine_sim (the masked loss is taken against the un-normalised input, vqp:1319)")
            if any(not vq.return_zeros_for_masked_padding for vq in self.layers):
                _unsupported("ResidualVQ.forward(mask=) with return_zeros_for_masked_padding=False")
            if self.training and any(b.has_dead_code_replacement for b in books):
                _unsupported("ResidualVQ.forward(mask=) with dead-code replacement")
            # The reference hands the mask to every layer (rvq:495): a layer searches every row, but masked rows take no part
            # in its statistics or loss (vqp:599-600, :1317-1325) and come back as zeros / index -1 (vqp:1378-1396), so their
            # residual is never reduced and their running sum stays zero.  That is exactly the forward over the COMPACTED
            # unmasked rows with zeros / -1 scattered around it (stage-wise: the row count changes from call to call, a
            # cached program per count would not pay).  With gradients the layered path runs on those rows, gathered and
            # scattered under autograd, so project_in / project_out and the input get the gradients of the reference.
            assert x.ndim == 3 and mask.shape == x.shape[:2]
            rows = mask.reshape(-1).nonzero(as_tuple=True)[0]  # host sync (the reference's masked path syncs as well)
            masked = (rows, torch.zeros((mask.numel(), D), dtype=x.dtype, device=x.device),
                      torch.full((mask.numel(), Q), -1, dtype=torch.int64, device=x.device))

        if rows is not None and rows.numel() == 0:   # nothing to quantize: no quantizer runs, not even the dropout draw
            quantized = indices = None
            losses = torch.zeros((Q,), dtype=torch.float32, device=x.device)
            if self._takes_layered(x):   # zero losses and rows that stay in the graph: a zero gradient, as in VectorQuantize
                quantized = x.reshape(-1, D)[rows]
                indices = torch.empty((0, Q), dtype=torch.int64, device=x.device)
                losses = quantized.float().sum().repeat(Q)   # the sum over no rows is an exact zero
        elif self._takes_layered(x):
            xl = x.reshape(-1, D)[rows] if rows is not None else x
            quantized, indices, losses = self._quantize_layered(xl, freeze_codebook, self._active_layers(dropout_seed, x.device))
        else:
            if x.dtype not in _DTYPES:
                raise TypeError(f"vqb200 supports float32 and bfloat16 inputs, got {x.dtype}")
            flat = x.detach().reshape(-1, D)
            flat = flat[rows] if rows is not None else flat.contiguous()
            n_run = self._active_layers(dropout_seed, x.device)   # < Q: quantize dropout skips the layers after it
            do_update = self._do_update(books, freeze_codebook, n_run)
            if rows is None and n_run == Q and self._program_ok(books, do_update):
                quantized, indices, losses = _run_program(self, [self], [flat], [(books, do_update)])[0]
            else:
                rows0 = flat.shape[0] // shape[0] if (rows is None and len(shape) > 2) else flat.shape[0]
                quantized, indices, losses = self._quantize_stagewise(flat, books, do_update, n_run, freeze_codebook, rows0,
                                                                      pending)

        return self._tail(x, masked, quantized, indices, losses, return_all_codes)

    def _tail(self, x, masked, quantized, indices, losses, return_all_codes):
        """Rows out: the compacted rows scattered into zeros / index -1 (vqp:1378-1396), DiVeQ (rvq:603-606, in every mode),
        project_out (rvq:610) and the codes of `return_all_codes`."""
        shape = x.shape
        if masked is not None:
            rows, quantized_all, indices_all = masked
            if quantized is not None:
                quantized_all[rows] = quantized
                indices_all[rows] = indices
            quantized, indices = quantized_all, indices_all
        quantized = quantized.reshape(shape)
        if self.diveq:
            quantized = directional_reparam(x, quantized)
        ret = (self.project_out(quantized), indices.reshape(*shape[:-1], self.num_quantizers), losses)
        if return_all_codes:
            ret = (*ret, self.get_codes_from_indices(ret[1]))
        return ret

    def _active_layers(self, fixed_seed, device) -> int:
        """Number of leading layers that quantize in this forward: all, or in training with quantize_dropout (rvq:423-439) the
        cut `dropout_cut` draws."""
        if not (self.training and self.quantize_dropout):
            return self.num_quantizers
        return dropout_cut(self, fixed_seed, device)

    def _codebooks_need_grad(self):
        return any(vq._codebook.embed.requires_grad for vq in self.layers)

    def _program_ok(self, books, do_update):
        """One-call path (ops.RvqProgram): every stage deferred, no collective, no dead-code expiry, nothing parked on `.grad`
        (accum_ema_update), codebooks initialised and stackable.  Returns the program's op count (stages, running sum, one EMA
        op per updated stage, peer barrier, update_ema of a shared codebook), 0 when the forward cannot run as a program."""
        n_ops = len(books) + 1 + sum(do_update) + 2
        if os.environ.get("VQB_RVQ_PROGRAM", "1") == "0":
            return 0
        if ops.PROFILE_EVENTS is not None or not self.uniform_codebook_size:
            return 0
        if n_ops > ops.RvqProgram.MAX_OPS:
            return 0
        for b, u in zip(books, do_update):
            if not b._initted_host:
                return 0
            if u and (b.has_dead_code_replacement or b.cluster_size.grad is not None or b.embed_avg.grad is not None):
                return 0
        ddp = [b.use_ddp for b, u in zip(books, do_update) if u]
        if any(ddp):
            # multi-GPU: the statistics go to symmetric memory and the EMA ops sum over the ranks (barrier + peer loads inside
            # the program); without peer memory the stage-wise path does ONE NCCL all-reduce instead
            if not all(ddp):
                return 0
            dev, D = books[0].embed.device, books[0].embed.shape[-1]
            numel = sum(ops.stats_floats(b.codebook_size, D) for b, u in zip(books, do_update) if u)
            if self._peer_reducer(numel, dev) is None:
                return 0
        return n_ops

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

    def _quantize_stagewise(self, flat, books, do_update, n_run, freeze_codebook, rows0, pending):
        """One search call per active stage (rvq:469); the codebook updates follow the running sum."""
        N, D = flat.shape
        Q = self.num_quantizers
        dev = flat.device
        training = self.training
        losses = self._ensure_loss_buf(dev)
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
        updates = _CodebookUpdates(self, books, do_update, D, dev)
        updates.begin()
        updates.rows0 = rows0
        residual = flat  # rvq:411 (never written: stage 0 reads the caller's tensor)
        inline_embeds = []   # the shared codebook as each inline stage searched it
        for q, book in enumerate(books[:n_run]):  # rvq:469
            nxt = (bufs[q] if keep_inputs else bufs[q & 1]) if q + 1 < n_run else None
            if keep_inputs:
                updates.stage_inputs.append(residual)
            if updates.inline[q]:
                if not book._initted_host:   # k-means init precedes the search (quantize_rows would run it next)
                    book.init_embed_(book.transform_input(residual).float())
                inline_embeds.append(book.embed[0].clone())
            want_loss = training and self.layers[q].has_commitment_loss
            book.quantize_rows(
                residual, update=do_update[q], idx64_out=all_idx[:, q], idx_stride=Q,
                loss_out=losses[q:q + 1] if want_loss else None, loss_weight=self.layers[q].commitment_weight,
                resid_out=nxt, stats_out=updates.stats(q), defer_ema=not updates.inline[q])
            residual = nxt

        # quantized_out (rvq:410, :525): rebuilt from the indices of the stages that ran, in one pass over the codebooks they
        # searched, instead of a read-modify-write of (N x D) in every stage.  Only inline stages change a codebook between
        # stages.  Codebooks of different sizes are zero-padded to the largest: every index of a stage is below its own size.
        if inline_embeds:
            searched = torch.stack(inline_embeds)
        elif self.shared_codebook:
            searched = books[0].embed[0]
        else:
            searched = torch.nn.utils.rnn.pad_sequence([b.embed[0] for b in books[:n_run]], batch_first=True)
        quantized = ops.rvq_accumulate(searched, all_idx[:, :n_run].contiguous(), flat.dtype)

        if any(do_update):
            if pending is not None:
                pending.append(updates)
            else:
                _CodebookUpdates.apply_all([updates])
        return quantized, all_idx, losses.clone()

    def _quantize_layered(self, x, freeze_codebook, n_run):
        """Differentiable path: the reference's Python loop (rvq:469-568) over our VectorQuantize layers.
        n_run < Q: quantize dropout (rvq:473-476)."""
        quantized_out = torch.zeros_like(x)
        residual = x
        all_idx, all_losses = [], []
        for q, vq in enumerate(self.layers):
            if q >= n_run:
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
        D, Q = x.shape[-1], self.num_quantizers
        return quantized_out.reshape(-1, D), torch.stack(all_idx, dim=-1).reshape(-1, Q), torch.stack(all_losses)


class GroupedResidualVQ(GroupedResidual):
    def __init__(self, *, dim, groups=1, accept_image_fmap=False, **kwargs):
        if accept_image_fmap:
            _unsupported("GroupedResidualVQ(accept_image_fmap=True)")
        super().__init__(ResidualVQ, dim=dim, groups=groups, accept_image_fmap=accept_image_fmap, **kwargs)  # rvq:646-658

    def _program_ok(self, xs, freeze_codebook):
        """All groups in one ops.RvqProgram: every group takes its own program path (ResidualVQ._program_ok), and the op list
        fits.  Returns every group's (codebooks, stages that update), or None."""
        if any(rvq.diveq or rvq._takes_layered(x) or not x.is_cuda or x.dtype not in _DTYPES for rvq, x in zip(self.rvqs, xs)):
            return None
        plan, n_ops = [], 0
        for rvq in self.rvqs:
            books = rvq._stage_plan()
            upd = rvq._do_update(books, freeze_codebook, rvq.num_quantizers)
            n = rvq._program_ok(books, upd)
            if not n:
                return None
            plan.append((books, upd))
            n_ops += n
        return plan if n_ops <= ops.RvqProgram.MAX_OPS else None

    def forward(self, x, indices=None, return_all_codes=False, sample_codebook_temp=None, freeze_codebook=False, mask=None):
        if indices is not None:
            _unsupported("GroupedResidualVQ.forward(indices=)")
        assert x.shape[-1] == self.dim
        chunks = x.chunk(self.groups, dim=-1)  # rvq:690
        if self.training:
            # the reference draws one torch.randint here even without quantize-dropout (rvq:701 -> :96-103);
            # consume it too so that seeded runs stay aligned with the reference's RNG stream.
            seed = sync_seed(x.device)
        dropout_seed = None
        if self.training and any(rvq.quantize_dropout for rvq in self.rvqs):
            dropout_seed = int(seed.item())   # rvq:701: the SAME dropout index in every group
        if mask is not None:   # rvq:698: every group receives the mask
            outs = [rvq(c, mask=mask, freeze_codebook=freeze_codebook, return_all_codes=return_all_codes,
                        rand_quantize_dropout_fixed_seed=dropout_seed) for rvq, c in zip(self.rvqs, chunks)]
        else:
            xs = [rvq.project_in(c) for rvq, c in zip(self.rvqs, chunks)]
            plan = self._program_ok(xs, freeze_codebook) if dropout_seed is None else None
            if plan is not None:   # every group in ONE call; the groups' cat / stack copy the plan's persistent outputs
                flats = [xp.detach().reshape(-1, xp.shape[-1]) for xp in xs]   # strided views of the groups' columns
                outs = [rvq._tail(xp, None, *o, return_all_codes)
                        for rvq, xp, o in zip(self.rvqs, xs, _run_program(self, self.rvqs, flats, plan, persistent_io=True))]
            else:
                pending = []
                outs = [rvq._forward_projected(xp, None, return_all_codes, freeze_codebook, dropout_seed, pending)
                        for rvq, xp in zip(self.rvqs, xs)]  # rvq:706
                _CodebookUpdates.apply_all(pending)   # without peer memory: ONE NCCL collective for every group
        quantized = torch.cat([o[0] for o in outs], dim=-1)  # rvq:719-721
        all_indices = torch.stack([o[1] for o in outs])
        commit_losses = torch.stack([o[2] for o in outs])
        ret = (quantized, all_indices, commit_losses)
        if return_all_codes:
            ret = (*ret, torch.stack([o[3] for o in outs]))
        return ret
