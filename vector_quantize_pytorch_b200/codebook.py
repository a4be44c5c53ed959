"""`Codebook` — host-side mirror of the reference's `Codebook` (vector_quantize_pytorch.py:349-791).

Same constructor arguments, same persistent buffers (`initted`, `cluster_size`, `embed_avg`, `embed`
with a leading num_codebooks=1 dim, vqp:415-423) so reference checkpoints load unchanged.  The
arithmetic of `forward` runs in the sm_90a kernels (`ops.py`); anything that is not on the hot
path (SURVEY.md §8) raises NotImplementedError instead of silently taking a slow path.
"""
from __future__ import annotations

import torch
import torch.distributed as distributed
import torch.nn.functional as F
from torch import nn

from . import ops
from .dist import allreduce_packed, PeerReducer


def _uniform_init(*shape):
    # same RNG consumption as the reference (vqp:112-115): kaiming_uniform_ on an (H, K, D) tensor
    t = torch.empty(shape)
    nn.init.kaiming_uniform_(t)
    return t


def _unsupported(what):
    raise NotImplementedError(f"vqb200: {what} is outside the accelerated hot path (SURVEY.md §8) and is not implemented")


class _LearnableCodebook(torch.autograd.Function):
    """Makes the kernels' `quantize` (and the commitment loss) differentiable w.r.t. a learnable `embed` (1, K, D).

    The reference's `quantize = onehot @ embed` (vqp:766) — and its gathers from `embed` (vqp:779-781, :998-1018) — send every
    row's upstream gradient to its code: d embed[k] = sum of the gradient rows n with idx(n) = k, taken by the statistics chain
    (ops.ema_stats) on those rows.  `valid` (bool per row, optional): rows whose index was -1 (zeros, no code) send nothing.
    The commitment loss `mse(quantize, x)` (vqp:1214-1216, :1327) adds scale * (count_k c_k - sum_{n -> k} x_n) per code, where
    `commit_rows` is that K x D difference, formed from the search's own statistics before any codebook change."""

    @staticmethod
    def forward(ctx, embed, q, loss, idx32, commit_rows, commit_scale, valid=None):
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(idx32, commit_rows, valid)
        ctx.commit_scale = commit_scale
        ctx.embed_shape = embed.shape
        return q, loss

    @staticmethod
    def backward(ctx, g_q, g_loss):
        idx32, rows, valid = ctx.saved_tensors
        H, K, D = ctx.embed_shape
        grad = None
        if g_q is not None:
            g = g_q.reshape(-1, D)
            if valid is not None:
                g = g.masked_fill(~valid[:, None], 0)
            stats = ops.ema_stats(g.contiguous(), idx32, K)
            off = ops.stats_offset(K)
            grad = stats[off:off + K * D].view(K, D)
        if rows is not None and g_loss is not None:
            part = rows * (g_loss.float() * ctx.commit_scale)
            grad = part if grad is None else grad + part
        return (None if grad is None else grad.view(H, K, D)), None, g_loss, None, None, None, None


class Codebook(nn.Module):
    def __init__(
        self,
        dim,
        codebook_size,
        num_codebooks=1,
        kmeans_init=False,
        kmeans_iters=10,
        sync_kmeans=True,
        decay=0.8,
        eps=1e-5,
        threshold_ema_dead_code=2,
        reset_cluster_size=None,
        use_ddp=False,
        learnable_codebook=False,
        gumbel_sample=None,
        sample_codebook_temp=1.,
        ema_update=True,
        manual_ema_update=False,
        affine_param=False,
        sync_affine_param=False,
        affine_param_batch_decay=0.99,
        affine_param_codebook_decay=0.9,
        use_cosine_sim=False,
        vq_bridge=None,
    ):
        super().__init__()
        if num_codebooks < 1:
            raise ValueError("num_codebooks must be >= 1")
        if kmeans_init and use_ddp and sync_kmeans:
            _unsupported("kmeans_init with distributed sampling (use_ddp + sync_kmeans, vqp:211-229)")
        if learnable_codebook and ema_update:
            _unsupported("learnable_codebook with ema_update (the reference rejects the combination, vqp:908)")
        if learnable_codebook and use_cosine_sim:
            _unsupported("learnable_codebook with use_cosine_sim (the reference rejects the combination, vqp:884)")
        if learnable_codebook and num_codebooks > 1:
            _unsupported("learnable_codebook with num_codebooks > 1 (separate codebooks per head)")
        if affine_param:
            _unsupported("affine_param")
        if vq_bridge is not None:
            _unsupported("vq_bridge")
        if gumbel_sample is not None:
            _unsupported("a custom gumbel_sample (stochastic code sampling)")
        if threshold_ema_dead_code > 0 and use_ddp and sync_kmeans:
            _unsupported("dead-code replacement with distributed sampling (use_ddp + sync_kmeans, vqp:211-229)")

        self.dim = dim
        self.decay = decay
        self.ema_update = ema_update
        self.manual_ema_update = manual_ema_update
        self.codebook_size = codebook_size
        self.num_codebooks = num_codebooks
        self.eps = eps
        self.threshold_ema_dead_code = threshold_ema_dead_code
        self.has_dead_code_replacement = threshold_ema_dead_code > 0
        self.reset_cluster_size = reset_cluster_size if reset_cluster_size is not None else threshold_ema_dead_code
        self.sample_codebook_temp = sample_codebook_temp
        self.use_ddp = use_ddp
        self.sync_kmeans = sync_kmeans
        self.learnable_codebook = learnable_codebook
        self.use_cosine_sim = use_cosine_sim

        self.kmeans_iters = kmeans_iters
        if kmeans_init:
            embed = torch.zeros(num_codebooks, codebook_size, dim)  # vqp:383
        else:
            embed = _uniform_init(num_codebooks, codebook_size, dim)  # vqp:385
            if use_cosine_sim:
                embed = F.normalize(embed, p=2, dim=-1, eps=1e-6)  # vqp:387-388
        self._initted_host = not kmeans_init   # host-side copy of `initted`: no device sync per forward once True

        self.register_buffer("initted", torch.tensor(not kmeans_init))  # vqp:415
        self.register_buffer("cluster_size", torch.ones(num_codebooks, codebook_size))  # vqp:416
        self.register_buffer("embed_avg", embed.clone())  # vqp:417
        if learnable_codebook:  # vqp:419-421: same state_dict key and shape, trained by the caller's optimizer
            self.embed = nn.Parameter(embed)
        else:
            self.register_buffer("embed", embed)  # vqp:423

        # num_codebooks > 1 (VectorQuantize(separate_codebook_per_head=True), vqp:1044-1049): every head is served by a light
        # view of this module (`head(i)`): same buffers, own slot, own operand cache
        self._slot = 0
        self._head_views = None
        self._operands: ops.CodebookOperands | None = None
        self._operands_key = None
        self._scratch = ops.Scratch()   # the search scratch of `quantize_rows` (a plain attribute: not in the state_dict)
        self._peer = None          # dist.PeerReducer of this codebook's packed statistics (use_ddp, created on first use)
        self._peer_tried = False

    # ------------------------------------------------------------------ operand cache
    def _state2d(self):
        """(cluster_size (K,), embed_avg (K, D), embed (K, D)) views sharing storage with the buffers."""
        i = self._slot
        return self.cluster_size[i], self.embed_avg[i], self.embed[i]

    def head(self, i: int) -> "Codebook":
        """The view of this module that works on codebook `i` of the (num_codebooks, K, D) buffers.  A shallow copy: it shares
        the buffer dict with its parent (so `.to()`, `load_state_dict` reach it) and keeps its own slot, operand cache and
        search scratch."""
        if self.num_codebooks == 1:
            return self
        if self._head_views is None:
            import copy
            views = []
            for j in range(self.num_codebooks):
                v = copy.copy(self)
                v._slot, v._head_views, v._operands, v._operands_key, v._peer, v._peer_tried = j, None, None, None, None, False
                v._scratch = ops.Scratch()
                views.append(v)
            self._head_views = views
        v = self._head_views[i]
        v.training = self.training
        return v

    def operands(self) -> ops.CodebookOperands:
        """bf16 hi/lo planes + bias of the current `embed`, rebuilt whenever `embed` was changed by
        anything other than our own EMA kernel (load_state_dict, `.codebook = ...`, `.to(device)`)."""
        embed = self.embed
        if not embed.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: move the module to a CUDA (H100) device")
        if embed.dtype != torch.float32 or not embed.is_contiguous():
            raise RuntimeError("vqb200: the `embed` buffer must be contiguous float32")
        key = (embed.data_ptr(), embed._version, embed.device)
        # a learnable codebook is written by the caller's optimizer, and not every optimizer step bumps `embed._version` (the
        # fused Adam kernels do not): its operands are rebuilt for every search
        if self._operands is None or self._operands_key != key or embed.requires_grad:
            reuse = self._operands if (self._operands is not None and self._operands.planes.device == embed.device) else None
            self._operands = ops.prepare_codebook(embed.detach()[self._slot], self.use_cosine_sim, out=reuse)
            self._operands_key = key
        return self._operands

    def _mark_operands_fresh(self):
        e = self.embed
        self._operands_key = (e.data_ptr(), e._version, e.device)

    def learns(self) -> bool:
        """True when this forward must carry a gradient to `embed` (learnable codebook, grad enabled)."""
        return torch.is_grad_enabled() and self.embed.requires_grad

    def decode(self, indices: torch.Tensor) -> torch.Tensor:
        """embed[slot][indices] (int64, -1 -> zeros) in fp32, shape indices.shape + (D,): the vqb_decode gather, differentiable
        w.r.t. a learnable `embed` like the reference's gather from the parameter (vqp:998-1018)."""
        codes = ops.decode(self.embed.detach()[self._slot], indices.unsqueeze(-1).contiguous())
        if self.learns():
            idx = indices.reshape(-1)
            codes, _ = _LearnableCodebook.apply(self.embed, codes, None, idx.clamp_min(0).to(torch.int32).contiguous(), None, 0.,
                                                idx >= 0)
        return codes

    # ------------------------------------------------------------------ reference surface
    def transform_input(self, t):  # vqp:376
        return F.normalize(t, p=2, dim=-1, eps=1e-6) if self.use_cosine_sim else t

    def peer_reducer(self):
        """Symmetric-memory statistics buffers for the fused multi-GPU EMA (csrc/vq_peer.cu); None -> NCCL all-reduce.
        Created on the first training forward (a collective rendezvous: every rank gets here in the same call)."""
        if not self._peer_tried:
            self._peer_tried = True
            if self.use_ddp and self.embed.is_cuda:
                self._peer = PeerReducer.create(ops.stats_floats(self.codebook_size, self.dim), self.embed.device)
        return self._peer

    def lerp_stats_peers(self, peer, peer_ptrs, slice_offset: int, normalise: bool):
        """`lerp_stats` with the sum over ranks taken inside the EMA kernels (call `peer.barrier()` first)."""
        cs, ea, emb = self._state2d()
        cb = self.operands()
        ops.ema_apply_peers(cs, ea, emb, peer, peer_ptrs, slice_offset, cb, decay=self.decay, eps=self.eps, do_normalise=normalise)
        if normalise:
            self._mark_operands_fresh()

    def sync_stats(self, stats: torch.Tensor) -> torch.Tensor:
        """The reference all-reduces cluster_size and embed_sum separately (vqp:603, :607); the packed
        buffer needs ONE all-reduce (NCCL over NVLink)."""
        if self.use_ddp:
            allreduce_packed(stats)
        return stats

    def _stat_views(self, stats: torch.Tensor):
        """(cluster_size (1, K), embed_sum (1, K, D)) views of a packed statistics buffer."""
        K, D = self.codebook_size, self.dim
        off = ops.stats_offset(K)
        return stats[:K].view(1, K), stats[off:off + K * D].view(1, K, D)

    def lerp_stats(self, stats: torch.Tensor, normalise: bool, ema_update_weight=None, accum_ema_update: bool = False):
        """track_cluster_size_and_embed_avg after the all-reduce (vqp:609-617): the custom per-code weight
        (tensor (K,) / (1, K) or callable of (embed_sum, cluster_size), vqp:86-97, :609-610), `accum_ema_update`
        (park the batch statistics on the buffers' `.grad`, vqp:70-74, :612-614 — folded into the next normal update,
        vqp:80-82), then ema_inplace of both buffers and, unless manual, update_ema (vqp:638-639).
        Returns False when the statistics were only accumulated (the reference then skips update_ema and expiry)."""
        cs_new, es_new = self._stat_views(stats)
        if callable(ema_update_weight):
            ema_update_weight = ema_update_weight(es_new, cs_new)
        if accum_ema_update:
            for buf, new in ((self.cluster_size, cs_new), (self.embed_avg, es_new)):
                if buf.grad is not None:
                    buf.grad.add_(new)
                else:
                    buf.grad = new.clone().detach()
            return False
        for buf, new in ((self.cluster_size, cs_new), (self.embed_avg, es_new)):  # vqp:80-82
            if buf.grad is not None:
                new.add_(buf.grad)
                buf.grad = None
        weight = None
        if ema_update_weight is not None:
            if torch.is_tensor(ema_update_weight):
                weight = ema_update_weight.to(device=stats.device, dtype=torch.float32).reshape(-1).contiguous()
                assert weight.numel() == self.codebook_size, "ema_update_weight must have one entry per code"
            else:  # a python scalar scales every code alike
                weight = torch.full((self.codebook_size,), float(ema_update_weight), dtype=torch.float32, device=stats.device)
        cs, ea, emb = self._state2d()
        cb = self.operands()
        ops.ema_apply(cs, ea, emb, stats, cb, decay=self.decay, eps=self.eps, do_lerp=True, do_normalise=normalise,
                      code_weight=weight)
        if normalise:
            self._mark_operands_fresh()
        return True

    def updates(self, training: bool, freeze_codebook: bool, ema_update=None) -> bool:
        """Whether a forward changes this codebook: in training, not frozen, with an EMA update or dead-code replacement to do
        (vqp:628-641).  `ema_update` None: the module's setting."""
        ema_update = self.ema_update if ema_update is None else ema_update
        return training and not freeze_codebook and (ema_update or self.has_dead_code_replacement)

    def apply_stats(self, stats: torch.Tensor, samples, ema_update=None, ema_update_weight=None, accum_ema_update: bool = False):
        """One EMA step from a batch's packed statistics: all-reduce, lerp (`lerp_stats`), then dead-code expiry (vqp:641) unless
        the statistics were only parked by `accum_ema_update`.  `samples()` gives expiry its rows; it is called only when codes
        can expire, so the fp32 copy of the batch is made only then."""
        ema_update = self.ema_update if ema_update is None else ema_update
        self.sync_stats(stats)
        if (self.lerp_stats(stats, normalise=ema_update and not self.manual_ema_update, ema_update_weight=ema_update_weight,
                            accum_ema_update=accum_ema_update) and self.has_dead_code_replacement):
            self.expire_codes_(samples())

    def update_ema(self):  # vqp:576-584
        cs, ea, emb = self._state2d()
        cb = self.operands()
        ops.ema_apply(cs, ea, emb, None, cb, decay=self.decay, eps=self.eps, do_lerp=False, do_normalise=True)
        self._mark_operands_fresh()

    @torch.no_grad()
    def init_embed_(self, data):
        """vqp:451-473 + :238-278: k-means initialisation from the first batch (`data`: the fp32 `flatten` of vqp:692-698,
        already l2-normalised for cosine).  Every Lloyd iteration is the hot path itself — tensor-core search with the
        exact re-score, then the counting-sort statistics — so the bucket of every sample follows the reference's
        argmax(-cdist) / argmax(dot) rule exactly; only the K x D mean update is torch glue."""
        if self._initted_host:
            return
        if bool(self.initted):  # e.g. a loaded checkpoint: one host sync, then never again
            self._initted_host = True
            return
        self._kmeans_init(data)
        self.initted.data.copy_(torch.tensor(True))
        self._initted_host = True

    @torch.no_grad()
    def _kmeans_init(self, data):
        """The Lloyd iterations of `init_embed_` for THIS slot (no `initted` bookkeeping)."""
        samples = data.reshape(-1, data.shape[-1]).float().contiguous()
        n, K = samples.shape[0], self.codebook_size
        # sample_vectors (vqp:156-163)
        picks = torch.randperm(n, device=samples.device)[:K] if n >= K else torch.randint(0, n, (K,), device=samples.device)
        means = samples[picks].contiguous()
        off = ops.stats_offset(K)
        bins = torch.zeros((K,), dtype=torch.float32, device=samples.device)
        cb = None
        for _ in range(self.kmeans_iters):
            cb = ops.prepare_codebook(means, self.use_cosine_sim, out=cb)
            res = ops.search(samples, cb, means, normalise=False)           # vqp:251-256
            stats = ops.ema_stats(samples, res.idx, K)                      # vqp:257, :265
            bins = stats[:K]
            sums = stats[off:off + K * samples.shape[1]].view(K, -1)
            new = sums / bins.clamp(min=1.)[:, None]                        # vqp:260-266
            if self.use_cosine_sim:
                new = F.normalize(new, p=2, dim=-1, eps=1e-6)               # vqp:269-270
            means = torch.where((bins == 0)[:, None], means, new).contiguous()  # vqp:272-276
        self.embed_avg.data[self._slot].copy_(means * bins[:, None])        # vqp:467-469
        self.cluster_size.data[self._slot].copy_(bins)                      # vqp:470
        self._operands_key = None
        self.update_ema()                                                   # vqp:471

    @torch.no_grad()
    def expire_codes_(self, batch_samples):  # vqp:544-574 (PyTorch glue: RNG-bound, cold, off by default)
        """`batch_samples` as the reference's call site passes them: the fp32 `flatten` from Codebook.forward (vqp:641),
        tensors in the input dtype from ResidualVQ's final expiry (rvq:601) — `replace` re-normalises in THAT dtype."""
        if not self.has_dead_code_replacement or not self.training:
            return
        expired = self.cluster_size[self._slot] < self.threshold_ema_dead_code
        if not torch.any(expired):  # host sync, exactly like the reference (vqp:570)
            return
        samples = batch_samples.reshape(-1, batch_samples.shape[-1])
        if self.use_cosine_sim:
            samples = F.normalize(samples, p=2, dim=-1, eps=1e-6)
        num = int(expired.sum().item())
        n = samples.shape[0]
        if n >= num:  # vqp:156-163 sample_vectors
            pick = torch.randperm(n, device=samples.device)[:num]
        else:
            pick = torch.randint(0, n, (num,), device=samples.device)
        sampled = samples[pick].to(self.embed.dtype)
        self.embed.data[self._slot][expired] = sampled
        self.cluster_size.data[self._slot][expired] = self.reset_cluster_size
        self.embed_avg.data[self._slot][expired] = sampled * self.reset_cluster_size
        # `.data[...] =` does not bump embed._version: without this the next search would still use the bf16 planes /
        # bias of the replaced rows
        self._operands_key = None

    @torch.no_grad()
    def update_indices(self, x, embed_ind, mask=None, ema_update_weight=None, accum_ema_update=False, ema_update=None):
        """vqp:643-668: EMA update from (x, indices) alone (tests/test_beam.py:8-45 of the reference)."""
        if mask is not None:
            _unsupported("update_indices with a mask")
        ema_update = self.ema_update if ema_update is None else ema_update
        if not ema_update and not self.has_dead_code_replacement:
            return
        flat = x.reshape(-1, x.shape[-1])
        if flat.dtype not in (torch.float32, torch.bfloat16):
            flat = flat.float()
        flat = flat.contiguous()
        idx = embed_ind.reshape(-1).to(torch.int32).clamp_min(0).contiguous()
        self.apply_stats(ops.ema_stats(flat, idx, self.codebook_size), flat.float, ema_update, ema_update_weight,
                         accum_ema_update)

    @torch.no_grad()
    def update_codebook(self, flatten, embed_onehot, mask=None, ema_update_weight=None, accum_ema_update=False,
                        ema_update=None):
        """vqp:619-641.  The reference passes the one-hot assignment; the kernels work from indices."""
        self.update_indices(flatten, embed_onehot.argmax(dim=-1), mask=mask, ema_update_weight=ema_update_weight,
                            accum_ema_update=accum_ema_update, ema_update=ema_update)

    @torch.no_grad()
    def track_cluster_size_and_embed_avg(self, flatten, embed_onehot, mask=None, ema_update_weight=None,
                                         accum_ema_update=False):
        """vqp:586-617: batch statistics -> (all-reduce) -> lerp of cluster_size / embed_avg, nothing else."""
        if mask is not None:
            _unsupported("track_cluster_size_and_embed_avg with a mask")
        flat = flatten.reshape(-1, flatten.shape[-1])
        flat = (flat if flat.dtype in (torch.float32, torch.bfloat16) else flat.float()).contiguous()
        idx = embed_onehot.argmax(dim=-1).reshape(-1).to(torch.int32).contiguous()
        stats = self.sync_stats(ops.ema_stats(flat, idx, self.codebook_size))
        self.lerp_stats(stats, normalise=False, ema_update_weight=ema_update_weight, accum_ema_update=accum_ema_update)

    update_ema_indices = update_indices

    # ------------------------------------------------------------------ the hot path
    @torch.no_grad()
    def quantize_rows(self, x: torch.Tensor, *, update: bool, q_out=None, idx64_out=None, idx_stride=1, loss_out=None,
                      loss_weight=1.0, resid_out=None, stats_out=None, defer_ema=False, margin=None,
                      ema_update=None, ema_update_weight=None, accum_ema_update=False,
                      row_mask=None, n_live=None, on_stats=None):
        """x (N, D) contiguous fp32/bf16 — the input BEFORE the cosine l2norm (done in-kernel).

        One C call: search (pre-update codebook, vqp:743-747) with the fused gather / loss / residual tail
        (vqp:766, :1178, :1327; rvq:524) -> batch statistics (vqp:602-607) -> EMA apply (vqp:616-617, :576-584).
        With defer_ema (or when the statistics must be all-reduced first) the EMA apply is left to the caller.
        row_mask (N,) uint8 + n_live (1,) int64: in-kernel padding mask (vqp:1116-1119; ops.vq_forward_args) — the caller has made
        sure that neither k-means init nor dead-code expiry (both sample from `x[mask]`) can run in this call.
        on_stats: called with this batch's statistics [count | sum of rows] right after the search, before any all-reduce or
        codebook change (the commitment gradient of a learnable codebook); the search then always produces them.
        Returns (idx32, stats or None).
        """
        if not self._initted_host:
            self.init_embed_(self.transform_input(x).float())   # vqp:703 (every mode, like the reference)
        cb = self.operands()
        ema_update = self.ema_update if ema_update is None else ema_update   # per-call override (vqp:628)
        custom = ema_update_weight is not None or accum_ema_update or any(
            b.grad is not None for b in (self.cluster_size, self.embed_avg))
        apply_here = update and not defer_ema and not self.use_ddp and not custom and on_stats is None
        mode = 0 if not (update or on_stats is not None) else (2 if apply_here else 1)
        normalise = ema_update and not self.manual_ema_update
        peer = peer_ptrs = None
        if update and not defer_ema and self.use_ddp and not custom and stats_out is None and on_stats is None:
            peer = self.peer_reducer()
            if peer is not None:   # multi-GPU step in ONE chain: statistics -> peer barrier -> reduce + EMA (vq_peer.cu)
                mode = 3
                stats_out, peer_ptrs = peer.next_buffer()
        idx32, stats = ops.vq_forward(
            x, cb, self._state2d(), update=mode, do_normalise=normalise, decay=self.decay, eps=self.eps, q_out=q_out,
            idx64_out=idx64_out, idx_stride=idx_stride, loss_out=loss_out, loss_weight=loss_weight, resid_out=resid_out,
            stats=stats_out, margin=margin, scratch=self._scratch,
            peer=peer, peer_ptrs=peer_ptrs, row_mask=row_mask, n_live=n_live)
        if mode >= 2 and normalise:
            self._mark_operands_fresh()
        if on_stats is not None:
            on_stats(stats)
        if update and not defer_ema:
            if mode == 1:
                self.apply_stats(stats, lambda: self.transform_input(x).float(), ema_update, ema_update_weight,
                                 accum_ema_update)
            elif self.has_dead_code_replacement:
                self.expire_codes_(self.transform_input(x).float())  # vqp:692: `flatten` is fp32
        return idx32, stats

    def forward(self, x, sample_codebook_temp=None, mask=None, freeze_codebook=False, codebook_transform_fn=None,
                ema_update_weight=None, accum_ema_update=False, ema_update=None, topk=None, update_usage=True):
        """Reference contract (vqp:674-686, :791): returns (quantize fp32, embed_ind int64, dist).

        `x` is the already-transformed input (the reference applies `transform_input` in the caller,
        vqp:1159).  `dist` — the (N x K) matrix the kernels never materialise — is returned as None.
        """
        if mask is not None:
            _unsupported("mask")
        if codebook_transform_fn is not None:
            _unsupported("codebook_transform_fn (implicit neural codebooks)")
        if topk is not None:
            _unsupported("topk")
        if self.num_codebooks > 1 and self._head_views is None and self._slot == 0 and x.ndim == 4:
            _unsupported("Codebook.forward on (h, b, n, d) inputs: go through VectorQuantize(separate_codebook_per_head=True)")
        shape = x.shape
        flat = x.reshape(-1, shape[-1])
        if flat.dtype not in (torch.float32, torch.bfloat16):
            flat = flat.float()
        flat = flat.contiguous()
        if not self._initted_host:
            self.init_embed_(flat.float())   # vqp:703
        cb = self.operands()
        embed2d = self.embed.detach()[self._slot]
        with torch.no_grad():
            res = ops.search(flat, cb, embed2d, normalise=False)  # the caller already applied transform_input
            q = torch.empty((flat.shape[0], shape[-1]), dtype=torch.float32, device=flat.device)
            idx64 = torch.empty((flat.shape[0],), dtype=torch.int64, device=flat.device)
            x32 = res.x_eff if res.x_eff.dtype == torch.float32 else res.x_eff.float()
            ops.gather(x32, embed2d, res.idx, q_out=q, idx64_out=idx64)
            if self.updates(self.training and update_usage, freeze_codebook, ema_update):
                self.apply_stats(ops.ema_stats(res.x_eff, res.idx, self.codebook_size), res.x_eff.float, ema_update,
                                 ema_update_weight, accum_ema_update)
        if self.learns():   # vqp:710, :766: `quantize` carries each row's gradient to its code
            q, _ = _LearnableCodebook.apply(self.embed, q, None, res.idx.clone(), None, 0.)
        return q.reshape(shape), idx64.reshape(shape[:-1]), None


class EuclideanCodebook(Codebook):
    """Legacy name (pre-1.2x releases of the reference); `Codebook` with use_cosine_sim=False."""

    def __init__(self, *args, **kwargs):
        kwargs["use_cosine_sim"] = False
        super().__init__(*args, **kwargs)


class CosineSimCodebook(Codebook):
    """Legacy name; `Codebook` with use_cosine_sim=True."""

    def __init__(self, *args, **kwargs):
        kwargs["use_cosine_sim"] = True
        super().__init__(*args, **kwargs)
