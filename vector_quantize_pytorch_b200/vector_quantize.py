"""`VectorQuantize` — drop-in for the reference module (vector_quantize_pytorch.py:802-1403) on the
default path: heads=1, no mask, Euclidean or cosine codebook with EMA updates.

forward(x) -> (quantize [x.dtype, x.shape], embed_ind [int64, x.shape[:-1]], loss [fp32 scalar]).
Layout handling, projections, STE / rotation trick stay PyTorch glue; the search, gather, commitment
loss and EMA run in the sm_90a kernels.  Unsupported constructor / forward options raise.
"""
from __future__ import annotations

import math
from collections import namedtuple

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .codebook import Codebook, _LearnableCodebook, _unsupported

LossBreakdown = namedtuple("LossBreakdown", ["commitment", "codebook_diversity", "orthogonal_reg", "inplace_optimize"])


def _is_distributed():
    import torch.distributed as dist
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def _safe_div(num, den, eps=1e-6):
    return num / den.clamp(min=eps)


def straight_through(src, tgt):  # vqp:282-283
    return src + (tgt - src).detach()


class _RotateTo(torch.autograd.Function):
    """Rotation-trick gradient estimator (arXiv:2410.06424 §4.2; reference vqp:287-318) on the sm_90a kernels: the forward
    value (numerically the quantized vector) and d/d src — the direction / norm factors are constants of the backward pass,
    exactly like the reference's `.detach()`s."""

    @staticmethod
    def forward(ctx, src, tgt):
        ctx.save_for_backward(src, tgt)
        return ops.rotate(src.detach(), tgt.detach())

    @staticmethod
    def backward(ctx, grad_out):
        src, tgt = ctx.saved_tensors
        return ops.rotate(src.detach(), tgt.detach(), grad_out.to(src.dtype)), None


def rotate_to(src, tgt):
    return _RotateTo.apply(src, tgt)


class _MaskedEstimator(torch.autograd.Function):
    """The estimator and commitment-loss gradient of a masked training step on the in-kernel masked search (vqb_rotate_masked).
    Forward: the searched codes on live rows, the padding value on padding rows (the values of the no-grad call, bit for bit)
    and the kernels' commitment loss.  Backward, in one kernel: the estimator's gradient plus
    2 w dL/dloss (x - q) / (n_live D) on live rows, 0 or the upstream gradient on padding rows.  n_live stays on the device."""

    @staticmethod
    def forward(ctx, x, q, commit, row_mask, n_live, estimator, pad_zeros, loss_weight):
        ctx.save_for_backward(x, q, row_mask, n_live)
        ctx.cfg = (estimator, pad_zeros, loss_weight, commit is not None)
        out = ops.rotate_masked(x.detach(), q, row_mask, estimator, pad_zeros)
        return out, (commit.clone() if commit is not None else torch.zeros((), dtype=torch.float32, device=x.device))

    @staticmethod
    def backward(ctx, grad_out, grad_loss):
        x, q, row_mask, n_live = ctx.saved_tensors
        estimator, pad_zeros, loss_weight, has_loss = ctx.cfg
        gl = grad_loss.float().reshape(1).contiguous() if has_loss else None
        dx = ops.rotate_masked(x.detach(), q, row_mask, estimator, pad_zeros, grad_out.to(x.dtype).contiguous(), gl, n_live,
                               loss_weight)
        return dx, None, None, None, None, None, None, None


def _with_grad_of(value, expr):
    """`value` carrying the gradient of `expr`, which equals it up to rounding (an estimator of it, or the same loss taken by
    autograd): the forward keeps the bits of the call without gradients."""
    return value + (expr - expr.detach())


def diveq_noise(like):
    """The N(0, 1) draw of DiVeQ (`torch.randn_like(error_dir)`, vqp:327), in `like`'s shape and dtype.  Every DiVeQ forward
    of this package draws through this one function."""
    return torch.randn_like(like)


class _DiVeQ(torch.autograd.Function):
    """DiVeQ estimator (vqp:323-330) on the vqb_diveq kernel: x + l2norm(q - x + s z) ||q - x|| with the direction detached.
    The backward recomputes the row scalars from (x, q, z)."""

    @staticmethod
    def forward(ctx, src, tgt, noise, scale):
        ctx.save_for_backward(src, tgt, noise)
        ctx.scale = scale
        return ops.diveq(src.detach(), tgt.detach(), noise, scale)

    @staticmethod
    def backward(ctx, grad_out):
        src, tgt, noise = ctx.saved_tensors
        dx, dq = ops.diveq(src.detach(), tgt.detach(), noise, ctx.scale, grad_out.to(src.dtype))
        return dx, dq.to(tgt.dtype), None, None


def directional_reparam(src, tgt, noise_variance=5e-3):
    """vqp:323-330; src and tgt in one dtype (the noise is drawn in it, after the codebook forward like the reference's)."""
    return _DiVeQ.apply(src, tgt, diveq_noise(tgt), math.sqrt(noise_variance))


def host_chunk_bounds(N: int, n_chunks: int):
    """Row boundaries [0, b1, ..., N] of the chunks `forward_host` streams through the GPU.

    Chunk sizes ramp up and down (1, 2, 3, 3, ..., 3, 2, 1 units): the first upload and the last download are not
    overlapped with anything, so they are kept short; the middle chunks are large to amortise per-chunk costs.
    Interior boundaries are multiples of 256 rows (whole CTA-pair tiles, 16-byte aligned row offsets)."""
    n_chunks = max(1, int(n_chunks))
    wts = [min(c + 1, n_chunks - c, 3) for c in range(n_chunks)]
    unit = N / sum(wts)
    bounds, acc = [0], 0.0
    for wgt in wts:
        acc += wgt * unit
        b_ = min(N, -(-int(round(acc)) // 256) * 256)
        if b_ > bounds[-1]:
            bounds.append(b_)
    bounds[-1] = N
    return bounds


class VectorQuantize(nn.Module):
    def __init__(
        self,
        dim,
        codebook_size,
        codebook_dim=None,
        heads=1,
        separate_codebook_per_head=False,
        decay=0.8,
        eps=1e-5,
        freeze_codebook=False,
        kmeans_init=False,
        kmeans_iters=10,
        sync_kmeans=True,
        use_cosine_sim=False,
        layernorm_after_project_in=False,
        threshold_ema_dead_code=0,
        channel_last=True,
        accept_image_fmap=False,
        accept_3d_fmap=False,
        commitment_weight=1.,
        commitment_use_cross_entropy_loss=False,
        orthogonal_reg_weight=0.,
        orthogonal_reg_active_codes_only=False,
        orthogonal_reg_max_codes=None,
        codebook_diversity_loss_weight=0.,
        codebook_diversity_temperature=100.,
        stochastic_sample_codes=False,
        sample_codebook_temp=1.,
        straight_through=False,
        rotation_trick=None,
        directional_reparam=False,
        directional_reparam_variance=5e-3,
        sync_codebook=None,
        sync_affine_param=False,
        ema_update=None,
        vq_bridge=None,
        manual_ema_update=False,
        learnable_codebook=None,
        in_place_codebook_optimizer=None,
        manual_in_place_optimizer_update=False,
        affine_param=False,
        affine_param_batch_decay=0.99,
        affine_param_codebook_decay=0.9,
        sync_update_v=0.,
        return_zeros_for_masked_padding=True,
        route_gradients_to_input=True,
    ):
        super().__init__()
        # ---- options outside the accelerated path fail loudly

        if vq_bridge is not None:
            _unsupported("vq_bridge")
        if in_place_codebook_optimizer is not None:
            _unsupported("in_place_codebook_optimizer")
        if affine_param:
            _unsupported("affine_param")
        if stochastic_sample_codes or straight_through:
            _unsupported("stochastic_sample_codes / gumbel straight_through")
        if commitment_use_cross_entropy_loss or orthogonal_reg_weight > 0 or codebook_diversity_loss_weight > 0:
            _unsupported("cross-entropy / orthogonal / diversity losses (they need the N x K distance matrix)")
        ema_update = (not directional_reparam) if ema_update is None else ema_update  # vqp:854
        learnable_codebook = directional_reparam if learnable_codebook is None else bool(learnable_codebook)  # vqp:855
        rotation_trick = (not directional_reparam and dim > 1) if rotation_trick is None else rotation_trick  # vqp:856
        # combinations the reference rejects (vqp:884, :908, :913)
        if learnable_codebook and ema_update:
            _unsupported("learnable_codebook together with ema_update")
        if learnable_codebook and use_cosine_sim:
            _unsupported("learnable_codebook together with use_cosine_sim")
        if sync_update_v > 0 and not learnable_codebook:
            _unsupported("sync_update_v without learnable_codebook")
        if learnable_codebook and separate_codebook_per_head and heads > 1:
            _unsupported("learnable_codebook with separate_codebook_per_head")
        assert 0 <= sync_update_v <= 1.  # vqp:912
        assert not (rotation_trick and directional_reparam)  # vqp:898
        assert not (directional_reparam and threshold_ema_dead_code == 0), \
            "periodic dead code replacement should be enabled when differential reparam method is turned on"  # vqp:901

        self.dim = dim
        self.heads = heads
        self.separate_codebook_per_head = separate_codebook_per_head
        codebook_dim = dim if codebook_dim is None else codebook_dim
        codebook_input_dim = codebook_dim * heads
        requires_projection = codebook_input_dim != dim
        if requires_projection:  # vqp:867-874
            layers = [nn.Linear(dim, codebook_input_dim)]
            if layernorm_after_project_in:
                layers.append(nn.LayerNorm(codebook_input_dim))
            self.project_in = layers[0] if len(layers) == 1 else nn.Sequential(*layers)
            self.project_out = nn.Linear(codebook_input_dim, dim)
        else:
            self.project_in = nn.Identity()
            self.project_out = nn.Identity()
        self.has_projections = requires_projection

        self.eps = eps
        self.has_commitment_loss = commitment_weight > 0. and not directional_reparam  # vqp:880
        self.commitment_weight = commitment_weight
        self.learnable_codebook = learnable_codebook
        self.rotation_trick = rotation_trick
        self.directional_reparam = directional_reparam
        self.directional_reparam_variance = directional_reparam_variance
        self.sync_update_v = sync_update_v
        self.route_gradients_to_input = route_gradients_to_input

        if sync_codebook is None:  # vqp:925-926
            sync_codebook = _is_distributed()

        self.use_cosine_sim = use_cosine_sim
        self._codebook = Codebook(
            dim=codebook_dim,
            num_codebooks=heads if separate_codebook_per_head else 1,  # vqp:931
            codebook_size=codebook_size,
            decay=decay,
            eps=eps,
            threshold_ema_dead_code=threshold_ema_dead_code,
            kmeans_init=kmeans_init,
            kmeans_iters=kmeans_iters,
            use_ddp=sync_codebook,
            sync_kmeans=sync_kmeans,
            sample_codebook_temp=sample_codebook_temp,
            ema_update=ema_update,
            manual_ema_update=manual_ema_update,
            use_cosine_sim=use_cosine_sim,
            learnable_codebook=learnable_codebook,
        )
        self.codebook_size = codebook_size
        self.accept_image_fmap = accept_image_fmap
        self.accept_3d_fmap = accept_3d_fmap
        self.channel_last = channel_last
        self.register_buffer("zero", torch.tensor(0.), persistent=False)  # vqp:970
        self.return_zeros_for_masked_padding = return_zeros_for_masked_padding
        self.freeze_codebook = freeze_codebook

    # ------------------------------------------------------------------ reference surface
    @property
    def ema_update(self):
        return self._codebook.ema_update

    @property
    def codebook(self):  # vqp:982-989
        if self.separate_codebook_per_head:
            return self._codebook.embed
        return self._codebook.embed[0]

    @codebook.setter
    @torch.no_grad()
    def codebook(self, codes):  # vqp:991-996
        self._codebook.embed.copy_(codes if self.separate_codebook_per_head else codes.unsqueeze(0))

    def get_codes_from_indices(self, indices):  # vqp:998-1018
        if self.separate_codebook_per_head:   # 'b * h' indices -> every head gathers from its own codebook -> 'b * (h d)'
            codes = torch.cat([ops.decode(self._codebook.embed[h], indices[..., h:h + 1].contiguous()) for h in range(self.heads)], dim=-1)
        else:
            codes = self._codebook.decode(indices)
        if not self.channel_last or self.accept_image_fmap or self.accept_3d_fmap:
            codes = codes.movedim(-1, 1)
        return codes

    def get_output_from_indices(self, indices):  # vqp:1020-1022
        return self.project_out(self.get_codes_from_indices(indices))

    def expire_codes_(self, x):
        self._codebook.expire_codes_(self._codebook.transform_input(x))

    def update_indices(self, x, indices, mask=None):  # vqp:1056-1091
        if mask is not None:
            _unsupported("update_indices with a mask")
        if self.heads > 1:
            _unsupported("update_indices with heads > 1")
        x, _ = self._to_rows_layout(x)
        x = self.project_in(x)
        x = self._codebook.transform_input(x)
        self._codebook.update_indices(x, indices.reshape(x.shape[:-1]))

    update_ema_indices = update_indices

    def _loss_scratch(self, device, n=1):
        """The persistent (n,) buffer the kernels write the commitment loss to (stable pointers for the graph cache); callers
        get a copy."""
        buf = getattr(self, "_loss_buf", None)
        if buf is None or buf.device != device or buf.numel() != n:
            buf = torch.zeros((n,), dtype=torch.float32, device=device)
            self._loss_buf = buf
        return buf

    # ------------------------------------------------------------------ layout glue (vqp:1136-1147)
    def _to_rows_layout(self, x):
        restore = None
        if self.accept_image_fmap:
            b, c, h, w = x.shape
            x = x.permute(0, 2, 3, 1).reshape(b, h * w, c)
            restore = ("image", (h, w))
        elif self.accept_3d_fmap:
            b, c, d, h, w = x.shape
            x = x.permute(0, 2, 3, 4, 1).reshape(b, d * h * w, c)
            restore = ("3d", (d, h, w))
        elif not self.channel_last:
            x = x.transpose(1, 2)
            restore = ("transpose", None)
        return x, restore

    # ------------------------------------------------------------------ host-resident batches
    @torch.no_grad()
    def forward_host(self, x_host: torch.Tensor, n_chunks: int = 8, out=None):
        """forward() for a batch that lives in (pinned) HOST memory; results are returned in host memory.

        The batch is streamed through the GPU in `n_chunks` row chunks on three streams — upload of chunk i+1,
        kernels of chunk i and download of chunk i-1 overlap, so the call costs ~max(H2D, D2H) over PCIe instead
        of H2D + kernels + D2H.  Same arithmetic as forward(): every chunk searches the pre-update codebook, the
        chunks' EMA statistics are summed and the codebook is updated once at the end (vqp:586-617).
        `out` = optional (quantize, indices, loss) host tensors to fill (pinned for full overlap).
        The device->host copies are ASYNCHRONOUS on an internal stream that the current stream waits for: synchronise
        the current stream (or the device) before reading the returned host tensors."""
        if self.has_projections or self.accept_image_fmap or self.accept_3d_fmap or not self.channel_last or self.heads > 1:
            _unsupported("forward_host with projections / feature-map layouts / heads > 1")
        cbk = self._codebook
        emb = cbk.embed
        if not emb.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: move the module to a CUDA (H100) device")
        if x_host.is_cuda or x_host.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError("forward_host expects a float32 / bfloat16 CPU tensor (pinned for full overlap)")
        dev = emb.device
        shape = x_host.shape
        D = shape[-1]
        xf = x_host.reshape(-1, D)
        N = xf.shape[0]
        training = self.training
        do_update = cbk.updates(training, self.freeze_codebook)
        want_loss = training and self.has_commitment_loss
        if out is None:
            out = (torch.empty(shape, dtype=x_host.dtype).pin_memory(), torch.empty(shape[:-1], dtype=torch.int64).pin_memory(),
                   torch.empty((), dtype=torch.float32).pin_memory())
        q_host, i_host, l_host = out
        qf, idf = q_host.reshape(-1, D), i_host.reshape(-1)
        bounds = host_chunk_bounds(N, n_chunks)
        n_chunks = len(bounds) - 1
        rows = max(bounds[c + 1] - bounds[c] for c in range(n_chunks))
        key = (N, D, x_host.dtype, tuple(bounds), dev)
        st = getattr(self, "_host_pipe", None)
        if st is None or st["key"] != key:
            # whole-batch device buffers (2 x 134 MB at BASELINE config 2): no upload ever waits for a buffer to be
            # recycled, so all uploads are enqueued up front and PCIe never idles on the host's enqueue pace
            st = dict(key=key, h2d=torch.cuda.Stream(dev), d2h=torch.cuda.Stream(dev),
                      x=torch.empty((N, D), dtype=x_host.dtype, device=dev),
                      q=torch.empty((N, D), dtype=x_host.dtype, device=dev),
                      i=torch.empty((N,), dtype=torch.int64, device=dev),
                      loss=torch.zeros((n_chunks,), dtype=torch.float32, device=dev),
                      stats=torch.empty((ops.stats_floats(cbk.codebook_size, D),), dtype=torch.float32, device=dev),
                      stats_chunk=torch.empty((ops.stats_floats(cbk.codebook_size, D),), dtype=torch.float32, device=dev))
            self._host_pipe = st
        cur = torch.cuda.current_stream(dev)
        up, down = st["h2d"], st["d2h"]
        up.wait_stream(cur)     # the previous call's kernels are done with x
        down.wait_stream(cur)
        ev_up = []
        with torch.cuda.stream(up):
            for c in range(n_chunks):
                r0, r1 = bounds[c], bounds[c + 1]
                st["x"][r0:r1].copy_(xf[r0:r1], non_blocking=True)
                e = torch.cuda.Event(); e.record(up); ev_up.append(e)
        weights = []
        for c in range(n_chunks):
            r0, r1 = bounds[c], bounds[c + 1]
            n = r1 - r0
            weights.append(n / N)
            cur.wait_event(ev_up[c])
            cbk.quantize_rows(st["x"][r0:r1], update=do_update, q_out=st["q"][r0:r1], idx64_out=st["i"][r0:r1],
                              loss_out=st["loss"][c:c + 1] if want_loss else None, loss_weight=self.commitment_weight,
                              stats_out=(st["stats"] if c == 0 else st["stats_chunk"]) if do_update else None,
                              defer_ema=True)
            if do_update and c > 0:
                st["stats"].add_(st["stats_chunk"])
            e = torch.cuda.Event(); e.record(cur)
            with torch.cuda.stream(down):
                down.wait_event(e)
                qf[r0:r1].copy_(st["q"][r0:r1], non_blocking=True)
                idf[r0:r1].copy_(st["i"][r0:r1], non_blocking=True)
        if do_update:   # dead-code expiry samples the whole batch, resident in st["x"] (vqp:641)
            cbk.apply_stats(st["stats"], lambda: cbk.transform_input(st["x"]).float())
        if want_loss:
            w = torch.tensor(weights, dtype=torch.float32, device=dev)
            loss = (st["loss"][:n_chunks] * w).sum()
            if x_host.dtype == torch.bfloat16:
                loss = loss.bfloat16().float()
            l_host.copy_(loss, non_blocking=True)
        else:
            l_host.zero_()
        cur.wait_stream(down)
        return q_host, i_host, l_host

    # ------------------------------------------------------------------ the codebook call of each forward variant
    # Each returns (quantize, embed_ind, commit, glue, learn): the quantized rows and int64 indices in the layout of its input
    # rows, the kernels' commitment loss (None: taken by the glue below), the glue loss's (quantize, target) when that is not
    # (quantize, transform_input(x)), and what _LearnableCodebook needs (idx32, commit_rows) for a learnable codebook.
    # want_q False: the quantized rows are neither written nor returned (None), for callers that keep only the indices.
    def _quantize_shared(self, x, update, ema_update, loss_weight, fused_loss, commit_grad, ema_update_weight, accum_ema_update,
                         want_q=True):
        """One search over all rows; with shared heads every head's sub-vector is a row (vqp:1044-1049)."""
        cbk, shape = self._codebook, x.shape
        flat = x.detach().reshape(-1, shape[-1]).contiguous()
        q = torch.empty_like(flat) if want_q else None
        idx64 = torch.empty((flat.shape[0],), dtype=torch.int64, device=flat.device)
        loss_buf = self._loss_scratch(flat.device) if fused_loss else None
        # a learnable codebook (vqp:710) gets the gradient of `quantize` and, in training, of the commitment loss (vqp:1214-1216)
        learns = cbk.learns()
        commit_rows = []

        def take_commit_rows(stats):   # count_k c_k - sum_{n -> k} x_n, with the codebook the rows were searched in
            # the reference differentiates mse(quantize.type(dtype), x) (vqp:1178, :1327): the code as rounded to x's dtype
            count, sums = cbk._stat_views(stats)
            commit_rows.append(count[0, :, None] * cbk.embed.detach()[0].to(x.dtype).float() - sums[0])

        idx32, _ = cbk.quantize_rows(flat, update=update, q_out=q, idx64_out=idx64, loss_out=loss_buf, loss_weight=loss_weight,
                                     ema_update=ema_update, ema_update_weight=ema_update_weight,
                                     accum_ema_update=accum_ema_update,
                                     on_stats=take_commit_rows if learns and commit_grad else None)
        commit = loss_buf.clone().reshape(()) if fused_loss else None
        # the search's index buffer is reused by the next forward
        learn = (idx32.clone(), commit_rows[0] if commit_rows else None) if learns else None
        return None if q is None else q.reshape(shape), idx64.reshape(shape[:-1]), commit, None, learn

    def _quantize_heads(self, x, update, ema_update, loss_weight, fused_loss, want_q=True):
        """separate_codebook_per_head, x (b, n, h, d) (vqp:1044-1049 'b n (h d) -> h b n d', Codebook(num_codebooks=h)): head i
        searches / updates codebook i of the (h, K, d) buffers — h independent chains on the same kernels, in head order (k-means
        init and dead-code expiry draw from the RNG head by head, like the reference's batched_sample_vectors)."""
        cbk, heads, d = self._codebook, self.heads, x.shape[-1]
        views = [cbk.head(i) for i in range(heads)]
        xs = [x[..., i, :].detach().reshape(-1, d).contiguous() for i in range(heads)]
        if not cbk._initted_host:   # vqp:703: every head's k-means on the first batch, then ONE `initted` flag
            if not bool(cbk.initted):
                for v, xi in zip(views, xs):
                    v._kmeans_init(v.transform_input(xi).float())
                cbk.initted.data.copy_(torch.tensor(True))
            cbk._initted_host = True
        for v in views:
            v._initted_host = True
        loss_buf = self._loss_scratch(x.device, heads) if fused_loss else None
        embed_ind = torch.empty(x.shape[:-1], dtype=torch.int64, device=x.device)   # 'h b n -> b n h' (vqp:1266-1268)
        qs = []
        for i, (v, xi) in enumerate(zip(views, xs)):
            q = torch.empty_like(xi) if want_q else None
            v.quantize_rows(xi, update=update, q_out=q, idx64_out=embed_ind[..., i], idx_stride=heads,
                            loss_out=loss_buf[i:i + 1] if fused_loss else None, loss_weight=loss_weight, ema_update=ema_update)
            if want_q:
                qs.append(q.reshape(x.shape[:-2] + (d,)))
        # one mse over all heads (vqp:1327) == the mean of the heads' (equal-sized) means
        commit = loss_buf.mean() if fused_loss else None
        return torch.stack(qs, dim=2) if want_q else None, embed_ind, commit, None, None

    def _quantize_masked(self, x, mask, update, ema_update, loss_weight, want_loss):
        """mask (B, N) bool (vqp:599-600, :1317-1325, :1378-1396).  Masked positions take no part in the statistics or the loss
        (the reference zeroes their one-hot rows, vqp:599-600, and averages the loss over the unmasked elements against the
        ORIGINAL input, vqp:1317-1325) and come back as zeros / index -1.  Euclidean codebooks: the search kernel takes the mask
        (row_mask of vqb_vq_forward).  Cosine codebooks, pending k-means init, dead-code expiry: the kernels run on the
        compacted unmasked rows.

        When x requires grad, the rows come back with the estimator of vqp:1225-1233 on the live rows (the padding rows pass
        no gradient, or the upstream gradient when they return the input) and the commitment loss differentiable w.r.t. x;
        every forward value stays that of the call without gradients.  The in-kernel path takes _MaskedEstimator (no host
        sync); the compacted path gathers and scatters the rows under autograd."""
        cbk = self._codebook
        B, N, D = x.shape
        pad_zeros = self.return_zeros_for_masked_padding
        grad = x.requires_grad and torch.is_grad_enabled()
        x_rows = x.reshape(-1, D).contiguous()
        flat = x_rows.detach()
        estimator = ops.ESTIMATOR_NONE
        if self.training and self.route_gradients_to_input:
            estimator = ops.ESTIMATOR_ROTATE if self.rotation_trick else ops.ESTIMATOR_STE
        if grad:   # padding rows are written by _MaskedEstimator / the scatter below
            quantize = torch.empty_like(flat)
        else:
            quantize = torch.zeros_like(flat) if pad_zeros else flat.clone()
        embed_ind = torch.full((B * N,), -1, dtype=torch.int64, device=x.device)
        loss_buf = commit = glue = None
        if not self.use_cosine_sim and cbk._initted_host and not (update and cbk.has_dead_code_replacement):
            # in-kernel mask: every row is searched (like the reference), the merge step of the search kernel drops the padding
            # rows — index -1, outputs left as pre-filled here, no loss term, no statistics — and the loss is divided by the
            # unmasked element count on the device: no host sync, no compaction pass.  (Cosine: the masked loss is taken
            # against the UN-normalised input, vqp:1319; k-means init / expiry sample from x[mask]: those take the path below.)
            row_mask = mask.reshape(-1).contiguous().view(torch.uint8)
            n_live = row_mask.sum(dtype=torch.int64).reshape(1)
            loss_buf = self._loss_scratch(x.device) if want_loss else None
            cbk.quantize_rows(flat, update=update, q_out=quantize, idx64_out=embed_ind, loss_out=loss_buf, loss_weight=loss_weight,
                              ema_update=ema_update, row_mask=row_mask, n_live=n_live)
            if grad:
                loss = loss_buf.clone().reshape(()) if loss_buf is not None else None
                quantize, commit = _MaskedEstimator.apply(x_rows, quantize, loss, row_mask, n_live, estimator, pad_zeros,
                                                          loss_weight)
                loss_buf = None
                if loss is None:
                    commit = None
        else:
            rows = mask.reshape(-1).nonzero(as_tuple=True)[0]  # host sync (the reference's masked path syncs as well)
            if grad:   # the padding rows: no gradient, or the input's own (vqp:1378-1389)
                base = torch.zeros_like(flat) if pad_zeros else x_rows
            if rows.numel() > 0:
                x_live = x_rows[rows] if grad else None
                xc = flat[rows].contiguous()
                qc = torch.empty_like(xc)
                ic = torch.empty((xc.shape[0],), dtype=torch.int64, device=x.device)
                # euclid: the original input IS what the codebook saw; cosine: the glue takes the un-normalised input (vqp:1319)
                loss_buf = self._loss_scratch(x.device) if want_loss and not self.use_cosine_sim else None
                cbk.quantize_rows(xc, update=update, q_out=qc, idx64_out=ic, loss_out=loss_buf, loss_weight=loss_weight,
                                  ema_update=ema_update)
                embed_ind[rows] = ic
                glue = (qc, x_live if grad else xc)
                if grad:
                    live = qc
                    if estimator != ops.ESTIMATOR_NONE:
                        x_t = cbk.transform_input(x_live)
                        live = _with_grad_of(qc, rotate_to(x_t, qc) if estimator == ops.ESTIMATOR_ROTATE
                                             else straight_through(x_t, qc))
                    quantize = base.index_put((rows,), live)
                    if loss_buf is not None:   # the kernels' loss with the gradient of the same mse taken by autograd
                        commit = _with_grad_of(loss_buf.clone().reshape(()), loss_weight * F.mse_loss(qc, x_live))
                        loss_buf = None
                else:
                    quantize[rows] = qc
            else:   # no unmasked row: no loss term.  With gradients both outputs stay in the graph and pass x a zero gradient,
                # like the in-kernel path (the sum over no rows is an exact zero)
                none = x_rows[rows] if grad else None
                if grad:
                    quantize = base.index_put((rows,), none)
                if want_loss:
                    commit = none.float().sum() if grad else torch.zeros((), dtype=torch.float32, device=x.device)
        if loss_buf is not None:
            commit = loss_buf.clone().reshape(())
        return quantize.reshape(B, N, D), embed_ind.reshape(B, N), commit, glue, None

    def _split_heads(self, x):
        """(b, n, h d) rows after project_in as the codebook calls take them (vqp:1044-1049); returns (rows, separate)."""
        heads, batch, n = self.heads, x.shape[0], x.shape[1]
        separate = heads > 1 and self.separate_codebook_per_head
        if separate:     # 'b n (h d) -> b n h d': head i is searched in codebook i
            x = x.reshape(batch, n, heads, -1)
        elif heads > 1:  # 'b n (h d) -> 1 (b h) n d' — every head's sub-vector is a row for the ONE codebook
            x = x.reshape(batch, n, heads, -1).transpose(1, 2).reshape(batch * heads, n, -1)
        return x, separate

    @torch.no_grad()
    def eval_indices(self, x):
        """The indices an eval-mode forward(x) returns for channel-last x (b, n, dim) without a mask, computed without
        writing the quantized rows or running project_out, and with no loss: project_in, the head split and one search per
        codebook (k-means init included, vqp:703).  For callers that keep only the codes (RandomProjectionQuantizer)."""
        if x.ndim != 3:
            raise TypeError(f"eval_indices expects (batch, seq, dim) rows, got shape {tuple(x.shape)}")
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        batch, n = x.shape[0], x.shape[1]
        x, separate = self._split_heads(self.project_in(x))
        if x.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"vqb200 supports float32 and bfloat16 inputs, got {x.dtype}")
        cbk = self._codebook
        if separate:
            _, embed_ind, _, _, _ = self._quantize_heads(x, False, cbk.ema_update, 1., False, want_q=False)
        else:
            _, embed_ind, _, _, _ = self._quantize_shared(x, False, cbk.ema_update, 1., False, False, None, False, want_q=False)
            if self.heads > 1:   # '1 (b h) n -> b n h'
                embed_ind = embed_ind.reshape(batch, self.heads, n).transpose(1, 2)
        return embed_ind

    def forward(self, x, indices=None, mask=None, lens=None, topk=None, sample_codebook_temp=None, freeze_codebook=None,
                return_loss_breakdown=False, codebook_transform_fn=None, ema_update_weight=None, accum_ema_update=False,
                ema_update=None):
        """vqp:1093-1403 as one pipeline: the input as rows (layout, project_in, heads), the codebook call of the variant (all
        rows, one search per separate head, or a masked batch), then one tail: commitment loss, codebook gradient, gradient
        estimator and the rows back in the input's layout."""
        if indices is not None:
            _unsupported("forward(indices=...) cross-entropy loss")
        if mask is not None and lens is not None:
            raise AssertionError("pass either mask or lens")  # vqp:1116
        if lens is not None:  # vqp:1118-1119, :99-101
            mask = torch.arange(x.shape[1], device=lens.device) < lens[:, None]
        if mask is not None:
            if self.learnable_codebook:
                _unsupported("mask / lens with a learnable codebook")
            if self.directional_reparam and x.requires_grad and torch.is_grad_enabled():
                # the masked estimators are the rotation trick and straight-through; DiVeQ's is not among them
                _unsupported("mask / lens with directional_reparam on inputs that require grad")
            if self.has_projections or self.accept_image_fmap or self.accept_3d_fmap or not self.channel_last or self.heads > 1:
                _unsupported("mask / lens together with projections, feature-map layouts or heads > 1")
        elif topk is not None or codebook_transform_fn is not None:
            _unsupported("topk / codebook_transform_fn")
        if not x.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: inputs must live on a CUDA (H100, sm_90) device")
        if mask is not None:
            assert x.ndim == 3 and mask.shape == x.shape[:2]

        freeze_codebook = self.freeze_codebook if freeze_codebook is None else freeze_codebook
        cbk = self._codebook
        ema_update = cbk.ema_update if ema_update is None else ema_update
        training = self.training

        # ---- rows in (vqp:1136-1151)
        only_one = x.ndim == 2
        if only_one:
            x = x.unsqueeze(1)
        x, restore = self._to_rows_layout(x)
        x = self.project_in(x)  # vqp:1151
        heads, batch, n = self.heads, x.shape[0], x.shape[1]
        x, separate = self._split_heads(x)
        # decided AFTER project_in: with a projection the commitment loss must stay differentiable w.r.t. its weights
        # even when the raw input carries no grad (vqp:1151, :1327)
        input_requires_grad = x.requires_grad and torch.is_grad_enabled()
        dtype = x.dtype
        if dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"vqb200 supports float32 and bfloat16 inputs, got {dtype}")

        # ---- the codebook call
        want_loss = training and self.has_commitment_loss
        fused_loss = want_loss and not input_requires_grad
        # the kernels return weight * mse already rounded like F.mse_loss in x.dtype (vqp:1327-1329); LossBreakdown.commitment
        # is the UNweighted mse: ask them for weight 1 then
        # (a masked call always takes the kernels' loss, with or without gradients)
        split_weight = (fused_loss or (want_loss and mask is not None)) and return_loss_breakdown and self.commitment_weight != 1.
        update = cbk.updates(training, freeze_codebook, ema_update)
        loss_weight = 1. if split_weight else self.commitment_weight
        if mask is not None:
            quantize, embed_ind, commit, glue, learn = self._quantize_masked(x, mask, update, ema_update, loss_weight, want_loss)
        elif separate:
            if accum_ema_update or ema_update_weight is not None:
                _unsupported("ema_update_weight / accum_ema_update with separate_codebook_per_head")
            quantize, embed_ind, commit, glue, learn = self._quantize_heads(x, update, ema_update, loss_weight, fused_loss)
        else:
            quantize, embed_ind, commit, glue, learn = self._quantize_shared(
                x, update, ema_update, loss_weight, fused_loss, want_loss and not freeze_codebook, ema_update_weight,
                accum_ema_update)

        # ---- commitment loss (vqp:1282, :1317-1329)
        fused = commit is not None
        if fused:
            weighted = commit
            if split_weight:  # commit * weight in the input dtype, promoted by the fp32 accumulator (vqp:1329, :1282)
                weighted = (commit.to(dtype) * self.commitment_weight).float()
            # vqp:1282: `loss` is a fresh fp32 scalar that requires grad in training mode
            loss = weighted.requires_grad_(torch.is_grad_enabled())
        else:
            loss = torch.tensor(0., device=x.device, requires_grad=training and torch.is_grad_enabled())  # vqp:1282
            if want_loss:   # differentiable w.r.t. the input: PyTorch glue on the kernel's outputs
                q_rows, target = glue or (quantize, cbk.transform_input(x))
                commit = F.mse_loss(q_rows.detach(), target)
        if learn is not None:
            idx32, commit_rows = learn
            if commit_rows is None:
                quantize, _ = _LearnableCodebook.apply(cbk.embed, quantize, None, idx32, None, 0.)
            elif fused:   # `loss` is already weight * mse
                quantize, loss = _LearnableCodebook.apply(cbk.embed, quantize, loss, idx32, commit_rows,
                                                          2. * self.commitment_weight / x.numel())
            else:
                quantize, commit = _LearnableCodebook.apply(cbk.embed, quantize, commit, idx32, commit_rows, 2. / x.numel())
        if training:
            if want_loss and not fused:
                loss = loss + commit * self.commitment_weight
            # ---- gradient estimator (vqp:1225-1237); a masked call ran it on its live rows already
            if input_requires_grad and self.route_gradients_to_input and mask is None:
                x_t = cbk.transform_input(x)
                if self.rotation_trick:
                    quantize = rotate_to(x_t, quantize)
                elif self.directional_reparam:
                    quantize = directional_reparam(x_t, quantize, self.directional_reparam_variance)
                else:
                    quantize = straight_through(x_t, quantize)
            if self.sync_update_v > 0.:
                quantize = quantize + self.sync_update_v * (quantize - quantize.detach())

        # ---- rows out (vqp:1354-1373, :1265-1275)
        if separate:     # 'b n h d -> b n (h d)'
            quantize = quantize.reshape(batch, n, -1)
        elif heads > 1:  # '1 (b h) n d -> b n (h d)', '1 (b h) n -> b n h'
            quantize = quantize.reshape(batch, heads, n, -1).transpose(1, 2).reshape(batch, n, -1)
            embed_ind = embed_ind.reshape(batch, heads, n).transpose(1, 2)
        quantize = self.project_out(quantize)  # vqp:1360
        if restore is not None:
            kind, dims = restore
            if kind == "transpose":
                quantize = quantize.transpose(1, 2)
            else:
                quantize = quantize.reshape(batch, *dims, quantize.shape[-1]).movedim(-1, 1)
                embed_ind = embed_ind.reshape(batch, *dims, *embed_ind.shape[2:])
        if only_one:
            quantize = quantize.squeeze(1)
            embed_ind = embed_ind.squeeze(1)

        if not return_loss_breakdown:
            return quantize, embed_ind, loss
        return quantize, embed_ind, loss, LossBreakdown(self.zero if commit is None else commit, self.zero, self.zero, self.zero)
