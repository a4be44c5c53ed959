"""Functional layer over the C ABI: torch tensors in, torch tensors out, everything enqueued on the
current CUDA stream.  Mirrors the arithmetic steps of `Codebook.forward`
(reference vector_quantize_pytorch.py:674-791); the nn.Modules in this package are glue around these.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import torch

from . import _C
from ._C import lib, check

# A row is certified by the tensor-core passes when its best score leads all others by more than the band
#   2 * (||x|| * cres + xaux * caux + margin * ||x|| * max||c|| [+ 2^-21 max||c||^2]) + (tag slack, sqrt-collapse width):
# Cauchy-Schwarz on the EXACT norms of what the bf16 hi / lo passes leave out (csrc/code_operands.cuh, vq_assign.cu):
# cres = max_k ||c - hi - lo||, and for fp32 inputs xaux = ||x_lo|| with caux = 2^-8 max||c|| + max||c_lo|| — plus `margin` for
# the fp32 accumulation in the tensor core alone (2^-18; its room is measured on the GPU by the test below).
# tests/test_parity_gpu.py::test_score_error_inside_margin asserts the bound on randn, heavy-tailed, tiny, unit-norm and
# default-init data.  See DESIGN.md 4.1.
DEFAULT_MARGIN = 2.0 ** -18

_DT = {torch.float32: _C.DTYPE_F32, torch.bfloat16: _C.DTYPE_BF16}

# bench.py instrumentation: when PROFILE_EVENTS is a list, `search` brackets the search kernel with CUDA
# events on the launching stream; LAUNCHES counts the kernels this library enqueues.
PROFILE_EVENTS = None
LAUNCHES = 0


def _count(n):
    global LAUNCHES
    LAUNCHES += n


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise TypeError(f"vqb200 supports float32 and bfloat16 inputs, got {t.dtype}") from None


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("vqb200 has no CPU path: tensors must live on a CUDA (H100, sm_90) device")


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms(dev) -> int:
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _aligned(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t.clone() if t.data_ptr() % 16 else t   # a contiguous view at an offset (the kernels move rows in 16-byte vectors)


def _queried(n: int, name: str) -> int:
    """A count returned by a query entry point, which returns a negative error code instead when it fails."""
    check(min(n, 0), name)
    return n


def _index_strides(idx: torch.Tensor) -> tuple:
    """(row, group, stage) element strides of an (N, G, Q) view of an index tensor (a size-1 axis has stride 0)."""
    return tuple(0 if n == 1 else s for n, s in zip(idx.shape, idx.stride()))


_fsq_strides = _index_strides   # the name FSQ's kernel tests import


def _check_index_dtype(indices: torch.Tensor, family: str):
    if indices.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"{family} indices must be int32 or int64, got {indices.dtype}")


# ---- what the scalar quantizer modules (FSQ, LFQ, FSP, BinaryMapper) share ----

FLOAT_DTYPES = (torch.float32, torch.bfloat16)


def float_input(t: torch.Tensor, family: str, what: str = "inputs", work_dtype: torch.dtype | None = None) -> torch.Tensor:
    """A module's input to the row kernels: fp32 or bf16 (TypeError; so must `work_dtype` be, the dtype of the module's chain
    when it differs from the input's) on a CUDA device (RuntimeError), returned contiguous and 16-byte aligned."""
    if t.dtype not in FLOAT_DTYPES or (work_dtype is not None and work_dtype not in FLOAT_DTYPES):
        chain = f" (quantizer chain in {work_dtype})" if work_dtype is not None else ""
        raise TypeError(f"vqb200 {family} supports float32 and bfloat16 {what}, got {t.dtype}{chain}")
    if not t.is_cuda:
        raise RuntimeError(f"vqb200 has no CPU path: {what} must live on a CUDA (H100, sm_90) device")
    return _aligned(t)


class DeviceTables:
    """Per-device copies of a module's kernel tables, made on first use by `make()` (the tables follow from non-persistent
    buffers fixed at construction; `key` names what may still change them, such as the buffers' dtype after `.to(dtype)`)."""

    def __init__(self, make):
        self.make = make
        self.cache = {}

    def get(self, device, key=()):
        k = (device, key)
        t = self.cache.get(k)
        if t is None:
            t = self.cache[k] = tuple(x.to(device) if x is not None else None for x in self.make())
        return t


def padded_codes(K: int) -> int:
    return lib.vqb_padded_codes(K)


@dataclass
class CodebookOperands:
    """Tensor-core view of one codebook (see vqb_codebook_prepare in include/vqb200.h)."""
    planes: torch.Tensor  # 2-byte (2, Kpad, D): bf16 hi, bf16 lo (bit patterns) (csrc/code_operands.cuh)
    bext: torch.Tensor  # bf16 (Kpad, 16): -bias as three bf16 terms (the operand of the "bias MMA")
    bias: torch.Tensor  # f32 (Kpad,)
    cnorm2: torch.Tensor  # f32 (K,)
    cmax: torch.Tensor  # f32 (3,): max||c||, max||c - bf16 hi - bf16 lo||, max||bf16 lo||
    scratch: torch.Tensor  # f32 (2,)
    K: int
    D: int
    cosine: bool

    @staticmethod
    def allocate(K: int, D: int, cosine: bool, device) -> "CodebookOperands":
        Kpad = padded_codes(K)
        return CodebookOperands(
            planes=torch.empty((2, Kpad, D), dtype=torch.float16, device=device),
            bext=torch.empty((Kpad, 16), dtype=torch.bfloat16, device=device),
            bias=torch.empty((Kpad,), dtype=torch.float32, device=device),
            cnorm2=torch.empty((K,), dtype=torch.float32, device=device),
            cmax=torch.zeros((3,), dtype=torch.float32, device=device),
            scratch=torch.zeros((2,), dtype=torch.float32, device=device),
            K=K, D=D, cosine=cosine)


def prepare_codebook(embed: torch.Tensor, cosine: bool, out: CodebookOperands | None = None) -> CodebookOperands:
    """embed (K, D) fp32 contiguous -> operands for `search`."""
    _require_cuda(embed)
    assert embed.dtype == torch.float32 and embed.dim() == 2 and embed.is_contiguous()
    K, D = embed.shape
    ops = out if out is not None else CodebookOperands.allocate(K, D, cosine, embed.device)
    with torch.cuda.device(embed.device):
        check(lib.vqb_codebook_prepare(_p(embed), K, D, int(cosine), _p(ops.planes), _p(ops.bext), _p(ops.bias), _p(ops.cnorm2),
                                       _p(ops.cmax), _stream()), "vqb_codebook_prepare")
    _count(1)
    return ops


@dataclass
class SearchResult:
    idx: torch.Tensor  # int32 (N,)
    x_eff: torch.Tensor  # (N, D) input as the codebook sees it (l2-normalised for cosine), in x.dtype
    flag_count: torch.Tensor  # int32 (1,) rows re-scored exactly
    flagged: torch.Tensor  # int32 (N, 8): (row, count, cand0, cand1, cand2, pad x 3) — vqb_flag_entry
    best: torch.Tensor | None = None
    rescan_count: torch.Tensor | None = None  # int32 (1,) rows re-scanned whole (entries at the back of `flagged`)


def search(x: torch.Tensor, ops: CodebookOperands, embed: torch.Tensor, *, margin: float | None = None, n_passes: int = 0,
           debug_best: bool = False, fix: bool = True, normalise: bool = True, fused: dict | None = None) -> SearchResult:
    """Nearest code of every row of x (N, D).  Replaces cdist/einsum + argmax (vqp:58-62, :741-747, :130-145).

    fused: optional dict(q_out=, idx64_out=, idx_stride=, loss_sum=, resid_out=, planes_out=) of output tensors — the
    gather / commitment-loss / residual tail (see `gather`) then runs INSIDE the search kernel (store warps) and
    the re-score kernels, and no separate gather launch is needed.  planes_out (fp32 rows with resid_out): 2-byte
    [2][N][D], the bf16 hi / lo split of the residual (the next ResidualVQ stage's A operand)."""
    _require_cuda(x, embed)
    assert x.dim() == 2 and x.is_contiguous()
    N, D = x.shape
    assert D == ops.D
    dt = _dtype_code(x)
    cosine = ops.cosine
    l2 = cosine and normalise  # normalise=False: the caller already applied l2norm (Codebook.forward contract)
    dev = x.device
    margin = DEFAULT_MARGIN if margin is None else margin
    with torch.cuda.device(dev):
        st = _stream()
        if x.dtype == torch.bfloat16:
            if l2:  # l2norm in bf16 (vqp:1159 -> :376); the normalised bf16 rows are the A operand
                x_eff = torch.empty_like(x)
                check(lib.vqb_input_prepare(_p(x), dt, N, D, 1, _p(x_eff), None, 0, st), "vqb_input_prepare")
                _count(1)
            else:
                x_eff = x
            a_planes, n_a = x_eff, 1
        else:
            a_planes = torch.empty((2, N, D), dtype=torch.bfloat16, device=dev)   # bf16 hi / lo split of the fp32 input
            x_eff = torch.empty_like(x) if l2 else x
            check(lib.vqb_input_prepare(_p(x), dt, N, D, int(l2), _p(x_eff) if l2 else None, _p(a_planes), 2, st),
                  "vqb_input_prepare")
            _count(1)
            n_a = 2
        idx = torch.empty((N,), dtype=torch.int32, device=dev)
        flagged = torch.empty((N, 8), dtype=torch.int32, device=dev)
        count = torch.zeros((2,), dtype=torch.int32, device=dev)   # [rows with 2 / 3 candidates, rows re-scanned whole]
        best = torch.empty((N,), dtype=torch.float32, device=dev) if debug_best else None
        fo = None
        if fused is not None:
            fo = _C.FusedOutputs(x_eff=_p(x_eff), embed=_p(embed), q_out=_p(fused.get("q_out")),
                                 idx64_out=_p(fused.get("idx64_out")), idx_stride=int(fused.get("idx_stride", 1)),
                                 loss_sum=_p(fused.get("loss_sum")), x_raw=_p(x) if x_eff is not x else None,
                                 resid_out=_p(fused.get("resid_out")), stats_cnt=None, stats_sum=None, dtype=dt,
                                 planes_out=_p(fused.get("planes_out")),
                                 qsum=_p(fused.get("qsum")))   # reserved: vqb_assign refuses a running sum, not ignores it
        fo_ref = ctypes.byref(fo) if fo is not None else None
        prof = PROFILE_EVENTS
        if prof is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        check(lib.vqb_assign_ex(_p(a_planes), n_a, N, D, _p(ops.planes), _p(ops.bext), _p(ops.cmax), ops.K, float(margin),
                                int(n_passes), _p(idx), _p(flagged), _p(count), _p(best), fo_ref, int(cosine),
                                _p(ops.cnorm2), st), "vqb_assign")
        if prof is not None:
            ev1.record()
            prof.append((ev0, ev1))
        _count(1 + 3 * int(fix))
        if fix:
            check(lib.vqb_fix_flagged(_p(x_eff), dt, N, D, _p(embed), _p(ops.cnorm2), ops.K, int(cosine), _p(flagged),
                                      _p(count), _p(idx), fo_ref, st), "vqb_fix_flagged")
    return SearchResult(idx, x_eff, count[:1], flagged, best, count[1:])


class Scratch:
    """The two device scratch buffers of `vq_forward_args` (the int32 index row and the workspace) for ONE owner: a `Codebook`
    for its eager calls, an `RvqProgram` lane for the stage ops it freezes.  Reused from call to call (calls of one owner are
    ordered on its stream), so the pointers stay stable and the CUDA-graph cache of vqb_vq_forward keeps replaying; grown when a
    call needs more bytes or another device, so a batch whose row count changes does not pin a buffer per count.  A grown
    buffer is dropped, so whoever froze a pointer into the old one must hold it itself.  Never copied or pickled with its
    owner: a copy starts empty."""

    def __init__(self):
        self.idx = None
        self.ws = None

    def __deepcopy__(self, memo):
        return Scratch()

    def __reduce__(self):
        return (Scratch, ())

    @staticmethod
    def _fit(buf, nbytes, device):
        if buf is None or buf.numel() < nbytes or buf.device != device:
            buf = torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=device)
        return buf

    def take(self, idx_bytes: int, ws_bytes: int, device) -> tuple[torch.Tensor, torch.Tensor]:
        """(index buffer, workspace) of at least these sizes (uint8) on `device`."""
        self.idx = self._fit(self.idx, idx_bytes, device)
        self.ws = self._fit(self.ws, ws_bytes, device)
        return self.idx, self.ws


def vq_forward_args(x: torch.Tensor, ops: CodebookOperands, state: tuple, *, update: int, do_normalise: bool, decay: float,
                    eps: float, q_out=None, idx64_out=None, idx_stride: int = 1, loss_out=None, loss_weight: float = 1.0,
                    resid_out=None, stats=None, margin: float | None = None, already_normalised: bool = False,
                    scratch: Scratch | None = None, peer=None, peer_ptrs=None, peer_slice_offset: int = 0,
                    a_planes_in=None, planes_out=None, row_mask=None, n_live=None):
    """The argument block of one vqb_vq_forward call (also one VQB_RVQ_STAGE op of vqb_rvq_forward).
    scratch: the caller's `Scratch` (None: a fresh one, freed after the call — for one-off calls).
    row_mask (N,) uint8 / n_live (1,) int64 on the device: a masked batch (vqp:1116-1119) — padding rows (0) keep the values
    q_out / idx64_out were pre-filled with and stay out of the loss and the statistics (include/vqb200.h).
    Returns (args, idx32, stats, n_launches)."""
    if row_mask is not None:
        assert row_mask.dtype == torch.uint8 and row_mask.is_contiguous() and row_mask.numel() == x.shape[0] and row_mask.is_cuda
        assert n_live is None or (n_live.dtype == torch.int64 and n_live.numel() == 1 and n_live.is_cuda)
    _require_cuda(x, state[2])
    assert x.dim() == 2 and x.is_contiguous()
    N, D = x.shape
    K = ops.K
    dt = _dtype_code(x)
    dev = x.device
    cs, ea, emb = state
    nbytes = lib.vqb_vq_forward_workspace(N, D, K, dt, int(ops.cosine), int(update))
    idx_buf, ws = (scratch or Scratch()).take(4 * N, nbytes, dev)
    idx32 = idx_buf[:4 * N].view(torch.int32)
    if update and stats is None:
        stats = torch.empty((stats_floats(K, D),), dtype=torch.float32, device=dev)
    a = _C.VQForwardArgs(
        x=_p(x), dtype=dt, metric=int(ops.cosine), N=N, D=D, K=K, already_normalised=int(already_normalised),
        cluster_size=_p(cs), embed_avg=_p(ea), embed=_p(emb), planes=_p(ops.planes), bext=_p(ops.bext), bias=_p(ops.bias),
        cnorm2=_p(ops.cnorm2), cmax=_p(ops.cmax), scratch=_p(ops.scratch), q_out=_p(q_out), idx64_out=_p(idx64_out),
        idx_stride=int(idx_stride), loss_out=_p(loss_out), loss_weight=float(loss_weight), resid_out=_p(resid_out),
        idx32=_p(idx32), update=int(update), stats_mode=1, do_normalise=int(do_normalise), decay=float(decay),
        eps=float(eps), stats=_p(stats), margin_rel=float(DEFAULT_MARGIN if margin is None else margin),
        workspace=_p(ws), workspace_bytes=nbytes, ev_search_begin=None, ev_search_end=None,
        a_planes_in=_p(a_planes_in), planes_out=_p(planes_out), row_mask=_p(row_mask), n_live=_p(n_live))
    if update == 3:  # multi-GPU: statistics -> peer barrier -> EMA kernels summing every rank's statistics (vq_peer.cu)
        a.peer_stats = ctypes.cast(peer_ptrs, ctypes.c_void_p)
        a.peer_flags = ctypes.cast(peer.flag_ptrs, ctypes.c_void_p)
        a.peer_epoch = peer.epoch.data_ptr()
        a.peer_rank, a.peer_world, a.peer_slice_offset = peer.rank, peer.world, int(peer_slice_offset)
    n_launch = (4 + (1 if dt == _C.DTYPE_F32 or ops.cosine else 0) + (1 if loss_out is not None else 0) + (5 if update else 0)
                + (2 if update == 2 else 0) + (3 if update == 3 else 0))
    return a, idx32, stats, n_launch


def vq_forward(x: torch.Tensor, ops: CodebookOperands, state: tuple, **kw) -> tuple[torch.Tensor, torch.Tensor | None]:
    """ONE C call for the arithmetic of VectorQuantize.forward / one ResidualVQ stage (vqb_vq_forward).

    state = (cluster_size (K,), embed_avg (K, D), embed (K, D)).  update: 0 none, 1 statistics only (returned
    packed; the caller all-reduces and calls `ema_apply`), 2 statistics + EMA apply.  Returns (idx32, stats)."""
    a, idx32, stats, n_launch = vq_forward_args(x, ops, state, **kw)
    with torch.cuda.device(x.device):
        prof = PROFILE_EVENTS
        if prof is not None:  # bench instrumentation: CUDA events around the search kernel, recorded from C
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(); ev1.record()  # materialise the handles
            a.ev_search_begin, a.ev_search_end = ev0.cuda_event, ev1.cuda_event
            prof.append((ev0, ev1))
        check(lib.vqb_vq_forward(ctypes.byref(a), _stream()), "vqb_vq_forward")
    _count(n_launch)
    return idx32, stats


class RvqProgram:
    """The op list of one vqb_rvq_forward call: a whole ResidualVQ / GroupedResidualVQ forward — stages, running sum, deferred
    EMA updates — enqueued by ONE FFI call and replayed from one CUDA graph.  Ops of one lane run in order; lanes (the groups
    of GroupedResidualVQ) run on parallel streams."""
    MAX_OPS = 62

    def __init__(self, device):
        self.device = device
        self.ops = []
        self.keep = []       # tensors the ops point into
        # the stage ops' scratch: one per lane (the ops of a lane run in order, every stage joins its side stream before the
        # next op; lanes run in parallel), and every buffer an op was handed, even one a later stage of its lane outgrew
        self.scratch = {}
        self.scratch_bufs = []
        self.launches = 0

    def stage(self, lane, x, cb_ops, state, **kw):
        scratch = self.scratch.setdefault(lane, Scratch())
        a, idx32, stats, n = vq_forward_args(x, cb_ops, state, scratch=scratch, **kw)
        op = _C.RvqOp(kind=_C.RVQ_STAGE, lane=lane)
        op.stage = a
        self.ops.append(op)
        self.keep.append((x, cb_ops, state, kw, idx32, stats))
        self.scratch_bufs += [scratch.idx, scratch.ws]
        self.launches += n
        return idx32, stats

    def ema(self, lane, cluster_size, embed_avg, embed, stats, cb_ops, *, decay, eps, do_lerp, do_normalise, n_lerp=1, slice_stride=0):
        K, D = embed.shape
        op = _C.RvqOp(kind=_C.RVQ_EMA, lane=lane)
        op.ema = _C.RvqEmaArgs(cluster_size=_p(cluster_size), embed_avg=_p(embed_avg), embed=_p(embed), stats=_p(stats), K=K, D=D,
                               decay=float(decay), eps=float(eps), metric=int(cb_ops.cosine), do_lerp=int(do_lerp),
                               do_normalise=int(do_normalise), planes=_p(cb_ops.planes), bext=_p(cb_ops.bext), bias=_p(cb_ops.bias),
                               cnorm2=_p(cb_ops.cnorm2), cmax=_p(cb_ops.cmax), scratch=_p(cb_ops.scratch),
                               n_lerp=int(n_lerp), slice_stride=int(slice_stride))
        self.ops.append(op)
        self.keep.append((cluster_size, embed_avg, embed, stats, cb_ops))
        self.launches += 2

    def barrier(self, lane, peer):
        op = _C.RvqOp(kind=_C.RVQ_BARRIER, lane=lane)
        op.bar = _C.RvqBarArgs(flags=ctypes.cast(peer.flag_ptrs, ctypes.c_void_p), epoch=peer.epoch.data_ptr(), rank=peer.rank,
                               world=peer.world)
        self.ops.append(op)
        self.keep.append(peer)
        self.launches += 1

    def ema_peers(self, lane, cluster_size, embed_avg, embed, peer, peer_ptrs, slice_offset, cb_ops, *, decay, eps, do_normalise,
                  n_lerp=1, slice_stride=0):
        K, D = embed.shape
        op = _C.RvqOp(kind=_C.RVQ_EMA_PEERS, lane=lane)
        op.emap = _C.RvqEmaPeersArgs(cluster_size=_p(cluster_size), embed_avg=_p(embed_avg), embed=_p(embed),
                                     peer_stats=ctypes.cast(peer_ptrs, ctypes.c_void_p), slice_offset=int(slice_offset),
                                     world=peer.world, K=K, D=D, decay=float(decay), eps=float(eps), metric=int(cb_ops.cosine),
                                     do_normalise=int(do_normalise), planes=_p(cb_ops.planes), bext=_p(cb_ops.bext),
                                     bias=_p(cb_ops.bias), cnorm2=_p(cb_ops.cnorm2), cmax=_p(cb_ops.cmax), scratch=_p(cb_ops.scratch),
                                     n_lerp=int(n_lerp), slice_stride=int(slice_stride))
        self.ops.append(op)
        self.keep.append((cluster_size, embed_avg, embed, peer, peer_ptrs, cb_ops))
        self.launches += 2

    def accumulate(self, lane, embeds, indices, out):
        N, Q = indices.shape
        if embeds.dim() == 2:
            K, D = embeds.shape
            stride = 0
        else:
            _, K, D = embeds.shape
            stride = K * D
        op = _C.RvqOp(kind=_C.RVQ_ACCUMULATE, lane=lane)
        op.acc = _C.RvqAccArgs(embeds=_p(embeds), embed_stride=stride, Q=Q, K=K, D=D, idx=_p(indices), N=N, out=_p(out),
                               dtype=_DT[out.dtype])
        self.ops.append(op)
        self.keep.append((embeds, indices, out))
        self.launches += 1

    def simvq_tail(self, lane, r, codes, idx32, *, rotation, r_next, qsum, first, idx64_out, idx_stride, loss_sum, loss_out,
                   input_weight, weight):
        """One ResidualSimVQ stage tail (vqb_rsimvq_tail) after that stage's `stage` op: r (N, D) fp32, codes (K, D) fp32."""
        N, D = r.shape
        op = _C.RvqOp(kind=_C.RVQ_SIMVQ_TAIL, lane=lane)
        op.simvq = _C.RvqSimvqArgs(r=_p(r), codes=_p(codes), idx=_p(idx32), N=N, D=D, rotation=int(rotation), r_next=_p(r_next),
                                   qsum=_p(qsum), first=int(first), idx64_out=_p(idx64_out), idx_stride=int(idx_stride),
                                   loss_sum=_p(loss_sum), loss_out=_p(loss_out), input_weight=float(input_weight),
                                   weight=float(weight))
        self.ops.append(op)
        self.keep.append((r, codes, idx32, r_next, qsum, idx64_out, loss_sum, loss_out))
        self.launches += 3 if loss_out is not None else 1

    def freeze(self):
        """Materialise the op array once; afterwards only `arr` is patched (cached programs: residual_vq.py)."""
        n = len(self.ops)
        assert 0 < n <= self.MAX_OPS
        self.arr = (_C.RvqOp * n)(*self.ops)
        self.n = n
        self.ops = None
        # whoever freezes a pointer owns the memory behind it: the program keeps the scratch its stage ops point into (freed
        # with the program), the owner of a cached program keeps its other persistent tensors alive itself (and re-binds the rest)
        self.keep = None
        return self

    def run(self):
        if getattr(self, "arr", None) is None:
            self.freeze()
        with torch.cuda.device(self.device):
            check(lib.vqb_rvq_forward(ctypes.cast(self.arr, ctypes.c_void_p), self.n, _stream()), "vqb_rvq_forward")
        _count(self.launches)


def gather(x_eff: torch.Tensor, embed: torch.Tensor, idx: torch.Tensor, *, q_out: torch.Tensor | None = None,
           idx64_out: torch.Tensor | None = None, idx_stride: int = 1, loss_sum: torch.Tensor | None = None,
           x_raw: torch.Tensor | None = None, resid_out: torch.Tensor | None = None) -> None:
    """quantize = embed[idx].type(x.dtype) (vqp:766/:779-781, :1178) fused with the mse partial sum (vqp:1327)
    and, for ResidualVQ, residual -= q (rvq:524)."""
    _require_cuda(x_eff, embed, idx)
    N, D = x_eff.shape
    with torch.cuda.device(x_eff.device):
        check(lib.vqb_gather(_p(x_eff), _dtype_code(x_eff), N, D, _p(embed), _p(idx), _p(q_out), _p(idx64_out),
                             int(idx_stride), _p(loss_sum), _p(x_raw), _p(resid_out), None, _stream()), "vqb_gather")
    _count(1)


def loss_finalize(loss_sum: torch.Tensor, numel: int, dtype: torch.dtype, weight: float, out: torch.Tensor) -> None:
    with torch.cuda.device(loss_sum.device):
        check(lib.vqb_loss_finalize(_p(loss_sum), int(numel), _DT[dtype], float(weight), _p(out), _stream()),
              "vqb_loss_finalize")
    _count(1)


def stats_floats(K: int, D: int) -> int:
    return lib.vqb_stats_floats(K, D)


def stats_offset(K: int) -> int:
    return lib.vqb_stats_offset(K)


def ema_stats(x_eff: torch.Tensor, idx: torch.Tensor, K: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """Packed [cluster_size | embed_sum] of this batch (vqp:602, :605) — ready for ONE all-reduce."""
    _require_cuda(x_eff, idx)
    N, D = x_eff.shape
    dev = x_eff.device
    stats = out if out is not None else torch.empty((stats_floats(K, D),), dtype=torch.float32, device=dev)
    ws_bytes = lib.vqb_ema_stats_workspace(N, K)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(lib.vqb_ema_stats(_p(x_eff), _dtype_code(x_eff), N, D, _p(idx), K, _p(stats), _p(ws), ws_bytes, _stream()),
              "vqb_ema_stats")
    _count(4)
    return stats


def ema_apply(cluster_size: torch.Tensor, embed_avg: torch.Tensor, embed: torch.Tensor, stats: torch.Tensor | None,
              ops: CodebookOperands, *, decay: float, eps: float, do_lerp: bool, do_normalise: bool,
              code_weight: torch.Tensor | None = None) -> None:
    """lerp_ of cluster_size / embed_avg (vqp:616-617) and update_ema (vqp:576-584); refreshes `ops`.
    code_weight (K,) fp32: the reference's per-code `ema_update_weight` (vqp:86-97)."""
    _require_cuda(cluster_size, embed_avg, embed, code_weight)
    K, D = embed.shape
    if code_weight is not None:
        assert code_weight.dtype == torch.float32 and code_weight.is_contiguous() and code_weight.numel() == K
    with torch.cuda.device(embed.device):
        check(lib.vqb_ema_apply_weighted(_p(cluster_size), _p(embed_avg), _p(embed), _p(stats), K, D, float(decay), float(eps),
                                         int(ops.cosine), int(do_lerp), int(do_normalise), _p(code_weight), _p(ops.planes),
                                         _p(ops.bext), _p(ops.bias), _p(ops.cnorm2), _p(ops.cmax), _p(ops.scratch), _stream()),
              "vqb_ema_apply")
    _count(2)


def decode(embeds: torch.Tensor, indices: torch.Tensor, out_dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """sum_q embeds[q][indices[..., q]] with -1 -> zeros (rvq:324-382).  embeds (Q, K, D) fp32 or (K, D)."""
    _require_cuda(embeds, indices)
    if embeds.dim() == 2:
        embeds = embeds.unsqueeze(0)
    Q, K, D = embeds.shape
    assert indices.shape[-1] == Q and indices.dtype == torch.int64
    embeds = embeds.contiguous()
    flat = indices.reshape(-1, Q).contiguous()
    N = flat.shape[0]
    out = torch.empty((N, D), dtype=out_dtype, device=embeds.device)
    with torch.cuda.device(embeds.device):
        check(lib.vqb_decode(_p(embeds), K * D, Q, K, D, _p(flat), N, _p(out), _DT[out_dtype], _stream()), "vqb_decode")
    _count(1)
    return out.reshape(*indices.shape[:-1], D)


def rvq_accumulate(embeds: torch.Tensor, indices: torch.Tensor, out_dtype: torch.dtype) -> torch.Tensor:
    """ResidualVQ's `quantized_out` from the stage indices (N, Q): the rounded running sum of rvq:525 in ONE pass.
    embeds (Q, K, D) fp32 — the codebooks the stages SEARCHED (pre-update), or (K, D) for a shared codebook."""
    _require_cuda(embeds, indices)
    assert indices.dim() == 2 and indices.dtype == torch.int64 and indices.is_contiguous()
    N, Q = indices.shape
    if embeds.dim() == 2:
        K, D = embeds.shape
        stride = 0
    else:
        assert embeds.shape[0] == Q
        _, K, D = embeds.shape
        stride = K * D
    embeds = embeds.contiguous()
    out = torch.empty((N, D), dtype=out_dtype, device=embeds.device)
    with torch.cuda.device(embeds.device):
        check(lib.vqb_rvq_accumulate(_p(embeds), stride, Q, K, D, _p(indices), N, _p(out), _DT[out_dtype], _stream()),
              "vqb_rvq_accumulate")
    _count(1)
    return out


def peer_barrier(peer) -> None:
    """Cross-GPU barrier kernel on the current stream (dist.PeerReducer; csrc/vq_peer.cu)."""
    with torch.cuda.device(peer.device):
        check(lib.vqb_peer_barrier(ctypes.cast(peer.flag_ptrs, ctypes.c_void_p), peer.rank, peer.world, peer.epoch.data_ptr(),
                                   _stream()), "vqb_peer_barrier")
    _count(1)


def ema_apply_peers(cluster_size: torch.Tensor, embed_avg: torch.Tensor, embed: torch.Tensor, peer, peer_ptrs, slice_offset: int,
                    ops: CodebookOperands, *, decay: float, eps: float, do_normalise: bool,
                    code_weight: torch.Tensor | None = None) -> None:
    """`ema_apply` with the statistics summed over every rank's symmetric buffer inside the kernels (after `peer_barrier`)."""
    _require_cuda(cluster_size, embed_avg, embed, code_weight)
    K, D = embed.shape
    with torch.cuda.device(embed.device):
        check(lib.vqb_ema_apply_peers(_p(cluster_size), _p(embed_avg), _p(embed), ctypes.cast(peer_ptrs, ctypes.c_void_p), peer.world,
                                      int(slice_offset), K, D, float(decay), float(eps), int(ops.cosine), int(do_normalise),
                                      _p(code_weight), _p(ops.planes), _p(ops.bext), _p(ops.bias), _p(ops.cnorm2), _p(ops.cmax),
                                      _p(ops.scratch), _stream()), "vqb_ema_apply_peers")
    _count(2)


def rsimvq_backward(x: torch.Tensor, codes: torch.Tensor, indices: torch.Tensor, rotation: bool, grad_q: torch.Tensor | None,
                    grad_loss: torch.Tensor | None) -> torch.Tensor:
    """d loss / d x of a whole ResidualSimVQ forward (vqb_rsimvq_backward).  x (N, D) fp32; codes (n_active, K, D) fp32, the
    codebooks of the stages that ran; indices (N, Q) int64; grad_loss (n_active,) fp32 already scaled by
    2 * weight * input_weight / (N * D)."""
    _require_cuda(x, codes, indices, grad_q, grad_loss)
    N, D = x.shape
    n_active, K, _ = codes.shape
    Q = indices.shape[1]
    for t in (x, codes, indices, grad_q, grad_loss):
        assert t is None or t.is_contiguous()
    gx = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.vqb_rsimvq_backward(_p(x), _p(codes), Q, K, _p(indices), N, D, n_active, int(rotation), _p(grad_q),
                                      _p(grad_loss), _p(gx), _stream()), "vqb_rsimvq_backward")
    _count(1)
    return gx


def rotate(src: torch.Tensor, tgt: torch.Tensor, grad_out: torch.Tensor | None = None) -> torch.Tensor:
    """Rotation-trick estimator (vqp:287-318): forward value (grad_out None) or the gradient w.r.t. src."""
    _require_cuda(src, tgt, grad_out)
    shape = src.shape
    s2 = src.reshape(-1, shape[-1]).contiguous()
    t2 = tgt.reshape(-1, shape[-1]).contiguous()
    g2 = grad_out.reshape(-1, shape[-1]).contiguous() if grad_out is not None else None
    assert s2.dtype == t2.dtype and (g2 is None or g2.dtype == s2.dtype)
    out = torch.empty_like(s2)
    with torch.cuda.device(s2.device):
        check(lib.vqb_rotate(_p(s2), _p(t2), _p(g2), s2.shape[0], s2.shape[1], _dtype_code(s2), _p(out), _stream()), "vqb_rotate")
    _count(1)
    return out.reshape(shape)


ESTIMATOR_NONE, ESTIMATOR_STE, ESTIMATOR_ROTATE = 0, 1, 2   # VQB_ESTIMATOR_*


def rotate_masked(src: torch.Tensor, tgt: torch.Tensor, row_mask: torch.Tensor, estimator: int, pad_zeros: bool,
                  grad_out: torch.Tensor | None = None, grad_loss: torch.Tensor | None = None,
                  n_live: torch.Tensor | None = None, loss_weight: float = 1.) -> torch.Tensor:
    """Estimator of a masked training step (vqb_rotate_masked).  src, tgt, grad_out (N, D) in one dtype; row_mask (N,) uint8;
    grad_out None: the forward (live rows tgt, padding rows 0 or src); else d/d src of the estimator on live rows plus
    2 loss_weight grad_loss (src - tgt) / (n_live D), and on padding rows 0 or grad_out.  grad_loss f32 (1,) and n_live
    int64 (1,) stay on the device."""
    _require_cuda(src, tgt, row_mask, grad_out, grad_loss, n_live)
    N, D = src.shape
    assert tgt.shape == src.shape and tgt.dtype == src.dtype and (grad_out is None or grad_out.dtype == src.dtype)
    assert row_mask.dtype == torch.uint8 and row_mask.shape == (N,)
    assert grad_loss is None or (grad_loss.dtype == torch.float32 and n_live is not None and n_live.dtype == torch.int64)
    for t in (src, tgt, grad_out, row_mask, grad_loss, n_live):
        assert t is None or t.is_contiguous()
    out = torch.empty_like(src)
    if N == 0:
        return out
    with torch.cuda.device(src.device):
        check(lib.vqb_rotate_masked(_p(src), _p(tgt), _p(grad_out), _p(grad_loss), _p(row_mask), _p(n_live), float(loss_weight),
                                    int(estimator), int(bool(pad_zeros)), N, D, _dtype_code(src), _p(out), _stream()),
              "vqb_rotate_masked")
    _count(1)
    return out


def diveq(x: torch.Tensor, q: torch.Tensor, noise: torch.Tensor, noise_scale: float, grad_out: torch.Tensor | None = None):
    """DiVeQ estimator (vqp:323-330, vqb_diveq): the forward value x + l2norm(q - x + noise_scale * noise) * ||q - x|| when
    grad_out is None, else (dx in x.dtype, dq fp32).  x, q, noise, grad_out: (..., D) in one dtype."""
    _require_cuda(x, q, noise, grad_out)
    shape = x.shape
    D = shape[-1]
    rows = [t.reshape(-1, D).contiguous() if t is not None else None for t in (x, q, noise, grad_out)]
    assert all(t is None or t.dtype == x.dtype for t in rows)
    x2, q2, z2, g2 = rows
    out = torch.empty_like(x2)
    dq = torch.empty(x2.shape, dtype=torch.float32, device=x2.device) if g2 is not None else None
    with torch.cuda.device(x2.device):
        check(lib.vqb_diveq(_p(x2), _p(q2), _p(z2), _p(g2), x2.shape[0], D, _dtype_code(x2), float(noise_scale), _p(out), _p(dq),
                            _stream()), "vqb_diveq")
    _count(1)
    if g2 is None:
        return out.reshape(shape)
    return out.reshape(shape), dq.reshape(shape)


def fsq_forward(z: torch.Tensor, work_dtype: torch.dtype, Q: int, n_active: int, sym: bool, hard: bool, consts: torch.Tensor,
                scales: torch.Tensor | None, clampv: torch.Tensor | None, indices: torch.Tensor) -> torch.Tensor:
    """vqb_fsq_forward: z (N, G, D) contiguous in fp32 / bf16 -> out (N, G, D) in `work_dtype`; writes the indices into
    `indices`, an (N, G, Q) view (int32 / int64, any strides) of the caller's index tensor.  consts (7, D), scales (2, Q, D), clampv (2, D): fp32 tables
    of the module (include/vqb200.h)."""
    _require_cuda(z, consts, scales, clampv, indices)
    N, G, D = z.shape
    out = torch.empty(z.shape, dtype=work_dtype, device=z.device)
    s_row, s_g, s_q = _index_strides(indices)
    with torch.cuda.device(z.device):
        check(lib.vqb_fsq_forward(_p(z), _dtype_code(z), _DT[work_dtype], N, G, D, Q, n_active, int(sym), int(hard), _p(consts),
                                  _p(scales), _p(clampv), _p(out), _p(indices), int(indices.dtype == torch.int64), s_row, s_g, s_q,
                                  _stream()), "vqb_fsq_forward")
    _count(1)
    return out


def fsq_backward(z: torch.Tensor, grad_out: torch.Tensor, Q: int, n_active: int, sym: bool, hard: bool, consts: torch.Tensor,
                 scales: torch.Tensor | None, clampv: torch.Tensor | None) -> torch.Tensor:
    """vqb_fsq_backward: d z (z's dtype) of fsq_forward's output given its gradient (N, G, D) in the work dtype."""
    _require_cuda(z, grad_out, consts, scales, clampv)
    N, G, D = z.shape
    gz = torch.empty_like(z)
    g = _aligned(grad_out)
    with torch.cuda.device(z.device):
        check(lib.vqb_fsq_backward(_p(z), _dtype_code(z), _dtype_code(g), N, G, D, Q, n_active, int(sym), int(hard), _p(consts),
                                   _p(scales), _p(clampv), _p(g), _p(gz), _stream()), "vqb_fsq_backward")
    _count(1)
    return gz


def fsq_decode(indices: torch.Tensor, D: int, work_dtype: torch.dtype, sym: bool, consts: torch.Tensor, levels_basis: torch.Tensor,
               scales: torch.Tensor | None, want_sum: bool, want_codes: bool):
    """vqb_fsq_decode: indices, an (N, G, Q) view (any strides) -> (sum over the stages (N, G, D) or None, stage codes
    (Q, N, G, D) or None) in `work_dtype`."""
    _require_cuda(indices, consts, levels_basis, scales)
    _check_index_dtype(indices, "FSQ")
    N, G, Q = indices.shape
    dev = indices.device
    out = torch.empty((N, G, D), dtype=work_dtype, device=dev) if want_sum else None
    codes = torch.empty((Q, N, G, D), dtype=work_dtype, device=dev) if want_codes else None
    s_row, s_g, s_q = _index_strides(indices)
    with torch.cuda.device(dev):
        check(lib.vqb_fsq_decode(_p(indices), int(indices.dtype == torch.int64), s_row, s_g, s_q, N, G, D, Q, _DT[work_dtype], int(sym),
                                 _p(consts), _p(levels_basis), _p(scales), _p(out), _p(codes), _stream()), "vqb_fsq_decode")
    _count(1)
    return out, codes


# ---- lookup-free quantization (csrc/vq_lfq.cu) ----

def lfq_forward(z: torch.Tensor, Q: int, n_active: int, residual: bool, training: bool, spherical: bool, params: torch.Tensor,
                indices: torch.Tensor, want_entropy: bool, rowmask: torch.Tensor | None, want_commit: bool):
    """vqb_lfq_forward: z (N, G, D) contiguous fp32 / bf16 -> (out (N, G, D) in z's dtype, entropy input (n_active, N, G, D) fp32
    or None, commitment sums (n_active,) fp64 or None); writes the int64 indices into `indices`, an (N, G, Q) view (any strides).
    params (3, Q) fp32: per-stage scale, code magnitude, soft-clamp value (0: none)."""
    _require_cuda(z, params, indices, rowmask)
    if indices.dtype != torch.int64:
        raise TypeError("LFQ indices are int64")
    N, G, D = z.shape
    dev = z.device
    out = torch.empty(z.shape, dtype=z.dtype, device=dev)
    ent = torch.empty((n_active, N, G, D), dtype=torch.float32, device=dev) if want_entropy else None
    s_row, s_g, s_q = _index_strides(indices)
    with torch.cuda.device(dev):
        blocks = _queried(lib.vqb_lfq_forward_blocks(N, G), "vqb_lfq_forward_blocks")
        commit = torch.empty((n_active, blocks), dtype=torch.float64, device=dev) if want_commit else None
        check(lib.vqb_lfq_forward(_p(z), _dtype_code(z), N, G, D, Q, n_active, int(residual), int(training), int(spherical), _p(params),
                                  _p(out), _p(indices), s_row, s_g, s_q, _p(ent), _p(rowmask), _p(commit), blocks, _stream()),
              "vqb_lfq_forward")
    _count(1)
    return out, ent, (commit.sum(1) if commit is not None else None)


def lfq_backward(z: torch.Tensor, grad_out: torch.Tensor, Q: int, n_active: int, residual: bool, training: bool, spherical: bool,
                 params: torch.Tensor, grad_ent: torch.Tensor | None, cc: torch.Tensor | None, rowmask: torch.Tensor | None):
    """vqb_lfq_backward: d z (z's dtype) of lfq_forward's outputs: grad_out (N, G, D) for `out`, grad_ent for the entropy input,
    cc (n_active,) fp32 (the gradient of each stage's commitment sum, times 2) for the commitment sums."""
    _require_cuda(z, grad_out, params, grad_ent, cc, rowmask)
    N, G, D = z.shape
    gz = torch.empty_like(z)
    g = grad_out.to(z.dtype).contiguous()
    ge = grad_ent.contiguous() if grad_ent is not None else None
    with torch.cuda.device(z.device):
        check(lib.vqb_lfq_backward(_p(z), _dtype_code(z), N, G, D, Q, n_active, int(residual), int(training), int(spherical),
                                   _p(params), _p(g), _p(ge), _p(cc), _p(rowmask), _p(gz), _stream()), "vqb_lfq_backward")
    _count(1)
    return gz


def lfq_entropy_plan(R: int, SG: int, D: int, sms: int, want_colsum: bool) -> tuple[int, int]:
    """(chunks, ksplit) of the entropy kernels for R rows in each of SG (stage, group) pairs of 2^D codes on `sms` SMs (host
    only).  chunks (vqb_lfq_entropy): row chunks, enough CTAs for 4 per SM, at most one per 32-row batch, and with the column
    sums at most 8 Mi floats of per-chunk partials.  ksplit (vqb_lfq_entropy_backward): the K split, doubled while the CTAs
    are under 4 per SM and each split keeps at least 2048 codes."""
    K = 1 << D
    tiles = _queried(lib.vqb_lfq_entropy_tiles(D), "vqb_lfq_entropy_tiles")
    chunks = -(-4 * sms // (tiles * SG))
    chunks = max(1, min(chunks, -(-R // 32), 65535))
    if want_colsum:
        chunks = max(1, min(chunks, (8 << 20) // (SG * K)))   # partial column sums <= 32 MiB
    blocks = -(-R // 128) * SG
    ksplit = 1
    while blocks * ksplit < 4 * sms and K // (2 * ksplit) >= 2048:
        ksplit *= 2
    return chunks, ksplit


def lfq_entropy(x: torch.Tensor, rows: torch.Tensor | None, R: int, m: torch.Tensor, tau: float, want_colsum: bool,
                chunks: int | None = None):
    """vqb_lfq_entropy over x (S, N, G, D) fp32: -> (sum of h(p) per (s, g) (S * G,) fp64, column sums of p (S * G, K) fp32 or
    None).  rows: int32 (S * G, R) or (R,) row lists, or None for rows 0..R-1.  chunks: the plan's by default."""
    _require_cuda(x, rows, m)
    S, N, G, D = x.shape
    SG, K, dev = S * G, 1 << D, x.device
    tiles = _queried(lib.vqb_lfq_entropy_tiles(D), "vqb_lfq_entropy_tiles")
    if chunks is None:
        chunks = lfq_entropy_plan(R, SG, D, _sms(dev), want_colsum)[0]
    rs = 0 if rows is None or rows.dim() == 1 else rows.shape[1]
    pse = torch.empty((SG, chunks, tiles), dtype=torch.float64, device=dev)
    col = torch.empty((chunks, SG, K), dtype=torch.float32, device=dev) if want_colsum else None
    with torch.cuda.device(dev):
        check(lib.vqb_lfq_entropy(_p(x), N, G, D, S, _p(rows), R, rs, _p(m), float(tau), chunks, _p(pse), _p(col), _stream()),
              "vqb_lfq_entropy")
    _count(1)
    return pse.sum((1, 2)), (col.sum(0) if col is not None else None)


def lfq_entropy_backward(x: torch.Tensor, rows: torch.Tensor | None, R: int, m: torch.Tensor, tau: float, cp: torch.Tensor,
                         V: torch.Tensor | None, ksplit: int | None = None) -> torch.Tensor:
    """vqb_lfq_entropy_backward: d/dx (x's layout, zero outside the listed rows) given dL/dp = cp[sg] h'(p) + V[sg, k].
    ksplit: the plan's by default."""
    _require_cuda(x, rows, m, cp, V)
    S, N, G, D = x.shape
    SG, dev = S * G, x.device
    if ksplit is None:
        ksplit = lfq_entropy_plan(R, SG, D, _sms(dev), False)[1]
    rs = 0 if rows is None or rows.dim() == 1 else rows.shape[1]
    work = torch.empty((ksplit, SG, R, D + 1), dtype=torch.float32, device=dev)
    grad = torch.zeros_like(x)
    cp = cp.float().contiguous()
    V = V.float().contiguous() if V is not None else None
    with torch.cuda.device(dev):
        check(lib.vqb_lfq_entropy_backward(_p(x), N, G, D, S, _p(rows), R, rs, _p(m), float(tau), _p(cp), _p(V), ksplit, _p(work),
                                           _p(grad), _stream()), "vqb_lfq_entropy_backward")
    _count(2)
    return grad


def lfq_decode(indices: torch.Tensor, D: int, vals: torch.Tensor, want_sum: bool, want_codes: bool):
    """vqb_lfq_decode: indices, an (N, G, Q) view (any strides, int32 / int64, -1 = dropped) -> (sum over the stages (N, G, D) or
    None, codes (Q, N, G, D) or None), fp32."""
    _require_cuda(indices, vals)
    _check_index_dtype(indices, "LFQ")
    N, G, Q = indices.shape
    dev = indices.device
    out = torch.empty((N, G, D), dtype=torch.float32, device=dev) if want_sum else None
    codes = torch.empty((Q, N, G, D), dtype=torch.float32, device=dev) if want_codes else None
    s_row, s_g, s_q = _index_strides(indices)
    with torch.cuda.device(dev):
        check(lib.vqb_lfq_decode(_p(indices), int(indices.dtype == torch.int64), s_row, s_g, s_q, N, G, D, Q, _p(vals), _p(out),
                                 _p(codes), _stream()), "vqb_lfq_decode")
    _count(1)
    return out, codes


# ---- finite scalar perturbation (csrc/vq_fsp.cu) ----

def fsp_forward(z: torch.Tensor, act: int, inv: bool, levels: torch.Tensor, clamp_hi: float, u1: torch.Tensor | None,
                u2: torch.Tensor | None, qrate: float, inv_lo: float, inv_hi: float):
    """vqb_fsp_forward: z (N, D) contiguous, 16-byte aligned, fp32 / bf16 -> (out (N, D), fp32 when perturbing else z's dtype;
    indices (N,) int32; level indices (N, D) in z's dtype; the accepted-proposal count (int64 scalar) or None).  u1, u2: the
    two (N, D) draws in z's dtype, or None for no perturbation."""
    _require_cuda(z, levels, u1, u2)
    N, D = z.shape
    dev = z.device
    out = torch.empty((N, D), dtype=torch.float32 if u1 is not None else z.dtype, device=dev)
    idx = torch.empty((N,), dtype=torch.int32, device=dev)
    lev = torch.empty((N, D), dtype=z.dtype, device=dev)
    with torch.cuda.device(dev):
        blocks = _queried(lib.vqb_fsp_blocks(N), "vqb_fsp_blocks")
        acc = torch.empty((blocks,), dtype=torch.int32, device=dev) if u1 is not None else None
        check(lib.vqb_fsp_forward(_p(z), _dtype_code(z), N, D, act, int(inv), _p(levels), clamp_hi, _p(u1), _p(u2), qrate, inv_lo,
                                  inv_hi, _p(out), _p(idx), _p(lev), _p(acc), blocks, _stream()), "vqb_fsp_forward")
    _count(1)
    return out, idx, lev, (acc.sum(dtype=torch.int64) if acc is not None else None)


def _norm_arg(norm) -> ctypes.Array:
    return (ctypes.c_double * 8)(*[float(v) for v in norm])


def fsp_stats(z: torch.Tensor, norm):
    """vqb_fsp_stats: z (N, D) -> (stats (4, D) = mean, variance, skewness, kurtosis in z's dtype, norm loss () in z's dtype,
    aux (D, 8) fp64 for fsp_backward).  norm: (l1_target, l1_weight, ..., l4_target, l4_weight)."""
    _require_cuda(z)
    N, D = z.shape
    dev = z.device
    stats = torch.empty((4, D), dtype=z.dtype, device=dev)
    loss = torch.empty((), dtype=z.dtype, device=dev)
    aux = torch.empty((D, 8), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        blocks = _queried(lib.vqb_fsp_blocks(N), "vqb_fsp_blocks")
        work = torch.empty((4 * blocks + 1, D), dtype=torch.float64, device=dev)
        check(lib.vqb_fsp_stats(_p(z), _dtype_code(z), N, D, _norm_arg(norm), _p(work), blocks, _p(stats), _p(loss), _p(aux),
                                _stream()), "vqb_fsp_stats")
    _count(4)
    return stats, loss, aux


def fsp_backward(z: torch.Tensor, act: int, inv: bool, grad_q: torch.Tensor | None, aux: torch.Tensor,
                 grad_stats: torch.Tensor | None, grad_loss: torch.Tensor | None, norm) -> torch.Tensor:
    """vqb_fsp_backward: d z (z's dtype) given the gradients of fsp_forward's out (N, D) and of fsp_stats' stats (4, D) and
    loss (), each None for zero."""
    _require_cuda(z, grad_q, aux, grad_stats, grad_loss)
    N, D = z.shape
    gz = torch.empty_like(z)
    g = _aligned(grad_q) if grad_q is not None else None
    gs = grad_stats.float().contiguous() if grad_stats is not None else None
    gl = grad_loss.float().reshape(1) if grad_loss is not None else None
    with torch.cuda.device(z.device):
        check(lib.vqb_fsp_backward(_p(z), _dtype_code(z), N, D, act, int(inv), _p(g), _dtype_code(g) if g is not None else 0,
                                   _p(aux), _p(gs), _p(gl), _norm_arg(norm), _p(gz), _stream()), "vqb_fsp_backward")
    _count(1)
    return gz


def fsp_decode(indices: torch.Tensor, D: int, act: int, inv: bool, levels: torch.Tensor, lo: float, hi: float, want_act: bool,
               want_codes: bool):
    """vqb_fsp_decode: indices (any shape, int32 / int64) -> (act values, codes), each (*indices.shape, D) fp32 or None."""
    _require_cuda(indices, levels)
    _check_index_dtype(indices, "FSP")
    idx = indices.contiguous()
    N = idx.numel()
    dev = idx.device
    shape = (*indices.shape, D)
    act_out = torch.empty(shape, dtype=torch.float32, device=dev) if want_act else None
    codes = torch.empty(shape, dtype=torch.float32, device=dev) if want_codes else None
    if N == 0:
        return act_out, codes
    with torch.cuda.device(dev):
        check(lib.vqb_fsp_decode(_p(idx), int(idx.dtype == torch.int64), N, D, act, int(inv), _p(levels), lo, hi, _p(act_out),
                                 _p(codes), _stream()), "vqb_fsp_decode")
    _count(1)
    return act_out, codes


# ---- BinaryMapper (csrc/vq_binmap.cu) ----

def binmap_hot(out: torch.Tensor, logits: torch.Tensor | None, indices: torch.Tensor) -> torch.Tensor:
    """vqb_binmap_hot: writes the hot element of every row of the zero-filled out (rows, 2^bits) fp32 in place: 1, or with
    logits (rows, bits) fp32 contiguous the straight-through value fl(fl(1 + s) - s).  indices: (rows,) int64."""
    _require_cuda(out, logits, indices)
    rows, K = out.shape
    if rows == 0:
        return out
    idx = indices.to(torch.int64).contiguous()
    with torch.cuda.device(out.device):
        check(lib.vqb_binmap_hot(_p(logits), _p(idx), rows, K.bit_length() - 1, _p(out), _stream()), "vqb_binmap_hot")
    _count(1)
    return out


def binmap_backward_plan(rows: int, bits: int, sms: int) -> tuple[int, int]:
    """(ksplit, codes per segment) of vqb_binmap_backward for (rows, bits) on `sms` SMs."""
    plan = (ctypes.c_int * 2)()
    check(lib.vqb_binmap_backward_plan(rows, bits, sms, plan), "vqb_binmap_backward_plan")
    return plan[0], plan[1]


def binmap_backward(logits: torch.Tensor, g: torch.Tensor, ksplit: int | None = None) -> torch.Tensor:
    """vqb_binmap_backward: d logits (rows, bits) fp32 of sum(out * g) through the soft codes.  logits (rows, bits) fp32
    contiguous; g (rows, 2^bits) fp32 with any non-negative strides and offset (read in place).  ksplit: the plan's by default."""
    _require_cuda(logits, g)
    rows, bits = logits.shape
    dl = torch.empty((rows, bits), dtype=torch.float32, device=logits.device)
    if rows == 0:
        return dl
    if g.dtype != torch.float32:
        g = g.float()
    with torch.cuda.device(logits.device):
        if ksplit is None:
            ksplit = binmap_backward_plan(rows, bits, _sms(logits.device))[0]
        work = torch.empty((rows, ksplit, 2 * bits), dtype=torch.float64, device=logits.device) if ksplit > 1 else None
        check(lib.vqb_binmap_backward(_p(logits), rows, bits, _p(g), g.stride(0), g.stride(1), ksplit, _p(work), _p(dl),
                                      _stream()), "vqb_binmap_backward")
    _count(1 if ksplit == 1 else 2)
    return dl


# ---- HierarchicalVQ (csrc/vq_hvq.cu) ----
# Images are (B, D, H, W) NCHW contiguous fp32; `rows` are the channel-last (B, s, s, D) contiguous maps the search reads and
# writes, handed around as their (B, D, s, s) views.

def _hvq_image(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise TypeError(f"vqb200 HierarchicalVQ supports float32 {what}, got {t.dtype}")
    _require_cuda(t)
    return t.contiguous()


def _hvq_rows(t: torch.Tensor, what: str) -> torch.Tensor:
    """A (B, D, s, s) map as its channel-last rows (B, s, s, D) contiguous: free for the search's own outputs."""
    if t.dtype != torch.float32:
        raise TypeError(f"vqb200 HierarchicalVQ supports float32 {what}, got {t.dtype}")
    _require_cuda(t)
    return t.permute(0, 2, 3, 1).contiguous()


def hvq_pool(x: torch.Tensor, s: int) -> torch.Tensor:
    """vqb_hvq_pool: adaptive_avg_pool2d(x, (s, s)) of x (B, D, H, W), returned as the (B, D, s, s) view of channel-last rows."""
    x = _hvq_image(x, "inputs")
    B, D, H, W = x.shape
    rows = torch.empty((B, s, s, D), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.vqb_hvq_pool(_p(x), B, D, H, W, s, _p(rows), _stream()), "vqb_hvq_pool")
    _count(1)
    return rows.permute(0, 3, 1, 2)


def hvq_pool_backward(g: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """vqb_hvq_pool_backward: d x (B, D, H, W) from the gradient g (B, D, s, s) of hvq_pool's output."""
    g = _hvq_rows(g, "gradients")
    B, s, _, D = g.shape
    gx = torch.empty((B, D, H, W), dtype=torch.float32, device=g.device)
    with torch.cuda.device(g.device):
        check(lib.vqb_hvq_pool_backward(_p(g), B, D, H, W, s, _p(gx), _stream()), "vqb_hvq_pool_backward")
    _count(1)
    return gx


def hvq_upsample(q: torch.Tensor, H: int, W: int, recon=None, resid=None, want_q=True, want_recon=False, want_resid=False):
    """vqb_hvq_upsample: u = bilinear(q (B, D, s, s), (H, W)) (q itself when (s, s) == (H, W)).  Returns (u, recon + u,
    resid - u), each None unless asked for; recon None counts as zero."""
    rows = _hvq_rows(q, "inputs")
    B, s, _, D = rows.shape
    outs = [torch.empty((B, D, H, W), dtype=torch.float32, device=q.device) if want else None
            for want in (want_q, want_recon, want_resid)]
    recon = None if recon is None else _hvq_image(recon, "reconstructions")
    resid = None if resid is None else _hvq_image(resid, "residuals")
    with torch.cuda.device(q.device):
        check(lib.vqb_hvq_upsample(_p(rows), B, D, s, H, W, _p(outs[0]), _p(recon), _p(resid), _p(outs[1]), _p(outs[2]),
                                   _stream()), "vqb_hvq_upsample")
    _count(1)
    return tuple(outs)


def hvq_upsample_backward(g_a, g_b, s: int) -> torch.Tensor:
    """vqb_hvq_upsample_backward: d q (B, D, s, s), as the view of channel-last rows, from g_a - g_b (B, D, H, W) (either
    None: zero, not both)."""
    g_a = None if g_a is None else _hvq_image(g_a, "gradients")
    g_b = None if g_b is None else _hvq_image(g_b, "gradients")
    ref = g_a if g_a is not None else g_b
    B, D, H, W = ref.shape
    g_rows = torch.empty((B, s, s, D), dtype=torch.float32, device=ref.device)
    with torch.cuda.device(ref.device):
        check(lib.vqb_hvq_upsample_backward(_p(g_a), _p(g_b), B, D, s, H, W, _p(g_rows), _stream()),
              "vqb_hvq_upsample_backward")
    _count(1)
    return g_rows.permute(0, 3, 1, 2)


def hvq_blend_update(up: torch.Tensor, conv: torch.Tensor, r: float, recon=None, resid=None, want_resid=True):
    """vqb_hvq_blend_update: q = (1 - r) up + r conv; returns (recon + q, resid - q or None).  recon None counts as zero."""
    up, conv = _hvq_image(up, "inputs"), _hvq_image(conv, "inputs")
    recon = None if recon is None else _hvq_image(recon, "reconstructions")
    resid = None if resid is None else _hvq_image(resid, "residuals")
    recon_out = torch.empty_like(up)
    resid_out = torch.empty_like(up) if want_resid else None
    with torch.cuda.device(up.device):
        check(lib.vqb_hvq_blend_update(_p(up), _p(conv), up.numel(), float(r), _p(recon), _p(resid), _p(recon_out),
                                       _p(resid_out), _stream()), "vqb_hvq_blend_update")
    _count(1)
    return recon_out, resid_out


def hvq_blend_backward(g_recon, g_resid, r: float):
    """vqb_hvq_blend_backward: (d up, d conv) from the gradients of recon + q and resid - q (either None: zero, not both)."""
    g_recon = None if g_recon is None else _hvq_image(g_recon, "gradients")
    g_resid = None if g_resid is None else _hvq_image(g_resid, "gradients")
    ref = g_recon if g_recon is not None else g_resid
    g_up, g_conv = torch.empty_like(ref), torch.empty_like(ref)
    with torch.cuda.device(ref.device):
        check(lib.vqb_hvq_blend_backward(_p(g_recon), _p(g_resid), ref.numel(), float(r), _p(g_up), _p(g_conv), _stream()),
              "vqb_hvq_blend_backward")
    _count(1)
    return g_up, g_conv


# ---- RandomProjectionQuantizer (csrc/vq_rpq.cu) ----

def rpq_norm_project(x: torch.Tensor, proj: torch.Tensor, norm: bool) -> torch.Tensor:
    """vqb_rpq_norm_project: LN(x) @ proj for x (..., dim) and proj (H, dim, E) (`rand_projs`), returned as fp32 rows
    (prod(x.shape[:-1]), H * E) packed head-major like the reference's 'b n h e -> b n (h e)'; norm False skips the LN."""
    if x.dtype != torch.float32 or proj.dtype != torch.float32:
        raise TypeError(f"vqb200 RandomProjectionQuantizer supports float32 inputs, got {x.dtype} (projection {proj.dtype})")
    _require_cuda(x, proj)
    if x.device != proj.device:
        raise RuntimeError(f"vqb200 RandomProjectionQuantizer: inputs on {x.device}, projection on {proj.device}")
    H, dim, E = proj.shape
    assert x.shape[-1] == dim, (x.shape, proj.shape)
    x = x.reshape(-1, dim).contiguous()
    proj = proj.contiguous()
    rows = torch.empty((x.shape[0], H * E), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.vqb_rpq_norm_project(_p(x), x.shape[0], dim, _p(proj), H, E, int(bool(norm)), _p(rows), _stream()),
              "vqb_rpq_norm_project")
    _count(1)
    return rows


# ---- LatentQuantize (csrc/vq_lq.cu) ----

def lq_quantize(z: torch.Tensor, C: int, vals: torch.Tensor, meta: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """vqb_lq_quantize: z (N, C * D) fp32 / bf16 -> (codes (N, C * D) fp32, indices (N, C) int32).  vals: the D value tables
    concatenated, fp32; meta (3, D) int32: table lengths, half widths, basis; both on z's device."""
    z = float_input(z, "LatentQuantize")
    _require_cuda(vals, meta)
    N, CD = z.shape
    D = CD // C
    codes = torch.empty((N, CD), dtype=torch.float32, device=z.device)
    idx = torch.empty((N, C), dtype=torch.int32, device=z.device)
    if N == 0:
        return codes, idx
    with torch.cuda.device(z.device):
        check(lib.vqb_lq_quantize(_p(z), _dtype_code(z), N, C, D, _p(vals), vals.numel(), _p(meta), _p(codes), _p(idx),
                                  _stream()), "vqb_lq_quantize")
    _count(1)
    return codes, idx


def _lq_loss_operands(x, out, wc, wq):
    """The loss kernels' operands: x fp32 / bf16 and out fp32, contiguous, of one size; wc, wq one-element fp32 tensors; all on
    one CUDA device (TypeError / ValueError / RuntimeError otherwise)."""
    if x.dtype not in FLOAT_DTYPES or out.dtype != torch.float32 or wc.dtype != torch.float32 or wq.dtype != torch.float32:
        raise TypeError(f"vqb200 LatentQuantize loss takes fp32 / bf16 x and fp32 out and weights, got {x.dtype}, {out.dtype}, "
                        f"{wc.dtype}, {wq.dtype}")
    if x.numel() != out.numel() or wc.numel() != 1 or wq.numel() != 1 or not (x.is_contiguous() and out.is_contiguous()):
        raise ValueError("vqb200 LatentQuantize loss: x and out contiguous of one size, one-element weights")
    _require_cuda(x, out, wc, wq)
    if len({t.device for t in (x, out, wc, wq)}) != 1:
        raise RuntimeError("vqb200 LatentQuantize loss: operands on different devices")


def lq_loss(x: torch.Tensor, out: torch.Tensor, wc: torch.Tensor, wq: torch.Tensor, use_c: bool, use_q: bool) -> torch.Tensor:
    """vqb_lq_loss: w_c mse + w_q mse of x (fp32 / bf16) and out (fp32), contiguous and of the same shape, as an fp32 scalar; a
    term counts only when its host flag is set.  wc, wq: fp32 scalars on the device."""
    _lq_loss_operands(x, out, wc, wq)
    n = x.numel()
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        blocks = _queried(lib.vqb_lq_loss_blocks(n), "vqb_lq_loss_blocks")
        partial = torch.empty(blocks, dtype=torch.float64, device=x.device)
        check(lib.vqb_lq_loss(_p(x), _dtype_code(x), _p(out), n, _p(wc), _p(wq), int(use_c), int(use_q), _p(partial), blocks,
                              _p(loss), _stream()), "vqb_lq_loss")
    _count(2)
    return loss


def lq_loss_backward(x: torch.Tensor, out: torch.Tensor, g_loss: torch.Tensor, wc: torch.Tensor, wq: torch.Tensor, use_c: bool,
                     use_q: bool, want_gx: bool = True, want_gout: bool = True):
    """vqb_lq_loss_backward: (d x in x's dtype or None, d out fp32 or None) of lq_loss for dL/dloss g_loss (fp32 scalar on the
    device)."""
    _lq_loss_operands(x, out, wc, wq)
    _require_cuda(g_loss)
    gx = torch.empty_like(x) if want_gx else None
    gout = torch.empty_like(out) if want_gout else None
    g_loss = g_loss.float().contiguous()
    with torch.cuda.device(x.device):
        check(lib.vqb_lq_loss_backward(_p(x), _dtype_code(x), _p(out), x.numel(), _p(g_loss), _p(wc), _p(wq), int(use_c),
                                       int(use_q), _p(gx), _p(gout), _stream()), "vqb_lq_loss_backward")
    _count(1)
    return gx, gout
