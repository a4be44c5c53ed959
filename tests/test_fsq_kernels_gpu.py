"""The FSQ kernels (csrc/vq_fsq.cu: vqb_fsq_forward, vqb_fsq_backward, vqb_fsq_decode) called through their C entry points, against
the numpy restatement the FSQ suite trusts (oracle/fsq_oracle.py: float32 in the reference's order, rounding boundaries and the
gradient bound in float64), on every path they take:

(a) every template instantiation: d = 1..16 for each (input, chain) dtype pair (f32, f32), (bf16, f32), (bf16, bf16), with
    sym / non-sym, hard / tanh, soft clamp on / off and n_active < Q rotated over the 48 cases;
(b) more than one grid wave (the grid stops at 16 CTAs per SM): forward and decode once per dtype pair, the backward once per
    block size of its thread ladder, including n_active * d = 768 (its limit) and Q = 64;
(c) planted rounding boundaries: adjacent float32 inputs across which the oracle's stage code changes (exact ties included),
    clamp inputs of exactly +-1, +-0, subnormals, +-FLT_MAX and +-inf;
(d) the index layouts of the modules (ResidualFSQ (N, Q), GroupedResidualFSQ (G, N, Q) permuted, FSQ(num_codebooks=c) with a
    stage stride of 0) in int32 and int64, forward and decode;
(e) arguments the host refuses before any launch;
(f) ResidualFSQ and GroupedResidualFSQ past one grid wave, and inputs and upstream gradients at a 4-byte offset.

The acceptance rule is DESIGN.md §4.9: a row whose index differs from the oracle's must be near a rounding boundary, and the
hard-clamp paths without a soft clamp may not flip at all; outputs are bit-exact on every other row; gradients are exact where
the oracle's bound is 0 and inside it elsewhere.  Every output buffer carries guard rows (and the index tensors padded slots)
holding a sentinel that must survive."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import fsq_oracle as O
from fsq_golden import _key, _unkey, boundary_pairs, exact_ties, flipped_rows, stage_values

import vector_quantize_pytorch_b200 as vqb
from vector_quantize_pytorch_b200 import _C, ops
from vector_quantize_pytorch_b200._C import lib
from vector_quantize_pytorch_b200.fsq import fsq_tables

pytestmark = pytest.mark.gpu

DEV = "cuda"
F32, BF16 = torch.float32, torch.bfloat16
CODE = {F32: _C.DTYPE_F32, BF16: _C.DTYPE_BF16}
PAIRS = [(F32, F32), (BF16, F32), (BF16, BF16)]   # (input, chain): the pairs torch's promotion can produce
PAIR_ID = {(F32, F32): "f32", (BF16, F32): "bf16in", (BF16, BF16): "bf16"}
GUARD = 3                 # guard rows after row N of every output buffer
SENT_F = -12345.678       # sentinel of the float outputs
SENT_I = -7               # sentinel of the index slots outside the view
BWD_SMEM = 96 * 1024      # the backward's per-block budget for its parked stage gradients
E_INVALID, E_UNSUPPORTED, E_ALIGN = -1, -2, -3


def bwd_threads(n_active, d):
    """The backward's block size: 256, lowered in steps of 32 until threads * n_active * d * 4 B fits (vqb_fsq_backward)."""
    t = 256
    while t > 32 and t * n_active * d * 4 > BWD_SMEM:
        t -= 32
    return t if t * n_active * d * 4 <= BWD_SMEM else None


def wave(threads):
    """Items one full grid of `threads`-thread blocks covers in one pass (16 CTAs per SM)."""
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * threads


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Spec:
    """One kernel configuration: levels, stages, bound, scaling and dtypes, with the module's tables on the device."""

    def __init__(self, levels, Q, n_active, sym, hard, scaled, soft, in_dt=F32, work_dt=F32):
        assert scaled or not soft
        self.levels, self.d, self.Q, self.n_active = list(levels), len(levels), Q, n_active
        self.sym, self.hard, self.in_dt, self.work_dt = sym, hard, in_dt, work_dt
        self.w_bf16 = work_dt == BF16
        L = torch.tensor(self.levels)
        scales = torch.stack([L.float() ** -q for q in range(Q)]) if scaled else None
        clampv = (1 + 1 / (L - 1)).float() if soft else None
        if self.w_bf16:   # the buffers of a module moved to bf16
            scales = scales.bfloat16().float() if scales is not None else None
            clampv = clampv.bfloat16().float() if clampv is not None else None
        self.scales = scales.numpy() if scales is not None else None
        self.clampv = clampv.numpy() if clampv is not None else None
        consts, ints = fsq_tables(torch.tensor(self.levels, dtype=torch.int32),
                                  torch.cumprod(torch.tensor([1] + self.levels[:-1]), 0, dtype=torch.int32), sym, hard)
        self.consts, self.ints = consts.to(DEV), ints.to(DEV)
        self.sc_t = torch.stack([scales, 1 / scales]).contiguous().to(DEV) if scales is not None else None
        self.cl_t = torch.stack([clampv, 1 / clampv]).contiguous().to(DEV) if clampv is not None else None

    def label(self):
        return (f"d={self.d} L={self.levels} Q={self.Q} n_active={self.n_active} {'sym' if self.sym else 'nonsym'} "
                f"{'hard' if self.hard else 'tanh'}{' scaled' if self.scales is not None else ''}"
                f"{' soft' if self.clampv is not None else ''} {PAIR_ID[(self.in_dt, self.work_dt)]}")


def levels_for(rng, d, sym, hi):
    """d random levels in [2 (sym) or 3, hi], their product kept below 2^24 where the lower limit allows it."""
    lo = 2 if sym else 3
    levels = [int(v) for v in rng.integers(lo, hi + 1, size=d)]
    while np.prod(levels, dtype=np.float64) >= 2 ** 24 and max(levels) > lo:
        levels[int(np.argmax(levels))] -= 1
    return levels


def random_z(rng, N, G, d, in_dt):
    z = (rng.standard_normal((N, G, d)) * 1.3).astype(np.float32)
    return O.bf16_round(z) if in_dt == BF16 else z


def bits_equal(a, b):
    if a.dtype == BF16:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def guarded(shape, dt):
    return torch.full(shape, SENT_F, dtype=dt, device=DEV)


def assert_guard(buf, n, what):
    assert bits_equal(buf[n:], torch.full_like(buf[n:], SENT_F)), f"{what}: guard rows were written"


# ---- index layouts: (big sentinel-filled tensor shape, the (N, G, Q) view of it) ----

def _layout(layout, N, G, Q):
    if layout == "contig":      # (N, G, Q) with a padded stage axis
        return (N + GUARD, G, Q + 1), lambda t: t[:N, :, :Q]
    if layout == "rfsq":        # ResidualFSQ: (N, Q) viewed as (N, 1, Q)
        assert G == 1
        return (N + GUARD, Q + 2), lambda t: t[:N, :Q].unsqueeze(1)
    if layout == "grouped":     # GroupedResidualFSQ: (G, N, Q) permuted to (N, G, Q)
        return (G, N + GUARD, Q + 2), lambda t: t[:, :N, :Q].permute(1, 0, 2)
    if layout == "codebooks":   # FSQ(num_codebooks=G): (N, G) viewed as (N, G, 1), stage stride 0
        assert Q == 1
        return (N + GUARD, G + 1, 2), lambda t: t[:N, :G, :1]
    raise ValueError(layout)


def index_buffer(layout, N, G, Q, dtype):
    """A sentinel-filled index tensor, its (N, G, Q) view and the mask of the view's slots."""
    shape, view = _layout(layout, N, G, Q)
    big = torch.full(shape, SENT_I, dtype=dtype, device=DEV)
    mask = torch.zeros(shape, dtype=torch.bool, device=DEV)
    view(mask).fill_(True)
    return big, view(big), mask


# ---- the three entry points, with guarded outputs ----

def kernel_forward(s: Spec, zt, layout="contig", idx_dtype=torch.int64):
    N, G, d = zt.shape
    big, view, mask = index_buffer(layout, N, G, s.Q, idx_dtype)
    out = guarded((N + GUARD, G, d), s.work_dt)
    rc = lib.vqb_fsq_forward(zt.data_ptr(), CODE[zt.dtype], CODE[s.work_dt], N, G, d, s.Q, s.n_active, int(s.sym), int(s.hard),
                             s.consts.data_ptr(), _p(s.sc_t), _p(s.cl_t), out.data_ptr(), view.data_ptr(),
                             int(idx_dtype == torch.int64), *ops._fsq_strides(view), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(out, N, "forward out")
    assert (big[~mask] == SENT_I).all(), "forward wrote an index slot outside its view"
    return out[:N], view


def kernel_decode(s: Spec, view):
    N, G, Q = view.shape
    out = guarded((N + GUARD, G, s.d), s.work_dt)
    codes = guarded((Q * N * G + GUARD, s.d), s.work_dt)
    rc = lib.vqb_fsq_decode(view.data_ptr(), int(view.dtype == torch.int64), *ops._fsq_strides(view), N, G, s.d, Q,
                            CODE[s.work_dt], int(s.sym), s.consts.data_ptr(), s.ints.data_ptr(), _p(s.sc_t), out.data_ptr(),
                            codes.data_ptr(), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(out, N, "decode out")
    assert_guard(codes, Q * N * G, "decode codes")
    return out[:N], codes[:Q * N * G].view(Q, N, G, s.d)


def kernel_backward(s: Spec, zt, g):
    N, G, d = zt.shape
    gz = guarded((N + GUARD, G, d), zt.dtype)
    rc = lib.vqb_fsq_backward(zt.data_ptr(), CODE[zt.dtype], CODE[s.work_dt], N, G, d, s.Q, s.n_active, int(s.sym), int(s.hard),
                              s.consts.data_ptr(), _p(s.sc_t), _p(s.cl_t), g.data_ptr(), gz.data_ptr(), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(gz, N, "backward grad_z")
    return gz[:N]


def check_kernels(s: Spec, z, label, layout="contig", idx_dtype=torch.int64, seed=0):
    """Forward, decode (from the forward's own index view) and backward of z (N, G, d) against the oracle."""
    N, G, d = z.shape
    zt = torch.from_numpy(z).to(s.in_dt).to(DEV)
    out, view = kernel_forward(s, zt, layout, idx_dtype)
    idx = view.cpu().numpy().astype(np.int64)
    fwd = O.forward(z, s.levels, s.Q, s.n_active, s.sym, s.hard, s.scales, s.clampv, s.w_bf16)
    rows, excused = flipped_rows(idx, fwd["idx"], fwd["near"])
    print(f"{label} [{s.label()}] N={N} G={G}: {int(rows.sum())} flipped rows of {rows.size}, "
          f"{int(excused.sum())} near a rounding boundary")
    assert (rows == excused).all(), "index differs away from any rounding boundary"
    if s.hard and s.clampv is None:
        assert not rows.any(), "the hard-clamp path without a soft clamp must match bit for bit"
    np.testing.assert_array_equal(out.float().cpu().numpy()[~rows], fwd["out"][~rows])
    assert (idx[..., s.n_active:] == -1).all()

    dsum, dcodes = kernel_decode(s, view)
    osum, ocodes = O.decode(idx, s.levels, s.sym, s.scales, s.w_bf16)
    np.testing.assert_array_equal(dsum.float().cpu().numpy(), osum)
    np.testing.assert_array_equal(dcodes.float().cpu().numpy(), ocodes)

    g = torch.randn((N, G, d), generator=torch.Generator().manual_seed(seed)).to(s.work_dt)
    gz = kernel_backward(s, zt, g.to(DEV))
    dz, bound = O.backward(z, g.float().numpy(), s.levels, s.Q, s.n_active, s.sym, s.hard, s.scales, s.clampv, s.w_bf16,
                           s.in_dt == BF16)
    err = np.abs(gz.float().cpu().numpy().astype(np.float64) - dz)[~rows]
    b = bound[~rows]
    assert (err[b == 0] == 0).all(), "a gradient made of exact factors must match bit for bit"
    ratio = float((err[b > 0] / b[b > 0]).max()) if (b > 0).any() else 0.0
    print(f"{label}: gradient elements exact {int((b == 0).sum())}, largest error / bound on the rest {ratio:.3g}")
    assert (err <= b).all()
    return rows


# ---- (a) every instantiation ----

def _matrix():
    cases = []
    for p, (in_dt, work_dt) in enumerate(PAIRS):
        order = np.random.default_rng(100 + p).permutation(16)   # each (sym, hard, soft, n_active < Q) once per pair
        for d in range(1, 17):
            k = int(order[d - 1])
            cases.append((in_dt, work_dt, d, k % 2 == 0, (k // 2) % 2 == 0, (k // 4) % 2 == 1, (k // 8) % 2 == 1))
    return cases


MATRIX = _matrix()


@pytest.mark.parametrize("case", MATRIX, ids=[f"{PAIR_ID[(c[0], c[1])]}_d{c[2]}" for c in MATRIX])
def test_instantiation(case):
    in_dt, work_dt, d, sym, hard, soft, partial = case
    rng = np.random.default_rng(1000 + d + 17 * PAIRS.index((in_dt, work_dt)))
    if partial:
        Q, n_active = 4, 2
    else:
        Q = n_active = 3 if soft else 1 + d % 3
    scaled = soft or Q > 1 or d % 4 == 0   # Q = 1 without scales is a plain FSQ
    s = Spec(levels_for(rng, d, sym, 9), Q, n_active, sym, hard, scaled, soft, in_dt, work_dt)
    G = 3 if d % 2 else 1
    N = 97 + 13 * d
    check_kernels(s, random_z(rng, N, G, d, in_dt), f"instantiation {PAIR_ID[(in_dt, work_dt)]} d={d}",
                  idx_dtype=torch.int32 if d % 3 == 0 else torch.int64, seed=d)


# ---- (b) more than one grid wave ----

WAVE_CASES = [   # (input, chain, d, G, Q, n_active, sym, hard, soft)
    (F32, F32, 5, 3, 3, 3, True, True, False),
    (BF16, F32, 7, 1, 4, 3, False, False, False),
    (BF16, BF16, 6, 1, 5, 5, True, True, True),
]


@pytest.mark.parametrize("case", WAVE_CASES, ids=[PAIR_ID[(c[0], c[1])] for c in WAVE_CASES])
def test_forward_decode_past_one_wave(case):
    """items = one full forward / decode grid (256 threads) + a ragged remainder: some threads loop twice, some once."""
    in_dt, work_dt, d, G, Q, n_active, sym, hard, soft = case
    rng = np.random.default_rng(d)
    s = Spec(levels_for(rng, d, sym, 8), Q, n_active, sym, hard, True, soft, in_dt, work_dt)
    N = (wave(256) + 101) // G + 1
    assert wave(256) < N * G < 2 * wave(256)
    check_kernels(s, random_z(rng, N, G, d, in_dt), f"wave {PAIR_ID[(in_dt, work_dt)]}", seed=d)


RUNGS = [   # (threads, d, Q, n_active, sym, hard, soft, input, chain): every block size of the backward's ladder
    (256, 16, 6, 6, True, True, False, F32, F32),
    (224, 10, 10, 10, False, True, False, BF16, F32),
    (192, 16, 9, 7, True, False, True, BF16, BF16),
    (160, 12, 12, 12, True, True, True, F32, F32),
    (128, 16, 12, 12, False, False, False, F32, F32),
    (96, 16, 16, 16, True, True, False, BF16, BF16),
    (64, 16, 30, 24, True, True, False, BF16, F32),
    (32, 12, 64, 64, True, True, False, F32, F32),   # n_active * d = 768, the limit; Q = 64, the most stages
]


@pytest.mark.parametrize("case", RUNGS, ids=[f"t{c[0]}" for c in RUNGS])
def test_backward_rung_past_one_wave(case):
    """items = one full backward grid at the block size the case lands on + a ragged remainder; forward and decode run on
    the same data.  Levels stay <= 4 (<= 3 past 32 stages) so that every stage scale L^-q is a normal float and the stage
    gradients A_q = (...) / scale_q stay finite."""
    threads, d, Q, n_active, sym, hard, soft, in_dt, work_dt = case
    assert bwd_threads(n_active, d) == threads
    rng = np.random.default_rng(threads)
    s = Spec(levels_for(rng, d, sym, 3 if Q > 32 else 4), Q, n_active, sym, hard, True, soft, in_dt, work_dt)
    N = wave(threads) + 37
    check_kernels(s, random_z(rng, N, 1, d, in_dt), f"rung {threads}", seed=threads)


# ---- (c) planted boundaries ----

PLANT_LEVELS = {True: [2, 3, 4, 5], False: [3, 4, 5, 8]}
FLT_MAX = float(np.finfo(np.float32).max)
SPECIAL = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-39, -3e-39, FLT_MAX, -FLT_MAX, np.inf, -np.inf], np.float32)


def clamp_edges(shift):
    """Around each of -1 and +1: the outermost input z whose clamp input z + shift (float32) is still inside [-1, 1], and the
    next float beyond it.  Returns them and how many of the inside ones are exactly -1 or +1 (always both when shift = 0)."""
    out, exact = [], 0
    for p in (np.float32(-1), np.float32(1)):
        cand = _unkey(_key(np.float32(p - shift)) + np.arange(-8, 9))
        pre = (cand + shift).astype(np.float32)
        inside = cand[pre >= -1].min() if p < 0 else cand[pre <= 1].max()
        exact += int(np.float32(inside + shift) == p)
        out += [inside, np.nextafter(inside, np.float32(2 * p))]
    return np.array(out, np.float32), exact


@pytest.mark.parametrize("variant", ["plain", "scaled", "soft"])
@pytest.mark.parametrize("hard", [True, False], ids=["hard", "tanh"])
@pytest.mark.parametrize("sym", [True, False], ids=["sym", "nonsym"])
def test_planted_boundaries(sym, hard, variant):
    """Both sides of every adjacent float32 pair across which the oracle's stage-0 (and last-stage) code of an element
    changes, planted one value per row.  The hard paths without a soft clamp must agree bit for bit on both sides, gradients
    included: among the pairs are pre-round values of exactly k + 1/2 (rintf and roundf round some of those apart) and
    pre-floor values of exactly an integer.  Clamp inputs of exactly +-1 pin the closed interval of the backward's mask.
    NaN is left out: the reference's .round().to(int32) of NaN is undefined, so there is no index to compare with."""
    levels = PLANT_LEVELS[sym]
    d = len(levels)
    Q = 1 if variant == "plain" else 3
    s = Spec(levels, Q, Q, sym, hard, variant != "plain", variant == "soft")
    t = O.tables(levels, sym, hard)
    rng = np.random.default_rng(7)
    planted, ties, apart = [], 0, 0
    for q in sorted({0, Q - 1}):
        for j in range(d):
            a, b = boundary_pairs(levels, Q, q, j, sym, hard, s.scales, s.clampv)
            for v in (a, b):
                _, br, _ = stage_values(v, j, levels, Q, q, sym, hard, s.scales, s.clampv)
                tie = exact_ties(br, sym)
                ties += int(tie.sum())
                if not sym:   # ties that round half to even and half away from zero put in different codes
                    k = br[tie].astype(np.float64)
                    apart += int((np.rint(k) != np.sign(k) * np.floor(np.abs(k) + 0.5)).sum())
                planted += [(j, x) for x in v]
    edges = 0
    for j in range(d):
        zs, exact = clamp_edges(t["shift"][j])
        edges += exact
        planted += [(j, x) for x in zs]
        planted += [(j, x) for x in SPECIAL]
    z = random_z(rng, len(planted), 1, d, F32)
    for r, (j, x) in enumerate(planted):
        z[r, 0, j] = x
    print(f"planted {len(planted)} values, {ties} exact ties ({apart} that rintf and roundf round apart), "
          f"{edges} clamp inputs of exactly -1 or +1")
    assert edges >= 2
    if hard:
        assert ties > 0, "no exact tie was planted"
        if not sym:
            assert apart > 0, "no tie that rounding half away from zero would move"
    with np.errstate(over="ignore", invalid="ignore"):
        check_kernels(s, z, f"planted {variant}")


# ---- (d) index layouts ----

LAYOUTS = [   # (layout, G, Q, n_active, sym, hard, scaled, soft)
    ("rfsq", 1, 5, 3, True, True, True, True),
    ("grouped", 3, 4, 4, True, True, True, False),
    ("codebooks", 3, 1, 1, False, False, False, False),
]


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("case", LAYOUTS, ids=[c[0] for c in LAYOUTS])
def test_index_layouts(case, idx_dtype):
    """Forward into, and decode from, the modules' strided index views inside a larger sentinel-filled tensor: a wrong
    stride writes a slot outside the view (or reads a sentinel)."""
    layout, G, Q, n_active, sym, hard, scaled, soft = case
    rng = np.random.default_rng(G * 10 + Q)
    s = Spec(levels_for(rng, 5, sym, 7), Q, n_active, sym, hard, scaled, soft)
    check_kernels(s, random_z(rng, 1001, G, 5, F32), f"layout {layout}", layout, idx_dtype)


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("layout", ["contig", "rfsq", "grouped"])
def test_decode_dropped_stages(layout, idx_dtype):
    """Decode of random indices with -1 (a dropped stage) anywhere, through a strided view, in both chain dtypes."""
    G = 1 if layout == "rfsq" else 2
    Q, N = 6, 777
    rng = np.random.default_rng(3)
    for work_dt in (F32, BF16):
        s = Spec(levels_for(rng, 4, True, 5), Q, Q, True, True, True, False, BF16 if work_dt == BF16 else F32, work_dt)
        idx = rng.integers(0, int(np.prod(s.levels)), size=(N, G, Q))
        idx[rng.random((N, G, Q)) < 0.3] = -1
        big, view, mask = index_buffer(layout, N, G, Q, idx_dtype)
        view.copy_(torch.from_numpy(idx))
        dsum, dcodes = kernel_decode(s, view)
        assert (big[~mask] == SENT_I).all()
        osum, ocodes = O.decode(idx, s.levels, True, s.scales, s.w_bf16)
        np.testing.assert_array_equal(dsum.float().cpu().numpy(), osum)
        np.testing.assert_array_equal(dcodes.float().cpu().numpy(), ocodes)


# ---- (e) limits the host refuses before any launch ----

def test_limits_are_refused_before_launch():
    N, G = 64, 1
    z = torch.randn((N + 1) * 17 * 2, device=DEV)   # room for d = 17 and an offset view
    buf = lambda: guarded((N * 17 * 65 + 64,), F32)   # noqa: E731
    idx = torch.full((N * 65 + 8,), SENT_I, dtype=torch.int64, device=DEV)
    big_sc = torch.ones((2, 65, 17), device=DEV)
    consts = torch.ones((7, 17), device=DEV)
    ints = torch.ones((2, 17), dtype=torch.int32, device=DEV)

    def fwd(zp, in_dt, w_dt, D, Q, n_active, out, sc=big_sc):
        return lib.vqb_fsq_forward(zp, in_dt, w_dt, N, G, D, Q, n_active, 1, 1, consts.data_ptr(), sc.data_ptr(), None,
                                   out, idx.data_ptr(), 1, Q, 0, 1, _stream())

    def bwd(zp, in_dt, w_dt, D, Q, n_active, gout, gz):
        return lib.vqb_fsq_backward(zp, in_dt, w_dt, N, G, D, Q, n_active, 1, 1, consts.data_ptr(), big_sc.data_ptr(), None,
                                    gout, gz, _stream())

    def dec(D, Q, w_dt, out, codes):
        return lib.vqb_fsq_decode(idx.data_ptr(), 1, Q, 0, 1, N, G, D, Q, w_dt, 1, consts.data_ptr(), ints.data_ptr(),
                                  big_sc.data_ptr(), out, codes, _stream())

    out, gz, gout, codes = buf(), buf(), buf(), buf()
    zp, f, b = z.data_ptr(), _C.DTYPE_F32, _C.DTYPE_BF16
    assert fwd(zp, f, f, 3, 65, 65, out.data_ptr()) == E_UNSUPPORTED
    assert fwd(zp, f, f, 17, 2, 2, out.data_ptr()) == E_UNSUPPORTED
    assert fwd(zp, f, f, 3, 2, 0, out.data_ptr()) == E_INVALID
    assert fwd(zp, f, f, 3, 2, 3, out.data_ptr()) == E_INVALID
    assert fwd(zp, f, b, 3, 2, 2, out.data_ptr()) == E_UNSUPPORTED
    assert fwd(zp + 4, f, f, 3, 2, 2, out.data_ptr()) == E_ALIGN
    assert fwd(zp, f, f, 3, 2, 2, out.data_ptr() + 4) == E_ALIGN
    assert bwd(zp, f, f, 3, 65, 65, gout.data_ptr(), gz.data_ptr()) == E_UNSUPPORTED
    assert bwd(zp, f, f, 17, 2, 2, gout.data_ptr(), gz.data_ptr()) == E_UNSUPPORTED
    assert bwd(zp, f, f, 3, 2, 0, gout.data_ptr(), gz.data_ptr()) == E_INVALID
    assert bwd(zp, f, f, 3, 2, 3, gout.data_ptr(), gz.data_ptr()) == E_INVALID
    assert bwd(zp, f, b, 3, 2, 2, gout.data_ptr(), gz.data_ptr()) == E_UNSUPPORTED
    assert bwd(zp + 4, f, f, 3, 2, 2, gout.data_ptr(), gz.data_ptr()) == E_ALIGN
    assert bwd(zp, f, f, 3, 2, 2, gout.data_ptr() + 4, gz.data_ptr()) == E_ALIGN
    assert bwd(zp, f, f, 3, 2, 2, gout.data_ptr(), gz.data_ptr() + 4) == E_ALIGN
    assert bwd_threads(60, 13) is None
    assert bwd(zp, f, f, 13, 60, 60, gout.data_ptr(), gz.data_ptr()) == E_UNSUPPORTED   # n_active * d = 780 > 768
    assert dec(3, 65, f, out.data_ptr(), codes.data_ptr()) == E_UNSUPPORTED
    assert dec(17, 2, f, out.data_ptr(), codes.data_ptr()) == E_UNSUPPORTED
    assert dec(3, 2, f, out.data_ptr() + 4, None) == E_ALIGN
    assert dec(3, 2, f, None, codes.data_ptr() + 4) == E_ALIGN
    torch.cuda.synchronize()
    for t in (out, gz, codes):
        assert bits_equal(t, torch.full_like(t, SENT_F)), "a refused call wrote its output"
    assert (idx == SENT_I).all(), "a refused call wrote indices"


# ---- (f) the modules at size, and offset inputs and gradients ----

class _Fixed(nn.Module):
    """Stands in for project_in: returns the module's own project_in output as a leaf, so its gradient can be read."""

    def __init__(self, z):
        super().__init__()
        self.z = z

    def forward(self, x):
        return self.z


class _Capture(nn.Module):
    """Stands in for project_out: keeps its input (the quantizer's output) and passes it on."""

    def __init__(self, sink):
        super().__init__()
        self.sink = sink

    def forward(self, q):
        self.sink.append(q)
        return q


@pytest.mark.parametrize("train", [True, False], ids=["train_dropout", "eval"])
@pytest.mark.parametrize("grouped", [False, True], ids=["rfsq", "grfsq"])
def test_module_past_one_wave(grouped, train):
    """ResidualFSQ (hard clamp, so a soft clamp) and GroupedResidualFSQ (G = 4, tanh) with projections, past one grid wave:
    against the oracle on their own project_in output; quantize dropout gives int64 indices with -1 stages;
    get_output_from_indices and the stage-order sum of return_all_codes equal the forward."""
    torch.manual_seed(0)
    levels, Q = ([4, 4, 3, 2], 6) if not grouped else ([4, 3, 3], 5)
    d = len(levels)
    if grouped:
        G = 4
        m = vqb.GroupedResidualFSQ(dim=G * (d + 1), groups=G, levels=levels, num_quantizers=Q, quantize_dropout=True,
                                   bound_hard_clamp=False)
        parts = list(m.rvqs)
    else:
        G = 1
        m = vqb.ResidualFSQ(dim=d + 4, levels=levels, num_quantizers=Q, quantize_dropout=True)
        parts = [m]
    m = m.to(DEV).train(train)
    N = wave(256) // G + 333
    x = torch.randn(1, N, m.dim if grouped else d + 4, device=DEV)
    chunks = x.chunk(G, dim=-1)
    sink, leaves = [], []
    for p, c in zip(parts, chunks):
        z = p.project_in(c).detach().requires_grad_(True)
        leaves.append(z)
        p.project_in = _Fixed(z)
        p.project_out = _Capture(sink)
    kw = {}
    if train:   # a dropout cut below Q: n_active < Q and int64 indices
        from vector_quantize_pytorch_b200.residual_fsq import get_maybe_sync_seed
        for seed in range(100):
            torch.manual_seed(seed)
            cut = parts[0]._n_active(get_maybe_sync_seed(DEV) if grouped else seed, DEV)[0]
            if cut < Q:
                break
        torch.manual_seed(seed)
        if not grouped:
            kw = dict(rand_quantize_dropout_fixed_seed=seed)
    res = m(x, return_all_codes=True, **kw)
    quantized, ind = res[0], res[1]
    sink = list(sink)   # the forward's outputs (decoding below passes through project_out as well)
    assert ind.dtype == (torch.int64 if train else torch.int32)
    idx = (ind.permute(1, 2, 0, 3).reshape(N, G, Q) if grouped else ind.reshape(N, 1, Q)).cpu().numpy().astype(np.int64)
    n_active = int((idx != -1).reshape(-1, Q).all(axis=0).sum())
    assert (idx[..., n_active:] == -1).all() and (n_active < Q) == train

    z_np = np.stack([z.detach().reshape(N, d).cpu().numpy() for z in leaves], axis=1)
    scales, clampv = parts[0]._make_scale_tables()
    hard = parts[0].layers[0].bound_hard_clamp
    cl = clampv[0].numpy() if clampv is not None else None
    fwd = O.forward(z_np, levels, Q, n_active, True, hard, scales[0].numpy(), cl)
    rows, excused = flipped_rows(idx, fwd["idx"], fwd["near"])
    print(f"{'grfsq' if grouped else 'rfsq'} {'train' if train else 'eval'} N={N} G={G} n_active={n_active}: "
          f"{int(rows.sum())} flipped rows of {rows.size}, {int(excused.sum())} near a rounding boundary")
    assert (rows == excused).all()
    out = torch.stack([q.detach().reshape(N, d) for q in sink], dim=1)
    np.testing.assert_array_equal(out.cpu().numpy()[~rows], fwd["out"][~rows])

    assert torch.equal(m.get_output_from_indices(ind), quantized.detach())
    codes = torch.stack(res[2]) if grouped else res[2][None]   # (G, Q, 1, N, d)
    acc = codes[:, 0]
    for q in range(1, Q):   # fp32, in stage order, as the forward's running sum
        acc = acc + codes[:, q]
    assert torch.equal(acc.reshape(G, N, d).permute(1, 0, 2), out)

    g = [torch.randn_like(q) for q in sink]
    grads = torch.autograd.grad(sink, leaves, g)
    gz = np.stack([t.reshape(N, d).cpu().numpy() for t in grads], axis=1)
    g_np = np.stack([t.reshape(N, d).cpu().numpy() for t in g], axis=1)
    dz, bound = O.backward(z_np, g_np, levels, Q, n_active, True, hard, scales[0].numpy(), cl)
    err = np.abs(gz.astype(np.float64) - dz)[~rows]
    b = bound[~rows]
    assert (err[b == 0] == 0).all()
    assert (err <= b).all()


def _unprojected(kind):
    if kind == "rfsq":
        return vqb.ResidualFSQ(levels=[4, 4, 3, 2], num_quantizers=4).to(DEV), (2, 700, 4)
    return vqb.FSQ([8, 5, 5, 3]).to(DEV), (2, 700, 4)


def _offset_view(shape):
    """A contiguous fp32 tensor 4 bytes past a 16-byte boundary (a view into a larger buffer)."""
    n = int(np.prod(shape))
    big = torch.randn(n + 8, device=DEV)
    v = big.view(-1)[1:1 + n].view(shape)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


@pytest.mark.parametrize("kind", ["rfsq", "fsq"])
def test_offset_input_matches_aligned_copy(kind):
    m, shape = _unprojected(kind)
    x = _offset_view(shape)
    xo = x.detach().requires_grad_(True)
    xa = x.detach().clone().requires_grad_(True)
    assert xo.data_ptr() % 16 == 4 and xa.data_ptr() % 16 == 0
    oo, io = m(xo)
    oa, ia = m(xa)
    assert bits_equal(oo, oa) and torch.equal(io, ia)
    g = torch.randn_like(oa)
    assert bits_equal(torch.autograd.grad(oo, xo, g)[0], torch.autograd.grad(oa, xa, g)[0])


@pytest.mark.parametrize("kind", ["rfsq", "fsq"])
def test_offset_upstream_gradient(kind):
    """An upstream gradient that is a contiguous view 4 bytes past a 16-byte boundary.  ops.fsq_backward used to hand it to
    vqb_fsq_backward as it was, which refused it (VQB_E_ALIGN) and raised; it now copies it to an aligned buffer."""
    m, shape = _unprojected(kind)
    x = torch.randn(shape, device=DEV, requires_grad=True)
    out, _ = m(x)
    g = _offset_view(out.shape)
    go = torch.autograd.grad(out, x, g, retain_graph=True)[0]
    ga = torch.autograd.grad(out, x, g.clone())[0]
    assert bits_equal(go, ga)
