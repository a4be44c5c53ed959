"""Search indices bit for bit against the reference's fp32 distance formula, near ties included (run on an H100: `pytest -m gpu`).

The search certifies a row when its best tensor-core score leads every other by more than the band W, and re-scores every
other row with the reference's formula (vqb_fix_flagged: pair / triple re-score, whole-row rescan with its 64-bit arg-max
key).  The other GPU tests excuse near ties, because the reference sums in an order nobody can reproduce.  Here the oracle
is the formula the re-score evaluates, with exactly rounded sums, so no row is excused:

    score(k) = -sqrt_rn(max(fl(fl(x2f + cnorm2[k]) + fl(-2 * xyf)), 1e-8))    (Euclidean)
    score(k) = xyf                                                            (cosine)

xyf, x2f and cnorm2 are exact sums rounded once to fp32, and the winner is the first maximal index (vqp:58-62, :140).  The
kernel sums its dots in float64 in its own order, so a row may differ only where an involved sum lies within that sum's
error bound of an fp32 rounding midpoint and the kernel's index wins under one of the admissible roundings; such rows are
counted apart (expected 0).  Any other differing row fails.

The data drives every path: a ladder of exact score gaps t * W across the certify / flag boundary, the reference's sqrt
collapse at large norms, its 1e-8 clamp floor on small-norm codebooks and zero rows, tie groups across the 128-code chunks
of the whole-row rescan at K = 16384, negative cosine scores, and the default-init codebook at a BASELINE shape.
"""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import vq_oracle as O
from test_band_model import kernel_band
from test_search_plans_gpu import assert_loss_sum, bits, mse_sum

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}
F32 = np.float32
CLAMP = F32(1e-8)


# ------------------------------------------------------------------------------------------------------------------------
# exact oracle
# ------------------------------------------------------------------------------------------------------------------------

def r32(parts):
    """Sum of exact float64 terms rounded once to fp32 (nearest, ties to even).  fsum rounds the exact sum to float64; that
    second rounding only matters when it lands on an fp32 midpoint, and then the sign of the exact remainder decides."""
    m = math.fsum(parts)
    f = F32(m)
    if float(f) != m and np.isfinite(f):
        g = np.nextafter(f, F32(np.inf) if m > float(f) else F32(-np.inf))
        if m == (float(f) + float(g)) / 2:
            r = math.fsum(list(parts) + [-m])
            if r != 0:
                f = max(f, g) if r > 0 else min(f, g)
    return f


def r32_admissible(parts):
    """fp32 values a float64 sum of `parts` in any order may round to: the exact sum moved by the bound of such a sum,
    (n - 1) 2^-53 sum |p|, in either direction."""
    b = (len(parts) - 1) * 2.0 ** -53 * math.fsum(abs(p) for p in parts)
    return sorted({r32(list(parts) + [-b]), r32(parts), r32(list(parts) + [b])})


def formula(x2f, cn2f, xyf, cosine):
    """The reference's fp32 score from the three rounded sums: fp32 adds and product, sqrt in float64 rounded to fp32
    (correctly rounded: float64 has more than twice fp32's precision)."""
    if cosine:
        return F32(xyf)
    d2 = (F32(x2f) + F32(cn2f)) + F32(-2.0) * F32(xyf)
    return -F32(np.sqrt(np.float64(max(d2, CLAMP))))


def first_max(scores):
    best, bk = None, -1
    for k, s in scores:
        if best is None or s > best:
            best, bk = s, k
    return bk


def check_cnorm2(c, cnorm2):
    """cnorm2 of the operands (what the re-score trusts) against the exactly rounded ||c||^2.  Returns the exact values."""
    c64 = c.double()
    s = (c64 * c64).sum(-1)
    bound = c.shape[1] * 2.0 ** -52 * s          # float64 sum on the device, any order
    exact = s.float()
    unsure = ((s - bound).float() != (s + bound).float()).nonzero()[:, 0].tolist()
    got = cnorm2.cpu().numpy()
    ex = exact.cpu().numpy().copy()
    cn = c.cpu().double().numpy()
    bad = []
    for k in unsure:
        parts = (cn[k] * cn[k]).tolist()
        ex[k] = r32(parts)
        if got[k] not in r32_admissible(parts):
            bad.append(k)
    sure = np.ones(len(ex), bool)
    sure[unsure] = False
    bad += np.nonzero(sure & (got != ex))[0].tolist()
    assert not bad, f"cnorm2 differs from the exactly rounded ||c||^2 at codes {bad[:8]}: {got[bad[:8]]} vs {ex[bad[:8]]}"
    return ex


def candidates(xe, c, cn2, cosine):
    """Per row, every code whose fp32 score may equal the row's maximum: float64 GEMM on the device, the fp32 formula's
    rounding errors bounded by 2^-21 of the magnitudes that enter it, widened by an fp32 ulp of the score so that values
    the final rounding merges are kept together.  Returns (first, count, {row: sorted candidate list} for count > 1)."""
    N, D = xe.shape
    K = c.shape[0]
    x64, c64 = xe.double(), c.double()
    cn2d = torch.from_numpy(np.asarray(cn2, np.float64)).to(DEV)
    floor = float(CLAMP)
    first, count, lists = [], [], {}
    step = max(1, (1 << 24) // K)
    for i in range(0, N, step):
        g = x64[i:i + step] @ c64.T
        if cosine:
            tol = 2.0 ** -21 * g.abs() + 1e-300
            lo, hi = g - tol, g + tol
        else:
            x2 = (x64[i:i + step] ** 2).sum(-1)[:, None]
            d2 = x2 + cn2d[None] - 2.0 * g
            tol = 2.0 ** -21 * (x2 + cn2d[None] + 2.0 * g.abs() + d2.abs())
            lo = -(d2 + tol).clamp_min(floor).sqrt()
            hi = -(d2 - tol).clamp_min(floor).sqrt()
        lo = lo - 2.0 ** -22 * lo.abs()
        hi = hi + 2.0 ** -22 * hi.abs()
        m = lo.max(-1, keepdim=True).values
        cand = hi >= m
        n = cand.sum(-1)
        first.append(lo.argmax(-1))
        count.append(n)
        for r in (n > 1).nonzero()[:, 0].tolist():
            lists[i + r] = cand[r].nonzero()[:, 0].tolist()
    return torch.cat(first).cpu().numpy(), torch.cat(count).cpu().numpy(), lists


class Oracle:
    """The reference formula with exactly rounded sums over rows xe (as searched) and codebook c."""

    def __init__(self, xe, c, cnorm2, cosine):
        self.cosine = cosine
        self.cn2 = check_cnorm2(c, cnorm2)
        self.first, self.count, self.lists = candidates(xe, c, self.cn2, cosine)
        self.x = xe.double().cpu().numpy()
        self.c = c.double().cpu().numpy()
        self.idx = self.first.astype(np.int64)
        for row, ks in self.lists.items():   # rows resolved by exact recomputation
            xr = self.x[row]
            x2 = r32((xr * xr).tolist())
            self.idx[row] = first_max([(k, formula(x2, self.cn2[k], r32((xr * self.c[k]).tolist()), cosine)) for k in ks])

    def admissible_winners(self, row):
        """Winners under every rounding a float64 sum in another order may give (the kernel's warp_sum)."""
        ks = self.lists.get(row, [int(self.first[row])])
        xr = self.x[row]
        x2s = r32_admissible((xr * xr).tolist()) if not self.cosine else [F32(0)]
        xys = [r32_admissible((xr * self.c[k]).tolist()) for k in ks]
        win = set()
        for x2 in x2s:
            for combo in itertools.islice(itertools.product(*xys), 4096):
                win.add(first_max([(k, formula(x2, self.cn2[k], xy, self.cosine)) for k, xy in zip(ks, combo)]))
        return win


def band(xe, cb, dt, cosine):
    """W of every row (test_band_model.kernel_band) from the operands' cmax and the row norms."""
    cm = cb.cmax.cpu().double().numpy()
    x = xe.cpu().numpy()
    x64 = x.astype(np.float64)
    x2 = (x64 * x64).sum(-1)
    if dt == "fp32":
        xlo = x64 - O.bf16_round(x).astype(np.float64)
        xlo_norm = np.sqrt((xlo * xlo).sum(-1))
        caux = float.fromhex("0x1.02p-8") * cm[0] + cm[2]
    else:
        xlo_norm, caux = np.zeros_like(x2), 0.0
    return kernel_band(x2, xlo_norm, cm[0], cm[1], caux, not cosine)


def exact_scores(o, row, ks):
    """The kernel's score x.c - ||c||^2 / 2 (x.c for cosine) in float64."""
    xr = o.x[row]
    return [float(xr @ o.c[k]) - (0.0 if o.cosine else 0.5 * float(o.c[k] @ o.c[k])) for k in ks]


def check_indices(got, o, what, flagged=None, W=None):
    """Indices against the oracle: equal, or attributable to the kernel's summation order.  Returns the attributed count."""
    got = np.asarray(got, np.int64)
    diff = np.nonzero(got != o.idx)[0]
    order, bad = 0, []
    for row in diff.tolist():
        if int(got[row]) in o.admissible_winners(row):
            order += 1
            print(f"{what}: row {row} -> {int(got[row])} (oracle {int(o.idx[row])}) within the float64 summation bound")
            continue
        sg, so = exact_scores(o, row, [int(got[row]), int(o.idx[row])])
        info = f"row {row}: kernel {int(got[row])}, oracle {int(o.idx[row])}"
        if W is not None:
            info += f", gap (oracle - kernel) {(so - sg) / W[row]:.3g} W"
        if flagged is not None:
            info += f", flag entry {flagged.get(row)}"
        bad.append(info)
    assert not bad, f"{what}: {len(bad)} rows differ from the exact formula: " + "; ".join(bad[:6])
    return order


def check_flags(res, N, K, idx):
    """The flag list: counts 2-3 at the front, > 3 at the back, no row twice, candidates in range, and every flagged row
    ended on one of its candidates (front) or on the index its rescan key encodes (back).  Returns {row: entry}."""
    nf, nb = res.flag_count.item(), res.rescan_count.item()
    assert 0 <= nf and 0 <= nb and nf + nb <= N
    fl = res.flagged.cpu().numpy()
    front, back = fl[:nf], fl[N - nb:]
    rows = np.concatenate([front[:, 0], back[:, 0]])
    assert len(np.unique(rows)) == len(rows) and ((rows >= 0) & (rows < N)).all()
    assert ((front[:, 1] >= 2) & (front[:, 1] <= 3)).all(), "front entries must have 2 or 3 candidates"
    assert (back[:, 1] > 3).all(), "back entries must have more than 3 candidates"
    for e in front:
        cs = e[2:2 + e[1]]
        assert len(set(cs.tolist())) == e[1] and ((cs >= 0) & (cs < K)).all(), e
        assert idx[e[0]] in cs, (e, idx[e[0]])
    for e in back:
        k = 0xFFFFFFFF - (int(e[2]) & 0xFFFFFFFF)
        assert k == idx[e[0]], (e, k, idx[e[0]])
    out = {int(e[0]): ("pair/triple", e[2:2 + e[1]].tolist()) for e in front}
    out.update({int(e[0]): ("rescan", int(e[1])) for e in back})
    return out, nf, nb


def run_case(x, c, dt, cosine, what):
    """Search x (N, D) against c (K, D): indices vs the oracle, flag list, and the fused copy / residual tails of every row
    (the re-scored ones included) against torch arithmetic on the oracle's indices."""
    from vector_quantize_pytorch_b200 import ops
    N, D = x.shape
    K = c.shape[0]
    x = x.to(TDT[dt]).to(DEV).contiguous()
    c = c.to(DEV).contiguous()
    cb = ops.prepare_codebook(c, cosine)
    res = ops.search(x, cb, c)
    torch.cuda.synchronize()
    xe = res.x_eff.float()
    o = Oracle(xe, c, cb.cnorm2, cosine)
    W = band(xe, cb, dt, cosine)
    idx = res.idx.cpu().numpy().astype(np.int64)
    flags, nf, nb = check_flags(res, N, K, idx)
    order = check_indices(idx, o, what, flags, W)
    print(f"{what}: N={N} K={K} D={D} flagged {nf} + rescanned {nb}, resolved exactly {len(o.lists)}, "
          f"attributed to the float64 summation order {order}")

    oi = torch.from_numpy(o.idx).to(DEV)
    q_ref = c[oi].to(TDT[dt])
    l_ref = mse_sum(q_ref, xe, dt)
    # copy tail: q, int64 indices, loss
    q_buf = torch.empty_like(x)
    i_buf = torch.full((N,), -7, dtype=torch.int64, device=DEV)
    l_copy = torch.zeros(1, dtype=torch.float64, device=DEV)
    r1 = ops.search(x, cb, c, fused=dict(q_out=q_buf, idx64_out=i_buf, loss_sum=l_copy))
    # residual tail: r = x - q rounded once, loss
    r_buf = torch.empty_like(x)
    l_res = torch.zeros(1, dtype=torch.float64, device=DEV)
    r2 = ops.search(x, cb, c, fused=dict(resid_out=r_buf, loss_sum=l_res))
    torch.cuda.synchronize()
    for r in (r1, r2):
        assert np.array_equal(r.idx.cpu().numpy(), idx), f"{what}: indices of a fused search differ from the plain one"
    assert torch.equal(bits(q_buf), bits(q_ref)), f"{what}: copy tail q_out"
    assert torch.equal(i_buf, oi), f"{what}: copy tail idx64_out"
    assert torch.equal(bits(r_buf), bits((x.float() - q_ref.float()).to(TDT[dt]))), f"{what}: residual tail resid_out"
    assert_loss_sum(l_copy.item(), l_ref, dt, False, f"{what}: copy tail loss")
    assert_loss_sum(l_res.item(), l_ref, dt, cosine, f"{what}: residual tail loss")
    return o, res


# ------------------------------------------------------------------------------------------------------------------------
# data
# ------------------------------------------------------------------------------------------------------------------------

def as_dt(a, dt):
    return O.bf16_round(a) if dt == "bf16" else np.asarray(a, F32)


def unit(rng, n, D):
    u = rng.standard_normal((n, D))
    return u / np.linalg.norm(u, axis=-1, keepdims=True)


LADDER = [0.0, 0.25, 0.5, 0.9, 1.1, 2.0, 8.0]


def ladder_data(dt, cosine, D, rng, K=1024, reps=2):
    """Rows whose two best codes' exact score gap is t * W.  Row i sits near code a; code b = a + beta (x - a) is placed so
    that score(b) - score(a) = t W; b is the higher index on half the rows and the lower one on the others."""
    c = rng.standard_normal((K, D)).astype(F32)
    if cosine:
        c = (c / np.linalg.norm(c, axis=-1, keepdims=True)).astype(F32)
    n_lad = len(LADDER) * 2 * reps
    x = np.empty((n_lad + 200, D), F32)
    cn = np.linalg.norm(c.astype(np.float64), axis=-1)
    cmax = float(cn.max()) * 1.01
    plan = []
    for i, (t, hi_closer, _) in enumerate(itertools.product(LADDER, (True, False), range(reps))):
        lo_k, hi_k = 3 * i, K - 1 - 3 * i
        a, b = (lo_k, hi_k) if hi_closer else (hi_k, lo_k)
        x[i] = as_dt(c[a] + 0.3 * cn[a] * unit(rng, 1, D)[0], dt)
        plan.append((i, a, b, t))
    x[n_lad:] = as_dt(rng.standard_normal((200, D)) * (1.0 / np.sqrt(D) if cosine else 1.0), dt)
    xe = O.l2norm(x, dt) if cosine else x
    for i, a, b, t in plan:
        xr = xe[i].astype(np.float64)
        x2 = float(xr @ xr)
        cres = 2.0 ** -16 * cmax
        caux = (float.fromhex("0x1.02p-8") * cmax + 2.0 ** -8 * cmax) if dt == "fp32" else 0.0
        xlo = 2.0 ** -8 * math.sqrt(x2) if dt == "fp32" else 0.0
        alpha = t * float(kernel_band(np.array([x2]), np.array([xlo]), cmax, cres, caux, not cosine)[0])
        g = xr - c[a].astype(np.float64)
        if cosine:
            beta = alpha / float(xr @ g)
        else:
            r2 = float(g @ g)
            beta = 1.0 - math.sqrt(1.0 - 2.0 * alpha / r2)
        c[b] = (c[a].astype(np.float64) + beta * g).astype(F32)
    return torch.from_numpy(x), torch.from_numpy(c)


def collapse_data(dt, D, rng, K=1024):
    """Rows of norm ~1e3 (d^2 ~ 1e6) and code pairs whose d^2 differ by 2^-30 .. 2^-21 relative, the HIGHER index closer:
    where the reference's fp32 d^2 and sqrt merge the two, the lower index must win."""
    c = rng.standard_normal((K, D)).astype(F32)
    rels = [2.0 ** -30, 2.0 ** -27, 2.0 ** -25, 2.0 ** -24, 2.0 ** -23, 2.0 ** -21]
    reps = 4
    x = as_dt(1e3 * unit(rng, len(rels) * reps + 100, D), dt)
    for i, (rel, _) in enumerate(itertools.product(rels, range(reps))):
        a, b = 5 * i + 1, K - 2 - 5 * i
        x[i] = as_dt(1e3 * c[a] / np.linalg.norm(c[a]) + unit(rng, 1, D)[0], dt)   # code a is the nearest
        xr = x[i].astype(np.float64)
        g = xr - c[a].astype(np.float64)
        r2 = float(g @ g)
        alpha = 0.5 * rel * r2                      # score units: half the d^2 difference
        beta = 1.0 - math.sqrt(1.0 - 2.0 * alpha / r2)
        c[b] = (c[a].astype(np.float64) + beta * g).astype(F32)
    return torch.from_numpy(x), torch.from_numpy(c)


GROUPS = [(5, 700), (130, 131), (9, 400, 1000), (2, 3, 250, 600, 1023), (60, 61, 62)]
EPS = [1e-5, 3e-5, 1e-4]


def floor_data(dt, D, rng, scale, K=1024):
    """Codebook of max norm ~scale holding near-duplicate groups 1e-5 .. 1e-4 apart, rows on (and 1e-7 off) the
    highest-index member of each group.  For scale <= 1e-2 these rows sit at the reference's clamp floor: every member
    within 1e-4 scores -1e-4 and the lowest index wins.  scale = 1 is the normal-norm codebook, where the band is wide.
    bf16: the codes the rows sit on are bf16 values, so that the rows can sit exactly on them."""
    c = as_dt(rng.standard_normal((K, D)) * scale / np.sqrt(D), dt)
    rows = []
    for gi, grp in enumerate(GROUPS):
        for j, k in enumerate(grp[1:]):
            eps = EPS[(gi + j) % len(EPS)]
            c[k] = as_dt(c[grp[0]] + eps * unit(rng, 1, D)[0], dt)
        top = c[grp[-1]]
        rows += [top, top, as_dt(top + 1e-7 * unit(rng, 1, D)[0], dt)]
    x = np.concatenate([np.stack(rows), as_dt(rng.standard_normal((100, D)) * scale / np.sqrt(D), dt)])
    return torch.from_numpy(x.astype(F32)), torch.from_numpy(c.astype(F32))


def zero_rows_data(dt, D, rng, K=1024):
    """Zero rows (a ResidualVQ stage after an exact match) against a codebook of norm ~3e-3 holding codes of norm 5e-5,
    1e-6, 3e-5 and 0: all four are at the clamp floor for a zero row, so the lowest (1) wins, not the closest (700)."""
    c = rng.standard_normal((K, D)) * 3e-3 / np.sqrt(D)
    for k, nrm in ((1, 5e-5), (3, 1e-6), (K - 2, 3e-5), (700, 0.0)):
        c[k] = nrm * unit(rng, 1, D)[0]
    x = np.concatenate([np.zeros((16, D)), rng.standard_normal((64, D)) * 3e-3 / np.sqrt(D)])
    return torch.from_numpy(as_dt(x, dt)), torch.from_numpy(c.astype(F32))


DS = [8, 136, 256, 1000, 1024]


@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("dt,cosine", [("bf16", False), ("fp32", False), ("bf16", True), ("fp32", True)])
def test_gap_ladder(dt, cosine, D):
    """Exact score gaps 0 .. 8 W between the two best codes: rows just inside the band go to the re-score, rows just outside
    are certified; either way the index is the reference formula's."""
    rng = np.random.default_rng(D * 13 + 2 * cosine + (dt == "fp32"))
    x, c = ladder_data(dt, cosine, D, rng)
    run_case(x, c, dt, cosine, f"ladder {dt} {'cosine' if cosine else 'euclid'} D={D}")


@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_sqrt_collapse(dt, D):
    rng = np.random.default_rng(D * 17 + (dt == "fp32"))
    x, c = collapse_data(dt, D, rng)
    run_case(x, c, dt, False, f"sqrt collapse {dt} D={D}")


@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("scale", [1e-2, 3e-3, 1e-3, 1.0])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_clamp_floor(dt, scale, D):
    rng = np.random.default_rng(D * 19 + int(1 / scale) + (dt == "fp32"))
    x, c = floor_data(dt, D, rng, scale)
    o, _ = run_case(x, c, dt, False, f"clamp floor {dt} max|c|~{scale:g} D={D}")
    if scale < 1.0:   # the data reaches the floor: the rows on a group's top member take a lower member
        n = 3 * len(GROUPS)
        tops = np.repeat([g[-1] for g in GROUPS], 3)
        assert (o.idx[:n] < tops).sum() >= len(GROUPS), "the rows did not reach the clamp floor"


@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_clamp_floor_zero_rows(dt, D):
    rng = np.random.default_rng(D * 23 + (dt == "fp32"))
    x, c = zero_rows_data(dt, D, rng)
    o, _ = run_case(x, c, dt, False, f"zero rows {dt} D={D}")
    assert (o.idx[:16] == 1).all(), o.idx[:16]


def size_data(cosine, K, rng, D=1024, N=2048):
    """K = 16384 / 16383 codes (128 rescan chunks of 128, the last ragged), D = 1024 (the rescan's MAXJ).  Tie groups with
    members in the first, a middle and the last chunk: exact duplicates (3: the pair / triple re-score) and a five-fold
    near-duplicate group (the whole-row rescan), so the lowest index must win through the atomicMax key.  Cosine: every
    code leans towards +e0 and the rows point to -e0, so the best scores are negative (orderable() on negative floats)."""
    dup3 = (7, 8200, K - 1)
    five = (100, 127, 128, 9000, K - 2)
    if cosine:
        c = rng.standard_normal((K, D))
        c[:, 0] = 0.0
        c = c / np.linalg.norm(c, axis=-1, keepdims=True)
        c[:, 0] = 1.5
        c = c / np.linalg.norm(c, axis=-1, keepdims=True)        # e0 component 0.83
        dirs = []
        for grp in (dup3, five):
            w = rng.standard_normal(D)
            w[0] = 0.0
            w /= np.linalg.norm(w)
            g = 0.3 * np.eye(D)[0] + math.sqrt(1 - 0.09) * w       # e0 component 0.3: the best code for a row near -e0
            for k in grp:
                c[k] = g
            dirs.append(w)
        for k in five[1:]:
            c[k] = c[k] + 1e-7 * unit(rng, 1, D)[0]
        x = -np.eye(D)[0][None] + 0.3 * rng.standard_normal((N, D)) / np.sqrt(D)
        for j, w in enumerate(dirs):
            x[64 * j:64 * j + 64] = -np.eye(D)[0] + 0.05 * w + 1e-3 * rng.standard_normal((64, D)) / np.sqrt(D)
    else:
        c = rng.standard_normal((K, D))
        for k in dup3[1:]:
            c[k] = c[dup3[0]]
        for k in five[1:]:
            c[k] = c[five[0]] + 1e-5 * unit(rng, 1, D)[0]
        x = rng.standard_normal((N, D))
        for j, grp in enumerate((dup3, five)):
            x[64 * j:64 * j + 64] = c[grp[-1]] + 1e-2 * rng.standard_normal((64, D)) / np.sqrt(D)
    return torch.from_numpy(x.astype(F32)), torch.from_numpy(c.astype(F32))


@pytest.mark.parametrize("K", [16384, 16383])
@pytest.mark.parametrize("dt,cosine", [("bf16", False), ("fp32", False), ("bf16", True), ("fp32", True)])
def test_whole_row_rescan_at_size(dt, cosine, K):
    rng = np.random.default_rng(K + 2 * cosine + (dt == "fp32"))
    x, c = size_data(cosine, K, rng)
    five = (100, 127, 128, 9000, K - 2)
    o, res = run_case(x, c, dt, cosine, f"rescan {dt} {'cosine' if cosine else 'euclid'} K={K}")
    assert res.rescan_count.item() >= 64 and res.flag_count.item() >= 64
    assert (o.idx[:64] == 7).all() and np.isin(o.idx[64:128], five).all()
    if cosine:
        best = [formula(0, 0, r32((o.x[r] * o.c[o.idx[r]]).tolist()), True) for r in range(128)]
        assert max(best) < 0


@pytest.mark.parametrize("dt,cosine", [("bf16", False), ("fp32", False), ("bf16", True)])
def test_default_init_baseline_shape(dt, cosine):
    """Kaiming codebook (a default-constructed module) with K = 1024, D = 256 and randn rows at N = 65536: the regime where
    the other tests excuse up to 2e-3 of the rows.  None is excused here."""
    torch.manual_seed(11 + 2 * cosine + (dt == "fp32"))
    e = torch.empty(1, 1024, 256)
    torch.nn.init.kaiming_uniform_(e)
    c = e[0]
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    x = torch.randn(65536, 256)
    run_case(x, c, dt, cosine, f"default init {dt} {'cosine' if cosine else 'euclid'}")


# ------------------------------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_vector_quantize_step_on_near_ties(dt):
    """Two training steps of VectorQuantize (vqb_vq_forward; the second replays the cached graph) on clamp-floor data: indices equal the oracle's, cluster_size equals the lerp of bincount(oracle indices) exactly (the re-scored rows
    enter the statistics through the flagged-row path), embed_avg matches float64."""
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    rng = np.random.default_rng(31 + (dt == "fp32"))
    D, K = 256, 1024
    x, c = floor_data(dt, D, rng, 3e-3)
    decay = 0.5
    vq = m.VectorQuantize(dim=D, codebook_size=K, decay=decay).to(DEV)
    with torch.no_grad():
        vq._codebook.embed[0].copy_(c)
        vq._codebook.embed_avg[0].copy_(c)
    xd = x.to(TDT[dt]).to(DEV)[None]
    vq.train()
    for step in range(2):
        pre = vq._codebook.embed[0].clone()
        cs0 = vq._codebook.cluster_size[0].double().clone()
        ea0 = vq._codebook.embed_avg[0].double().clone()
        q, ind, loss = vq(xd)
        torch.cuda.synchronize()
        o = Oracle(xd[0].float(), pre, ops.prepare_codebook(pre, False).cnorm2, False)
        check_indices(ind[0].cpu().numpy(), o, f"VectorQuantize {dt} step {step}")
        oi = torch.from_numpy(o.idx).to(DEV)
        assert torch.equal(q[0], pre[oi].to(TDT[dt]))
        cnt = torch.bincount(oi, minlength=K).double()
        assert torch.equal(vq._codebook.cluster_size[0].double(), cs0 + (1 - decay) * (cnt - cs0)), f"step {step}: cluster_size"
        es = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, oi, xd[0].double())
        ea_ref = ea0 + (1 - decay) * (es - ea0)
        torch.testing.assert_close(vq._codebook.embed_avg[0].double(), ea_ref, rtol=1e-6, atol=1e-6 * ea_ref.abs().max().item())


@pytest.mark.parametrize("program", ["1", "0"])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_residual_vq_zero_residuals(dt, program, monkeypatch):
    """ResidualVQ (Q = 2) whose stage-0 codebook holds the rows exactly: stage 1 sees zero residuals against a small-norm
    codebook with codes at the clamp floor.  Both stages' indices equal the oracle along the residual recurrence."""
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    monkeypatch.setenv("VQB_RVQ_PROGRAM", program)
    rng = np.random.default_rng(41 + (dt == "fp32"))
    D, K, N = 256, 1024, 2048
    c0 = torch.from_numpy(as_dt(rng.standard_normal((K, D)), dt))
    _, c1 = zero_rows_data(dt, D, rng, K)
    j = torch.from_numpy(rng.integers(0, K, N))
    x = c0[j].clone()
    x[N // 2:] += torch.from_numpy(rng.standard_normal((N // 2, D)).astype(F32)) * 1e-2   # rows off the codes too
    rvq = m.ResidualVQ(dim=D, num_quantizers=2, codebook_size=K).to(DEV)
    with torch.no_grad():
        for layer, c in zip(rvq.layers, (c0, c1)):
            layer._codebook.embed[0].copy_(c)
            layer._codebook.embed_avg[0].copy_(c)
    books = [layer._codebook.embed[0].clone() for layer in rvq.layers]
    xd = x.to(TDT[dt]).to(DEV)[None]
    rvq.train()
    out, ind, losses = rvq(xd)
    torch.cuda.synchronize()
    r = xd[0]
    for s, book in enumerate(books):
        o = Oracle(r.float(), book, ops.prepare_codebook(book, False).cnorm2, False)
        check_indices(ind[0, :, s].cpu().numpy(), o, f"ResidualVQ {dt} program={program} stage {s}")
        if s == 1:
            assert (o.idx[:N // 2] == 1).all()   # zero residuals: the lowest code at the floor
        r = (r.float() - book[torch.from_numpy(o.idx).to(DEV)]).to(TDT[dt])


# ------------------------------------------------------------------------------------------------------------------------
# operand preparation
# ------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K,D,scale", [(1024, 8, 1.0), (1000, 136, 3e-3), (1024, 256, 1e-2), (333, 1000, 1.0),
                                       (16383, 1024, 1e-3), (37, 24, 1.0)])
@pytest.mark.parametrize("cosine", [False, True])
def test_codebook_prepare(K, D, scale, cosine):
    """vqb_codebook_prepare against an independent reference: bext sums to -bias exactly, bias = cnorm2 / 2 (0 for cosine),
    cnorm2 is exactly rounded, padded codes hold zeros, +inf bias and a -3e38 seed, and cmax bounds the norms."""
    from vector_quantize_pytorch_b200 import ops
    rng = np.random.default_rng(K + D)
    c = rng.standard_normal((K, D)) * scale / np.sqrt(D)
    c[K // 2] = 0.0
    if cosine:
        c[K // 2] = 1.0
        c = c / np.linalg.norm(c, axis=-1, keepdims=True)
    c = torch.from_numpy(c.astype(F32)).to(DEV).contiguous()
    cb = ops.prepare_codebook(c, cosine)
    torch.cuda.synchronize()
    Kpad = ops.padded_codes(K)
    ex = check_cnorm2(c, cb.cnorm2)
    bias = cb.bias.cpu().numpy()
    assert np.array_equal(bias[:K], np.zeros(K, F32) if cosine else F32(0.5) * ex)
    assert np.isposinf(bias[K:]).all()
    bext = cb.bext.float().cpu().double().numpy()
    assert np.array_equal(bext[:K, :3].sum(-1), -bias[:K].astype(np.float64)), "bext[:, 0:3] must sum to -bias exactly"
    assert (bext[:K, 3:] == 0).all()
    assert (bext[K:, 0] == float(torch.tensor(-3.0e38).bfloat16().float())).all() and (bext[K:, 1:] == 0).all()
    planes = cb.planes.view(torch.int16)
    assert (planes[:, K:] == 0).all()
    hi = planes[0, :K].view(torch.bfloat16).float()
    lo = planes[1, :K].view(torch.bfloat16).float()
    assert torch.equal(hi, c.bfloat16().float()) and torch.equal(lo, (c - hi).bfloat16().float())
    c64 = c.double()
    nmax = c64.norm(dim=-1).max().item()
    cm = cb.cmax.cpu().numpy()
    assert abs(float(cm[0]) - nmax) <= float(np.spacing(F32(nmax))), (cm[0], nmax)
    assert cm[1] >= (c64 - hi.double() - lo.double()).norm(dim=-1).max().item()
    assert cm[2] >= lo.double().norm(dim=-1).max().item()
