"""The gather-sum kernels (ResidualVQ's running sum and the decode) and the rotation trick, against plain references
(run on an H100: `pytest -m gpu`).

(a) vqb_rvq_accumulate builds `quantized_out` of ResidualVQ / GroupedResidualVQ: every partial sum rounded to the dtype where
    the reference's `quantized_out = quantized_out + quantized` rounds.  It must equal, bit for bit, torch's own recurrence
    `acc = acc + embed_q[idx[:, q]].to(dtype)` from zeros (fp32: the same IEEE adds in the same order; bf16: add.rn.bf16x2 of
    two bf16 values is torch's round(fp32(a + b))).
(b) vqb_decode (get_output_from_indices / get_codes_from_indices) must equal the sequential fp32 sum of the gathered rows,
    index -1 adding nothing, rounded once to the output dtype.
    Both run on every slice plan of rvq_accumulate_smem_kernel (tests/test_gather_sum_plan.py has the table): 4 lane-per-row
    widths x 2 staged element sizes, shared and stacked codebooks, Q > lanes per row (the stage-chunk loop), a row count
    that leaves the last row group ragged (the next-row index prefetch runs off the end) — and on the L2 kernel.  Every
    output buffer carries guard rows holding a sentinel that must survive.
(c) The modules' `quantized` and get_output_from_indices against (a) and (b), on both forward paths.
(d) vqb_rotate (vqp:287-318), forward value and gradient, against a float64 restatement of the reference formula and its
    float64 autograd, within a first-order bound of the fp32 evaluation that torch's own fp32 evaluation meets as well.
"""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}
GUARD = 5                    # guard rows after row N in every output buffer
SENT = -12345.678            # their sentinel
SMEM = 196608


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gather_plan(nbooks, K, D, esz, N):
    from vector_quantize_pytorch_b200 import _C
    out = (ctypes.c_int * 3)()
    assert _C.lib.vqb_debug_gather_sum_plan(nbooks, K, D, esz, N, sms(), ctypes.cast(out, ctypes.c_void_p)) == 0
    return tuple(out)


# ------------------------------------------------------------------------------------------------ references
def running_sum_ref(E, idx, dt):
    """rvq:525 on the device: acc = acc + embed_q[idx[:, q]].to(dt), from zeros.  E (nbooks, K, D) fp32."""
    acc = torch.zeros(idx.shape[0], E.shape[-1], dtype=dt, device=DEV)
    for q in range(idx.shape[1]):
        acc = acc + E[q if E.shape[0] > 1 else 0][idx[:, q]].to(dt)
    return acc


def decode_ref(E, idx, dt):
    """Sequential fp32 sum over q of the gathered rows, index -1 adding nothing, one rounding to dt."""
    acc = torch.zeros(idx.shape[0], E.shape[-1], dtype=torch.float32, device=DEV)
    for q in range(idx.shape[1]):
        k = idx[:, q]
        acc = torch.where((k >= 0)[:, None], acc + E[q if E.shape[0] > 1 else 0][k.clamp_min(0)], acc)
    return acc.to(dt)


def run_abi(fn, E, stacked, idx, dt):
    """vqb_rvq_accumulate / vqb_decode on (N + GUARD) output rows; the guard rows must keep the sentinel."""
    from vector_quantize_pytorch_b200 import _C
    N, Q = idx.shape
    _, K, D = E.shape
    out = torch.full((N + GUARD, D), SENT, dtype=dt, device=DEV)
    code = _C.DTYPE_F32 if dt == torch.float32 else _C.DTYPE_BF16
    rc = getattr(_C.lib, fn)(E.data_ptr(), K * D if stacked else 0, Q, K, D, idx.data_ptr(), N, out.data_ptr(), code,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, fn
    torch.cuda.synchronize()
    assert torch.equal(out[N:], torch.full_like(out[N:], SENT)), f"{fn} wrote past row N"
    return out[:N]


def codebooks(nbooks, K, D, gen):
    """Code rows of widely varying magnitude, so that a reordered or re-rounded sum shows."""
    e = torch.randn(nbooks, K, D, generator=gen, device=DEV)
    return e * torch.exp(2 * torch.randn(nbooks, K, 1, generator=gen, device=DEV))


def with_dropped(idx, rpw, gen):
    """Index -1 (a dropped stage) as every pattern the decode meets: whole trailing columns (quantize dropout), scattered
    entries, whole rows, and the first stage of the first row of a warp's row group (read from the prefetched indices)."""
    N, Q = idx.shape
    idx = idx.clone()
    band = N // 4
    keep = torch.randint(0, Q, (band,), generator=gen, device=DEV)
    idx[:band][torch.arange(Q, device=DEV)[None, :] >= keep[:, None]] = -1
    idx[band:2 * band][torch.rand(band, Q, generator=gen, device=DEV) < 0.3] = -1
    rows = torch.arange(N, device=DEV)
    idx[rows % 97 == 5] = -1
    idx[(rows >= 2 * band) & (rows % rpw == 0), 0] = -1
    return idx, rows % 97 == 5


# ------------------------------------------------------------------------------------------------ (a), (b): slice plans
def slice_case(esz, lpr, stacked):
    """A case whose plan is (esz, lanes per row): D = 3 W (W the widest power of two dividing it), Q = lpr + 1 stages (the
    stage-chunk loop runs twice, the second chunk ragged), K as large as the slice allows, N past one row step + ragged."""
    W = 16 * lpr // esz
    D, Q = 3 * W, lpr + 1
    nb = Q if stacked else 1
    K = min(1536, SMEM // (nb * W * esz))
    W_, slices, cps = gather_plan(nb, K, D, esz, 1 << 20)
    assert W_ == W, (esz, lpr, stacked)
    step = cps * 32 * (32 // lpr)          # rows per iteration of all the CTAs of one slice
    N = (4096 // step + 1) * step + 37
    assert gather_plan(nb, K, D, esz, N)[0] == W and N % step != 0
    return D, Q, K, N, W


@pytest.mark.parametrize("stacked", [False, True], ids=["shared", "stacked"])
@pytest.mark.parametrize("lpr", [4, 8, 16, 32])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_running_sum_slice_plans(dt, lpr, stacked):
    gen = torch.Generator(device=DEV).manual_seed(lpr * 2 + stacked)
    D, Q, K, N, W = slice_case(2 if dt == "bf16" else 4, lpr, stacked)
    E = codebooks(Q if stacked else 1, K, D, gen)
    idx = torch.randint(0, K, (N, Q), generator=gen, device=DEV)
    got = run_abi("vqb_rvq_accumulate", E, stacked, idx, TDT[dt])
    ref = running_sum_ref(E, idx, TDT[dt])
    bad = (got != ref).any(-1)
    assert not bad.any(), f"W={W} D={D} Q={Q} K={K} N={N}: {int(bad.sum())} rows differ, first {int(bad.nonzero()[0])}"


@pytest.mark.parametrize("stacked", [False, True], ids=["shared", "stacked"])
@pytest.mark.parametrize("lpr", [4, 8, 16, 32])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_decode_slice_plans(dt, lpr, stacked):
    gen = torch.Generator(device=DEV).manual_seed(100 + lpr * 2 + stacked)
    D, Q, K, N, W = slice_case(4, lpr, stacked)      # the decode stages fp32 codes for either output dtype
    E = codebooks(Q if stacked else 1, K, D, gen)
    idx, empty = with_dropped(torch.randint(0, K, (N, Q), generator=gen, device=DEV), 32 // lpr, gen)
    got = run_abi("vqb_decode", E, stacked, idx, TDT[dt])
    ref = decode_ref(E, idx, TDT[dt])
    bad = (got != ref).any(-1)
    assert not bad.any(), f"W={W} D={D} Q={Q} K={K} N={N}: {int(bad.sum())} rows differ, first {int(bad.nonzero()[0])}"
    assert not got[empty].signbit().any() and not got[empty].any(), "a row of -1 must decode to +0"


# ------------------------------------------------------------------------------------------------ (a), (b): L2 kernel
L2_CASES = [
    # Q,  K,     D,   stacked    rvq_accumulate_kernel: stages in batches of 8, indices in chunks of 32
    (1, 16384, 264, True),       # one stage; D = 264: 31 of 32 lanes idle in the second 256-column pass
    (8, 16384, 264, True),       # one batch of 8
    (9, 16384, 264, True),       # two batches, the second of one stage
    (33, 16384, 264, True),      # two index chunks
    (8, 1000, 264, False),       # shared codebook, D with no 64-byte row piece
    (3, 16384, 256, True),       # D = 256: every lane active; three codebooks of 16384 fit no slice
]


@pytest.mark.parametrize("kind", ["running_sum", "decode"])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
@pytest.mark.parametrize("Q,K,D,stacked", L2_CASES)
def test_l2_kernel(Q, K, D, stacked, dt, kind):
    gen = torch.Generator(device=DEV).manual_seed(Q * 7 + D)
    N = 5003
    assert gather_plan(Q if stacked else 1, K, D, 4, N)[0] == 0 and gather_plan(Q if stacked else 1, K, D, 2, N)[0] == 0
    E = codebooks(Q if stacked else 1, K, D, gen)
    idx = torch.randint(0, K, (N, Q), generator=gen, device=DEV)
    if kind == "running_sum":
        got, ref = run_abi("vqb_rvq_accumulate", E, stacked, idx, TDT[dt]), running_sum_ref(E, idx, TDT[dt])
    else:
        idx, empty = with_dropped(idx, 1, gen)
        got, ref = run_abi("vqb_decode", E, stacked, idx, TDT[dt]), decode_ref(E, idx, TDT[dt])
        assert not got[empty].signbit().any() and not got[empty].any(), "a row of -1 must decode to +0"
    bad = (got != ref).any(-1)
    assert not bad.any(), f"{int(bad.sum())} rows differ, first {int(bad.nonzero()[0])}"


@pytest.mark.parametrize("kind,dt", [("running_sum", "bf16"), ("running_sum", "fp32"), ("decode", "fp32")])
def test_row_threshold_kernels_agree(kind, dt):
    """4095 rows take the L2 kernel and 4096 the slice kernel: on the same data they must agree bit for bit."""
    gen = torch.Generator(device=DEV).manual_seed(5)
    K, D, Q = 1024, 256, 8
    esz = 2 if (kind, dt) == ("running_sum", "bf16") else 4
    assert gather_plan(1, K, D, esz, 4095)[0] == 0 and gather_plan(1, K, D, esz, 4096)[0] == (64 if esz == 2 else 32)
    E = codebooks(1, K, D, gen)
    idx = torch.randint(0, K, (4096, Q), generator=gen, device=DEV)
    fn = "vqb_rvq_accumulate" if kind == "running_sum" else "vqb_decode"
    if kind == "decode":
        idx, _ = with_dropped(idx, 4, gen)
    a = run_abi(fn, E, False, idx[:4095].contiguous(), TDT[dt])
    b = run_abi(fn, E, False, idx, TDT[dt])
    assert torch.equal(a, b[:4095])
    ref = running_sum_ref(E, idx, TDT[dt]) if kind == "running_sum" else decode_ref(E, idx, TDT[dt])
    assert torch.equal(b, ref)


# ------------------------------------------------------------------------------------------------ (c): the modules
@pytest.mark.parametrize("program", ["1", "0"], ids=["program", "stagewise"])
@pytest.mark.parametrize("dt", ["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["rvq_shared", "rvq_separate", "grvq"])
def test_module_running_sum_and_decode(kind, dt, program, monkeypatch):
    """`quantized` of a training forward is the recurrence (a) on the module's own indices and the codebooks the stages
    searched (before the deferred EMA update); get_output_from_indices is the decode (b) on the updated codebooks."""
    m = vqb()
    monkeypatch.setenv("VQB_RVQ_PROGRAM", program)
    torch.manual_seed(3)
    if kind == "grvq":
        mod = m.GroupedResidualVQ(dim=256, groups=2, num_quantizers=3, codebook_size=128).to(DEV)
        rvqs, dim = list(mod.rvqs), 256
    else:
        shared = kind == "rvq_shared"
        mod = m.ResidualVQ(dim=128, num_quantizers=4, codebook_size=512 if shared else 256, shared_codebook=shared).to(DEV)
        rvqs, dim = [mod], 128
    for step in range(2):   # step 0 initialises the codebooks (stage-wise); step 1 runs the cached program when allowed
        pre = [torch.stack([layer._codebook.embed[0] for layer in r.layers]).clone() for r in rvqs]
        x = torch.randn(2, 4096, dim, device=DEV).to(TDT[dt])
        q, ind, _ = mod(x)
        torch.cuda.synchronize()
        inds = ind if kind == "grvq" else ind[None]
        Q = inds.shape[-1]
        ref = torch.cat([running_sum_ref(E, i.reshape(-1, Q), TDT[dt]) for E, i in zip(pre, inds)], -1)
        assert torch.equal(q.reshape(-1, dim), ref), f"step {step}: quantized is not the rounded running sum"
        post = [torch.stack([layer._codebook.embed[0] for layer in r.layers]) for r in rvqs]
        dec = torch.cat([decode_ref(E, i.reshape(-1, Q), torch.float32) for E, i in zip(post, inds)], -1)
        assert torch.equal(mod.get_output_from_indices(ind).reshape(-1, dim), dec), f"step {step}: decode differs"
    assert (len(mod.__dict__.get("_plans", {})) >= 1) == (program == "1")


# ------------------------------------------------------------------------------------------------ (d): rotation trick
EPS32 = 2.0 ** -24
ANTI = [1e-1, 1e-2, 1e-3, 2e-4, 1e-5, 0.0]
ROW_KINDS = ["randn", "close", "orthogonal", "equal", "zero_src", "zero_tgt", "tiny"] + [f"anti_{a:g}" for a in ANTI]


def rotation_rows(kind, n, D, gen):
    """(src, tgt) float64 rows of one kind, before rounding to the input dtype."""
    def rn(*shape):
        return torch.randn(*shape, generator=gen, device=DEV, dtype=torch.float64)
    scale = lambda: 10.0 ** (4 * torch.rand(n, 1, generator=gen, device=DEV, dtype=torch.float64) - 2)
    t = rn(n, D) * scale()
    if kind == "randn":
        return rn(n, D) * scale(), t
    if kind == "close":        # an input next to its code, as with a trained codebook
        return t * (1 + 0.1 * rn(n, 1)) + 0.02 * rn(n, D) * t.norm(dim=-1, keepdim=True) / math.sqrt(D), t
    if kind == "orthogonal":
        s = rn(n, D)
        return (s - (s * t).sum(-1, keepdim=True) / (t * t).sum(-1, keepdim=True) * t) * scale(), t
    if kind == "equal":
        return t.clone(), t
    if kind == "zero_src":
        return torch.zeros_like(t), t
    if kind == "zero_tgt":
        return t, torch.zeros_like(t)
    if kind == "tiny":         # both norms below the 1e-6 clamps of safe_div
        unit = lambda v: v / v.norm(dim=-1, keepdim=True)
        return unit(rn(n, D)) * 3e-7, unit(t) * 5e-7
    m = float(kind.split("_")[1])
    if m == 0.0:               # exactly antipodal in any dtype: src = -2 tgt
        return -2 * t, t
    qh = t / t.norm(dim=-1, keepdim=True)
    p = rn(n, D)
    p = p - (p * qh).sum(-1, keepdim=True) * qh
    p = p / p.norm(dim=-1, keepdim=True)
    th = 2 * math.asin(m / 2)  # ||u + q|| = 2 sin(theta / 2) for u = -cos(theta) q + sin(theta) p
    return (-math.cos(th) * qh + math.sin(th) * p) * scale(), t


def rotate_formula(src, tgt):
    """vqp:287-318 restated: safe_div with eps 1e-6, l2norm eps 1e-6, w / u / q / the norm factor detached."""
    norm_src = src.norm(dim=-1, keepdim=True)
    norm_tgt = tgt.norm(dim=-1, keepdim=True)
    u = src / norm_src.clamp(min=1e-6)
    q = tgt / norm_tgt.clamp(min=1e-6)
    e = src[:, None, :]
    w = torch.nn.functional.normalize(u + q, p=2, dim=1, eps=1e-6).detach()
    out = e - 2 * (e @ w[:, :, None] @ w[:, None, :]) + 2 * (e @ u.detach()[:, :, None] @ q.detach()[:, None, :])
    return out[:, 0, :] * (norm_tgt / norm_src.clamp(min=1e-6)).detach()


def rotate_eval(src, tgt, grad):
    """Forward value and d/d src of rotate_formula, in the dtype of src."""
    s = src.detach().clone().requires_grad_(True)
    out = rotate_formula(s, tgt)
    (ds,) = torch.autograd.grad(out, s, grad)
    return out.detach(), ds


def rotate_bound(s, t, g, D):
    """First-order bound on |fp32 evaluation - exact| per element of the forward value (g None) or of the gradient, for any
    evaluation that forms u = s ins, q = t int_, w = (u + q) / ||u + q|| elementwise in fp32 and the dot products by sums
    of D products (the kernel: D / 32 terms per lane, then a 5-level tree).  u + q is formed from rounded u and q, so w
    carries a direction error ~ 2^-24 |u_i| / ||u + q||: the conditioning of the problem itself near antipodal rows."""
    rho = (math.ceil(D / 32) + 8) * EPS32               # relative error of a reduction of D terms (of their |sum|)
    d1 = rho + 3 * EPS32                                # of ins / int_: a reduction, sqrt, reciprocal
    ns, nt = s.norm(dim=-1, keepdim=True), t.norm(dim=-1, keepdim=True)
    ins, int_ = 1 / ns.clamp(min=1e-6), 1 / nt.clamp(min=1e-6)
    u, q = s * ins, t * int_
    m = (u + q).norm(dim=-1, keepdim=True)
    mc = m.clamp(min=1e-6)
    w = (u + q) / mc
    du, dq = (d1 + EPS32) * u.abs(), (d1 + EPS32) * q.abs()
    dp = du + dq + EPS32 * (u + q).abs()
    dm = dp.norm(dim=-1, keepdim=True) + rho * m + EPS32 * m
    dw = dp / mc + w.abs() * (dm / mc + 2 * EPS32)
    lam = nt * ins
    dlam = (2 * d1 + EPS32) * lam
    if g is None:   # out = lam (s - 2 (s.w) w + 2 (s.u) q)
        e, bv, dbv, v, dv = s, u, du, q, dq
    else:           # d_s = lam (g - 2 (g.w) w + 2 (g.q) u)
        e, bv, dbv, v, dv = g, q, dq, u, du
    a = (e * w).sum(-1, keepdim=True)
    b = (e * bv).sum(-1, keepdim=True)
    da = (e.abs() * dw).sum(-1, keepdim=True) + rho * (e * w).abs().sum(-1, keepdim=True)
    db = (e.abs() * dbv).sum(-1, keepdim=True) + rho * (e * bv).abs().sum(-1, keepdim=True)
    r = e - 2 * a * w + 2 * b * v
    # da * dw: both errors grow as 1 / ||u + q||, so their product outgrows the first-order terms below ||u + q|| ~ 2^-12
    dr = 2 * da * (w.abs() + dw) + 2 * a.abs() * dw + 2 * db * v.abs() + 2 * b.abs() * dv \
        + 4 * EPS32 * (e.abs() + 2 * (a * w).abs() + 2 * (b * v).abs())
    return lam * dr + (dlam + EPS32 * lam) * r.abs()


def half_ulp_bf16(x):
    """Half a bf16 ulp of |x| (0 at 0)."""
    _, ex = torch.frexp(x.abs())
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), ex - 9))


def ratio(got, ref, bound):
    """Worst |got - ref| / bound; an exact zero error on a zero bound counts 0."""
    err = (got.double() - ref).abs()
    return torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))


@pytest.mark.parametrize("D,rows", [(8, 16), (24, 16), (200, 16), (256, 16), (1000, 16), (1024, 16),
                                    (256, "grid")])
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_rotate_against_float64(dt, D, rows):
    """ops.rotate forward and backward on every row kind; rows = "grid": more rows than one grid of warps (16 CTAs per SM
    x 8 rows), so the grid-stride loop runs."""
    from vector_quantize_pytorch_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(D)
    n = 16 if rows != "grid" else -(-3 * 16 * sms() * 8 // len(ROW_KINDS))
    parts = [rotation_rows(k, n, D, gen) for k in ROW_KINDS]
    tdt = TDT[dt]
    s = torch.cat([p[0] for p in parts]).to(tdt)
    t = torch.cat([p[1] for p in parts]).to(tdt)
    g = torch.randn(s.shape, generator=gen, device=DEV).to(tdt)
    kind = torch.arange(len(ROW_KINDS), device=DEV).repeat_interleave(n)
    s64, t64, g64 = s.double(), t.double(), g.double()
    ref_f, ref_b = rotate_eval(s64, t64, g64)
    got_f, got_b = ops.rotate(s, t), ops.rotate(s, t, g)
    tor_f, tor_b = rotate_eval(s.float(), t.float(), g.float())     # torch's fp32 evaluation of the same formula
    torch.cuda.synchronize()
    m = (s64 / s64.norm(dim=-1, keepdim=True).clamp(min=1e-6) + t64 / t64.norm(dim=-1, keepdim=True).clamp(min=1e-6)).norm(dim=-1)
    worst = {}
    for what, ref, got, tor, gg in (("fwd", ref_f, got_f, tor_f, None), ("bwd", ref_b, got_b, tor_b, g64)):
        bound = rotate_bound(s64, t64, gg, D)
        if dt == "bf16":
            tor = tor.to(tdt)
            bound = bound + half_ulp_bf16(ref.abs() + bound)
        rk, rt = ratio(got, ref, bound).amax(-1), ratio(tor, ref, bound).amax(-1)
        for j, name in enumerate(ROW_KINDS):
            sel = kind == j
            worst[(what, name)] = (float(rk[sel].max()), float(rt[sel].max()), float(m[sel].min()), float(m[sel].max()))
    print(f"\n{dt} D={D} N={s.shape[0]}: worst |error| / bound, kernel | torch fp32   (||u + q|| of the rows)")
    for (what, name), (k_, t_, lo, hi) in worst.items():
        print(f"  {what} {name:11s} {k_:9.3g} | {t_:9.3g}   ({lo:.3g} .. {hi:.3g})")
    # 2: room for the second-order terms the first-order bound leaves out
    assert all(v[1] <= 2 for v in worst.values()), "torch's fp32 evaluation exceeds the bound: the bound is too tight"
    bad = {k: v[0] for k, v in worst.items() if not v[0] <= 2}
    assert not bad, f"vqb_rotate outside the bound: {bad}"
