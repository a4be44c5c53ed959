"""vqb_fsp_forward / _stats / _backward / _decode called directly against the float64 oracle (oracle/fsp_oracle.py): every d
from 1 to 16 x every CDF x need_inv_act x fp32 / bf16, sentinel guard rows around every output of the four entry points, more
than one grid wave, planted floor / clamp / accept / choice boundaries and extreme inputs (+-0, subnormals, +-FLT_MAX, +-inf,
NaN) against exactly rounded restatements, the moments of a far-offset column at 2^22 rows, a constant column and run-to-run
bit equality."""
import numpy as np
import pytest
import torch

from oracle import fsp_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 4   # sentinel rows on each side of every output (4 rows of d fp32 keep the view 16-byte aligned)


def _ops():
    from vector_quantize_pytorch_b200 import ops
    return ops


def _guarded(shape, dtype, fill):
    """A view of `shape` inside a buffer with GUARD sentinel rows before and after."""
    buf = torch.full((shape[0] + 2 * GUARD, *shape[1:]), fill, dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + shape[0]]


def _levels(d, seed):
    g = np.random.default_rng(seed)
    lv = g.integers(2, 9, size=d)
    while np.prod(lv.astype(np.float64)) >= 2 ** 31:
        lv[np.argmax(lv)] -= 1
    return [int(v) for v in lv]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("inv", [False, True], ids=["fwd", "inv"])
@pytest.mark.parametrize("act", O.ACTS)
@pytest.mark.parametrize("d", range(1, 17))
def test_instantiation(d, act, inv, dtype):
    ops = _ops()
    N = 3000
    levels = _levels(d, d * 7 + O.ACTS.index(act))
    lv = torch.tensor(levels, dtype=torch.int32, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(d)
    z = (torch.randn(N, d, device=DEV, generator=g) * 1.7).to(dtype)
    u1 = torch.rand(N, d, device=DEV, generator=g).to(dtype)
    u2 = torch.rand(N, d, device=DEV, generator=g).to(dtype)
    eps = float(torch.finfo(dtype).eps)
    f64 = lambda t: t.double().cpu().numpy()   # noqa: E731
    for pert in (False, True):
        out_dt = torch.float32 if pert else dtype
        ca = lambda v, dt: torch.tensor(v, dtype=torch.float64).to(dt).item()   # noqa: E731
        out, idx, lev, acc = ops.fsp_forward(z, O.ACTS.index(act), inv, lv, ca(1 - eps, dtype), u1 if pert else None,
                                             u2 if pert else None, ca(0.5, dtype), ca(eps, out_dt), ca(1 - eps, out_dt))
        q64, idx64, lev64, acc64 = O.row_chain(f64(z), levels, act, inv, eps, f64(u1) if pert else None, f64(u2) if pert else None,
                                               ca(0.5, dtype))
        rel = 2. ** -19 if dtype == torch.float32 else 2. ** -6   # bf16 rounds act and act L to 8 bits
        near = O.near_integer(O.pre_floor(f64(z), levels, act, eps), rel)
        ok = ~near.any(-1)
        a64 = O.act_f64(act, f64(z))
        if pert:   # proposals within the act error of 0 or 1 may be accepted on one side and not on the other
            prop = a64 + (f64(u1) * 2 - 1) / (2 * np.array(levels))
            ok &= ~((np.abs(prop) <= 2 * rel) | (np.abs(1 - prop) <= 2 * rel)).any(-1)
        if inv:    # the inverse CDF's slope amplifies act's last-bit differences without bound near 0 and 1
            ok &= ((a64 > 0.01) & (a64 < 0.99)).all(-1) & (np.abs(q64) < 100).all(-1)
        np.testing.assert_array_equal(f64(lev)[~near], lev64[~near])
        np.testing.assert_array_equal(idx.cpu().numpy()[~near.any(-1)], idx64[~near.any(-1)])
        exact = (f64(lev).astype(np.int64) * O.basis(levels)).sum(-1)
        np.testing.assert_array_equal(idx.cpu().numpy(), exact)
        if pert:
            assert abs(int(acc) - int(acc64.sum())) <= near.sum() + 2
        tol = (2e-5 if dtype == torch.float32 else 3e-2) * (10 if inv else 1)
        np.testing.assert_allclose(f64(out)[ok], q64[ok], rtol=tol, atol=tol)
    # statistics and the backward
    norm = O.PRESETS["kurt"]
    stats, loss, aux = ops.fsp_stats(z, norm)
    s64 = O.moments(f64(z))
    for k in range(4):
        np.testing.assert_allclose(f64(stats[k]), s64[k], rtol=1e-5 if dtype == torch.float32 else 1e-2, atol=1e-6)
    gq = torch.randn(N, d, device=DEV, generator=g).to(dtype)
    gs = torch.randn(4, d, device=DEV, generator=g)
    gl = torch.tensor(0.7, device=DEV)
    gz = ops.fsp_backward(z, O.ACTS.index(act), inv, gq, aux, gs, gl, norm)
    G = f64(gs) + 0.7 * O.norm_loss_grad_weights(s64, norm, d)
    qpath = f64(gq) if inv else f64(gq) / O.UNIT_STD * O.act_grad_f64(act, f64(z))
    ref = qpath + O.stats_grad(f64(z), G)
    np.testing.assert_allclose(f64(gz), ref, rtol=2e-4 if dtype == torch.float32 else 2e-2,
                               atol=(2e-5 if dtype == torch.float32 else 2e-2) * np.abs(ref).max())
    # decode
    bufa, a = _guarded((N, d), torch.float32, 7.0)
    bufc, c = _guarded((N, d), torch.float32, 7.0)
    ix = idx.clone()
    lib = ops.lib
    with torch.cuda.device(z.device):
        ops.check(lib.vqb_fsp_decode(ix.data_ptr(), 0, N, d, O.ACTS.index(act), int(inv), lv.data_ptr(), 1e-6, 1 - 1e-6,
                                     a.data_ptr(), c.data_ptr(), ops._stream()), "decode")
    torch.cuda.synchronize()
    assert (bufa[:GUARD] == 7).all() and (bufa[-GUARD:] == 7).all() and (bufc[:GUARD] == 7).all() and (bufc[-GUARD:] == 7).all()
    digits = (ix.cpu().numpy()[:, None] // O.basis(levels)) % np.array(levels)
    np.testing.assert_array_equal(a.cpu().numpy(), ((digits + 0.5) / np.array(levels)).astype(np.float32))
    code64 = O.inv_act_f64(act, np.clip((digits + 0.5) / np.array(levels), 1e-6, 1 - 1e-6)) if inv else \
        ((digits + 0.5) / np.array(levels) - 0.5) / O.UNIT_STD
    np.testing.assert_allclose(c.cpu().numpy(), code64, rtol=2e-6, atol=2e-6)


def test_forward_over_several_waves():
    """The forward's indices and accept count at a row count several grid waves deep."""
    ops = _ops()
    N, d = 600_000, 4
    lv = torch.tensor([8, 5, 5, 5], dtype=torch.int32, device=DEV)
    z = torch.randn(N, d, device=DEV)
    u1, u2 = torch.rand(N, d, device=DEV), torch.rand(N, d, device=DEV)
    out, idx, lev, acc = ops.fsp_forward(z, 0, False, lv, 1 - 2 ** -23, u1, u2, 0.5, 2 ** -23, 1 - 2 ** -23)
    q64, idx64, lev64, acc64 = O.row_chain(z.double().cpu().numpy(), [8, 5, 5, 5], "tanh", False, 2 ** -23,
                                           u1.double().cpu().numpy(), u2.double().cpu().numpy(), 0.5)
    near = O.near_integer(O.pre_floor(z.double().cpu().numpy(), [8, 5, 5, 5], "tanh", 2 ** -23)).any(-1)
    np.testing.assert_array_equal(idx.cpu().numpy()[~near], idx64[~near])
    assert abs(int(acc) - int(acc64.sum())) <= 4
    assert lib_blocks(N) * 256 < N


def lib_blocks(N):
    return _ops().lib.vqb_fsp_blocks(N)


def test_moments_far_offset_column():
    """2^22 rows, a column at mean 1e3 with sigma 1: the two-pass fp64 moments stay at float64 accuracy."""
    ops = _ops()
    N = 1 << 22
    g = torch.Generator(device=DEV).manual_seed(3)
    z = torch.randn(N, 4, device=DEV, generator=g)
    z[:, 0] += 1000.
    stats, loss, _ = ops.fsp_stats(z, O.PRESETS["kurt"])
    s64 = O.moments(z.double().cpu().numpy())
    for k in range(4):
        np.testing.assert_allclose(stats[k].double().cpu().numpy(), s64[k], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(float(loss), O.norm_loss(s64, O.PRESETS["kurt"]), rtol=1e-5)


def test_constant_column():
    ops = _ops()
    z = torch.randn(1000, 3, device=DEV)
    z[:, 1] = 0.25
    stats, loss, aux = ops.fsp_stats(z, O.PRESETS["kurt"])
    assert stats[1, 1].item() == 0. and stats[2, 1].item() == 0. and stats[3, 1].item() == -3.
    G = torch.randn(4, 3, device=DEV)
    gz = ops.fsp_backward(z, 0, True, None, aux, G, None, O.PRESETS["kurt"])
    ref = O.stats_grad(z.double().cpu().numpy(), G.double().cpu().numpy())
    np.testing.assert_allclose(gz.double().cpu().numpy(), ref, rtol=1e-4, atol=1e-6 * np.abs(ref).max())


def test_run_to_run_bit_equality():
    ops = _ops()
    N, d = 300_000, 5
    lv = torch.tensor([8, 5, 5, 5, 3], dtype=torch.int32, device=DEV)
    z = torch.randn(N, d, device=DEV).bfloat16()
    u1, u2 = torch.rand(N, d, device=DEV).bfloat16(), torch.rand(N, d, device=DEV).bfloat16()
    runs = []
    for _ in range(2):
        out, idx, lev, acc = ops.fsp_forward(z, 2, True, lv, 0.9921875, u1, u2, 0.5, 0.0078125, 0.9921875)
        stats, loss, aux = ops.fsp_stats(z, O.PRESETS["kurt"])
        gz = ops.fsp_backward(z, 2, False, out, aux, stats.float(), loss.float(), O.PRESETS["kurt"])
        runs.append((out, idx, lev, acc, stats, loss, aux, gz))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ---- every output inside sentinel rows, through the raw entry points ----

SENT = 8   # sentinel rows (or elements) on each side: 8 rows keep every [N][D] view 16-byte aligned for fp32 and bf16


def _sentinel(n, inner, dtype, fill):
    buf = torch.full((n + 2 * SENT, *inner), fill, dtype=dtype, device=DEV)
    return buf, buf[SENT:SENT + n]


def _intact(buf, fill):
    head, tail = buf[:SENT], buf[-SENT:]
    return bool((head == fill).all()) and bool((tail == fill).all())


@pytest.mark.parametrize("d,act,inv,dtype", [(3, "tanh", False, torch.bfloat16), (5, "cauchy", True, torch.float32),
                                             (16, "sigmoid", False, torch.bfloat16), (1, "laplace", True, torch.float32),
                                             (7, "normal", False, torch.float32)])
def test_guard_rows_around_every_output(d, act, inv, dtype):
    """vqb_fsp_forward (out, idx, level_idx, accept), vqb_fsp_stats (stats, loss, aux) and vqb_fsp_backward (grad_z) write
    into views with sentinel rows around them: the sentinels stay, and every view holds the bits the ops wrappers return
    (vqb_fsp_decode's act and codes are guarded in test_instantiation)."""
    ops = _ops()
    lib = ops.lib
    N = 70_000
    a = O.ACTS.index(act)
    levels = _levels(d, 5)
    lv = torch.tensor(levels, dtype=torch.int32, device=DEV)
    z = (torch.randn(N, d, device=DEV) * 1.5).to(dtype)
    u1, u2 = torch.rand(N, d, device=DEV).to(dtype), torch.rand(N, d, device=DEV).to(dtype)
    eps = float(torch.finfo(dtype).eps)
    blocks = lib.vqb_fsp_blocks(N)
    norm = O.PRESETS["kurt"]
    dt = ops._dtype_code(z)
    st = ops._stream()
    for pert in (False, True):
        odt = torch.float32 if pert else dtype
        hi, lo, ohi = 1 - eps, eps, 1 - eps
        ref = ops.fsp_forward(z, a, inv, lv, hi, u1 if pert else None, u2 if pert else None, 0.5, lo, ohi)
        bo, out = _sentinel(N, (d,), odt, 7.0)
        bi, idx = _sentinel(N, (), torch.int32, -77)
        bl, lev = _sentinel(N, (d,), dtype, 7.0)
        ba, acc = _sentinel(blocks, (), torch.int32, -77)
        with torch.cuda.device(z.device):
            ops.check(lib.vqb_fsp_forward(z.data_ptr(), dt, N, d, a, int(inv), lv.data_ptr(), hi, u1.data_ptr() if pert else None,
                                          u2.data_ptr() if pert else None, 0.5, lo, ohi, out.data_ptr(), idx.data_ptr(),
                                          lev.data_ptr(), acc.data_ptr() if pert else None, blocks, st), "forward")
        torch.cuda.synchronize()
        assert _intact(bo, 7.0) and _intact(bi, -77) and _intact(bl, 7.0) and _intact(ba, -77)
        assert torch.equal(out, ref[0]) and torch.equal(idx, ref[1]) and torch.equal(lev, ref[2])
        if pert:
            assert int(acc.sum()) == int(ref[3])
    stats_ref, loss_ref, aux_ref = ops.fsp_stats(z, norm)
    work = torch.empty((4 * blocks + 1, d), dtype=torch.float64, device=DEV)
    bs, stats = _sentinel(4 * d, (), dtype, 7.0)
    bL, loss = _sentinel(1, (), dtype, 7.0)
    bx, aux = _sentinel(d * 8, (), torch.float64, 7.0)
    with torch.cuda.device(z.device):
        ops.check(lib.vqb_fsp_stats(z.data_ptr(), dt, N, d, ops._norm_arg(norm), work.data_ptr(), blocks, stats.data_ptr(),
                                    loss.data_ptr(), aux.data_ptr(), st), "stats")
    torch.cuda.synchronize()
    assert _intact(bs, 7.0) and _intact(bL, 7.0) and _intact(bx, 7.0)
    assert torch.equal(stats, stats_ref.reshape(-1)) and torch.equal(loss, loss_ref.reshape(1)) and torch.equal(aux, aux_ref.reshape(-1))
    g = torch.randn(N, d, device=DEV).to(dtype)
    gs, gl = torch.randn(4, d, device=DEV), torch.tensor([0.3], device=DEV)
    gz_ref = ops.fsp_backward(z, a, inv, g, aux_ref, gs, gl, norm)
    bg, gz = _sentinel(N, (d,), dtype, 7.0)
    with torch.cuda.device(z.device):
        ops.check(lib.vqb_fsp_backward(z.data_ptr(), dt, N, d, a, int(inv), g.data_ptr(), dt, aux_ref.data_ptr(), gs.data_ptr(),
                                       gl.data_ptr(), ops._norm_arg(norm), gz.data_ptr(), st), "backward")
    torch.cuda.synchronize()
    assert _intact(bg, 7.0) and torch.equal(gz, gz_ref)


# ---- planted boundaries and extreme inputs, against the kernel's formula restated in exactly rounded numpy ----

F32 = np.float32
UNIT = F32(O.UNIT_STD)


def _bf16(v):
    return torch.from_numpy(np.asarray(v, np.float32)).bfloat16().float().numpy()


def _expected_row(act, L, hi, bf, u1=None, u2=None, qrate=F32(0.5)):
    """The forward's level, accept flag and output for one element whose CDF value `act` is exact: each op of the kernel
    (include/vqb200.h, DESIGN 4.11) in correctly rounded float32, rounded to bf16 where the chain runs in bf16."""
    r = _bf16 if bf else (lambda v: F32(v))
    L = F32(L)
    c = act if np.isnan(act) else min(act, hi)
    lev = np.floor(r(F32(c) * L))
    mid = r(r(lev + F32(0.5)) / L)
    q = r(act + r(mid - act))
    acc = None
    ro = r
    if u1 is not None:
        ro = lambda v: F32(v)   # noqa: E731  (the fp32 p_max_norm promotes the output chain)
        rr = r(r(F32(u1) * F32(2)) - F32(1))
        prop = F32(act + F32(F32(1) / F32(2 * L)) * rr)
        acc = bool(prop > 0 and prop < 1)
        if F32(u2) > qrate:
            q = prop if acc else F32(act)
    out = ro(ro(F32(q) - F32(0.5)) / UNIT)
    return lev, acc, out


def _run_rows(z, levels, act, dtype, hi, u1=None, u2=None, qrate=0.5, inv=False):
    ops = _ops()
    zt = torch.tensor(z, dtype=torch.float32, device=DEV).to(dtype)
    lv = torch.tensor(levels, dtype=torch.int32, device=DEV)
    ut = [torch.tensor(u, dtype=torch.float32, device=DEV).to(dtype) if u is not None else None for u in (u1, u2)]
    return ops.fsp_forward(zt, O.ACTS.index(act), inv, lv, hi, ut[0], ut[1], qrate, 1e-6, 1 - 1e-6)


TINY = [0., -0., 2. ** -23, -(2. ** -24), 2. ** -22, 1e-40, -1e-40]   # tanh(z) = z here on any libm: act = (1 + z) / 2 in fp32
BIG = [3.4028234663852886e38, -3.4028234663852886e38, float("inf"), float("-inf"), 20., -20.]   # act exactly 1 or 0


def _tanh_act(z):
    return F32(F32(F32(np.tanh(F32(z))) + F32(1)) * F32(0.5)) if abs(z) < 1 else F32(1.0 if z > 0 else 0.0)


@pytest.mark.parametrize("hi", [1 - 2. ** -23, 0.5 - 2. ** -25, 0.5 + 2. ** -24], ids=["clamp_1-eps", "clamp_below_half", "clamp_at_act"])
def test_planted_floor_boundaries(hi):
    """act L exactly an integer (act = 1/2, L = 8) and one ulp either side; the clamp with act exactly at, above and below it;
    act = 1 and 0 (clamped to 1 - eps): levels and output bits exactly as the float32 restatement gives them."""
    z = TINY + BIG
    rows = [[v, v, v, v] for v in z]
    levels = [8, 2, 6, 5]
    out, idx, lev, _ = _run_rows(rows, levels, "tanh", torch.float32, hi)
    for i, v in enumerate(z):
        act = _tanh_act(v)
        for j, L in enumerate(levels):
            el, _, eo = _expected_row(act, L, F32(hi), False)
            assert lev[i, j].item() == el, (v, L)
            assert out[i, j].cpu().numpy().view(np.int32) == np.float32(eo).view(np.int32), (v, L, out[i, j].item(), eo)
    np.testing.assert_array_equal(idx.cpu().numpy(), (lev.cpu().numpy().astype(np.int64) * O.basis(levels)).sum(-1))


def test_planted_proposals_and_choice():
    """Proposals exactly 0 and 1 (rejected: the accept test is the open interval), one just inside, and u2 exactly equal
    to quantize_rate (not perturbed: the choice is strict) and one ulp above it."""
    up = float(np.nextafter(F32(0.5), F32(1)))
    # (z, u1, u2) per element; L = 1 gives p_max_norm = 1/2, so act = 1/2 with u1 = 0 or 1 proposes exactly 0 or 1
    cases = [(0., 0., 1.), (0., 1., 1.), (0., 0.75, 1.), (float("-inf"), 0.5, 1.), (float("inf"), 0.5, 1.),
             (0., 0.25, 0.5), (0., 0.25, up), (2. ** -23, 0.9, up)]
    levels = [1, 1, 1, 1]
    z = [[c[0]] * 4 for c in cases]
    u1 = [[c[1]] * 4 for c in cases]
    u2 = [[c[2]] * 4 for c in cases]
    out, idx, lev, acc = _run_rows(z, levels, "tanh", torch.float32, 1 - 2. ** -23, u1, u2, 0.5)
    n_acc = 0
    for i, (v, a1, a2) in enumerate(cases):
        el, ea, eo = _expected_row(_tanh_act(v), 1, F32(1 - 2. ** -23), False, a1, a2)
        n_acc += 4 * ea
        assert lev[i, 0].item() == el
        assert out[i, 0].cpu().numpy().view(np.int32) == np.float32(eo).view(np.int32), (v, a1, a2, out[i, 0].item(), eo)
    assert int(acc) == n_acc


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("act", O.ACTS)
def test_extreme_inputs(act, dtype):
    """+-0, subnormals, +-FLT_MAX and +-inf give act exactly 1/2, 1 or 0 for every CDF: levels, index and output bits as the
    restatement gives them; NaN stays NaN in the level and the output and adds digit 0 to the index; the backward's
    quantized path at the finite extremes matches float64."""
    ops = _ops()
    bf = dtype == torch.bfloat16
    vals = [0., -0., 1e-40, -1e-40, 3.4028234663852886e38, -3.4028234663852886e38, float("inf"), float("-inf")]
    if bf:
        vals[2:6] = [1e-39, -1e-39, 3.3895313892515355e38, -3.3895313892515355e38]   # bf16 subnormals and largest finite
    acts = [0.5, 0.5, 0.5, 0.5, 1., 0., 1., 0.]
    levels = [8, 5, 2, 7]
    eps = float(torch.finfo(dtype).eps)
    hi = torch.tensor(1 - eps, dtype=torch.float64).to(dtype).item()
    rows = [[v] * 4 for v in vals] + [[float("nan"), 0., 0., 0.]]
    out, idx, lev, _ = _run_rows(rows, levels, act, dtype, hi)
    for i, a in enumerate(acts):
        for j, L in enumerate(levels):
            el, _, eo = _expected_row(F32(a), L, F32(hi), bf)
            assert lev[i, j].item() == el, (vals[i], L)
            assert out[i, j].float().cpu().numpy().view(np.int32) == np.float32(eo).view(np.int32), (vals[i], L)
    assert torch.isnan(lev[-1, 0]) and torch.isnan(out[-1, 0]).item()
    exact = (np.nan_to_num(lev.float().cpu().numpy()).astype(np.int64) * O.basis(levels)).sum(-1)
    np.testing.assert_array_equal(idx.cpu().numpy(), exact)
    # the backward's quantized path at the finite extremes (statistics from a benign z, no upstream statistics gradient)
    zf = torch.tensor([[v] * 4 for v in vals[:6]], dtype=torch.float32, device=DEV).to(dtype)
    _, _, aux = ops.fsp_stats(torch.randn(64, 4, device=DEV).to(dtype), O.PRESETS["none"])
    g = torch.full_like(zf, 0.75)
    gz = ops.fsp_backward(zf, O.ACTS.index(act), False, g, aux, None, None, O.PRESETS["none"])
    ref = 0.75 / O.UNIT_STD * O.act_grad_f64(act, zf.double().cpu().numpy())
    np.testing.assert_allclose(gz.double().cpu().numpy(), ref, rtol=1e-2 if bf else 1e-6, atol=1e-30)
