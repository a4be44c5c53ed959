"""The row kernels' float64 reference and bounds (oracle/lfq_oracle.py::chain_reference, check_rows) on the CPU: they hold
for a restatement of the kernels' fp32 and bf16 arithmetic, and each seeded defect falls outside them."""
import pytest
import torch

from oracle import lfq_oracle as O

DEFECTS = ["no_tanh_jacobian", "no_projection", "projection_below_clamp", "entropy_grad_dropped", "entropy_grad_wrong_stage",
           "commit_on_masked_row", "bit_order_reversed", "residual_off_by_one", "stage0_smallest_bit_flipped"]


def _rw(v, bf):
    return v.bfloat16().float() if bf else v


def emulate(z, params, Q, n_active, residual, training, spherical, gout, gent, cc, rowmask, grid, defect=None):
    """vqb_lfq_forward and vqb_lfq_backward restated on the CPU: fp32 ops, each result rounded to the chain's dtype where
    the kernels round (the norm as a sequential fp32 sum of squares, torch's tanh for tanhf).  `defect` seeds one wrong
    step.  -> (indices (N, G, Q), out (N, G, d), entropy inputs (n_active, N, G, d), commitment partials (n_active, grid),
    d z (N, G, d)), in the kernels' output dtypes."""
    bf = z.dtype == torch.bfloat16
    N, G, d = z.shape
    p = params.float()
    eps = _rw(torch.tensor(1e-12), bf)
    live = torch.ones(N) if rowmask is None else (rowmask != 0).float()
    if defect == "commit_on_masked_row":
        live = torch.ones(N)
    live = live[:, None]

    def stage_input(r, q):
        s, c = p[0, q], p[2, q]
        x, t, nrm, proj = r.clone(), None, None, None
        if c != 0:
            t = _rw(torch.tanh(_rw(x / c, bf)), bf)
            x = _rw(t * c, bf)
        if spherical:
            ss = torch.zeros((N, G))
            for j in range(d):
                ss = ss + x[..., j] * x[..., j]
            rn = _rw(ss.sqrt(), bf)[..., None]
            nrm = torch.maximum(rn, eps)
            proj = rn >= eps
            x = _rw(_rw(x / nrm, bf) * s, bf)
        return x, t, nrm, proj

    def stage_output(x, q):
        m = p[1, q]
        qv = torch.where(x > 0, m, -m)
        return qv, _rw(x + (qv - x), bf) if training else _rw(qv, bf)

    bitw = 2 ** (torch.arange(d) if defect == "bit_order_reversed" else torch.arange(d - 1, -1, -1))
    r = z.float()
    o = torch.zeros_like(r)
    idx = torch.full((N, G, Q), -1, dtype=torch.int64)
    ents, items = [], []
    for q in range(n_active):
        x, _, _, _ = stage_input(r, q)
        qv, ov = stage_output(x, q)
        idx[..., q] = ((x > 0).long() * bitw).sum(-1)
        if defect == "stage0_smallest_bit_flipped" and q == 0:   # the bit of each item's element nearest to zero
            idx[..., q] ^= 1 << (d - 1 - x.abs().argmin(-1))
        ents.append(x)
        e = x - qv
        items.append(torch.where(live != 0, (e * e).double().sum(-1), 0.))   # masked rows add nothing (inf * 0 would)
        if not (defect == "residual_off_by_one" and q == 0):
            r = _rw(r - ov, bf)
        o = _rw(o + ov, bf) if residual else ov
    blk = O.item_blocks(N, G, grid).flatten()
    commit = torch.zeros((n_active, grid), dtype=torch.float64).index_add_(1, blk, torch.stack(items).flatten(1))
    # backward: every stage recomputed from z
    r = z.float()
    acc = torch.zeros_like(r)
    for q in range(n_active):
        s, c = p[0, q], p[2, q]
        x, t, nrm, proj = stage_input(r, q)
        qv, ov = stage_output(x, q)
        gi = gout.float() if training else torch.zeros_like(x)
        if gent is not None and not (defect == "entropy_grad_dropped" and q == n_active - 1):
            gi = gi + gent[(q + 1) % n_active if defect == "entropy_grad_wrong_stage" else q]
        if cc is not None:
            gi = gi + cc[q] * live[..., None] * (x - qv)
        g = _rw(gi, bf)
        gx = g
        if spherical:
            g = _rw(g * s, bf)
            y = x / s
            dot = torch.zeros((N, G, 1))
            for j in range(d):
                dot = dot + g[..., j:j + 1] * y[..., j:j + 1]
            if defect == "no_projection":
                proj = torch.zeros_like(proj)
            elif defect == "projection_below_clamp":
                proj = torch.ones_like(proj)
            gx = torch.where(proj, g - y * dot, g) / nrm
        if c != 0 and defect != "no_tanh_jacobian":
            gx = gx * (1 - t * t)
        acc = acc + _rw(gx, bf)
        if not (defect == "residual_off_by_one" and q == 0):
            r = _rw(r - ov, bf)
    gz = acc.to(z.dtype)
    return idx, o.to(z.dtype), torch.stack(ents), commit, gz


def _params(Q, d, spherical, clamp):
    from vector_quantize_pytorch_b200.lfq import code_magnitude
    s = [0.75 * 2.0 ** -q for q in range(Q)]
    m = [code_magnitude(v, d, spherical) for v in s]
    c = [(1.5 * 0.5 ** q if (clamp == "all" or (clamp == "some" and q % 2 == 0)) else 0.) for q in range(Q)]
    return torch.tensor([s, m, c], dtype=torch.float32)


def _inputs(N, G, d, Q, n_active, dtype, seed, planted=True):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn((N, G, d), generator=g) * 1.2
    if planted:
        z[0] = 0.
        z[1] = 3e-13 / d ** 0.5          # norm below the l2norm clamp 1e-12
        z[2, :, 0] = 0.75                # stage 0 input exactly m (non-spherical): the next residual is exactly 0
        z[3] = 40.                       # tanh saturates
        z[4] = 2.0 ** -140               # subnormal
    z = z.to(dtype)
    gout = torch.randn((N, G, d), generator=g).to(dtype)
    gent = torch.randn((n_active, N, G, d), generator=g) * 0.3
    cc = torch.linspace(0.4, 0.9, Q)
    rowmask = (torch.rand(N, generator=g) > 0.3).to(torch.uint8)
    return z, gout, gent, cc, rowmask


def _run(z, params, Q, n_active, residual, training, spherical, gout, gent, cc, rowmask, grid=3, defect=None):
    _, it, xt, _ = O.chain(z, params, Q, n_active, residual, training, spherical)
    ref = O.chain_reference(z, params, Q, n_active, residual, training, spherical, gout, gent, cc, rowmask, signs=xt > 0)
    ik, ok, ek, ck, gk = emulate(z, params, Q, n_active, residual, training, spherical, gout, gent, cc, rowmask, grid, defect)
    return O.check_rows(ref, n_active, it, xt, ik, ok, ek, ck, grid, rowmask, gk, spherical, params)


CASES = [(dt, sph, clamp, training) for dt in ("f32", "bf16") for sph in (False, True) for clamp in ("none", "some", "all")
         for training in (True, False)]


@pytest.mark.parametrize("dt,sph,clamp,training", CASES)
@pytest.mark.parametrize("d", [1, 3, 8])
def test_bounds_hold_for_the_kernel_arithmetic(dt, sph, clamp, training, d):
    dtype = torch.bfloat16 if dt == "bf16" else torch.float32
    Q, na = 5, 4
    z, gout, gent, cc, rowmask = _inputs(120, 2, d, Q, na, dtype, d)
    params = _params(Q, d, sph, clamp)
    rep = _run(z, params, Q, na, True, training, sph, gout, gent, cc, rowmask)
    assert not rep.violations, rep.violations
    if not sph or not training:   # exactly reproducible arithmetic: no excused row
        assert rep.excused == 0
    assert rep.ratios["grad"] <= 1 and rep.ratios["out"] <= 1


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_deep_spherical_chain_is_checkable(dt):
    """64 spherical stages (scales 2^-q), the clamp on even stages: the rule excuses no item of the restated kernel, whose
    signs follow the torch chain's on every stage, and a bit flipped at stage 0 is still caught."""
    Q = 64
    dtype = torch.bfloat16 if dt == "bf16" else torch.float32
    params = _params(Q, 5, True, "some")
    z, gout, gent, cc, rowmask = _inputs(200, 1, 5, Q, Q, dtype, 11, planted=False)
    rep = _run(z, params, Q, Q, True, True, True, gout, gent, cc, rowmask)
    assert not rep.violations, rep.violations
    assert rep.excused == 0
    assert _run(z, params, Q, Q, True, True, True, gout, gent, cc, rowmask, defect="stage0_smallest_bit_flipped").violations


def test_no_sign_window_where_the_stage_input_is_exact():
    """bf16, spherical, training, d = 16, no clamp: stage 0 normalises z itself, so its sign is z's and no correct kernel
    can differ from torch on any stage-0 bit.  The slack is that of the value before the l2norm (0 here), not the stage
    input's bound (about 2^-8 s), so no stage-0 element lies inside it, and flipping each item's stage-0 bit nearest to
    zero is a violation rather than an excused item."""
    d, Q = 16, 3
    params = _params(Q, d, True, "none")
    z, gout, gent, cc, rowmask = _inputs(800, 1, d, Q, Q, torch.bfloat16, 2, planted=False)
    _, it, xt, _ = O.chain(z, params, Q, Q, True, True, True)
    ref = O.chain_reference(z, params, Q, Q, True, True, True, gout, gent, cc, rowmask, signs=xt > 0)
    assert int((xt[0].double().abs() <= 2 * ref.sign_b[0]).sum()) == 0
    assert float(ref.sign_b[0].max()) < 1e-30
    ok = _run(z, params, Q, Q, True, True, True, gout, gent, cc, rowmask)
    assert not ok.violations and ok.excused == 0
    bad = _run(z, params, Q, Q, True, True, True, gout, gent, cc, rowmask, defect="stage0_smallest_bit_flipped")
    assert any("index bit" in v for v in bad.violations)


def _teeth_case(defect):
    """A case in which the defect changes the answer: the stage it touches is there and matters."""
    sph = defect in ("no_projection", "projection_below_clamp", "stage0_smallest_bit_flipped")
    clamp = "none" if sph else "all"   # stage Jacobians that differ, so that a gradient on the wrong stage shows
    d, Q, na = 4, 3, 3
    z, gout, gent, cc, rowmask = _inputs(64, 2, d, Q, na, torch.float32, 5)
    return z, _params(Q, d, sph, clamp), Q, na, True, True, sph, gout, gent, cc, rowmask


@pytest.mark.parametrize("defect", DEFECTS)
def test_bounds_have_teeth(defect):
    args = _teeth_case(defect)
    assert not _run(*args).violations
    rep = _run(*args, defect=defect)
    assert rep.violations, defect


def test_projection_below_clamp_is_caught_on_the_small_norm_row():
    """The clamp branch alone: only row 1 (||z|| = 3e-13 < 1e-12) differs, and it falls outside its bound."""
    z, params, Q, na, res, tr, sph, gout, gent, cc, rowmask = _teeth_case("projection_below_clamp")
    ok = emulate(z, params, Q, na, res, tr, sph, gout, gent, cc, rowmask, 3)[4]
    bad = emulate(z, params, Q, na, res, tr, sph, gout, gent, cc, rowmask, 3, "projection_below_clamp")[4]
    rows = (ok != bad).flatten(1).any(1).nonzero().flatten().tolist()
    assert rows == [1]
    rep = _run(z, params, Q, na, res, tr, sph, gout, gent, cc, rowmask, defect="projection_below_clamp")
    assert any("gradient" in v for v in rep.violations)
