"""The LFQ entropy kernels (vqb_lfq_entropy, vqb_lfq_entropy_backward) against the float64 dense oracle, every codebook
dimension d = 1..20, row lists, regimes on both sides of the 1e-5 clamp, determinism, and the d = 18 / 16384-row scale case."""
import pytest
import torch

from oracle import lfq_oracle as O
from vector_quantize_pytorch_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case(S, N, G, d, scale, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((S, N, G, d), generator=g, device=DEV) * scale
    m = torch.rand(S, generator=g, device=DEV) + 0.5
    return x, m


def _check(x, m, tau, rows=None):
    S, N, G, d = x.shape
    R = N if rows is None else rows.shape[-1]
    pse, col = ops.lfq_entropy(x, rows, R, m, tau, True)
    cp = torch.linspace(0.5, 1.5, S * G, device=DEV)
    V = torch.randn((S * G, 1 << d), device=DEV) * 1e-2
    gx = ops.lfq_entropy_backward(x, rows, R, m, tau, cp, V)
    chunks, ksplit = ops.lfq_entropy_plan(R, S * G, d, torch.cuda.get_device_properties(0).multi_processor_count, True)
    for s in range(S):
        for g in range(G):
            sg = s * G + g
            r = rows if rows is None or rows.dim() == 1 else rows[sg]
            xs = x[s, :, g] if r is None else x[s, r.long(), g]
            hs, cs = O.dense_stats(xs, float(m[s]), tau)
            torch.testing.assert_close(pse[sg], hs, rtol=2e-5, atol=1e-6 * R)
            torch.testing.assert_close(col[sg].double(), cs, rtol=2e-5, atol=1e-7 * R)
            # per-element float64 bounds of the plan that ran (oracle/lfq_oracle.py::entropy_reference)
            ref = O.entropy_reference(xs, float(m[s]), tau, float(cp[sg]), V[sg])
            pb, cb, gb = ref.bounds(chunks, ksplit)
            assert abs(float(pse[sg]) - float(ref.pse)) <= pb
            assert ((col[sg].double() - ref.colsum).abs() <= cb).all()
            got = gx[s, :, g] if r is None else gx[s, r.long(), g]
            assert ((got.double() - ref.grad).abs() <= gb).all()
    if rows is not None:   # rows outside the lists get no gradient
        hit = torch.zeros((S * G, N), dtype=torch.bool, device=DEV)
        for sg in range(S * G):
            hit[sg, (rows if rows.dim() == 1 else rows[sg]).long()] = True
        assert (gx.permute(0, 2, 1, 3).reshape(S * G, N, d)[~hit] == 0).all()


@pytest.mark.parametrize("d", list(range(1, 21)))
def test_every_d(d):
    N = 300 if d <= 12 else (40 if d <= 16 else 5)
    x, m = _case(2, N, 1, d, 1.0, d)
    _check(x, m, 1.0)


@pytest.mark.parametrize("tau,scale", [(100., 1.), (1e-3, 1.), (0.35, 0.1)], ids=["peaked", "flat", "straddle"])
def test_regimes(tau, scale):
    x, m = _case(1, 70, 2, 16, scale, 5)
    _check(x, m, tau)


def test_row_lists_shared_and_per_group():
    x, m = _case(2, 500, 3, 9, 1.0, 11)
    _check(x, m, 2.0, torch.tensor([3, 4, 99, 250, 499, 17, 18], dtype=torch.int32, device=DEV))
    per = torch.stack([torch.randperm(500, device=DEV)[:61].sort().values for _ in range(6)]).int()
    _check(x, m, 2.0, per)


def test_many_waves_of_rows():
    x, m = _case(1, 9000, 1, 10, 1.0, 3)
    _check(x, m, 3.0)


def test_deterministic():
    x, m = _case(3, 2000, 2, 12, 1.0, 9)
    a = ops.lfq_entropy(x, None, 2000, m, 5.0, True)
    b = ops.lfq_entropy(x, None, 2000, m, 5.0, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    cp = torch.ones(6, device=DEV)
    V = torch.randn(6, 4096, device=DEV)
    assert torch.equal(ops.lfq_entropy_backward(x, None, 2000, m, 5.0, cp, V), ops.lfq_entropy_backward(x, None, 2000, m, 5.0, cp, V))


def test_scale_d18_16k_rows():
    d, N, tau = 18, 16384, 100.
    x, m = _case(1, N, 1, d, 0.3, 18)
    V = torch.randn(1, 1 << d, device=DEV) * 1e-6
    cp = torch.ones(1, device=DEV) / N
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    pse, col = ops.lfq_entropy(x, None, N, m, tau, True)
    gx = ops.lfq_entropy_backward(x, None, N, m, tau, cp, V)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 64 << 20, extra
    href = torch.zeros((), dtype=torch.float64, device=DEV)
    cref = torch.zeros(1 << d, dtype=torch.float64, device=DEV)
    for i in range(0, N, 512):
        hs, cs = O.dense_stats(x[0, i:i + 512, 0], float(m[0]), tau)
        href += hs
        cref += cs
    torch.testing.assert_close(pse[0], href, rtol=2e-5, atol=0)
    torch.testing.assert_close(col[0].double(), cref, rtol=2e-5, atol=1e-7 * N)
    ref = O.entropy_reference(x[0, :, 0], float(m[0]), tau, float(cp[0]), V[0])
    pb, cb, gb = ref.bounds(*ops.lfq_entropy_plan(N, 1, d, torch.cuda.get_device_properties(0).multi_processor_count, True))
    assert abs(float(pse[0]) - float(ref.pse)) <= pb
    assert ((col[0].double() - ref.colsum).abs() <= cb).all()
    assert ((gx[0, :, 0].double() - ref.grad).abs() <= gb).all()


# ---- the row kernels: vqb_lfq_forward, vqb_lfq_backward, vqb_lfq_decode, called directly with sentinel-guarded outputs ----

from vector_quantize_pytorch_b200 import _C   # noqa: E402

GUARD = 3
SENT_F = 7.0e30
SENT_I = -77


def _guarded(shape, dtype, fill):
    """A tensor of `shape` inside a larger one: GUARD sentinel rows before and after (first axis) -> (inner view, whole)."""
    whole = torch.full((shape[0] + 2 * GUARD, *shape[1:]), fill, dtype=dtype, device=DEV)
    return whole[GUARD:GUARD + shape[0]], whole


def _guards_intact(whole, fill):
    g = torch.cat([whole[:GUARD].flatten(), whole[-GUARD:].flatten()])
    return bool((g == fill).all())


def _params(Q, d, spherical, clamp):
    from vector_quantize_pytorch_b200.lfq import code_magnitude
    s = [2.0 ** -q for q in range(Q)]
    m = [code_magnitude(v, d, spherical) for v in s]
    c = [(2.0 * 0.5 ** q if clamp else 0.) for q in range(Q)]
    return torch.tensor([s, m, c], dtype=torch.float32, device=DEV)


def _forward(z, params, Q, n_active, residual, training, spherical, rowmask=None, commit=True):
    N, G, d = z.shape
    dt = _C.DTYPE_BF16 if z.dtype == torch.bfloat16 else _C.DTYPE_F32
    out, out_w = _guarded((N, G, d), z.dtype, SENT_F)
    idx_w = torch.full((N + 2 * GUARD, G, Q + 2), SENT_I, dtype=torch.int64, device=DEV)   # strided: 2 spare columns per row
    idx = idx_w[GUARD:GUARD + N, :, 1:1 + Q]
    ent, ent_w = _guarded((n_active, N, G, d), torch.float32, SENT_F) if training else (None, None)
    blocks = _C.lib.vqb_lfq_forward_blocks(N, G)
    com, com_w = _guarded((n_active, blocks), torch.float64, SENT_F) if commit else (None, None)
    rc = _C.lib.vqb_lfq_forward(z.data_ptr(), dt, N, G, d, Q, n_active, int(residual), int(training), int(spherical), params.data_ptr(),
                                out.data_ptr(), idx.data_ptr(), idx.stride(0), idx.stride(1), idx.stride(2),
                                ent.data_ptr() if ent is not None else None, rowmask.data_ptr() if rowmask is not None else None,
                                com.data_ptr() if com is not None else None, blocks, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(out_w, SENT_F)
    spare = torch.cat([idx_w[:GUARD].flatten(), idx_w[-GUARD:].flatten(), idx_w[:, :, 0].flatten(), idx_w[:, :, -1].flatten()])
    assert bool((spare == SENT_I).all())
    if ent is not None:
        assert _guards_intact(ent_w, SENT_F)
    if com is not None:
        assert _guards_intact(com_w, SENT_F)
    return out, idx, ent, (com.sum(1) if com is not None else None)


def _cases():
    out = []
    for d in range(1, 21):
        bf = d % 3 == 0
        plain = d % 7 == 0
        Q = 1 if plain else 2 + d % 4
        out.append(dict(d=d, bf=bf, sph=d % 2 == 0, clamp=d % 4 in (1, 2), Q=Q, n_active=Q if plain else Q - d % 2,
                        training=d % 5 != 0, G=1 + d % 3, residual=not plain, N=97 + 13 * d))
    # 64 stages: the residual shrinks by 2^-q and a spherical chain's signs then hang on rounding, so these two are not spherical
    out.append(dict(d=6, bf=False, sph=False, clamp=True, Q=64, n_active=50, training=True, G=2, residual=True, N=301))
    out.append(dict(d=9, bf=True, sph=False, clamp=True, Q=64, n_active=64, training=True, G=1, residual=True, N=150))
    out.append(dict(d=4, bf=False, sph=False, clamp=False, Q=2, n_active=2, training=True, G=2, residual=True, N=300000))   # waves
    return out


def _id(c):
    return f"d{c['d']}_{'bf16' if c['bf'] else 'f32'}_q{c['n_active']}of{c['Q']}_n{c['N']}{'_sph' if c['sph'] else ''}" \
           f"{'_clamp' if c['clamp'] else ''}{'' if c['training'] else '_eval'}"


@pytest.mark.parametrize("c", _cases(), ids=_id)
def test_row_kernels_against_oracle(c):
    d, Q, na, G, N = c["d"], c["Q"], c["n_active"], c["G"], c["N"]
    g = torch.Generator(device=DEV).manual_seed(d * 1000 + Q)
    dtype = torch.bfloat16 if c["bf"] else torch.float32
    z = (torch.randn((N, G, d), generator=g, device=DEV) * 1.5).to(dtype)
    params = _params(Q, d, c["sph"], c["clamp"])
    rowmask = (torch.rand(N, generator=g, device=DEV) > 0.25).to(torch.uint8)
    out, idx, ent, com = _forward(z, params, Q, na, c["residual"], c["training"], c["sph"], rowmask)
    ro, ri, rent, rq = O.chain(z, params, Q, na, c["residual"], c["training"], c["sph"])
    # indices and values follow the signs and the explicitly rounded chain: exact, except that the l2norm's sum order and
    # bf16 rounding of the norm may differ from torch's reduction by an ulp (spherical)
    if c["sph"]:
        assert (idx != ri).float().mean() <= 1e-3
        torch.testing.assert_close(out.float(), ro.float(), rtol=2e-2 if c["bf"] else 2e-6, atol=1e-6)
    else:
        assert torch.equal(idx, ri)
        assert torch.equal(out, ro)
        if c["training"]:
            assert torch.equal(ent, rent)
    if c["training"]:
        cref = ((rent.double() - rq.double()) ** 2 * rowmask.double()[None, :, None, None]).sum((1, 2, 3))
        torch.testing.assert_close(com, cref, rtol=1e-5 if not c["sph"] else 1e-3, atol=1e-9)
    # backward: grad_out, an entropy gradient and commitment coefficients, against float64 autograd of the chain
    gout = torch.randn((N, G, d), generator=g, device=DEV).to(dtype)
    gent = torch.randn((na, N, G, d), generator=g, device=DEV) * 0.1 if c["training"] else None
    cc = torch.linspace(0.1, 0.3, Q, device=DEV) if c["training"] else None
    gz, gz_w = _guarded((N, G, d), dtype, SENT_F)
    dt = _C.DTYPE_BF16 if c["bf"] else _C.DTYPE_F32
    go = gout.contiguous()
    rc = _C.lib.vqb_lfq_backward(z.data_ptr(), dt, N, G, d, Q, na, int(c["residual"]), int(c["training"]), int(c["sph"]),
                                 params.data_ptr(), go.data_ptr(), gent.data_ptr() if gent is not None else None,
                                 cc.data_ptr() if cc is not None else None, rowmask.data_ptr(), gz.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(gz_w, SENT_F)
    # float64 gradient along the discrete path (the signs) of the chain in its own dtype
    ref_w, qs = _chain_grad(z, z.dtype, params, Q, na, c, gout, gent, cc, rowmask)   # the reference's own ops, in its dtype
    ref64, _ = _chain_grad(z, torch.float64, params, Q, na, c, gout, gent, cc, rowmask, force_q=qs)
    # no worse than the reference's own ops in the chain's dtype, measured against float64 (2e-5 of the largest value at least).
    # A bf16 chain may reach 1.5 times torch's deviation: the kernel rounds its backward at other points than autograd's
    # per-op bf16 rounding (DESIGN §4.10 gives the measured ratio)
    factor = 1.5 if c["bf"] else 1.0
    bound = max(factor * float((ref_w - ref64).abs().max()), 2e-5 * float(ref64.abs().max()), 1e-9)
    err = float((gz.double() - ref64).abs().max())
    assert err <= bound, (err, bound)


def _chain_grad(z, dtype, params, Q, na, c, gout, gent, cc, rowmask, force_q=None):
    zz = z.detach().to(dtype).requires_grad_(True) if dtype == torch.float64 else z.detach().clone().requires_grad_(True)
    o, _, e, qv = O.chain(zz, params, Q, na, c["residual"], c["training"], c["sph"], dtype=dtype, force_q=force_q)
    if not c["training"]:
        return torch.zeros(z.shape, dtype=torch.float64, device=DEV), qv   # eval: the output is q, no gradient reaches z
    L = (o.to(e.dtype) * gout.to(e.dtype)).sum() + (e * gent.to(e.dtype)).sum()
    L = L + ((cc[:na].to(e.dtype) / 2)[:, None, None, None] * (e - qv.detach()) ** 2 * rowmask.to(e.dtype)[None, :, None, None]).sum()
    L.backward()
    return zz.grad.double(), qv.detach()


@pytest.mark.parametrize("idx64", [False, True])
@pytest.mark.parametrize("d", [1, 7, 13, 20])
def test_decode_against_oracle(d, idx64):
    N, G, Q = 211, 2, 5
    g = torch.Generator(device=DEV).manual_seed(d)
    itype = torch.int64 if idx64 else torch.int32
    ind = torch.randint(0, 1 << d, (N, G, Q), generator=g, device=DEV)
    ind[torch.rand((N, G, Q), generator=g, device=DEV) < 0.1] = -1
    whole = torch.full((N + 2 * GUARD, Q + 3, G), SENT_I, dtype=itype, device=DEV)   # strided (row, stage, group) layout
    view = whole[GUARD:GUARD + N, 1:1 + Q].permute(0, 2, 1)
    view.copy_(ind)
    vals = torch.tensor([1.0, 0.5, 0.3, 0.25, 0.125], device=DEV)
    out, out_w = _guarded((N, G, d), torch.float32, SENT_F)
    cbuf, cbuf_w = _guarded((Q * N, G, d), torch.float32, SENT_F)
    rc = _C.lib.vqb_lfq_decode(view.data_ptr(), int(idx64), view.stride(0), view.stride(1), view.stride(2), N, G, d, Q,
                               vals.data_ptr(), out.data_ptr(), cbuf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(out_w, SENT_F) and _guards_intact(cbuf_w, SENT_F)
    bits = ((ind[..., None] >> torch.arange(d - 1, -1, -1, device=DEV)) & 1).float() * 2 - 1
    ref = torch.where(ind[..., None] == -1, torch.zeros_like(bits), bits * vals[None, None, :, None])   # (N, G, Q, d)
    assert torch.equal(cbuf.view(Q, N, G, d), ref.permute(2, 0, 1, 3))
    acc = torch.zeros((N, G, d), device=DEV)
    for q in range(Q):
        acc = acc + ref[:, :, q]
    assert torch.equal(out, acc)


def test_module_scale_d18_16k_rows_memory():
    """LFQ(codebook_size=2^18) training forward and backward on 16384 rows: the whole module, row kernels included."""
    import vector_quantize_pytorch_b200 as vqb
    torch.manual_seed(0)
    mod = vqb.LFQ(codebook_size=1 << 18).to(DEV).train()
    x = (torch.randn(1, 16384, 18, device=DEV) * 0.3).requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out, _, aux = mod(x)
    (out.sum() + aux).backward()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 64 << 20, extra
    assert torch.isfinite(x.grad).all()
