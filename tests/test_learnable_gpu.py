"""GPU checks of codebooks learnt by gradient (learnable_codebook, sync_update_v, DiVeQ on VectorQuantize and ResidualVQ):

(a) replay of the reference's training steps (tests/golden/learnable/, oracle/gen_golden_learnable.py), chained with our own SGD
    steps; the reference's RNG draws (k-means / dead-code samples, DiVeQ noise) are substituted for ours;
(b) the vqb_diveq kernel, forward and backward, against float64 over several waves of rows, every D class, both dtypes and
    rows with e = q - x = 0;
(c) the codebook gradient (statistics chain) against float64 at N = 262144;
(d) an optimizer step between two forwards: the next search (layered and one-call ResidualVQ) uses the updated codebook.
"""
import numpy as np
import pytest
import torch

from learnable_golden import Fixture, names

pytestmark = pytest.mark.gpu
DEV = "cuda"
U_BF16 = 2.0 ** -8
U_F32 = 2.0 ** -24


class _Replay:
    """Hands out the reference's recorded draws in call order in place of torch.randperm / torch.randint / the DiVeQ noise."""

    def __init__(self, draws):
        self.draws = list(draws)

    def take(self, kind, device, dtype=None):
        assert self.draws, f"the module drew more from the RNG than the reference ({kind})"
        k, a = self.draws.pop(0)
        assert k == kind, (k, kind)
        t = torch.from_numpy(np.array(a)).to(device)
        return t.to(dtype) if dtype is not None else t


def _install(monkeypatch, replay):
    import vector_quantize_pytorch_b200.vector_quantize as vqm
    monkeypatch.setattr(torch, "randperm", lambda *a, device=None, **k: replay.take("randperm", device))
    monkeypatch.setattr(torch, "randint", lambda *a, device=None, **k: replay.take("randint", device))
    monkeypatch.setattr(vqm, "diveq_noise", lambda like: replay.take("randn_like", like.device, like.dtype))


def _bf16_grad_bound(f, s, x_rows, G_rows, idx, K, q_rows):
    """One bf16 rounding per summed term: the reference rounds every gradient row to bf16 before the fp32 sum over the rows of
    a code, so |ours - reference| <= 2^-8 * sum_{n -> k} |row_n| per element, doubled for the bf16 sum of two such rows (output
    path + commitment), plus the fp32 chain."""
    kw = f.kw
    numel = x_rows.size
    mag = np.abs(G_rows) * (1.0 + kw.get("sync_update_v", 0.0))
    if kw.get("directional_reparam") or kw.get("diveq"):
        e = q_rows - x_rows
        ne = np.linalg.norm(e, axis=-1, keepdims=True)
        mag = mag + np.linalg.norm(G_rows, axis=-1, keepdims=True) * np.abs(e) / np.maximum(ne, 1e-30)
    mag = mag + 2.0 * f.meta["lw"] * np.abs(q_rows - x_rows) / numel
    out = np.zeros((K, x_rows.shape[1]))
    np.add.at(out, idx, mag)
    return 2.0 * U_BF16 * out + 1e-6


@pytest.mark.parametrize("name", names())
def test_learnable_replays_reference(name, monkeypatch):
    import vector_quantize_pytorch_b200 as m
    f = Fixture(name)
    bf16 = f.meta["dtype"] == "bfloat16"
    dt = torch.bfloat16 if bf16 else torch.float32
    mod = f.build(m).to(DEV)
    mod.load_state_dict({k: torch.from_numpy(v) for k, v in f.state().items()})
    mod.train()
    opt = torch.optim.SGD(mod.parameters(), lr=f.meta["lr"])
    params = dict(mod.named_parameters())
    for s in range(f.meta["steps"]):
        if bf16 and s:
            # bf16: each step starts from the reference's state — the (bounded) bf16 gradient differences would otherwise
            # compound into the next step's codebook; the fp32 replays chain our own SGD steps
            mod.load_state_dict({k: torch.from_numpy(v) for k, v in f.state(s).items()})
        replay = _Replay(f.draws(s))
        with monkeypatch.context() as mp:
            _install(mp, replay)
            x = torch.from_numpy(f[f"x_{s}"]).to(DEV, dt).requires_grad_(f.meta["x_grad"])
            G = torch.from_numpy(f[f"G_{s}"]).to(DEV)
            opt.zero_grad(set_to_none=True)
            out, ind, loss = mod(x)
        assert not replay.draws, "the module drew less from the RNG than the reference"
        ((out.float() * G).sum() + f.meta["lw"] * loss.float().sum()).backward()
        pg_ref = f.pgrads(s)
        if bf16:
            targets = _check_bf16_step(f, s, out, ind, x.grad, params, pg_ref, loss.detach().float().cpu().numpy())
        else:
            assert torch.equal(ind.cpu(), torch.from_numpy(f[f"ind_{s}"])), f"indices differ at step {s}"
            tol = dict(rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(out.detach().float().cpu().numpy(), f[f"out_{s}"], **tol)
            np.testing.assert_allclose(loss.detach().float().cpu().numpy(), f[f"loss_{s}"], **tol)
            if f.meta["x_grad"]:
                np.testing.assert_allclose(x.grad.float().cpu().numpy(), f[f"xgrad_{s}"], **tol)
            for n, p in params.items():
                got = p.grad.cpu().numpy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
                np.testing.assert_allclose(got, pg_ref[n], **tol, err_msg=f"{n} step {s}")
        opt.step()
        post = mod.state_dict()
        for k, v in f.post(s).items():
            got = post[k].float().cpu().numpy()
            if bf16 and f.kw.get("shared_codebook") and k.endswith("_codebook.embed"):
                k_param = "layers.0._codebook.embed"     # every layer's `embed` key is the one shared parameter
            else:
                k_param = k
            if bf16 and k_param in targets:
                # SGD from the reference's pre-step state: |ours - target| <= lr * (gradient bound) + the fp32 rounding of each
                # side's update; the target is the reference's step (or, where later-stage rows took the other side of a near
                # tie, the step with the oracle's gradient for our own indices)
                want, gb = targets[k_param]
                err = np.abs(got - want)
                assert np.all(err <= f.meta["lr"] * gb + 2.0 ** -23 * np.abs(want) + 1e-30), f"{k} after step {s}"
            else:
                np.testing.assert_allclose(got, v.astype(np.float32), rtol=1e-5, atol=1e-5, err_msg=f"{k} after step {s}")


# ---- bf16 bounds.  U = 2^-8: every value torch computes in bf16 is rounded once per op to a relative 2^-8.  The reference's
# rotation trick is a chain of 8 such ops per element (norms, divisions, two dot products, two scaled terms, the sum, the scale),
# which vqb_rotate evaluates in fp32 and rounds once: 8 U per summed term for the estimator values and their backward.
EST_OPS = 8


def _rotation_terms(r, c, G):
    """Per-element magnitude of the terms of the rotation trick's backward (vqp:287-318) at (r, c): lam (|g| + 2 |g|.|w| |w|
    + 2 |g|.|q| |u|), float64 rows."""
    nr = np.linalg.norm(r, axis=-1, keepdims=True)
    nc = np.linalg.norm(c, axis=-1, keepdims=True)
    u, q = r / np.maximum(nr, 1e-6), c / np.maximum(nc, 1e-6)
    w = (u + q) / np.maximum(np.linalg.norm(u + q, axis=-1, keepdims=True), 1e-6)
    lam = nc / np.maximum(nr, 1e-6)
    aG = np.abs(G)
    return lam * (aG + 2 * (aG * np.abs(w)).sum(-1, keepdims=True) * np.abs(w) + 2 * (aG * np.abs(q)).sum(-1, keepdims=True) * np.abs(u))


def _value_terms(f, r, c):
    """Per-element magnitude of the terms of a stage's estimator VALUE, scaled so that EST_OPS * U * terms bounds its bf16
    rounding: the rotation trick's terms (its 8 ops), straight-through's x + (q - x) (2 ops), or the code itself (exact)."""
    if not f.meta["x_grad"] or f.kw.get("route_gradients_to_input") is False or f.kw.get("diveq"):
        return np.zeros_like(r)
    if f.kw.get("rotation_trick", True):
        return _rotation_terms(r, c, r)
    return (np.abs(r) + np.abs(c)) * 2 / EST_OPS


def _est_terms(f, r, c, G):
    kw = f.kw
    if not f.meta["x_grad"] or kw.get("route_gradients_to_input") is False or kw.get("diveq"):
        return np.zeros_like(r)
    if kw.get("directional_reparam"):
        e = c - r
        ne = np.linalg.norm(e, axis=-1, keepdims=True)
        return np.abs(G) + np.linalg.norm(G, axis=-1, keepdims=True) * np.abs(e) / np.maximum(ne, 1e-30)
    if kw.get("rotation_trick", True):
        return _rotation_terms(r, c, G)
    return np.abs(G)


def _sums(rows, idx, K):
    out = np.zeros((K, rows.shape[1]))
    np.add.at(out, idx, rows)
    return out


def _check_bf16_step(f, s, out, ind, xgrad, params, pg_ref, loss):
    """Checks one bf16 step against the reference with per-element bounds; returns {param: (post-step target, gradient bound)}."""
    from oracle import learnable_oracle as O
    kw, lw, U = f.kw, f.meta["lw"], U_BF16
    x, G = f[f"x_{s}"].astype(np.float64), f[f"G_{s}"].astype(np.float64)
    ref_ind, ref_out = f[f"ind_{s}"], f[f"out_{s}"].astype(np.float64)
    state = f.state(s)
    got_ind = ind.cpu().numpy()
    got_out = out.detach().float().cpu().numpy().astype(np.float64)
    got_xg = xgrad.float().cpu().numpy().astype(np.float64) if xgrad is not None else None
    ref_xg = f[f"xgrad_{s}"].astype(np.float64) if f.meta["x_grad"] else None
    w = kw.get("commitment_weight", 1.0) if not (kw.get("directional_reparam") or kw.get("diveq")) else 0.0
    if f.meta["cls"] == "VectorQuantize":
        assert np.array_equal(got_ind, ref_ind), f"indices differ at step {s}"
        xr, Gr, idx = f.vq_rows(x), f.vq_rows(G), f.vq_index_rows(ref_ind)
        key = "_codebook.embed"
        C = state[key][0].astype(np.float64)
        c = O.round_bf16(C[idx])
        commit = 2.0 * lw * w * np.abs(c - xr) / xr.size
        # output: x and the code (DiVeQ: x + u ||e||)
        b_out = EST_OPS * U * (np.abs(xr) + np.abs(c)) + 1e-30
        b_xg = EST_OPS * U * (_est_terms(f, xr, c, Gr) + commit)
        assert np.all(np.abs(f.vq_rows(got_out) - f.vq_rows(ref_out)) <= b_out), f"output step {s}"
        if ref_xg is not None:
            assert np.all(np.abs(f.vq_rows(got_xg) - f.vq_rows(ref_xg)) <= b_xg + 1e-30), f"x.grad step {s}"
        gb = _bf16_grad_bound(f, s, xr, Gr, idx, C.shape[0], c)
        grads = {key: (pg_ref[key][0], gb)}
        # the mse and its weighting are each rounded to bf16 once
        np.testing.assert_allclose(loss, f[f"loss_{s}"], rtol=2 * U, err_msg=f"loss step {s}")
        all_agree = True
    else:
        Q = kw["num_quantizers"]
        D = x.shape[-1]
        xr, Gr = x.reshape(-1, D), G.reshape(-1, D)
        gi, ri = got_ind.reshape(-1, Q), ref_ind.reshape(-1, Q)
        keys = [f"layers.{0 if kw.get('shared_codebook') else q}._codebook.embed" for q in range(Q)]
        books = [state[k][0].astype(np.float64) for k in keys]
        assert np.array_equal(gi[:, 0], ri[:, 0]), f"stage 0 indices differ at step {s}"
        # stage q searches r_q, which carries the estimator values of the stages before it: ours and the reference's each lie
        # within dR_q = sum_{p<q} 8 U (terms of stage p's estimator value) of the residual the oracle forms with the codes; a row
        # whose first disagreeing stage has its two candidates within that perturbation of a tie is excused (4 ||dR|| ||c1 - c2||
        # on the squared distances)
        r, T, dR = xr.copy(), np.abs(xr), np.zeros_like(xr)
        losses_ref = f[f"loss_{s}"]
        agree = np.ones(len(xr), bool)
        est, commit_rows, Ts = np.zeros_like(xr), [], []
        for q in range(Q):
            C = books[q]
            if q:
                new = agree & (gi[:, q] != ri[:, q])
                if new.any():
                    rr, c1, c2 = r[new], C[gi[new, q]], C[ri[new, q]]
                    gap = np.abs(((rr - c1) ** 2).sum(-1) - ((rr - c2) ** 2).sum(-1))
                    dr = np.linalg.norm(dR[new], axis=-1)
                    slack = 4 * dr * np.linalg.norm(c1 - c2, axis=-1) + 2.0 ** -20 * ((rr ** 2).sum(-1) + (c1 ** 2).sum(-1))
                    assert np.all(gap <= slack), f"stage {q} indices differ beyond a near tie at step {s}"
                    agree &= ~new
            c = O.round_bf16(C[gi[:, q]])
            est += _est_terms(f, r, c, Gr)
            commit_rows.append(2.0 * lw * w * np.abs(c - r) / xr.size)
            Ts.append(dR.copy())
            # stage loss w mse(c, r): its perturbation through r, plus the bf16 rounding of the mse and its weighting
            b_loss = w * 2.0 * (np.abs(c - r) * dR)[agree].sum() / xr.size + 2 * U * abs(losses_ref[q]) + 1e-9
            if agree.all():
                assert abs(loss[q] - losses_ref[q]) <= b_loss, f"stage {q} loss step {s}"
            dR = dR + EST_OPS * U * _value_terms(f, r, c)
            r = O.round_bf16(r - c)
            T = T + np.abs(c)
        # quantized_out: the stages' values (within dR) summed in bf16, one rounding per partial sum
        b_out = dR + 2 * U * (T + np.abs(ref_out.reshape(-1, D)))
        err = np.abs(got_out.reshape(-1, D) - ref_out.reshape(-1, D))
        assert np.all(err[agree] <= b_out[agree]), f"output step {s}"
        if ref_xg is not None:
            b_xg = EST_OPS * U * (est + sum(commit_rows)) + sum(2.0 * lw * w / xr.size * t for t in Ts)
            err = np.abs(got_xg.reshape(-1, D) - ref_xg.reshape(-1, D))
            assert np.all(err[agree] <= b_xg[agree] + 1e-30), f"x.grad step {s}"
        # codebook gradients: against the reference when every row agrees, else against the oracle's gradient for our indices;
        # one bf16 rounding per summed row (doubled: the bf16 sum of two rows) plus the residual perturbation of each commit row
        all_agree = bool(agree.all())
        noise = f.noise(s)
        _, _, _, _, o_grads = O.rvq_rows(xr, Gr, books, x_grad=f.meta["x_grad"], lw=lw, bf16=True, given_idx=gi, commit_weight=w,
                                         diveq_var=5e-3 if kw.get("diveq") else None,
                                         noise=None if noise is None else noise.reshape(-1, D))
        grads = {}
        for q, k in enumerate(keys):
            K = books[q].shape[0]
            # one bf16 rounding per summed commitment row, plus each row's perturbation through its residual (within dR_q)
            gb = 2.0 * U * _sums(commit_rows[q], gi[:, q], K) + _sums(2.0 * lw * w / xr.size * Ts[q], gi[:, q], K) + 1e-9
            want = pg_ref[k][0] if all_agree else o_grads[q]
            if k in grads:
                grads[k] = (grads[k][0] if all_agree else grads[k][0] + want, grads[k][1] + gb)
            else:
                grads[k] = (want, gb)
    targets = {}
    for k, (want, gb) in grads.items():
        got = params[k].grad[0].cpu().numpy()
        excess = np.abs(got - want) - gb
        assert np.all(excess <= 0), f"{k} step {s}: worst excess {excess.max():.3g}"
        # the reference's post-step state, or its pre-step state moved by the oracle's gradient for our indices
        target = f.post(s)[k] if all_agree else state[k] - f.meta["lr"] * want[None]
        targets[k] = (target.astype(np.float64), gb[None])
    return targets


# ------------------------------------------------------------------------------------------------ (b) vqb_diveq vs float64
def _diveq64(x, q, z, g, scale):
    e = q - x
    ne = e.norm(dim=-1, keepdim=True)
    n = e + scale * z
    u = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    out = x + u * ne
    s = (g * u).sum(-1, keepdim=True)
    de = torch.where(ne > 0, s / torch.where(ne > 0, ne, 1.0), 0.0) * e
    return out, g - de, de, ne


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("D", [8, 24, 136, 256, 1000, 1024])
def test_diveq_kernel_against_float64(dt, D):
    from vector_quantize_pytorch_b200 import ops
    # one wave of rows = 16 CTAs of 8 warps per SM: more than two waves, ending ragged
    N = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 16 * 8 + 77
    gen = torch.Generator(device=DEV).manual_seed(D * 3 + (dt == torch.bfloat16))
    x = torch.randn(N, D, device=DEV, generator=gen).to(dt)
    q = (x.float() + 0.3 * torch.randn(N, D, device=DEV, generator=gen)).to(dt)
    q[::97] = x[::97]                                    # e = 0 exactly: x equal to its code
    z = torch.randn(N, D, device=DEV, generator=gen).to(dt)
    g = torch.randn(N, D, device=DEV, generator=gen).to(dt)
    scale = float(np.sqrt(5e-3))
    out = ops.diveq(x, q, z, scale)
    dx, dq = ops.diveq(x, q, z, scale, g)
    assert dq.dtype == torch.float32 and dx.dtype == dt and out.dtype == dt
    X, Qn, Z, Gn = (t.double() for t in (x, q, z, g))
    r_out, r_dx, r_dq, ne = _diveq64(X, Qn, Z, Gn, float(np.float32(scale)))
    u = U_BF16 if dt == torch.bfloat16 else U_F32
    # every value is a short chain of rounded ops (<= 8 roundings in the row dtype): 16 u times its operands' magnitudes
    de_mag = Gn.norm(dim=-1, keepdim=True) * (Qn - X).abs() / ne.clamp_min(1e-30)
    checks = ((out, r_out, 16 * u * (X.abs() + ne)), (dq, r_dq, 16 * u * de_mag), (dx, r_dx, 16 * u * (Gn.abs() + de_mag)))
    for got, ref, bound in checks:
        err = (got.double() - ref).abs()
        assert bool((err <= bound).all()), float((err - bound).max())
    zero = ne[:, 0] == 0
    assert bool(zero[::97].all())
    assert torch.equal(out[zero], x[zero]) and bool((dq[zero] == 0).all()) and torch.equal(dx[zero], g[zero])


def test_diveq_rejects_bad_arguments():
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    x = torch.zeros(4, 2048, device=DEV)
    p = x.data_ptr()
    assert lib.vqb_diveq(None, p, p, None, 4, 8, 0, 0.1, p, None, None) == -1          # VQB_E_INVALID
    assert lib.vqb_diveq(p, p, p, p, 4, 8, 0, 0.1, p, None, None) == -1                # backward without grad_q
    assert lib.vqb_diveq(p, p, p, None, 4, 2048, 0, 0.1, p, None, None) == -2          # VQB_E_UNSUPPORTED: D > 1024
    assert lib.vqb_diveq(p + 2, p, p, None, 4, 8, 0, 0.1, p, None, None) == -3         # VQB_E_ALIGN


# ------------------------------------------------------------------------------------------------ (c) codebook gradient
@pytest.mark.parametrize("K", [5, 1024, 16384])
def test_codebook_gradient_against_float64(K):
    """d embed of sum(quantize * G) + loss for an input without grad: output path + commitment term, both from the statistics
    chain, against float64 sums over the module's own indices.  Bound: the longest fp32 addition chain of a code (its row count)."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(K)
    N, D = 262144, 64
    vq = m.VectorQuantize(dim=D, codebook_size=K, learnable_codebook=True, ema_update=False, commitment_weight=0.5).to(DEV).train()
    x = torch.randn(4, N // 4, D, device=DEV)
    G = torch.randn_like(x)
    C = vq._codebook.embed.detach()[0].double().clone()
    out, ind, loss = vq(x)
    ((out * G).sum() + loss).backward()
    idx = ind.reshape(-1)
    X, Gd = x.reshape(-1, D).double(), G.reshape(-1, D).double()
    rows = Gd + 2 * 0.5 * (C[idx] - X) / (N * D)
    ref = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, idx, rows)
    mag = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, idx, Gd.abs() + (C[idx].abs() + X.abs()) / (N * D))
    count = torch.bincount(idx, minlength=K).double()[:, None]
    bound = (count + 4) * U_F32 * mag + 1e-12
    err = (vq._codebook.embed.grad[0].double() - ref).abs()
    assert bool((err <= bound).all()), float((err - bound).max())


# ------------------------------------------------------------------------------------------------ (d) optimizer step
@pytest.mark.parametrize("opt_kind", ["sgd", "adam_foreach", "adam_fused"])
def test_optimizer_step_reaches_next_search(opt_kind):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(5)
    D, K = 64, 256
    vq = m.VectorQuantize(dim=D, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV).train()
    rvq = m.ResidualVQ(dim=D, num_quantizers=3, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV).train()
    params = list(vq.parameters()) + list(rvq.parameters())
    opt = {"sgd": lambda: torch.optim.SGD(params, lr=200.),
           "adam_foreach": lambda: torch.optim.Adam(params, lr=0.5, foreach=True),
           "adam_fused": lambda: torch.optim.Adam(params, lr=0.5, fused=True)}[opt_kind]()
    x = torch.randn(2, 2048, D, device=DEV, requires_grad=True)
    G = torch.randn_like(x)
    for mod in (vq, rvq):
        out, ind0, loss = mod(x)
        ((out * G).sum() + loss.sum()).backward()
    with torch.no_grad():
        _, before, _ = vq(x)
        _, rbefore, _ = rvq.eval()(x)
    rvq.train()
    opt.step()
    fresh = m.VectorQuantize(dim=D, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV)
    fresh.load_state_dict(vq.state_dict())
    rfresh = m.ResidualVQ(dim=D, num_quantizers=3, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV)
    rfresh.load_state_dict(rvq.state_dict())
    _, want, _ = fresh(x.detach())
    _, got, _ = vq(x)                            # training, layered on grad
    assert torch.equal(got, want) and not torch.equal(got, before)
    with torch.no_grad():
        _, got_ng, _ = vq(x)
    assert torch.equal(got_ng, want)
    _, rwant, _ = rfresh.eval()(x.detach())
    _, rgot, _ = rvq(x)                          # layered path
    assert torch.equal(rgot, rwant) and not torch.equal(rgot, rbefore)
    with torch.no_grad():
        _, rgot_ng, _ = rvq.eval()(x)            # one-call program
    assert torch.equal(rgot_ng, rwant)


# ------------------------------------------------------------------------------------------------ (e) other differentiable surfaces
def _code_sums64(rows, idx, K):
    """float64 per-code sums of gradient rows; rows with index -1 send nothing."""
    keep = idx >= 0
    out = torch.zeros(K, rows.shape[-1], dtype=torch.float64, device=rows.device)
    return out.index_add_(0, idx[keep], rows[keep].double())


def _check_sums(got, rows, idx, K):
    ref = _code_sums64(rows, idx, K)
    mag = _code_sums64(rows.abs(), idx, K)
    count = torch.bincount(idx[idx >= 0], minlength=K).double()[:, None]
    bound = (count + 1) * U_F32 * mag          # the fp32 addition chain of each code
    assert bool(((got.double() - ref).abs() <= bound).all())


def test_codebook_forward_carries_gradient_to_embed():
    """Codebook.forward (vqp:674-791) of a learnable codebook: `quantize` sends each row's gradient to its code."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(21)
    cb = m.Codebook(dim=32, codebook_size=40, learnable_codebook=True, ema_update=False, threshold_ema_dead_code=0).to(DEV)
    x = torch.randn(3, 500, 32, device=DEV)
    G = torch.randn(3, 500, 32, device=DEV)
    q, ind, _ = cb(x)
    assert q.requires_grad
    (q * G).sum().backward()
    _check_sums(cb.embed.grad[0], G.reshape(-1, 32), ind.reshape(-1), 40)
    assert torch.equal(q.detach(), cb.embed.detach()[0][ind])


def test_decoders_carry_gradient_to_embed():
    """get_codes_from_indices / get_output_from_indices of learnable codebooks gather from the parameter (vqp:998-1022,
    rvq:324-382): each code receives the sum of the gradient rows that gathered it; index -1 (a dropped layer) sends nothing."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(22)
    D, K, Q = 32, 48, 3
    vq = m.VectorQuantize(dim=D, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV)
    ind = torch.randint(0, K, (4, 300), device=DEV)
    G = torch.randn(4, 300, D, device=DEV)
    (vq.get_output_from_indices(ind) * G).sum().backward()
    _check_sums(vq._codebook.embed.grad[0], G.reshape(-1, D), ind.reshape(-1), K)
    for shared in (False, True):
        rvq = m.ResidualVQ(dim=D, num_quantizers=Q, codebook_size=K, learnable_codebook=True, ema_update=False,
                           shared_codebook=shared, quantize_dropout=True).to(DEV)
        idx = torch.randint(0, K, (4, 300, Q), device=DEV)
        idx[..., 2][::2] = -1
        G = torch.randn(4, 300, D, device=DEV)
        Gs = torch.randn(Q, 4, 300, D, device=DEV)
        ((rvq.get_output_from_indices(idx) * G).sum() + (rvq.get_codes_from_indices(idx) * Gs).sum()).backward()
        flat = idx.reshape(-1, Q)
        rows = [G.reshape(-1, D) + Gs[q].reshape(-1, D) for q in range(Q)]
        if shared:
            got = rvq.layers[0]._codebook.embed.grad[0]
            _check_sums(got, torch.cat(rows), flat.t().reshape(-1), K)
        else:
            for q in range(Q):
                _check_sums(rvq.layers[q]._codebook.embed.grad[0], rows[q], flat[:, q], K)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_diveq_rvq_without_grad(dt, monkeypatch):
    """ResidualVQ(diveq=True) outside autograd (rvq:603-606 applies DiVeQ in every mode): the one-call program (eval), the
    stage-wise path (quantize dropout in training) and GroupedResidualVQ, each = vqb_diveq(x, quantized_out(indices), z)."""
    import vector_quantize_pytorch_b200 as m
    import vector_quantize_pytorch_b200.vector_quantize as vqm
    from vector_quantize_pytorch_b200 import ops
    torch.manual_seed(23)
    D, K, Q = 64, 128, 3
    drawn = []

    def noise(like):
        z = torch.randn_like(like)
        drawn.append(z)
        return z
    monkeypatch.setattr(vqm, "diveq_noise", noise)
    x = torch.randn(2, 1500, D, device=DEV).to(dt)
    scale = float(np.sqrt(5e-3))

    def expect(rvq, xin, idx, z):
        d = xin.shape[-1]
        n = int((idx.reshape(-1, Q)[0] >= 0).sum())
        books = torch.stack([layer._codebook.embed.detach()[0] for layer in rvq.layers[:n]])
        qout = ops.rvq_accumulate(books, idx.reshape(-1, Q)[:, :n].contiguous(), xin.dtype)
        return ops.diveq(xin.reshape(-1, d), qout, z.reshape(-1, d), scale).reshape(xin.shape)

    rvq = m.ResidualVQ(dim=D, num_quantizers=Q, codebook_size=K, diveq=True, quantize_dropout=True).to(DEV)
    with torch.no_grad():
        out, idx, _ = rvq.eval()(x)                                              # one-call program
        assert torch.equal(out, expect(rvq, x, idx, drawn[-1]))
        out, idx, _ = rvq.train()(x, rand_quantize_dropout_fixed_seed=1)         # stage-wise path, dropped layers
        assert bool((idx[..., -1] == -1).all())
        assert torch.equal(out, expect(rvq, x, idx, drawn[-1]))
    grvq = m.GroupedResidualVQ(dim=D, groups=2, num_quantizers=Q, codebook_size=K, diveq=True).to(DEV).eval()
    with torch.no_grad():
        drawn.clear()
        out, idx, _ = grvq(x)
        assert len(drawn) == 2
        for g, (r, z) in enumerate(zip(grvq.rvqs, drawn)):
            xs = x[..., g * D // 2:(g + 1) * D // 2]
            assert torch.equal(out[..., g * D // 2:(g + 1) * D // 2], expect(r, xs, idx[g], z))
