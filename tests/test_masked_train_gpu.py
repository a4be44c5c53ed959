"""GPU checks of masked training steps (mask= / lens= with gradients) of VectorQuantize, ResidualVQ and GroupedResidualVQ:

(a) replay of the reference's masked step (tests/golden/masked_train/, oracle/gen_golden_masked_train.py): indices equal, the
    outputs, losses, x.grad, projection gradients and the codebook buffers after the step within the tolerances of the
    learnable-codebook replays (fp32 1e-5; bf16 per-element bounds of 8 bf16 roundings per summed term), padding rows exactly
    the padding value with exactly zero or exactly the upstream gradient, and nothing non-finite anywhere;
(b) the Euclidean VectorQuantize step (in-kernel mask, vqb_rotate_masked) runs with no host synchronisation;
(c) the same masked call with and without requires_grad gives the same forward bits: rows, indices, loss, code counts (the
    EMA's row sums add re-scored rows with vector reductions in no fixed order, so those buffers agree to fp32 rounding);
(d) a batch with no live row, and the configurations that stay refused.
"""
import copy

import numpy as np
import pytest
import torch

from masked_train_golden import Fixture, names
from test_learnable_gpu import EST_OPS, U_BF16, _Replay, _install, _rotation_terms

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _build(f):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(f.meta["init_seed"])
    mod = getattr(m, f.cls)(**f.kw).to(DEV)
    mod.load_state_dict({k: torch.from_numpy(v) for k, v in f.state().items()})
    return mod.train()


def _run(f, mod, monkeypatch, x_grad=True):
    """One forward (+ backward when x requires grad) of the fixture's step; the reference's RNG draws replace ours."""
    dt = torch.bfloat16 if f.bf16 else torch.float32
    x = torch.from_numpy(f["x"]).to(DEV, dt).requires_grad_(x_grad)
    G = torch.from_numpy(f["G"]).to(DEV)
    kw = dict(f.meta["fwd"])
    if f.meta["how"] == "lens":
        kw["lens"] = torch.from_numpy(f["lens"]).to(DEV)
    else:
        kw["mask"] = torch.from_numpy(f["mask"]).to(DEV)
    replay = _Replay(f.draws())
    with monkeypatch.context() as mp:
        _install(mp, replay)
        out, ind, loss = mod(x, **kw)
    assert not replay.draws, "the module drew less from the RNG than the reference"
    if x_grad:
        ((out.float() * G).sum() + f.meta["lw"] * loss.float().sum()).backward()
    return x, out, ind, loss


def _np(t):
    return t.detach().float().cpu().numpy()


def _bf16_vq_bounds(f):
    """Per-element bounds of a bf16 VectorQuantize step: output and x.grad, 8 bf16 roundings of each summed term (the
    reference's estimator is a chain of such ops; the kernels round once)."""
    from oracle.masked_train_oracle import l2norm
    kw = f.kw
    D = f["x"].shape[-1]
    x, G = f["x"].astype(np.float64).reshape(-1, D), f["G"].astype(np.float64).reshape(-1, D)
    live = f["mask"].reshape(-1)
    C = f.state()["_codebook.embed"][0].astype(np.float64)
    c = np.zeros_like(x)
    c[live] = C[f["ind"].reshape(-1)[live]]
    xt = l2norm(x.astype(np.float32)).astype(np.float64) if kw.get("use_cosine_sim") else x
    terms = _rotation_terms(xt, c, G) if kw.get("rotation_trick", True) else np.abs(G)
    if kw.get("use_cosine_sim"):   # through l2norm's backward
        n = np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), 1e-12)
        u = np.abs(x) / n
        terms = (terms + (terms * u).sum(-1, keepdims=True) * u) / n
    n_live = max(int(live.sum()), 1)
    commit = 2.0 * f.meta["lw"] * kw.get("commitment_weight", 1.0) * np.abs(c - x) / (n_live * D)
    b_out = EST_OPS * U_BF16 * (np.abs(x) + np.abs(c)) + 1e-30
    b_xg = EST_OPS * U_BF16 * (terms + commit) + 1e-30
    return b_out.reshape(f["x"].shape), b_xg.reshape(f["x"].shape)


@pytest.mark.parametrize("name", names())
def test_masked_train_replays_reference(name, monkeypatch):
    f = Fixture(name)
    mod = _build(f)
    x, out, ind, loss = _run(f, mod, monkeypatch)
    got = dict(out=_np(out), loss=_np(loss), xgrad=_np(x.grad))
    for k, v in got.items():
        assert np.isfinite(v).all(), f"non-finite {k}"
    np.testing.assert_array_equal(ind.cpu().numpy(), f["ind"])
    if f.bf16:
        b_out, b_xg = _bf16_vq_bounds(f)
        assert np.all(np.abs(got["out"] - f["out"]) <= b_out), "output"
        assert np.all(np.abs(got["xgrad"] - f["xgrad"]) <= b_xg), "x.grad"
        np.testing.assert_allclose(got["loss"], f["loss"], rtol=2 * U_BF16)
    else:
        tol = dict(rtol=1e-5, atol=1e-5)
        for k, v in got.items():
            np.testing.assert_allclose(v, f[k], **tol, err_msg=k)
        ref = f.pgrads()
        for n, p in mod.named_parameters():
            g = p.grad.cpu().numpy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
            np.testing.assert_allclose(g, ref[n], **tol, err_msg=n)
    post = mod.state_dict()
    for k, v in f.post().items():
        np.testing.assert_allclose(post[k].float().cpu().numpy(), v.astype(np.float32), rtol=1e-5, atol=1e-5, err_msg=k)
    # padding rows: exactly the padding value / no gradient, or the input and the upstream gradient
    pad = ~f["mask"]
    if f.cls == "VectorQuantize":
        assert (ind.cpu().numpy()[pad] == -1).all()
        if f.kw.get("return_zeros_for_masked_padding", True):
            assert (got["out"][pad] == 0).all() and (got["xgrad"][pad] == 0).all()
        else:
            np.testing.assert_array_equal(got["out"][pad], _np(x)[pad])
            np.testing.assert_array_equal(got["xgrad"][pad], f["G"][pad])
    else:
        assert (got["xgrad"][pad] == 0).all()


def _vq(**kw):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    return m.VectorQuantize(dim=64, codebook_size=256, **kw).to(DEV).train()


def _batch(dt, zero_pad=True, B=8, N=512, D=64, seed=1):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    lens = torch.randint(0, N + 1, (B,), generator=gen, device=DEV)
    lens[0], lens[1] = N, 0
    mask = torch.arange(N, device=DEV) < lens[:, None]
    x = torch.randn(B, N, D, generator=gen, device=DEV)
    if zero_pad:
        x = x * mask[..., None]
    return x.to(dt), mask, torch.randn(B, N, D, generator=gen, device=DEV)


@pytest.mark.parametrize("rotation", [True, False])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_euclidean_masked_step_has_no_host_sync(dt, rotation):
    vq = _vq(rotation_trick=rotation)
    x, mask, G = _batch(dt)
    for step in range(2):    # the first step reads the `initted` flag once
        xr = x.clone().requires_grad_(True)
        mode = "error" if step else "default"
        torch.cuda.set_sync_debug_mode(mode)
        try:
            out, ind, loss = vq(xr, mask=mask)
            ((out.float() * G).sum() + loss).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(xr.grad).all() and (xr.grad[~mask] == 0).all() and (out[~mask] == 0).all()


_BITWISE = [
    dict(),                                                          # in-kernel, rotation trick
    dict(rotation_trick=False, return_zeros_for_masked_padding=False),
    dict(use_cosine_sim=True),                                       # compacted rows
    dict(threshold_ema_dead_code=2),                                 # compacted rows: expiry pending
    dict(commitment_weight=0.3),
]


@pytest.mark.parametrize("kw", _BITWISE, ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()) or "default")
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_gradient_changes_no_forward_bit(dt, kw):
    base = _vq(**kw)
    x, mask, _ = _batch(dt, zero_pad=False)
    res = []
    for x_grad in (False, True):
        vq = copy.deepcopy(base)
        torch.manual_seed(3)
        out, ind, loss, br = vq(x.clone().requires_grad_(x_grad), mask=mask, return_loss_breakdown=True)
        res.append((out.detach(), ind, loss.detach(), br.commitment.detach(),
                    {k: v.clone() for k, v in vq.state_dict().items()}))
    (o0, i0, l0, c0, s0), (o1, i1, l1, c1, s1) = res
    assert torch.equal(o0.view(torch.int16 if dt == torch.bfloat16 else torch.int32),
                       o1.view(torch.int16 if dt == torch.bfloat16 else torch.int32))
    assert torch.equal(i0, i1)
    assert torch.equal(l0, l1) and torch.equal(c0, c1)
    for k in s0:
        if k.endswith("embed_avg") or k.endswith("embed"):
            torch.testing.assert_close(s0[k], s1[k], rtol=1e-5, atol=1e-5, msg=lambda m: f"{k}: {m}")
        else:
            assert torch.equal(s0[k], s1[k]), k


@pytest.mark.parametrize("kw", [dict(), dict(rotation_trick=False), dict(return_zeros_for_masked_padding=False),
                                dict(use_cosine_sim=True), dict(use_cosine_sim=True, return_zeros_for_masked_padding=False),
                                dict(kmeans_init=True)],
                         ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()) or "default")
def test_no_live_row(kw):
    """An all-padding batch, on the in-kernel path and on the compacted one (cosine, k-means pending): a zero loss, and x gets
    a zero gradient (or the upstream one through pass-through padding) from the rows and from the loss alone."""
    vq = _vq(**kw)
    x, _, G = _batch(torch.float32)
    mask = torch.zeros(x.shape[:2], dtype=torch.bool, device=DEV)
    want = G if kw.get("return_zeros_for_masked_padding") is False else torch.zeros_like(G)
    xr = x.clone().requires_grad_(True)
    out, ind, loss = vq(xr, mask=mask)
    ((out * G).sum() + loss).backward()
    assert float(loss.detach()) == 0.0 and (ind == -1).all()
    assert xr.grad is not None and torch.equal(xr.grad, want)
    xr = x.clone().requires_grad_(True)
    vq(xr, mask=mask)[2].backward()
    assert xr.grad is not None and torch.equal(xr.grad, torch.zeros_like(G))


@pytest.mark.parametrize("cls", ["ResidualVQ", "GroupedResidualVQ"])
@pytest.mark.parametrize("proj", [False, True])
def test_rvq_no_live_row(cls, proj):
    """An all-padding batch through ResidualVQ / GroupedResidualVQ with gradients: zero losses and x (and project_in) get a
    zero gradient, from the rows and from the losses alone."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    kw = dict(dim=64, num_quantizers=3, codebook_size=64, codebook_dim=32 if proj else None)
    if cls == "GroupedResidualVQ":
        kw.update(groups=2, codebook_dim=16 if proj else None)
    mod = getattr(m, cls)(**kw).to(DEV).train()
    x, _, G = _batch(torch.float32)
    mask = torch.zeros(x.shape[:2], dtype=torch.bool, device=DEV)
    for with_rows in (True, False):
        xr = x.clone().requires_grad_(True)
        out, ind, losses = mod(xr, mask=mask)
        assert (ind == -1).all() and torch.equal(losses.detach(), torch.zeros_like(losses))
        (((out * G).sum() if with_rows else 0) + losses.sum()).backward()
        assert xr.grad is not None and torch.equal(xr.grad, torch.zeros_like(G))
        if proj:
            ins = [mod.project_in] if cls == "ResidualVQ" else [r.project_in for r in mod.rvqs]
            assert all(torch.equal(p.weight.grad, torch.zeros_like(p.weight)) for p in ins)
            mod.zero_grad(set_to_none=True)


def test_rvq_masked_projections_train():
    """A masked ResidualVQ with projections at a larger shape, shared and separate codebooks: finite gradients for x and both projections, zero on padding rows."""
    import vector_quantize_pytorch_b200 as m
    for shared in (False, True):
        torch.manual_seed(0)
        rvq = m.ResidualVQ(dim=64, codebook_dim=32, num_quantizers=4, codebook_size=128, shared_codebook=shared).to(DEV).train()
        x, mask, G = _batch(torch.float32)
        xr = x.clone().requires_grad_(True)
        out, ind, losses = rvq(xr, mask=mask)
        ((out * G).sum() + losses.sum()).backward()
        assert torch.isfinite(xr.grad).all() and (xr.grad[~mask] == 0).all() and (ind[~mask] == -1).all()
        for p in (rvq.project_in.weight, rvq.project_out.weight):
            assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0


def test_masked_training_refusals():
    import vector_quantize_pytorch_b200 as m
    x, mask, _ = _batch(torch.float32)
    x = x.requires_grad_(True)
    refused = [
        m.VectorQuantize(dim=64, codebook_size=64, learnable_codebook=True, ema_update=False),
        m.VectorQuantize(dim=64, codebook_size=64, directional_reparam=True, threshold_ema_dead_code=2),
        m.VectorQuantize(dim=64, codebook_size=64, directional_reparam=True, learnable_codebook=False, threshold_ema_dead_code=2),
        m.VectorQuantize(dim=64, codebook_size=64, codebook_dim=32),
        m.VectorQuantize(dim=64, codebook_size=64, heads=2, codebook_dim=32),
        m.ResidualVQ(dim=64, num_quantizers=2, codebook_size=64, use_cosine_sim=True),
        m.ResidualVQ(dim=64, num_quantizers=2, codebook_size=64, return_zeros_for_masked_padding=False),
        m.ResidualVQ(dim=64, num_quantizers=2, codebook_size=64, learnable_codebook=True, ema_update=False),
        m.ResidualVQ(dim=64, num_quantizers=2, codebook_size=64, threshold_ema_dead_code=2),
    ]
    for mod in refused:
        with pytest.raises(NotImplementedError):
            mod.to(DEV).train()(x, mask=mask)
