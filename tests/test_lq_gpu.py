"""LatentQuantize on the GPU: the reference's fixtures replayed (tests/golden/lq/), the reference's own test classes, a training
step without host syncs, and values loaded after construction.

Without projections the quantized output and the indices must equal the reference bit for bit.  With projections cuBLAS and
the CPU's GEMMs round differently, so the indices must equal the decision the oracle takes on our own z (project_in on the
GPU), and values and gradients must lie within the bound of a length-K fp32 dot product (gamma_K = K u / (1 - K u), u = 2^-24,
on the sum of absolute products, for each of the two implementations) of the float64 recomputation from the fixture."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lq_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "lq")
FIXTURES = sorted(p[:-4] for p in os.listdir(GOLDEN) if p.endswith(".npz"))
U = 2.0 ** -24


def load(name):
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    return f, json.loads(bytes(f["meta"]).decode())


def gamma(k):
    return k * U / (1 - k * U)


def build(name, device="cuda"):
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    torch.manual_seed(meta["seed"])
    lq = m.LatentQuantize(**meta["kw"])
    if meta["loaded"]:
        with torch.no_grad():
            for i, v in enumerate(lq.values_per_latent):
                v.copy_(torch.from_numpy(f[f"table_{i}"]))
    return f, meta, lq.to(device)


def step(lq, f, meta):
    dtype = getattr(torch, meta["dtype"])
    x = torch.from_numpy(f["x"]).to(dtype).cuda().requires_grad_()
    lq.train()
    out, ind, loss = lq(x)
    g = torch.from_numpy(f["g"]).cuda()
    obj = (out * g).sum()
    if meta["loss_backward"] and loss.requires_grad:
        obj = obj + loss
    obj.backward()
    return x, out, ind, loss


@pytest.mark.parametrize("name", FIXTURES)
def test_replay_fixture(name):
    f, meta, lq = build(name)
    x, out, ind, loss = step(lq, f, meta)
    assert out.dtype == torch.float32 and ind.dtype == torch.int32 and loss.dtype == torch.float32
    assert out.shape == f["out"].shape and ind.shape == f["indices"].shape and loss.shape == ()
    kw = meta["kw"]
    wc, wq = kw.get("commitment_loss_weight", 0.1), kw.get("quantization_loss_weight", 0.1)
    x_rows = np.moveaxis(f["x"], 1, -1).reshape(-1, f["x"].shape[1]).astype(np.float64)
    if not lq.has_projections:
        np.testing.assert_array_equal(out.detach().cpu().numpy(), f["out"])
        np.testing.assert_array_equal(ind.cpu().numpy(), f["indices"])
        out_rows = np.moveaxis(f["out"], 1, -1).reshape(-1)
        l64, bound = O.loss64(x_rows.ravel(), out_rows, wc, wq, wc != 0, wq != 0)
        assert abs(loss.item() - l64) <= bound + abs(l64) * 2.0 ** -22
        # x.grad = g + 2 w_c (out - x) / M g_loss (through the codes) + 2 w_q (x - out) / M (the quantization term), fp32
        gx = x.grad.float().cpu().numpy()
        if meta["dtype"] == "float32":
            err = np.abs(gx - f["x_grad"])
            scale = np.abs(f["g"]) + 4 * (wc + wq) * np.abs(f["x"] - f["out"]) / f["x"].size
            assert (err <= 4 * U * scale + 1e-45).all()
        else:   # the reference raises in its mse backward on bf16 inputs: ours is the bf16 rounding of the fp32 gradient
            np.testing.assert_array_equal(gx, torch.from_numpy(f["g"]).bfloat16().float().numpy())
    else:
        check_projected(f, meta, lq, x, out, ind, x_rows, wc, wq)
    # eval: same decisions, zero loss
    lq.eval()
    with torch.no_grad():
        eo, ei, el = lq(x.detach())
    assert torch.equal(ei, ind) and el.item() == 0.0 and el.device == x.device
    assert torch.equal(eo, out.detach())


def decision_margin_rows(f, lq, x_rows):
    """Rows whose fixture z lies farther from every decision midpoint of its tables than the two project_in roundings can
    move it (2 gamma_{K+1} (|x| |W_in|^T + |b_in|), K = dim): there our z must take the reference's decisions."""
    z = f["z"].reshape(-1, lq.num_codebooks, lq.codebook_dim).astype(np.float64)
    Wi = lq.project_in.weight.detach().cpu().double().numpy()
    bi = lq.project_in.bias.detach().cpu().double().numpy()
    bz = (2 * gamma(Wi.shape[1] + 1) * (np.abs(x_rows) @ np.abs(Wi.T) + np.abs(bi))).reshape(z.shape)
    marg = np.full(z.shape, np.inf)
    for i in range(lq.codebook_dim):
        v = np.sort(f[f"table_{i}"].astype(np.float64))
        marg[..., i] = np.min(np.abs(z[..., i, None] - (v[1:] + v[:-1]) / 2), -1)
    return (marg > bz).all(-1).all(-1)


def step_grads64(x_rows, out_rows, codes, g_rows, Wo, Wi, wc, wq, M):
    """float64 gradients of sum(out * g) + loss from one forward's fp32 values, and their bounds: every quantity is a short
    chain of fp32 sums and GEMMs, bounded by 4 gamma_k of the same chain over absolute values (k the longest sum plus the
    chain's depth)."""
    d_out = 2 * wc * (out_rows - x_rows) / M
    go = g_rows + d_out
    ago = np.abs(g_rows) + np.abs(d_out)
    gz = go @ Wo
    dq = 2 * wq * (x_rows - out_rows) / M
    R, dim = x_rows.shape
    kr, kd = 4 * gamma(R + 8), 4 * gamma(Wo.shape[0] + Wi.shape[1] + 8)
    ref = dict(x=gz @ Wi + dq, pout_w=go.T @ codes, pout_b=go.sum(0), pin_w=gz.T @ x_rows, pin_b=gz.sum(0))
    agz = ago @ np.abs(Wo)
    bnd = dict(x=kd * (agz @ np.abs(Wi) + np.abs(dq)), pout_w=kr * (ago.T @ np.abs(codes)), pout_b=kr * ago.sum(0),
               pin_w=(kr + kd) * (agz.T @ np.abs(x_rows)), pin_b=(kr + kd) * agz.sum(0))
    return ref, bnd


def check_projected(f, meta, lq, x, out, ind, x_rows, wc, wq):
    """Projections: decisions equal the oracle's on our own z, and the reference's on every row outside the project_in
    rounding band (every row of every fixture here); outputs within the project_out bound; the gradients of x and of both
    projections' weights and biases, ours and the reference's, each within its bound of the float64 recomputation from its own
    forward."""
    R, C, D = x_rows.shape[0], lq.num_codebooks, lq.codebook_dim
    z = lq.project_in(torch.from_numpy(x_rows.astype(np.float32)).cuda()).detach().cpu().numpy()
    tables = [f[f"table_{i}"] for i in range(D)]
    levels, basis = lq._levels.cpu().numpy(), lq._basis.cpu().numpy()
    codes, idx = O.quantize(z.reshape(R, C, D), tables, levels, basis)
    np.testing.assert_array_equal(ind.cpu().numpy().reshape(idx.shape), idx)
    same = (idx.reshape(f["indices"].shape) == f["indices"]).reshape(R, C).all(-1)
    clear = decision_margin_rows(f, lq, x_rows)
    assert clear.all(), "a fixture row lies inside the project_in rounding band"
    assert same[clear].all()
    Wo = lq.project_out.weight.detach().cpu().double().numpy()
    bo = lq.project_out.bias.detach().cpu().double().numpy()
    c64 = codes.reshape(R, -1).astype(np.float64)
    bound = 2 * gamma(Wo.shape[1] + 1) * (np.abs(c64) @ np.abs(Wo.T) + np.abs(bo))
    out_rows = np.moveaxis(out.detach().cpu().numpy(), 1, -1).reshape(R, -1).astype(np.float64)
    ref_rows = np.moveaxis(f["out"], 1, -1).reshape(R, -1).astype(np.float64)
    assert (np.abs(out_rows - ref_rows) <= bound).all()
    Wi = lq.project_in.weight.detach().cpu().double().numpy()
    M = f["x"].size
    g_rows = np.moveaxis(f["g"], 1, -1).reshape(R, -1).astype(np.float64)
    ref_codes, _ = O.quantize(f["z"].reshape(R, C, D), tables, levels, basis)
    ours = dict(x=np.moveaxis(x.grad.cpu().numpy(), 1, -1).reshape(R, -1), pout_w=lq.project_out.weight.grad.cpu().numpy(),
                pout_b=lq.project_out.bias.grad.cpu().numpy(), pin_w=lq.project_in.weight.grad.cpu().numpy(),
                pin_b=lq.project_in.bias.grad.cpu().numpy())
    theirs = dict(x=np.moveaxis(f["x_grad"], 1, -1).reshape(R, -1), pout_w=f["pout_w_grad"], pout_b=f["pout_b_grad"],
                  pin_w=f["pin_w_grad"], pin_b=f["pin_b_grad"])
    for got, o_rows, cds in ((ours, out_rows, c64), (theirs, ref_rows, ref_codes.reshape(R, -1).astype(np.float64))):
        ref, bnd = step_grads64(x_rows, o_rows, cds, g_rows, Wo, Wi, wc, wq, M)
        for k in ref:
            assert (np.abs(got[k] - ref[k]) <= bnd[k] + 1e-30).all(), k


def _quantized_roundtrip(lq, x):
    quantized, indices, _ = lq(x)
    assert x.shape == quantized.shape
    assert (quantized == lq.indices_to_codes(indices)).all()
    return indices


# the reference's five test classes (tests/test_latent_quantization.py), on the GPU

@pytest.mark.parametrize("shape", [(1, 16, 32, 32), (1, 16, 10, 32, 32), (1, 16, 64)])
def test_reference_default(shape):
    import vector_quantize_pytorch_b200 as m
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=16, commitment_loss_weight=0.1, quantization_loss_weight=0.1).cuda()
    _quantized_roundtrip(lq, torch.randn(*shape, device="cuda"))


def test_reference_no_optim():
    import vector_quantize_pytorch_b200 as m
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=16, optimize_values=False).cuda()
    _quantized_roundtrip(lq, torch.randn(1, 16, 32, 32, device="cuda"))


def test_reference_same_level_and_int():
    import vector_quantize_pytorch_b200 as m
    for kw in (dict(levels=[5, 5, 5]), dict(levels=5, codebook_dim=3)):
        lq = m.LatentQuantize(dim=16, **kw).cuda()
        _quantized_roundtrip(lq, torch.randn(1, 16, 32, 32, device="cuda"))
    with pytest.raises(RuntimeError):
        m.LatentQuantize(levels=5, dim=16)


def test_reference_multi_codebook():
    import vector_quantize_pytorch_b200 as m
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=16, num_codebooks=4).cuda()
    x = torch.randn(1, 16, 64, device="cuda", requires_grad=True)
    quantized, indices, loss = lq(x)
    assert indices.shape[-1] == 4
    assert (quantized == lq.indices_to_codes(indices)).all()
    loss.backward()
    assert x.grad is not None and lq.project_in.weight.grad is not None
    assert all(v.grad is None for v in lq.values_per_latent)


def test_training_step_makes_no_host_sync():
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=16).cuda().train()
    x = torch.randn(4, 16, 8, 8, device="cuda", requires_grad=True)
    lq(x)   # first use: the per-device index tables are copied from the host once
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, ind, loss = lq(x)
        (out.square().mean() + loss).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(x.grad).all()


def test_loaded_values_change_next_forward():
    import vector_quantize_pytorch_b200 as m
    for optimize in (True, False):
        lq = m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=optimize).cuda()
        x = torch.full((2, 3, 4), 0.3, device="cuda")
        out1, ind1, _ = lq(x)
        assert torch.allclose(out1, torch.tensor([0.25, 0.25, 0.25], device="cuda").view(1, 3, 1).expand_as(out1))
        new = [torch.tensor([0.3, -0.5, 0.0, 0.1, 0.5]), torch.tensor([0.5, 0.0, -0.5, 0.28, 0.31]),
               torch.arange(8) / 8 - 0.5]
        if optimize:
            lq.load_state_dict({f"values_per_latent.{i}": v for i, v in enumerate(new)})
        else:
            for v, n in zip(lq.values_per_latent, new):
                v.copy_(n)
        out2, ind2, _ = lq(x)
        want = torch.tensor([0.3, 0.31, 0.25], device="cuda").view(1, 3, 1).expand_as(out2)
        assert torch.allclose(out2, want, rtol=0, atol=1e-7)
        assert not torch.equal(ind1, ind2)


def test_data_edits_change_next_forward():
    """Edits through `.data` move no version counter; the next forward still quantizes against the edited values, for
    tables on the device and for the plain CPU list."""
    import vector_quantize_pytorch_b200 as m
    for optimize in (True, False):
        lq = m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=optimize).cuda()
        x = torch.full((2, 3, 4), 0.3, device="cuda")
        out1, ind1, _ = lq(x)
        v = lq.values_per_latent[0]
        before = (v._version, v.data_ptr())
        v.data.copy_(torch.tensor([0.3, -0.5, 0.0, 0.1, 0.5], device=v.device))
        lq.values_per_latent[1].data.mul_(-1.0)
        assert (v._version, v.data_ptr()) == before
        out2, ind2, _ = lq(x)
        assert out2[:, 0].eq(0.3).all() and out2[:, 1].eq(0.25).all() and out2[:, 2].eq(0.25).all()
        assert not torch.equal(out2, out1)
        assert torch.equal(ind2, lq.codes_to_indices(out2.movedim(1, -1)))   # the index follows the new codes


@pytest.mark.parametrize("cast", ["bfloat16", "double"])
def test_dtype_cast_module(cast):
    """A module cast with .bfloat16() / .double() (optimize_values=False and no projection leave nothing else to cast): the
    kernels take the weights as fp32, so the loss equals an fp32 module's whose weights hold the cast values, in the
    reference's promoted dtype (w * mse: fp32 for bf16 weights, fp64 for fp64 weights)."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    lq = getattr(m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=False, commitment_loss_weight=0.1,
                                  quantization_loss_weight=0.3), cast)().cuda().train()
    assert lq.commitment_loss_weight.dtype == getattr(torch, cast)
    ref = m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=False, commitment_loss_weight=0.1,
                           quantization_loss_weight=0.3).cuda().train()
    with torch.no_grad():
        ref.commitment_loss_weight.copy_(lq.commitment_loss_weight.float())
        ref.quantization_loss_weight.copy_(lq.quantization_loss_weight.float())
    xdt = torch.bfloat16 if cast == "bfloat16" else torch.float32
    x = torch.randn(4, 3, 64, device="cuda").to(xdt)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    out, ind, loss = lq(xa)
    out_r, ind_r, loss_r = ref(xb)
    assert loss.dtype == (torch.float32 if cast == "bfloat16" else torch.float64)
    assert torch.equal(out, out_r) and torch.equal(ind, ind_r)
    assert torch.equal(loss, loss_r.to(loss.dtype))
    loss.backward()
    loss_r.backward()
    assert torch.equal(xa.grad, xb.grad)
    lq.eval()
    assert lq(x)[2].dtype == loss.dtype


@pytest.mark.parametrize("kw,shape", [(dict(levels=[5, 5, 8], dim=16), (2, 16, 6, 7)),
                                      (dict(levels=[4, 8, 16], dim=9, num_codebooks=3), (2, 9, 20))])
def test_quantize_and_project_matches_forward(kw, shape):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(1)
    lq = m.LatentQuantize(**kw).cuda().eval()
    x = torch.randn(*shape, device="cuda")
    out, ind, _ = lq(x)
    b, d = shape[0], shape[1]
    z = lq.project_in(x.movedim(1, -1).reshape(b, -1, d)).reshape(b, -1, lq.num_codebooks, lq.codebook_dim)
    codes, out2, ind2 = lq.quantize_and_project(z, len(shape) >= 4, [torch.Size(shape[2:])])
    assert codes.shape == (b, z.shape[1], lq.effective_codebook_dim)
    assert torch.equal(out2, out) and torch.equal(ind2, ind)
    assert torch.equal(lq.quantize(z).reshape(codes.shape), codes)
