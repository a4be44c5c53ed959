"""ResidualSimVQ on the GPU (`pytest -m gpu` on an H100): the reference's outputs and gradients (tests/golden/residual_simvq/),
the README invariant, coarse-index decode, a user-sized shape against float64, and the cached graph of the forward program."""
import ctypes

import numpy as np
import pytest
import torch

from residual_simvq_golden import Fixture, names

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def loaded(f):
    mod = f.build(vqb())
    mod.load_state_dict({k: torch.from_numpy(v) for k, v in f.state().items()})
    return mod.to(DEV).train()


@pytest.mark.parametrize("name", names())
def test_residual_simvq_matches_reference(name):
    f = Fixture(name)
    mod = loaded(f)
    x = torch.from_numpy(f["x"]).to(DEV).requires_grad_(True)
    G = torch.from_numpy(f["G"]).to(DEV)
    Lw = torch.from_numpy(f["Lw"]).to(DEV)
    q, ind, losses = mod(x, rand_quantize_dropout_fixed_seed=f.meta["dropout_seed"])
    ((q * G).sum() + (losses * Lw).sum()).backward()
    assert ind.dtype == torch.int64 and losses.shape == (mod.num_quantizers,)
    assert np.array_equal(ind.cpu().numpy(), f["indices"])
    np.testing.assert_allclose(q.detach().cpu().numpy(), f["quantized"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(losses.detach().cpu().numpy(), f["losses"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(x.grad.cpu().numpy(), f["xgrad"], rtol=1e-4, atol=2e-5)
    params = dict(mod.named_parameters())
    assert list(params) == f.meta["param_names"]
    for j, n in enumerate(f.meta["param_names"]):
        grad = params[n].grad
        got = grad.cpu().numpy() if grad is not None else np.zeros(tuple(params[n].shape), np.float32)
        np.testing.assert_allclose(got, f[f"pgrad_{j}"], rtol=1e-4, atol=2e-5, err_msg=n)
    # README invariant: the summed codes of the indices are the quantized output (dropped stages: index -1, zeros)
    with torch.no_grad():
        dec = mod.get_output_from_indices(ind)
    assert torch.allclose(q.detach(), dec, atol=1e-6)


def test_residual_simvq_codes_and_coarse_indices():
    m = vqb()
    torch.manual_seed(0)
    mod = m.ResidualSimVQ(dim=32, num_quantizers=4, codebook_size=48, quantize_dropout=True, channel_first=True).to(DEV).eval()
    x = torch.randn(2, 32, 5, 7, device=DEV)
    with torch.no_grad():
        q, ind, losses, all_codes = mod(x, return_all_codes=True)
        assert q.shape == x.shape and ind.shape == (2, 5, 7, 4) and all_codes.shape == (4, 2, 32, 5, 7)
        books = mod.codebooks
        for s in range(4):
            ref = books[s][ind[..., s]].movedim(-1, 1)
            assert torch.equal(all_codes[s], ref)
        assert torch.allclose(all_codes.sum(0), q, atol=1e-6)
        coarse = mod.get_output_from_indices(ind[..., :2])   # rsv:111-115: missing stages are padded with -1 (zeros)
        assert torch.allclose(coarse, all_codes[:2].sum(0), atol=1e-6)
    with pytest.raises(TypeError):
        mod(x.bfloat16())


def _stage_reference(x, books, indices, rotation, G, Lw, weight=1.0, input_weight=0.25):
    """rsv:182-203 as torch ops with the given stage indices (autograd runs in the dtype of x and books)."""
    r = x
    qout = 0.
    losses = []
    for s in range(indices.shape[1]):
        c = books[s][indices[:, s]]
        losses.append((torch.nn.functional.mse_loss(r.detach(), c) + torch.nn.functional.mse_loss(r, c.detach()) * input_weight) * weight)
        if rotation:
            ns, nt = r.norm(dim=-1, keepdim=True), c.norm(dim=-1, keepdim=True)
            u, qn = r / ns.clamp(min=1e-6), c / nt.clamp(min=1e-6)
            w = torch.nn.functional.normalize(u + qn, dim=-1, eps=1e-6).detach()
            e = r
            out = e - 2 * (e * w).sum(-1, keepdim=True) * w + 2 * (e * u.detach()).sum(-1, keepdim=True) * qn.detach()
            out = out * (nt / ns.clamp(min=1e-6)).detach()
        else:
            out = (c - r).detach() + r
        r = r - out.detach()
        qout = qout + out
    losses = torch.stack(losses)
    return qout, losses, (qout * G).sum() + (losses * Lw).sum()


# (D, stages, codes, rows): the user-sized shape, and rows that fill 2, 8 and 32 register slots per lane with a partial last slot
# (D = 40, 200) or the widest row (D = 1024, the backward's largest register footprint)
SHAPES = [(512, 4, 1024, 65536), (40, 3, 96, 4096), (200, 3, 160, 4096), (1024, 2, 256, 4096)]


@pytest.mark.parametrize("rotation", [True, False])
@pytest.mark.parametrize("D,Q,K,N", SHAPES)
def test_residual_simvq_user_shape_against_float64(D, Q, K, N, rotation):
    """Every stage's index is the float64 arg-min of its residual (rows whose two best distances lie within 1e-5 relative of each
    other excepted and counted), and the outputs, losses and the gradients to x and to the code transform match a float64 autograd
    run of the reference's op sequence with those indices."""
    m = vqb()
    torch.manual_seed(11)
    mod = m.ResidualSimVQ(dim=D, num_quantizers=Q, codebook_size=K, rotation_trick=rotation).to(DEV).train()
    x = torch.randn(8, N // 8, D, device=DEV).requires_grad_(True)
    G = torch.randn_like(x)
    Lw = torch.rand(Q, device=DEV) + 0.5
    q, ind, losses = mod(x)
    ((q * G).sum() + (losses * Lw).sum()).backward()
    idx = ind.reshape(N, Q)

    mod64 = m.ResidualSimVQ(dim=D, num_quantizers=Q, codebook_size=K, rotation_trick=rotation)
    mod64.load_state_dict(mod.state_dict())
    mod64 = mod64.to(DEV).double()
    x64 = x.detach().double().reshape(N, D).requires_grad_(True)
    books64 = [layer.codebook for layer in mod64.layers]
    near = 0
    with torch.no_grad():
        r = x64.detach()
        for s in range(Q):
            d = torch.cdist(r, books64[s])
            two = d.topk(2, largest=False)
            bad = idx[:, s] != two.indices[:, 0]
            gap = (two.values[:, 1] - two.values[:, 0]) / two.values[:, 1].clamp(min=1e-30)
            assert not (bad & (gap >= 1e-5)).any(), f"stage {s}: index differs from the float64 arg-min outside near ties"
            near += int(bad.sum())
            c = books64[s][idx[:, s]]
            r = r - c   # the estimator's value equals c up to rounding; the residual of the next stage's search
    assert near <= max(4, N // 1000), near
    q64, l64, total = _stage_reference(x64, books64, idx, rotation, G.double().reshape(N, D), Lw.double())
    total.backward()
    np.testing.assert_allclose(q.detach().reshape(N, D).cpu().numpy(), q64.detach().cpu().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(losses.detach().cpu().numpy(), l64.detach().cpu().numpy(), rtol=1e-5)
    gx, gx64 = x.grad.reshape(N, D).double(), x64.grad
    assert ((gx - gx64).abs().max() / gx64.abs().max()).item() < 1e-4
    for (n, p), (_, p64) in zip(mod.named_parameters(), mod64.named_parameters()):
        err = ((p.grad.double() - p64.grad).abs().max() / p64.grad.abs().max()).item()
        assert err < 1e-4, (n, err)


def test_residual_simvq_forward_replays_graph():
    """A repeated forward with the same shapes is served from the cached CUDA graph of its program."""
    m = vqb()
    from vector_quantize_pytorch_b200 import _C
    torch.manual_seed(1)
    mod = m.ResidualSimVQ(dim=64, num_quantizers=3, codebook_size=128).to(DEV).eval()
    x = torch.randn(4, 256, 64, device=DEV)

    def stats():
        out = (ctypes.c_longlong * 4)()
        _C.lib.vqb_debug_graph_stats(out)
        return list(out)

    with torch.no_grad():
        first = mod(x)
        for _ in range(3):
            out = mod(x)
            del out
        before = stats()
        again = mod(x)
        after = stats()
    torch.cuda.synchronize()
    assert after[0] == before[0] + 1 and after[2] == before[2], (before, after)
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1]) and torch.equal(first[2], again[2])
    assert len(mod.__dict__["_plans"]) == 1


def test_residual_simvq_plan_memory_lives_on_the_input_device():
    """A cached plan owns device memory, so it is keyed by the input's device; its buffers live there."""
    m = vqb()
    torch.manual_seed(2)
    devices = [torch.device("cuda", i) for i in range(min(2, torch.cuda.device_count()))]
    mod = m.ResidualSimVQ(dim=64, num_quantizers=3, codebook_size=128).eval()
    for dev in devices:
        mod = mod.to(dev)
        with torch.no_grad():
            q, ind, losses = mod(torch.randn(2, 128, 64, device=dev))
        assert q.device == ind.device == losses.device == dev
    plans = mod.__dict__["_plans"]
    assert sorted(k[0].index for k in plans) == [d.index for d in devices]
    for key, plan in plans.items():
        bufs = plan.bufs + [plan.loss_sum] + plan.prog.scratch_bufs + [o.planes for o in plan.operands]
        assert all(b.device == key[0] for b in bufs)


def test_residual_simvq_plan_memory_is_freed_with_the_plans():
    """Forwards over many distinct row counts keep at most 8 plans, and clearing the plans returns the device memory they held,
    their search scratch included."""
    import gc
    m = vqb()
    torch.manual_seed(3)
    mod = m.ResidualSimVQ(dim=128, num_quantizers=3, codebook_size=256).to(DEV).train()
    # the first forward and backward allocate library workspaces that live on (cuBLAS, for the code transform): before the baseline
    q, _, losses = mod(torch.randn(1, 64, 128, device=DEV, requires_grad=True))
    (q.sum() + losses.sum()).backward()
    del q, losses
    mod.__dict__["_plans"].clear()
    for p in mod.parameters():
        p.grad = None
    torch.cuda.synchronize()
    gc.collect()
    base = torch.cuda.memory_allocated()
    for n in range(20):
        x = torch.randn(1, 1000 + 37 * n, 128, device=DEV, requires_grad=True)
        q, _, losses = mod(x)
        (q.sum() + losses.sum()).backward()
        assert len(mod.__dict__["_plans"]) <= 8
    del x, q, losses
    mod.__dict__["_plans"].clear()
    torch.cuda.synchronize()
    gc.collect()
    # what remains is the parameters' gradients (allocated by the first backward)
    grads = sum(p.grad.numel() * 4 for p in mod.parameters() if p.grad is not None)
    assert torch.cuda.memory_allocated() - base <= grads + (1 << 20)


def test_residual_simvq_layers_must_agree_on_the_estimator():
    m = vqb()
    mod = m.ResidualSimVQ(dim=32, num_quantizers=2, codebook_size=16).to(DEV)
    mod.layers[1].rotation_trick = False
    with pytest.raises(ValueError, match="same gradient estimator"):
        mod(torch.randn(1, 8, 32, device=DEV))
