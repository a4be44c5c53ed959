"""Cross-path equivalences of VectorQuantize.forward that hold by construction, checked bit for bit (outputs, losses, gradients;
the codebook state after an EMA step to fp32 reordering, because the statistics add with atomics):

(a) separate codebooks per head == one VectorQuantize(dim=d) per head, run in head order on the head's slice with that head's
    codebook slot;
(b) heads sharing one codebook == a heads=1 module on the 'b n (h d) -> (b h) n d' rows; image, 3-D, channel-first and 2-D
    inputs == the rows module on the permuted input;
(c) LossBreakdown.commitment is the unweighted mse over the unmasked rows and `loss` is it weighted as vqp:1329, shared and
    masked (in-kernel mask, compacted Euclidean rows, compacted cosine rows);
(d) separate heads with DiVeQ == per-head DiVeQ modules, with the noise substituted through `diveq_noise`.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
K = 256
DTYPES = [torch.float32, torch.bfloat16]


def _vq(**kw):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    return m.VectorQuantize(codebook_size=K, **kw).to(DEV).train()


def _state(mod, slot=0):
    c = mod._codebook
    return [t[slot].detach().clone() for t in (c.cluster_size, c.embed_avg, c.embed)]


def _load(mod, state):
    c = mod._codebook
    with torch.no_grad():
        for buf, v in zip((c.cluster_size, c.embed_avg, c.embed), state):
            buf[0].copy_(v)


def _assert_state(got, want):
    for g, w in zip(got, want):
        torch.testing.assert_close(g, w, rtol=1e-6, atol=1e-5)


def _run(mod, x, grad, G, with_loss=True):
    """One training forward; with `grad` also the backward of <out, G> (+ loss).  Returns (out, ind, loss, x.grad)."""
    x = x.detach().clone().requires_grad_(grad)
    out, ind, loss = mod(x)
    if grad:
        ((out.float() * G).sum() + (loss if with_loss else 0.)).backward()
    return out.detach(), ind, loss.detach(), x.grad


def _equal(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a, b), f"{what}: {(a.float() - b.float()).abs().max().item()}"


# ------------------------------------------------------------------------------------------------ (a) separate heads
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("heads", [2, 4])
@pytest.mark.parametrize("grad,rotation", [(False, True), (True, True), (True, False)])
def test_separate_heads_equal_per_head_modules(dt, heads, grad, rotation):
    d, B, N = 64, 2, 1024
    sep = _vq(dim=heads * d, codebook_dim=d, heads=heads, separate_codebook_per_head=True, rotation_trick=rotation)
    per = [_vq(dim=d, rotation_trick=rotation) for _ in range(heads)]
    for i, m in enumerate(per):
        _load(m, _state(sep, i))
    gen = torch.Generator(device=DEV).manual_seed(heads * 10 + grad)
    x = torch.randn(B, N, heads * d, device=DEV, generator=gen).to(dt)
    G = torch.randn(B, N, heads * d, device=DEV, generator=gen)
    # the loss is one mean over all heads: its gradient is not the per-head modules' — the backward takes the output only
    out, ind, loss, xg = _run(sep, x, grad, G, with_loss=False)
    losses = []
    for i, m in enumerate(per):
        cols = slice(i * d, (i + 1) * d)
        o, j, l, g = _run(m, x[..., cols], grad, G[..., cols], with_loss=False)
        _equal(out[..., cols], o, f"quantize head {i}")
        _equal(ind[..., i], j, f"indices head {i}")
        if grad:
            _equal(xg[..., cols], g, f"x.grad head {i}")
        _assert_state(_state(sep, i), _state(m))
        losses.append(l)
    if not grad:   # kernel loss per head; one mse over all heads == the mean of the heads' (equal-sized) means
        _equal(loss, torch.stack(losses).mean(), "loss")


# ------------------------------------------------------------------------------------------------ (b) shared heads, layouts
def _heads_to_rows(t, h):
    b, n, hd = t.shape
    return t.reshape(b, n, h, hd // h).transpose(1, 2).reshape(b * h, n, hd // h)


LAYOUTS = {
    # name: (module kwargs, input shape, input -> rows, rows-module quantize -> output, rows-module indices -> output)
    "heads": (dict(dim=128, heads=2, codebook_dim=64), (2, 512, 128), lambda t: _heads_to_rows(t, 2),
              lambda q: q.reshape(2, 2, 512, 64).transpose(1, 2).reshape(2, 512, 128),
              lambda i: i.reshape(2, 2, 512).transpose(1, 2)),
    "image": (dict(dim=64, accept_image_fmap=True), (2, 64, 16, 32), lambda t: t.permute(0, 2, 3, 1).reshape(2, 512, 64),
              lambda q: q.reshape(2, 16, 32, 64).permute(0, 3, 1, 2), lambda i: i.reshape(2, 16, 32)),
    "3d": (dict(dim=64, accept_3d_fmap=True), (2, 64, 4, 8, 16), lambda t: t.permute(0, 2, 3, 4, 1).reshape(2, 512, 64),
           lambda q: q.reshape(2, 4, 8, 16, 64).permute(0, 4, 1, 2, 3), lambda i: i.reshape(2, 4, 8, 16)),
    "channel_first": (dict(dim=64, channel_last=False), (2, 64, 512), lambda t: t.transpose(1, 2),
                      lambda q: q.transpose(1, 2), lambda i: i),
    "2d": (dict(dim=64), (1024, 64), lambda t: t.unsqueeze(1), lambda q: q.squeeze(1), lambda i: i.squeeze(1)),
}


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("grad", [False, True])
def test_layouts_equal_rows_module(dt, layout, grad):
    kw, shape, to_rows, q_back, i_back = LAYOUTS[layout]
    mod = _vq(**kw)
    rows = _vq(dim=64)
    _load(rows, _state(mod))
    gen = torch.Generator(device=DEV).manual_seed(len(layout) * 2 + grad)
    x = torch.randn(shape, device=DEV, generator=gen).to(dt)
    G = torch.randn(shape, device=DEV, generator=gen)
    out, ind, loss, xg = _run(mod, x, grad, G)
    o, j, l, g = _run(rows, to_rows(x), grad, to_rows(G))
    _equal(out, q_back(o), "quantize")
    _equal(ind, i_back(j), "indices")
    _equal(loss, l, "loss")
    if grad:
        _equal(to_rows(xg), g, "x.grad")
    _assert_state(_state(mod), _state(rows))


# ------------------------------------------------------------------------------------------------ (c) LossBreakdown
BREAKDOWN = {
    # name: (module kwargs, masked)
    "shared": (dict(), False),
    "masked_in_kernel": (dict(), True),
    "masked_compacted": (dict(threshold_ema_dead_code=2), True),   # dead-code expiry samples x[mask]: compacted rows
    "masked_cosine": (dict(use_cosine_sim=True), True),            # mse against the un-normalised input (vqp:1319)
}


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", list(BREAKDOWN))
def test_loss_breakdown_is_unweighted_mse(dt, case):
    kw, masked = BREAKDOWN[case]
    mod = _vq(dim=64, commitment_weight=0.5, **kw)
    with torch.no_grad():
        mod._codebook.cluster_size.fill_(100.)   # no code expires
    gen = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(4, 300, 64, device=DEV, generator=gen).to(dt)
    lens = torch.tensor([300, 17, 256, 129], device=DEV)
    mask = torch.arange(300, device=DEV) < lens[:, None]
    out, ind, loss, bd = mod(x, mask=mask if masked else None, return_loss_breakdown=True)
    live = mask if masked else torch.ones_like(mask)
    mse = ((out[live].double() - x[live].double()) ** 2).mean().item()
    commit = bd.commitment.item()
    if dt == torch.float32:
        assert abs(commit - mse) <= 1e-5 * mse, (commit, mse)
    else:   # rounded once to bf16, like F.mse_loss in bf16: within one bf16 ulp
        assert abs(commit - mse) <= 2.0 ** -7 * mse, (commit, mse)
    # vqp:1329: commit_loss * commitment_weight in the input dtype, added to the fp32 `loss`
    want = (bd.commitment.to(dt) * 0.5).float()
    assert loss.dtype == torch.float32 and torch.equal(loss.detach(), want), (loss.item(), want.item())


# ------------------------------------------------------------------------------------------------ (d) separate heads + DiVeQ
@pytest.mark.parametrize("dt", DTYPES)
def test_separate_heads_diveq_equal_per_head_modules(dt, monkeypatch):
    import vector_quantize_pytorch_b200.vector_quantize as vqm
    heads, d, B, N = 2, 64, 2, 1024
    kw = dict(directional_reparam=True, learnable_codebook=False, threshold_ema_dead_code=2)
    sep = _vq(dim=heads * d, codebook_dim=d, heads=heads, separate_codebook_per_head=True, **kw)
    per = [_vq(dim=d, **kw) for _ in range(heads)]
    with torch.no_grad():
        sep._codebook.cluster_size.fill_(100.)   # no code expires: no RNG draw besides the noise
    for i, m in enumerate(per):
        _load(m, _state(sep, i))
    gen = torch.Generator(device=DEV).manual_seed(11)
    x = torch.randn(B, N, heads * d, device=DEV, generator=gen).to(dt)
    G = torch.randn(B, N, heads * d, device=DEV, generator=gen)
    Z = torch.randn(B, N, heads, d, device=DEV, generator=gen).to(dt)
    draws = [Z] + [Z[:, :, i] for i in range(heads)]   # the separate-heads module first, then the heads in order

    def noise(like):
        z = draws.pop(0)
        assert z.shape == like.shape and z.dtype == like.dtype
        return z.contiguous()

    monkeypatch.setattr(vqm, "diveq_noise", noise)
    out, ind, loss, xg = _run(sep, x, True, G, with_loss=False)
    for i, m in enumerate(per):
        cols = slice(i * d, (i + 1) * d)
        o, j, _, g = _run(m, x[..., cols], True, G[..., cols], with_loss=False)
        _equal(ind[..., i], j, f"indices head {i}")
        _equal(out[..., cols], o, f"quantize head {i}")
        _equal(xg[..., cols], g, f"x.grad head {i}")
        _assert_state(_state(sep, i), _state(m))
    assert not draws
