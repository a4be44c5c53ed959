"""The HierarchicalVQ kernels (csrc/vq_hvq.cu) called through the C ABI against float64 and against torch's own
adaptive_avg_pool2d / interpolate on the device, with sentinel guard rows around every output and every backward run twice
(the gather-form adjoints must give the same bits).

Per-element bounds, u = 2^-24, for a map y = sum_t w_t v_t evaluated in fp32 with n terms:
    |y - y64| <= (n + c) u sum_t |w_t v_t|
which is the map applied to |v| in float64 times (n + c) u.  The pool has n = kh kw and c = 3 (two divisions).  The bilinear
map and its adjoint take their taps' weights from a source index src <= s computed in fp32 (torch's float64 reference in
float64), which moves a weight by up to 4 (s + 1) u whatever the weight: that term is bounded with the largest |v| of the
element's (b, d) plane, times the number of terms.  The upsample has 4 terms plus 8 roundings; its adjoint at most
(ceil(H / s) + 4)(ceil(W / s) + 4) terms.  torch's fp32 result is held to twice the bound.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
GUARD = 67   # floats of sentinel before and after every output
SENTINEL = -1.2345678e30

SIDES = list(range(1, 18)) + [32, 64]


def _lib():
    from vector_quantize_pytorch_b200._C import lib
    return lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Guarded:
    """An fp32 output of n elements inside sentinel guards."""

    def __init__(self, shape):
        n = 1
        for v in shape:
            n *= v
        self.buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32, device=DEV)
        self.shape = shape
        self.n = n

    @property
    def ptr(self):
        return self.buf.data_ptr() + 4 * GUARD

    def value(self):
        g = torch.cat([self.buf[:GUARD], self.buf[GUARD + self.n:]])
        assert bool((g == SENTINEL).all()), "a kernel wrote outside its output"
        return self.buf[GUARD:GUARD + self.n].view(self.shape)


def check_bound(ours, ref64, bound, what):
    err = (ours.double() - ref64).abs()
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements over the bound, worst ratio {float((err / bound).max()):.3g}"
    return float((err / bound).max())


def pool(x, s):
    B, D, H, W = x.shape
    out = Guarded((B, s, s, D))
    assert _lib().vqb_hvq_pool(x.data_ptr(), B, D, H, W, s, out.ptr, _stream()) == 0
    return out.value().permute(0, 3, 1, 2)


def pool_bwd(g_rows, H, W):
    B, s, _, D = g_rows.shape
    out = Guarded((B, D, H, W))
    assert _lib().vqb_hvq_pool_backward(g_rows.data_ptr(), B, D, H, W, s, out.ptr, _stream()) == 0
    return out.value()


def upsample(rows, H, W, recon=None, resid=None, outs=(True, False, False)):
    B, s, _, D = rows.shape
    g = [Guarded((B, D, H, W)) if w else None for w in outs]
    p = [x.ptr if x is not None else None for x in g]
    rc = _lib().vqb_hvq_upsample(rows.data_ptr(), B, D, s, H, W, p[0], None if recon is None else recon.data_ptr(),
                                 None if resid is None else resid.data_ptr(), p[1], p[2], _stream())
    assert rc == 0
    return [x.value() if x is not None else None for x in g]


def upsample_bwd(ga, gb, s):
    ref = ga if ga is not None else gb
    B, D, H, W = ref.shape
    out = Guarded((B, s, s, D))
    rc = _lib().vqb_hvq_upsample_backward(None if ga is None else ga.data_ptr(), None if gb is None else gb.data_ptr(), B, D, s,
                                          H, W, out.ptr, _stream())
    assert rc == 0
    return out.value().permute(0, 3, 1, 2)


def up64(q, H, W):
    """torch's float64 bilinear map (its source index in float64: the bound carries the kernels' fp32 source index)."""
    s = q.shape[-1]
    if (s, s) == (H, W):
        return q.double()
    return F.interpolate(q.double(), size=(H, W), mode="bilinear", align_corners=False)


def up_adj64(g, s):
    H, W = g.shape[-2:]
    if (s, s) == (H, W):
        return g.double()
    q = torch.zeros(g.shape[:2] + (s, s), dtype=torch.float64, device=DEV, requires_grad=True)
    F.interpolate(q, size=(H, W), mode="bilinear", align_corners=False).backward(g.double())
    return q.grad


def pool_adj64(g, H, W):
    x = torch.zeros(g.shape[:2] + (H, W), dtype=torch.float64, device=DEV, requires_grad=True)
    F.adaptive_avg_pool2d(x, g.shape[-2:]).backward(g.double())
    return x.grad


def plane_max(t):
    """The largest |value| of each (b, d) plane, broadcast over the plane, in float64."""
    return t.abs().double().amax(dim=(-2, -1), keepdim=True)


def _windows(n, s):
    return [(i * n) // s for i in range(s)], [-(-((i + 1) * n) // s) for i in range(s)]


def run_shape(B, D, H, W, s, gen):
    x = torch.randn(B, D, H, W, device=DEV, generator=gen)
    # pool
    p = pool(x, s)
    p64 = F.adaptive_avg_pool2d(x.double(), (s, s))
    st, en = _windows(H, s)
    kh = max(e - a for a, e in zip(st, en))
    st, en = _windows(W, s)
    kw = max(e - a for a, e in zip(st, en))
    bound = (kh * kw + 3) * U * F.adaptive_avg_pool2d(x.abs().double(), (s, s)) + 1e-37
    check_bound(p, p64, bound, f"pool {H}x{W}->{s}")
    check_bound(F.adaptive_avg_pool2d(x, (s, s)), p64, 2 * bound, "torch pool")
    # pool backward, twice
    g_rows = torch.randn(B, s, s, D, device=DEV, generator=gen)
    gx = pool_bwd(g_rows, H, W)
    assert torch.equal(gx, pool_bwd(g_rows, H, W)), "pool backward is not repeatable"
    g_img = g_rows.permute(0, 3, 1, 2)
    n_terms = (-(-s // H) + 1) * (-(-s // W) + 1)
    bound = (n_terms + 3) * U * pool_adj64(g_img.abs(), H, W) + 1e-37
    check_bound(gx, pool_adj64(g_img, H, W), bound, f"pool backward {H}x{W}->{s}")
    # upsample from the rows
    rows = torch.randn(B, s, s, D, device=DEV, generator=gen)
    q_img = rows.permute(0, 3, 1, 2)
    (u,) = [v for v in upsample(rows, H, W) if v is not None]
    lam = 4 * (s + 1) * U
    bound = 12 * U * up64(q_img.abs(), H, W) + 4 * lam * plane_max(q_img) + 1e-37
    if (s, s) == (H, W):
        assert torch.equal(u, q_img), "the same-size upsample is a copy"
    else:
        check_bound(u, up64(q_img, H, W), bound, f"upsample {s}->{H}x{W}")
        check_bound(F.interpolate(q_img, size=(H, W), mode="bilinear", align_corners=False), up64(q_img, H, W), 2 * bound,
                    "torch interpolate")
    # upsample backward, twice; with both gradients (g_a - g_b)
    ga = torch.randn(B, D, H, W, device=DEV, generator=gen)
    gb = torch.randn(B, D, H, W, device=DEV, generator=gen)
    n_terms = (-(-H // s) + 4) * (-(-W // s) + 4)
    for a, b in ((ga, None), (ga, gb), (None, gb)):
        gq = upsample_bwd(a, b, s)
        assert torch.equal(gq, upsample_bwd(a, b, s)), "upsample backward is not repeatable"
        g = (a.double() if a is not None else 0) - (b.double() if b is not None else 0)
        gabs = (a.abs().double() if a is not None else 0) + (b.abs().double() if b is not None else 0)
        bound = (n_terms + 12) * U * up_adj64(gabs, s) + n_terms * lam * plane_max(gabs) + 1e-37
        check_bound(gq, up_adj64(g, s), bound, f"upsample backward {s}->{H}x{W}")
    return u


def test_every_side_and_scale_d8():
    gen = torch.Generator(device=DEV).manual_seed(0)
    for H in SIDES:
        for W in (H, SIDES[(SIDES.index(H) + 5) % len(SIDES)]):
            for s in range(1, max(H, W) + 3):
                run_shape(2, 8, H, W, s, gen)


@pytest.mark.parametrize("D", [32, 256, 1024])
def test_wide_rows_several_waves(D):
    """Enough elements for several grid-stride waves (the grid is capped at 8 CTAs of 256 threads per SM)."""
    gen = torch.Generator(device=DEV).manual_seed(D)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wave = sms * 8 * 256
    for H, W, scales in ((16, 16, (1, 2, 3, 5, 8, 13, 16, 18)), (17, 9, (4, 17, 19)), (32, 32, (7, 31, 32)), (64, 64, (1, 13, 64))):
        B = max(1, -(-3 * wave // (D * H * W)))
        B = min(B, max(1, (1 << 27) // (D * H * W)))
        for s in scales:
            run_shape(B, D, H, W, s, gen)


@pytest.mark.parametrize("H,W,s", [(7, 7, 4), (9, 12, 5), (6, 6, 6), (5, 5, 7), (16, 16, 1)])
def test_fused_updates(H, W, s):
    """upsample's recon + u / resid - u, and the blend (1 - r) up + r conv with its updates and backward, bit for bit against
    the same fp32 operations in torch (no fma: each is one correctly rounded operation)."""
    gen = torch.Generator(device=DEV).manual_seed(H * W * s)
    B, D = 3, 32
    rows = torch.randn(B, s, s, D, device=DEV, generator=gen)
    recon = torch.randn(B, D, H, W, device=DEV, generator=gen)
    resid = torch.randn(B, D, H, W, device=DEV, generator=gen)
    u, ro, so = upsample(rows, H, W, recon, resid, outs=(True, True, True))
    assert torch.equal(ro, recon + u) and torch.equal(so, resid - u)
    _, r0, none = upsample(rows, H, W, None, None, outs=(False, True, False))
    assert none is None and torch.equal(r0, torch.zeros_like(u) + u)
    lib = _lib()
    conv = torch.randn(B, D, H, W, device=DEV, generator=gen)
    for r in (0.5, 0.25, 0.1, 1.0 / 3.0):
        a, rf = torch.tensor(1.0 - r, dtype=torch.float32).item(), torch.tensor(r, dtype=torch.float32).item()
        q = u * a + conv * rf
        out_r, out_s = Guarded((B, D, H, W)), Guarded((B, D, H, W))
        assert lib.vqb_hvq_blend_update(u.data_ptr(), conv.data_ptr(), u.numel(), r, recon.data_ptr(), resid.data_ptr(),
                                        out_r.ptr, out_s.ptr, _stream()) == 0
        assert torch.equal(out_r.value(), recon + q) and torch.equal(out_s.value(), resid - q)
        out_r = Guarded((B, D, H, W))
        assert lib.vqb_hvq_blend_update(u.data_ptr(), conv.data_ptr(), u.numel(), r, None, None, out_r.ptr, None,
                                        _stream()) == 0
        assert torch.equal(out_r.value(), torch.zeros_like(q) + q)
        for g_r, g_s in ((recon, resid), (recon, None), (None, resid)):
            gu, gc = Guarded((B, D, H, W)), Guarded((B, D, H, W))
            assert lib.vqb_hvq_blend_backward(None if g_r is None else g_r.data_ptr(), None if g_s is None else g_s.data_ptr(),
                                              u.numel(), r, gu.ptr, gc.ptr, _stream()) == 0
            gq = (g_r if g_r is not None else 0) - (g_s if g_s is not None else 0)
            if g_r is None:
                gq = -g_s
            assert torch.equal(gu.value(), gq * a) and torch.equal(gc.value(), gq * rf)
