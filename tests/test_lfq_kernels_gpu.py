"""The LFQ entropy kernels (vqb_lfq_entropy, vqb_lfq_entropy_backward) against the float64 dense oracle, every codebook
dimension d = 1..20, row lists, regimes on both sides of the 1e-5 clamp, determinism, and the d = 18 / 16384-row scale case.
The row kernels (forward, backward, decode) are tested in test_lfq_row_kernels_gpu.py."""
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
