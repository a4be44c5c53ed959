"""The RandomProjectionQuantizer kernel (csrc/vq_rpq.cu, vqb_rpq_norm_project) called through the C ABI against float64, with
sentinel guards around the output and every case run twice (the same bits both times).

Bound (oracle/rpq_oracle.py, u = 2^-24, g(n) = n u / (1 - n u)), per element of row r, column c, with xn the float64 layer
norm of x and rstd its 1 / sqrt(var + 1e-5):
    2 [ g(dim) sum_d |xn_d P_dc| + sum_d ((er + 2u) |xn_d| + 2 dm rstd) |P_dc| ]
where dm = g(dim + 1) sum_d |x_d| / dim bounds the fp32 mean's error and er = 1.5 g(dim + 4) + 2u the relative error of the
fp32 rstd; without the norm only the product's g(dim) term remains.  Computed here in float64 on the device.
Rows span at least three waves of CTAs (two per SM) with a ragged last row tile.
"""
import pytest
import torch

from oracle import rpq_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 67
SENTINEL = -1.2345678e30
DIMS = [1, 7, 8, 81, 320, 512, 1024, 4096]
# output width H E -> (H, E): one head, several heads, wide heads
WIDTHS = {8: (1, 8), 16: (2, 8), 64: (4, 16), 256: (16, 16), 1024: (4, 256)}


def rows_for_waves(W, sms):
    """Row count that spans >= 3 waves of CTAs (2 per SM) and leaves the last row tile ragged."""
    bm, bn = (64, 16) if W <= 16 else (128, 64)
    col = -(-W // bn)
    tiles = -(-3 * 2 * sms // col) + 1
    return tiles * bm - 5


def run(x, proj, norm):
    from vector_quantize_pytorch_b200._C import lib
    N, dim = x.shape
    H, _, E = proj.shape
    buf = torch.full((N * H * E + 2 * GUARD,), SENTINEL, dtype=torch.float32, device=DEV)
    rc = lib.vqb_rpq_norm_project(x.data_ptr(), N, dim, proj.data_ptr(), H, E, int(norm), buf.data_ptr() + 4 * GUARD,
                                  torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    g = torch.cat([buf[:GUARD], buf[GUARD + N * H * E:]])
    assert bool((g == SENTINEL).all()), "the kernel wrote outside its output"
    return buf[GUARD:GUARD + N * H * E].view(N, H * E)


def reference64(x, proj, norm):
    """(float64 rows, per-element bound) on the device, as oracle/rpq_oracle.py computes them."""
    x = x.double()
    H, dim, E = proj.shape
    P = proj.double().permute(1, 0, 2).reshape(dim, H * E)
    Pa = P.abs()
    if norm:
        mean = x.mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + O.EPS)
        xn = (x - mean) * rstd
    else:
        xn = x
    b = O.gamma(dim) * (xn.abs() @ Pa)
    if norm:
        dm = O.gamma(dim + 1) * x.abs().sum(-1, keepdim=True) / dim
        er = 1.5 * O.gamma(dim + 4) + 2 * O.U
        b = b + ((er + 2 * O.U) * xn.abs() + 2 * dm * rstd) @ Pa
    return xn @ P, O.SAFETY * b


@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("W", sorted(WIDTHS))
@pytest.mark.parametrize("dim", DIMS)
def test_against_float64(dim, W, norm):
    H, E = WIDTHS[W]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = rows_for_waves(W, sms)
    g = torch.Generator(device=DEV).manual_seed(1000 * dim + W + int(norm))
    # rows with an offset and a spread of their own, so the mean matters
    x = torch.randn(N, dim, device=DEV, generator=g) * (0.5 + torch.rand(N, 1, device=DEV, generator=g) * 3) \
        + torch.randn(N, 1, device=DEV, generator=g) * 2
    proj = torch.randn(H, dim, E, device=DEV, generator=g) * (2.0 / (dim + E)) ** 0.5
    ours = run(x, proj, norm)
    ref, bound = reference64(x, proj, norm)
    err = (ours.double() - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert ratio <= 1.0, f"dim {dim} W {W} norm {norm}: worst error / bound {ratio:.3g}"
    again = run(x, proj, norm)
    assert torch.equal(ours.view(torch.int32), again.view(torch.int32)), "a rerun gave different bits"


def test_ops_wrapper_matches_entry_point():
    import vector_quantize_pytorch_b200.ops as ops
    x = torch.randn(3, 100, 81, device=DEV)
    proj = torch.randn(2, 81, 8, device=DEV)
    rows = ops.rpq_norm_project(x, proj, True)
    assert rows.shape == (300, 16)
    assert torch.equal(rows, run(x.reshape(300, 81), proj, True))
    with pytest.raises(TypeError):
        ops.rpq_norm_project(x.bfloat16(), proj, True)
