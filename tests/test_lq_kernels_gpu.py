"""vqb_lq_quantize / vqb_lq_loss / vqb_lq_loss_backward on the GPU against oracle/lq_oracle.py.

Quantize: table sizes 2 to the cap (VQB_LQ_MAX_VALUES), sorted, unsorted and duplicated, fp32 and bf16 rows, planted midpoints,
on-table values, +-0, |z| of 1e4 and 1e8, NaN and +-inf.  Codes and indices must equal the fp32 oracle bit for bit.  A NaN z
has NaN distances only, so index 0 wins and its code is NaN; +-inf give infinite distances everywhere, index 0, and the code
inf + (v - inf) = NaN.  The packed index of a row with a NaN code is 0 (cvt.rzi of NaN; x86 gives INT_MIN for the reference
on the CPU).  Launches span at least three passes of the grid-stride loop with a ragged tail, outputs sit between sentinel
guards, and a second run must give the same bits.  Loss: within the float64 bound, the same bits twice; backward: the
elementwise formula in fp32."""
import numpy as np
import pytest
import torch

from oracle import lq_oracle as O

pytestmark = pytest.mark.gpu

GUARD = 4096
SENT_F, SENT_I = 0x7FA5A5A5, -0x5A5A5A5B


def _lib():
    from vector_quantize_pytorch_b200._C import lib
    return lib


def grid_items():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256   # capped_grid(items, 256, 8) x 256 threads


def make_tables(L, D, order, gen):
    out = []
    for i in range(D):
        Li = max(2, L - i)
        v = (torch.rand(Li, generator=gen) - 0.5).float()
        if order == "sorted":
            v = v.sort().values
        elif order == "dup":
            v[Li // 2:] = v[: Li - Li // 2].clone()
            v[0] = v[-1]
        out.append(v)
    return out


def planted_rows(tables, N, C, D, gen):
    z = torch.randn(N, C, D, generator=gen) * 0.4
    flat = z.view(-1, D)
    for i, v in enumerate(tables):
        s = np.sort(v.numpy())
        mids = ((s[:-1].astype(np.float64) + s[1:]) / 2).astype(np.float32)
        special = np.concatenate([mids[:512], s[:512], np.float32([0.0, -0.0, 1e4, -1e4, 1e8, -1e8, np.nan, np.inf,
                                                                    -np.inf, 3e38, -3e38])])
        rows = (np.arange(len(special)) * 13 + 5 * i) % flat.shape[0]
        flat[rows, i] = torch.from_numpy(special)
    return z


def run_quantize(z, C, tables, levels, basis):
    lib = _lib()
    dev = z.device
    N, D = z.shape[0], len(tables)
    vals = torch.cat(tables).to(dev)
    meta = torch.tensor([[t.numel() for t in tables], [l // 2 for l in levels], basis], dtype=torch.int32).to(dev)
    codes_buf = torch.full((N * C * D + 2 * GUARD,), SENT_F, dtype=torch.int32, device=dev).view(torch.float32)
    idx_buf = torch.full((N * C + 2 * GUARD,), SENT_I, dtype=torch.int32, device=dev)
    codes = codes_buf[GUARD:GUARD + N * C * D]
    idx = idx_buf[GUARD:GUARD + N * C]
    dt = 1 if z.dtype == torch.bfloat16 else 0
    rc = lib.vqb_lq_quantize(z.data_ptr(), dt, N, C, D, vals.data_ptr(), vals.numel(), meta.data_ptr(), codes.data_ptr(),
                             idx.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    cb = codes_buf.view(torch.int32)
    assert (cb[:GUARD] == SENT_F).all() and (cb[-GUARD:] == SENT_F).all(), "codes guard overwritten"
    assert (idx_buf[:GUARD] == SENT_I).all() and (idx_buf[-GUARD:] == SENT_I).all(), "index guard overwritten"
    return codes.clone(), idx.clone()


CASES = [(2, 3, 1), (3, 3, 2), (7, 5, 1), (12, 3, 4), (64, 4, 1), (1000, 2, 1), (8192, 1, 1), (4096, 2, 1)]


@pytest.mark.parametrize("L,D,C", CASES)
@pytest.mark.parametrize("order", ["sorted", "unsorted", "dup"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_quantize_matches_oracle(L, D, C, order, dtype):
    gen = torch.Generator().manual_seed(L * 1000 + D * 10 + C)
    tables = make_tables(L, D, order, gen)
    levels = [t.numel() for t in tables]
    basis = np.cumprod([1] + levels[:-1]).tolist()
    if np.prod(levels, dtype=np.float64) >= 2 ** 31:
        basis = [1] * D
    # three passes of the grid-stride loop and a ragged tail for the small tables; fewer rows where the oracle's
    # (rows x table) distance matrix would not fit
    items = 3 * grid_items() + 77 if sum(levels) <= 64 else 4099
    N = (items + C - 1) // C
    z = planted_rows(tables, N, C, D, gen).to(dtype)
    zc = z.cuda().contiguous()
    codes, idx = run_quantize(zc, C, tables, levels, basis)
    zo = z.float().numpy()
    ref_codes, ref_idx = O.quantize(zo, [t.numpy() for t in tables], levels, basis)
    got = codes.view(N, C, D).cpu().numpy()
    nan = np.isnan(ref_codes)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got.view(np.uint32)[~nan], ref_codes.view(np.uint32)[~nan])   # bits: signed zeros too
    np.testing.assert_array_equal(idx.view(N, C).cpu().numpy(), ref_idx)
    nan_rows = np.isnan(ref_codes).any(-1)
    assert nan_rows.any() and (ref_idx[nan_rows] == 0).all()
    codes2, idx2 = run_quantize(zc, C, tables, levels, basis)
    assert torch.equal(codes.view(torch.int32), codes2.view(torch.int32)) and torch.equal(idx, idx2)


def test_large_index_rounding_and_huge_z():
    """levels [256, 256, 257]: every lattice point's fp32 sum, rounded above 2^24, and rows at |z| 1e8 whose codes leave the
    lattice."""
    gen = torch.Generator().manual_seed(7)
    levels = [256, 256, 257]
    tables = [torch.arange(256) / 256 - 0.5, torch.arange(256) / 256 - 0.5, torch.linspace(-0.5, 0.5, 257)]
    basis = [1, 256, 65536]
    k = torch.stack([torch.randint(0, l, (1 << 20,), generator=gen) for l in levels], -1)
    z = torch.stack([tables[i][k[:, i]] for i in range(3)], -1)
    z[::97] = 1e8
    z[1::97] = -1e8
    codes, idx = run_quantize(z.cuda().contiguous(), 1, [t.float() for t in tables], levels, basis)
    ref_codes, ref_idx = O.quantize(z.numpy()[:, None, :], [t.float().numpy() for t in tables], levels, basis)
    np.testing.assert_array_equal(codes.view(-1, 1, 3).cpu().numpy(), ref_codes)
    np.testing.assert_array_equal(idx.view(-1, 1).cpu().numpy(), ref_idx)
    assert (ref_idx[:, 0] != (k * torch.tensor(basis)).sum(-1).numpy()).any()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 1000, 8192, 8193, 3 * 1024 * 8192 + 5])
@pytest.mark.parametrize("use", [(1, 1), (1, 0), (0, 1)])
def test_loss_and_backward(dtype, n, use):
    from vector_quantize_pytorch_b200 import ops
    gen = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=gen).to(dtype).cuda()
    out = (torch.randn(n, generator=gen) * 0.5).cuda()
    wc = torch.tensor(0.1, device="cuda")
    wq = torch.tensor(0.25, device="cuda")
    loss = ops.lq_loss(x, out, wc, wq, *map(bool, use))
    loss2 = ops.lq_loss(x, out, wc, wq, *map(bool, use))
    assert torch.equal(loss.view(torch.int32), loss2.view(torch.int32))
    l64, bound = O.loss64(x.float().cpu().numpy(), out.cpu().numpy(), 0.1, 0.25, *use)
    assert abs(loss.item() - l64) <= bound + abs(l64) * 2.0 ** -22   # the fp32 weights against their decimal values
    g = torch.tensor(1.7, device="cuda")
    gx, gout = ops.lq_loss_backward(x, out, g, wc, wq, *map(bool, use))
    norm = torch.tensor(2.0 / n, dtype=torch.float32)
    xf, of = x.float().cpu(), out.cpu()
    ref_gx = (norm * (xf - of)) * (wq.cpu() * g.cpu()) if use[1] else torch.zeros(n)
    ref_go = (norm * (of - xf)) * (wc.cpu() * g.cpu()) if use[0] else torch.zeros(n)
    assert torch.equal(gx.cpu(), ref_gx.to(dtype))
    assert torch.equal(gout.cpu(), ref_go)
