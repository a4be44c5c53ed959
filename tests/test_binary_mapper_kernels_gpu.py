"""The vqb_binmap_* kernels called directly against float64: every bits value, ragged and multi-wave row counts, every
backward plan, saturated soft codes, the non-finite patterns, strided and offset upstream gradients, offsets past 2^31 and
the memory the forward and backward allocate."""
import numpy as np
import pytest
import torch

from oracle import binary_mapper_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from vector_quantize_pytorch_b200 import ops
    return ops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hot_f32(l: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """fl(fl(1 + s) - s), s = exp of the float32 sum of the hot code's log-sigmoids."""
    lt = torch.from_numpy(l.astype(np.float32))
    c = torch.from_numpy(O.index_bits(idx, l.shape[1]))
    s = torch.where(c, torch.nn.functional.logsigmoid(lt), torch.nn.functional.logsigmoid(-lt)).sum(-1).exp()
    return ((1.0 + s) - s).numpy()


def _forward(l: torch.Tensor, idx: torch.Tensor, st=True):
    rows, bits = l.shape
    out = torch.zeros((rows, 1 << bits), dtype=torch.float32, device=DEV)
    _ops().binmap_hot(out, l if st else None, idx)
    return out


def _check_forward(l, idx, out, st=True):
    rows = l.shape[0]
    r = torch.arange(rows, device=DEV)
    hot = out[r, idx].cpu().numpy()
    assert int(torch.count_nonzero(out)) == int(torch.count_nonzero(out[r, idx]))
    if st:
        ref = _hot_f32(l.cpu().numpy(), idx.cpu().numpy())
        assert (np.abs(hot.astype(np.float64) - ref) <= 2.0 ** -23).all()
    else:
        assert (hot == 1.0).all()


def _dl64(l: np.ndarray, g: np.ndarray):
    """float64 closed form and the per-row scale sum_k |g_k s_k| (rows with a non-finite logit: NaN)."""
    w = np.abs(g.astype(np.float64)) * O.soft_codes(l)
    return O.st_grad(l, g), w.sum(-1)


def _check_backward(dl: torch.Tensor, l: torch.Tensor, g: torch.Tensor):
    ref, scale = _dl64(l.cpu().numpy().astype(np.float64), g.cpu().numpy())
    ours = dl.cpu().numpy().astype(np.float64)
    np.testing.assert_array_equal(np.isnan(ours), np.isnan(ref))
    ok = ~np.isnan(ref)
    err = np.where(ok, np.abs(ours - np.nan_to_num(ref)), 0.0)
    assert (err <= 1e-5 * scale[:, None] + 1e-30).all(), f"max relative error {(err / scale[:, None]).max():.3g}"


def _data(rows, bits, seed, scale=2.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    l = torch.randn(rows, bits, device=DEV, generator=g) * scale
    idx = torch.randint(0, 1 << bits, (rows,), device=DEV, generator=g)
    G = torch.randn(rows, 1 << bits, device=DEV, generator=g)
    return l, idx, G


@pytest.mark.parametrize("bits", list(range(1, 21)))
def test_every_bits_value(bits):
    rows = max(1, min(129, (1 << 22) >> bits))
    l, idx, G = _data(rows, bits, bits)
    for st in (True, False):
        _check_forward(l, idx, _forward(l, idx, st), st)
    _check_backward(_ops().binmap_backward(l, G), l, G)


@pytest.mark.parametrize("rows", [1, 7, 129, 70001])
@pytest.mark.parametrize("bits", [3, 8])
def test_ragged_rows_and_grid_waves(rows, bits):
    l, idx, G = _data(rows, bits, rows + bits)
    _check_forward(l, idx, _forward(l, idx))
    ks, _ = _ops().binmap_backward_plan(rows, bits, _sms())
    assert rows < 70001 or (rows * ks + 127) // 128 > 2 * _sms(), "several waves of CTAs"
    _check_backward(_ops().binmap_backward(l, G), l, G)


@pytest.mark.parametrize("bits", [1, 2, 3, 4, 5, 6, 9, 13])
def test_every_split(bits):
    """Every K split the ABI accepts (a power of two up to the segment count) gives the float64 result, and every segment
    width (2 to 32 codes) is reached."""
    l, idx, G = _data(33, bits, 100 + bits)
    nseg = max(1, (1 << bits) // 32)
    ks = 1
    while ks <= nseg:
        _check_backward(_ops().binmap_backward(l, G, ksplit=ks), l, G)
        ks *= 2


@pytest.mark.parametrize("rows,bits", [(1, 20), (3, 18), (64, 14), (1024, 12), (8192, 10), (1 << 15, 8)])
def test_planned_shapes(rows, bits):
    """Shapes on which the planner picks different splits, run with the plan."""
    ks, seg = _ops().binmap_backward_plan(rows, bits, _sms())
    print(f"rows {rows} bits {bits}: ksplit {ks}, segment {seg}")
    l, idx, G = _data(rows, bits, rows * 31 + bits)
    sel = torch.arange(0, rows, max(1, rows // 64), device=DEV)
    dl = _ops().binmap_backward(l, G)
    _check_backward(dl[sel], l[sel], G[sel])


@pytest.mark.parametrize("bits", [4, 8, 16])
def test_saturated_soft_codes(bits):
    """Logits +-30: the hot soft code is near 1 or near 0; sigmoid(l) rounds to 1 in float32."""
    rows = 64
    g = torch.Generator(device=DEV).manual_seed(bits)
    l = torch.where(torch.randn(rows, bits, device=DEV, generator=g) > 0, 30.0, -30.0)
    l[1::2] *= torch.rand(rows // 2, bits, device=DEV, generator=g)
    likely = ((l > 0).long() << torch.arange(bits, device=DEV)).sum(-1)
    idx = torch.where(torch.arange(rows, device=DEV) % 4 == 0, likely ^ 1, likely)   # some rows hot on an unlikely code
    out = _forward(l, idx)
    _check_forward(l, idx, out)
    G = torch.randn(rows, 1 << bits, device=DEV, generator=g)
    _check_backward(_ops().binmap_backward(l, G), l, G)


@pytest.mark.parametrize("bits", [1, 3, 8, 17])
def test_nonfinite_rows(bits):
    rows = 6
    l, idx, G = _data(rows, bits, 7 * bits)
    l[0, 0] = float("nan")
    l[1, bits - 1] = float("inf")
    l[2, 0] = -float("inf")
    if bits > 1:
        l[3, 0], l[3, 1] = float("inf"), -float("inf")
    out = _forward(l, idx).cpu().numpy()
    ln = l.cpu().numpy().astype(np.float64)
    c = O.codes(bits)
    nan = np.isnan(ln).any(-1)[:, None] | (c[None] & (ln[:, None, :] == np.inf)).any(-1) | \
        (~c[None] & (ln[:, None, :] == -np.inf)).any(-1)
    np.testing.assert_array_equal(np.isnan(out), nan)
    hot = np.zeros_like(nan)
    hot[np.arange(rows), idx.cpu().numpy()] = True
    assert (out[~nan & ~hot] == 0).all() and not np.signbit(out[~nan & ~hot]).any()
    fin = np.isfinite(ln).all(-1)
    _check_forward(l[torch.from_numpy(fin).to(DEV)], idx[torch.from_numpy(fin).to(DEV)],
                   torch.from_numpy(out[fin]).to(DEV))
    dl = _ops().binmap_backward(l, G).cpu().numpy()
    assert np.isnan(dl[~fin]).all() and np.isfinite(dl[fin]).all()


def test_upstream_layouts_give_identical_bits():
    """g contiguous, broadcast over rows (row stride 0), offset by one float, and a column stride of 0 (out.sum().backward()):
    the kernel reads each in place and gives the same bits as the contiguous copy."""
    rows, bits = 300, 12
    K = 1 << bits
    l, _, _ = _data(rows, bits, 5)
    row = torch.randn(K, device=DEV)
    ops = _ops()
    for ks in (1, 4):
        a = ops.binmap_backward(l, row.expand(rows, K).contiguous(), ksplit=ks)
        b = ops.binmap_backward(l, row.expand(rows, K), ksplit=ks)
        buf = torch.empty(rows * K + 1, device=DEV)
        buf[1:] = row.repeat(rows)
        c = ops.binmap_backward(l, buf[1:].view(rows, K), ksplit=ks)
        assert torch.equal(a, b) and torch.equal(a, c)
        d = ops.binmap_backward(l, torch.ones((), device=DEV).expand(rows, K), ksplit=ks)
        e = ops.binmap_backward(l, torch.ones(rows, K, device=DEV), ksplit=ks)
        assert torch.equal(d, e)
        f = ops.binmap_backward(l, torch.ones(rows, 2 * K, device=DEV)[:, ::2], ksplit=ks)   # column stride 2
        assert torch.equal(f, e)
    _check_backward(a, l, row.expand(rows, K))
    again = ops.binmap_backward(l, row.expand(rows, K).contiguous(), ksplit=4)
    assert torch.equal(a, again), "identical calls give identical bits"


def test_offsets_past_2_31():
    """32769 rows at 16 bits: 2^31 + 2^16 output elements (8 GiB); the last rows are checked."""
    rows, bits = 32769, 16
    K = 1 << bits
    g = torch.Generator(device=DEV).manual_seed(11)
    l = torch.randn(rows, bits, device=DEV, generator=g) * 2
    idx = torch.randint(0, K, (rows,), device=DEV, generator=g)
    x = l.clone().requires_grad_(True)
    from vector_quantize_pytorch_b200.binary_mapper import _BinaryMapperST
    out = _BinaryMapperST.apply(x, idx, K)
    assert out.numel() > 2 ** 31
    tail = torch.arange(rows - 5, rows, device=DEV)
    _check_forward(l[tail], idx[tail], out.detach()[tail])
    assert int(torch.count_nonzero(out)) == rows
    out.sum().backward()   # the upstream gradient is a (rows, K) view of one float
    del out
    torch.cuda.empty_cache()
    _check_backward(x.grad[tail], l[tail], torch.ones(5, K, device=DEV))


def test_peak_memory_at_16_bits():
    """8192 rows at 16 bits: the forward allocates its (rows, 2^16) output and O(rows * bits) beyond it; the backward
    dlogits, the plan's workspace and O(rows * bits)."""
    import vector_quantize_pytorch_b200 as vqb
    rows, bits = 8192, 16
    K = 1 << bits
    m = vqb.BinaryMapper(bits=bits).to(DEV).train()
    x = torch.randn(rows, bits, device=DEV, requires_grad=True)
    G = torch.randn(rows, K, device=DEV)
    small = 64 * rows * bits * 4   # generous room for the O(rows * bits) torch ops of the draw, the index and the aux loss
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out, aux = m(x)
    torch.cuda.synchronize()
    fwd = torch.cuda.max_memory_allocated() - base
    out_bytes = rows * K * 4
    print(f"forward peak beyond inputs: {fwd / 2**20:.1f} MiB (output {out_bytes / 2**20:.0f} MiB)")
    assert fwd <= out_bytes + small
    ks, _ = _ops().binmap_backward_plan(rows, bits, _sms())
    work = rows * ks * 2 * bits * 8 if ks > 1 else 0
    for how in ("kernel", "autograd"):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        if how == "kernel":
            dx = _ops().binmap_backward(x.detach(), G)
        else:
            (dx,) = torch.autograd.grad(out, x, G, retain_graph=True)
        torch.cuda.synchronize()
        bwd = torch.cuda.max_memory_allocated() - base
        print(f"backward peak ({how}): {bwd / 2**20:.2f} MiB (workspace {work / 2**20:.1f} MiB, ksplit {ks})")
        assert bwd <= rows * bits * 4 + work + small
        del dx
    dx = _ops().binmap_backward(x.detach(), G)
    sel = torch.arange(0, rows, 512, device=DEV)
    _check_backward(dx[sel], x.detach()[sel], G[sel])
