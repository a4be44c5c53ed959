"""FSQ, ResidualFSQ and GroupedResidualFSQ on the GPU (csrc/vq_fsq.cu): every reference fixture replays through the modules,
seeded kernel cases against the numpy restatement (oracle/fsq_oracle.py, rounding boundaries recomputed in float64), the
reference's two invariants, the backward, and one forward launch for all groups.  Contract: DESIGN.md §4.9."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import fsq_oracle as O
from fsq_golden import FIXTURES, Case, fixture_id, flipped_rows, part_rows

import vector_quantize_pytorch_b200 as vqb
from vector_quantize_pytorch_b200 import ops
from vector_quantize_pytorch_b200.fsq import fsq_tables

pytestmark = pytest.mark.gpu

DEV = "cuda"
CLASSES = {"FSQ": vqb.FSQ, "ResidualFSQ": vqb.ResidualFSQ, "GroupedResidualFSQ": vqb.GroupedResidualFSQ}
DT = {"fp32": torch.float32, "bf16": torch.bfloat16, "float32": torch.float32, "bfloat16": torch.bfloat16}


def build(c: Case):
    torch.manual_seed(c.meta["init_seed"])
    m = CLASSES[c.cls](**c.meta["kw"])
    if c.meta["module_dtype"] == "bf16":
        m = m.to(torch.bfloat16)
    return m.to(DEV).train(c.meta["train"])


class _Fixed(nn.Module):
    """Stands in for project_in: returns the reference's own project_in output (a leaf, so its gradient can be read)."""

    def __init__(self, z):
        super().__init__()
        self.z = z

    def forward(self, x):
        return self.z


class _Capture(nn.Module):
    """Stands in for project_out: keeps its input (the quantizer's output) and passes it on."""

    def __init__(self, sink):
        super().__init__()
        self.sink = sink

    def forward(self, q):
        self.sink.append(q)
        return q


@pytest.mark.parametrize("path", FIXTURES, ids=fixture_id)
def test_fixture_module_replay(path):
    """The module on x: output / index dtypes and shapes equal the reference's; then the quantizer proper on the reference's
    own project_in output: indices and quantized_out bit for bit (tanh paths: flips only at rounding boundaries), and d z of
    the reference's upstream gradient against the reference's (exact where every factor is exact, else inside the bound)."""
    c = Case(path)
    m = build(c)
    x = torch.tensor(c.a["x"]).to(DT[c.meta["x_dtype"]]).to(DEV)
    res = m(x, **c.meta["forward_kw"])
    out, ind = res[0], res[1]
    assert str(out.dtype).replace("torch.", "") == c.meta["out_dtype"] and list(out.shape) == c.meta["out_shape"]
    assert str(ind.dtype).replace("torch.", "") == c.meta["indices_dtype"] and list(ind.shape) == c.meta["indices_shape"]
    # the projections are torch matmuls, a few ulps apart between devices, and later stages magnify that by 1 / scale_q
    agree = (c.index_rows(ind.cpu().numpy())[..., 0] == c.index_rows()[..., 0]).mean()
    assert agree > 0.97, agree

    parts = list(m.rvqs) if c.cls == "GroupedResidualFSQ" else [m]
    sink, leaves = [], []
    for k, p in enumerate(parts):
        z = torch.tensor(c.a["z"][k]).to(DT[c.meta["z_dtype"]]).to(DEV).requires_grad_(True)
        leaves.append(z)
        p.project_in = _Fixed(z)
        p.project_out = _Capture(sink)
    res = m(x, **c.meta["forward_kw"])
    ind = res[1].cpu().numpy()
    z_np = c.rows("z")
    fwd = O.forward(z_np, c.levels, c.Q, c.n_active, c.sym, c.hard, c.scales, c.clampv, c.w_bf16)
    rows, excused = flipped_rows(c.index_rows(ind), c.index_rows(), fwd["near"])
    print(f"{fixture_id(path)}: {int(rows.sum())} flipped rows of {rows.size}, {int(excused.sum())} near a rounding boundary")
    assert (rows == excused).all()
    if c.hard and c.clampv is None:
        assert not rows.any()
    q = np.stack([s.detach().float().cpu().numpy() for s in sink])
    assert str(sink[0].dtype).replace("torch.", "") == c.meta["qsum_dtype"]
    qrows = part_rows(q, c.d)
    np.testing.assert_array_equal(qrows[~rows], c.rows("qsum")[~rows])
    if "all_codes" in c.a:   # (Q, b, n, d) of a ResidualFSQ
        ac, ref = res[2].float().cpu().numpy(), c.a["all_codes"]
        keep = ~rows[:, 0]
        np.testing.assert_array_equal(ac.reshape(c.Q, -1, c.d)[:, keep], ref.reshape(c.Q, -1, c.d)[:, keep])
    grads = torch.autograd.grad(sink, leaves, [torch.tensor(c.a["qgrad"][k]).to(sink[k].dtype).to(DEV) for k in range(len(sink))])
    gz = np.stack([g.float().cpu().numpy() for g in grads])
    gz_rows = part_rows(gz, c.d)
    _, bound = O.backward(z_np, c.rows("qgrad"), c.levels, c.Q, c.n_active, c.sym, c.hard, c.scales, c.clampv, c.w_bf16,
                          c.in_bf16)
    err = np.abs(gz_rows.astype(np.float64) - c.rows("zgrad"))[~rows]
    b = bound[~rows]
    assert (err[b == 0] == 0).all()
    ratio = float((err[b > 0] / b[b > 0]).max()) if (b > 0).any() else 0.0
    print(f"{fixture_id(path)}: gradient elements exact {int((b == 0).sum())}, largest error / bound on the rest {ratio:.3g}")
    assert (err <= b).all()


def _seeded(seed, N, G, d, Q, n_active, sym, hard, in_dt, work_dt, soft):
    rng = np.random.default_rng(seed)
    lo = 2 if sym else 3
    levels = [int(v) for v in rng.integers(lo, 10, size=d)]
    if d > 1:
        levels[0] = 2 if sym else 4
        levels[-1] = 7
    while np.prod(levels) >= 2 ** 23:   # codes_to_indices sums index terms in fp32 (fsq:224): exact below 2^24
        j = int(np.argmax(levels))
        levels[j] -= 1
    z = (rng.standard_normal((N, G, d)) * 1.3).astype(np.float32)
    if in_dt == torch.bfloat16:
        z = O.bf16_round(z)
    L = torch.tensor(levels)
    scales = torch.stack([L.float() ** -q for q in range(Q)]) if Q > 1 or soft else None
    clampv = (1 + 1 / (L - 1)) if soft else None
    if work_dt == torch.bfloat16:
        scales = scales.bfloat16().float() if scales is not None else None
        clampv = clampv.bfloat16().float() if clampv is not None else None
    return levels, z, scales, clampv


CASES = [
    # (seed, N, G, d, Q, n_active, sym, hard, input dtype, chain dtype, soft clamp)
    (1, 1037, 1, 1, 1, 1, True, True, torch.float32, torch.float32, False),
    (2, 999, 3, 2, 1, 1, False, False, torch.float32, torch.float32, False),
    (3, 1531, 1, 3, 12, 12, True, True, torch.float32, torch.float32, True),
    (4, 777, 2, 4, 8, 5, True, True, torch.float32, torch.float32, True),
    (5, 1001, 1, 5, 3, 3, True, False, torch.float32, torch.float32, False),
    (6, 513, 1, 6, 4, 4, False, True, torch.float32, torch.float32, False),
    (7, 1200, 1, 7, 6, 2, True, True, torch.bfloat16, torch.float32, False),
    (8, 640, 1, 8, 8, 8, True, True, torch.bfloat16, torch.bfloat16, True),
    (9, 333, 2, 9, 2, 2, False, False, torch.bfloat16, torch.bfloat16, False),
    (10, 257, 1, 11, 5, 5, True, True, torch.bfloat16, torch.float32, True),
    (11, 129, 1, 13, 7, 7, True, False, torch.float32, torch.float32, True),
    (12, 300, 1, 15, 3, 1, True, True, torch.float32, torch.float32, False),
    (13, 1029, 1, 16, 12, 12, True, True, torch.float32, torch.float32, True),
    (14, 401, 1, 14, 4, 4, False, False, torch.bfloat16, torch.bfloat16, False),
]


@pytest.mark.parametrize("case", CASES, ids=[f"s{c[0]}_d{c[3]}_q{c[4]}" for c in CASES])
def test_kernels_against_oracle(case):
    seed, N, G, d, Q, n_active, sym, hard, in_dt, work_dt, soft = case
    levels, z, scales, clampv = _seeded(seed, N, G, d, Q, n_active, sym, hard, in_dt, work_dt, soft)
    consts, ints = fsq_tables(torch.tensor(levels, dtype=torch.int32),
                              torch.cumprod(torch.tensor([1] + levels[:-1]), 0, dtype=torch.int32), sym, hard)
    sc_t = torch.stack([scales, 1 / scales]).contiguous().to(DEV) if scales is not None else None
    cl_t = torch.stack([clampv, 1 / clampv]).contiguous().to(DEV) if clampv is not None else None
    zt = torch.tensor(z).to(in_dt).to(DEV)
    idx = torch.empty((N, G, Q), dtype=torch.int64, device=DEV)
    out = ops.fsq_forward(zt, work_dt, Q, n_active, sym, hard, consts.to(DEV), sc_t, cl_t, idx)
    s_np = scales.numpy() if scales is not None else None
    c_np = clampv.numpy() if clampv is not None else None
    w_bf16 = work_dt == torch.bfloat16
    fwd = O.forward(z, levels, Q, n_active, sym, hard, s_np, c_np, w_bf16)
    rows, excused = flipped_rows(idx.cpu().numpy(), fwd["idx"], fwd["near"])
    print(f"case {seed}: {int(rows.sum())} flipped rows of {rows.size}, {int(excused.sum())} near a rounding boundary")
    assert (rows == excused).all()
    if hard and not soft:
        assert not rows.any()
    np.testing.assert_array_equal(out.float().cpu().numpy()[~rows], fwd["out"][~rows])
    # decode: quantized_out == the codes of its indices (exact), stage by stage
    dsum, dcodes = ops.fsq_decode(idx, d, work_dt, sym, consts.to(DEV), ints.to(DEV), sc_t, True, True)
    osum, ocodes = O.decode(idx.cpu().numpy(), levels, sym, s_np, w_bf16)
    np.testing.assert_array_equal(dsum.float().cpu().numpy(), osum)
    np.testing.assert_array_equal(dcodes.float().cpu().numpy(), ocodes)
    if not w_bf16:
        np.testing.assert_array_equal(dsum.cpu().numpy(), out.cpu().numpy())
    # backward against the straight-through chain
    g = torch.randn((N, G, d), generator=torch.Generator().manual_seed(seed)).to(work_dt)
    gz = ops.fsq_backward(zt, g.to(DEV), Q, n_active, sym, hard, consts.to(DEV), sc_t, cl_t)
    dz, bound = O.backward(z, g.float().numpy(), levels, Q, n_active, sym, hard, s_np, c_np, w_bf16, in_dt == torch.bfloat16)
    err = np.abs(gz.float().cpu().numpy().astype(np.float64) - dz)[~rows]
    b = bound[~rows]
    assert (err[b == 0] == 0).all()
    ratio = float((err[b > 0] / b[b > 0]).max()) if (b > 0).any() else 0.0
    print(f"case {seed}: largest gradient error / bound {ratio:.3g}")
    assert (err <= b).all()


def test_readme_fsq_invariant():
    """Reference tests/test_readme.py::test_fsq: xhat == indices_to_codes(indices)."""
    quantizer = vqb.FSQ([8, 5, 5, 5]).to(DEV)
    x = torch.randn(1, 1024, 4, device=DEV)
    xhat, indices = quantizer(x)
    assert xhat.shape == x.shape and indices.shape == (1, 1024) and indices.dtype == torch.int32
    assert torch.all(xhat == quantizer.indices_to_codes(indices))
    q2 = vqb.FSQ([8, 5, 5, 5], return_indices=False).to(DEV)
    out, none = q2(x)
    assert none is None and out.shape == x.shape


def test_readme_rfsq_invariant():
    """Reference tests/test_readme.py::test_rfsq: quantized == get_output_from_indices(indices), in eval, and training runs."""
    residual_fsq = vqb.ResidualFSQ(dim=256, levels=[8, 5, 5, 3], num_quantizers=8).to(DEV)
    x = torch.randn(1, 1024, 256, device=DEV)
    residual_fsq.eval()
    quantized, indices = residual_fsq(x)
    assert quantized.shape == (1, 1024, 256) and indices.shape == (1, 1024, 8)
    quantized_out = residual_fsq.get_output_from_indices(indices)
    assert torch.all(quantized == quantized_out)
    residual_fsq.train()
    xg = x.clone().requires_grad_(True)
    q, _ = residual_fsq(xg)
    q.sum().backward()
    assert torch.isfinite(xg.grad).all()


def test_grouped_runs_one_forward_launch():
    m = vqb.GroupedResidualFSQ(dim=64, groups=4, levels=[8, 5, 5, 3], num_quantizers=6).to(DEV)
    x = torch.randn(2, 100, 64, device=DEV, requires_grad=True)
    before = ops.LAUNCHES
    q, ind = m(x)
    assert ops.LAUNCHES - before == 1
    assert ind.shape == (4, 2, 100, 6)
    before = ops.LAUNCHES
    q.sum().backward()
    assert ops.LAUNCHES - before == 1


def test_bad_dtype_raises():
    with pytest.raises(TypeError):
        vqb.FSQ([8, 5, 5, 5]).to(DEV)(torch.randn(1, 8, 4, device=DEV, dtype=torch.float16))
