"""The LFQ entropy kernels (vqb_lfq_entropy, vqb_lfq_entropy_backward) on every launch plan, called directly, against the
float64 oracle with the per-element error bounds of oracle/lfq_oracle.py::entropy_reference.

For every d = 1..20 the rows span at least three full 32-row batches and a short one when the rows form one chunk, and the
forward runs with chunks in {1, 2, 3, ceil(R / 32), the plan's on this device, R}, each with and without column sums; the
backward runs with every power-of-two K split from 1 to min(K / 16, 32768), so at d >= 12 splits of fewer than, exactly and
more than 2048 codes (the gradient table's shared-memory step).  Row sets: none, one shared unsorted list with gaps, and one
list per (stage, group) with a row stride of R + 5 whose padding names a row of large values.  Temperatures: flat (1e-3),
moderate (1) and peaked (100), on generic rows, zero rows, rows with codes at the 1e-5 clamp and rows whose |a| = 40 flushes
most p to zero.  Every output lies inside a sentinel-filled buffer; the gradient buffer starts as sentinels, so a row outside
the lists must never be written.
"""
import math

import pytest
import torch

from oracle import lfq_oracle as O
from vector_quantize_pytorch_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64       # sentinel elements before and after every output
SENT = 7.0e30
TAUS = {"flat": 1e-3, "moderate": 1.0, "peaked": 100.0}


def _guarded(shape, dtype):
    n = math.prod(shape)
    whole = torch.full((n + 2 * GUARD,), SENT, dtype=dtype, device=DEV)
    return whole[GUARD:GUARD + n].view(shape), whole


def _guards_intact(whole):
    return bool((whole[:GUARD] == SENT).all() and (whole[-GUARD:] == SENT).all())


def _clamp_alpha(d):
    """|a| at which the codes one bit away from a row's most likely code have p = 1e-5 (on the decreasing branch)."""
    def f(al):
        return -math.log1p(math.exp(2 * al)) - (d - 1) * math.log1p(math.exp(-2 * al)) - math.log(1e-5)
    lo, hi = 0.5 * math.log(max(d - 1, 1)), 30.0
    for _ in range(100):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if f(mid) > 0 else (lo, mid)
    return lo


def _rows_for(d):
    return 32 * 3 + 17 if d >= 17 else 32 * 9 + 17


def _case(d, kind):
    """-> (S, G, N, R, m (S,), row list or None, rows per (s, g) as index tensors, special row indices)."""
    R = _rows_for(d)
    S, G = (2, 3) if kind == "per_group" else (1, 2)
    N = R + 40 if kind != "none" else R + 7
    g = torch.Generator(device="cpu").manual_seed(1000 * d + len(kind))
    m = torch.tensor([0.8125, 1.375][:S], dtype=torch.float32, device=DEV)
    special = list(range(5, 5 + 9))   # zero rows, clamp rows, large rows (3 each)
    if kind == "none":
        return S, G, N, R, m, None, [torch.arange(R, device=DEV)] * (S * G), special
    pool = [i for i in range(N - 1) if i not in special]   # row N - 1 holds the padding's large values
    if kind == "shared":
        pick = torch.tensor(pool)[torch.randperm(len(pool), generator=g)[:R - len(special)]].tolist() + special
        lst = torch.tensor(pick)[torch.randperm(R, generator=g)].to(torch.int32).to(DEV)
        return S, G, N, R, m, lst, [lst.long()] * (S * G), special
    rows = torch.full((S * G, R + 5), N - 1, dtype=torch.int32)
    for sg in range(S * G):
        pick = torch.tensor(pool)[torch.randperm(len(pool), generator=g)[:R - len(special)]].tolist() + special
        rows[sg, :R] = torch.tensor(pick)[torch.randperm(R, generator=g)].to(torch.int32)
    rows = rows.to(DEV)
    return S, G, N, R, m, rows, [rows[sg, :R].long() for sg in range(S * G)], special


def _inputs(d, S, G, N, m, tau, special, seed):
    """x (S, N, G, d) fp32: generic rows on a log scale of magnitudes, then per stage 3 zero rows, 3 rows with codes at the
    clamp and 3 rows with |a| = 40 (a = 2 tau m x); row N - 1 has |x| = 1e4 / (2 tau m)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((S, N, G, d), generator=g, device=DEV) * torch.logspace(-1.5, 0.5, N, device=DEV)[None, :, None, None]
    sgn = torch.randint(0, 2, (S, N, G, d), generator=g, device=DEV).float() * 2 - 1
    al = _clamp_alpha(d)
    tau32 = float(torch.tensor(tau, dtype=torch.float32))
    for s in range(S):
        tm = 2 * tau32 * float(m[s])
        x[s, special[0:3]] = 0.
        x[s, special[3:6]] = sgn[s, special[3:6]] * (al / tm)
        x[s, special[6:9]] = sgn[s, special[6:9]] * (40. / tm)
        x[s, N - 1] = sgn[s, N - 1] * (1e4 / tm)
    return x.contiguous()


def _fwd(x, m, tau, rows, R, rs, chunks, want_colsum):
    S, N, G, d = x.shape
    SG, K = S * G, 1 << d
    tiles = ops.lib.vqb_lfq_entropy_tiles(d)
    pse, pse_w = _guarded((SG, chunks, tiles), torch.float64)
    col, col_w = _guarded((chunks, SG, K), torch.float32) if want_colsum else (None, None)
    rc = ops.lib.vqb_lfq_entropy(x.data_ptr(), N, G, d, S, rows.data_ptr() if rows is not None else None, R, rs, m.data_ptr(),
                                 tau, chunks, pse.data_ptr(), col.data_ptr() if col is not None else None,
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(pse_w) and bool((pse != SENT).all())
    if col is not None:
        assert _guards_intact(col_w) and bool(torch.isfinite(col).all())
    return pse, col


def _bwd(x, m, tau, rows, R, rs, cp, V, ksplit):
    S, N, G, d = x.shape
    SG = S * G
    work, work_w = _guarded((ksplit, SG, R, d + 1), torch.float32)
    grad, grad_w = _guarded(tuple(x.shape), torch.float32)
    rc = ops.lib.vqb_lfq_entropy_backward(x.data_ptr(), N, G, d, S, rows.data_ptr() if rows is not None else None, R, rs,
                                          m.data_ptr(), tau, cp.data_ptr(), V.data_ptr() if V is not None else None, ksplit,
                                          work.data_ptr(), grad.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(work_w) and bool(torch.isfinite(work).all())
    assert _guards_intact(grad_w)
    return grad


def _ratio(err, bound):
    err, bound = err.abs().double(), torch.as_tensor(bound, dtype=torch.float64, device=err.device).expand_as(err)
    assert bool((err <= bound).all()), float((err - bound).max())
    r = torch.where(bound > 0, err / bound, torch.zeros_like(err))
    return float(r.max())


@pytest.mark.parametrize("kind", ["none", "shared", "per_group"])
@pytest.mark.parametrize("d", list(range(1, 21)))
def test_entropy_plans(d, kind):
    S, G, N, R, m, rows, sg_rows, special = _case(d, kind)
    SG, K = S * G, 1 << d
    rs = R + 5 if kind == "per_group" else 0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    chunk_set = sorted({c for c in (1, 2, 3, -(-R // 32), R, ops.lfq_entropy_plan(R, SG, d, sms, True)[0],
                                    ops.lfq_entropy_plan(R, SG, d, sms, False)[0]) if 1 <= c <= min(R, 65535)})
    ksplits = [1 << e for e in range(0, 16) if (1 << e) <= max(1, min(K // 16, 32768))]
    cp_on = torch.linspace(0.5, 1.5, SG, device=DEV)
    V = torch.randn((SG, K), generator=torch.Generator(device=DEV).manual_seed(d), device=DEV) * 1e-2
    grad_inputs = [(cp_on, V), (torch.zeros(SG, device=DEV), V), (cp_on, None)]
    worst = dict(pse=0., col=0., grad=0.)
    listed = torch.zeros((S, N, G), dtype=torch.bool, device=DEV)
    for sg in range(SG):
        listed[sg // G, sg_rows[sg], sg % G] = True
    for ti, (regime, tau) in enumerate(TAUS.items()):
        tau = float(torch.tensor(tau, dtype=torch.float32))
        x = _inputs(d, S, G, N, m, tau, special, seed=d * 10 + ti)
        xs = [x[sg // G, sg_rows[sg], sg % G] for sg in range(SG)]
        refs = [[O.entropy_reference(xs[sg], float(m[sg // G]), tau, float(cp[sg]), V[sg] if V is not None else None)
                 for sg in range(SG)] for cp, V in grad_inputs]
        # forward: every chunks value, with and without the column sums
        for chunks in chunk_set:
            pse_c, col = _fwd(x, m, tau, rows, R, rs, chunks, True)
            pse_n, _ = _fwd(x, m, tau, rows, R, rs, chunks, False)
            assert torch.equal(pse_c, pse_n), (regime, chunks)   # the column sums do not change the PSE bits
            pse_2, col_2 = _fwd(x, m, tau, rows, R, rs, chunks, True)
            assert torch.equal(pse_c, pse_2) and torch.equal(col, col_2), (regime, chunks)
            for sg in range(SG):
                ref = refs[0][sg]
                pb, cb, _ = ref.bounds(chunks, 1)
                worst["pse"] = max(worst["pse"], _ratio(pse_c[sg].sum() - ref.pse.to(DEV), pb))
                worst["col"] = max(worst["col"], _ratio(col[:, sg].sum(0, dtype=torch.float64) - ref.colsum, cb))
            del col, col_2
        # backward: every K split, every gradient input
        for gi, (cp, Vg) in enumerate(grad_inputs):
            for ksplit in ksplits:
                grad = _bwd(x, m, tau, rows, R, rs, cp, Vg, ksplit)
                assert bool((grad[~listed] == SENT).all()), (regime, gi, ksplit)   # rows outside the lists: never written
                assert torch.equal(grad, _bwd(x, m, tau, rows, R, rs, cp, Vg, ksplit)), (regime, gi, ksplit)
                for sg in range(SG):
                    ref = refs[gi][sg]
                    _, _, gb = ref.bounds(1, ksplit)
                    got = grad[sg // G, sg_rows[sg], sg % G]
                    worst["grad"] = max(worst["grad"], _ratio(got.double() - ref.grad, gb))
    print(f"\nRATIO d={d} kind={kind} R={R} chunks={chunk_set} ksplits={len(ksplits)} "
          f"pse={worst['pse']:.3g} col={worst['col']:.3g} grad={worst['grad']:.3g}")
