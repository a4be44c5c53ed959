"""vqb_rotate_masked (the estimator of a masked training step) against float64 on every instantiation: fp32 and bf16, forward
and backward, the rotation trick, straight-through and no estimator, both padding modes, with and without the commitment
term.  D from 8 to 1024; row counts over several waves of the grid (16 CTAs of 8 row-warps per SM) and a single row; n_live
= 0, a ragged mask and n_live = N.

Forward: live rows must be the code bit for bit, padding rows the padding value bit for bit.  Backward: padding rows exactly
0 or the upstream gradient; live rows within the rotation bound of test_decode_rotate_gpu (the kernel evaluates the same
arithmetic) plus the commitment term's rounding, and every value finite, zero-norm codes and inputs included.  Rows the
masked search leaves unwritten are planted with NaN in the code buffer: no output may read them.
"""
import pytest
import torch

from test_decode_rotate_gpu import EPS32, ROW_KINDS, half_ulp_bf16, ratio, rotate_bound, rotate_eval, rotation_rows, sms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}
EST = {"none": 0, "ste": 1, "rotate": 2}


def _rows(D, n_rows, gen, dt):
    per = -(-n_rows // len(ROW_KINDS))
    parts = [rotation_rows(k, per, D, gen) for k in ROW_KINDS]
    s = torch.cat([p[0] for p in parts])[:n_rows].to(TDT[dt])
    t = torch.cat([p[1] for p in parts])[:n_rows].to(TDT[dt])
    return s, t


def _mask(kind, n, gen):
    if kind == "none_live":
        return torch.zeros(n, dtype=torch.uint8, device=DEV)
    if kind == "all_live":
        return torch.ones(n, dtype=torch.uint8, device=DEV)
    return (torch.rand(n, generator=gen, device=DEV) < 0.6).to(torch.uint8)


def waves():
    """Three grids of row-warps and a ragged rest."""
    return 3 * 16 * sms() * 8 + 37


@pytest.mark.parametrize("D,rows", [(8, "waves"), (24, 1), (32, "waves"), (200, 300), (256, "waves"), (1000, 300),
                                    (1024, "waves")])
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_rotate_masked_against_float64(dt, D, rows):
    from vector_quantize_pytorch_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(1000 + D)
    n = waves() if rows == "waves" else rows
    if rows == "waves" and D == 1024:
        n = 16 * sms() * 8 + 37     # one grid and a ragged rest (the rotation kinds are all represented)
    s, t = _rows(D, n, gen, dt)
    g = torch.randn(s.shape, generator=gen, device=DEV).to(TDT[dt])
    s64, g64 = s.double(), g.double()
    worst = {}
    for mkind in ("ragged", "none_live", "all_live"):
        m = _mask(mkind, n, gen)
        live = m.bool()
        n_live = m.sum(dtype=torch.int64).reshape(1)
        # the masked search leaves padding rows of the code buffer unwritten: plant NaN there
        tq = torch.where(live[:, None], t, torch.full_like(t, float("nan")))
        t64 = torch.where(live[:, None], t.double(), torch.zeros_like(t, dtype=torch.float64))
        gl = torch.rand(1, generator=gen, device=DEV) + 0.5
        w = 0.7
        sl, tl, gg = s64[live], t64[live], g64[live]
        rot = (rotate_eval(sl, tl, gg)[1], rotate_bound(sl, tl, gg, D)) if live.any() else None
        for pad_zeros in (True, False):
            fwd = ops.rotate_masked(s, tq, m, EST["rotate"], pad_zeros)
            want = torch.where(live[:, None], t, torch.zeros_like(t) if pad_zeros else s)
            assert torch.equal(fwd.view(torch.uint8), want.view(torch.uint8)), f"forward {mkind} pad_zeros={pad_zeros}"
            for est in ("rotate", "ste", "none"):
                for with_loss in (True, False):
                    got = ops.rotate_masked(s, tq, m, EST[est], pad_zeros, g, gl if with_loss else None,
                                            n_live, w)
                    assert torch.isfinite(got).all(), f"non-finite gradient {est} {mkind}"
                    pad = ~live
                    want_pad = torch.zeros_like(g[pad]) if pad_zeros else g[pad]
                    assert torch.equal(got[pad].view(torch.uint8), want_pad.view(torch.uint8)), f"padding rows {est}"
                    if not live.any():
                        continue
                    c = 2.0 * w * float(gl) / (int(n_live) * D) if with_loss else 0.0
                    if est == "rotate":
                        ref, bound = rot
                    else:
                        ref = gg if est == "ste" else torch.zeros_like(gg)
                        bound = torch.zeros_like(gg)
                    ref = ref + c * (sl - tl)
                    # c (s - t): c and s - t rounded once each, the product and the sum once more
                    bound = bound + 4 * EPS32 * abs(c) * (sl - tl).abs() + 2 * EPS32 * ref.abs()
                    if dt == "bf16":
                        bound = bound + half_ulp_bf16(ref.abs() + bound)
                    r = float(ratio(got[live], ref, bound).max())
                    worst[(mkind, pad_zeros, est, with_loss)] = r
    print(f"\n{dt} D={D} N={n}: worst |error| / bound " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v <= 2}
    assert not bad, f"vqb_rotate_masked outside the bound: {bad}"

