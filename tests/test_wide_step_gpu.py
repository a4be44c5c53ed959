"""The search kernel's 256-code step against float64 and the reference's fp32 formula (run on an H100: `pytest -m gpu`).

Where the launch plan allows it (A resident, an even number of ring stages, the 8 KiB seed slots and the step's static
shared memory inside 227 KiB, more than 128 padded codes), the kernel sweeps the codebook 256 codes per step: one
m64n256k16 wgmma per k16 step over two adjacent ring stages.  The cases below cover the wide step at a multiple of 256
codes, at a K whose padded codes sit in the last 256-wide step, and at a tiny codebook (Kpad < 256: one padded step), and
two plans that keep the 128-code step.  Exact ties are planted inside each 128-code half of one step and on the column
pair that straddles the halves (columns 127 / 128 of the step), so that the merge of the halves' groups and the tagged
top-3 decide between codes of both halves.

Each case prints the step width it launched with, derived from the launch plan by the rule the host applies.
"""
import ctypes
import math

import pytest
import torch

from test_exact_rescore_gpu import run_case
from test_search_plans_gpu import TIE_TOL, ref_search

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SMEM_LIMIT = 232448
SEED_BYTES = 128 * 32          # bext of 128 codes
WIDE_STATIC_SMEM = 3072        # the wide step's static shared memory (loss sums, bias-MMA ones)
SCHEMES = {"bf16": (1, 2), "fp32": (2, 3)}


def step_width(dt, D, K):
    """Codes per step the search launches with for (dtype, D, K): the host's rule applied to vqb_debug_assign_plan."""
    from vector_quantize_pytorch_b200 import _C
    n_a, n_passes = SCHEMES[dt]
    out = (ctypes.c_int * 6)()
    assert _C.lib.vqb_debug_assign_plan(n_a, D, n_passes, ctypes.cast(out, ctypes.c_void_p)) == 0
    stream_a, stages, n_seed, n_items, _, smem = tuple(out)
    kpad = _C.lib.vqb_padded_codes(K)
    if stream_a or stages % 2 or kpad <= 128:
        return 128
    seeds = math.ceil(stages // 2 / n_items)
    wide_smem = smem - n_seed * SEED_BYTES + seeds * 2 * SEED_BYTES
    return 256 if wide_smem + WIDE_STATIC_SMEM <= SMEM_LIMIT else 128


CASES = [
    # dtype, D,   K,    cosine, expected step width
    ("bf16", 256, 1024, False, 256),   # config 2's plan
    ("fp32", 128, 1024, True, 256),    # config 5's plan
    ("bf16", 256, 700, False, 256),    # Kpad = 768: codes 700..767 are padding inside the last 256-wide step
    ("bf16", 136, 200, True, 256),     # Kpad = 208 < 256: one padded step
    ("fp32", 24, 37, False, 128),      # Kpad = 48 <= 128: one 128-code step
    ("bf16", 512, 1024, False, 128),   # 5 ring stages: the 128-code step
]


def plant(K, D, cosine, gen, n_rows):
    """Codebook with exact ties inside both 128-code halves of one step and across its halves, and rows on top of them."""
    c = torch.randn(K, D, generator=gen)
    base = 256 if K >= 512 else 0
    pairs = [(base + 127, base + 128),                                   # the column pair that straddles the halves
             (base + 10, base + 60), (base + 140, base + 190),           # inside the first half, inside the second half
             (base + 30, base + 180)]                                    # one code in each half
    pairs = [(a, b) for a, b in pairs if b < K]
    for a, b in pairs:
        c[b] = c[a]
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    x = torch.randn(n_rows, D, generator=gen)
    scale = 1.0 / D ** 0.5 if cosine else 1.0
    planted = {}
    for j, (a, b) in enumerate(pairs):
        for r in range(3):
            row = 128 * (7 * j + 2 * r) + 5 * j + r                      # spread over tiles and rows of both warpgroups
            x[row] = c[a] + 1e-2 * scale * torch.randn(D, generator=gen)
            planted[row] = a
    return x, c, planted


@pytest.mark.parametrize("dt,D,K,cosine,width", CASES)
def test_wide_step(dt, D, K, cosine, width):
    got = step_width(dt, D, K)
    print(f"{dt} D={D} K={K}: {got}-code steps")
    assert got == width
    N = 128 * 40 + 77
    gen = torch.Generator().manual_seed(D * 131 + K)
    x, c, planted = plant(K, D, cosine, gen, N)
    o, res = run_case(x, c, dt, cosine, f"{dt} D={D} K={K} ({got}-code steps)")
    idx = res.idx.long()
    for row, code in planted.items():   # equal codes: the lowest index wins (vqp:140), after the exact re-score
        assert idx[row].item() == code, (row, idx[row].item(), code)
    ref_idx, gap = ref_search(res.x_eff.float(), c.to(DEV), cosine)
    mism = idx != ref_idx
    assert not (mism & (gap >= TIE_TOL)).any(), f"{int((mism & (gap >= TIE_TOL)).sum())} mismatches against float64 outside ties"
