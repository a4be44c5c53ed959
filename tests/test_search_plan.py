"""The shared-memory launch plan of the search kernel (vqb_debug_assign_plan, the arithmetic vqb_assign launches with).

Host only: no device is needed.  For every supported D of both production pass schemes the plan must fit in the 227 KiB a
CTA may opt into, keep the ring deep enough to overlap TMA and MMA, and size the seed slots so that a slot is refilled only
after every consumer released the first item of the code step that last used it (DESIGN.md 4.1).  The table of distinct
plans is pinned, so that a change to the sizing shows up in review as a changed table.
"""
import ctypes

import pytest

SMEM_LIMIT = 232448          # 227 KiB opt-in maximum per CTA on sm_90
MAX_A_SUB = 8                # stationary A: at most 8 (plane, k-block) sub-tiles of 16 KiB
SCHEMES = {"bf16": (1, 2), "fp32": (2, 3)}   # (n_a, n_passes) the library selects

# dtype, D range, stream_a, stages, seed slots
PLANS = [
    ("bf16", 8, 64, 0, 8, 4),
    ("bf16", 72, 192, 0, 8, 2),
    ("bf16", 200, 320, 0, 8, 1),
    ("bf16", 328, 384, 0, 7, 1),
    ("bf16", 392, 448, 0, 6, 1),
    ("bf16", 456, 512, 0, 5, 1),
    ("bf16", 520, 1024, 1, 6, 1),
    ("fp32", 8, 64, 0, 8, 3),
    ("fp32", 72, 128, 0, 8, 2),
    ("fp32", 136, 192, 0, 7, 1),
    ("fp32", 200, 256, 0, 5, 1),
    ("fp32", 264, 1024, 1, 6, 1),
]


def plan(n_a, D, n_passes):
    from vector_quantize_pytorch_b200 import _C
    out = (ctypes.c_int * 6)()
    rc = _C.lib.vqb_debug_assign_plan(n_a, D, n_passes, ctypes.cast(out, ctypes.c_void_p))
    return rc, tuple(out)


@pytest.mark.parametrize("dt", sorted(SCHEMES))
def test_plan_invariants_for_every_D(dt):
    n_a, n_passes = SCHEMES[dt]
    for D in range(8, 1025, 8):
        rc, (stream_a, stages, n_seed, n_items, KB, smem) = plan(n_a, D, n_passes)
        assert rc == 0, (dt, D, rc)
        assert KB == (D + 63) // 64 and n_items == KB * n_passes, (dt, D)
        assert smem <= SMEM_LIMIT and stages >= 2, (dt, D, smem, stages)
        # a seed slot is reused n_seed code steps later; the ring runs at most `stages` items ahead
        assert n_seed * n_items >= stages, (dt, D)
        assert n_seed == -(-stages // n_items), (dt, D)
        assert stream_a == int(n_a * KB > MAX_A_SUB), (dt, D)
        if not stream_a:
            assert n_a * KB <= MAX_A_SUB, (dt, D)
        # the sizing is tight: one more stage (with the seed slots it needs) would not fit
        if stages < 8:
            a_bytes = 0 if stream_a else n_a * KB * 16384
            stage_bytes = 16384 * (2 if stream_a else 1)
            fixed = smem - a_bytes - stages * stage_bytes - n_seed * 4096
            more = fixed + a_bytes + (stages + 1) * stage_bytes + -(-(stages + 1) // n_items) * 4096
            assert more > SMEM_LIMIT, (dt, D)


def test_distinct_plans_are_the_table():
    got = {}
    for dt, (n_a, n_passes) in SCHEMES.items():
        for D in range(8, 1025, 8):
            _, (stream_a, stages, n_seed, _, _, _) = plan(n_a, D, n_passes)
            key = (dt, stream_a, stages, n_seed)
            lo, hi = got.get(key, (D, D))
            got[key] = (min(lo, D), max(hi, D))
    want = {(dt, s, st, ns): (lo, hi) for dt, lo, hi, s, st, ns in PLANS}
    assert got == want


def test_plan_rejects_what_the_search_rejects():
    VQB_E_INVALID, VQB_E_UNSUPPORTED = -1, -2
    assert plan(1, 0, 2)[0] == VQB_E_INVALID
    assert plan(3, 64, 4)[0] == VQB_E_INVALID
    assert plan(1, 60, 2)[0] == VQB_E_UNSUPPORTED      # D % 8 != 0
    assert plan(2, 64, 2)[0] == VQB_E_UNSUPPORTED      # the fp32 split needs three passes
    assert plan(1, 64, 3)[0] == VQB_E_UNSUPPORTED
    assert plan(1, 64, 1)[0] == VQB_E_UNSUPPORTED      # one pass is not a scheme the search runs
    assert plan(1, 64, 0)[1] == plan(1, 64, 2)[1]       # 0 = automatic: n_a + 1 passes
    assert plan(2, 512, 0)[1] == plan(2, 512, 3)[1]
    from vector_quantize_pytorch_b200 import _C
    assert _C.lib.vqb_debug_assign_plan(1, 64, 2, None) == VQB_E_INVALID
