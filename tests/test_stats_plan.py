"""The counting-sort plan of the EMA statistics (vqb_debug_stats_plan, the arithmetic vqb_ema_stats and vqb_vq_forward launch with).

Host only: no device is needed.  Few rows per code (or a codebook too large for a K-int histogram in shared memory) take the
global-atomic kernels; otherwise every CTA owns a slab of 128 << shift rows — whole row tiles of the search kernel, which
counts its winners per slab — with at most one slab per SM (the scatter is one wave), at most 256 slabs (colscan_kernel scans
32 warps x 8 slabs from registers) and at most 2^22 histogram cells.  The workspace is sized for a device-independent slab
bound, so a plan above that bound would write past it.
"""
import ctypes

import pytest

SORT_MAX_K = 16384
MAX_CELLS = 1 << 22
SMS = [1, 78, 114, 132, 256, 300]
NS = sorted({1, 2, 127, 128, 129, 511, 512, 513, 4095, 32768, 65537, 262144, 262145, 1 << 20, 3_000_001, 1 << 24,
             (1 << 27) - 1, 1 << 27} | {1 << e for e in range(0, 28, 3)})
KS = [1, 2, 31, 33, 100, 1000, 1024, 4097, 8192, 8193, 16383, 16384, 16385, 65536]


def plan(N, K, sms):
    from vector_quantize_pytorch_b200 import _C
    out = (ctypes.c_int * 3)()
    rc = _C.lib.vqb_debug_stats_plan(N, K, sms, ctypes.cast(out, ctypes.c_void_p))
    return rc, tuple(out)


@pytest.mark.parametrize("sms", SMS)
def test_stats_plan_invariants(sms):
    n_cta = 0
    for N in NS:
        for K in KS:
            rc, (G, shift, bound) = plan(N, K, sms)
            assert rc == 0, (N, K, sms, rc)
            assert bound == max(1, min(-(-N // 512), 512, MAX_CELLS // K)), (N, K)
            if K > SORT_MAX_K or N < 32 * K:
                assert (G, shift) == (0, 31), (N, K, sms)
                continue
            n_cta += 1
            slab = 128 << shift
            assert 1 <= G <= min(sms, 256), (N, K, sms, G)
            assert G * K <= MAX_CELLS, (N, K, sms, G)
            assert shift >= 2, (N, K, sms, shift)              # slabs of at least 512 rows
            assert G * slab >= N, (N, K, sms, G, shift)        # the slabs cover every row ...
            assert (G - 1) * slab < N, (N, K, sms, G, shift)   # ... and none is empty
            assert G <= bound, (N, K, sms, G, bound)           # carve() sizes the histograms for `bound` slabs
            # the smallest slab that keeps G under the caps
            if shift > 2:
                cap = min(sms, 256, MAX_CELLS // K)
                assert -(-N // (slab // 2)) > cap, (N, K, sms, G, shift)
    assert n_cta > 50


def test_stats_plan_examples():
    assert plan(262144, 1024, 132)[1][:2] == (128, 4)     # BASELINE config 2: 2048 row tiles in 128 slabs of 16
    assert plan(262144, 1024, 114)[1][:2] == (64, 5)
    assert plan(4096, 1024, 132)[1][:2] == (0, 31)        # N / K = 4: global cursors
    assert plan(1 << 20, 16385, 132)[1][:2] == (0, 31)    # K over the shared-memory histogram
    assert plan(1 << 20, 16384, 132)[1][:2] == (128, 6)   # the largest K that still sorts in CTAs
    assert plan(1 << 20, 16384, 300)[1][:2] == (256, 5)   # 256 slabs: the cell cap and the column scan's cap at once
    assert plan(32768, 1024, 132)[1][:2] == (64, 2)


def test_stats_plan_rejects():
    VQB_E_INVALID, VQB_E_UNSUPPORTED = -1, -2
    assert plan(0, 16, 132)[0] == VQB_E_INVALID
    assert plan(16, 0, 132)[0] == VQB_E_INVALID
    assert plan(16, 16, 0)[0] == VQB_E_INVALID
    assert plan(1 << 31, 16, 132)[0] == VQB_E_UNSUPPORTED
    from vector_quantize_pytorch_b200 import _C
    assert _C.lib.vqb_debug_stats_plan(16, 16, 132, None) == VQB_E_INVALID
