"""The slice plan of the gather-sum kernels (vqb_debug_gather_sum_plan, the arithmetic vqb_decode and vqb_rvq_accumulate
launch with).

Host only: no device is needed.  rvq_accumulate_smem_kernel stages a W-column slice of every codebook it reads in shared
memory (bf16 for the rounded bf16 running sum, fp32 otherwise) and serves a row with LPR = W * esz / 16 adjacent lanes of
16 bytes each.  W is the widest power of two that divides D with a row piece of 64..512 bytes (LPR 4..32) and a slice of at
most 192 KiB; when none fits, or below 4096 rows, the L2 kernel (rvq_accumulate_kernel) runs instead.  The slices split
the SMs between them, at least one CTA each.

tests/test_decode_rotate_gpu.py runs both kernels on these plans (132 SMs):
    esz  LPR  W    D    K      nbooks   slices  CTAs/slice
    2    4    32   96   1536   1        3       44
    2    8    64   192  1536   1        3       44
    2    16   128  384  768    1        3       44
    2    32   256  768  384    1        3       44
    4    4    16   48   1536   1        3       44
    4    8    32   96   1536   1        3       44
    4    16   64   192  768    1        3       44
    4    32   128  384  384    1        3       44
    (the stacked cases shrink K to fit nbooks = Q = LPR + 1 codebooks; D = 264, or K = 16384 stacked, or N = 4095: W = 0, the L2 kernel)
"""
import ctypes

import pytest

SMEM = 196608
NBOOKS = [1, 2, 8, 16]
KS = [5, 16, 100, 256, 384, 1000, 1024, 1536, 4096, 16384]
DS = list(range(8, 1025, 8))
NS = [1, 4095, 4096, 4097, 1 << 20]
SMS = [1, 78, 132]


def plan(nbooks, K, D, esz, N, sms):
    from vector_quantize_pytorch_b200 import _C
    out = (ctypes.c_int * 3)()
    rc = _C.lib.vqb_debug_gather_sum_plan(nbooks, K, D, esz, N, sms, ctypes.cast(out, ctypes.c_void_p))
    return rc, tuple(out)


def widest_slice(nbooks, K, D, esz):
    """The rule, restated: the widest power of two W dividing D with 64 <= W * esz <= 512 whose slice fits; 0 if none."""
    fits = [w for w in (2 ** e for e in range(12)) if D % w == 0 and 64 <= w * esz <= 512 and nbooks * K * w * esz <= SMEM]
    return max(fits, default=0)


@pytest.mark.parametrize("esz", [2, 4])
@pytest.mark.parametrize("nbooks", NBOOKS)
def test_gather_sum_plan_invariants(nbooks, esz):
    n_smem = n_l2 = 0
    for K in KS:
        for D in DS:
            rule = widest_slice(nbooks, K, D, esz)
            for N in NS:
                for sms in SMS:
                    rc, (W, slices, cps) = plan(nbooks, K, D, esz, N, sms)
                    case = (nbooks, K, D, esz, N, sms)
                    assert rc == 0, case
                    if N < 4096 or rule == 0:
                        assert (W, slices, cps) == (0, 0, 0), case
                        n_l2 += 1
                        continue
                    n_smem += 1
                    assert W == rule, case
                    assert W * esz // 16 in (4, 8, 16, 32), case        # lanes per row: a power of two that divides a warp
                    assert slices * W == D, case
                    assert nbooks * K * W * esz <= SMEM, case            # the dynamic smem request
                    assert cps == max(1, sms // slices), case
                    assert slices * cps <= max(sms, slices), case        # one wave (one CTA per SM: the slice fills its smem)
    assert n_smem > 50 and n_l2 > 1000


def test_gather_sum_plan_examples():
    assert plan(1, 1024, 256, 4, 262144, 132)[1] == (32, 8, 16)    # BASELINE config 3, fp32: LPR 8
    assert plan(1, 1024, 256, 2, 262144, 132)[1] == (64, 4, 33)    # the same in bf16: LPR 8
    assert plan(1, 1024, 256, 2, 4095, 132)[1] == (0, 0, 0)        # too few rows
    assert plan(8, 1024, 128, 4, 32768, 132)[1] == (0, 0, 0)       # 8 separate codebooks of 1024 do not fit
    assert plan(1, 256, 1024, 4, 4096, 132)[1] == (128, 8, 16)     # the widest fp32 slice: LPR 32
    assert plan(1, 256, 1024, 2, 4096, 132)[1] == (256, 4, 33)     # the widest bf16 slice: LPR 32
    assert plan(1, 100, 264, 4, 1 << 20, 132)[1] == (0, 0, 0)      # D = 8 x 33: no row piece of 64 bytes
    assert plan(1, 100, 1024, 4, 4096, 1)[1] == (128, 8, 1)        # fewer SMs than slices: one CTA each


def test_gather_sum_plan_rejects():
    VQB_E_INVALID = -1
    for args in [(0, 16, 64, 4, 4096, 132), (1, 0, 64, 4, 4096, 132), (1, 16, 0, 4, 4096, 132), (1, 16, 64, 3, 4096, 132),
                 (1, 16, 64, 4, 0, 132), (1, 16, 64, 4, 4096, 0)]:
        assert plan(*args)[0] == VQB_E_INVALID, args
    from vector_quantize_pytorch_b200 import _C
    assert _C.lib.vqb_debug_gather_sum_plan(1, 16, 64, 4, 4096, 132, None) == VQB_E_INVALID
