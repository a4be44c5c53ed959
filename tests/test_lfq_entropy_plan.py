"""The launch plan of the LFQ entropy kernels (ops.lfq_entropy_plan) and the argument checks of vqb_lfq_entropy and
vqb_lfq_entropy_backward that guard a plan given by hand.

Host only: no device is needed.  vqb_lfq_entropy streams the 2^d codes in tiles over `chunks` row chunks (32-row batches
within a chunk); with column sums each chunk writes a (SG, K) fp32 partial.  vqb_lfq_entropy_backward splits K over `ksplit`
CTAs of Kc = K / ksplit codes; the kernel steps through Kc 16 codes at a time, so a split needs Kc >= 16.  The plan splits
only while the CTAs are under 4 per SM and each split keeps 2048 codes (one shared-memory step of the gradient table).
"""
import itertools

import pytest

from vector_quantize_pytorch_b200 import ops

SMS = [1, 78, 114, 132, 256]
RS = sorted({1, 2, 31, 32, 33, 113, 300, 1000, 4097, 16384, 100_000, 1 << 20} | {1 << e for e in range(0, 21, 4)})
SGS = [1, 2, 3, 6, 64]
MAX_COLSUM = 8 << 20   # floats of per-chunk column-sum partials
E_INVALID = -1


def _tiles(D):
    """K tiles of the forward kernel: 16 k_hi values x 2^min(D, 8) codes each."""
    return 1 << max(0, D - 12)


def test_lfq_entropy_tiles():
    assert [ops.lib.vqb_lfq_entropy_tiles(D) for D in range(1, 21)] == [_tiles(D) for D in range(1, 21)]


@pytest.mark.parametrize("sms", SMS)
def test_lfq_entropy_plan_invariants(sms):
    for R, SG, D, want_colsum in itertools.product(RS, SGS, range(1, 21), (False, True)):
        case = (R, SG, D, sms, want_colsum)
        chunks, ksplit = ops.lfq_entropy_plan(R, SG, D, sms, want_colsum)
        K = 1 << D
        assert 1 <= chunks <= min(R, -(-R // 32), 65535), case
        if want_colsum and chunks > 1:
            assert chunks * SG * K <= MAX_COLSUM, case
        # as many chunks as the caps allow, up to the 4-CTAs-per-SM target
        cap = min(-(-R // 32), 65535, *((max(1, MAX_COLSUM // (SG * K)),) if want_colsum else ()))
        assert chunks == min(cap, -(-4 * sms // (_tiles(D) * SG))), case
        assert ksplit & (ksplit - 1) == 0 and K % ksplit == 0 and ksplit <= 65535, case
        Kc = K // ksplit
        blocks = -(-R // 128) * SG
        if ksplit > 1:
            assert Kc >= 2048, case
            assert blocks * (ksplit // 2) < 4 * sms, case   # minimal: half the split is under the CTA target
        # and maximal: doubling it would reach the target or leave a split under 2048 codes
        assert blocks * ksplit >= 4 * sms or Kc // 2 < 2048, case
        assert ops.lfq_entropy_plan(R, SG, D, sms, not want_colsum)[1] == ksplit, case


# (R, SG, D, sms, want_colsum) -> (chunks, ksplit), as the kernel tests launch them on a 132-SM H100, and a few extremes
PINNED = [
    ((300, 2, 1, 132, True), (10, 1)),        # test_every_d, d <= 12: one 30-row batch per chunk
    ((300, 2, 8, 132, True), (10, 1)),
    ((300, 2, 11, 132, True), (10, 1)),
    ((300, 2, 12, 132, True), (10, 2)),
    ((40, 2, 13, 132, True), (2, 4)),         # d = 13...20: Kc = 2048
    ((40, 2, 16, 132, True), (2, 32)),
    ((5, 2, 17, 132, True), (1, 64)),
    ((5, 2, 20, 132, True), (1, 512)),
    ((70, 2, 16, 132, True), (3, 32)),        # test_regimes
    ((500, 6, 9, 132, True), (16, 1)),        # test_row_lists_shared_and_per_group
    ((61, 6, 9, 132, True), (2, 1)),
    ((7, 6, 9, 132, True), (1, 1)),
    ((9000, 1, 10, 132, True), (282, 1)),     # test_many_waves_of_rows
    ((2000, 6, 12, 132, True), (63, 2)),      # test_deterministic
    ((16384, 1, 18, 132, True), (9, 8)),      # test_scale_d18_16k_rows: 57 batches per chunk, Kc = 32768
    ((16384, 1, 18, 114, True), (8, 4)),
    ((4096, 4, 14, 78, True), (20, 4)),
    ((113, 6, 20, 132, False), (1, 128)),
    ((1 << 20, 1, 20, 132, True), (3, 1)),    # colsum cap: 3 x 2^20 floats
    ((1 << 20, 1, 20, 132, False), (3, 1)),   # 64 tiles: 3 chunks reach 4 CTAs per SM
    ((1 << 20, 64, 20, 132, True), (1, 1)),
    ((1 << 20, 64, 1, 256, False), (16, 1)),
    ((1, 1, 1, 1, True), (1, 1)),
]


@pytest.mark.parametrize("args,expect", PINNED, ids=[str(a) for a, _ in PINNED])
def test_lfq_entropy_plan_pinned(args, expect):
    assert ops.lfq_entropy_plan(*args) == expect


def _fwd(D, R, chunks, N=None):
    """vqb_lfq_entropy on stand-in addresses: a refused plan returns before anything touches them or the device."""
    a = 1 << 20
    return ops.lib.vqb_lfq_entropy(a, N or R, 1, D, 1, None, R, 0, a, 1.0, chunks, a, None, None)


def _bwd(D, ksplit, R=4):
    a = 1 << 20
    return ops.lib.vqb_lfq_entropy_backward(a, R, 1, D, 1, None, R, 0, a, 1.0, a, None, ksplit, a, a, None)


def test_lfq_entropy_plan_refusals():
    assert _fwd(8, 5, 6) == E_INVALID                    # chunks > R
    assert _fwd(8, 1 << 17, 65536) == E_INVALID          # chunks > 65535 (grid y)
    assert _fwd(8, 5, 0) == E_INVALID
    for ks in (3, 6, 12, 24, 65535):                     # not a power of two
        assert _bwd(20, ks) == E_INVALID, ks
    assert _bwd(5, 4) == E_INVALID                       # Kc = 8 < 16 with ksplit > 1
    assert _bwd(8, 32) == E_INVALID                      # Kc = 8
    assert _bwd(4, 2) == E_INVALID                       # Kc = 8
    assert _bwd(3, 2) == E_INVALID                       # K = 8 < 16
    assert _bwd(20, 1 << 16) == E_INVALID                # ksplit > 65535 (grid z), although Kc = 16
    assert _bwd(8, 512) == E_INVALID                     # ksplit > K
    assert _bwd(8, 0) == E_INVALID
