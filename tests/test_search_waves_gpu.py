"""Search over more row tiles than one wave of persistent CTAs (run on an H100: `pytest -m gpu`).

Every CTA sweeps several tiles, so the per-tile state (x refill and its L2 prefetch, the shared-memory seed slots that
rotate over code steps across tile boundaries) is exercised, and the odd tile count leaves a last tile with one row.
Same checks as the search cases of test_parity_gpu.py.
"""
import pytest

from test_parity_gpu import test_search_gather_stats_match_oracle as _search_case

pytestmark = pytest.mark.gpu

WAVE_CASES = [
    # N,                 D,  K,   dtype,  cosine
    (128 * (2 * 132) + 1, 64, 256, "bf16", False),
]


@pytest.mark.parametrize("N,D,K,dt,cosine", WAVE_CASES)
def test_search_multi_wave_matches_oracle(N, D, K, dt, cosine):
    _search_case(N, D, K, dt, cosine)
