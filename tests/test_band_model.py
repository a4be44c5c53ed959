"""CPU model of the certification band's reference-facing terms (csrc/vq_assign.cu, `sc.init(...)`; DESIGN.md 4.1).

The search kernel certifies a row when its best tensor-core score leads every other score by more than
    W = 2 (||x|| cres + ||x_lo|| caux + m ||x|| cmax + 2^-21 cmax^2)          <- what the MMA passes can be off by (GPU test:
                                                                                 test_score_error_inside_margin)
      + 2^-18 (||x|| cmax + cmax^2 / 2) + 2^-22 (||x||^2 + cmax^2)            <- tag slack + the width over which the REFERENCE's
                                                                                 own fp32 formula (vqp:58-62: sqrt of a rounded
                                                                                 d^2, first maximal index) departs from exact
and sends every other row to the exact re-score, which evaluates the reference formula itself.  The first line is a property
of the tensor core and is asserted on the GPU.  The second line is a property of the reference's arithmetic and can be checked
here: whenever the reference's fp32 arg-max differs from the exact (float64) arg-max of x.c - |c|^2/2, the exact score gap
between the two winners must lie inside that slack — then the kernel cannot certify such a row with the non-reference index
(round-1 VERDICT weak #2: with the default-init codebook 4 of 32768 rows escaped the old band).
"""
import numpy as np
import pytest
import torch

from oracle import vq_oracle as O


def reference_slack(x2, cmax):
    """The band's last two terms, float64 evaluation of the fp32 expression in vq_assign.cu (Euclidean metric)."""
    xc = np.sqrt(x2) * cmax
    return 2.0 ** -18 * (xc + 0.5 * cmax * cmax) + 2.0 ** -22 * (x2 + cmax * cmax)


def codebook(kind, K, D):
    if kind == "default":  # vqp:112-115, :385: kaiming_uniform_ on the (1, K, D) tensor -> |c| <= sqrt(6 / (K D))
        e = torch.empty(1, K, D)
        torch.nn.init.kaiming_uniform_(e)
        return e[0].numpy()
    if kind == "warm":
        return torch.randn(K, D).numpy()
    if kind == "tiny_and_huge":  # norms spread over four decades
        return (torch.randn(K, D) * torch.logspace(-2, 2, K)[:, None]).numpy()
    raise ValueError(kind)


def rows(kind, N, D):
    x = torch.randn(N, D)
    if kind == "heavy":  # one dominant coordinate per row
        x[torch.arange(N), torch.randint(0, D, (N,))] *= 300.0
    elif kind == "scaled":
        x = x * torch.logspace(-2, 2, N)[:, None]
    return x.numpy().astype(np.float32)


CASES = [
    # K,    D,   N,     codebook,        rows
    (1024, 256, 16384, "default", "randn"),     # BASELINE config 2, first training step of a default-constructed module
    (1024, 256, 8192, "default", "scaled"),
    (1024, 256, 8192, "default", "heavy"),
    (1024, 256, 8192, "warm", "randn"),
    (1024, 256, 4096, "warm", "scaled"),
    (1024, 128, 8192, "default", "randn"),      # config 5 stage shape
    (4096, 512, 2048, "default", "randn"),      # towards config 4's size (Euclidean variant)
    (333, 64, 8192, "tiny_and_huge", "randn"),
    (96, 64, 8192, "default", "randn"),         # the shape of the small cold-init fixture
]


@pytest.mark.parametrize("K,D,N,cb_kind,row_kind", CASES)
def test_reference_departures_lie_inside_the_band(K, D, N, cb_kind, row_kind):
    torch.manual_seed(K * 7 + D + N)
    e = codebook(cb_kind, K, D)
    x = rows(row_kind, N, D)
    ref = O.argmax_first(O.neg_cdist(x, e))                     # the reference's fp32 formula and tie rule (vqp:58-62, :140)
    x64, e64 = x.astype(np.float64), e.astype(np.float64)
    s = x64 @ e64.T - 0.5 * (e64 * e64).sum(-1)[None]           # the kernel's score, exact
    best = s.argmax(-1)
    ar = np.arange(N)
    gap = s[ar, best] - s[ar, ref]
    x2 = (x64 * x64).sum(-1)
    cmax = float(np.sqrt((e64 * e64).sum(-1).max()))
    slack = reference_slack(x2, cmax)
    differing = ref != best
    # every departure of the reference from the exact arg-max is a near tie well inside the slack (factor 1.5 in hand)
    assert (gap[differing] * 1.5 <= slack[differing]).all(), (
        f"{int(differing.sum())} rows differ, worst gap / slack = {(gap[differing] / slack[differing]).max():.3f}")
    # and these two terms alone do not send a trained codebook's rows to the re-score wholesale
    top2 = np.partition(s, -2, axis=-1)[:, -2:]
    frac = float(((top2[:, 1] - top2[:, 0]) < slack).mean())
    if cb_kind == "warm" and row_kind == "randn":
        assert frac < 1e-3, frac


# ------------------------------------------------------------------------------------------------------------------------
# The whole certificate: split-precision operands + worst-case accumulation noise + the band -> the reference's winner is
# always among the candidates the kernel hands to the exact re-score (or the row is certified with that very winner).
# ------------------------------------------------------------------------------------------------------------------------

MARGIN = 2.0 ** -18   # ops.DEFAULT_MARGIN: the share of the band reserved for the tensor core's fp32 accumulation


def split_bf16(a):
    hi = O.bf16_round(a)
    lo = O.bf16_round((a - hi).astype(np.float32))
    return hi, lo


FLOOR = 1e-8   # the band's clamp-floor term (Euclid): the reference's d^2 clamp, vqp:58-62


def kernel_band(x2, xlo_norm, cmax, cres, caux, euclid):
    """W of vq_assign.cu (`sc.init`), float64 evaluation."""
    xn = np.sqrt(x2)
    xc = xn * cmax
    e = 1.0 if euclid else 0.0
    return (2.0 * (xn * cres + xlo_norm * caux + MARGIN * xc + e * 2.0 ** -21 * cmax * cmax)
            + 2.0 ** -18 * (xc + e * 0.5 * cmax * cmax) + e * (2.0 ** -22 * (x2 + cmax * cmax) + FLOOR))


def _floor_case(kind, rng):
    """(rows, codebook) of the clamp-floor regime.  The reference clamps d^2 at 1e-8, so every code within 1e-4 of a row
    scores exactly -1e-4 and the LOWEST such index wins, even when a higher index is strictly closer."""
    K, D = 1024, 256
    if kind == "zero_rows":   # a ResidualVQ stage after an exact match: zero residuals, two codes of norm below 1e-4
        e = (rng.standard_normal((K, D)) * 3e-3 / np.sqrt(D)).astype(np.float32)
        e[1] = (rng.standard_normal(D) * 5e-5 / np.sqrt(D)).astype(np.float32)
        e[3] = (rng.standard_normal(D) * 1e-6 / np.sqrt(D)).astype(np.float32)
        return np.zeros((8, D), np.float32), e
    scale = {"pair_3e-3": 3e-3, "pair_1e-2": 1e-2}[kind]   # small-norm codebook, a pair 5e-5 apart, rows on the higher index
    e = (rng.standard_normal((K, D)) * scale / np.sqrt(D)).astype(np.float32)
    e[700] = e[5] + (rng.standard_normal(D) * 5e-5 / np.sqrt(D)).astype(np.float32)
    x = (e[700] + rng.standard_normal((64, D)) * 1e-6 / np.sqrt(D)).astype(np.float32)
    return x, e


@pytest.mark.parametrize("kind", ["zero_rows", "pair_3e-3", "pair_1e-2"])
def test_clamp_floor_departures_lie_inside_the_band(kind):
    """At the clamp floor the reference's winner departs from the exact arg-max on every row of these cases (the departure
    is asserted, so the case keeps testing the floor); the exact score gap between the two must still lie inside W, or
    the kernel would certify the exact winner instead of the reference's.  Without the band's FLOOR term the zero rows
    (gap ~30 W) and the pair at max||c|| ~ 3e-3 (~5 W) would be certified with the exact winner; at ~1e-2 the norm-scaled
    terms alone still cover the floor."""
    x, e = _floor_case(kind, np.random.default_rng(1))
    ref = O.argmax_first(O.neg_cdist(x, e))
    x64, e64 = x.astype(np.float64), e.astype(np.float64)
    s = x64 @ e64.T - 0.5 * (e64 * e64).sum(-1)[None]
    best = s.argmax(-1)
    assert (ref != best).all() and (ref < best).all()
    ar = np.arange(len(x))
    gap = s[ar, best] - s[ar, ref]
    x2 = (x64 * x64).sum(-1)
    cmax = float(np.sqrt((e64 * e64).sum(-1).max()))
    c_hi, c_lo = split_bf16(e)
    cres = float(np.sqrt(((e64 - c_hi.astype(np.float64) - c_lo.astype(np.float64)) ** 2).sum(-1)).max())
    W = kernel_band(x2, np.zeros_like(x2), cmax, cres, 0.0, True)   # bf16 rows: no x_lo term
    assert (gap * 1.5 <= W).all(), f"worst gap / W = {np.max(gap / W):.3f}"


@pytest.mark.parametrize("dtype", ["bf16", "fp32"])
@pytest.mark.parametrize("cb_kind,row_kind,cosine", [("default", "randn", False), ("warm", "randn", False), ("warm", "heavy", False),
                                                      ("default", "scaled", False), ("warm", "randn", True)])
def test_reference_winner_is_always_a_candidate(dtype, cb_kind, row_kind, cosine):
    """Emulates what the search kernel sees — bf16 hi / lo codebook planes, for fp32 rows the (x_hi, x_lo) split without the
    x_lo . c_lo and residual terms, scores off by up to MARGIN ||x|| cmax from the accumulation (injected at full amplitude with
    random signs) — and checks the certificate: the index the REFERENCE formula picks is never farther than W below the best
    emulated score.  Hence a row is either certified with the reference's index or re-scored with the reference's formula."""
    K, D, N = 1024, 256, 8192
    rng = np.random.default_rng(11)
    torch.manual_seed(5 + int(cosine))
    e = codebook(cb_kind, K, D)
    x = rows(row_kind, N, D)
    if dtype == "bf16":
        x = O.bf16_round(x)
    if cosine:
        e = O.l2norm(e)
        x = O.l2norm(x, dtype)                                   # vqp:1159: in the input dtype
    ref = O.argmax_first(O.scores(x, e, cosine))                 # the reference's fp32 evaluation and tie rule
    c_hi, c_lo = split_bf16(e)
    e64 = e.astype(np.float64)
    bias = 0.0 if cosine else 0.5 * (e64 * e64).sum(-1)
    csum = c_hi.astype(np.float64) + c_lo.astype(np.float64)
    if dtype == "bf16":
        x_hi, x_lo = x, np.zeros_like(x)
        s = x_hi.astype(np.float64) @ csum.T                      # passes (x, c_hi) + (x, c_lo)
    else:
        x_hi, x_lo = split_bf16(x)
        s = x_hi.astype(np.float64) @ csum.T + x_lo.astype(np.float64) @ c_hi.astype(np.float64).T   # + (x_lo, c_hi)
    s = s - (bias[None] if not cosine else 0.0)
    x2 = (x.astype(np.float64) ** 2).sum(-1)
    cn = np.sqrt((e64 * e64).sum(-1))
    cmax = float(cn.max())
    cres = float(np.sqrt(((e64 - csum) ** 2).sum(-1)).max())                    # cmax[1]
    clo = float(np.sqrt((c_lo.astype(np.float64) ** 2).sum(-1)).max())          # cmax[2]
    caux = (float.fromhex("0x1.02p-8") * cmax + clo) if dtype == "fp32" else 0.0
    xlo_norm = np.sqrt((x_lo.astype(np.float64) ** 2).sum(-1))
    s = s + rng.choice([-1.0, 1.0], size=s.shape) * (MARGIN * np.sqrt(x2) * cmax)[:, None]   # accumulation error, full amplitude
    W = kernel_band(x2, xlo_norm, cmax, cres, caux, not cosine)
    ar = np.arange(N)
    behind = s.max(-1) - s[ar, ref]
    assert (behind <= W).all(), f"{int((behind > W).sum())} rows would be certified with a non-reference index; worst {np.max(behind / W):.3f} W"
    # cost of exactness: how many rows the band sends to the re-score (pairs within W of the emulated best)
    flagged = float(((s > (s.max(-1) - W)[:, None]).sum(-1) > 1).mean())
    if cb_kind == "warm" and row_kind == "randn":
        assert flagged < 0.02, flagged
