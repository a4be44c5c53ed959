"""Float64 restatement of RandomProjectionQuantizer's forward (random_projection_quantizer.py, "rpq") and the per-element bound
of the fp32 rows csrc/vq_rpq.cu writes (TEST INFRASTRUCTURE ONLY; numpy).

rows = LN(x) @ P with LN(v) = (v - mean) / sqrt(var + eps), biased var, P[d, h E + j] = rand_projs[h, d, j].  The kernel takes
the mean and the variance in fp32 (two passes, any summation order), rstd = 1 / sqrt(var + eps) correctly rounded, stages
xn_d = (x_d - mean) rstd and sums xn_d P_dc over d with fmas.  With u = 2^-24 and g(n) = n u / (1 - n u):
    |mean - mean64| <= dm = g(dim + 1) sum_d |x_d| / dim
    rstd relative error <= er = g(dim + 4) / 2 + g(dim + 4) + 2 u   (the variance sums dim squares of deviations each off by
                                                                    dm, and sqrt, the division and the eps add round once)
    |xn_d - xn64_d| <= (er + 2 u) |xn64_d| + 2 dm rstd64
    |row_c - row64_c| <= g(dim) sum_d |xn64_d P_dc| + sum_d |xn_d - xn64_d| |P_dc|   (first order; times a safety factor 2)
Without the norm, xn = x exactly and only the product's g(dim) term remains.
"""
import numpy as np

U = 2.0 ** -24
EPS = 1e-5
SAFETY = 2.0


def gamma(n):
    return n * U / (1 - n * U)


def proj_matrix(rand_projs):
    """(H, dim, E) -> (dim, H E), head-major columns like the reference's pack of 'b n h e'."""
    H, dim, E = rand_projs.shape
    return np.asarray(rand_projs, np.float64).transpose(1, 0, 2).reshape(dim, H * E)


def layer_norm(x, norm=True):
    x = np.asarray(x, np.float64)
    if not norm:
        return x, np.ones(x.shape[:-1] + (1,))
    mean = x.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((x - mean) ** 2).mean(-1, keepdims=True) + EPS)
    return (x - mean) * rstd, rstd


def norm_project(x, rand_projs, norm=True):
    """float64 rows (..., H E)."""
    xn, _ = layer_norm(x, norm)
    return xn @ proj_matrix(rand_projs)


def row_bound(x, rand_projs, norm=True):
    """Per-element bound of |fp32 kernel rows - float64 rows|, shape (..., H E)."""
    x = np.asarray(x, np.float64)
    P = np.abs(proj_matrix(rand_projs))
    dim = x.shape[-1]
    xn, rstd = layer_norm(x, norm)
    b = gamma(dim) * (np.abs(xn) @ P)
    if norm:
        dm = gamma(dim + 1) * np.abs(x).sum(-1, keepdims=True) / dim
        er = 1.5 * gamma(dim + 4) + 2 * U
        b = b + ((er + 2 * U) * np.abs(xn) + 2 * dm * rstd) @ P
    return SAFETY * b


def linear_bound(y, y_bound, weight):
    """Bound of an fp32 nn.Linear(y) against float64 when y is off by y_bound: |W| y_bound plus the product's own rounding."""
    W = np.abs(np.asarray(weight, np.float64))
    n = W.shape[1]
    return y_bound @ W.T + SAFETY * (gamma(n + 1) * (np.abs(y) @ W.T) + U)


def cosine_search(rows, embed):
    """rows (N, D), embed (K, D): (argmax of l2norm(rows) . embed, its lead over the best DISTINCT code vector)."""
    r = np.asarray(rows, np.float64)
    r = r / np.maximum(np.linalg.norm(r, axis=-1, keepdims=True), 1e-300)
    c = np.asarray(embed, np.float64)
    s = r @ c.T
    best = s.argmax(1)
    same = (c[best][:, None, :] == c[None, :, :]).all(-1)
    other = np.where(same, -np.inf, s).max(1)
    return best, s[np.arange(len(r)), best] - other


def lead_bound(rows, row_err):
    """How far a cosine score of a row can move when the row is off by row_err (elementwise bound), against unit codes:
    |l2norm(r + e) - l2norm(r)| <= 2 |e| / |r|, twice over for the two scores a lead compares."""
    n = np.linalg.norm(np.asarray(rows, np.float64), axis=-1)
    return 4.0 * np.linalg.norm(row_err, axis=-1) / np.maximum(n, 1e-300)


def forward(x, rand_projs, norm, embeds, project_in=None):
    """The eval forward in float64.  embeds (H, K, D); project_in = (weight, bias) for H > 1.  Returns (rows, rows after
    project_in, indices (N, H), leads (N, H))."""
    H = embeds.shape[0]
    rows = norm_project(x, rand_projs, norm).reshape(-1, rand_projs.shape[0] * rand_projs.shape[2])
    y = rows if project_in is None else rows @ np.asarray(project_in[0], np.float64).T + np.asarray(project_in[1], np.float64)
    D = y.shape[1] // H
    idx, lead = [], []
    for h in range(H):
        i, g = cosine_search(y[:, h * D:(h + 1) * D], embeds[h])
        idx.append(i)
        lead.append(g)
    return rows, y, np.stack(idx, 1), np.stack(lead, 1)
