"""Float64 oracle of HierarchicalVQ's per-scale maps (hierarchical_vq.py, "hvq"), in numpy, written from ATen's definitions:

    pool(x, s)            adaptive_avg_pool2d: cell (i, j) averages rows [floor(i H / s), ceil((i + 1) H / s)), same for W;
    pool_adjoint(g, H, W) each pixel sums g / (kh kw) over every window that contains it;
    upsample(q, H, W)     bilinear, align_corners = False: src = max((in / out) (dst + 0.5) - 0.5, 0), lower tap floor(src),
                          upper tap +1 unless at the last input; identity when the size already matches (hvq:105);
    upsample_adjoint      the transpose of that map;
    choose_phi            the phi index of a scale (hvq:87-102, Python's round);
    phi(up, w, b, r)      (1 - r) up + r conv3x3(up) (hvq:25);
    forward(...)          the whole chain with given per-scale codes (the rows each search returned).

Images are (B, D, H, W); pooled maps and codes are (B, D, s, s) here.
"""
import numpy as np


def windows(n: int, s: int):
    """ATen's adaptive windows [start, end) of the s output cells over n inputs."""
    return [((i * n) // s, -(-((i + 1) * n) // s)) for i in range(s)]


def pool_matrix(n: int, s: int) -> np.ndarray:
    """(s, n): row i averages its window."""
    m = np.zeros((s, n))
    for i, (a, b) in enumerate(windows(n, s)):
        m[i, a:b] = 1.0 / (b - a)
    return m


def upsample_matrix(n_in: int, n_out: int) -> np.ndarray:
    """(n_out, n_in): the bilinear taps of each output (align_corners = False), with the source index computed in fp32 like
    ATen (scale = in / out rounded to fp32)."""
    m = np.zeros((n_out, n_in))
    if n_in == n_out:
        return np.eye(n_in)
    scale = np.float32(n_in) / np.float32(n_out)
    for d in range(n_out):
        src = max(np.float32(scale * np.float32(np.float32(d) + np.float32(0.5)) - np.float32(0.5)), np.float32(0.0))
        i0 = int(src)
        p = 1 if i0 < n_in - 1 else 0
        lam = float(np.float32(src - np.float32(i0)))
        m[d, i0] += 1.0 - lam
        m[d, i0 + p] += lam
    return m


def pool(x: np.ndarray, s: int) -> np.ndarray:
    H, W = x.shape[-2:]
    return np.einsum("ih,bdhw,jw->bdij", pool_matrix(H, s), np.asarray(x, np.float64), pool_matrix(W, s))


def pool_adjoint(g: np.ndarray, H: int, W: int) -> np.ndarray:
    s = g.shape[-1]
    return np.einsum("ih,bdij,jw->bdhw", pool_matrix(H, s), np.asarray(g, np.float64), pool_matrix(W, s))


def upsample(q: np.ndarray, H: int, W: int) -> np.ndarray:
    s = q.shape[-1]
    if (s, s) == (H, W):
        return np.asarray(q, np.float64).copy()
    return np.einsum("hi,bdij,wj->bdhw", upsample_matrix(s, H), np.asarray(q, np.float64), upsample_matrix(s, W))


def upsample_adjoint(g: np.ndarray, s: int) -> np.ndarray:
    H, W = g.shape[-2:]
    if (s, s) == (H, W):
        return np.asarray(g, np.float64).copy()
    return np.einsum("hi,bdhw,wj->bdij", upsample_matrix(s, H), np.asarray(g, np.float64), upsample_matrix(s, W))


def choose_phi(n_scales: int, n_phi: int, scale_index: int) -> int:
    """hvq:87-102 for phi_levels of length n_phi (the shared phi is index 0 of one)."""
    if n_phi == n_scales:
        return scale_index
    if n_scales == 1:
        return 0
    position = scale_index / float(n_scales - 1)
    return max(0, min(n_phi - 1, round(position * (n_phi - 1))))


def n_phis(n_scales: int, share_quant_resi: int) -> int:
    if share_quant_resi == 1:
        return 1
    return n_scales if share_quant_resi <= 0 else min(n_scales, int(share_quant_resi))


def conv3x3(x: np.ndarray, w: np.ndarray, b: np.ndarray) -> np.ndarray:
    """nn.Conv2d(D, D, 3, padding=1) in float64: x (B, D, H, W), w (D, D, 3, 3), b (D,)."""
    x = np.asarray(x, np.float64)
    B, D, H, W = x.shape
    xp = np.zeros((B, D, H + 2, W + 2))
    xp[:, :, 1:-1, 1:-1] = x
    out = np.broadcast_to(np.asarray(b, np.float64)[None, :, None, None], (B, w.shape[0], H, W)).copy()
    for u in range(3):
        for v in range(3):
            out += np.einsum("oc,bchw->bohw", np.asarray(w[:, :, u, v], np.float64), xp[:, :, u:u + H, v:v + W])
    return out


def phi(up: np.ndarray, w, b, r: float) -> np.ndarray:
    r = abs(float(r))
    if r <= 1e-8:
        return up
    return (1.0 - r) * up + r * conv3x3(up, w, b)


def forward(x: np.ndarray, scales, codes, phis, share_quant_resi: int, full_hw=None):
    """The chain of hvq:128-147 in float64 with the per-scale codes given (codes[k]: (B, D, s, s), the rows scale k's search
    returned).  phis: list of (weight, bias, r).  Returns (recon, pooled inputs per scale)."""
    x = np.asarray(x, np.float64)
    H, W = x.shape[-2:] if full_hw is None else full_hw
    residual, recon, pooled = x, np.zeros(x.shape[:2] + (H, W)), []
    for k, s in enumerate(scales):
        pooled.append(pool(residual, s))
        w, b, r = phis[choose_phi(len(scales), len(phis), k)]
        q = phi(upsample(codes[k], H, W), w, b, r)
        recon = recon + q
        residual = residual - q
    return recon, pooled
