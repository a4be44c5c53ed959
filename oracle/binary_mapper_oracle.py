"""float64 numpy restatement of BinaryMapper (binary_mapper.py of the reference, "bm")  —  TEST INFRASTRUCTURE ONLY.

Everything is given the sampled indices (the discrete path), so it replays a fixture whatever generator drew them:
  codes(bits)            (2^bits, bits) bool, codes[k, j] = bit j of k (least significant first, bm:57-58)
  soft_codes(l)          (rows, 2^bits) exp(sum_j log P(bit_j = codes[k, j])): the reference's soft_G (bm:173-176)
  aux_rows(l, thr)       relu(bits ln 2 - H(l) - thr) per row (bm:28-31, :75-87)
  log_prob(l, idx)       sum_j log P(bit_j = bit_j(idx)), or per bit (bm:89-122)
and the gradients:
  st_grad(l, G)          d/dl of sum(soft_G * G): S1_j - sigmoid(l_j) S, S = sum_k G_k s_k, S1_j = sum_{bit_j(k) = 1} G_k s_k
  aux_grad(l, thr, mean) d/dl of aux (mean over rows, or the per-row sum): l p (1 - p) where the relu is on
  log_prob_grad(l, idx)  d/dl of sum_rows log_prob: bit_j(idx) - sigmoid(l_j)
"""
from __future__ import annotations

import numpy as np

NAT = float(np.log(2.0))


def log_sigmoid(x):
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.minimum(x, 0.0) - np.log1p(np.exp(-np.abs(x)))


def sigmoid(x):
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-x))


def codes(bits: int) -> np.ndarray:
    k = np.arange(1 << bits)[:, None]
    return ((k >> np.arange(bits)) & 1).astype(bool)


def index_bits(idx, bits: int) -> np.ndarray:
    return ((np.asarray(idx, np.int64).reshape(-1, 1) >> np.arange(bits)) & 1).astype(bool)


def soft_codes(l) -> np.ndarray:
    l = np.asarray(l, np.float64)
    c = codes(l.shape[1]).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return np.exp(log_sigmoid(l) @ c.T + log_sigmoid(-l) @ (1.0 - c).T)


def binary_entropy(l) -> np.ndarray:
    p = sigmoid(l)
    with np.errstate(invalid="ignore"):
        return -(p * log_sigmoid(l) + (1.0 - p) * log_sigmoid(-l)).sum(-1)


def aux_rows(l, thr) -> np.ndarray:
    l = np.asarray(l, np.float64)
    return np.maximum(l.shape[1] * NAT - binary_entropy(l) - thr, 0.0)


def aux_grad(l, thr, mean: bool) -> np.ndarray:
    l = np.asarray(l, np.float64)
    on = (l.shape[1] * NAT - binary_entropy(l) - thr) > 0.0   # relu'(0) = 0, as torch takes it
    p = sigmoid(l)
    return l * p * (1.0 - p) * on[:, None] / (l.shape[0] if mean else 1.0)


def log_prob(l, idx, sum_bits: bool = True) -> np.ndarray:
    l = np.asarray(l, np.float64)
    per_bit = np.where(index_bits(idx, l.shape[1]), log_sigmoid(l), log_sigmoid(-l))
    return per_bit.sum(-1) if sum_bits else per_bit


def log_prob_grad(l, idx, H) -> np.ndarray:
    l = np.asarray(l, np.float64)
    return (index_bits(idx, l.shape[1]) - sigmoid(l)) * np.asarray(H, np.float64).reshape(-1, 1)


def st_grad(l, G) -> np.ndarray:
    """The closed form, evaluated as sigmoid(-l) S1 - sigmoid(l) S0 (no cancellation when sigmoid(l) is near 1); rows with a
    non-finite logit are NaN, as the reference's autograd gives them."""
    l = np.asarray(l, np.float64)
    w = np.asarray(G, np.float64) * soft_codes(l)
    c = codes(l.shape[1]).astype(np.float64)
    with np.errstate(invalid="ignore"):
        S1 = w @ c
        S0 = w @ (1.0 - c)
        out = sigmoid(-l) * S1 - sigmoid(l) * S0
    out[~np.isfinite(l).all(-1)] = np.nan
    return out


def st_grad_plain(l, G) -> np.ndarray:
    """S1_j - sigmoid(l_j) S, as the closed form is usually written."""
    l = np.asarray(l, np.float64)
    w = np.asarray(G, np.float64) * soft_codes(l)
    return w @ codes(l.shape[1]).astype(np.float64) - sigmoid(l) * w.sum(-1, keepdims=True)


def grad_total(l, idx, G, H, *, st: bool, aux_kind: str, thr: float) -> np.ndarray:
    """d/dl of sum(out * G) [straight-through] + aux [mean, or summed per-row] + sum(log_prob(indices) * H)."""
    g = log_prob_grad(l, idx, H)
    if st:
        g = g + st_grad(l, G)
    if aux_kind != "zero":
        g = g + aux_grad(l, thr, aux_kind == "mean")
    return g
