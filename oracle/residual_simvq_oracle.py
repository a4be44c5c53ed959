"""numpy restatement of ResidualSimVQ (residual_sim_vq.py:182-203 over sim_vq.py:100-138) — TEST INFRASTRUCTURE ONLY.

Forward: per stage the cdist arg-min of the residual against the stage's implicit codebook, the two commitment terms, the
rotation-trick / straight-through value `out`, then r <- r - out and quantized_out <- quantized_out + out.  Backward to x: every
stage's residual depends on x through the identity (the reference detaches `out` in the recurrence), so
d/dx = sum_q [estimator backward of G at (r_q, c_q) + dL/dloss_q * weight * input_weight * 2 (r_q - c_q) / numel].
All arithmetic in fp32 like the reference (pinned by tests/test_residual_simvq_oracle.py against its outputs).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
EPS = F32(1e-6)   # safe_div / l2norm eps (vector_quantize_pytorch.py:37-41)


def linear(x, weight, bias=None):
    y = (x.astype(F32) @ weight.astype(F32).T).astype(F32)
    return y if bias is None else (y + bias.astype(F32)).astype(F32)


def implicit_codebooks(state: dict, n_layers: int, transform: str | None):
    """C_q = code_transform(frozen_codebook) (sim_vq.py:81-83) from a ResidualSimVQ state_dict of numpy arrays."""
    books = []
    for q in range(n_layers):
        frozen = state[f"layers.{q}.frozen_codebook"]
        if transform == "mlp":   # Linear -> ReLU -> Linear, one module shared by every layer
            h = np.maximum(linear(frozen, state[f"layers.{q}.code_transform.0.weight"], state[f"layers.{q}.code_transform.0.bias"]), 0)
            books.append(linear(h, state[f"layers.{q}.code_transform.2.weight"], state[f"layers.{q}.code_transform.2.bias"]))
        else:
            books.append(linear(frozen, state[f"layers.{q}.code_transform.weight"]))
    return books


def _rotation_terms(s, t):
    ns = np.linalg.norm(s, axis=-1, keepdims=True).astype(F32)
    nt = np.linalg.norm(t, axis=-1, keepdims=True).astype(F32)
    u = (s / np.maximum(ns, EPS)).astype(F32)
    q = (t / np.maximum(nt, EPS)).astype(F32)
    w = (u + q).astype(F32)
    w = (w / np.maximum(np.linalg.norm(w, axis=-1, keepdims=True), EPS)).astype(F32)
    lam = (nt / np.maximum(ns, EPS)).astype(F32)
    return u, q, w, lam


def rotate_to(s, t):
    """vector_quantize_pytorch.py:287-318: (s - 2 (s.w) w + 2 (s.u) q) * ||t|| / ||s||."""
    u, q, w, lam = _rotation_terms(s, t)
    out = s - 2 * (s * w).sum(-1, keepdims=True) * w + 2 * (s * u).sum(-1, keepdims=True) * q
    return (out * lam).astype(F32)


def rotate_to_backward(s, t, g):
    """d/ds of sum(g * rotate_to(s, t)): only `e = s` carries gradient (w, u, q and the scale are detached)."""
    u, q, w, lam = _rotation_terms(s, t)
    d = g - 2 * (g * w).sum(-1, keepdims=True) * w + 2 * (g * q).sum(-1, keepdims=True) * u
    return (d * lam).astype(F32)


def forward(x, books, n_active, rotation, input_weight=0.25, commitment_weight=1.0, G=None, loss_grad=None):
    """x (N, D) fp32 rows, books [Q] of (K, D) fp32.  Returns (quantized_out, indices (N, Q) int64 with -1 for the dropped
    stages, losses (Q,), and — when G (N, D) and loss_grad (Q,) are given — d/dx of sum(quantized_out * G) + sum(losses *
    loss_grad))."""
    x = x.astype(F32)
    N, D = x.shape
    Q = len(books)
    r = x
    qout = np.zeros_like(x)
    idx = np.full((N, Q), -1, dtype=np.int64)
    losses = np.zeros((Q,), dtype=F32)
    gx = np.zeros_like(x) if G is not None else None
    for q in range(n_active):
        C = books[q].astype(F32)
        x2 = (r * r).sum(-1, dtype=F32)[:, None]
        y2 = (C * C).sum(-1, dtype=F32)[None, :]
        d2 = np.maximum((x2 + y2).astype(F32) - (F32(2) * (r @ C.T)).astype(F32), F32(0))
        k = np.argmin(np.sqrt(d2), axis=-1)                    # first minimum, like torch.argmin (sim_vq.py:112-113)
        idx[:, q] = k
        c = C[k]
        mse = np.mean((r - c).astype(F32) ** 2, dtype=F32)
        losses[q] = F32(mse + mse * F32(input_weight)) * F32(commitment_weight)   # sim_vq.py:121-124, :138
        out = rotate_to(r, c) if rotation else ((c - r).astype(F32) + r).astype(F32)
        if gx is not None:
            est = rotate_to_backward(r, c, G) if rotation else G
            gx = (gx + est + F32(loss_grad[q] * commitment_weight * input_weight * 2.0 / x.size) * (r - c)).astype(F32)
        qout = (qout + out).astype(F32)                         # rsv:196 (0. + out for the first stage)
        r = (r - out).astype(F32)                               # rsv:195: the estimator's forward value, detached
    return qout, idx, losses, gx
