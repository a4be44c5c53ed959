"""Numpy restatement (float64) of one training step of a codebook learnt by gradient (tests/golden/learnable/*.npz): the
forward value, indices, loss, d/dx and d/d embed of sum(out * G) + LW * sum(loss), then the SGD step of the codebook.

    VectorQuantize (vqp:1212-1237, :1327): q = C[argmin_k ||x - c_k||]; with x requiring grad the estimator (rotation trick,
    straight-through or DiVeQ) decides where G goes; without it G reaches the codes; sync_update_v scales that by 1 + v;
    the commitment loss adds 2 w (q - x) / numel per row to the code's gradient (and its negative to x).
    ResidualVQ (rvq:469-606): the same per stage on the residual, DiVeQ of (x, sum of the stages' codes) at the end.
"""
import numpy as np

from oracle.residual_simvq_oracle import rotate_to_backward

F64 = np.float64


def round_bf16(a):
    """Round-to-nearest-even to bfloat16 (finite values), returned as float64."""
    b = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32).astype(F64)


def search(r, C):
    """argmax(-cdist) of the reference (vqp:58-62, :743) in its fp32 arithmetic: near-ties fall as they fall there."""
    r, C = np.asarray(r, np.float32), np.asarray(C, np.float32)
    F32 = np.float32
    x2 = (r * r).sum(-1, dtype=F32)[:, None]
    y2 = (C * C).sum(-1, dtype=F32)[None, :]
    d2 = np.maximum((x2 + y2).astype(F32) + (F32(-2) * (r @ C.T)).astype(F32), F32(1e-8))
    return np.argmin(np.sqrt(d2), axis=-1)


def code_sums(rows, idx, K):
    out = np.zeros((K, rows.shape[1]), F64)
    np.add.at(out, idx, rows)
    return out


def diveq(x, q, z, variance):
    """vqp:323-330: value and the backward pieces (u, e, ||e||)."""
    e = q - x
    ne = np.sqrt((e * e).sum(-1, keepdims=True))
    n = e + np.sqrt(variance) * z
    u = n / np.maximum(np.sqrt((n * n).sum(-1, keepdims=True)), 1e-6)
    return x + u * ne, (u, e, ne)


def diveq_backward(G, parts):
    u, e, ne = parts
    s = (G * u).sum(-1, keepdims=True)
    de = np.where(ne > 0, s / np.where(ne > 0, ne, 1.0), 0.0) * e
    return G - de, de


def vq_rows(x, G, C, *, x_grad, rotation, diveq_var=None, noise=None, commit_weight=1.0, sync_v=0.0, lw=1.0):
    """One VectorQuantize step on rows.  Returns (idx, out, loss, xgrad, egrad)."""
    x, G, C = (np.asarray(a, F64) for a in (x, G, C))
    K = C.shape[0]
    numel = x.size
    idx = search(x, C)
    q = C[idx]
    has_commit = commit_weight > 0 and diveq_var is None
    loss = commit_weight * ((q - x) ** 2).mean() if has_commit else 0.0
    Gv = G * (1.0 + sync_v)
    xgrad = np.zeros_like(x)
    g_code = np.zeros_like(x)
    if x_grad and diveq_var is not None:
        out, parts = diveq(x, q, np.asarray(noise, F64), diveq_var)
        xgrad, g_code = diveq_backward(Gv, parts)
    elif x_grad and rotation:
        out = q
        xgrad = rotate_to_backward(x, q, Gv)
    elif x_grad:
        out = q
        xgrad = Gv.copy()
    else:
        out = q
        g_code = Gv
    if has_commit:
        c = lw * commit_weight * 2.0 * (q - x) / numel
        g_code = g_code + c
        xgrad = xgrad - c
    return idx, out, loss, xgrad, code_sums(g_code, idx, K)


def rvq_rows(x, G, books, *, x_grad, rotation=True, diveq_var=None, noise=None, commit_weight=1.0, lw=1.0, bf16=False,
             given_idx=None):
    """One ResidualVQ step on rows; books: one (K, D) array per stage (the same array for a shared codebook).  bf16: the
    residual and the running sum are bf16 tensors in the reference (rvq:524-525), rounded after every stage.  given_idx (N, Q):
    take these codes instead of searching (bf16 with the rotation trick: the reference subtracts the estimator's bf16 value,
    whose rounding this restatement does not reproduce, so its later stages search slightly different residuals).
    Returns (idx (N, Q), out, losses (Q,), xgrad, egrads per stage)."""
    x, G = np.asarray(x, F64), np.asarray(G, F64)
    numel = x.size
    r = x.copy()
    qsum = np.zeros_like(x)
    idxs, losses, egrads = [], [], []
    xgrad = np.zeros_like(x)
    for q, C in enumerate(books):
        C = np.asarray(C, F64)
        idx = search(r, C) if given_idx is None else given_idx[:, q]
        c = round_bf16(C[idx]) if bf16 else C[idx]
        g_code = np.zeros_like(x)
        if diveq_var is None:
            losses.append(commit_weight * ((c - r) ** 2).mean())
            if x_grad:
                xgrad += rotate_to_backward(r, c, G) if rotation else G
            cg = lw * commit_weight * 2.0 * (c - r) / numel
            g_code += cg
            xgrad -= cg
        else:
            losses.append(0.0)
        idxs.append(idx)
        egrads.append((idx, g_code))
        r = round_bf16(r - c) if bf16 else r - c
        qsum = round_bf16(qsum + c) if bf16 else qsum + c
    out = qsum
    if diveq_var is not None:
        out, parts = diveq(x, qsum, np.asarray(noise, F64), diveq_var)
        dx, dq = diveq_backward(G, parts)
        xgrad = dx
        egrads = [(idx, g + dq) for idx, g in egrads]
    K = [np.asarray(C).shape[0] for C in books]
    return (np.stack(idxs, axis=1), out, np.asarray(losses), xgrad,
            [code_sums(g, idx, k) for (idx, g), k in zip(egrads, K)])
