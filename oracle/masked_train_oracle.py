"""numpy restatement of one masked training step of VectorQuantize, ResidualVQ and GroupedResidualVQ (vqp:1093-1403, rvq:384-630,
:688-724) — TEST INFRASTRUCTURE ONLY.

Every row is searched, but only the live rows (mask True) matter: the padding rows return 0 (or the input, with
return_zeros_for_masked_padding=False) and index -1, take no part in the loss, and pass no gradient (or the upstream one).
Backward to x on a live row: the estimator's backward of the upstream gradient at (transform_input(x), q) — rotate_to or the
identity, through l2norm for cosine codebooks — plus the masked commitment-loss term 2 w dL/dloss (x - q) / (n_live D).
ResidualVQ: every layer gets the mask (rvq:495), the residual chain passes the identity to x (the reference detaches the
quantized rows in it), and project_in / project_out wrap the layers.  Codebook updates are not restated here (the EMA
oracles cover them): every search uses the codebooks of the state_dict before the step, as the reference does within one
forward.  All arithmetic in fp32 (pinned by tests/test_masked_train_oracle.py against the reference's own outputs).
"""
from __future__ import annotations

import random

import numpy as np

from oracle.residual_simvq_oracle import linear, rotate_to, rotate_to_backward

F32 = np.float32


def l2norm(x):
    return (x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), F32(1e-12))).astype(F32)


def l2norm_backward(x, g):
    """d/dx of sum(g * l2norm(x)) (F.normalize above its eps)."""
    n = np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), F32(1e-12)).astype(F32)
    u = (x / n).astype(F32)
    return ((g - (g * u).sum(-1, keepdims=True) * u) / n).astype(F32)


def search(r, C, cosine):
    """Indices of the reference's search: the cdist arg-min (vqp:58-62) or the arg-max of l2norm(r) . C (vqp:741)."""
    if cosine:
        return np.argmax(l2norm(r) @ C.T, axis=-1)
    x2 = (r * r).sum(-1, dtype=F32)[:, None]
    y2 = (C * C).sum(-1, dtype=F32)[None, :]
    d2 = np.maximum((x2 + y2).astype(F32) - (F32(2) * (r @ C.T)).astype(F32), F32(0))
    return np.argmin(np.sqrt(d2), axis=-1)


def vq_step(x, mask, C, G, *, cosine=False, rotation=True, pad_zeros=True, commit_weight=1.0, lw=1.0):
    """VectorQuantize (b, n, d) channel-last, one codebook C (K, d).  Returns (out, indices, loss, x.grad) of a backward of
    sum(out * G) + lw * loss."""
    x = x.astype(F32)
    shape, D = x.shape, x.shape[-1]
    xr, Gr, live = x.reshape(-1, D), G.astype(F32).reshape(-1, D), mask.reshape(-1)
    n_live = int(live.sum())
    out = np.zeros_like(xr) if pad_zeros else xr.copy()
    idx = np.full((xr.shape[0],), -1, dtype=np.int64)
    gx = np.zeros_like(xr) if pad_zeros else Gr.copy()
    loss = F32(0)
    if n_live:
        xl, gl = xr[live], Gr[live]
        k = search(xl, C, cosine)
        q = C[k].astype(F32)
        idx[live], out[live] = k, q
        loss = F32(np.mean((q - xl) ** 2, dtype=F32) * F32(commit_weight))
        xt = l2norm(xl) if cosine else xl
        est = rotate_to_backward(xt, q, gl) if rotation else gl
        if cosine:
            est = l2norm_backward(xl, est)
        gx[live] = est + F32(2.0 * lw * commit_weight / (n_live * D)) * (xl - q)
    return out.reshape(shape), idx.reshape(shape[:-1]), loss, gx.reshape(shape)


def rvq_step(x, mask, state, G, *, num_quantizers, shared_codebook=False, rotation=True, commit_weight=1.0, lw=1.0,
             n_run=None, prefix=""):
    """ResidualVQ on (b, n, dim) with the state_dict `state` (numpy arrays).  Returns (out, indices (b, n, Q), losses (Q,),
    x.grad, {parameter name: grad}) of a backward of sum(out * G) + lw * sum(losses)."""
    x = x.astype(F32)
    shape, Q = x.shape, num_quantizers
    n_run = Q if n_run is None else n_run
    proj = f"{prefix}project_in.weight" in state
    xr, Gr, live = x.reshape(-1, shape[-1]), G.astype(F32).reshape(-1, shape[-1]), mask.reshape(-1)
    xp = linear(xr, state[f"{prefix}project_in.weight"], state[f"{prefix}project_in.bias"]) if proj else xr
    N, D = xp.shape
    n_live = int(live.sum())
    g_q = (Gr @ state[f"{prefix}project_out.weight"].astype(F32)).astype(F32) if proj else Gr   # d/d quantized_out
    qout = np.zeros((N, D), F32)
    idx = np.full((N, Q), -1, dtype=np.int64)
    losses = np.zeros((Q,), F32)
    gxp = np.zeros((N, D), F32)
    if n_live:
        r, g = xp[live], g_q[live]
        acc, gacc = np.zeros_like(r), np.zeros_like(r)
        for q in range(n_run):
            C = state[f"{prefix}layers.{0 if shared_codebook else q}._codebook.embed"][0].astype(F32)
            k = search(r, C, False)
            c = C[k].astype(F32)
            idx[live, q] = k
            losses[q] = F32(np.mean((c - r) ** 2, dtype=F32) * F32(commit_weight))
            val = rotate_to(r, c) if rotation else ((c - r).astype(F32) + r).astype(F32)
            gacc = gacc + (rotate_to_backward(r, c, g) if rotation else g) + F32(2.0 * lw * commit_weight / (n_live * D)) * (r - c)
            acc = (acc + val).astype(F32)
            r = (r - val).astype(F32)
        qout[live], gxp[live] = acc, gacc
    grads = {}
    if proj:
        w_out = state[f"{prefix}project_out.weight"].astype(F32)
        out = linear(qout, w_out, state[f"{prefix}project_out.bias"])
        grads[f"{prefix}project_out.weight"] = (Gr.T @ qout).astype(F32)
        grads[f"{prefix}project_out.bias"] = Gr.sum(0).astype(F32)
        grads[f"{prefix}project_in.weight"] = (gxp.T @ xr).astype(F32)
        grads[f"{prefix}project_in.bias"] = gxp.sum(0).astype(F32)
        gx = (gxp @ state[f"{prefix}project_in.weight"].astype(F32)).astype(F32)
    else:
        out, gx = qout, gxp
    return out.reshape(shape), idx.reshape(*shape[:-1], Q), losses, gx.reshape(shape), grads


def dropout_layers(seed, cutoff, Q):
    """Layers a quantize-dropout forward runs with rand_quantize_dropout_fixed_seed=seed (rvq:423-439, multiple_of 1)."""
    return random.Random(seed).randrange(cutoff, Q) + 1


def grvq_step(x, mask, state, G, *, groups, **kw):
    """GroupedResidualVQ: `groups` ResidualVQs over the feature chunks (rvq:688-724), each given the mask."""
    xs, Gs = np.split(x, groups, axis=-1), np.split(G, groups, axis=-1)
    res = [rvq_step(xg, mask, state, gg, prefix=f"rvqs.{g}.", **kw) for g, (xg, gg) in enumerate(zip(xs, Gs))]
    grads = {}
    for r in res:
        grads.update(r[4])
    return (np.concatenate([r[0] for r in res], -1), np.stack([r[1] for r in res]), np.stack([r[2] for r in res]),
            np.concatenate([r[3] for r in res], -1), grads)
