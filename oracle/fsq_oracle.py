"""numpy restatement of finite scalar quantization (TEST INFRASTRUCTURE ONLY): the reference's FSQ and ResidualFSQ stage loop
(finite_scalar_quantization.py "fsq", residual_fsq.py "rfsq"), element by element in the reference's operation order, in
float32 (numpy rounds every float32 op once, as torch does), with the bf16 chain of a bf16 module emulated by rounding after
every op.  Written from the reference's semantics; no reference source is copied.

Rows are (N, G, d): G groups (FSQ codebooks or GroupedResidualFSQ groups) of d = len(levels) values.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def bf16_round(a):
    """Round float32 values to bfloat16 (nearest, ties to even), returned as float32."""
    a = np.ascontiguousarray(a, dtype=F32)
    b = a.view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    out = (b & 0xFFFFFFFF).astype(np.uint32).view(F32)
    return np.where(np.isnan(a), a, out)


def _rw(a, bf):
    a = np.asarray(a, dtype=F32)
    return bf16_round(a) if bf else a


def tables(levels, sym, hard):
    """The per-dimension constants of fsq:152-156 / :165-166 (float32), as the kernels take them (include/vqb200.h rows)."""
    L = np.asarray(levels, dtype=np.int64)
    hw = (L // 2).astype(F32)
    if sym:
        a = (L - 1).astype(F32)
        b = (F32(2.) / (L - 1).astype(F32)).astype(F32)
        shift = np.zeros_like(a)
    else:
        a = ((L - 1).astype(F32) * F32(1 + 1e-3) / F32(2)).astype(F32)
        b = np.where(L % 2 == 0, F32(0.5), F32(0.0)).astype(F32)
        shift = (b / a).astype(F32) if hard else np.arctanh((b / a).astype(F32)).astype(F32)
    basis = np.cumprod([1] + list(L[:-1])).astype(F32)
    return dict(a=a, b=b, shift=shift, hw=hw, basis=basis, levels=L)


def _clamp1(v):
    return np.where(np.isnan(v), v, np.minimum(np.maximum(v, F32(-1)), F32(1))).astype(F32)


def stage(u, t, sym, hard):
    """One FSQ quantize on fp32 u (fsq:147-169): (code, pre (clamp/tanh input), h (its output), boundary value (pre-floor or
    pre-round))."""
    if sym:
        pre = u
        h = _clamp1(u) if hard else np.tanh(u).astype(F32)
        br = ((t["a"] * (h + F32(1))) / F32(2) + F32(0.5)).astype(F32)
        fl = (br + (np.floor(br) - br)).astype(F32)
        code = (t["b"] * fl - F32(1)).astype(F32)
    else:
        pre = (u + t["shift"]).astype(F32)
        h = _clamp1(pre) if hard else np.tanh(pre).astype(F32)
        br = (h * t["a"] - t["b"]).astype(F32)
        r = (br + (np.round(br) - br)).astype(F32)   # np.round: half to even, as torch.round
        code = (r / t["hw"]).astype(F32)
    return code, pre, h, br


def codes_to_indices(code, t, sym):
    """fsq:220-224: (N, G, d) fp32 codes -> int64 indices (N, G)."""
    if sym:
        s = ((code + F32(1)) / t["b"]).astype(F32)
    else:
        s = (code * t["hw"] + t["hw"]).astype(F32)
    terms = (s * t["basis"]).astype(F32)
    acc = np.zeros(code.shape[:-1], F32)
    for j in range(code.shape[-1]):
        acc = (acc + terms[..., j]).astype(F32)
    return np.round(acc).astype(np.int64)


def near_boundary(br, u, t, sym, hard, amp=None):
    """Elements whose boundary value (pre-floor for sym, pre-round otherwise), recomputed in float64 from the stage input u,
    lies within a few float32 ulps of a rounding boundary — where CUDA's tanhf and the CPU's tanh (an ulp apart at most) may
    round to different codes.  `amp` (same shape) widens the window by the absolute uncertainty of u itself (a soft-clamp ulp
    scaled up by 1 / scale_q)."""
    u64 = u.astype(np.float64)
    bound = (lambda v: np.clip(v, -1, 1)) if hard else np.tanh
    if sym:
        b64 = t["a"] * (bound(u64) + 1) / 2 + 0.5
        dist = np.abs(b64 - np.round(b64))
        slope = t["a"] / 2
    else:
        b64 = bound(u64 + t["shift"]) * t["a"] - t["b"]
        dist = np.abs(np.abs(b64 - np.floor(b64)) - 0.5)
        slope = t["a"]
    tol = 2.0 ** -19 * np.maximum(1.0, np.abs(b64))
    if amp is not None:
        tol = tol + slope * amp
    return dist <= tol


def forward(z, levels, Q, n_active, sym, hard, scales=None, clampv=None, w_bf16=False):
    """The ResidualFSQ stage loop (rfsq:193-241) on float32 z (N, G, d) (a plain FSQ: Q = 1, scales None, clampv None).  Returns
    dict(out (N, G, d) float32 values of the chain dtype, idx (N, G, Q) int64 with -1 for dropped stages, codes (Q, N, G, d)
    scaled stage codes, near (N, G, Q) bool: some element of the stage is near a rounding boundary, u (Q, N, G, d) stage inputs)."""
    t = tables(levels, sym, hard)
    N, G, d = z.shape
    r = np.asarray(z, F32)
    if clampv is not None:   # rfsq:193-195
        c = np.asarray(clampv, F32)
        r = _rw((_rw(np.tanh(_rw(r / c, w_bf16)), w_bf16)) * c, w_bf16)
    r0 = r.copy()
    out = np.zeros((N, G, d), F32)
    idx = np.full((N, G, Q), -1, np.int64)
    codes = np.zeros((Q, N, G, d), F32)
    near = np.zeros((N, G, Q), bool)
    us = np.zeros((Q, N, G, d), F32)
    for q in range(n_active):
        s = None if scales is None else np.asarray(scales[q], F32)
        u = r if s is None else _rw(r / s, w_bf16)
        code, pre, h, br = stage(u, t, sym, hard)
        idx[..., q] = codes_to_indices(code, t, sym)
        cw = _rw(code, w_bf16)
        qv = cw if s is None else _rw(cw * s, w_bf16)
        codes[q] = qv
        r = _rw(r - qv, w_bf16)
        out = qv.copy() if q == 0 else _rw(out + qv, w_bf16)
        us[q] = u
        if not hard or clampv is not None:
            amp = None
            if clampv is not None:
                amp = 2.0 ** -19 * np.maximum(np.abs(r0.astype(np.float64)), 1.0) / (1.0 if s is None else s.astype(np.float64))
            near[..., q] = near_boundary(br, u, t, sym, hard, amp).any(axis=-1)
    return dict(out=out, idx=idx, codes=codes, near=near, u=us, r0=r0)


def backward(z, g, levels, Q, n_active, sym, hard, scales=None, clampv=None, w_bf16=False, in_bf16=False):
    """d z of the chain given d out (N, G, d), as autograd takes it: per stage A_q = (chain of the stage's straight-through
    backward on g * scale_q) / scale_q; d r_q = A_q + d r_{q+1} (nested from the last stage); then the soft clamp's backward.
    Returns (dz float32 values of z's dtype, bound (N, G, d) float64): `bound` is zero where every factor is exact (hard clamp,
    no soft clamp) and otherwise the per-element room for tanh's last-ulp differences between CUDA and the CPU."""
    t = tables(levels, sym, hard)
    r = np.asarray(z, F32)
    g = np.asarray(g, F32)
    tc = None
    if clampv is not None:
        c = np.asarray(clampv, F32)
        tc = _rw(np.tanh(_rw(r / c, w_bf16)), w_bf16)
        r = _rw(tc * c, w_bf16)
    # a soft-clamp output a few ulps off (plus the roundings of the residual chain after it) moves stage q's input by that
    # much over scale_q: it moves tanh's derivative, and a hard clamp's mask where the input is that close to +-1
    du0 = 16 * np.spacing(np.maximum(np.abs(r), 1)).astype(np.float64) if clampv is not None else None
    A = []
    room = np.zeros(z.shape, np.float64)
    for q in range(n_active):
        s = None if scales is None else np.asarray(scales[q], F32)
        u = r if s is None else _rw(r / s, w_bf16)
        code, pre, h, br = stage(u, t, sym, hard)
        gc = g if s is None else _rw(g * s, w_bf16)
        if sym:
            gh = (((gc * t["b"]) / F32(2)) * t["a"]).astype(F32)
        else:
            gh = ((gc / t["hw"]) * t["a"]).astype(F32)
        if hard:
            gu = np.where((pre >= -1) & (pre <= 1), gh, F32(0)).astype(F32)
            if du0 is not None:
                sd = 1.0 if s is None else s.astype(np.float64)
                edge = np.abs(np.abs(pre.astype(np.float64)) - 1) <= du0 / sd
                room += np.where(edge, np.abs(gh.astype(np.float64)) / sd, 0.0)
        else:
            gu = (gh * (F32(1) - h * h)).astype(F32)
            # d(1 - h^2) for an h 2 ulps off, plus the product's own rounding
            h64 = np.abs(h.astype(np.float64))
            dh = 2 * np.spacing(np.abs(h)).astype(np.float64)
            if du0 is not None:
                dh = dh + (1 - h64 * h64) * du0 / (1.0 if s is None else s.astype(np.float64))
            room += np.abs(gh.astype(np.float64)) * (2 * h64 * dh + 2.0 ** -22) / (1.0 if s is None else s.astype(np.float64))
        gu = _rw(gu, w_bf16)
        A.append(gu if s is None else _rw(gu / s, w_bf16))
        cw = _rw(code, w_bf16)
        qv = cw if s is None else _rw(cw * s, w_bf16)
        r = _rw(r - qv, w_bf16)
    last = n_active - 1
    d = A[last]
    for q in range(last - 1, 0, -1):
        d = _rw(A[q] + d, w_bf16)
    if last >= 1:
        if in_bf16 and not w_bf16 and clampv is None and scales is not None:   # r_0 is bf16: each gradient rounds first
            d = bf16_round(bf16_round(A[0]) + bf16_round(d))
        else:
            d = _rw(A[0] + d, w_bf16)
    if clampv is not None:
        gt = _rw(d * c, w_bf16)
        ga = _rw(gt * (F32(1) - tc * tc), w_bf16)
        room = room + np.abs(gt.astype(np.float64)) * (2 * np.abs(tc.astype(np.float64)) * 2 * np.spacing(np.abs(tc)).astype(np.float64)
                                                      + 2.0 ** -22) / c.astype(np.float64) * 2
        d = _rw(ga / c, w_bf16)
    if room.any():   # the chain's own roundings after a perturbed term: a few ulps of the largest term
        mag = np.abs(np.stack(A).astype(np.float64)).sum(axis=0)
        room = room + (n_active + 4) * 2.0 ** -23 * mag
        if clampv is not None:
            room = room + 4 * 2.0 ** -23 * np.abs(d.astype(np.float64))
    if in_bf16 or w_bf16:
        room = np.where(room > 0, room + np.abs(d.astype(np.float64)) * 2.0 ** -7, room)
        d = bf16_round(d)
    return d, room


def decode(idx, levels, sym, scales=None, w_bf16=False):
    """indices (N, G, Q) (-1 = dropped) -> (sum over stages rounded once to the chain dtype, codes (Q, N, G, d)) (rfsq:131-171;
    fsq:202-218)."""
    t = tables(levels, sym, False)
    L = t["levels"]
    basis = np.cumprod([1] + list(L[:-1])).astype(np.int64)
    N, G, Q = idx.shape
    d = len(L)
    codes = np.zeros((Q, N, G, d), F32)
    for q in range(Q):
        ix = idx[..., q]
        lv = (np.maximum(ix, 0)[..., None] // basis) % L
        if sym:
            c = (lv.astype(F32) * t["b"] - F32(1)).astype(F32)
        else:
            c = ((lv - (L // 2)).astype(F32) / (L // 2).astype(F32)).astype(F32)
        c = _rw(c, w_bf16)
        if scales is not None:
            c = _rw(c * np.asarray(scales[q], F32), w_bf16)
        codes[q] = np.where((ix == -1)[..., None], F32(0), c)
    acc = np.zeros((N, G, d), F32)
    for q in range(Q):
        acc = (acc + codes[q]).astype(F32)
    return _rw(acc, w_bf16), codes
