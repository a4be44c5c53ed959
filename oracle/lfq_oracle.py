"""Float64 dense restatement of the LFQ entropy loss (lookup_free_quantization.py:347-403 of the reference) and of its
factorised form (DESIGN §4.10).  TEST INFRASTRUCTURE ONLY: torch float64 on whichever device the inputs live on.

`dense_stats` builds the (rows, K) probabilities: the definition.  `factored_stats` uses ln p[k] = sum_j l_j(bit_j(k)) with
l_j(1) = -softplus(-2 a_j), l_j(0) = -softplus(2 a_j), a_j = 2 tau m x_j: what the kernels compute.  Gradients come from
float64 autograd through the dense form.  `entropy_reference` restates the entropy kernels' outputs in float64 with
per-element error bounds derived from their fp32 arithmetic.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F


def codebook_signs(d, device="cpu"):
    """(K, d) float64 signs: bit j of code k is 2^(d-1-j) (dimension 0 is the most significant bit)."""
    k = torch.arange(1 << d, device=device)
    mask = 2 ** torch.arange(d - 1, -1, -1, device=device)
    return ((k[:, None] & mask) != 0).double() * 2 - 1


def log_probs_dense(x, m, tau):
    """x (R, d) float64 -> log softmax over the codes of 2 tau (x . m sgn_k), (R, K)."""
    logits = 2 * tau * (x.double() @ (m * codebook_signs(x.shape[-1], x.device)).t())
    return logits.log_softmax(-1)


def h(p):
    return -p * p.clamp(min=1e-5).log()


def dense_stats(x, m, tau):
    """x (R, d) -> (sum over rows and codes of h(p), column sums of p (K,)), float64."""
    p = log_probs_dense(x, m, tau).exp()
    return h(p).sum(), p.sum(0)


def factored_log_probs(x, m, tau):
    a = 2 * tau * m * x.double()
    l1 = -F.softplus(-2 * a)
    l0 = -F.softplus(2 * a)
    bits = (codebook_signs(x.shape[-1], x.device) > 0)
    return torch.where(bits[None], l1[:, None, :], l0[:, None, :]).sum(-1)


def factored_stats(x, m, tau):
    p = factored_log_probs(x, m, tau).exp()
    return h(p).sum(), p.sum(0)


def loss_and_grad(x, m, tau, cp, V, chunk=256):
    """L = cp * sum h(p) + sum_k V[k] * colsum_k (the linearisation the entropy backward receives) and dL/dx, float64, the rows
    in chunks of `chunk` so that the (rows, K) matrix stays small."""
    total = torch.zeros((), dtype=torch.float64, device=x.device)
    grads = []
    V = V.double() if V is not None else None
    for i in range(0, x.shape[0], chunk):
        xc = x[i:i + chunk].double().detach().requires_grad_(True)
        p = log_probs_dense(xc, m, tau).exp()
        L = cp * h(p).sum()
        if V is not None:
            L = L + (p.sum(0) * V).sum()
        L.backward()
        total += L.detach()
        grads.append(xc.grad)
    return total, torch.cat(grads)


# ---- float64 error bounds of the entropy kernels (vqb_lfq_entropy, vqb_lfq_entropy_backward in csrc/vq_lfq.cu) ----

U = 2.0 ** -24             # fp32 unit roundoff
EX2_REL = 2.0 ** -22       # ex2.approx.ftz.f32: maximum relative error (PTX ISA); results below 2^-126 flush to zero
FLT_MIN = 2.0 ** -126
SAFETY = 2.0               # on the first-order bounds: covers the neglected products of two error terms (O(u^2) relative)
LN2 = math.log(2.0)
LN_EPS, LOG2_EPS = math.log(1e-5), math.log2(1e-5)


def _F32(v):
    return float(np.float32(v))


# the kernel's clamp in fp32: its threshold log2(1e-5) and its value ln(1e-5), each rounded once
THR2 = abs(_F32(LOG2_EPS) - LOG2_EPS)                # log2 units
THR = abs(_F32(LN_EPS) - LN_EPS) + LN2 * THR2
ENT_THREADS, ENT_RB = 256, 32                         # entropy forward: threads per CTA, rows per batch


def gamma(n, u=U):
    """The bound n u / (1 - n u) on the relative error of n roundings (a recursive sum of n + 1 terms)."""
    n = max(n, 0)
    return n * u / (1 - n * u)


def _code_bits(d, device):
    k = torch.arange(1 << d, device=device)
    return ((k[:, None] >> torch.arange(d - 1, -1, -1, device=device)) & 1).double()   # (K, d): bit j = 2^(d-1-j)


def entropy_block(x, m, tau, cp=None, V=None):
    """Dense float64 quantities of the entropy kernels for the rows x (n, d), with their per-element first-order error terms.

    The kernels take tau, m, cp and V in fp32; so does this (each rounded to fp32 first), and x holds fp32 values.  Errors
    are bounded from the kernels' arithmetic, u = 2^-24, gamma_n = n u / (1 - n u):

    * ell.  The kernels compute l_j(b) = -softplus(y) / ln 2 with y = -+2 fl(fl(2 tau m) x_j) as
      -(max(y, 0) + log1pf(expf(-|y|))) * LOG2E: expf (2 ulp = 4u), log1pf (1 ulp = 2u, and z / ((1 + z) log1p(z)) <= 1
      carries expf's error at most 1:1), the add, the fp32 LOG2E and the multiply give 9u |l_j|; the two roundings in y give
      gamma_2 |y| sigma(y) / ln 2 (the derivative times the argument error).  That is e_j(b), in log2 units.
    * log2 p.  Every l_j <= 0, so the fp32 sum of the d terms (TA + TB in any order) adds gamma_{d-1} |log2 p_k|:
      B_k = gamma_{d-1} |log2 p_k| + sum_j e_j(bit_j(k)).  ex2.approx then gives the relative error of p_k
      eps_k = expm1(ln2 B_k) (1 + 2^-22) + 2^-22, and dp_k = p_k eps_k, plus p_k itself where the result flushes to zero.
    * h(p) = -p max(ln p, ln 1e-5).  The kernel takes lp >= fl(log2 1e-5) ? fl(lp LN2) : fl(ln 1e-5).  The clamped log is
      continuous in p, so even on the wrong side of the threshold its error is at most ln2 B_k + 2u |max(ln p, ln 1e-5)| +
      THR (the two fp32 constants).  Per term: dT = dp |L| + p dL.
    * h'(p) = -(ln p + 1) above the clamp, -ln 1e-5 below, a jump of 1 at p = 1e-5: where |log2 p - log2 1e-5| <= B_k +
      THR2 the kernel may take the other side, and dh' gains 1.  u_k = fl(cp h' + V_k) (one fma): du = |cp| dh' + u |u_k|;
      w_k = p_k u_k: dw = |u_k| dp + p du + u |w|.

    Returns a dict of (n, K) tensors p, lnp, w (or None), and the per-element terms pse_d (dT), pse_m (p |L|), col_d (dp),
    w_d (dw) (or None)."""
    d = x.shape[-1]
    dev = x.device
    tau, m = _F32(tau), _F32(m)
    tm = 2 * tau * m
    x = x.double()
    lnp = log_probs_dense(x, m, tau)
    p = lnp.exp()
    bits = _code_bits(d, dev)
    a = tm * x
    sp1, sp0 = F.softplus(-2 * a), F.softplus(2 * a)                          # -ln sigma for bit 1 / bit 0
    e1 = (9 * U * sp1 + gamma(2) * (2 * a).abs() * torch.sigmoid(-2 * a)) / LN2
    e0 = (9 * U * sp0 + gamma(2) * (2 * a).abs() * torch.sigmoid(2 * a)) / LN2
    E = e0.sum(-1, keepdim=True) + (e1 - e0) @ bits.t()
    lp2 = lnp / LN2
    B = gamma(d - 1) * lp2.abs() + E
    eps = torch.expm1(LN2 * B) * (1 + EX2_REL) + EX2_REL
    zero = torch.zeros_like(p)
    dp = torch.where(p > 0, p * eps, zero)   # p = 0 in float64: far below fp32's range, where ex2 flushes to zero too
    dp = dp + torch.where(p < 2 * FLT_MIN, p, zero)
    L = lnp.clamp(min=LN_EPS)
    dL = LN2 * B + 2 * U * L.abs() + THR
    out = dict(p=p, lnp=lnp, pse_d=dp * L.abs() + p * dL, pse_m=p * L.abs(), col_d=dp, w=None, w_d=None)
    if cp is None and V is None:
        return out
    cp = _F32(cp) if cp is not None else 0.
    hp = torch.where(p >= 1e-5, -(lnp + 1), torch.full_like(p, -LN_EPS))
    uk = cp * hp
    if V is not None:
        uk = uk + V.float().double()[None, :]
    w = p * uk
    jump = ((lp2 - LOG2_EPS).abs() <= B + THR2).double()
    dhp = LN2 * B + 2 * U * (L.abs() + 1) + THR + jump
    du = abs(cp) * dhp + U * uk.abs()
    out.update(w=w, w_d=uk.abs() * dp + p * du + U * w.abs())
    return out


@dataclass
class EntropyRef:
    """Float64 reference values of the entropy kernels for one (stage, group) row set, and the plan-independent parts of
    their error bounds; `bounds(chunks, ksplit)` adds the plan's summation terms."""
    d: int
    R: int
    pse: torch.Tensor       # ()   sum of h(p)
    colsum: torch.Tensor    # (K,) column sums of p
    grad: torch.Tensor      # (R, d) d/dx of cp sum h(p) + sum_k V_k colsum_k, or None
    pse_d: float
    pse_m: float
    col_d: torch.Tensor
    col_m: torch.Tensor
    g_d: torch.Tensor       # (R,) sum_k dw
    g_abs: torch.Tensor     # (R,) sum_k |w|
    g_tot: torch.Tensor     # (R,) sum_k w
    tm: float
    t: torch.Tensor         # (R, d) tanh(a)
    a: torch.Tensor         # (R, d)

    def bounds(self, chunks, ksplit):
        """Per-element float64 bounds on |kernel - reference| of pse (), colsum (K,) and grad (R, d) for the plan.

        pse: each thread sums h over its <= 16 codes of a row with fp32 fmas (gamma_16), then fp64 over rows, threads, CTAs
        and the torch sum of the partials.  colsum: a thread's fp32 column sum runs over the rows of its chunk (or, at d < 8,
        its lane's share of every 32-row batch, then the `lanes` lane sums), and torch adds the `chunks` partials in fp32.
        grad: each 16-code step sums w and +-w in fp32 (gamma_15) into fp64, a split's sums are rounded to fp32 (u), the
        fin kernel adds the `ksplit` splits in fp32 (gamma_{ksplit-1}) and forms fl(2 tau m) (s_j - S tanhf(fl(fl(2 tau m)
        x_j))) (the products, the difference, tm: 5u; tanhf: 2 ulp = 4u |t|; its argument: gamma_2 |a| (1 - t^2)).  So
        |dg_j| <= tm (1 + |t_j|) (sum_k dw_k + (gamma_15 + gamma_{ksplit-1} + 5u) sum_k |w_k|) + tm |sum_k w_k| dt_j."""
        d, R, K = self.d, self.R, 1 << self.d
        ud = 2.0 ** -53
        tiles = 1 << max(0, d - 12)
        pse = self.pse_d + (gamma(16) + gamma(R * tiles + ENT_THREADS + chunks * tiles, ud)) * (self.pse_m + self.pse_d)
        chunk_rows = -(-R // chunks)
        lanes = ENT_THREADS >> min(d, 8)
        per_thread = chunk_rows if lanes == 1 else -(-chunk_rows // ENT_RB) * -(-ENT_RB // lanes)
        col = self.col_d + gamma(per_thread + lanes + chunks) * (self.col_m + self.col_d)
        grad = None
        if self.grad is not None:
            s = self.g_d + (gamma(15) + gamma(ksplit - 1) + 5 * U + gamma(K, ud)) * self.g_abs
            dt = 4 * U * self.t.abs() + gamma(2) * self.a.abs() * (1 - self.t ** 2)
            grad = self.tm * (1 + self.t.abs()) * s[:, None] + self.tm * self.g_tot.abs()[:, None] * dt
            grad = SAFETY * grad
        return SAFETY * pse, SAFETY * col, grad


def entropy_reference(x, m, tau, cp=None, V=None, chunk=None):
    """EntropyRef for the rows x (R, d) (fp32 values) with code magnitude m and temperature tau; with cp and / or V (K,) also
    the gradient the backward receives dL/dp = cp h'(p) + V.  The (rows, K) blocks have `chunk` rows (<= 256 MiB each by
    default).  The gradient is the closed form 2 tau m (sum_k w_k sgn_kj - (sum_k w_k) tanh(a_j)), w = p dL/dp."""
    R, d = x.shape
    K = 1 << d
    chunk = chunk or max(1, (1 << 25) // K)
    want_grad = cp is not None or V is not None
    tm = 2 * _F32(tau) * _F32(m)
    signs = codebook_signs(d, x.device)
    acc = dict(pse=0., pse_d=0., pse_m=0., col=0., col_d=0.)
    gs, gd, gabs, gtot = [], [], [], []
    for i in range(0, R, chunk):
        b = entropy_block(x[i:i + chunk], m, tau, cp, V)
        acc["pse"] += float(h(b["p"]).sum())
        acc["pse_d"] += float(b["pse_d"].sum())
        acc["pse_m"] += float(b["pse_m"].sum())
        acc["col"] = acc["col"] + b["p"].sum(0)
        acc["col_d"] = acc["col_d"] + b["col_d"].sum(0)
        if want_grad:
            w = b["w"]
            gs.append(w @ signs)
            gd.append(b["w_d"].sum(1))
            gabs.append(w.abs().sum(1))
            gtot.append(w.sum(1))
        del b
    a = tm * x.double()
    t = a.tanh()
    grad = g_d = g_abs = g_tot = None
    if want_grad:
        g_tot = torch.cat(gtot)
        grad = tm * (torch.cat(gs) - g_tot[:, None] * t)
        g_d, g_abs = torch.cat(gd), torch.cat(gabs)
    return EntropyRef(d, R, torch.tensor(acc["pse"], dtype=torch.float64), acc["col"], grad, acc["pse_d"], acc["pse_m"],
                      acc["col_d"], acc["col"], g_d, g_abs, g_tot, tm, t, a)


def chain(z, params, Q, n_active, residual, training, spherical, dtype=None, force_q=None):
    """Restatement of the row chain with the reference's torch ops (lfq:295-343 per stage, rlfq:179-190 around them) on z
    (N, G, d): soft clamp, l2norm, sign, index bits, x + (q - x), residual and running sum, in `dtype` (z's by default; float64
    for a gradient oracle).  params (3, Q): scale, magnitude, clamp (0: none).  -> (out, indices (N, G, Q) int64, stage
    inputs (n_active, N, G, d) fp32-or-dtype, quantized (n_active, N, G, d)); the straight-through value is differentiable.
    force_q: the quantized values of another run (n_active, N, G, d), used instead of this run's signs, so that a float64
    gradient follows the same discrete path as the fp32 / bf16 chain it checks."""
    dt = dtype or z.dtype
    r = z.to(dt)
    d = z.shape[-1]
    bitw = 2 ** torch.arange(d - 1, -1, -1, device=z.device)
    out = None
    idx = torch.full((*z.shape[:-1], Q), -1, dtype=torch.int64, device=z.device)
    ents, qs = [], []
    p = params.double().cpu().tolist()
    for q in range(n_active):
        s, m, c = p[0][q], p[1][q], p[2][q]
        x = r
        if c != 0.:
            x = (x / c).tanh() * c
        if spherical:
            x = F.normalize(x, dim=-1) * s
        xf = x.float() if dt != torch.float64 else x
        qv = torch.where(xf > 0, torch.full_like(xf, m), torch.full_like(xf, -m)) if force_q is None else force_q[q].to(xf.dtype)
        idx[..., q] = ((qv > 0).long() * bitw).sum(-1)
        o = (xf + (qv - xf).detach()) if training else qv
        o = o.to(dt)
        ents.append(xf)
        qs.append(qv)
        r = r - o.detach()
        out = o if out is None else out + o
    return out, idx, torch.stack(ents), torch.stack(qs)
