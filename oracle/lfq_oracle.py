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


# ---- float64 reference of the row kernels (vqb_lfq_forward, vqb_lfq_backward in csrc/vq_lfq.cu) with per-element bounds ----

LFQ_THREADS = 256          # the row kernels' CTA size: item `it` runs in block (it mod (grid * 256)) / 256


def l2norm_eps(bf):
    """F.normalize's eps = 1e-12 in the chain's dtype, the clamp the forward compares the rounded norm with."""
    e = torch.tensor(1e-12, dtype=torch.float32)
    return float(e.bfloat16().float()) if bf else float(e)


@dataclass
class RowRef:
    """Float64 values of the row chain along one discrete path, and bounds on |computed - value| for a chain that rounds as
    the kernels do.  Stage tensors are (n_active, N, G, d); items are (N, G)."""
    x: torch.Tensor          # stage inputs: the values the sign is taken of, and the entropy input
    x_b: torch.Tensor
    sign_b: torch.Tensor     # how far from zero a computed stage input can lie on the other side of x's sign (<= x_b)
    pos: torch.Tensor        # the path: x > 0 (bool)
    idx: torch.Tensor        # (N, G, Q) int64 indices of the path, -1 past n_active
    out: torch.Tensor        # (N, G, d)
    out_b: torch.Tensor
    commit: torch.Tensor     # (n_active, N, G) one item's term sum_j (x_j - q_j)^2 of each stage (rowmask not applied)
    commit_b: torch.Tensor
    grad: torch.Tensor       # (N, G, d) d z, or None
    grad_b: torch.Tensor
    clamp_side_unsure: torch.Tensor   # (n_active, N, G) spherical: the rounded norm may fall on either side of the l2norm clamp


def chain_reference(z, params, Q, n_active, residual, training, spherical, gout=None, gent=None, cc=None, rowmask=None,
                    signs=None):
    """The row chain of `chain` in float64, along the signs `signs` ((n_active, N, G, d) bool, the path of another run) or its
    own, with per-element bounds on how far a chain that rounds like the kernels can be from it.

    z (N, G, d) fp32 or bf16 (the chain's dtype W), params (3, Q) fp32 (scale s, magnitude m, clamp c), gout (N, G, d),
    gent (n_active, N, G, d), cc (n_active,) and rowmask (N,) as vqb_lfq_backward takes them.  The gradient is that of
    <out, gout> (training only: in eval out is q) + <x_q, gent_q> + cc_q / 2 sum over live rows of |x_q - q|^2, torch's
    autograd in float64: the l2norm's projection applies where ||x|| >= eps (clamp_min passes the gradient there), else the
    Jacobian is I s / eps.

    The bounds follow the kernels' arithmetic (csrc/vq_lfq.cu), first order, each rounding contributing u |value|
    (u = 2^-24 for an fp32 op; ur = 2^-24 + 2^-8 for an fp32 op followed by the round to bf16 of a bf16 chain; plus an
    absolute 2^-149 / 2^-133 where a result may be subnormal; |value| is that of the computed result, the float64 value plus
    its bound), and the error of each operand carried through the operation (its derivative times the operand's bound; for
    tanh the image of the operand's interval, and a normalised element never moves by more than to the edge of [-1, 1]):
    * stage_input: y = __fdiv_rn(x, c) (ur), tanhf (2 ulp = 4u, then ur), t c (__fmul_rn, ur); the norm's sequential
      __fmaf_rn sum of d squares (gamma_d relative, 2 |x| e_x carried), __fsqrt_rn (u, then ur), the clamp max(., eps)
      (1-Lipschitz; exact where the norm plus its bound is below eps), x / nrm (__fdiv_rn, ur) and * s (__fmul_rn, ur).
    * the stage output fl(x + fl(q - x)) equals q up to u (|q - x| + e_x) + ur |q| (eval: q rounded to W, 2^-8 |q| in bf16);
      the residual r - ov and the running sum o + ov add ur of their result.  The stage input is the entropy input.
    * the commitment term: fl(x - q) (u), its fp32 square (u), the rest fp64 (the block sums: negligible, gamma(n, 2^-53)).
    * the backward, per stage: gi = go + gent + cc (x - q) in fp32 (gamma_4 on the magnitudes, cc e_x carried), rounded to
      W; spherical: g s (ur), y = x / s (u), the fp32 dot product (gamma_{d+1}), (g - y dot) / nrm (gamma_2, u, the norm's
      bound carried), and where the norm may lie on either side of the clamp the whole projection term |y dot| / nrm; the
      clamp: (1 - t^2) (2 |t| e_t + u), the product (u); rounded to W; the stages added in fp32 (gamma_{n_active - 1}) and
      rounded once at the store (bf16: 2^-8).
    * the sign: x / nrm * s has the sign of the value v before the l2norm (times the sign of s), so a computed stage input
      can have the other sign only if v's bound e_v reaches zero; it then lies within e_v |s| / (nrm - e_nrm) of zero
      (plus u for the division and the product, and the underflow of x / nrm).  That is sign_b: 0 at a spherical
      stage 0 without a clamp, where v = z exactly; the stage input's own bound x_b where there is no l2norm.
    Every bound carries SAFETY = 2 for the neglected second-order terms.  Non-finite inputs have no bound (inf / NaN)."""
    bf = z.dtype == torch.bfloat16
    uw = 2.0 ** -8 if bf else 0.
    ur = U + uw
    eta = 2.0 ** -133 if bf else 2.0 ** -149
    eps = l2norm_eps(bf)
    N, G, d = z.shape
    dev = z.device
    p = params.double().cpu().tolist()
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=dev)
    r = z.double()
    er = torch.zeros_like(r)
    o = eo = None
    bitw = 2 ** torch.arange(d - 1, -1, -1, device=dev)
    idx = torch.full((N, G, Q), -1, dtype=torch.int64, device=dev)
    xs, xbs, sbs, poss, cts, cbs, unsure, saved = [], [], [], [], [], [], [], []
    for q in range(n_active):
        s, m, c = p[0][q], p[1][q], p[2][q]
        x, ex = r, er
        t = et = None
        if c != 0.:
            y = x / c
            ey = ex / abs(c)
            ey = ey + ur * (y.abs() + ey) + eta
            t = torch.tanh(y)
            # tanh is monotone: the image of [y - ey, y + ey], not its first-order slope, which vanishes where the float64
            # value saturates and the computed one need not
            et = torch.maximum((torch.tanh(y + ey) - t).abs(), (torch.tanh(y - ey) - t).abs())
            et = et + (4 * U + ur) * (t.abs() + et) + eta
            x = t * c
            ex = abs(c) * et
            ex = ex + ur * (x.abs() + ex) + eta
        nrm = enrm = proj = yv = None
        sb = None
        if spherical:
            ss = (x * x).sum(-1, keepdim=True)
            ess = gamma(d) * ss + (2 * x.abs() * ex + ex * ex).sum(-1, keepdim=True) + d * 2.0 ** -149
            rn = ss.sqrt()
            ern = torch.minimum(ess.sqrt(), torch.where(rn > 0, ess / rn, inf)) + (U + ur) * rn + eta
            nrm = rn.clamp_min(eps)
            enrm = torch.where(rn + ern < eps, torch.zeros_like(ern), ern)
            proj = rn >= eps
            unsure.append(((rn - eps).abs() <= ern)[..., 0])
            den = torch.where(nrm > enrm, nrm - enrm, torch.zeros_like(nrm))
            yv = x / nrm
            sb = torch.where(den > 0, ex * abs(s) / den, inf) * (1 + 3 * ur) + 2 * eta * max(abs(s), 1.)
            ey = torch.where(den > 0, ex / den + x.abs() * enrm / (nrm * den), inf)
            ey = torch.minimum(ey, yv.abs() + 1)   # a normalised element lies in [-1, 1]
            ey = ey + ur * (yv.abs() + ey) + eta
            x = yv * s
            ex = abs(s) * ey
            ex = ex + ur * (x.abs() + ex) + eta
        pos = (x > 0) if signs is None else signs[q].to(dev).bool()
        qv = torch.where(pos, m, -m).double()
        idx[..., q] = (pos.long() * bitw).sum(-1)
        xs.append(x)
        xbs.append(ex)
        sbs.append(ex if sb is None else torch.minimum(sb.expand_as(ex), ex))
        poss.append(pos)
        e = x - qv
        ee = ex + U * e.abs()
        cts.append((e * e).sum(-1))
        cbs.append(((2 * e.abs() + ee) * ee + U * (e.abs() + ee) ** 2).sum(-1) + gamma(d, 2.0 ** -53) * (e * e).sum(-1))
        if training:
            eov = U * ((qv - x).abs() + ex) + ur * qv.abs() + eta
        else:
            eov = torch.full_like(x, uw * abs(m))
        saved.append((s, c, x, ex, t, et, nrm, enrm, proj, yv, qv, unsure[-1] if spherical else None))
        r = r - qv
        er = er + eov
        er = er + ur * (r.abs() + er) + eta
        if o is None or not residual:
            o, eo = qv, eov
        else:
            o = o + qv
            eo = eo + eov
            eo = eo + ur * (o.abs() + eo) + eta
    grad = grad_b = None
    if gout is not None or gent is not None or cc is not None:
        live = torch.ones(N, dtype=torch.float64, device=dev) if rowmask is None else (rowmask != 0).double()
        live = live[:, None, None]
        acc = torch.zeros_like(r)
        eacc = torch.zeros_like(r)
        sabs = torch.zeros_like(r)
        for q, (s, c, x, ex, t, et, nrm, enrm, proj, yv, qv, uns) in enumerate(saved):
            terms = []
            if training and gout is not None:
                terms.append(gout.double())
            if gent is not None:
                terms.append(gent[q].double())
            ccq = float(cc[q]) if cc is not None else 0.
            if ccq != 0.:
                terms.append(ccq * live * (x - qv))
            gi = sum(terms) if terms else torch.zeros_like(x)
            mag = sum(v.abs() for v in terms) if terms else torch.zeros_like(x)
            eg = abs(ccq) * live * ex + gamma(4) * mag + uw * gi.abs() + eta
            gx, egx = gi, eg
            if spherical:
                g2 = gi * s
                eg2 = abs(s) * eg + ur * g2.abs() + eta
                eyk = ex / abs(s) + U * yv.abs()
                dot = (g2 * yv).sum(-1, keepdim=True)
                edot = (eg2 * yv.abs() + g2.abs() * eyk).sum(-1, keepdim=True) + gamma(d + 1) * (g2 * yv).abs().sum(-1, keepdim=True)
                pterm = yv * dot
                num = torch.where(proj, g2 - pterm, g2)
                enum = torch.where(proj, eg2 + eyk * dot.abs() + yv.abs() * edot + gamma(2) * (g2.abs() + pterm.abs()), eg2)
                enum = enum + torch.where(uns[..., None], pterm.abs(), torch.zeros_like(pterm))
                den = torch.where(nrm > enrm, nrm - enrm, torch.zeros_like(nrm))
                gx = num / nrm
                egx = torch.where(den > 0, enum / den + num.abs() * enrm / (nrm * den), inf) + U * gx.abs() + eta
            if c != 0.:
                tt = 1 - t * t
                ett = (2 * t.abs() + et) * et + U * (t * t + tt.abs())
                g3 = gx * tt
                egx = (egx + gx.abs()) * (tt.abs() + ett) - gx.abs() * tt.abs() + U * g3.abs() + eta
                gx = g3
            egx = egx + uw * gx.abs() + eta
            acc = acc + gx
            eacc = eacc + egx
            sabs = sabs + gx.abs() + egx
        grad = acc
        grad_b = eacc + gamma(n_active - 1) * sabs + uw * (acc.abs() + eacc) + eta
    def fin(b):   # an unbounded operand times a zero (inf * 0) leaves the result unbounded
        return None if b is None else torch.nan_to_num(SAFETY * b, nan=float("inf"))

    return RowRef(torch.stack(xs), fin(torch.stack(xbs)), fin(torch.stack(sbs)), torch.stack(poss), idx, o, fin(eo), torch.stack(cts),
                  fin(torch.stack(cbs)), grad, fin(grad_b),
                  torch.stack(unsure) if spherical else torch.zeros((n_active, N, G), dtype=torch.bool, device=dev))


def item_blocks(N, G, grid, device="cpu"):
    """(N, G) the CTA of vqb_lfq_forward that handles each item: the grid-stride loop gives item it to thread
    it mod (grid * 256)."""
    it = torch.arange(N * G, device=device)
    return ((it % (grid * LFQ_THREADS)) // LFQ_THREADS).view(N, G)


@dataclass
class RowReport:
    """The outcome of `check_rows`: violations (empty when every check held), the rows excused by the sign rule and the
    largest error / bound ratio of each output."""
    violations: list
    excused: int
    first_excused: torch.Tensor   # (N, G) the first stage an item is excused from (n_active: none)
    ratios: dict


def _ratio(err, bound):
    """max err / bound; an error where the bound is 0 counts as inf, 0 / 0 as 0."""
    if err.numel() == 0:
        return 0.
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(r.max())


def check_rows(ref, n_active, idx_t, x_t, idx_k, out_k=None, ent_k=None, commit_k=None, grid=None, rowmask=None, grad_k=None,
               spherical=False, params=None):
    """The sign rule and the bounds of one chain run.

    idx_t / x_t: indices (N, G, Q) and stage inputs (n_active, N, G, d) of the same-dtype torch chain (`chain`), whose
    signs `ref` follows.  idx_k, out_k, ent_k (n_active, N, G, d), commit_k (n_active, grid) per-block partials and grad_k
    (N, G, d): the run under test, any of them None when not produced.

    Sign rule: an index bit may differ from the torch chain's only where that chain's stage input lies within
    delta = 2 sign_b of zero: two computed chains can take different signs only where both lie within sign_b of zero
    (for a spherical chain that is the bound of the value before the l2norm, carried into normalised units: 0 at stage 0
    without a clamp, where every bit must match).  An item is excused from the first stage with such a bit onwards; every
    bit of every other stage must match, and past n_active the index is -1.  The entropy inputs are checked up to and
    including the item's first excused stage (they depend only on earlier stages), the output and the gradient on items
    never excused, and the
    commitment partials block by block, an excused (live) item adding its largest possible term d (|s| + m)^2, for which
    the stage inputs of a spherical chain (|x_j| <= |s|) give the room."""
    viol = []
    N, G, Q = idx_k.shape
    d = ref.x.shape[-1]
    dev = ref.x.device
    sh = torch.arange(d - 1, -1, -1, device=dev)
    past = idx_k[..., n_active:]
    if not bool((past == -1).all()):
        viol.append("index past n_active is not -1")
    bk = (idx_k[..., :n_active].permute(2, 0, 1)[..., None] >> sh) & 1
    bt = (idx_t[..., :n_active].to(dev).permute(2, 0, 1)[..., None] >> sh) & 1
    differ = bk != bt                                                        # (n_active, N, G, d)
    near = x_t.to(dev).double().abs() <= 2 * ref.sign_b
    stage_diff = differ.any(-1)                                              # (n_active, N, G)
    q_of = torch.arange(n_active, device=dev)[:, None, None].expand_as(stage_diff)
    first = torch.where(stage_diff, q_of, torch.full_like(q_of, n_active)).amin(0)   # (N, G)
    at_first = (q_of == first[None]) & stage_diff
    far = (differ & ~near).any(-1) & at_first
    if bool(far.any()):
        n, g = [int(v) for v in far.nonzero()[0, 1:]]
        q = int(first[n, g])
        viol.append(f"index bit differs away from the sign boundary: stage {q} item ({n}, {g}) kernel {int(idx_k[n, g, q])} "
                    f"torch {int(idx_t[n, g, q])} x {x_t[q, n, g].tolist()} delta {(2 * ref.sign_b[q, n, g]).tolist()}")
    if not spherical and bool(stage_diff.any()):
        viol.append("non-spherical chain: an index bit differs from the torch chain")
    ok_stage = q_of < first[None]                                            # (n_active, N, G): checked stages
    clean = first == n_active
    ratios = {}
    if ent_k is not None:
        err = (ent_k.double() - ref.x).abs()
        sel = (q_of <= first[None])[..., None].expand_as(err)
        ratios["ent"] = _ratio(err[sel], ref.x_b[sel])
        if not bool((err[sel] <= ref.x_b[sel]).all()):
            viol.append(f"entropy input outside its bound (ratio {ratios['ent']:.3g})")
    if out_k is not None:
        err = (out_k.double() - ref.out).abs()
        sel = clean[..., None].expand_as(err)
        ratios["out"] = _ratio(err[sel], ref.out_b[sel])
        if not bool((err[sel] <= ref.out_b[sel]).all()):
            viol.append(f"output outside its bound (ratio {ratios['out']:.3g})")
    if commit_k is not None:
        live = torch.ones(N, dtype=torch.bool, device=dev) if rowmask is None else rowmask.to(dev) != 0
        live = live[None, :, None]
        blk = item_blocks(N, G, grid, dev).flatten()
        if spherical:
            p = params.double().cpu()
            slack = (d * (p[0, :n_active].abs() * (1 + 2.0 ** -6) + p[1, :n_active].abs()) ** 2).to(dev)[:, None, None]
        else:
            slack = torch.full((n_active, 1, 1), float("inf"), dtype=torch.float64, device=dev)
        zero = torch.zeros_like(ref.commit)
        val = torch.where(live, ref.commit, zero)
        bnd = torch.where(live, torch.where(ok_stage, ref.commit_b, slack.expand_as(ref.commit_b)), zero)
        sums = torch.zeros((n_active, grid), dtype=torch.float64, device=dev).index_add_(1, blk, val.flatten(1))
        bsum = torch.zeros((n_active, grid), dtype=torch.float64, device=dev).index_add_(1, blk, bnd.flatten(1))
        err = (commit_k.double() - sums).abs()
        ratios["commit"] = _ratio(err, bsum)
        if not bool((err <= bsum).all()):
            viol.append(f"commitment partial outside its bound (ratio {ratios['commit']:.3g})")
    if grad_k is not None:
        err = (grad_k.double() - ref.grad).abs()
        sel = clean[..., None].expand_as(err)
        ratios["grad"] = _ratio(err[sel], ref.grad_b[sel])
        if not bool((err[sel] <= ref.grad_b[sel]).all()):
            bad = ((err > ref.grad_b) & sel).nonzero()[0].tolist()
            viol.append(f"gradient outside its bound at {bad}: {float(grad_k[tuple(bad)])} vs {float(ref.grad[tuple(bad)])} "
                        f"bound {float(ref.grad_b[tuple(bad)])} (ratio {ratios['grad']:.3g})")
    return RowReport(viol, int((~clean).sum()), first, ratios)
