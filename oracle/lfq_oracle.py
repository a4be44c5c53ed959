"""Float64 dense restatement of the LFQ entropy loss (lookup_free_quantization.py:347-403 of the reference) and of its
factorised form (DESIGN §4.10).  TEST INFRASTRUCTURE ONLY: torch float64 on whichever device the inputs live on.

`dense_stats` builds the (rows, K) probabilities: the definition.  `factored_stats` uses ln p[k] = sum_j l_j(bit_j(k)) with
l_j(1) = -softplus(-2 a_j), l_j(0) = -softplus(2 a_j), a_j = 2 tau m x_j: what the kernels compute.  Gradients come from
float64 autograd through the dense form.
"""
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
