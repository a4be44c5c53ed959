"""Time one training step — forward, backward, optimizer.step — of a codebook learnt by gradient, against an eager-torch
restatement of the reference's step (vector_quantize_pytorch.py:674-791, :1212-1237, :1327; residual_vq.py:469-606), with CUDA
events after warm-up.  Prints the card's name, power limit and maximum SM clock with the numbers (one JSON line per step kind).

    python tools/bench_learnable.py [--steps 10] [--warmup 3]

    A: VectorQuantize(256, 1024, learnable_codebook=True, ema_update=False), x (64, 4096, 256) bf16 requiring grad
    B: ResidualVQ(256, 8 quantizers, 1024, learnable_codebook=True, ema_update=False), x (32, 8192, 256) fp32 requiring grad
    C: VectorQuantize DiVeQ (directional_reparam=True, threshold_ema_dead_code=2) on A's shapes
"""
import argparse
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vector_quantize_pytorch_b200 as vqb  # noqa: E402
from gpu_measure import gpu_info, time_ms  # noqa: E402

DEV = "cuda"


# ---------------------------------------------------------------- eager restatement of the reference's step
def cdist(x, y, eps=1e-8):   # vqp:58-62
    x2 = (x ** 2).sum(-1)
    y2 = (y ** 2).sum(-1)
    return (x2[:, None] + y2[None, :] - 2 * x @ y.t()).clamp(min=eps).sqrt()


def rotate_to(src, tgt):   # vqp:287-318
    def sdiv(a, b):
        return a / b.clamp(min=1e-6)
    ns, nt = src.norm(dim=-1, keepdim=True), tgt.norm(dim=-1, keepdim=True)
    u, q, e = sdiv(src, ns), sdiv(tgt, nt), src
    w = F.normalize(u + q, dim=-1, eps=1e-6).detach()
    out = e - 2 * (e * w).sum(-1, keepdim=True) * w + 2 * (e * u.detach()).sum(-1, keepdim=True) * q.detach()
    return out * sdiv(nt, ns).detach()


def directional_reparam(src, tgt, var=5e-3):   # vqp:323-330
    e = tgt - src
    u = F.normalize(e + math.sqrt(var) * torch.randn_like(e), dim=-1, eps=1e-6).detach()
    return src + u * e.norm(dim=-1, keepdim=True)


class EagerVQ(torch.nn.Module):
    def __init__(self, embed, diveq=False, decay=0.8, threshold=2):
        super().__init__()
        K = embed.shape[0]
        self.embed = torch.nn.Parameter(embed.clone())
        self.register_buffer("cluster_size", torch.ones(K, device=embed.device))
        self.register_buffer("embed_avg", embed.clone())
        self.diveq, self.decay, self.threshold = diveq, decay, threshold

    def forward(self, x):
        flat = x.reshape(-1, x.shape[-1])
        f32 = flat.float()
        idx = (-cdist(f32.detach(), self.embed.detach())).argmax(-1)
        onehot = F.one_hot(idx, self.embed.shape[0]).float()
        quantize = (onehot @ self.embed).type(x.dtype)                      # vqp:766, :1178
        if self.diveq:   # update_codebook without EMA: lerp of the statistics, dead-code expiry (vqp:586-641)
            with torch.no_grad():
                self.cluster_size.lerp_(onehot.sum(0), 1 - self.decay)
                self.embed_avg.lerp_(onehot.t() @ f32, 1 - self.decay)
                expired = self.cluster_size < self.threshold
                if torch.any(expired):
                    n = int(expired.sum().item())
                    self.embed.data[expired] = f32[torch.randperm(f32.shape[0], device=x.device)[:n]]
            return directional_reparam(flat, quantize).reshape(x.shape), torch.zeros((), device=x.device)
        loss = F.mse_loss(quantize, flat)                                    # vqp:1327 (commitment weight 1)
        return rotate_to(flat, quantize).reshape(x.shape), loss


class EagerRVQ(torch.nn.Module):
    def __init__(self, embeds):
        super().__init__()
        self.layers = torch.nn.ModuleList([EagerVQ(e) for e in embeds])

    def forward(self, x):
        residual, out, losses = x, torch.zeros_like(x), []
        for layer in self.layers:
            q, loss = layer(residual)
            residual = residual - q.detach()
            out = out + q
            losses.append(loss)
        return out, torch.stack(losses)


# ---------------------------------------------------------------- timing
def make_step(mod, x, G, fwd):
    opt = torch.optim.SGD(mod.parameters(), lr=1e-3)

    def step():
        opt.zero_grad(set_to_none=True)
        out, loss = fwd(mod, x)
        ((out.float() * G).sum() + loss.sum()).backward()
        opt.step()
    return step


def ours_fwd(mod, x):
    out, _, loss = mod(x)
    return out, loss


def eager_fwd(mod, x):
    return mod(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_learnable: needs a CUDA device")
    torch.manual_seed(0)
    gpu = ", ".join(gpu_info())
    cases = []
    D, K = 256, 1024
    xa = torch.randn(64, 4096, D, device=DEV).bfloat16().requires_grad_(True)
    Ga = torch.randn(64, 4096, D, device=DEV)
    a = vqb.VectorQuantize(dim=D, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV).train()
    cases.append(("A_vq_bf16", a, EagerVQ(a._codebook.embed.detach()[0]), xa, Ga))
    xb = torch.randn(32, 8192, D, device=DEV).requires_grad_(True)
    Gb = torch.randn(32, 8192, D, device=DEV)
    b = vqb.ResidualVQ(dim=D, num_quantizers=8, codebook_size=K, learnable_codebook=True, ema_update=False).to(DEV).train()
    cases.append(("B_rvq8_fp32", b, EagerRVQ([layer._codebook.embed.detach()[0] for layer in b.layers]), xb, Gb))
    c = vqb.VectorQuantize(dim=D, codebook_size=K, directional_reparam=True, threshold_ema_dead_code=2).to(DEV).train()
    cases.append(("C_diveq_bf16", c, EagerVQ(c._codebook.embed.detach()[0], diveq=True), xa, Ga))
    for name, ours, eager, x, G in cases:
        eager = eager.to(DEV).train()
        t_ours = time_ms(make_step(ours, x, G, ours_fwd), None, args.warmup, iters=args.steps)
        t_eager = time_ms(make_step(eager, x, G, eager_fwd), None, args.warmup, iters=args.steps)
        print(json.dumps({"case": name, "rows": x.numel() // D, "ms_per_step": round(t_ours, 3), "eager_ms_per_step": round(t_eager, 3),
                          "speedup": round(t_eager / t_ours, 2), "gpu": gpu}), flush=True)
        del eager
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
