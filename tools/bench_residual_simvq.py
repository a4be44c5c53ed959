"""Forward and forward + backward time of ResidualSimVQ against an eager-torch restatement of the reference's stage loop.

    python tools/bench_residual_simvq.py [--dim 512] [--stages 4] [--codes 1024] [--rows 65536] [--iters 20] [--warmup 5]

fp32 with TF32 off (the reference's only dtype), CUDA events around `iters` calls after `warmup` calls of the same shape.  The
eager arm is residual_sim_vq.py:182-203 over sim_vq.py:100-138 as the reference writes it: per stage torch.cdist + argmin, the
gather, two mse terms, the rotation trick (or straight-through), the residual update and the running sum; autograd for the
backward.  Prints one JSON line with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_measure import gpu_info, time_ms  # noqa: E402


def rotate_to(src, tgt):   # vector_quantize_pytorch.py:287-318
    ns, nt = src.norm(dim=-1, keepdim=True), tgt.norm(dim=-1, keepdim=True)
    u, q = src / ns.clamp(min=1e-6), tgt / nt.clamp(min=1e-6)
    w = (u + q) / (u + q).norm(dim=-1, keepdim=True).clamp(min=1e-6)
    w = w.detach()
    out = src - 2 * (src * w).sum(-1, keepdim=True) * w + 2 * (src * u.detach()).sum(-1, keepdim=True) * q.detach()
    return out * (nt / ns.clamp(min=1e-6)).detach()


def eager_forward(layers, x, rotation):
    """The reference's loop with the same layers (their code_transform and frozen codebooks)."""
    import torch
    import torch.nn.functional as F
    r, qout, losses, idx = x, 0., [], []
    for layer in layers:
        books = layer.code_transform(layer.frozen_codebook)
        with torch.no_grad():
            ind = torch.cdist(r, books).argmin(dim=-1)
        c = books[ind]
        losses.append((F.mse_loss(r.detach(), c) + F.mse_loss(r, c.detach()) * 0.25) * 1.)
        out = rotate_to(r, c) if rotation else (c - r).detach() + r
        r = r - out.detach()
        qout = qout + out
        idx.append(ind)
    return qout, torch.stack(idx, -1), torch.stack(losses)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--stages", type=int, default=4)
    ap.add_argument("--codes", type=int, default=1024)
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ste", action="store_true", help="straight-through estimator instead of the rotation trick")
    args = ap.parse_args()

    import torch
    import vector_quantize_pytorch_b200 as vqb
    if not torch.cuda.is_available():
        raise SystemExit("bench_residual_simvq needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda:0"
    torch.manual_seed(0)
    rotation = not args.ste
    mod = vqb.ResidualSimVQ(dim=args.dim, num_quantizers=args.stages, codebook_size=args.codes, rotation_trick=rotation).to(dev).train()
    x = torch.randn(8, args.rows // 8, args.dim, device=dev)
    G = torch.randn_like(x)
    flat_x, flat_g = x.reshape(-1, args.dim), G.reshape(-1, args.dim)

    def ours_fwd():
        with torch.no_grad():
            mod(x)

    def ours_fwd_bwd():
        xr = x.detach().requires_grad_(True)
        q, _, losses = mod(xr)
        ((q * G).sum() + losses.sum()).backward()

    def eager_fwd():
        with torch.no_grad():
            eager_forward(mod.layers, flat_x, rotation)

    def eager_fwd_bwd():
        xr = flat_x.detach().requires_grad_(True)
        q, _, losses = eager_forward(mod.layers, xr, rotation)
        ((q * flat_g).sum() + losses.sum()).backward()

    # same indices on both arms (up to near ties) before timing anything
    with torch.no_grad():
        _, i_ours, _ = mod(x)
        _, i_eager, _ = eager_forward(mod.layers, flat_x, rotation)
    agree = (i_ours.reshape(-1, args.stages) == i_eager).float().mean().item()

    res = {}
    for name, fn in (("ours_fwd_ms", ours_fwd), ("eager_fwd_ms", eager_fwd), ("ours_fwd_bwd_ms", ours_fwd_bwd),
                     ("eager_fwd_bwd_ms", eager_fwd_bwd)):
        res[name] = round(time_ms(fn, None, args.warmup, iters=args.iters), 3)
    gpu, power, clock = gpu_info()
    res.update(gpu=gpu, power_limit=power, max_sm_clock=clock, dim=args.dim, stages=args.stages, codes=args.codes, rows=args.rows,
               rotation_trick=rotation, index_agreement=round(agree, 6),
               fwd_speedup=round(res["eager_fwd_ms"] / res["ours_fwd_ms"], 2),
               fwd_bwd_speedup=round(res["eager_fwd_bwd_ms"] / res["ours_fwd_bwd_ms"], 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
