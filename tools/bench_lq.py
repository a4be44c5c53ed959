"""A LatentQuantize training step (forward + backward) against an eager-torch restatement of the reference's forward.

    python tools/bench_lq.py [--rounds 7] [--seconds 0.5] [--warmup 5]

Workloads (fp32, training):
  readme    levels [5, 5, 8], dim 16 (projections), x (256, 16, 32, 32)
  noproj    levels [4, 8, 16], dim 9, 3 codebooks (no projection), x (256, 9, 64, 64)
  encoder   levels [8, 8, 8, 6, 5], dim 512 (projections), x (64, 512, 32, 32)
Each round times the module's step and the eager step (the reference's per-latent argmin, gather, straight-through, index sum
and mse losses, latent_quantization.py:148-192, :227-310, with the module's own projections) with CUDA events, alternating the
two; reports the median and range over rounds, each arm's peak memory above the input, and the quantize kernel alone with its
achieved bytes/s from shapes (z read, fp32 codes and int32 indices written).  One JSON line with the GPU's name and power
limit, which belong with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_measure import gpu_info, peak_mib, time_ms  # noqa: E402

WORKLOADS = {
    "readme": (dict(levels=[5, 5, 8], dim=16), (256, 16, 32, 32)),
    "noproj": (dict(levels=[4, 8, 16], dim=9, num_codebooks=3), (256, 9, 64, 64)),
    "encoder": (dict(levels=[8, 8, 8, 6, 5], dim=512), (64, 512, 32, 32)),
}


def eager_forward(m, x):
    """The reference's forward (lq:227-310) in eager torch ops on the module's parameters and buffers."""
    import torch
    import torch.nn.functional as F
    b, d = x.shape[0], x.shape[1]
    z = x.movedim(1, -1).reshape(b, -1, d)
    z = m.project_in(z)
    z = z.reshape(*z.shape[:2], m.num_codebooks, m.codebook_dim)
    vals = m.values_per_latent
    index = torch.stack([torch.argmin(torch.abs(z[..., i, None] - vals[i]), dim=-1) for i in range(m.codebook_dim)], dim=-1)
    q = torch.stack([vals[i][index[..., i]] for i in range(m.codebook_dim)], dim=-1)
    codes = z + (q - z).detach()
    hw = m._levels // 2
    indices = ((codes * 2 * hw + hw) * m._basis).sum(dim=-1).to(torch.int32)
    out = m.project_out(codes.reshape(*codes.shape[:2], -1))
    out = out.reshape(b, *x.shape[2:], d).movedim(-1, 1)
    loss = m.commitment_loss_weight * F.mse_loss(x.detach(), out) + m.quantization_loss_weight * F.mse_loss(out.detach(), x)
    return out, indices, loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import ops

    torch.backends.cuda.matmul.allow_tf32 = False
    name, power, clock = gpu_info()
    res = dict(gpu=name, power_limit=power, max_sm_clock=clock)
    for wl in args.workloads.split(","):
        kw, shape = WORKLOADS[wl]
        torch.manual_seed(0)
        m = vqb.LatentQuantize(**kw).cuda().train()
        x = torch.randn(*shape, device="cuda", requires_grad=True)
        g = torch.randn(*shape, device="cuda")

        def ours():
            out, _, loss = m(x)
            ((out * g).sum() + loss).backward()

        def eager():
            out, _, loss = eager_forward(m, x)
            ((out * g).sum() + loss).backward()

        t_ours, t_eager = [], []
        for _ in range(args.rounds):
            t_ours.append(time_ms(ours, args.seconds, args.warmup, min_iters=3))
            t_eager.append(time_ms(eager, args.seconds, args.warmup, min_iters=3))
        # both arms decide the same indices on the same z
        with torch.no_grad():
            _, i_ours, _ = m(x)
            _, i_eager, _ = eager_forward(m, x)
        agree = float((i_ours.reshape(-1) == i_eager.reshape(-1)).float().mean())
        b, d = shape[0], shape[1]
        with torch.no_grad():
            z = m.project_in(x.movedim(1, -1).reshape(b, -1, d)).reshape(-1, m.effective_codebook_dim).contiguous()
        vals, meta = m._kernel_tables(z.device)
        N, C = z.shape[0], m.num_codebooks
        kq = time_ms(lambda: ops.lq_quantize(z, C, vals, meta), args.seconds, args.warmup, min_iters=10)
        q_bytes = z.numel() * z.element_size() + z.numel() * 4 + N * C * 4
        res[wl] = dict(
            shape=list(shape), kw=kw,
            step_ms_median=statistics.median(t_ours), step_ms_range=[min(t_ours), max(t_ours)],
            eager_step_ms_median=statistics.median(t_eager), eager_step_ms_range=[min(t_eager), max(t_eager)],
            speedup=statistics.median(t_eager) / statistics.median(t_ours),
            peak_mib=peak_mib(ours), eager_peak_mib=peak_mib(eager),
            quantize_kernel_ms=kq, quantize_kernel_bytes=q_bytes, quantize_kernel_gbps=q_bytes / (kq * 1e-3) / 1e9,
            index_agreement=agree)
        x.grad = None
        m.zero_grad(set_to_none=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
