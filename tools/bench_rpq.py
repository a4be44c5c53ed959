"""RandomProjectionQuantizer: the fused forward (vqb_rpq_norm_project, then project_in and the search) against the eager
composition a user would otherwise write (nn.LayerNorm, torch.einsum with `rand_projs`, then the same VectorQuantize in eval),
and the layer-norm + projection prologue alone on both sides.

    python tools/bench_rpq.py [--seconds 1.0] [--warmup 3] [--frames 262144]

Configurations: BEST-RQ-like (dim 320, one codebook of 8192 16-wide codes) and USM-like (dim 512, 16 codebooks of 1024
codes, codebook_dim 16), each over --frames frames (64 sequences).  Times are CUDA-event means per call.  The prologue
kernel's device time comes from torch.profiler in a separate pass; its algorithmic bytes (x read once, the rows written
once, the projection read once) and FLOP (2 N dim H E) over that time are set against the H100 SXM data sheet's 3.35 TB/s
and 67 TFLOP/s FP32, and the larger of the two lower bounds names what limits it.  One JSON line; the GPU's name, power limit
and max SM clock read in the same run belong with the numbers.
"""
import argparse
import json
import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_measure import gpu_info, time_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP32_FLOP_PER_S = 67e12
CONFIGS = [
    ("bestrq_like", dict(dim=320, codebook_size=8192, codebook_dim=16)),
    ("usm_like", dict(dim=512, codebook_size=1024, codebook_dim=16, num_codebooks=16)),
]


def eager_prologue(ln, rand_projs, x):
    b, n, _ = x.shape
    return torch.einsum("b n d, h d e -> b n h e", ln(x), rand_projs).reshape(b, n, -1)


def kernel_ms(fn, name, reps=10):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    times = [e.device_time_total for e in prof.events() if name in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    assert times, f"no {name} in the trace"
    return sum(times) / len(times) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=1 << 18)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rpq measures on a CUDA device"
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    name, power, clock = gpu_info()
    out = dict(gpu=name, power_limit=power, max_sm_clock=clock, frames=args.frames, tf32=torch.backends.cuda.matmul.allow_tf32)
    B = 64
    n = args.frames // B
    for cname, kw in CONFIGS:
        torch.manual_seed(0)
        rpq = m.RandomProjectionQuantizer(**kw).to("cuda")
        ln = nn.LayerNorm(kw["dim"], elementwise_affine=False).to("cuda")
        x = torch.randn(B, n, kw["dim"], device="cuda")
        H, dim, E = rpq.rand_projs.shape

        def eager():
            rpq.vq.eval()
            return rpq.vq(eager_prologue(ln, rpq.rand_projs, x))[1]

        with torch.no_grad():
            same = bool((rpq(x) == eager()).float().mean() > 0.999)   # the two paths round differently only near ties
            r = dict(fused_ms=time_ms(lambda: rpq(x), args.seconds, args.warmup),
                     eager_ms=time_ms(eager, args.seconds, args.warmup),
                     prologue_fused_ms=time_ms(lambda: ops.rpq_norm_project(x, rpq.rand_projs, True), args.seconds, args.warmup),
                     prologue_eager_ms=time_ms(lambda: eager_prologue(ln, rpq.rand_projs, x), args.seconds, args.warmup),
                     indices_agree=same)
            k = kernel_ms(lambda: ops.rpq_norm_project(x, rpq.rand_projs, True), "rpq_norm_project_kernel")
        N = B * n
        nbytes = 4 * (N * dim + N * H * E + H * dim * E)
        flop = 2 * N * dim * H * E
        t_hbm, t_fp32 = nbytes / HBM_BYTES_PER_S, flop / FP32_FLOP_PER_S
        r.update(kernel_ms=k, kernel_bytes=nbytes, kernel_flop=flop, kernel_bound="hbm" if t_hbm >= t_fp32 else "fp32",
                 kernel_share_of_bound=max(t_hbm, t_fp32) / (k / 1e3), kernel_gb_s=nbytes / (k / 1e3) / 1e9,
                 kernel_tflop_s=flop / (k / 1e3) / 1e12)
        out[cname] = r
        del rpq, x
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
