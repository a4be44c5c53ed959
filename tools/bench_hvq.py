"""HierarchicalVQ eval forward and training forward + backward against the same module with its pool, upsample and residual
update done by eager ATen (F.adaptive_avg_pool2d, F.interpolate, the blend and the adds of hierarchical_vq.py:104-147), so
that only the new kernels differ: the search, the EMA update, expiry and phi's conv are the same calls on both sides.

    python tools/bench_hvq.py [--seconds 1.0] [--warmup 3]

Configurations: the reference's test (dim 32, K 128, scales (1, 2, 4, 7), 7x7, batch 1), and a VAR-like one (dim 32, K 4096,
16x16, scales (1, 2, 3, 4, 5, 6, 8, 10, 13, 16), batch 64), each with quant_resi 0.5 (blended phi) and 0 (identity).  Then
each kernel alone over the VAR-like scales, summed over the scales: its device time from torch.profiler (the mean over
repeated launches, so the host's launch overhead is not counted) and the algorithmic HBM bytes (every operand read once,
every output written once) over that time against the H100's 3.35 TB/s.  One JSON line; the GPU's name, power limit and max
SM clock read in the same run belong with the numbers.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_measure import gpu_info, time_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
CONFIGS = [
    ("reference_test", dict(dim=32, codebook_size=128, scales=(1, 2, 4, 7)), (1, 32, 7, 7)),
    ("var_like", dict(dim=32, codebook_size=4096, scales=(1, 2, 3, 4, 5, 6, 8, 10, 13, 16)), (64, 32, 16, 16)),
]


def eager_forward(hq, x):
    """hvq:128-150 on eager ATen around the same `vq` and phi modules."""
    B, D, H, W = x.shape
    residual, recon, losses, indices = x, torch.zeros_like(x), [], []
    for k, s in enumerate(hq.scales):
        q, ind, loss = hq.vq(F.adaptive_avg_pool2d(residual, (s, s)))
        if q.shape[-2:] != (H, W):
            q = F.interpolate(q, size=(H, W), mode="bilinear", align_corners=False)
        phi = hq._choose_phi(k)
        if phi.resi_ratio > 1e-8:
            q = (1. - phi.resi_ratio) * q + phi.resi_ratio * phi.conv(q)
        recon = recon + q
        residual = residual - q
        losses.append(loss)
        indices.append(ind)
    return recon, tuple(indices), torch.stack(losses).mean()


def module_times(m, kw, shape, quant_resi, seconds, warmup):
    torch.manual_seed(0)
    hq = m.HierarchicalVQ(**kw, quant_resi=quant_resi, accept_image_fmap=True).cuda()
    x = torch.randn(*shape, device="cuda")
    G = torch.randn(*shape, device="cuda")
    hq.train()
    hq(x)   # k-means init

    def train(fwd):
        def step():
            xg = x.clone().requires_grad_(True)
            recon, _, loss = fwd(hq, xg)
            ((recon * G).sum() + loss).backward()
        return step

    out = {}
    out["train_ms"] = time_ms(train(lambda h, v: h(v)), seconds, warmup)
    out["train_eager_ms"] = time_ms(train(eager_forward), seconds, warmup)
    hq.eval()
    with torch.no_grad():
        out["eval_ms"] = time_ms(lambda: hq(x), seconds, warmup)
        out["eval_eager_ms"] = time_ms(lambda: eager_forward(hq, x), seconds, warmup)
        r0 = hq(x)[0]
        r1 = eager_forward(hq, x)[0]
        out["eval_max_abs_diff_vs_eager"] = float((r0 - r1).abs().max())
    out["eval_speedup"] = out["eval_eager_ms"] / out["eval_ms"]
    out["train_speedup"] = out["train_eager_ms"] / out["train_ms"]
    return out


def device_ms(fn, kernel, reps=50):
    """Mean device time in ms of the kernels whose name contains `kernel` over `reps` calls of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    t = [e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and kernel in e.name]
    assert len(t) == reps, (kernel, len(t))
    return sum(t) / len(t) / 1e3


def kernel_times(ops, shape, scales):
    B, D, H, W = shape
    N = B * D * H * W
    x = torch.randn(B, D, H, W, device="cuda")
    recon, resid, conv = torch.randn_like(x), torch.randn_like(x), torch.randn_like(x)
    ga, gb = torch.randn_like(x), torch.randn_like(x)
    acc = {}

    def add(name, ms, nbytes):
        t = acc.setdefault(name, [0.0, 0])
        t[0] += ms
        t[1] += nbytes

    for s in scales:
        R = B * s * s * D
        rows = ops.hvq_pool(x, s)
        g_rows = torch.randn_like(rows)
        add("pool", device_ms(lambda: ops.hvq_pool(x, s), "hvq_pool_kernel"), 4 * (N + R))
        add("pool_backward", device_ms(lambda: ops.hvq_pool_backward(g_rows, H, W), "hvq_pool_bwd_kernel"), 4 * (R + N))
        add("upsample", device_ms(lambda: ops.hvq_upsample(rows, H, W), "hvq_up_kernel"), 4 * (R + N))
        add("upsample_update", device_ms(lambda: ops.hvq_upsample(rows, H, W, recon, resid, want_q=False, want_recon=True,
                                                                  want_resid=True), "hvq_up_kernel"), 4 * (R + 4 * N))
        add("upsample_backward", device_ms(lambda: ops.hvq_upsample_backward(ga, gb, s), "hvq_up_bwd_kernel"),
            4 * (2 * N + R))
        add("blend_update", device_ms(lambda: ops.hvq_blend_update(x, conv, 0.5, recon, resid), "hvq_blend_kernel"), 4 * 6 * N)
        add("blend_backward", device_ms(lambda: ops.hvq_blend_backward(ga, gb, 0.5), "hvq_blend_bwd_kernel"), 4 * 4 * N)
    return {k: dict(ms=ms, hbm_bytes=nb, tb_per_s=nb / (ms * 1e-3) / 1e12, share_of_hbm_peak=nb / (ms * 1e-3) / HBM_BYTES_PER_S)
            for k, (ms, nb) in acc.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hvq needs a CUDA device")
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    name, power, clock = gpu_info()
    res = dict(tool="bench_hvq", gpu=name, power_limit=power, max_sm_clock=clock, configs={})
    for cname, kw, shape in CONFIGS:
        for r in (0.5, 0.0):
            res["configs"][f"{cname}_resi{r}"] = module_times(m, kw, shape, r, a.seconds, a.warmup)
    var = CONFIGS[1]
    res["kernels_var_like"] = kernel_times(ops, var[2], var[1]["scales"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
