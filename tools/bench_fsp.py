"""Training forward and forward + backward time of FSP against the reference's formula written as eager torch on the same GPU
(oracle/fsp_oracle.py `eager_forward`, with the same projections around it).

    python tools/bench_fsp.py [--seconds 1.0] [--warmup 3]

Configurations: FSP(levels=[8, 5, 5, 5], dim=256, quantize_rate=0.5, vector_norm='kurt') on x (64, 4096, 256), fp32 and a bf16
module under autocast; a projection-free FSP([8, 5, 5, 5]) on 2^24 rows (z of 256 MiB in fp32, beyond L2), fp32.  For each:
ms per call (CUDA events) of the module forward (train) and forward + backward, the eager formula's, and each vqb_fsp kernel
alone; HBM bytes from the shapes (the kernels' reads and writes of the (N, 4) planes) and their share of 3.35 TB/s.  One JSON
line; the GPU's name and power limit read in the same run belong with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_measure import gpu_info, time_ms  # noqa: E402

HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import ops
    from oracle import fsp_oracle as O

    assert torch.cuda.is_available(), "bench_fsp needs a CUDA device"
    name, power, clock = gpu_info()
    dev = "cuda"
    rows = []
    configs = [("proj256_fp32", (64, 4096, 256), 256, torch.float32, False),
               ("proj256_bf16_autocast", (64, 4096, 256), 256, torch.bfloat16, True),
               ("noproj_2^24_fp32", (1, 1 << 24, 4), None, torch.float32, False)]
    for label, shape, dim, dt, amp in configs:
        torch.manual_seed(0)
        m = vqb.FSP(levels=[8, 5, 5, 5], dim=dim, quantize_rate=0.5, vector_norm="kurt").to(dev).train()
        if amp:
            m = m.to(dt)
        x = torch.randn(*shape, device=dev, dtype=dt, requires_grad=True)
        norm = m.vector_norm.norm_args()

        def fwd():
            with torch.no_grad(), torch.autocast("cuda", dtype=dt, enabled=amp):
                return m(x)

        def fwdbwd():
            with torch.autocast("cuda", dtype=dt, enabled=amp):
                q, _, loss, _ = m(x)
            (q.float().sum() + loss).backward()

        def eager(backward):
            def run():
                with torch.autocast("cuda", dtype=dt, enabled=amp):
                    z = m.project_in(x.reshape(-1, shape[-1]))
                    q, _, loss, _, _ = O.eager_forward(z, [8, 5, 5, 5], "tanh", False, 0.5, norm)
                    q = m.project_out(q)
                if backward:
                    (q.float().sum() + loss).backward()
            if backward:
                return run
            return lambda: torch.no_grad()(run)()

        r = dict(config=label, rows=shape[0] * shape[1])
        r["fwd_ms"] = time_ms(fwd, args.seconds, args.warmup)
        r["fwd_bwd_ms"] = time_ms(fwdbwd, args.seconds, args.warmup)
        try:
            r["eager_fwd_ms"] = time_ms(eager(False), args.seconds, args.warmup)
            r["eager_fwd_bwd_ms"] = time_ms(eager(True), args.seconds, args.warmup)
        except torch.OutOfMemoryError:
            r["eager_fwd_ms"] = r["eager_fwd_bwd_ms"] = "does not fit"
        x.grad = None
        # each kernel alone, on the z the module quantizes
        with torch.no_grad(), torch.autocast("cuda", dtype=dt, enabled=amp):
            z = m.project_in(x.reshape(-1, shape[-1])).contiguous()
        N, d = z.shape
        u1, u2 = torch.rand_like(z), torch.rand_like(z)
        eb = z.element_size()
        fw = lambda: ops.fsp_forward(z, 0, False, m._levels, 1 - float(torch.finfo(z.dtype).eps), u1, u2, 0.5, 0., 1.)  # noqa: E731
        st = lambda: ops.fsp_stats(z, norm)  # noqa: E731
        _, _, aux = st()
        g = torch.randn(N, d, device=dev)
        bw = lambda: ops.fsp_backward(z, 0, False, g, aux, None, torch.ones((), device=dev), norm)  # noqa: E731
        kern = {"vqb_fsp_forward": (fw, N * d * (3 * eb + 4 + eb) + 4 * N),   # z, u1, u2 in; q fp32, level indices, index out
                "vqb_fsp_stats": (st, 2 * N * d * eb),                         # z read twice
                "vqb_fsp_backward": (bw, N * d * (eb + 4 + eb))}               # z, g in; dz out
        for k, (fn, nbytes) in kern.items():
            ms = time_ms(fn, args.seconds, args.warmup)
            r[k + "_ms"] = ms
            r[k + "_hbm_share"] = nbytes / (ms * 1e-3) / HBM
        rows.append(r)
        del x, z, u1, u2, g, m
        torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=name, power_limit=power, max_sm_clock=clock, results=rows)))


if __name__ == "__main__":
    main()
