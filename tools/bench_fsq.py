"""Forward and forward + backward time of ResidualFSQ against an eager-torch restatement of the reference's stage loop.

    python tools/bench_fsq.py [--dim 256] [--levels 8,5,5,3] [--stages 8] [--shape 64,4096] [--seconds 1.5] [--warmup 10]

For fp32 and bf16 inputs (a bf16 input runs in a module moved to bf16, as the reference needs for its bf16 projections):
CUDA events around enough calls to fill `seconds` after `warmup` calls.  Reports the module's forward and forward + backward,
the fused forward and backward kernels alone with their algorithmic HBM bytes (z read, out and int32 indices written; z and
d out read, d z written) and the share of 3.35 TB/s, and the same workload as the reference's eager stage loop
(residual_fsq.py:193-241 over finite_scalar_quantization.py:161-169, :220-224, with the same projections).  One JSON line;
the GPU's name and power limit belong with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_measure import gpu_info, time_ms  # noqa: E402

HBM = 3.35e12


def eager_forward(m, x):
    """The reference's loop (rfsq:189-245, fsq:161-169 with the hard clamp, fsq:220-224), eager torch ops."""
    import torch
    lv = m.layers[0]._levels
    basis = m.layers[0]._basis
    x = m.project_in(x)
    c = m.soft_clamp_input_value
    x = (x / c).tanh() * c
    qout, r, idx = 0., x, []
    for scale in m.scales:
        z = (r / scale).float()
        lm1 = lv - 1
        br = (lm1 * (z.clamp(-1., 1.) + 1) / 2.) + 0.5
        br = br + (br.floor() - br).detach()
        code = (2. / lm1) * br - 1.
        idx.append((((code + 1.) / (2. / lm1)) * basis).sum(dim=-1).round().to(torch.int32))
        q = code.to(r.dtype) * scale
        r = r - q.detach()
        qout = qout + q
    return m.project_out(qout), torch.stack(idx, dim=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--levels", default="8,5,5,3")
    ap.add_argument("--stages", type=int, default=8)
    ap.add_argument("--shape", default="64,4096")
    ap.add_argument("--seconds", type=float, default=1.5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import ops

    torch.backends.cuda.matmul.allow_tf32 = False
    levels = [int(v) for v in args.levels.split(",")]
    b, n = (int(v) for v in args.shape.split(","))
    d, Q = len(levels), args.stages
    name, power, clock = gpu_info()
    res = dict(gpu=name, power_limit=power, max_sm_clock=clock, dim=args.dim, levels=levels, stages=Q, shape=[b, n, args.dim])

    def ms(fn):
        return time_ms(fn, args.seconds, args.warmup, min_iters=10)

    for dt_name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        torch.manual_seed(0)
        m = vqb.ResidualFSQ(dim=args.dim, levels=levels, num_quantizers=Q).to("cuda", dt).train()
        x = torch.randn(b, n, args.dim, device="cuda", dtype=dt, requires_grad=True)
        g = torch.randn(b, n, args.dim, device="cuda", dtype=dt)

        def fwd():
            with torch.no_grad():
                m(x)

        def fwd_bwd():
            q, _ = m(x)
            q.backward(g)

        def eager_fwd():
            with torch.no_grad():
                eager_forward(m, x)

        def eager_fwd_bwd():
            q, _ = eager_forward(m, x)
            q.backward(g)

        # the fused kernels alone, on the module's own rows
        N = b * n
        with torch.no_grad():
            z = m.project_in(x).reshape(N, 1, d).contiguous()
        consts, _, scales, clampv = m._tables(z.device)
        work = m._chain_dtype(z.dtype)
        idx = torch.empty((N, Q), dtype=torch.int32, device="cuda")
        gout = torch.randn(N, 1, d, device="cuda").to(work)
        hard = m.layers[0].bound_hard_clamp

        def kern_fwd():
            ops.fsq_forward(z, work, Q, Q, True, hard, consts, scales, clampv, idx.view(N, 1, Q))

        def kern_bwd():
            ops.fsq_backward(z, gout, Q, Q, True, hard, consts, scales, clampv)

        ez = z.element_size()
        ew = torch.empty((), dtype=work).element_size()
        fwd_bytes = N * d * ez + N * d * ew + N * Q * 4
        bwd_bytes = N * d * ez + N * d * ew + N * d * ez
        kf, kb = ms(kern_fwd), ms(kern_bwd)
        res[dt_name] = dict(
            forward_ms=ms(fwd), forward_backward_ms=ms(fwd_bwd),
            eager_forward_ms=ms(eager_fwd),
            eager_forward_backward_ms=ms(eager_fwd_bwd),
            kernel_forward_ms=kf, kernel_forward_bytes=fwd_bytes, kernel_forward_hbm_share=fwd_bytes / (kf * 1e-3) / HBM,
            kernel_backward_ms=kb, kernel_backward_bytes=bwd_bytes, kernel_backward_hbm_share=bwd_bytes / (kb * 1e-3) / HBM)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
