"""Training forward and forward + backward time of LFQ / ResidualLFQ against an eager-torch restatement of the reference's
entropy loss (lookup_free_quantization.py:347-403: the dense (rows, K) distances, softmax and entropies).

    python tools/bench_lfq.py [--seconds 1.0] [--warmup 3]

Configurations: the README LFQ (codebook 65536, dim 16, image (1, 16, 32, 32)); ResidualLFQ(dim=256, codebook_size=1024,
num_quantizers=8) on x (64, 4096, 256); LFQ with codebook 2^18 on 16384 rows.  For each: ms per call (CUDA events), ex2 per
second (two per (row, code) over forward + backward, one in the forward) and the share of the SFU bound (16 ex2 / clock / SM,
the CUDA programming guide's throughput table for compute capability 9.0, at the clock read in the run).  The eager path is
run where its (rows, K) tensors fit in memory and reported as "does not fit" otherwise.  One JSON line; the GPU's name and power
limit read in the same run belong with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_measure import gpu_info, time_ms  # noqa: E402


def eager_entropy(x, scale, tau, gamma=1.):
    """The reference's dense entropy loss on x (rows, c, d): distances, softmax, per-sample and batch entropy."""
    import torch
    d = x.shape[-1]
    k = torch.arange(1 << d, device=x.device)
    mask = 2 ** torch.arange(d - 1, -1, -1, device=x.device)
    codebook = ((k[:, None] & mask) != 0).float() * scale * 2 - scale
    prob = (2 * torch.einsum('...id,jd->...ij', x, codebook) * tau).softmax(-1)
    ent = lambda p: (-p * p.clamp(min=1e-5).log()).sum(-1)
    return ent(prob).mean() - gamma * ent(prob.mean(0)).mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    name, power, clock = gpu_info()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        sfu = 16 * sms * float(clock.split()[0]) * 1e6
    except ValueError:
        sfu = float("nan")
    torch.manual_seed(0)
    cfgs = [
        ("lfq_readme", lambda: vqb.LFQ(codebook_size=65536, dim=16), (1, 16, 32, 32), 1024, 65536, 1, 1.),
        ("rlfq_1024x8", lambda: vqb.ResidualLFQ(dim=256, codebook_size=1024, num_quantizers=8), (64, 4096, 256), 64 * 4096, 1024, 8,
         None),
        ("lfq_d18_16k", lambda: vqb.LFQ(codebook_size=1 << 18), (1, 16384, 18), 16384, 1 << 18, 1, 1.),
    ]
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "sfu_ex2_per_s": sfu, "configs": {}}
    for cname, make, shape, rows, K, stages, scale in cfgs:
        mod = make().cuda().train()
        x = torch.randn(*shape, device="cuda", requires_grad=True)

        def fwd():
            with torch.no_grad():
                mod(x)

        def fwdbwd():
            out = mod(x)
            (out[0].sum() + out[2].sum()).backward()
        r = {}
        ex2 = rows * K * stages
        r["fwd_ms"] = time_ms(fwd, args.seconds, args.warmup)
        r["fwdbwd_ms"] = time_ms(fwdbwd, args.seconds, args.warmup)
        r["fwd_ex2_per_s"] = ex2 / (r["fwd_ms"] * 1e-3)
        r["fwdbwd_ex2_per_s"] = 2 * ex2 / (r["fwdbwd_ms"] * 1e-3)
        r["fwdbwd_share_of_sfu"] = r["fwdbwd_ex2_per_s"] / sfu
        dense_bytes = rows * K * 4 * 6   # the eager stages run one after another
        free = torch.cuda.mem_get_info()[0]
        if scale is not None and dense_bytes < 0.8 * free:
            xe = torch.randn(rows, 1, K.bit_length() - 1, device="cuda", requires_grad=True)
            r["eager_entropy_fwd_ms"] = time_ms(lambda: eager_entropy(xe.detach(), scale, 100.), args.seconds, args.warmup)
            r["eager_entropy_fwdbwd_ms"] = time_ms(lambda: eager_entropy(xe, scale, 100.).backward(), args.seconds, args.warmup)
        elif scale is None and dense_bytes < 0.8 * free:   # ResidualLFQ: the reference's loss per stage, codebook scale 2^-q
            xe = torch.randn(rows, 1, K.bit_length() - 1, device="cuda", requires_grad=True)
            per_stage = lambda f: [f(q) for q in range(stages)]
            r["eager_entropy_fwd_ms"] = time_ms(lambda: per_stage(lambda q: eager_entropy(xe.detach(), 2.0 ** -q, 100.)),
                                                args.seconds, args.warmup)
            r["eager_entropy_fwdbwd_ms"] = time_ms(lambda: sum(per_stage(lambda q: eager_entropy(xe, 2.0 ** -q, 100.))).backward(),
                                                   args.seconds, args.warmup)
        else:
            r["eager"] = f"does not fit: (rows, K) fp32 tensors need about {dense_bytes / 2**30:.1f} GiB"
        res["configs"][cname] = r
        del mod, x
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
