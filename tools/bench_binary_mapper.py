"""Training forward and forward + backward time and peak memory of BinaryMapper against an eager-torch restatement of the
reference's formulas (binary_mapper.py:148-180: the dense one-hot and the (rows, 2^bits) soft codes of its straight-through).

    python tools/bench_binary_mapper.py [--seconds 1.0] [--warmup 3]

Configurations: bits 16 on logits (8, 1024, 16); bits 8 on (64, 4096, 8); bits 20 on (1, 1024, 20).  For each: ms per
training forward and per forward + backward (CUDA events), the peak memory each allocates beyond its inputs, and each
kernel's bytes over its time against the H100's 3.35 TB/s: the forward writes the output (rows * 2^bits * 4 bytes: the memset
and the hot-element kernel), the backward reads the upstream gradient once and writes d logits.  The eager path runs where its
temporaries fit in memory and is reported as "does not fit" otherwise.  One JSON line; the GPU's name, power limit and max SM
clock read in the same run belong with the numbers.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_measure import gpu_info, time_ms, peak_mib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def eager_reference(x, bits, power_two, codes, temperature=1.0, threshold=math.log(2)):
    """The reference's training forward restated in eager torch: the draw, the dense one-hot, the aux loss and the
    straight-through through the dense soft codes exp(logsigmoid(x) @ codes^T + logsigmoid(-x) @ (1 - codes)^T)."""
    import torch
    import torch.nn.functional as F
    prob = (x / temperature).sigmoid()
    idx = (power_two * prob.bernoulli().long()).sum(-1)
    one_hot = F.one_hot(idx, 1 << bits).float()
    p = x.sigmoid()
    entropy = -(p * F.logsigmoid(x) + (1 - p) * F.logsigmoid(-x)).sum(-1)
    aux = F.relu(bits * math.log(2) - entropy - threshold).mean()
    soft = (F.logsigmoid(x) @ codes.t() + F.logsigmoid(-x) @ (1 - codes).t()).exp()
    return one_hot + soft - soft.detach(), aux


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import ops
    name, power, clock = gpu_info()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "hbm_bytes_per_s": HBM_BYTES_PER_S, "configs": {}}
    torch.manual_seed(0)
    for cname, shape in (("bits16_8x1024", (8, 1024, 16)), ("bits8_64x4096", (64, 4096, 8)), ("bits20_1x1024", (1, 1024, 20))):
        bits = shape[-1]
        rows, K = math.prod(shape[:-1]), 1 << bits
        m = vqb.BinaryMapper(bits=bits).cuda().train()
        x = torch.randn(*shape, device="cuda", requires_grad=True)
        G = torch.randn(*shape[:-1], K, device="cuda")
        r = {"rows": rows, "codes": K, "backward_plan": list(ops.binmap_backward_plan(rows, bits, sms))}

        def fwd():
            with torch.no_grad():
                m(x, straight_through=True)

        def fwdbwd():
            out, aux = m(x)
            torch.autograd.backward((out, aux), (G, None))
        r["fwd_ms"] = time_ms(fwd, args.seconds, args.warmup)
        r["fwdbwd_ms"] = time_ms(fwdbwd, args.seconds, args.warmup)
        r["fwdbwd_peak_mib"] = peak_mib(fwdbwd)
        # the kernels alone: the output write (memset + hot element), and the backward's read of g plus d logits
        lf = x.detach().reshape(rows, bits).contiguous()
        idx = torch.randint(0, K, (rows,), device="cuda")
        Gf = G.reshape(rows, K)
        out_bytes = rows * K * 4
        r["fwd_kernel_ms"] = time_ms(lambda: ops.binmap_hot(torch.zeros((rows, K), device="cuda"), lf, idx), args.seconds,
                                     args.warmup)
        r["fwd_kernel_hbm_share"] = out_bytes / (r["fwd_kernel_ms"] * 1e-3) / HBM_BYTES_PER_S
        r["bwd_kernel_ms"] = time_ms(lambda: ops.binmap_backward(lf, Gf), args.seconds, args.warmup)
        r["bwd_kernel_hbm_share"] = (out_bytes + rows * bits * 4) / (r["bwd_kernel_ms"] * 1e-3) / HBM_BYTES_PER_S
        # eager: about nine (rows, K) fp32 temporaries in the forward and as many again in the backward
        xe = x.detach().reshape(rows, bits).clone().requires_grad_(True)
        codes = m.codes.float()
        need = 20 * out_bytes
        if need < 0.8 * torch.cuda.mem_get_info()[0]:
            try:
                def efwd():
                    with torch.no_grad():
                        eager_reference(xe, bits, m.power_two, codes)

                def efwdbwd():
                    out, aux = eager_reference(xe, bits, m.power_two, codes)
                    torch.autograd.backward((out, aux), (Gf, None))
                r["eager_fwd_ms"] = time_ms(efwd, args.seconds, args.warmup)
                r["eager_fwdbwd_ms"] = time_ms(efwdbwd, args.seconds, args.warmup)
                r["eager_fwdbwd_peak_mib"] = peak_mib(efwdbwd)
            except torch.OutOfMemoryError:
                r["eager"] = "does not fit"
        else:
            r["eager"] = f"does not fit: its (rows, 2^bits) fp32 temporaries need about {need / 2**30:.0f} GiB"
        res["configs"][cname] = r
        del m, x, G, Gf, xe
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
