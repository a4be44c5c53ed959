"""Time one masked training step — forward and backward, input requiring grad — against the same step without a mask, with
CUDA events after warm-up.  Prints the card's name, power limit and maximum SM clock with the numbers (one JSON line per case).

    python tools/bench_masked_train.py [--steps 50] [--warmup 3] [--repeats 7]

    VectorQuantize(256, 1024), x (64, 4096, 256) bf16 (BASELINE config 2): 0 %, 10 % and 50 % padding rows, each sequence
        padded at its end; the Euclidean codebook takes the in-kernel mask and vqb_rotate_masked (no host sync)
    ResidualVQ(256, 8 quantizers, 1024, shared codebook), x (32, 8192, 256) fp32 (BASELINE config 3) at 10 % padding: the
        layered path on the gathered live rows
The unmasked step of the same module and input is timed alongside each case, alternating with the masked one `--repeats`
times (each timing a mean over `--steps` steps); the median and the range over the repeats are printed.  The two steps do not
compute the same forward: a masked step returns the searched codes on live rows, the unmasked one the estimator's value
rotate_to(x, q), and the unmasked step with gradients takes its loss and estimator value through PyTorch glue.
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import vector_quantize_pytorch_b200 as vqb  # noqa: E402
from gpu_measure import gpu_info, time_ms  # noqa: E402

DEV = "cuda"


def padded_mask(B, N, frac, gen):
    """(B, N) mask whose sequences end in padding: lengths uniform around N (1 - frac), mean padding fraction `frac`."""
    if frac == 0:
        return torch.ones(B, N, dtype=torch.bool, device=DEV)
    lo, hi = max(0, int(N * (1 - 2 * frac))), N
    lens = torch.randint(lo, hi + 1, (B,), generator=gen, device=DEV)
    return torch.arange(N, device=DEV) < lens[:, None]


def make_step(mod, x, G, mask):
    def step():
        xr = x.detach().requires_grad_(True)
        out, _, loss = mod(xr, mask=mask) if mask is not None else mod(xr)
        ((out.float() * G).sum() + loss.float().sum()).backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_masked_train: needs a CUDA device")
    torch.manual_seed(0)
    gen = torch.Generator(device=DEV).manual_seed(0)
    gpu = ", ".join(gpu_info())
    D, K = 256, 1024
    cases = []
    vq = vqb.VectorQuantize(dim=D, codebook_size=K).to(DEV).train()
    xa = torch.randn(64, 4096, D, device=DEV).bfloat16()
    Ga = torch.randn(64, 4096, D, device=DEV)
    for frac in (0.0, 0.1, 0.5):
        cases.append((f"vq_bf16_pad{int(frac * 100)}", vq, xa, Ga, padded_mask(64, 4096, frac, gen)))
    rvq = vqb.ResidualVQ(dim=D, num_quantizers=8, codebook_size=K, shared_codebook=True).to(DEV).train()
    xb = torch.randn(32, 8192, D, device=DEV)
    Gb = torch.randn(32, 8192, D, device=DEV)
    cases.append(("rvq8_fp32_pad10", rvq, xb, Gb, padded_mask(32, 8192, 0.1, gen)))
    for name, mod, x, G, mask in cases:
        masked, plain = make_step(mod, x, G, mask), make_step(mod, x, G, None)
        t = {"masked": [], "unmasked": []}
        for r in range(args.repeats):   # alternated, so that drift on a shared host hits both alike
            warm = args.warmup if r == 0 else 1
            t["masked"].append(time_ms(masked, None, warm, iters=args.steps))
            t["unmasked"].append(time_ms(plain, None, warm, iters=args.steps))
        line = {"case": name, "rows": x.numel() // D, "live_fraction": round(float(mask.float().mean()), 4),
                "steps": args.steps, "repeats": args.repeats}
        for k, v in t.items():
            line[f"{k}_ms_median"] = round(statistics.median(v), 3)
            line[f"{k}_ms_range"] = [round(min(v), 3), round(max(v), 3)]
        line["gpu"] = gpu
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
