"""Per-role cycle accounting of the search kernel (vq_assign_kernel) on the config-2 workload.

    VQB_PROFILE=1 python -m vector_quantize_pytorch_b200.build --force   # counters are compiled in only then
    python tools/search_roles.py [--json OUT]

Runs the training-mode forward of VectorQuantize(dim=256, codebook_size=1024) on a bf16 batch of (64, 4096, 256) — the
bench.py config-2 step — with the profile buffer armed, and prints each counter as kcycles (mean and max over the CTAs).
Counters (`[grid][16]` int64, one row per CTA, written by the producer lane and by the first thread of consumer warpgroup 0):
  0 producer: waits on b_empty (ring stage free)          1 producer: total
  2 consumer: waits on b_full (ring stage loaded)          3 consumer: total
  4 consumer: issue gap between code steps (last wgmma commit of a step -> first barrier wait of the next one; scan,
    seeding and, once per tile, the row merge)
  5 consumer: waits on a_full (x tile loaded)              6 producer: waits on a_empty (x sub-tile released)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NAMES = {0: "producer b_empty wait", 1: "producer total", 6: "producer a_empty wait",
         2: "consumer b_full wait", 5: "consumer a_full wait", 4: "consumer step gap", 3: "consumer total"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    ap.add_argument("--calls", type=int, default=5, help="forward calls before the profiled one")
    args = ap.parse_args()

    import torch
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import _C

    dev = "cuda:0"
    torch.manual_seed(0)
    vq = vqb.VectorQuantize(dim=256, codebook_size=1024).to(dev)
    with torch.no_grad():
        e = torch.randn(1, 1024, 256, device=dev)
        vq._codebook.embed.copy_(e)
        vq._codebook.embed_avg.copy_(e)
    vq.train()
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(64, 4096, 256, generator=gen).bfloat16().to(dev)

    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros((max(n_sm, 1024), 16), dtype=torch.int64, device=dev)
    for _ in range(args.calls):
        vq(x)
    torch.cuda.synchronize()
    _C.lib.vqb_debug_set_profile_buffer(buf.data_ptr())
    try:
        vq(x)
        torch.cuda.synchronize()
    finally:
        _C.lib.vqb_debug_set_profile_buffer(None)
    rows = buf.cpu()
    rows = rows[rows[:, 1] > 0]   # CTAs that ran (producer total is always > 0 on a profiling build)
    if rows.shape[0] == 0:
        sys.exit("no counters written: build with VQB_PROFILE=1 first")
    out = {"ctas": int(rows.shape[0]), "gpu": torch.cuda.get_device_name(0), "kcycles": {}}
    print(f"{out['gpu']}: {out['ctas']} CTAs, kcycles per CTA")
    print(f"{'counter':<26}{'mean':>10}{'max':>10}")
    for i, name in NAMES.items():
        col = rows[:, i].double() / 1e3
        out["kcycles"][name] = {"mean": round(col.mean().item(), 1), "max": round(col.max().item(), 1)}
        print(f"{name:<26}{col.mean().item():>10.1f}{col.max().item():>10.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
