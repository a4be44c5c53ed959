"""Peak device memory of the benchmark steps, and the memory a ResidualVQ holds with a training and an eval program cached.

    python tools/peak_memory.py [--steps 5]

torch.cuda.max_memory_allocated() from the module's creation over 2 x `steps` training forwards, above what was allocated
before (the input), of
- cfg2: VectorQuantize(dim=256, codebook_size=1024), x (64, 4096, 256) bf16 (bench.py's default workload);
- cfg5: GroupedResidualVQ(dim=256, groups=2, num_quantizers=8, codebook_size=1024), x (64, 4096, 256) fp32 (bench.py --workload
  cfg5);
- rvq_shared_train_eval: ResidualVQ(dim=256, num_quantizers=8, codebook_size=1024, shared_codebook=True), x (32, 8192, 256)
  fp32: one training and one eval forward (two cached programs), the peak, and the memory still allocated for the module once
  its outputs are gone (`held_bytes`: buffers, plans and their scratch).
Prints one JSON line with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_measure import gpu_info  # noqa: E402


def measure(make, x, schedule):
    """(peak bytes over the forwards of `schedule` (training flags), bytes still allocated for the module afterwards), both
    above what was allocated before the module was made (the input, and anything an earlier workload left behind)."""
    import torch
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    mod = make()
    with torch.no_grad():
        for training in schedule:
            mod.train(training)
            out = mod(x)
            del out
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    held = torch.cuda.memory_allocated() - base
    del mod
    gc.collect()
    return peak, held


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import vector_quantize_pytorch_b200 as vqb
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(1234)
    steps = [True] * (2 * args.steps)
    res = {}
    x = torch.randn(64, 4096, 256, device=dev).bfloat16()
    res["cfg2_peak_bytes"], _ = measure(lambda: vqb.VectorQuantize(dim=256, codebook_size=1024).to(dev), x, steps)
    x = torch.randn(64, 4096, 256, device=dev)
    res["cfg5_peak_bytes"], _ = measure(
        lambda: vqb.GroupedResidualVQ(dim=256, groups=2, num_quantizers=8, codebook_size=1024).to(dev), x, steps)
    x = torch.randn(32, 8192, 256, device=dev)
    res["rvq_shared_train_eval_peak_bytes"], res["rvq_shared_train_eval_held_bytes"] = measure(
        lambda: vqb.ResidualVQ(dim=256, num_quantizers=8, codebook_size=1024, shared_codebook=True).to(dev), x, [True, False])
    gpu, power, clock = gpu_info()
    res.update(gpu=gpu, power_limit=power, max_sm_clock=clock, steps=args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
