"""Generate tests/golden/lfq/*.npz by running the UNMODIFIED reference's LFQ / ResidualLFQ / GroupedResidualLFQ on CPU (TEST
INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_lfq.py

Per case: the constructor kwargs and the construction seed, the state_dict, x, an upstream gradient G, the forward seed, one
forward (train or eval) with its outputs, the loss breakdown (LFQ) and the gradient of sum(out * G) + sum(losses) w.r.t. x.
It also keeps z, the project_in output of every (Residual)LFQ, the gradient there, and q, the project_out input, so the
kernels can be checked on the rows the reference quantized (the projections are torch matmuls, whose summation order differs
between devices).  The same forward and backward are then repeated in float64 (the module and x in double,
force_quantization_f32 off so nothing is rounded to fp32): its losses and gradients at z are stored as `losses64` / `gz64_j`,
and the fp32 reference's own deviation from them sets the tolerance of the replay.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "lfq")

# (name, class, kwargs, x shape, x dtype, train, forward kwargs, x scale, mask kind)
CASES = [
    ("lfq_readme_image", "LFQ", dict(codebook_size=65536, dim=16), (1, 16, 8, 8), "fp32", True, dict(inv_temperature=100.), 1.0, None),
    ("lfq_proj_c4", "LFQ", dict(codebook_size=4096, dim=16, num_codebooks=4), (2, 24, 16), "fp32", True, {}, 1.0, None),
    ("lfq_spherical", "LFQ", dict(codebook_size=1024, spherical=True, codebook_scale=1.5), (2, 32, 10), "fp32", True, {}, 1.0, None),
    ("lfq_softclamp_softplus_commit", "LFQ", dict(codebook_size=256, soft_clamp_input_value=2.0, experimental_softplus_entropy_loss=True,
                                                  commitment_loss_weight=0.25), (2, 32, 8), "fp32", True, {}, 3.0, None),
    ("lfq_mask", "LFQ", dict(codebook_size=512, num_codebooks=2, commitment_loss_weight=0.1), (2, 20, 18), "fp32", True, {}, 1.0, "mask"),
    ("lfq_frac", "LFQ", dict(codebook_size=256, frac_per_sample_entropy=0.5), (2, 32, 8), "fp32", True, {}, 1.0, None),
    ("lfq_frac_mask", "LFQ", dict(codebook_size=256, num_codebooks=2, frac_per_sample_entropy=0.5), (2, 20, 16), "fp32", True, {}, 1.0,
     "mask"),
    ("lfq_eval", "LFQ", dict(codebook_size=4096, dim=32), (2, 16, 32), "fp32", False, {}, 1.0, None),
    ("lfq_bf16", "LFQ", dict(codebook_size=1024), (2, 32, 10), "bf16", True, {}, 1.0, None),
    ("lfq_rot_cosine", "LFQ", dict(codebook_size=256, dim=32, orthogonal_rotation=True, cosine_sim_project_in=True,
                                   soft_clamp_input_value=1.5), (2, 16, 32), "fp32", True, {}, 1.0, None),
    ("lfq_flat_d16", "LFQ", dict(codebook_size=65536), (1, 24, 16), "fp32", True, dict(inv_temperature=1e-3), 1.0, None),
    ("lfq_flat_d17", "LFQ", dict(codebook_size=131072), (1, 16, 17), "fp32", True, dict(inv_temperature=1e-3), 1.0, None),
    ("rlfq_readme_train", "ResidualLFQ", dict(dim=256, codebook_size=256, num_quantizers=8), (2, 32, 256), "fp32", True, {}, 1.0, None),
    ("rlfq_readme_eval", "ResidualLFQ", dict(dim=256, codebook_size=256, num_quantizers=8), (2, 32, 256), "fp32", False, {}, 1.0, None),
    ("rlfq_dropout_clamp_mask", "ResidualLFQ", dict(dim=64, codebook_size=256, num_quantizers=6, quantize_dropout=True,
                                                    soft_clamp_input_value=4.0, commitment_loss_weight=0.2),
     (2, 24, 64), "fp32", True, dict(rand_quantize_dropout_fixed_seed=7), 1.0, "mask"),
    ("rlfq_frac", "ResidualLFQ", dict(dim=32, codebook_size=1024, num_quantizers=3, frac_per_sample_entropy=0.5), (2, 24, 32), "fp32",
     True, {}, 1.0, None),
    ("grlfq_frac_mask", "GroupedResidualLFQ", dict(dim=32, groups=2, codebook_size=256, num_quantizers=3, frac_per_sample_entropy=0.5,
                                                          diversity_gamma=0.5),
     (2, 24, 32), "fp32", True, {}, 1.0, "mask"),
    ("grlfq_groups2", "GroupedResidualLFQ", dict(dim=64, groups=2, codebook_size=512, num_quantizers=4), (2, 24, 64), "fp32", True, {},
     1.0, None),
]


def to_np(t):
    if t.dtype == torch.bfloat16:
        return t.float().numpy()
    return t.detach().numpy()


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, cls, kwargs, shape, xdt, train, fkw, scale, mkind) in enumerate(CASES):
        seed = 1000 + i
        torch.manual_seed(seed)
        mod = getattr(ref, cls)(**kwargs)
        mod.train(train)
        sd = {k: v.clone() for k, v in mod.state_dict().items()}
        g = torch.Generator().manual_seed(seed + 1)
        x = (torch.randn(*shape, generator=g) * scale)
        if xdt == "bf16":
            x = x.bfloat16()
        x.requires_grad_(True)
        mask = None
        if mkind == "mask":
            mask = torch.rand(shape[0], shape[1], generator=g) > 0.3
            fkw = dict(fkw, mask=mask)
        # z and its gradient at every project_in
        fwd_seed = seed + 2
        G = None

        def run(mod, x):
            zs, qs = [], []

            def hook(_m, _inp, out):
                out.retain_grad()
                zs.append(out)
            if cls == "GroupedResidualLFQ":
                pis, pos = [r.project_in for r in mod.rvqs], [r.project_out for r in mod.rvqs]
            else:
                pis, pos = [mod.project_in], [mod.project_out]
            hs = [p.register_forward_hook(hook) for p in pis]
            hs += [p.register_forward_pre_hook(lambda _m, inp: qs.append(inp[0].detach().clone())) for p in pos]
            torch.manual_seed(fwd_seed)
            if cls == "LFQ":
                (out, idx, aux), bd = mod(x, return_loss_breakdown=True, **fkw)
                losses = aux
            else:
                out, idx, losses = mod(x, **fkw)
                bd = None
            for h in hs:
                h.remove()
            return out, idx, losses, bd, zs, qs

        out, idx, losses, bd, zs, qs = run(mod, x)
        G = torch.randn(out.shape, generator=g).to(out.dtype)
        total = (out.float() * G.float()).sum() + (losses.float().sum() if train else 0.)
        total.backward()
        # the same step in float64
        torch.manual_seed(seed)
        mod64 = getattr(ref, cls)(**kwargs)
        mod64.load_state_dict(sd)
        mod64 = mod64.double().train(train)
        for sub in mod64.modules():
            if hasattr(sub, "force_quantization_f32"):
                sub.force_quantization_f32 = False
        x64 = x.detach().double().requires_grad_(True)
        out64, _, losses64, _, zs64, _ = run(mod64, x64)
        total64 = (out64 * G.double()).sum() + (losses64.sum() if train else 0.)
        total64.backward()
        rec = dict(kwargs=np.array(json.dumps(kwargs)), cls=np.array(cls), seed=np.array(seed), fwd_seed=np.array(fwd_seed),
                   train=np.array(train), xdtype=np.array(xdt), fkw=np.array(json.dumps({k: v for k, v in fkw.items() if k != "mask"})),
                   x=to_np(x.detach()), G=to_np(G), out=to_np(out.detach()), out_dtype=np.array(str(out.dtype)),
                   indices=idx.numpy(), idx_dtype=np.array(str(idx.dtype)), losses=to_np(losses.detach().reshape(-1).float()),
                   dx=to_np(x.grad.float()) if x.grad is not None else np.zeros(x.shape, np.float32))
        if mask is not None:
            rec["mask"] = mask.numpy()
        if bd is not None:
            rec["breakdown"] = np.array([float(v.detach()) for v in bd])
        for k, v in sd.items():
            rec["sd." + k] = to_np(v)
        rec["losses64"] = losses64.detach().reshape(-1).numpy()
        for j, z in enumerate(zs):
            rec[f"z{j}"] = to_np(z.detach().float())
            rec[f"gz{j}"] = to_np(z.grad.float()) if z.grad is not None else np.zeros(1)
            rec[f"gz64_{j}"] = zs64[j].grad.numpy() if zs64[j].grad is not None else np.zeros(1)
        for j, q in enumerate(qs):
            rec[f"q{j}"] = to_np(q.float())
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print(name, "indices", tuple(idx.shape), "losses", rec["losses"][:4], "breakdown", rec.get("breakdown"))


if __name__ == "__main__":
    main()
