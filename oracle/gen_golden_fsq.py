"""Generate tests/golden/fsq/*.npz by running the UNMODIFIED reference's FSQ / ResidualFSQ / GroupedResidualFSQ on CPU
(TEST INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_fsq.py

Per case: the constructor kwargs and the construction seed, the state_dict, x, an upstream gradient G, and one forward (train or
eval) with the outputs, their dtypes and shapes, and the gradient of sum(out * G) w.r.t. x.  Around the quantizer proper it also
keeps, per ResidualFSQ (per group for GroupedResidualFSQ): z = the project_in output, qsum = the project_out input, and the
gradients at both, so the kernels can be checked on the exact rows the reference quantized (the projections are torch's
matmuls, whose summation order differs between devices).  The per-dimension constants are the reference's own expressions.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "fsq")

L8553 = [8, 5, 5, 5]
L8553R = [8, 5, 5, 3]

# (name, class, kwargs, x shape, x dtype, module dtype, train, forward kwargs, x scale)
CASES = [
    ("fsq_plain_fp32", "FSQ", dict(levels=L8553), (2, 64, 4), "fp32", "fp32", True, {}, 1.5),
    ("fsq_sym_fp32", "FSQ", dict(levels=L8553, preserve_symmetry=True), (2, 64, 4), "fp32", "fp32", True, {}, 1.5),
    ("fsq_hard_fp32", "FSQ", dict(levels=L8553, bound_hard_clamp=True), (2, 64, 4), "fp32", "fp32", True, {}, 1.5),
    ("fsq_sym_hard_fp32", "FSQ", dict(levels=L8553, preserve_symmetry=True, bound_hard_clamp=True), (2, 64, 4), "fp32", "fp32",
     True, {}, 1.5),
    ("fsq_plain_bf16", "FSQ", dict(levels=L8553), (2, 64, 4), "bf16", "fp32", True, {}, 1.5),
    ("fsq_proj_c2_fp32", "FSQ", dict(levels=L8553, dim=32, num_codebooks=2), (2, 48, 32), "fp32", "fp32", True, {}, 1.0),
    ("fsq_image_fp32", "FSQ", dict(levels=L8553, dim=16), (2, 16, 6, 5), "fp32", "fp32", True, {}, 1.0),
    ("rfsq_readme_fp32", "ResidualFSQ", dict(dim=256, levels=L8553R, num_quantizers=8), (2, 32, 256), "fp32", "fp32", True, {}, 1.0),
    ("rfsq_readme_bf16", "ResidualFSQ", dict(dim=256, levels=L8553R, num_quantizers=8), (2, 32, 256), "bf16", "bf16", True, {}, 1.0),
    ("rfsq_eval_allcodes_fp32", "ResidualFSQ", dict(dim=256, levels=L8553R, num_quantizers=8), (2, 32, 256), "fp32", "fp32", False,
     dict(return_all_codes=True), 1.0),
    ("rfsq_dropout_fp32", "ResidualFSQ", dict(dim=32, levels=L8553R, num_quantizers=8, quantize_dropout=True,
                                              quantize_dropout_cutoff_index=1, quantize_dropout_multiple_of=4), (2, 48, 32), "fp32",
     "fp32", True, dict(rand_quantize_dropout_fixed_seed=1), 1.0),
    ("rfsq_chfirst_fp32", "ResidualFSQ", dict(dim=32, levels=L8553R, num_quantizers=4, is_channel_first=True), (2, 32, 6, 5), "fp32",
     "fp32", True, {}, 1.0),
    ("rfsq_bf16in_noproj", "ResidualFSQ", dict(levels=L8553R, num_quantizers=4), (2, 64, 4), "bf16", "fp32", True, {}, 1.5),
    ("rfsq_softclamp_tanh_fp32", "ResidualFSQ", dict(levels=L8553R, num_quantizers=4, bound_hard_clamp=False,
                                                     soft_clamp_input_value=1.5), (2, 64, 4), "fp32", "fp32", True, {}, 1.5),
    ("grfsq_fp32", "GroupedResidualFSQ", dict(dim=64, groups=2, levels=L8553R, num_quantizers=4), (2, 40, 64), "fp32", "fp32", True,
     {}, 1.0),
    ("grfsq_image_fp32", "GroupedResidualFSQ", dict(dim=64, groups=2, levels=L8553R, num_quantizers=4, accept_image_fmap=True,
                                                    is_channel_first=True), (2, 64, 6, 5), "fp32", "fp32", True, {}, 1.0),
]

DT = {"fp32": torch.float32, "bf16": torch.bfloat16}


def f32(t):
    return t.detach().float().cpu().numpy().astype(np.float32)


def rfsq_parts(m):
    """The ResidualFSQ modules of a case (one, or one per group) and the FSQ whose projections bracket the quantizer."""
    if hasattr(m, "rvqs"):
        return list(m.rvqs)
    return [m]


def fsq_constants(layer):
    """The reference's per-dimension constants (fsq:152-156, :165-166), by its own expressions."""
    lv = layer._levels
    out = dict(half_l=(lv - 1) * (1 + 1e-3) / 2, offset=torch.where(lv % 2 == 0, 0.5, 0.0), half_width=lv // 2,
               sym_scale=2. / (lv - 1), basis=layer._basis)
    out["shift_atanh"] = torch.atanh(out["offset"] / out["half_l"])
    out["shift_hard"] = out["offset"] / out["half_l"]
    return {k: v.float().numpy() for k, v in out.items()}


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, cls, kw, x_shape, xdt, mdt, train, fkw, xs) in enumerate(CASES):
        init_seed = 300 + i
        torch.manual_seed(init_seed)
        m = getattr(ref, cls)(**kw)
        if mdt == "bf16":
            m = m.to(torch.bfloat16)
        m.train(train)
        sd = m.state_dict()
        store = {f"sd_{j}": v.float().numpy().copy() for j, v in enumerate(sd.values())}
        gen = torch.Generator().manual_seed(7100 + i)
        x = (torch.randn(*x_shape, generator=gen) * xs).to(DT[xdt]).requires_grad_(True)
        G = torch.randn(*x_shape, generator=gen)
        # capture z (project_in output) and qsum (project_out input) of every ResidualFSQ / the FSQ
        parts = rfsq_parts(m)
        cap = [dict() for _ in parts]

        def hook_in(k):
            def h(mod, inp, out):
                out.retain_grad()
                cap[k]["z"] = out
            return h

        def hook_out(k):
            def h(mod, inp):
                inp[0].retain_grad()
                cap[k]["qsum"] = inp[0]
            return h

        handles = []
        for k, p in enumerate(parts):
            handles.append(p.project_in.register_forward_hook(hook_in(k)))
            handles.append(p.project_out.register_forward_pre_hook(hook_out(k)))
        res = m(x, **fkw)
        for h in handles:
            h.remove()
        out, ind = res[0], res[1]
        (out.float() * G).sum().backward()
        store.update(x=f32(x), G=f32(G), out=f32(out), xgrad=f32(x.grad))
        if ind is not None:
            store["indices"] = ind.numpy().astype(np.int64)
        if len(res) > 2:
            ac = res[2]
            store["all_codes"] = f32(torch.stack(list(ac)) if isinstance(ac, tuple) else ac)
        store["z"] = np.stack([f32(c["z"]) for c in cap])
        store["qsum"] = np.stack([f32(c["qsum"]) for c in cap])
        store["zgrad"] = np.stack([f32(c["z"].grad) for c in cap])
        store["qgrad"] = np.stack([f32(c["qsum"].grad) for c in cap])
        layer = parts[0].layers[0] if hasattr(parts[0], "layers") else parts[0]
        for k, v in fsq_constants(layer).items():
            store[f"const_{k}"] = v
        if hasattr(parts[0], "scales"):
            store["scales"] = f32(parts[0].scales)
            scv = parts[0].soft_clamp_input_value
            if scv is not None:
                store["soft_clamp"] = f32(scv.expand(len(parts[0].levels)))
        if cls == "ResidualFSQ" and not train:
            store["decoded"] = f32(m.get_output_from_indices(ind))
        meta = dict(kind="fsq", name=name, cls=cls, kw=kw, x_shape=list(x_shape), x_dtype=xdt, module_dtype=mdt, train=train,
                    forward_kw=fkw, x_scale=xs, init_seed=init_seed, state_dict_keys=list(sd), torch=torch.__version__,
                    out_dtype=str(out.dtype).replace("torch.", ""), out_shape=list(out.shape),
                    indices_dtype=None if ind is None else str(ind.dtype).replace("torch.", ""),
                    indices_shape=None if ind is None else list(ind.shape),
                    z_dtype=str(cap[0]["z"].dtype).replace("torch.", ""), qsum_dtype=str(cap[0]["qsum"].dtype).replace("torch.", ""),
                    xgrad_dtype=str(x.grad.dtype).replace("torch.", ""))
        store["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **store)
        print(f"fsq/{name}: {os.path.getsize(path) / 1024:.0f} KiB out {meta['out_dtype']} {meta['out_shape']} "
              f"idx {meta['indices_dtype']} {meta['indices_shape']}")


if __name__ == "__main__":
    main()
