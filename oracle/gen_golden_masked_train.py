"""Generate tests/golden/masked_train/*.npz: one masked training step of the UNMODIFIED reference on CPU (TEST INFRASTRUCTURE
ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_masked_train.py

Per case: the initial state_dict under a seed, seeded x (requires grad), a mask (or lens), an upstream gradient G, one training
forward and a backward of sum(out * G) + LW * sum(loss).  Stored: x, mask, G, the output, indices, loss, x.grad, every
parameter's .grad (the projections of ResidualVQ), the state_dict after the step (the EMA codebook buffers) and every draw the
reference made from torch.randperm / torch.randint during the forward (k-means samples), so a replay can substitute them.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402
from gen_golden_learnable import RngRecorder, f32  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "masked_train")
LW = 0.7

_VQ = dict(dim=32, codebook_size=48)
_RVQ = dict(dim=32, num_quantizers=3, codebook_size=32)
# (name, class, construction kwargs, x shape, dtype, lens of the batch's sequences, how the mask is passed, padding rows,
#  forward kwargs)
#   lens: the mask is arange(n) < lens; "mask": passed as mask=, "lens": as lens=
#   padding: "rand" (x as drawn) or "zero" (padding rows exactly zero)
CASES = [
    ("vq_rotation_fp32", "VectorQuantize", dict(_VQ), (3, 40, 32), "float32", (40, 23, 7), "mask", "rand", {}),
    ("vq_ste_fp32", "VectorQuantize", dict(_VQ, rotation_trick=False, commitment_weight=0.5), (3, 40, 32), "float32",
     (31, 40, 12), "mask", "rand", {}),
    ("vq_rotation_bf16", "VectorQuantize", dict(_VQ), (3, 40, 32), "bfloat16", (40, 23, 7), "mask", "rand", {}),
    ("vq_ste_bf16", "VectorQuantize", dict(_VQ, rotation_trick=False), (3, 40, 32), "bfloat16", (17, 33, 40), "mask", "rand",
     {}),
    ("vq_lens_fp32", "VectorQuantize", dict(_VQ), (4, 24, 32), "float32", (24, 1, 13, 20), "lens", "rand", {}),
    ("vq_passthrough_fp32", "VectorQuantize", dict(_VQ, return_zeros_for_masked_padding=False), (3, 40, 32), "float32",
     (40, 23, 7), "mask", "rand", {}),
    ("vq_passthrough_ste_fp32", "VectorQuantize", dict(_VQ, return_zeros_for_masked_padding=False, rotation_trick=False),
     (3, 40, 32), "float32", (9, 40, 30), "mask", "rand", {}),
    ("vq_allpad_fp32", "VectorQuantize", dict(_VQ), (3, 40, 32), "float32", (40, 0, 25), "mask", "rand", {}),
    ("vq_zeropad_fp32", "VectorQuantize", dict(_VQ), (3, 40, 32), "float32", (40, 11, 29), "mask", "zero", {}),
    ("vq_zeropad_bf16", "VectorQuantize", dict(_VQ), (3, 40, 32), "bfloat16", (3, 40, 29), "mask", "zero", {}),
    ("vq_cosine_fp32", "VectorQuantize", dict(_VQ, use_cosine_sim=True), (3, 40, 32), "float32", (40, 23, 7), "mask", "rand",
     {}),
    ("vq_cosine_ste_bf16", "VectorQuantize", dict(_VQ, use_cosine_sim=True, rotation_trick=False), (3, 40, 32), "bfloat16",
     (12, 40, 27), "lens", "rand", {}),
    ("vq_kmeans_fp32", "VectorQuantize", dict(_VQ, kmeans_init=True, kmeans_iters=4), (3, 40, 32), "float32", (40, 23, 7),
     "mask", "rand", {}),
    ("rvq_separate_proj_fp32", "ResidualVQ", dict(_RVQ, codebook_dim=16), (3, 40, 32), "float32", (40, 23, 7), "mask", "rand",
     {}),
    ("rvq_shared_fp32", "ResidualVQ", dict(_RVQ, shared_codebook=True), (3, 40, 32), "float32", (19, 40, 5), "mask", "rand",
     {}),
    ("rvq_shared_proj_fp32", "ResidualVQ", dict(_RVQ, codebook_dim=24, shared_codebook=True), (3, 40, 32), "float32",
     (40, 0, 30), "mask", "zero", {}),
    ("rvq_dropout_fp32", "ResidualVQ", dict(_RVQ, num_quantizers=4, quantize_dropout=True), (3, 40, 32), "float32",
     (40, 23, 7), "mask", "rand", dict(rand_quantize_dropout_fixed_seed=5)),
    ("grvq_fp32", "GroupedResidualVQ", dict(_RVQ, groups=2), (3, 40, 32), "float32", (40, 23, 7), "mask", "rand", {}),
]


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, cls, kw, x_shape, dtype, lens, how, padding, fwd) in enumerate(CASES):
        init_seed = 500 + i
        torch.manual_seed(init_seed)
        m = getattr(ref, cls)(**kw)
        m.train()
        sd = m.state_dict()
        store = {f"sd_{j}": v.numpy().copy() for j, v in enumerate(sd.values())}
        params = [n for n, _ in m.named_parameters()]
        gen = torch.Generator().manual_seed(6161 + i)
        dt = getattr(torch, dtype)
        lens_t = torch.tensor(lens, dtype=torch.int64)
        mask = torch.arange(x_shape[1]) < lens_t[:, None]
        x = torch.randn(*x_shape, generator=gen)
        if padding == "zero":
            x = x * mask[..., None]
        x = x.to(dt).requires_grad_(True)
        G = torch.randn(*x_shape, generator=gen)
        torch.manual_seed(7000 + 13 * i)
        with RngRecorder() as rec:
            if how == "lens":
                out, ind, loss = m(x, lens=lens_t, **fwd)
            else:
                out, ind, loss = m(x, mask=mask, **fwd)
        ((out.float() * G).sum() + LW * loss.float().sum()).backward()
        store.update({"x": f32(x), "mask": mask.numpy(), "lens": lens_t.numpy(), "G": f32(G), "out": f32(out),
                      "ind": ind.numpy().astype(np.int64), "loss": f32(loss), "xgrad": f32(x.grad)})
        for j, (n, p) in enumerate(m.named_parameters()):
            store[f"pgrad_{j}"] = f32(p.grad) if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
        for j, v in enumerate(m.state_dict().values()):
            store[f"post_{j}"] = v.numpy().copy()
        kinds = []
        for j, (kind, t) in enumerate(rec.draws):
            store[f"rng_{j}"] = t.float().numpy() if t.is_floating_point() else t.numpy().astype(np.int64)
            kinds.append(kind)
        meta = dict(kind="masked_train", name=name, cls=cls, kw=kw, x_shape=list(x_shape), dtype=dtype, lens=list(lens),
                    how=how, padding=padding, fwd=fwd, lw=LW, init_seed=init_seed, state_dict_keys=list(sd), param_names=params,
                    rng=kinds, torch=torch.__version__)
        store["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **store)
        print(f"masked_train/{name}: {os.path.getsize(path) / 1024:.0f} KiB rng={kinds} "
              f"nan={bool(np.isnan(store['xgrad']).any())}")


if __name__ == "__main__":
    main()
