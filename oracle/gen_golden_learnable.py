"""Generate tests/golden/learnable/*.npz by training the UNMODIFIED reference on CPU for a few steps with a codebook learnt by
gradient (TEST INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_learnable.py

Per case: the initial state_dict under a seed, then per step one training forward with seeded x and upstream gradient G, a
backward of sum(out * G) + LW * sum(loss), and a plain SGD step (lr LR) over every parameter.  Stored per step s: x_s, G_s,
the indices, output, loss, x.grad, every parameter's .grad, the post-step state_dict, and every draw the reference made from
torch's RNG in that step (`rng_s_j`: the k-means / dead-code samples of torch.randperm / torch.randint, and the DiVeQ noise of
torch.randn_like), so that a replay can substitute the reference's draws for its own.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "learnable")
LR = 0.1
LW = 0.7
STEPS = 3

_L = dict(learnable_codebook=True, ema_update=False)
# (name, class, construction kwargs, x shape, dtype, x requires grad)
CASES = [
    ("vq_rotation_fp32", "VectorQuantize", dict(dim=32, codebook_size=48, **_L), (2, 64, 32), "float32", True),
    ("vq_ste_fp32", "VectorQuantize", dict(dim=32, codebook_size=48, rotation_trick=False, **_L), (2, 64, 32), "float32", True),
    ("vq_nograd_fp32", "VectorQuantize", dict(dim=32, codebook_size=48, **_L), (2, 64, 32), "float32", False),
    ("vq_rotation_bf16", "VectorQuantize", dict(dim=32, codebook_size=48, **_L), (2, 64, 32), "bfloat16", True),
    ("vq_ste_bf16", "VectorQuantize", dict(dim=32, codebook_size=48, rotation_trick=False, **_L), (2, 64, 32), "bfloat16", True),
    ("vq_nograd_bf16", "VectorQuantize", dict(dim=32, codebook_size=48, **_L), (2, 64, 32), "bfloat16", False),
    ("vq_syncv_fp32", "VectorQuantize", dict(dim=32, codebook_size=48, sync_update_v=1., **_L), (2, 64, 32), "float32", False),
    ("vq_heads2_fp32", "VectorQuantize", dict(dim=32, codebook_dim=16, heads=2, codebook_size=40, **_L), (2, 48, 32), "float32",
     True),
    ("vq_image_fp32", "VectorQuantize", dict(dim=32, codebook_size=40, accept_image_fmap=True, **_L), (2, 32, 6, 5), "float32",
     True),
    ("vq_kmeans_expire_fp32", "VectorQuantize", dict(dim=32, codebook_size=40, kmeans_init=True, kmeans_iters=4,
                                                     threshold_ema_dead_code=2, **_L), (2, 64, 32), "float32", True),
    ("vq_diveq_fp32", "VectorQuantize", dict(dim=32, codebook_size=40, directional_reparam=True, threshold_ema_dead_code=2),
     (2, 64, 32), "float32", True),
    ("vq_diveq_bf16", "VectorQuantize", dict(dim=32, codebook_size=40, directional_reparam=True, threshold_ema_dead_code=2),
     (2, 64, 32), "bfloat16", True),
    ("rvq_separate_fp32", "ResidualVQ", dict(dim=32, num_quantizers=3, codebook_size=32, **_L), (2, 64, 32), "float32", True),
    ("rvq_separate_bf16", "ResidualVQ", dict(dim=32, num_quantizers=3, codebook_size=32, **_L), (2, 64, 32), "bfloat16", True),
    ("rvq_shared_fp32", "ResidualVQ", dict(dim=32, num_quantizers=3, codebook_size=32, shared_codebook=True, **_L), (2, 64, 32),
     "float32", True),
    ("rvq_shared_bf16", "ResidualVQ", dict(dim=32, num_quantizers=3, codebook_size=32, shared_codebook=True, **_L), (2, 64, 32),
     "bfloat16", True),
    ("rvq_diveq_fp32", "ResidualVQ", dict(dim=32, num_quantizers=3, codebook_size=32, diveq=True), (2, 64, 32), "float32", True),
    ("grvq_fp32", "GroupedResidualVQ", dict(dim=32, groups=2, num_quantizers=2, codebook_size=24, **_L), (2, 48, 32), "float32",
     True),
]


def f32(t):
    return t.detach().float().cpu().numpy().astype(np.float32)


class RngRecorder:
    """Records, in call order, what torch.randperm / torch.randint / torch.randn_like return while it is active."""

    def __init__(self):
        self.draws = []
        self._orig = {}

    def __enter__(self):
        for name in ("randperm", "randint", "randn_like"):
            fn = getattr(torch, name)
            self._orig[name] = fn

            def wrap(*a, _fn=fn, _name=name, **k):
                out = _fn(*a, **k)
                self.draws.append((_name, out.detach().clone()))
                return out
            setattr(torch, name, wrap)
        return self

    def __exit__(self, *exc):
        for name, fn in self._orig.items():
            setattr(torch, name, fn)


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, cls, kw, x_shape, dtype, x_grad) in enumerate(CASES):
        init_seed = 300 + i
        torch.manual_seed(init_seed)
        m = getattr(ref, cls)(**kw)
        m.train()
        sd = m.state_dict()
        store = {f"sd_{j}": v.numpy().copy() for j, v in enumerate(sd.values())}
        params = [n for n, _ in m.named_parameters()]
        opt = torch.optim.SGD(m.parameters(), lr=LR)
        gen = torch.Generator().manual_seed(4242 + i)
        dt = getattr(torch, dtype)
        rng_kinds = []
        for s in range(STEPS):
            x = torch.randn(*x_shape, generator=gen).to(dt).requires_grad_(x_grad)
            G = torch.randn(*x_shape, generator=gen)
            opt.zero_grad(set_to_none=True)
            torch.manual_seed(9000 + 17 * i + s)
            with RngRecorder() as rec:
                out, ind, loss = m(x)
            ((out.float() * G).sum() + LW * loss.float().sum()).backward()
            store.update({f"x_{s}": f32(x), f"G_{s}": f32(G), f"out_{s}": f32(out), f"ind_{s}": ind.numpy().astype(np.int64),
                          f"loss_{s}": f32(loss)})
            if x_grad:
                store[f"xgrad_{s}"] = f32(x.grad)
            for j, (n, p) in enumerate(m.named_parameters()):
                store[f"pgrad_{s}_{j}"] = f32(p.grad) if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
            opt.step()
            for j, v in enumerate(m.state_dict().values()):
                store[f"post_{s}_{j}"] = v.numpy().copy()
            kinds = []
            for j, (kind, t) in enumerate(rec.draws):
                store[f"rng_{s}_{j}"] = t.float().numpy() if t.is_floating_point() else t.numpy().astype(np.int64)
                kinds.append(kind)
            rng_kinds.append(kinds)
        meta = dict(kind="learnable", name=name, cls=cls, kw=kw, x_shape=list(x_shape), dtype=dtype, x_grad=x_grad, steps=STEPS,
                    lr=LR, lw=LW, init_seed=init_seed, state_dict_keys=list(sd), param_names=params, rng=rng_kinds,
                    torch=torch.__version__)
        store["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **store)
        print(f"learnable/{name}: {os.path.getsize(path) / 1024:.0f} KiB rng={rng_kinds}")


if __name__ == "__main__":
    main()
