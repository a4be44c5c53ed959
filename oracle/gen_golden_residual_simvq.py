"""Generate tests/golden/residual_simvq/*.npz by running the UNMODIFIED reference's ResidualSimVQ on CPU
(TEST INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_residual_simvq.py

Per case (residual_sim_vq.py:51-203, "rsv"): the initial state_dict under a seed, then one training forward with seeded x,
upstream gradient G and per-stage loss weights Lw; the outputs and the gradients of sum(quantized * G) + sum(losses * Lw)
with respect to x and to every parameter.  The directory is not globbed by the flat-fixture replays (tests/golden_util.py).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "residual_simvq")


def f32(t):
    return t.detach().float().cpu().numpy().astype(np.float32)


def make_transform(kind, dim):
    """The code_transform of a case: None (each SimVQ layer makes its own nn.Linear) or one MLP that every layer shares (the
    reference passes the same module to all of them, rsv:83).  Built right after torch.manual_seed(init_seed), before the
    quantizer, here and in the tests."""
    if kind == "mlp":
        return torch.nn.Sequential(torch.nn.Linear(dim, 2 * dim), torch.nn.ReLU(), torch.nn.Linear(2 * dim, dim))
    return None


# (name, construction kwargs, x shape, code_transform kind, rand_quantize_dropout_fixed_seed)
CASES = [
    ("q2_rotation", dict(dim=32, num_quantizers=2, codebook_size=40), (2, 48, 32), None, None),
    ("q4_ste", dict(dim=32, num_quantizers=4, codebook_size=40, rotation_trick=False), (2, 48, 32), None, None),
    ("q4_chfirst_rotation", dict(dim=32, num_quantizers=4, codebook_size=48, channel_first=True), (2, 32, 6, 5), None, None),
    ("q2_mlp_ste", dict(dim=32, num_quantizers=2, codebook_size=40, rotation_trick=False), (2, 40, 32), "mlp", None),
    ("q4_mlp_rotation", dict(dim=32, num_quantizers=4, codebook_size=40, commitment_weight=0.5), (2, 40, 32), "mlp", None),
    ("q4_dropout_rotation", dict(dim=32, num_quantizers=4, codebook_size=40, quantize_dropout=True), (2, 48, 32), None, 3),
    ("q4_dropout_mult2_ste", dict(dim=32, num_quantizers=4, codebook_size=40, quantize_dropout=True, quantize_dropout_cutoff_index=1,
                                  quantize_dropout_multiple_of=2, rotation_trick=False), (2, 48, 32), None, 1),
]


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, kw, x_shape, transform, seed) in enumerate(CASES):
        init_seed = 100 + i
        torch.manual_seed(init_seed)
        t = make_transform(transform, kw["dim"])
        m = ref.ResidualSimVQ(**kw, **({"codebook_transform": t} if t is not None else {}))
        m.train()
        sd = m.state_dict()
        store = {f"sd_{j}": v.numpy().copy() for j, v in enumerate(sd.values())}
        gen = torch.Generator().manual_seed(9753 + i)
        x = torch.randn(*x_shape, generator=gen).requires_grad_(True)
        G = torch.randn(*x_shape, generator=gen)
        Lw = torch.rand(kw["num_quantizers"], generator=gen) + 0.5
        q, ind, losses = m(x, rand_quantize_dropout_fixed_seed=seed)
        ((q * G).sum() + (losses * Lw).sum()).backward()
        store.update(x=f32(x), G=f32(G), Lw=f32(Lw), quantized=f32(q), indices=ind.numpy().astype(np.int64), losses=f32(losses),
                     xgrad=f32(x.grad))
        names = []
        for j, (n, p) in enumerate(m.named_parameters()):
            names.append(n)
            store[f"pgrad_{j}"] = f32(p.grad) if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
        meta = dict(kind="residual_simvq", name=name, kw=kw, x_shape=list(x_shape), transform=transform, dropout_seed=seed,
                    init_seed=init_seed, state_dict_keys=list(sd), param_names=names, torch=torch.__version__)
        store["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **store)
        print(f"residual_simvq/{name}: {os.path.getsize(path) / 1024:.0f} KiB", ind.reshape(-1, kw["num_quantizers"])[0].tolist())


if __name__ == "__main__":
    main()
