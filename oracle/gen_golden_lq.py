"""Generate tests/golden/lq/*.npz by running the UNMODIFIED reference's LatentQuantize on the CPU (TEST INFRASTRUCTURE ONLY;
needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_lq.py

Per case: the constructor kwargs, the seed, the seeded state_dict (keys and tensors), the value tables the forward used
(`table_i`, after any loaded values), and
  - one training step: x, the upstream gradient g of `out`, out, indices, loss, the z the reference quantized (`z`, after
    project_in), and the gradients of x and of the projections for the objective sum(out * g) + loss (sum(out * g) alone
    when `loss_backward` is false: with a bf16 input the reference's mse backward raises on its mixed dtypes);
  - one eval step on the same x: `eval_out`, `eval_indices`, `eval_loss`.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "lq")
README = dict(levels=[5, 5, 8], dim=16, commitment_loss_weight=0.1, quantization_loss_weight=0.1)


def planted(tables, n_rows, D, gen):
    """Rows of z (n_rows, D): randn, then per latent the fp32 midpoints of neighbouring table values, the values themselves,
    +-0 and +-1e4, +-1e8 planted down the rows."""
    z = torch.randn(n_rows, D, generator=gen) * 0.4
    for i, v in enumerate(tables):
        s = np.sort(v.numpy())
        mids = ((s[:-1].astype(np.float64) + s[1:]) / 2).astype(np.float32)
        special = np.concatenate([mids, s, np.float32([0.0, -0.0, 1e4, -1e4, 1e8, -1e8])])
        col = z[:, i].numpy()
        rows = (np.arange(len(special)) * 7 + i) % n_rows
        col[rows] = special
        z[:, i] = torch.from_numpy(col)
    return z


# (name, kwargs, x shape, dtype, x maker ('randn' or 'planted'), loaded tables or None)
CASES = [
    ("readme_image", README, (2, 16, 8, 8), torch.float32, "randn", None),
    ("readme_video", README, (1, 16, 3, 4, 4), torch.float32, "randn", None),
    ("readme_series", README, (2, 16, 24), torch.float32, "randn", None),
    ("readme_2d", README, (6, 16), torch.float32, "randn", None),
    ("codebooks4", dict(README, num_codebooks=4), (2, 16, 20), torch.float32, "randn", None),
    ("int_levels", dict(levels=5, dim=16, codebook_dim=3), (2, 16, 6, 6), torch.float32, "randn", None),
    ("no_optimize", dict(README, optimize_values=False), (2, 16, 6, 6), torch.float32, "randn", None),
    ("noproj_3cb", dict(levels=[4, 8, 16], dim=9, num_codebooks=3), (2, 9, 10), torch.float32, "randn", None),
    ("bf16_noproj", dict(levels=[5, 5, 8], dim=3), (2, 3, 8, 8), torch.bfloat16, "randn", None),
    ("weights_zero_c", dict(levels=[5, 5, 8], dim=3, commitment_loss_weight=0.0, quantization_loss_weight=0.25),
     (2, 3, 40), torch.float32, "randn", None),
    ("weights_zero_both", dict(levels=[5, 5, 8], dim=3, commitment_loss_weight=0.0, quantization_loss_weight=0.0),
     (2, 3, 40), torch.float32, "randn", None),
    ("nondyadic", dict(levels=[6, 7, 12], dim=3), (1, 3, 96), torch.float32, "planted", None),
    ("unsorted", dict(levels=[5, 5, 8], dim=3), (1, 3, 64), torch.float32, "planted",
     [[0.3, -0.5, 0.3, 0.0, -0.25], [0.5, 0.25, 0.25, -0.5, 0.1], [0.125, -0.375, 0.375, 0.125, -0.5, 0.0, 0.25, -0.125]]),
    ("levels_2p24", dict(levels=[256, 256, 257], dim=3), (1, 3, 2048), torch.float32, "planted", None),
]


def run_case(ref, name, kw, shape, dtype, maker, loaded, seed):
    torch.manual_seed(seed)
    m = ref.LatentQuantize(**kw)
    sd = m.state_dict()
    rec = dict(sd_keys=np.array(json.dumps(list(sd))))
    for j, v in enumerate(sd.values()):
        rec[f"sd_{j}"] = v.numpy().copy()
    if loaded is not None:
        with torch.no_grad():
            for i, v in enumerate(loaded):
                m.values_per_latent[i].copy_(torch.tensor(v, dtype=torch.float32))
    tables = [v.detach().clone() for v in m.values_per_latent]
    for i, v in enumerate(tables):
        rec[f"table_{i}"] = v.numpy()
    gen = torch.Generator().manual_seed(seed + 1)
    if maker == "randn":
        x = torch.randn(*shape, generator=gen)
    else:
        b, d, n = shape
        x = planted(tables, b * n, d, gen).reshape(b, n, d).movedim(-1, 1).contiguous()
    x = x.to(dtype).requires_grad_()
    seen = {}
    if m.has_projections:
        m.project_in.register_forward_hook(lambda mod, inp, out: seen.update(z=out.detach().float().numpy().copy()))
    m.train()
    out, indices, loss = m(x)
    g = torch.randn(out.shape, generator=gen)
    loss_backward = dtype == torch.float32
    obj = (out * g).sum() + (loss if loss_backward and loss.requires_grad else 0.0)
    obj.backward()
    rec.update(x=x.detach().float().numpy(), g=g.numpy(), out=out.detach().numpy(), indices=indices.numpy(),
               loss=np.float32(loss.item()), x_grad=x.grad.float().numpy())
    rec["z"] = seen["z"] if m.has_projections else x.detach().float().movedim(1, -1).reshape(x.shape[0], -1, x.shape[1]).numpy()
    if m.has_projections:
        for nm, p in (("pin_w", m.project_in.weight), ("pin_b", m.project_in.bias), ("pout_w", m.project_out.weight),
                      ("pout_b", m.project_out.bias)):
            rec[f"{nm}_grad"] = p.grad.numpy().copy()
    m.eval()
    with torch.no_grad():
        eo, ei, el = m(x.detach())
    rec.update(eval_out=eo.numpy(), eval_indices=ei.numpy(), eval_loss=np.float32(el.item()))
    meta = dict(name=name, kw=kw, shape=list(shape), dtype=str(dtype).replace("torch.", ""), seed=seed,
                loss_backward=loss_backward, loaded=loaded is not None, torch=torch.__version__)
    rec["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    return rec


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, kw, shape, dtype, maker, loaded) in enumerate(CASES):
        rec = run_case(ref, name, kw, shape, dtype, maker, loaded, 11000 + 100 * i)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"lq/{name}: {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
