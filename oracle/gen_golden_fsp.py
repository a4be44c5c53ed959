"""Generate tests/golden/fsp/*.npz by running the UNMODIFIED reference's FSP on the CPU (TEST INFRASTRUCTURE ONLY; needs the
reference, oracle/ref_loader.py):

    python oracle/gen_golden_fsp.py

Per case: the constructor kwargs, the construction and forward seeds, the state_dict, x, the two perturbation draws (recorded
by wrapping torch.rand_like during the call: the wrapper calls the real function and keeps a copy), z (the project_in
output), every output (q_z, indices, norm_loss, level_indices, norm_info, p_accept_prob), and the gradients of
sum(q_z * G) + norm_loss + sum_k norm_info[k] . H[k] with respect to x and z.  The same step is then rerun in float64 with the
same draws cast to double; its outputs and gradients (`*64`) set the tolerance of the replay.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "fsp")
STATS = ("mean", "variance", "skewness", "kurtosis")

# (name, kwargs, x shape, dtype, train, forward eps, x scale, column offset)
CASES = [(f"act_{a}{'_inv' if inv else ''}", dict(levels=[8, 5, 5, 5], act_name=a, need_inv_act=inv, quantize_rate=0.5),
          (2, 256, 4), "fp32", True, None, 1.5, 0.) for a in ("tanh", "sigmoid", "normal", "laplace", "cauchy") for inv in (False, True)]
CASES += [(f"norm_{v}", dict(levels=[7, 6, 5], vector_norm=v), (1, 300, 3), "fp32", True, None, 1.0, 0.)
          for v in ("none", "var", "kurt", "var_tanh", "var_sigmoid", "var_laplace")]
CASES += [
    ("rate0", dict(levels=[8, 5, 5, 5], quantize_rate=0.0), (1, 512, 4), "fp32", True, None, 1.0, 0.),
    ("rate1", dict(levels=[8, 5, 5, 5], quantize_rate=1.0), (1, 512, 4), "fp32", True, None, 1.0, 0.),
    ("eval", dict(levels=[8, 5, 5, 5], quantize_rate=0.5), (1, 512, 4), "fp32", False, None, 1.0, 0.),
    ("image_channel_first", dict(levels=[8, 5, 5, 5], dim=4, channel_first=True), (2, 4, 8, 8), "fp32", True, None, 1.0, 0.),
    ("proj_dim256", dict(levels=[8, 5, 5, 5], dim=256, quantize_rate=0.5, vector_norm="kurt"), (1, 32, 256), "fp32", True, None, 1.0, 0.),
    ("levels_2_mixed", dict(levels=[2, 3, 4, 2, 7, 16], act_name="normal"), (1, 400, 6), "fp32", True, None, 1.0, 0.),
    ("explicit_eps", dict(levels=[8, 5, 5, 5], need_inv_act=True, act_name="sigmoid"), (1, 256, 4), "fp32", True, 1e-3, 3.0, 0.),
    ("readme_basic", dict(levels=[8, 5, 5, 5], act_name="normal", vector_norm="none"), (1, 1024, 4), "fp32", True, None, 1.0, 0.),
    ("readme_eval", dict(levels=[8, 5, 5, 5]), (1, 1024, 4), "fp32", False, None, 1.0, 0.),
    ("bf16_eval", dict(levels=[8, 5, 5, 5]), (1, 4096, 4), "bf16", False, None, 1.0, 0.),
    ("bf16_train", dict(levels=[8, 5, 5, 5], quantize_rate=0.5, vector_norm="kurt"), (1, 1024, 4), "bf16", True, None, 1.0, 0.),
    ("large_offset", dict(levels=[8, 5, 5, 5], vector_norm="kurt"), (1, 2048, 4), "fp32", True, None, 1.0, 1000.),
]


def to_np(t):
    return t.detach().float().numpy() if t.dtype == torch.bfloat16 else t.detach().numpy()


def run(ref, kwargs, sd, x, train, eps, draws, G, H):
    """One forward and backward; `draws` None records the draws, a list replays them (cast to x's dtype)."""
    mod = ref.FSP(**kwargs)
    mod.load_state_dict(sd, strict=False)
    mod = mod.to(x.dtype).train(train)
    x = x.detach().clone().requires_grad_(True)
    zs, rec = [], []
    real = torch.rand_like

    def rand_like(t, *a, **k):
        if draws is None:
            u = real(t, *a, **k)
            rec.append(u.clone())
            return u
        u = draws[len(rec)]
        rec.append(u)
        return u.to(t.dtype)

    def hook(_m, _i, out):
        out.retain_grad()
        zs.append(out)
    h = mod.project_in.register_forward_hook(hook)
    torch.rand_like = rand_like
    try:
        q, idx, loss, info = mod(x, eps) if eps is not None else mod(x)
    finally:
        torch.rand_like = real
        h.remove()
    total = (q * G.to(q.dtype)).sum() + loss
    for k, s in enumerate(STATS):
        total = total + (info["norm_info"][s] * H[k].to(q.dtype)).sum()
    total.backward()
    return q, idx, loss, info, x.grad, zs[0], rec


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, kwargs, shape, xdt, train, eps, scale, offset) in enumerate(CASES):
        seed = 3000 + i
        torch.manual_seed(seed)
        mod = ref.FSP(**kwargs)
        sd = {k: v.clone() for k, v in mod.state_dict().items()}
        g = torch.Generator().manual_seed(seed + 1)
        x = torch.randn(*shape, generator=g) * scale
        if offset:
            x[..., 0] += offset
        dt = torch.bfloat16 if xdt == "bf16" else torch.float32
        x = x.to(dt)
        G = torch.randn(*shape, generator=g)
        d = len(kwargs["levels"])
        H = torch.randn(4, d, generator=g) * 0.1
        fwd_seed = seed + 2
        torch.manual_seed(fwd_seed)
        q, idx, loss, info, dx, z, draws = run(ref, kwargs, sd, x, train, eps, None, G, H)
        q64, _, loss64, info64, dx64, z64, _ = run(ref, kwargs, sd, x.double(), train, eps if eps is not None else
                                                    torch.finfo(dt).eps, [u.double() for u in draws], G.double(), H.double())
        rec = dict(kwargs=np.array(json.dumps(kwargs)), seed=np.array(seed), fwd_seed=np.array(fwd_seed), train=np.array(train),
                   xdtype=np.array(xdt), eps=np.array(np.nan if eps is None else eps), x=to_np(x), G=G.numpy(), H=H.numpy(),
                   q=to_np(q), q_dtype=np.array(str(q.dtype)), indices=idx.numpy(), loss=np.array(float(loss)),
                   level_indices=to_np(info["level_indices"]), dx=to_np(dx), dz=to_np(z.grad),
                   q64=q64.detach().numpy(), loss64=np.array(float(loss64)), dx64=dx64.numpy(), dz64=z64.grad.numpy())
        for s in STATS:
            rec["stat_" + s] = to_np(info["norm_info"][s])
            rec["stat64_" + s] = info64["norm_info"][s].detach().numpy()
        if "p_accept_prob" in info:
            rec["p_accept_prob"] = np.array(float(info["p_accept_prob"]))
        for j, u in enumerate(draws):
            rec[f"u{j + 1}"] = to_np(u)
        for k, v in sd.items():
            rec["sd." + k] = v.numpy()
        rec["z"] = to_np(z.detach())
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print(name, "indices", tuple(idx.shape), "loss", float(loss), "draws", len(draws))


if __name__ == "__main__":
    main()
