"""Generate tests/golden/rpq/*.npz by running the UNMODIFIED reference's RandomProjectionQuantizer on the CPU (TEST
INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_rpq.py

Per case: the constructor kwargs, the seed, the initial state_dict (its tensors when they total at most 4 MiB, and always
their sha256 digests), and per call s: x_s, the packed rows the reference's
VectorQuantize received (`rows_s`), the rows after its project_in (`proj_in_s`, more than one codebook only), the indices,
the codebooks searched when k-means init changed them (`embed_s`), every draw the reference made from torch.randperm / torch.randint
(`rng_s_j`, so a replay can substitute them for its own), and the float64 rerun (rpq_oracle.forward on the searched
codebooks): `rows64_s`, `proj_in64_s`, `indices64_s` and each row's top-2 lead `lead64_s`.

A seed is refused, and the next one tried, when some row's float64 lead over the best distinct code is under GAP_REL (cosine
scores, so relative to 1), or when the float64 search does not give the reference's indices.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402
from gen_golden_hvq import RngRecorder  # noqa: E402
import rpq_oracle as O  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "rpq")
GAP_REL = 2e-5
SD_MAX_BYTES = 4 << 20   # larger state_dicts are stored as per-tensor sha256 digests: a seeded construction rebuilds them

# (name, constructor kwargs, x shape, calls (a .train() between consecutive calls))
CASES = [
    ("bestrq", dict(dim=320, codebook_size=8192, codebook_dim=16), (1, 24, 320), 1),
    ("no_norm", dict(dim=64, codebook_size=256, codebook_dim=16, norm=False), (2, 20, 64), 1),
    ("dim81", dict(dim=81, codebook_size=512, codebook_dim=16), (2, 20, 81), 1),
    ("h2_e16", dict(dim=64, codebook_size=1024, codebook_dim=16, num_codebooks=2), (2, 12, 64), 1),
    ("h4_e8", dict(dim=48, codebook_size=256, codebook_dim=8, num_codebooks=4), (2, 12, 48), 1),
    ("usm", dict(dim=512, codebook_size=1024, codebook_dim=16, num_codebooks=16), (1, 6, 512), 1),
    ("kmeans", dict(dim=64, codebook_size=32, codebook_dim=8, num_codebooks=2, kmeans_init=True), (2, 40, 64), 1),
    ("train_between", dict(dim=64, codebook_size=256, codebook_dim=16), (2, 16, 64), 2),
    ("b1_n1", dict(dim=64, codebook_size=256, codebook_dim=16), (1, 1, 64), 1),
]


def f32(t):
    return t.detach().float().cpu().numpy().astype(np.float32)


def run_case(ref, name, kw, shape, calls, seed):
    torch.manual_seed(seed)
    rpq = ref.RandomProjectionQuantizer(**kw)
    sd = rpq.state_dict()
    rec = dict(sd_keys=np.array(json.dumps(list(sd))),
               sd_sha256=np.array(json.dumps([hashlib.sha256(v.numpy().tobytes()).hexdigest() for v in sd.values()])))
    if sum(v.numel() * v.element_size() for v in sd.values()) <= SD_MAX_BYTES:
        for j, v in enumerate(sd.values()):
            rec[f"sd_{j}"] = v.numpy().copy()
    seen = {}
    rpq.vq.register_forward_pre_hook(lambda mod, inp: seen.update(rows=f32(inp[0])))
    H = rpq.num_codebooks
    if H > 1:
        rpq.vq.project_in.register_forward_hook(lambda mod, inp, out: seen.update(proj_in=f32(out)))
    gen = torch.Generator().manual_seed(seed + 1)
    ok, min_lead = True, np.inf
    for s in range(calls):
        if s > 0:
            rpq.train()
        x = torch.randn(*shape, generator=gen)
        torch.manual_seed(seed + 100 + s)
        with RngRecorder() as rng:
            indices = rpq(x)
        ind = indices.numpy().astype(np.int64)
        embeds = rpq.vq._codebook.embed.detach().numpy().astype(np.float64)
        pin = None
        if H > 1:
            pin = (rpq.vq.project_in.weight.detach().numpy(), rpq.vq.project_in.bias.detach().numpy())
        rows64, y64, idx64, lead64 = O.forward(f32(x), f32(rpq.rand_projs), kw.get("norm", True), embeds, pin)
        ok &= bool((lead64 >= GAP_REL).all()) and np.array_equal(idx64.reshape(ind.shape), ind)
        min_lead = min(min_lead, float(lead64.min()))
        rec.update({f"x_{s}": f32(x), f"rows_{s}": seen["rows"].reshape(-1, seen["rows"].shape[-1]), f"indices_{s}": ind,
                    f"rows64_{s}": rows64, f"indices64_{s}": idx64,
                    f"lead64_{s}": lead64})
        if kw.get("kmeans_init", False):
            rec[f"embed_{s}"] = embeds.astype(np.float32)
        if H > 1:
            rec[f"proj_in_{s}"] = seen["proj_in"].reshape(-1, seen["proj_in"].shape[-1])
            rec[f"proj_in64_{s}"] = y64
        for j, (kind, t) in enumerate(rng.draws):
            rec[f"rng_{s}_{j}"] = t.numpy().astype(np.int64)
        rec[f"rng_kinds_{s}"] = np.array(json.dumps([k for k, _ in rng.draws]))
    meta = dict(name=name, kw=kw, shape=list(shape), calls=calls, seed=seed, min_lead=min_lead, torch=torch.__version__)
    rec["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    return ok, rec, min_lead


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, kw, shape, calls) in enumerate(CASES):
        for attempt in range(200):
            seed = 9000 + 1000 * i + attempt
            ok, rec, lead = run_case(ref, name, kw, shape, calls, seed)
            if ok:
                break
        else:
            raise RuntimeError(f"{name}: no seed with every row's lead above {GAP_REL}")
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"rpq/{name}: seed {seed} min lead {lead:.3g} {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
