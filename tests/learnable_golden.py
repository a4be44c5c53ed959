"""Replay helpers of tests/golden/learnable/*.npz (oracle/gen_golden_learnable.py, written by the reference)."""
import glob
import json
import os

import numpy as np

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "learnable")


def names():
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(DIR, "*.npz")))


class Fixture:
    def __init__(self, name):
        self.z = np.load(os.path.join(DIR, name + ".npz"))
        self.meta = json.loads(bytes(self.z["meta"]).decode())
        self.kw = self.meta["kw"]

    def __getitem__(self, k):
        return self.z[k]

    def state(self, step=None):
        """The reference's state_dict before step `step` (the initial one for step 0 or None), key order kept."""
        keys = self.meta["state_dict_keys"]
        if not step:
            return {k: self.z[f"sd_{j}"] for j, k in enumerate(keys)}
        return {k: self.z[f"post_{step - 1}_{j}"] for j, k in enumerate(keys)}

    def post(self, step):
        return {k: self.z[f"post_{step}_{j}"] for j, k in enumerate(self.meta["state_dict_keys"])}

    def pgrads(self, step):
        return {n: self.z[f"pgrad_{step}_{j}"] for j, n in enumerate(self.meta["param_names"])}

    def draws(self, step):
        """The reference's RNG draws of step `step`, in call order: [(kind, array)]."""
        return [(kind, self.z[f"rng_{step}_{j}"]) for j, kind in enumerate(self.meta["rng"][step])]

    def noise(self, step):
        d = [a for kind, a in self.draws(step) if kind == "randn_like"]
        return d[0] if d else None

    def build(self, mod):
        """The module of package `mod` built like the reference was (same seed, same construction)."""
        import torch
        torch.manual_seed(self.meta["init_seed"])
        return getattr(mod, self.meta["cls"])(**self.kw)

    # ---- VectorQuantize layouts: (x layout) <-> rows in the order the one codebook sees them
    def vq_rows(self, a):
        kw = self.kw
        if kw.get("accept_image_fmap"):
            b, c, h, w = a.shape
            return np.moveaxis(a, 1, -1).reshape(-1, c)
        heads = kw.get("heads", 1)
        if heads > 1:   # 'b n (h d) -> (b h) n d'
            b, n, hd = a.shape
            return a.reshape(b, n, heads, hd // heads).transpose(0, 2, 1, 3).reshape(-1, hd // heads)
        return a.reshape(-1, a.shape[-1])

    def vq_from_rows(self, r, shape):
        kw = self.kw
        if kw.get("accept_image_fmap"):
            b, c, h, w = shape
            return np.moveaxis(r.reshape(b, h, w, c), -1, 1)
        heads = kw.get("heads", 1)
        if heads > 1:
            b, n, hd = shape
            return r.reshape(b, heads, n, hd // heads).transpose(0, 2, 1, 3).reshape(shape)
        return r.reshape(shape)

    def vq_index_rows(self, ind):
        heads = self.kw.get("heads", 1)
        if heads > 1:   # (b, n, h) -> '(b h) n'
            return ind.transpose(0, 2, 1).reshape(-1)
        return ind.reshape(-1)
