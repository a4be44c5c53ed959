"""Replay helpers of tests/golden/residual_simvq/*.npz (oracle/gen_golden_residual_simvq.py, written by the reference)."""
import glob
import json
import os

import numpy as np

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "residual_simvq")


def names():
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(DIR, "*.npz")))


class Fixture:
    def __init__(self, name):
        self.z = np.load(os.path.join(DIR, name + ".npz"))
        self.meta = json.loads(bytes(self.z["meta"]).decode())

    def __getitem__(self, k):
        return self.z[k]

    def state(self):
        """The reference's initial state_dict, key order kept."""
        return {k: self.z[f"sd_{j}"] for j, k in enumerate(self.meta["state_dict_keys"])}

    def build(self, mod):
        """ResidualSimVQ of package `mod` built like the reference was (same seed, same construction order)."""
        import torch
        from oracle.gen_golden_residual_simvq import make_transform
        m = self.meta
        torch.manual_seed(m["init_seed"])
        t = make_transform(m["transform"], m["kw"]["dim"])
        return mod.ResidualSimVQ(**m["kw"], **({"codebook_transform": t} if t is not None else {}))

    def rows(self, a):
        """(b, ..., d) or channel-first (b, d, ...) array -> (N, d) rows in the order the quantizer packs them."""
        if self.meta["kw"].get("channel_first"):
            a = np.moveaxis(a, 1, -1)
        return a.reshape(-1, a.shape[-1])
