"""Fixtures of tests/golden/masked_train/*.npz (oracle/gen_golden_masked_train.py, written by the reference)."""
import glob
import json
import os

import numpy as np

DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "masked_train")


def names(prefix=""):
    return sorted(n for n in (os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(DIR, "*.npz")))
                  if n.startswith(prefix))


class Fixture:
    def __init__(self, name):
        self.z = np.load(os.path.join(DIR, name + ".npz"))
        self.meta = json.loads(bytes(self.z["meta"]).decode())
        self.kw = self.meta["kw"]
        self.cls = self.meta["cls"]
        self.bf16 = self.meta["dtype"] == "bfloat16"

    def __getitem__(self, k):
        return self.z[k]

    def state(self):
        return {k: self.z[f"sd_{j}"] for j, k in enumerate(self.meta["state_dict_keys"])}

    def post(self):
        return {k: self.z[f"post_{j}"] for j, k in enumerate(self.meta["state_dict_keys"])}

    def pgrads(self):
        return {n: self.z[f"pgrad_{j}"] for j, n in enumerate(self.meta["param_names"])}

    def draws(self):
        return [(kind, self.z[f"rng_{j}"]) for j, kind in enumerate(self.meta["rng"])]

    def n_run(self):
        """Layers the reference ran (quantize dropout with its fixed seed), for ResidualVQ fixtures."""
        from oracle.masked_train_oracle import dropout_layers
        seed = self.meta["fwd"].get("rand_quantize_dropout_fixed_seed")
        Q = self.kw["num_quantizers"]
        if not self.kw.get("quantize_dropout") or seed is None:
            return Q
        return dropout_layers(seed, self.kw.get("quantize_dropout_cutoff_index", 0), Q)

    def oracle(self):
        """(out, indices, loss(es), x.grad, parameter grads) of the numpy restatement on this fixture's inputs."""
        from oracle import masked_train_oracle as O
        kw, x, mask, G, lw = self.kw, self["x"], self["mask"], self["G"], self.meta["lw"]
        if self.cls == "VectorQuantize":
            out, idx, loss, gx = O.vq_step(
                x, mask, self.state()["_codebook.embed"][0], G, cosine=kw.get("use_cosine_sim", False),
                rotation=kw.get("rotation_trick", True), pad_zeros=kw.get("return_zeros_for_masked_padding", True),
                commit_weight=kw.get("commitment_weight", 1.0), lw=lw)
            return out, idx, loss, gx, {}
        common = dict(num_quantizers=kw["num_quantizers"], shared_codebook=kw.get("shared_codebook", False), lw=lw,
                      n_run=self.n_run())
        if self.cls == "ResidualVQ":
            return O.rvq_step(x, mask, self.state(), G, **common)
        return O.grvq_step(x, mask, self.state(), G, groups=kw["groups"], **common)
