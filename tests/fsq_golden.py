"""Shared loading of the FSQ fixtures (tests/golden/fsq/*.npz, oracle/gen_golden_fsq.py) for the CPU oracle replay and the GPU
replay.  The quantizer proper sees rows (N, G, d): G = the FSQ's codebooks or the GroupedResidualFSQ's groups."""
from __future__ import annotations

import glob
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fsq", "*.npz")))


def fixture_id(path):
    return os.path.splitext(os.path.basename(path))[0]


class Case:
    def __init__(self, path):
        f = np.load(path)
        self.a = {k: f[k] for k in f.files}
        self.meta = json.loads(bytes(self.a["meta"]).decode())
        m = self.meta
        kw = m["kw"]
        self.cls = m["cls"]
        self.levels = kw["levels"]
        self.d = len(self.levels)
        if self.cls == "FSQ":
            self.Q = 1
            self.sym = kw.get("preserve_symmetry", False)
            self.hard = kw.get("bound_hard_clamp", False)
            self.scales = None
            self.clampv = None
        else:
            self.Q = kw["num_quantizers"]
            self.sym = True
            self.hard = kw.get("bound_hard_clamp", True)
            self.scales = self.a["scales"]
            self.clampv = self.a.get("soft_clamp")
        self.chfirst = kw.get("is_channel_first", False)
        self.w_bf16 = m["qsum_dtype"] == "bfloat16"
        self.in_bf16 = m["z_dtype"] == "bfloat16"

    def rows(self, key):
        return part_rows(self.a[key], self.d)

    def index_rows(self, ind=None):
        """The case's indices as (N, G, Q)."""
        ind = self.a["indices"] if ind is None else ind
        Q = self.Q
        if self.cls == "FSQ":
            G = self.meta["kw"].get("num_codebooks", 1)
            return ind.reshape(-1, G)[..., None]
        if self.cls == "ResidualFSQ":
            if self.chfirst:
                ind = np.moveaxis(ind, 1, -1)
            return ind.reshape(-1, Q)[:, None, :]
        G = ind.shape[0]
        if self.chfirst:
            ind = np.moveaxis(ind, 2, -1)
        return np.ascontiguousarray(ind.reshape(G, -1, Q).transpose(1, 0, 2))

    @property
    def n_active(self):
        idx = self.index_rows()
        live = (idx != -1).reshape(-1, self.Q).all(axis=0)
        return int(live.sum())


def part_rows(t, d):
    """(P, b, ..., D) per-part arrays (one part per ResidualFSQ of a group, or the one quantizer) -> (N, G, d)."""
    P = t.shape[0]
    t = t.reshape(P, -1, t.shape[-1])
    if P == 1:
        return np.ascontiguousarray(t[0].reshape(t.shape[1], -1, d))
    return np.ascontiguousarray(t.transpose(1, 0, 2))


def flipped_rows(idx, ref_idx, near):
    """Rows (N, G) whose indices differ, and whether each is excused: the first differing stage is near a rounding boundary
    (oracle.forward's `near`); later stages of such a row are excused with it."""
    diff = idx != ref_idx
    rows = diff.any(axis=-1)
    first = np.argmax(diff, axis=-1)
    excused = np.take_along_axis(near, first[..., None], axis=-1)[..., 0] & rows
    return rows, excused
