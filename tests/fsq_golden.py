"""Shared loading of the FSQ fixtures (tests/golden/fsq/*.npz, oracle/gen_golden_fsq.py) for the CPU oracle replay and the GPU
replay, and the rounding-boundary finder of the kernel tests.  The quantizer proper sees rows (N, G, d): G = the FSQ's codebooks
or the GroupedResidualFSQ's groups."""
from __future__ import annotations

import glob
import json
import os

import numpy as np

from oracle import fsq_oracle as O

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


def _key(f):
    """float32 -> int64 keys ordered like the values (adjacent floats differ by 1; -0 and +0 share 0)."""
    b = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF), b)


def _unkey(k):
    k = np.asarray(k, np.int64)
    return np.where(k < 0, (-k) | 0x80000000, k).astype(np.uint32).view(np.float32)


def stage_values(z, j, levels, Q, q, sym, hard, scales=None, clampv=None, w_bf16=False):
    """The oracle's stage-q (code, pre-floor / pre-round value, stage input u) of element j for 1-D float32 inputs z of that
    element (each element's chain is independent of the others, which are left 0)."""
    zz = np.zeros((len(z), 1, len(levels)), np.float32)
    zz[:, 0, j] = z
    f = O.forward(zz, levels, Q, q + 1, sym, hard, scales, clampv, w_bf16)
    u = f["u"][q][:, 0, :]
    code, _, _, br = O.stage(u, O.tables(levels, sym, hard), sym, hard)
    return code[:, j], br[:, j], u[:, j]


def boundary_pairs(levels, Q, q, j, sym, hard, scales=None, clampv=None, w_bf16=False, lo=-2.5, hi=2.5, n=2001):
    """Adjacent float32 inputs (a, b = the next float after a) of element j across which the oracle's stage-q code changes:
    every sign change of the code on an n-point grid of [lo, hi], bisected on the float32 bit pattern down to one ulp.  The
    bisection keeps code(a) != code(b), so it needs no monotone chain."""
    def code(z):
        return stage_values(z, j, levels, Q, q, sym, hard, scales, clampv, w_bf16)[0]

    grid = np.linspace(lo, hi, n, dtype=np.float32)
    c = code(grid)
    k = np.nonzero(c[:-1] != c[1:])[0]
    a, b, ca = _key(grid[k]), _key(grid[k + 1]), c[k]
    while (b - a > 1).any():
        wide = b - a > 1
        m = a + (b - a) // 2
        same = code(_unkey(m)) == ca
        a = np.where(wide & same, m, a)
        b = np.where(wide & ~same, m, b)
    return _unkey(a), _unkey(b)


def exact_ties(br, sym):
    """Pre-floor values that are exactly an integer (sym) or pre-round values exactly k + 1/2 (non-sym)."""
    br = np.asarray(br, np.float64)
    return br == np.floor(br) if sym else br - np.floor(br) == 0.5


def flipped_rows(idx, ref_idx, near):
    """Rows (N, G) whose indices differ, and whether each is excused: the first differing stage is near a rounding boundary
    (oracle.forward's `near`); later stages of such a row are excused with it."""
    diff = idx != ref_idx
    rows = diff.any(axis=-1)
    first = np.argmax(diff, axis=-1)
    excused = np.take_along_axis(near, first[..., None], axis=-1)[..., 0] & rows
    return rows, excused
