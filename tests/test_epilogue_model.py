"""CPU model of the search kernel's epilogue arithmetic (csrc/epilogue.cuh: ScanReg, RowState::insert, merge_slices).

Each row is split over the four threads of a quad; per row slice the CUDA epilogue keeps the exact running maximum t1 and
a skip threshold thr = (maximum over the row's four slices) - W.  A 16-score group (the values one thread holds for the
row across eight 8-column wgmma blocks: columns base + 8 (e / 2) + (e % 2)) whose maximum beats thr is a potential
candidate: if it beats t1 by more than W it REPLACES the live group (and empties the queue), otherwise it is queued next to it (a near tie; at most CAP groups, overflow -> exact re-scan).  At
the end of the row sweep the exact tagged top-3 (4 low mantissa bits = 15 - position inside the group; compare-exchange minima
recovered with min = a + b - max) is rebuilt from the live groups only, and the column slices are merged into up to three
candidates.  This file restates that arithmetic bit for bit in numpy and checks the CERTIFICATE the parity argument rests
on (DESIGN.md 4.1) against brute force on adversarial score matrices:

  * every code NOT reported as a candidate scores at least W - 2*(tag slack) below the exact row maximum, so the exact
    arg-max is always among the reported candidates (1: certified; 2 / 3: exact re-score of those codes; > 3: whole-row rescan);
  * reported indices are valid and distinct; the exact winning score (`best`, feeds the loss) is the true maximum.

It is a model of the algorithm (test infrastructure), not of the GPU: the CUDA code itself is checked on the device by
tests/test_parity_gpu.py.
"""
import numpy as np
import pytest

NEG = np.float32(-3.4e38)
CAP = 4


def f2u(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def u2f(x):
    return np.ascontiguousarray(x, dtype=np.uint32).view(np.float32)


class RowState:
    """Exact tagged top-3 of one slice, vectorised over rows (epilogue.cuh: struct RowState)."""

    def __init__(self, W):
        R = W.shape[0]
        self.W = W.astype(np.float32)
        self.t1 = np.full(R, NEG, np.float32)
        self.t2 = np.full(R, NEG, np.float32)
        self.t3 = np.full(R, NEG, np.float32)
        self.t4 = np.full(R, NEG, np.float32)               # value only: "is there a fourth candidate"
        self.j1 = np.zeros(R, np.int64)
        self.j2 = np.zeros(R, np.int64)
        self.j3 = np.zeros(R, np.int64)

    def insert(self, r, cbase, act):
        """r: (R, 16) float32 scores of one group; cbase: (R,) first column; act: rows that insert it."""
        t1, t2, t3, t4 = self.t1.copy(), self.t2.copy(), self.t3.copy(), self.t4.copy()
        o1, o2, o3 = t1.copy(), t2.copy(), t3.copy()
        bits = f2u(r)
        with np.errstate(over="ignore"):
            for e in range(16):
                ku = (bits[:, e] & np.uint32(0xFFFFFFF0)) | np.uint32(15 - e)
                n1 = np.maximum(t1, u2f(ku))
                lo1 = (f2u(t1) + ku - f2u(n1)).astype(np.uint32)          # min(t1, k) = t1 + k - max(t1, k), mod 2^32
                n2 = np.maximum(t2, u2f(lo1))
                lo2 = (f2u(t2) + lo1 - f2u(n2)).astype(np.uint32)
                n3 = np.maximum(t3, u2f(lo2))
                lo3 = (f2u(t3) + lo2 - f2u(n3)).astype(np.uint32)
                t4 = np.maximum(t4, u2f(lo3))
                t1, t2, t3 = n1, n2, n3
        k1, k2, k3 = self.j1, self.j2, self.j3
        m1 = t1 == o1                                       # greedy attribution of the new slots to the old ones
        j1 = np.where(m1, k1, cbase)
        q2 = np.where(m1, o2, o1)
        m2 = t2 == q2
        j2 = np.where(m2, np.where(m1, k2, k1), cbase)
        used = m1.astype(np.int64) + m2.astype(np.int64)
        q3 = np.where(used == 0, o1, np.where(used == 1, o2, o3))
        j3 = np.where(t3 == q3, np.where(used == 0, k1, np.where(used == 1, k2, k3)), cbase)
        for name, new in (("t1", t1), ("t2", t2), ("t3", t3), ("t4", t4), ("j1", j1), ("j2", j2), ("j3", j3)):
            setattr(self, name, np.where(act, new, getattr(self, name)))


def group_col(e):
    """Column offset of element e of a group (epilogue.cuh: group_col)."""
    return ((e >> 1) << 3) | (e & 1)


GROUP_COLS = group_col(np.arange(16))


def col(t, j):
    return j + group_col(15 - (f2u(t) & np.uint32(15)).astype(np.int64))


class Scan:
    """Hot loop of one slice (epilogue.cuh: struct ScanReg): running maximum, skip threshold, live group + queue."""

    def __init__(self, W):
        R = W.shape[0]
        self.W = W.astype(np.float32)
        self.t1 = np.full(R, NEG, np.float32)
        self.thr = np.full(R, NEG, np.float32)
        self.kill = np.full(R, NEG, np.float32)
        self.cnt = np.zeros(R, np.int64)
        self.lcol = np.full(R, -1, np.int64)
        self.live = np.full((R, 16), NEG, np.float32)
        self.qv = np.full((R, CAP + 1, 16), NEG, np.float32)
        self.qc = np.zeros((R, CAP + 1), np.int64)

    def raise_(self, other):
        self.thr = np.maximum(self.thr, (other - self.W).astype(np.float32))

    def scan16(self, r, cbase):
        m = r.max(axis=1)
        p = m > self.thr
        if not p.any():                                   # the warp-uniform skip
            return
        reset = m > self.kill
        tie = p & ~reset
        rows = np.nonzero(tie)[0]
        slot = np.minimum(self.cnt[rows], CAP)
        self.qv[rows, slot] = r[rows]
        self.qc[rows, slot] = cbase
        self.cnt[rows] = np.minimum(self.cnt[rows] + 1, CAP + 1)
        self.live = np.where(reset[:, None], r, self.live)
        self.lcol = np.where(reset, cbase, self.lcol)
        self.cnt = np.where(reset, 0, self.cnt)
        self.t1 = np.maximum(self.t1, m)                  # unconditional inside the taken branch, like the kernel
        self.thr = np.maximum(self.thr, (self.t1 - self.W).astype(np.float32))
        self.kill = (self.t1 + self.W).astype(np.float32)

    def finish(self):
        st = RowState(self.W)
        st.bexact = self.t1.copy()
        st.insert(self.live, self.lcol, self.lcol >= 0)
        lv = (self.t1 - self.W).astype(np.float32)
        for i in range(CAP):
            v = self.qv[:, i]
            act = (i < np.minimum(self.cnt, CAP)) & (v.max(axis=1) > lv)
            st.insert(v, self.qc[:, i], act)
        ovf = self.cnt > CAP
        st.t2 = np.where(ovf, st.t1, st.t2)
        st.t3 = np.where(ovf, st.t1, st.t3)
        st.t4 = np.where(ovf, st.t1, st.t4)
        return st


def merge(slices):
    """(i0, i1, i2, n, best) per row (epilogue.cuh: merge_slices, Top3::offer); slices[0] is the merging thread's."""
    R = slices[0].t1.shape[0]
    v = np.full((R, 3), NEG, np.float32)
    ix = np.zeros((R, 3), np.int64)

    def offer(val, idx):
        for r in range(R):                                 # small R in the tests: clarity over speed
            x, i = val[r], idx[r]
            if x > v[r, 0] or (x == v[r, 0] and i < ix[r, 0]):
                v[r, 2], ix[r, 2] = v[r, 1], ix[r, 1]; v[r, 1], ix[r, 1] = v[r, 0], ix[r, 0]; v[r, 0], ix[r, 0] = x, i
            elif x > v[r, 1] or (x == v[r, 1] and i < ix[r, 1]):
                v[r, 2], ix[r, 2] = v[r, 1], ix[r, 1]; v[r, 1], ix[r, 1] = x, i
            elif x > v[r, 2] or (x == v[r, 2] and i < ix[r, 2]):
                v[r, 2], ix[r, 2] = x, i

    for s in slices:
        offer(s.t1, col(s.t1, s.j1)); offer(s.t2, col(s.t2, s.j2)); offer(s.t3, col(s.t3, s.j3))
    best = np.maximum.reduce([s.bexact for s in slices])
    tb = np.maximum.reduce([s.t1 for s in slices])
    band = (tb - slices[0].W).astype(np.float32)
    n = sum((t > band).astype(np.int64) for s in slices for t in (s.t1, s.t2, s.t3, s.t4))
    return ix[:, 0], ix[:, 1], ix[:, 2], n, best


WN = 128   # codes per MMA step of the search kernel


def epilogue(V, W, share=True):
    """(i0, i1, i2, n, best) per row, as the kernel produces them.  V: (R, Kpad) float32; columns past Kpad score -3e38
    (the kernel seeds them so), up to a whole number of 128-code steps."""
    R, Kpad = V.shape
    steps = -(-Kpad // WN)
    Vp = np.full((R, steps * WN), np.float32(-3e38), np.float32)
    Vp[:, :Kpad] = V
    quad = [Scan(W) for _ in range(4)]                     # slice q: columns 2q, 2q + 1 of every 8-column block
    for ct in range(steps):
        if share and ct > 0:                               # the row's running maximum over the quad (two shuffles)
            m = np.maximum.reduce([s.t1 for s in quad])
            for s in quad:
                s.raise_(m)
        for q in range(4):
            for g in range(2):                             # group g: 8-column blocks 8g .. 8g + 7 of the step
                c0 = ct * WN + 64 * g + 2 * q
                quad[q].scan16(Vp[:, c0 + GROUP_COLS], c0)
    return merge([s.finish() for s in quad])


def make_scores(kind, R, K, rng):
    V = rng.standard_normal((R, K)).astype(np.float32) * np.float32(16.0) - np.float32(100.0)
    if kind == "mixed_sign":
        V = rng.standard_normal((R, K)).astype(np.float32) * np.float32(3.0)
    elif kind == "near_ties":          # several codes within a few float32 ulps .. 1e-3 of the row maximum
        top = V.max(axis=1, keepdims=True)
        for _ in range(4):
            cols = rng.integers(0, K, size=R)
            eps = (rng.random(R).astype(np.float32) ** 4) * np.float32(2e-3)
            V[np.arange(R), cols] = (top[:, 0] - eps * np.abs(top[:, 0])).astype(np.float32)
    elif kind == "exact_ties":         # exact duplicates of the maximum, in the same piece and in other pieces
        top = V.max(axis=1)
        for _ in range(3):
            cols = rng.integers(0, K, size=R)
            V[np.arange(R), cols] = top
    elif kind == "ascending":          # every element is a new maximum: the most updates possible
        V = np.sort(V, axis=1)
    elif kind == "descending":
        V = -np.sort(-V, axis=1)
    elif kind == "constant":
        V[:] = np.float32(-7.25)
    return V


@pytest.mark.parametrize("kind", ["random", "mixed_sign", "near_ties", "exact_ties", "ascending", "descending", "constant"])
@pytest.mark.parametrize("K,BN", [(1024, 256), (300, 256), (48, 48)])
@pytest.mark.parametrize("w_rel", [0.0, 2.0 ** -16, 2.0 ** -10])
def test_epilogue_certificate(kind, K, BN, w_rel):
    rng = np.random.default_rng(hash((kind, K, int(w_rel * 2 ** 20))) % (2 ** 32))
    R = 192
    V = make_scores(kind, R, K, rng)
    Kpad = -(-K // BN) * BN
    Vp = np.full((R, Kpad), np.float32(-3e38), np.float32)   # padded codes: bias -3e38, never candidates
    Vp[:, :K] = V
    vmax_abs = np.abs(V).max(axis=1)
    slack = (np.float32(2.0 ** -18) * vmax_abs).astype(np.float32)        # 2 * (16 ulp <= 2^-19 |score|)
    W = (np.float32(w_rel) * vmax_abs + slack + np.float32(1e-30)).astype(np.float32)
    i0, i1, i2, n, best = epilogue(Vp, W)

    exact_best = V.max(axis=1)
    assert np.array_equal(best, exact_best), "bexact must be the exact row maximum"
    assert ((i0 >= 0) & (i0 < K)).all(), "winner must be a real code"
    two = (n == 2) | (n == 3)
    three = n == 3
    assert ((i1[two] >= 0) & (i1[two] < K) & (i1[two] != i0[two])).all(), "second candidate must be a distinct real code"
    assert ((i2[three] >= 0) & (i2[three] < K) & (i2[three] != i0[three]) & (i2[three] != i1[three])).all(), "third candidate"

    # the certificate: a code that is not a reported candidate is at least (W - slack) below the exact maximum
    V64 = V.astype(np.float64)
    lim = exact_best.astype(np.float64) - (W.astype(np.float64) - slack.astype(np.float64))
    reported = np.zeros((R, K), bool)
    reported[np.arange(R), i0] = True
    reported[two, i1[two]] = True
    reported[three, i2[three]] = True
    many = n > 3                                   # whole-row rescan: nothing to certify
    unreported_high = (V64 > lim[:, None]) & ~reported & ~many[:, None]
    assert not unreported_high.any(), f"{int(unreported_high.any(axis=1).sum())} rows hide a candidate from the re-score"
    # hence the exact arg-max is always among the candidates handed on
    am = V64.argmax(axis=1)
    ok = many | (am == i0) | (two & (am == i1)) | (three & (am == i2)) | (V64[np.arange(R), i0] == V64[np.arange(R), am])
    assert ok.all()
    # certified rows have a strict, unique exact maximum at i0
    one = n == 1
    others = V64.copy()
    others[np.arange(R), i0] = -np.inf
    assert (others[one].max(axis=1) < V64[np.arange(R), i0][one]).all()


def test_constant_rows_go_to_the_whole_row_rescan():
    V = np.full((8, 256), np.float32(1.5), np.float32)
    W = np.full(8, np.float32(1e-6), np.float32)
    _, _, _, n, best = epilogue(V, W)
    assert (n > 3).all() and (best == np.float32(1.5)).all()
