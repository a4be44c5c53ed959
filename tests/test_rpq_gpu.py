"""RandomProjectionQuantizer on the GPU: replay of the reference's calls (tests/golden/rpq/, oracle/gen_golden_rpq.py) with the
reference's k-means draws substituted for ours; the BEST-RQ and USM-like shapes over many rows against a float64 search; and
Sequential against calling its layers by hand.

At the large shapes the kernel's rows must lie within its bound (oracle/rpq_oracle.py) of the float64 rows, and the indices
must equal the float64 search's wherever the float64 lead exceeds the error propagated from the rows: their measured error,
through project_in with its own fp32 rounding bound (|W| e + 2 g(n + 1) (|W| |r| + |b|) + 2u), then 2 |e| / |r| per cosine
score, twice for a lead, plus the error of the search's own scores.  That last term: every row gets the index of the
reference's fp32 formula (DESIGN §4.1-4.2: certified by the band or re-scored with that formula), l2norm(r) . c in fp32.
The l2norm moves each element by at most g(D / 2 + 3) relative (a D-term sum of squares, a sqrt and a division), and the
D-term dot adds g(D) sum |r_d c_d| <= g(D) |c|, so a score is within g(3D / 2 + 3) max|c| of float64 to first order, and a
lead within twice that; it enters with the safety factor 2.  Rows under the whole bound are counted and printed; where such
a row's index differs, its code's float64 score must lie within the bound of the best.
"""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import rpq_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "rpq")
FIXTURES = sorted(p[:-4] for p in os.listdir(GOLDEN) if p.endswith(".npz"))


class _Replay:
    def __init__(self, kinds, arrays):
        self.draws = list(zip(kinds, arrays))

    def take(self, kind, device):
        assert self.draws, f"the module drew more from the RNG than the reference ({kind})"
        k, a = self.draws.pop(0)
        assert k == kind, (k, kind)
        return torch.from_numpy(a).to(device)


@pytest.fixture(autouse=True)
def full_fp32_matmul(monkeypatch):
    """project_in is torch's nn.Linear and follows torch's precision settings; the fp32 reference ran it in fp32."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.mark.parametrize("name", FIXTURES)
def test_replays_reference(name, monkeypatch):
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(bytes(f["meta"]).decode())
    torch.manual_seed(meta["seed"])
    rpq = m.RandomProjectionQuantizer(**meta["kw"])
    digests = json.loads(str(f["sd_sha256"]))
    assert [hashlib.sha256(v.numpy().tobytes()).hexdigest() for v in rpq.state_dict().values()] == digests
    rpq = rpq.to(DEV)
    norm = meta["kw"].get("norm", True)
    P = rpq.rand_projs.cpu().numpy()
    for s in range(meta["calls"]):
        if s > 0:
            rpq.train()
        kinds = json.loads(str(f[f"rng_kinds_{s}"]))
        replay = _Replay(kinds, [f[f"rng_{s}_{j}"] for j in range(len(kinds))])
        x = torch.from_numpy(f[f"x_{s}"]).to(DEV)
        with monkeypatch.context() as mp:
            mp.setattr(torch, "randperm", lambda *a, device=None, **k: replay.take("randperm", device))
            mp.setattr(torch, "randint", lambda *a, device=None, **k: replay.take("randint", device))
            ind = rpq(x)
        assert not replay.draws, "the module drew less from the RNG than the reference"
        assert not rpq.vq.training
        assert ind.dtype == torch.int64 and ind.shape == f[f"indices_{s}"].shape
        np.testing.assert_array_equal(ind.cpu().numpy(), f[f"indices_{s}"], err_msg=f"call {s}")
        rows = ops.rpq_norm_project(x, rpq.rand_projs, norm).cpu().numpy()
        xf = f[f"x_{s}"].reshape(-1, P.shape[1])
        assert (np.abs(rows - f[f"rows64_{s}"]) <= O.row_bound(xf, P, norm)).all(), f"call {s}: rows outside the bound"


def _large(kw, B, n, seed):
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import ops
    torch.manual_seed(seed)
    rpq = m.RandomProjectionQuantizer(**kw).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, n, kw["dim"], device=DEV, generator=g) * 1.5 + 0.25
    ind = rpq(x).reshape(B * n, -1)
    # float64 rows, their bound, project_in, its bound
    proj = rpq.rand_projs
    H, dim, E = proj.shape
    xd = x.reshape(-1, dim).double()
    P = proj.double().permute(1, 0, 2).reshape(dim, H * E)
    mean = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mean) ** 2).mean(-1, keepdim=True) + O.EPS)
    xn = (xd - mean) * rstd
    rows = xn @ P
    dm = O.gamma(dim + 1) * xd.abs().sum(-1, keepdim=True) / dim
    er = 1.5 * O.gamma(dim + 4) + 2 * O.U
    bound = O.SAFETY * (O.gamma(dim) * (xn.abs() @ P.abs()) + ((er + 2 * O.U) * xn.abs() + 2 * dm * rstd) @ P.abs())
    ours_rows = ops.rpq_norm_project(x, proj, True).double()
    assert bool(((ours_rows - rows).abs() <= bound).all())
    # from here on the rows' measured error, which the line above holds within the kernel's bound
    bound = (ours_rows - rows).abs()
    if H > 1:
        Wt, b = rpq.vq.project_in.weight.double(), rpq.vq.project_in.bias.double()
        y = rows @ Wt.T + b
        bound = bound @ Wt.abs().T + O.SAFETY * (O.gamma(Wt.shape[1] + 1) * (rows.abs() @ Wt.abs().T + b.abs()) + O.U)
        rows = y
    embeds = rpq.vq._codebook.embed.double()
    D = rows.shape[1] // H
    n_close = 0
    for h in range(H):
        r, e = rows[:, h * D:(h + 1) * D], bound[:, h * D:(h + 1) * D]
        rn = r.norm(dim=-1)
        scores = (r / rn[:, None]) @ embeds[h].T
        top2 = scores.topk(2, dim=-1)
        lead = top2.values[:, 0] - top2.values[:, 1]
        search = O.SAFETY * 2 * O.gamma(1.5 * D + 3) * float(embeds[h].norm(dim=-1).max())
        slack = 4 * e.norm(dim=-1) / rn + search
        ours = ind[:, h]
        sure = lead > slack
        assert torch.equal(ours[sure], top2.indices[sure, 0]), f"head {h}: {int((ours[sure] != top2.indices[sure, 0]).sum())} rows"
        close = ~sure
        n_close += int(close.sum())
        got = scores[close].gather(1, ours[close][:, None])[:, 0]
        assert bool((top2.values[close, 0] - got <= slack[close]).all()), f"head {h}: a close row's code is outside the bound"
    print(f"{kw}: {B * n} rows x {H} heads, {n_close} under the bound")


def test_bestrq_shape_against_float64():
    """dim 320, one codebook of 8192 16-wide codes (the first search at D = 16, K = 8192), 2^16 frames."""
    _large(dict(dim=320, codebook_size=8192, codebook_dim=16), 16, 4096, 1)


def test_usm_shape_against_float64():
    """dim 512, 16 codebooks of 1024 codes; each head searches 256-wide rows after project_in (256 -> 4096), 2^15 frames."""
    _large(dict(dim=512, codebook_size=1024, codebook_dim=16, num_codebooks=16), 8, 4096, 2)


def test_sequential_matches_layers_by_hand():
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(3)
    pre = torch.nn.Linear(24, 64).to(DEV)
    rpq = m.RandomProjectionQuantizer(dim=64, codebook_size=128, codebook_dim=8, num_codebooks=2).to(DEV)
    x = torch.randn(2, 50, 24, device=DEV)
    with torch.no_grad():
        want = rpq(pre(x))
        out = m.Sequential(pre, rpq)(x)
    # the reference's `x, *rest = fn(x)` unpacks RPQ's bare index tensor along its first axis
    assert len(out) == 2 and torch.equal(out[0], want[0]) and torch.equal(out[1], want[1])

    vq = m.VectorQuantize(dim=64, codebook_size=128).to(DEV).eval()
    post = torch.nn.Linear(64, 8).to(DEV)
    with torch.no_grad():
        q, i, loss = vq(pre(x))
        q = post(q)
        got = m.Sequential(pre, vq, post)(x)
    assert len(got) == 3 and torch.equal(got[0], q) and torch.equal(got[1], i) and torch.equal(got[2], loss)


_LAYOUTS = [
    dict(),                                                          # one head
    dict(heads=4, codebook_dim=16),                                  # heads sharing one codebook: '1 (b h) n -> b n h'
    dict(heads=4, codebook_dim=16, separate_codebook_per_head=True),  # one codebook per head
    dict(heads=2, codebook_dim=16),                                  # project_in (64 -> 32), shared codebook
    dict(heads=2, codebook_dim=16, separate_codebook_per_head=True, kmeans_init=True),
]


# project_in is an fp32 nn.Linear, which takes fp32 inputs only: bf16 goes with the layouts without it
@pytest.mark.parametrize("kw,dtype", [(kw, torch.float32) for kw in _LAYOUTS]
                         + [(kw, torch.bfloat16) for kw in _LAYOUTS[:3]])
def test_eval_indices_equal_eval_forward(kw, dtype):
    """VectorQuantize.eval_indices returns what an eval forward returns as its indices, on every head layout (k-means init
    included: two copies of the module, each initialised by its own first call with the same draws)."""
    import copy
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(5)
    vq = m.VectorQuantize(dim=64, codebook_size=256, use_cosine_sim=True, **kw).to(DEV).eval()
    other = copy.deepcopy(vq)
    x = torch.randn(3, 300, 64, device=DEV).to(dtype)
    with torch.no_grad():
        torch.manual_seed(6)
        _, want, _ = vq(x)
        torch.manual_seed(6)
        got = other.eval_indices(x)
    assert got.dtype == torch.int64 and got.shape == want.shape
    assert torch.equal(got, want)
