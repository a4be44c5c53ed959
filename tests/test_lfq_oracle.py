"""CPU checks of the LFQ oracle, fixtures, module surface and argument refusals (no GPU needed)."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import lfq_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "lfq", "*.npz")))


@pytest.mark.parametrize("d", [1, 2, 5, 8, 11])
@pytest.mark.parametrize("tau", [1e-3, 1.0, 100.0])
def test_factorised_equals_dense(d, tau):
    g = torch.Generator().manual_seed(d)
    x = torch.randn(7, d, generator=g, dtype=torch.float64)
    hd, cd = O.dense_stats(x, 0.75, tau)
    hf, cf = O.factored_stats(x, 0.75, tau)
    torch.testing.assert_close(hf, hd, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(cf, cd, rtol=1e-12, atol=1e-12)


def test_fixtures_exist():
    names = {os.path.basename(f)[:-4] for f in FIXTURES}
    assert {"lfq_readme_image", "lfq_mask", "lfq_frac_mask", "rlfq_readme_train", "grlfq_groups2", "rlfq_frac",
            "grlfq_frac_mask"} <= names
    for path in FIXTURES:   # the float64 run that sets each fixture's tolerance
        f = np.load(path)
        assert "losses64" in f and all(f"gz64_{j}" in f for j in range(sum(k.startswith("gz64_") for k in f.files)))


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_reproduces_fixture_breakdown(path):
    """PSE and CBE of the fixture's LFQ from z through the float64 oracle (no mask, no sampling, no projection-free rotation)."""
    f = np.load(path)
    if str(f["cls"]) != "LFQ" or "breakdown" not in f or not bool(f["train"]) or "mask" in f:
        pytest.skip("oracle replay covers unmasked, unsampled LFQ training cases")
    kw = json.loads(str(f["kwargs"]))
    if kw.get("frac_per_sample_entropy", 1.) < 1 or kw.get("orthogonal_rotation") or kw.get("spherical") \
            or kw.get("soft_clamp_input_value"):
        pytest.skip("input transform before the entropy is not restated here")
    tau = json.loads(str(f["fkw"])).get("inv_temperature", 100.)
    d = int(np.log2(kw["codebook_size"]))
    c = kw.get("num_codebooks", 1)
    z = torch.from_numpy(f["z0"]).double().reshape(-1, c, d) if "z0" in f else \
        torch.from_numpy(f["x"]).double().movedim(1, -1).reshape(-1, c, d)
    s = kw.get("codebook_scale", 1.)
    pse, cbe = 0., 0.
    for g in range(c):
        hs, col = O.dense_stats(z[:, g], s, tau)
        pse += float(hs) / (z.shape[0] * c)
        cbe += float(O.h(col / z.shape[0]).sum()) / c
    np.testing.assert_allclose([pse, cbe], f["breakdown"][:2], rtol=2e-5, atol=1e-7)


def test_state_dict_keys_and_buffers():
    import vector_quantize_pytorch_b200 as vqb
    torch.manual_seed(0)
    m = vqb.LFQ(codebook_size=256, dim=32, orthogonal_rotation=True)
    assert list(m.state_dict().keys()) == ["orthogonal_rot", "mask", "project_in.weight", "project_in.bias", "project_out.weight",
                                           "project_out.bias"]
    assert m.codebook.shape == (256, 8) and m.codebook.dtype == torch.float32
    r = vqb.ResidualLFQ(dim=64, codebook_size=256, num_quantizers=3, soft_clamp_input_value=4.)
    assert [l.codebook_scale for l in r.layers] == [1, 0.5, 0.25]
    assert [l.soft_clamp_input_value for l in r.layers] == [4., 2., 1.]
    assert r.codebooks.shape == (3, 256, 8)


def test_fixture_state_dicts_load():
    import vector_quantize_pytorch_b200 as vqb
    for path in FIXTURES:
        f = np.load(path)
        kw = json.loads(str(f["kwargs"]))
        torch.manual_seed(int(f["seed"]))
        mod = getattr(vqb, str(f["cls"]))(**kw)
        sd = {k[3:]: torch.from_numpy(f[k]) for k in f.files if k.startswith("sd.")}
        for k, v in mod.state_dict().items():   # a seeded construction gives the reference's weights
            assert torch.equal(v, sd[k].to(v.dtype)), (path, k)
        assert set(sd) == set(mod.state_dict())


def test_refusals():
    import vector_quantize_pytorch_b200 as vqb
    with pytest.raises(NotImplementedError):
        vqb.LFQ(codebook_size=16, straight_through_activation=torch.nn.Tanh())
    with pytest.raises(NotImplementedError):
        vqb.LFQ(codebook_size=16, force_quantization_f32=False)
    with pytest.raises(NotImplementedError):
        vqb.LFQ(codebook_size=2 ** 21)
    with pytest.raises(NotImplementedError):
        vqb.ResidualLFQ(dim=8, codebook_size=256, num_quantizers=2, orthogonal_rotation=True)
    with pytest.raises(NotImplementedError):
        vqb.ResidualLFQ(dim=8, codebook_size=256, num_quantizers=65)


def test_abi_argument_errors():
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    E_INVALID, E_UNSUPPORTED = -1, -2
    assert lib.vqb_lfq_forward(None, 0, 4, 1, 4, 1, 1, 0, 1, 0, None, None, None, 0, 0, 0, None, None, None, 0, None) == E_INVALID
    assert lib.vqb_lfq_forward(1 << 20, 0, 4, 1, 21, 1, 1, 0, 1, 0, 1 << 20, 1 << 20, 1 << 20, 0, 0, 0, None, None, None, 0,
                               None) == E_UNSUPPORTED
    assert lib.vqb_lfq_entropy(None, 4, 1, 4, 1, None, 4, 0, None, 1.0, 1, None, None, None) == E_INVALID
    assert lib.vqb_lfq_entropy(1 << 20, 4, 1, 21, 1, None, 4, 0, 1 << 20, 1.0, 1, 1 << 20, None, None) == E_UNSUPPORTED
    assert lib.vqb_lfq_entropy_backward(1 << 20, 4, 1, 4, 1, None, 4, 0, 1 << 20, 1.0, 1 << 20, None, 3, 1 << 20, 1 << 20,
                                        None) == E_INVALID   # ksplit not a power of two
    assert lib.vqb_lfq_decode(None, 1, 0, 0, 0, 4, 1, 4, 1, None, None, None, None) == E_INVALID
    assert lib.vqb_lfq_entropy_tiles(0) == E_UNSUPPORTED and lib.vqb_lfq_entropy_tiles(18) == 64
    # the row kernels' shape checks run before the device check: Q, n_active, N * G, and the backward's own pointers
    P = 1 << 20

    def fwd(N=4, G=1, D=4, Q=2, na=2):
        return lib.vqb_lfq_forward(P, 0, N, G, D, Q, na, 1, 1, 0, P, P, P, 0, 0, 0, None, None, None, 0, None)

    def bwd(N=4, G=1, D=4, Q=2, na=2, gout=P, gz=P):
        return lib.vqb_lfq_backward(P, 0, N, G, D, Q, na, 1, 1, 0, P, gout, None, None, None, gz, None)

    for f in (fwd, bwd):
        assert f(Q=65, na=1) == E_UNSUPPORTED
        assert f(na=0) == E_INVALID and f(na=3) == E_INVALID and f(Q=0, na=0) == E_INVALID
        assert f(N=1 << 30, G=2) == E_UNSUPPORTED   # N * G = 2^31
        assert f(D=0) == E_UNSUPPORTED and f(N=0) == E_INVALID
    assert lib.vqb_lfq_forward(P, 2, 4, 1, 4, 2, 2, 1, 1, 0, P, P, P, 0, 0, 0, None, None, None, 0, None) == E_INVALID   # fp16
    assert lib.vqb_lfq_forward(P, 0, 4, 1, 4, 2, 2, 1, 1, 0, P, P, P, 0, 0, 0, None, None, P, 0, None) == E_INVALID   # no blocks
    assert bwd(gout=None) == E_INVALID and bwd(gz=None) == E_INVALID
    assert lib.vqb_lfq_decode(P, 1, 0, 0, 0, 4, 1, 4, 65, P, P, None, None) == E_UNSUPPORTED
    assert lib.vqb_lfq_decode(P, 1, 0, 0, 0, 1 << 30, 2, 4, 1, P, P, None, None) == E_UNSUPPORTED
    assert lib.vqb_lfq_decode(P, 1, 0, 0, 0, 4, 1, 21, 1, P, P, None, None) == E_UNSUPPORTED
    assert lib.vqb_lfq_decode(P, 1, 0, 0, 0, 4, 1, 4, 0, P, P, None, None) == E_INVALID
    assert lib.vqb_lfq_decode(P, 1, 0, 0, 0, 4, 1, 4, 1, P, None, None, None) == E_INVALID   # neither out nor codes


# ---- the entropy kernels' error bounds (oracle/lfq_oracle.py::entropy_reference): they hold for fp32 arithmetic and have teeth

def _rows(d, R, seed):
    """Generic rows, zero rows and rows whose every |a_j| puts codes on both sides of the 1e-5 clamp, fp32 values."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, d, generator=g, dtype=torch.float64) * torch.logspace(-1, 0.5, R, dtype=torch.float64)[:, None]
    x[R // 3] = 0.
    return x.float().double()


def _emulate(x, m, tau, cp, V, chunks, ksplit):
    """The kernels' arithmetic restated in fp32 on the CPU (torch's expf / log1pf / exp2 / tanh stand in for CUDA's), in one
    of the summation orders the bounds allow.  -> (pse, colsum (K,), grad (R, d)), float64 views of the fp32 results."""
    f = torch.float32
    R, d = x.shape
    K = 1 << d
    x = x.float()
    tm = torch.tensor(2 * tau, dtype=f) * torch.tensor(m, dtype=f)
    av = tm * x
    log2e, ln2 = torch.tensor(1.4426950408889634, dtype=f), torch.tensor(0.6931471805599453, dtype=f)
    lo2, lne = torch.tensor(O.LOG2_EPS, dtype=f), torch.tensor(O.LN_EPS, dtype=f)

    def nsp2(y):
        return -(y.clamp(min=0) + torch.log1p(torch.exp(-y.abs()))) * log2e

    l1, l0 = nsp2(-2 * av), nsp2(2 * av)
    bits = O._code_bits(d, "cpu").bool()
    lp = torch.zeros((R, K), dtype=f)
    for j in range(d):
        lp = lp + torch.where(bits[:, j], l1[:, j:j + 1], l0[:, j:j + 1])
    p = torch.exp2(lp)
    hs = -p * torch.where(lp >= lo2, lp * ln2, lne)
    pse = hs.double().sum()
    cr = -(-R // chunks)
    col = torch.zeros(K, dtype=f)
    for c in range(chunks):
        part = torch.zeros(K, dtype=f)
        for r in range(c * cr, min(R, (c + 1) * cr)):
            part = part + p[r]
        col = col + part
    hp = torch.where(lp >= lo2, -(lp.double() * ln2.double() + 1).float(), -lne)
    u = (float(np.float32(cp)) * hp.double() + V.double()[None]).float()   # one fma
    w = p * u
    sgn = O.codebook_signs(d).float()
    L = min(K, 16)
    seg = w.view(R, K // L, L, 1) * sgn.view(1, K // L, L, d)
    s16 = torch.zeros((R, K // L, d + 1), dtype=f)
    for i in range(L):   # the 16-code fp32 sums of w sgn_kj and of w
        s16 = s16 + torch.cat([seg[:, :, i], w.view(R, K // L, L)[:, :, i, None]], -1)
    parts = s16.double().view(R, ksplit, -1, d + 1).sum(2).float()
    tot = torch.zeros((R, d + 1), dtype=f)
    for k in range(ksplit):
        tot = tot + parts[:, k]
    grad = tm * (tot[:, :d] - tot[:, d:] * torch.tanh(tm * x))
    return pse, col.double(), grad.double()


@pytest.mark.parametrize("d,R,chunks,ksplit", [(2, 40, 3, 1), (5, 90, 2, 2), (9, 70, 3, 8), (12, 33, 2, 16)])
@pytest.mark.parametrize("tau", [1e-3, 1.0, 100.0])
def test_entropy_bounds_hold_for_fp32(d, R, chunks, ksplit, tau):
    tau = float(np.float32(tau))
    x = _rows(d, R, d)
    g = torch.Generator().manual_seed(1)
    V = (torch.randn(1 << d, generator=g) * 1e-2).float()
    cp, m = 0.75, 0.8125
    ref = O.entropy_reference(x, m, tau, cp, V)
    _, gref = O.loss_and_grad(x, m, tau, cp, V)
    torch.testing.assert_close(ref.grad, gref, rtol=1e-10, atol=1e-12 * float(gref.abs().max()))   # float64 autograd's gradient
    hs, cs = O.dense_stats(x, m, tau)
    torch.testing.assert_close(ref.pse, hs, rtol=1e-12, atol=0)
    torch.testing.assert_close(ref.colsum, cs, rtol=1e-12, atol=0)
    pb, cb, gb = ref.bounds(chunks, ksplit)
    pse, col, grad = _emulate(x, m, tau, cp, V, chunks, ksplit if (1 << d) // ksplit >= 16 else 1)
    assert abs(float(pse - ref.pse)) <= pb
    assert ((col - ref.colsum).abs() <= cb).all()
    assert ((grad - ref.grad).abs() <= gb).all()


def test_entropy_bounds_have_teeth():
    """Each wrong answer below falls outside the bound, on every row of a moderate batch (d = 10, tau = 1)."""
    d, R, tau, m, cp = 10, 48, 1.0, 0.8125, 0.75
    K = 1 << d
    chunks, ksplit = 2, 2
    g = torch.Generator().manual_seed(3)
    x = torch.randn(R, d, generator=g, dtype=torch.float64).float().double()
    V = (torch.randn(K, generator=g) * 1e-2).float()
    ref = O.entropy_reference(x, m, tau, cp, V)
    pb, cb, gb = ref.bounds(chunks, ksplit)
    b = O.entropy_block(x, m, tau, cp, V)
    p, w = b["p"], b["w"]
    sgn = O.codebook_signs(d)
    contrib = ref.tm * (w[:, :, None] * (sgn[None] - ref.t[:, None, :]))   # (R, K, d): code k's part of grad[r, j]

    def outside(err, bound):
        return bool((err.abs() > bound).any())

    for r in range(R):
        # one row's contribution missing from its chunk's column sums
        assert outside(p[r], cb), r
        assert abs(float(O.h(p[r]).sum())) > pb, r
        # one 16-code segment (the row's largest) and one K split missing from the row's gradient
        segs = contrib[r].view(K // 16, 16, d).sum(1)
        assert outside(segs[segs.abs().amax(1).argmax()], gb[r]), r
        for half in contrib[r].view(ksplit, K // ksplit, d).sum(1):
            assert outside(half, gb[r]), r
        # one code's probability doubled (the row's most likely code)
        k = int(p[r].argmax())
        assert outside(p[r, k:k + 1], cb[k:k + 1]), r
        # the row's gradient replaced by 0
        assert outside(ref.grad[r], gb[r]), r
