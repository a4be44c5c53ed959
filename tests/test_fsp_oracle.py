"""CPU checks of the FSP oracle, fixtures, module surface and argument refusals (no GPU needed)."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import fsp_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fsp", "*.npz")))
STATS = ("mean", "variance", "skewness", "kurtosis")


def fixture_setup(f):
    """(kwargs, eps, z (N, d) float64, the upstream gradient at project_out's input (N, d), the draws, qrate)."""
    kw = json.loads(str(f["kwargs"]))
    d = len(kw["levels"])
    dt = torch.bfloat16 if str(f["xdtype"]) == "bf16" else torch.float32
    eps = float(f["eps"]) if np.isfinite(f["eps"]) else float(torch.finfo(dt).eps)
    z = f["z"].astype(np.float64).reshape(-1, d)
    G = f["G"].astype(np.float64)
    if kw.get("channel_first"):
        G = np.moveaxis(G, 1, -1)
    G = G.reshape(-1, G.shape[-1])
    if "sd.project_out.weight" in f:
        G = G @ f["sd.project_out.weight"].astype(np.float64)
    draws = (f["u1"].astype(np.float64), f["u2"].astype(np.float64)) if "u1" in f else (None, None)
    qrate = kw.get("quantize_rate", 0.) if bool(f["train"]) else 1.
    return kw, eps, z, G, draws, qrate


def test_fixtures_exist():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert {f"act_{a}{s}" for a in O.ACTS for s in ("", "_inv")} <= names
    assert {f"norm_{v}" for v in O.PRESETS} <= names
    assert {"rate0", "rate1", "eval", "image_channel_first", "proj_dim256", "levels_2_mixed", "explicit_eps", "readme_basic",
            "readme_eval", "bf16_eval", "bf16_train", "large_offset"} <= names


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_reproduces_fixture(path):
    """The float64 oracle against the reference's float64 rerun: the row chain away from bin edges, the moments, the loss and
    the gradient at z (the closed form plus the CDF derivative)."""
    f = np.load(path)
    kw, eps, z, G, (u1, u2), qrate = fixture_setup(f)
    levels, act, inv = kw["levels"], kw.get("act_name", "tanh"), kw.get("need_inv_act", False)
    norm = O.PRESETS[kw.get("vector_norm", "var_tanh")]
    d = len(levels)
    q, idx, lev, _ = O.row_chain(z, levels, act, inv, eps, u1, u2, qrate)
    bf16 = str(f["xdtype"]) == "bf16"
    far = ~O.near_integer(O.pre_floor(z, levels, act, eps), 2. ** -6 if bf16 else 2. ** -19)   # bf16 rounds act L to 8 bits
    assert far.mean() > 0.7
    np.testing.assert_array_equal(lev[far], f["level_indices"].reshape(-1, d)[far])
    proj = kw.get("dim") not in (None, d)
    rows = far.all(-1)
    if not proj:
        q64 = f["q64"]
        if kw.get("channel_first"):
            q64 = np.moveaxis(q64, 1, -1)
        np.testing.assert_allclose(q[rows], q64.reshape(-1, d)[rows], rtol=1e-9, atol=1e-9)
    # with projections the float64 rerun's z is the double matmul, not the fp32 z stored here
    tol = 1e-5 if proj else 1e-9
    stats = O.moments(z)
    for k, s in enumerate(STATS):
        np.testing.assert_allclose(stats[k], f["stat64_" + s], rtol=tol, atol=tol)
    np.testing.assert_allclose(O.norm_loss(stats, norm), float(f["loss64"]), rtol=tol, atol=1e-12)
    Gs = f["H"].astype(np.float64) + O.norm_loss_grad_weights(stats, norm, d)
    gq = G if inv else G / O.UNIT_STD * O.act_grad_f64(act, z)
    dz = gq + O.stats_grad(z, Gs)
    dz64 = f["dz64"].reshape(-1, d)
    np.testing.assert_allclose(dz, dz64, rtol=1e-4 if proj else 1e-7, atol=(1e-5 if proj else 1e-9) * np.abs(dz64).max())


@pytest.mark.parametrize("case", ["randn", "offset", "constant", "tiny", "two_rows"])
def test_closed_form_gradient_matches_autograd(case):
    g = np.random.default_rng(7)
    z = g.standard_normal((64, 5))
    if case == "offset":
        z[:, 1] += 1e3
    elif case == "constant":
        z[:, 2] = 0.25                    # std 0: the clamp at 1e-8 is active (mask 0)
    elif case == "tiny":
        z[:, 3] = 0.5 + 1e-10 * z[:, 3]   # std ~1e-10, clamped
    elif case == "two_rows":
        z = z[:2]
    G = g.standard_normal((4, z.shape[1]))
    ref = O.stats_grad_autograd(z, G)
    ours = O.stats_grad(z, G)
    if case == "constant":   # autograd meets sqrt'(0) = inf times the clamp's zero gradient: NaN; the closed form masks it
        assert np.isnan(ref[:, 2]).all() and np.isfinite(ours).all()
        ref, ours = np.delete(ref, 2, 1), np.delete(ours, 2, 1)
    np.testing.assert_allclose(ours, ref, rtol=1e-9, atol=1e-9 * max(np.abs(ref).max(), 1.))


def test_bf16_fixture_pins_the_index_deviation():
    """The reference's bf16 indices are the bf16 sum of level_indices * basis; ours are the exact mixed-radix index."""
    f = np.load(os.path.join(HERE, "golden", "fsp", "bf16_eval.npz"))
    lev = f["level_indices"].reshape(-1, 4).astype(np.int64)
    exact = (lev * O.basis([8, 5, 5, 5])).sum(-1)
    assert (exact != f["indices"].reshape(-1)).sum() > 1000


def _make(kw, seed):
    import vector_quantize_pytorch_b200 as vqb
    torch.manual_seed(seed)
    return vqb.FSP(**kw)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_state_dict_and_seeded_weights(path):
    f = np.load(path)
    m = _make(json.loads(str(f["kwargs"])), int(f["seed"]))
    sd = {k[3:]: f[k] for k in f.files if k.startswith("sd.")}
    assert sorted(m.state_dict().keys()) == sorted(sd.keys())
    for k, v in m.state_dict().items():
        np.testing.assert_array_equal(v.numpy(), sd[k])


def test_module_surface():
    m = _make(dict(levels=[8, 5, 5, 5], dim=16, act_name="laplace", vector_norm="kurt"), 0)
    assert m.codebook_size == 1000 and m.codebook_dim == 4 and m.has_projections
    assert m._levels.tolist() == [8, 5, 5, 5] and m._basis.tolist() == [1, 8, 40, 200]
    assert "_levels" not in m.state_dict() and "_basis" not in m.state_dict()
    assert (m.vector_norm.l3_weight, m.vector_norm.l4_weight, m.vector_norm.l2_target) == (0.06, 0.05, 1.0)
    assert repr(m).splitlines()[1:] == ["  levels=[8, 5, 5, 5],", "  codebook_size=1000,", "  codebook_dim=4,", "  dim=16,",
                                        "  act_name='laplace',", "  need_inv_act=False,", "  quantize_rate=0.0", ")"]
    li = torch.tensor([[[7, 4, 4, 4]]])
    assert m.level_indices_to_indices(li).item() == 7 + 4 * 8 + 4 * 40 + 4 * 200
    assert torch.equal(m.indices_to_level_indices(m.level_indices_to_indices(li)), li)


def test_refusals():
    import vector_quantize_pytorch_b200 as vqb
    with pytest.raises(NotImplementedError):
        vqb.FSP(levels=[2] * 17)
    with pytest.raises(NotImplementedError):
        vqb.FSP(levels=[65536, 32768])
    with pytest.raises(AssertionError):
        vqb.FSP(levels=[8, 5], act_name="softsign")
    with pytest.raises(AssertionError):
        vqb.FSP(levels=[8, 5], vector_norm="skew")
    with pytest.raises(AssertionError):
        vqb.FSP(levels=[8, 5], quantize_rate=1.5)
    m = vqb.FSP(levels=[8, 5])
    with pytest.raises(TypeError):
        m(torch.randn(4, 2, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.randn(4, 2))


def test_fsp_argument_errors_are_return_codes_not_crashes():
    """vqb_fsp_* refuse null pointers, d > 16, unknown dtypes and CDFs, and unaligned planes before any CUDA call."""
    import ctypes
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced
    f = _C.DTYPE_F32
    norm = (ctypes.c_double * 8)()

    def fwd(z=p, dt=f, D=4, act=0, levels=p, u1=None, u2=None, out=p, idx=p, lev=p, acc=None):
        return lib.vqb_fsp_forward(z, dt, 8, D, act, 0, levels, 0.99, u1, u2, 0.5, 1e-6, 0.99, out, idx, lev, acc, 1, None)

    def stats(z=p, dt=f, D=4, work=p, st=p, loss=p, aux=p, nrm=norm):
        return lib.vqb_fsp_stats(z, dt, 8, D, nrm, work, 1, st, loss, aux, None)

    def bwd(z=p, dt=f, D=4, act=0, g=p, gdt=f, aux=p, gz=p, nrm=norm):
        return lib.vqb_fsp_backward(z, dt, 8, D, act, 0, g, gdt, aux, None, None, nrm, gz, None)

    def dec(idx=p, D=4, act=0, levels=p, a=p, c=None):
        return lib.vqb_fsp_decode(idx, 0, 8, D, act, 1, levels, 1e-6, 0.99, a, c, None)

    for call in (fwd, stats, bwd):
        assert call(z=None) == -1 and call(dt=7) == -1 and call(D=17) == -2 and call(D=0) == -1
        assert call(z=p + 4) == -3
    for call in (fwd, bwd, dec):
        assert call(act=5) == -1 and call(act=-1) == -1
    assert fwd(levels=None) == -1 and fwd(out=None) == -1 and fwd(idx=None) == -1
    assert fwd(u1=p) == -1 and fwd(u1=p, u2=p) == -1   # one draw alone; draws without accept counts
    assert fwd(out=p + 4) == -3 and fwd(lev=p + 8) == -3 and fwd(u1=p + 4, u2=p, acc=p) == -3
    assert stats(work=None) == -1 and stats(st=None) == -1 and stats(loss=None) == -1 and stats(aux=None) == -1
    assert stats(nrm=None) == -1
    assert bwd(aux=None) == -1 and bwd(gz=None) == -1 and bwd(gdt=7) == -1 and bwd(g=p + 4) == -3 and bwd(gz=p + 4) == -3
    assert dec(idx=None) == -1 and dec(levels=None) == -1 and dec(a=None) == -1 and dec(D=17) == -2
    assert dec(a=p + 4) == -3 and dec(a=None, c=p + 4) == -3
    assert lib.vqb_fsp_blocks(0) == -1 and lib.vqb_fsp_blocks(1 << 31) == -2
