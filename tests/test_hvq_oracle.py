"""CPU checks of HierarchicalVQ: the float64 oracle (oracle/hvq_oracle.py) against the reference's fixtures and against autograd
of torch's own pool / interpolate, the phi mapping, seeded state_dict parity, the refusals and the C ABI's argument errors
(all returned before any CUDA call)."""
import glob
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hvq_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "hvq", "*.npz")))
IDS = [os.path.basename(p)[:-4] for p in FIXTURES]


def load(path):
    f = np.load(path)
    return f, json.loads(bytes(f["meta"]).decode())


def phis_of(f, meta):
    """(weight, bias, r) of every phi, from the fixture's initial state_dict (phi is not trained by the step)."""
    keys = json.loads(str(f["sd_keys"]))
    sd = {k: f[f"sd_{j}"] for j, k in enumerate(keys)}
    r = abs(float(meta["kw"].get("quant_resi", 0.5)))
    if "phi_shared.conv.weight" in sd:
        return [(sd["phi_shared.conv.weight"], sd["phi_shared.conv.bias"], r)]
    return [(sd[f"phi_levels.{i}.conv.weight"], sd[f"phi_levels.{i}.conv.bias"], r) for i in range(meta["n_phi"])]


def test_fixtures_exist():
    assert {"ref_train", "ref_eval", "ref_two_steps", "share0_5s", "share1_5s", "share2_5s", "share3_5s", "resi0", "resi_neg05",
            "nonsquare_9x12", "scale_above_h", "dup_scales", "rotation", "no_kmeans_no_expiry"} <= set(IDS)


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_oracle_reproduces_fixture(path):
    """The float64 chain on the reference's codes: the pooled input of every scale within fp32 rounding of the reference's, the
    indices the nearest codes of the searched codebook, the reconstruction within the fp32 reference's distance of the stored
    float64 rerun, and get_output_from_indices at (scales[-1], scales[-1])."""
    f, meta = load(path)
    scales, phis = meta["scales"], phis_of(f, meta)
    for s in range(meta["steps"]):
        x = f[f"x_{s}"]
        B, D = x.shape[:2]
        codes = [f[f"s{s}_k{k}_codes"].astype(np.float64).reshape(B, sc, sc, D).transpose(0, 3, 1, 2)
                 for k, sc in enumerate(scales)]
        recon, pooled = O.forward(x, scales, codes, phis, 0)
        for k, sc in enumerate(scales):
            p_ref = f[f"s{s}_k{k}_pooled"]
            np.testing.assert_allclose(pooled[k], p_ref, rtol=0, atol=1e-5 * max(np.abs(pooled[k]).max(), 1.0))
            rows = p_ref.astype(np.float64).transpose(0, 2, 3, 1).reshape(-1, D)
            cb = f[f"s{s}_k{k}_searched"].astype(np.float64)
            d = ((rows[:, None] - cb[None]) ** 2).sum(-1)
            ind = f[f"s{s}_k{k}_indices"].reshape(-1)
            np.testing.assert_array_equal(d[np.arange(len(ind)), ind], d.min(1))
            np.testing.assert_array_equal(f[f"s{s}_k{k}_codes"].reshape(-1, D), cb[ind].astype(np.float32))
        r64 = f[f"recon64_{s}"]
        np.testing.assert_allclose(recon, r64, rtol=0, atol=1e-12 * max(np.abs(r64).max(), 1.0))
        err = np.abs(f[f"recon_{s}"] - r64).max()
        assert err <= 1e-5 * np.abs(r64).max(), err
    np.testing.assert_allclose(f["gofi"], f["gofi64"], rtol=0, atol=1e-5 * np.abs(f["gofi64"]).max())


SHAPES = [(1, 1, 1), (3, 3, 1), (7, 7, 4), (7, 5, 3), (5, 5, 7), (9, 12, 5), (2, 3, 5), (16, 16, 13), (4, 17, 6)]


@pytest.mark.parametrize("H,W,s", SHAPES)
def test_pool_and_adjoint_match_autograd(H, W, s):
    g = torch.Generator().manual_seed(H * 100 + W * 10 + s)
    x = torch.randn(2, 3, H, W, dtype=torch.float64, generator=g, requires_grad=True)
    y = F.adaptive_avg_pool2d(x, (s, s))
    np.testing.assert_allclose(O.pool(x.detach().numpy(), s), y.detach().numpy(), rtol=1e-13, atol=1e-13)
    gy = torch.randn(y.shape, dtype=torch.float64, generator=g)
    y.backward(gy)
    np.testing.assert_allclose(O.pool_adjoint(gy.numpy(), H, W), x.grad.numpy(), rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("H,W,s", SHAPES)
def test_upsample_and_adjoint_match_autograd(H, W, s):
    """torch's float64 interpolate takes its source index in float64, the oracle (like the fp32 kernels) in fp32: the taps'
    weights differ by fp32 rounding of the source index."""
    g = torch.Generator().manual_seed(H * 100 + W * 10 + s + 1)
    q = torch.randn(2, 3, s, s, dtype=torch.float64, generator=g, requires_grad=True)
    u = q if (s, s) == (H, W) else F.interpolate(q, size=(H, W), mode="bilinear", align_corners=False)
    np.testing.assert_allclose(O.upsample(q.detach().numpy(), H, W), u.detach().numpy(), rtol=0, atol=1e-6)
    gu = torch.randn(u.shape, dtype=torch.float64, generator=g)
    u.backward(gu)
    np.testing.assert_allclose(O.upsample_adjoint(gu.numpy(), s), q.grad.numpy(), rtol=0, atol=1e-5)
    # the adjoint is the exact transpose of the oracle's own map
    v = np.random.default_rng(s).standard_normal((2, 3, s, s))
    w = np.random.default_rng(H).standard_normal((2, 3, H, W))
    assert abs((O.upsample(v, H, W) * w).sum() - (v * O.upsample_adjoint(w, s)).sum()) < 1e-10 * np.abs(w).sum() * np.abs(v).max()


def test_conv_matches_torch():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 5, 6, dtype=torch.float64, generator=g)
    w = torch.randn(8, 8, 3, 3, dtype=torch.float64, generator=g)
    b = torch.randn(8, dtype=torch.float64, generator=g)
    np.testing.assert_allclose(O.conv3x3(x.numpy(), w.numpy(), b.numpy()), F.conv2d(x, w, b, padding=1).numpy(), rtol=1e-12,
                               atol=1e-12)


@pytest.mark.parametrize("n_scales", [1, 2, 3, 4, 5, 7, 10])
@pytest.mark.parametrize("share", [1, 0, -1, 2, 3, 4, 20])
def test_choose_phi_matches_reference_rule(n_scales, share):
    import vector_quantize_pytorch_b200 as m
    hq = m.HierarchicalVQ(dim=8, codebook_size=4, scales=range(1, n_scales + 1), share_quant_resi=share, accept_image_fmap=True)
    phis = [hq.phi_shared] if hq.phi_shared is not None else list(hq.phi_levels)
    assert len(phis) == O.n_phis(n_scales, share)
    for k in range(n_scales):
        assert hq._choose_phi(k) is phis[O.choose_phi(n_scales, len(phis), k)]


def test_choose_phi_ties_round_half_to_even():
    """5 scales over 2 phis: scale 2 sits at position 0.5, which Python's round sends to phi 0."""
    import vector_quantize_pytorch_b200 as m
    hq = m.HierarchicalVQ(dim=8, codebook_size=4, scales=(1, 2, 3, 4, 5), share_quant_resi=2, accept_image_fmap=True)
    assert [list(hq.phi_levels).index(hq._choose_phi(k)) for k in range(5)] == [0, 0, 0, 1, 1]
    hq = m.HierarchicalVQ(dim=8, codebook_size=4, scales=(1, 2, 3, 4, 5), share_quant_resi=4, accept_image_fmap=True)
    # positions 0, .75, 1.5, 2.25, 3: 1.5 rounds to 2
    assert [list(hq.phi_levels).index(hq._choose_phi(k)) for k in range(5)] == [0, 1, 2, 2, 3]


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_seeded_state_dict_matches_reference(path):
    """Construction in the reference's order draws the same numbers: same keys, same bits; and the reference's state loads."""
    import vector_quantize_pytorch_b200 as m
    f, meta = load(path)
    torch.manual_seed(meta["seed"])
    hq = m.HierarchicalVQ(**meta["kw"], accept_image_fmap=True)
    sd = hq.state_dict()
    keys = json.loads(str(f["sd_keys"]))
    assert list(sd) == keys
    for j, k in enumerate(keys):
        ours = sd[k].numpy()
        assert ours.dtype == f[f"sd_{j}"].dtype and ours.shape == f[f"sd_{j}"].shape, k
        assert ours.tobytes() == f[f"sd_{j}"].tobytes(), k
    other = m.HierarchicalVQ(**meta["kw"], accept_image_fmap=True)
    other.load_state_dict({k: torch.from_numpy(f[f"sd_{j}"]) for j, k in enumerate(keys)})
    for k, v in other.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_surface():
    import vector_quantize_pytorch_b200 as m
    hq = m.HierarchicalVQ(dim=16, codebook_size=8, scales=[1.0, 2, 3], quant_resi=-0.25, share_quant_resi=0,
                          accept_image_fmap=True)
    assert hq.dim == 16 and hq.scales == (1, 2, 3) and isinstance(hq.vq, m.VectorQuantize) and hq.phi_shared is None
    assert len(hq.phi_levels) == 3 and all(p.resi_ratio == 0.25 for p in hq.phi_levels)
    assert hq.vq.accept_image_fmap
    hq0 = m.HierarchicalVQ(dim=16, codebook_size=8, scales=[2], quant_resi=0.0, accept_image_fmap=True)
    assert hq0.phi_shared.resi_ratio == 0.0 and hq0.phi_shared.conv.weight.shape == (16, 16, 3, 3)


def test_refusals():
    import vector_quantize_pytorch_b200 as m
    kw = dict(dim=16, codebook_size=8, scales=(1, 2))
    with pytest.raises(AssertionError):
        m.HierarchicalVQ(**kw)
    for scales in ((), (2, 1), (0, 1), (-1, 2)):
        with pytest.raises(AssertionError):
            m.HierarchicalVQ(**dict(kw, scales=scales), accept_image_fmap=True)
    with pytest.raises(NotImplementedError):
        m.HierarchicalVQ(**kw, stochastic_sample_codes=True, accept_image_fmap=True)
    with pytest.raises(NotImplementedError):
        m.HierarchicalVQ(**kw, orthogonal_reg_weight=0.1, accept_image_fmap=True)
    for dim in (12, 1032):
        with pytest.raises(NotImplementedError):
            m.HierarchicalVQ(**dict(kw, dim=dim), accept_image_fmap=True)
    hq = m.HierarchicalVQ(**kw, accept_image_fmap=True)
    for dt in (torch.bfloat16, torch.float16, torch.float64):
        with pytest.raises(TypeError):
            hq(torch.zeros(1, 16, 4, 4, dtype=dt))
    with pytest.raises(RuntimeError):
        hq(torch.zeros(1, 16, 4, 4))
    with pytest.raises(AssertionError):
        hq(torch.zeros(1, 16, 4, 4), indices=torch.zeros(1, 4, 4, dtype=torch.long))
    with pytest.raises(AssertionError):
        hq(torch.zeros(16, 4, 4))


VQB_E_INVALID, VQB_E_UNSUPPORTED, VQB_E_ALIGN = -1, -2, -3
P = 256   # a stand-in device pointer: the argument checks never dereference it


def test_abi_errors_before_any_cuda_call():
    from vector_quantize_pytorch_b200._C import lib
    # pool / pool backward: (ptr, B, D, H, W, s, out, stream)
    for fn in (lib.vqb_hvq_pool, lib.vqb_hvq_pool_backward):
        assert fn(None, 1, 8, 4, 4, 2, P, None) == VQB_E_INVALID
        assert fn(P, 1, 8, 4, 4, 2, None, None) == VQB_E_INVALID
        for bad in ((0, 8, 4, 4, 2), (1, 0, 4, 4, 2), (1, 8, 0, 4, 2), (1, 8, 4, -1, 2), (1, 8, 4, 4, 0)):
            assert fn(P, *bad, P, None) == VQB_E_INVALID, bad
        assert fn(P, 1, 8, 1 << 17, 4, 2, P, None) == VQB_E_UNSUPPORTED
        assert fn(P, 1, 8, 4, 4, 1 << 17, P, None) == VQB_E_UNSUPPORTED
        assert fn(P, 1 << 30, 1024, 64, 64, 2, P, None) == VQB_E_UNSUPPORTED
        assert fn(P + 2, 1, 8, 4, 4, 2, P, None) == VQB_E_ALIGN
        assert fn(P, 1, 8, 4, 4, 2, P + 1, None) == VQB_E_ALIGN
    # upsample: (rows, B, D, s, H, W, q, recon, resid, recon_out, resid_out, stream)
    up = lib.vqb_hvq_upsample
    assert up(None, 1, 8, 2, 4, 4, P, None, None, None, None, None) == VQB_E_INVALID
    assert up(P, 1, 8, 2, 4, 4, None, None, None, None, None, None) == VQB_E_INVALID      # no output
    assert up(P, 1, 8, 2, 4, 4, None, None, None, None, P, None) == VQB_E_INVALID         # resid_out without resid
    assert up(P, 1, 8, 0, 4, 4, P, None, None, None, None, None) == VQB_E_INVALID
    assert up(P, 1, 8, 2, 4, 4, P, P + 2, None, P, None, None) == VQB_E_ALIGN
    # upsample backward: (g_a, g_b, B, D, s, H, W, g_rows, stream)
    ub = lib.vqb_hvq_upsample_backward
    assert ub(None, None, 1, 8, 2, 4, 4, P, None) == VQB_E_INVALID
    assert ub(P, None, 1, 8, 2, 4, 4, None, None) == VQB_E_INVALID
    assert ub(None, P + 1, 1, 8, 2, 4, 4, P, None) == VQB_E_ALIGN
    # blend: (up, conv, n, r, recon, resid, recon_out, resid_out, stream)
    bl = lib.vqb_hvq_blend_update
    assert bl(None, P, 16, 0.5, None, None, P, None, None) == VQB_E_INVALID
    assert bl(P, P, 0, 0.5, None, None, P, None, None) == VQB_E_INVALID
    assert bl(P, P, 16, 0.5, None, None, None, None, None) == VQB_E_INVALID
    assert bl(P, P, 16, 0.5, None, None, None, P, None) == VQB_E_INVALID
    assert bl(P, P, 1 << 40, 0.5, None, None, P, None, None) == VQB_E_UNSUPPORTED
    assert bl(P, P + 3, 16, 0.5, None, None, P, None, None) == VQB_E_ALIGN
    bb = lib.vqb_hvq_blend_backward   # (g_recon, g_resid, n, r, g_up, g_conv, stream)
    assert bb(None, None, 16, 0.5, P, P, None) == VQB_E_INVALID
    assert bb(P, None, 16, 0.5, None, P, None) == VQB_E_INVALID
    assert bb(P, None, -4, 0.5, P, P, None) == VQB_E_INVALID
    assert bb(P, None, 16, 0.5, P, P + 2, None) == VQB_E_ALIGN
