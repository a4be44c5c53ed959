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
