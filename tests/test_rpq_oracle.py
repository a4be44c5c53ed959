"""RandomProjectionQuantizer on the CPU: the float64 oracle (oracle/rpq_oracle.py) against the reference's fixtures
(tests/golden/rpq/, oracle/gen_golden_rpq.py), seeded state_dict parity, loading the reference's state_dicts, Sequential's
one-quantizer rule, the refusals and the C ABI's argument errors."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import rpq_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "rpq")
FIXTURES = sorted(p[:-4] for p in os.listdir(GOLDEN) if p.endswith(".npz"))


def load(name):
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    return f, json.loads(bytes(f["meta"]).decode())


def seeded(m, meta):
    torch.manual_seed(meta["seed"])
    return m.RandomProjectionQuantizer(**meta["kw"])


def test_fixtures_exist():
    assert {"bestrq", "no_norm", "dim81", "h2_e16", "h4_e8", "usm", "kmeans", "train_between", "b1_n1"} <= set(FIXTURES)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_fixture(name):
    """The reference's fp32 rows lie within the kernel's bound of the float64 rows, and the float64 search on the float64 rows
    (through a float64 project_in) gives the reference's indices, with every lead over the fixture's threshold."""
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    rpq = seeded(m, meta)
    kw = meta["kw"]
    norm = kw.get("norm", True)
    P = rpq.rand_projs.numpy()
    H = rpq.num_codebooks
    for s in range(meta["calls"]):
        x = f[f"x_{s}"].reshape(-1, kw["dim"])
        rows64 = O.norm_project(x, P, norm)
        np.testing.assert_allclose(rows64, f[f"rows64_{s}"], rtol=1e-12, atol=1e-12)
        err = np.abs(f[f"rows_{s}"] - rows64)
        assert (err <= O.row_bound(x, P, norm)).all(), f"call {s}: reference rows outside the bound"
        embeds = f[f"embed_{s}"] if f"embed_{s}" in f else rpq.vq._codebook.embed.numpy()
        pin = (rpq.vq.project_in.weight.detach().numpy(), rpq.vq.project_in.bias.detach().numpy()) if H > 1 else None
        _, y64, idx, lead = O.forward(x, P, norm, embeds.astype(np.float64), pin)
        if H > 1:
            np.testing.assert_allclose(f[f"proj_in_{s}"], y64, rtol=0, atol=1e-4 * np.abs(y64).max())
        np.testing.assert_array_equal(idx.reshape(f[f"indices_{s}"].shape), f[f"indices_{s}"])
        assert (lead > 2e-5).all()


@pytest.mark.parametrize("name", FIXTURES)
def test_seeded_state_dict_matches_reference(name):
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    sd = seeded(m, meta).state_dict()
    assert list(sd) == json.loads(str(f["sd_keys"]))
    digests = json.loads(str(f["sd_sha256"]))
    for j, (k, v) in enumerate(sd.items()):
        assert hashlib.sha256(v.numpy().tobytes()).hexdigest() == digests[j], k
        if f"sd_{j}" in f:
            np.testing.assert_array_equal(v.numpy(), f[f"sd_{j}"], err_msg=k)


def test_loads_reference_state_dict():
    import vector_quantize_pytorch_b200 as m
    f, meta = load("h2_e16")
    keys = json.loads(str(f["sd_keys"]))
    torch.manual_seed(123)
    rpq = m.RandomProjectionQuantizer(**meta["kw"])
    rpq.load_state_dict({k: torch.from_numpy(f[f"sd_{j}"]) for j, k in enumerate(keys)})
    for j, (k, v) in enumerate(rpq.state_dict().items()):
        np.testing.assert_array_equal(v.numpy(), f[f"sd_{j}"], err_msg=k)


def test_surface():
    import vector_quantize_pytorch_b200 as m
    from vector_quantize_pytorch_b200 import utils
    assert m.RandomProjectionQuantizer is utils.RandomProjectionQuantizer and m.Sequential is utils.Sequential
    assert len(utils.QUANTIZE_KLASSES) == 14 and m.BinaryMapper not in utils.QUANTIZE_KLASSES
    rpq = m.RandomProjectionQuantizer(dim=32, codebook_size=64, codebook_dim=8, num_codebooks=2, norm=False)
    assert isinstance(rpq.norm, torch.nn.Identity) and rpq.rand_projs.shape == (2, 32, 8)
    assert rpq.vq.heads == 2 and rpq.vq.separate_codebook_per_head and rpq.vq.use_cosine_sim
    assert tuple(rpq.vq.project_in.weight.shape) == (32, 16)


def test_sequential_holds_exactly_one_quantizer():
    import vector_quantize_pytorch_b200 as m
    vq = m.VectorQuantize(dim=16, codebook_size=32)
    rpq = m.RandomProjectionQuantizer(dim=16, codebook_size=32, codebook_dim=8)
    m.Sequential(torch.nn.Linear(16, 16), vq)
    m.Sequential(rpq)
    with pytest.raises(AssertionError, match="exactly one quantizer"):
        m.Sequential(torch.nn.Linear(16, 16))
    with pytest.raises(AssertionError, match="exactly one quantizer"):
        m.Sequential(vq, rpq)


def test_refusals():
    import vector_quantize_pytorch_b200 as m
    for kw in (dict(codebook_dim=12), dict(codebook_dim=256, num_codebooks=16), dict(codebook_dim=2048),
               dict(codebook_dim=3, num_codebooks=2)):
        with pytest.raises(NotImplementedError, match="per-head width"):
            m.RandomProjectionQuantizer(dim=512, codebook_size=64, **kw)
    rpq = m.RandomProjectionQuantizer(dim=16, codebook_size=32, codebook_dim=8)
    with pytest.raises(NotImplementedError, match="cross-entropy"):
        rpq(torch.randn(1, 4, 16), indices=torch.zeros(1, 4, dtype=torch.long))
    with pytest.raises(TypeError, match="float32"):
        rpq(torch.randn(1, 4, 16).bfloat16())
    with pytest.raises(TypeError, match="batch, seq, dim"):
        rpq(torch.randn(4, 16))
    with pytest.raises(TypeError, match="batch, seq, dim"):
        rpq(torch.randn(1, 2, 4, 16))


VQB_E_INVALID, VQB_E_UNSUPPORTED, VQB_E_ALIGN = -1, -2, -3


def test_abi_errors_before_any_cuda_call():
    from vector_quantize_pytorch_b200._C import lib
    fn = lib.vqb_rpq_norm_project
    P = 1 << 20
    assert fn(None, 4, 16, P, 1, 8, 1, P, None) == VQB_E_INVALID
    assert fn(P, 4, 16, None, 1, 8, 1, P, None) == VQB_E_INVALID
    assert fn(P, 4, 16, P, 1, 8, 1, None, None) == VQB_E_INVALID
    for bad in ((0, 16, 1, 8, 1), (-1, 16, 1, 8, 1), (4, 0, 1, 8, 1), (4, 16, 0, 8, 1), (4, 16, 1, 0, 1), (4, 16, 1, 8, 2),
                (4, 16, 1, 8, -1)):
        N, dim, H, E, norm = bad
        assert fn(P, N, dim, P, H, E, norm, P, None) == VQB_E_INVALID, bad
    assert fn(P, 4, 16, P, 1, 1025, 1, P, None) == VQB_E_UNSUPPORTED
    assert fn(P, 4, 16, P, 33, 32, 1, P, None) == VQB_E_UNSUPPORTED
    assert fn(P, 4, (1 << 16) + 1, P, 1, 8, 1, P, None) == VQB_E_UNSUPPORTED
    assert fn(P, 1 << 30, 4096, P, 1, 8, 1, P, None) == VQB_E_UNSUPPORTED
    assert fn(P, 1 << 31, 8, P, 1, 1024, 1, P, None) == VQB_E_UNSUPPORTED
    assert fn(P + 2, 4, 16, P, 1, 8, 1, P, None) == VQB_E_ALIGN
    assert fn(P, 4, 16, P + 1, 1, 8, 1, P, None) == VQB_E_ALIGN
    assert fn(P, 4, 16, P, 1, 8, 1, P + 3, None) == VQB_E_ALIGN
