"""CPU checks of ResidualSimVQ: the numpy restatement (oracle/residual_simvq_oracle.py) against the reference's own outputs and
gradients (tests/golden/residual_simvq/), and the module's construction against the reference's state_dict."""
import numpy as np
import pytest
import torch

from oracle import residual_simvq_oracle as R
from residual_simvq_golden import Fixture, names


@pytest.mark.parametrize("name", names())
def test_residual_simvq_oracle_matches_reference(name):
    f = Fixture(name)
    kw = f.meta["kw"]
    Q = kw["num_quantizers"]
    books = R.implicit_codebooks(f.state(), Q, f.meta["transform"])
    n_active = int((f["indices"].reshape(-1, Q)[0] >= 0).sum())
    q, idx, losses, gx = R.forward(f.rows(f["x"]), books, n_active, kw.get("rotation_trick", True),
                                   commitment_weight=kw.get("commitment_weight", 1.0), G=f.rows(f["G"]), loss_grad=f["Lw"])
    assert np.array_equal(idx, f["indices"].reshape(-1, Q))
    np.testing.assert_allclose(q, f.rows(f["quantized"]), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(losses, f["losses"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(gx, f.rows(f["xgrad"]), rtol=1e-4, atol=2e-5)


@pytest.mark.parametrize("name", names())
def test_residual_simvq_state_dict_matches_reference(name):
    """Same RNG use at construction: the reference's state_dict keys in order, identical initial tensors, and it loads."""
    import vector_quantize_pytorch_b200 as m
    f = Fixture(name)
    ref = {k: torch.from_numpy(v) for k, v in f.state().items()}
    ours = f.build(m).state_dict()
    assert list(ours) == list(ref)
    for k in ref:
        assert torch.equal(ours[k], ref[k]), k
    f.build(m).load_state_dict(ref)


def test_residual_simvq_surface():
    import vector_quantize_pytorch_b200 as m
    rsv = m.ResidualSimVQ(dim=32, num_quantizers=3, codebook_size=16)
    assert rsv.codebook_size == 16 and rsv.codebooks.shape == (3, 16, 32)
    with pytest.raises(AssertionError):
        m.ResidualSimVQ(dim=32, num_quantizers=2, codebook_size=16, heads=2)   # rsv:67
    with pytest.raises(RuntimeError, match="no CPU path"):
        rsv(torch.randn(1, 8, 32))
    assert not m.ResidualSimVQ(dim=32, num_quantizers=1, codebook_size=16, quantize_dropout=True).quantize_dropout
    with pytest.raises(AssertionError):   # coarse indices need quantize dropout (rsv:115)
        rsv.get_codes_from_indices(torch.zeros(1, 4, 2, dtype=torch.long))
