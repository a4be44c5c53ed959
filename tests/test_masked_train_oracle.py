"""CPU checks of the numpy restatement of a masked training step (oracle/masked_train_oracle.py) against the reference's own
step (tests/golden/masked_train/, oracle/gen_golden_masked_train.py): outputs, indices, losses, x.grad and the projection
gradients of every fixture.  Also pins what the fixtures cover."""
import numpy as np
import pytest

from masked_train_golden import Fixture, names


def _tol(f):
    # bf16 inputs: the reference rounds every elementwise step to bf16 (relative 2^-8); fp32 within its own rounding
    return (3e-2, 3e-2) if f.bf16 else (1e-4, 1e-5)


@pytest.mark.parametrize("name", names())
def test_masked_train_oracle_matches_reference(name):
    f = Fixture(name)
    if f.kw.get("kmeans_init"):
        pytest.skip("the restatement searches the state_dict's codebook; this fixture's search used its k-means init")
    rtol, atol = _tol(f)
    out, idx, loss, gx, grads = f.oracle()
    np.testing.assert_array_equal(idx, f["ind"])
    np.testing.assert_allclose(out, f["out"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(np.asarray(loss, np.float32).reshape(f["loss"].shape), f["loss"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(gx, f["xgrad"], rtol=rtol, atol=atol)
    ref = f.pgrads()
    for n, g in grads.items():
        np.testing.assert_allclose(g, ref[n], rtol=rtol, atol=atol, err_msg=n)
    # the padding rows: index -1, and exactly the padding value / no gradient (or the upstream one)
    pad = ~f["mask"]
    if f.cls == "VectorQuantize":
        assert (f["ind"][pad] == -1).all()
        if f.kw.get("return_zeros_for_masked_padding", True):
            assert (f["out"][pad] == 0).all() and (f["xgrad"][pad] == 0).all()
        else:
            np.testing.assert_array_equal(f["out"][pad], f["x"][pad])
            np.testing.assert_array_equal(f["xgrad"][pad], f["G"][pad])
    else:
        assert (f["xgrad"][pad] == 0).all()


def test_masked_train_fixtures_cover_the_cases():
    metas = [Fixture(n).meta for n in names()]
    vq = [m for m in metas if m["cls"] == "VectorQuantize"]
    assert any(m["kw"].get("rotation_trick", True) for m in vq) and any(not m["kw"].get("rotation_trick", True) for m in vq)
    assert {m["dtype"] for m in vq} == {"float32", "bfloat16"}
    assert any(m["how"] == "lens" for m in vq)
    assert any(not m["kw"].get("return_zeros_for_masked_padding", True) for m in vq)
    assert any(0 in m["lens"] for m in vq)                       # a sequence that is all padding
    assert any(m["padding"] == "zero" for m in vq)               # padding rows exactly zero
    assert any(m["kw"].get("use_cosine_sim") for m in vq)
    rvq = [m for m in metas if m["cls"] == "ResidualVQ"]
    assert any(m["kw"].get("shared_codebook") for m in rvq) and any(not m["kw"].get("shared_codebook") for m in rvq)
    assert any("codebook_dim" in m["kw"] for m in rvq) and any(m["kw"].get("quantize_dropout") for m in rvq)
    assert any(m["cls"] == "GroupedResidualVQ" for m in metas)
    for m in metas:
        assert m["lens"] and min(m["lens"]) < m["x_shape"][1]    # every fixture has padding rows


def test_rotate_masked_argument_errors_are_return_codes():
    """vqb_rotate_masked refuses, before any CUDA call, null pointers, a loss gradient without n_live, an unknown estimator or
    dtype and an empty batch."""
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null; never dereferenced
    assert lib.vqb_rotate_masked(None, p, None, None, p, None, 1.0, 2, 1, 8, 8, 0, p, None) == -1   # no src
    assert lib.vqb_rotate_masked(p, p, None, None, None, None, 1.0, 2, 1, 8, 8, 0, p, None) == -1   # no mask
    assert lib.vqb_rotate_masked(p, p, p, p, p, None, 1.0, 2, 1, 8, 8, 0, p, None) == -1            # grad_loss, no n_live
    assert lib.vqb_rotate_masked(p, p, None, None, p, None, 1.0, 3, 1, 8, 8, 0, p, None) == -1      # bad estimator
    assert lib.vqb_rotate_masked(p, p, None, None, p, None, 1.0, 2, 1, 8, 8, 2, p, None) == -1      # bad dtype
    assert lib.vqb_rotate_masked(p, p, None, None, p, None, 1.0, 2, 1, 0, 8, 0, p, None) == -1      # N = 0
