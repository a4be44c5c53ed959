"""CPU checks of finite scalar quantization: every reference fixture (tests/golden/fsq) replays through the numpy restatement
(oracle/fsq_oracle.py) under the exactness contract of DESIGN.md §4.9; the torch-computed kernel constants equal the reference's;
a seeded construction gives the reference's weights and state_dict keys; the unsupported options raise."""
import numpy as np
import pytest
import torch

from oracle import fsq_oracle as O
from fsq_golden import FIXTURES, Case, _key, boundary_pairs, fixture_id, flipped_rows, stage_values

import vector_quantize_pytorch_b200 as vqb
from vector_quantize_pytorch_b200.fsq import fsq_tables

CLASSES = {"FSQ": vqb.FSQ, "ResidualFSQ": vqb.ResidualFSQ, "GroupedResidualFSQ": vqb.GroupedResidualFSQ}


def replay(c: Case):
    z = c.rows("z")
    n_active = c.n_active
    fwd = O.forward(z, c.levels, c.Q, n_active, c.sym, c.hard, c.scales, c.clampv, c.w_bf16)
    return z, n_active, fwd


@pytest.mark.parametrize("path", FIXTURES, ids=fixture_id)
def test_forward_replays_through_oracle(path):
    c = Case(path)
    z, n_active, fwd = replay(c)
    ref_idx = c.index_rows()
    rows, excused = flipped_rows(fwd["idx"], ref_idx, fwd["near"])
    print(f"{fixture_id(path)}: {int(rows.sum())} flipped rows of {rows.size}, {int(excused.sum())} near a rounding boundary")
    assert (rows == excused).all(), "index differs away from any rounding boundary"
    if c.hard and c.clampv is None:
        assert not rows.any(), "the hard-clamp path without soft clamp must match bit for bit"
    qsum = c.rows("qsum")
    keep = ~rows
    np.testing.assert_array_equal(fwd["out"][keep], qsum[keep])


@pytest.mark.parametrize("path", FIXTURES, ids=fixture_id)
def test_backward_replays_through_oracle(path):
    c = Case(path)
    z, n_active, fwd = replay(c)
    rows, _ = flipped_rows(fwd["idx"], c.index_rows(), fwd["near"])
    dz, bound = O.backward(z, c.rows("qgrad"), c.levels, c.Q, n_active, c.sym, c.hard, c.scales, c.clampv, c.w_bf16, c.in_bf16)
    ref = c.rows("zgrad")
    keep = ~rows
    err = np.abs(dz.astype(np.float64) - ref)[keep]
    b = bound[keep]
    exact = b == 0
    assert (err[exact] == 0).all(), "a gradient made of exact factors must match bit for bit"
    ratio = float((err[~exact] / b[~exact]).max()) if (~exact).any() else 0.0
    print(f"{fixture_id(path)}: {int(exact.sum())} exact gradient elements, largest error / bound on the rest {ratio:.3g}")
    assert (err <= b).all()


@pytest.mark.parametrize("path", [p for p in FIXTURES if "decoded" in np.load(p).files or "all_codes" in np.load(p).files],
                         ids=fixture_id)
def test_decode_replays_through_oracle(path):
    c = Case(path)
    idx = c.index_rows()
    s, codes = O.decode(idx, c.levels, True, c.scales, c.w_bf16)
    if "decoded" in c.a:
        np.testing.assert_array_equal(s, c.rows("qsum"))   # quantized == get_output_from_indices(indices)
    ac = c.a["all_codes"]   # (Q, b, n, d)
    np.testing.assert_array_equal(codes.reshape(ac.shape), ac)


@pytest.mark.parametrize("path", FIXTURES, ids=fixture_id)
def test_constants_equal_reference(path):
    c = Case(path)
    for sym in (False, True):
        if not sym and 2 in c.levels:
            continue
        for hard in (False, True):
            consts, ints = fsq_tables(torch.tensor(c.levels, dtype=torch.int32),
                                      torch.tensor(c.a["const_basis"]).int(), sym, hard)
            a, b, shift, hw, basis, rb, rhw = consts.numpy()
            np.testing.assert_array_equal(hw, c.a["const_half_width"])
            np.testing.assert_array_equal(basis, c.a["const_basis"])
            np.testing.assert_array_equal(rhw, (1 / torch.tensor(c.a["const_half_width"])).numpy())
            if sym:
                np.testing.assert_array_equal(b, c.a["const_sym_scale"])
                np.testing.assert_array_equal(rb, (1 / torch.tensor(c.a["const_sym_scale"])).numpy())
            else:
                np.testing.assert_array_equal(a, c.a["const_half_l"])
                np.testing.assert_array_equal(b, c.a["const_offset"])
                np.testing.assert_array_equal(shift, c.a["const_shift_hard" if hard else "const_shift_atanh"])
            np.testing.assert_array_equal(ints.numpy()[0], np.asarray(c.levels))
    if c.scales is not None:
        m = CLASSES[c.cls](**c.meta["kw"])
        if c.meta["module_dtype"] == "bf16":
            m = m.to(torch.bfloat16)
        part = m.rvqs[0] if c.cls == "GroupedResidualFSQ" else m
        scales, clampv = part._make_scale_tables()
        np.testing.assert_array_equal(scales[0].numpy(), c.scales)
        if c.clampv is not None:
            np.testing.assert_array_equal(clampv[0].numpy(), c.clampv)


@pytest.mark.parametrize("path", FIXTURES, ids=fixture_id)
def test_seeded_construction_matches_reference(path):
    c = Case(path)
    torch.manual_seed(c.meta["init_seed"])
    m = CLASSES[c.cls](**c.meta["kw"])
    if c.meta["module_dtype"] == "bf16":
        m = m.to(torch.bfloat16)
    sd = m.state_dict()
    assert list(sd) == c.meta["state_dict_keys"]
    for j, v in enumerate(sd.values()):
        np.testing.assert_array_equal(v.float().numpy(), c.a[f"sd_{j}"])
    # the RNG is left where the reference leaves it
    after = torch.randn(3)
    torch.manual_seed(c.meta["init_seed"])
    CLASSES[c.cls](**c.meta["kw"])
    np.testing.assert_array_equal(torch.randn(3).numpy(), after.numpy())


@pytest.mark.parametrize("sym", [True, False], ids=["sym", "nonsym"])
@pytest.mark.parametrize("hard", [True, False], ids=["hard", "tanh"])
@pytest.mark.parametrize("soft", [False, True], ids=["nosoft", "soft"])
def test_boundary_finder(sym, hard, soft):
    """fsq_golden.boundary_pairs (the planted boundaries of tests/test_fsq_kernels_gpu.py): across every pair it returns the
    oracle's stage code changes, and the pre-floor / pre-round value recomputed in float64 from each side's stage input lies
    within one float32 step of a rounding boundary (plus, on the tanh paths, tanhf's two-ulp error times the slope)."""
    levels = [2, 3, 4, 5] if sym else [3, 4, 5, 8]
    Q = 3
    L = np.asarray(levels, np.float32)
    scales = np.stack([L ** -q for q in range(Q)]).astype(np.float32)
    clampv = (1 + 1 / (L - 1)).astype(np.float32) if soft else None
    t = O.tables(levels, sym, hard)
    bound = (lambda v: np.clip(v, -1, 1)) if hard else np.tanh
    total = 0
    for q in (0, Q - 1):
        for j in range(len(levels)):
            a, b = boundary_pairs(levels, Q, q, j, sym, hard, scales, clampv)
            assert len(a) >= 1
            np.testing.assert_array_equal(_key(b) - _key(a), 1)
            sides = [stage_values(z, j, levels, Q, q, sym, hard, scales, clampv) for z in (a, b)]
            assert (sides[0][0] != sides[1][0]).all(), "the code does not change across a pair"
            b64 = []
            tol = 0.0
            for _, br, u in sides:
                x = bound(u.astype(np.float64) + t["shift"][j])
                b64.append(t["a"][j] * (x + 1) / 2 + 0.5 if sym else x * t["a"][j] - t["b"][j])
                tol = np.maximum(tol, np.spacing(np.abs(br).astype(np.float32)).astype(np.float64))
                if not hard:
                    h = np.abs(np.tanh((u + t["shift"][j]).astype(np.float32)))
                    tol = tol + 2 * np.spacing(h).astype(np.float64) * t["a"][j] * (0.5 if sym else 1.0)
            lo, hi = np.minimum(*b64), np.maximum(*b64)
            k = np.floor(lo) + np.arange(-1, 3)[:, None] + (0.0 if sym else 0.5)   # the boundaries around the pair
            dist = np.maximum(0.0, np.maximum(k - hi, lo - k)).min(axis=0)
            assert (dist <= tol).all(), float((dist / tol).max())
            total += len(a)
    print(f"{total} pairs")


def test_codebook_and_helpers_match_reference_expressions():
    f = vqb.FSQ([8, 5, 5, 5])
    assert f.codebook_size == 1000 and f.implicit_codebook.shape == (1000, 4)
    assert f.implicit_codebook.dtype == torch.float32
    idx = f.codes_to_indices(f.implicit_codebook)
    assert idx.dtype == torch.int32
    np.testing.assert_array_equal(idx.numpy(), np.arange(1000))
    lv = f.indices_to_level_indices(torch.arange(1000))
    np.testing.assert_array_equal(lv.numpy(), (np.arange(1000)[:, None] // np.array([1, 8, 40, 200])) % np.array([8, 5, 5, 5]))
    r = vqb.ResidualFSQ(levels=[8, 5, 5, 3], num_quantizers=3)
    assert r.codebooks.shape == (3, 600, 4)
    assert not any(k in r.state_dict() for k in ("scales", "soft_clamp_input_value"))


@pytest.mark.parametrize("kw", [dict(noise_dropout=0.1, preserve_symmetry=True), dict(orthogonal_rotation=True),
                                dict(force_quantization_f32=False)], ids=["noise_dropout", "orthogonal_rotation", "no_force_f32"])
def test_unsupported_options_raise(kw):
    with pytest.raises(NotImplementedError, match="SURVEY"):
        vqb.FSQ([8, 5, 5, 5], **kw)
    with pytest.raises(NotImplementedError, match="SURVEY"):
        vqb.ResidualFSQ(levels=[8, 5, 5, 5], num_quantizers=2, **{k: v for k, v in kw.items() if k != "preserve_symmetry"})


def test_level_two_needs_symmetry():
    with pytest.raises(AssertionError):
        vqb.FSQ([2, 5])
    vqb.FSQ([2, 5], preserve_symmetry=True)


def test_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        vqb.FSQ([8, 5, 5, 5])(torch.randn(1, 4, 4))
