"""CPU checks of the BinaryMapper oracle, fixtures, module surface, refusals and C ABI argument errors (no GPU needed)."""
import glob
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import binary_mapper_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "binary_mapper", "*.npz")))


def upstream(f) -> np.ndarray:
    """The fixture's G (rows, 2^bits), regenerated from its seed and checked against its checksum."""
    rows, K = int(np.prod(f["lead"], dtype=np.int64)), 1 << int(f["bits"])
    G = torch.randn(rows, K, generator=torch.Generator().manual_seed(int(f["g_seed"])))
    assert hashlib.sha256(G.numpy().tobytes()).hexdigest()[:16] == str(f["g_digest"]), "the seeded recipe of G drifted"
    return G.numpy()


def close_to_f64(ours, ref, ref64):
    """ours no further from float64 than the fp32 reference is, or 2e-5 of the largest value; NaNs where the reference's."""
    ours, ref, ref64 = (np.asarray(a, np.float64) for a in (ours, ref, ref64))
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(ours), nan)
    ours, ref, ref64 = ours[~nan], ref[~nan], ref64[~nan]
    if ours.size == 0:
        return
    floor = 2e-5 * max(np.abs(ref64).max(), 1e-30)
    bad = np.abs(ours - ref64) > np.abs(ref - ref64) + floor
    assert not bad.any(), f"{bad.sum()} elements: ours {ours[bad][:4]} ref {ref[bad][:4]} f64 {ref64[bad][:4]}"


def test_fixtures_exist():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert {f"train_b{b}" for b in (1, 3, 8, 12, 16)} <= names
    assert {"eval_b8", "eval_det_on_eval_b8", "train_deterministic_b12", "eval_st_b8", "temp05_b8", "temp2_b3", "thr0_b8",
            "thr100_b8", "noreduce_image_b3", "single_row_b8", "bf16_eval_b8", "bf16_no_st_b8", "nonfinite_b3", "nonfinite_b8",
            "tiny_b8"} <= names


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_reproduces_fixture(path):
    """The float64 oracle on the reference's indices against the reference: the aux loss, log_prob (with indices= and
    one_hot=, summed and per bit) and the gradient, each within the fp32 reference's own distance from float64."""
    f = np.load(path)
    bits, lead = int(f["bits"]), tuple(int(v) for v in f["lead"])
    ckw, fkw = json.loads(str(f["ckw"])), json.loads(str(f["fkw"]))
    rows = int(np.prod(lead, dtype=np.int64))
    l = f["x"].astype(np.float64).reshape(rows, bits)
    idx = f["indices"].reshape(rows)
    bf16 = str(f["xdtype"]) == "bf16"
    tol = dict(rtol=1e-2, atol=1e-2) if bf16 else dict(rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(O.log_prob(l, idx).reshape(lead), f["lp"], **tol)
    np.testing.assert_allclose(O.log_prob(l, idx, sum_bits=False).reshape(*lead, bits), f["lp_bits"], **tol)
    np.testing.assert_array_equal(np.isnan(f["lp_onehot"]), np.isnan(f["lp"]))
    finite_rows = np.isfinite(l).all(-1)
    np.testing.assert_array_equal(f["lp_onehot"].reshape(-1)[finite_rows], f["lp"].reshape(-1)[finite_rows])
    if not bf16:
        close_to_f64(f["lp64"], f["lp"], f["lp64"])
    thr = ckw.get("kl_loss_threshold", O.NAT)
    if str(f["aux_kind"]) != "zero":
        a = O.aux_rows(l, thr)
        a = a.mean() if str(f["aux_kind"]) == "mean" else a.reshape(lead)
        # bf16: the difference bits ln 2 - H of bf16 terms of size ~ln 2 is off by a few bf16 ulps of bits ln 2
        np.testing.assert_allclose(a, f["aux"], **(dict(rtol=0.0, atol=0.02 * bits) if bf16 else tol))
    else:
        assert float(f["aux"]) == 0.0
    st = fkw.get("straight_through", bool(f["train"]))
    G = upstream(f) if st else None
    dx = O.grad_total(l, idx, G, f["H"], st=st, aux_kind=str(f["aux_kind"]), thr=thr).reshape(*lead, bits)
    np.testing.assert_array_equal(dx, f["dx64"])
    if bf16:
        np.testing.assert_allclose(dx, f["dx"], rtol=2e-2, atol=2e-2 * np.abs(dx).max())
    else:
        np.testing.assert_allclose(f["dx"][np.isfinite(dx)], dx[np.isfinite(dx)], rtol=1e-4, atol=1e-5 * np.nanmax(np.abs(dx)))
    # the deterministic bit is sigmoid(l / t) > 0.5, so a tiny positive logit can give bit 0
    if fkw.get("deterministic") or (ckw.get("deterministic_on_eval") and not bool(f["train"])):
        t = fkw.get("temperature", 1.0)
        p = torch.sigmoid(torch.from_numpy(f["x"].reshape(rows, bits)).float() / t)
        np.testing.assert_array_equal(O.index_bits(idx, bits), (p > 0.5).numpy())


@pytest.mark.parametrize("bits", [1, 3, 8])
@pytest.mark.parametrize("case", ["randn", "wide", "saturated"])
def test_closed_form_gradient_matches_autograd(bits, case):
    """S1_j - sigmoid(l_j) S (and the two-sum form the kernel evaluates) against float64 autograd of the reference formula:
    exp(logsigmoid(l) @ codes^T + logsigmoid(-l) @ (1 - codes)^T) contracted with G."""
    g = np.random.default_rng(bits)
    l = g.standard_normal((16, bits)) * {"randn": 1.0, "wide": 6.0, "saturated": 30.0}[case]
    G = g.standard_normal((16, 1 << bits))
    lt = torch.from_numpy(l).requires_grad_(True)
    c = torch.from_numpy(O.codes(bits).astype(np.float64))
    soft = (torch.nn.functional.logsigmoid(lt) @ c.T + torch.nn.functional.logsigmoid(-lt) @ (1 - c).T).exp()
    (soft * torch.from_numpy(G)).sum().backward()
    ref = lt.grad.numpy()
    np.testing.assert_allclose(O.st_grad(l, G), ref, rtol=1e-9, atol=1e-12 * max(np.abs(ref).max(), 1e-300))
    if case != "saturated":   # the one-sum form cancels when sigmoid(l) is near 1
        np.testing.assert_allclose(O.st_grad_plain(l, G), ref, rtol=1e-7, atol=1e-10 * np.abs(ref).max())


def test_oracle_nan_pattern_matches_fixture():
    """The reference's NaN elements: all codes of a NaN row; under +inf at bit j the codes with bit j set; under -inf the
    codes with bit j clear."""
    for name in ("nonfinite_b3", "nonfinite_b8"):
        f = np.load(os.path.join(HERE, "golden", "binary_mapper", name + ".npz"))
        bits = int(f["bits"])
        l = f["x"].astype(np.float64).reshape(-1, bits)
        c = O.codes(bits)
        nan = np.isnan(l).any(-1)[:, None] | (c[None] & (l[:, None, :] == np.inf)).any(-1) | \
            (~c[None] & (l[:, None, :] == -np.inf)).any(-1)
        idx = f["indices"].reshape(-1)
        nonhot = nan.copy()
        nonhot[np.arange(len(idx)), idx] = False
        np.testing.assert_array_equal(np.flatnonzero(nonhot.reshape(-1)), f["nan_pos"])
        np.testing.assert_array_equal(np.isnan(f["hot"]), nan[np.arange(len(idx)), idx])


def test_module_surface_and_cpu_methods():
    """Buffers, attributes and the torch-only methods match the fixtures on the CPU."""
    import vector_quantize_pytorch_b200 as vqb
    m = vqb.BinaryMapper(bits=5, kl_loss_threshold=0.5, deterministic_on_eval=True)
    assert m.num_codes == 32 and m.bits == 5 and m.kl_loss_threshold == 0.5 and m.deterministic_on_eval
    assert m.power_two.tolist() == [1, 2, 4, 8, 16] and m.power_two.dtype == torch.int64
    assert m.codes.dtype == torch.bool and m.codes.shape == (32, 5) and m.codes[6].tolist() == [False, True, True, False, False]
    assert m.zero.dtype == torch.float32 and m.zero.item() == 0.0
    assert m.state_dict() == {}
    for path in FIXTURES:
        f = np.load(path)
        if str(f["xdtype"]) != "fp32":
            continue
        ckw = json.loads(str(f["ckw"]))
        fkw = json.loads(str(f["fkw"]))
        mod = vqb.BinaryMapper(bits=int(f["bits"]), **ckw)
        x = torch.from_numpy(f["x"])
        idx = torch.from_numpy(f["indices"])
        np.testing.assert_array_equal(mod.log_prob(x, indices=idx).numpy(), f["lp"])
        np.testing.assert_array_equal(mod.log_prob(x, indices=idx, sum_bits=False).numpy(), f["lp_bits"])
        if str(f["aux_kind"]) != "zero":
            aux = mod.calc_aux_loss(x, reduce_aux_kl_loss=fkw.get("reduce_aux_kl_loss", True))
            np.testing.assert_allclose(aux.numpy(), f["aux"], rtol=1e-6, atol=1e-7)


def test_refusals():
    import vector_quantize_pytorch_b200 as vqb
    with pytest.raises(NotImplementedError):
        vqb.BinaryMapper(bits=21)
    with pytest.raises(NotImplementedError):
        vqb.BinaryMapper(bits=0)
    m = vqb.BinaryMapper(bits=4)
    with pytest.raises(TypeError):
        m(torch.randn(3, 4, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.randn(3, 4))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.eval()(torch.randn(3, 4).bfloat16())


def test_binmap_argument_errors_are_return_codes_not_crashes():
    """vqb_binmap_* refuse null pointers, bits outside [1, 20], bad plans and misaligned pointers before any CUDA call."""
    import ctypes
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced

    def hot(lg=p, idx=p, rows=8, bits=4, out=p):
        return lib.vqb_binmap_hot(lg, idx, rows, bits, out, None)

    def bwd(lg=p, rows=8, bits=8, g=p, rs=256, cs=1, ks=1, work=None, dl=p):
        return lib.vqb_binmap_backward(lg, rows, bits, g, rs, cs, ks, work, dl, None)

    assert hot(idx=None) == -1 and hot(out=None) == -1 and hot(rows=0) == -1 and hot(bits=0) == -1
    assert hot(bits=21) == -2
    assert hot(out=p + 4) == -3 and hot(out=p + 8) == -3 and hot(idx=p + 4) == -3 and hot(lg=p + 2) == -3
    assert bwd(lg=None) == -1 and bwd(g=None) == -1 and bwd(dl=None) == -1 and bwd(rows=0) == -1 and bwd(bits=0) == -1
    assert bwd(bits=21) == -2 and bwd(rs=-1) == -1 and bwd(cs=-1) == -1
    assert bwd(ks=0) == -1 and bwd(ks=3) == -1 and bwd(ks=2) == -1   # ks > 1 needs the workspace
    assert bwd(bits=8, ks=16, work=p) == -1   # 8 segments of 32 codes: at most 8 chunks
    assert bwd(g=p + 2) == -3 and bwd(dl=p + 1) == -3 and bwd(ks=2, work=p + 4) == -3
    plan = (ctypes.c_int * 2)()
    assert lib.vqb_binmap_backward_plan(0, 8, 132, plan) == -1 and lib.vqb_binmap_backward_plan(8, 0, 132, plan) == -1
    assert lib.vqb_binmap_backward_plan(8, 21, 132, plan) == -2 and lib.vqb_binmap_backward_plan(8, 8, 0, plan) == -1
    assert lib.vqb_binmap_backward_plan(8, 8, 132, None) == -1


def _plan(rows, bits, sms):
    from vector_quantize_pytorch_b200 import ops
    return ops.binmap_backward_plan(rows, bits, sms)


def test_backward_plan_space():
    """Every plan is valid, and the space is covered: every segment width, every power-of-two split up to the largest."""
    seen = set()
    for bits in range(1, 21):
        for rows in (1, 2, 7, 64, 129, 1000, 8192, 1 << 16, 1 << 20, 1 << 30):
            for sms in (1, 16, 132, 144):
                ks, seg = _plan(rows, bits, sms)
                nseg = (1 << bits) // seg
                assert seg == min(32, 1 << bits)
                assert ks >= 1 and ks & (ks - 1) == 0 and nseg % ks == 0
                assert ks == 1 or nseg // ks >= 8, "a chunk keeps at least 8 segments"
                assert ks == 1 or rows * (ks // 2) < sms * 1024, "the split stops once the threads fill the GPU"
                seen.add((ks, seg))
    assert {s for _, s in seen} == {2, 4, 8, 16, 32}
    splits = {k for k, _ in seen}
    assert splits == {1 << i for i in range(max(splits).bit_length())} and max(splits) == 1 << 12
    # the bench and test shapes on a 132-SM H100
    assert _plan(64 * 4096, 8, 132) == (1, 32)
    assert _plan(8 * 1024, 16, 132) == (32, 32)
    assert _plan(1024, 20, 132) == (256, 32)
    assert _plan(1, 20, 132) == (4096, 32)
