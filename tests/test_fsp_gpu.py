"""FSP on the GPU: replay of the reference fixtures (tests/golden/fsp) under the DESIGN 4.11 rules, RNG parity with the eager
formula on the same device, and the reference's own test cases."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import fsp_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "fsp", "*.npz")))
STATS = ("mean", "variance", "skewness", "kurtosis")
DEV = "cuda"


def _vqb():
    import vector_quantize_pytorch_b200 as vqb
    return vqb


def _module(f):
    vqb = _vqb()
    kw = json.loads(str(f["kwargs"]))
    torch.manual_seed(int(f["seed"]))
    m = vqb.FSP(**kw)
    m.load_state_dict({k[3:]: torch.from_numpy(f[k]) for k in f.files if k.startswith("sd.")}, strict=False)
    dt = torch.bfloat16 if str(f["xdtype"]) == "bf16" else torch.float32
    return kw, m.to(DEV).to(dt).train(bool(f["train"])), dt


def _run(m, x, eps, draws, G, H, monkeypatch):
    from vector_quantize_pytorch_b200 import fsp as fsp_mod
    it = iter(draws)
    monkeypatch.setattr(fsp_mod, "_rand", lambda z: next(it).to(z.device, z.dtype).reshape(z.shape).contiguous())
    zs = []

    def hook(_m, _i, out):
        out.retain_grad()
        zs.append(out)
    h = m.project_in.register_forward_hook(hook)
    x = x.clone().requires_grad_(True)
    q, idx, loss, info = m(x, eps) if eps is not None else m(x)
    h.remove()
    total = (q * G.to(q.dtype)).sum() + loss
    for k, s in enumerate(STATS):
        total = total + (info["norm_info"][s] * H[k].to(q.dtype)).sum()
    total.backward()
    return q, idx, loss, info, x.grad, zs[0]


def _close_to_f64(ours, ref, ref64, bf16):
    """ours no further from float64 than the reference is (bf16: 1.5 times), or 2e-5 of the largest value."""
    ours, ref, ref64 = (np.asarray(a, np.float64) for a in (ours, ref, ref64))
    floor = 2e-5 * max(np.abs(ref64).max(), 1e-30)
    if bf16:   # the largest deviation, as LFQ's bf16 rule takes it
        assert np.abs(ours - ref64).max() <= 1.5 * np.abs(ref - ref64).max() + floor
        return
    bad = np.abs(ours - ref64) > np.abs(ref - ref64) + floor
    assert not bad.any(), f"{bad.sum()} elements: ours {ours[bad][:4]} ref {ref[bad][:4]} f64 {ref64[bad][:4]}"


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_replay(path, monkeypatch):
    f = np.load(path)
    kw, m, dt = _module(f)
    bf16 = dt == torch.bfloat16
    eps = float(f["eps"]) if np.isfinite(f["eps"]) else None
    draws = [torch.from_numpy(f[k]) for k in ("u1", "u2") if k in f]
    x = torch.from_numpy(f["x"]).to(DEV, dt)
    q, idx, loss, info, dx, z = _run(m, x, eps, draws, torch.from_numpy(f["G"]).to(DEV), torch.from_numpy(f["H"]).to(DEV),
                                     monkeypatch)
    d = len(kw["levels"])
    assert str(q.dtype) == str(f["q_dtype"]) and idx.dtype == torch.int32 and loss.dtype == dt
    assert tuple(idx.shape) == f["indices"].shape and tuple(q.shape) == f["q"].shape
    assert info["level_indices"].dtype == dt and all(info["norm_info"][s].dtype == dt for s in STATS)
    assert ("p_accept_prob" in info) == ("p_accept_prob" in f)
    act, inv = kw.get("act_name", "tanh"), kw.get("need_inv_act", False)
    epsv = eps if eps is not None else float(torch.finfo(dt).eps)
    zf = z.detach().float().cpu().numpy().reshape(-1, d)
    lev = info["level_indices"].float().cpu().numpy().reshape(-1, d)
    lev_ref = f["level_indices"].reshape(-1, d)
    # fp32 and the CPU's math functions differ in the last ulps; bf16 rounds act and act L to 8 bits
    near = O.near_integer(O.pre_floor(zf, kw["levels"], act, epsv), 2. ** -6 if bf16 else 2. ** -19)
    diff = lev != lev_ref
    print(f"{os.path.basename(path)}: {near.sum()} elements near a bin edge, {diff.sum()} level indices differ")
    assert not (diff & ~near).any()
    exact = (lev.astype(np.int64) * O.basis(kw["levels"])).sum(-1)
    np.testing.assert_array_equal(idx.cpu().numpy().reshape(-1), exact)
    if not bf16:
        np.testing.assert_array_equal(idx.cpu().numpy().reshape(-1)[~near.any(-1)], f["indices"].reshape(-1)[~near.any(-1)])
    else:   # the pinned deviation: the reference's bf16 index sum is not the mixed-radix index of its own level indices
        ref_exact = (lev_ref.astype(np.int64) * O.basis(kw["levels"])).sum(-1)
        print(f"bf16 reference indices off their own level indices: {(ref_exact != f['indices'].reshape(-1)).sum()}")
    qv = q.detach().float().cpu().numpy()
    if not m.has_projections:
        qr = f["q"]
        if kw.get("channel_first"):
            qv, qr = np.moveaxis(qv, 1, -1), np.moveaxis(qr, 1, -1)
        qv, qr = qv.reshape(-1, d), qr.reshape(-1, d)
        exactq = ~diff
        if draws:
            exactq &= ~(f["u2"].reshape(-1, d) > (kw.get("quantize_rate", 0.) if bool(f["train"]) else 1.))
        if not inv:
            # act + (q - act) rounds like the reference's wherever the device's act has the CPU's bits; where the device math
            # function gives act one ulp apart, the sum may land one ulp apart
            ulps = np.abs(qv[exactq].view(np.int32).astype(np.int64) - qr[exactq].view(np.int32).astype(np.int64))
            print(f"unperturbed q_z one ulp apart: {(ulps == 1).sum()} of {exactq.sum()}")
            assert ulps.max(initial=0) <= 1 and (ulps == 1).sum() <= max(1, 0.01 * ulps.size)
        # perturbed and inverse-CDF elements: the device functions' ulps, amplified by the inverse CDF's slope
        np.testing.assert_allclose(qv[~diff], qr[~diff], rtol=2e-3 if inv else 1e-5, atol=1e-5 if inv else 1e-6)
    else:
        np.testing.assert_allclose(qv, f["q"], rtol=1e-4, atol=1e-4)
    if "p_accept_prob" in f:
        assert abs(float(info["p_accept_prob"]) - float(f["p_accept_prob"])) <= 2. / zf.size
    for s in STATS:
        _close_to_f64(info["norm_info"][s].detach().float().cpu().numpy(), f["stat_" + s], f["stat64_" + s], bf16)
    _close_to_f64([float(loss)], [float(f["loss"])], [float(f["loss64"])], bf16)
    _close_to_f64(z.grad.float().cpu().numpy().reshape(-1), f["dz"].reshape(-1), f["dz64"].reshape(-1), bf16)
    _close_to_f64(dx.float().cpu().numpy().reshape(-1), f["dx"].reshape(-1), f["dx64"].reshape(-1), bf16)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("act,inv", [("tanh", False), ("normal", True), ("cauchy", False)])
def test_seeded_run_matches_eager_and_generator(act, inv, dtype):
    """Same seed, same device: q_z as the eager formula gives it, and the generator left where two rand_like calls leave it."""
    vqb = _vqb()
    m = vqb.FSP(levels=[8, 5, 5, 5], act_name=act, need_inv_act=inv, quantize_rate=0.5).to(DEV).train()
    z = torch.randn(4096, 4, device=DEV).to(dtype)
    torch.cuda.manual_seed(11)
    q, idx, loss, info = m(z)
    after = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(11)
    qe, leve, losse, _, pe = O.eager_forward(z, [8, 5, 5, 5], act, inv, 0.5)
    torch.cuda.manual_seed(11)
    torch.rand_like(z)
    torch.rand_like(z)
    assert torch.equal(after, torch.cuda.get_rng_state())
    same = (info["level_indices"] == leve).all(-1)
    assert same.float().mean() > 0.999
    torch.testing.assert_close(q[same].float(), qe[same].float(), rtol=2e-5, atol=2e-5)
    assert abs(float(info["p_accept_prob"]) - float(pe)) <= 2. / z.numel()


def test_eval_and_rate_one_draw_nothing():
    vqb = _vqb()
    for m in (vqb.FSP(levels=[8, 5, 5, 5], quantize_rate=1.0).to(DEV).train(), vqb.FSP(levels=[8, 5, 5, 5]).to(DEV).eval()):
        z = torch.randn(1, 64, 4, device=DEV)
        before = torch.cuda.get_rng_state()
        out1, *_ = m(z)
        out2, *_, info = m(z)
        assert torch.equal(before, torch.cuda.get_rng_state()) and torch.equal(out1, out2) and "p_accept_prob" not in info


def test_reference_basic():
    m = _vqb().FSP(levels=[8, 5, 5, 5], act_name="normal", vector_norm="none").to(DEV)
    x = torch.randn(1, 1024, 4, device=DEV)
    q, idx, loss, info = m(x)
    assert q.shape == x.shape and idx.shape == (1, 1024) and loss.item() == 0.0 and isinstance(info, dict)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_reference_eval_roundtrip(dtype):
    m = _vqb().FSP(levels=[8, 5, 5, 5]).to(DEV).to(dtype).eval()
    x = torch.randn(1, 1024, 4, device=DEV, dtype=dtype)
    q, idx, *_ = m(x)
    rec = m.indices_to_codes(idx)
    torch.testing.assert_close(q.float(), rec.float(), atol=1e-5 if dtype == torch.float32 else 2e-2, rtol=0)
    assert torch.equal(m.indices_to_level_indices(idx), m.indices_to_level_indices(m.level_indices_to_indices(
        m.indices_to_level_indices(idx))))


def test_reference_index_encoding():
    m = _vqb().FSP(levels=[8, 5, 5, 5]).to(DEV)
    li = torch.tensor([[[7, 4, 4, 4]]], device=DEV)
    flat = m.level_indices_to_indices(li)
    assert flat.item() == 999 and torch.equal(m.indices_to_level_indices(flat), li)
    zero = torch.zeros(1, 1, 4, dtype=torch.int64, device=DEV)
    assert m.level_indices_to_indices(zero).item() == 0
    act = m.indices_to_act_value(flat)
    torch.testing.assert_close(act, (li.float() + 0.5) / m._levels)


def test_reference_image_input():
    m = _vqb().FSP(levels=[8, 5, 5, 5], dim=4, channel_first=True).to(DEV).eval()
    x = torch.randn(2, 4, 8, 8, device=DEV)
    q, idx, *_ = m(x)
    assert q.shape == x.shape and idx.shape == (2, 8, 8)
    rec = m.indices_to_codes(idx)
    assert rec.shape == x.shape
    torch.testing.assert_close(q, rec, atol=1e-5, rtol=0)


def test_reference_projection():
    m = _vqb().FSP(levels=[8, 5, 5, 5], dim=256).to(DEV).eval()
    assert m.has_projections
    x = torch.randn(1, 64, 256, device=DEV)
    q, idx, _, _ = m(x)
    assert q.shape == x.shape and idx.shape == (1, 64)
    torch.testing.assert_close(q, m.indices_to_codes(idx), atol=1e-4, rtol=0)


@pytest.mark.parametrize("dtype,autocast", [(torch.float32, False), (torch.bfloat16, True)])
def test_reference_training(dtype, autocast):
    vqb = _vqb()
    model = torch.nn.Sequential(torch.nn.Linear(256, 256), vqb.FSP(levels=[8, 5, 5, 5], dim=256),
                                torch.nn.Linear(256, 256)).to(DEV).to(dtype).train()
    x = torch.randn(2, 64, 256, dtype=dtype, device=DEV, requires_grad=True)
    with torch.autocast("cuda", dtype=dtype, enabled=autocast):
        h = model[0](x)
        q, idx, loss, info = model[1](h)
        out = model[2](q)
    assert q.dtype == dtype and idx.dtype == torch.int32
    assert (idx >= 0).all() and (idx < model[1].codebook_size).all()
    (out.sum() + loss).backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    for p in model.parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all()


def test_gradient_through_variance_only():
    """A loss on norm_info['variance'] alone reaches z through the statistics path (2 u / (N - 1) per unit gradient)."""
    m = _vqb().FSP(levels=[8, 5, 5, 5]).to(DEV).train()
    z = torch.randn(777, 4, device=DEV, dtype=torch.float64).float().requires_grad_(True)
    _, _, _, info = m(z)
    info["norm_info"]["variance"].sum().backward()
    zd = z.detach().double()
    ref = 2. * (zd - zd.mean(0)) / (zd.shape[0] - 1)
    torch.testing.assert_close(z.grad.double(), ref, rtol=1e-5, atol=1e-8)


def test_fp16_raises():
    m = _vqb().FSP(levels=[8, 5, 5, 5]).to(DEV)
    with pytest.raises(TypeError):
        m(torch.randn(1, 16, 4, device=DEV, dtype=torch.float16))


def test_deterministic():
    m = _vqb().FSP(levels=[8, 5, 5, 5], dim=32, quantize_rate=0.5, vector_norm="kurt").to(DEV).train()
    x = torch.randn(8, 1000, 32, device=DEV)
    outs = []
    for _ in range(2):
        torch.cuda.manual_seed(5)
        xx = x.clone().requires_grad_(True)
        q, idx, loss, info = m(xx)
        (q.square().sum() + loss).backward()
        outs.append([q, idx, loss, info["level_indices"], info["p_accept_prob"], *info["norm_info"].values(), xx.grad])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
