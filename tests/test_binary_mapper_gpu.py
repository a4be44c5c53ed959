"""BinaryMapper on the GPU: replay of the reference fixtures (tests/golden/binary_mapper) under the DESIGN 4.12 rules, the
refusals, and the Bernoulli draw against an eager restatement of the reference's sampling on the same device."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import binary_mapper_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "binary_mapper", "*.npz")))
DEV = "cuda"


def _vqb():
    import vector_quantize_pytorch_b200 as vqb
    return vqb


def _close_to_f64(ours, ref, ref64, bf16=False):
    """ours no further from float64 than the reference is (bf16: 1.5 times the largest deviation), or 2e-5 of the largest
    value; NaN exactly where the reference has NaN."""
    ours, ref, ref64 = (np.asarray(a, np.float64) for a in (ours, ref, ref64))
    np.testing.assert_array_equal(np.isnan(ours), np.isnan(ref))
    keep = ~np.isnan(ref)
    ours, ref, ref64 = ours[keep], ref[keep], ref64[keep]
    if ours.size == 0:
        return
    floor = 2e-5 * max(np.abs(ref64).max(), 1e-30)
    if bf16:
        assert np.abs(ours - ref64).max() <= 1.5 * np.abs(ref - ref64).max() + floor
        return
    bad = np.abs(ours - ref64) > np.abs(ref - ref64) + floor
    assert not bad.any(), f"{bad.sum()} elements: ours {ours[bad][:4]} ref {ref[bad][:4]} f64 {ref64[bad][:4]}"


def _upstream(f):
    rows, K = int(np.prod(f["lead"], dtype=np.int64)), 1 << int(f["bits"])
    return torch.randn(rows, K, generator=torch.Generator().manual_seed(int(f["g_seed"])))


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_replay(path, monkeypatch):
    from vector_quantize_pytorch_b200 import binary_mapper as bm_mod
    f = np.load(path)
    bits, lead = int(f["bits"]), tuple(int(v) for v in f["lead"])
    rows, K = int(np.prod(lead, dtype=np.int64)), 1 << bits
    ckw, fkw = json.loads(str(f["ckw"])), json.loads(str(f["fkw"]))
    bf16 = str(f["xdtype"]) == "bf16"
    dt = torch.bfloat16 if bf16 else torch.float32
    ref_idx = f["indices"].reshape(rows)
    recorded = torch.from_numpy(O.index_bits(ref_idx, bits))
    drawn = []

    def bernoulli(prob):   # the reference's draw, as recorded in its indices
        drawn.append(prob.shape)
        return recorded.to(prob.device, prob.dtype).reshape(prob.shape)
    monkeypatch.setattr(bm_mod, "_bernoulli", bernoulli)
    m = _vqb().BinaryMapper(bits=bits, **ckw).to(DEV).train(bool(f["train"]))
    x = torch.from_numpy(f["x"]).to(DEV, dt).requires_grad_(True)
    out, idx, aux = m(x, return_indices=True, **fkw)
    det = fkw.get("deterministic", ckw.get("deterministic_on_eval", False) and not bool(f["train"]))
    assert len(drawn) == (0 if det else 1)
    assert out.dtype == torch.float32 and tuple(out.shape) == (*lead, K)
    assert idx.dtype == torch.int64 and tuple(idx.shape) == lead
    st = fkw.get("straight_through", bool(f["train"]))
    assert out.requires_grad == st
    total = (out * _upstream(f).to(DEV).reshape(out.shape)).sum() if st else 0.0
    if aux.requires_grad:
        total = total + aux.sum()
    lp = m.log_prob(x, indices=idx)
    (total + (lp * torch.from_numpy(f["H"]).to(DEV, lp.dtype)).sum()).backward()

    # indices: bit for bit, except deterministic entries within 2^-22 of the threshold (sigmoid's last ulp)
    ours = idx.reshape(rows).cpu().numpy()
    tiny = np.zeros((rows, bits), bool)
    if det:
        tiny = np.abs(f["x"].reshape(rows, bits).astype(np.float64) / fkw.get("temperature", 1.0)) < 2.0 ** -22
    diff = O.index_bits(ours, bits) != O.index_bits(ref_idx, bits)
    print(f"{os.path.basename(path)}: {tiny.sum()} deterministic entries near the threshold, {diff.sum()} bits differ")
    assert not (diff & ~tiny).any()
    same_row = ~diff.any(-1)
    # output: non-hot elements exactly the reference's (0, or NaN at its NaN positions); hot within 2^-23
    o = out.detach().reshape(rows, K).cpu()
    hot = o[torch.arange(rows), torch.from_numpy(ours)].numpy()
    rest = o.clone()
    rest[torch.arange(rows), torch.from_numpy(ours)] = 0.0
    np.testing.assert_array_equal(torch.nonzero(torch.isnan(rest).reshape(-1)).reshape(-1).numpy(), f["nan_pos"])
    assert not (rest.nan_to_num(0.0) != 0).any() and not torch.signbit(rest.nan_to_num(0.0)).any()
    np.testing.assert_array_equal(np.isnan(hot), np.isnan(f["hot"]))
    fin = ~np.isnan(hot) & same_row
    hd = np.abs(hot[fin].astype(np.float64) - f["hot"][fin]) > 0
    print(f"hot elements differing from the reference's: {hd.sum()} of {fin.sum()}")
    assert (np.abs(hot[fin].astype(np.float64) - f["hot"][fin]) <= 2.0 ** -23).all()
    if not st:
        assert (hot == 1.0).all()
    # aux loss, log_prob and the gradient against the float64 rerun; rows whose bits differ are left out
    kind = str(f["aux_kind"])
    if kind == "zero":
        assert aux is m.zero
    else:
        assert aux.dtype == dt and tuple(aux.shape) == (() if kind == "mean" else lead)
        _close_to_f64(aux.detach().float().cpu().numpy(), f["aux"], f["aux64"], bf16)
    assert lp.dtype == dt
    sel = same_row.reshape(lead) if lead else bool(same_row[0])
    _close_to_f64(lp.detach().float().cpu().numpy()[sel], f["lp"][sel], f["lp64"][sel], bf16)
    lpb = m.log_prob(x, indices=idx, sum_bits=False).detach().float().cpu().numpy()
    _close_to_f64(lpb[sel], f["lp_bits"][sel], f["lp_bits64"][sel], bf16)
    # one_hot= takes the argmax, which lands on a NaN in a row with a non-finite logit (in the reference as well)
    fin = np.isfinite(f["x"].reshape(rows, bits)).all(-1) & same_row
    fin = fin.reshape(lead) if lead else bool(fin[0])
    lpo = m.log_prob(x, one_hot=out).detach().float().cpu().numpy()
    np.testing.assert_array_equal(lpo[fin], lp.detach().float().cpu().numpy()[fin])
    np.testing.assert_array_equal(m.log_prob(x, one_hot=out, sum_bits=False).detach().float().cpu().numpy()[fin], lpb[fin])
    assert x.grad.dtype == dt
    _close_to_f64(x.grad.float().cpu().numpy()[sel], f["dx"][sel], f["dx64"][sel], bf16)


def test_two_output_form_and_shapes():
    m = _vqb().BinaryMapper(bits=8).to(DEV)
    x = torch.randn(3, 4, 8, device=DEV)
    one_hot, aux = m(x)
    assert one_hot.shape == (3, 4, 256) and aux.shape == ()
    sparse, idx, aux = m(x, return_indices=True, reduce_aux_kl_loss=False)
    assert idx.shape == (3, 4) and aux.shape == (3, 4)
    np.testing.assert_allclose(m.log_prob(x, indices=idx).cpu(), m.log_prob(x, one_hot=sparse).cpu())
    m.eval()
    a, _ = m(x, deterministic=True)
    b, _ = m(x, deterministic=True)
    assert torch.equal(a, b) and not a.requires_grad
    e = m(torch.randn(0, 8, device=DEV), return_indices=True)
    assert e[0].shape == (0, 256) and e[1].shape == (0,)


def test_refusals_on_the_gpu():
    vqb = _vqb()
    m = vqb.BinaryMapper(bits=6).to(DEV)
    xb = torch.randn(4, 6, device=DEV).bfloat16()
    with pytest.raises(TypeError, match="reference"):
        m.train()(xb)
    with pytest.raises(TypeError, match="reference"):
        m.eval()(xb, straight_through=True)
    out, aux = m.eval()(xb)   # no straight-through: bf16 runs
    assert out.dtype == torch.float32
    with pytest.raises(TypeError):
        m(torch.randn(4, 6, device=DEV).half())
    with pytest.raises(NotImplementedError):
        vqb.BinaryMapper(bits=21)
    x = torch.randn(4, 6, device=DEV, requires_grad=True)
    out, _ = m.train()(x)
    (g,) = torch.autograd.grad((out * out).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):   # double backward is not supported
        g.sum().backward()


def _eager_indices(logits, temperature, power_two):
    """The reference's sampling restated in eager torch (bm:148-157)."""
    prob = (logits / temperature).sigmoid()
    return (power_two * prob.bernoulli().long()).sum(dim=-1)


@pytest.mark.parametrize("bits,shape,temperature", [(1, (64, 1), 1.0), (8, (4, 256, 8), 1.0), (16, (2, 64, 16), 0.5),
                                                     (20, (3, 20), 2.0)])
def test_seeded_draw_matches_eager_torch(bits, shape, temperature):
    m = _vqb().BinaryMapper(bits=bits).to(DEV).train()
    x = torch.randn(*shape, device=DEV) * 2
    torch.manual_seed(1234)
    _, idx, _ = m(x, temperature=temperature, return_indices=True)
    after = torch.cuda.get_rng_state()
    torch.manual_seed(1234)
    ref = _eager_indices(x.reshape(-1, bits), temperature, m.power_two).reshape(shape[:-1])
    assert torch.equal(idx, ref)
    assert torch.equal(torch.cuda.get_rng_state(), after), "the module consumes the generator as the reference does"


def test_two_seeded_runs_are_identical():
    m = _vqb().BinaryMapper(bits=12).to(DEV).train()
    x0 = torch.randn(64, 12, device=DEV)
    G = torch.randn(64, 4096, device=DEV)
    res = []
    for _ in range(2):
        torch.manual_seed(7)
        x = x0.clone().requires_grad_(True)
        out, idx, aux = m(x, return_indices=True)
        ((out * G).sum() + aux).backward()
        res.append((out.detach(), idx, aux.detach(), x.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_bit_frequencies_follow_prob():
    """A chi-square test at a fixed seed: each bit's count of ones over 2^18 rows against sigmoid(logit / t)."""
    bits, rows, t = 8, 1 << 18, 1.5
    m = _vqb().BinaryMapper(bits=bits).to(DEV).train()
    logit = torch.linspace(-3.0, 3.0, bits, device=DEV)
    torch.manual_seed(2024)
    _, idx, _ = m(logit.expand(rows, bits).contiguous(), temperature=t, return_indices=True)
    ones = ((idx[:, None] >> torch.arange(bits, device=DEV)) & 1).sum(0).double().cpu().numpy()
    p = torch.sigmoid(logit / t).double().cpu().numpy()
    chi2 = (((ones - rows * p) ** 2) / (rows * p * (1 - p))).sum()
    print(f"chi-square {chi2:.2f} with {bits} degrees of freedom")
    assert chi2 < 30.0   # the 99.98th percentile of chi-square(8) is about 30
