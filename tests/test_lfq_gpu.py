"""Module replay of the reference fixtures (oracle/gen_golden_lfq.py) on the GPU: LFQ, ResidualLFQ, GroupedResidualLFQ.

The fixture's z (the project_in output the reference quantized) is fed in through a hook on project_in, so the kernels see the
reference's rows, and the quantizer's output is taken at the project_out input (the projections are torch matmuls whose
summation order differs by device).  Indices and eval outputs must match bit for bit, training outputs too except where the
input passes a soft clamp, an l2norm or a rotation matmul (DESIGN §4.10).  Losses and gradients at z are held to the fixture's
own bound: their distance from the reference's float64 run may not exceed max(the fp32 reference's distance from it, 2e-5 of
the largest value)."""
import glob
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "lfq", "*.npz")))
DEV = "cuda"


def _build(f):
    import vector_quantize_pytorch_b200 as vqb
    kw = json.loads(str(f["kwargs"]))
    torch.manual_seed(int(f["seed"]))
    mod = getattr(vqb, str(f["cls"]))(**kw)
    sd = {k[3:]: torch.from_numpy(f[k]) for k in f.files if k.startswith("sd.")}
    mod.load_state_dict(sd, strict=True)
    mod = mod.to(DEV)
    mod.train(bool(f["train"]))
    return mod, kw


def _project_ins(mod):
    cls = type(mod).__name__
    if cls == "GroupedResidualLFQ":
        return [r.project_in for r in mod.rvqs]
    return [mod.project_in]


def _replay(f):
    mod, kw = _build(f)
    dt = torch.bfloat16 if str(f["xdtype"]) == "bf16" else torch.float32
    x = torch.from_numpy(f["x"]).to(DEV, dt).requires_grad_(True)
    zs, qs = [], []
    for j, pi in enumerate(_project_ins(mod)):
        z = torch.from_numpy(f[f"z{j}"]).to(DEV, dt).requires_grad_(True)
        zs.append(z)
        pi.register_forward_hook(lambda _m, _i, _o, z=z: z.reshape(_o.shape) + 0 * _o.sum())
    pos = [r.project_out for r in mod.rvqs] if type(mod).__name__ == "GroupedResidualLFQ" else [mod.project_out]
    for po in pos:
        po.register_forward_pre_hook(lambda _m, inp: qs.append(inp[0].detach().clone()))
    fkw = json.loads(str(f["fkw"]))
    if "mask" in f:
        fkw["mask"] = torch.from_numpy(f["mask"]).to(DEV)
    torch.manual_seed(int(f["fwd_seed"]))
    cls = str(f["cls"])
    if cls == "GroupedResidualLFQ" and bool(f["train"]):
        # the fixture ran on the CPU, where the group seed (rlfq:275, torch.randint on x's device) came from the CPU generator
        # before the frac draws; on the GPU it comes from the CUDA generator, so replay the CPU draw the reference made
        torch.randint(0, 10_000, ())
    if cls == "LFQ":
        (out, idx, aux), bd = mod(x, return_loss_breakdown=True, **fkw)
        losses = aux
    else:
        out, idx, losses = mod(x, **fkw)
        bd = None
    return mod, x, zs, qs, out, idx, losses, bd


def _within_fixture_bound(got, ref32, ref64, what):
    """|got - ref64| <= max(|ref32 - ref64|, 2e-5 max|ref64|) (largest elements compared)."""
    got, ref32, ref64 = got.double(), ref32.double(), ref64.double()
    bound = max(float((ref32 - ref64).abs().max()), 2e-5 * float(ref64.abs().max()), 1e-9)
    err = float((got - ref64).abs().max())
    assert err <= bound, (what, err, bound)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_replay(path):
    f = np.load(path)
    mod, x, zs, qs, out, idx, losses, bd = _replay(f)
    kw = json.loads(str(f["kwargs"]))
    train = bool(f["train"])
    assert str(idx.dtype) == str(f["idx_dtype"]) and str(out.dtype) == str(f["out_dtype"])
    assert torch.equal(idx.cpu(), torch.from_numpy(f["indices"]))
    inexact = bool(kw.get("soft_clamp_input_value") or kw.get("spherical") or kw.get("orthogonal_rotation"))
    for j, q in enumerate(qs):
        ref = torch.from_numpy(f[f"q{j}"])
        got = q.float().cpu()
        if kw.get("orthogonal_rotation"):   # the rotation back is a torch matmul
            torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6)
        elif not train or not inexact:
            assert torch.equal(got, ref), (j, int((got != ref).sum()))
        else:   # the documented rounding positions: a few ulps where the clamp / l2norm / rotation rounds differently
            diff = (got - ref).abs() > 0
            assert diff.float().mean() <= 0.02, float(diff.float().mean())
            torch.testing.assert_close(got, ref, rtol=4e-7 if got.dtype == torch.float32 else 1e-2, atol=1e-7)
    ref_l = torch.from_numpy(f["losses"])
    _within_fixture_bound(losses.detach().reshape(-1).cpu(), ref_l, torch.from_numpy(f["losses64"]), "losses")
    if bd is not None:
        got = torch.tensor([float(v.detach()) for v in bd], dtype=torch.float64)
        torch.testing.assert_close(got, torch.from_numpy(f["breakdown"]), rtol=2e-5, atol=2e-6)
    if not train:
        return
    G = torch.from_numpy(f["G"]).to(DEV, out.dtype)
    total = (out.float() * G.float()).sum() + losses.float().sum()
    total.backward()
    for j, z in enumerate(zs):
        _within_fixture_bound(z.grad.cpu(), torch.from_numpy(f[f"gz{j}"]), torch.from_numpy(f[f"gz64_{j}"]), f"grad z{j}")


def test_readme_invariants():
    import vector_quantize_pytorch_b200 as vqb
    torch.manual_seed(0)
    q = vqb.LFQ(codebook_size=65536, dim=16, entropy_loss_weight=0.1, diversity_gamma=1.).to(DEV).eval()
    image = torch.randn(1, 16, 32, 32, device=DEV)
    quantized, indices, _ = q(image)
    assert quantized.shape == image.shape and indices.shape == (1, 32, 32)
    assert torch.equal(quantized, q.indices_to_codes(indices))
    r = vqb.ResidualLFQ(dim=256, codebook_size=256, num_quantizers=8).to(DEV).eval()
    x = torch.randn(1, 1024, 256, device=DEV)
    out, ind, loss = r(x)
    assert ind.shape == (1, 1024, 8) and loss.shape == (8,)
    torch.testing.assert_close(r.get_output_from_indices(ind), out, rtol=1e-6, atol=1e-6)
    s = vqb.LFQ(codebook_size=1024, spherical=True, codebook_scale=1.5).to(DEV).eval()
    xs = torch.randn(4, 50, 10, device=DEV)
    qs, ids, _ = s(xs)
    assert torch.equal(qs, s.indices_to_codes(ids))


def test_grouped_one_forward_launch():
    import vector_quantize_pytorch_b200 as vqb
    from vector_quantize_pytorch_b200 import ops
    torch.manual_seed(0)
    m = vqb.GroupedResidualLFQ(dim=64, groups=2, codebook_size=512, num_quantizers=4).to(DEV).train()
    x = torch.randn(2, 100, 64, device=DEV, requires_grad=True)
    before = ops.LAUNCHES
    out, idx, losses = m(x)
    assert ops.LAUNCHES - before == 2   # one row-chain launch and one entropy launch for both groups and all stages
    assert idx.shape == (2, 2, 100, 4) and losses.shape == (2, 4)
    before = ops.LAUNCHES
    (out.sum() + losses.sum()).backward()
    assert ops.LAUNCHES - before == 3   # the entropy backward (two kernels) and one row-chain backward
