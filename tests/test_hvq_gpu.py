"""HierarchicalVQ on the GPU: replay of the reference's steps (tests/golden/hvq/, oracle/gen_golden_hvq.py) with the reference's
k-means / dead-code draws substituted for ours, the reference's own test_hq, and the kernels an eval forward launches.

Per step of a fixture: the indices equal at every scale; the reconstruction, the loss and x.grad no further from the float64
rerun than the fp32 reference is, or 2e-5 of the largest value; the codebook buffers after every scale's call within 1e-5 of
the reference's (relative to the largest; the EMA sums our own pooled rows, which differ from the reference's by fp32
rounding); get_output_from_indices against its float64 value, and in eval at (scales[-1], scales[-1]) bit for bit equal to
the forward.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(p for p in os.listdir(os.path.join(HERE, "golden", "hvq")) if p.endswith(".npz"))


class _Replay:
    """Hands out the reference's recorded draws in call order in place of torch.randperm / torch.randint."""

    def __init__(self, kinds, arrays):
        self.draws = list(zip(kinds, arrays))

    def take(self, kind, device):
        assert self.draws, f"the module drew more from the RNG than the reference ({kind})"
        k, a = self.draws.pop(0)
        assert k == kind, (k, kind)
        return torch.from_numpy(a).to(device)


@pytest.fixture(autouse=True)
def full_fp32_conv(monkeypatch):
    """phi's conv is torch's nn.Conv2d and follows torch's precision settings, whose default lets cuDNN use TF32; the fp32
    reference these tests compare with ran it in fp32."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def close_to_f64(ours, ref, ref64, what):
    ours, ref, ref64 = (np.asarray(a, np.float64) for a in (ours, ref, ref64))
    floor = 2e-5 * max(np.abs(ref64).max(), 1e-30)
    bad = np.abs(ours - ref64) > np.abs(ref - ref64) + floor
    assert not bad.any(), f"{what}: {bad.sum()} elements, ours {ours[bad][:4]} ref {ref[bad][:4]} f64 {ref64[bad][:4]}"


def build(m, f, meta):
    keys = json.loads(str(f["sd_keys"]))
    hq = m.HierarchicalVQ(**meta["kw"], accept_image_fmap=True)
    hq.load_state_dict({k: torch.from_numpy(f[f"sd_{j}"]) for j, k in enumerate(keys)})
    return hq.to(DEV).train(meta["train"])


@pytest.mark.parametrize("name", [p[:-4] for p in FIXTURES])
def test_replays_reference(name, monkeypatch):
    import vector_quantize_pytorch_b200 as m
    f = np.load(os.path.join(HERE, "golden", "hvq", name + ".npz"))
    meta = json.loads(bytes(f["meta"]).decode())
    hq = build(m, f, meta)
    train, scales = meta["train"], meta["scales"]
    cb = hq.vq._codebook
    after = []
    hq.vq.register_forward_hook(lambda mod, inp, out: after.append(
        (out[1].cpu().numpy(), cb.cluster_size[0].cpu().numpy(), cb.embed_avg[0].cpu().numpy(), cb.embed[0].cpu().numpy())))
    for s in range(meta["steps"]):
        kinds = json.loads(str(f[f"rng_kinds_{s}"]))
        replay = _Replay(kinds, [f[f"rng_{s}_{j}"] for j in range(len(kinds))])
        after.clear()
        x = torch.from_numpy(f[f"x_{s}"]).to(DEV).requires_grad_(train)
        with monkeypatch.context() as mp:
            mp.setattr(torch, "randperm", lambda *a, device=None, **k: replay.take("randperm", device))
            mp.setattr(torch, "randint", lambda *a, device=None, **k: replay.take("randint", device))
            recon, indices, loss = hq(x)
        assert not replay.draws, "the module drew less from the RNG than the reference"
        assert len(indices) == len(scales) and len(after) == len(scales)
        for k, sc in enumerate(scales):
            assert indices[k].shape == (x.shape[0], sc, sc) and indices[k].dtype == torch.int64
            np.testing.assert_array_equal(indices[k].cpu().numpy(), f[f"s{s}_k{k}_indices"], err_msg=f"step {s} scale {k}")
            for got, key in zip(after[k][1:], ("cluster_size", "embed_avg", "embed")):
                want = f[f"s{s}_k{k}_{key}"]
                np.testing.assert_allclose(got, want, rtol=0, atol=1e-5 * max(np.abs(want).max(), 1.0),
                                           err_msg=f"{key} after step {s} scale {k}")
        assert recon.shape == x.shape and recon.dtype == torch.float32
        close_to_f64(recon.detach().cpu().numpy(), f[f"recon_{s}"], f[f"recon64_{s}"], f"recon step {s}")
        close_to_f64(loss.detach().cpu().numpy(), f[f"loss_{s}"], f[f"loss64_{s}"], f"loss step {s}")
        if train:
            ((recon * torch.from_numpy(f[f"G_{s}"]).to(DEV)).sum() + loss).backward()
            close_to_f64(x.grad.cpu().numpy(), f[f"xgrad_{s}"], f[f"xgrad64_{s}"], f"x.grad step {s}")
    last = tuple(torch.from_numpy(f[f"s{meta['steps'] - 1}_k{k}_indices"]).to(DEV) for k in range(len(scales)))
    with torch.no_grad():
        gofi = hq.get_output_from_indices(last)
    S = scales[-1]
    assert gofi.shape == (x.shape[0], x.shape[1], S, S)
    close_to_f64(gofi.cpu().numpy(), f["gofi"], f["gofi64"], "get_output_from_indices")
    if not train and tuple(x.shape[-2:]) == (S, S):
        assert torch.equal(gofi, recon), "eval forward and get_output_from_indices differ"


@pytest.mark.parametrize("quant_resi,share", [(0.5, 1), (0.0, 1), (0.5, 0), (0.5, 2)])
def test_eval_forward_equals_output_from_indices(quant_resi, share):
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    hq = m.HierarchicalVQ(dim=32, codebook_size=256, scales=(1, 2, 3, 5, 8), quant_resi=quant_resi, share_quant_resi=share,
                          accept_image_fmap=True).to(DEV)
    x = torch.randn(4, 32, 8, 8, device=DEV)
    hq.train()
    hq(x)
    hq.eval()
    with torch.no_grad():
        recon, indices, loss = hq(x)
        again = hq.get_output_from_indices(indices)
    assert torch.equal(recon, again) and float(loss) == 0.0


def test_hq():
    """The reference's own test (tests/test_readme.py::test_hq)."""
    from vector_quantize_pytorch_b200 import HierarchicalVQ
    hq = HierarchicalVQ(dim=32, codebook_size=128, accept_image_fmap=True, scales=(1, 2, 4, 7), quant_resi=0.5,
                        share_quant_resi=1).to(DEV)
    x = torch.randn(1, 32, 7, 7, device=DEV)
    quantized, indices, commit_loss = hq(x)
    reconstructed = hq.get_output_from_indices(indices)
    assert quantized.shape == x.shape
    assert reconstructed.shape == x.shape
    assert len(indices) == 4
    assert torch.isfinite(commit_loss).all()


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and not e.name.startswith(("Memcpy", "Memset"))}


@pytest.mark.parametrize("quant_resi", [0.5, 0.0])
def test_eval_forward_launches_only_vqb_and_conv_kernels(quant_resi):
    """Every kernel of a (warm) eval forward is one of this package's or one that phi's nn.Conv2d launches on its own on the
    same input (cuDNN's kernels and the bias add)."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(1)
    hq = m.HierarchicalVQ(dim=32, codebook_size=512, scales=(1, 2, 3, 4, 6, 8, 12, 16), quant_resi=quant_resi,
                          accept_image_fmap=True).to(DEV)
    x = torch.randn(8, 32, 16, 16, device=DEV)
    hq.train()
    hq(x)
    hq.eval()
    with torch.no_grad():
        for _ in range(2):
            hq(x)
        conv = _kernels(lambda: hq.phi_shared.conv(x)) if quant_resi else set()
        seen = _kernels(lambda: hq(x))
    ours = {k for k in seen if "vqb" in k}
    assert any("hvq_pool_kernel" in k for k in ours) and any("hvq_up_kernel" in k for k in ours)
    assert seen - ours <= conv, f"kernels outside the package and the conv: {sorted(seen - ours - conv)}"
