"""GPU tests of the EMA options and adjacent paths of SURVEY §8 (a8, a10, f1) — `pytest -m gpu` on an H100.

  * `ema_update_weight` (tensor / callable) and `accum_ema_update`: the reference's own tests
    (tests/test_readme.py:434-465, :467-492 of the reference) restated, plus the post-state against the oracle;
  * dead-code expiry (`threshold_ema_dead_code > 0`): post-state against the oracle given the same sampled rows
    (the oracle itself is pinned to the reference by the `expire_*` goldens, tests/test_oracle_golden.py);
  * decode (`get_output_from_indices`) against the oracle, including -1 entries;
  * the commitment loss stays differentiable w.r.t. `project_in` (vqp:1151, :1327).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import GOLDEN_DIR, Golden, grad_golden_names, simvq_golden_names
from oracle import vq_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def oracle_state(cb):
    return O.CodebookState(cb.embed[0].cpu().numpy().copy(), cb.embed_avg[0].cpu().numpy().copy(),
                           cb.cluster_size[0].cpu().numpy().copy())


def assert_state(cb, st, tol=1e-5):
    np.testing.assert_allclose(cb.cluster_size[0].cpu().numpy(), st.cluster_size, rtol=tol, atol=tol)
    np.testing.assert_allclose(cb.embed_avg[0].cpu().numpy(), st.embed_avg, rtol=tol, atol=tol)
    np.testing.assert_allclose(cb.embed[0].cpu().numpy(), st.embed, rtol=tol, atol=tol)


# ------------------------------------------------------------------------------------------------ ema_update_weight
@pytest.mark.parametrize("use_cosine_sim", (False, True))
@pytest.mark.parametrize("use_callable", (False, True))
def test_vq_custom_ema_update_weighting(use_cosine_sim, use_callable):
    """Reference tests/test_readme.py:434-465, same shapes; then the whole post-state against the oracle."""
    torch.manual_seed(11)
    vq = vqb().VectorQuantize(dim=256, use_cosine_sim=use_cosine_sim, codebook_dim=128, codebook_size=8, decay=0.8).to(DEV)
    x = torch.randn(16, 1024, 256, device=DEV)
    codebook_before = vq.codebook.clone()
    st = oracle_state(vq._codebook)
    weights = torch.tensor([0., 1., 1., 0., 1., 0., 0., 1.], device=DEV)
    seen = {}

    def update_weights_callable(embed_sum, cluster_size):
        seen["shapes"] = (tuple(embed_sum.shape), tuple(cluster_size.shape))
        return weights

    quantized, indices, loss = vq(x, ema_update_weight=update_weights_callable if use_callable else weights)
    torch.cuda.synchronize()
    codebook_after = vq.codebook
    did_update = weights.bool()
    assert torch.allclose(codebook_before[~did_update], codebook_after[~did_update], atol=1e-6)
    assert (codebook_before[did_update] != codebook_after[did_update]).all()
    if use_callable:  # the callable sees (embed_sum (h, c, d), cluster_size (h, c)) like vqp:609-610
        assert seen["shapes"] == ((1, 8, 128), (1, 8))
    # oracle EMA on the projected input (project_in is a random nn.Linear: evaluate it with torch, vqp:1151), from the module's
    # own indices: a near tie the two searches break differently must not skip the state check
    with torch.no_grad():
        xp = vq.project_in(x).cpu().numpy().reshape(-1, 128)
    if use_cosine_sim:
        xp = O.l2norm(xp)
    O.track_stats(st, xp, indices.reshape(-1).cpu().numpy(), 0.8, ema_update_weight=weights.cpu().numpy())
    O.update_ema(st, 1e-5, use_cosine_sim)
    assert_state(vq._codebook, st, 2e-5)


def test_accum_ema_update():
    """Reference tests/test_readme.py:467-492, then the folded update against the oracle."""
    torch.manual_seed(12)
    vq = vqb().VectorQuantize(dim=256, use_cosine_sim=True, codebook_dim=128, codebook_size=8, decay=0.8,
                              commitment_weight=1.).to(DEV)
    x = torch.randn(16, 1024, 256, device=DEV)
    codebook_before = vq.codebook.clone()
    st = oracle_state(vq._codebook)
    vq.train()
    _ = vq(x, accum_ema_update=True)
    _ = vq(x, accum_ema_update=True)
    assert torch.allclose(codebook_before, vq.codebook, atol=1e-6)
    assert vq._codebook.cluster_size.grad is not None and vq._codebook.embed_avg.grad is not None
    _ = vq(x)
    torch.cuda.synchronize()
    assert not torch.allclose(codebook_before, vq.codebook, atol=1e-6)
    assert vq._codebook.cluster_size.grad is None and vq._codebook.embed_avg.grad is None
    with torch.no_grad():
        xp = vq.project_in(x).cpu().numpy()
    cfg = O.VQConfig(dim=128, codebook_size=8, use_cosine_sim=True)
    acc = {}
    O.vq_forward(xp, "fp32", st, cfg, accum=acc, accum_ema_update=True)
    O.vq_forward(xp, "fp32", st, cfg, accum=acc, accum_ema_update=True)
    O.vq_forward(xp, "fp32", st, cfg, accum=acc)
    assert_state(vq._codebook, st, 2e-5)


def test_per_call_ema_update_override():
    """forward(ema_update=False) on a module with dead-code replacement tracks cluster_size / embed_avg but leaves
    `embed` alone (vqp:628-639); ema_update=True on a module built with ema_update=False updates it."""
    torch.manual_seed(13)
    m = vqb()
    x = torch.randn(4, 256, 64, device=DEV)
    vq = m.VectorQuantize(dim=64, codebook_size=32, threshold_ema_dead_code=1e-6).to(DEV)
    e0, cs0 = vq.codebook.clone(), vq._codebook.cluster_size.clone()
    vq(x, ema_update=False)
    assert torch.equal(e0, vq.codebook) and not torch.equal(cs0, vq._codebook.cluster_size)
    vq2 = m.VectorQuantize(dim=64, codebook_size=32, ema_update=False).to(DEV)
    e0 = vq2.codebook.clone()
    vq2(x)
    assert torch.equal(e0, vq2.codebook)
    vq2(x, ema_update=True)
    assert not torch.equal(e0, vq2.codebook)


def test_codebook_surface_names():
    """Codebook.update_codebook / track_cluster_size_and_embed_avg (vqp:586-641) bind and match update_indices."""
    torch.manual_seed(14)
    m = vqb()
    a, b = m.Codebook(dim=32, codebook_size=16, threshold_ema_dead_code=0).to(DEV), m.Codebook(dim=32, codebook_size=16, threshold_ema_dead_code=0).to(DEV)
    b.load_state_dict(a.state_dict())
    x = torch.randn(1, 512, 32, device=DEV)
    _, ind, _ = a(x)
    onehot = F.one_hot(ind, 16).float()
    c = m.Codebook(dim=32, codebook_size=16, threshold_ema_dead_code=0).to(DEV)
    c.load_state_dict(b.state_dict())
    b.update_codebook(x, onehot)
    assert torch.allclose(a.embed, b.embed, atol=1e-6) and torch.allclose(a.cluster_size, b.cluster_size, atol=1e-6)
    c.track_cluster_size_and_embed_avg(x, onehot)
    assert torch.allclose(a.embed_avg, c.embed_avg, atol=1e-6) and not torch.allclose(a.embed, c.embed, atol=1e-6)


# ------------------------------------------------------------------------------------------------ dead-code expiry
def cuda_pick_fn(n, num):
    """The product draws sample_vectors (vqp:156-163) on the CUDA generator; the test re-seeds it and replays."""
    p = torch.randperm(n, device=DEV)[:num] if n >= num else torch.randint(0, n, (num,), device=DEV)
    return p.cpu().numpy()


@pytest.mark.parametrize("name", ["expire_vq_fp32", "expire_vq_cosine_bf16", "expire_rvq_shared_fp32", "expire_rvq_separate_fp32"])
def test_dead_code_expiry_matches_oracle(name):
    """Same inputs / initial state as the reference-generated `expire_*` goldens; the sampled rows differ from the
    golden's (CPU vs CUDA generator), so the comparison is against the oracle replaying OUR draws."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    kw = dict(dim=meta["dim"], codebook_size=meta["codebook_size"], threshold_ema_dead_code=meta["threshold_ema_dead_code"])
    if meta.get("use_cosine_sim"):
        kw["use_cosine_sim"] = True
    if meta["kind"] == "vq":
        module = m.VectorQuantize(**kw).to(DEV)
    else:
        module = m.ResidualVQ(num_quantizers=meta["num_quantizers"], shared_codebook=meta["shared_codebook"], **kw).to(DEV)
    books = []
    for sub in module.modules():
        if isinstance(sub, m.Codebook) and all(sub is not b for b in books):
            books.append(sub)
    for i, cb in enumerate(books):
        st = g.state("s0_pre", i)
        with torch.no_grad():
            cb.embed.copy_(torch.from_numpy(st.embed)[None]); cb.embed_avg.copy_(torch.from_numpy(st.embed_avg)[None])
            cb.cluster_size.copy_(torch.from_numpy(st.cluster_size)[None])
    states = g.states("s0_pre")
    flat = g.flat_states(states)
    dt = meta["dtype"]
    module.train()
    replaced_total = 0
    for step in range(len(meta["steps"])):
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(torch.bfloat16 if dt == "bf16" else torch.float32)
        before = [cb.embed.clone() for cb in books]
        torch.manual_seed(9000 + step)
        q, ind, loss = module(x)[:3]
        torch.cuda.synchronize()
        torch.manual_seed(9000 + step)
        if meta["kind"] == "vq":
            qo, io, lo, _ = O.vq_forward(g[f"s{step}_x"], dt, states, g.cfg, pick_fn=cuda_pick_fn)
        else:
            qo, io, lo, _ = O.rvq_forward(g[f"s{step}_x"], dt, states, g.cfg, shared_codebook=meta["shared_codebook"],
                                          pick_fn=cuda_pick_fn)
        assert np.array_equal(ind.cpu().numpy(), io), f"{name} step {step}: indices differ (stale operands after expiry?)"
        np.testing.assert_allclose(q.float().cpu().numpy(), qo, rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-5 if dt == "fp32" else 8e-3)
        for cb, st in zip(books, flat):
            assert_state(cb, st, 2e-5)
        replaced_total += sum(int((cb.cluster_size[0] == meta["threshold_ema_dead_code"]).sum()) for cb in books)
    assert replaced_total > 0, "the fixture is meant to replace dead codes"


@pytest.mark.parametrize("name", ["kmeans_vq_fp32", "kmeans_vq_cosine_bf16"])
def test_kmeans_init_matches_oracle(name):
    """kmeans_init=True (vqp:238-278, :451-473): every Lloyd iteration runs the search + statistics kernels.  Inputs as in
    the reference-generated `kmeans_*` goldens (which pin the oracle); sampled seeds replayed from the CUDA generator."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    kw = dict(dim=meta["dim"], codebook_size=meta["codebook_size"], kmeans_init=True, kmeans_iters=meta["kmeans_iters"])
    if meta.get("use_cosine_sim"):
        kw["use_cosine_sim"] = True
    module = m.VectorQuantize(**kw).to(DEV)
    state = g.states("s0_pre")
    assert not state.initted and not bool(module._codebook.initted)
    dt = meta["dtype"]
    module.train()
    for step in range(len(meta["steps"])):
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(torch.bfloat16 if dt == "bf16" else torch.float32)
        torch.manual_seed(9100 + step)
        q, ind, loss = module(x)
        torch.cuda.synchronize()
        torch.manual_seed(9100 + step)
        qo, io, lo, _ = O.vq_forward(g[f"s{step}_x"], dt, state, g.cfg, pick_fn=cuda_pick_fn)
        assert bool(module._codebook.initted)
        assert np.array_equal(ind.cpu().numpy(), io), f"{name} step {step}"
        np.testing.assert_allclose(loss.item(), float(lo), rtol=1e-5 if dt == "fp32" else 8e-3)
        assert_state(module._codebook, state, 3e-5)


def test_forward_host_expires_dead_codes():
    torch.manual_seed(15)
    vq = vqb().VectorQuantize(dim=64, codebook_size=64, threshold_ema_dead_code=2).to(DEV)
    x = (torch.randn(8, 1, 64).repeat(1, 512, 1) + 0.05 * torch.randn(8, 512, 64)).pin_memory()  # 8 clusters
    vq.forward_host(x, n_chunks=2)
    torch.cuda.synchronize()
    assert int((vq._codebook.cluster_size[0] == 2).sum()) > 0


# ------------------------------------------------------------------------------------------------ decode (f1)
def test_decode_matches_oracle_with_dropout_entries():
    torch.manual_seed(16)
    m = vqb()
    rvq = m.ResidualVQ(dim=64, num_quantizers=5, codebook_size=96).to(DEV)
    with torch.no_grad():
        for layer in rvq.layers:
            layer._codebook.embed.copy_(torch.randn(1, 96, 64))
    idx = torch.randint(0, 96, (3, 77, 5), device=DEV)
    idx[0, :10, 3:] = -1   # quantize-dropout style -1 entries contribute zeros (rvq:341-342, :371)
    idx[2, 5, 0] = -1
    out = rvq.get_output_from_indices(idx)
    embeds = [layer._codebook.embed[0].cpu().numpy() for layer in rvq.layers]
    ref = O.rvq_output_from_indices(embeds, idx.cpu().numpy())
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-6, atol=1e-6)
    codes = rvq.get_codes_from_indices(idx)
    assert codes.shape == (5, 3, 77, 64)
    # large batches take the shared-memory slice kernel (N >= 4096): same sums, -1 entries included; shared codebook too
    big = torch.randint(-1, 96, (4, 1500, 5), device=DEV)
    out = rvq.get_output_from_indices(big)
    ref = O.rvq_output_from_indices(embeds, big.cpu().numpy())
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-6, atol=1e-5)
    shared = m.ResidualVQ(dim=64, num_quantizers=4, codebook_size=200, shared_codebook=True).to(DEV)
    big = torch.randint(0, 200, (2, 3000, 4), device=DEV)
    ref = O.rvq_output_from_indices([shared.layers[0]._codebook.embed[0].cpu().numpy()] * 4, big.cpu().numpy())
    np.testing.assert_allclose(shared.get_output_from_indices(big).cpu().numpy(), ref, rtol=1e-6, atol=1e-5)
    vq = m.VectorQuantize(dim=64, codebook_size=96).to(DEV)
    i1 = torch.randint(0, 96, (2, 33), device=DEV)
    np.testing.assert_array_equal(vq.get_codes_from_indices(i1).cpu().numpy(),
                                  O.vq_codes_from_indices(vq.codebook.cpu().numpy(), i1.cpu().numpy()))
    g = m.GroupedResidualVQ(dim=64, groups=2, num_quantizers=3, codebook_size=48).to(DEV)
    gi = torch.randint(0, 48, (2, 4, 19, 3), device=DEV)
    out = g.get_output_from_indices(gi).cpu().numpy()
    ref = np.concatenate([O.rvq_output_from_indices([l._codebook.embed[0].cpu().numpy() for l in r.layers], gi[k].cpu().numpy())
                          for k, r in enumerate(g.rvqs)], axis=-1)
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------ project_in gradient
def test_commit_loss_trains_project_in():
    """Raw input without grad + codebook_dim != dim: the loss must reach project_in (vqp:1151, :1327)."""
    torch.manual_seed(17)
    vq = vqb().VectorQuantize(dim=64, codebook_dim=32, codebook_size=40).to(DEV)
    x = torch.randn(2, 100, 64, device=DEV)
    q, ind, loss = vq(x, freeze_codebook=True)   # frozen: the codes the kernel gathered are still in the codebook
    assert loss.requires_grad
    loss.backward()
    gw = vq.project_in.weight.grad
    assert gw is not None and torch.isfinite(gw).all() and gw.abs().sum() > 0
    # reference gradient: mse(quantize.detach(), project_in(x)) with the indices the kernel chose
    w = vq.project_in.weight.detach().clone().requires_grad_(True)
    b = vq.project_in.bias.detach().clone().requires_grad_(True)
    F.mse_loss(vq.get_codes_from_indices(ind).detach(), F.linear(x, w, b)).backward()
    assert torch.allclose(gw, w.grad, rtol=1e-4, atol=1e-7)
    rvq = vqb().ResidualVQ(dim=64, codebook_dim=32, num_quantizers=3, codebook_size=40).to(DEV)
    _, _, losses = rvq(x)
    losses.sum().backward()
    assert rvq.project_in.weight.grad is not None and rvq.project_in.weight.grad.abs().sum() > 0


# ------------------------------------------------------------------------------------------------ gradient estimators (f2)
@pytest.mark.parametrize("name", grad_golden_names())
def test_gradient_estimators_match_reference(name):
    """Rotation trick (default) / straight-through (vqp:282-318, :1225-1233): d(sum(quantize * G) + loss)/dx against the
    gradient the UNMODIFIED reference computed for the same x, G and codebook (oracle/gen_golden.py --grad).  The rotation
    trick's forward and backward run in the vqb_rotate kernel."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    kw = dict(dim=meta["dim"], codebook_size=meta["codebook_size"])
    for k in ("use_cosine_sim", "rotation_trick"):
        if k in meta:
            kw[k] = meta[k]
    if meta["kind"] == "vq":
        module = m.VectorQuantize(**kw).to(DEV)
    else:
        module = m.ResidualVQ(num_quantizers=meta["num_quantizers"], shared_codebook=meta["shared_codebook"], **kw).to(DEV)
    books = []
    for sub in module.modules():
        if isinstance(sub, m.Codebook) and all(sub is not b for b in books):
            books.append(sub)
    for i, cb in enumerate(books):
        st = g.state("s0_pre", i)
        with torch.no_grad():
            cb.embed.copy_(torch.from_numpy(st.embed)[None]); cb.embed_avg.copy_(torch.from_numpy(st.embed_avg)[None])
            cb.cluster_size.copy_(torch.from_numpy(st.cluster_size)[None])
    dt = torch.bfloat16 if meta["dtype"] == "bf16" else torch.float32
    x = torch.from_numpy(g["s0_x"]).to(DEV).to(dt).requires_grad_(True)
    G = torch.from_numpy(g["s0_G"]).to(DEV).to(dt)
    module.train()
    q, ind, loss = module(x, freeze_codebook=True)
    ((q * G).sum() + loss.sum().to(q.dtype)).backward()
    torch.cuda.synchronize()
    assert np.array_equal(ind.cpu().numpy(), g["s0_indices"])
    tol = 2e-5 if meta["dtype"] == "fp32" else 3e-2
    np.testing.assert_allclose(q.detach().float().cpu().numpy(), g["s0_quantize"], rtol=tol, atol=tol)
    np.testing.assert_allclose(loss.detach().float().cpu().numpy(), g["s0_loss"], rtol=1e-5 if meta["dtype"] == "fp32" else 8e-3, atol=1e-7)
    ref = g["s0_xgrad"]
    got = x.grad.float().cpu().numpy()
    scale = np.abs(ref).max()
    np.testing.assert_allclose(got, ref, rtol=tol, atol=tol * scale)


# ------------------------------------------------------------------------------------------------ vqb_rvq_forward
@pytest.mark.parametrize("kind", ["rvq_shared_bf16", "rvq_separate_fp32", "rvq_cosine_fp32", "grvq_fp32", "rvq_eval_bf16"])
def test_rvq_program_equals_stagewise_path(kind, monkeypatch):
    """One vqb_rvq_forward call (cached op list, one CUDA graph, groups on parallel lanes) must give the results of the
    stage-by-stage path bit for bit: same kernels, same order (residual_vq.py:469-568, :593-601, :690-724)."""
    import copy
    m = vqb()
    torch.manual_seed(11)
    cosine = "cosine" in kind
    dt = torch.bfloat16 if "bf16" in kind else torch.float32
    if kind.startswith("grvq"):
        mod = m.GroupedResidualVQ(dim=128, groups=2, num_quantizers=3, codebook_size=96).to(DEV)
        width = 128
    else:
        mod = m.ResidualVQ(dim=64, num_quantizers=4, codebook_size=200, shared_codebook="shared" in kind or "eval" in kind,
                           use_cosine_sim=cosine).to(DEV)
        width = 64
    ref = copy.deepcopy(mod)
    if "eval" in kind:
        mod.eval(); ref.eval()
    for step in range(4):   # step 0 initialises (stage-wise in both), later steps replay the cached program
        x = torch.randn(3, 1500, width, device=DEV).to(dt)
        monkeypatch.setenv("VQB_RVQ_PROGRAM", "1")
        q1, i1, l1 = mod(x)[:3]
        monkeypatch.setenv("VQB_RVQ_PROGRAM", "0")
        q0, i0, l0 = ref(x)[:3]
        torch.cuda.synchronize()
        assert torch.equal(i1, i0), f"step {step}: indices differ"
        assert torch.equal(q1, q0), f"step {step}: quantized differs"
        assert torch.equal(l1, l0), f"step {step}: losses differ"
        # the statistics add a code's re-scored rows with atomics: two such rows on one code may land in either order
        for a, b in zip(mod.buffers(), ref.buffers()):
            torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6, msg=f"step {step}: codebook state differs")
        ref.load_state_dict(mod.state_dict())   # identical pre-state for the next step: outputs must then be bit-equal
    assert len(mod.__dict__.get("_plans", {})) >= 1, "the program path was not taken"


# ------------------------------------------------------------------------------------------------ SimVQ (sim_vq.py)
@pytest.mark.parametrize("name", simvq_golden_names())
def test_simvq_matches_reference(name):
    """SimVQ on the search kernel: indices, quantized, loss and the gradients to x and to the codebook transform against the
    reference's (sim_vq.py:99-139); plus a config-2-sized search against brute-force fp64 arg-min."""
    import json, os
    m = vqb()
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = json.loads(bytes(g["meta"]).decode())
    mod = m.SimVQ(dim=meta["dim"], codebook_size=meta["codebook_size"], rotation_trick=meta["rotation_trick"]).to(DEV)
    with torch.no_grad():
        mod.frozen_codebook.copy_(torch.from_numpy(g["frozen"]))
        mod.code_transform.weight.copy_(torch.from_numpy(g["weight"]))
    x = torch.from_numpy(g["s0_x"]).to(DEV).requires_grad_(True)
    G = torch.from_numpy(g["s0_G"]).to(DEV)
    q, ind, loss = mod(x)
    ((q * G).sum() + loss).backward()
    assert np.array_equal(ind.cpu().numpy(), g["s0_indices"])
    np.testing.assert_allclose(q.detach().cpu().numpy(), g["s0_quantize"], rtol=1e-5, atol=2e-5)
    np.testing.assert_allclose(loss.item(), float(g["s0_loss"]), rtol=1e-5)
    np.testing.assert_allclose(x.grad.cpu().numpy(), g["s0_xgrad"], rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(mod.code_transform.weight.grad.cpu().numpy(), g["s0_wgrad"], rtol=1e-4, atol=2e-5)
    codes = mod.indices_to_codes(ind)
    np.testing.assert_allclose(codes.detach().cpu().numpy(), (torch.from_numpy(g["frozen"]) @ torch.from_numpy(g["weight"]).T)[g["s0_indices"]].numpy(),
                               rtol=1e-5, atol=1e-5)
    if name.endswith("rotation_fp32"):   # one larger search: exact arg-min up to fp64 near-ties
        torch.manual_seed(3)
        big = m.SimVQ(dim=256, codebook_size=1024).to(DEV)
        xb = torch.randn(4, 4096, 256, device=DEV)
        _, ib, _ = big(xb)
        cb = big.codebook.detach().double()
        d = torch.cdist(xb.reshape(-1, 256).double(), cb)
        best = d.argmin(-1)
        bad = ib.reshape(-1) != best
        if bad.any():
            two = d[bad].topk(2, largest=False).values
            assert ((two[:, 1] - two[:, 0]) / two[:, 1] < 1e-5).all(), "SimVQ index differs from the fp64 arg-min outside near ties"

