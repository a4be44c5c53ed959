"""CPU checks of codebooks learnt by gradient: the numpy restatement (oracle/learnable_oracle.py) against the reference's own
steps (tests/golden/learnable/), the module surface against the reference's construction rules, and the state_dict."""
import numpy as np
import pytest
import torch

from learnable_golden import Fixture, names
from oracle import learnable_oracle as O


def _tol(f):
    # bf16 inputs: the reference rounds every elementwise step to bf16 (relative 2^-8); fp32 within its own rounding
    return (3e-2, 3e-2) if f.meta["dtype"] == "bfloat16" else (1e-4, 1e-5)


def _replay_vq(f, s, C):
    kw = f.kw
    x, G = f[f"x_{s}"], f[f"G_{s}"]
    noise = f.noise(s)
    idx, out, loss, xg, eg = O.vq_rows(
        f.vq_rows(x), f.vq_rows(G), C, x_grad=f.meta["x_grad"], rotation=kw.get("rotation_trick", not kw.get("directional_reparam")),
        diveq_var=5e-3 if kw.get("directional_reparam") else None, noise=None if noise is None else f.vq_rows(noise),
        commit_weight=kw.get("commitment_weight", 1.0), sync_v=kw.get("sync_update_v", 0.0), lw=f.meta["lw"])
    return idx, f.vq_from_rows(out, x.shape), loss, (f.vq_from_rows(xg, x.shape) if f.meta["x_grad"] else None), {
        "_codebook.embed": eg[None]}, f.vq_index_rows(f[f"ind_{s}"])


def _replay_rvq(f, s, state, prefix, x, G, noise):
    kw = f.kw
    Q = kw["num_quantizers"]
    keys = [f"{prefix}layers.{0 if kw.get('shared_codebook') else q}._codebook.embed" for q in range(Q)]
    books = [state[k][0] for k in keys]
    D = x.shape[-1]
    idx, out, losses, xg, egs = O.rvq_rows(x.reshape(-1, D), G.reshape(-1, D), books, x_grad=f.meta["x_grad"],
                                           diveq_var=5e-3 if kw.get("diveq") else None,
                                           noise=None if noise is None else noise.reshape(-1, D), lw=f.meta["lw"],
                                           bf16=f.meta["dtype"] == "bfloat16",
                                           given_idx=f[f"ind_{s}"].reshape(-1, Q) if f.meta["dtype"] == "bfloat16" else None)
    grads = {}
    for k, g in zip(keys, egs):
        grads[k] = grads.get(k, 0) + g[None]
    return idx, out.reshape(x.shape), losses, xg.reshape(x.shape), grads


@pytest.mark.parametrize("name", names())
def test_learnable_oracle_matches_reference(name):
    f = Fixture(name)
    rtol, atol = _tol(f)
    kmeans = f.kw.get("kmeans_init", False)
    for s in range(f.meta["steps"]):
        if kmeans and s == 0:
            continue   # step 0 searches the k-means initialised codebook, which the fixture does not hold
        state = f.state(s)
        cls = f.meta["cls"]
        if cls == "VectorQuantize":
            idx, out, loss, xg, grads, ref_idx = _replay_vq(f, s, state["_codebook.embed"][0])
            assert np.array_equal(idx, ref_idx), s
        else:
            x, G, noise = f[f"x_{s}"], f[f"G_{s}"], f.noise(s)
            if cls == "ResidualVQ":
                idx, out, loss, xg, grads = _replay_rvq(f, s, state, "", x, G, noise)
            else:   # GroupedResidualVQ: each group a ResidualVQ on its slice of the features (rvq:690-721)
                g = f.kw["groups"]
                d = x.shape[-1] // g
                parts = [_replay_rvq(f, s, state, f"rvqs.{i}.", x[..., i * d:(i + 1) * d], G[..., i * d:(i + 1) * d], None)
                         for i in range(g)]
                idx = np.stack([p[0] for p in parts])
                out = np.concatenate([p[1] for p in parts], axis=-1)
                loss = np.stack([p[2] for p in parts])
                xg = np.concatenate([p[3] for p in parts], axis=-1)
                grads = {k: v for p in parts for k, v in p[4].items()}
            assert np.array_equal(idx.reshape(-1), f[f"ind_{s}"].reshape(-1)), s
        np.testing.assert_allclose(out, f[f"out_{s}"], rtol=rtol, atol=atol)
        np.testing.assert_allclose(loss, f[f"loss_{s}"], rtol=rtol, atol=1e-6)
        if f.meta["x_grad"]:
            np.testing.assert_allclose(xg, f[f"xgrad_{s}"], rtol=rtol, atol=atol)
        ref_grads = f.pgrads(s)
        post = f.post(s)
        for k, g in grads.items():
            np.testing.assert_allclose(g, ref_grads[k], rtol=rtol, atol=atol, err_msg=f"{k} step {s}")
            if not f.kw.get("threshold_ema_dead_code"):   # SGD step (expired codes are replaced after it)
                np.testing.assert_allclose(post[k], state[k] - f.meta["lr"] * ref_grads[k], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("name", names())
def test_learnable_state_dict_matches_reference(name):
    """The reference's state_dict keys in order and its initial tensors (embed is a Parameter), and it loads."""
    import vector_quantize_pytorch_b200 as m
    f = Fixture(name)
    ref = {k: torch.from_numpy(v) for k, v in f.state().items()}
    mod = f.build(m)
    ours = mod.state_dict()
    assert list(ours) == list(ref)
    for k in ref:
        assert torch.equal(ours[k], ref[k]), k
    assert [n for n, _ in mod.named_parameters()] == f.meta["param_names"]
    mod.load_state_dict(ref)


def test_learnable_construction_rules():
    import vector_quantize_pytorch_b200 as m
    vq = m.VectorQuantize(dim=16, codebook_size=8, learnable_codebook=True, ema_update=False)
    assert isinstance(vq._codebook.embed, torch.nn.Parameter) and vq._codebook.embed.shape == (1, 8, 16)
    dv = m.VectorQuantize(dim=16, codebook_size=8, directional_reparam=True, threshold_ema_dead_code=2)   # vqp:854-856, :880
    assert dv.learnable_codebook and not dv.ema_update and not dv.rotation_trick and not dv.has_commitment_loss
    rvq = m.ResidualVQ(dim=16, num_quantizers=2, codebook_size=8, diveq=True)                            # rvq:222-232, :268
    assert rvq.quant_grad_frac == 1. and all(vq.learnable_codebook and not vq.ema_update for vq in rvq.layers)
    assert all(not vq.route_gradients_to_input and not vq.has_commitment_loss for vq in rvq.layers)
    for kw in (dict(learnable_codebook=True),                                   # with EMA (vqp:908)
               dict(learnable_codebook=True, ema_update=False, use_cosine_sim=True),   # vqp:884
               dict(sync_update_v=0.5),                                        # vqp:913
               dict(learnable_codebook=True, ema_update=False, heads=2, separate_codebook_per_head=True),
               dict(learnable_codebook=True, ema_update=False, in_place_codebook_optimizer=torch.optim.SGD),
               dict(learnable_codebook=True, ema_update=False, orthogonal_reg_weight=1.)):
        with pytest.raises(NotImplementedError):
            m.VectorQuantize(dim=16, codebook_size=8, **kw)
    with pytest.raises(NotImplementedError):   # one learnable codebook per module: no separate codebooks per head
        m.Codebook(dim=16, codebook_size=8, num_codebooks=2, learnable_codebook=True, ema_update=False)
    cb = m.Codebook(dim=16, codebook_size=8, learnable_codebook=True, ema_update=False)
    assert isinstance(cb.embed, torch.nn.Parameter) and list(cb.state_dict()) == ["embed", "initted", "cluster_size", "embed_avg"]
    with pytest.raises(AssertionError):   # vqp:901
        m.VectorQuantize(dim=16, codebook_size=8, directional_reparam=True)
    for kw in (dict(quant_grad_frac=0.5), dict(implicit_neural_codebook=True)):
        with pytest.raises(NotImplementedError):
            m.ResidualVQ(dim=16, num_quantizers=2, codebook_size=8, learnable_codebook=True, ema_update=False, **kw)
