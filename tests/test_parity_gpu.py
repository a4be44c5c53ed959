"""GPU parity tests (run on an H100: `pytest -m gpu`).

The CUDA path (through the C ABI) is compared with
  * the committed golden fixtures generated from the real reference (tests/golden/*.npz),
  * the numpy oracle on seeded inputs at sizes it finishes in seconds,
  * size-independent invariants at BASELINE.json's full sizes.
Bars: indices bit-exact (except rows the reference itself resolves inside fp32 rounding noise, which are
counted and classified with a float64 top-2 gap); values within 1e-5 (fp32) / one bf16 ulp (bf16).
"""
import numpy as np
import os

import pytest
import torch

from golden_util import Golden, dropout_golden_names, golden_names, layout_golden_names, mask_golden_names, near_tie_rows, replayable_on_gpu
from oracle import vq_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def ours_codebooks(module):
    m = vqb()
    seen, out = set(), []
    for sub in module.modules():
        if isinstance(sub, m.Codebook) and id(sub) not in seen:
            seen.add(id(sub))
            out.append(sub)
    return out


def build_module(meta):
    m = vqb()
    kw = {}
    for k in ("use_cosine_sim", "decay", "eps", "commitment_weight", "heads", "codebook_dim", "separate_codebook_per_head"):
        if k in meta:
            kw[k] = meta[k]
    if meta["kind"] == "vq":
        return m.VectorQuantize(dim=meta["dim"], codebook_size=meta["codebook_size"], **kw)
    if meta["kind"] == "rvq":
        return m.ResidualVQ(dim=meta["dim"], num_quantizers=meta["num_quantizers"], codebook_size=meta["codebook_size"],
                            shared_codebook=meta["shared_codebook"], **kw)
    return m.GroupedResidualVQ(dim=meta["dim"], groups=meta["groups"], num_quantizers=meta["num_quantizers"],
                               codebook_size=meta["codebook_size"], shared_codebook=meta["shared_codebook"], **kw)


def codebook_slots(module):
    """(Codebook module, slot) for every (K, D) codebook: a Codebook with num_codebooks > 1 (separate_codebook_per_head) has several."""
    return [(cb, j) for cb in ours_codebooks(module) for j in range(cb.embed.shape[0])]


def load_state(module, g, tag):
    for i, (cb, j) in enumerate(codebook_slots(module)):
        st = g.state(tag, i)
        with torch.no_grad():
            cb.embed[j].copy_(torch.from_numpy(st.embed))
            cb.embed_avg[j].copy_(torch.from_numpy(st.embed_avg))
            cb.cluster_size[j].copy_(torch.from_numpy(st.cluster_size))


@pytest.mark.parametrize("name", replayable_on_gpu(golden_names()))
def test_modules_match_reference_goldens(name):
    g = Golden(name)
    m = g.meta
    module = build_module(m).to(DEV)
    load_state(module, g, "s0_pre")
    dt = m["dtype"]
    vtol = 1e-5 if dt == "fp32" else 8e-3
    for step, mode in enumerate(m["steps"]):
        module.train(mode == "train")
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(TDT[dt])
        q, ind, loss = module(x)
        torch.cuda.synchronize()
        assert q.dtype == x.dtype and q.shape == x.shape and ind.dtype == torch.int64 and loss.dtype == torch.float32
        ref_ind = g[f"s{step}_indices"]
        mism = ind.cpu().numpy() != ref_ind
        if "coldinit" in name:
            # degenerate kaiming codebook: the reference itself sits on fp32 ties (SURVEY 7.2); only near ties may differ
            pre = g.state("s0_pre", 0) if step == 0 else g.state(f"s{step - 1}_post", 0)
            tie = near_tie_rows(g[f"s{step}_x"].reshape(-1, m["dim"]), pre.embed, False, tol=2e-5).reshape(mism.shape)
            assert not (mism & ~tie).any()
            assert mism.mean() < 0.05
            load_state(module, g, f"s{step}_post")
            continue
        assert mism.sum() == 0, f"{name} step {step}: {mism.sum()} index mismatches"
        np.testing.assert_allclose(q.float().cpu().numpy(), g[f"s{step}_quantize"], rtol=vtol, atol=vtol)
        np.testing.assert_allclose(loss.detach().cpu().numpy(), g[f"s{step}_loss"], rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-7)
        for i, (cb, j) in enumerate(codebook_slots(module)):
            ref = g.state(f"s{step}_post", i)
            np.testing.assert_allclose(cb.cluster_size[j].cpu().numpy(), ref.cluster_size, rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(cb.embed_avg[j].cpu().numpy(), ref.embed_avg, rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(cb.embed[j].cpu().numpy(), ref.embed, rtol=1e-5, atol=1e-5)


SEARCH_CASES = [
    # N,    D,   K,    dtype,  cosine
    (3000, 256, 1024, "bf16", False),
    (3000, 256, 1024, "fp32", False),
    (1111, 128, 1000, "fp32", False),   # K not a tile multiple
    (2049, 64, 333, "bf16", False),
    (515, 32, 5, "fp32", False),        # tiger-sized codebook
    (4096, 8, 64, "fp32", False),       # minimum D
    (1500, 256, 2048, "bf16", True),
    (1500, 192, 700, "fp32", True),
    (1024, 512, 4096, "bf16", True),    # config-4 shape family
    (1, 64, 17, "fp32", False),         # single row
    (1024, 512, 4096, "fp32", True),    # config 4 in fp32: A planes streamed through the ring (n_a * ceil(D/64) > 8)
    (700, 384, 600, "fp32", False),     # streamed A, ragged K
    (515, 1024, 300, "bf16", False),    # maximum D (16 k-blocks, streamed)
    (333, 520, 96, "fp32", False),      # streamed A with a ragged last k-block (D % 64 != 0)
]


@pytest.mark.parametrize("N,D,K,dt,cosine", SEARCH_CASES)
def test_search_gather_stats_match_oracle(N, D, K, dt, cosine):
    from vector_quantize_pytorch_b200 import ops
    gen = torch.Generator().manual_seed(N * 7 + D * 3 + K)
    x = torch.randn(N, D, generator=gen).to(TDT[dt])
    c = torch.randn(K, D, generator=gen)
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    xd, cd = x.to(DEV), c.to(DEV).contiguous()
    cb = ops.prepare_codebook(cd, cosine)
    res = ops.search(xd, cb, cd, debug_best=True)
    torch.cuda.synchronize()
    x_np = O.cast_like(x.float().numpy(), dt)
    if cosine:
        x_np = O.l2norm(x_np, dt)
    np.testing.assert_allclose(res.x_eff.float().cpu().numpy(), x_np, rtol=0, atol=1e-6 if dt == "fp32" else 0)
    ref_idx = O.argmax_first(O.scores(x_np, c.numpy(), cosine))
    mism = res.idx.cpu().numpy() != ref_idx
    tie = near_tie_rows(x_np, c.numpy(), cosine)
    assert not (mism & ~tie).any(), f"{(mism & ~tie).sum()} non-tie mismatches"
    assert mism.sum() <= max(2, N // 500)
    # tensor-core score error stays inside the certified margin
    s64 = x_np.astype(np.float64) @ c.numpy().astype(np.float64).T
    if not cosine:
        s64 -= 0.5 * (c.numpy().astype(np.float64) ** 2).sum(-1)[None]
    # gather / loss
    q = torch.empty_like(xd)
    i64 = torch.empty(N, dtype=torch.int64, device=DEV)
    ls = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.gather(res.x_eff, cd, res.idx, q_out=q, idx64_out=i64, loss_sum=ls)
    idx_np = res.idx.cpu().numpy().astype(np.int64)
    q_ref = O.cast_like(c.numpy()[idx_np], dt)
    assert np.array_equal(q.float().cpu().numpy(), q_ref)
    assert np.array_equal(i64.cpu().numpy(), idx_np)
    _, l32 = O.mse_loss(q_ref, x_np, dt)
    assert abs(ls.item() / (N * D) - float(l32)) <= 1e-5 * max(float(l32), 1e-12)
    # statistics
    st = ops.ema_stats(res.x_eff, res.idx, K)
    off = ops.stats_offset(K)
    cs_ref, es_ref = O.batch_stats(x_np, idx_np, K)
    assert np.array_equal(st[:K].cpu().numpy(), cs_ref)
    np.testing.assert_allclose(st[off:].view(K, D).cpu().numpy(), es_ref, rtol=1e-5, atol=1e-5)


SCORE_CASES = [
    # dtype, D, K, distribution
    ("bf16", 256, 1024, "randn"), ("fp32", 256, 1024, "randn"), ("bf16", 512, 512, "randn"), ("fp32", 64, 4096, "randn"),
    ("bf16", 256, 1024, "heavy"),     # heavy-tailed rows: one coordinate 1e3 x the rest
    ("fp32", 256, 1024, "heavy"),
    ("bf16", 200, 777, "randn"),      # D not a multiple of 64 (zero-filled last k-block), ragged K
    ("fp32", 520, 300, "randn"),      # streamed A planes, ragged last k-block
    ("bf16", 512, 16384, "unit"),     # config-4 shape family: unit-norm rows and codes
    ("fp32", 512, 16384, "unit"),
    ("bf16", 256, 1024, "tiny"),      # |x| ~ 1e-6: below the fp16 normal range (the 2^-25 per-element term of the band)
    ("bf16", 256, 1024, "cold"),      # default-init codebook: |c| ~ 5e-3
]


@pytest.mark.parametrize("dt,D,K,dist", SCORE_CASES)
def test_score_error_inside_margin(dt, D, K, dist):
    """The band that certifies a row must bound the real tensor-core error of the bf16 hi / lo passes with room to spare:
    |score_mma - score_exact| <= ||x|| * cres + ||x_lo|| * caux + margin * ||x|| * max||c|| + 2^-21 max||c||^2, by
    Cauchy-Schwarz on the exact residual norms the operand-preparation kernel reports (ops.CodebookOperands.cmax)."""
    from vector_quantize_pytorch_b200 import ops
    torch.manual_seed(5)
    N = 8192 if K <= 4096 else 2048
    x = torch.randn(N, D)
    c = torch.randn(K, D) * 2
    if dist == "heavy":
        x[:, 3] *= 1e3
        c[:, 3] *= 30
    elif dist == "unit":
        x, c = torch.nn.functional.normalize(x, dim=-1), torch.nn.functional.normalize(c, dim=-1)
    elif dist == "tiny":
        x = x * 1e-6
    elif dist == "cold":
        c = (torch.rand(K, D) * 2 - 1) * (6.0 / (K * D)) ** 0.5
    x = (x * (1 if dist != "randn" else 3)).to(TDT[dt]).to(DEV)
    c = c.to(DEV).contiguous()
    cb = ops.prepare_codebook(c, False)
    n_a = 1 if dt == "bf16" else 2
    res = ops.search(x, cb, c, debug_best=True, fix=False, n_passes=n_a + 1)
    torch.cuda.synchronize()
    s = x.double() @ c.double().T - 0.5 * (c.double() ** 2).sum(-1)[None]
    got = s.gather(1, res.idx.long()[:, None])[:, 0]
    err = (res.best.double() - got).abs()
    xd = x.double()
    xn = xd.norm(dim=-1)
    cmax = c.double().norm(dim=-1).max()
    cm = cb.cmax.cpu().double()   # max||c||, max||c - hi - lo||, max||lo||
    # the residual norms are what the kernel believes: they must be true upper bounds of what the operand planes leave out
    hi = cb.planes[0, :K].view(torch.bfloat16).float().double()
    lo = cb.planes[1, :K].view(torch.bfloat16).float().double()
    assert (c.double() - hi - lo).norm(dim=-1).max().item() <= cm[1].item()
    assert lo.norm(dim=-1).max().item() <= cm[2].item()
    # the kernel's per-score allowance (half of its band without the tag / sqrt terms), vq_assign.cu
    allow = ops.DEFAULT_MARGIN * xn * cmax + 2.0 ** -21 * cmax * cmax
    allow = allow + xn * cm[1]
    if dt == "fp32":
        xhi = x.bfloat16().float()
        xlo = (x - xhi).bfloat16().double().norm(dim=-1)
        allow = allow + xlo * (2.0 ** -8 * 1.01 * cmax + cm[2])
    worst = (err / allow.clamp_min(1e-300)).max().item()
    print(f"{dt} D={D} K={K} {dist}: worst error / allowance = {worst:.3f}")
    assert worst < 1.0, (dt, D, K, dist, worst)


def test_flagged_rows_are_rescored_exactly():
    """Force near ties: duplicate codes (exact ties -> lowest index must win, vqp:140) and near-duplicates."""
    from vector_quantize_pytorch_b200 import ops
    torch.manual_seed(11)
    K, D, N = 512, 128, 4096
    c = torch.randn(K, D)
    c[300] = c[7]                        # exact duplicate: index 7 must always beat 300
    c[301] = c[7]                        # ... a third copy: three candidates -> exact re-score of the triple
    c[302] = c[7]
    c[303] = c[7]                        # ... five copies: > 3 candidates -> whole-row rescan path
    c[500] = c[13]
    c[501] = c[13]                       # a clean triple (13, 500, 501)
    c[400] = c[9] * (1 + 3e-7)           # inside fp32 noise of code 9
    c[401] = c[11] + 1e-4 * torch.randn(D)  # resolvable only by the exact re-score
    x = torch.randn(N, D)
    x[:64] = c[7] + 0.01 * torch.randn(64, D)
    x[64:128] = c[11] + 0.01 * torch.randn(64, D)
    x[128:192] = c[13] + 0.01 * torch.randn(64, D)
    for dt in ("fp32", "bf16"):
        xd = x.to(TDT[dt]).to(DEV)
        cd = c.to(DEV)
        cb = ops.prepare_codebook(cd, False)
        res = ops.search(xd, cb, cd)
        idx = res.idx.cpu().numpy()
        n_front, n_back = res.flag_count.item(), res.rescan_count.item()
        assert n_front >= 128 and n_back >= 64
        front = res.flagged[:n_front].cpu().numpy()  # (row, count, cand0, cand1, cand2, ...)
        back = res.flagged[N - n_back:].cpu().numpy()
        assert ((front[:, 1] == 2) | (front[:, 1] == 3)).all() and (front[:, 1] == 3).sum() >= 64, "triples are re-scored directly"
        assert (back[:, 1] > 3).all(), "the five-fold tie must take the whole-row rescan path"
        assert (idx[:64] == 7).all() and (idx[128:192] == 13).all()
        x_np = O.cast_like(x.numpy(), dt)
        ref = O.argmax_first(O.scores(x_np, c.numpy(), False))
        tie = near_tie_rows(x_np, c.numpy(), False)
        assert not ((idx != ref) & ~tie).any()


def test_codebook_forward_contract_and_update_indices():
    """Reference tests/test_beam.py:8-45: stats from (x, indices) alone reproduce a normal EMA step."""
    m = vqb()
    torch.manual_seed(3)
    vq1 = m.VectorQuantize(dim=64, codebook_size=128).to(DEV)
    vq2 = m.VectorQuantize(dim=64, codebook_size=128).to(DEV)
    with torch.no_grad():
        e = torch.randn(1, 128, 64, device=DEV)
        vq1._codebook.embed.copy_(e); vq1._codebook.embed_avg.copy_(e)
    vq2.load_state_dict(vq1.state_dict())
    x = torch.randn(2, 300, 64, device=DEV)
    q1, i1, _ = vq1(x)
    vq2.eval()
    q2, i2, l2 = vq2(x)
    assert torch.equal(i1, i2) and torch.equal(q1, q2) and l2.item() == 0.0
    vq2.train()
    vq2.update_indices(x, i2)
    for name in ("cluster_size", "embed_avg", "embed"):
        a, b = getattr(vq1._codebook, name), getattr(vq2._codebook, name)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), name
    # Codebook.forward contract: (quantize fp32, int64 indices, dist None)
    cbk = vq1._codebook
    cbk.eval()
    q, ind, dist = cbk(x)
    assert q.dtype == torch.float32 and ind.dtype == torch.int64 and dist is None
    assert torch.equal(q, cbk.embed[0][ind])
    # eval: quantized == get_output_from_indices(indices)   (reference tests/test_readme.py:33-47)
    assert torch.allclose(vq1.get_output_from_indices(ind), q)


@pytest.mark.parametrize("dt,cosine", [("bf16", False), ("fp32", False), ("bf16", True)])
def test_forward_host_matches_forward(dt, cosine):
    """The chunk-pipelined host API must be the same function as forward() (one EMA update from summed statistics)."""
    m = vqb()
    torch.manual_seed(9)
    a = m.VectorQuantize(dim=64, codebook_size=200, use_cosine_sim=cosine).to(DEV)
    b = m.VectorQuantize(dim=64, codebook_size=200, use_cosine_sim=cosine).to(DEV)
    _warm_codebook(a, 64, 200, cosine)
    b.load_state_dict(a.state_dict())
    x = torch.randn(7, 1000, 64).to(TDT[dt])
    qa, ia, la = a(x.to(DEV))
    qh, ih, lh = b.forward_host(x.pin_memory(), n_chunks=5)
    torch.cuda.synchronize()
    assert not qh.is_cuda and qh.shape == x.shape and ih.shape == x.shape[:-1]
    assert torch.equal(ia.cpu(), ih) and torch.equal(qa.cpu(), qh)
    assert abs(la.item() - lh.item()) <= (1e-5 if dt == "fp32" else 8e-3) * la.item()
    for name in ("cluster_size", "embed_avg", "embed"):
        assert torch.allclose(getattr(a._codebook, name), getattr(b._codebook, name), rtol=1e-5, atol=1e-5), name
    # second call reuses the pipeline buffers
    qh2, ih2, _ = b.forward_host(x.pin_memory(), n_chunks=5)
    qa2, ia2, _ = a(x.to(DEV))
    assert torch.equal(ia2.cpu(), ih2)


def test_lens_mask_matches_unmasked_prefix():
    """Reference tests/test_readme.py:49-72: a `lens`-masked call equals the call on the unpadded prefix; padding
    comes back as zeros / index -1; masked rows take no part in the EMA update."""
    m = vqb()
    torch.manual_seed(2)
    a = m.VectorQuantize(dim=64, codebook_size=100).to(DEV)
    b = m.VectorQuantize(dim=64, codebook_size=100).to(DEV)
    _warm_codebook(a, 64, 100)
    b.load_state_dict(a.state_dict())
    x = torch.randn(1, 300, 64, device=DEV)
    lens = torch.tensor([211], device=DEV)
    qm, im, lm = a(x, lens=lens)
    qp, ip, lp = b(x[:, :211])
    assert torch.equal(im[:, :211], ip) and (im[:, 211:] == -1).all()
    assert torch.equal(qm[:, :211], qp) and (qm[:, 211:] == 0).all()
    assert abs(lm.item() - lp.item()) <= 1e-6 * lp.item()
    for name in ("cluster_size", "embed_avg", "embed"):
        assert torch.allclose(getattr(a._codebook, name), getattr(b._codebook, name), rtol=1e-6, atol=1e-6), name
    # boolean mask, eval mode, padding returned as the input
    c = m.VectorQuantize(dim=64, codebook_size=100, return_zeros_for_masked_padding=False).to(DEV).eval()
    mask = torch.rand(2, 50, device=DEV) > 0.3
    y = torch.randn(2, 50, 64, device=DEV)
    qc, ic, lc = c(y, mask=mask)
    assert torch.equal(qc[~mask], y[~mask]) and (ic[~mask] == -1).all() and (ic[mask] >= 0).all() and lc.item() == 0.0


def test_rvq_decode_invariant():
    """Reference tests/test_readme.py:74-103: sum of gathered codes == quantized_out (frozen codebook)."""
    m = vqb()
    torch.manual_seed(0)
    for shared in (False, True):
        for cosine in (False, True):
            rvq = m.ResidualVQ(dim=32, num_quantizers=8, codebook_size=128, shared_codebook=shared, use_cosine_sim=cosine).to(DEV)
            x = torch.randn(1, 256, 32, device=DEV)
            rvq.train()
            q, ind, loss = rvq(x, freeze_codebook=True)
            out = rvq.get_output_from_indices(ind)
            assert ind.shape == (1, 256, 8) and loss.shape == (8,)
            # fp32: the rounded running sum and the decode are the same fp32 adds in the same order
            assert torch.equal(q, out)


def test_gradients_route_through_glue():
    m = vqb()
    torch.manual_seed(0)
    for rot in (True, False):
        vq = m.VectorQuantize(dim=64, codebook_size=64, rotation_trick=rot).to(DEV)
        x = torch.randn(2, 50, 64, device=DEV, requires_grad=True)
        q, ind, loss = vq(x)
        (q.sum() + loss).backward()
        assert x.grad is not None and torch.isfinite(x.grad).all()


def test_graph_replay_and_patch_match_direct_enqueue():
    """vqb_vq_forward replays / patches CUDA graphs when a call structure repeats (vq_forward.cu).  Twin modules see the
    same batches: one through the graph cache (outputs kept alive in different patterns, so pointer sets repeat, alternate
    and appear new), one with profiling events requested, which forces the launch-by-launch path.  Everything — outputs
    and the EMA-updated codebook — must stay identical step after step (a stale pointer in a patched graph would not).
    Run on torch's default stream (the legacy stream, on which CUDA refuses stream capture: the cache must fall back
    cleanly) and on a side stream (where capture is legal)."""
    import ctypes
    m = vqb()
    from vector_quantize_pytorch_b200 import _C, ops

    def graph_stats():
        out = (ctypes.c_longlong * 4)()
        assert _C.lib.vqb_debug_graph_stats(ctypes.cast(out, ctypes.c_void_p)) == 0
        return list(out)

    def twin_run(dim, K):
        torch.manual_seed(7)
        a = m.VectorQuantize(dim=dim, codebook_size=K).to(DEV)
        b = m.VectorQuantize(dim=dim, codebook_size=K).to(DEV)
        _warm_codebook(a, dim, K)
        b.load_state_dict(a.state_dict())
        keep = []
        for step in range(10):
            x = torch.randn(4, 1024, dim, device=DEV).bfloat16()
            qa, ia, la = a(x)
            ops.PROFILE_EVENTS = []
            try:
                qb, ib, lb = b(x)
            finally:
                ops.PROFILE_EVENTS = None
            torch.cuda.current_stream().synchronize()
            assert torch.equal(ia, ib), f"indices differ at step {step}"
            assert torch.equal(qa, qb), f"quantized differs at step {step}"
            assert torch.allclose(la, lb, rtol=1e-6, atol=0), f"loss differs at step {step}"
            # float atomics in the statistics make them order-dependent in the last bits
            torch.testing.assert_close(a._codebook.embed, b._codebook.embed, rtol=1e-5, atol=1e-6)
            b.load_state_dict(a.state_dict())   # keep the twins in lock step
            if step % 3 == 0:
                keep.append((qa, ia))            # hold some outputs: the allocator hands out new blocks
            elif step % 3 == 2:
                keep.clear()

    s0 = graph_stats()
    twin_run(64, 256)
    s1 = graph_stats()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        twin_run(96, 320)
    side.synchronize()
    s2 = graph_stats()
    names = ("replayed", "patched", "instantiated", "fell_back")
    print("graph cache, default stream:", dict(zip(names, (y - x for x, y in zip(s0, s1)))),
          "| side stream:", dict(zip(names, (y - x for x, y in zip(s1, s2)))))


# ------------------------------------------------------------------------------------------------
# BASELINE.json full sizes: size-independent properties
# ------------------------------------------------------------------------------------------------

def _warm_codebook(vq, D, K, cosine=False):
    with torch.no_grad():
        e = torch.randn(1, K, D, device=DEV)
        if cosine:
            e = torch.nn.functional.normalize(e, dim=-1)
        vq._codebook.embed.copy_(e)
        vq._codebook.embed_avg.copy_(e)


def test_config2_full_size_properties():
    """VectorQuantize dim=256 K=1024, x=(64,4096,256) bf16, EMA on."""
    m = vqb()
    torch.manual_seed(1234)
    vq = m.VectorQuantize(dim=256, codebook_size=1024).to(DEV)
    _warm_codebook(vq, 256, 1024)
    pre = vq._codebook.embed[0].clone()
    x = torch.randn(64, 4096, 256, device=DEV).bfloat16()
    q, ind, loss = vq(x)
    torch.cuda.synchronize()
    N = 64 * 4096
    # (1) quantize is exactly the gathered PRE-update code cast to bf16 (vqp:766, :1178)
    assert torch.equal(q, pre[ind].bfloat16())
    # (2) a sample of rows agrees with the numpy oracle
    sel = torch.randperm(N, device=DEV)[:4096]
    xs = x.reshape(-1, 256)[sel].float().cpu().numpy()
    ref = O.argmax_first(O.scores(xs, pre.cpu().numpy(), False))
    got = ind.reshape(-1)[sel].cpu().numpy()
    tie = near_tie_rows(xs, pre.cpu().numpy(), False)
    assert not ((got != ref) & ~tie).any()
    # (3) loss == mean((q - x)^2) in bf16 semantics
    l_ref = ((q.float() - x.float()) ** 2).bfloat16().float().mean()
    assert abs(loss.item() - l_ref.bfloat16().float().item()) <= 8e-3 * l_ref.item()
    # (4) EMA bookkeeping: cluster_size sums to decay*K + (1-decay)*N ; embed_avg row sums follow the same lerp
    cs = vq._codebook.cluster_size[0]
    assert abs(cs.sum().item() - (0.8 * 1024 + 0.2 * N)) < 1e-2 * N * 0.2 * 1e-2 + 1.0
    flat = x.reshape(-1, 256).float()
    es = torch.zeros(1024, 256, device=DEV, dtype=torch.float64).index_add_(0, ind.reshape(-1), flat.double())
    ea_ref = pre.double() * 0.8 + 0.2 * es
    assert torch.allclose(vq._codebook.embed_avg[0].double(), ea_ref, rtol=1e-5, atol=1e-4)
    # (5) idempotence in eval: the codes themselves quantize to themselves
    vq.eval()
    codes = vq._codebook.embed[0].clone()
    q2, ind2, l2 = vq(codes[None])
    assert torch.equal(ind2[0], torch.arange(1024, device=DEV)) and torch.equal(q2[0], codes)


def test_config3_full_size_properties():
    """ResidualVQ Q=8 shared codebook K=1024, x=(32,8192,256)."""
    m = vqb()
    torch.manual_seed(1234)
    rvq = m.ResidualVQ(dim=256, num_quantizers=8, codebook_size=1024, shared_codebook=True).to(DEV)
    _warm_codebook(rvq.layers[0], 256, 1024)
    pre = rvq.layers[0]._codebook.embed[0].clone()
    x = torch.randn(32, 8192, 256, device=DEV)
    q, ind, losses = rvq(x)
    torch.cuda.synchronize()
    assert ind.shape == (32, 8192, 8) and losses.shape == (8,)
    # decode invariant with the PRE-update codebook: every stage searched and gathered it (rvq:302-306, SURVEY 3.2)
    acc = torch.zeros_like(x)
    for s in range(8):
        acc = acc + pre[ind[..., s]]
    assert torch.equal(q, acc)   # the running sum of rvq:525, rounded where the reference rounds
    # commitment losses equal mse(residual_s, code_s) along the residual recurrence
    l = losses.cpu().numpy()
    resid = x.clone()
    for s in range(8):
        code = pre[ind[..., s]]
        ref = ((code - resid) ** 2).mean().item()
        assert abs(l[s] - ref) <= 1e-4 * ref
        resid = resid - code
    # stage-0 indices of a row sample agree with the oracle
    sel = torch.randperm(32 * 8192, device=DEV)[:2048]
    xs = x.reshape(-1, 256)[sel].cpu().numpy()
    ref0 = O.argmax_first(O.scores(xs, pre.cpu().numpy(), False))
    tie = near_tie_rows(xs, pre.cpu().numpy(), False)
    got0 = ind.reshape(-1, 8)[sel, 0].cpu().numpy()
    assert not ((got0 != ref0) & ~tie).any()


@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_config4_full_size_properties(dt):
    """cosine dim=512 K=16384, x=(16,4096,512), bf16 and fp32 (fp32 at D=512: the A planes are streamed, vq_assign.cu)."""
    m = vqb()
    torch.manual_seed(1234)
    vq = m.VectorQuantize(dim=512, codebook_size=16384, use_cosine_sim=True).to(DEV)
    _warm_codebook(vq, 512, 16384, cosine=True)
    pre = vq._codebook.embed[0].clone()
    x = torch.randn(16, 4096, 512, device=DEV).to(TDT[dt])
    q, ind, loss = vq(x)
    torch.cuda.synchronize()
    assert torch.equal(q, pre[ind].to(TDT[dt]))
    sel = torch.randperm(16 * 4096, device=DEV)[:1024]
    xs = O.l2norm(x.reshape(-1, 512)[sel].float().cpu().numpy(), dt)
    ref = O.argmax_first(O.scores(xs, pre.cpu().numpy(), True))
    tie = near_tie_rows(xs, pre.cpu().numpy(), True)
    got = ind.reshape(-1)[sel].cpu().numpy()
    assert not ((got != ref) & ~tie).any()
    # codebook rows stay unit-norm after the EMA step (vqp:581-582)
    n = vq._codebook.embed[0].norm(dim=-1)
    assert torch.allclose(n, torch.ones_like(n), atol=1e-5)


def test_config5_grouped_single_gpu_shard():
    """GroupedResidualVQ groups=2 Q=8 K=1024 on one 1/8 shard x=(8,4096,256)."""
    m = vqb()
    torch.manual_seed(1234)
    g = m.GroupedResidualVQ(dim=256, groups=2, num_quantizers=8, codebook_size=1024).to(DEV)
    for rvq in g.rvqs:
        for layer in rvq.layers:
            _warm_codebook(layer, 128, 1024)
    x = torch.randn(8, 4096, 256, device=DEV)
    g.train()
    q, ind, losses = g(x, freeze_codebook=True)
    assert q.shape == x.shape and ind.shape == (2, 8, 4096, 8) and losses.shape == (2, 8)
    assert torch.equal(q, g.get_output_from_indices(ind))   # fp32: the running sum is the decode's sequential sum


# ------------------------------------------------------------------------------------------------ mask / lens (vqp:1116-1119)
@pytest.mark.parametrize("name", mask_golden_names())
def test_masked_calls_match_reference(name):
    """`mask` / `lens` calls against the reference's own outputs (oracle/gen_golden.py --mask / --mask-rvq): indices (-1 on the
    padding), quantized (zeros / the input on the padding), the loss over the unmasked elements (vqp:1317-1325) and the codebooks
    after the masked EMA update (vqp:599-600) — VectorQuantize, ResidualVQ (rvq:495) and GroupedResidualVQ (rvq:698)."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    if meta["kind"] == "vq":
        kw = {k: meta[k] for k in ("use_cosine_sim", "commitment_weight", "return_zeros_for_masked_padding") if k in meta}
        mod = m.VectorQuantize(dim=meta["dim"], codebook_size=meta["codebook_size"], **kw).to(DEV)
    else:
        mod = build_module(meta).to(DEV)
    load_state(mod, g, "s0_pre")
    dt = meta["dtype"]
    vtol = 1e-5 if dt == "fp32" else 8e-3
    for step, mode in enumerate(meta["steps"]):
        mod.train(mode == "train")
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(TDT[dt])
        mask = g[f"s{step}_mask"]
        if meta["how"] == "lens":
            q, ind, loss = mod(x, lens=torch.from_numpy(g[f"s{step}_lens"]).to(DEV))
        else:
            q, ind, loss = mod(x, mask=torch.from_numpy(mask).to(DEV))
        torch.cuda.synchronize()
        assert q.dtype == x.dtype and q.shape == x.shape and ind.dtype == torch.int64 and loss.dtype == torch.float32
        assert tuple(ind.shape) == g[f"s{step}_indices"].shape and tuple(loss.shape) == g[f"s{step}_loss"].shape
        assert np.array_equal(ind.cpu().numpy(), g[f"s{step}_indices"]), f"{name} step {step}"
        np.testing.assert_allclose(q.float().cpu().numpy(), g[f"s{step}_quantize"], rtol=vtol, atol=vtol)
        np.testing.assert_allclose(loss.detach().cpu().numpy(), g[f"s{step}_loss"], rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-7)
        for i, (cb, j) in enumerate(codebook_slots(mod)):
            ref = g.state(f"s{step}_post", i)
            np.testing.assert_allclose(cb.cluster_size[j].cpu().numpy(), ref.cluster_size, rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(cb.embed_avg[j].cpu().numpy(), ref.embed_avg, rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(cb.embed[j].cpu().numpy(), ref.embed, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ input layouts (vqp:1121-1147)
@pytest.mark.parametrize("name", layout_golden_names())
def test_input_layouts_match_reference(name):
    """accept_image_fmap / accept_3d_fmap / channel_last=False / one token per batch element against the reference's own
    outputs (oracle/gen_golden.py --layout): shapes and values of quantize and indices, the loss, the codebook afterwards."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    kw = {k: meta[k] for k in ("use_cosine_sim", "heads", "codebook_dim") if k in meta}
    kw.update({"image": dict(accept_image_fmap=True), "3d": dict(accept_3d_fmap=True), "channel_first": dict(channel_last=False),
               "single": {}}[meta["layout"]])
    mod = m.VectorQuantize(dim=meta["dim"], codebook_size=meta["codebook_size"], **kw).to(DEV)
    load_state(mod, g, "s0_pre")
    cb = mod._codebook
    dt = meta["dtype"]
    vtol = 1e-5 if dt == "fp32" else 8e-3
    for step, mode in enumerate(meta["steps"]):
        mod.train(mode == "train")
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(TDT[dt])
        q, ind, loss = mod(x)
        torch.cuda.synchronize()
        assert q.dtype == x.dtype and q.shape == x.shape and ind.dtype == torch.int64
        assert tuple(ind.shape) == g[f"s{step}_indices"].shape
        assert np.array_equal(ind.cpu().numpy(), g[f"s{step}_indices"]), f"{name} step {step}"
        np.testing.assert_allclose(q.float().cpu().numpy(), g[f"s{step}_quantize"], rtol=vtol, atol=vtol)
        np.testing.assert_allclose(loss.detach().cpu().numpy(), g[f"s{step}_loss"], rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-7)
        ref = g.state(f"s{step}_post", 0)
        np.testing.assert_allclose(cb.cluster_size[0].cpu().numpy(), ref.cluster_size, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(cb.embed[0].cpu().numpy(), ref.embed, rtol=1e-5, atol=1e-5)
        if mode == "eval" and meta.get("heads", 1) == 1:  # decode restores the layout too (vqp:1015-1016)
            codes = mod.get_codes_from_indices(ind)
            assert codes.shape == q.shape
            np.testing.assert_allclose(codes.float().cpu().numpy(), g[f"s{step}_quantize"], rtol=vtol, atol=vtol)


# ------------------------------------------------------------------------------------------------ quantize dropout (rvq:423-439, :473-476)
@pytest.mark.parametrize("name", dropout_golden_names())
def test_quantize_dropout_matches_reference(name):
    """ResidualVQ(quantize_dropout=True) with the reference's explicit per-step seeds (oracle/gen_golden.py --dropout): the
    same layers are skipped (index -1, loss 0, codebook untouched), everything else as usual; coarse indices decode
    (rvq:333-339)."""
    m = vqb()
    g = Golden(name)
    meta = g.meta
    kw = {k: meta[k] for k in ("quantize_dropout", "quantize_dropout_cutoff_index", "quantize_dropout_multiple_of") if k in meta}
    mod = m.ResidualVQ(dim=meta["dim"], num_quantizers=meta["num_quantizers"], codebook_size=meta["codebook_size"],
                       shared_codebook=meta["shared_codebook"], **kw).to(DEV)
    load_state(mod, g, "s0_pre")
    dt = meta["dtype"]
    vtol = 1e-5 if dt == "fp32" else 8e-3
    for step, mode in enumerate(meta["steps"]):
        mod.train(mode == "train")
        x = torch.from_numpy(g[f"s{step}_x"]).to(DEV).to(TDT[dt])
        q, ind, loss = mod(x, rand_quantize_dropout_fixed_seed=meta["seeds"][step])
        torch.cuda.synchronize()
        assert np.array_equal(ind.cpu().numpy(), g[f"s{step}_indices"]), f"{name} step {step}"
        np.testing.assert_allclose(q.float().cpu().numpy(), g[f"s{step}_quantize"], rtol=vtol, atol=vtol)
        np.testing.assert_allclose(loss.detach().cpu().numpy(), g[f"s{step}_loss"], rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-7)
        for i, (cb, j) in enumerate(codebook_slots(mod)):
            ref = g.state(f"s{step}_post", i)
            np.testing.assert_allclose(cb.cluster_size[j].cpu().numpy(), ref.cluster_size, rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(cb.embed[j].cpu().numpy(), ref.embed, rtol=1e-5, atol=1e-5)
    # coarse indices (the first two layers only) decode to the sum of those layers' codes
    mod.eval()
    coarse = mod.get_output_from_indices(ind[..., :2])
    full = ind.clone()
    full[..., 2:] = -1
    assert torch.equal(coarse, mod.get_output_from_indices(full))


def test_grouped_quantize_dropout_shares_the_index():
    """GroupedResidualVQ draws ONE dropout seed per forward and hands it to every group (rvq:701): the same layers are skipped in
    all groups; the output is the sum of the active layers' codes."""
    m = vqb()
    torch.manual_seed(7)
    g = m.GroupedResidualVQ(dim=64, groups=2, num_quantizers=4, codebook_size=32, quantize_dropout=True).to(DEV)
    for rvq in g.rvqs:
        for layer in rvq.layers:
            _warm_codebook(layer, 32, 32)
    g.train()
    seen = set()
    for _ in range(6):
        x = torch.randn(2, 50, 64, device=DEV)
        q, ind, losses = g(x, freeze_codebook=True)
        assert ind.shape == (2, 2, 50, 4) and losses.shape == (2, 4)
        active = (ind >= 0).all(dim=1).all(dim=1)          # (G, Q): a layer is active for all rows or for none
        dropped = (ind == -1).all(dim=1).all(dim=1)
        assert (active | dropped).all() and torch.equal(active[0], active[1])
        n = int(active[0].sum())
        assert active[0, :n].all() and (losses[:, n:] == 0).all()
        seen.add(n)
        assert torch.allclose(q, g.get_output_from_indices(ind), atol=1e-5)
    g.eval()
    _, ind, _ = g(torch.randn(2, 50, 64, device=DEV))
    assert (ind >= 0).all()                                  # no dropout in eval mode


@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_in_kernel_mask_equals_compacted_rows(dt):
    """The row mask inside the search kernel (vqb_vq_forward_args.row_mask) at a many-tile size: a masked training step equals
    the same step on the compacted unmasked rows — indices, quantized rows, loss, codebook afterwards — and the padding comes
    back as zeros / -1.  (Tiles mix live and padding rows; flagged rows, the in-kernel histogram and the sort all see the mask.)
    Bit-equality between the two modules is asserted while their codebooks are bit-identical, i.e. in the first step: the
    segmented sums run in a different order on the compacted batch, so the EMA-updated codebooks may differ in the last
    bits afterwards (observed for fp32 rows; sums of bf16 rows are mostly exact in fp32 and stayed identical)."""
    m = vqb()
    torch.manual_seed(99)
    B, N, D, K = 4, 3000, 256, 1024
    a = m.VectorQuantize(dim=D, codebook_size=K).to(DEV)
    _warm_codebook(a, D, K)
    b = m.VectorQuantize(dim=D, codebook_size=K).to(DEV)
    b.load_state_dict(a.state_dict())
    x = torch.randn(B, N, D, device=DEV).to(TDT[dt])
    mask = torch.rand(B, N, device=DEV) < 0.7
    mask[0, :200] = False            # whole tiles of padding
    mask[1] = True                   # and a fully live sequence
    for step, mode in enumerate(["train", "train", "eval"]):
        a.train(mode == "train"); b.train(mode == "train")
        exact = step == 0      # (bf16 rows usually stay bit-identical later on too — their sums are mostly exact in fp32 — but not provably)
        ea, eb = a.codebook.clone(), b.codebook.clone()    # the codebooks this step searches (pre-update, vqp:766)
        qa, ia, la = a(x, mask=mask)
        qb, ib, lb = b(x[mask][None])
        torch.cuda.synchronize()
        assert (ia[~mask] == -1).all() and (qa[~mask] == 0).all()
        same = ia[mask] == ib[0]
        assert same.all() if exact else (~same).sum() <= 2     # last-bit codebook differences may flip an fp32 near tie
        # every live row is exactly its winning code of the module's OWN codebook
        assert torch.equal(qa[mask], ea[ia[mask]].to(qa.dtype)) and torch.equal(qb[0], eb[ib[0]].to(qb.dtype))
        if exact:
            assert torch.equal(qa[mask], qb[0])
        vt = 1e-5 if dt == "fp32" else 8e-3
        torch.testing.assert_close(qa[mask][same].float(), qb[0][same].float(), rtol=vt, atol=vt)
        if mode == "eval":
            assert la.item() == 0.0
        elif same.all():
            torch.testing.assert_close(la, lb, rtol=1e-5 if dt == "fp32" else 8e-3, atol=1e-7)
            for u, v in zip(a.buffers(), b.buffers()):
                torch.testing.assert_close(u, v, rtol=1e-5, atol=1e-5)
        else:
            break    # a flipped near tie moved a row between two codes: the two trajectories legitimately part here
        x = torch.randn(B, N, D, device=DEV).to(TDT[dt])
