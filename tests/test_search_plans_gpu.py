"""Every launch plan of the search kernel over several waves of row tiles, against float64 (run on an H100: `pytest -m gpu`).

The host sizes the kernel's shared memory from (n_a, D): A resident or streamed through the ring, 5-8 ring stages, 1-4 seed
slots (tests/test_search_plan.py pins the table).  One case per plan (two more where the seed slots can be told apart)
runs N = 128 * (2 * SMs + 1) + r rows, so every CTA
sweeps two or three row tiles — the seed slots rotate across tile boundaries, A is refilled on its `a_empty` parity and the
next tile is prefetched into L2 — and the last tile is ragged.  Near ties are planted in the first tile, in a tile of the
second wave and in the last tile, so that rows finished by the exact re-score (vqb_fix_flagged) are spread over the waves.

Each case runs the three store-warp tails of the fused search (copy, residual, generic) and checks them bit for bit against
torch arithmetic on the kernel's own indices; the indices against a float64 search; the loss against a float64 sum with
F.mse_loss's rounding; every output buffer carries guard rows (and strided index gaps) holding a sentinel that must survive.
"""
import numpy as np
import pytest
import torch

from oracle import vq_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}
GUARD = 5                    # guard rows after row N in every output buffer
SENT_F = -12345.678          # sentinel of the float outputs (exact in neither dtype's arithmetic of these tests)
SENT_I = -7                  # sentinel of the int64 index slots
SENT_P = 0x7F7B              # sentinel bit pattern of the bf16 planes
TIE_TOL = 2e-6               # relative float64 top-2 gap below which the reference's own fp32 evaluation may pick either code


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


PLAN_CASES = [
    # dtype, D,    K,    cosine, r       plan (stream_a, stages, seed slots)
    ("bf16", 64, 256, False, 1),       # 0 8 4
    ("bf16", 136, 100, True, 77),      # 0 8 2   tiny codebook: Kpad = 112 < 128 fills the seed slot partly
    ("bf16", 200, 4096, False, 1),     # 0 8 1   32 code steps through one seed slot
    ("bf16", 384, 700, False, 77),     # 0 7 1   ragged K: padded codes in the last step
    ("bf16", 424, 1024, True, 1),      # 0 6 1
    ("bf16", 512, 333, False, 77),     # 0 5 1
    ("bf16", 1000, 256, False, 1),     # 1 6 1   streamed A
    ("fp32", 24, 37, False, 77),       # 0 8 3   tiny codebook
    ("fp32", 128, 1000, True, 1),      # 0 8 2
    ("fp32", 184, 4096, False, 77),    # 0 7 1
    ("fp32", 256, 300, False, 1),      # 0 5 1   exactly 227 KiB of shared memory
    ("fp32", 520, 700, True, 77),      # 1 6 1   streamed A
    # Code steps per tile not a multiple of the seed slots: from the second tile on, slot (step % slots) holds another
    # step's seeds, so only these cases see a seed slot chosen by the step within the tile instead of the global step.
    # (K >= 256 pads to a multiple of 256 codes: an even step count, which two slots cannot tell apart.)
    ("bf16", 40, 700, False, 77),      # 0 8 4   6 steps
    ("fp32", 64, 512, False, 1),       # 0 8 3   4 steps (Euclidean: cosine seeds are all 0)
]


def ref_search(xe, c, cosine):
    """float64 arg-max of the reference's scores (x.c, or -(||x||^2 + ||c||^2 - 2 x.c)) and the relative top-2 gap."""
    c64 = c.double()
    c2 = (c64 * c64).sum(-1)
    idx, gap = [], []
    for i in range(0, xe.shape[0], 8192):
        xs = xe[i:i + 8192].double()
        s = xs @ c64.T
        if cosine:
            scale = torch.ones(xs.shape[0], dtype=torch.float64, device=xs.device)
        else:
            x2 = (xs * xs).sum(-1)
            s = -(x2[:, None] + c2[None] - 2.0 * s)
            scale = x2.clamp_min(1e-30)
        top = s.topk(2, dim=-1).values
        gap.append((top[:, 0] - top[:, 1]) / scale)
        idx.append(s.argmax(-1))
    return torch.cat(idx), torch.cat(gap)


def mse_sum(q, xe, dt):
    """sum((q - x)^2) with F.mse_loss's rounding (oracle mse_loss): fp32 difference and square, bf16-rounded squares for
    bf16 tensors, summed in float64."""
    d = q.float() - xe.float()
    sq = d * d
    if dt == "bf16":
        sq = sq.bfloat16().float()
    return sq.double().sum().item()


def assert_loss_sum(got, ref, dt, rounded, what):
    """fp32: 1e-5 relative.  bf16: a tail that rounds every square like F.mse_loss (the generic one) to 1e-5 relative; the copy
    and residual tails read the loss off ||x||^2 - 2 * score without that per-element rounding, so their sum only has to give
    the same bf16 mean: within half a bf16 ulp of it."""
    tol = 1e-5 if dt == "fp32" or rounded else 2.0 ** -9
    assert abs(got - ref) <= tol * ref, (what, got, ref, abs(got - ref) / ref)


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def guarded(N, D, dt):
    """(N + GUARD, D) buffer holding the sentinel; rows >= N must keep it."""
    return torch.full((N + GUARD, D), SENT_F, dtype=TDT[dt], device=DEV)


def assert_guard(buf, N, what):
    sent = torch.full_like(buf[N:], SENT_F)
    assert torch.equal(bits(buf[N:]), bits(sent)), f"{what}: guard rows after row N were written"


def plant_ties(N, D, K, cosine, gen):
    """Codebook with duplicated codes and rows on top of them.  Returns (c, x_plants {row: (kind, code)})."""
    c = torch.randn(K, D, generator=gen)
    pair = (1, K - 2)                                      # K - 2: in the last code step (padded codes for ragged K)
    five = (2, 3, K // 2, K // 2 + 1, K - 1)               # > 3 candidates: the whole-row exact rescan
    near = (4, K // 3)
    c[pair[1]] = c[pair[0]]
    for k in five[1:]:
        c[k] = c[five[0]]
    c[near[1]] = c[near[0]] + 1e-4 * torch.randn(D, generator=gen)
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    s = sms()
    plants = {}
    for tile, off in ((0, 5), (s + 3, 40), (2 * s + 1, 0)):   # first tile, second wave, ragged last tile
        row = tile * 128 + off
        for j, (kind, code) in enumerate((("five", five[0]), ("pair", pair[0]), ("near", near[0]))):
            if row + j < N:
                plants[row + j] = (kind, code)
    return c, plants


@pytest.mark.parametrize("dt,D,K,cosine,r", PLAN_CASES)
def test_search_plan_fused_tails(dt, D, K, cosine, r):
    from vector_quantize_pytorch_b200 import ops
    N = 128 * (2 * sms() + 1) + r
    gen = torch.Generator().manual_seed(D * 7919 + K * 31 + r)
    c, plants = plant_ties(N, D, K, cosine, gen)
    x = torch.randn(N, D, generator=gen)
    scale = 1.0 / D ** 0.5 if cosine else 1.0
    for row, (_, code) in plants.items():
        x[row] = c[code] + 1e-2 * scale * torch.randn(D, generator=gen)
    x = x.to(TDT[dt]).to(DEV)
    c = c.to(DEV).contiguous()
    cb = ops.prepare_codebook(c, cosine)
    if cosine:
        xe_ref = torch.from_numpy(O.l2norm(x.float().cpu().numpy(), dt)).to(DEV)
    else:
        xe_ref = x.float()

    # ---- copy tail: q <- code row, int64 indices at a stride of 3, loss from the scores
    q_buf = guarded(N, D, dt)
    i_buf = torch.full(((N + GUARD) * 3,), SENT_I, dtype=torch.int64, device=DEV)
    l_copy = torch.zeros(1, dtype=torch.float64, device=DEV)
    res = ops.search(x, cb, c, fused=dict(q_out=q_buf[:N], idx64_out=i_buf, idx_stride=3, loss_sum=l_copy))
    torch.cuda.synchronize()
    torch.testing.assert_close(res.x_eff.float(), xe_ref, rtol=0, atol=1e-6 if dt == "fp32" else 0)
    xe = res.x_eff.float()      # the rows as searched: loss and statistics are taken against them
    idx = res.idx.long()

    # indices against float64
    ref_idx, gap = ref_search(xe_ref, c, cosine)
    mism = idx != ref_idx
    tie = gap < TIE_TOL
    assert not (mism & ~tie).any(), f"{int((mism & ~tie).sum())} mismatches outside near ties, rows {torch.nonzero(mism & ~tie)[:8, 0].tolist()}"
    assert int(mism.sum()) <= max(2, N // 500)
    # planted ties: the lowest of equal codes wins (vqp:140), and the rows went through the exact re-score
    n_front, n_back = res.flag_count.item(), res.rescan_count.item()
    assert n_front > 0 and n_back > 0
    front = set(res.flagged[:n_front, 0].tolist())
    back = set(res.flagged[N - n_back:, 0].tolist())
    for row, (kind, code) in plants.items():
        if kind == "near":
            continue
        assert idx[row].item() == code, (row, kind, idx[row].item(), code)
        assert row in (back if kind == "five" else front | back), (row, kind)
    assert N - 1 in plants or r > 1

    q_ref = c[idx].to(TDT[dt])
    assert torch.equal(bits(q_buf[:N]), bits(q_ref)), "copy tail: q_out"
    assert_guard(q_buf, N, "copy tail: q_out")
    iv = i_buf.view(N + GUARD, 3)
    assert torch.equal(iv[:N, 0], idx), "copy tail: idx64_out"
    assert (iv[:N, 1:] == SENT_I).all() and (iv[N:] == SENT_I).all(), "copy tail: idx64_out gaps / guard written"
    l_ref = mse_sum(q_ref, xe, dt)
    assert_loss_sum(l_copy.item(), l_ref, dt, False, "copy tail: loss")

    # ---- residual tail: r <- x - q rounded once (+ the bf16 hi / lo planes of r for fp32 rows), loss.  Cosine: the residual
    # is taken from the raw rows, so this runs the generic tail (x_raw != x_eff).
    r_buf = guarded(N, D, dt)
    l_res = torch.zeros(1, dtype=torch.float64, device=DEV)
    fused = dict(resid_out=r_buf[:N], loss_sum=l_res)
    if dt == "fp32":
        p_buf = torch.full((2 * N * D + GUARD * D,), SENT_P, dtype=torch.int16, device=DEV)
        fused["planes_out"] = p_buf
    res2 = ops.search(x, cb, c, fused=fused)
    torch.cuda.synchronize()
    assert torch.equal(res2.idx, res.idx)
    r_ref = (x.float() - q_ref.float()).to(TDT[dt])
    assert torch.equal(bits(r_buf[:N]), bits(r_ref)), "residual tail: resid_out"
    assert_guard(r_buf, N, "residual tail: resid_out")
    if dt == "fp32":
        hi = r_ref.bfloat16()
        lo = (r_ref - hi.float()).bfloat16()
        assert torch.equal(p_buf[:N * D].view(N, D), hi.view(torch.int16)), "residual tail: planes_out hi"
        assert torch.equal(p_buf[N * D:2 * N * D].view(N, D), lo.view(torch.int16)), "residual tail: planes_out lo"
        assert (p_buf[2 * N * D:] == SENT_P).all(), "residual tail: planes_out guard written"
    assert_loss_sum(l_res.item(), l_ref, dt, cosine, "residual tail: loss")   # cosine: the generic tail

    # ---- generic tail (q_out and resid_out together): q_out, r <- x - q, int64 indices at a stride of 2, loss from x
    q2_buf = guarded(N, D, dt)
    r2_buf = guarded(N, D, dt)
    i2_buf = torch.full(((N + GUARD) * 2,), SENT_I, dtype=torch.int64, device=DEV)
    l_gen = torch.zeros(1, dtype=torch.float64, device=DEV)
    res3 = ops.search(x, cb, c, fused=dict(q_out=q2_buf[:N], resid_out=r2_buf[:N], idx64_out=i2_buf, idx_stride=2, loss_sum=l_gen))
    torch.cuda.synchronize()
    assert torch.equal(res3.idx, res.idx)
    assert torch.equal(bits(r2_buf[:N]), bits(r_ref)), "generic tail: resid_out"
    assert_guard(r2_buf, N, "generic tail: resid_out")
    assert torch.equal(bits(q2_buf[:N]), bits(q_ref)), "generic tail: q_out"
    assert_guard(q2_buf, N, "generic tail: q_out")
    iv2 = i2_buf.view(N + GUARD, 2)
    assert torch.equal(iv2[:N, 0], idx) and (iv2[:N, 1] == SENT_I).all() and (iv2[N:] == SENT_I).all(), "generic tail: idx64_out"
    assert_loss_sum(l_gen.item(), l_ref, dt, True, "generic tail: loss")

    # the running-sum output (qsum) is retired: asking for it is refused before the search kernel runs, not ignored
    from vector_quantize_pytorch_b200._C import VQBError
    s_buf = guarded(N, D, dt)
    with pytest.raises(VQBError, match="vqb_assign"):
        ops.search(x, cb, c, fused=dict(q_out=s_buf[:N], qsum=s_buf[:N]))
    torch.cuda.synchronize()
    assert (bits(s_buf) == bits(guarded(N, D, dt))).all(), "refused running sum: a buffer was written"

    # ---- EMA statistics of this batch
    st = ops.ema_stats(res.x_eff, res.idx, K)
    off = ops.stats_offset(K)
    assert torch.equal(st[:K], torch.bincount(idx, minlength=K).float())
    xe64 = xe.double()
    es_ref = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, idx, xe64)
    es_abs = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, idx, xe64.abs())
    err = (st[off:off + K * D].view(K, D).double() - es_ref).abs()
    assert (err <= 1e-5 * es_abs + 1e-6).all(), f"embed_sum: worst error {err.max().item():.3e}"


@pytest.mark.parametrize("dt", ["bf16", "fp32"])
def test_in_kernel_mask_across_waves(dt):
    """The row mask inside the search kernel over more than two waves of row tiles: whole padding tiles in the second wave and
    padding inside the ragged last tile.  Padding comes back as zeros / -1; live rows match the float64 search; after one
    training step cluster_size and embed_avg equal a float64 EMA over the live rows only."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(23)
    B, n, D, K = 3, 23000, 256, 1024
    N = B * n
    s = sms()
    assert N > 128 * 2 * s and N % 128 != 0
    decay = 0.8
    vq = m.VectorQuantize(dim=D, codebook_size=K, decay=decay).to(DEV)
    with torch.no_grad():
        e = torch.randn(1, K, D, device=DEV)
        vq._codebook.embed.copy_(e)
        vq._codebook.embed_avg.copy_(e)
    cs0 = vq._codebook.cluster_size[0].double().clone()
    ea0 = vq._codebook.embed_avg[0].double().clone()
    embed = vq._codebook.embed[0].clone()
    x = torch.randn(B, n, D, device=DEV).to(TDT[dt])
    mask = torch.rand(B, n, device=DEV) < 0.7
    flat = mask.view(-1)
    flat[128 * (s + 2):128 * (s + 6)] = False         # whole padding tiles in the second wave
    last = (N // 128) * 128
    flat[last + 1:last + 5] = False                   # padding inside the ragged last tile (live rows around it)
    flat[last] = True
    flat[-1] = True
    vq.train()
    q, ind, loss = vq(x, mask=mask)
    torch.cuda.synchronize()
    assert (ind[~mask] == -1).all() and (q[~mask] == 0).all()
    live = flat.nonzero()[:, 0]
    xs = x.reshape(-1, D)[live]
    got = ind.reshape(-1)[live]
    ref, gap = ref_search(xs.float(), embed, False)
    mism = got != ref
    assert not (mism & (gap >= TIE_TOL)).any() and int(mism.sum()) <= max(2, live.numel() // 500)
    assert torch.equal(q.reshape(-1, D)[live], embed[got].to(TDT[dt]))
    cnt = torch.bincount(got, minlength=K).double()
    es = torch.zeros(K, D, dtype=torch.float64, device=DEV).index_add_(0, got, xs.double())
    cs_ref = cs0 + (1 - decay) * (cnt - cs0)
    ea_ref = ea0 + (1 - decay) * (es - ea0)
    torch.testing.assert_close(vq._codebook.cluster_size[0].double(), cs_ref, rtol=1e-6, atol=1e-5)
    torch.testing.assert_close(vq._codebook.embed_avg[0].double(), ea_ref, rtol=1e-5, atol=1e-4)


def _loss_ref(q, xe, dt):
    """F.mse_loss(q, x) as the reference returns it: float64 sum with the dtype's rounding, mean in fp32, bf16-rounded."""
    mean = torch.tensor(mse_sum(q, xe, dt) / q.numel(), dtype=torch.float32)
    return mean.bfloat16().float().item() if dt == "bf16" else mean.item()


def _check_loss(got, ref, dt, what):
    if dt == "fp32":
        rel = abs(got - ref) / ref
        print(f"commitment loss {what}: relative error {rel:.3e}")
        assert rel <= 1e-5, (what, got, ref, rel)
    else:
        ulp = 2.0 ** (np.floor(np.log2(ref)) - 7)
        print(f"commitment loss {what}: error {abs(got - ref) / ulp:.2f} bf16 ulp")
        assert abs(got - ref) <= ulp, (what, got, ref)


def _near_code_rows(c, n_rows, eps, gen):
    """Rows x = c[j] + noise with ||noise||^2 = eps * ||c[j]||^2, j drawn at random: a trained codebook's view of its data."""
    K, D = c.shape
    j = torch.randint(0, K, (n_rows,), generator=gen)
    noise = torch.nn.functional.normalize(torch.randn(n_rows, D, generator=gen), dim=-1)
    return c[j] + noise * (eps ** 0.5) * c[j].norm(dim=-1, keepdim=True), j


EPS = [1e-1, 1e-2, 1e-3]


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("dt,cosine", [("fp32", False), ("bf16", False), ("fp32", True), ("bf16", True)])
def test_commitment_loss_close_to_codes_vq(dt, cosine, eps):
    """VectorQuantize's fused loss (copy tail) when the rows lie close to their codes, eps = ||x - q||^2 / ||x||^2 small:
    the loss must not be read off ||x||^2 - 2 * score where that difference cancels."""
    import vector_quantize_pytorch_b200 as m
    D, K, N = 256, 1024, 8192
    gen = torch.Generator().manual_seed(int(1 / eps) + 2 * cosine)
    c = torch.randn(K, D, generator=gen)
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    x, j = _near_code_rows(c, N, eps, gen)
    vq = m.VectorQuantize(dim=D, codebook_size=K, use_cosine_sim=cosine).to(DEV)
    with torch.no_grad():
        vq._codebook.embed[0].copy_(c)
        vq._codebook.embed_avg[0].copy_(c)
    xd = x.to(TDT[dt]).to(DEV)[None]
    vq.train()
    q, ind, loss = vq(xd)
    torch.cuda.synchronize()
    assert torch.equal(ind[0].cpu(), j)
    q_ref = c.to(DEV)[j.to(DEV)].to(TDT[dt])
    assert torch.equal(q[0], q_ref)
    xe = torch.from_numpy(O.l2norm(xd[0].float().cpu().numpy(), dt)).to(DEV) if cosine else xd[0].float()
    _check_loss(loss.item(), _loss_ref(q_ref, xe, dt), dt, f"VectorQuantize {dt} {'cosine' if cosine else 'euclid'} eps={eps:g}")


@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
def test_commitment_loss_close_to_codes_rvq(dt, eps):
    """ResidualVQ(num_quantizers=2): the first stage runs the residual tail (and, for fp32, hands the next stage the bf16
    planes of the residual); both stages' losses against float64 along the residual recurrence."""
    import vector_quantize_pytorch_b200 as m
    D, K, N = 256, 1024, 8192
    gen = torch.Generator().manual_seed(int(1 / eps) + 7)
    books = [torch.randn(K, D, generator=gen) for _ in range(2)]
    x, j = _near_code_rows(books[0], N, eps, gen)
    rvq = m.ResidualVQ(dim=D, num_quantizers=2, codebook_size=K).to(DEV)
    with torch.no_grad():
        for layer, c in zip(rvq.layers, books):
            layer._codebook.embed[0].copy_(c)
            layer._codebook.embed_avg[0].copy_(c)
    xd = x.to(TDT[dt]).to(DEV)[None]
    rvq.train()
    out, ind, losses = rvq(xd)
    torch.cuda.synchronize()
    assert torch.equal(ind[0, :, 0].cpu(), j)
    q0 = books[0].to(DEV)[ind[0, :, 0]].to(TDT[dt])
    r1 = (xd[0].float() - q0.float()).to(TDT[dt])
    q1 = books[1].to(DEV)[ind[0, :, 1]].to(TDT[dt])
    _check_loss(losses[0].item(), _loss_ref(q0, xd[0].float(), dt), dt, f"ResidualVQ stage 0 {dt} eps={eps:g}")
    _check_loss(losses[1].item(), _loss_ref(q1, r1.float(), dt), dt, f"ResidualVQ stage 1 {dt} eps={eps:g}")
