"""The EMA codebook update against float64 on every path it takes (run on an H100: `pytest -m gpu`).

(a) Batch statistics.  The production chain (search kernel's slab histogram + provisional indices, sort on the side stream,
    exact re-score rows added by stats_add_flagged) and the stand-alone chain (ops.ema_stats: hist_kernel with shared or
    global atomics) against float64 sums over the kernel's own final indices.  Counts are exact; each embed_sum element is within (L + 2) * 2^-24 * sum|x| of the float64 sum, where
    L is the longest chain of fp32 additions the kernels give that element.
(b) ops.ema_apply from a given statistics buffer against float64 evaluations of the same formulas, with an error bound that
    follows every fp32 rounding; the refreshed tensor-core operands bit for bit against vqb_codebook_prepare of the new
    codebook, padded rows included, after the step shrank the code norms (a cmax that is not reset stays too large).
(c) The same checks through VectorQuantize and ResidualVQ (shared codebook: Q lerps and one normalise in one launch).
"""
import ctypes

import pytest
import torch

from oracle import vq_oracle as O
from test_search_plans_gpu import TIE_TOL, ref_search

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"fp32": torch.float32, "bf16": torch.bfloat16}
U = 2.0 ** -24               # unit roundoff of fp32
SEG_CHUNK = 512              # rows per work item of the segmented sums (csrc/vq_ema.cu)
SEG_THREADS = 256
SENT16 = 0x5A5A              # sentinel bit pattern of the 2-byte operand planes and bext
SENT_F = -12345.678


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stats_plan(N, K):
    """(G, shift) of the counting sort on this device: G = 0 is the global-atomic path."""
    from vector_quantize_pytorch_b200 import _C
    out = (ctypes.c_int * 3)()
    assert _C.lib.vqb_debug_stats_plan(N, K, sms(), ctypes.cast(out, ctypes.c_void_p)) == 0
    return out[0], out[1]


def seg_lanes(dt, D):
    """NY: rows summed side by side in one segsum CTA (TX = D / VEC threads across a row)."""
    return SEG_THREADS // (D // (8 if dt == "bf16" else 4))


def chain_sorted(cnt, n_flag, NY):
    """Longest fp32 addition chain of an embed_sum element of the sort path: a row lane sums ceil(rows / NY) rows of its work
    item, the NY lanes are summed in order, and every work item of the code (ceil(sorted / 512)) and every re-scored row of it
    (stats_add_flagged) lands on the element by atomicAdd."""
    srt = cnt - n_flag
    return torch.ceil(srt.clamp(max=SEG_CHUNK) / NY) + NY + torch.ceil(srt / SEG_CHUNK) + n_flag


def ref_stats(xe, idx, K):
    x64 = xe.double()
    cnt = torch.bincount(idx, minlength=K).double()
    es = torch.zeros(K, xe.shape[1], dtype=torch.float64, device=DEV).index_add_(0, idx, x64)
    ab = torch.zeros_like(es).index_add_(0, idx, x64.abs())
    return cnt, es, ab


def unpack(st, K, D):
    from vector_quantize_pytorch_b200 import ops
    off = ops.stats_offset(K)
    return st[:K], st[off:off + K * D].view(K, D)


def check_stats(st, xe, idx, K, L, what):
    cnt, es, ab = ref_stats(xe, idx, K)
    cs_got, es_got = unpack(st, K, xe.shape[1])
    assert torch.equal(cs_got.double(), cnt), f"{what}: cluster_size"
    err = (es_got.double() - es).abs()
    tol = (L[:, None] + 2) * U * ab
    bad = err > tol
    assert not bad.any(), f"{what}: embed_sum off at {int(bad.sum())} elements, worst {float((err / tol.clamp_min(1e-300)).max()):.2f} x the bound"
    return float((err / tol.clamp_min(1e-300)).max())


def tie_codebook(K, D, cosine, gen):
    """Duplicated codes (as in test_search_plans_gpu.plant_ties): rows on a pair go to the front flag list (2 candidates),
    rows on five equal codes to the back list (whole-row rescan)."""
    c = torch.randn(K, D, generator=gen)
    pair, five, near = (1, K - 2), (2, 3, K // 2, K // 2 + 1, K - 1), (4, K // 3)
    c[pair[1]] = c[pair[0]]
    for k in five[1:]:
        c[k] = c[five[0]]
    c[near[1]] = c[near[0]] + 1e-4 * torch.randn(D, generator=gen)
    return c, (("five", five[0]), ("pair", pair[0]), ("near", near[0]))


def plant_rows(x, c, kinds, rows, cosine, gen):
    scale = 1.0 / x.shape[1] ** 0.5 if cosine else 1.0
    plants = {}
    for r0 in rows:
        for j, (kind, code) in enumerate(kinds):
            x[r0 + j] = c[code] + 1e-2 * scale * torch.randn(x.shape[1], generator=gen)
            plants[r0 + j] = (kind, code)
    return plants


# ------------------------------------------------------------------------------------------------ (a) statistics
# name, dtype, D, K, N ("cap": 8 row tiles per SM), cosine, skew, expected sort path
STATS_CASES = [
    ("global_d8", "bf16", 8, 1000, 20000, False, True, "global"),           # N < 32 K; ema_stats: hist_kernel in smem
    ("global_k10000_d24", "fp32", 24, 10000, 60000, False, True, "global"),  # K > 8192: hist_kernel's global atomics; TX = 6
    ("cta_g24_d1000", "bf16", 1000, 300, 12000, True, False, "g<32"),       # fewer slabs than the column scan's 32 warps
    ("cta_g79_d1024", "fp32", 1024, 1000, 40000, False, True, "g%32"),      # G not a multiple of 32; NY = 1
    ("cta_cap_d256", "bf16", 256, 1000, "cap", False, True, "cap"),         # G = SMs, shift 3
    ("cta_cap_cosine", "bf16", 256, 777, "cap", True, False, "cap"),
]


def stats_case(dt, D, K, N, cosine, skew, gen):
    """Rows and codebook of a statistics case.  Skewed cases plant rows around three far-away codes (exactly 512, exactly
    513 and about 40 % of N rows: one work item, a split into two, many) and move three more codes as far without planting
    rows: they stay empty."""
    c, kinds = tie_codebook(K, D, cosine, gen)
    x = torch.randn(N, D, generator=gen)
    tie_rows = [N * j // 5 + 11 for j in range(5)] + [N - 3]     # several slabs, the last rows included
    skew_codes, empty = {}, []
    if skew:
        a, b, big = K // 5, K // 5 + 1, (3 * K) // 4
        empty = [K // 5 + 2, K // 5 + 3, K - 5]
        # 4x the norm of a randn code: far from every randn row, and still small enough that the certification band (it grows
        # with max ||c||^2) leaves the rows on two equal codes in the front flag list
        for k in (a, b, big, *empty):
            c[k] = 4.0 * torch.randn(D, generator=gen)
        free = torch.ones(N, dtype=torch.bool)
        for r0 in tie_rows:
            free[r0:r0 + 3] = False
        perm = torch.nonzero(free)[:, 0][torch.randperm(int(free.sum()), generator=gen)]
        n_big = int(0.4 * N)
        at = 0
        for k, n in ((a, 512), (b, 513), (big, n_big)):
            rows = perm[at:at + n]
            at += n
            x[rows] = c[k] + 0.05 * torch.randn(n, D, generator=gen)
            skew_codes[k] = n
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    plants = plant_rows(x, c, kinds, tie_rows, cosine, gen)
    return x.to(TDT[dt]).to(DEV), c.to(DEV).contiguous(), plants, skew_codes, empty


@pytest.mark.parametrize("name,dt,D,K,N,cosine,skew,path", STATS_CASES, ids=[c[0] for c in STATS_CASES])
def test_counting_sort_statistics_within_bound(name, dt, D, K, N, cosine, skew, path):
    from vector_quantize_pytorch_b200 import ops
    s = sms()
    if N == "cap":
        N = 8 * 128 * min(s, 256) - 77
    G, shift = stats_plan(N, K)
    if path == "global":
        assert G == 0
    elif path == "g<32":
        assert 0 < G < 32
    elif path == "g%32":
        assert G > 32 and G % 32 != 0
    else:
        assert G == min(s, 256) and shift >= 3
    gen = torch.Generator().manual_seed(K * 131 + D)
    x, c, plants, skew_codes, empty = stats_case(dt, D, K, N, cosine, skew, gen)
    cb = ops.prepare_codebook(c, cosine)

    # the rows as searched, the final indices and both flag lists
    res = ops.search(x, cb, c)
    torch.cuda.synchronize()
    idx = res.idx.long()
    xe = res.x_eff
    n_front, n_back = res.flag_count.item(), res.rescan_count.item()
    front = set(res.flagged[:n_front, 0].tolist())
    back = set(res.flagged[N - n_back:, 0].tolist())
    for row, (kind, code) in plants.items():   # the lowest of equal codes wins (vqp:140)
        if kind == "five":
            assert row in back and idx[row].item() == code, (row, kind)
        elif kind == "pair":
            assert row in front | back and idx[row].item() == code, (row, kind)
    assert front and back, "stats_add_flagged must carry rows of both flag lists"
    flag_rows = torch.tensor(sorted(front | back), dtype=torch.long, device=DEV)
    n_flag = torch.bincount(idx[flag_rows], minlength=K).double()
    cnt = torch.bincount(idx, minlength=K).double()
    for k, n in skew_codes.items():
        assert cnt[k].item() == n, (k, cnt[k].item(), n)
    for k in empty:
        assert cnt[k].item() == 0

    NY = seg_lanes(dt, D)
    zero = torch.zeros_like(cnt)
    state = (torch.ones(K, device=DEV), c.clone(), c)
    worst = {}
    idx32, st = ops.vq_forward(x, cb, state, update=1, do_normalise=False, decay=0.8, eps=1e-5)
    torch.cuda.synchronize()
    assert torch.equal(idx32.long(), idx), "vq_forward: indices differ from the search"
    # segment chains + one atomicAdd per work item and per re-scored row
    worst["vq_forward"] = check_stats(st, xe, idx, K, chain_sorted(cnt, n_flag, NY), f"{name} vq_forward stats")
    st = ops.ema_stats(xe, res.idx, K)
    torch.cuda.synchronize()
    worst["ema_stats"] = check_stats(st, xe, idx, K, chain_sorted(cnt, zero, NY), f"{name} ema_stats")
    if empty:
        assert (unpack(st, K, D)[1][empty] == 0).all()
    print(f"{name}: N={N} G={G} shift={shift} flagged {n_front}+{n_back}; worst error / bound: "
          + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------ (b) apply
def lerp_b(a, ea, b, eb, w):
    """torch.lerp(a, b, w) for 0 <= w <= 1 in float64 and a bound on the fp32 kernel's error, given bounds ea / eb on its
    inputs: three roundings (b - a, the product, the sum; 1 - w is exact for w >= 1/2)."""
    v = a + w * (b - a)
    return v, (1 - w) * ea + w * eb + U * (v.abs() + 2 * (b - a).abs())


def ema_ref(cs, ea, batches, w, K, eps, cosine, normalise=True):
    """float64 EMA of vector_quantize_pytorch (lerp of each batch in order, then embed = embed_avg / laplace-smoothed sizes,
    l2norm for cosine) with running bounds on the fp32 kernels' error.  batches: [(cnt, embed_sum, embed_sum error bound)];
    w (K,) the fp32 per-code lerp weight.  Returns ((cs, ecs), (ea, eea), (embed, eembed) or None)."""
    ecs, eea = torch.zeros_like(cs), torch.zeros_like(ea)
    for cnt, es, ees in batches:
        cs, ecs = lerp_b(cs, ecs, cnt, 0.0, w)
        ea, eea = lerp_b(ea, eea, es, ees, w[:, None])
    if not normalise:
        return (cs, ecs), (ea, eea), None
    epsf = float(torch.tensor(eps, dtype=torch.float32))
    kepsf = float(torch.tensor(K * eps, dtype=torch.float32))
    T = cs.sum()
    eT = ecs.sum() + U * T                                   # summed in double, rounded once
    num, den = cs + epsf, T + kepsf
    rel = (ecs + U * num) / num + (eT + U * den) / den + U + eT / T + U    # (cs + eps) / (T + K eps) * T
    denom = num / den * T
    emb = ea / denom[:, None]
    eemb = emb.abs() * (rel[:, None] + U) + eea / denom[:, None]
    if cosine:
        n = emb.norm(dim=-1).clamp_min(1e-6)[:, None]
        E = eemb.norm(dim=-1)[:, None]
        emb = emb / n
        eemb = eemb / n + emb.abs() * (E / n + 3 * U)        # norm: double sum, sqrt, fp32 rounding; the division
    return (cs, ecs), (ea, eea), (emb, eemb)


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > 2 * bound     # 2: room for the second-order terms the first-order bound leaves out
    assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the bound, worst {float((err / bound.clamp_min(1e-300)).max()):.2f} x"
    return float((err / bound.clamp_min(1e-300)).max())


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def assert_operands(got, embed, cosine, what):
    """Every operand tensor bit for bit against vqb_codebook_prepare of `embed`, padded rows included."""
    from vector_quantize_pytorch_b200 import ops
    ref = ops.prepare_codebook(embed.contiguous(), cosine)
    torch.cuda.synchronize()
    for f in ("planes", "bext", "bias", "cnorm2", "cmax"):
        a, b = getattr(got, f), getattr(ref, f)
        assert a.shape == b.shape and torch.equal(bits(a), bits(b)), f"{what}: {f} differs from vqb_codebook_prepare"


def w32(decay, weight, K):
    w = torch.full((K,), 1.0 - decay, dtype=torch.float32, device=DEV)
    if weight is not None:
        w = w * weight
    return w.double()


# D, K, cosine, code_weight, do_lerp, do_normalise, NV of ema_rows_kernel (float4 of the row per lane: 4 for D <= 512, else 8)
APPLY_CASES = [
    (64, 1000, False, None, True, True, 4),
    (64, 37, True, "zeros", True, True, 4),
    (512, 700, True, None, True, True, 4),
    (512, 300, False, "zeros", True, True, 4),
    (520, 333, True, "zeros", True, True, 8),
    (520, 1000, False, None, False, True, 8),     # update_ema of the k-means init: no lerp
    (1024, 100, True, None, False, True, 8),
    (1024, 257, False, "zeros", True, True, 8),
    (64, 1000, True, None, False, True, 4),
    (520, 100, True, None, True, False, 8),       # lerp only (track_cluster_size_and_embed_avg): embed, operands untouched
    (256, 100, False, "zeros", True, False, 4),
]


@pytest.mark.parametrize("D,K,cosine,weight,do_lerp,do_normalise,nv", APPLY_CASES)
def test_ema_apply(D, K, cosine, weight, do_lerp, do_normalise, nv):
    from vector_quantize_pytorch_b200 import ops
    assert nv == (4 if D <= 512 else 8)
    Kpad = ops.padded_codes(K)
    decay, eps = 0.8, 1e-5
    gen = torch.Generator().manual_seed(D * 1009 + K)
    c0 = torch.randn(K, D, generator=gen)
    if cosine:
        c0 = torch.nn.functional.normalize(c0, dim=-1)
    # the operands (and `embed`) of a codebook 10x longer than the EMA state: the step shrinks every code norm, even where
    # the weight is zero, so a cmax that is not reset stays visibly too large
    embed0 = (10.0 * c0).to(DEV)
    cs0 = (torch.rand(K, generator=gen) * 20 + 0.5).to(DEV)
    ea0 = (c0.to(DEV) * cs0[:, None]).contiguous()
    target = torch.randn(K, D, generator=gen)
    cnt = torch.randint(0, 60, (K,), generator=gen).float()
    cnt[::7] = 0
    es = cnt[:, None] * target + cnt.sqrt()[:, None] * torch.randn(K, D, generator=gen)
    st = torch.zeros(ops.stats_floats(K, D), dtype=torch.float32, device=DEV)
    cnt, es = cnt.to(DEV), es.to(DEV)
    off = ops.stats_offset(K)
    st[:K] = cnt
    st[off:off + K * D] = es.reshape(-1)
    cw = None
    if weight == "zeros":
        cw = torch.rand(K, generator=gen).to(DEV)
        cw[::3] = 0.0
    cb = ops.prepare_codebook(embed0, cosine)
    cmax0 = cb.cmax.clone()
    for t in (cb.planes, cb.bext):
        t.view(torch.int16).fill_(SENT16)
    cb.bias.fill_(SENT_F)
    cb.cnorm2.fill_(SENT_F)
    sent = {f: getattr(cb, f).clone() for f in ("planes", "bext", "bias", "cnorm2", "cmax")}
    cs, ea, emb = cs0.clone(), ea0.clone(), embed0.clone()
    ops.ema_apply(cs, ea, emb, st if do_lerp else None, cb, decay=decay, eps=eps, do_lerp=do_lerp, do_normalise=do_normalise,
                  code_weight=cw)
    torch.cuda.synchronize()

    w = w32(decay, cw, K)
    batches = [(cnt.double(), es.double(), torch.zeros(K, D, dtype=torch.float64, device=DEV))] if do_lerp else []
    (cs_r, ecs), (ea_r, eea), e = ema_ref(cs0.double(), ea0.double(), batches, w, K, eps, cosine, do_normalise)
    worst = [assert_within(cs, cs_r, ecs, "cluster_size"), assert_within(ea, ea_r, eea, "embed_avg")]
    if not do_lerp:
        assert torch.equal(cs, cs0) and torch.equal(ea, ea0)
    if cw is not None:   # a zero weight leaves the code's EMA state exactly as it was
        z = cw == 0
        assert torch.equal(cs[z], cs0[z]) and torch.equal(ea[z], ea0[z])
    if not do_normalise:
        assert torch.equal(emb, embed0)
        for f, t in sent.items():
            assert torch.equal(bits(getattr(cb, f)), bits(t)), f"{f} written without do_normalise"
        return
    worst.append(assert_within(emb, e[0], e[1], "embed"))
    assert_operands(cb, emb, cosine, f"D={D} K={K} (Kpad {Kpad}) NV={nv}")
    assert cb.cmax[0] < cmax0[0], "the step should have shrunk the largest code norm"
    print(f"D={D} K={K} Kpad={Kpad} {'cosine' if cosine else 'euclid'} NV={nv}: worst error / bound "
          + " ".join(f"{v:.3f}" for v in worst))


# ------------------------------------------------------------------------------------------------ (c) through the modules
def stats_bound(dt, D, K, N, idx, xe):
    """(cnt, embed_sum, bound) of one batch through the sort path, with every row counted as possibly re-scored (f <= count:
    the module does not return its flag lists)."""
    G, _ = stats_plan(N, K)
    assert G > 0
    cnt, es, ab = ref_stats(xe, idx, K)
    L = chain_sorted(cnt, torch.zeros_like(cnt), seg_lanes(dt, D)) + cnt   # >= the chain for any f <= count
    return cnt, es, (L[:, None] + 2) * U * ab


def check_module_codebook(book, cs0, ea0, batches, K, D, cosine, decay, ops_before, what):
    from vector_quantize_pytorch_b200 import ops
    cs, ea, emb = book._state2d()
    (cs_r, ecs), (ea_r, eea), (e_r, ee) = ema_ref(cs0, ea0, batches, w32(decay, None, K), K, book.eps, cosine)
    assert_within(cs, cs_r, ecs, f"{what}: cluster_size")
    assert_within(ea, ea_r, eea, f"{what}: embed_avg")
    assert_within(emb, e_r, ee, f"{what}: embed")
    n0 = ops.LAUNCHES
    got = book.operands()
    assert got is ops_before and ops.LAUNCHES == n0, f"{what}: the operands were not refreshed by the EMA kernel"
    assert_operands(got, emb.clone(), cosine, what)


VQ_CASES = [
    ("bf16", 256, 1024, 262144, False),    # config 2: CTA sort, 128 slabs of 16 row tiles on 132 SMs
    ("bf16", 256, 1000, 65536, True),
    ("fp32", 640, 500, 40000, False),      # D > 512: ema_rows_kernel with 8 float4 per lane
]


@pytest.mark.parametrize("dt,D,K,N,cosine", VQ_CASES)
def test_vector_quantize_ema_step(dt, D, K, N, cosine):
    import vector_quantize_pytorch_b200 as m
    G, shift = stats_plan(N, K)
    assert G > 0
    if N == 262144 and K == 1024:
        assert shift == 4 or sms() < 128
    decay = 0.8
    gen = torch.Generator().manual_seed(N + D + K)
    c, kinds = tie_codebook(K, D, cosine, gen)
    if cosine:
        c = torch.nn.functional.normalize(c, dim=-1)
    x = torch.randn(N, D, generator=gen)
    plant_rows(x, c, kinds, [N * j // 7 + 5 for j in range(7)], cosine, gen)
    x = x.to(TDT[dt]).to(DEV)
    c = c.to(DEV)
    vq = m.VectorQuantize(dim=D, codebook_size=K, decay=decay, use_cosine_sim=cosine).to(DEV)
    book = vq._codebook
    with torch.no_grad():
        book.embed[0].copy_(c)
        book.embed_avg[0].copy_(c)
    ops_before = book.operands()
    cmax0 = ops_before.cmax.clone()
    cs0, ea0 = book.cluster_size[0].double().clone(), book.embed_avg[0].double().clone()
    vq.train()
    _, ind, _ = vq(x[None])
    torch.cuda.synchronize()
    idx = ind[0]
    xe = torch.from_numpy(O.l2norm(x.float().cpu().numpy(), dt)).to(DEV) if cosine else x.float()
    check_module_codebook(book, cs0, ea0, [stats_bound(dt, D, K, N, idx, xe)], K, D, cosine, decay, ops_before,
                          f"VectorQuantize {dt} D={D} K={K}")
    if not cosine:
        assert ops_before.cmax[0] < cmax0[0]
    # the next search runs on the refreshed operands
    embed1 = book.embed[0].clone()
    vq.eval()
    _, ind2, _ = vq(x[None])
    torch.cuda.synchronize()
    ref, gap = ref_search(xe, embed1, cosine)
    mism = ind2[0] != ref
    assert not (mism & (gap >= TIE_TOL)).any() and int(mism.sum()) <= max(2, N // 500)


def residuals(x, dt, books, idx):
    """Stage inputs of a ResidualVQ rebuilt from its indices: r <- (r - q).to(dtype), q = code row in the input dtype."""
    r, out = x, []
    for q, c in enumerate(books):
        out.append(r)
        qv = c[idx[:, q]].to(TDT[dt])
        r = (r.float() - qv.float()).to(TDT[dt])
    return out


@pytest.mark.parametrize("shared", [True, False], ids=["shared", "separate"])
def test_residual_vq_ema_step(shared):
    import vector_quantize_pytorch_b200 as m
    if shared:   # Q lerps of one codebook and one normalise: a single EMA op with n_lerp = Q
        dt, D, K, N, Q = "fp32", 64, 250, 16384, 8
    else:
        dt, D, K, N, Q = "bf16", 128, 300, 20000, 3
    decay = 0.8
    gen = torch.Generator().manual_seed(Q * 1000 + D)
    rvq = m.ResidualVQ(dim=D, num_quantizers=Q, codebook_size=K, shared_codebook=shared, decay=decay).to(DEV)
    books = [rvq.layers[0]._codebook] if shared else [layer._codebook for layer in rvq.layers]
    if shared:
        assert all(layer._codebook is books[0] for layer in rvq.layers) and books[0].manual_ema_update
    init = []
    with torch.no_grad():
        for b in books:
            c = torch.randn(K, D, generator=gen).to(DEV) * (0.5 if shared else 1.0)
            b.embed[0].copy_(c)
            b.embed_avg[0].copy_(c)
            init.append((b.cluster_size[0].double().clone(), b.embed_avg[0].double().clone(), c.clone(), b.operands()))
    x = torch.randn(N, D, generator=gen).to(TDT[dt]).to(DEV)
    rvq.train()
    _, ind, _ = rvq(x[None])
    torch.cuda.synchronize()
    idx = ind[0]
    searched = [init[0][2]] * Q if shared else [i[2] for i in init]
    rs = residuals(x, dt, searched, idx)
    batches = [stats_bound(dt, D, K, N, idx[:, q], rs[q].float()) for q in range(Q)]
    if shared:
        cs0, ea0, _, ops0 = init[0]
        check_module_codebook(books[0], cs0, ea0, batches, K, D, False, decay, ops0, f"shared codebook Q={Q}")
    else:
        for q, (b, (cs0, ea0, _, ops0)) in enumerate(zip(books, init)):
            check_module_codebook(b, cs0, ea0, [batches[q]], K, D, False, decay, ops0, f"stage {q}")
