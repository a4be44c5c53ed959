"""The ResidualSimVQ kernels (csrc/vq_rsimvq.cu) against float64 on every path they take (run on an H100: `pytest -m gpu`).

(1) vqb_rsimvq_tail, one stage at a time, on every row kind of the rotation test plus the residuals late stages see (a few ulps
    of the code, norm 1e-7: the 1e-6 clamp branch).  Straight-through values bit for bit against torch fp32, rotation values
    within the first-order bound of test_decode_rotate_gpu; r_next and qsum exact given the value; the loss sum and its
    rounding to fp32; every optional output (r_next, loss_out) left out; guard rows and the gaps of a strided index output.
(2) vqb_rsimvq_backward on four stages built with the tail: against float64 on the tail's own residuals; the residual
    recompute bit-identical to the forward's (DESIGN §4.7); grad_q / grad_loss NULL; quantize dropout (index -1 columns).
(3) ResidualSimVQ: the cached program against direct calls, bit for bit; quantize dropout at size; the codebook and transform
    gradients; a backward through only the losses or only the output; rows that sit on a stage-0 code.

D takes one value per register-slot count J (the smallest power of two with 32 J >= D) with a full and a partial last slot,
and an odd D: 8 -> 1, 33, 40, 64 -> 2, 100 -> 4, 200, 256 -> 8, 300, 512 -> 16, 520, 1024 -> 32.  Row counts: 1, 7, and more
than two grids of warps (16 CTAs per SM x 8 rows), ragged, so that the grid-stride loop runs.

Every float64 reference is evaluated on the kernels' own fp32 residuals cast to float64, never on a float64 recurrence: a
residual of a few ulps rotates with lambda = ||c|| / 1e-6, and a float64 recurrence would drift from the kernel's residual by
up to 1e6 ulps and say nothing about the kernel.
"""
import numpy as np
import pytest
import torch

from test_decode_rotate_gpu import ROW_KINDS, ratio, rotate_bound, rotate_eval, rotation_rows

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS32 = 2.0 ** -24
GUARD = 5                        # guard rows after row N in every output buffer
SENT = -12345.678                # their sentinel (fp32 buffers)
ISENT = -777                     # int64 sentinel
LSENT = 123.25                   # loss_sum sentinel
IW, W = 0.3, 1.7                 # input_weight and weight: not the defaults 0.25 and 1
CHUNK = 1024                     # rows per chunk of the float64 references
D_SLOTS = {8: 1, 33: 2, 40: 2, 64: 2, 100: 4, 200: 8, 256: 8, 300: 16, 512: 16, 520: 32, 1024: 32}
# the multi-wave row count takes up to 0.7 GB of device memory at D = 520 and would take twice that at D = 1024; D = 520
# already runs the J = 32 instantiation through the grid-stride loop
CASES = [(D, rows) for D in D_SLOTS for rows in ("1", "7", "waves") if not (rows == "waves" and D > 520)]
KINDS = ROW_KINDS + ["ulp_res", "tiny_res"]


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def n_rows(rows):
    if rows != "waves":
        return int(rows)
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 16 * 8 + 37


def chunks(N):
    return [slice(a, min(a + CHUNK, N)) for a in range(0, N, CHUNK)]


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def ptr(t):
    return None if t is None else t.data_ptr()


def tail_call(r, codes, idx32, rotation, r_next, qsum, first, idx64, stride, loss_sum, loss_out, iw=IW, w=W):
    from vector_quantize_pytorch_b200 import _C
    N, D = r.shape
    rc = _C.lib.vqb_rsimvq_tail(ptr(r), ptr(codes), ptr(idx32), N, D, int(rotation), ptr(r_next), ptr(qsum), int(first),
                                ptr(idx64), stride, ptr(loss_sum), ptr(loss_out), float(iw), float(w),
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc


def raw_backward(x, codes, idx, n_active, rotation, grad_q, grad_loss):
    """vqb_rsimvq_backward into N + GUARD rows; the guard rows must keep the sentinel."""
    from vector_quantize_pytorch_b200 import _C
    N, D = x.shape
    gx = torch.full((N + GUARD, D), SENT, device=DEV)
    rc = _C.lib.vqb_rsimvq_backward(ptr(x), ptr(codes), idx.shape[1], codes.shape[1], ptr(idx), N, D, n_active, int(rotation),
                                    ptr(grad_q), ptr(grad_loss), ptr(gx), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert torch.equal(gx[N:], torch.full_like(gx[N:], SENT)), "vqb_rsimvq_backward wrote past row N"
    return gx[:N]


def backward_reference(Rs, Cs, G, gl, rotation):
    """float64 d/dx of one chunk of rows: sum_q [rotation backward of G at (r_q, c_q), or G] + gl[q] (r_q - c_q), on the fp32
    stage residuals Rs[q] and codes Cs[q]; and a per-element bound on the kernel's fp32 evaluation: the rotate_bound of every
    stage, fl(r - c) and fl(gl (r - c)) (and gl itself rounded to fp32), and the 2 fp32 adds per stage of the accumulation."""
    D = Rs[0].shape[1]
    g64 = None if G is None else G.double()
    ref = bnd = mag = 0.0
    for s, t, glq in zip(Rs, Cs, gl):
        s64, t64 = s.double(), t.double()
        if g64 is None:
            de, bd = torch.zeros_like(s64), 0.0
        elif rotation:
            de, bd = rotate_eval(s64, t64, g64)[1], rotate_bound(s64, t64, g64, D)
        else:
            de, bd = g64, 0.0
        lt = glq * (s64 - t64)
        ref = ref + de + lt
        mag = mag + de.abs() + bd + lt.abs()
        bnd = bnd + bd + 4 * EPS32 * lt.abs()
    return ref, bnd + 2 * len(Rs) * EPS32 * mag


# ------------------------------------------------------------------------------------------------ (1) the stage tail
def kind_rows(kind, n, D, gen):
    """(residual, code) float64 rows of one kind."""
    if kind in ROW_KINDS:
        return rotation_rows(kind, n, D, gen)
    t = torch.randn(n, D, generator=gen, device=DEV, dtype=torch.float64).float().double()
    if kind == "ulp_res":      # what a row that sat on its code leaves behind: a few ulps of the code
        return t * torch.randint(-2, 3, (n, D), generator=gen, device=DEV).double() * 2.0 ** -23, t
    unit = torch.randn(n, D, generator=gen, device=DEV, dtype=torch.float64)
    return 1e-7 * unit / unit.norm(dim=-1, keepdim=True), t     # "tiny_res": norm 1e-7 against a normal code


def tail_inputs(D, N, gen):
    """N residual rows r, a codebook of N + 3 rows holding their codes at a random permutation, the int32 indices, and the row
    kind of every row.  Kinds are interleaved (every warp meets several), starting at a D-dependent kind so N = 1 varies."""
    nk = len(KINDS)
    n = -(-N // nk)
    off = D % nk
    order = KINDS[off:] + KINDS[:off]
    parts = [[v.float() for v in kind_rows(k, n, D, gen)] for k in order]
    s = torch.stack([p[0] for p in parts], 1).reshape(-1, D)[:N].contiguous()
    t = torch.stack([p[1] for p in parts], 1).reshape(-1, D)[:N]
    del parts
    kind = torch.tensor([KINDS.index(k) for k in order], device=DEV).repeat(n)[:N]
    perm = torch.randperm(N + 3, generator=gen, device=DEV)[:N]
    codes = torch.randn(N + 3, D, generator=gen, device=DEV)
    codes[perm] = t
    return s, codes, perm.int(), kind


def tail_buffers(N, D):
    return dict(r_next=torch.full((N + GUARD, D), SENT, device=DEV), qsum=torch.full((N + GUARD, D), SENT, device=DEV),
                idx64=torch.full((3 * N + GUARD,), ISENT, dtype=torch.int64, device=DEV),
                loss_sum=torch.full((1,), LSENT, dtype=torch.float64, device=DEV), loss_out=torch.full((3,), SENT, device=DEV))


def run_tail(r, codes, idx32, rotation, b, first=1, with_r_next=True, with_loss=True):
    """One tail call into the buffers b: idx64_out at stride 3, loss_out its middle element."""
    tail_call(r, codes, idx32, rotation, b["r_next"] if with_r_next else None, b["qsum"], first, b["idx64"], 3, b["loss_sum"],
              b["loss_out"][1:2] if with_loss else None)
    torch.cuda.synchronize()
    N = r.shape[0]
    for name in ("r_next", "qsum"):
        assert torch.equal(b[name][N:], torch.full_like(b[name][N:], SENT)), f"{name}: guard rows overwritten"
    iv = b["idx64"][:3 * N].view(N, 3)
    assert torch.equal(iv[:, 0], idx32.long()), "idx64_out"
    assert (iv[:, 1:] == ISENT).all() and (b["idx64"][3 * N:] == ISENT).all(), "idx64_out written between its strided entries"
    assert b["loss_out"][0].item() == b["loss_out"][2].item() == np.float32(SENT), "loss_out written outside its element"


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
@pytest.mark.parametrize("D,rows", CASES)
def test_tail_against_float64(D, rows, rotation):
    N = n_rows(rows)
    gen = torch.Generator(device=DEV).manual_seed(7919 * D + N)
    r, codes, idx32, kind = tail_inputs(D, N, gen)
    c = codes[idx32.long()]

    a = tail_buffers(N, D)                      # first stage: qsum holds the sentinel and must come out as 0 + out
    run_tail(r, codes, idx32, rotation, a)
    out = a["qsum"][:N]
    assert torch.isfinite(out).all()
    assert same_bits(a["r_next"][:N], r - out), "r_next != r - out"
    if rotation:
        rk = torch.cat([ratio(out[sl], rotate_eval(r[sl].double(), c[sl].double(), torch.zeros_like(r[sl], dtype=torch.float64))[0],
                              rotate_bound(r[sl].double(), c[sl].double(), None, D)).amax(-1) for sl in chunks(N)])
        worst = {name: float(rk[kind == j].max()) for j, name in enumerate(KINDS) if bool((kind == j).any())}
        print(f"\ntail D={D} (J={D_SLOTS[D]}) N={N}: worst |error| / bound of the rotation value per row kind")
        print("  " + "  ".join(f"{k} {v:.3g}" for k, v in worst.items()))
        bad = {k: v for k, v in worst.items() if not v <= 2}
        assert not bad, f"rotation value outside the bound: {bad}"
    else:
        assert same_bits(out, torch.zeros_like(out) + ((c - r) + r)), "straight-through value != (c - r) + r"

    # loss: the double sum of exact squares of fp32 differences, then the fp32 roundings of torch's (mse + mse iw) w.  The CTAs
    # add their partial sums with atomics, so only the order of the double additions is free (and varies from run to run)
    ref = sum(float(((r[sl] - c[sl]).double() ** 2).sum()) for sl in chunks(N))

    def check_loss(b):
        ls = b["loss_sum"].item()
        assert abs(ls - ref) <= 1e-9 * ref, (ls, ref)
        mse = np.float32(ls / (N * D))
        want = np.float32(np.float32(mse + np.float32(mse * np.float32(IW))) * np.float32(W))
        got = b["loss_out"][1:2].cpu().numpy()
        assert got.view(np.int32)[0] == np.array([want]).view(np.int32)[0], (got[0], want)
    check_loss(a)

    b = tail_buffers(N, D)                      # a later stage: qsum + out onto a prefilled running sum
    prior = torch.randn(N, D, generator=gen, device=DEV)
    b["qsum"][:N] = prior
    run_tail(r, codes, idx32, rotation, b, first=0)
    assert same_bits(b["qsum"][:N], prior + out), "qsum != qsum + out"
    assert same_bits(b["r_next"], a["r_next"])
    del b, prior

    d = tail_buffers(N, D)                      # the last stage: no r_next; nothing else changes
    run_tail(r, codes, idx32, rotation, d, with_r_next=False)
    assert torch.equal(d["r_next"], torch.full_like(d["r_next"], SENT))
    assert same_bits(d["qsum"], a["qsum"]) and torch.equal(d["idx64"], a["idx64"])
    check_loss(d)
    del d

    e = tail_buffers(N, D)                      # no loss_out: loss_sum is not touched
    run_tail(r, codes, idx32, rotation, e, with_loss=False)
    assert e["loss_sum"].item() == LSENT and torch.equal(e["loss_out"], torch.full_like(e["loss_out"], SENT))
    assert same_bits(e["r_next"], a["r_next"]) and same_bits(e["qsum"], a["qsum"]) and torch.equal(e["idx64"], a["idx64"])


# ------------------------------------------------------------------------------------------------ (2) the backward
Q, K = 4, 64
GL = [0.75, -1.25, 2.5, 0.375]          # per-stage grad_loss, distinct and exact in fp32
# planted rows: (stage, rows, code as a function of the row's residual at that stage)
PLANTS = [(1, [0, 2, 4, 6], lambda r: r),            # the code equals the residual
          (2, [1, 3, 5], lambda r: -2 * r),          # an antiparallel code
          (3, [0], lambda r: -2 * r)]                # antiparallel to the few-ulp residual row 0 has left after stage 1


def stage_chain(D, N, rotation, gen):
    """x, Q codebooks of K codes and the kernel's own residuals R[0..Q-1] (R[0] = x), built stage by stage with the tail.
    Each index is the float64 arg-min over the kernel's residual, except for the planted rows (codes K - 4 ..)."""
    x = torch.randn(N, D, generator=gen, device=DEV) * torch.exp(torch.randn(N, 1, generator=gen, device=DEV))
    codes = torch.randn(Q, K, D, generator=gen, device=DEV) * (0.6 ** torch.arange(Q, device=DEV))[:, None, None]
    idx = torch.empty((N, Q), dtype=torch.int64, device=DEV)
    qsum = torch.empty_like(x)
    R = [x]
    for q in range(Q):
        r = R[q]
        k = torch.cat([torch.cdist(r[sl].double(), codes[q].double()).argmin(1) for sl in chunks(N)])
        for stage, rows, f in PLANTS:
            if stage == q:
                for j, i in enumerate(i for i in rows if i < N):
                    codes[q, K - 4 + j] = f(r[i])
                    k[i] = K - 4 + j
        idx[:, q] = k
        nxt = torch.empty_like(x) if q + 1 < Q else None
        tail_call(r, codes[q], k.int(), rotation, nxt, qsum, int(q == 0), None, 1, None, None)
        if nxt is not None:
            R.append(nxt)
    torch.cuda.synchronize()
    return x, codes, idx, R


def backward_case(D, rows, rotation):
    """The stage chain of (D, rows) and G."""
    N = n_rows(rows)
    gen = torch.Generator(device=DEV).manual_seed(104729 * D + N)
    x, codes, idx, R = stage_chain(D, N, rotation, gen)
    return x, codes, idx, R, torch.randn(N, D, generator=gen, device=DEV)


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
@pytest.mark.parametrize("D,rows", CASES)
def test_backward_against_float64(D, rows, rotation):
    from vector_quantize_pytorch_b200 import ops
    x, codes, idx, R, G = backward_case(D, rows, rotation)
    N = x.shape[0]
    gl = torch.tensor(GL, device=DEV)
    gx = raw_backward(x, codes, idx, Q, rotation, G, gl)
    assert torch.equal(gx, ops.rsimvq_backward(x, codes, idx, rotation, G, gl))
    rk = torch.cat([ratio(gx[sl], *backward_reference([r[sl] for r in R], [codes[q][idx[sl, q]] for q in range(Q)], G[sl], GL,
                                                      rotation)).amax(-1) for sl in chunks(N)])
    planted = torch.arange(N, device=DEV) < 8
    worst = {"planted": float(rk[planted].max()), "arg-min": float(rk[~planted].max()) if N > 8 else 0.0}
    print(f"\nbackward D={D} (J={D_SLOTS[D]}) N={N} {'rotation' if rotation else 'straight'}: worst |error| / bound "
          + "  ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert all(v <= 2 for v in worst.values()), worst


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
@pytest.mark.parametrize("D,rows", CASES)
def test_backward_recompute_is_bit_identical(D, rows, rotation):
    """DESIGN §4.7: the backward recomputes every r_q bit-identical to the forward's.  With grad_q NULL (G = 0) every other
    term is an exact zero, so grad_loss = one-hot(q) gives grad_x = fl(r_q - c_q), r_q the tail's own output; with grad_loss
    NULL as well grad_x is zero."""
    from vector_quantize_pytorch_b200 import ops
    x, codes, idx, R, _ = backward_case(D, rows, rotation)
    for q in range(Q):
        got = ops.rsimvq_backward(x, codes, idx, rotation, None, torch.eye(Q, device=DEV)[q].contiguous())
        want = R[q] - codes[q][idx[:, q]]
        if not torch.equal(got, want):
            bad = (got != want).any(-1).nonzero()[:, 0]
            pytest.fail(f"stage {q}: recomputed residual differs from the tail's on {bad.numel()} rows, first {int(bad[0])}")
    assert torch.equal(ops.rsimvq_backward(x, codes, idx, rotation, None, None), torch.zeros_like(x))


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
@pytest.mark.parametrize("D,rows", CASES)
def test_backward_quantize_dropout(D, rows, rotation):
    """Columns >= n_active hold -1 and are never read: the result equals a run over the active stages alone, and n_active = 0
    (which the module never runs; called directly, since an empty codes tensor may have no storage) gives +0."""
    from vector_quantize_pytorch_b200 import ops
    x, codes, idx, _, G = backward_case(D, rows, rotation)
    gl = torch.tensor(GL, device=DEV)
    for n in (1, Q - 1):
        dropped = idx.clone()
        dropped[:, n:] = -1
        got = ops.rsimvq_backward(x, codes[:n], dropped, rotation, G, gl[:n])
        want = ops.rsimvq_backward(x, codes[:n], idx[:, :n].contiguous(), rotation, G, gl[:n])
        assert same_bits(got, want), f"n_active = {n}"
    none = raw_backward(x, codes, torch.full_like(idx, -1), 0, rotation, G, gl)
    assert same_bits(none, torch.zeros_like(x)), "n_active = 0 must give +0"


# ------------------------------------------------------------------------------------------------ (3) the module
SEED = 1    # random.Random(1).randrange(0, 4) == 1: two of four stages run


def rsimvq(D, nq, K, rotation, dropout=False, seed=0):
    torch.manual_seed(seed)
    return vqb().ResidualSimVQ(dim=D, num_quantizers=nq, codebook_size=K, rotation_trick=rotation, quantize_dropout=dropout,
                               input_to_quantize_commit_loss_weight=IW, commitment_weight=W).to(DEV).train()


def replay(mod, flat, n_active, indices=None):
    """ResidualSimVQ.forward stage by stage with direct calls: ops.prepare_codebook and ops.search on the fp32 residual (or the
    given indices), then vqb_rsimvq_tail.  Returns (out, indices (N, Q), losses (Q,), residuals R[0..n_active-1], codebooks)."""
    from vector_quantize_pytorch_b200 import ops
    N, D = flat.shape
    nq = mod.num_quantizers
    books = [layer.codebook.detach().float().contiguous() for layer in mod.layers[:n_active]]
    out = torch.empty_like(flat)
    idx = torch.full((N, nq), -1, dtype=torch.int64, device=DEV)
    losses = torch.zeros((nq,), device=DEV)
    R = [flat]
    for q in range(n_active):
        layer, r = mod.layers[q], R[q]
        if indices is None:
            idx32 = ops.search(r, ops.prepare_codebook(books[q], False), books[q]).idx
        else:
            idx32 = indices[:, q].int().contiguous()
        nxt = torch.empty_like(flat) if q + 1 < n_active else None
        tail_call(r, books[q], idx32, layer.rotation_trick, nxt, out, int(q == 0), idx[:, q], nq,
                  torch.zeros((1,), dtype=torch.float64, device=DEV), losses[q:q + 1],
                  layer.input_to_quantize_commit_loss_weight, layer.commitment_weight)
        if nxt is not None:
            R.append(nxt)
    torch.cuda.synchronize()
    return out, idx, losses, R, books


PROGRAM_CASES = [(128, 4, 256, 15003, True), (40, 3, 96, 1001, False), (520, 2, 128, 4099, False)]


@pytest.mark.parametrize("grad", [True, False], ids=["grad", "no_grad"])
@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
@pytest.mark.parametrize("D,nq,K,N,dropout", PROGRAM_CASES)
def test_program_matches_direct_calls(D, nq, K, N, dropout, rotation, grad):
    """The cached program's output, indices and losses equal, bit for bit, direct stage-by-stage calls: the first forward builds
    the program, the second runs it with every per-call pointer (input, codebooks, idx64_out + 8 q, loss_out + 4 q, the
    statistics slice) patched into the frozen op array."""
    mod = rsimvq(D, nq, K, rotation, dropout)
    n_active = mod._active_layers(SEED, torch.device(DEV))
    assert (n_active < nq) == dropout
    for step in range(2):
        x = torch.randn(1, N, D, device=DEV).requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            q, ind, losses = mod(x, rand_quantize_dropout_fixed_seed=SEED)
        with torch.no_grad():
            out, idx, lo, _, _ = replay(mod, x.detach().reshape(N, D), n_active)
        assert torch.equal(ind.reshape(N, nq), idx), f"step {step}: indices"
        assert same_bits(q.detach().reshape(N, D), out), f"step {step}: quantized"
        assert same_bits(losses.detach(), lo), f"step {step}: losses"
    assert len(mod.__dict__["_plans"]) == 1


def capture_codebooks(mod):
    """The implicit codebook tensor each layer's code_transform produces in a forward, with its gradient retained."""
    got = {}

    def hook(i):
        def f(module, inp, out):
            if out.requires_grad:
                out.retain_grad()
            got[i] = out
        return f
    handles = [layer.code_transform.register_forward_hook(hook(i)) for i, layer in enumerate(mod.layers)]
    return got, handles


def check_module(mod, x, G, Lw, seed=None):
    """Forward and backward of (q * G).sum() + (losses * Lw).sum() (a term left out when G or Lw is None), checked against
    float64 on the kernels' own residuals (direct tail calls with the module's indices, which reproduce the forward bit for bit):
    every index is the float64 arg-min of its residual outside 1e-5 near ties; grad_x, every active codebook's gradient (from the
    search statistics) and its code_transform's within per-element bounds; dropped layers get no gradient.  Returns the worst
    |error| / bound of (grad_x, codebooks, transforms) and the number of near-tie rows."""
    nq = mod.num_quantizers
    N, D = x.shape[0] * x.shape[1], x.shape[2]
    caught, handles = capture_codebooks(mod)
    xr = x.detach().clone().requires_grad_(True)
    try:
        q, ind, losses = mod(xr, rand_quantize_dropout_fixed_seed=seed)
    finally:
        for h in handles:
            h.remove()
    total = 0.
    if G is not None:
        total = total + (q * G).sum()
    if Lw is not None:
        total = total + (losses * Lw).sum()
    total.backward()
    assert torch.isfinite(q).all() and torch.isfinite(losses).all() and torch.isfinite(xr.grad).all()
    n = mod._active_layers(seed, torch.device(DEV))
    idx = ind.reshape(N, nq)
    assert (idx[:, n:] == -1).all() and (idx[:, :n] >= 0).all() and (losses[n:] == 0).all()
    with torch.no_grad():
        out, _, lo, R, books = replay(mod, xr.detach().reshape(N, D), n, idx)
    assert same_bits(q.detach().reshape(N, D), out) and same_bits(losses.detach(), lo)

    near = 0
    for s in range(n):
        two = torch.cat([torch.cdist(R[s][sl].double(), books[s].double()) for sl in chunks(N)]).topk(2, largest=False)
        bad = idx[:, s] != two.indices[:, 0]
        gap = (two.values[:, 1] - two.values[:, 0]) / two.values[:, 1].clamp(min=1e-30)
        assert not (bad & (gap >= 1e-5)).any(), f"stage {s}: index differs from the float64 arg-min outside near ties"
        near += int(bad.sum())

    lw = [0.0] * n if Lw is None else [float(v) for v in Lw[:n]]
    gl = [lw[s] * 2 * IW * W / (N * D) for s in range(n)]
    Gf = None if G is None else G.reshape(N, D)
    gx = xr.grad.reshape(N, D)
    wx = max(float(ratio(gx[sl], *backward_reference([r[sl] for r in R], [books[s][idx[sl, s]] for s in range(n)],
                                                     None if Gf is None else Gf[sl], gl, mod.layers[0].rotation_trick)).max())
             for sl in chunks(N))
    wc = wt = 0.0
    for s in range(n):
        Kq = books[s].shape[0]
        C64, r64, k = books[s].double(), R[s].double(), idx[:, s]
        count = torch.bincount(k, minlength=Kq).double()[:, None]
        S = torch.zeros_like(C64).index_add_(0, k, r64)
        A = torch.zeros_like(C64).index_add_(0, k, r64.abs())
        scale = lw[s] * 2 * W / (N * D)
        refC = scale * (count * C64 - S)
        # the statistics sum each code's rows in fp32 in any order: the longest addition chain is the code's row count
        bC = abs(scale) * (count + 4) * EPS32 * (count * C64.abs() + A) + 4 * EPS32 * refC.abs()
        wc = max(wc, float(ratio(caught[s].grad, refC, bC).max()))
        F64 = mod.layers[s].frozen_codebook.double()
        refW = refC.t() @ F64
        bW = bC.t() @ F64.abs() + (Kq + 2) * EPS32 * (refC.abs().t() @ F64.abs())
        wt = max(wt, float(ratio(mod.layers[s].code_transform.weight.grad, refW, bW).max()))
    for s in range(n, nq):
        assert mod.layers[s].code_transform.weight.grad is None, f"dropped layer {s} got a gradient"
    return (wx, wc, wt), near


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
def test_quantize_dropout_at_size(rotation):
    D, nq, K, N = 128, 4, 256, 3 * 5001
    mod = rsimvq(D, nq, K, rotation, dropout=True, seed=4)
    x = torch.randn(3, N // 3, D, device=DEV)
    G = torch.randn_like(x)
    Lw = torch.rand(nq, device=DEV) + 0.5
    assert mod._active_layers(SEED, torch.device(DEV)) == 2
    worst, near = check_module(mod, x, G, Lw, SEED)
    print(f"\ndropout D={D} N={N}: worst |error| / bound grad_x {worst[0]:.3g} codebooks {worst[1]:.3g} "
          f"transforms {worst[2]:.3g}; near-tie rows {near}")
    assert all(v <= 2 for v in worst) and near <= max(4, N // 1000), (worst, near)


@pytest.mark.parametrize("half", ["losses", "output"])
@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
def test_backward_through_one_output(rotation, half):
    """losses.sum().backward() and (q * G).sum().backward(): each matches its half of the float64 gradient (the unused output's
    gradient reaches the backward as zeros)."""
    D, nq, K, N = 200, 3, 160, 4099
    mod = rsimvq(D, nq, K, rotation, seed=5)
    x = torch.randn(1, N, D, device=DEV)
    G = torch.randn_like(x) if half == "output" else None
    Lw = torch.ones(nq, device=DEV) if half == "losses" else None
    worst, near = check_module(mod, x, G, Lw)
    print(f"\n{half} only: worst |error| / bound grad_x {worst[0]:.3g} codebooks {worst[1]:.3g} transforms {worst[2]:.3g}")
    assert all(v <= 2 for v in worst) and near <= 4, (worst, near)


@pytest.mark.parametrize("rotation", [True, False], ids=["rotation", "straight"])
def test_rows_on_stage0_codes(rotation):
    """Rows that sit exactly on a stage-0 code, so that stage 1 on sees residuals of a few ulps (rotation: lambda = ||c|| / 1e-6)
    or exact zeros (straight-through); every fourth row is a plain random row."""
    D, nq, K, N = 128, 4, 256, 4099
    mod = rsimvq(D, nq, K, rotation, seed=6)
    gen = torch.Generator(device=DEV).manual_seed(6)
    with torch.no_grad():
        x = mod.layers[0].codebook.detach()[torch.randint(0, K, (N,), generator=gen, device=DEV)]
        x[::4] = torch.randn(x[::4].shape, generator=gen, device=DEV) * 0.3
    x = x[None].contiguous()
    G = torch.randn(x.shape, generator=gen, device=DEV)
    Lw = torch.rand(nq, generator=gen, device=DEV) + 0.5
    worst, near = check_module(mod, x, G, Lw)
    print(f"\nrows on codes: worst |error| / bound grad_x {worst[0]:.3g} codebooks {worst[1]:.3g} transforms {worst[2]:.3g}; "
          f"near-tie rows {near}")
    assert all(v <= 2 for v in worst), worst
