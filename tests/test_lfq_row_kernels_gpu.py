"""The LFQ row kernels (vqb_lfq_forward, vqb_lfq_backward, vqb_lfq_decode) called directly, every output inside sentinel
guards, against the same-dtype torch chain (`oracle/lfq_oracle.py::chain`) and the float64 reference with per-element bounds
(`chain_reference`, `check_rows`): the sign rule for the indices, bounds for the output, the entropy input, the commitment
partials block by block and the gradient.  Each case prints its excused rows and its largest error / bound ratios."""
import itertools
import math

import pytest
import torch

from oracle import lfq_oracle as O
from vector_quantize_pytorch_b200 import _C
from vector_quantize_pytorch_b200.lfq import code_magnitude

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 3
SENT_F = 7.0e30
SENT_I = -77
E_INVALID = -1
DS = [1, 2, 7, 16, 20]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(shape, dtype, fill):
    """A tensor of `shape` inside a larger one: GUARD sentinel rows before and after (first axis) -> (inner view, whole)."""
    whole = torch.full((shape[0] + 2 * GUARD, *shape[1:]), fill, dtype=dtype, device=DEV)
    return whole[GUARD:GUARD + shape[0]], whole


def _guards_intact(whole, fill):
    g = torch.cat([whole[:GUARD].flatten(), whole[-GUARD:].flatten()])
    return bool((g == fill).all())


def _params(Q, d, spherical, clamp, pow2=False, pow2_clamp=True):
    """Per-stage scale, magnitude and soft clamp; clamp is "all", "some" (even stages) or "none", of about 1.75 * 0.6^q.
    With pow2_clamp the clamp values are rounded to powers of two, as the modules' halving clamps are for a power-of-two
    soft_clamp_input_value: on CUDA torch divides by a Python scalar as a multiply by its reciprocal, which equals the
    kernel's correctly rounded division only then, and the exact comparisons with the torch chain need the same operations.
    Where the bounds alone decide (spherical training) the clamps are not powers of two."""
    s = [2.0 ** -q if pow2 else 0.8 * 0.55 ** q for q in range(Q)]
    m = [code_magnitude(v, d, spherical) for v in s]
    c = [1.75 * 0.6 ** q if clamp == "all" or (clamp == "some" and q % 2 == 0) else 0. for q in range(Q)]
    if pow2_clamp:
        c = [2.0 ** round(math.log2(v)) if v else 0. for v in c]
    return torch.tensor([s, m, c], dtype=torch.float32, device=DEV)


def _dt(z):
    return _C.DTYPE_BF16 if z.dtype == torch.bfloat16 else _C.DTYPE_F32


def forward(z, params, Q, na, residual, training, sph, rowmask=None, want_ent=True, want_commit=True):
    """vqb_lfq_forward with guarded outputs and a strided int64 index view inside a sentinel-filled tensor.
    -> (out, indices (N, G, Q), entropy input or None, commitment partials (na, blocks) or None, blocks)."""
    N, G, d = z.shape
    out, out_w = _guarded((N, G, d), z.dtype, SENT_F)
    idx_w = torch.full((N + 2 * GUARD, G, Q + 2), SENT_I, dtype=torch.int64, device=DEV)   # 2 spare columns per row
    idx = idx_w[GUARD:GUARD + N, :, 1:1 + Q]
    ent, ent_w = _guarded((na, N, G, d), torch.float32, SENT_F) if want_ent else (None, None)
    blocks = _C.lib.vqb_lfq_forward_blocks(N, G)
    assert blocks > 0
    com, com_w = _guarded((na, blocks), torch.float64, SENT_F) if want_commit else (None, None)
    rc = _C.lib.vqb_lfq_forward(z.data_ptr(), _dt(z), N, G, d, Q, na, int(residual), int(training), int(sph), params.data_ptr(),
                                out.data_ptr(), idx.data_ptr(), idx.stride(0), idx.stride(1), idx.stride(2),
                                ent.data_ptr() if ent is not None else None, rowmask.data_ptr() if rowmask is not None else None,
                                com.data_ptr() if com is not None else None, blocks, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(out_w, SENT_F)
    spare = torch.cat([idx_w[:GUARD].flatten(), idx_w[-GUARD:].flatten(), idx_w[:, :, 0].flatten(), idx_w[:, :, -1].flatten()])
    assert bool((spare == SENT_I).all())
    if ent is not None:
        assert _guards_intact(ent_w, SENT_F)
    if com is not None:
        assert _guards_intact(com_w, SENT_F)
    return out, idx, ent, com, blocks


def backward(z, params, Q, na, residual, training, sph, gout, gent=None, cc=None, rowmask=None):
    N, G, d = z.shape
    gz, gz_w = _guarded((N, G, d), z.dtype, SENT_F)
    rc = _C.lib.vqb_lfq_backward(z.data_ptr(), _dt(z), N, G, d, Q, na, int(residual), int(training), int(sph), params.data_ptr(),
                                 gout.data_ptr(), gent.data_ptr() if gent is not None else None,
                                 cc.data_ptr() if cc is not None else None, rowmask.data_ptr() if rowmask is not None else None,
                                 gz.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert _guards_intact(gz_w, SENT_F)
    return gz


def _report(label, rep, n_active):
    r = " ".join(f"{k} {v:.3g}" for k, v in rep.ratios.items())
    first = int(rep.first_excused.min()) if rep.excused else n_active
    print(f"[lfq-rows] {label}: excused {rep.excused} (first at stage {first}) | {r}")


def run_case(z, params, Q, na, residual, training, sph, rowmask, label, gent_cc=((True, True),), outputs=((True, True),),
             gen=None, max_excused=0, min_excused_stage=None):
    """Every output of one configuration: the forward once per (entropy input, commitment) request, which must not change
    the output or the indices, the backward once per (gent, cc) presence, all under the sign rule and the bounds.  At most
    `max_excused` items may be excused, none before stage `min_excused_stage`."""
    N, G, d = z.shape
    ro, it, xt, _ = O.chain(z, params, Q, na, residual, training, sph)
    runs = [forward(z, params, Q, na, residual, training, sph, rowmask, e, c) for e, c in outputs]
    out, idx, ent, com, blocks = runs[0]
    ent = next((r[2] for r in runs if r[2] is not None), None)
    com = next((r[3] for r in runs if r[3] is not None), None)
    for r in runs[1:]:
        assert torch.equal(r[0], out) and torch.equal(r[1], idx)
    gout = torch.randn(z.shape, generator=gen, device=DEV).to(z.dtype)
    gent_all = torch.randn((na, N, G, d), generator=gen, device=DEV) * 0.3
    cc_all = torch.linspace(0.3, 0.9, Q, device=DEV)
    worst = None
    for with_gent, with_cc in gent_cc:
        gent = gent_all if with_gent else None
        cc = cc_all if with_cc else None
        gz = backward(z, params, Q, na, residual, training, sph, gout, gent, cc, rowmask)
        ref = O.chain_reference(z, params, Q, na, residual, training, sph, gout, gent, cc, rowmask, signs=xt > 0)
        rep = O.check_rows(ref, na, it, xt, idx, out, ent, com, blocks, rowmask, gz, sph, params)
        _report(f"{label} gent={int(with_gent)} cc={int(with_cc)}", rep, na)
        assert not rep.violations, (label, rep.violations)
        assert rep.excused <= max_excused, (label, rep.excused)
        if rep.excused:
            assert int(rep.first_excused.min()) >= min_excused_stage, label
        if not sph or not training:   # exactly reproducible arithmetic: every bit and every value as the torch chain
            assert rep.excused == 0
            assert torch.equal(idx, it) and torch.equal(out, ro)
        if not sph and ent is not None:
            assert torch.equal(ent, xt.float())
        if not training and not with_gent:   # eval: only the commitment term reaches z, and never on a masked row
            if not with_cc:
                assert bool((gz == 0).all())
            elif rowmask is not None:
                assert bool((gz[rowmask == 0] == 0).all())
        worst = rep
    return worst


# ---- every path: dtype x residual x training x spherical x clamp x rowmask x (gent, cc) x (ent, commit) ----

@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("sph", [False, True], ids=["plain", "sph"])
@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_every_path(bf, sph, training):
    dtype = torch.bfloat16 if bf else torch.float32
    gen = torch.Generator(device=DEV).manual_seed(1000 * bf + 100 * sph + training)
    both = list(itertools.product([False, True], repeat=2))
    for k, (residual, clamp, mask) in enumerate(itertools.product([True, False], ["all", "some", "none"], ["none", "part", "zero"])):
        d, G = DS[k % len(DS)], (1, 3)[(k // len(DS)) % 2]
        Q, na = (4, 4 - k % 2) if residual else (1, 1)   # without the residual the kernels run one stage (LFQ)
        N = 211 + 17 * k
        z = (torch.randn((N, G, d), generator=gen, device=DEV) * 1.5).to(dtype)
        rowmask = None if mask == "none" else \
            (torch.rand(N, generator=gen, device=DEV) > 0.3).to(torch.uint8) if mask == "part" else \
            torch.zeros(N, dtype=torch.uint8, device=DEV)
        params = _params(Q, d, sph, clamp, pow2_clamp=not (sph and training))
        run_case(z, params, Q, na, residual, training, sph, rowmask,
                 f"{'bf16' if bf else 'f32'} d{d} G{G} q{na}/{Q} res{int(residual)} train{int(training)} sph{int(sph)} "
                 f"clamp={clamp} mask={mask}", gent_cc=both, outputs=both, gen=gen)


@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_every_d(bf):
    dtype = torch.bfloat16 if bf else torch.float32
    gen = torch.Generator(device=DEV).manual_seed(7 + bf)
    for d in range(1, 21):
        sph, training = d % 2 == 0, d % 3 != 0
        z = (torch.randn((157, 2, d), generator=gen, device=DEV) * 1.5).to(dtype)
        rowmask = (torch.rand(157, generator=gen, device=DEV) > 0.25).to(torch.uint8)
        run_case(z, _params(3, d, sph, "some", pow2_clamp=not (sph and training)), 3, 3, True, training, sph, rowmask,
                 f"{'bf16' if bf else 'f32'} d{d} sph{int(sph)} train{int(training)}", gen=gen)


# ---- depth: 64 stages, spherical included ----

@pytest.mark.parametrize("na", [50, 64])
@pytest.mark.parametrize("sph", [False, True], ids=["plain", "sph"])
@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_64_stages(bf, sph, na):
    dtype = torch.bfloat16 if bf else torch.float32
    gen = torch.Generator(device=DEV).manual_seed(na + 2 * sph + bf)
    d = 6 if na == 50 else 9
    z = (torch.randn((301, 2, d), generator=gen, device=DEV) * 1.5).to(dtype)
    rowmask = (torch.rand(301, generator=gen, device=DEV) > 0.25).to(torch.uint8)
    for training in (True, False):
        # an fp32 spherical training chain's late residuals are at the level of its rounding (0.55^q against 2^-24), and
        # their signs with them: those items may be excused, from stage 16 on and at most two thirds of them.  Every other
        # chain excuses none.
        deep = sph and training and not bf
        run_case(z, _params(64, d, sph, "some", pow2_clamp=not (sph and training)), 64, na, True, training, sph, rowmask,
                 f"{'bf16' if bf else 'f32'} d{d} q{na}/64 sph{int(sph)} train{int(training)}", gen=gen,
                 max_excused=2 * z.shape[0] * z.shape[1] // 3 if deep else 0, min_excused_stage=16)


# ---- more than one grid wave, G > 1: the commitment partials block by block, and determinism ----

@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("sph", [False, True], ids=["plain", "sph"])
@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_waves(bf, sph, training):
    dtype = torch.bfloat16 if bf else torch.float32
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    G, d, Q = 3, 5, 3
    N = (2 * sms * 8 * 256) // G + 4099           # more than two full waves of the capped grid, and a ragged remainder
    gen = torch.Generator(device=DEV).manual_seed(31 + 4 * bf + 2 * sph + training)
    z = (torch.randn((N, G, d), generator=gen, device=DEV) * 1.5).to(dtype)
    rowmask = (torch.rand(N, generator=gen, device=DEV) > 0.25).to(torch.uint8)
    params = _params(Q, d, sph, "some", pow2_clamp=not (sph and training))
    assert _C.lib.vqb_lfq_forward_blocks(N, G) == sms * 8
    rep = run_case(z, params, Q, Q, True, training, sph, rowmask,
                   f"waves {'bf16' if bf else 'f32'} N{N} G{G} sph{int(sph)} train{int(training)}", gen=gen)
    assert rep is not None
    # two runs give identical bits: the commitment partials (fixed-order block sums) and the backward
    a = forward(z, params, Q, Q, True, training, sph, rowmask)
    b = forward(z, params, Q, Q, True, training, sph, rowmask)
    assert all(torch.equal(x, y) for x, y in zip(a[:4], b[:4]))
    gout = torch.randn(z.shape, generator=gen, device=DEV).to(dtype)
    gent = torch.randn((Q, N, G, d), generator=gen, device=DEV)
    cc = torch.linspace(0.3, 0.9, Q, device=DEV)
    assert torch.equal(backward(z, params, Q, Q, True, training, sph, gout, gent, cc, rowmask),
                       backward(z, params, Q, Q, True, training, sph, gout, gent, cc, rowmask))


# ---- planted rows ----

def _planted(dtype, d, m0, sph):
    """Rows at the edges of the chain: signed zeros, the smallest subnormal and normal, subnormals, the largest finite value,
    values next to and at the stage-0 magnitude (the next residual is exactly 0 or one ulp), tanh-saturating values, and for
    a spherical chain norms of 0, inside (0, eps), exactly eps and on either side of it.  -> (rows (R, d), finite-rows mask)."""
    fi = torch.finfo(dtype)
    tiny_sub = float(torch.tensor(fi.tiny, dtype=dtype) / 2 ** (7 if dtype == torch.bfloat16 else 23))
    m = float(torch.tensor(m0, dtype=dtype))
    up = float(torch.nextafter(torch.tensor(m, dtype=dtype), torch.tensor(2.0, dtype=dtype)))
    eps = O.l2norm_eps(dtype == torch.bfloat16)
    vals = [0., -0., tiny_sub, -tiny_sub, fi.tiny, -fi.tiny, 3 * tiny_sub, -5 * tiny_sub, m, -m, up, -up, 60., -60., 1e4]
    if sph:
        vals += [1e18, -1e18, eps, 3e-13, 2 * eps, eps / 2]
    else:
        vals += [fi.max, -fi.max]
    rows = [torch.full((d,), v) for v in vals]
    one = [torch.zeros(d) for _ in range(len(vals))]   # the same values alone in an otherwise zero row
    for r, v in zip(one, vals):
        r[d // 2] = v
    if sph:
        rows.append(torch.full((d,), 3e-13 / d ** 0.5))     # ||x|| = 3e-13 < eps
        rows.append(torch.tensor([eps] + [0.] * (d - 1)))   # ||x|| = eps exactly: fp32 sqrt(eps^2) = eps, as in float64
    z = torch.stack(rows + one).to(dtype)
    return z


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("sph", [False, True], ids=["plain", "sph"])
@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_planted_rows(bf, sph, training):
    dtype = torch.bfloat16 if bf else torch.float32
    gen = torch.Generator(device=DEV).manual_seed(5)
    for d, clamp in ((1, "none"), (4, "some"), (13, "all")):
        Q = 3
        params = _params(Q, d, sph, clamp, pow2_clamp=not (sph and training))
        z = _planted(dtype, d, float(params[0, 0]) if clamp == "none" else 0.5, sph)
        N = z.shape[0]
        z = z.view(N, 1, d).to(DEV)
        # rows holding the largest finite value are masked: their fp32 commitment square overflows, as torch's would
        rowmask = ((torch.arange(N, device=DEV) % 3 != 1) & (z.float().abs().amax((1, 2)) < 1e30)).to(torch.uint8)
        run_case(z, params, Q, Q, True, training, sph, rowmask,
                 f"planted {'bf16' if bf else 'f32'} d{d} clamp={clamp} sph{int(sph)} train{int(training)}",
                 gent_cc=((True, True), (False, False)), gen=gen)


@pytest.mark.parametrize("bf", [False, True], ids=["f32", "bf16"])
def test_nonfinite_rows_match_the_torch_chain(bf):
    """+-inf and NaN on the non-spherical paths: every index, output and entropy input as the torch chain (NaN > 0 is
    false: bit 0)."""
    dtype = torch.bfloat16 if bf else torch.float32
    inf, nan = float("inf"), float("nan")
    for d, clamp in ((3, "none"), (5, "all")):
        rows = [[inf] * d, [-inf] * d, [nan] * d, [inf, nan] + [1.] * (d - 2), [-inf] + [0.5] * (d - 1)]
        z = torch.tensor(rows, dtype=torch.float32).to(dtype).view(len(rows), 1, d).to(DEV)
        params = _params(3, d, False, clamp)
        for training in (True, False):
            out, idx, ent, _, _ = forward(z, params, 3, 3, True, training, False)
            ro, ri, rx, _ = O.chain(z, params, 3, 3, True, training, False)
            assert torch.equal(idx, ri)
            assert torch.equal(out.float().nan_to_num(nan=7.), ro.float().nan_to_num(nan=7.))
            assert torch.equal(ent.nan_to_num(nan=7.), rx.float().nan_to_num(nan=7.))
            assert int(idx[2, 0, 0]) == 0   # NaN row: no bit set


# ---- decode ----

def _decode(ind, d, vals, itype, want_out, want_codes, stride0_g=False):
    """vqb_lfq_decode on a strided (row, stage, group) view inside a sentinel-filled tensor; with stride0_g the size-1 group
    axis has stride 0."""
    N, G, Q = ind.shape
    whole = torch.full((N + 2 * GUARD, Q + 3, G), SENT_I, dtype=itype, device=DEV)
    view = whole[GUARD:GUARD + N, 1:1 + Q].permute(0, 2, 1)
    view.copy_(ind)
    if stride0_g:
        assert G == 1
        s_g = 0
    else:
        s_g = view.stride(1)
    out, out_w = _guarded((N, G, d), torch.float32, SENT_F) if want_out else (None, None)
    codes, codes_w = _guarded((Q * N, G, d), torch.float32, SENT_F) if want_codes else (None, None)
    rc = _C.lib.vqb_lfq_decode(view.data_ptr(), int(itype == torch.int64), view.stride(0), s_g, view.stride(2), N, G, d, Q,
                               vals.data_ptr(), out.data_ptr() if out is not None else None,
                               codes.data_ptr() if codes is not None else None, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(whole[:GUARD], torch.full_like(whole[:GUARD], SENT_I))
    assert torch.equal(whole[-GUARD:], torch.full_like(whole[-GUARD:], SENT_I))
    assert bool((whole[:, 0] == SENT_I).all()) and bool((whole[:, -2:] == SENT_I).all())
    if out is not None:
        assert _guards_intact(out_w, SENT_F)
    if codes is not None:
        assert _guards_intact(codes_w, SENT_F)
        codes = codes.view(Q, N, G, d)
    return out, codes


def _decode_ref(ind, d, vals, want_codes=True):
    """The codes (Q, N, G, d) (or None) and their fp32 sum over the stages in stage order; -1 gives 0."""
    sh = torch.arange(d - 1, -1, -1, device=ind.device)
    codes = []
    acc = torch.zeros((*ind.shape[:2], d), dtype=torch.float32, device=ind.device)
    for q in range(ind.shape[2]):
        iq = ind[..., q, None]
        c = torch.where(iq == -1, 0., torch.where(((iq >> sh) & 1) == 1, vals[q], -vals[q])).float()
        acc = acc + c
        if want_codes:
            codes.append(c)
    return (torch.stack(codes) if want_codes else None), acc


@pytest.mark.parametrize("d", list(range(1, 21)))
def test_decode_every_d(d):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator(device=DEV).manual_seed(d)
    Q = (1, 7, 64)[d % 3]
    G = 2
    N = (sms * 8 * 256) // G + 333 if d % 4 == 0 else 257            # past one grid wave on every fourth d
    ind = torch.randint(0, 1 << d, (N, G, Q), generator=gen, device=DEV)
    ind[torch.rand((N, G, Q), generator=gen, device=DEV) < 0.1] = -1
    ind[0], ind[1], ind[2] = 0, (1 << d) - 1, -1
    vals = (torch.rand(Q, generator=gen, device=DEV) + 0.1) * torch.where(torch.arange(Q, device=DEV) % 5 == 4, -1., 1.)
    big = N * G * Q * d > (1 << 27)   # the codes of a many-wave, 64-stage case would be gigabytes: the sum covers those
    codes_ref, out_ref = _decode_ref(ind, d, vals, not big)
    modes = [(True, False)] if big else [(True, False), (False, True), (True, True)]
    for itype, (want_out, want_codes) in itertools.product([torch.int32, torch.int64], modes):
        out, codes = _decode(ind, d, vals, itype, want_out, want_codes)
        if want_out:
            assert torch.equal(out, out_ref)
        if want_codes:
            assert torch.equal(codes, codes_ref)


@pytest.mark.parametrize("itype", [torch.int32, torch.int64], ids=["i32", "i64"])
def test_decode_stride0_group_axis(itype):
    gen = torch.Generator(device=DEV).manual_seed(3)
    N, Q, d = 999, 5, 11
    ind = torch.randint(-1, 1 << d, (N, 1, Q), generator=gen, device=DEV)
    vals = torch.tensor([1.0, 0.5, 0.3, 0.25, 0.125], device=DEV)
    codes_ref, out_ref = _decode_ref(ind, d, vals)
    out, codes = _decode(ind, d, vals, itype, True, True, stride0_g=True)
    assert torch.equal(out, out_ref) and torch.equal(codes, codes_ref)


@pytest.mark.parametrize("na", [24, 17])
def test_round_trip_forward_decode(na):
    """fp32, power-of-two scales, Q <= 24, non-spherical eval: the forward's output equals the decode of its own indices bit
    for bit (every partial sum is exact)."""
    gen = torch.Generator(device=DEV).manual_seed(na)
    Q, G = 24, 2
    for d in (1, 8, 20):
        z = torch.randn((500, G, d), generator=gen, device=DEV) * 1.5
        params = _params(Q, d, False, "none", pow2=True)
        out, idx, _, _, _ = forward(z, params, Q, na, True, False, False, want_ent=False, want_commit=False)
        dec, _ = _decode(idx, d, params[1].contiguous(), torch.int64, True, False)
        assert torch.equal(out, dec)


# ---- offsets past 2^31 elements ----

BIG_N, BIG_D = 110_000_000, 20


def _free_enough(nbytes):
    free, _ = torch.cuda.mem_get_info()
    return free > nbytes + (2 << 30)


def _big_rows():
    """Items around element 2^31 and the last items."""
    b = (1 << 31) // BIG_D
    return torch.cat([torch.arange(b - 64, b + 64), torch.arange(BIG_N - 64, BIG_N)]).to(DEV)


def test_forward_past_2_31_elements():
    """bf16 eval forward, d = 20, N = 1.1e8 (2.2e9 elements): the rows around element 2^31 and the last rows against the
    torch chain, exactly."""
    need = BIG_N * BIG_D * 2 * 2 + BIG_N * 2 * 8
    if not _free_enough(need):
        pytest.skip("needs ~10 GiB of free device memory")
    try:
        gen = torch.Generator(device=DEV).manual_seed(2)
        z = torch.randn((BIG_N, 1, BIG_D), generator=gen, device=DEV, dtype=torch.bfloat16)
        params = _params(2, BIG_D, False, "some")
        out = torch.empty_like(z)
        idx = torch.empty((BIG_N, 1, 2), dtype=torch.int64, device=DEV)
        rc = _C.lib.vqb_lfq_forward(z.data_ptr(), _C.DTYPE_BF16, BIG_N, 1, BIG_D, 2, 2, 1, 0, 0, params.data_ptr(), out.data_ptr(),
                                    idx.data_ptr(), idx.stride(0), idx.stride(1), idx.stride(2), None, None, None, 0, _stream())
        assert rc == 0
        torch.cuda.synchronize()
        rows = _big_rows()
        ro, ri, _, _ = O.chain(z[rows], params, 2, 2, True, False, False)
        assert torch.equal(out[rows], ro) and torch.equal(idx[rows], ri)
    finally:
        z = out = idx = None
        torch.cuda.empty_cache()


def test_decode_past_2_31_elements():
    need = BIG_N * BIG_D * 4 + BIG_N * 4
    if not _free_enough(need):
        pytest.skip("needs ~9 GiB of free device memory")
    try:
        gen = torch.Generator(device=DEV).manual_seed(4)
        ind = torch.randint(-1, 1 << BIG_D, (BIG_N, 1, 1), generator=gen, device=DEV, dtype=torch.int32)
        vals = torch.tensor([0.75], device=DEV)
        out = torch.full((BIG_N, 1, BIG_D), SENT_F, device=DEV)
        rc = _C.lib.vqb_lfq_decode(ind.data_ptr(), 0, 1, 1, 1, BIG_N, 1, BIG_D, 1, vals.data_ptr(), out.data_ptr(), None,
                                   _stream())
        assert rc == 0
        torch.cuda.synchronize()
        rows = _big_rows()
        _, ref = _decode_ref(ind[rows].long(), BIG_D, vals, False)
        assert torch.equal(out[rows], ref)
    finally:
        ind = out = None
        torch.cuda.empty_cache()


# ---- refusals after the device check ----

def test_commit_blocks_must_be_the_grid():
    N, G, d, Q = 5000, 2, 4, 2
    z = torch.randn((N, G, d), device=DEV)
    params = _params(Q, d, False, "none")
    out = torch.empty_like(z)
    idx = torch.empty((N, G, Q), dtype=torch.int64, device=DEV)
    blocks = _C.lib.vqb_lfq_forward_blocks(N, G)
    com = torch.full((Q, blocks + 1), SENT_F, dtype=torch.float64, device=DEV)
    for wrong in (blocks - 1, blocks + 1):
        rc = _C.lib.vqb_lfq_forward(z.data_ptr(), _C.DTYPE_F32, N, G, d, Q, Q, 1, 1, 0, params.data_ptr(), out.data_ptr(),
                                    idx.data_ptr(), idx.stride(0), idx.stride(1), idx.stride(2), None, None, com.data_ptr(), wrong,
                                    _stream())
        assert rc == E_INVALID
    torch.cuda.synchronize()
    assert bool((com == SENT_F).all())
