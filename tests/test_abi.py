"""CPU-side checks of the drop-in boundary: the C-ABI library builds/loads without a GPU and exports
every symbol include/vqb200.h declares; argument errors are reported through return codes; the Python
host layer fails loudly instead of falling back to a CPU path."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    text = open(os.path.join(ROOT, "include", "vqb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vqb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from vector_quantize_pytorch_b200 import _C
    names = declared_functions()
    assert len(names) >= 14
    lib = ctypes.CDLL(_C.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/vqb200.h but not exported"
        assert n in _C.SIGNATURES, f"{n} has no ctypes signature in _C.py"
    assert _C.lib.vqb_version() == 100


def test_host_only_entry_points():
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    assert lib.vqb_padded_codes(1024) == 1024
    assert lib.vqb_padded_codes(1000) == 1024
    assert lib.vqb_padded_codes(5) == 16
    assert lib.vqb_padded_codes(96) == 96
    assert lib.vqb_stats_offset(5) == 8 and lib.vqb_stats_floats(5, 8) == 48
    assert lib.vqb_ema_stats_workspace(1000, 64) > 1000 * 4
    assert b"ok" in lib.vqb_strerror(0)
    assert b"aligned" in lib.vqb_strerror(-3)


def test_argument_errors_are_return_codes_not_crashes():
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    assert lib.vqb_codebook_prepare(None, 10, 8, 0, None, None, None, None, None, None) == -1
    assert lib.vqb_assign(None, 1, 10, 8, None, None, None, 4, 0.0, 0, None, None, None, None, None, None) == -1
    assert lib.vqb_gather(None, 0, 1, 8, None, None, None, None, 1, None, None, None, None, None) == -1
    assert lib.vqb_ema_stats(None, 0, 1, 8, None, 4, None, None, 0, None) == -1
    assert lib.vqb_decode(None, 0, 1, 1, 8, None, 1, None, 0, None) == -1
    # D > 1024 (the longest row a warp keeps in registers) is rejected before any CUDA call
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced
    assert lib.vqb_codebook_prepare(p, 10, 1032, 0, p, p, p, p, p, None) == -2
    assert lib.vqb_ema_apply_weighted(p, p, p, p, 10, 1032, 0.8, 1e-5, 0, 1, 1, None, p, p, p, p, p, p, None) == -2


def test_fsq_argument_errors_are_return_codes_not_crashes():
    """vqb_fsq_forward / _backward / _decode refuse, before any CUDA call, more than 64 stages, d > 16, null pointers, unknown
    dtypes, an fp32 input with a bf16 chain (torch would promote it) and an unaligned z or decode output."""
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced
    f, b = _C.DTYPE_F32, _C.DTYPE_BF16

    def fwd(z=p, in_dt=f, w_dt=f, D=4, Q=2, n_active=2, consts=p, out=p, idx=p):
        return lib.vqb_fsq_forward(z, in_dt, w_dt, 8, 1, D, Q, n_active, 1, 1, consts, None, None, out, idx, 1, Q, 0, 1, None)

    def bwd(z=p, in_dt=f, w_dt=f, D=4, Q=2, n_active=2, consts=p, gout=p, gz=p):
        return lib.vqb_fsq_backward(z, in_dt, w_dt, 8, 1, D, Q, n_active, 1, 1, consts, None, None, gout, gz, None)

    def dec(idx=p, D=4, Q=2, w_dt=f, consts=p, ints=p, out=p, codes=None):
        return lib.vqb_fsq_decode(idx, 1, Q, 0, 1, 8, 1, D, Q, w_dt, 1, consts, ints, None, out, codes, None)

    for call in (fwd, bwd):
        assert call(Q=65, n_active=65) == -2
        assert call(D=17) == -2
        assert call(z=None) == -1 and call(consts=None) == -1
        assert call(n_active=0) == -1 and call(n_active=3) == -1
        assert call(in_dt=7) == -1 and call(w_dt=7) == -1
        assert call(w_dt=b) == -2
        assert call(z=p + 4) == -3
    assert fwd(out=None) == -1 and fwd(idx=None) == -1
    assert bwd(gout=None) == -1 and bwd(gz=None) == -1
    assert dec(Q=65) == -2 and dec(D=17) == -2
    assert dec(idx=None) == -1 and dec(consts=None) == -1 and dec(ints=None) == -1 and dec(out=None) == -1
    assert dec(w_dt=7) == -1
    assert dec(out=p + 4) == -3 and dec(out=None, codes=p + 4) == -3


def test_struct_layout_is_pinned():
    """The ctypes mirrors have the layout of include/vqb200.h (the library static_asserts the same sizes); fields that no
    longer select anything keep their place."""
    from vector_quantize_pytorch_b200 import _C
    assert ctypes.sizeof(_C.VQForwardArgs) == 328
    assert ctypes.sizeof(_C.FusedOutputs) == 104
    assert ctypes.sizeof(_C.RvqOp) == 808
    offsets = {(_C.VQForwardArgs, "stats_mode"): 180, (_C.VQForwardArgs, "stats_accumulate"): 184,
               (_C.VQForwardArgs, "row_mask"): 312, (_C.VQForwardArgs, "n_live"): 320, (_C.VQForwardArgs, "qsum"): 160,
               (_C.FusedOutputs, "qsum"): 64, (_C.FusedOutputs, "stats_cnt"): 72, (_C.FusedOutputs, "stats_sum"): 80, (_C.FusedOutputs, "planes_out"): 96}
    for (cls, field), off in offsets.items():
        assert getattr(cls, field).offset == off, (cls.__name__, field)


def test_retired_statistics_options_are_rejected():
    """Statistics always come from the counting sort: a call that asks the search tail to accumulate them, or asks
    vqb_vq_forward to add onto `stats`, is refused before any CUDA call instead of being ignored."""
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced
    a = _C.VQForwardArgs(x=p, dtype=_C.DTYPE_BF16, N=1024, D=64, K=64, cluster_size=p, embed_avg=p, embed=p, planes=p,
                         bext=p, bias=p, cnorm2=p, cmax=p, scratch=p, idx32=p, update=1, stats_mode=1,
                         stats_accumulate=1, stats=p, workspace=p, workspace_bytes=1 << 30)
    assert lib.vqb_vq_forward(ctypes.byref(a), None) == -2
    for field in ("stats_cnt", "stats_sum"):
        f = _C.FusedOutputs(x_eff=p, embed=p, q_out=p, dtype=_C.DTYPE_BF16, **{field: p})
        assert lib.vqb_assign(p, 1, 1024, 64, p, p, p, 64, 0.0, 0, p, p, p, None, ctypes.byref(f), None) == -2


def test_retired_running_sum_is_rejected():
    """ResidualVQ rebuilds quantized_out from the indices (vqb_rvq_accumulate): a non-NULL `qsum` — the running sum the
    stage tail used to add into — is refused before any CUDA call by every entry point that takes one."""
    from vector_quantize_pytorch_b200 import _C
    lib = _C.lib
    p = 0x10000   # non-null, 16-byte aligned; never dereferenced
    a = _C.VQForwardArgs(x=p, dtype=_C.DTYPE_BF16, N=1024, D=64, K=64, embed=p, planes=p, bext=p, bias=p, cnorm2=p, cmax=p,
                         scratch=p, idx64_out=p, idx_stride=1, resid_out=p, qsum=p, idx32=p, workspace=p,
                         workspace_bytes=1 << 30)
    assert lib.vqb_vq_forward(ctypes.byref(a), None) == -2
    op = _C.RvqOp(kind=_C.RVQ_STAGE, lane=0)
    op.stage = a
    assert lib.vqb_rvq_forward(ctypes.byref(op), 1, None) == -2
    f = _C.FusedOutputs(x_eff=p, embed=p, resid_out=p, qsum=p, dtype=_C.DTYPE_BF16)
    assert lib.vqb_assign(p, 1, 1024, 64, p, p, p, 64, 0.0, 0, p, p, p, None, ctypes.byref(f), None) == -2
    assert lib.vqb_gather(p, _C.DTYPE_BF16, 1024, 64, p, p, None, p, 1, None, None, p, p, None) == -2


def test_no_cpu_fallback():
    import vector_quantize_pytorch_b200 as m
    vq = m.VectorQuantize(dim=64, codebook_size=32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        vq(torch.randn(1, 8, 64))
    rvq = m.ResidualVQ(dim=32, num_quantizers=2, codebook_size=16)
    with pytest.raises(RuntimeError, match="no CPU path"):
        rvq(torch.randn(1, 8, 32))
    from vector_quantize_pytorch_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.prepare_codebook(torch.randn(16, 8), False)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "vector_quantize_pytorch_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("the oracle", ""), fn


def test_state_dict_layout_matches_reference():
    """SURVEY 5: buffer names/shapes/dtypes must match so reference checkpoints load."""
    import vector_quantize_pytorch_b200 as m
    sd = m.VectorQuantize(dim=64, codebook_size=32).state_dict()
    assert list(sd) == ["_codebook.initted", "_codebook.cluster_size", "_codebook.embed_avg", "_codebook.embed"]
    assert sd["_codebook.cluster_size"].shape == (1, 32) and sd["_codebook.embed"].shape == (1, 32, 64)
    assert sd["_codebook.initted"].dtype == torch.bool and bool(sd["_codebook.initted"])
    assert torch.equal(sd["_codebook.cluster_size"], torch.ones(1, 32))
    assert torch.equal(sd["_codebook.embed"], sd["_codebook.embed_avg"])
    rvq = m.ResidualVQ(dim=32, num_quantizers=3, codebook_size=16, shared_codebook=True)
    keys = list(rvq.state_dict())
    assert "layers.0._codebook.embed" in keys and "layers.2._codebook.embed" in keys
    assert rvq.layers[0]._codebook is rvq.layers[2]._codebook
    g = m.GroupedResidualVQ(dim=64, groups=2, num_quantizers=2, codebook_size=16)
    assert "rvqs.1.layers.1._codebook.cluster_size" in g.state_dict()


def test_reference_state_dict_loads(tmp_path):
    """The reference's state_dict (keys and initial buffers under seed 0, tests/golden/state_dict/reference_init.npz, written by
    `oracle/gen_golden.py --state-dicts`) must equal ours key-for-key and load into ours."""
    import json
    import numpy as np
    from oracle.gen_golden import STATE_DICT_BUILDS
    import vector_quantize_pytorch_b200 as m
    z = np.load(os.path.join(ROOT, "tests", "golden", "state_dict", "reference_init.npz"))
    keys = json.loads(z["keys"].tobytes().decode())
    assert len(keys) == len(STATE_DICT_BUILDS)
    for i, build in enumerate(STATE_DICT_BUILDS):
        sa = {k: torch.from_numpy(z[f"m{i}_{j}"]) for j, k in enumerate(keys[i])}
        torch.manual_seed(0)
        b = build(m)
        sb = b.state_dict()
        assert list(sa) == list(sb)
        for k in sa:  # same RNG consumption at construction -> identical initial codebooks
            assert torch.equal(sa[k], sb[k]), k
        b.load_state_dict(sa)


def test_unsupported_options_raise():
    import vector_quantize_pytorch_b200 as m
    for kw in (dict(learnable_codebook=True), dict(stochastic_sample_codes=True),
               dict(orthogonal_reg_weight=1.0), dict(affine_param=True)):
        with pytest.raises(NotImplementedError):
            m.VectorQuantize(dim=64, codebook_size=32, **kw)
    vq = m.VectorQuantize(dim=64, codebook_size=32, kmeans_init=True, kmeans_iters=3)   # supported since round 2
    assert not bool(vq._codebook.initted) and float(vq._codebook.embed.abs().sum()) == 0.0   # vqp:383, :415
    rvq = m.ResidualVQ(dim=32, num_quantizers=2, codebook_size=16, quantize_dropout=True)   # supported since round 2
    assert rvq.quantize_dropout and not m.ResidualVQ(dim=32, num_quantizers=1, codebook_size=16, quantize_dropout=True).quantize_dropout  # rvq:253
    with pytest.raises(NotImplementedError):
        m.ResidualVQ(dim=32, num_quantizers=2, codebook_size=16, beam_size=4)
