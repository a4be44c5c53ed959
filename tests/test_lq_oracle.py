"""LatentQuantize on the CPU: the numpy oracle (oracle/lq_oracle.py) against the reference's fixtures (tests/golden/lq/,
oracle/gen_golden_lq.py), seeded state_dict parity, loading the reference's state_dicts, the refusals and the C ABI's
argument errors."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lq_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "lq")
FIXTURES = sorted(p[:-4] for p in os.listdir(GOLDEN) if p.endswith(".npz"))


def load(name):
    f = np.load(os.path.join(GOLDEN, name + ".npz"))
    return f, json.loads(bytes(f["meta"]).decode())


def seeded(m, meta):
    torch.manual_seed(meta["seed"])
    return m.LatentQuantize(**meta["kw"])


def tables(f):
    return [f[k] for k in sorted((k for k in f.files if k.startswith("table_")), key=lambda k: int(k[6:]))]


def test_fixtures_exist():
    assert {"readme_image", "readme_video", "readme_series", "readme_2d", "codebooks4", "int_levels", "no_optimize",
            "noproj_3cb", "bf16_noproj", "weights_zero_c", "weights_zero_both", "nondyadic", "unsorted",
            "levels_2p24"} <= set(FIXTURES)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_fixture(name):
    """Indices bit for bit from the reference's z; without projections the output is the oracle's codes bit for bit; the loss
    lies within the float64 bound widened by the reference's own fp32 sum; the eval step gives the same indices and a zero
    loss."""
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    lq = seeded(m, meta)
    C, D = lq.num_codebooks, lq.codebook_dim
    z = f["z"].reshape(-1, C, D)
    codes, idx = O.quantize(z, tables(f), lq._levels.numpy(), lq._basis.numpy())
    ind = f["indices"]
    np.testing.assert_array_equal(idx.reshape(ind.shape), ind)
    np.testing.assert_array_equal(f["eval_indices"], ind)
    x = f["x"]
    x_rows = np.moveaxis(x, 1, -1).reshape(-1)
    out_rows = np.moveaxis(f["out"], 1, -1).reshape(-1)
    if not lq.has_projections:
        np.testing.assert_array_equal(out_rows, codes.reshape(-1))
    kw = meta["kw"]
    wc, wq = kw.get("commitment_loss_weight", 0.1), kw.get("quantization_loss_weight", 0.1)
    l64, bound = O.loss64(x_rows, out_rows, wc, wq, wc != 0, wq != 0)
    n = x_rows.size
    slack = (abs(wc) + abs(wq)) * np.mean((x_rows.astype(np.float64) - out_rows) ** 2) * np.log2(n) * 2.0 ** -23
    assert abs(float(f["loss"]) - l64) <= bound + slack
    assert float(f["eval_loss"]) == 0.0


@pytest.mark.parametrize("name", ["readme_image", "codebooks4", "int_levels", "noproj_3cb", "nondyadic", "levels_2p24"])
def test_decode_matches_oracle(name):
    """indices_to_codes(project_out=False) is the fixed lattice, and with dyadic tables, no projection and moderate |z| it gives
    the forward's output back (not for 7 levels, whose linspace values are off the lattice, nor above 2^24, where the fp32
    index rounds)."""
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    lq = seeded(m, meta)
    ind = torch.from_numpy(f["indices"])
    codes = lq.indices_to_codes(ind, project_out=False).numpy()
    ref = O.decode(f["indices"], lq._levels.numpy(), lq._basis.numpy())
    if lq.keep_num_codebooks_dim:
        ref = ref.reshape(*ref.shape[:-2], -1)
    np.testing.assert_array_equal(codes, np.moveaxis(ref, -1, 1))
    if name == "noproj_3cb":
        np.testing.assert_array_equal(codes, f["out"])


def test_oracle_quirks():
    """The cases the reference's fp32 arithmetic decides: first minimum at exact midpoints and duplicates, the code at huge |z|
    (z + (q - z) = 0 while q = -0.5), sums above 2^24 rounded before the truncation, and a linspace value just below its
    lattice point truncating to the index below."""
    lv, basis = [7], [1]
    t = [torch.linspace(-0.5, 0.5, 7).numpy()]
    assert t[0][3] != 0.0
    codes, idx = O.quantize(np.float32([[[1e8]]]), t, lv, basis)
    assert codes[0, 0, 0] == 0.0 and idx[0, 0] == 3
    mid = np.float32((np.float64(t[0][1]) + t[0][2]) / 2)
    codes, _ = O.quantize(np.float32([[[mid]]]), t, lv, basis)
    assert codes[0, 0, 0] in (t[0][1], t[0][2])
    dup = [np.float32([0.25, -0.5, 0.25])]
    _, idx = O.quantize(np.float32([[[0.3]]]), dup, [3], [1])
    assert idx[0, 0] == int(np.float32(0.25) * 2 * 1 + 1)
    big = [np.arange(256, dtype=np.float32) / 256 - 0.5] * 2 + [np.linspace(-0.5, 0.5, 257).astype(np.float32)]
    z = np.float32([[[255 / 256 - 0.5, 255 / 256 - 0.5, 0.5]]])
    _, idx = O.quantize(z, big, [256, 256, 257], [1, 256, 65536])
    assert idx[0, 0] == np.float32(65535 + 256 * 65536) and idx[0, 0] != 65535 + 256 * 65536


@pytest.mark.parametrize("name", FIXTURES)
def test_seeded_state_dict_matches_reference(name):
    import vector_quantize_pytorch_b200 as m
    f, meta = load(name)
    sd = seeded(m, meta).state_dict()
    assert list(sd) == json.loads(str(f["sd_keys"]))
    for j, (k, v) in enumerate(sd.items()):
        assert v.dtype == torch.from_numpy(f[f"sd_{j}"]).dtype, k
        np.testing.assert_array_equal(v.numpy(), f[f"sd_{j}"], err_msg=k)


def test_buffers_match_reference_layout():
    import vector_quantize_pytorch_b200 as m
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=16)
    assert [n for n, _ in lq.named_buffers()] == ["commitment_loss_weight", "quantization_loss_weight", "_levels", "_basis",
                                                  "implicit_codebook"]
    # torch.cumprod promotes the int32 levels: the reference's basis is int64
    assert lq._levels.dtype == torch.int32 and lq._basis.dtype == torch.int64 and lq._basis.tolist() == [1, 5, 25]
    assert lq.implicit_codebook.shape == (200, 3) and lq.implicit_codebook.dtype == torch.float32
    assert lq.codebook_size == 200 and not lq.keep_num_codebooks_dim
    assert m.LatentQuantize(levels=[5, 5, 8], dim=16, num_codebooks=2).keep_num_codebooks_dim
    plain = m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=False)
    assert isinstance(plain.values_per_latent, list) and list(plain.state_dict()) == []


def test_loads_reference_state_dict():
    import vector_quantize_pytorch_b200 as m
    f, meta = load("unsorted")
    keys = json.loads(str(f["sd_keys"]))
    torch.manual_seed(123)
    lq = m.LatentQuantize(**meta["kw"])
    lq.load_state_dict({k: torch.from_numpy(f[f"sd_{j}"]) for j, k in enumerate(keys)})
    for j, (k, v) in enumerate(lq.state_dict().items()):
        np.testing.assert_array_equal(v.numpy(), f[f"sd_{j}"], err_msg=k)
    f2, meta2 = load("readme_image")
    keys2 = json.loads(str(f2["sd_keys"]))
    lq2 = m.LatentQuantize(**meta2["kw"])
    lq2.load_state_dict({k: torch.from_numpy(f2[f"sd_{j}"]) for j, k in enumerate(keys2)})
    for j, (k, v) in enumerate(lq2.state_dict().items()):
        np.testing.assert_array_equal(v.numpy(), f2[f"sd_{j}"], err_msg=k)


def test_refusals():
    import vector_quantize_pytorch_b200 as m
    with pytest.raises(NotImplementedError, match="in_place_codebook_optimizer"):
        m.LatentQuantize(levels=[5, 5, 8], dim=16, in_place_codebook_optimizer=torch.optim.SGD)
    with pytest.raises(NotImplementedError, match="2\\^31"):
        m.LatentQuantize(levels=[65536, 32768], dim=2)
    with pytest.raises(NotImplementedError, match="shared-memory cap"):
        m.LatentQuantize(levels=[8193], dim=1)
    with pytest.raises(NotImplementedError, match="shared-memory cap"):
        m.LatentQuantize(levels=[1] * 257, dim=257)
    lq = m.LatentQuantize(levels=[5, 5, 8], dim=3)
    for dt in (torch.float16, torch.float64):
        with pytest.raises(NotImplementedError, match="float32 and bfloat16"):
            lq(torch.randn(1, 3, 4).to(dt))
    # the reference's own exceptions: an int level without codebook_dim, a wrong input width
    with pytest.raises(RuntimeError):
        m.LatentQuantize(levels=5, dim=16)
    with pytest.raises(AssertionError, match="expected dimension of 3"):
        lq(torch.randn(1, 4, 4))


VQB_E_INVALID, VQB_E_UNSUPPORTED, VQB_E_ALIGN = -1, -2, -3


def test_abi_errors_before_any_cuda_call():
    from vector_quantize_pytorch_b200._C import lib
    P = 1 << 20
    q = lib.vqb_lq_quantize
    assert q(None, 0, 4, 1, 3, P, 16, P, P, P, None) == VQB_E_INVALID
    assert q(P, 0, 4, 1, 3, None, 16, P, P, P, None) == VQB_E_INVALID
    assert q(P, 0, 4, 1, 3, P, 16, None, P, P, None) == VQB_E_INVALID
    assert q(P, 0, 4, 1, 3, P, 16, P, None, P, None) == VQB_E_INVALID
    assert q(P, 0, 4, 1, 3, P, 16, P, P, None, None) == VQB_E_INVALID
    for N, C, D, total, dt in ((0, 1, 3, 16, 0), (4, 0, 3, 16, 0), (4, 1, 0, 16, 0), (4, 1, 3, 2, 0), (4, 1, 3, 16, 2),
                               (4, 1, 3, 16, -1)):
        assert q(P, dt, N, C, D, P, total, P, P, P, None) == VQB_E_INVALID, (N, C, D, total, dt)
    assert q(P, 0, 4, 1, 257, P, 300, P, P, P, None) == VQB_E_UNSUPPORTED
    assert q(P, 0, 4, 1, 3, P, 8193, P, P, P, None) == VQB_E_UNSUPPORTED
    assert q(P, 0, 1 << 40, 1, 3, P, 16, P, P, P, None) == VQB_E_UNSUPPORTED
    assert q(P, 0, 1 << 38, 4, 3, P, 16, P, P, P, None) == VQB_E_UNSUPPORTED
    assert q(P, 0, (1 << 40) - 1, (1 << 31) - 1, 256, P, 300, P, P, P, None) == VQB_E_UNSUPPORTED   # no overflowing N C D
    assert q(P, 0, 1 << 30, (1 << 31) - 1, 2, P, 16, P, P, P, None) == VQB_E_UNSUPPORTED
    assert q(P + 2, 0, 4, 1, 3, P, 16, P, P, P, None) == VQB_E_ALIGN
    assert q(P + 1, 1, 4, 1, 3, P, 16, P, P, P, None) == VQB_E_ALIGN
    assert q(P, 0, 4, 1, 3, P + 2, 16, P, P, P, None) == VQB_E_ALIGN
    assert q(P, 0, 4, 1, 3, P, 16, P, P + 2, P, None) == VQB_E_ALIGN
    assert q(P, 0, 4, 1, 3, P, 16, P, P, P + 2, None) == VQB_E_ALIGN

    assert lib.vqb_lq_loss_blocks(0) == VQB_E_INVALID
    assert lib.vqb_lq_loss_blocks(1 << 40) == VQB_E_UNSUPPORTED
    assert lib.vqb_lq_loss_blocks(1) == 1 and lib.vqb_lq_loss_blocks(8193) == 2 and lib.vqb_lq_loss_blocks(1 << 30) == 1024
    ls = lib.vqb_lq_loss
    assert ls(None, 0, P, 16, P, P, 1, 1, P, 1, P, None) == VQB_E_INVALID
    assert ls(P, 0, P, 16, P, P, 1, 1, None, 1, P, None) == VQB_E_INVALID
    assert ls(P, 0, P, 0, P, P, 1, 1, P, 1, P, None) == VQB_E_INVALID
    assert ls(P, 0, P, 16, P, P, 2, 1, P, 1, P, None) == VQB_E_INVALID
    assert ls(P, 0, P, 16, P, P, 1, 1, P, 2, P, None) == VQB_E_INVALID
    assert ls(P, 3, P, 16, P, P, 1, 1, P, 1, P, None) == VQB_E_INVALID
    assert ls(P, 0, P, 1 << 40, P, P, 1, 1, P, 1024, P, None) == VQB_E_UNSUPPORTED
    assert ls(P, 0, P, 16, P, P, 1, 1, P + 4, 1, P, None) == VQB_E_ALIGN
    assert ls(P + 2, 0, P, 16, P, P, 1, 1, P, 1, P, None) == VQB_E_ALIGN
    lb = lib.vqb_lq_loss_backward
    assert lb(P, 0, P, 16, P, P, P, 1, 1, None, None, None) == VQB_E_INVALID
    assert lb(P, 0, P, 16, None, P, P, 1, 1, P, P, None) == VQB_E_INVALID
    assert lb(P, 0, P, 16, P, P, P, 1, -1, P, P, None) == VQB_E_INVALID
    assert lb(P, 0, P, 1 << 40, P, P, P, 1, 1, P, P, None) == VQB_E_UNSUPPORTED
    assert lb(P, 1, P, 16, P, P, P, 1, 1, P + 1, P, None) == VQB_E_ALIGN
    assert lb(P, 0, P, 16, P, P, P, 1, 1, P, P + 2, None) == VQB_E_ALIGN


def test_codebook_dim_mismatch_raises_the_references_exceptions():
    """codebook_dim longer than the levels: the reference's quantize indexes past its tables (IndexError); shorter: its
    codes_to_indices fails to broadcast (RuntimeError).  Both before any device work."""
    import vector_quantize_pytorch_b200 as m
    with pytest.raises(IndexError):
        m.LatentQuantize(levels=[5, 5, 8], dim=4, codebook_dim=4)(torch.randn(1, 4, 6))
    with pytest.raises(RuntimeError):
        m.LatentQuantize(levels=[5, 5, 8], dim=2, codebook_dim=2)(torch.randn(1, 2, 6))


def test_loss_weights_follow_a_module_cast():
    """.bfloat16() / .double() cast the weight buffers: the kernels get fp32 copies of the cast values, and the loss takes the
    reference's promoted dtype."""
    import vector_quantize_pytorch_b200 as m
    for cast, dt in (("bfloat16", torch.float32), ("double", torch.float64), ("float", torch.float32)):
        lq = getattr(m.LatentQuantize(levels=[5, 5, 8], dim=3, optimize_values=False), cast)()
        wc, wq, loss_dtype = lq._loss_weights()
        assert wc.dtype == wq.dtype == torch.float32 and loss_dtype == dt
        assert wc.item() == lq.commitment_loss_weight.float().item()


def test_loss_ops_refuse_other_operand_dtypes():
    from vector_quantize_pytorch_b200 import ops
    x, out = torch.zeros(8), torch.zeros(8)
    w = torch.tensor(0.1)
    for args in ((x, out, w.bfloat16(), w), (x, out, w, w.double()), (x, out.bfloat16(), w, w), (x.half(), out, w, w)):
        with pytest.raises(TypeError):
            ops.lq_loss(*args, True, True)
        with pytest.raises(TypeError):
            ops.lq_loss_backward(*args[:2], w, *args[2:], True, True)
    with pytest.raises(ValueError):
        ops.lq_loss(x, torch.zeros(9), w, w, True, True)
    with pytest.raises(ValueError):
        ops.lq_loss(x, out, torch.zeros(2), w, True, True)
