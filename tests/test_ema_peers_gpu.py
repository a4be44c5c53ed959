"""The multi-GPU EMA update on one GPU (run on an H100: `pytest -m gpu`).

The peer kernels sum every rank's statistics with loads through pointers into the other ranks' symmetric buffers.  On one GPU
the "ranks" are distinct local buffers, and a load through a local pointer is a plain load, so the whole peer path runs here:
  * ops.ema_apply_peers over world = 1, 2, 3 buffers (statistics at a nonzero slice offset) is bit-identical to ops.ema_apply on
    the fp32 sum of the ranks' statistics in rank order, ((0 + s0) + s1) + s2 — the state, the codebook and every operand;
  * RvqProgram.ema_peers with three statistics slices (a shared codebook) is bit-identical to RvqProgram.ema on the summed slices;
  * ops.vq_forward(update=3) with world = 1 (the barrier waits on its own flag only) meets the float64 bounds of the EMA step.
"""
import ctypes
import types

import pytest
import torch

from test_ema_update_gpu import APPLY_CASES, DEV, assert_operands, assert_within, bits, ema_ref, stats_bound, w32

pytestmark = pytest.mark.gpu

OPERANDS = ("planes", "bext", "bias", "cnorm2", "cmax")
SLICE_OFFSET = 4 * 37          # floats in front of this codebook's statistics in every rank's buffer
CASES = list(dict.fromkeys(c[:4] for c in APPLY_CASES))   # D, K, cosine, code weight


def make_peer(world):
    """A stand-in for dist.PeerReducer: rank 0 of `world`, with zeroed barrier flags and epoch on this GPU."""
    flags = torch.zeros((64,), dtype=torch.int32, device=DEV)
    return types.SimpleNamespace(world=world, rank=0, flags=flags, flag_ptrs=(ctypes.c_void_p * 1)(flags.data_ptr()),
                                 epoch=torch.zeros((1,), dtype=torch.int32, device=DEV), device=torch.device(DEV))


def rank_buffers(world, floats, gen):
    """One buffer per rank: junk in front of the slice and behind it, random statistics inside."""
    bufs = []
    for _ in range(world):
        b = torch.randn(SLICE_OFFSET + floats + 8, generator=gen) * 1e3
        bufs.append(b.to(DEV))
    return bufs


def fill_stats(buf, K, D, gen, at=SLICE_OFFSET):
    from vector_quantize_pytorch_b200 import ops
    off = ops.stats_offset(K)
    cnt = torch.randint(0, 60, (K,), generator=gen).float()
    cnt[::7] = 0
    es = cnt[:, None] * torch.randn(K, D, generator=gen) + cnt.sqrt()[:, None] * torch.randn(K, D, generator=gen)
    buf[at:at + K] = cnt.to(DEV)
    buf[at + off:at + off + K * D] = es.reshape(-1).to(DEV)


def rank_sum(bufs, lo, hi):
    """The fp32 sum over ranks in rank order, starting from zero, as the peer kernels add them."""
    acc = torch.zeros(hi - lo, dtype=torch.float32, device=DEV)
    for b in bufs:
        acc = acc + b[lo:hi]
    return acc


def codebook_state(K, D, cosine, gen):
    from vector_quantize_pytorch_b200 import ops
    c0 = torch.randn(K, D, generator=gen)
    if cosine:
        c0 = torch.nn.functional.normalize(c0, dim=-1)
    embed0 = (10.0 * c0).to(DEV)
    cs0 = (torch.rand(K, generator=gen) * 20 + 0.5).to(DEV)
    ea0 = (c0.to(DEV) * cs0[:, None]).contiguous()
    return cs0, ea0, embed0, ops.prepare_codebook(embed0, cosine)


def copy_operands(cb):
    from vector_quantize_pytorch_b200 import ops
    return ops.CodebookOperands(**{f: getattr(cb, f).clone() for f in OPERANDS + ("scratch",)}, K=cb.K, D=cb.D, cosine=cb.cosine)


def assert_same(got, ref, what):
    for name, a, b in zip(("cluster_size", "embed_avg", "embed"), got[:3], ref[:3]):
        assert torch.equal(bits(a), bits(b)), f"{what}: {name} differs"
    for f in OPERANDS:
        assert torch.equal(bits(getattr(got[3], f)), bits(getattr(ref[3], f))), f"{what}: {f} differs"


@pytest.mark.parametrize("do_normalise", [True, False], ids=["normalise", "lerp"])
@pytest.mark.parametrize("D,K,cosine,weight", CASES)
def test_ema_apply_peers_matches_local(D, K, cosine, weight, do_normalise):
    from vector_quantize_pytorch_b200 import ops
    decay, eps = 0.8, 1e-5
    floats = ops.stats_floats(K, D)
    for world in (1, 2, 3):
        gen = torch.Generator().manual_seed(D * 1009 + K + world)
        cs0, ea0, embed0, cb0 = codebook_state(K, D, cosine, gen)
        bufs = rank_buffers(world, floats, gen)
        for b in bufs:
            fill_stats(b, K, D, gen)
        cw = None
        if weight == "zeros":
            cw = torch.rand(K, generator=gen).to(DEV)
            cw[::3] = 0.0
        ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in bufs])
        peer = make_peer(world)
        got = (cs0.clone(), ea0.clone(), embed0.clone(), copy_operands(cb0))
        ops.ema_apply_peers(*got[:3], peer, ptrs, SLICE_OFFSET, got[3], decay=decay, eps=eps, do_normalise=do_normalise,
                            code_weight=cw)
        summed = rank_sum(bufs, SLICE_OFFSET, SLICE_OFFSET + floats)
        ref = (cs0.clone(), ea0.clone(), embed0.clone(), copy_operands(cb0))
        ops.ema_apply(*ref[:3], summed, ref[3], decay=decay, eps=eps, do_lerp=True, do_normalise=do_normalise, code_weight=cw)
        torch.cuda.synchronize()
        assert_same(got, ref, f"world={world}")
        assert not torch.equal(got[1], ea0)


@pytest.mark.parametrize("D,K,cosine", [(64, 250, False), (640, 300, True)])
def test_rvq_ema_peers_matches_ema(D, K, cosine):
    from vector_quantize_pytorch_b200 import ops
    decay, eps, n_lerp, world = 0.8, 1e-5, 3, 3
    floats = ops.stats_floats(K, D)
    stride = (floats + 7) // 4 * 4        # slices of the stages of a shared codebook, 4-aligned and apart
    gen = torch.Generator().manual_seed(D + K)
    cs0, ea0, embed0, cb0 = codebook_state(K, D, cosine, gen)
    bufs = []
    for _ in range(world):
        b = torch.randn(SLICE_OFFSET + n_lerp * stride + 8, generator=gen).to(DEV) * 1e3
        for j in range(n_lerp):
            fill_stats(b, K, D, gen, at=SLICE_OFFSET + j * stride)
        bufs.append(b)
    ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in bufs])
    got = (cs0.clone(), ea0.clone(), embed0.clone(), copy_operands(cb0))
    prog = ops.RvqProgram(DEV)
    prog.ema_peers(0, *got[:3], make_peer(world), ptrs, SLICE_OFFSET, got[3], decay=decay, eps=eps, do_normalise=True,
                   n_lerp=n_lerp, slice_stride=stride)
    prog.run()
    summed = rank_sum(bufs, SLICE_OFFSET, SLICE_OFFSET + n_lerp * stride)
    ref = (cs0.clone(), ea0.clone(), embed0.clone(), copy_operands(cb0))
    prog = ops.RvqProgram(DEV)
    prog.ema(0, *ref[:3], summed, ref[3], decay=decay, eps=eps, do_lerp=True, do_normalise=True, n_lerp=n_lerp,
             slice_stride=stride)
    prog.run()
    torch.cuda.synchronize()
    assert_same(got, ref, f"D={D} K={K} n_lerp={n_lerp}")


def test_vq_forward_peer_update_on_one_rank():
    from vector_quantize_pytorch_b200 import ops
    D, K, N, decay, eps = 256, 512, 65536, 0.8, 1e-5
    gen = torch.Generator().manual_seed(N + K + 1)
    c = torch.randn(K, D, generator=gen).to(DEV)
    x = torch.randn(N, D, generator=gen).to(torch.bfloat16).to(DEV)
    cs0 = (torch.rand(K, generator=gen) * 20 + 0.5).to(DEV)
    ea0 = (c * cs0[:, None]).contiguous()
    cb = ops.prepare_codebook(c, False)
    state = (cs0.clone(), ea0.clone(), c.clone())
    buf = torch.full((SLICE_OFFSET + ops.stats_floats(K, D) + 8,), -7.0, device=DEV)
    peer = make_peer(1)
    ptrs = (ctypes.c_void_p * 1)(buf.data_ptr())
    idx32, _ = ops.vq_forward(x, cb, state, update=3, do_normalise=True, decay=decay, eps=eps,
                              stats=buf[SLICE_OFFSET:SLICE_OFFSET + ops.stats_floats(K, D)], peer=peer, peer_ptrs=ptrs,
                              peer_slice_offset=SLICE_OFFSET)
    torch.cuda.synchronize()
    assert peer.epoch.item() == 2   # one barrier per EMA launch group
    idx = idx32.long()
    (cs_r, ecs), (ea_r, eea), (e_r, ee) = ema_ref(cs0.double(), ea0.double(), [stats_bound("bf16", D, K, N, idx, x.float())],
                                                  w32(decay, None, K), K, eps, False)
    cs, ea, emb = state
    assert_within(cs, cs_r, ecs, "cluster_size")
    assert_within(ea, ea_r, eea, "embed_avg")
    assert_within(emb, e_r, ee, "embed")
    assert_operands(cb, emb.clone(), False, "vq_forward update=3")
