"""`ops.Scratch`, the search scratch of one owner (no GPU needed): reuse and growth, and that it never travels with a copy or a
pickle of its owner."""
import copy
import pickle

import torch


def test_scratch_reuses_grows_and_follows_the_device():
    from vector_quantize_pytorch_b200.ops import Scratch
    s = Scratch()
    idx, ws = s.take(4000, 10000, torch.device("cpu"))
    assert idx.dtype == ws.dtype == torch.uint8 and idx.numel() >= 4000 and ws.numel() >= 10000
    for n_idx, n_ws in ((4000, 10000), (400, 100), (0, 0)):   # equal and smaller sizes: the same buffers
        i2, w2 = s.take(n_idx, n_ws, torch.device("cpu"))
        assert i2 is idx and w2 is ws
    i3, w3 = s.take(4000, 10001, torch.device("cpu"))   # a larger workspace: it grows, the index buffer stays
    assert i3 is idx and w3 is not ws and w3.numel() >= 10001
    i4, w4 = s.take(4001, 10001, torch.device("cpu"))
    assert i4 is not idx and i4.numel() >= 4001 and w4 is w3
    i5, w5 = s.take(16, 16, torch.device("meta"))   # another device: both reallocated there, even though they are big enough
    assert i5.device.type == w5.device.type == "meta" and s.idx is i5 and s.ws is w5


def test_scratch_is_never_copied_or_pickled():
    from vector_quantize_pytorch_b200.ops import Scratch
    s = Scratch()
    s.take(1 << 20, 1 << 20, torch.device("cpu"))
    for dup in (copy.deepcopy(s), pickle.loads(pickle.dumps(s))):
        assert isinstance(dup, Scratch) and dup.idx is None and dup.ws is None
    assert s.idx is not None and s.ws is not None


def test_modules_copy_without_their_scratch():
    """deepcopy / pickle of a module starts every codebook (and every head view) with an empty scratch, and the scratch is no
    part of the state_dict."""
    import vector_quantize_pytorch_b200 as m
    torch.manual_seed(0)
    mods = [m.VectorQuantize(dim=32, codebook_size=16),
            m.VectorQuantize(dim=32, codebook_size=16, heads=2, separate_codebook_per_head=True),
            m.ResidualVQ(dim=32, num_quantizers=3, codebook_size=16),
            m.ResidualVQ(dim=32, num_quantizers=3, codebook_size=16, shared_codebook=True)]
    for mod in mods:
        keys = list(mod.state_dict())
        books = [mod._codebook] if hasattr(mod, "_codebook") else [layer._codebook for layer in mod.layers]
        cb = books[0]
        if cb.num_codebooks > 1:
            books += [cb.head(i) for i in range(cb.num_codebooks)]
        assert len({id(b._scratch) for b in books}) == len({id(b) for b in books}), "codebooks share a scratch"
        for b in books:
            b._scratch.take(4096, 4096, torch.device("cpu"))
        for dup in (copy.deepcopy(mod), pickle.loads(pickle.dumps(mod))):
            assert list(dup.state_dict()) == keys
            dup_books = [dup._codebook] if hasattr(dup, "_codebook") else [layer._codebook for layer in dup.layers]
            dup_books += dup_books[0]._head_views or []
            for b in dup_books:
                assert b._scratch.idx is None and b._scratch.ws is None
        assert all(b._scratch.ws is not None for b in books)
