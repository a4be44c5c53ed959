"""ResidualVQ / GroupedResidualVQ: the one-call program, the stage-wise path and the masked path against each other, through
the public module surface only (run on an H100: `pytest -m gpu`).

(a) program == stage-wise (`VQB_RVQ_PROGRAM=0`) bit for bit in indices, quantized and losses, and in the codebook state up to
    the order of the statistics atomics: with projections, DiVeQ (noise fixed through `diveq_noise`), a frozen codebook, and a
    bf16 GroupedResidualVQ with a shared codebook in training and in eval;
(b) the multi-GPU codebook-update schedule on one GPU: `dist.PeerReducer.create` hands out a world-1 peer built on local
    buffers, whose sum over ranks is the local statistics bit for bit, so a `sync_codebook=True` module must equal a twin
    without sync on either path, over enough steps to use both parity buffers; without peer memory a GroupedResidualVQ
    forward makes exactly one `allreduce_packed` for all its groups;
(c) a masked forward == a twin's forward over the compacted rows, scattered into zeros and -1; an all-masked batch changes
    nothing, not even the RNG state;
(d) what a forward costs on each path: kernel launches, FFI calls and graph-cache events.
"""
import copy
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def _equal(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a, b), f"{what}: {(a.float() - b.float()).abs().max().item()}"


def _same_state(mod, ref, what):
    """Codebook state up to the order in which the statistics atomics add a code's rows; then `ref` takes `mod`'s state so that
    the next step starts from identical codebooks."""
    for (n, a), (_, b) in zip(mod.named_buffers(), ref.named_buffers()):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6, msg=f"{what}: {n} differs")
    for (n, a), (_, b) in zip(mod.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6, msg=f"{what}: {n} differs")
    ref.load_state_dict(mod.state_dict())


def _compare_outputs(o1, o0, what):
    for name, a, b in zip(("quantized", "indices", "losses"), o1, o0):
        _equal(a, b, f"{what}: {name}")


# ------------------------------------------------------------------------------------------------ (a) program vs stage-wise
PROGRAM_CASES = {
    "projections": dict(grouped=False, dt=torch.float32, width=96, kw=dict(codebook_dim=64)),
    "diveq_no_grad": dict(grouped=False, dt=torch.float32, width=64, kw=dict(diveq=True)),
    "diveq_no_grad_bf16": dict(grouped=False, dt=torch.bfloat16, width=64, kw=dict(diveq=True)),
    "freeze_codebook": dict(grouped=False, dt=torch.float32, width=64, kw={}, call=dict(freeze_codebook=True)),
    "grvq_shared_bf16": dict(grouped=True, dt=torch.bfloat16, width=128, kw=dict(shared_codebook=True)),
    "grvq_shared_bf16_eval": dict(grouped=True, dt=torch.bfloat16, width=128, kw=dict(shared_codebook=True), eval=True),
    # (training, rows per batch element) of each step: an eval plan is cached before training needs more scratch, and replayed
    "eval_train_rows_eval": dict(grouped=False, dt=torch.float32, width=64, kw={},
                                 schedule=[(False, 700), (True, 700), (True, 1400), (False, 700)]),
}


def _build(grouped, width, **kw):
    m = vqb()
    torch.manual_seed(11)
    if grouped:
        return m.GroupedResidualVQ(dim=width, groups=2, num_quantizers=3, codebook_size=96, **kw).to(DEV)
    return m.ResidualVQ(dim=width, num_quantizers=4, codebook_size=200, **kw).to(DEV)


@pytest.mark.parametrize("case", list(PROGRAM_CASES))
def test_program_equals_stagewise(case, monkeypatch):
    from vector_quantize_pytorch_b200 import vector_quantize as vqm
    c = PROGRAM_CASES[case]
    mod = _build(c["grouped"], c["width"], **c["kw"])
    ref = copy.deepcopy(mod)
    noise = {}
    monkeypatch.setattr(vqm, "diveq_noise", lambda like: noise["z"].to(like.dtype))
    with torch.no_grad():
        for step, (training, rows) in enumerate(c.get("schedule", [(not c.get("eval"), 700)] * 4)):
            mod.train(training), ref.train(training)
            gen = torch.Generator(device=DEV).manual_seed(100 + step)
            x = torch.randn(3, rows, c["width"], device=DEV, generator=gen).to(c["dt"])
            noise["z"] = torch.randn(3, rows, 64, device=DEV, generator=gen)
            monkeypatch.setenv("VQB_RVQ_PROGRAM", "1")
            o1 = mod(x, **c.get("call", {}))
            monkeypatch.setenv("VQB_RVQ_PROGRAM", "0")
            o0 = ref(x, **c.get("call", {}))
            torch.cuda.synchronize()
            _compare_outputs(o1, o0, f"step {step}")
            _same_state(mod, ref, f"step {step}")
    owners = mod.rvqs if c["grouped"] else [mod]
    assert len(mod.__dict__.get("_plans", {})) >= 1 or any(r.__dict__.get("_plans") for r in owners), "no program ran"


# ------------------------------------------------------------------------------------------------ (b) the peer schedule
def _world1_create(made):
    """A stand-in for dist.PeerReducer.create: a world-1 reducer on local buffers (its peer loads are plain loads)."""
    from vector_quantize_pytorch_b200 import dist

    def create(numel, device, group=None):
        numel = (int(numel) + 3) // 4 * 4
        pr = object.__new__(dist.PeerReducer)
        pr.numel, pr.device, pr.world, pr.rank = numel, torch.device(device), 1, 0
        pr.bufs = [torch.zeros((numel,), dtype=torch.float32, device=device) for _ in range(2)]
        pr.stats_ptrs = [(ctypes.c_void_p * 1)(b.data_ptr()) for b in pr.bufs]
        pr._flags = torch.zeros((64,), dtype=torch.int32, device=device)
        pr.flag_ptrs = (ctypes.c_void_p * 1)(pr._flags.data_ptr())
        pr.epoch = torch.zeros((1,), dtype=torch.int32, device=device)
        pr.step = 0
        made.append(pr)
        return pr
    return create


PEER_CASES = {
    "separate": dict(grouped=False, kw={}),
    "shared": dict(grouped=False, kw=dict(shared_codebook=True)),
    "grouped": dict(grouped=True, kw={}),
    "grouped_shared": dict(grouped=True, kw=dict(shared_codebook=True)),
}


@pytest.mark.parametrize("program", ["1", "0"])
@pytest.mark.parametrize("case", list(PEER_CASES))
def test_peer_schedule_equals_local(case, program, monkeypatch):
    from vector_quantize_pytorch_b200 import dist
    c = PEER_CASES[case]
    made = []
    monkeypatch.setattr(dist.PeerReducer, "create", staticmethod(_world1_create(made)))
    monkeypatch.setenv("VQB_RVQ_PROGRAM", program)
    width = 128 if c["grouped"] else 64
    mod = _build(c["grouped"], width, sync_codebook=True, **c["kw"])
    ref = _build(c["grouped"], width, sync_codebook=False, **c["kw"])
    ref.load_state_dict(mod.state_dict())
    with torch.no_grad():
        for step in range(5):
            x = torch.randn(2, 900, width, device=DEV)
            o1, o0 = mod(x), ref(x)
            torch.cuda.synchronize()
            _compare_outputs(o1, o0, f"step {step}")
            _same_state(mod, ref, f"step {step}")
    assert made, "no peer reducer was asked for"
    assert all(pr.step >= 4 for pr in made), [pr.step for pr in made]   # both parity buffers were used, twice each
    owners = mod.rvqs if c["grouped"] else [mod]
    assert all(r._peer is not None for r in owners)


@pytest.mark.parametrize("grouped", [False, True])
def test_no_peer_memory_one_allreduce(grouped, monkeypatch):
    m = vqb()
    from vector_quantize_pytorch_b200 import codebook, dist, residual_vq
    monkeypatch.setattr(dist.PeerReducer, "create", staticmethod(lambda numel, device, group=None: None))
    calls = []

    def counting(packed, group=None):
        calls.append(packed.numel())
        return packed
    for mod_ in (dist, residual_vq, codebook):
        if hasattr(mod_, "allreduce_packed"):
            monkeypatch.setattr(mod_, "allreduce_packed", counting)
    width = 128 if grouped else 64
    mod = _build(grouped, width, sync_codebook=True)
    ref = _build(grouped, width, sync_codebook=False)
    ref.load_state_dict(mod.state_dict())
    with torch.no_grad():
        for step in range(3):
            x = torch.randn(2, 900, width, device=DEV)
            calls.clear()
            o1 = mod(x)
            assert len(calls) == 1, f"step {step}: {len(calls)} all-reduces"
            o0 = ref(x)
            assert len(calls) == 1
            torch.cuda.synchronize()
            _compare_outputs(o1, o0, f"step {step}")
            _same_state(mod, ref, f"step {step}")
    owners = mod.rvqs if grouped else [mod]
    assert all(r._peer is None for r in owners)


# ------------------------------------------------------------------------------------------------ (c) masks
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("proj", [False, True])
def test_masked_equals_compacted(dt, proj, monkeypatch):
    m = vqb()
    torch.manual_seed(5)
    D = 64
    width = 96 if proj else D
    mod = m.ResidualVQ(dim=width, codebook_dim=D, num_quantizers=4, codebook_size=128).to(DEV).train()
    mod.project_in.to(dt), mod.project_out.to(dt)
    twin = m.ResidualVQ(dim=D, num_quantizers=4, codebook_size=128).to(DEV).train()
    twin.layers.load_state_dict(mod.layers.state_dict())
    B, N = 3, 500
    with torch.no_grad():
        for step in range(3):
            x = torch.randn(B, N, width, device=DEV).to(dt)
            mask = torch.rand(B, N, device=DEV) < 0.6
            monkeypatch.setenv("VQB_RVQ_PROGRAM", "1")
            q, idx, loss = mod(x, mask=mask)
            xp = mod.project_in(x)
            rows = mask.reshape(-1).nonzero(as_tuple=True)[0]
            qc, ic, lc = twin(xp.reshape(-1, D)[rows].unsqueeze(0))
            want_q = torch.zeros((B * N, D), dtype=xp.dtype, device=DEV)
            want_q[rows] = qc[0]
            want_i = torch.full((B * N, 4), -1, dtype=torch.int64, device=DEV)
            want_i[rows] = ic[0]
            torch.cuda.synchronize()
            _equal(idx, want_i.reshape(B, N, 4), f"step {step}: indices")
            _equal(q, mod.project_out(want_q.reshape(B, N, D)), f"step {step}: quantized")
            _equal(loss, lc, f"step {step}: losses")
            _same_state(mod.layers, twin.layers, f"step {step}")


def test_all_masked_changes_nothing():
    m = vqb()
    torch.manual_seed(6)
    mod = m.ResidualVQ(dim=64, num_quantizers=4, codebook_size=128, quantize_dropout=True).to(DEV).train()
    with torch.no_grad():
        mod(torch.randn(2, 300, 64, device=DEV), mask=torch.ones(2, 300, dtype=torch.bool, device=DEV))   # initialise
    state = copy.deepcopy(mod.state_dict())
    x = torch.randn(2, 300, 64, device=DEV)
    mask = torch.zeros(2, 300, dtype=torch.bool, device=DEV)
    cpu_rng, cuda_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    with torch.no_grad():
        q, idx, loss = mod(x, mask=mask)
    torch.cuda.synchronize()
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    _equal(q, torch.zeros_like(x), "quantized")
    _equal(idx, torch.full((2, 300, 4), -1, dtype=torch.int64, device=DEV), "indices")
    _equal(loss, torch.zeros((4,), dtype=torch.float32, device=DEV), "losses")
    for k, v in mod.state_dict().items():
        _equal(v, state[k], k)


# ------------------------------------------------------------------------------------------------ (d) cost accounting
def _cost_case(name):
    """(module, forward kwargs, input requires grad, VQB_RVQ_PROGRAM) of one cost case."""
    m = vqb()
    torch.manual_seed(3)
    rvq = dict(dim=64, num_quantizers=8, codebook_size=256)
    if name.startswith("grvq"):
        mod = m.GroupedResidualVQ(groups=2, **rvq)
    elif name == "rvq_shared_dead_code":
        mod = m.ResidualVQ(shared_codebook=True, threshold_ema_dead_code=2, **rvq)
    elif name == "rvq_dropout":
        mod = m.ResidualVQ(quantize_dropout=True, **rvq)
    else:
        mod = m.ResidualVQ(**rvq)
    mod = mod.to(DEV).train()
    if name.endswith("eval"):
        mod.eval()
    call = {}
    if name == "rvq_masked":
        call["mask"] = torch.arange(1024, device=DEV)[None] % 3 != 0
    if name == "rvq_dropout":
        call["rand_quantize_dropout_fixed_seed"] = 4
    return mod, call, name == "rvq_layered", "0" if "stagewise" in name else "1"


COST_CASES = ["rvq_program_train", "rvq_program_eval", "rvq_stagewise_train", "rvq_stagewise_eval", "rvq_layered", "rvq_masked",
              "rvq_dropout", "rvq_shared_dead_code", "grvq_program_train", "grvq_program_eval", "grvq_stagewise_train"]

# per warmed forward: (ops.LAUNCHES delta, vqb_rvq_forward calls, vqb_vq_forward calls,
#                      graph stats delta (replayed, updated, instantiated, direct)), recorded on the parent of the
# one-row-pipeline refactor of ResidualVQ
COST = {
    "rvq_program_train": (105, 1, 0, (1, 0, 0, 0)),
    "rvq_program_eval": (41, 1, 0, (1, 0, 0, 0)),
    "rvq_stagewise_train": (105, 0, 8, (8, 0, 0, 0)),
    "rvq_stagewise_eval": (41, 0, 8, (8, 0, 0, 0)),
    "rvq_layered": (112, 0, 8, (8, 0, 0, 0)),
    "rvq_masked": (105, 0, 8, (8, 0, 0, 0)),
    "rvq_dropout": (53, 0, 4, (4, 0, 0, 0)),
    "rvq_shared_dead_code": (115, 0, 8, (8, 0, 0, 0)),
    "grvq_program_train": (210, 1, 0, (1, 0, 0, 0)),
    "grvq_program_eval": (82, 1, 0, (1, 0, 0, 0)),
    "grvq_stagewise_train": (210, 0, 16, (16, 0, 0, 0)),
}


@pytest.mark.parametrize("name", COST_CASES)
def test_forward_cost(name, monkeypatch):
    from vector_quantize_pytorch_b200 import _C, ops
    mod, call, grad, program = _cost_case(name)
    monkeypatch.setenv("VQB_RVQ_PROGRAM", program)
    counts = {"vqb_rvq_forward": 0, "vqb_vq_forward": 0}
    for fn in counts:
        real = getattr(ops.lib, fn)

        def wrapped(*a, _real=real, _fn=fn):
            counts[_fn] += 1
            return _real(*a)
        monkeypatch.setattr(ops.lib, fn, wrapped)

    def graph_stats():
        out = (ctypes.c_longlong * 4)()
        assert _C.lib.vqb_debug_graph_stats(ctypes.cast(out, ctypes.c_void_p)) == 0
        return list(out)

    gen = torch.Generator(device=DEV).manual_seed(9)
    xs = [torch.randn(1, 1024, 64, device=DEV, generator=gen) for _ in range(2)]

    def forward(x):
        x = x.detach().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            out = mod(x, **call)
            if grad:
                out[0].float().sum().backward()

    stream = torch.cuda.Stream()   # graph capture is legal on a side stream (not on the legacy default stream)
    with torch.cuda.stream(stream):
        for i in range(6):
            forward(xs[i % 2])
        stream.synchronize()
        launches, g0 = ops.LAUNCHES, graph_stats()
        for fn in counts:
            counts[fn] = 0
        forward(xs[0])
        stream.synchronize()
        got = (ops.LAUNCHES - launches, counts["vqb_rvq_forward"], counts["vqb_vq_forward"],
               tuple(b - a for a, b in zip(g0, graph_stats())))
    assert got == COST.get(name), f"{name}: {got}"
