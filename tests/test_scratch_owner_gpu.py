"""Whoever freezes a pointer owns the memory behind it (run on an H100: `pytest -m gpu`).

(a) every cached program — ResidualVQ, GroupedResidualVQ, ResidualSimVQ — holds the search scratch (index row and workspace) its
    stage ops point into, even after calls that needed more scratch (training after eval, more rows), and the parallel lanes of a
    grouped program share no scratch;
(b) deleting a module returns all the device memory its forwards took, its codebooks' scratch and its plans' included.
"""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (training, rows per batch element) of each forward: an eval plan is cached first, then training needs more workspace (the
# statistics), then more rows need more of everything, then the eval plan is replayed
SCHEDULE = [(False, 700), (True, 700), (True, 1400), (False, 700)]

PLAN_CASES = {
    "rvq_separate_fp32": (dict(num_quantizers=4), torch.float32),
    "rvq_shared_fp32": (dict(num_quantizers=4, shared_codebook=True), torch.float32),
    "rvq_separate_bf16": (dict(num_quantizers=4), torch.bfloat16),
    "rvq_shared_bf16": (dict(num_quantizers=4, shared_codebook=True), torch.bfloat16),
    "grvq_fp32": (dict(num_quantizers=3, groups=2), torch.float32),
    "rsimvq": (dict(num_quantizers=3), torch.float32),
}


def vqb():
    import vector_quantize_pytorch_b200 as m
    return m


def _held(plan):
    """{storage start: end} of every tensor reachable from a cached plan through lists, tuples, dicts and the attributes of the
    package's own objects.  Modules are not entered: the plan itself must hold what its ops point into."""
    held, seen, todo = {}, set(), [plan]
    while todo:
        o = todo.pop()
        if id(o) in seen or isinstance(o, torch.nn.Module):
            continue
        seen.add(id(o))
        if isinstance(o, torch.Tensor):
            st = o.untyped_storage()
            held[st.data_ptr()] = st.data_ptr() + st.nbytes()
        elif isinstance(o, dict):
            todo += list(o.values())
        elif isinstance(o, (list, tuple)):
            todo += list(o)
        elif type(o).__module__.startswith("vector_quantize_pytorch_b200") and hasattr(o, "__dict__"):
            todo += list(vars(o).values())
    return held


def _check_plans(owner):
    """Every stage op's idx32 and workspace lie inside a tensor its plan holds; lanes share none.  Returns the lane counts."""
    from vector_quantize_pytorch_b200 import _C
    plans = owner.__dict__.get("_plans") or {}
    assert plans, "no program ran"
    n_lanes = []
    for key, plan in plans.items():
        prog = plan[0] if isinstance(plan, tuple) else plan.prog
        held = _held(plan)
        lanes = {}
        for i in range(prog.n):
            op = prog.arr[i]
            if op.kind != _C.RVQ_STAGE:
                continue
            for what, ptr, nbytes in (("idx32", op.stage.idx32, 4 * op.stage.N),
                                      ("workspace", op.stage.workspace, op.stage.workspace_bytes)):
                inside = [s for s, e in held.items() if s <= ptr and ptr + nbytes <= e]
                assert inside, f"plan {key}: op {i} ({what}) points into memory the plan does not hold"
                lanes.setdefault(op.lane, set()).update(inside)
        bufs = list(lanes.values())
        for a in range(len(bufs)):
            for b in range(a + 1, len(bufs)):
                assert not bufs[a] & bufs[b], f"plan {key}: two lanes share a scratch buffer"
        n_lanes.append(len(lanes))
    return n_lanes


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_cached_programs_hold_their_scratch(case):
    m = vqb()
    kw, dt = PLAN_CASES[case]
    torch.manual_seed(21)
    if case == "rsimvq":
        mod = m.ResidualSimVQ(dim=64, codebook_size=128, **kw)
    elif case.startswith("grvq"):
        mod = m.GroupedResidualVQ(dim=128, codebook_size=96, **kw)
    else:
        mod = m.ResidualVQ(dim=64, codebook_size=200, **kw)
    mod = mod.to(DEV)
    width = 128 if case.startswith("grvq") else 64
    for training, rows in SCHEDULE:
        mod.train(training)
        x = torch.randn(3, rows, width, device=DEV).to(dt)
        # ResidualSimVQ: training with gradient-carrying codebooks makes its stages produce statistics (a larger workspace)
        with torch.set_grad_enabled(training and case == "rsimvq"):
            mod(x)
    torch.cuda.synchronize()
    n_lanes = _check_plans(mod)
    assert all(n == (2 if case.startswith("grvq") else 1) for n in n_lanes), n_lanes


LEAK_CASES = {
    "vq": (lambda m: m.VectorQuantize(dim=64, codebook_size=128), {}),
    "vq_heads2_separate": (lambda m: m.VectorQuantize(dim=64, codebook_size=128, heads=2, separate_codebook_per_head=True), {}),
    "rvq_stagewise_dropout": (lambda m: m.ResidualVQ(dim=64, num_quantizers=4, codebook_size=128, quantize_dropout=True),
                              dict(rand_quantize_dropout_fixed_seed=1)),
    "rvq_program": (lambda m: m.ResidualVQ(dim=64, num_quantizers=4, codebook_size=128), {}),
}


@pytest.mark.parametrize("case", list(LEAK_CASES))
def test_deleting_a_module_frees_its_scratch(case):
    m = vqb()
    make, call = LEAK_CASES[case]
    torch.manual_seed(22)

    def run(mod):
        with torch.no_grad():
            for rows in (700, 1400):
                mod(torch.randn(2, rows, 64, device=DEV), **call)
        return bool(mod.__dict__.get("_plans"))

    # the first calls of a kind allocate library workspaces that live on (cuBLAS, for project_in): a twin takes them before
    # the baseline, and stays alive so that no object id of the measured module can be one of its
    twin = make(m).to(DEV).train()
    run(twin)
    torch.cuda.synchronize()
    gc.collect()
    base = torch.cuda.memory_allocated()
    mod = make(m).to(DEV).train()
    ran_program = run(mod)
    assert ran_program == (case == "rvq_program"), ran_program
    del mod
    torch.cuda.synchronize()
    gc.collect()
    assert torch.cuda.memory_allocated() - base <= 1 << 20, torch.cuda.memory_allocated() - base
