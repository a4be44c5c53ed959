"""LFQ on two GPUs (`pytest -m gpu`, skipped below 2 GPUs): one process per GPU, the batch sharded over the ranks.  Every
rank's per-sample entropy is the mean over its own rows and the batch entropy is that of the cross-rank mean of the (c, K)
averages, as the full batch gives it; the gradient at each rank's rows is float64 autograd of the sum of both ranks' losses
over the full batch (the all-reduce's backward sums the ranks' gradients of the shared mean)."""
import os
import socket
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = textwrap.dedent('''
    import os, sys
    import torch
    import torch.distributed as dist
    sys.path.insert(0, os.environ["VQB_ROOT"])
    import vector_quantize_pytorch_b200 as vqb
    from oracle import lfq_oracle as O

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    d, c, rows, tau, gamma = 8, 2, 64, 2.0, 0.7
    torch.manual_seed(0)
    mod = vqb.LFQ(codebook_size=1 << d, num_codebooks=c, entropy_loss_weight=1., diversity_gamma=gamma).to(dev).train()
    full = torch.randn(world * rows, c * d, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    x = full[rank * rows:(rank + 1) * rows].float().to(dev)[None].requires_grad_(True)
    (_, _, aux), (pse, cbe, _) = mod(x, inv_temperature=tau, return_loss_breakdown=True)
    aux.backward()
    # float64 full-batch oracle
    xf = full.reshape(world, rows, c, d).requires_grad_(True)
    pses = []
    for r in range(world):
        pses.append(sum(O.h(O.log_probs_dense(xf[r, :, g], 1.0, tau).exp()).sum() for g in range(c)) / (rows * c))
    avg = torch.stack([sum(O.log_probs_dense(xf[r, :, g], 1.0, tau).exp().sum(0) for r in range(world)) / (world * rows)
                       for g in range(c)])
    cbe64 = O.h(avg).sum(-1).mean()
    total = sum(pses) - gamma * world * cbe64
    total.backward()
    ok = abs(float(pse) - float(pses[rank])) <= 2e-5 * abs(float(pses[rank])) + 1e-7
    ok &= abs(float(cbe) - float(cbe64)) <= 2e-5 * float(cbe64)
    g64 = xf.grad[rank].reshape(rows, c * d)
    err = float((x.grad[0].double().cpu() - g64).abs().max())
    ok &= err <= 1e-4 * float(g64.abs().max())
    print(f"RESULT rank={rank} ok={ok} pse={float(pse):.7f}/{float(pses[rank]):.7f} cbe={float(cbe):.7f}/{float(cbe64):.7f} "
          f"grad_err={err:.3e}", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)
''')


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_lfq_two_ranks_equal_full_batch_oracle(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, VQB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    out = res.stdout + res.stderr
    assert res.returncode == 0, out[-4000:]
    assert out.count("ok=True") == 2, out[-2000:]
