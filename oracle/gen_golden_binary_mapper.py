"""Generate tests/golden/binary_mapper/*.npz by running the UNMODIFIED reference's BinaryMapper on the CPU (TEST
INFRASTRUCTURE ONLY; needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_binary_mapper.py

Per case: the constructor and forward kwargs, the seeds, the logits, the indices (they carry the reference's Bernoulli
draws), the output as its hot values plus the flat positions of its NaNs (every other element is checked to be exactly 0
here), the aux loss, log_prob with indices= and with one_hot=, summed and per bit, and the gradient of
sum(out * G) + aux + sum(log_prob(indices) * H) with respect to the logits.  G (rows, 2^bits) is regenerated from its seed
(`upstream`), the fixture keeps its checksum.  The float64 oracle's rerun on the same indices (`*64`) sets the tolerance.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402
import binary_mapper_oracle as O  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "binary_mapper")

# (name, bits, constructor kwargs, train, forward kwargs, leading dims, dtype, logits kind)
CASES = [
    ("train_b1", 1, {}, True, {}, (4, 32), "fp32", "randn"),
    ("train_b3", 3, {}, True, {}, (2, 64), "fp32", "randn"),
    ("train_b8", 8, {}, True, {}, (4, 16), "fp32", "randn"),
    ("train_b12", 12, {}, True, {}, (2, 8), "fp32", "randn"),
    ("train_b16", 16, {}, True, {}, (1, 16), "fp32", "randn"),
    ("eval_b8", 8, {}, False, {}, (4, 16), "fp32", "randn"),
    ("eval_det_on_eval_b8", 8, dict(deterministic_on_eval=True), False, {}, (4, 16), "fp32", "randn"),
    ("train_deterministic_b12", 12, {}, True, dict(deterministic=True), (2, 8), "fp32", "randn"),
    ("eval_st_b8", 8, {}, False, dict(straight_through=True), (4, 16), "fp32", "randn"),
    ("eval_st_b16", 16, dict(deterministic_on_eval=True), False, dict(straight_through=True), (1, 8), "fp32", "randn"),
    ("temp05_b8", 8, {}, True, dict(temperature=0.5), (4, 16), "fp32", "randn"),
    ("temp2_b3", 3, {}, True, dict(temperature=2.0), (2, 64), "fp32", "randn"),
    ("thr0_b8", 8, dict(kl_loss_threshold=0.0), True, {}, (4, 16), "fp32", "randn"),
    ("thr100_b8", 8, dict(kl_loss_threshold=100.0), True, {}, (4, 16), "fp32", "randn"),
    ("noreduce_image_b3", 3, {}, True, dict(reduce_aux_kl_loss=False), (2, 3, 5), "fp32", "randn"),
    ("noreduce_image_b8", 8, dict(kl_loss_threshold=0.0), True, dict(reduce_aux_kl_loss=False), (2, 2, 4), "fp32", "randn"),
    ("single_row_b8", 8, {}, True, {}, (), "fp32", "randn"),
    ("single_row_b16", 16, {}, True, dict(reduce_aux_kl_loss=False), (), "fp32", "randn"),
    ("bf16_eval_b8", 8, {}, False, {}, (4, 16), "bf16", "randn"),
    ("bf16_no_st_b8", 8, {}, True, dict(straight_through=False), (4, 16), "bf16", "randn"),
    ("bf16_no_st_noreduce_b3", 3, {}, True, dict(straight_through=False, reduce_aux_kl_loss=False), (2, 64), "bf16", "randn"),
    ("nonfinite_b3", 3, {}, True, dict(deterministic=True, calc_aux_loss=False), (4, 8), "fp32", "nonfinite"),
    ("nonfinite_b8", 8, {}, True, dict(deterministic=True, calc_aux_loss=False), (2, 8), "fp32", "nonfinite"),
    ("saturated_b8", 8, {}, True, {}, (4, 16), "fp32", "saturated"),
    ("tiny_b8", 8, {}, True, dict(deterministic=True), (4, 16), "fp32", "tiny"),
    ("tiny_temp2_b3", 3, dict(deterministic_on_eval=True), False, dict(temperature=2.0, straight_through=True), (2, 64), "fp32",
     "tiny"),
]


def upstream(seed: int, rows: int, K: int) -> torch.Tensor:
    """G, the upstream gradient of the output (rows, K) fp32, from its seed."""
    return torch.randn(rows, K, generator=torch.Generator().manual_seed(seed))


def digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()[:16]


def make_logits(kind, shape, g):
    x = torch.randn(*shape, generator=g) * 2.0
    flat = x.view(-1, shape[-1])
    if kind == "nonfinite":   # +inf, -inf, NaN, and both infinities, on the first rows; the rest stays finite
        flat[0, 1] = float("inf")
        flat[1, 0] = -float("inf")
        flat[2, -1] = float("nan")
        flat[3, 0], flat[3, -1] = float("inf"), -float("inf")
    elif kind == "saturated":   # soft code of the hot element near 1 (all large) and rows of mixed +-30
        flat[:] = torch.where(flat >= 0, 30.0, -30.0)
        flat[1::2] *= torch.rand(flat[1::2].shape, generator=g)
    elif kind == "tiny":   # around the deterministic threshold: sigmoid(6e-8) > 0.5 is False, sigmoid(1e-7) > 0.5 is True
        vals = torch.tensor([6e-8, 1e-7, -6e-8, -1e-7, 3e-8, 2e-7, 0.0, 1e-6])
        flat[:] = vals[torch.randint(0, len(vals), flat.shape, generator=g)]
    return x


def run(ref, bits, ckw, train, fkw, x, G, H):
    mod = ref.BinaryMapper(bits=bits, **ckw).train(train)
    x = x.detach().clone().requires_grad_(True)
    out, idx, aux = mod(x, return_indices=True, **fkw)
    total = (out * G.reshape(out.shape).to(out.dtype)).sum() if out.requires_grad else 0.0
    if aux.requires_grad:
        total = total + aux.sum()
    lp = mod.log_prob(x, indices=idx)
    total = total + (lp * H.to(lp.dtype)).sum()
    total.backward()
    with torch.no_grad():
        extra = dict(lp_bits=mod.log_prob(x, indices=idx, sum_bits=False), lp_onehot=mod.log_prob(x, one_hot=out),
                     lp_onehot_bits=mod.log_prob(x, one_hot=out, sum_bits=False))
    return out, idx, aux, lp, x.grad, extra


def to_np(t):
    t = t.detach()
    return t.float().numpy() if t.dtype == torch.bfloat16 else t.numpy()


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, bits, ckw, train, fkw, lead, xdt, kind) in enumerate(CASES):
        seed = 5000 + 10 * i
        g = torch.Generator().manual_seed(seed)
        dt = torch.bfloat16 if xdt == "bf16" else torch.float32
        x = make_logits(kind, (*lead, bits), g).to(dt)
        rows, K = int(np.prod(lead, dtype=np.int64)), 1 << bits
        G = upstream(seed + 1, rows, K)
        H = torch.randn(lead, generator=g)
        torch.manual_seed(seed + 2)
        out, idx, aux, lp, dx, extra = run(ref, bits, ckw, train, fkw, x, G, H)
        assert out.dtype == torch.float32 and out.shape == (*lead, K) and idx.shape == lead
        o = out.detach().reshape(rows, K)
        fi = idx.reshape(rows)
        hot = o[torch.arange(rows), fi]
        rest = o.clone()
        rest[torch.arange(rows), fi] = 0.0
        nan_pos = torch.nonzero(torch.isnan(rest).reshape(-1)).reshape(-1)
        assert not (rest.nan_to_num(0.0) != 0).any() and not torch.signbit(rest.nan_to_num(0.0)).any()
        aux_kind = "zero" if not fkw.get("calc_aux_loss", train) else "mean" if fkw.get("reduce_aux_kl_loss", True) else "rows"
        st = fkw.get("straight_through", train)
        thr = ckw.get("kl_loss_threshold", O.NAT)
        l64 = x.double().numpy().reshape(rows, bits)
        fi_np = fi.numpy()
        rec = dict(bits=np.array(bits), ckw=np.array(json.dumps(ckw)), fkw=np.array(json.dumps(fkw)), train=np.array(train),
                   xdtype=np.array(xdt), lead=np.array(lead, np.int64), seed=np.array(seed), fwd_seed=np.array(seed + 2),
                   g_seed=np.array(seed + 1), g_digest=np.array(digest(G)), x=to_np(x), H=H.numpy(), indices=idx.numpy(),
                   hot=hot.numpy(), nan_pos=nan_pos.numpy(), aux_kind=np.array(aux_kind), aux=to_np(aux), lp=to_np(lp),
                   lp_bits=to_np(extra["lp_bits"]), lp_onehot=to_np(extra["lp_onehot"]),
                   lp_onehot_bits=to_np(extra["lp_onehot_bits"]), dx=to_np(dx))
        a64 = O.aux_rows(l64, thr)
        rec["aux64"] = (a64.mean() if aux_kind == "mean" else a64.reshape(lead)) if aux_kind != "zero" else np.array(0.0)
        rec["lp64"] = O.log_prob(l64, fi_np).reshape(lead)
        rec["lp_bits64"] = O.log_prob(l64, fi_np, sum_bits=False).reshape(*lead, bits)
        rec["dx64"] = O.grad_total(l64, fi_np, G.numpy() if st else None, H.numpy(), st=st, aux_kind=aux_kind,
                                   thr=thr).reshape(*lead, bits)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print(name, "rows", rows, "K", K, "aux", aux_kind, "st", st, "nan elements", len(nan_pos))


if __name__ == "__main__":
    main()
