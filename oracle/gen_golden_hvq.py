"""Generate tests/golden/hvq/*.npz by running the UNMODIFIED reference's HierarchicalVQ on the CPU (TEST INFRASTRUCTURE ONLY;
needs the reference, oracle/ref_loader.py):

    python oracle/gen_golden_hvq.py

Per case: the constructor kwargs, the seed, the initial state_dict, and per step s: x_s, the upstream gradient G_s of the
reconstruction, the reconstruction, the loss, x.grad of sum(recon * G) + loss (training), the codebook buffers after the step,
every draw the reference made from torch.randperm / torch.randint (`rng_s_j`, so a replay can substitute them for its own),
and per scale k: the pooled input the search saw, the codebook it searched, the codes it returned, the indices, the loss and
the codebook buffers after the call.  After the last step, get_output_from_indices of the last indices.  `*64` arrays: the
same step in float64 (hvq_oracle, with the reference's codes).

A seed is refused, and the next one tried, when some searched row's float64 squared distance to its best code leads the
nearest DISTINCT code vector by less than 1e-4 relative: the replay then has to find the same index at every scale.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402
import hvq_oracle as O  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "hvq")
GAP_REL = 1e-4

_REF = dict(dim=32, codebook_size=128, scales=(1, 2, 4, 7), quant_resi=0.5, share_quant_resi=1)
_FIVE = dict(dim=32, codebook_size=64, scales=(1, 2, 3, 4, 6))
# (name, constructor kwargs, x shape, train, steps)
CASES = [
    ("ref_train", _REF, (2, 32, 7, 7), True, 1),
    ("ref_eval", _REF, (2, 32, 7, 7), False, 1),
    ("ref_two_steps", _REF, (2, 32, 7, 7), True, 2),
    ("share1_5s", dict(_FIVE, share_quant_resi=1), (2, 32, 6, 6), True, 1),
    ("share0_5s", dict(_FIVE, share_quant_resi=0), (2, 32, 6, 6), True, 1),
    ("share2_5s", dict(_FIVE, share_quant_resi=2), (2, 32, 6, 6), True, 1),
    ("share3_5s", dict(_FIVE, share_quant_resi=3), (2, 32, 6, 6), True, 1),
    ("resi0", dict(_REF, quant_resi=0.0), (2, 32, 7, 7), True, 1),
    ("resi_neg05", dict(_REF, quant_resi=-0.5), (2, 32, 7, 7), True, 1),
    ("nonsquare_9x12", dict(dim=32, codebook_size=64, scales=(1, 3, 5, 9)), (2, 32, 9, 12), True, 1),
    ("scale_above_h", dict(dim=32, codebook_size=64, scales=(1, 3, 7)), (2, 32, 5, 5), True, 1),
    ("dup_scales", dict(dim=32, codebook_size=64, scales=(1, 1, 2)), (3, 32, 4, 4), True, 1),
    ("rotation", dict(_REF, rotation_trick=True), (2, 32, 7, 7), True, 1),
    ("no_kmeans_no_expiry", dict(_REF, kmeans_init=False, threshold_ema_dead_code=0), (2, 32, 7, 7), True, 2),
    ("eval_quirk_8x8", dict(dim=32, codebook_size=64, scales=(1, 2, 4)), (2, 32, 8, 8), False, 1),
    ("dim64_train", dict(dim=64, codebook_size=96, scales=(1, 2, 4, 8)), (2, 64, 8, 8), True, 1),
]


def f32(t):
    return t.detach().float().cpu().numpy().astype(np.float32)


class RngRecorder:
    """Records, in call order, what torch.randperm / torch.randint return while it is active."""

    def __init__(self):
        self.draws = []
        self._orig = {}

    def __enter__(self):
        for name in ("randperm", "randint"):
            fn = getattr(torch, name)
            self._orig[name] = fn

            def wrap(*a, _fn=fn, _name=name, **k):
                out = _fn(*a, **k)
                self.draws.append((_name, out.detach().clone()))
                return out
            setattr(torch, name, wrap)
        return self

    def __exit__(self, *exc):
        for name, fn in self._orig.items():
            setattr(torch, name, fn)


class ScaleRecorder:
    """Per vq call: the pooled input, the codebook searched (after any k-means init), the codes returned by the search, the
    indices, the loss and the buffers after the call."""

    def __init__(self, hq):
        self.calls = []
        self.hq = hq
        cb = hq.vq._codebook
        orig = cb.init_embed_

        def init_embed_(*a, **k):
            out = orig(*a, **k)
            self.calls.append(dict(searched=f32(cb.embed[0])))
            return out
        cb.init_embed_ = init_embed_
        cb.register_forward_hook(lambda mod, inp, out: self.calls[-1].update(codes=f32(out[0])))
        hq.vq.register_forward_hook(self._after_vq)

    def _after_vq(self, mod, inp, out):
        cb = mod._codebook
        self.calls[-1].update(pooled=f32(inp[0]), indices=out[1].numpy().astype(np.int64), loss=f32(out[2]),
                              cluster_size=f32(cb.cluster_size[0]), embed_avg=f32(cb.embed_avg[0]), embed=f32(cb.embed[0]))


def gap_ok(pooled, searched):
    """Each row's float64 lead of its best code over the nearest distinct code vector, relative to the row's scale."""
    x = pooled.astype(np.float64).transpose(0, 2, 3, 1).reshape(-1, pooled.shape[1])
    c = searched.astype(np.float64)
    d = ((x[:, None, :] - c[None, :, :]) ** 2).sum(-1)
    best = d.argmin(1)
    same = (c[best][:, None, :] == c[None, :, :]).all(-1)
    other = np.where(same, np.inf, d).min(1)
    lead = other - d[np.arange(len(x)), best]
    scale = np.maximum((x ** 2).sum(-1), (c ** 2).sum(-1).max())
    return bool((lead >= GAP_REL * scale).all()), float((lead / scale).min())


def rerun64(ref, hq, x, G, calls, train, kw):
    """The step in float64 with the reference's codes: reconstruction, mean commitment loss and x.grad."""
    from vector_quantize_pytorch.vector_quantize_pytorch import rotate_to
    scales = hq.scales
    B, D, H, W = x.shape
    phis = [(p.conv.weight.detach().double(), p.conv.bias.detach().double(), p.resi_ratio)
            for p in ([hq.phi_shared] if hq.phi_shared is not None else list(hq.phi_levels))]
    xd = torch.from_numpy(x.astype(np.float64)).requires_grad_(train)
    residual, recon, losses = xd, torch.zeros(B, D, H, W, dtype=torch.float64), []
    for k, s in enumerate(scales):
        ph, pw = torch.from_numpy(O.pool_matrix(H, s)), torch.from_numpy(O.pool_matrix(W, s))
        pooled = torch.einsum("ih,bdhw,jw->bdij", ph, residual, pw)
        codes = torch.from_numpy(calls[k]["codes"].astype(np.float64)).reshape(B, s, s, D).permute(0, 3, 1, 2)
        if train:
            rows = pooled.permute(0, 2, 3, 1).reshape(B, s * s, D)
            crow = codes.permute(0, 2, 3, 1).reshape(B, s * s, D)
            q = rotate_to(rows, crow) if kw.get("rotation_trick", False) else rows + (crow - rows).detach()
            q = q.reshape(B, s, s, D).permute(0, 3, 1, 2)
            losses.append(kw.get("commitment_weight", 1.0) * F.mse_loss(codes, pooled))
        else:
            q = codes
        uh, uw = torch.from_numpy(O.upsample_matrix(s, H)), torch.from_numpy(O.upsample_matrix(s, W))
        up = torch.einsum("hi,bdij,wj->bdhw", uh, q, uw)
        w, b, r = phis[O.choose_phi(len(scales), len(phis), k)]
        if r > 1e-8:
            up = (1.0 - r) * up + r * F.conv2d(up, w, b, padding=1)
        recon = recon + up
        residual = residual - up
    loss = torch.stack(losses).mean() if train else torch.zeros((), dtype=torch.float64)
    if train:
        ((recon * torch.from_numpy(G.astype(np.float64))).sum() + loss).backward()
    return recon.detach().numpy(), float(loss), (xd.grad.numpy() if train else None)


def run_case(ref, i, name, kw, shape, train, steps, seed):
    ckw = dict(kw, accept_image_fmap=True)
    torch.manual_seed(seed)
    hq = ref.HierarchicalVQ(**ckw)
    sd = hq.state_dict()
    rec = dict(sd_keys=np.array(json.dumps(list(sd))))
    for j, v in enumerate(sd.values()):
        rec[f"sd_{j}"] = v.numpy().copy()
    hq.train(train)
    recorder = ScaleRecorder(hq)
    gen = torch.Generator().manual_seed(seed + 1)
    min_lead = np.inf
    ok = True
    for s in range(steps):
        x = torch.randn(*shape, generator=gen)
        G = torch.randn(*shape, generator=gen)
        recorder.calls.clear()
        torch.manual_seed(seed + 100 + s)
        xg = x.clone().requires_grad_(train)
        with RngRecorder() as rng:
            recon, indices, loss = hq(xg)
        if train:
            ((recon * G).sum() + loss).backward()
        calls = list(recorder.calls)
        assert len(calls) == len(hq.scales)
        for k, c in enumerate(calls):
            good, lead = gap_ok(c["pooled"], c["searched"])
            ok &= good
            min_lead = min(min_lead, lead)
            for key in ("pooled", "searched", "codes", "indices", "loss", "cluster_size", "embed_avg", "embed"):
                rec[f"s{s}_k{k}_{key}"] = c[key]
        rec.update({f"x_{s}": f32(x), f"G_{s}": f32(G), f"recon_{s}": f32(recon), f"loss_{s}": f32(loss)})
        if train:
            rec[f"xgrad_{s}"] = f32(xg.grad)
        for j, (kind, t) in enumerate(rng.draws):
            rec[f"rng_{s}_{j}"] = t.numpy().astype(np.int64)
        rec[f"rng_kinds_{s}"] = np.array(json.dumps([k for k, _ in rng.draws]))
        r64, l64, g64 = rerun64(ref, hq, f32(x), f32(G), calls, train, kw)
        rec[f"recon64_{s}"] = r64
        rec[f"loss64_{s}"] = np.array(l64)
        if train:
            rec[f"xgrad64_{s}"] = g64
    last = tuple(torch.from_numpy(rec[f"s{steps - 1}_k{k}_indices"]) for k in range(len(hq.scales)))
    with torch.no_grad():
        rec["gofi"] = f32(hq.get_output_from_indices(last))
    cb = hq.vq._codebook
    phis = [hq.phi_shared] if hq.phi_shared is not None else list(hq.phi_levels)
    codes = [cb.embed[0].detach().numpy().astype(np.float64)[rec[f"s{steps - 1}_k{k}_indices"]].transpose(0, 3, 1, 2)
             for k in range(len(hq.scales))]
    S = hq.scales[-1]
    rec["gofi64"], _ = O.forward(np.zeros(shape[:2] + (S, S)), hq.scales, codes,
                                 [(p.conv.weight.detach().numpy(), p.conv.bias.detach().numpy(), p.resi_ratio) for p in phis],
                                 0, full_hw=(S, S))
    meta = dict(name=name, kw=kw, shape=list(shape), train=train, steps=steps, seed=seed, scales=list(hq.scales),
                n_phi=len(phis), min_lead=min_lead, torch=torch.__version__)
    rec["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    return ok, rec, min_lead


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    for i, (name, kw, shape, train, steps) in enumerate(CASES):
        for attempt in range(64):
            seed = 7000 + 100 * i + attempt
            ok, rec, lead = run_case(ref, i, name, kw, shape, train, steps, seed)
            if ok:
                break
        else:
            raise RuntimeError(f"{name}: no seed with every search lead above {GAP_REL}")
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"hvq/{name}: seed {seed} min lead {lead:.3g} {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
