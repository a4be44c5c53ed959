"""numpy restatement of LatentQuantize (latent_quantization.py, "lq") for the tests: the quantize and index steps exactly in
fp32 (every operation rounded as the reference and vqb_lq_quantize round it), the loss in float64 with the bound the kernel's
fp32 result must lie within.

    quantize(z, tables, levels, basis) -> (codes, indices)   z (M, C, D) fp32; per latent the first argmin of |z - v| (NaN
                                                             first), codes z + (v - z), index sum_i ((c * 2) * hw + hw) * basis
                                                             in fp32 left to right, truncated as the GPU converts (NaN -> 0,
                                                             saturating)
    decode(indices, levels, basis) -> codes                  the fixed lattice of indices_to_codes (lq:194-200)
    loss64(x, out, wc, wq, use_c, use_q) -> (loss, bound)    float64 loss and the kernel's error bound
"""
import numpy as np

F32 = np.float32


def to_int32_gpu(s):
    """fp32 -> int32 as cvt.rzi.s32.f32: truncation, NaN -> 0, saturating at the int32 range."""
    s = np.asarray(s, dtype=np.float32)
    out = np.zeros(s.shape, dtype=np.int64)
    fin = ~np.isnan(s)
    out[fin] = np.clip(np.trunc(s[fin].astype(np.float64)), -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)
    return out.astype(np.int32)


def argmin_first(dist):
    """torch.argmin over the last axis: the first NaN if there is one, else the first minimum."""
    nan = np.isnan(dist)
    idx = np.argmin(np.where(nan, np.inf, dist), axis=-1)
    has_nan = nan.any(-1)
    idx[has_nan] = np.argmax(nan, axis=-1)[has_nan]
    # all-inf rows: np.argmin gives the first inf, the first minimum
    return idx


def quantize(z, tables, levels, basis):
    z = np.asarray(z, dtype=np.float32)
    D = len(tables)
    codes = np.empty_like(z)
    hw = (np.asarray(levels, dtype=np.int64) // 2).astype(np.float32)
    bf = np.asarray(basis, dtype=np.int64).astype(np.float32)
    s = None
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(D):
            v = np.asarray(tables[i], dtype=np.float32)
            zi = z[..., i]
            j = argmin_first(np.abs(zi[..., None] - v))
            c = zi + (v[j] - zi)
            codes[..., i] = c
            t = ((c * F32(2)) * hw[i] + hw[i]) * bf[i]
            s = t if s is None else (s + t).astype(np.float32)
    return codes, to_int32_gpu(s)


def decode(indices, levels, basis):
    """indices (...) int -> codes (..., D) fp32: ((idx // basis) % levels - hw) / hw / 2."""
    lv = np.asarray(levels, dtype=np.int64)
    hw = lv // 2
    k = (np.asarray(indices, dtype=np.int64)[..., None] // np.asarray(basis, dtype=np.int64)) % lv
    with np.errstate(divide="ignore", invalid="ignore"):
        return (((k - hw).astype(np.float32) / hw.astype(np.float32)) / F32(2)).astype(np.float32)


def loss64(x, out, wc, wq, use_c, use_q):
    """The loss w_c m + w_q m in float64 (m the mean of (x - out)^2 over x's elements, a term 0 unless its flag is set) and a
    bound on |kernel - float64|: each difference and square rounded to fp32 (relative 3 u each), the fp64 sum, and the
    fp32 roundings of m, the two products and the sum (u = 2^-24)."""
    x = np.asarray(x, dtype=np.float64).ravel()
    out = np.asarray(out, dtype=np.float64).ravel()
    m = np.mean((x - out) ** 2)
    u = 2.0 ** -24
    w = abs(float(wc)) * use_c + abs(float(wq)) * use_q
    loss = float(wc) * m * use_c + float(wq) * m * use_q
    bound = w * m * (3 * u + x.size * 2.0 ** -52) + w * m * 2 * u + abs(loss) * 2 * u + 1e-45
    return loss, bound
