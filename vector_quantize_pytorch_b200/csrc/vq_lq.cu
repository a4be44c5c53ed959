// LatentQuantize (latent_quantization.py, "lq"): the per-latent value search with its straight-through codes and packed
// index, and the two-sided mse loss with its gradient.  Three kernels:
//
//   lq_quantize_kernel    one thread per (row, codebook) item, the value tables staged in shared memory.  Per latent i:
//                         the first j minimising |z_i - v_i[j]| in fp32 (torch.argmin: a NaN distance is the minimum, the
//                         first one wins), codes_i = z_i + (v_i[j] - z_i) (lq:174) and the index sum_i ((codes_i * 2) * hw_i
//                         + hw_i) * basis_i in fp32, added left to right and truncated to int32 (lq:180-181, :188-192).
//                         Every operation is a separately rounded IEEE op (no fma contraction), so a code that is not on
//                         the lattice (z + (q - z) != q at large |z|) and sums above 2^24 give the reference's index.
//   lq_loss_kernel        per-CTA fp64 partial sums of (x - out)^2 (each difference and square rounded to fp32, as mse_loss
//                         computes them), then one CTA adds the partials in a fixed order (each thread a strided run of
//                         partials, then a shared-memory tree): loss = w_c m + w_q m (lq:293-308)
//                         with m the mean, a term present only when its host flag is set.  No atomics: reruns give the same bits.
//   lq_loss_bwd_kernel    gx = (2/M) (x - out) (w_q g) and gout = (2/M) (out - x) (w_c g), one pass.
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int LQ_THREADS = 256;
constexpr int LQ_CTAS_PER_SM = 8;
constexpr int LOSS_THREADS = 256;
constexpr int LOSS_PER_CTA = 8192;   // elements per loss CTA before the CTA count caps at VQB_LQ_MAX_LOSS_BLOCKS

// Loads element i of an fp32 / bf16 array as fp32.
__device__ __forceinline__ float ld(const void* p, int dtype, int64_t i) {
  return dtype == VQB_DTYPE_BF16 ? Elem<VQB_DTYPE_BF16>::load(p, i) : Elem<VQB_DTYPE_F32>::load(p, i);
}

// Shared memory: the concatenated tables vals[total], then per latent its first table slot, length, hw and basis (as fp32,
// the reference's int32 -> fp32 promotion).
struct LqShared {
  float* vals;
  int* off;
  int* len;
  float* hw;
  float* basis;
};

__device__ __forceinline__ LqShared lq_shared(int D, int total) {
  extern __shared__ float smem[];
  LqShared s;
  s.vals = smem;
  s.off = reinterpret_cast<int*>(smem + total);
  s.len = s.off + D;
  s.hw = reinterpret_cast<float*>(s.len + D);
  s.basis = s.hw + D;
  return s;
}

__global__ void __launch_bounds__(LQ_THREADS) lq_quantize_kernel(const void* __restrict__ z, int dtype, int64_t items, int D,
                                                                  const float* __restrict__ vals, int total,
                                                                  const int32_t* __restrict__ meta, float* __restrict__ codes,
                                                                  int32_t* __restrict__ idx) {
  const LqShared s = lq_shared(D, total);
  for (int k = threadIdx.x; k < total; k += blockDim.x) s.vals[k] = vals[k];
  if (threadIdx.x == 0) {   // table offsets: a prefix sum of the lengths, clamped so that no read leaves the staged tables
    int o = 0;
    for (int i = 0; i < D; ++i) {
      const int off = o < total ? o : total - 1;
      const int room = total - off, L = meta[i];
      s.off[i] = off;
      s.len[i] = L < 1 ? 1 : L > room ? room : L;
      o += L > 0 ? L : 0;
    }
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    s.hw[i] = __int2float_rn(meta[D + i]);
    s.basis[i] = __int2float_rn(meta[2 * D + i]);
  }
  __syncthreads();
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < items; it += stride) {
    const int64_t base = it * D;
    float sum = 0.f;
#pragma unroll 1
    for (int i = 0; i < D; ++i) {
      const float x = ld(z, dtype, base + i);
      const float* v = s.vals + s.off[i];
      const int L = s.len[i];
      float best = fabsf(__fsub_rn(x, v[0]));
      int bj = 0;
      if (!isnan(best)) {
#pragma unroll 4
        for (int j = 1; j < L; ++j) {
          const float dj = fabsf(__fsub_rn(x, v[j]));
          if (isnan(dj)) {   // torch.argmin: the first NaN is the minimum
            bj = j;
            break;
          }
          if (dj < best) {
            best = dj;
            bj = j;
          }
        }
      }
      const float c = __fadd_rn(x, __fsub_rn(v[bj], x));
      codes[base + i] = c;
      const float t = __fmul_rn(__fadd_rn(__fmul_rn(__fmul_rn(c, 2.f), s.hw[i]), s.hw[i]), s.basis[i]);
      sum = i == 0 ? t : __fadd_rn(sum, t);
    }
    idx[it] = __float2int_rz(sum);   // cvt.rzi: NaN -> 0, saturating outside the int32 range
  }
}

__global__ void __launch_bounds__(LOSS_THREADS) lq_loss_kernel(const void* __restrict__ x, int dtype, const float* __restrict__ out,
                                                               int64_t n, double* __restrict__ partial) {
  __shared__ double red[LOSS_THREADS / 32];
  double acc = 0.0;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const float d = __fsub_rn(ld(x, dtype, i), out[i]);
    acc += static_cast<double>(__fmul_rn(d, d));
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < LOSS_THREADS / 32; ++w) t += red[w];
    partial[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(LOSS_THREADS) lq_loss_fin_kernel(const double* __restrict__ partial, int blocks, int64_t n,
                                                                   const float* __restrict__ wc, const float* __restrict__ wq,
                                                                   int use_c, int use_q, float* __restrict__ loss) {
  __shared__ double red[LOSS_THREADS];
  double t = 0.0;
  for (int b = threadIdx.x; b < blocks; b += LOSS_THREADS) t += partial[b];
  red[threadIdx.x] = t;
  __syncthreads();
  for (int h = LOSS_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float m = static_cast<float>(red[0] / static_cast<double>(n));
    // lq:305-308: w_c * (commitment or 0) + w_q * (quantization or 0); both mse terms are the same mean
    loss[0] = __fadd_rn(__fmul_rn(*wc, use_c ? m : 0.f), __fmul_rn(*wq, use_q ? m : 0.f));
  }
}

__global__ void __launch_bounds__(LOSS_THREADS) lq_loss_bwd_kernel(const void* __restrict__ x, int dtype, const float* __restrict__ out,
                                                                   int64_t n, const float* __restrict__ g_loss,
                                                                   const float* __restrict__ wc, const float* __restrict__ wq,
                                                                   int use_c, int use_q, void* __restrict__ gx,
                                                                   float* __restrict__ gout) {
  const float g = *g_loss;
  const float norm = static_cast<float>(2.0 / static_cast<double>(n));   // mse_loss_backward's 2 / numel
  const float gq = use_q ? __fmul_rn(*wq, g) : 0.f;
  const float gc = use_c ? __fmul_rn(*wc, g) : 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const float xv = ld(x, dtype, i), ov = out[i];
    if (gx) {
      const float v = use_q ? __fmul_rn(__fmul_rn(norm, __fsub_rn(xv, ov)), gq) : 0.f;
      if (dtype == VQB_DTYPE_BF16) Elem<VQB_DTYPE_BF16>::store(gx, i, v);
      else Elem<VQB_DTYPE_F32>::store(gx, i, v);
    }
    if (gout) gout[i] = use_c ? __fmul_rn(__fmul_rn(norm, __fsub_rn(ov, xv)), gc) : 0.f;
  }
}

int loss_blocks(int64_t n) {
  const int64_t b = (n + LOSS_PER_CTA - 1) / LOSS_PER_CTA;
  return static_cast<int>(b < VQB_LQ_MAX_LOSS_BLOCKS ? b : VQB_LQ_MAX_LOSS_BLOCKS);
}

bool bad_dtype(int dtype) { return dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16; }

}  // namespace
}  // namespace vqb

extern "C" int vqb_lq_quantize(const void* z, int dtype, int64_t N, int C, int D, const float* vals, int total,
                               const int32_t* meta, float* codes, int32_t* idx, void* stream) {
  using namespace vqb;
  if (!z || !vals || !meta || !codes || !idx || N <= 0 || C <= 0 || D <= 0 || total < D || bad_dtype(dtype)) return VQB_E_INVALID;
  // bounded step by step so no product overflows: N < 2^40, then N C <= 2^40, then N C D <= 2^48
  if (D > VQB_LQ_MAX_DIM || total > VQB_LQ_MAX_VALUES || N >= (int64_t{1} << 40) || C > (int64_t{1} << 40) / N ||
      N * C * D >= (int64_t{1} << 40))
    return VQB_E_UNSUPPORTED;
  if (!aligned(z, dtype == VQB_DTYPE_BF16 ? 2 : 4) || !aligned(vals, 4) || !aligned(meta, 4) || !aligned(codes, 4) ||
      !aligned(idx, 4))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int64_t items = N * C;
  const size_t smem = (static_cast<size_t>(total) + 4 * static_cast<size_t>(D)) * sizeof(float);
  const int grid = capped_grid(items, LQ_THREADS, LQ_CTAS_PER_SM);
  lq_quantize_kernel<<<grid, LQ_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(z, dtype, items, D, vals, total, meta, codes,
                                                                                     idx);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lq_loss_blocks(int64_t n) {
  if (n <= 0) return VQB_E_INVALID;
  if (n >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  return vqb::loss_blocks(n);
}

extern "C" int vqb_lq_loss(const void* x, int dtype, const float* out, int64_t n, const float* wc, const float* wq, int use_c,
                           int use_q, double* partial, int blocks, float* loss, void* stream) {
  using namespace vqb;
  if (!x || !out || !wc || !wq || !partial || !loss || n <= 0 || bad_dtype(dtype) || (use_c | use_q) & ~1) return VQB_E_INVALID;
  if (n >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  if (blocks != loss_blocks(n)) return VQB_E_INVALID;
  if (!aligned(x, dtype == VQB_DTYPE_BF16 ? 2 : 4) || !aligned(out, 4) || !aligned(wc, 4) || !aligned(wq, 4) ||
      !aligned(partial, 8) || !aligned(loss, 4))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  lq_loss_kernel<<<blocks, LOSS_THREADS, 0, s>>>(x, dtype, out, n, partial);
  lq_loss_fin_kernel<<<1, LOSS_THREADS, 0, s>>>(partial, blocks, n, wc, wq, use_c, use_q, loss);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lq_loss_backward(const void* x, int dtype, const float* out, int64_t n, const float* g_loss, const float* wc,
                                    const float* wq, int use_c, int use_q, void* gx, float* gout, void* stream) {
  using namespace vqb;
  if (!x || !out || !g_loss || !wc || !wq || (!gx && !gout) || n <= 0 || bad_dtype(dtype) || (use_c | use_q) & ~1)
    return VQB_E_INVALID;
  if (n >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  const int ea = dtype == VQB_DTYPE_BF16 ? 2 : 4;
  if (!aligned(x, ea) || !aligned(out, 4) || !aligned(g_loss, 4) || !aligned(wc, 4) || !aligned(wq, 4) ||
      (gx && !aligned(gx, ea)) || (gout && !aligned(gout, 4)))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(n, LOSS_THREADS, 8);
  lq_loss_bwd_kernel<<<grid, LOSS_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(x, dtype, out, n, g_loss, wc, wq, use_c, use_q,
                                                                                    gx, gout);
  return static_cast<int>(cudaGetLastError());
}
