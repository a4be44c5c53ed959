// Finite scalar perturbation: FSP (finite_scalar_perturbation.py, "fsp").  One thread owns one row, its D <= 16 values in
// registers; the CDF and need_inv_act are template parameters.  Five kernels:
//
//   fsp_forward_kernel   the CDF activation (fsp:31-72), clamp_max(1 - eps), floor(act L), the midpoint (l + 1/2) / L and the
//                        straight-through value (fsp:276-281); in training with quantize_rate < 1 the proposal act + (2 u1 - 1)
//                        / (2 L), its accept test and the u2 > quantize_rate choice (fsp:332-341); the output map (fsp:343-348),
//                        the exact int32 index and the level indices, and a per-CTA accept count.
//   fsp_moments_kernel   the batch moments of z over the rows (fsp:93-99): pass 0 the column sums, pass 1 the central sums
//                        of u^2, u^3, u^4 around the mean, both in fp64, one partial per CTA; fsp_mean_kernel between them
//                        adds pass 0's partials in a fixed order (one warp per column).
//   fsp_stats_kernel     one CTA: pass 1's partials added in a fixed order, then the unbiased variance, the clamped
//                        std, the skewness, the kurtosis - 3 and the weighted norm loss (fsp:126-133).
//   fsp_backward_kernel  d z = the quantized-output path (the CDF derivative, or the identity with need_inv_act) plus the
//                        statistics path, a cubic in t = (z - m) / std with per-column coefficients (DESIGN 4.11).
//   fsp_decode_kernel    indices -> act values (l + 1/2) / L -> codes (fsp:286-307), digits (index // basis) % L.
//
// Every operation is rounded explicitly (no contraction).  torch runs the reference's chain in z's dtype up to the `where`
// of the perturbation, whose fp32 `p_max_norm` promotes everything after it to fp32; `rw` rounds to z's dtype, `rwo` to the
// dtype of the output chain (fp32 when perturbing).  Scalars keep fp32 precision in arithmetic and are cast to the tensor's
// dtype in comparisons and clamps, as torch does; the host passes those casts in (include/vqb200.h).
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int FSP_THREADS = 256;
constexpr int FSP_CTAS_PER_SM = 8;   // grid cap; vqb_fsp_blocks reports the grid, which orders the partial sums
constexpr int FSP_MAX_D = 16;
constexpr float SQRT2F = 1.41421356237309515f;   // fsp:47, as fp32
constexpr float PIF = 3.14159265358979312f;      // torch.pi, as fp32
constexpr float UNIT_STD = 0.28867513459481287f; // fsp:348, as fp32
constexpr float R_SQRT2F = 1.f / SQRT2F;          // the reciprocals, rounded to nearest, for divc
constexpr float R_PIF = 1.f / PIF;
constexpr float R_UNIT_STD = 1.f / UNIT_STD;

enum { ACT_TANH = 0, ACT_SIGMOID = 1, ACT_NORMAL = 2, ACT_LAPLACE = 3, ACT_CAUCHY = 4 };

__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : v); }   // torch.sign keeps 0 and NaN

// 1 / x in fp64 for a normal, finite x != 0: the hardware estimate refined by three Newton steps (each squares the relative
// error, which ends at the fp64 rounding), with no call to the division's slow path (whose calling convention spills).
__device__ __forceinline__ double rcp64(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#pragma unroll
  for (int i = 0; i < 3; ++i) r = __fma_rn(r, __fma_rn(-x, r, 1.0), r);
  return r;
}

// torch.sigmoid's 1 / (1 + e), e = exp(-z) in [0, inf], correctly rounded to fp32: 1 + e >= 1 is normal, and the fp64 quotient
// is within 2^-52 relative of 1 / (1 + e), which is never that close to an fp32 rounding midpoint (a quotient 1 / x of an
// fp32 x lies at least 2^-49 relative from any such midpoint), so rounding it once gives the correctly rounded result.
__device__ __forceinline__ float sigmoid_rcp(float e) {
  const float x = __fadd_rn(1.f, e);
  return isinf(x) ? 0.f : __double2float_rn(rcp64(static_cast<double>(x)));
}

// a / b, correctly rounded, for finite a and a normal, finite b: the fp64 product a (1 / b) is within 2^-51 relative of the
// quotient, and a quotient of two fp32 values is never that close to an fp32 rounding midpoint.
__device__ __forceinline__ float div64(float a, float b) {
  return __double2float_rn(static_cast<double>(a) * rcp64(static_cast<double>(b)));
}

// tan(b) for |b| <= pi / 2 + 1 ulp (the clamped inverse Cauchy argument): sin(pi x) / cos(pi x) with x = b / pi in fp64, whose
// argument reduction is exact, so there is no large-argument path (tanf's would spill); the fp64 quotient is far inside one fp32
// ulp of tan(b) even where cos(b) ~ 1e-7.
__device__ __forceinline__ float tan_halfpi(float b) {
  double sn, cs;
  sincospi(static_cast<double>(b) * 0.31830988618379067, &sn, &cs);   // b / pi; its last bit does not reach the fp32 result
  return __double2float_rn(sn * rcp64(cs));   // |cs| >= 4e-8: normal
}

// The CDF activations, (-inf, inf) -> [0, 1], each op rounded to z's dtype.
template <int ACT, bool BF>
__device__ __forceinline__ float cdf(float z) {
  if constexpr (ACT == ACT_TANH) {            // (tanh(z) + 1) / 2
    return rw<BF>(__fmul_rn(rw<BF>(__fadd_rn(rw<BF>(tanhf(z)), 1.f)), 0.5f));
  } else if constexpr (ACT == ACT_SIGMOID) {  // torch.sigmoid: 1 / (1 + exp(-z)), one rounding
    return rw<BF>(sigmoid_rcp(expf(-z)));
  } else if constexpr (ACT == ACT_NORMAL) {   // (1 + erf(z / sqrt 2)) / 2
    const float e = rw<BF>(erff(rw<BF>(divc(z, SQRT2F, R_SQRT2F))));
    return rw<BF>(__fmul_rn(rw<BF>(__fadd_rn(1.f, e)), 0.5f));
  } else if constexpr (ACT == ACT_LAPLACE) {  // 0.5 (1 + sign(z) (1 - exp(-|z|)))
    const float m = rw<BF>(__fsub_rn(1.f, rw<BF>(expf(-fabsf(z)))));
    return rw<BF>(__fmul_rn(0.5f, rw<BF>(__fadd_rn(1.f, rw<BF>(__fmul_rn(sgn(z), m))))));
  } else {                                    // arctan(z) / pi + 0.5
    return rw<BF>(__fadd_rn(rw<BF>(divc(rw<BF>(atanf(z)), PIF, R_PIF)), 0.5f));
  }
}

// The inverse CDFs (0, 1) -> (-inf, inf), each op rounded by R (the output chain's dtype).
template <int ACT, typename R>
__device__ __forceinline__ float inv_cdf(float p, R r) {
  if constexpr (ACT == ACT_TANH) {            // arctanh(2 p - 1)
    return r(atanhf(r(__fsub_rn(r(__fmul_rn(p, 2.f)), 1.f))));
  } else if constexpr (ACT == ACT_SIGMOID) {  // torch.logit: log(p / (1 - p)), one rounding
    return r(logf(div64(p, __fsub_rn(1.f, p))));   // 1 - p >= eps: normal
  } else if constexpr (ACT == ACT_NORMAL) {   // erfinv(2 p - 1) sqrt 2
    return r(__fmul_rn(r(erfinvf(r(__fsub_rn(r(__fmul_rn(2.f, p)), 1.f)))), SQRT2F));
  } else if constexpr (ACT == ACT_LAPLACE) {  // -sign(p - 0.5) log(1 - 2 |p - 0.5|)
    const float a = r(__fsub_rn(p, 0.5f));
    const float l = r(logf(r(__fsub_rn(1.f, r(__fmul_rn(2.f, fabsf(a)))))));
    return r(__fmul_rn(-sgn(a), l));
  } else {                                    // tan((p - 0.5) pi)
    return r(tan_halfpi(r(__fmul_rn(r(__fsub_rn(p, 0.5f)), PIF))));
  }
}

// d act / d z times g, in autograd's order (fp32).  y: the activation's saved output where autograd uses it.
template <int ACT, bool BF>
__device__ __forceinline__ float cdf_bwd(float g, float z) {
  if constexpr (ACT == ACT_TANH) {            // / 2, then tanh_backward g (1 - y^2)
    const float y = rw<BF>(tanhf(z));
    return __fmul_rn(__fmul_rn(g, 0.5f), __fsub_rn(1.f, __fmul_rn(y, y)));
  } else if constexpr (ACT == ACT_SIGMOID) {  // sigmoid_backward g (1 - y) y
    const float y = rw<BF>(sigmoid_rcp(expf(-z)));
    return __fmul_rn(__fmul_rn(g, __fsub_rn(1.f, y)), y);
  } else if constexpr (ACT == ACT_NORMAL) {   // / 2, erf' = 2 / sqrt(pi) exp(-u^2), / sqrt 2
    const float u = rw<BF>(divc(z, SQRT2F, R_SQRT2F));
    const float d = __fmul_rn(1.12837916709551257f, expf(-__fmul_rn(u, u)));
    return divc(__fmul_rn(__fmul_rn(g, 0.5f), d), SQRT2F, R_SQRT2F);
  } else if constexpr (ACT == ACT_LAPLACE) {  // * 0.5, * sign(z), exp backward, abs backward (sign(z), 0 at 0)
    const float s = sgn(z);
    return __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(g, 0.5f), s), rw<BF>(expf(-fabsf(z)))), s);
  } else {                                    // / pi, atan backward g / (1 + z^2)
    const float d = __fadd_rn(1.f, __fmul_rn(z, z));   // >= 1
    const float gp = divc(g, PIF, R_PIF);
    return isinf(d) ? __fmul_rn(gp, 0.f) : div64(gp, d);
  }
}

struct FwdArgs {
  const void* z;
  const void* u1;   // [N][D] in z's dtype, or null: no perturbation
  const void* u2;
  const int32_t* levels;
  int64_t N;
  float clamp_hi;   // 1 - eps in z's dtype
  float qrate;      // quantize_rate in z's dtype
  float inv_lo, inv_hi;   // eps, 1 - eps in the output chain's dtype
  void* out;        // [N][D], fp32 when perturbing, else z's dtype
  int32_t* idx;     // [N]
  void* lev_out;    // [N][D] in z's dtype, or null
  int32_t* accept;  // [gridDim.x], or null
};

struct LevelTable {
  int lev[FSP_MAX_D];
  int basis[FSP_MAX_D];
  float pmax[FSP_MAX_D];   // 1.0 / (2 L) in fp32 (fsp:333)
  float rlev[FSP_MAX_D];   // RN(1 / L), for divc
  int64_t size;            // prod(levels)
};

template <int D>
__device__ __forceinline__ void load_levels(LevelTable& t, const int32_t* levels) {
  if (threadIdx.x == 0) {
    int b = 1;
    for (int j = 0; j < D; ++j) {
      t.lev[j] = levels[j];
      t.basis[j] = b;
      t.pmax[j] = __frcp_rn(static_cast<float>(2 * levels[j]));
      t.rlev[j] = __frcp_rn(static_cast<float>(levels[j]));
      b *= levels[j];   // the host refuses prod(levels) >= 2^31
    }
    t.size = b;
  }
  __syncthreads();
}

template <int ACT, bool INV, bool BF, int D>
__global__ void __launch_bounds__(FSP_THREADS) fsp_forward_kernel(FwdArgs a) {
  __shared__ LevelTable t;
  __shared__ int warp_cnt[FSP_THREADS / 32];
  load_levels<D>(t, a.levels);
  constexpr int DT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  const bool pert = a.u1 != nullptr;
  const bool obf = BF && !pert;   // the output chain runs in z's dtype unless the perturbation promoted it to fp32
  const auto rwo = [obf](float v) { return obf ? bf16_round(v) : v; };
  int cnt = 0;
  for (int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; row < a.N; row += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float z[D], q[D], l[D];
    load_item<DT, D>(a.z, row, z);
    int index = 0;
#pragma unroll
    for (int j = 0; j < D; ++j) {
      const float act = cdf<ACT, BF>(z[j]);
      const float L = static_cast<float>(t.lev[j]);
      const float c = act != act ? act : fminf(act, a.clamp_hi);            // clamp_max keeps NaN
      l[j] = floorf(rw<BF>(__fmul_rn(c, L)));
      index += static_cast<int>(l[j]) * t.basis[j];                         // exact (DESIGN 4.11)
      const float mid = rw<BF>(divc(rw<BF>(__fadd_rn(l[j], 0.5f)), L, t.rlev[j]));
      q[j] = rw<BF>(__fadd_rn(act, rw<BF>(__fsub_rn(mid, act))));           // act + (q - act).detach()
    }
    a.idx[row] = index;
    if (a.lev_out) store_item<DT, D>(a.lev_out, row, l);
    if (pert) {
      float u1[D], u2[D];
      load_item<DT, D>(a.u1, row, u1);
      load_item<DT, D>(a.u2, row, u2);
#pragma unroll
      for (int j = 0; j < D; ++j) {
        const float act = cdf<ACT, BF>(z[j]);
        const float r = rw<BF>(__fsub_rn(rw<BF>(__fmul_rn(u1[j], 2.f)), 1.f));
        const float prop = __fadd_rn(act, __fmul_rn(t.pmax[j], r));         // fp32 from here on
        const bool acc = prop > 0.f && prop < 1.f;
        cnt += acc;
        if (u2[j] > a.qrate) q[j] = acc ? prop : act;
      }
    }
#pragma unroll
    for (int j = 0; j < D; ++j) {
      if constexpr (INV) {
        const float p = q[j] != q[j] ? q[j] : fminf(fmaxf(q[j], a.inv_lo), a.inv_hi);
        const float v = inv_cdf<ACT>(p, rwo);
        q[j] = rwo(__fadd_rn(z[j], rwo(__fsub_rn(v, z[j]))));               // z + (q_z - z).detach()
      } else {
        q[j] = rwo(divc(rwo(__fsub_rn(q[j], 0.5f)), UNIT_STD, R_UNIT_STD));
      }
    }
    if (obf) store_item<VQB_DTYPE_BF16, D>(a.out, row, q);
    else store_item<VQB_DTYPE_F32, D>(a.out, row, q);
  }
  if (a.accept) {
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int s = 0;
      for (int w = 0; w < FSP_THREADS / 32; ++w) s += warp_cnt[w];
      a.accept[blockIdx.x] = s;
    }
  }
}

// The column sums of z (PASS 0), or of u^2, u^3, u^4 with u = z - mean (PASS 1, the mean from fsp_mean_kernel), over the
// rows this CTA visits: part[blockIdx.x][k][D].  Per thread, then per warp (shuffles), then the warps in order: no atomics.
template <bool BF, int D, int PASS>
__global__ void __launch_bounds__(FSP_THREADS) fsp_moments_kernel(const void* __restrict__ zp, int64_t N, const double* __restrict__ colmean,
                                                                   double* __restrict__ part) {
  constexpr int K = PASS == 0 ? 1 : 3;
  constexpr int DT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  __shared__ double mean[D];
  __shared__ double red[FSP_THREADS / 32][K * D];
  if (PASS == 1) {
    if (threadIdx.x < D) mean[threadIdx.x] = colmean[threadIdx.x];
    __syncthreads();
  }
  double acc[K * D];
#pragma unroll
  for (int i = 0; i < K * D; ++i) acc[i] = 0.;
  for (int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; row < N; row += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float z[D];
    load_item<DT, D>(zp, row, z);
#pragma unroll
    for (int j = 0; j < D; ++j) {
      if constexpr (PASS == 0) {
        acc[j] += static_cast<double>(z[j]);
      } else {
        const double u = static_cast<double>(z[j]) - mean[j], u2 = u * u;
        acc[j] += u2;
        acc[D + j] += u2 * u;
        acc[2 * D + j] += u2 * u2;
      }
    }
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < K * D; ++i) {
    const double v = warp_sum(acc[i]);
    if (lane == 0) red[w][i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * D; i += blockDim.x) {
    double s = 0.;
    for (int v = 0; v < FSP_THREADS / 32; ++v) s += red[v][i];
    part[static_cast<int64_t>(blockIdx.x) * K * D + i] = s;
  }
}

// The sum over b < blocks of part[b * stride + j] by one warp, in a fixed order: lane l adds b = l, l + 32, ..., then the
// lanes are added by the xor-shuffle tree.  Equal partials give equal bits.
__device__ __forceinline__ double warp_colsum(const double* part, int blocks, int stride, int j) {
  double s = 0.;
  for (int b = threadIdx.x & 31; b < blocks; b += 32) s += part[static_cast<int64_t>(b) * stride + j];
  return warp_sum(s);
}

// Warp j: the mean of column j from pass 0's partials.
__global__ void fsp_mean_kernel(int64_t N, int D, int blocks, const double* __restrict__ part0, double* __restrict__ colmean) {
  const int j = threadIdx.x >> 5;
  const double s = warp_colsum(part0, blocks, D, j);
  if ((threadIdx.x & 31) == 0) colmean[j] = s / static_cast<double>(N);
}

struct NormW {
  double t[4], w[4];   // VectorNorm targets and weights (fsp:120-123)
};

// aux f64 [D][FSP_AUX]: what the backward needs of the statistics.
enum { AUX_MEAN = 0, AUX_STD = 1, AUX_SKEW = 2, AUX_KURT = 3, AUX_A2 = 4, AUX_MASK = 5, AUX_VAR = 6, FSP_AUX = 8 };

// One CTA, warp j for column j: pass 1's partials added in a fixed order, then the moments, the aux row and the loss terms.
template <bool BF>
__global__ void fsp_stats_kernel(int64_t N, int D, int blocks, const double* __restrict__ colmean, const double* __restrict__ part1,
                                 NormW nw, void* __restrict__ stats, void* __restrict__ loss, double* __restrict__ aux) {
  __shared__ double terms[4][FSP_MAX_D];
  const int j = threadIdx.x >> 5;
  const double m2 = warp_colsum(part1, blocks, 3 * D, j);
  const double m3 = warp_colsum(part1 + D, blocks, 3 * D, j);
  const double m4 = warp_colsum(part1 + 2 * D, blocks, 3 * D, j);
  if ((threadIdx.x & 31) == 0) {
    const double n = static_cast<double>(N);
    const double mean = colmean[j], var = m2 / (n - 1.);
    const double sd = sqrt(var);
    const double std = sd != sd ? sd : fmax(sd, 1e-8);   // clamp_min keeps NaN
    const double s2 = std * std;
    const double skew = m3 / n / (s2 * std), kurt = m4 / n / (s2 * s2) - 3.;
    const double v[4] = {mean, var, skew, kurt};
    for (int k = 0; k < 4; ++k) {
      const float f = static_cast<float>(v[k]);
      if (BF) reinterpret_cast<uint16_t*>(stats)[k * D + j] = float_to_bf16_bits(f);
      else reinterpret_cast<float*>(stats)[k * D + j] = f;
      const double e = v[k] - nw.t[k];
      terms[k][j] = e * e;
    }
    double* x = aux + j * FSP_AUX;
    x[AUX_MEAN] = mean; x[AUX_STD] = std; x[AUX_SKEW] = skew; x[AUX_KURT] = kurt;
    x[AUX_A2] = m2 / n / s2; x[AUX_MASK] = sd >= 1e-8 ? 1. : 0.; x[AUX_VAR] = var; x[7] = 0.;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double l = 0.;
    for (int k = 0; k < 4; ++k) {
      double s = 0.;
      for (int i = 0; i < D; ++i) s += terms[k][i];
      l += s / D * nw.w[k];
    }
    const float f = static_cast<float>(l);
    if (BF) *reinterpret_cast<uint16_t*>(loss) = float_to_bf16_bits(f);
    else *reinterpret_cast<float*>(loss) = f;
  }
}

struct BwdArgs {
  const void* z;
  const void* g;         // [N][D] upstream gradient of the output, or null
  int g_bf16;            // its dtype
  const double* aux;
  const float* g_stats;  // f32 [4][D] upstream gradients of mean, variance, skewness, kurtosis, or null
  const float* g_loss;   // f32 [1] upstream gradient of norm_loss, or null
  NormW nw;
  int64_t N;
  void* gz;
};

// dz = d_q(z) + a0 + t (a1 + t (a2 + t a3)), t = (z - m) / std (DESIGN 4.11).
template <int ACT, bool INV, bool BF, int D>
__global__ void __launch_bounds__(FSP_THREADS) fsp_backward_kernel(BwdArgs a) {
  __shared__ double cf[6][FSP_MAX_D];   // a0..a3, mean, 1 / std
  constexpr int DT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  if (threadIdx.x < D) {
    const int j = threadIdx.x;
    const double* x = a.aux + j * FSP_AUX;
    const double n = static_cast<double>(a.N), m = x[AUX_MEAN], sd = x[AUX_STD], s = x[AUX_SKEW], k = x[AUX_KURT];
    const double gl = a.g_loss ? static_cast<double>(*a.g_loss) : 0.;
    const double st[4] = {m, x[AUX_VAR], s, k};
    double G[4];
    for (int i = 0; i < 4; ++i)   // d norm_loss / d stat_i = 2 w_i (stat_i - target_i) / D
      G[i] = (a.g_stats ? static_cast<double>(a.g_stats[i * D + j]) : 0.) + gl * 2. * a.nw.w[i] * (st[i] - a.nw.t[i]) / D;
    const double c = x[AUX_MASK], nsd = n * sd, n1sd = (n - 1.) * sd;
    cf[0][j] = G[0] / n - 3. * G[2] * x[AUX_A2] / nsd - 4. * G[3] * s / nsd;
    cf[1][j] = 2. * G[1] * sd / (n - 1.) - c * 3. * G[2] * s / n1sd - c * 4. * G[3] * (k + 3.) / n1sd;
    cf[2][j] = 3. * G[2] / nsd;
    cf[3][j] = 4. * G[3] / nsd;
    cf[4][j] = m;
    cf[5][j] = 1. / sd;
  }
  __syncthreads();
  for (int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; row < a.N; row += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float z[D], g[D];
    load_item<DT, D>(a.z, row, z);
    if (a.g) {
      if (a.g_bf16) load_item<VQB_DTYPE_BF16, D>(a.g, row, g);
      else load_item<VQB_DTYPE_F32, D>(a.g, row, g);
    }
#pragma unroll
    for (int j = 0; j < D; ++j) {
      float dq = 0.f;
      if (a.g) dq = INV ? g[j] : cdf_bwd<ACT, BF>(divc(g[j], UNIT_STD, R_UNIT_STD), z[j]);
      const double t = (static_cast<double>(z[j]) - cf[4][j]) * cf[5][j];
      const double ds = cf[0][j] + t * (cf[1][j] + t * (cf[2][j] + t * cf[3][j]));
      z[j] = static_cast<float>(static_cast<double>(dq) + ds);
    }
    store_item<DT, D>(a.gz, row, z);
  }
}

// (ix // basis_j) % L_j depends only on ix mod C (C = prod(levels) < 2^31, a multiple of basis_j L_j), in Python's floor
// semantics.  Each step subtracts q C for the fp64 estimate q of floor(m / C) (m times the Newton-refined 1 / C), in wrapping uint64 arithmetic (the true
// difference is small, so the wrap is exact): for |m| up to 2^63 the estimate's error leaves |m| < 2^13 C, which fp64 holds
// exactly, so the next step is off by at most one and the loop ends within three steps, with no 64-bit division.
__device__ __forceinline__ int64_t floor_mod(int64_t ix, int64_t C) {
  int64_t m = ix;
  while (m < 0 || m >= C) {
    const int64_t q = static_cast<int64_t>(floor(static_cast<double>(m) * rcp64(static_cast<double>(C))));
    m = static_cast<int64_t>(static_cast<uint64_t>(m) - static_cast<uint64_t>(q) * static_cast<uint64_t>(C));
    if (q == 0) m += m < 0 ? C : -C;   // the estimate rounded across an integer
  }
  return m;
}

// indices (int32 / int64, contiguous [N]) -> act values f32 [N][D] (act_out, or null) and codes f32 [N][D] (codes, or null).
template <int ACT, bool INV, int D>
__global__ void __launch_bounds__(FSP_THREADS) fsp_decode_kernel(const void* __restrict__ idx, int idx64, int64_t N, const int32_t* levels,
                                                                  float lo, float hi, float* __restrict__ act_out, float* __restrict__ codes) {
  __shared__ LevelTable t;
  load_levels<D>(t, levels);
  const auto id = [](float v) { return v; };
  for (int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; row < N; row += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t ix = load_index(idx, idx64, row);
    const int64_t m = floor_mod(ix, t.size);
    float p[D], c[D];
#pragma unroll
    for (int j = 0; j < D; ++j) {
      const uint32_t r = (static_cast<uint32_t>(m) / static_cast<uint32_t>(t.basis[j])) % static_cast<uint32_t>(t.lev[j]);
      const float L = static_cast<float>(t.lev[j]);
      p[j] = divc(__fadd_rn(static_cast<float>(r), 0.5f), L, t.rlev[j]);
      if constexpr (INV) c[j] = inv_cdf<ACT>(fminf(fmaxf(p[j], lo), hi), id);
      else c[j] = divc(__fsub_rn(p[j], 0.5f), UNIT_STD, R_UNIT_STD);
    }
    if (act_out) store_item<VQB_DTYPE_F32, D>(act_out, row, p);
    if (codes) store_item<VQB_DTYPE_F32, D>(codes, row, c);
  }
}

int fsp_shape(int64_t N, int D, int dtype) {
  if (N <= 0 || D < 1) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D > FSP_MAX_D || N >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  return VQB_OK;
}

NormW norm_weights(const double* norm) {
  NormW w;
  for (int k = 0; k < 4; ++k) { w.t[k] = norm[2 * k]; w.w[k] = norm[2 * k + 1]; }
  return w;
}

// ACT and INV as template arguments; with need_inv_act the backward does not depend on the CDF (one instantiation).
#define VQB_FSP_SWITCH_ACT(CALL, DD, BFV)                                                                                   \
  if (inv) {                                                                                                                \
    switch (act) {                                                                                                          \
      case ACT_TANH: CALL(ACT_TANH, true, BFV, DD); break; case ACT_SIGMOID: CALL(ACT_SIGMOID, true, BFV, DD); break;       \
      case ACT_NORMAL: CALL(ACT_NORMAL, true, BFV, DD); break; case ACT_LAPLACE: CALL(ACT_LAPLACE, true, BFV, DD); break;   \
      default: CALL(ACT_CAUCHY, true, BFV, DD); break;                                                                      \
    }                                                                                                                       \
  } else {                                                                                                                  \
    switch (act) {                                                                                                          \
      case ACT_TANH: CALL(ACT_TANH, false, BFV, DD); break; case ACT_SIGMOID: CALL(ACT_SIGMOID, false, BFV, DD); break;     \
      case ACT_NORMAL: CALL(ACT_NORMAL, false, BFV, DD); break; case ACT_LAPLACE: CALL(ACT_LAPLACE, false, BFV, DD); break; \
      default: CALL(ACT_CAUCHY, false, BFV, DD); break;                                                                     \
    }                                                                                                                       \
  }

}  // namespace
}  // namespace vqb

extern "C" int vqb_fsp_blocks(int64_t N) {
  using namespace vqb;
  if (N <= 0) return VQB_E_INVALID;
  if (N >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if (const int rc = check_device()) return rc;
  return capped_grid(N, FSP_THREADS, FSP_CTAS_PER_SM);
}

extern "C" int vqb_fsp_forward(const void* z, int dtype, int64_t N, int D, int act, int inv, const int32_t* levels, float clamp_hi,
                               const void* u1, const void* u2, float qrate, float inv_lo, float inv_hi, void* out, int32_t* idx,
                               void* level_idx, int32_t* accept, int accept_blocks, void* stream) {
  using namespace vqb;
  if (!z || !levels || !out || !idx || (!u1 != !u2) || (u1 && !accept)) return VQB_E_INVALID;
  if (act < ACT_TANH || act > ACT_CAUCHY) return VQB_E_INVALID;
  if (const int rc = fsp_shape(N, D, dtype)) return rc;
  if (!aligned(z, 16) || !aligned(out, 16) || (u1 && (!aligned(u1, 16) || !aligned(u2, 16))) ||
      (level_idx && !aligned(level_idx, 16)))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(N, FSP_THREADS, FSP_CTAS_PER_SM);
  if (accept && accept_blocks != grid) return VQB_E_INVALID;   // vqb_fsp_blocks() sizes the counts
  const FwdArgs a{z, u1, u2, levels, N, clamp_hi, qrate, inv_lo, inv_hi, out, idx, level_idx, u1 ? accept : nullptr};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool bf = dtype == VQB_DTYPE_BF16;
#define VQB_FSP_FWD_LAUNCH(A, I, B, DD) fsp_forward_kernel<A, I, B, DD><<<grid, FSP_THREADS, 0, s>>>(a)
#define VQB_FSP_FWD(DD)                                                \
  if (bf) { VQB_FSP_SWITCH_ACT(VQB_FSP_FWD_LAUNCH, DD, true) }         \
  else { VQB_FSP_SWITCH_ACT(VQB_FSP_FWD_LAUNCH, DD, false) }
  VQB_SWITCH_D(VQB_FSP_FWD)
#undef VQB_FSP_FWD
#undef VQB_FSP_FWD_LAUNCH
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fsp_stats(const void* z, int dtype, int64_t N, int D, const double* norm, double* work, int blocks, void* stats,
                             void* loss, double* aux, void* stream) {
  using namespace vqb;
  if (!z || !norm || !work || !stats || !loss || !aux) return VQB_E_INVALID;
  if (const int rc = fsp_shape(N, D, dtype)) return rc;
  if (!aligned(z, 16)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  // work f64 [4 * blocks + 1][D], sized by vqb_fsp_blocks()
  if (blocks != capped_grid(N, FSP_THREADS, FSP_CTAS_PER_SM)) return VQB_E_INVALID;
  double* part0 = work;
  double* part1 = work + static_cast<int64_t>(blocks) * D;
  double* colmean = work + static_cast<int64_t>(4 * blocks) * D;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool bf = dtype == VQB_DTYPE_BF16;
#define VQB_FSP_MOM(DD)                                                                                  \
  if (bf) {                                                                                              \
    fsp_moments_kernel<true, DD, 0><<<blocks, FSP_THREADS, 0, s>>>(z, N, nullptr, part0);                \
    fsp_mean_kernel<<<1, 32 * DD, 0, s>>>(N, DD, blocks, part0, colmean);                                \
    fsp_moments_kernel<true, DD, 1><<<blocks, FSP_THREADS, 0, s>>>(z, N, colmean, part1);                \
  } else {                                                                                               \
    fsp_moments_kernel<false, DD, 0><<<blocks, FSP_THREADS, 0, s>>>(z, N, nullptr, part0);               \
    fsp_mean_kernel<<<1, 32 * DD, 0, s>>>(N, DD, blocks, part0, colmean);                                \
    fsp_moments_kernel<false, DD, 1><<<blocks, FSP_THREADS, 0, s>>>(z, N, colmean, part1);               \
  }
  VQB_SWITCH_D(VQB_FSP_MOM)
#undef VQB_FSP_MOM
  const NormW nw = norm_weights(norm);
  if (bf) fsp_stats_kernel<true><<<1, 32 * D, 0, s>>>(N, D, blocks, colmean, part1, nw, stats, loss, aux);
  else fsp_stats_kernel<false><<<1, 32 * D, 0, s>>>(N, D, blocks, colmean, part1, nw, stats, loss, aux);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fsp_backward(const void* z, int dtype, int64_t N, int D, int act, int inv, const void* grad_q, int grad_dtype,
                                const double* aux, const float* grad_stats, const float* grad_loss, const double* norm, void* grad_z,
                                void* stream) {
  using namespace vqb;
  if (!z || !aux || !norm || !grad_z) return VQB_E_INVALID;
  if (act < ACT_TANH || act > ACT_CAUCHY) return VQB_E_INVALID;
  if (grad_q && grad_dtype != VQB_DTYPE_F32 && grad_dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (const int rc = fsp_shape(N, D, dtype)) return rc;
  if (!aligned(z, 16) || !aligned(grad_z, 16) || (grad_q && !aligned(grad_q, 16))) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const BwdArgs a{z, grad_q, grad_dtype == VQB_DTYPE_BF16, aux, grad_stats, grad_loss, norm_weights(norm), N, grad_z};
  const int grid = capped_grid(N, FSP_THREADS, FSP_CTAS_PER_SM);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool bf = dtype == VQB_DTYPE_BF16;
#define VQB_FSP_BWD(DD)                                                                                                     \
  if (inv) {                                                                                                                \
    if (bf) fsp_backward_kernel<ACT_TANH, true, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);                                  \
    else fsp_backward_kernel<ACT_TANH, true, false, DD><<<grid, FSP_THREADS, 0, s>>>(a);                                    \
  } else {                                                                                                                  \
    switch (act) {                                                                                                          \
      case ACT_TANH: if (bf) fsp_backward_kernel<ACT_TANH, false, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);                \
                     else fsp_backward_kernel<ACT_TANH, false, false, DD><<<grid, FSP_THREADS, 0, s>>>(a); break;           \
      case ACT_SIGMOID: if (bf) fsp_backward_kernel<ACT_SIGMOID, false, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);          \
                        else fsp_backward_kernel<ACT_SIGMOID, false, false, DD><<<grid, FSP_THREADS, 0, s>>>(a); break;     \
      case ACT_NORMAL: if (bf) fsp_backward_kernel<ACT_NORMAL, false, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);            \
                       else fsp_backward_kernel<ACT_NORMAL, false, false, DD><<<grid, FSP_THREADS, 0, s>>>(a); break;       \
      case ACT_LAPLACE: if (bf) fsp_backward_kernel<ACT_LAPLACE, false, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);          \
                        else fsp_backward_kernel<ACT_LAPLACE, false, false, DD><<<grid, FSP_THREADS, 0, s>>>(a); break;     \
      default: if (bf) fsp_backward_kernel<ACT_CAUCHY, false, true, DD><<<grid, FSP_THREADS, 0, s>>>(a);                    \
               else fsp_backward_kernel<ACT_CAUCHY, false, false, DD><<<grid, FSP_THREADS, 0, s>>>(a); break;               \
    }                                                                                                                       \
  }
  VQB_SWITCH_D(VQB_FSP_BWD)
#undef VQB_FSP_BWD
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fsp_decode(const void* idx, int idx64, int64_t N, int D, int act, int inv, const int32_t* levels, float lo,
                              float hi, float* act_out, float* codes, void* stream) {
  using namespace vqb;
  if (!idx || !levels || (!act_out && !codes)) return VQB_E_INVALID;
  if (act < ACT_TANH || act > ACT_CAUCHY) return VQB_E_INVALID;
  if (const int rc = fsp_shape(N, D, VQB_DTYPE_F32)) return rc;
  if ((act_out && !aligned(act_out, 16)) || (codes && !aligned(codes, 16))) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(N, FSP_THREADS, FSP_CTAS_PER_SM);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define VQB_FSP_DEC_LAUNCH(A, I, DD) fsp_decode_kernel<A, I, DD><<<grid, FSP_THREADS, 0, s>>>(idx, idx64, N, levels, lo, hi, act_out, codes)
#define VQB_FSP_DEC(DD)                                                                                                     \
  if (!inv) VQB_FSP_DEC_LAUNCH(ACT_TANH, false, DD);                                                                        \
  else switch (act) {                                                                                                       \
    case ACT_TANH: VQB_FSP_DEC_LAUNCH(ACT_TANH, true, DD); break; case ACT_SIGMOID: VQB_FSP_DEC_LAUNCH(ACT_SIGMOID, true, DD); break; \
    case ACT_NORMAL: VQB_FSP_DEC_LAUNCH(ACT_NORMAL, true, DD); break; case ACT_LAPLACE: VQB_FSP_DEC_LAUNCH(ACT_LAPLACE, true, DD); break; \
    default: VQB_FSP_DEC_LAUNCH(ACT_CAUCHY, true, DD); break;                                                               \
  }
  VQB_SWITCH_D(VQB_FSP_DEC)
#undef VQB_FSP_DEC
#undef VQB_FSP_DEC_LAUNCH
  return static_cast<int>(cudaGetLastError());
}
