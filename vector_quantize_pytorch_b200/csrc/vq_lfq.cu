// Lookup-free quantization: LFQ (lookup_free_quantization.py, "lfq"), ResidualLFQ and GroupedResidualLFQ (residual_lfq.py,
// "rlfq").  Five kernels:
//
//   lfq_forward_kernel         one thread per (row, group) item, its D <= 20 values in registers, every stage q < n_active:
//                              soft clamp (lfq:295-297), spherical l2norm (lfq:308), sign and index bits (lfq:326-331), the
//                              straight-through value x + (q - x) (lfq:341), the residual and the running sum (rlfq:189-190);
//                              in training it also writes the stage's entropy input and the commitment partial sums.
//   lfq_entropy_kernel         the entropy statistics of lfq:365-398 without the (N, K) matrix: the softmax over {+-m}^D
//                              factorises into per-bit Bernoullis, ln p[k] = TA[k_hi] + TB[k_lo] (DESIGN 4.10), so a CTA streams
//                              a K tile for a chunk of rows with one ex2 per (row, code), and writes the sum of h(p) and the
//                              column sums of p.
//   lfq_entropy_bwd_kernel     d/d(entropy input) given the gradients of those two outputs: one thread per row streams its K
//                              range, accumulating the sign-weighted sums of w = p u; lfq_entropy_fin_kernel adds the K splits.
//   lfq_backward_kernel        d z of the whole chain: grad_out, the entropy gradient and the commitment gradient through the
//                              l2norm, the soft clamp and the residual chain, every stage recomputed from z.
//   lfq_decode_kernel          indices -> +-m codes and / or their sum over the stages (lfq:228-263, rlfq:101-136).
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int LFQ_THREADS = 256;
constexpr int LFQ_CTAS_PER_SM = 8;   // grid cap; vqb_lfq_forward_blocks reports the grid, which orders the partial sums
constexpr int LFQ_MAX_D = 20;
constexpr int LFQ_MAX_Q = 64;
constexpr int ENT_THREADS = 256;   // entropy forward: codes across threads
constexpr int ENT_RB = 32;         // rows staged per batch
constexpr int ENT_HT = 16;         // k_hi values per thread (a tile is ENT_HT x 2^l codes)
constexpr int EB_THREADS = 128;    // entropy backward: rows across threads
constexpr int EB_VT = 2048;        // codes of the gradient table staged per step
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;
constexpr float LOG2_EPS = -16.609640474436812f;   // log2(1e-5): p >= 1e-5  <=>  log2 p >= LOG2_EPS
constexpr float LN_EPS = -11.512925464970229f;     // ln(1e-5)

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// -softplus(y) / ln 2, the log2 of sigmoid(-y)
__device__ __forceinline__ float neg_softplus2(float y) { return -(fmaxf(y, 0.f) + log1pf(expf(-fabsf(y)))) * LOG2E; }

struct StageParams {   // per stage, in shared memory
  float s[LFQ_MAX_Q];    // codebook_scale
  float m[LFQ_MAX_Q];    // code magnitude: s, or the reference's l2norm(+-s) * s when spherical
  float c[LFQ_MAX_Q];    // soft-clamp value (0: none)
};

__device__ __forceinline__ void load_params(StageParams& p, const float* params, int Q) {
  for (int i = threadIdx.x; i < 3 * Q; i += blockDim.x) (&p.s[0])[(i / Q) * LFQ_MAX_Q + i % Q] = params[i];
  __syncthreads();
}

// One stage's input transform, in the work dtype W (rounded after every op as torch does): the soft clamp tanh(x / c) * c,
// then the spherical x / max(||x||, 1e-12) * s.  Returns ||x|| rounded to W, before the clamp, for the backward; t receives
// the tanh.
template <bool BF>
__device__ __forceinline__ float stage_input(float (&x)[LFQ_MAX_D], float (&t)[LFQ_MAX_D], int D, float c, bool sph, float s) {
  if (c != 0.f) {
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j)
      if (j < D) {
        t[j] = rw<BF>(tanhf(rw<BF>(__fdiv_rn(x[j], c))));
        x[j] = rw<BF>(__fmul_rn(t[j], c));
      }
  }
  float rn = 1.f;
  if (sph) {
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j)
      if (j < D) ss = __fmaf_rn(x[j], x[j], ss);
    rn = rw<BF>(__fsqrt_rn(ss));
    const float nrm = fmaxf(rn, rw<BF>(1e-12f));
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j)
      if (j < D) x[j] = rw<BF>(__fmul_rn(rw<BF>(__fdiv_rn(x[j], nrm)), s));
  }
  return rn;
}

struct FwdArgs {
  const void* z;
  int64_t N;
  int G, D, Q, n_active, residual, training, sph;
  const float* params;   // [3][Q]: s, m, c
};

template <int DT, bool BF>
__global__ void __launch_bounds__(LFQ_THREADS) lfq_forward_kernel(FwdArgs a, void* __restrict__ out, void* __restrict__ idx, int idx64,
                                                                  int64_t s_row, int64_t s_g, int64_t s_q, float* __restrict__ ent,
                                                                  const uint8_t* __restrict__ rowmask, double* __restrict__ commit) {
  __shared__ StageParams P;
  __shared__ double red[LFQ_THREADS / 32];
  load_params(P, a.params, a.Q);
  constexpr int WT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  const int D = a.D;
  const int64_t items = a.N * a.G;
  // the commitment partials, one per stage (n_active <= LFQ_MAX_Q, indexed by the stage: local memory, touched once per item
  // and stage)
  double cacc[LFQ_MAX_Q];
  for (int q = 0; q < a.n_active; ++q) cacc[q] = 0.0;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = it / a.G, g = it - row * a.G;
    const bool live = rowmask == nullptr || rowmask[row] != 0;
    float r[LFQ_MAX_D], o[LFQ_MAX_D], x[LFQ_MAX_D], t[LFQ_MAX_D];
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j) {
      r[j] = j < D ? Elem<DT>::load(a.z, it * D + j) : 0.f;
      o[j] = 0.f;
    }
    const int64_t ibase = row * s_row + g * s_g;
    for (int q = 0; q < a.n_active; ++q) {
      const float s = P.s[q], m = P.m[q];
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j) x[j] = r[j];
      stage_input<BF>(x, t, D, P.c[q], a.sph, s);
      int64_t index = 0;
      double cq = 0.0;
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < D) {
          const float xi = x[j];   // original_input (fp32; exact from W)
          const bool pos = xi > 0.f;
          const float qv = pos ? m : -m;
          if (pos) index |= int64_t{1} << (D - 1 - j);
          const float ov = rw<BF>(a.training ? __fadd_rn(xi, __fsub_rn(qv, xi)) : qv);   // lfq:341, then .type(orig_dtype)
          if (ent) ent[(static_cast<int64_t>(q) * items + it) * D + j] = xi;
          const float e = __fsub_rn(xi, qv);
          cq += static_cast<double>(__fmul_rn(e, e));
          r[j] = rw<BF>(__fsub_rn(r[j], ov));                                        // rlfq:189
          o[j] = a.residual ? rw<BF>(__fadd_rn(o[j], ov)) : ov;                      // rlfq:190 (0. + q at stage 0)
        }
      if (live) cacc[q] += cq;
      reinterpret_cast<int64_t*>(idx)[ibase + q * s_q] = index;
    }
    for (int q = a.n_active; q < a.Q; ++q) reinterpret_cast<int64_t*>(idx)[ibase + q * s_q] = -1;   // rlfq:182-185
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j)
      if (j < D) Elem<WT>::store(out, it * D + j, o[j]);
  }
  (void)idx64;
  if (commit) {   // fixed-order block sums: commit[q][blockIdx.x]
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int q = 0; q < a.n_active; ++q) {
      double v = warp_sum(cacc[q]);
      if (lane == 0) red[w] = v;
      __syncthreads();
      if (threadIdx.x == 0) {
        double tsum = 0.0;
        for (int i = 0; i < LFQ_THREADS / 32; ++i) tsum += red[i];
        commit[static_cast<int64_t>(q) * gridDim.x + blockIdx.x] = tsum;
      }
      __syncthreads();
    }
  }
}

// ---- entropy statistics ----

struct EntArgs {
  const float* x;        // [S][N][G][D] entropy inputs (fp32)
  int64_t N;
  int G, D, SG;
  const int32_t* rows;   // [SG][rs] row list or null (rows 0..R-1)
  int64_t R, rs;
  const float* m;        // [S] code magnitude
  float tau;
};

__device__ __forceinline__ const float* ent_row(const EntArgs& a, int sg, int64_t r) {
  const int s = sg / a.G, g = sg - s * a.G;
  const int64_t n = a.rows ? a.rows[sg * a.rs + r] : r;
  return a.x + ((static_cast<int64_t>(s) * a.N + n) * a.G + g) * a.D;
}

// grid (ntiles, nchunks, SG).  Thread t: k_lo = t % 2^l, row lane t / 2^l; k = (hi0 + i) 2^l + k_lo for i < HT.
__global__ void __launch_bounds__(ENT_THREADS) lfq_entropy_kernel(EntArgs a, int64_t chunk_rows, double* __restrict__ pse,
                                                                  float* __restrict__ colsum) {
  __shared__ float ell[ENT_RB][LFQ_MAX_D][2];
  __shared__ float ta[ENT_RB][ENT_HT];
  __shared__ double red[ENT_THREADS / 32];
  __shared__ float lanesum[ENT_THREADS];
  const int D = a.D, l = D < 8 ? D : 8, h = D - l, L = 1 << l, lanes = ENT_THREADS / L;
  const int HT = (1 << h) < ENT_HT ? (1 << h) : ENT_HT;
  const int tile = blockIdx.x, chunk = blockIdx.y, sg = blockIdx.z;
  const int hi0 = tile * HT;
  const int t = threadIdx.x, klo = t % L, lane = t / L;
  const float tm = __fmul_rn(__fmul_rn(2.f, a.tau), a.m[sg / a.G]);
  const int64_t r0 = chunk * chunk_rows;
  const int64_t r1 = r0 + chunk_rows < a.R ? r0 + chunk_rows : a.R;
  float col[ENT_HT];
#pragma unroll
  for (int i = 0; i < ENT_HT; ++i) col[i] = 0.f;
  double hacc = 0.0;
  for (int64_t rb = r0; rb < r1; rb += ENT_RB) {
    const int nb = static_cast<int>(r1 - rb < ENT_RB ? r1 - rb : ENT_RB);
    __syncthreads();
    for (int i = t; i < nb * D; i += ENT_THREADS) {
      const int rr = i / D, j = i - rr * D;
      const float av = __fmul_rn(tm, ent_row(a, sg, rb + rr)[j]);
      ell[rr][j][1] = neg_softplus2(-2.f * av);
      ell[rr][j][0] = neg_softplus2(2.f * av);
    }
    __syncthreads();
    for (int i = t; i < nb * HT; i += ENT_THREADS) {
      const int rr = i / HT, hi = hi0 + i % HT;
      float v = 0.f;
      for (int j = 0; j < h; ++j) v += ell[rr][j][(hi >> (h - 1 - j)) & 1];
      ta[rr][i % HT] = v;
    }
    __syncthreads();
    for (int rr = lane; rr < nb; rr += lanes) {
      float tb = 0.f;
      for (int j = h; j < D; ++j) tb += ell[rr][j][(klo >> (D - 1 - j)) & 1];
      float hs = 0.f;
#pragma unroll
      for (int i = 0; i < ENT_HT; ++i)
        if (i < HT) {
          const float lp = ta[rr][i] + tb;   // log2 p
          const float p = ex2(lp);
          col[i] += p;
          hs = __fmaf_rn(-p, lp >= LOG2_EPS ? lp * LN2 : LN_EPS, hs);
        }
      hacc += static_cast<double>(hs);
    }
  }
  // PSE partial: fixed-order block reduction
  const double hv = warp_sum(hacc);
  if ((t & 31) == 0) red[t >> 5] = hv;
  __syncthreads();
  if (t == 0) {
    double v = 0.0;
    for (int i = 0; i < ENT_THREADS / 32; ++i) v += red[i];
    pse[(static_cast<int64_t>(sg) * gridDim.y + chunk) * gridDim.x + tile] = v;
  }
  if (!colsum) return;
  const int64_t K = int64_t{1} << D;
  float* dst = colsum + (static_cast<int64_t>(chunk) * a.SG + sg) * K;
  if (lanes == 1) {
#pragma unroll
    for (int i = 0; i < ENT_HT; ++i)
      if (i < HT) dst[static_cast<int64_t>(hi0 + i) * L + klo] = col[i];
    return;
  }
  // several row lanes (D < 8): add the lanes in lane order.  HT = 1 here (h = 0).
  lanesum[t] = col[0];
  __syncthreads();
  if (t < L) {
    float v = 0.f;
    for (int ln = 0; ln < lanes; ++ln) v += lanesum[ln * L + t];
    dst[t] = v;
  }
}

// Entropy backward.  grid (ceil(R / EB_THREADS), SG, ksplit); thread = one row, codes [ks Kc, (ks + 1) Kc).
// u[k] = cp[sg] h'(p[k]) + V[sg][k] (h'(p) = -(ln p + 1), or -ln 1e-5 below the clamp); w = p u.
// part[ks][sg][r][0..D-1] = sum_k w sgn_kj, part[..][D] = sum_k w.
__global__ void __launch_bounds__(EB_THREADS) lfq_entropy_bwd_kernel(EntArgs a, const float* __restrict__ cp, const float* __restrict__ V,
                                                                     int64_t Kc, float* __restrict__ part) {
  __shared__ float vt[EB_VT];
  const int D = a.D, l = D < 4 ? D : 4, h = D - l, L = 1 << l;
  const int sg = blockIdx.y, ks = blockIdx.z;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * EB_THREADS + threadIdx.x;
  const bool valid = r < a.R;
  const int64_t K = int64_t{1} << D;
  const float tm = __fmul_rn(__fmul_rn(2.f, a.tau), a.m[sg / a.G]);
  const float c = cp[sg];
  float l1[LFQ_MAX_D], l0[LFQ_MAX_D];
  const float* xr = valid ? ent_row(a, sg, r) : nullptr;
#pragma unroll
  for (int j = 0; j < LFQ_MAX_D; ++j) {
    const float av = (valid && j < D) ? __fmul_rn(tm, xr[j]) : 0.f;
    l1[j] = neg_softplus2(-2.f * av);
    l0[j] = neg_softplus2(2.f * av);
  }
  float tb[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    float v = 0.f;
#pragma unroll
    for (int b = 0; b < 4; ++b)
      if (b < l) {
        const int j = D - 1 - b;
        float sel = 0.f;
#pragma unroll
        for (int jj = 0; jj < LFQ_MAX_D; ++jj)
          if (jj == j) sel = ((i >> b) & 1) ? l1[jj] : l0[jj];
        v += sel;
      }
    tb[i] = v;
  }
  // fp32 sums over the 16 codes of one k_hi step, added to fp64 accumulators (K can be 2^20 terms per row)
  double acc[LFQ_MAX_D], accl[4] = {0.0, 0.0, 0.0, 0.0}, tot = 0.0;
#pragma unroll
  for (int j = 0; j < LFQ_MAX_D; ++j) acc[j] = 0.0;
  const float* Vs = V ? V + static_cast<int64_t>(sg) * K : nullptr;
  for (int64_t k0 = ks * Kc; k0 < (ks + 1) * Kc; k0 += EB_VT) {
    const int nv = static_cast<int>(Kc < EB_VT ? Kc : EB_VT);
    __syncthreads();
    for (int i = threadIdx.x; i < nv; i += EB_THREADS) vt[i] = Vs ? Vs[k0 + i] : 0.f;
    __syncthreads();
    if (!valid) continue;
    for (int kk = 0; kk < nv; kk += L) {
      const int64_t hi = (k0 + kk) >> l;
      float ta = 0.f;
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < h) ta += ((hi >> (h - 1 - j)) & 1) ? l1[j] : l0[j];
      float S = 0.f, sl[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 16; ++i)
        if (i < L) {
          const float lp = ta + tb[i];
          const float p = ex2(lp);
          const float hp = lp >= LOG2_EPS ? -__fmaf_rn(lp, LN2, 1.f) : -LN_EPS;
          const float w = p * __fmaf_rn(c, hp, vt[kk + i]);
          S += w;
#pragma unroll
          for (int b = 0; b < 4; ++b) sl[b] += ((i >> b) & 1) ? w : -w;   // k_lo bit b is dimension D - 1 - b
        }
#pragma unroll
      for (int b = 0; b < 4; ++b) accl[b] += static_cast<double>(sl[b]);
      tot += static_cast<double>(S);
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < h) acc[j] += static_cast<double>(((hi >> (h - 1 - j)) & 1) ? S : -S);
    }
  }
  if (!valid) return;
  float* dst = part + ((static_cast<int64_t>(ks) * a.SG + sg) * a.R + r) * (D + 1);
#pragma unroll
  for (int j = 0; j < LFQ_MAX_D; ++j)
    if (j < h) dst[j] = static_cast<float>(acc[j]);
#pragma unroll
  for (int b = 0; b < 4; ++b)
    if (b < l) dst[D - 1 - b] = static_cast<float>(accl[b]);
  dst[D] = static_cast<float>(tot);
}

// grad[row] = 2 tau m (sum_k w sgn_kj - (sum_k w) tanh(a_j)), the K splits added in order.
__global__ void lfq_entropy_fin_kernel(EntArgs a, const float* __restrict__ part, int ksplit, float* __restrict__ grad) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= a.SG * a.R) return;
  const int sg = static_cast<int>(i / a.R);
  const int64_t r = i - static_cast<int64_t>(sg) * a.R;
  const int D = a.D;
  const float tm = __fmul_rn(__fmul_rn(2.f, a.tau), a.m[sg / a.G]);
  const float* xr = ent_row(a, sg, r);
  float* gr = grad + (xr - a.x);
  float tot = 0.f;
  for (int ks = 0; ks < ksplit; ++ks) tot += part[((static_cast<int64_t>(ks) * a.SG + sg) * a.R + r) * (D + 1) + D];
  for (int j = 0; j < D; ++j) {
    float sj = 0.f;
    for (int ks = 0; ks < ksplit; ++ks) sj += part[((static_cast<int64_t>(ks) * a.SG + sg) * a.R + r) * (D + 1) + j];
    gr[j] = tm * (sj - tot * tanhf(__fmul_rn(tm, xr[j])));
  }
}

// ---- backward of the row chain ----

template <int DT, bool BF>
__global__ void __launch_bounds__(LFQ_THREADS) lfq_backward_kernel(FwdArgs a, const void* __restrict__ gout, const float* __restrict__ gent,
                                                                   const float* __restrict__ cc, const uint8_t* __restrict__ rowmask,
                                                                   void* __restrict__ gz) {
  __shared__ StageParams P;
  load_params(P, a.params, a.Q);
  constexpr int WT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  const int D = a.D;
  const int64_t items = a.N * a.G;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = it / a.G;
    const bool live = rowmask == nullptr || rowmask[row] != 0;
    float r[LFQ_MAX_D], go[LFQ_MAX_D], acc[LFQ_MAX_D], x[LFQ_MAX_D], t[LFQ_MAX_D], g[LFQ_MAX_D];
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j) {
      r[j] = j < D ? Elem<DT>::load(a.z, it * D + j) : 0.f;
      go[j] = j < D ? Elem<WT>::load(gout, it * D + j) : 0.f;
      acc[j] = 0.f;
      t[j] = 0.f;
    }
    for (int q = 0; q < a.n_active; ++q) {
      const float s = P.s[q], m = P.m[q], c = P.c[q];
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j) x[j] = r[j];
      const float rn = stage_input<BF>(x, t, D, c, a.sph, s);
      const float nrm = fmaxf(rn, rw<BF>(1e-12f));
      const float ccq = (cc && live) ? cc[q] : 0.f;
      // d original_input: the straight-through gradient, the entropy gradient, the commitment gradient (2 (x - q) per unit)
      float dot = 0.f;
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < D) {
          const float qv = x[j] > 0.f ? m : -m;
          float gi = a.training ? go[j] : 0.f;   // in eval the value is q itself: no gradient reaches x
          if (gent) gi += gent[(static_cast<int64_t>(q) * items + it) * D + j];
          if (ccq != 0.f) gi += ccq * (x[j] - qv);
          g[j] = rw<BF>(gi);                       // x.float() backward: the gradient returns in W
          if (a.sph) {
            g[j] = rw<BF>(g[j] * s);               // * codebook_scale
            dot += g[j] * (x[j] / s);              // y = x / s is the normalised vector
          }
        }
      // below the clamp x / eps is linear in x: clamp_min passes the norm's gradient only where ||x|| >= eps, so no projection
      if (!(rn >= rw<BF>(1e-12f))) dot = 0.f;
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < D) {
          float gx = g[j];
          if (a.sph) gx = (g[j] - (x[j] / s) * dot) / nrm;   // F.normalize backward
          if (c != 0.f) gx = gx * (1.f - t[j] * t[j]);     // tanh(x / c) * c backward
          acc[j] += rw<BF>(gx);
          const float qv = x[j] > 0.f ? m : -m;
          const float ov = rw<BF>(a.training ? __fadd_rn(x[j], __fsub_rn(qv, x[j])) : qv);
          r[j] = rw<BF>(__fsub_rn(r[j], ov));
        }
    }
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j)
      if (j < D) Elem<DT>::store(gz, it * D + j, acc[j]);
  }
}

// indices -> codes.  vals [Q]: the +-value of stage q's codes.  codes [Q][N][G][D] and / or out [N][G][D] (sum over q), fp32.
__global__ void __launch_bounds__(LFQ_THREADS) lfq_decode_kernel(const void* __restrict__ idx, int idx64, int64_t s_row, int64_t s_g,
                                                                 int64_t s_q, int64_t N, int G, int D, int Q, const float* __restrict__ vals,
                                                                 float* __restrict__ out, float* __restrict__ codes) {
  const int64_t items = N * G;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = it / G, g = it - row * G;
    float acc[LFQ_MAX_D];
#pragma unroll
    for (int j = 0; j < LFQ_MAX_D; ++j) acc[j] = 0.f;
    for (int q = 0; q < Q; ++q) {
      const int64_t ix = load_index(idx, idx64, row * s_row + g * s_g + q * s_q);
      const float v = vals[q];
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < D) {
          const float c = ix == -1 ? 0.f : (((ix >> (D - 1 - j)) & 1) ? v : -v);
          if (codes) codes[(static_cast<int64_t>(q) * items + it) * D + j] = c;
          acc[j] = __fadd_rn(acc[j], c);
        }
    }
    if (out) {
#pragma unroll
      for (int j = 0; j < LFQ_MAX_D; ++j)
        if (j < D) out[it * D + j] = acc[j];
    }
  }
}

int check_fwd(const FwdArgs& a, int in_dtype, int work_dtype) {
  if (!a.z || !a.params || a.N <= 0 || a.G <= 0 || a.Q <= 0 || a.n_active < 1 || a.n_active > a.Q) return VQB_E_INVALID;
  if (a.D < 1 || a.D > LFQ_MAX_D || a.Q > LFQ_MAX_Q || a.N * a.G >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if ((in_dtype != VQB_DTYPE_F32 && in_dtype != VQB_DTYPE_BF16) || (work_dtype != VQB_DTYPE_F32 && work_dtype != VQB_DTYPE_BF16))
    return VQB_E_INVALID;
  if (in_dtype != work_dtype) return VQB_E_UNSUPPORTED;   // the reference's chain runs in the input dtype
  return VQB_OK;
}

int check_ent(const EntArgs& a) {
  if (!a.x || !a.m || a.N <= 0 || a.G <= 0 || a.SG <= 0 || a.R <= 0 || a.SG % a.G != 0) return VQB_E_INVALID;
  if (a.D < 1 || a.D > LFQ_MAX_D || a.R >= (int64_t{1} << 31) || a.SG > 65535) return VQB_E_UNSUPPORTED;
  if (!a.rows && a.R > a.N) return VQB_E_INVALID;
  if (a.rs < 0) return VQB_E_INVALID;
  return VQB_OK;
}

}  // namespace
}  // namespace vqb

extern "C" int vqb_lfq_forward(const void* z, int dtype, int64_t N, int G, int D, int Q, int n_active, int residual, int training,
                               int spherical, const float* params, void* out, void* idx, int64_t idx_s_row, int64_t idx_s_g,
                               int64_t idx_s_q, float* ent, const uint8_t* rowmask, double* commit, int commit_blocks, void* stream) {
  using namespace vqb;
  const FwdArgs a{z, N, G, D, Q, n_active, residual, training, spherical, params};
  if (!out || !idx) return VQB_E_INVALID;
  if (const int rc = check_fwd(a, dtype, dtype)) return rc;
  if (commit && commit_blocks <= 0) return VQB_E_INVALID;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(N * G, LFQ_THREADS, LFQ_CTAS_PER_SM);
  if (commit && commit_blocks != grid) return VQB_E_INVALID;   // vqb_lfq_forward_blocks() sizes the partials
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == VQB_DTYPE_F32)
    lfq_forward_kernel<VQB_DTYPE_F32, false><<<grid, LFQ_THREADS, 0, s>>>(a, out, idx, 1, idx_s_row, idx_s_g, idx_s_q, ent, rowmask, commit);
  else
    lfq_forward_kernel<VQB_DTYPE_BF16, true><<<grid, LFQ_THREADS, 0, s>>>(a, out, idx, 1, idx_s_row, idx_s_g, idx_s_q, ent, rowmask, commit);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lfq_forward_blocks(int64_t N, int G) {
  if (N <= 0 || G <= 0) return VQB_E_INVALID;
  if (const int rc = vqb::check_device()) return rc;
  return vqb::capped_grid(N * G, vqb::LFQ_THREADS, vqb::LFQ_CTAS_PER_SM);
}

extern "C" int vqb_lfq_entropy(const float* x, int64_t N, int G, int D, int S, const int32_t* rows, int64_t R, int64_t rows_stride,
                               const float* m, float tau, int chunks, double* pse, float* colsum, void* stream) {
  using namespace vqb;
  const EntArgs a{x, N, G, D, S * G, rows, R, rows_stride, m, tau};
  if (!pse || S <= 0 || chunks < 1) return VQB_E_INVALID;
  if (const int rc = check_ent(a)) return rc;
  if (chunks > 65535 || chunks > R) return VQB_E_INVALID;
  if (const int rc = check_device()) return rc;
  const int l = D < 8 ? D : 8, h = D - l;
  const int HT = (1 << h) < ENT_HT ? (1 << h) : ENT_HT;
  const int ntiles = (1 << h) / HT;
  const int64_t chunk_rows = (R + chunks - 1) / chunks;
  const dim3 grid(ntiles, chunks, a.SG);
  lfq_entropy_kernel<<<grid, ENT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a, chunk_rows, pse, colsum);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lfq_entropy_tiles(int D) {
  if (D < 1 || D > vqb::LFQ_MAX_D) return VQB_E_UNSUPPORTED;
  const int l = D < 8 ? D : 8, h = D - l;
  const int HT = (1 << h) < vqb::ENT_HT ? (1 << h) : vqb::ENT_HT;
  return (1 << h) / HT;
}

extern "C" int vqb_lfq_entropy_backward(const float* x, int64_t N, int G, int D, int S, const int32_t* rows, int64_t R,
                                        int64_t rows_stride, const float* m, float tau, const float* cp, const float* V, int ksplit,
                                        float* work, float* grad, void* stream) {
  using namespace vqb;
  const EntArgs a{x, N, G, D, S * G, rows, R, rows_stride, m, tau};
  if (!cp || !work || !grad || S <= 0 || ksplit < 1) return VQB_E_INVALID;
  if (const int rc = check_ent(a)) return rc;
  const int64_t K = int64_t{1} << D;
  const int64_t Kc = K / ksplit;
  if (Kc * ksplit != K || (ksplit & (ksplit - 1)) || (Kc < 16 && ksplit > 1) || ksplit > 65535) return VQB_E_INVALID;
  if (const int rc = check_device()) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dim3 grid(static_cast<unsigned>((R + EB_THREADS - 1) / EB_THREADS), a.SG, ksplit);
  lfq_entropy_bwd_kernel<<<grid, EB_THREADS, 0, s>>>(a, cp, V, Kc, work);
  const int64_t n = static_cast<int64_t>(a.SG) * R;
  lfq_entropy_fin_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(a, work, ksplit, grad);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lfq_backward(const void* z, int dtype, int64_t N, int G, int D, int Q, int n_active, int residual, int training,
                                int spherical, const float* params, const void* grad_out, const float* grad_ent, const float* cc,
                                const uint8_t* rowmask, void* grad_z, void* stream) {
  using namespace vqb;
  const FwdArgs a{z, N, G, D, Q, n_active, residual, training, spherical, params};
  if (!grad_out || !grad_z) return VQB_E_INVALID;
  if (const int rc = check_fwd(a, dtype, dtype)) return rc;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(N * G, LFQ_THREADS, LFQ_CTAS_PER_SM);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == VQB_DTYPE_F32)
    lfq_backward_kernel<VQB_DTYPE_F32, false><<<grid, LFQ_THREADS, 0, s>>>(a, grad_out, grad_ent, cc, rowmask, grad_z);
  else
    lfq_backward_kernel<VQB_DTYPE_BF16, true><<<grid, LFQ_THREADS, 0, s>>>(a, grad_out, grad_ent, cc, rowmask, grad_z);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_lfq_decode(const void* idx, int idx64, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, int64_t N, int G, int D,
                              int Q, const float* vals, float* out, float* codes, void* stream) {
  using namespace vqb;
  if (!idx || !vals || (!out && !codes) || N <= 0 || G <= 0 || Q <= 0) return VQB_E_INVALID;
  if (D < 1 || D > LFQ_MAX_D || Q > LFQ_MAX_Q || N * G >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(N * G, LFQ_THREADS, LFQ_CTAS_PER_SM);
  lfq_decode_kernel<<<grid, LFQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(idx, idx64, idx_s_row, idx_s_g, idx_s_q, N, G, D, Q,
                                                                                 vals, out, codes);
  return static_cast<int>(cudaGetLastError());
}
