// RandomProjectionQuantizer (random_projection_quantizer.py, "rpq"): the layer norm and the random projection in front of the
// cosine search, in one fp32 pass over x (rpq:49-53):
//
//   rows[r, h E + j] = sum_d LN(x[r, :])[d] * proj[h, d, j]      LN(v) = (v - mean) / sqrt(var + 1e-5), biased var
//
// One CTA owns a tile of BM rows and BN output columns.  It first takes the mean and the biased variance of each of its rows
// (two passes over the row, warp per row, fp32), then runs a tiled fp32 product on the CUDA cores over `dim` in steps of BK:
// the x tile is normalised as it is written to shared memory, so the normalised x never reaches global memory, and the
// projection is read in its (H, dim, E) layout, so the (dim, H E) matrix of the einsum is never formed.  No TF32: the
// reference's einsum is a full fp32 product.  The column tiles of one row tile are adjacent in launch order, so the x rows of
// the statistics pass and of the product (and of every column tile) are one read from HBM and re-reads from L2.
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int RPQ_THREADS = 256;
constexpr int RPQ_MAX_WIDTH = 1024;     // H E: the widest rows the search takes
constexpr int RPQ_MAX_DIM = 1 << 16;
constexpr float RPQ_EPS = 1e-5f;        // nn.LayerNorm's default

// Row (column) of a thread's i-th accumulator: 8-wide thread tiles are split into two 4-wide halves BM/2 apart, so the float4
// reads of a quarter warp from shared memory hit distinct banks.
template <int B, int T>
__device__ __forceinline__ int tile_pos(int t, int i) {
  if constexpr (T == 8) return (i >> 2) * (B / 2) + t * 4 + (i & 3);
  return t * T + i;
}

template <int BM, int BN, int TM, int TN, int BK>
__global__ void __launch_bounds__(RPQ_THREADS, 2) rpq_norm_project_kernel(const float* __restrict__ x, int64_t N, int dim,
                                                                       const float* __restrict__ proj, int H, int E, int norm,
                                                                       float* __restrict__ rows) {
  static_assert((BM / TM) * (BN / TN) == RPQ_THREADS, "one accumulator tile per thread");
  static_assert((BK * BM) % RPQ_THREADS == 0 && (BK * BN) % RPQ_THREADS == 0, "whole staging loads per thread");
  constexpr int A_LOADS = BK * BM / RPQ_THREADS, B_LOADS = BK * BN / RPQ_THREADS;
  constexpr int AS = BM + 4;   // padded row of the transposed x tile: 16-byte aligned, at most 2-way conflicts on the store
  __shared__ __align__(16) float sA[BK][AS];
  __shared__ __align__(16) float sB[BK][BN];
  __shared__ float s_mean[BM], s_rstd[BM];

  const int W = H * E;
  const int n_col = (W + BN - 1) / BN;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x / n_col) * BM;
  const int c0 = (blockIdx.x % n_col) * BN;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- row statistics: mean, then the mean of the squared deviations (two passes, no cancellation)
  for (int m = warp; m < BM; m += RPQ_THREADS / 32) {
    const int64_t r = r0 + m;
    float mean = 0.f, rstd = 0.f;
    if (r < N) {
      if (norm) {
        const float* xr = x + r * dim;
        float s = 0.f;
        for (int k = lane; k < dim; k += 32) s += xr[k];
        mean = warp_sum(s) / static_cast<float>(dim);
        float ss = 0.f;
        for (int k = lane; k < dim; k += 32) {
          const float d = xr[k] - mean;
          ss += d * d;
        }
        rstd = 1.f / sqrtf(warp_sum(ss) / static_cast<float>(dim) + RPQ_EPS);
      } else {
        rstd = 1.f;   // (v - 0) * 1 == v: the staging below passes x through unchanged
      }
    }
    if (lane == 0) {
      s_mean[m] = mean;
      s_rstd[m] = rstd;
    }
  }
  __syncthreads();

  // staging: a thread loads column a_k of rows a_m + i (THREADS / BK) of the (BM x BK) x tile (16 consecutive floats of a row
  // per 16 threads), and column b_c of rows b_k + i (THREADS / BN) of the (BK x BN) projection tile
  static_assert(RPQ_THREADS % BK == 0 && RPQ_THREADS % BN == 0, "a fixed staging column per thread");
  const int a_k = tid % BK, a_m = tid / BK, b_c = tid % BN, b_k = tid / BN;
  const float* xa = x + (r0 + a_m) * dim + a_k;
  const int64_t a_rows = N - r0 - a_m;   // rows a_m + i (THREADS / BK) < a_rows exist
  const int bc = c0 + b_c;
  const float* pb = proj + (bc < W ? (static_cast<int64_t>(bc / E) * dim) * E + bc % E : 0);
  float ra[A_LOADS], rb[B_LOADS];
  auto load = [&](int k0) {
#pragma unroll
    for (int i = 0; i < A_LOADS; ++i) {
      const int m = i * (RPQ_THREADS / BK);
      ra[i] = (m < a_rows && k0 + a_k < dim) ? xa[static_cast<int64_t>(m) * dim + k0] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < B_LOADS; ++i) {
      const int k = k0 + b_k + i * (RPQ_THREADS / BN);
      rb[i] = (k < dim && bc < W) ? pb[static_cast<int64_t>(k) * E] : 0.f;
    }
  };
  auto stage = [&]() {
#pragma unroll
    for (int i = 0; i < A_LOADS; ++i) {
      const int m = a_m + i * (RPQ_THREADS / BK);
      sA[a_k][m] = (ra[i] - s_mean[m]) * s_rstd[m];   // rows past N: (0 - 0) * 0
    }
#pragma unroll
    for (int i = 0; i < B_LOADS; ++i) sB[b_k + i * (RPQ_THREADS / BN)][b_c] = rb[i];
  };

  const int tn = tid % (BN / TN), tm = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load(0);
  for (int k0 = 0; k0 < dim; k0 += BK) {
    stage();
    __syncthreads();
    if (k0 + BK < dim) load(k0 + BK);   // the next tile's global reads overlap this tile's FMAs
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&sA[k][tile_pos<BM, TM>(tm, i)]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
      if constexpr (TN % 4 == 0) {
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&sB[k][tile_pos<BN, TN>(tn, j)]);
          b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = sB[k][tile_pos<BN, TN>(tn, j)];
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t r = r0 + tile_pos<BM, TM>(tm, i);
    if (r >= N) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int c = c0 + tile_pos<BN, TN>(tn, j);
      if (c < W) rows[r * W + c] = acc[i][j];
    }
  }
}

template <int BM, int BN, int TM, int TN, int BK>
int launch(const float* x, int64_t N, int dim, const float* proj, int H, int E, int norm, float* rows, cudaStream_t stream) {
  const int64_t W = static_cast<int64_t>(H) * E;
  const int64_t ctas = ((N + BM - 1) / BM) * ((W + BN - 1) / BN);
  if (ctas > 0x7fffffff) return VQB_E_UNSUPPORTED;
  rpq_norm_project_kernel<BM, BN, TM, TN, BK><<<static_cast<unsigned>(ctas), RPQ_THREADS, 0, stream>>>(x, N, dim, proj, H, E, norm,
                                                                                                  rows);
  return static_cast<int>(cudaGetLastError());
}

bool aligned4(const void* p) { return aligned(p, 4); }

}  // namespace
}  // namespace vqb

extern "C" int vqb_rpq_norm_project(const float* x, int64_t N, int dim, const float* proj, int H, int E, int norm, float* rows,
                                    void* stream) {
  using namespace vqb;
  if (!x || !proj || !rows || N <= 0 || dim <= 0 || H <= 0 || E <= 0 || (norm != 0 && norm != 1)) return VQB_E_INVALID;
  const int64_t W = static_cast<int64_t>(H) * E;
  if (W > RPQ_MAX_WIDTH || dim > RPQ_MAX_DIM) return VQB_E_UNSUPPORTED;
  const int64_t lim = int64_t{1} << 40;
  if (N > lim / dim || N > lim / W) return VQB_E_UNSUPPORTED;
  if (!aligned4(x) || !aligned4(proj) || !aligned4(rows)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // a 16-wide projection (BEST-RQ) reads x at the HBM rate without spending FMAs on padding columns; wider ones take 8 x 4
  // thread tiles, the widest that keep every kernel within 128 registers without spills (two CTAs per SM)
  if (W <= 16) return launch<64, 16, 4, 1, 16>(x, N, dim, proj, H, E, norm, rows, s);
  return launch<128, 64, 8, 4, 16>(x, N, dim, proj, H, E, norm, rows, s);
}
