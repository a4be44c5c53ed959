// ResidualSimVQ (residual_sim_vq.py:182-203 over sim_vq.py:100-138): the stage tail that follows each stage's search, and one
// backward kernel for all stages.  A warp per row, the row held in registers (element lane + 32 j in slot j).
//
// The reference subtracts the gradient estimator's FORWARD value from the residual (rsv:195), which is a few ulps away from
// the code row.  The backward recomputes every stage's residual from x instead of keeping Q x N x D of them, so the tail and
// the backward share `stage_value` below, written with explicitly rounded operations (no contraction the compiler could choose
// differently in the two kernels): the recomputed residuals are bit-identical to the forward's.
#include "vqb_common.cuh"

namespace vqb {
namespace {

constexpr int RS_THREADS = 256;   // 8 rows in flight per CTA
constexpr float RS_EPS = 1e-6f;   // safe_div / l2norm eps (vqp:37-41)

template <int J>
__device__ __forceinline__ void load_row(float (&v)[J], const float* __restrict__ p, int D, int lane) {
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const int i = lane + 32 * j;
    v[j] = i < D ? p[i] : 0.f;
  }
}

// Scalars of the rotation trick (vqp:287-318) for src s and tgt t, as in vq_aux.cu's rotate_kernel:
//   u = s / max(||s||, eps), q = t / max(||t||, eps), w = (u + q) / max(||u + q||, eps), lam = ||t|| / max(||s||, eps)
//   forward  out = (s - 2 (s.w) w + 2 (s.u) q) lam      backward  d_s = (g - 2 (g.w) w + 2 (g.q) u) lam
// Row reductions in double (exact products, see rotate_kernel for why fp32 is not enough near s = -t).
struct Rot {
  float ins, int_, inw, lam;
  float fa, fb;   // forward: s.w, s.u
  float ba, bb;   // backward: g.w, g.q
};

template <int J, bool BWD>
__device__ __forceinline__ Rot rot_setup(const float (&s)[J], const float (&t)[J], const float (&g)[J]) {
  double ss = 0.0, tt = 0.0, st = 0.0, gs = 0.0, gt = 0.0;
#pragma unroll
  for (int j = 0; j < J; ++j) {
    const double a = s[j], b = t[j];
    ss = __fma_rn(a, a, ss); tt = __fma_rn(b, b, tt); st = __fma_rn(a, b, st);
    if (BWD) { const double c = g[j]; gs = __fma_rn(c, a, gs); gt = __fma_rn(c, b, gt); }
  }
  ss = warp_sum(ss); tt = warp_sum(tt); st = warp_sum(st);
  if (BWD) { gs = warp_sum(gs); gt = warp_sum(gt); }
  Rot r;
  const float ns = static_cast<float>(sqrt(ss)), nt = static_cast<float>(sqrt(tt));
  r.ins = __frcp_rn(fmaxf(ns, RS_EPS));
  r.int_ = __frcp_rn(fmaxf(nt, RS_EPS));
  const double dins = r.ins, dint = r.int_;
  const double nw2 = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(ss, dins), dins), __dmul_rn(__dmul_rn(tt, dint), dint)),
                               __dmul_rn(__dmul_rn(__dmul_rn(2.0, st), dins), dint));
  const double dinw = __drcp_rn(fmax(sqrt(fmax(nw2, 0.0)), static_cast<double>(RS_EPS)));
  r.inw = static_cast<float>(dinw);
  r.lam = __fmul_rn(nt, r.ins);
  r.fa = static_cast<float>(__dmul_rn(__dadd_rn(__dmul_rn(ss, dins), __dmul_rn(st, dint)), dinw));
  r.fb = static_cast<float>(__dmul_rn(ss, dins));
  if (BWD) {
    r.ba = static_cast<float>(__dmul_rn(__dadd_rn(__dmul_rn(gs, dins), __dmul_rn(gt, dint)), dinw));
    r.bb = static_cast<float>(__dmul_rn(gt, dint));
  }
  return r;
}

// The value stage q adds to quantized_out and subtracts from the residual: rotate_to(s, t) (sim_vq.py:126-128) or the
// straight-through value (t - s) + s (sim_vq.py:130).  u and w are returned for the backward.
__device__ __forceinline__ float stage_value(float s, float t, bool rotation, const Rot& r, float* u_out, float* w_out) {
  if (!rotation) return __fadd_rn(__fsub_rn(t, s), s);
  const float u = __fmul_rn(s, r.ins), q = __fmul_rn(t, r.int_);
  const float w = __fmul_rn(__fadd_rn(u, q), r.inw);
  *u_out = u;
  *w_out = w;
  const float v = __fadd_rn(__fsub_rn(s, __fmul_rn(2.f * r.fa, w)), __fmul_rn(2.f * r.fb, q));
  return __fmul_rn(v, r.lam);
}

// Stage tail: c = codes[idx], out = stage_value(r, c); r_next = r - out; qsum = 0 + out (first stage) or qsum + out
// (rsv:195-196); idx64_out[row * idx_stride] = idx; loss_sum += sum((r - c)^2) (sim_vq.py:121-124).
template <int J>
__global__ void __launch_bounds__(RS_THREADS, 1) rsimvq_tail_kernel(const float* __restrict__ r, const float* __restrict__ codes,
                                                                 const int32_t* __restrict__ idx, int64_t N, int D, int rotation,
                                                                 float* __restrict__ r_next, float* __restrict__ qsum, int first,
                                                                 int64_t* __restrict__ idx64_out, int64_t idx_stride,
                                                                 double* __restrict__ loss_sum) {
  __shared__ double part[RS_THREADS / 32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  double sq = 0.0;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + wib; row < N; row += static_cast<int64_t>(gridDim.x) * wpb) {
    const int k = idx[row];
    float s[J], t[J];
    load_row<J>(s, r + row * D, D, lane);
    load_row<J>(t, codes + static_cast<int64_t>(k) * D, D, lane);
    Rot rt = {};
    if (rotation) rt = rot_setup<J, false>(s, t, t);
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int i = lane + 32 * j;
      if (i >= D) break;
      float u, w;
      const float o = stage_value(s[j], t[j], rotation, rt, &u, &w);
      const double d = __fsub_rn(s[j], t[j]);
      sq = __fma_rn(d, d, sq);
      const int64_t e = row * D + i;
      if (r_next) r_next[e] = __fsub_rn(s[j], o);
      qsum[e] = first ? __fadd_rn(0.f, o) : __fadd_rn(qsum[e], o);
    }
    if (idx64_out && lane == 0) idx64_out[row * idx_stride] = k;
  }
  if (!loss_sum) return;
  sq = warp_sum(sq);
  if (lane == 0) part[wib] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int i = 0; i < wpb; ++i) b += part[i];
    atomicAdd(loss_sum, b);
  }
}

// loss = (mse + mse * input_weight) * weight, each step rounded to fp32 as torch does (sim_vq.py:121-124, :138)
__global__ void rsimvq_loss_kernel(const double* loss_sum, int64_t numel, float input_weight, float weight, float* loss_out) {
  const float mse = static_cast<float>(*loss_sum / static_cast<double>(numel));
  *loss_out = __fmul_rn(__fadd_rn(mse, __fmul_rn(mse, input_weight)), weight);
}

// Backward of all stages.  The residual enters stage q as r_q = x - sum_{j<q} out_j (detached), so d/dx of every stage
// reaches x through the identity: grad_x = sum_q [ estimator backward of G at (r_q, c_q) + gl[q] (r_q - c_q) ], where
// gl[q] = dL/dloss_q * 2 weight input_weight / numel (the second commitment term; the first one carries gradient to the code
// only).  Stages q >= n_active were dropped (quantize dropout) and add nothing.
template <int J>
__global__ void __launch_bounds__(RS_THREADS, 1) rsimvq_backward_kernel(const float* __restrict__ x, const float* __restrict__ codes,
                                                                     int64_t book_stride, int Q, int n_active,
                                                                     const int64_t* __restrict__ idx, int64_t N, int D, int rotation,
                                                                     const float* __restrict__ grad_q, const float* __restrict__ gl,
                                                                     float* __restrict__ grad_x) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N; row += static_cast<int64_t>(gridDim.x) * wpb) {
    float s[J], g[J], dx[J];
    load_row<J>(s, x + row * D, D, lane);
    if (grad_q) load_row<J>(g, grad_q + row * D, D, lane);
#pragma unroll
    for (int j = 0; j < J; ++j) {
      if (!grad_q) g[j] = 0.f;
      dx[j] = 0.f;
    }
    for (int q = 0; q < n_active; ++q) {
      const int64_t k = idx[row * Q + q];
      float t[J];
      load_row<J>(t, codes + q * book_stride + k * D, D, lane);
      const float glq = gl ? gl[q] : 0.f;
      Rot rt = {};
      if (rotation) rt = rot_setup<J, true>(s, t, g);
#pragma unroll
      for (int j = 0; j < J; ++j) {
        float u = 0.f, w = 0.f;
        const float o = stage_value(s[j], t[j], rotation, rt, &u, &w);
        const float de = rotation ? __fmul_rn(__fadd_rn(__fsub_rn(g[j], __fmul_rn(2.f * rt.ba, w)), __fmul_rn(2.f * rt.bb, u)), rt.lam)
                                  : g[j];
        dx[j] = __fadd_rn(dx[j], __fadd_rn(de, __fmul_rn(glq, __fsub_rn(s[j], t[j]))));
        s[j] = __fsub_rn(s[j], o);
      }
    }
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int i = lane + 32 * j;
      if (i < D) grad_x[row * D + i] = dx[j];
    }
  }
}

// registers per lane: the smallest power of two J with 32 J >= D
int rs_slots(int D) {
  int J = 1;
  while (32 * J < D) J <<= 1;
  return J;
}

}  // namespace
}  // namespace vqb

extern "C" int vqb_rsimvq_tail(const float* r, const float* codes, const int32_t* idx, int64_t N, int D, int rotation, float* r_next,
                               float* qsum, int first, int64_t* idx64_out, int64_t idx_stride, double* loss_sum, float* loss_out,
                               float input_weight, float weight, void* stream) {
  using namespace vqb;
  if (!r || !codes || !idx || !qsum || N <= 0 || D <= 0 || (loss_out && !loss_sum)) return VQB_E_INVALID;
  if (D > 1024) return VQB_E_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (loss_out) {
    const cudaError_t e = cudaMemsetAsync(loss_sum, 0, sizeof(double), s);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  double* ls = loss_out ? loss_sum : nullptr;
  const int g = capped_grid(N, RS_THREADS / 32, 16);
  switch (rs_slots(D)) {
#define VQB_RS_TAIL(JJ) \
  case JJ: rsimvq_tail_kernel<JJ><<<g, RS_THREADS, 0, s>>>(r, codes, idx, N, D, rotation, r_next, qsum, first, idx64_out, idx_stride, ls); break;
    VQB_RS_TAIL(1) VQB_RS_TAIL(2) VQB_RS_TAIL(4) VQB_RS_TAIL(8) VQB_RS_TAIL(16) VQB_RS_TAIL(32)
#undef VQB_RS_TAIL
  }
  if (loss_out) rsimvq_loss_kernel<<<1, 1, 0, s>>>(loss_sum, N * D, input_weight, weight, loss_out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_rsimvq_backward(const float* x, const float* codes, int Q, int K, const int64_t* idx, int64_t N, int D,
                                   int n_active, int rotation, const float* grad_q, const float* grad_loss, float* grad_x,
                                   void* stream) {
  using namespace vqb;
  if (!x || !codes || !idx || !grad_x || Q <= 0 || K <= 0 || N <= 0 || D <= 0 || n_active < 0 || n_active > Q) return VQB_E_INVALID;
  if (D > 1024) return VQB_E_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t stride = static_cast<int64_t>(K) * D;
  const int g = capped_grid(N, RS_THREADS / 32, 16);
  switch (rs_slots(D)) {
#define VQB_RS_BWD(JJ) \
  case JJ: rsimvq_backward_kernel<JJ><<<g, RS_THREADS, 0, s>>>(x, codes, stride, Q, n_active, idx, N, D, rotation, grad_q, grad_loss, grad_x); break;
    VQB_RS_BWD(1) VQB_RS_BWD(2) VQB_RS_BWD(4) VQB_RS_BWD(8) VQB_RS_BWD(16) VQB_RS_BWD(32)
#undef VQB_RS_BWD
  }
  return static_cast<int>(cudaGetLastError());
}
