// DiVeQ, the directional reparameterization gradient estimator (vector_quantize_pytorch.py:323-330), forward and backward,
// one warp per row:
//   e = q - x,  u = l2norm(e + s z) (detached),  out = x + u ||e||
//   backward, with g = d loss / d out:  de = (g.u) e / ||e|| (0 where ||e|| = 0, as torch's norm backward),
//   dx = g - de,  dq = de
// Every intermediate is rounded to the row dtype exactly where torch rounds it in the reference's expression (each
// elementwise op of a bf16 tensor, and each row reduction once, from an fp32 accumulator): the bf16 results are torch's to
// within the order of the row sums.  The row sums are taken in double (products of fp32 values are exact there).
// The backward recomputes e, u and ||e|| from (x, q, z): no per-row state is kept between the two passes.
#include "vqb_common.cuh"

namespace vqb {
namespace {

constexpr int DV_THREADS = 256;   // 8 rows in flight per CTA
constexpr float DV_EPS = 1e-6f;   // l2norm eps (vqp:37-38)

struct DvRow {
  float ne;    // ||e||, rounded to the row dtype
  float den;   // max(||e + s z||, eps) in the row dtype (the divisor of F.normalize): u = R(n / den)
};

template <int DT>
__device__ __forceinline__ float dv_e(const void* x, const void* q, int64_t i) {
  using E = Elem<DT>;
  return E::round(__fsub_rn(E::load(q, i), E::load(x, i)));
}

template <int DT>
__device__ __forceinline__ float dv_n(float e, const void* z, int64_t i, float scale) {
  using E = Elem<DT>;
  return E::round(__fadd_rn(e, E::round(__fmul_rn(scale, E::load(z, i)))));
}

template <int DT>
__device__ __forceinline__ DvRow dv_setup(const void* x, const void* q, const void* z, int64_t base, int D, int lane, float scale) {
  using E = Elem<DT>;
  double ee = 0.0, nn = 0.0;
  for (int i = lane; i < D; i += 32) {
    const float e = dv_e<DT>(x, q, base + i);
    const float n = dv_n<DT>(e, z, base + i, scale);
    ee = __fma_rn(static_cast<double>(e), static_cast<double>(e), ee);
    nn = __fma_rn(static_cast<double>(n), static_cast<double>(n), nn);
  }
  ee = warp_sum(ee);
  nn = warp_sum(nn);
  DvRow r;
  r.ne = E::round(static_cast<float>(sqrt(ee)));
  r.den = E::round(fmaxf(E::round(static_cast<float>(sqrt(nn))), DV_EPS));
  return r;
}

template <int DT, bool BWD>
__global__ void __launch_bounds__(DV_THREADS) diveq_kernel(const void* __restrict__ x, const void* __restrict__ q,
                                                           const void* __restrict__ z, const void* __restrict__ grad, int64_t N,
                                                           int D, float scale, void* __restrict__ out, float* __restrict__ dq) {
  using E = Elem<DT>;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb) {
    const int64_t base = row * D;
    const DvRow r = dv_setup<DT>(x, q, z, base, D, lane, scale);
    if (!BWD) {
      for (int i = lane; i < D; i += 32) {
        const float e = dv_e<DT>(x, q, base + i);
        const float u = E::round(__fdiv_rn(dv_n<DT>(e, z, base + i, scale), r.den));
        E::store(out, base + i, __fadd_rn(E::load(x, base + i), E::round(__fmul_rn(u, r.ne))));
      }
      continue;
    }
    // d ||e|| = sum_i g_i u_i (the mul backward of `u * ||e||` rounds each product, the sum is rounded once)
    double gu = 0.0;
    for (int i = lane; i < D; i += 32) {
      const float e = dv_e<DT>(x, q, base + i);
      const float u = E::round(__fdiv_rn(dv_n<DT>(e, z, base + i, scale), r.den));
      gu += static_cast<double>(E::round(__fmul_rn(E::load(grad, base + i), u)));
    }
    gu = warp_sum(gu);
    // torch's norm backward: e * (grad / ||e||), with the quotient zeroed where ||e|| = 0
    const float c = r.ne == 0.f ? 0.f : E::round(__fdiv_rn(E::round(static_cast<float>(gu)), r.ne));
    for (int i = lane; i < D; i += 32) {
      const float de = E::round(__fmul_rn(dv_e<DT>(x, q, base + i), c));
      E::store(out, base + i, __fsub_rn(E::load(grad, base + i), de));
      dq[base + i] = de;
    }
  }
}

}  // namespace
}  // namespace vqb

using namespace vqb;

extern "C" int vqb_diveq(const void* x, const void* q, const void* noise, const void* grad_out, int64_t N, int D, int dtype,
                         float noise_scale, void* out, float* grad_q, void* stream) {
  if (!x || !q || !noise || !out || N <= 0 || D <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (grad_out && !grad_q) return VQB_E_INVALID;
  if (D > 1024) return VQB_E_UNSUPPORTED;
  const uintptr_t esz = dtype == VQB_DTYPE_F32 ? 4 : 2;
  const uintptr_t any = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(noise) |
                        reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(out);
  if ((any & (esz - 1)) || (reinterpret_cast<uintptr_t>(grad_q) & 3)) return VQB_E_ALIGN;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = capped_grid(N, DV_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32) {
    if (grad_out) diveq_kernel<VQB_DTYPE_F32, true><<<g, DV_THREADS, 0, s>>>(x, q, noise, grad_out, N, D, noise_scale, out, grad_q);
    else diveq_kernel<VQB_DTYPE_F32, false><<<g, DV_THREADS, 0, s>>>(x, q, noise, nullptr, N, D, noise_scale, out, nullptr);
  } else {
    if (grad_out) diveq_kernel<VQB_DTYPE_BF16, true><<<g, DV_THREADS, 0, s>>>(x, q, noise, grad_out, N, D, noise_scale, out, grad_q);
    else diveq_kernel<VQB_DTYPE_BF16, false><<<g, DV_THREADS, 0, s>>>(x, q, noise, nullptr, N, D, noise_scale, out, nullptr);
  }
  return static_cast<int>(cudaGetLastError());
}
