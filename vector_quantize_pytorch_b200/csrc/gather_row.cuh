// Per-row tail of VectorQuantize.forward / one ResidualVQ stage, executed by ONE WARP for one row:
//   q = embed[k].type(dtype)                      vqp:766/:779-781, :1178
//   loss partial += sum((q - x)^2) in dtype        vqp:1327
//   residual = x_raw - q                           rvq:524
// (ResidualVQ's quantized_out += q, rvq:525, is rebuilt from the indices afterwards: vqb_rvq_accumulate.)
// Shared by the stand-alone gather kernel, the store warps of the fused search kernel and the exact
// re-score kernels (which finish the rows the search kernel could not certify).
#pragma once
#include "vqb_common.cuh"

namespace vqb {

struct FusedOut {  // device-side copy of vqb_fused_outputs
  const void* x_eff;
  const float* embed;
  void* q_out;
  int64_t* idx64_out;
  int64_t idx_stride;
  double* loss_sum;
  const void* x_raw;
  void* resid_out;
  int dtype;
  int enabled;
  uint16_t* planes_out;   // optional (fp32 rows): bf16 hi / lo split of the residual, [2][N][D]
  int64_t planes_stride;  // N * D
};

inline int make_fused(FusedOut* o, const vqb_fused_outputs* f, int D, int64_t N = 0) {
  *o = FusedOut{};  // every pointer null, enabled = 0: a disabled tail must be inert wherever the kernels test a field
  if (!f) return VQB_OK;
  if (!f->x_eff || !f->embed) return VQB_E_INVALID;
  if (f->dtype != VQB_DTYPE_F32 && f->dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D % 8 != 0) return VQB_E_UNSUPPORTED;
  // reserved fields: the tail accumulates no statistics and no running sum
  if (f->stats_cnt || f->stats_sum || f->qsum) return VQB_E_UNSUPPORTED;
  const uintptr_t all = reinterpret_cast<uintptr_t>(f->x_eff) | reinterpret_cast<uintptr_t>(f->embed) |
                        reinterpret_cast<uintptr_t>(f->q_out) | reinterpret_cast<uintptr_t>(f->x_raw) |
                        reinterpret_cast<uintptr_t>(f->resid_out);
  if (all & 15) return VQB_E_ALIGN;
  o->x_eff = f->x_eff; o->embed = f->embed; o->q_out = f->q_out; o->idx64_out = f->idx64_out;
  o->idx_stride = f->idx_stride; o->loss_sum = f->loss_sum; o->x_raw = f->x_raw ? f->x_raw : f->x_eff;
  o->resid_out = f->resid_out; o->dtype = f->dtype; o->enabled = 1;
  if (f->planes_out) {  // the split rides on the fp32 residual
    if (f->dtype != VQB_DTYPE_F32 || !f->resid_out || N <= 0 || (reinterpret_cast<uintptr_t>(f->planes_out) & 15)) return VQB_E_INVALID;
    o->planes_out = static_cast<uint16_t*>(f->planes_out);
    o->planes_stride = N * D;
  }
  return VQB_OK;
}

// bf16 hi / lo split of four fp32 values (the same arithmetic as input_prepare_kernel) -> the two operand planes
__device__ __forceinline__ void store_planes4(uint16_t* planes, int64_t stride, int64_t at, const float* v) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    h[e] = float_to_bf16_bits(v[e]);
    l[e] = float_to_bf16_bits(v[e] - bf16_bits_to_float(static_cast<uint16_t>(h[e])));
  }
  *reinterpret_cast<uint2*>(planes + at) = make_uint2(h[0] | (h[1] << 16), h[2] | (h[3] << 16));
  *reinterpret_cast<uint2*>(planes + stride + at) = make_uint2(l[0] | (l[1] << 16), l[2] | (l[3] << 16));
}

template <int DT>
__device__ __forceinline__ void unpack16(const uint4& u, float* v) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  if (DT == VQB_DTYPE_BF16) {
#pragma unroll
    for (int e = 0; e < 4; ++e) { v[2 * e] = __uint_as_float(w[e] << 16); v[2 * e + 1] = __uint_as_float(w[e] & 0xFFFF0000u); }
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = __uint_as_float(w[e]);
  }
}
template <int DT>
__device__ __forceinline__ uint4 pack16(const float* v) {
  uint32_t w[4];
  if (DT == VQB_DTYPE_BF16) {
#pragma unroll
    for (int e = 0; e < 4; ++e) w[e] = float_to_bf16_bits(v[2 * e]) | (uint32_t(float_to_bf16_bits(v[2 * e + 1])) << 16);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) w[e] = __float_as_uint(v[e]);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// B rows (ks[b] their codes) per call.  A batch (B > 1, the store warps of the search kernel, latency-bound otherwise) issues
// all its loads before any use/store, so a warp keeps ~3*B independent 16-byte requests in flight; rows[b] < 0 marks an
// empty slot.  The row kernels pass one row (rows[0] >= 0) and read x_raw where it is used: hoisting that load costs them
// registers, and the re-score kernels run next to the statistics sort.  All 32 lanes must call.  Returns
// this lane's partial of sum((q - x)^2) (0 if no loss is requested).
template <int DT, int B>
__device__ __forceinline__ float gather_rows(const FusedOut& o, const int64_t (&rows)[B], const int (&ks)[B], int D, int lane) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr int VEC = 16 / sizeof(T);  // elements per 16-byte access: 8 (bf16) or 4 (fp32)
  auto ld = [](const void* p, int64_t off) { return *reinterpret_cast<const uint4*>(static_cast<const T*>(p) + off); };
  float lsum = 0.f;
  if (o.idx64_out && lane < B) {
#pragma unroll
    for (int b = 0; b < B; ++b)
      if (lane == b && (B == 1 || rows[b] >= 0)) o.idx64_out[rows[b] * o.idx_stride] = ks[b];
  }
  for (int i = lane * VEC; i < D; i += 32 * VEC) {
    float4 cq[B][VEC / 4];
    uint4 xq[B], rq[B];
#pragma unroll
    for (int b = 0; b < B; ++b) {
      if (B > 1 && rows[b] < 0) continue;
      const float* c = o.embed + static_cast<int64_t>(ks[b]) * D + i;
#pragma unroll
      for (int e = 0; e < VEC / 4; ++e) cq[b][e] = __ldg(reinterpret_cast<const float4*>(c) + e);
      const int64_t off = rows[b] * D + i;
      xq[b] = ld(o.x_eff, off);
      if (B > 1 && o.resid_out && o.x_raw != o.x_eff) rq[b] = ld(o.x_raw, off);
    }
#pragma unroll
    for (int b = 0; b < B; ++b) {
      if (B > 1 && rows[b] < 0) continue;
      const int64_t off = rows[b] * D + i;
      float xv[8], qv[8];
      unpack16<DT>(xq[b], xv);
#pragma unroll
      for (int e = 0; e < VEC / 4; ++e) {
        qv[4 * e] = E::round(cq[b][e].x); qv[4 * e + 1] = E::round(cq[b][e].y);
        qv[4 * e + 2] = E::round(cq[b][e].z); qv[4 * e + 3] = E::round(cq[b][e].w);
      }
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const float d = qv[e] - xv[e];
        lsum += E::round(d * d);
      }
      if (o.q_out) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(o.q_out) + off) = pack16<DT>(qv);
      if (o.resid_out) {
        float rv[8];
        if (o.x_raw != o.x_eff) unpack16<DT>(B > 1 ? rq[b] : ld(o.x_raw, off), rv);
        else {
#pragma unroll
          for (int e = 0; e < VEC; ++e) rv[e] = xv[e];
        }
#pragma unroll
        for (int e = 0; e < VEC; ++e) rv[e] -= qv[e];
        *reinterpret_cast<uint4*>(reinterpret_cast<T*>(o.resid_out) + off) = pack16<DT>(rv);
        if (DT == VQB_DTYPE_F32 && o.planes_out) store_planes4(o.planes_out, o.planes_stride, off, rv);
      }
    }
  }
  return lsum;
}

}  // namespace vqb
