// Helpers of the one-thread-per-row kernels (vq_fsq.cu, vq_lfq.cu, vq_fsp.cu, vq_binmap.cu): row moves with the D values of
// one item in registers, the rounding and division primitives, index access and the host's alignment test and D dispatch.
#pragma once
#include "vqb_common.cuh"

namespace vqb {
namespace {

// Rounds to the chain's work dtype: bf16 when BF, else fp32 (no-op).
template <bool BF> __device__ __forceinline__ float rw(float v) { return BF ? bf16_round(v) : v; }

// a / b, correctly rounded, for a divisor b with rb = RN(1 / b) (Markstein: q0 = RN(a rb) is within an ulp of a / b, the
// remainder a - b q0 is exact in one fma, and RN(q0 + rem rb) = RN(a / b) while nothing over- or underflows; an infinite or
// NaN q0 is returned as it is).  Every division by a constant goes through it, with the reciprocal computed by the caller, so no
// kernel carries a call to the division's slow path (whose calling convention spills).
__device__ __forceinline__ float divc(float a, float b, float rb) {
  const float q0 = __fmul_rn(a, rb);
  if (!isfinite(q0)) return q0;
  return __fmaf_rn(__fmaf_rn(-b, q0, a), rb, q0);
}

// Element `off` of an int32 (idx64 = 0) or int64 index array.
__device__ __forceinline__ int64_t load_index(const void* idx, int idx64, int64_t off) {
  return idx64 ? reinterpret_cast<const int64_t*>(idx)[off] : static_cast<int64_t>(reinterpret_cast<const int32_t*>(idx)[off]);
}

__device__ __forceinline__ void store_index(void* idx, int idx64, int64_t off, int64_t v) {
  if (idx64) reinterpret_cast<int64_t*>(idx)[off] = v;
  else reinterpret_cast<int32_t*>(idx)[off] = static_cast<int32_t>(v);
}

// Whether p is a multiple of n bytes (the host's check of what a kernel's widest access needs).
inline bool aligned(const void* p, int n) { return reinterpret_cast<uintptr_t>(p) % n == 0; }

// CALL(D) for the row width D = 1..16 the kernels are instantiated for; any other D returns VQB_E_UNSUPPORTED.
#define VQB_SWITCH_D(CALL)                                                                                                  \
  switch (D) {                                                                                                              \
    case 1: CALL(1); break; case 2: CALL(2); break; case 3: CALL(3); break; case 4: CALL(4); break;                         \
    case 5: CALL(5); break; case 6: CALL(6); break; case 7: CALL(7); break; case 8: CALL(8); break;                         \
    case 9: CALL(9); break; case 10: CALL(10); break; case 11: CALL(11); break; case 12: CALL(12); break;                   \
    case 13: CALL(13); break; case 14: CALL(14); break; case 15: CALL(15); break; case 16: CALL(16); break;                 \
    default: return VQB_E_UNSUPPORTED;                                                                                      \
  }

// The D values of one item as 32-bit words, moved with the widest accesses the row size allows (the host checks the 16-byte
// alignment of every base pointer); bf16 rows of odd D move element by element.
template <int DT, int D>
struct Row {
  static constexpr int B = D * static_cast<int>(sizeof(typename Elem<DT>::T));
  static constexpr int W = (B + 3) / 4;   // 32-bit words
  static constexpr int C = B % 16 == 0 ? 16 : B % 8 == 0 ? 8 : B % 4 == 0 ? 4 : 2;   // access width in bytes
};

template <int DT, int D>
__device__ __forceinline__ void load_item(const void* base, int64_t item, float (&v)[D]) {
  using R = Row<DT, D>;
  if constexpr (R::C == 2) {
#pragma unroll
    for (int j = 0; j < D; ++j) v[j] = Elem<DT>::load(base, item * D + j);
  } else {
    uint32_t w[R::W];
    const char* p = reinterpret_cast<const char*>(base) + item * R::B;
#pragma unroll
    for (int k = 0; k < R::B / R::C; ++k) {
      if constexpr (R::C == 16) {
        const uint4 c = __ldg(reinterpret_cast<const uint4*>(p) + k);
        w[4 * k] = c.x; w[4 * k + 1] = c.y; w[4 * k + 2] = c.z; w[4 * k + 3] = c.w;
      } else if constexpr (R::C == 8) {
        const uint2 c = __ldg(reinterpret_cast<const uint2*>(p) + k);
        w[2 * k] = c.x; w[2 * k + 1] = c.y;
      } else {
        w[k] = __ldg(reinterpret_cast<const unsigned int*>(p) + k);
      }
    }
#pragma unroll
    for (int j = 0; j < D; ++j) {
      if constexpr (DT == VQB_DTYPE_F32) v[j] = __uint_as_float(w[j]);
      else v[j] = bf16_bits_to_float(static_cast<uint16_t>(w[j / 2] >> (16 * (j % 2))));
    }
  }
}

template <int DT, int D>
__device__ __forceinline__ void store_item(void* base, int64_t item, const float (&v)[D]) {
  using R = Row<DT, D>;
  if constexpr (R::C == 2) {
#pragma unroll
    for (int j = 0; j < D; ++j) Elem<DT>::store(base, item * D + j, v[j]);
  } else {
    uint32_t w[R::W];
#pragma unroll
    for (int j = 0; j < D; ++j) {
      if constexpr (DT == VQB_DTYPE_F32) w[j] = __float_as_uint(v[j]);
      else if (j % 2 == 0) w[j / 2] = float_to_bf16_bits(v[j]);
      else w[j / 2] |= static_cast<uint32_t>(float_to_bf16_bits(v[j])) << 16;
    }
    char* p = reinterpret_cast<char*>(base) + item * R::B;
#pragma unroll
    for (int k = 0; k < R::B / R::C; ++k) {
      if constexpr (R::C == 16) reinterpret_cast<uint4*>(p)[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
      else if constexpr (R::C == 8) reinterpret_cast<uint2*>(p)[k] = make_uint2(w[2 * k], w[2 * k + 1]);
      else reinterpret_cast<unsigned int*>(p)[k] = w[k];
    }
  }
}

}  // namespace
}  // namespace vqb
