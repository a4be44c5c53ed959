// Row moves of the one-thread-per-row kernels (vq_fsq.cu, vq_fsp.cu): the D values of one item in registers.
#pragma once
#include "vqb_common.cuh"

namespace vqb {
namespace {

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
