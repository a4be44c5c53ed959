// Tensor-core operands of one codebook row (shared by vqb_codebook_prepare and the EMA apply step, vq_ema.cu).
#pragma once
#include "vqb_common.cuh"

namespace vqb {

// One warp owns one (padded) code row.  Lane l holds elements [128 j + 4 l, +4) of the row in c[j]: NV float4 cover
// D <= 128 NV, so NV = 8 covers every D the library supports.
constexpr int CODE_ROW_MAX_D = 8 * 128;

template <int NV>
__device__ __forceinline__ void load_code_row(const float* row, int D, int lane, float4 (&c)[NV]) {
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = j * 128 + lane * 4;
    c[j] = i < D ? *reinterpret_cast<const float4*>(row + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// planes (two bf16 planes of [Kpad][D]):
//   [0] hi = bf16(c)        B operand of every pass; ALSO the row `quantize = embed[ind].type(bf16)` copies
//   [1] lo = bf16(c - hi)   B operand of the (x, c_lo) pass (hi + lo carries 16 mantissa bits)
// cmax[CMAX_NORM] = max_k ||c||, cmax[CMAX_RES] = max_k ||c - hi - lo|| and cmax[CMAX_LO] = max_k ||lo||: the certification band
// of the search (vq_assign.cu) is a Cauchy-Schwarz bound on these exact norms, not an empirical constant (a single heavy
// coordinate reaches it).
template <int NV>
__device__ __forceinline__ void write_code_operands(const float4 (&c)[NV], int k, int Kpad, int D, int metric, uint16_t* planes,
                                                    uint16_t* bext, float* bias, float* cnorm2, float* cmax, int lane) {
  uint16_t* hi = planes + static_cast<int64_t>(k) * D;
  uint16_t* lo = planes + (static_cast<int64_t>(Kpad) + k) * D;
  double n2 = 0.0;
  float r2 = 0.f, l2 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = j * 128 + lane * 4;
    if (i >= D) continue;
    const float v[4] = {c[j].x, c[j].y, c[j].z, c[j].w};
    uint16_t h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      h[e] = float_to_bf16_bits(v[e]);
      const float dl = v[e] - bf16_bits_to_float(h[e]);
      l[e] = float_to_bf16_bits(dl);
      const float d2 = dl - bf16_bits_to_float(l[e]);
      r2 = fmaf(d2, d2, r2);
      l2 = fmaf(bf16_bits_to_float(l[e]), bf16_bits_to_float(l[e]), l2);
      n2 += static_cast<double>(v[e]) * static_cast<double>(v[e]);
    }
    *reinterpret_cast<uint2*>(hi + i) = make_uint2(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16));
    *reinterpret_cast<uint2*>(lo + i) = make_uint2(l[0] | (uint32_t(l[1]) << 16), l[2] | (uint32_t(l[3]) << 16));
  }
  n2 = warp_sum(n2);
  r2 = warp_sum(r2);
  l2 = warp_sum(l2);
  if (lane == 0) {
    const float n2f = static_cast<float>(n2);
    cnorm2[k] = n2f;
    const float b = (metric == VQB_METRIC_EUCLID) ? 0.5f * n2f : 0.f;
    bias[k] = b;
    // -bias as three bf16 terms (8+8+8 mantissa bits = the exact fp32 value): the K=16 "bias MMA" of the
    // search kernel multiplies them by [1 1 1 0...] and so seeds the accumulator with -0.5||c||^2.
    const uint16_t b1 = float_to_bf16_bits(b);
    const float q1 = b - bf16_bits_to_float(b1);
    const uint16_t b2 = float_to_bf16_bits(q1);
    const uint16_t b3 = float_to_bf16_bits(q1 - bf16_bits_to_float(b2));
    uint16_t* row = bext + k * 16;
    row[0] = b1 ^ 0x8000; row[1] = b2 ^ 0x8000; row[2] = b3 ^ 0x8000;  // sign flip = negate
#pragma unroll
    for (int j = 3; j < 16; ++j) row[j] = 0;
    // valid as unsigned-int maxima: the values are >= 0.  The residual norms are rounded UP (they are error bounds).
    atomicMax(reinterpret_cast<unsigned int*>(cmax + CMAX_NORM), __float_as_uint(sqrtf(n2f)));
    atomicMax(reinterpret_cast<unsigned int*>(cmax + CMAX_RES), __float_as_uint(__fsqrt_ru(r2) * 1.0001f));
    atomicMax(reinterpret_cast<unsigned int*>(cmax + CMAX_LO), __float_as_uint(__fsqrt_ru(l2) * 1.0001f));
  }
}

// Padding row k >= K: never wins (bias = +inf, accumulator seed -3e38) and contributes zeros to the MMA.
__device__ __forceinline__ void write_padding_operands(int k, int Kpad, int D, uint16_t* planes, uint16_t* bext, float* bias,
                                                       int lane) {
  uint16_t* hi = planes + static_cast<int64_t>(k) * D;
  uint16_t* lo = planes + (static_cast<int64_t>(Kpad) + k) * D;
  for (int i = lane; i < D; i += 32) { hi[i] = 0; lo[i] = 0; }
  if (lane == 0) bias[k] = INFINITY;
  if (lane < 16) bext[k * 16 + lane] = (lane == 0) ? float_to_bf16_bits(-3.0e38f) : 0;
}

}  // namespace vqb
