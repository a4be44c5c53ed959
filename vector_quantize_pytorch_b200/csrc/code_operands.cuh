// Tensor-core operands of one codebook row (shared by vqb_codebook_prepare and vqb_ema_apply).
#pragma once
#include "vqb_common.cuh"
#include <cuda_fp16.h>

namespace vqb {

// ---------------------------------------------------------------------------------------------
// codebook operands.  Shared by vqb_codebook_prepare and vqb_ema_apply (vq_ema.cu).
// One warp owns one (padded) code row.  `vals(i)` yields c[i] in fp32.
// ---------------------------------------------------------------------------------------------
// planes (three 2-byte planes of [Kpad][D]):
//   [0] bf16 hi = bf16(c)        B operand of the bf16 pass schemes; ALSO the row `quantize = embed[ind].type(bf16)` copies
//   [1] bf16 lo = bf16(c - hi)   B operand of the (x, c_lo) pass of the bf16 schemes (hi + lo carries 16 mantissa bits)
//   [2] fp16(c)                  B operand of the MIXED scheme (bf16 rows x fp16 codes, products exact in fp32): 11 instead of 8
//                                mantissa bits at the same tensor-core rate, i.e. a residual of 2^-12 ||c|| that certifies ~97 %
//                                of the rows at K ~ 1e3 with ONE pass per A plane; values beyond +-65504 are clamped.
//                                cmax[1] = max_k ||c - fp16 plane|| is the exact norm of everything the plane leaves out
//                                (clamp included) and sizes the certification band of that scheme (vq_assign.cu).
// cmax[2] = max_k ||c - hi - lo|| and cmax[3] = max_k ||lo|| do the same for the bf16 split schemes: the band is a
// Cauchy-Schwarz bound on exact norms, not an empirical constant (a single heavy coordinate reaches it).
__device__ __forceinline__ void write_code_operands(const float* crow /*K x D row or nullptr for padding*/, int k, int K, int Kpad, int D,
                                    int metric, uint16_t* planes, uint16_t* bext, float* bias, float* cnorm2, float* cmax, int lane) {
  uint16_t* hi = planes + static_cast<int64_t>(k) * D;
  uint16_t* lo = planes + (static_cast<int64_t>(Kpad) + k) * D;
  uint16_t* qr = planes + (static_cast<int64_t>(2) * Kpad + k) * D;   // the fp16 plane
  if (crow == nullptr) {  // padding row: never wins (bias = +inf), contributes zeros to the MMA
    for (int i = lane; i < D; i += 32) { hi[i] = 0; lo[i] = 0; qr[i] = 0; }
    if (lane == 0) bias[k] = INFINITY;
    if (lane < 16) bext[k * 16 + lane] = (lane == 0) ? float_to_bf16_bits(-3.0e38f) : 0;  // score = -huge: never wins
    return;
  }
  double n2 = 0.0;
  float r1 = 0.f, r2 = 0.f, l2 = 0.f;
  for (int i = lane * 4; i < D; i += 128) {
    const float4 c = *reinterpret_cast<const float4*>(crow + i);
    const float v[4] = {c.x, c.y, c.z, c.w};
    uint16_t h[4], l[4], q[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      h[e] = float_to_bf16_bits(v[e]);
      const float dl = v[e] - bf16_bits_to_float(h[e]);
      l[e] = float_to_bf16_bits(dl);
      const float d2 = dl - bf16_bits_to_float(l[e]);
      r2 = fmaf(d2, d2, r2);
      l2 = fmaf(bf16_bits_to_float(l[e]), bf16_bits_to_float(l[e]), l2);
      const __half hh = __float2half_rn(fminf(fmaxf(v[e], -65504.f), 65504.f));
      const float d1 = v[e] - __half2float(hh);
      q[e] = __half_as_ushort(hh);
      r1 = fmaf(d1, d1, r1);
      n2 += static_cast<double>(v[e]) * static_cast<double>(v[e]);
    }
    *reinterpret_cast<uint2*>(hi + i) = make_uint2(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16));
    *reinterpret_cast<uint2*>(lo + i) = make_uint2(l[0] | (uint32_t(l[1]) << 16), l[2] | (uint32_t(l[3]) << 16));
    *reinterpret_cast<uint2*>(qr + i) = make_uint2(q[0] | (uint32_t(q[1]) << 16), q[2] | (uint32_t(q[3]) << 16));
  }
  n2 = warp_sum(n2);
  r1 = warp_sum(r1);
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
    atomicMax(reinterpret_cast<unsigned int*>(cmax), __float_as_uint(sqrtf(n2f)));
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 1), __float_as_uint(__fsqrt_ru(r1) * 1.0001f));   // ||c - fp16 plane||
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 2), __float_as_uint(__fsqrt_ru(r2) * 1.0001f));   // ||c - bf16 hi - bf16 lo||
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 3), __float_as_uint(__fsqrt_ru(l2) * 1.0001f));   // ||bf16 lo||
  }
}

// Same, with the row in registers: lane l holds elements [128 j + 4 l, +4) in c[j] (D <= 128 NV).  Bit-identical results.
template <int NV>
__device__ __forceinline__ void write_code_operands_regs(const float4 (&crow_regs)[NV], int k, int K, int Kpad, int D,
                                    int metric, uint16_t* planes, uint16_t* bext, float* bias, float* cnorm2, float* cmax, int lane) {
  uint16_t* hi = planes + static_cast<int64_t>(k) * D;
  uint16_t* lo = planes + (static_cast<int64_t>(Kpad) + k) * D;
  uint16_t* qr = planes + (static_cast<int64_t>(2) * Kpad + k) * D;   // the fp16 plane
  double n2 = 0.0;
  float r1 = 0.f, r2 = 0.f, l2 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = j * 128 + lane * 4;
    if (i >= D) continue;
    const float4 c = crow_regs[j];
    const float v[4] = {c.x, c.y, c.z, c.w};
    uint16_t h[4], l[4], q[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      h[e] = float_to_bf16_bits(v[e]);
      const float dl = v[e] - bf16_bits_to_float(h[e]);
      l[e] = float_to_bf16_bits(dl);
      const float d2 = dl - bf16_bits_to_float(l[e]);
      r2 = fmaf(d2, d2, r2);
      l2 = fmaf(bf16_bits_to_float(l[e]), bf16_bits_to_float(l[e]), l2);
      const __half hh = __float2half_rn(fminf(fmaxf(v[e], -65504.f), 65504.f));
      const float d1 = v[e] - __half2float(hh);
      q[e] = __half_as_ushort(hh);
      r1 = fmaf(d1, d1, r1);
      n2 += static_cast<double>(v[e]) * static_cast<double>(v[e]);
    }
    *reinterpret_cast<uint2*>(hi + i) = make_uint2(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16));
    *reinterpret_cast<uint2*>(lo + i) = make_uint2(l[0] | (uint32_t(l[1]) << 16), l[2] | (uint32_t(l[3]) << 16));
    *reinterpret_cast<uint2*>(qr + i) = make_uint2(q[0] | (uint32_t(q[1]) << 16), q[2] | (uint32_t(q[3]) << 16));
  }
  n2 = warp_sum(n2);
  r1 = warp_sum(r1);
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
    atomicMax(reinterpret_cast<unsigned int*>(cmax), __float_as_uint(sqrtf(n2f)));
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 1), __float_as_uint(__fsqrt_ru(r1) * 1.0001f));   // ||c - fp16 plane||
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 2), __float_as_uint(__fsqrt_ru(r2) * 1.0001f));   // ||c - bf16 hi - bf16 lo||
    atomicMax(reinterpret_cast<unsigned int*>(cmax + 3), __float_as_uint(__fsqrt_ru(l2) * 1.0001f));   // ||bf16 lo||
  }
}


}  // namespace vqb
