// Shared host/device helpers for the vqb200 kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#include "../../include/vqb200.h"

namespace vqb {

// Slots of a codebook's cmax (f32 [3], code_operands.cuh): the exact norms that size the search's certification band.
enum CmaxSlot { CMAX_NORM = 0 /* max ||c|| */, CMAX_RES = 1 /* max ||c - hi - lo|| */, CMAX_LO = 2 /* max ||lo|| */, CMAX_SLOTS = 3 };

// MMA N-tile (codes per accumulator): 256 for real codebooks, the 16-rounded size for tiny ones.
__host__ __device__ inline int code_tile(int K) { return K >= 256 ? 256 : ((K + 15) / 16) * 16; }

inline int device_props(int* sms, int* major) {
  static int cached_dev = -1, c_sms = 0, c_major = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return VQB_E_NO_DEVICE;
  if (dev != cached_dev) {
    if (cudaDeviceGetAttribute(&c_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return VQB_E_NO_DEVICE;
    if (cudaDeviceGetAttribute(&c_major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return VQB_E_NO_DEVICE;
    cached_dev = dev;
  }
  *sms = c_sms;
  *major = c_major;
  return VQB_OK;
}
inline int check_device() {
  int sms, major;
  int rc = device_props(&sms, &major);
  if (rc) return rc;
  return major == 9 ? VQB_OK : VQB_E_NO_DEVICE;   // the library carries sm_90a code only
}
inline int num_sms() {
  int sms = 1, major;
  device_props(&sms, &major);
  return sms;
}
// CTAs of a grid-stride loop over `items` at `per_cta` items per CTA: enough to cover them, at most `ctas_per_sm` per SM, at
// least one.
inline int capped_grid(int64_t items, int64_t per_cta, int ctas_per_sm) {
  const int64_t need = (items + per_cta - 1) / per_cta;
  const int64_t cap = static_cast<int64_t>(num_sms()) * ctas_per_sm;
  const int64_t g = need < cap ? need : cap;
  return static_cast<int>(g > 1 ? g : 1);
}

__device__ __forceinline__ float bf16_bits_to_float(uint16_t b) { return __uint_as_float(static_cast<uint32_t>(b) << 16); }
// round-to-nearest-even float -> bf16 bits (finite inputs)
__device__ __forceinline__ uint16_t float_to_bf16_bits(float f) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}
__device__ __forceinline__ float bf16_round(float f) { return bf16_bits_to_float(float_to_bf16_bits(f)); }

template <int DT> struct Elem;
template <> struct Elem<VQB_DTYPE_F32> {
  using T = float;
  static __device__ __forceinline__ float load(const void* p, int64_t i) { return reinterpret_cast<const float*>(p)[i]; }
  static __device__ __forceinline__ void store(void* p, int64_t i, float v) { reinterpret_cast<float*>(p)[i] = v; }
  static __device__ __forceinline__ float round(float v) { return v; }
};
template <> struct Elem<VQB_DTYPE_BF16> {
  using T = uint16_t;
  static __device__ __forceinline__ float load(const void* p, int64_t i) { return bf16_bits_to_float(reinterpret_cast<const uint16_t*>(p)[i]); }
  static __device__ __forceinline__ void store(void* p, int64_t i, float v) { reinterpret_cast<uint16_t*>(p)[i] = float_to_bf16_bits(v); }
  static __device__ __forceinline__ float round(float v) { return bf16_round(v); }
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}


// ---- internal entry points shared between translation units (not part of the C ABI) ----
// vq_assign.cu: vqb_assign_ex plus an optional provisional index array (-1 for rows handed to the exact re-score)
int assign_launch(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
                  const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx, int32_t* idx_prov,
                  int32_t* hist, int hist_shift, vqb_flag_entry* flagged, int32_t* flag_count, float* dbg_best,
                  const vqb_fused_outputs* fused, int metric, const float* cnorm2, void* stream,
                  const uint8_t* row_mask = nullptr /* [N], 0 = padding row: index -1, no tail / loss / statistics */);
// vq_aux.cu: vqb_loss_finalize whose divisor is (*n_live rows) x D when n_live (device, i64[1]) is given — masked batches
int loss_finalize_launch(const double* loss_sum, int64_t numel, const int64_t* n_live, int D, int dtype, float weight,
                         float* loss_out, void* stream);
// vq_ema.cu: add the rows listed in `flagged` (final code = idx[row]) to packed statistics that were built from an
// index array in which those rows were marked -1
int stats_add_flagged(const void* x_eff, int dtype, int64_t N, int D, const vqb_flag_entry* flagged,
                      const int32_t* flag_count, const int32_t* idx, int K, float* stats, void* stream);
// vq_ema.cu: the statistics chain in three steps (vqb_ema_stats = all three, histogram by its own kernel).  With
// prehist the search kernel counts the certified winners into *hist (slabs of 128 << *hist_shift rows) itself.
// zero_before: bytes directly in front of the workspace zeroed by the same memset; stats_stream: optional stream for the
// memset of the statistics (they are not touched before the search ends).
int stats_begin(float* stats, int dtype, int64_t N, int D, int K, void* workspace, size_t workspace_bytes, int prehist,
                size_t zero_before, int32_t** hist, int* hist_shift, void* stats_stream, void* stream);
int stats_scan(const int32_t* idx, int dtype, int64_t N, int D, int K, float* stats, void* workspace, size_t workspace_bytes,
               int prehist, void* stream);
int stats_sum(const void* x_eff, int dtype, int64_t N, int D, const int32_t* idx, int K, float* stats, void* workspace,
              size_t workspace_bytes, void* stream);
// The statistics the EMA apply step lerps towards: one packed buffer p[0] (world == 0), or the sum of `world` ranks' packed
// buffers p[0..world-1] read over peer memory, each already offset to this codebook's slice.
constexpr int MAX_PEERS = 16;
struct EmaStats {
  const float* p[MAX_PEERS];
  int world;
};
inline EmaStats local_stats(const float* stats) {
  EmaStats s = {};
  s.p[0] = stats;
  return s;
}
// vq_peer.cu: the source of vqb_ema_apply_peers (checks the host array of peer pointers and the slice offset)
int peer_stats(EmaStats* src, const void* const* peer_stats_host, int world, int64_t slice_offset);
// vq_ema.cu: vqb_ema_apply_weighted / vqb_ema_apply_peers in two launches (part 1: cluster sizes — needs only the counts —,
// 2: rows, 3: both).  n_lerp statistics slices, slice_stride floats apart, are applied in order (0: no lerp, only the
// normalisation; local statistics only).
int ema_apply_part(int part, const EmaStats& src, float* cluster_size, float* embed_avg, float* embed, int K, int D,
                   double decay, double eps, int metric, int n_lerp, int do_normalise, const float* code_weight,
                   void* planes, void* bext, float* bias, float* cnorm2, float* cmax, float* scratch, void* stream,
                   int64_t slice_stride = 0);


}  // namespace vqb
