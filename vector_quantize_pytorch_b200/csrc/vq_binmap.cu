// BinaryMapper (binary_mapper.py, "bm"): the O(rows * 2^bits) part of the straight-through one-hot.  Three kernels:
//
//   binmap_hot_kernel       one thread per row: writes the hot element of the zero-filled output, 1 or, with straight-through,
//                           fl(fl(1 + s) - s) with s = exp(sum_j term_j) (bm:173-180).  A row with a non-finite logit writes
//                           the reference's whole row: NaN where a per-bit term is 0 * -inf, 0 elsewhere.
//   binmap_bwd_kernel       d logits of sum(out * g) without the (rows, K) soft codes: one thread per (row, K chunk), the
//                           warp stages 32 threads' g segments through shared memory so every load is coalesced.  soft_G
//                           factorises, s_k = TA[k >> lb] * TB[k & (seg - 1)], and the per-bit sums S1_j = sum_{bit_j(k)=1}
//                           g_k s_k and S0_j (bit 0) come from the segment column (low bits) and per-segment sums (high bits).
//   binmap_bwd_fin_kernel   adds the K chunks' fp64 partials in chunk order: d logit_j = sigmoid(-l_j) S1_j - sigmoid(l_j) S0_j.
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int BM_MAX_BITS = 20;
constexpr int HOT_THREADS = 256;
constexpr int BWD_THREADS = 128;
constexpr int BWD_WARPS = BWD_THREADS / 32;
constexpr int BWD_MIN_SEGS = 8;         // a K chunk holds at least 8 segments (256 codes) once K allows it
constexpr int BWD_THREADS_PER_SM = 1024;   // the K split grows until rows x ksplit reaches this many threads per SM

// log sigmoid(x) as torch's F.logsigmoid: min(x, 0) - log1p(exp(-|x|)); -inf at -inf, 0 at +inf, NaN at NaN
__device__ __forceinline__ float log_sigmoid(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }

// ---- forward: the hot element ----

__global__ void __launch_bounds__(HOT_THREADS) binmap_hot_kernel(const float* __restrict__ logits, const int64_t* __restrict__ idx,
                                                                  int64_t rows, int bits, float* __restrict__ out) {
  const int64_t K = int64_t{1} << bits;
  for (int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; r < rows; r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t hot = idx[r];
    if (hot < 0 || hot >= K) continue;
    float* o = out + r * K;
    if (!logits) {   // no straight-through: F.one_hot
      o[hot] = 1.f;
      continue;
    }
    const float* l = logits + r * bits;
    // per-bit term of the hot code, c ls(l) + (1 - c) ls(-l) with IEEE products (the two einsums of bm:173-176)
    float sum = 0.f;
    uint32_t pos = 0, neg = 0;
    bool nan = false;
    for (int j = 0; j < bits; ++j) {
      const float v = l[j];
      const float c = static_cast<float>((hot >> j) & 1);
      sum += c * log_sigmoid(v) + (1.f - c) * log_sigmoid(-v);
      nan |= isnan(v);
      if (isinf(v)) (v > 0.f ? pos : neg) |= 1u << j;
    }
    const float s = expf(sum);
    o[hot] = __fsub_rn(__fadd_rn(1.f, s), s);
    if (!(nan || pos || neg)) continue;
    // the slow row: code k's sum is NaN iff a term is (NaN logit; bit 1 under +inf; bit 0 under -inf), else 0 + s - s = 0
    const uint32_t kmask = static_cast<uint32_t>(K - 1);
    auto val = [&](int64_t k) {
      const uint32_t ku = static_cast<uint32_t>(k);
      return (nan || (ku & pos) || (~ku & kmask & neg)) ? __int_as_float(0x7fffffff) : 0.f;
    };
    const float hv = o[hot];
    if (K >= 4) {
      float4* o4 = reinterpret_cast<float4*>(o);
      for (int64_t k = 0; k < K; k += 4) o4[k >> 2] = make_float4(val(k), val(k + 1), val(k + 2), val(k + 3));
    } else {
      for (int64_t k = 0; k < K; ++k) o[k] = val(k);
    }
    o[hot] = hv;
  }
}

// ---- backward ----

struct BwdArgs {
  const float* logits;   // [rows][bits]
  const float* g;        // g[r * gs_row + k * gs_col]
  int64_t gs_row, gs_col;
  int64_t rows;
  int bits;
  int ksplit;            // K chunks per row
  int64_t segs_per_chunk;
  double* work;          // [rows][ksplit][2 bits] (S0_j, S1_j) when ksplit > 1
  float* dlogits;        // [rows][bits]
};

// Item = (row, chunk), one per thread, consecutive items in consecutive lanes.  A segment is SEG = 2^LB consecutive codes:
// the low LB bits of k are the column c inside it, the high bits the segment index.
template <int LB>
__global__ void __launch_bounds__(BWD_THREADS) binmap_bwd_kernel(BwdArgs a) {
  constexpr int SEG = 1 << LB;
  constexpr int HB = LB == 5 ? BM_MAX_BITS : LB;   // below 32 codes a row is one segment: no high bits
  constexpr int NH = HB - LB > 0 ? HB - LB : 1;
  __shared__ float stage[BWD_WARPS][32][SEG + 1];
  __shared__ int64_t base[BWD_WARPS][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t items = a.rows * a.ksplit;
  const int64_t item = static_cast<int64_t>(blockIdx.x) * BWD_THREADS + threadIdx.x;
  const bool valid = item < items;
  const int64_t row = valid ? item / a.ksplit : 0;
  const int chunk = valid ? static_cast<int>(item - row * a.ksplit) : 0;
  const int bits = a.bits;
  const int64_t seg0 = chunk * a.segs_per_chunk;   // global index of the chunk's first segment
  base[warp][lane] = valid ? row * a.gs_row + (seg0 << LB) * a.gs_col : -1;

  // per-bit log-sigmoids; the low bits go into the column table TB, the high ones into TA per segment
  float l1[HB], l0[HB];
  bool finite = true;
#pragma unroll
  for (int j = 0; j < HB; ++j) {
    const float v = (valid && j < bits) ? a.logits[row * bits + j] : 0.f;
    finite &= isfinite(v);
    l1[j] = log_sigmoid(v);
    l0[j] = log_sigmoid(-v);
  }
  float tb[SEG];
#pragma unroll
  for (int c = 0; c < SEG; ++c) {
    float t = 0.f;
#pragma unroll
    for (int b = 0; b < LB; ++b) t += ((c >> b) & 1) ? l1[b] : l0[b];
    tb[c] = expf(t);
  }
  // fp32 sums over one segment, added to fp64 accumulators (a row sums up to 2^20 terms)
  double lo1[LB], lo0[LB], hi1[NH], hi0[NH];   // hi*[j - LB]: bit j >= LB
#pragma unroll
  for (int b = 0; b < LB; ++b) lo1[b] = lo0[b] = 0.0;
#pragma unroll
  for (int j = 0; j < NH; ++j) hi1[j] = hi0[j] = 0.0;
  __syncwarp();

  for (int64_t s = 0; s < a.segs_per_chunk; ++s) {
    // stage the warp's 32 segments: 32 x SEG floats, SEG / 32 segments per load instruction
    float v[SEG];
#pragma unroll
    for (int t = 0; t < SEG; ++t) {
      const int e = t * 32 + lane, i = e >> LB, c = e & (SEG - 1);
      const int64_t b0 = base[warp][i];
      v[t] = b0 >= 0 ? a.g[b0 + ((s << LB) + c) * a.gs_col] : 0.f;
    }
#pragma unroll
    for (int t = 0; t < SEG; ++t) {
      const int e = t * 32 + lane;
      stage[warp][e >> LB][e & (SEG - 1)] = v[t];
    }
    __syncwarp();
    float s1[LB], s0[LB];
#pragma unroll
    for (int b = 0; b < LB; ++b) s1[b] = s0[b] = 0.f;
#pragma unroll
    for (int c = 0; c < SEG; ++c) {
      const float x = stage[warp][lane][c] * tb[c];
#pragma unroll
      for (int b = 0; b < LB; ++b) {
        if ((c >> b) & 1) s1[b] += x;
        else s0[b] += x;
      }
    }
    __syncwarp();
    const int64_t gs = seg0 + s;
    float la = 0.f;
#pragma unroll
    for (int j = LB; j < HB; ++j)
      if (j < bits) la += ((gs >> (j - LB)) & 1) ? l1[j] : l0[j];
    const double ta = static_cast<double>(expf(la));
#pragma unroll
    for (int b = 0; b < LB; ++b) {
      lo1[b] += ta * static_cast<double>(s1[b]);
      lo0[b] += ta * static_cast<double>(s0[b]);
    }
    const double tot = ta * static_cast<double>(s1[0] + s0[0]);
#pragma unroll
    for (int j = LB; j < HB; ++j)
      if (j < bits) {
        if ((gs >> (j - LB)) & 1) hi1[j - LB] += tot;
        else hi0[j - LB] += tot;
      }
  }
  if (!valid) return;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  auto S1 = [&](int j) { return !finite ? qnan : j < LB ? lo1[j] : hi1[j - LB]; };
  auto S0 = [&](int j) { return !finite ? qnan : j < LB ? lo0[j] : hi0[j - LB]; };
  if (a.ksplit == 1) {
#pragma unroll
    for (int j = 0; j < HB; ++j)
      if (j < bits) {
        const double x = static_cast<double>(a.logits[row * bits + j]);
        const double p = 1.0 / (1.0 + exp(-x)), q = 1.0 / (1.0 + exp(x));
        a.dlogits[row * bits + j] = static_cast<float>(q * S1(j) - p * S0(j));
      }
  } else {
    double* w = a.work + item * (2 * bits);
#pragma unroll
    for (int j = 0; j < HB; ++j)
      if (j < bits) {
        w[2 * j] = S0(j);
        w[2 * j + 1] = S1(j);
      }
  }
}

__global__ void binmap_bwd_fin_kernel(BwdArgs a) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= a.rows * a.bits) return;
  const int64_t row = i / a.bits;
  const int j = static_cast<int>(i - row * a.bits);
  const double* w = a.work + row * a.ksplit * (2 * a.bits) + 2 * j;
  double s0 = 0.0, s1 = 0.0;
  for (int c = 0; c < a.ksplit; ++c) {
    s0 += w[static_cast<int64_t>(c) * 2 * a.bits];
    s1 += w[static_cast<int64_t>(c) * 2 * a.bits + 1];
  }
  const double x = static_cast<double>(a.logits[i]);
  const double p = 1.0 / (1.0 + exp(-x)), q = 1.0 / (1.0 + exp(x));
  a.dlogits[i] = static_cast<float>(q * s1 - p * s0);
}

// The K split and the segment width for (rows, bits) on `sms` SMs.
void bwd_plan(int64_t rows, int bits, int sms, int* ksplit, int* seg) {
  const int lb = bits < 5 ? bits : 5;
  const int64_t nseg = int64_t{1} << (bits - lb);
  const int64_t max_split = nseg >= BWD_MIN_SEGS ? nseg / BWD_MIN_SEGS : 1;
  const int64_t target = static_cast<int64_t>(sms > 0 ? sms : 1) * BWD_THREADS_PER_SM;
  int64_t k = 1;
  while (k < max_split && rows * k < target) k <<= 1;
  *ksplit = static_cast<int>(k);
  *seg = 1 << lb;
}

}  // namespace
}  // namespace vqb

extern "C" int vqb_binmap_hot(const float* logits, const int64_t* idx, int64_t rows, int bits, float* out, void* stream) {
  using namespace vqb;
  if (!idx || !out || rows <= 0 || bits < 1) return VQB_E_INVALID;
  if (bits > BM_MAX_BITS || rows >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  if (!aligned(out, 16) || !aligned(idx, 8) || (logits && !aligned(logits, 4))) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(rows, HOT_THREADS, 16);
  binmap_hot_kernel<<<grid, HOT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(logits, idx, rows, bits, out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_binmap_backward_plan(int64_t rows, int bits, int sms, int* plan) {
  if (!plan || rows <= 0 || bits < 1 || sms < 1) return VQB_E_INVALID;
  if (bits > vqb::BM_MAX_BITS) return VQB_E_UNSUPPORTED;
  vqb::bwd_plan(rows, bits, sms, &plan[0], &plan[1]);
  return VQB_OK;
}

extern "C" int vqb_binmap_backward(const float* logits, int64_t rows, int bits, const float* g, int64_t g_row_stride,
                                   int64_t g_col_stride, int ksplit, double* work, float* dlogits, void* stream) {
  using namespace vqb;
  if (!logits || !g || !dlogits || rows <= 0 || bits < 1 || g_row_stride < 0 || g_col_stride < 0) return VQB_E_INVALID;
  if (bits > BM_MAX_BITS || rows >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  const int lb = bits < 5 ? bits : 5;
  const int64_t nseg = int64_t{1} << (bits - lb);
  if (ksplit < 1 || (ksplit & (ksplit - 1)) || ksplit > nseg || (ksplit > 1 && !work)) return VQB_E_INVALID;
  if (!aligned(logits, 4) || !aligned(g, 4) || !aligned(dlogits, 4) || (work && !aligned(work, 8))) return VQB_E_ALIGN;
  const int64_t items = rows * ksplit, blocks = (items + BWD_THREADS - 1) / BWD_THREADS;
  if (blocks >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if (const int rc = check_device()) return rc;
  const BwdArgs a{logits, g, g_row_stride, g_col_stride, rows, bits, ksplit, nseg / ksplit, work, dlogits};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>(blocks);
  switch (lb) {
    case 1: binmap_bwd_kernel<1><<<grid, BWD_THREADS, 0, s>>>(a); break;
    case 2: binmap_bwd_kernel<2><<<grid, BWD_THREADS, 0, s>>>(a); break;
    case 3: binmap_bwd_kernel<3><<<grid, BWD_THREADS, 0, s>>>(a); break;
    case 4: binmap_bwd_kernel<4><<<grid, BWD_THREADS, 0, s>>>(a); break;
    default: binmap_bwd_kernel<5><<<grid, BWD_THREADS, 0, s>>>(a); break;
  }
  if (ksplit > 1) {
    const int64_t n = rows * bits;
    binmap_bwd_fin_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(a);
  }
  return static_cast<int>(cudaGetLastError());
}
