// HBM-bound companions of the tensor-core search: operand preparation, exact re-score of flagged
// rows, gather + commitment-loss + residual update, decode.  All are "one warp per row" streaming
// kernels with 16-byte accesses; the codebook (<= a few MiB) stays L2-resident.
#include "vqb_common.cuh"
#include "code_operands.cuh"
#include "gather_row.cuh"

namespace vqb {

constexpr int ROW_THREADS = 256;  // 8 warps = 8 rows in flight per CTA

template <int NV>
__global__ void codebook_prepare_kernel(const float* __restrict__ embed, int K, int Kpad, int D, int metric,
                                        uint16_t* planes, uint16_t* bext, float* bias, float* cnorm2, float* cmax) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= Kpad) return;
  if (k >= K) {
    write_padding_operands(k, Kpad, D, planes, bext, bias, lane);
    return;
  }
  float4 c[NV];
  load_code_row<NV>(embed + static_cast<int64_t>(k) * D, D, lane, c);
  write_code_operands<NV>(c, k, Kpad, D, metric, planes, bext, bias, cnorm2, cmax, lane);
}

// ---------------------------------------------------------------------------------------------
// input staging: l2norm in the input dtype (cosine) and bf16 hi/lo split
// ---------------------------------------------------------------------------------------------
// Vector width: 4 elements per lane and step (16-byte fp32 loads / 8-byte bf16 stores); D % 4 == 0 (host-checked).
template <int DT>
__global__ void input_prepare_kernel(const void* __restrict__ x, int64_t N, int D, int metric, void* x_eff,
                                     uint16_t* planes, int n_planes) {
  using E = Elem<DT>;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const bool cosine = metric == VQB_METRIC_COSINE;
  auto load4 = [&](int64_t at, float* v) {
    if (DT == VQB_DTYPE_F32) {
      const float4 f = *reinterpret_cast<const float4*>(static_cast<const float*>(x) + at);
      v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
      const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(x) + at);
      v[0] = __uint_as_float(u.x << 16); v[1] = __uint_as_float(u.x & 0xFFFF0000u);
      v[2] = __uint_as_float(u.y << 16); v[3] = __uint_as_float(u.y & 0xFFFF0000u);
    }
  };
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb) {
    const int64_t base = row * D;
    float nrm = 1.f;
    if (cosine) {
      double s = 0.0;
      for (int i = lane * 4; i < D; i += 128) {
        float v[4];
        load4(base + i, v);
        s += static_cast<double>(v[0]) * v[0] + static_cast<double>(v[1]) * v[1] + static_cast<double>(v[2]) * v[2] +
             static_cast<double>(v[3]) * v[3];
      }
      s = warp_sum(s);
      nrm = E::round(static_cast<float>(sqrt(s)));  // F.normalize: norm in the tensor dtype ...
      nrm = fmaxf(nrm, 1e-6f);                      // ... clamp_min(eps)
    }
    for (int i = lane * 4; i < D; i += 128) {
      float v[4];
      load4(base + i, v);
      if (cosine) {
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = E::round(__fdiv_rn(v[e], nrm));  // ... x / norm, rounded to the dtype
      }
      if (x_eff) {
        if (DT == VQB_DTYPE_F32) {
          *reinterpret_cast<float4*>(static_cast<float*>(x_eff) + base + i) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
          const uint32_t w0 = float_to_bf16_bits(v[0]) | (static_cast<uint32_t>(float_to_bf16_bits(v[1])) << 16);
          const uint32_t w1 = float_to_bf16_bits(v[2]) | (static_cast<uint32_t>(float_to_bf16_bits(v[3])) << 16);
          *reinterpret_cast<uint2*>(static_cast<uint16_t*>(x_eff) + base + i) = make_uint2(w0, w1);
        }
      }
      if (planes) {
        uint16_t h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          h[e] = float_to_bf16_bits(v[e]);
          l[e] = float_to_bf16_bits(v[e] - bf16_bits_to_float(h[e]));
        }
        *reinterpret_cast<uint2*>(planes + base + i) = make_uint2(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16));
        if (n_planes == 2)
          *reinterpret_cast<uint2*>(planes + N * D + base + i) = make_uint2(l[0] | (uint32_t(l[1]) << 16), l[2] | (uint32_t(l[3]) << 16));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// exact re-score of flagged rows (reference formula and tie rule)
// ---------------------------------------------------------------------------------------------
// Six CTAs per SM (40 registers): the kernel runs next to the statistics sort of vqb_vq_forward's side stream.
template <int DT>
__global__ void __launch_bounds__(ROW_THREADS, 6)
fix_flagged_kernel(const void* __restrict__ x, int64_t N, int D, const float* __restrict__ embed,
                   const float* __restrict__ cnorm2, int K, int metric, vqb_flag_entry* __restrict__ flagged,
                   const int32_t* __restrict__ flag_count, int32_t* idx, const FusedOut fo) {
  using E = Elem<DT>;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  int64_t cnt = *flag_count;
  if (cnt > N) cnt = N;
  for (int64_t e = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); e < cnt;
       e += static_cast<int64_t>(gridDim.x) * wpb) {
    const vqb_flag_entry fe = flagged[e];
    const int64_t base = static_cast<int64_t>(fe.row) * D;
    double x2 = 0.0;
    for (int i = lane; i < D; i += 32) {
      const float v = E::load(x, base + i);
      x2 += static_cast<double>(v) * v;
    }
    const float x2f = static_cast<float>(warp_sum(x2));
    // score(k) exactly as the reference evaluates it in fp32 (vqp:58-62, :741-743); products/sums are
    // accumulated in f64 and rounded once, the "ideal" fp32 GEMM result.
    auto score = [&](int k) -> float {
      const float* c = embed + static_cast<int64_t>(k) * D;
      double xy = 0.0;
      for (int i = lane; i < D; i += 32) xy += static_cast<double>(E::load(x, base + i)) * static_cast<double>(__ldg(c + i));
      const float xyf = static_cast<float>(warp_sum(xy));
      if (metric == VQB_METRIC_COSINE) return xyf;
      const float d2 = __fadd_rn(__fadd_rn(x2f, __ldg(cnorm2 + k)), __fmul_rn(xyf, -2.f));
      return -__fsqrt_rn(fmaxf(d2, 1e-8f));
    };
    if (fe.count > 3 || fe.count < 2) continue;  // (rows with more candidates live at the back of the list: fix_overflow_kernel)
    // two or three candidates, visited in ascending index order: argmax keeps the FIRST maximal index (vqp:140)
    int k0 = fe.cand0, k1 = fe.cand1, k2 = fe.count == 3 ? fe.cand2 : 0x7FFFFFFF;
    if (k0 > k1) { const int t = k0; k0 = k1; k1 = t; }
    if (k1 > k2) { const int t = k1; k1 = k2; k2 = t; }
    if (k0 > k1) { const int t = k0; k0 = k1; k1 = t; }
    int best_k = k0;
    float sbest = score(k0);
    const float s1 = score(k1);
    if (s1 > sbest) { sbest = s1; best_k = k1; }
    if (fe.count == 3) {
      const float s2 = score(k2);
      if (s2 > sbest) { sbest = s2; best_k = k2; }
    }
    if (lane == 0) idx[fe.row] = best_k;
    if (fo.enabled) {  // finish the row the search kernel left to us: gather / loss / residual
      const double l = warp_sum(static_cast<double>(gather_rows<DT, 1>(fo, {int64_t{fe.row}}, {best_k}, D, lane)));
      if (fo.loss_sum && lane == 0) atomicAdd(fo.loss_sum, l);
    }
  }
}

// Rows with more than two codes inside the error band: exact rescan of the WHOLE codebook row.  Work items are
// (flagged entry, chunk of OVF_CHUNK codes) pairs spread over the grid, so one unlucky row of a 16384-code codebook
// is scanned by 128 CTAs in parallel instead of one.  Each item folds its chunk winner into the entry's 64-bit key
// [orderable(score) : ~index] with atomicMax (larger score wins; equal scores: the LOWER index, vqp:140);
// fix_finish_kernel then writes the index and the gather tail.  f64 accumulation, reference formula.
constexpr int OVF_CHUNK = 128;

__device__ __forceinline__ uint32_t orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <int DT>
__global__ void __launch_bounds__(256)
fix_overflow_kernel(const void* __restrict__ x, int64_t N, int D, const float* __restrict__ embed,
                    const float* __restrict__ cnorm2, int K, int metric, vqb_flag_entry* __restrict__ flagged,
                    const int32_t* __restrict__ flag_count) {
  using E = Elem<DT>;
  constexpr int MAXJ = 8;  // D <= 1024
  constexpr int CPI = 8;   // codes per warp iteration: independent L2 gathers in flight
  __shared__ unsigned long long s_key[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the rows to re-scan are the entries at the BACK of the list: flagged[N - 1 - j], j < flag_count[1]
  int64_t n_ovf = flag_count[1];
  if (n_ovf > N) n_ovf = N;
  const int n_chunks = (K + OVF_CHUNK - 1) / OVF_CHUNK;
  const int64_t items = n_ovf * n_chunks;
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int64_t e = N - 1 - it / n_chunks;
    const int chunk = static_cast<int>(it % n_chunks);
    const vqb_flag_entry fe = flagged[e];
    const int64_t base = static_cast<int64_t>(fe.row) * D;
    float xr[MAXJ][4];
    double x2 = 0.0;
#pragma unroll
    for (int j = 0; j < MAXJ; ++j) {
      const int i = lane * 4 + j * 128;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        xr[j][t] = (i + t < D) ? E::load(x, base + i + t) : 0.f;
        x2 += static_cast<double>(xr[j][t]) * xr[j][t];
      }
    }
    const float x2f = static_cast<float>(warp_sum(x2));
    unsigned long long key = 0ull;
    const int k_end = min(K, (chunk + 1) * OVF_CHUNK);
    for (int k0 = chunk * OVF_CHUNK + warp * CPI; k0 < k_end; k0 += 8 * CPI) {
      double acc[CPI];
#pragma unroll
      for (int u = 0; u < CPI; ++u) acc[u] = 0.0;
#pragma unroll
      for (int u = 0; u < CPI; ++u) {
        const int k = k0 + u;
        if (k < k_end) {
          const float* c = embed + static_cast<int64_t>(k) * D;
#pragma unroll
          for (int j = 0; j < MAXJ; ++j) {
            const int i = lane * 4 + j * 128;
            if (i < D) {
              const float4 cv = __ldg(reinterpret_cast<const float4*>(c + i));
              acc[u] += static_cast<double>(xr[j][0]) * cv.x + static_cast<double>(xr[j][1]) * cv.y +
                        static_cast<double>(xr[j][2]) * cv.z + static_cast<double>(xr[j][3]) * cv.w;
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < CPI; ++u) {
        const int k = k0 + u;
        const float xyf = static_cast<float>(warp_sum(acc[u]));
        if (k < k_end) {
          float sc;
          if (metric == VQB_METRIC_COSINE) {
            sc = xyf;
          } else {
            const float d2 = __fadd_rn(__fadd_rn(x2f, __ldg(cnorm2 + k)), __fmul_rn(xyf, -2.f));
            sc = -__fsqrt_rn(fmaxf(d2, 1e-8f));
          }
          const unsigned long long cand = (static_cast<unsigned long long>(orderable(sc)) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(k));
          key = cand > key ? cand : key;
        }
      }
    }
    if (lane == 0) s_key[warp] = key;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long kk = s_key[0];
      for (int w = 1; w < 8; ++w) kk = s_key[w] > kk ? s_key[w] : kk;
      atomicMax(reinterpret_cast<unsigned long long*>(&flagged[e].cand0), kk);
    }
    __syncthreads();
  }
}

// Five CTAs per SM (at most 48 registers): like fix_flagged_kernel, it runs next to the statistics sort.
template <int DT>
__global__ void __launch_bounds__(ROW_THREADS, 5)
fix_finish_kernel(int64_t N, int D, const vqb_flag_entry* __restrict__ flagged, const int32_t* __restrict__ flag_count,
                  int32_t* idx, const FusedOut fo) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  int64_t cnt = flag_count[1];
  if (cnt > N) cnt = N;
  for (int64_t j = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); j < cnt;
       j += static_cast<int64_t>(gridDim.x) * wpb) {
    const int64_t e = N - 1 - j;
    const vqb_flag_entry fe = flagged[e];
    const unsigned long long key = *reinterpret_cast<const unsigned long long*>(&flagged[e].cand0);
    const int k = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull));
    if (lane == 0) idx[fe.row] = k;
    if (fo.enabled) {
      const double l = warp_sum(static_cast<double>(gather_rows<DT, 1>(fo, {int64_t{fe.row}}, {k}, D, lane)));
      if (fo.loss_sum && lane == 0) atomicAdd(fo.loss_sum, l);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// gather + loss + residual update
// ---------------------------------------------------------------------------------------------
template <int DT>
__global__ void gather_kernel(int64_t N, int D, const int32_t* __restrict__ idx, const FusedOut fo) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  float lsum = 0.f;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb)
    lsum += gather_rows<DT, 1>(fo, {row}, {idx[row]}, D, lane);
  if (fo.loss_sum) {
    __shared__ double part[32];
    const double w = warp_sum(static_cast<double>(lsum));
    if (lane == 0) part[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int i = 0; i < wpb; ++i) s += part[i];
      atomicAdd(fo.loss_sum, s);
    }
  }
}

__global__ void loss_finalize_kernel(const double* loss_sum, int64_t numel, const int64_t* n_live, int D, int dtype, float weight,
                                     float* loss_out) {
  if (n_live) numel = max(*n_live, static_cast<int64_t>(1)) * D;   // masked batch: mean over the unmasked elements (vqp:1317-1325)
  float mean = static_cast<float>(*loss_sum / static_cast<double>(numel));
  if (dtype == VQB_DTYPE_BF16) {
    mean = bf16_round(mean);            // F.mse_loss returns a bf16 tensor
    mean = bf16_round(mean * weight);   // commit_loss * commitment_weight stays bf16
    *loss_out = 0.f + mean;             // promoted by the fp32 `loss` accumulator  vqp:1282, :1329
  } else {
    *loss_out = 0.f + mean * weight;
  }
}

// ---------------------------------------------------------------------------------------------
// decode: out[row] = sum_q embed_q[idx[row, q]]   (index -1 -> zeros)      rvq:324-382
// ---------------------------------------------------------------------------------------------
// quantized_out of ResidualVQ.forward rebuilt from the stage indices:  out = (((q_0) + q_1) + ...), q_j = embed_j[idx_j].type(dtype),
// every partial sum rounded to dtype exactly where the reference's `quantized_out = quantized_out + quantized` rounds
// (rvq:525, vqp:1178).  One pass over the indices, code rows from L2, ONE write of (N x D) instead of a read-modify-write
// of the running sum in every stage.
// A warp per row, 8 elements per lane; the Q indices of the row are read once (one lane each) and broadcast; the code rows
// of up to 8 stages are in flight together (the first version chained index load -> row load -> rounding per stage and was
// latency- and instruction-bound: 279 us at config 3 for a 134 MB write).  bf16: round(acc + round(c)) is one packed
// cvt.rn.bf16x2.f32 plus one add.rn.bf16x2 per element pair.
// ROUNDED = false is the decode of get_output_from_indices (rvq:324-382): plain fp32 sum of the gathered rows, index -1 (a
// dropped-out stage) contributes zeros, one rounding at the store.
template <int DT, bool ROUNDED>
__global__ void __launch_bounds__(256, 2) rvq_accumulate_kernel(const float* __restrict__ embeds, int64_t embed_stride, int Q, int D,
                                      const int64_t* __restrict__ idx, int64_t N, void* out) {
  constexpr int QB = 8;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb) {
    for (int i0 = 0; i0 < D; i0 += 256) {   // warp-uniform trip count (shuffles inside)
      const int i = i0 + lane * 8;
      const bool active = i < D;
      float accf[8];
      uint32_t acch[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int e = 0; e < 8; ++e) accf[e] = 0.f;
      for (int qc = 0; qc < Q; qc += 32) {   // indices of (up to) 32 stages: one lane each
        const int64_t kq = (qc + lane < Q) ? idx[row * Q + qc + lane] : 0;
        const int nq = min(32, Q - qc);
        for (int q0 = 0; q0 < nq; q0 += QB) {
          float4 c[QB][2];
          uint32_t skip = 0u;   // stages whose index is -1
#pragma unroll
          for (int b = 0; b < QB; ++b) {
            const int64_t k = __shfl_sync(0xffffffffu, kq, (q0 + b) & 31);
            if (k < 0) skip |= 1u << b;
            if (q0 + b < nq && active && k >= 0) {
              const float4* src = reinterpret_cast<const float4*>(embeds + (qc + q0 + b) * embed_stride + k * D + i);
              c[b][0] = __ldg(src);
              c[b][1] = __ldg(src + 1);
            }
          }
#pragma unroll
          for (int b = 0; b < QB; ++b) {
            if (q0 + b >= nq || !active) continue;
            if ((skip >> b) & 1u) continue;
            const float v[8] = {c[b][0].x, c[b][0].y, c[b][0].z, c[b][0].w, c[b][1].x, c[b][1].y, c[b][1].z, c[b][1].w};
            if (ROUNDED && DT == VQB_DTYPE_BF16) {
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                uint32_t h;
                asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(v[2 * e + 1]), "f"(v[2 * e]));   // round(c)
                asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(acch[e]) : "r"(acch[e]), "r"(h));              // round(acc + round(c))
              }
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) accf[e] += v[e];
            }
          }
        }
      }
      if (!active) continue;
      if (DT == VQB_DTYPE_BF16) {
        if (!ROUNDED) {
#pragma unroll
          for (int e = 0; e < 4; ++e) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(acch[e]) : "f"(accf[2 * e + 1]), "f"(accf[2 * e]));
        }
        *reinterpret_cast<uint4*>(static_cast<uint16_t*>(out) + row * D + i) = make_uint4(acch[0], acch[1], acch[2], acch[3]);
      } else {
        float4* dst = reinterpret_cast<float4*>(static_cast<float*>(out) + row * D + i);
        dst[0] = make_float4(accf[0], accf[1], accf[2], accf[3]);
        dst[1] = make_float4(accf[4], accf[5], accf[6], accf[7]);
      }
    }
  }
}

// Same result with the codebook slice in shared memory.  The kernel above reads Q code rows per output row from L2
// (config 3: 262144 x 8 x 1 KiB = 2.1 GB -> 250 us, L2-bandwidth bound for a 134 MB write).  When one W-column slice of
// every codebook the stages searched fits in smem (a shared codebook: K x W x esz <= 192 KiB), a CTA converts its slice
// once and then serves all its rows from smem: L2 traffic drops to the indices (re-read once per slice) and HBM to the
// output write.  A row is handled by LPR = W*esz/16 adjacent lanes (16 bytes each), 32/LPR rows per warp; 32 warps per
// CTA (one CTA per SM: the slice fills its smem) keep enough index loads in flight — with 8 warps the kernel was as slow as
// the L2 version (244 us: one dependent index load -> smem read chain per warp at a time).
// ROUNDED = false: the decode (fp32 slice, fp32 sum, index -1 contributes zeros, one rounding at the store).
template <int DT, bool ROUNDED>
__global__ void __launch_bounds__(1024, 1)
rvq_accumulate_smem_kernel(const float* __restrict__ embeds, int64_t embed_stride, int nbooks, int Q, int K, int D, int W,
                           const int64_t* __restrict__ idx, int64_t N, void* out, int ctas_per_slice) {
  extern __shared__ uint4 code_smem[];   // [nbooks][K][W] staged elements: bf16 for the rounded bf16 sum, fp32 otherwise
  constexpr bool HALF = ROUNDED && DT == VQB_DTYPE_BF16;
  constexpr int ESZ = HALF ? 2 : 4;                          // staged element
  constexpr int OSZ = DT == VQB_DTYPE_BF16 ? 2 : 4;          // output element
  const int slice = blockIdx.x / ctas_per_slice, part = blockIdx.x % ctas_per_slice;
  const int c0 = slice * W;
  {  // stage the slice: 4 consecutive columns per thread
    const int quads = nbooks * K * (W / 4);
    for (int e = threadIdx.x; e < quads; e += blockDim.x) {
      const int c = (e % (W / 4)) * 4;
      const int r = e / (W / 4);   // book * K + code
      const int book = r / K, code = r % K;
      const float4 v = __ldg(reinterpret_cast<const float4*>(embeds + book * embed_stride + static_cast<int64_t>(code) * D + c0 + c));
      uint8_t* dst = reinterpret_cast<uint8_t*>(code_smem) + (static_cast<size_t>(r) * W + c) * ESZ;
      if (HALF) {
        uint32_t h0, h1;
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h0) : "f"(v.y), "f"(v.x));
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h1) : "f"(v.w), "f"(v.z));
        *reinterpret_cast<uint2*>(dst) = make_uint2(h0, h1);
      } else {
        *reinterpret_cast<float4*>(dst) = v;
      }
    }
  }
  __syncthreads();
  const int LPR = W * ESZ / 16;             // lanes per row (power of two, 4..32) == uint4 per staged code row
  const int rpw = 32 / LPR;                 // rows per warp and iteration
  const int lane = threadIdx.x & 31;
  const int lir = lane & (LPR - 1), riw = lane / LPR;
  const int src_lane0 = riw * LPR;
  const int book_stride = nbooks > 1 ? K * LPR : 0;
  const int64_t gw = static_cast<int64_t>(part) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t step = static_cast<int64_t>(ctas_per_slice) * (blockDim.x >> 5) * rpw;
  const int opl = 16 / ESZ;                 // output elements per lane (8 or 4)
  // running pointers: no 64-bit multiplications in the loop
  const int64_t row0 = gw * rpw + riw;
  const int64_t* ip = idx + row0 * Q + lir;
  uint8_t* op = static_cast<uint8_t*>(out) + (row0 * D + c0 + lir * opl) * OSZ;
  const int64_t ip_step = step * Q;
  const int64_t op_step = step * D * OSZ;
  // the first chunk of indices of the NEXT iteration is requested before this one is consumed
  int kq_next = (row0 < N && lir < Q) ? static_cast<int>(*ip) : 0;
  for (int64_t row = row0, base = gw * rpw; base < N; base += step, row += step, ip += ip_step, op += op_step) {   // warp-uniform
    const bool active = row < N;
    uint32_t acch[4] = {0u, 0u, 0u, 0u};
    float accf[4] = {0.f, 0.f, 0.f, 0.f};
    const int kq_first = kq_next;
    kq_next = (row + step < N && lir < Q) ? static_cast<int>(ip[ip_step]) : 0;
    for (int qc = 0; qc < Q; qc += LPR) {
      const int kq = qc == 0 ? kq_first : ((active && qc + lir < Q) ? static_cast<int>(ip[qc]) : 0);
      const int nq = min(LPR, Q - qc);
      int sbase = qc * book_stride + lir;
      for (int b = 0; b < nq; ++b, sbase += book_stride) {
        const int k = __shfl_sync(0xffffffffu, kq, src_lane0 + b);
        if (!ROUNDED && k < 0) continue;    // (uniform per row group only; the load below is skipped per lane)
        const uint4 v = code_smem[sbase + k * LPR];
        if (HALF) {
          asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(acch[0]) : "r"(acch[0]), "r"(v.x));
          asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(acch[1]) : "r"(acch[1]), "r"(v.y));
          asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(acch[2]) : "r"(acch[2]), "r"(v.z));
          asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(acch[3]) : "r"(acch[3]), "r"(v.w));
        } else {
          accf[0] += __uint_as_float(v.x); accf[1] += __uint_as_float(v.y);
          accf[2] += __uint_as_float(v.z); accf[3] += __uint_as_float(v.w);
        }
      }
    }
    if (!active) continue;
    if (HALF) {
      *reinterpret_cast<uint4*>(op) = make_uint4(acch[0], acch[1], acch[2], acch[3]);
    } else if (DT == VQB_DTYPE_BF16) {
      uint32_t h0, h1;
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h0) : "f"(accf[1]), "f"(accf[0]));
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h1) : "f"(accf[3]), "f"(accf[2]));
      *reinterpret_cast<uint2*>(op) = make_uint2(h0, h1);
    } else {
      *reinterpret_cast<float4*>(op) = make_float4(accf[0], accf[1], accf[2], accf[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// rotation-trick gradient estimator (arXiv:2410.06424; vqp:287-318), forward and backward, one warp per row.
//   u = src / max(||src||, eps), q = tgt / max(||tgt||, eps), w = (u + q) / max(||u + q||, eps)   (all detached)
//   out  = (e - 2 (e.w) w + 2 (e.u) q) * ||tgt|| / max(||src||, eps)          with e = src
//   d_e  = (g - 2 (g.w) w + 2 (g.q) u) * ||tgt|| / max(||src||, eps)          (only `e` carries gradient)
// Every scalar follows from five row reductions (||s||^2, ||t||^2, s.t, g.s, g.t): one sweep for them, one for the row.
// The reductions and the scalars are taken in double: ||u + q||^2 = ||u||^2 + ||q||^2 + 2 u.q and e.(u + q) cancel when src
// points almost opposite to tgt, and in fp32 their rounding noise (~1e-7) swamps ||u + q||^2 below ||u + q|| ~ 5e-4, where the
// eps clamp could then scale the row by up to 1e6.  Products of fp32 values are exact in double, so the sums are exact to
// about D * 2^-53.  nw and the dot products are those of the vectors the second sweep forms with the fp32 ins / int_.
// ---------------------------------------------------------------------------------------------
// One row (one warp) of the estimator.  COMMIT (backward only): out += commit * (src - tgt), the commitment-loss gradient that
// rotate_masked_kernel adds in the same sweep.
template <int DT, bool BWD, bool COMMIT = false>
__device__ __forceinline__ void rotate_row(const void* __restrict__ src, const void* __restrict__ tgt,
                                           const void* __restrict__ grad, int64_t base, int D, int lane, float commit,
                                           void* out) {
  using E = Elem<DT>;
  constexpr float eps = 1e-6f;
  double ss = 0.0, tt = 0.0, st = 0.0, gs = 0.0, gt = 0.0;
  for (int i = lane; i < D; i += 32) {
    const double s = E::load(src, base + i), t = E::load(tgt, base + i);
    ss = fma(s, s, ss); tt = fma(t, t, tt); st = fma(s, t, st);
    if (BWD) { const double g = E::load(grad, base + i); gs = fma(g, s, gs); gt = fma(g, t, gt); }
  }
  ss = warp_sum(ss); tt = warp_sum(tt); st = warp_sum(st);
  if (BWD) { gs = warp_sum(gs); gt = warp_sum(gt); }
  const float ns = static_cast<float>(sqrt(ss)), nt = static_cast<float>(sqrt(tt));
  const float ins = 1.f / fmaxf(ns, eps), int_ = 1.f / fmaxf(nt, eps);        // safe_div (vqp:52-53)
  const double dins = ins, dint = int_;
  // ||u + q||^2 = ||u||^2 + ||q||^2 + 2 u.q
  const double nw = sqrt(fmax(ss * dins * dins + tt * dint * dint + 2.0 * st * dins * dint, 0.0));
  const double dinw = 1.0 / fmax(nw, static_cast<double>(eps));                // l2norm eps (vqp:37-38)
  const float inw = static_cast<float>(dinw);
  const float lam = nt * ins;
  // forward: a = e.w, b = e.u ; backward: a = g.w, b = g.q
  const float a = static_cast<float>(BWD ? (gs * dins + gt * dint) * dinw : (ss * dins + st * dint) * dinw);
  const float b = static_cast<float>(BWD ? gt * dint : ss * dins);
  for (int i = lane; i < D; i += 32) {
    const float s = E::load(src, base + i), t = E::load(tgt, base + i);
    const float u = s * ins, q = t * int_, w = (u + q) * inw;
    const float e = BWD ? E::load(grad, base + i) : s;
    const float r = BWD ? (e - 2.f * a * w + 2.f * b * u) : (e - 2.f * a * w + 2.f * b * q);
    E::store(out, base + i, COMMIT ? r * lam + commit * (s - t) : r * lam);
  }
}

template <int DT, bool BWD>
__global__ void rotate_kernel(const void* __restrict__ src, const void* __restrict__ tgt, const void* __restrict__ grad,
                              int64_t N, int D, void* out) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb)
    rotate_row<DT, BWD>(src, tgt, grad, row * D, D, lane, 0.f, out);
}

// ---------------------------------------------------------------------------------------------
// The estimator of VectorQuantize's masked training step (vqp:1225-1233, :1317-1325, :1378-1389), one warp per row.  Padding
// rows (row_mask 0) are written as the padding value and never reach the estimator: the masked search gives them no code, and
// rotate_to(x, 0) would divide by a zero norm.
//   forward:  live rows tgt (the value both estimators take), padding rows 0 (pad_zeros) or src
//   backward: live rows  estimator'(grad) + c (src - tgt),  c = 2 weight grad_loss[0] / (n_live[0] D)  (0 without grad_loss)
//             padding rows 0 (pad_zeros) or grad
// n_live and grad_loss are read on the device, so the host never waits for them.
// ---------------------------------------------------------------------------------------------
template <int DT, bool BWD>
__global__ void rotate_masked_kernel(const void* __restrict__ src, const void* __restrict__ tgt, const void* __restrict__ grad,
                                     const float* __restrict__ grad_loss, const uint8_t* __restrict__ row_mask,
                                     const int64_t* __restrict__ n_live, float loss_weight, int estimator, int pad_zeros,
                                     int64_t N, int D, void* out) {
  using E = Elem<DT>;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  float commit = 0.f;
  if (BWD && grad_loss) {
    const int64_t nl = *n_live;     // > 0 whenever a live row exists
    if (nl > 0) commit = static_cast<float>(2.0 * loss_weight * static_cast<double>(*grad_loss) / (static_cast<double>(nl) * D));
  }
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5); row < N;
       row += static_cast<int64_t>(gridDim.x) * wpb) {
    const int64_t base = row * D;
    if (!row_mask[row]) {
      const void* from = BWD ? grad : src;
      for (int i = lane; i < D; i += 32) E::store(out, base + i, pad_zeros ? 0.f : E::load(from, base + i));
    } else if (!BWD) {
      for (int i = lane; i < D; i += 32) E::store(out, base + i, E::load(tgt, base + i));
    } else if (estimator == VQB_ESTIMATOR_ROTATE) {
      rotate_row<DT, true, true>(src, tgt, grad, base, D, lane, commit, out);
    } else {
      const bool ste = estimator == VQB_ESTIMATOR_STE;
      for (int i = lane; i < D; i += 32) {
        const float d = commit * (E::load(src, base + i) - E::load(tgt, base + i));
        E::store(out, base + i, ste ? E::load(grad, base + i) + d : d);
      }
    }
  }
}

}  // namespace vqb

using namespace vqb;

extern "C" int vqb_version(void) { return VQB_VERSION; }

extern "C" const char* vqb_strerror(int code) {
  switch (code) {
    case VQB_OK: return "ok";
    case VQB_E_INVALID: return "vqb200: invalid argument (null pointer, non-positive size or bad enum)";
    case VQB_E_UNSUPPORTED: return "vqb200: shape not supported by the sm_90a kernels (need D % 8 == 0, D <= 1024)";
    case VQB_E_ALIGN: return "vqb200: pointer is not 16-byte aligned";
    case VQB_E_NO_DEVICE: return "vqb200: no CUDA device or device is not compute capability 9.x (H100)";
    case VQB_E_DRIVER: return "vqb200: cuTensorMapEncodeTiled unavailable or failed";
    case VQB_E_WORKSPACE: return "vqb200: workspace too small";
    default: break;
  }
  if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
  return "vqb200: unknown error";
}

extern "C" int vqb_codebook_prepare(const float* embed, int K, int D, int metric, void* planes, void* bext, float* bias,
                                    float* cnorm2, float* cmax, void* stream) {
  if (!embed || !planes || !bext || !bias || !cnorm2 || !cmax || K <= 0 || D <= 0) return VQB_E_INVALID;
  if (metric != VQB_METRIC_EUCLID && metric != VQB_METRIC_COSINE) return VQB_E_INVALID;
  if (D % 8 != 0 || D > CODE_ROW_MAX_D) return VQB_E_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(embed) | reinterpret_cast<uintptr_t>(planes)) & 15) return VQB_E_ALIGN;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(cmax, 0, CMAX_SLOTS * sizeof(float), s);
  if (e != cudaSuccess) return static_cast<int>(e);
  const int Kpad = vqb_padded_codes(K);
  const int wpb = ROW_THREADS / 32;
  auto kernel = D <= 4 * 128 ? codebook_prepare_kernel<4> : codebook_prepare_kernel<8>;
  kernel<<<(Kpad + wpb - 1) / wpb, ROW_THREADS, 0, s>>>(embed, K, Kpad, D, metric, static_cast<uint16_t*>(planes),
                                                        static_cast<uint16_t*>(bext), bias, cnorm2, cmax);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_input_prepare(const void* x, int dtype, int64_t N, int D, int metric, void* x_eff, void* a_planes,
                                 int n_planes, void* stream) {
  if (!x || N <= 0 || D <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (a_planes && n_planes != 1 && n_planes != 2) return VQB_E_INVALID;
  if (!x_eff && !a_planes) return VQB_E_INVALID;
  if (D % 4 != 0) return VQB_E_UNSUPPORTED;   // 4 elements per lane and step
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_eff) | reinterpret_cast<uintptr_t>(a_planes)) & 15) return VQB_E_ALIGN;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32)
    input_prepare_kernel<VQB_DTYPE_F32><<<g, ROW_THREADS, 0, s>>>(x, N, D, metric, x_eff, static_cast<uint16_t*>(a_planes), n_planes);
  else
    input_prepare_kernel<VQB_DTYPE_BF16><<<g, ROW_THREADS, 0, s>>>(x, N, D, metric, x_eff, static_cast<uint16_t*>(a_planes), n_planes);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fix_flagged(const void* x_eff, int dtype, int64_t N, int D, const float* embed, const float* cnorm2,
                               int K, int metric, vqb_flag_entry* flagged, const int32_t* flag_count,
                               int32_t* idx, const vqb_fused_outputs* fused, void* stream) {
  if (!x_eff || !embed || !cnorm2 || !flagged || !flag_count || !idx || N <= 0 || D <= 0 || K <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D > 1024) return VQB_E_UNSUPPORTED;
  FusedOut fo;
  int rc = make_fused(&fo, fused, D, N);
  if (rc) return rc;
  if (fo.enabled && fo.dtype != dtype) return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // flag_count is only known on the device: fixed grids stride over the list.  The pair / triple re-score is a chain of
  // dependent loads per row (entry -> x row in HBM -> code rows in L2): many warps in flight, about one row each.
  const int g = num_sms() * 2;
  const int gp = num_sms() * 8;
  if (dtype == VQB_DTYPE_F32) {
    fix_flagged_kernel<VQB_DTYPE_F32><<<gp, ROW_THREADS, 0, s>>>(x_eff, N, D, embed, cnorm2, K, metric, flagged, flag_count, idx, fo);
    fix_overflow_kernel<VQB_DTYPE_F32><<<g, 256, 0, s>>>(x_eff, N, D, embed, cnorm2, K, metric, flagged, flag_count);
    fix_finish_kernel<VQB_DTYPE_F32><<<g, ROW_THREADS, 0, s>>>(N, D, flagged, flag_count, idx, fo);
  } else {
    fix_flagged_kernel<VQB_DTYPE_BF16><<<gp, ROW_THREADS, 0, s>>>(x_eff, N, D, embed, cnorm2, K, metric, flagged, flag_count, idx, fo);
    fix_overflow_kernel<VQB_DTYPE_BF16><<<g, 256, 0, s>>>(x_eff, N, D, embed, cnorm2, K, metric, flagged, flag_count);
    fix_finish_kernel<VQB_DTYPE_BF16><<<g, ROW_THREADS, 0, s>>>(N, D, flagged, flag_count, idx, fo);
  }
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_gather(const void* x_eff, int dtype, int64_t N, int D, const float* embed, const int32_t* idx,
                          void* q_out, int64_t* idx64_out, int64_t idx_stride, double* loss_sum, const void* x_raw,
                          void* resid_out, void* qsum, void* stream) {
  if (!x_eff || !embed || !idx || N <= 0 || D <= 0) return VQB_E_INVALID;
  vqb_fused_outputs f = {};
  f.x_eff = x_eff; f.embed = embed; f.q_out = q_out; f.idx64_out = idx64_out; f.idx_stride = idx_stride;
  f.loss_sum = loss_sum; f.x_raw = x_raw; f.resid_out = resid_out; f.qsum = qsum; f.dtype = dtype;
  FusedOut fo;
  const int rc = make_fused(&fo, &f, D);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32) gather_kernel<VQB_DTYPE_F32><<<g, ROW_THREADS, 0, s>>>(N, D, idx, fo);
  else gather_kernel<VQB_DTYPE_BF16><<<g, ROW_THREADS, 0, s>>>(N, D, idx, fo);
  return static_cast<int>(cudaGetLastError());
}

int vqb::loss_finalize_launch(const double* loss_sum, int64_t numel, const int64_t* n_live, int D, int dtype, float weight,
                              float* loss_out, void* stream) {
  if (!loss_sum || !loss_out || numel <= 0) return VQB_E_INVALID;
  loss_finalize_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(loss_sum, numel, n_live, D, dtype, weight, loss_out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_loss_finalize(const double* loss_sum, int64_t numel, int dtype, float weight, float* loss_out,
                                 void* stream) {
  return vqb::loss_finalize_launch(loss_sum, numel, nullptr, 1, dtype, weight, loss_out, stream);
}

// Slice plan of the smem gather-sum for nbooks codebooks of K x D staged as esz-byte elements, N rows, `sms` SMs:
// out3 = {W, slices = D / W, CTAs per slice}.  W is the widest power-of-two column slice of all the codebooks that fits in
// 192 KiB with a row piece of 64..512 staged bytes (4..32 lanes x 16 bytes); W = 0 (the L2 kernel) when none fits or when
// N < 4096, where staging the slices costs more than the rows it serves.
static void gather_sum_plan(int nbooks, int K, int D, int esz, int64_t N, int sms, int* out3) {
  int W = 0;
  for (int w = 512 / esz; w * esz >= 64; w >>= 1)
    if (D % w == 0 && static_cast<size_t>(nbooks) * K * w * esz <= 196608) { W = w; break; }
  if (N < 4096) W = 0;
  out3[0] = W;
  out3[1] = W ? D / W : 0;
  out3[2] = W ? max(1, sms / (D / W)) : 0;
}

// smem variant of the gather-sum (rounded running sum / decode); false when the plan picks the L2 kernel
template <bool ROUNDED>
static bool gather_sum_smem(const float* embeds, int64_t embed_stride, int Q, int K, int D, const int64_t* idx, int64_t N, void* out,
                            int dtype, cudaStream_t s) {
  const int esz = (ROUNDED && dtype == VQB_DTYPE_BF16) ? 2 : 4;
  const int nbooks = embed_stride ? Q : 1;
  int plan[3];
  gather_sum_plan(nbooks, K, D, esz, N, num_sms(), plan);
  const int W = plan[0], slices = plan[1], cps = plan[2];
  if (!W) return false;
  const size_t smem = static_cast<size_t>(nbooks) * K * W * esz;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(rvq_accumulate_smem_kernel<VQB_DTYPE_F32, ROUNDED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 196608);
    cudaFuncSetAttribute(rvq_accumulate_smem_kernel<VQB_DTYPE_BF16, ROUNDED>, cudaFuncAttributeMaxDynamicSharedMemorySize, 196608);
    attr_set = true;
  }
  if (dtype == VQB_DTYPE_F32)
    rvq_accumulate_smem_kernel<VQB_DTYPE_F32, ROUNDED><<<slices * cps, 1024, smem, s>>>(embeds, embed_stride, nbooks, Q, K, D, W, idx, N, out, cps);
  else
    rvq_accumulate_smem_kernel<VQB_DTYPE_BF16, ROUNDED><<<slices * cps, 1024, smem, s>>>(embeds, embed_stride, nbooks, Q, K, D, W, idx, N, out, cps);
  return true;
}

extern "C" int vqb_decode(const float* embeds, int64_t embed_stride, int Q, int K, int D, const int64_t* idx, int64_t N,
                          void* out, int dtype, void* stream) {
  if (!embeds || !idx || !out || Q <= 0 || K <= 0 || D <= 0 || N <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D % 8 != 0) return VQB_E_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (gather_sum_smem<false>(embeds, embed_stride, Q, K, D, idx, N, out, dtype, s)) return static_cast<int>(cudaGetLastError());
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32)
    rvq_accumulate_kernel<VQB_DTYPE_F32, false><<<g, ROW_THREADS, 0, s>>>(embeds, embed_stride, Q, D, idx, N, out);
  else
    rvq_accumulate_kernel<VQB_DTYPE_BF16, false><<<g, ROW_THREADS, 0, s>>>(embeds, embed_stride, Q, D, idx, N, out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_rvq_accumulate(const float* embeds, int64_t embed_stride, int Q, int K, int D, const int64_t* idx, int64_t N,
                                  void* out, int dtype, void* stream) {
  if (!embeds || !idx || !out || Q <= 0 || K <= 0 || D <= 0 || N <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D % 8 != 0) return VQB_E_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (gather_sum_smem<true>(embeds, embed_stride, Q, K, D, idx, N, out, dtype, s)) return static_cast<int>(cudaGetLastError());
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32)
    rvq_accumulate_kernel<VQB_DTYPE_F32, true><<<g, ROW_THREADS, 0, s>>>(embeds, embed_stride, Q, D, idx, N, out);
  else
    rvq_accumulate_kernel<VQB_DTYPE_BF16, true><<<g, ROW_THREADS, 0, s>>>(embeds, embed_stride, Q, D, idx, N, out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_debug_gather_sum_plan(int nbooks, int K, int D, int esz, int64_t N, int sms, int* out3) {
  if (!out3 || nbooks <= 0 || K <= 0 || D <= 0 || N <= 0 || sms <= 0 || (esz != 2 && esz != 4)) return VQB_E_INVALID;
  gather_sum_plan(nbooks, K, D, esz, N, sms, out3);
  return VQB_OK;
}

extern "C" int vqb_rotate(const void* src, const void* tgt, const void* grad_out, int64_t N, int D, int dtype, void* out,
                          void* stream) {
  if (!src || !tgt || !out || N <= 0 || D <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  if (dtype == VQB_DTYPE_F32) {
    if (grad_out) rotate_kernel<VQB_DTYPE_F32, true><<<g, ROW_THREADS, 0, s>>>(src, tgt, grad_out, N, D, out);
    else rotate_kernel<VQB_DTYPE_F32, false><<<g, ROW_THREADS, 0, s>>>(src, tgt, nullptr, N, D, out);
  } else {
    if (grad_out) rotate_kernel<VQB_DTYPE_BF16, true><<<g, ROW_THREADS, 0, s>>>(src, tgt, grad_out, N, D, out);
    else rotate_kernel<VQB_DTYPE_BF16, false><<<g, ROW_THREADS, 0, s>>>(src, tgt, nullptr, N, D, out);
  }
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_rotate_masked(const void* src, const void* tgt, const void* grad_out, const float* grad_loss,
                                 const uint8_t* row_mask, const int64_t* n_live, float loss_weight, int estimator,
                                 int pad_zeros, int64_t N, int D, int dtype, void* out, void* stream) {
  if (!src || !tgt || !row_mask || !out || N <= 0 || D <= 0) return VQB_E_INVALID;
  if (grad_loss && !n_live) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (estimator != VQB_ESTIMATOR_NONE && estimator != VQB_ESTIMATOR_STE && estimator != VQB_ESTIMATOR_ROTATE)
    return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = capped_grid(N, ROW_THREADS / 32, 16);
  const int pz = pad_zeros ? 1 : 0;
  if (dtype == VQB_DTYPE_F32) {
    if (grad_out)
      rotate_masked_kernel<VQB_DTYPE_F32, true><<<g, ROW_THREADS, 0, s>>>(src, tgt, grad_out, grad_loss, row_mask, n_live,
                                                                          loss_weight, estimator, pz, N, D, out);
    else
      rotate_masked_kernel<VQB_DTYPE_F32, false><<<g, ROW_THREADS, 0, s>>>(src, tgt, nullptr, nullptr, row_mask, nullptr,
                                                                           0.f, estimator, pz, N, D, out);
  } else {
    if (grad_out)
      rotate_masked_kernel<VQB_DTYPE_BF16, true><<<g, ROW_THREADS, 0, s>>>(src, tgt, grad_out, grad_loss, row_mask, n_live,
                                                                           loss_weight, estimator, pz, N, D, out);
    else
      rotate_masked_kernel<VQB_DTYPE_BF16, false><<<g, ROW_THREADS, 0, s>>>(src, tgt, nullptr, nullptr, row_mask, nullptr,
                                                                            0.f, estimator, pz, N, D, out);
  }
  return static_cast<int>(cudaGetLastError());
}
