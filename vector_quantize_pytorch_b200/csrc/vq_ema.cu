// EMA codebook update:  batch statistics (cluster_size, embed_sum) and the lerp / Laplace-smoothed
// normalisation of vector_quantize_pytorch.py:76-97, :152-154, :576-617.
//
// The reference computes embed_sum with a third dense GEMM (x^T . one_hot, :605).  Here it is a
// segmented reduction: counting sort of the rows by code (CTA-local histograms + column scan + smem-cursor
// scatter: no global atomics), then one CTA sums the rows of one code with
// coalesced 8/16-byte loads — x is read exactly once, no float atomics on the common path (only codes
// with more than SEG_CHUNK rows are split and combined with atomicAdd).
#include "vqb_common.cuh"
#include "code_operands.cuh"

namespace vqb {

constexpr int SEG_CHUNK = 512;    // rows per work item (every item accumulates atomically: a finer split only balances the load)
constexpr int SEG_THREADS = 256;

struct StatsWs {  // carved out of the caller's workspace
  int32_t* counts;   // [K]
  int32_t* offsets;  // [K]   exclusive scan of counts
  int32_t* cursor;   // [K]   running insert position
  int32_t* nwork;    // [1]
  int32_t* perm;     // [N]   row ids grouped by code
  int4* work;        // [K + N/SEG_CHUNK + 1]  {code, begin, end, split}
  int32_t* ticket;      // [1] (64 ints reserved) directly in front of cta_counts: zeroed by the same memset
  int32_t* cta_counts;  // [sort_ctas][K]  per-CTA histograms -> (in place) each CTA's insert base inside a code's segment
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int64_t max_work_items(int64_t N, int K) { return K + N / SEG_CHUNK + 1; }

// CTA-local counting sort (K <= SORT_MAX_K): every CTA owns a contiguous slab of rows, histograms it in smem, and —
// after a column scan over the CTAs — scatters its row ids with smem cursors only.  No global atomics, and the
// 256-way contention of a global cursor per code (25 us at config 2) is gone.
constexpr int SORT_THREADS = 512;
constexpr int SORT_MAX_K = 16384;           // K ints of smem per CTA
constexpr int64_t SORT_MAX_CELLS = 1 << 22; // cap on sort_ctas * K (16 MiB of workspace)
// device-independent upper bound (workspace queries must not depend on the device)
static int64_t sort_ctas_bound(int64_t N, int K) {
  int64_t g = (N + 511) / 512;              // >= 512 rows per CTA
  if (g > 512) g = 512;
  if (g > SORT_MAX_CELLS / K) g = SORT_MAX_CELLS / K;
  return g < 1 ? 1 : g;
}
// Slabs of (128 << shift) rows — whole row tiles of the search kernel, which can therefore count its certified winners
// per slab itself (AssignParams::hist).  At most one slab per SM (`sms`; the scatter is a single wave), at least 512 rows each.
static int sort_ctas(int64_t N, int K, int sms, int* shift) {
  // Few rows per code: a global cursor per code sees little contention, while the per-CTA histograms would move
  // sort_ctas * K counters three times (config 4: N/K = 4, measured 1.58 -> 1.71 ms per step with the CTA-local path).
  if (K > SORT_MAX_K || N < 32 * static_cast<int64_t>(K)) { *shift = 31; return 0; }   // -> global-atomic kernels
  const int64_t tiles = (N + 127) / 128;
  int64_t cap = sms;
  if (cap > 256) cap = 256;   // colscan_kernel: 32 warps x 8 slabs in registers
  if (cap > SORT_MAX_CELLS / K) cap = SORT_MAX_CELLS / K;
  if (cap < 1) cap = 1;
  int sh = 2;
  while (((tiles + (1ll << sh) - 1) >> sh) > cap) ++sh;
  *shift = sh;
  return static_cast<int>((tiles + (1ll << sh) - 1) >> sh);
}

static size_t carve(StatsWs* ws, void* base, int64_t N, int K) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  // ticket block + slab histograms FIRST: vq_forward.cu zeroes its own counters (the 256 bytes in front of this workspace)
  // with the same memset
  const size_t o_cta = take(256 + sizeof(int32_t) * static_cast<size_t>(K <= SORT_MAX_K ? sort_ctas_bound(N, K) * K : 0));
  const size_t o_counts = take(sizeof(int32_t) * K);
  const size_t o_offsets = take(sizeof(int32_t) * K);
  const size_t o_cursor = take(sizeof(int32_t) * K);
  const size_t o_nwork = take(sizeof(int32_t));
  const size_t o_perm = take(sizeof(int32_t) * N);
  const size_t o_work = take(sizeof(int4) * max_work_items(N, K));
  if (ws && base) {
    uint8_t* b = static_cast<uint8_t*>(base);
    ws->counts = reinterpret_cast<int32_t*>(b + o_counts);
    ws->offsets = reinterpret_cast<int32_t*>(b + o_offsets);
    ws->cursor = reinterpret_cast<int32_t*>(b + o_cursor);
    ws->nwork = reinterpret_cast<int32_t*>(b + o_nwork);
    ws->perm = reinterpret_cast<int32_t*>(b + o_perm);
    ws->work = reinterpret_cast<int4*>(b + o_work);
    ws->ticket = reinterpret_cast<int32_t*>(b + o_cta);
    ws->cta_counts = reinterpret_cast<int32_t*>(b + o_cta + 256);
  }
  return off;
}

__global__ void hist_kernel(const int32_t* __restrict__ idx, int64_t N, int K, int32_t* counts) {
  extern __shared__ int32_t sh[];
  const bool use_sh = K <= 8192;
  if (use_sh) {
    for (int i = threadIdx.x; i < K; i += blockDim.x) sh[i] = 0;
    __syncthreads();
  }
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < N;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = idx[r];
    if (k < 0) continue;
    if (use_sh) atomicAdd(&sh[k], 1); else atomicAdd(&counts[k], 1);
  }
  if (use_sh) {
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x)
      if (sh[i]) atomicAdd(&counts[i], sh[i]);
  }
}

// CTA c histograms rows [c*rows_per_cta, (c+1)*rows_per_cta) into cta_counts[c][:]
__global__ void __launch_bounds__(SORT_THREADS)
hist_cta_kernel(const int32_t* __restrict__ idx, int64_t N, int K, int64_t rows_per_cta, int32_t* __restrict__ cta_counts) {
  extern __shared__ int32_t sh[];
  for (int i = threadIdx.x; i < K; i += SORT_THREADS) sh[i] = 0;
  __syncthreads();
  const int64_t b = blockIdx.x * rows_per_cta;
  const int64_t e = min(N, b + rows_per_cta);
  for (int64_t r = b + threadIdx.x; r < e; r += SORT_THREADS) {
    const int k = idx[r];
    if (k >= 0) atomicAdd(&sh[k], 1);   // -1: row accounted for elsewhere (stats_add_flagged)
  }
  __syncthreads();
  int32_t* out = cta_counts + static_cast<size_t>(blockIdx.x) * K;
  for (int i = threadIdx.x; i < K; i += SORT_THREADS) out[i] = sh[i];
}

// offsets = exclusive_scan(counts) over the codes; the work list of the segmented sums; the cluster_size part of the
// statistics (added atomically: the buffer was zeroed, and the re-scored rows may be added concurrently).  Runs on ONE
// block of any size (a multiple of 32 threads).
__device__ void scan_codes_block(const int32_t* counts, int K, int32_t* offsets, int32_t* cursor, int4* work, int32_t* nwork,
                                 float* stats) {
  __shared__ int32_t s_c[32], s_w[32];
  __shared__ int32_t carry_cnt, carry_wk, tot_cnt, tot_wk;
  const int nt = blockDim.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = nt >> 5;
  if (threadIdx.x == 0) { carry_cnt = 0; carry_wk = 0; }
  __syncthreads();
  for (int base = 0; base < K; base += nt) {
    const int k = base + threadIdx.x;
    const int c = k < K ? __ldcg(counts + k) : 0;
    const int w = (c + SEG_CHUNK - 1) / SEG_CHUNK;   // 0 for an empty code: its sums stay at the zero they were set to
    int ic = c, iw = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, ic, o), b = __shfl_up_sync(0xffffffffu, iw, o);
      if (lane >= o) { ic += a; iw += b; }
    }
    if (lane == 31) { s_c[warp] = ic; s_w[warp] = iw; }
    __syncthreads();
    if (warp == 0) {
      int a = lane < nwarps ? s_c[lane] : 0, b = lane < nwarps ? s_w[lane] : 0;
      const int a0 = a, b0 = b;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, a, o), y = __shfl_up_sync(0xffffffffu, b, o);
        if (lane >= o) { a += x; b += y; }
      }
      s_c[lane] = a - a0;   // exclusive prefix of the warps
      s_w[lane] = b - b0;
      if (lane == 31) { tot_cnt = a; tot_wk = b; }
    }
    __syncthreads();
    const int wc = s_c[warp], ww = s_w[warp];
    const int ex_cnt = carry_cnt + wc + ic - c;
    const int ex_wk = carry_wk + ww + iw - w;
    if (k < K) {
      offsets[k] = ex_cnt;
      if (cursor) cursor[k] = ex_cnt;
      if (c) atomicAdd(stats + k, static_cast<float>(c));  // cluster_size = onehot.sum(1)   vqp:602 (exact: integers < 2^24)
      for (int j = 0; j < w; ++j) {
        const int b = ex_cnt + j * SEG_CHUNK;
        const int e = min(ex_cnt + c, b + SEG_CHUNK);
        work[ex_wk + j] = make_int4(k, b, e, 0);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) { carry_cnt += tot_cnt; carry_wk += tot_wk; }
    __syncthreads();
  }
  if (threadIdx.x == 0) *nwork = carry_wk;
}

// Exclusive scan down the slab axis (in place) + each code's total, then — in the LAST block to finish (ticket) — the
// scan over the codes: one launch instead of two on the critical path of the step.  A block owns 32 adjacent codes
// (coalesced 128-byte rows of the [G][K] matrix); its 8 warps split the slab axis, scan their stretch, and are stitched
// together through smem — two short passes instead of one G-long dependent chain per code.
constexpr int CS_CODES = 32, CS_PARTS = 32, CS_PER = 8;   // 32 warps per block; a warp scans at most CS_PER slabs from registers
__global__ void __launch_bounds__(CS_CODES * CS_PARTS)
colscan_kernel(int32_t* __restrict__ cta_counts, int G, int K, int32_t* __restrict__ counts, int32_t* ticket,
               int32_t* offsets, int4* work, int32_t* nwork, float* stats) {
  __shared__ int32_t part[CS_PARTS][CS_CODES + 1];
  __shared__ int s_last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int k = blockIdx.x * CS_CODES + lane;
  const int per = (G + CS_PARTS - 1) / CS_PARTS;   // <= CS_PER (host: G <= CS_PARTS * CS_PER)
  const int g0 = min(G, w * per), g1 = min(G, g0 + per);
  // one round trip: every slab count of this warp's stretch is loaded before the first use and stays in registers
  int v[CS_PER];
  int sum = 0;
#pragma unroll
  for (int j = 0; j < CS_PER; ++j) {
    v[j] = (k < K && g0 + j < g1) ? __ldcg(cta_counts + static_cast<size_t>(g0 + j) * K + k) : 0;   // written by REDs: L2
    sum += v[j];
  }
  part[w][lane] = sum;
  __syncthreads();
  int run = 0, total = 0;
#pragma unroll 8
  for (int q = 0; q < CS_PARTS; ++q) { const int x = part[q][lane]; run += (q < w) ? x : 0; total += x; }
  if (k < K) {
#pragma unroll
    for (int j = 0; j < CS_PER; ++j) {
      if (g0 + j < g1) cta_counts[static_cast<size_t>(g0 + j) * K + k] = run;
      run += v[j];
    }
    if (w == 0) counts[k] = total;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1) == static_cast<int>(gridDim.x) - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) *ticket = 0;   // ready for the next launch
  scan_codes_block(counts, K, offsets, nullptr, work, nwork, stats);
}

// CTA c scatters the row ids of its slab: position = offsets[k] + (its base inside the code's segment) + smem cursor
__global__ void __launch_bounds__(SORT_THREADS)
scatter_cta_kernel(const int32_t* __restrict__ idx, int64_t N, int K, int64_t rows_per_cta,
                   const int32_t* __restrict__ cta_counts, const int32_t* __restrict__ offsets, int32_t* __restrict__ perm) {
  extern __shared__ int32_t sh[];
  const int32_t* base = cta_counts + static_cast<size_t>(blockIdx.x) * K;
  for (int i = threadIdx.x; i < K; i += SORT_THREADS) sh[i] = offsets[i] + base[i];
  __syncthreads();
  const int64_t b = blockIdx.x * rows_per_cta;
  const int64_t e = min(N, b + rows_per_cta);
  for (int64_t r = b + threadIdx.x; r < e; r += SORT_THREADS) {
    const int k = idx[r];
    if (k < 0) continue;
    const int pos = atomicAdd(&sh[k], 1);
    perm[pos] = static_cast<int32_t>(r);
  }
}

// single CTA (global-cursor path): offsets = exclusive_scan(counts); work list; cluster_size part of stats
__global__ void scan_kernel(const int32_t* __restrict__ counts, int K, int32_t* offsets, int32_t* cursor, int4* work,
                            int32_t* nwork, float* stats) {
  scan_codes_block(counts, K, offsets, cursor, work, nwork, stats);
}

__global__ void scatter_kernel(const int32_t* __restrict__ idx, int64_t N, int32_t* cursor, int32_t* perm) {
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; r < N;
       r += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = idx[r];
    if (k < 0) continue;
    const int pos = atomicAdd(&cursor[k], 1);
    perm[pos] = static_cast<int32_t>(r);
  }
}

// one CTA per work item: embed_sum[code] (+)= sum of the rows perm[begin:end]        vqp:605
// The row ids of the segment are staged in smem first, so the gather loop has a single dependent global
// load per row and keeps UNROLL independent 16-byte row loads in flight per thread.
template <int DT>
__global__ void __launch_bounds__(SEG_THREADS)
segsum_kernel(const void* __restrict__ x, int D, const int32_t* __restrict__ perm, const int4* __restrict__ work,
              const int32_t* __restrict__ nwork, float* embed_sum) {
  if (static_cast<int>(blockIdx.x) >= *nwork) return;
  constexpr int VEC = (DT == VQB_DTYPE_BF16) ? 8 : 4;  // elements per 16-byte load
  constexpr int UNROLL = 8;
  extern __shared__ __align__(16) uint8_t seg_smem[];
  int32_t* s_perm = reinterpret_cast<int32_t*>(seg_smem);                 // [SEG_CHUNK]
  float* red = reinterpret_cast<float*>(seg_smem + SEG_CHUNK * sizeof(int32_t));  // [NY][D]
  const int4 wk = work[blockIdx.x];
  const int nrows = wk.z - wk.y;
  for (int i = threadIdx.x; i < nrows; i += SEG_THREADS) s_perm[i] = perm[wk.y + i];
  __syncthreads();
  const int TX = D / VEC;               // threads across one row (D % 8 == 0)
  const int NY = SEG_THREADS / TX;      // row lanes
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  float acc[VEC];
#pragma unroll
  for (int e = 0; e < VEC; ++e) acc[e] = 0.f;
  if (ty < NY) {
    const uint8_t* xb = reinterpret_cast<const uint8_t*>(x) + static_cast<size_t>(tx) * 16;
    const size_t row_bytes = static_cast<size_t>(D) * (DT == VQB_DTYPE_BF16 ? 2 : 4);
    auto accumulate = [&](const uint4& u) {
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      if (DT == VQB_DTYPE_BF16) {
#pragma unroll
        for (int e = 0; e < 4; ++e) { acc[(2 * e) % VEC] += __uint_as_float(w[e] << 16); acc[(2 * e + 1) % VEC] += __uint_as_float(w[e] & 0xFFFF0000u); }
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e % VEC] += __uint_as_float(w[e]);
      }
    };
    int r = ty;
    for (; r + (UNROLL - 1) * NY < nrows; r += UNROLL * NY) {
      uint4 u[UNROLL];
#pragma unroll
      for (int q = 0; q < UNROLL; ++q) u[q] = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(s_perm[r + q * NY]) * row_bytes));
#pragma unroll
      for (int q = 0; q < UNROLL; ++q) accumulate(u[q]);
    }
    for (; r < nrows; r += NY) accumulate(__ldg(reinterpret_cast<const uint4*>(xb + static_cast<size_t>(s_perm[r]) * row_bytes)));
    float* dst = red + ty * D + tx * VEC;
#pragma unroll
    for (int e = 0; e < VEC; ++e) dst[e] = acc[e];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float s = 0.f;
    for (int y = 0; y < NY; ++y) s += red[y * D + i];
    float* out = embed_sum + static_cast<int64_t>(wk.x) * D + i;
    atomicAdd(out, s);   // onto zeros (or onto the re-scored rows of this code, added concurrently)
  }
}

// one warp per flagged row: cluster_size[k] += 1, embed_sum[k] += x[row]   (k = the row's final code)
template <int DT>
__global__ void stats_add_flagged_kernel(const void* __restrict__ x, int64_t N, int D, const vqb_flag_entry* __restrict__ flagged,
                                         const int32_t* __restrict__ flag_count, const int32_t* __restrict__ idx,
                                         float* stats, int64_t soff) {
  using E = Elem<DT>;
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  // front of the list: rows with 2 / 3 candidates; back of the list (from N - 1 downwards): the re-scanned rows
  int64_t cnt = flag_count[0], cnt_back = flag_count[1];
  if (cnt > N) cnt = N;
  if (cnt_back > N - cnt) cnt_back = N - cnt;
  for (int64_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < cnt + cnt_back; j += warps) {
    const int64_t e = j < cnt ? j : N - 1 - (j - cnt);
    const int row = flagged[e].row;
    const int k = idx[row];
    if (lane == 0) atomicAdd(stats + k, 1.f);
    float* dst = stats + soff + static_cast<int64_t>(k) * D;
    for (int i = lane * 4; i < D; i += 128) {   // 16-byte vector reductions (D % 8 == 0, rows 16-byte aligned)
      const int64_t o = static_cast<int64_t>(row) * D + i;
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + i), "f"(E::load(x, o)), "f"(E::load(x, o + 1)),
                   "f"(E::load(x, o + 2)), "f"(E::load(x, o + 3)) : "memory");
    }
  }
}

// ---------------------------------------------------------------------------------------------
// EMA apply
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float lerp_f32(float a, float b, float w) {  // torch.lerp
  return (fabsf(w) < 0.5f) ? a + w * (b - a) : b - (b - a) * (1.f - w);
}

// Statistics sources of the apply kernels: element i (float4 at i) of the packed statistics [cluster_size | embed_sum].
struct LocalStats {
  const float* p;
  __device__ __forceinline__ float load(int64_t i) const { return p[i]; }
  __device__ __forceinline__ float4 load4(int64_t i) const { return *reinterpret_cast<const float4*>(p + i); }
};
// The sum over the ranks' buffers (vqp:603, :607).  Every peer load is in flight before the first add (NVLink latency ~2 us),
// and the adds run in rank order from 0: every rank performs the identical fp32 additions, so the replicas stay bit-identical.
struct PeerStats {
  EmaStats s;
  __device__ __forceinline__ float load(int64_t i) const {
    float v[MAX_PEERS];
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < s.world) v[r] = s.p[r][i];
    float n = 0.f;
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < s.world) n += v[r];
    return n;
  }
  __device__ __forceinline__ float4 load4(int64_t i) const {
    float4 v[MAX_PEERS];
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < s.world) v[r] = *reinterpret_cast<const float4*>(s.p[r] + i);
    float4 n = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < s.world) { n.x += v[r].x; n.y += v[r].y; n.z += v[r].z; n.w += v[r].w; }
    return n;
  }
};

// single CTA: cluster_size.lerp_ (vqp:616) and its sum (vqp:577); zero cmax for the atomicMax that follows
// n_lerp statistics slices (slice_stride floats apart) are applied one after the other — the Q stages of a ResidualVQ that
// share one codebook (rvq:302-306: every layer lerps the same buffers in turn) in ONE launch.
template <class Src>
__global__ void ema_sizes_kernel(float* cluster_size, const Src src, int K, float w, const float* __restrict__ code_weight,
                                 int n_lerp, int64_t slice_stride, float* scratch, float* cmax) {
  __shared__ double part[32];
  double s = 0.0;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float c = cluster_size[k];
    if (n_lerp) {  // (1 - decay) * weight, an fp32 product (vqp:86-97)
      const float wk = code_weight ? __fmul_rn(w, code_weight[k]) : w;
      for (int j = 0; j < n_lerp; ++j) c = lerp_f32(c, src.load(j * slice_stride + k), wk);
      cluster_size[k] = c;
    }
    s += c;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += part[i];
    scratch[0] = static_cast<float>(t);
    if (cmax) { cmax[CMAX_NORM] = 0.f; cmax[CMAX_RES] = 0.f; cmax[CMAX_LO] = 0.f; }
  }
}

// one warp per (padded) code: embed_avg.lerp_ (vqp:617); embed = embed_avg / smoothed (vqp:576-584); refresh the tensor-core
// operands of that row.  The row stays in registers (D <= 128 NV): one round trip for the loads, and every later phase —
// lerp, divide, l2norm, operand split — works on registers (this kernel sits on the critical path of every step).
template <int NV, class Src>
__global__ void ema_rows_kernel(const float* __restrict__ cluster_size, float* embed_avg, float* embed, const Src src,
                                int64_t soff, int K, int Kpad, int D, float w, const float* __restrict__ code_weight, float eps,
                                float keps, int metric, int n_lerp, int64_t slice_stride, int do_normalise,
                                const float* __restrict__ scratch, uint16_t* planes, uint16_t* bext, float* bias, float* cnorm2,
                                float* cmax) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= Kpad) return;
  if (k >= K) {
    if (do_normalise) write_padding_operands(k, Kpad, D, planes, bext, bias, lane);
    return;
  }
  float* avg = embed_avg + static_cast<int64_t>(k) * D;
  float* emb = embed + static_cast<int64_t>(k) * D;
  float4 a[NV];
  load_code_row<NV>(avg, D, lane, a);
  if (code_weight) w = __fmul_rn(w, code_weight[k]);
  const int64_t roff = soff + static_cast<int64_t>(k) * D;
  for (int q = 0; q < n_lerp; ++q) {
    float4 b[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int i = j * 128 + lane * 4;
      if (i < D) b[j] = src.load4(q * slice_stride + roff + i);
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int i = j * 128 + lane * 4;
      if (i >= D) continue;
      a[j].x = lerp_f32(a[j].x, b[j].x, w); a[j].y = lerp_f32(a[j].y, b[j].y, w);
      a[j].z = lerp_f32(a[j].z, b[j].z, w); a[j].w = lerp_f32(a[j].w, b[j].w, w);
    }
  }
  if (n_lerp) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int i = j * 128 + lane * 4;
      if (i < D) *reinterpret_cast<float4*>(avg + i) = a[j];
    }
  }
  if (!do_normalise) return;
  // laplace_smoothing(cluster_size, K, eps) * cluster_size.sum()      vqp:152-154, :577
  const float total = scratch[0];
  const float denom = __fmul_rn(__fdiv_rn(__fadd_rn(cluster_size[k], eps), __fadd_rn(total, keps)), total);
  double n2 = 0.0;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = j * 128 + lane * 4;
    if (i >= D) continue;
    a[j] = make_float4(__fdiv_rn(a[j].x, denom), __fdiv_rn(a[j].y, denom), __fdiv_rn(a[j].z, denom), __fdiv_rn(a[j].w, denom));
    if (metric == VQB_METRIC_COSINE)
      n2 += static_cast<double>(a[j].x) * a[j].x + static_cast<double>(a[j].y) * a[j].y + static_cast<double>(a[j].z) * a[j].z +
            static_cast<double>(a[j].w) * a[j].w;
  }
  if (metric == VQB_METRIC_COSINE) {  // l2norm(embed_normalized)     vqp:581-582, eps 1e-6 (:37-38)
    const float nrm = fmaxf(static_cast<float>(sqrt(warp_sum(n2))), 1e-6f);
#pragma unroll
    for (int j = 0; j < NV; ++j)
      a[j] = make_float4(__fdiv_rn(a[j].x, nrm), __fdiv_rn(a[j].y, nrm), __fdiv_rn(a[j].z, nrm), __fdiv_rn(a[j].w, nrm));
  }
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int i = j * 128 + lane * 4;
    if (i < D) *reinterpret_cast<float4*>(emb + i) = a[j];
  }
  write_code_operands<NV>(a, k, Kpad, D, metric, planes, bext, bias, cnorm2, cmax, lane);
}

template <class Src>
static void ema_launch(int part, const Src& src, float* cluster_size, float* embed_avg, float* embed, int K, int D, float w,
                       const float* code_weight, float eps, float keps, int metric, int n_lerp, int64_t slice_stride,
                       int do_normalise, uint16_t* planes, uint16_t* bext, float* bias, float* cnorm2, float* cmax,
                       float* scratch, cudaStream_t s) {
  if (part & 1)
    ema_sizes_kernel<Src><<<1, 1024, 0, s>>>(cluster_size, src, K, w, code_weight, n_lerp, slice_stride, scratch,
                                             do_normalise ? cmax : nullptr);
  if (part & 2) {
    const int Kpad = vqb_padded_codes(K);
    const int wpb = 8;
    const int64_t soff = vqb_stats_offset(K);
    auto rows = D <= 4 * 128 ? ema_rows_kernel<4, Src> : ema_rows_kernel<8, Src>;
    rows<<<(Kpad + wpb - 1) / wpb, wpb * 32, 0, s>>>(cluster_size, embed_avg, embed, src, soff, K, Kpad, D, w, code_weight, eps, keps,
                                                    metric, n_lerp, slice_stride, do_normalise, scratch, planes, bext, bias, cnorm2,
                                                    cmax);
  }
}

}  // namespace vqb

using namespace vqb;

extern "C" int64_t vqb_stats_offset(int K) { return K <= 0 ? 0 : (static_cast<int64_t>(K) + 3) / 4 * 4; }
extern "C" int64_t vqb_stats_floats(int K, int D) { return (K <= 0 || D <= 0) ? 0 : vqb_stats_offset(K) + static_cast<int64_t>(K) * D; }

int vqb::stats_add_flagged(const void* x_eff, int dtype, int64_t N, int D, const vqb_flag_entry* flagged,
                           const int32_t* flag_count, const int32_t* idx, int K, float* stats, void* stream) {
  if (!x_eff || !flagged || !flag_count || !idx || !stats) return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int g = num_sms() * 8;
  const int64_t soff = vqb_stats_offset(K);
  if (dtype == VQB_DTYPE_F32) stats_add_flagged_kernel<VQB_DTYPE_F32><<<g, 256, 0, s>>>(x_eff, N, D, flagged, flag_count, idx, stats, soff);
  else stats_add_flagged_kernel<VQB_DTYPE_BF16><<<g, 256, 0, s>>>(x_eff, N, D, flagged, flag_count, idx, stats, soff);
  return static_cast<int>(cudaGetLastError());
}

extern "C" size_t vqb_ema_stats_workspace(int64_t N, int K) {
  if (N <= 0 || K <= 0) return 0;
  return carve(nullptr, nullptr, N, K);
}

// The sort plan of the statistics for (N, K) on a device with `sms` SMs: out3 = {slabs G (0: global-atomic path), shift
// (slabs of 128 << shift rows; 31 on the global path), the device-independent slab bound the workspace is sized with}.
extern "C" int vqb_debug_stats_plan(int64_t N, int K, int sms, int* out3) {
  if (!out3 || N <= 0 || K <= 0 || sms <= 0) return VQB_E_INVALID;
  if (N >= (static_cast<int64_t>(1) << 31)) return VQB_E_UNSUPPORTED;
  int shift = 31;
  out3[0] = sort_ctas(N, K, sms, &shift);
  out3[1] = shift;
  out3[2] = static_cast<int>(sort_ctas_bound(N, K));
  return VQB_OK;
}

// ---- the statistics chain in three steps, so that vq_forward.cu can interleave it with the search and the re-score:
//   stats_begin  (before the search)  zero the packed statistics and the histogram the search kernel counts into
//   stats_scan   (after the search)   [histogram, unless the search made it] + slab scan + code scan + cluster sizes
//   stats_sum    (after stats_scan)   scatter of the row ids + segmented row sums
static int stats_check(const void* x_eff, int dtype, int64_t N, int D, int K, const float* stats, const void* workspace,
                       size_t workspace_bytes, StatsWs* ws) {
  if (!stats || !workspace || N <= 0 || D <= 0 || K <= 0) return VQB_E_INVALID;
  if (dtype != VQB_DTYPE_F32 && dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (D % 8 != 0 || D > 4 * SEG_THREADS) return VQB_E_UNSUPPORTED;  // TX = D/VEC <= SEG_THREADS
  if (N >= (static_cast<int64_t>(1) << 31)) return VQB_E_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(x_eff) | reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(stats)) & 15)
    return VQB_E_ALIGN;
  if (carve(ws, const_cast<void*>(workspace), N, K) > workspace_bytes) return VQB_E_WORKSPACE;
  return VQB_OK;
}

int vqb::stats_begin(float* stats, int dtype, int64_t N, int D, int K, void* workspace, size_t workspace_bytes, int prehist,
                     size_t zero_before, int32_t** hist, int* hist_shift, void* stats_stream, void* stream) {
  StatsWs ws;
  int rc = stats_check(stats, dtype, N, D, K, stats, workspace, workspace_bytes, &ws);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // everything below accumulates onto zeros: the cluster sizes (scan), the row sums (segmented sums, split or not) and the
  // re-scored rows (stats_add_flagged), in any order.  Nothing touches the statistics before the search has finished, so
  // this memset may run on another stream next to it (stats_stream).
  cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(float) * static_cast<size_t>(vqb_stats_floats(K, D)),
                                  static_cast<cudaStream_t>(stats_stream ? stats_stream : stream));
  if (e != cudaSuccess) return static_cast<int>(e);
  int shift = 31;
  const int G = sort_ctas(N, K, num_sms(), &shift);
  // [caller's counters (zero_before bytes) | ticket block | slab histograms, when the search kernel counts into them]
  e = cudaMemsetAsync(reinterpret_cast<uint8_t*>(ws.ticket) - zero_before, 0,
                      zero_before + 256 + ((G > 0 && prehist) ? sizeof(int32_t) * static_cast<size_t>(G) * K : 0), s);
  if (e != cudaSuccess) return static_cast<int>(e);
  if (G == 0) {
    e = cudaMemsetAsync(ws.counts, 0, sizeof(int32_t) * K, s);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (hist) *hist = G > 0 ? ws.cta_counts : ws.counts;
  if (hist_shift) *hist_shift = shift;
  return VQB_OK;
}

int vqb::stats_scan(const int32_t* idx, int dtype, int64_t N, int D, int K, float* stats, void* workspace,
                    size_t workspace_bytes, int prehist, void* stream) {
  StatsWs ws;
  int rc = stats_check(stats, dtype, N, D, K, stats, workspace, workspace_bytes, &ws);
  if (rc) return rc;
  if (!idx) return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int shift = 31;
  const int G = sort_ctas(N, K, num_sms(), &shift);
  if (G > 0) {
    static bool attr_set = false;
    if (!attr_set) {  // K ints of dynamic smem: up to 64 KiB
      cudaFuncSetAttribute(hist_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_MAX_K * 4);
      cudaFuncSetAttribute(scatter_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_MAX_K * 4);
      attr_set = true;
    }
    const int64_t rows_per_cta = static_cast<int64_t>(128) << shift;
    if (!prehist) hist_cta_kernel<<<G, SORT_THREADS, static_cast<size_t>(K) * sizeof(int32_t), s>>>(idx, N, K, rows_per_cta, ws.cta_counts);
    colscan_kernel<<<(K + CS_CODES - 1) / CS_CODES, CS_CODES * CS_PARTS, 0, s>>>(ws.cta_counts, G, K, ws.counts, ws.ticket,
                                                                              ws.offsets, ws.work, ws.nwork, stats);
  } else {
    if (!prehist) {
      int g = static_cast<int>((N + 1023) / 1024);
      const int cap = num_sms() * 4;
      if (g > cap) g = cap;
      hist_kernel<<<g, 256, K <= 8192 ? K * sizeof(int32_t) : 0, s>>>(idx, N, K, ws.counts);
    }
    scan_kernel<<<1, 1024, 0, s>>>(ws.counts, K, ws.offsets, ws.cursor, ws.work, ws.nwork, stats);
  }
  return static_cast<int>(cudaGetLastError());
}

int vqb::stats_sum(const void* x_eff, int dtype, int64_t N, int D, const int32_t* idx, int K, float* stats, void* workspace,
                   size_t workspace_bytes, void* stream) {
  StatsWs ws;
  int rc = stats_check(x_eff, dtype, N, D, K, stats, workspace, workspace_bytes, &ws);
  if (rc) return rc;
  if (!x_eff || !idx) return VQB_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int shift = 31;
  const int G = sort_ctas(N, K, num_sms(), &shift);
  if (G > 0) {
    scatter_cta_kernel<<<G, SORT_THREADS, static_cast<size_t>(K) * sizeof(int32_t), s>>>(idx, N, K, static_cast<int64_t>(128) << shift,
                                                                                        ws.cta_counts, ws.offsets, ws.perm);
  } else {
    int g = static_cast<int>((N + 1023) / 1024);
    const int cap = num_sms() * 4;
    if (g > cap) g = cap;
    scatter_kernel<<<g, 256, 0, s>>>(idx, N, ws.cursor, ws.perm);
  }
  const int64_t soff = vqb_stats_offset(K);
  const int items = static_cast<int>(max_work_items(N, K));
  const int TX = D / (dtype == VQB_DTYPE_BF16 ? 8 : 4);
  const size_t red_bytes = SEG_CHUNK * sizeof(int32_t) + static_cast<size_t>(SEG_THREADS / TX) * D * sizeof(float);
  if (dtype == VQB_DTYPE_F32)
    segsum_kernel<VQB_DTYPE_F32><<<items, SEG_THREADS, red_bytes, s>>>(x_eff, D, ws.perm, ws.work, ws.nwork, stats + soff);
  else
    segsum_kernel<VQB_DTYPE_BF16><<<items, SEG_THREADS, red_bytes, s>>>(x_eff, D, ws.perm, ws.work, ws.nwork, stats + soff);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_ema_stats(const void* x_eff, int dtype, int64_t N, int D, const int32_t* idx, int K, float* stats,
                             void* workspace, size_t workspace_bytes, void* stream) {
  if (!x_eff || !idx) return VQB_E_INVALID;
  int rc = stats_begin(stats, dtype, N, D, K, workspace, workspace_bytes, 0, 0, nullptr, nullptr, nullptr, stream);
  if (rc) return rc;
  rc = stats_scan(idx, dtype, N, D, K, stats, workspace, workspace_bytes, 0, stream);
  if (rc) return rc;
  return stats_sum(x_eff, dtype, N, D, idx, K, stats, workspace, workspace_bytes, stream);
}

extern "C" int vqb_ema_apply(float* cluster_size, float* embed_avg, float* embed, const float* stats, int K, int D,
                             double decay, double eps, int metric, int do_lerp, int do_normalise, void* planes,
                             void* bext, float* bias, float* cnorm2, float* cmax, float* scratch, void* stream) {
  return vqb_ema_apply_weighted(cluster_size, embed_avg, embed, stats, K, D, decay, eps, metric, do_lerp, do_normalise,
                                nullptr, planes, bext, bias, cnorm2, cmax, scratch, stream);
}

extern "C" int vqb_ema_apply_weighted(float* cluster_size, float* embed_avg, float* embed, const float* stats, int K, int D,
                                      double decay, double eps, int metric, int do_lerp, int do_normalise,
                                      const float* code_weight, void* planes, void* bext, float* bias, float* cnorm2,
                                      float* cmax, float* scratch, void* stream) {
  return ema_apply_part(3, local_stats(stats), cluster_size, embed_avg, embed, K, D, decay, eps, metric, do_lerp ? 1 : 0,
                        do_normalise, code_weight, planes, bext, bias, cnorm2, cmax, scratch, stream);
}

extern "C" int vqb_ema_apply_peers(float* cluster_size, float* embed_avg, float* embed, const void* const* peer_stats_host,
                                   int world, int64_t slice_offset, int K, int D, double decay, double eps, int metric,
                                   int do_normalise, const float* code_weight, void* planes, void* bext, float* bias,
                                   float* cnorm2, float* cmax, float* scratch, void* stream) {
  EmaStats src;
  const int rc = peer_stats(&src, peer_stats_host, world, slice_offset);
  if (rc) return rc;
  return ema_apply_part(3, src, cluster_size, embed_avg, embed, K, D, decay, eps, metric, 1, do_normalise, code_weight, planes,
                        bext, bias, cnorm2, cmax, scratch, stream);
}

// part: 1 = the cluster sizes (needs only the counts of the statistics), 2 = the rows (needs part 1 and the row sums), 3 = both
int vqb::ema_apply_part(int part, const EmaStats& src, float* cluster_size, float* embed_avg, float* embed, int K, int D,
                        double decay, double eps, int metric, int n_lerp, int do_normalise, const float* code_weight,
                        void* planes, void* bext, float* bias, float* cnorm2, float* cmax, float* scratch, void* stream,
                        int64_t slice_stride) {
  if (!cluster_size || !embed_avg || !embed || !scratch || K <= 0 || D <= 0 || n_lerp < 0) return VQB_E_INVALID;
  if (n_lerp && (!src.p[0] || (slice_stride & 3))) return VQB_E_INVALID;
  if (!n_lerp && src.world) return VQB_E_INVALID;
  if (do_normalise && (!planes || !bext || !bias || !cnorm2 || !cmax)) return VQB_E_INVALID;
  if (D % 8 != 0 || D > CODE_ROW_MAX_D) return VQB_E_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(embed_avg) | reinterpret_cast<uintptr_t>(embed) | reinterpret_cast<uintptr_t>(planes)) & 15)
    return VQB_E_ALIGN;
  const int64_t soff = vqb_stats_offset(K);
  for (int r = 0; n_lerp && r < (src.world ? src.world : 1); ++r)
    if ((reinterpret_cast<uintptr_t>(src.p[r]) | reinterpret_cast<uintptr_t>(src.p[r] + soff)) & 15) return VQB_E_ALIGN;
  const float w = static_cast<float>(1.0 - decay);  // (1. - decay) evaluated in python float, then fp32 (vqp:97)
  const float epsf = static_cast<float>(eps);
  const float keps = static_cast<float>(static_cast<double>(K) * eps);  // n_categories * eps in python float (vqp:154)
  uint16_t* pl = static_cast<uint16_t*>(planes);
  uint16_t* be = static_cast<uint16_t*>(bext);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (src.world)
    ema_launch(part, PeerStats{src}, cluster_size, embed_avg, embed, K, D, w, code_weight, epsf, keps, metric, n_lerp, slice_stride,
               do_normalise, pl, be, bias, cnorm2, cmax, scratch, s);
  else
    ema_launch(part, LocalStats{src.p[0]}, cluster_size, embed_avg, embed, K, D, w, code_weight, epsf, keps, metric, n_lerp,
               slice_stride, do_normalise, pl, be, bias, cnorm2, cmax, scratch, s);
  return static_cast<int>(cudaGetLastError());
}
