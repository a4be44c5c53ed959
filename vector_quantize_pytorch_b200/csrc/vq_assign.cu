// Nearest-code search on the Hopper tensor cores (sm_90a: TMA, mbarrier, wgmma).
//
// Replaces the reference's   dist = -cdist(x, embed) | einsum(x, embed) ; ind = dist.argmax(-1)
// (vector_quantize_pytorch.py:58-62, :741-747, :130-145) without materialising the (N x K) matrix.
//
// Persistent CTAs, one 128-row tile of x at a time, three warpgroups (384 threads):
//   warp 0          TMA producer : x tile (A: 128 rows, stationary in smem for the whole code sweep, refilled k-block by
//                                  k-block as the last code step of the previous tile releases it) and codebook tiles
//                                  (B: 128 codes x 64 dims per ring stage) -> 128-byte-swizzled smem
//   warps 1..3      store warps  : fused gather tail (quantized rows, int64 indices, residuals) of the tile just certified
//   warpgroups 1, 2 consumers    : rows 0..63 / 64..127 of the tile.  Per step of 128 codes a bias MMA sets the
//                                  accumulators to -0.5||c||^2 (the three bf16 terms of bext times [1 1 1 0 ...]: the
//                                  exact value), then wgmma m64n128k16 accumulates the split-precision passes (a0,c_hi)+(a0,c_lo)
//                                  [+(a1,c_hi)] on top (bf16 x bf16 -> fp32), and the certified arg-max scan
//                                  (epilogue.cuh) reads the scores straight from the registers.  The two consumer
//                                  warpgroups share the tensor cores: one scans while the other's MMAs run.
//
// Exactness: the tensor-core score of a (row, code) pair differs from the exact fp32 value by at most
// tau = margin_rel * ||x|| * max||c||, and the epilogue's 4-bit column tag perturbs it by < 16 ulp.  A row is
// certified when its best (tagged) score leads every other score by more than W = 2*tau + 2*(tag slack) + the widths
// over which the reference's own fp32 formula ties distinct codes (its sqrt collapse and, Euclid, its 1e-8 clamp floor);
// otherwise (row, two best candidates, candidate count) goes to `flagged` and vqb_fix_flagged re-scores it with
// the reference's exact formula (count > 3: whole-row rescan).  Conservative: may over-flag, never under-flag.
#include <type_traits>
#include "ptx.cuh"
#include "vqb_common.cuh"
#include "gather_row.cuh"
#include "epilogue.cuh"

// Per-role cycle accounting (vqb_debug_set_profile_buffer): compile with -DVQB_PROFILE.  Off by default.
#ifdef VQB_PROFILE
#define PROF_CLOCK() clock64()
#else
#define PROF_CLOCK() 0ll
#endif

namespace vqb {

constexpr int BM = 128;         // rows of x per tile
constexpr int WM = 64;          // rows per consumer warpgroup (wgmma M)
constexpr int BN_STAGE = 128;   // codes per ring stage; a code step (wgmma N = WN, 128 or 256) spans WN / 128 stages
constexpr int BK = 64;          // bf16 elements per 128-byte swizzle row
constexpr int A_SUB_BYTES = BM * BK * 2;  // 16 KiB: one (plane, k-block) sub-tile of A
constexpr int B_SUB_BYTES = BN_STAGE * BK * 2;  // 16 KiB: one ring stage, 128 codes of one (plane, k-block)
constexpr int MAX_A_SUB = 8;    // n_a * ceil(D/64) <= 8  -> A <= 128 KiB
constexpr int MAX_STAGES = 8;
constexpr int NUM_CONSUMER_WARPS = 8;   // two warpgroups
constexpr int NUM_STORE_WARPS = 3;      // warps 1..3 (warp 0 is the TMA producer)
constexpr int NUM_THREADS = 128 + NUM_CONSUMER_WARPS * 32;
constexpr int SMEM_CTRL_BYTES = 14336;  // barriers + winner hand-off + merge area
constexpr int SMEM_LIMIT = 232448;      // 227 KiB opt-in maximum per CTA
constexpr int SEED_BYTES = BN_STAGE * 32;   // bext of 128 codes ([128][16] bf16); a seed slot holds WN / 128 of them:
                                            // B of the step's bias MMA

struct AssignParams {
  int64_t N;
  int D, K, Kpad;
  int n_a, n_passes;   // pass 0 (a0,c_hi), 1 (a0,c_lo), 2 (a1,c_hi): bf16 operands, fp32 accumulation
  int KB;              // ceil(D / 64)
  int n_stages;        // ring stages of 16 KiB; an item of a 256-code step takes two adjacent ones
  int n_seed;          // seed slots: ceil(ring items / items per code step), so that a slot is refilled only after every
                       // consumer released the first item of the step that last used it
  int stream_a;        // A does not fit in smem next to a useful B ring (fp32 split input with D > 256): its k-blocks travel
                       // through the ring together with the codebook k-blocks (re-read from L2 for every code step)
  const uint16_t* a_global;   // [n_a][N][D] bf16: the A planes in global memory (row norms)
  const uint16_t* bext;       // [Kpad][16] bf16: -0.5||c||^2 as three bf16 terms (code_operands.cuh)
  int num_row_tiles, num_code_steps;
  float margin_rel;
  const float* cmax;   // [CMAX_SLOTS] (code_operands.cuh)
  int32_t* idx;
  int32_t* idx_prov;   // optional: idx with -1 for flagged rows
  int32_t* hist;       // optional [slabs][K]: histogram of the certified winners per slab of (128 << hist_shift) rows — the
  int hist_shift;      // first step of the EMA counting sort (vq_ema.cu), folded into the merge step of the epilogue
  vqb_flag_entry* flagged;
  int32_t* flag_count;
  float* dbg_best;
  const uint8_t* row_mask;   // optional [N]: 0 = padding row (vqp:1116-1119): index -1, no tail, no loss, no statistics, never re-scored
  long long* prof;     // optional [gridDim][16] cycle counters (diagnostics)
  FusedOut fo;         // optional fused gather tail (fo.enabled)
  int copy_mode;       // tail = pure row copy q <- codebook row (+ loss from the scores); no x re-read
  int resid_mode;      // tail = residual only: r <- x - codebook row (+ loss from the scores): a ResidualVQ stage (rvq:524)
  int metric;
  const uint16_t* b_hi;     // bf16 hi plane [Kpad][D]: bf16(c) == the quantized row for bf16 inputs
  const float* cnorm2;      // [K] (cosine loss term)
  uint32_t tagmask, mul1, mulm1;  // 0xFFFFFFF0, 1, -1: constants the compiler must not fold (RowState::insert)
};

struct Ctrl {  // lives at the start of dynamic smem
  uint64_t a_full[MAX_A_SUB], a_empty[MAX_A_SUB];
  uint64_t b_full[MAX_STAGES], b_empty[MAX_STAGES];
  uint64_t g_full[2], g_empty[2];        // winners of a row tile handed to the store warps
  int gidx[2][BM];                       // certified winner per row (-1: flagged / out of range)
  MergeSlot merge[BM][3];                // slices 1..3 of each row, published for the quad's lane 0
  float x2[BM];                          // ||x||^2 of each row of the tile (kept out of the consumers' registers)
};
static_assert(sizeof(Ctrl) <= SMEM_CTRL_BYTES, "control block too large");

// Generic fused tail of one batch of rows (needs x again: running sum / cosine residual).  Kept out of line so that
// its register appetite does not set the allocation of the whole persistent kernel.
template <int GB>
__device__ __forceinline__ float tail_rows(const FusedOut& fo, const int64_t (&rows)[GB], const int (&ks)[GB], int D, int lane) {
  if (fo.dtype == VQB_DTYPE_BF16) return gather_rows<VQB_DTYPE_BF16, GB>(fo, rows, ks, D, lane);
  return gather_rows<VQB_DTYPE_F32, GB>(fo, rows, ks, D, lane);
}

// sum((q - x)^2) over one 16-byte chunk of a row and its code row, rounded like F.mse_loss in the rows' dtype (vqp:1327):
// the square of each fp32 difference, rounded to bf16 for bf16 rows.  The order of the difference does not change its square.
__device__ __forceinline__ float sq_diff16(const uint4& xa, const uint4& ca, bool bf) {
  const uint32_t xw[4] = {xa.x, xa.y, xa.z, xa.w}, cw[4] = {ca.x, ca.y, ca.z, ca.w};
  float s = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (bf) {
      const float d0 = __uint_as_float(xw[e] << 16) - __uint_as_float(cw[e] << 16);
      const float d1 = __uint_as_float(xw[e] & 0xFFFF0000u) - __uint_as_float(cw[e] & 0xFFFF0000u);
      s += bf16_round(d0 * d0);
      s += bf16_round(d1 * d1);
    } else {
      const float d = __uint_as_float(xw[e]) - __uint_as_float(cw[e]);
      s += d * d;
    }
  }
  return s;
}

// What the 256-code step keeps in static shared memory rather than in registers (its 128 accumulators leave 40 for
// everything else; ptxas of CUDA 12.9 needs both moves to stay at 168 registers with no spill):
//  - the per-thread sum of the commitment loss read off the scores (touched once per row);
//  - A of the bias MMA, a 64 x 16 bf16 tile of ones read from shared memory: the register form of that MMA needs four
//    A registers at the point where the accumulators are allocated.  Ones in every column are exact here: the bext
//    columns past the three bias terms are zero.
// The 128-code step keeps both in registers and has no static shared memory (its tightest plan uses all 227 KiB).
template <int WN>
struct StepLocals {
  float loss_ = 0.f;
  __device__ __forceinline__ float& loss() { return loss_; }
};
template <>
struct StepLocals<256> {
  static __device__ __forceinline__ float& loss() {
    __shared__ float s[NUM_CONSUMER_WARPS * 32];
    return s[threadIdx.x - 128];
  }
  static __device__ __forceinline__ uint32_t* bias_ones() {   // [64 rows][16] bf16 1.0, 32-byte swizzle (any layout: all ones)
    __shared__ __align__(256) uint32_t o[WM * 16 / 2];
    return o;
  }
  __device__ __forceinline__ StepLocals() { loss() = 0.f; }
};
constexpr int WIDE_STATIC_SMEM = NUM_CONSUMER_WARPS * 32 * 4 + WM * 16 * 2;   // 1 KiB + 2 KiB

// TAIL selects the work of the store warps at compile time (one instantiation each: the variants do not share a register
// budget): 0 = none / generic (x re-read: running sum, cosine residual), 1 = copy mode, 2 = resid mode.
// WN = codes per code step (wgmma N): 128, or 256 where the launch plan allows it (wide_step below).  A 256-code step pays
// the drain, the quad's shuffles and the restart of the MMA pipe once per 256 codes instead of once per 128, and reads A
// from shared memory half as often.  Its item is two adjacent ring stages (codes 0..127 and 128..255 of one k-block),
// filled by one 256-row TMA box on one barrier pair; its 128 accumulators leave no room for a register-resident live
// group, so its scan keeps live groups in the thread-local queue (ScanState<16>).
template <int TAIL, int WN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
vq_assign_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmS, const AssignParams p) {
  static_assert(WN == 128 || WN == 256, "code step width");
  constexpr int SPAN = WN / BN_STAGE;                  // ring stages per item
  constexpr uint32_t STEP_SEED_BYTES = SPAN * SEED_BYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  Ctrl* ctrl = reinterpret_cast<Ctrl*>(smem);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t a_base = (smem_base + SMEM_CTRL_BYTES + 1023u) & ~1023u;    // swizzled tiles need 1024 B alignment
  const bool stream_a = WN == 128 && p.stream_a;                              // the wide step keeps A resident
  const int n_sub = stream_a ? 0 : p.n_a * p.KB;                              // stationary A sub-tiles
  const uint32_t b_base = a_base + n_sub * A_SUB_BYTES;
  // ring item = [A k-block (stream_a only) | codebook k-block of the code step: SPAN stages of 128 codes, back to back]
  const uint32_t a_stage_bytes = stream_a ? A_SUB_BYTES : 0;
  const uint32_t stage_stride = a_stage_bytes + SPAN * B_SUB_BYTES;
  const int n_ring = p.n_stages / SPAN;                                       // ring items (the plan's stage count is even for WN = 256)
  const uint32_t seed_base = b_base + n_ring * stage_stride;                 // [n_seed][WN codes][16] bf16

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ------------------------------------------------------------------ one-time setup
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmS);
    for (int s = 0; s < n_sub; ++s) {
      mbar_init(smem_u32(&ctrl->a_full[s]), 1);
      mbar_init(smem_u32(&ctrl->a_empty[s]), NUM_CONSUMER_WARPS);
    }
    for (int s = 0; s < n_ring; ++s) {
      mbar_init(smem_u32(&ctrl->b_full[s]), 1);
      mbar_init(smem_u32(&ctrl->b_empty[s]), NUM_CONSUMER_WARPS);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(&ctrl->g_full[s]), NUM_CONSUMER_WARPS);
      mbar_init(smem_u32(&ctrl->g_empty[s]), NUM_STORE_WARPS);
    }
    fence_barrier_init();
  }
  if constexpr (WN == 256) {
    for (int i = threadIdx.x; i < WM * 16 / 2; i += NUM_THREADS) StepLocals<256>::bias_ones()[i] = 0x3F803F80u;
    fence_proxy_async_shared();   // generic-proxy stores, read by wgmma
  }
  __syncthreads();

  if (warp == 0) {
    // ================================================================ TMA producer
    if (lane == 0) {
      long long w_empty = 0, w_aempty = 0;
      const long long pstart = PROF_CLOCK();
      int stage = 0, gstep = 0;
      uint32_t ph = 0;
      for (int t = 0, tile = static_cast<int>(blockIdx.x); tile < p.num_row_tiles; ++t, tile += static_cast<int>(gridDim.x)) {
        const int row0 = tile * BM;
        if (!stream_a && tile + static_cast<int>(gridDim.x) < p.num_row_tiles) {   // the next tile's x into L2: its refill below then does not wait on HBM
          for (int ap = 0; ap < p.n_a; ++ap)
            for (int kb = 0; kb < p.KB; ++kb) tma_prefetch_l2_3d(&tmA, kb * BK, row0 + static_cast<int>(gridDim.x) * BM, ap);
        }
        for (int ct = 0; ct < p.num_code_steps; ++ct, ++gstep) {
          // k-block-major: all passes of a k-block back to back, so that in the LAST code step of a row tile an A sub-tile
          // is released (and refilled for the next row tile) as early as possible
          for (int kb = 0; kb < p.KB; ++kb) {
            for (int ps = 0; ps < p.n_passes; ++ps) {
              const int bplane = (ps == 1) ? 1 : 0;
              const int aplane = (ps == 2) ? 1 : 0;
              if (!stream_a && ct == 0 && (ps == 0 || ps == 2)) {  // refill this A sub-tile once the previous row tile released it
                const int sub = aplane * p.KB + kb;
                { const long long c0 = PROF_CLOCK(); mbar_wait(smem_u32(&ctrl->a_empty[sub]), (t & 1) ^ 1); w_aempty += PROF_CLOCK() - c0; }
                mbar_arrive_expect_tx(smem_u32(&ctrl->a_full[sub]), A_SUB_BYTES);
                tma_load_3d(a_base + sub * A_SUB_BYTES, &tmA, smem_u32(&ctrl->a_full[sub]), kb * BK, row0, aplane);
              }
              { const long long c0 = PROF_CLOCK(); mbar_wait(smem_u32(&ctrl->b_empty[stage]), ph ^ 1); w_empty += PROF_CLOCK() - c0; }
              // the step's seeds ride on the barrier of its first item (a whole box: rows past Kpad are zero-filled).
              // Seed-slot reuse: slot gstep % n_seed was last read by the bias MMA of step gstep - n_seed, committed with
              // that step's first item, n_seed * n_items ring items before this one.  The b_empty wait above proves that
              // every consumer warp released the item n_ring items back, and releases run in item order, so with
              // n_seed * n_items >= n_ring (n_seed = ceil(n_ring / n_items)) that first item — and the bias MMA — has
              // completed.  The rule counts ring items, not stages: a 256-code item is one item on one barrier pair.
              const bool seeds = kb == 0 && ps == 0;
              mbar_arrive_expect_tx(smem_u32(&ctrl->b_full[stage]), stage_stride + (seeds ? STEP_SEED_BYTES : 0));
              if (seeds)
                tma_load_3d(seed_base + (gstep % p.n_seed) * STEP_SEED_BYTES, &tmS, smem_u32(&ctrl->b_full[stage]), 0, ct * WN, 0);
              if (stream_a)
                tma_load_3d(b_base + stage * stage_stride, &tmA, smem_u32(&ctrl->b_full[stage]), kb * BK, row0, aplane);
              // one box of WN codes (the tensor map's box is WN rows): for WN = 256 it fills two adjacent 16 KiB stages
              tma_load_3d(b_base + stage * stage_stride + a_stage_bytes, &tmB, smem_u32(&ctrl->b_full[stage]), kb * BK,
                          ct * WN, bplane);
              if (++stage == n_ring) { stage = 0; ph ^= 1; }
            }
          }
        }
      }
      if (p.prof) {
        p.prof[blockIdx.x * 16 + 0] = w_empty;
        p.prof[blockIdx.x * 16 + 1] = PROF_CLOCK() - pstart;
        p.prof[blockIdx.x * 16 + 6] = w_aempty;
      }
    }
  } else if (warp <= NUM_STORE_WARPS) {
    // ================================================================ store warps: fused gather tail
    const int sw = warp - 1;
    float lsum = 0.f;
    for (int t = 0, tile = static_cast<int>(blockIdx.x); p.fo.enabled && tile < p.num_row_tiles; ++t, tile += static_cast<int>(gridDim.x)) {
      mbar_wait(smem_u32(&ctrl->g_full[t & 1]), (t >> 1) & 1);
      const int* gi = ctrl->gidx[t & 1];
      if (TAIL >= 1) {
        // copy mode: q[row] <- codebook row: bf16 inputs copy the bf16 hi plane (== embed.type(bf16)), fp32 inputs the fp32 row.
        // resid mode (a ResidualVQ stage): residual[row] <- x[row] - that same row, rounded once (rvq:524, vqp:1178); the x
        // rows were just read by the TMA (L2).
        constexpr int CB = 4;  // rows per batch: independent 16-byte loads in flight per lane
        const bool bf = p.fo.dtype == VQB_DTYPE_BF16;
        const int row_bytes = p.D * (bf ? 2 : 4);
        const uint8_t* src = bf ? reinterpret_cast<const uint8_t*>(p.b_hi) : reinterpret_cast<const uint8_t*>(p.fo.embed);
        const uint8_t* xin = static_cast<const uint8_t*>(p.fo.x_eff);
        uint8_t* dst = static_cast<uint8_t*>(TAIL == 2 ? p.fo.resid_out : p.fo.q_out);
        for (int r0 = sw * CB; r0 < BM; r0 += NUM_STORE_WARPS * CB) {
          int ks[CB];
          bool ex[CB];   // the row's loss is evaluated here, from x and the code row
#pragma unroll
          for (int b = 0; b < CB; ++b) {
            const int g = gi[r0 + b];
            ex[b] = g < -1;
            ks[b] = ex[b] ? -2 - g : g;
          }
          const int64_t row_base = static_cast<int64_t>(tile) * BM + r0;
          if (p.fo.idx64_out && lane < CB && ks[lane & (CB - 1)] >= 0) {
            int kk = 0;
#pragma unroll
            for (int b = 0; b < CB; ++b) kk = (lane == b) ? ks[b] : kk;
            p.fo.idx64_out[(row_base + lane) * p.fo.idx_stride] = kk;
          }
          if (dst || (ex[0] | ex[1] | ex[2] | ex[3])) {
            for (int off = lane * 16; off < row_bytes; off += 512) {
              uint4 v[CB];
#pragma unroll
              for (int b = 0; b < CB; ++b)
                if (ks[b] >= 0) v[b] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<int64_t>(ks[b]) * row_bytes + off));
              if (TAIL == 1) {
#pragma unroll
                for (int b = 0; b < CB; ++b)
                  if (ex[b]) lsum += sq_diff16(*reinterpret_cast<const uint4*>(xin + (row_base + b) * row_bytes + off), v[b], bf);
              }
              if (TAIL == 2) {
                uint4 x[CB];
#pragma unroll
                for (int b = 0; b < CB; ++b)
                  if (ks[b] >= 0) x[b] = *reinterpret_cast<const uint4*>(xin + (row_base + b) * row_bytes + off);
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                  if (ks[b] < 0) continue;
                  if (ex[b]) lsum += sq_diff16(x[b], v[b], bf);
                  const uint32_t xw[4] = {x[b].x, x[b].y, x[b].z, x[b].w}, cw[4] = {v[b].x, v[b].y, v[b].z, v[b].w};
                  uint32_t rw[4];
                  if (bf) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                      const float d0 = __uint_as_float(xw[e] << 16) - __uint_as_float(cw[e] << 16);
                      const float d1 = __uint_as_float(xw[e] & 0xFFFF0000u) - __uint_as_float(cw[e] & 0xFFFF0000u);
                      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(rw[e]) : "f"(d1), "f"(d0));
                    }
                  } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) rw[e] = __float_as_uint(__uint_as_float(xw[e]) - __uint_as_float(cw[e]));
                    if (p.fo.planes_out) {  // the next stage's MMA operand: bf16 hi / lo split of the residual
                      const float rf[4] = {__uint_as_float(rw[0]), __uint_as_float(rw[1]), __uint_as_float(rw[2]), __uint_as_float(rw[3])};
                      store_planes4(p.fo.planes_out, p.fo.planes_stride, ((row_base + b) * row_bytes + off) >> 2, rf);
                    }
                  }
                  v[b] = make_uint4(rw[0], rw[1], rw[2], rw[3]);
                }
              }
#pragma unroll
              for (int b = 0; b < CB; ++b)
                if (dst && ks[b] >= 0) *reinterpret_cast<uint4*>(dst + (row_base + b) * row_bytes + off) = v[b];
            }
          }
        }
      } else {
        constexpr int GB = 2;
        for (int r0 = sw * GB; r0 < BM; r0 += NUM_STORE_WARPS * GB) {
          int64_t rows[GB];
          int ks[GB];
          bool any = false;
#pragma unroll
          for (int b = 0; b < GB; ++b) {
            ks[b] = gi[r0 + b];
            rows[b] = ks[b] >= 0 ? static_cast<int64_t>(tile) * BM + r0 + b : -1;
            any |= ks[b] >= 0;
          }
          if (!any) continue;
          lsum += tail_rows<GB>(p.fo, rows, ks, p.D, lane);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&ctrl->g_empty[t & 1]));
    }
    if (p.fo.enabled && p.fo.loss_sum) {   // generic tail: every row; copy / resid: the rows left to the store warps
      const double w = warp_sum(static_cast<double>(lsum));
      if (lane == 0) atomicAdd(p.fo.loss_sum, w);
    }
  } else {
    // ================================================================ consumers (warpgroups 1 and 2)
    const int wg = (warp >> 2) - 1;                              // 0: rows 0..63, 1: rows 64..127
    const int q = lane & 3;                                      // column slice of the thread's rows
    const int rit0 = wg * WM + (warp & 3) * 16 + (lane >> 2);    // the thread's rows: rit0 and rit0 + 8
    const int n_items = p.KB * p.n_passes;
    const uint32_t a_row_off = wg * WM * 128;          // this warpgroup's 64 rows inside an A sub-tile (1024 B aligned)
    // A of the bias MMA: 1 at k = 0, 1, 2 of every row, 0 elsewhere (the thread's fragment holds columns 2q, 2q + 1)
    const uint32_t bias_a = q == 0 ? 0x3F803F80u : (q == 1 ? 0x00003F80u : 0u);
    long long w_full = 0, w_afull = 0, w_gap = 0, gap0 = -1;   // gap: last commit of a step -> first wait of the next
    const long long cstart = PROF_CLOCK();
    float acc[WN / 2];
    int stage = 0, gstep = 0;
    uint32_t ph = 0;
    StepLocals<WN> locals;
    auto release = [&](int st, int sub) {   // this warp's MMAs of a ring stage (and A sub-tile) have completed
      if (lane == 0) {
        mbar_arrive(smem_u32(&ctrl->b_empty[st]));
        if (sub >= 0) mbar_arrive(smem_u32(&ctrl->a_empty[sub]));
      }
    };
    // ||x||^2 of the thread's two rows (the quad splits each row), from the bf16 planes in global memory (L2: the TMA
    // just read them, or the producer prefetched them).  fp32 accumulation: the norm scales the certification band AND
    // carries the commitment loss (sum ||q - x||^2 = sum ||x||^2 - 2 score), so it must be as exact as the scores.
    // ||x||^2 goes to shared memory for the merge, ||x_lo||^2 to xlo.  WN = 128 runs this under the first code step's
    // last MMAs; the 256-code step's accumulators leave no registers for it there, so WN = 256 runs it before the
    // tile's first MMA (the rows are in L2: prefetched one tile ahead).
    auto row_norms = [&](int tile, float (&xlo)[2]) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = static_cast<int64_t>(tile) * BM + rit0 + 8 * h;
        float a = 0.f, alo = 0.f;
        if (row < p.N) {
          const uint16_t* hp = p.a_global + row * p.D;
          for (int c = q * 8; c < p.D; c += 32) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(hp + c));
            uint4 l = make_uint4(0u, 0u, 0u, 0u);
            if (p.n_a == 2) l = __ldg(reinterpret_cast<const uint4*>(hp + p.N * p.D + c));
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
            const uint32_t wl[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float h0 = __uint_as_float(w[e] << 16), h1 = __uint_as_float(w[e] & 0xFFFF0000u);
              const float l0 = __uint_as_float(wl[e] << 16), l1 = __uint_as_float(wl[e] & 0xFFFF0000u);
              a = fmaf(h0 + l0, h0 + l0, a);
              a = fmaf(h1 + l1, h1 + l1, a);
              alo = fmaf(l0, l0, alo);
              alo = fmaf(l1, l1, alo);
            }
          }
        }
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        alo += __shfl_xor_sync(0xffffffffu, alo, 1);
        alo += __shfl_xor_sync(0xffffffffu, alo, 2);
        if (q == 0) ctrl->x2[rit0 + 8 * h] = a;
        xlo[h] = alo;   // squared: the sqrt (a subroutine call) waits until no wgmma is in flight
      }
    };
    // The certification band W of the thread's two rows (after row_norms; the sqrt is a subroutine call, which must not
    // sit where a wgmma is in flight), and a fresh scan state.
    auto init_band = [&](auto (&sc)[2], float (&xlo)[2]) {
      const bool euclid = p.metric != VQB_METRIC_COSINE;
      const float cmax = __ldg(p.cmax + CMAX_NORM);
      // Exact norms of what the passes leave out of the codebook operand (code_operands.cuh): ||c - hi - lo||.  fp32 inputs
      // (x = hi + lo + res, |res| <= 2^-8 |lo| per element) add x_res . c and the omitted x_lo . c_lo:  ||x_lo|| * caux.
      const float cres = __ldg(p.cmax + CMAX_RES);
      const float caux = p.n_a == 2 ? 0x1.02p-8f * cmax + __ldg(p.cmax + CMAX_LO) : 0.f;
      __syncwarp();   // the quad's lane 0 wrote the norms
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x2 = ctrl->x2[rit0 + 8 * h];
        // band = 2 * (MMA error bound) + 2 * (tag perturbation: 16 ulp <= 2^-19 |score|, |score| <= |x||c| + |c|^2/2)
        // + (Euclid) the width over which the reference's own evaluation collapses distinct d^2 into one distance:
        // d = sqrt(fl(fl(x2 + y2) - 2xy)) has ~d^2 * 2^-23 of resolution in d^2 (vqp:58-62); with a small-norm codebook
        // (the default init) that exceeds the MMA band.  Rows inside it go to the exact re-score, which evaluates the
        // reference formula including the sqrt.  In score units (d^2 / 2), with a 2x safety factor.
        // 2 * |score error|: what the passes leave out of the codebook (||x|| * cres) and of the row (xaux * caux), both by
        // Cauchy-Schwarz on exact norms; the fp32 accumulation in the tensor core (margin_rel relative to ||x|| max||c||,
        // 2^-20 relative to the bias the bias MMA sums); then the tag slack and the sqrt-collapse width.
        // Last (Euclid), the clamp floor: the reference clamps d^2 at 1e-8 before the sqrt (vqp:58-62), so every code with
        // fp32 d^2 <= 1e-8 scores -1e-4 and the lowest such index wins, although their exact scores differ by up to
        // (1e-8 + the d^2 rounding) / 2.  The norm-scaled terms above are narrower than that once ||x|| and max||c|| fall
        // to ~1e-2 (late ResidualVQ stages, zero residuals); 1e-8 keeps those codes inside the band, and the band of a
        // normal-norm codebook (~1e-5 and up) does not notice it.
        const float xn = sqrtf(x2);
        const float xc = xn * cmax;
        xlo[h] = p.n_a == 2 ? sqrtf(xlo[h]) * 1.0001f : 0.f;
        sc[h].init(2.f * (xn * cres + xlo[h] * caux + p.margin_rel * xc + (euclid ? 0x1p-21f * cmax * cmax : 0.f)) +
                   0x1p-18f * (xc + (euclid ? 0.5f * cmax * cmax : 0.f)) +
                   (euclid ? 0x1p-22f * (x2 + cmax * cmax) + 1e-8f : 1e-30f));
      }
    };
    for (int t = 0, tile = static_cast<int>(blockIdx.x); tile < p.num_row_tiles; ++t, tile += static_cast<int>(gridDim.x)) {
      // hot-loop state of the two rows: running maximum (+ for WN = 128 the live group, in registers)
      typename std::conditional<WN == 128, ScanReg, ScanState<16>>::type sc[2];
      ScanQueue<16> sq[2];         // (further) live groups (thread-local memory, rarely touched)

      float xlo[2] = {0.f, 0.f};
      for (int ct = 0; ct < p.num_code_steps; ++ct) {
        const bool last_ct = ct == p.num_code_steps - 1;
        // The bias MMA (scale-d = 0) sets the accumulators to -0.5||c||^2 (Euclid; 0 for cosine, -3e38 for padding codes):
        // A = [1 1 1 0 ...] times the step's bext rows, which the producer loaded into a seed slot on the barrier of the
        // step's first item; b1 + b2 + b3 is exact in fp32.  It is committed with item 0, so the release of item 0's
        // stage also proves that the slot has been read.
        if (WN == 256 && ct == 0) {   // no accumulator is live and no wgmma in flight
          row_norms(tile, xlo);
          init_band(sc, xlo);
        }
        if (gap0 >= 0) w_gap += PROF_CLOCK() - gap0;
        { const long long c0 = PROF_CLOCK(); mbar_wait(smem_u32(&ctrl->b_full[stage]), ph); w_full += PROF_CLOCK() - c0; }
        wgmma_fence();
        const uint64_t sd = wgmma_desc_sw32(seed_base + (gstep % p.n_seed) * STEP_SEED_BYTES);
        if constexpr (WN == 128) wgmma_m64n128k16_bf16_rs_set(acc, bias_a, sd);
        else wgmma_m64n256k16_bf16_ss_set(acc, wgmma_desc_sw32(smem_u32(StepLocals<256>::bias_ones())), sd);
        // Items of a code step in k-block-major order (kb, ps) — the order the producer stages them in.  One wgmma group
        // stays in flight: the stage of item i - 1 is released once item i has been issued.
        int kb = 0, ps = 0;
        int pend_stage = -1, pend_sub = -1;
        for (int i = 0; i < n_items; ++i) {
          const int aplane = (ps == 2) ? 1 : 0;
          const int sub = aplane * p.KB + kb;
          if (ct == 0 && !stream_a) { const long long c0 = PROF_CLOCK(); mbar_wait(smem_u32(&ctrl->a_full[sub]), t & 1); w_afull += PROF_CLOCK() - c0; }
          if (i > 0) { const long long c0 = PROF_CLOCK(); mbar_wait(smem_u32(&ctrl->b_full[stage]), ph); w_full += PROF_CLOCK() - c0; }
          const uint32_t st_addr = b_base + stage * stage_stride;
          const uint32_t a_addr = (stream_a ? st_addr : a_base + sub * A_SUB_BYTES) + a_row_off;
          const uint64_t ad = wgmma_desc_sw128(a_addr);
          const uint64_t bd = wgmma_desc_sw128(st_addr + a_stage_bytes);   // WN rows of 128 B, 8-row groups 1024 B apart
          fence_regs(acc);
          wgmma_fence();
          // four K=16 steps, descriptors advance by 32 B.  A ragged last k-block (D % 64 != 0) runs them all too: the TMA
          // zero-fills both operands past D, so the extra steps add exact zeros (a data-dependent step count would make
          // ptxas serialise the wgmmas)
#pragma unroll
          for (int k = 0; k < 8; k += 2) {
            if constexpr (WN == 128) wgmma_m64n128k16_bf16(acc, ad + k, bd + k);
            else wgmma_m64n256k16_bf16(acc, ad + k, bd + k);
          }
          wgmma_commit();
          if (i == n_items - 1) gap0 = PROF_CLOCK();
          wgmma_wait<1>();
          fence_regs(acc);
          if (pend_stage >= 0) release(pend_stage, pend_sub);
          const bool last_use = last_ct && !stream_a && (aplane == 1 ? ps == 2 : ps == 1);  // pass 1: the last one of a k-block on A plane 0
          pend_stage = stage;
          pend_sub = last_use ? sub : -1;
          if (++stage == n_ring) { stage = 0; ph ^= 1; }
          if (++ps == p.n_passes) { ps = 0; ++kb; }
        }
        if (WN == 128 && ct == 0) row_norms(tile, xlo);   // while the last MMAs of the step run
        wgmma_wait<0>();
        fence_regs(acc);
        release(pend_stage, pend_sub);
        ++gstep;
        if ((ct + 1) * WN > p.Kpad) {   // tiny codebooks: codes past Kpad (zero-filled seeds and operands) score -3e38
#pragma unroll
          for (int j = 0; j < WN / 8; ++j)
#pragma unroll
            for (int b = 0; b < 2; ++b)
              if (ct * WN + 8 * j + 2 * q + b >= p.Kpad) { acc[4 * j + b] = -3.0e38f; acc[4 * j + 2 + b] = -3.0e38f; }
        }

        if (WN == 128 && ct == 0) {
          init_band(sc, xlo);
        } else if (ct > 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {  // the row's running maximum over the quad raises every slice's skip threshold
            float m = sc[h].t1;
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            sc[h].raise(m);
          }
        }
        // Per row, the thread holds WN / 64 groups of 16 scores: group g = 8-column blocks 8g..8g+7, columns 2q, 2q + 1 of each.
        // Group-major: the two rows' groups of a column block are scanned together and their accumulators die together.
#pragma unroll
        for (int g = 0; g < WN / 64; ++g) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t r[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) r[e] = __float_as_uint(acc[4 * (8 * g + (e >> 1)) + 2 * h + (e & 1)]);
            if constexpr (WN == 128) sc[h].template scan16<true, false>(sq[h], r, ct * WN + 64 * g + 2 * q, p.mul1);
            else sc[h].template scan16<true>(sq[h], r, ct * WN + 64 * g + 2 * q);
          }
        }
      }

      // ---- merge the four column slices of each row (lanes 1..3 of the quad publish, lane 0 finishes the row)
      if (p.fo.enabled) mbar_wait(smem_u32(&ctrl->g_empty[t & 1]), ((t >> 1) & 1) ^ 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rit = rit0 + 8 * h;
        RowState st;
        sc[h].finish(sq[h], st, p.tagmask, p.mul1, p.mulm1);
        MergeSlot* slots = ctrl->merge[rit];
        if (q != 0) publish(&slots[q - 1], st);
        __syncwarp();
        if (q == 0) {
          const RowResult rr = merge_slices(st, slots, 3, 1);
          const int n = rr.n, i0 = rr.i0, i1 = rr.i1;
          const float best = rr.best;
          const int64_t row = static_cast<int64_t>(tile) * BM + rit;
          // padding rows of a masked batch (vqp:1116-1119) are searched like any other row — the tile is dense — but take no
          // part in anything afterwards: index -1, no tail (the caller pre-filled their outputs), no loss (vqp:1317-1325), no
          // statistics (vqp:599-600: no histogram count, -1 in the provisional indices), never flagged
          const bool live = row < p.N && (p.row_mask == nullptr || __ldg(p.row_mask + row) != 0);
          bool exact_loss = false;
          if (TAIL >= 1 && p.fo.loss_sum && live && n < 2) {
            // ||q - x||^2 = ||x||^2 - 2(x.c - 0.5||c||^2)  — the score already holds it (cosine: bias is 0, add ||c||^2).
            // Its error is about the band W (the score's error bound, twice).  A row close to its code (a trained
            // codebook) cancels in this difference, so unless d2 leads W by 2^14 the store warps evaluate sum((q - x)^2)
            // from the rows themselves; randn-like rows (d2 ~ 6e4 W at config 2) never take that path.  Flagged rows get the exact
            // evaluation in vqb_fix_flagged.
            float d2 = ctrl->x2[rit] - 2.f * best;
            if (p.metric == VQB_METRIC_COSINE) d2 += __ldg(p.cnorm2 + i0);
            exact_loss = !(d2 >= 0x1p14f * st.W);
            if (!exact_loss) locals.loss() += d2;
          }
          // hand the certified winners to the store warps: k, or -2 - k when the row's loss is left to them
          if (p.fo.enabled) ctrl->gidx[t & 1][rit] = (live && n < 2) ? (exact_loss ? -2 - i0 : i0) : -1;
          if (row < p.N && !live) {
            p.idx[row] = -1;
            if (p.idx_prov) p.idx_prov[row] = -1;
          } else if (row < p.N) {
            p.idx[row] = i0;
            if (p.idx_prov) p.idx_prov[row] = (n < 2) ? i0 : -1;
            if (p.hist && n < 2) atomicAdd(p.hist + static_cast<size_t>(tile >> p.hist_shift) * p.K + i0, 1);   // RED, fire and forget
            if (p.dbg_best) p.dbg_best[row] = best;
            if (n >= 2) {
              // 2 or 3 candidates: front of the list (exact re-score of those codes); more: BACK of the list, growing
              // downwards (whole-row exact re-scan) — the two kinds never share a slot (at most N entries in total)
              const bool many = n > 3;
              const int s = many ? static_cast<int>(p.N) - 1 - atomicAdd(p.flag_count + 1, 1) : atomicAdd(p.flag_count, 1);
              vqb_flag_entry e;
              e.row = static_cast<int32_t>(row);
              e.cand0 = many ? 0 : i0;     // (cand0, cand1) of a re-scanned row is its 64-bit arg-max key: starts at 0
              e.cand1 = many ? 0 : i1;
              e.cand2 = rr.i2;
              e.count = n;
              e.pad[0] = e.pad[1] = e.pad[2] = 0;
              p.flagged[s] = e;
            }
          }
        }
        __syncwarp();   // the slots are reused by the next row / tile
      }
      if (p.fo.enabled && lane == 0) mbar_arrive(smem_u32(&ctrl->g_full[t & 1]));
    }
    if (TAIL >= 1 && p.fo.loss_sum) {
      const double w = warp_sum(static_cast<double>(locals.loss()));
      if (lane == 0) atomicAdd(p.fo.loss_sum, w);
    }
    if (p.prof && threadIdx.x == 128) {
      p.prof[blockIdx.x * 16 + 2] = w_full;
      p.prof[blockIdx.x * 16 + 3] = PROF_CLOCK() - cstart;
      p.prof[blockIdx.x * 16 + 4] = w_gap;
      p.prof[blockIdx.x * 16 + 5] = w_afull;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(f);
  }
  return fn;
}

// bf16 tensor [planes][rows][cols] (row-major) -> boxes of {box_cols, box_rows, 1}, swizzle span == box row bytes,
// out-of-bounds elements read as zero (ragged N / K / D are handled by the zero fill).
static int make_map(CUtensorMap* m, const void* base, int cols, int64_t rows, int planes, int box_cols, int box_rows,
                    CUtensorMapSwizzle swz) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return VQB_E_DRIVER;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(planes)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(cols) * 2, static_cast<cuuint64_t>(cols) * 2 * static_cast<cuuint64_t>(rows)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? VQB_OK : VQB_E_DRIVER;
}

// Shared-memory layout of one launch: whether A stays resident, ring stages, seed slots.  Host only, no device needed.
struct AssignPlan {
  int stream_a, n_stages, n_seed, n_items, KB, smem_bytes;
};

static int assign_plan(int n_a, int D, int n_passes, AssignPlan* pl) {
  if (D <= 0 || (n_a != 1 && n_a != 2)) return VQB_E_INVALID;
  // Passes (bf16 operands, fp32 accumulation): A = the input rows (n_a = 1) or the bf16 hi / lo planes of an fp32 input
  // (n_a = 2), B = the bf16 hi / lo codebook planes — (x,c_hi)+(x,c_lo) [+ (x_lo,c_hi)]: residual ~2^-17 ||x|| ||c||, carried
  // exactly by the band.  DESIGN.md section 8.
  if (n_passes == 0) n_passes = n_a + 1;
  if (n_passes != n_a + 1) return VQB_E_UNSUPPORTED;
  if (D % 8 != 0) return VQB_E_UNSUPPORTED;
  const int KB = (D + BK - 1) / BK;
  // A stationary in smem when it leaves room for a useful ring; else (fp32 split input with D > 256) its k-blocks are
  // streamed through the ring next to the codebook's (re-read from L2 for every code step)
  const int stream_a = n_a * KB > MAX_A_SUB ? 1 : 0;
  const int a_bytes = stream_a ? 0 : n_a * KB * A_SUB_BYTES;
  const int stage_bytes = B_SUB_BYTES + (stream_a ? A_SUB_BYTES : 0);
  const int fixed = SMEM_CTRL_BYTES + 1024 /*align*/ + a_bytes;
  // ring stages + seed slots (one slot per code step the ring can run ahead).  The tightest case, fp32 at D = 256, keeps
  // its 5 stages: 15 KiB + 128 KiB of A + 5 * 16 KiB + 4 KiB of seeds = exactly 227 KiB.
  const int n_items = KB * n_passes;
  int stages = MAX_STAGES;
  auto seed_slots = [&](int st) { return (st + n_items - 1) / n_items; };
  while (stages >= 2 && fixed + stages * stage_bytes + seed_slots(stages) * SEED_BYTES > SMEM_LIMIT) --stages;
  if (stages < 2) return VQB_E_UNSUPPORTED;
  pl->stream_a = stream_a;
  pl->n_stages = stages;
  pl->n_seed = seed_slots(stages);
  pl->n_items = n_items;
  pl->KB = KB;
  pl->smem_bytes = fixed + stages * stage_bytes + pl->n_seed * SEED_BYTES;
  return VQB_OK;
}

// The 256-code step on the same ring: an item takes two adjacent stages, so the stage count must be even, and the ring
// has n_stages / 2 items, each step's seeds take 8 KiB, and a slot is reused after ceil(ring items / items per step)
// steps.  It needs A resident (a streamed A k-block would sit between the two halves of B) and the larger seed slots
// and its 3 KiB of static shared memory (StepLocals) inside 227 KiB; and a codebook of more than 128 padded codes (Kpad <= 128 is one 128-code step, which the wide step
// could only double).  Config 2 (bf16, D = 256) and fp32 at D = 128 qualify: 8 stages, one 8 KiB seed slot.
// Fills the seed slots and dynamic shared memory of the wide step; the launch plan and its stage count are unchanged.
static bool wide_step(const AssignPlan& pl, int Kpad, int* n_seed, int* smem_bytes) {
  if (pl.stream_a || pl.n_stages % 2 != 0 || Kpad <= BN_STAGE) return false;
  const int ring = pl.n_stages / 2;
  const int seeds = (ring + pl.n_items - 1) / pl.n_items;
  const int bytes = pl.smem_bytes - pl.n_seed * SEED_BYTES + seeds * 2 * SEED_BYTES;
  if (bytes + WIDE_STATIC_SMEM > SMEM_LIMIT) return false;
  *n_seed = seeds;
  *smem_bytes = bytes;
  return true;
}

}  // namespace vqb

using namespace vqb;

// The launch plan vqb_assign would use for (n_a, D, n_passes): out6 = {stream_a, n_stages, n_seed, n_items, KB, smem_bytes}.
extern "C" int vqb_debug_assign_plan(int n_a, int D, int n_passes, int* out6) {
  if (!out6) return VQB_E_INVALID;
  AssignPlan pl;
  const int rc = assign_plan(n_a, D, n_passes, &pl);
  if (rc) return rc;
  out6[0] = pl.stream_a; out6[1] = pl.n_stages; out6[2] = pl.n_seed;
  out6[3] = pl.n_items; out6[4] = pl.KB; out6[5] = pl.smem_bytes;
  return VQB_OK;
}

extern "C" int vqb_padded_codes(int K) {
  if (K <= 0) return 0;
  const int BN = code_tile(K);
  return (K + BN - 1) / BN * BN;
}

// validate + copy the optional fused-tail description (shared with vq_aux.cu through vqb_common.cuh)
static long long* g_prof = nullptr;
static int g_dbg_mode = 0;
extern "C" int vqb_debug_set_mode(int mode) { g_dbg_mode = mode; return VQB_OK; }
extern "C" int vqb_debug_active(void) { return (g_prof != nullptr) || (g_dbg_mode != 0); }
// diagnostics: device buffer of [grid][16] int64 cycle counters filled by the next vqb_assign calls (NULL = off)
extern "C" int vqb_debug_set_profile_buffer(void* buf) { g_prof = static_cast<long long*>(buf); return VQB_OK; }

extern "C" int vqb_assign(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
                          const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx,
                          vqb_flag_entry* flagged, int32_t* flag_count, float* dbg_best,
                          const vqb_fused_outputs* fused, void* stream) {
  return vqb_assign_ex(a_planes, n_a, N, D, b_planes, bext, cmax, K, margin_rel, n_passes, idx, flagged, flag_count,
                       dbg_best, fused, VQB_METRIC_EUCLID, nullptr, stream);
}

// Same, with the metric and ||c||^2 needed for the in-kernel commitment loss of the cosine metric.
extern "C" int vqb_assign_ex(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
                             const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx,
                             vqb_flag_entry* flagged, int32_t* flag_count, float* dbg_best,
                             const vqb_fused_outputs* fused, int metric, const float* cnorm2, void* stream) {
  return vqb::assign_launch(a_planes, n_a, N, D, b_planes, bext, cmax, K, margin_rel, n_passes, idx, nullptr, nullptr, 0,
                            flagged, flag_count, dbg_best, fused, metric, cnorm2, stream);
}

// idx_prov (optional): like idx, but -1 for the rows handed to the exact re-score — lets the EMA sort start on the
// certified rows while vqb_fix_flagged is still running (vq_forward.cu).
int vqb::assign_launch(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
                       const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx, int32_t* idx_prov,
                       int32_t* hist, int hist_shift, vqb_flag_entry* flagged, int32_t* flag_count, float* dbg_best,
                       const vqb_fused_outputs* fused, int metric, const float* cnorm2, void* stream, const uint8_t* row_mask) {
  if (!a_planes || !b_planes || !bext || !cmax || !idx || !flagged || !flag_count) return VQB_E_INVALID;
  if (N <= 0 || K <= 0) return VQB_E_INVALID;
  AssignPlan plan;
  int rc = assign_plan(n_a, D, n_passes, &plan);
  if (rc) return rc;
  if (n_passes == 0) n_passes = n_a + 1;
  if (N > (static_cast<int64_t>(1) << 31) - BM) return VQB_E_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(a_planes) | reinterpret_cast<uintptr_t>(b_planes) | reinterpret_cast<uintptr_t>(bext)) & 15)
    return VQB_E_ALIGN;
  AssignParams p;
  rc = make_fused(&p.fo, fused, D, N);
  if (rc) return rc;
  rc = check_device();
  if (rc) return rc;

  p.N = N; p.D = D; p.K = K;
  p.Kpad = vqb_padded_codes(K);
  p.n_a = n_a; p.n_passes = n_passes; p.KB = plan.KB;
  p.num_row_tiles = static_cast<int>((N + BM - 1) / BM);
  int smem_bytes = plan.smem_bytes;
  p.n_seed = plan.n_seed;
  const bool wide = wide_step(plan, p.Kpad, &p.n_seed, &smem_bytes);
  const int WN = wide ? 256 : 128;   // codes per code step
  p.num_code_steps = (p.Kpad + WN - 1) / WN;
  p.margin_rel = margin_rel;
  p.cmax = cmax; p.idx = idx; p.idx_prov = idx_prov; p.hist = hist; p.hist_shift = hist_shift; p.flagged = flagged; p.flag_count = flag_count; p.dbg_best = dbg_best;
  p.row_mask = row_mask;
  p.prof = g_prof;
  p.tagmask = 0xFFFFFFF0u; p.mul1 = 1u; p.mulm1 = 0xFFFFFFFFu;
  p.metric = metric;
  p.cnorm2 = cnorm2;
  p.b_hi = static_cast<const uint16_t*>(b_planes);   // plane 0: bf16(c) == the quantized row for bf16 inputs
  p.bext = static_cast<const uint16_t*>(bext);
  // pure-copy tail: nothing needs x again (no residual); the cosine loss needs ||c||^2
  p.copy_mode = p.fo.enabled && !p.fo.resid_out && !(metric == VQB_METRIC_COSINE && p.fo.loss_sum && !cnorm2);
  // residual-only tail of a ResidualVQ stage on the raw rows (Euclidean, or inputs that were already unit vectors)
  p.resid_mode = p.fo.enabled && p.fo.resid_out && !p.fo.q_out &&
                 (!p.fo.x_raw || p.fo.x_raw == p.fo.x_eff) && !(metric == VQB_METRIC_COSINE && p.fo.loss_sum && !cnorm2);
  p.stream_a = plan.stream_a;
  p.a_global = static_cast<const uint16_t*>(a_planes);
  p.n_stages = plan.n_stages;

  CUtensorMap tmA, tmB, tmS;
  rc = make_map(&tmA, a_planes, D, N, n_a, BK, BM, CU_TENSOR_MAP_SWIZZLE_128B);  // plane stride = N*D either way
  if (rc) return rc;
  rc = make_map(&tmB, b_planes, D, p.Kpad, 2, BK, WN, CU_TENSOR_MAP_SWIZZLE_128B);   // planes: bf16 hi, bf16 lo
  if (rc) return rc;
  rc = make_map(&tmS, bext, 16, p.Kpad, 1, 16, WN, CU_TENSOR_MAP_SWIZZLE_32B);      // seeds: B of the bias MMA
  if (rc) return rc;

  static bool attr_set = false;
  if (!attr_set) {
    void (*const kernels[6])(CUtensorMap, CUtensorMap, CUtensorMap, AssignParams) = {
        vq_assign_kernel<0, 128>, vq_assign_kernel<1, 128>, vq_assign_kernel<2, 128>,
        vq_assign_kernel<0, 256>, vq_assign_kernel<1, 256>, vq_assign_kernel<2, 256>};
    for (int i = 0; i < 6; ++i) {   // dynamic + static shared memory <= 227 KiB
      const int dyn = i < 3 ? SMEM_LIMIT : SMEM_LIMIT - WIDE_STATIC_SMEM;
      const cudaError_t e = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
      if (e != cudaSuccess) return static_cast<int>(e);
    }
    attr_set = true;
  }
  const int grid = p.num_row_tiles < num_sms() ? p.num_row_tiles : num_sms();
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (wide) {
    if (p.copy_mode) vq_assign_kernel<1, 256><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
    else if (p.resid_mode) vq_assign_kernel<2, 256><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
    else vq_assign_kernel<0, 256><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
  } else {
    if (p.copy_mode) vq_assign_kernel<1, 128><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
    else if (p.resid_mode) vq_assign_kernel<2, 128><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
    else vq_assign_kernel<0, 128><<<grid, NUM_THREADS, smem_bytes, s>>>(tmA, tmB, tmS, p);
  }
  return static_cast<int>(cudaGetLastError());
}
