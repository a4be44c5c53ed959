/* vqb200 — C ABI of the H100 (sm_90a) vector-quantization hot path.
 *
 * The reference (lucidrains/vector-quantize-pytorch v1.31.0) is pure Python and has NO FFI for this
 * path; its boundary is `Codebook.forward` (vector_quantize_pytorch/vector_quantize_pytorch.py:674-791)
 * called from `VectorQuantize.forward` (:1176).  These entry points are what a binding for that path
 * would need; each one cites the reference lines it replaces.  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (torch tensors); the library never
 *     allocates, frees or retains device memory;
 *   - every call only ENQUEUES work on `stream` (a cudaStream_t / CUstream passed as void*), never
 *     synchronises the host, and may be captured in a CUDA graph;
 *   - return value: 0 = ok, < 0 = VQB_E_* argument / capability error detected before launch,
 *     > 0 = a cudaError_t raised by the launch.  No exceptions, no printing.
 *   - matrices are row-major and contiguous; N = number of vectors, D = codebook dim, K = codebook size.
 */
#ifndef VQB200_H
#define VQB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VQB_VERSION 100 /* 0.1.0 */

#define VQB_DTYPE_F32 0
#define VQB_DTYPE_BF16 1

#define VQB_METRIC_EUCLID 0 /* -cdist(x, c)        vector_quantize_pytorch.py:58-62, :743 */
#define VQB_METRIC_COSINE 1 /* l2norm(x) . c^T     vector_quantize_pytorch.py:37-38, :741, :1159 */

#define VQB_OK 0
#define VQB_E_INVALID -1     /* null pointer / non-positive size / bad enum */
#define VQB_E_UNSUPPORTED -2 /* shape outside what the kernels support (see vqb_assign) */
#define VQB_E_ALIGN -3       /* pointer not 16-byte aligned */
#define VQB_E_NO_DEVICE -4   /* no CUDA device, or device is not sm_90 */
#define VQB_E_DRIVER -5      /* cuTensorMapEncodeTiled unavailable / failed */
#define VQB_E_WORKSPACE -6   /* workspace too small */

typedef struct vqb_flag_entry { /* one row whose winner the tensor-core passes could not certify (32 bytes) */
  int32_t row;                  /* vector index                                                            */
  int32_t count;                /* candidates inside the band; > 3 means "rescan the whole row"              */
  int32_t cand0;                /* best candidate of the tensor-core passes                                */
  int32_t cand1;                /* second candidate (valid if count >= 2)                                   */
                                /* (cand0, cand1) double as a 64-bit arg-max key during a whole-row rescan  */
  int32_t cand2;                /* third candidate (valid if count == 3)                                    */
  int32_t pad[3];
} vqb_flag_entry;

/* Optional fused tail of the search (gather + loss + residual update, see vqb_gather for the meaning of
 * every field).  Passed to vqb_assign, the certified rows are finished by the kernel's store warps while the
 * tensor cores work on the next tile; pass the same struct to vqb_fix_flagged, which finishes the re-scored
 * rows.  Host struct of device pointers. */
typedef struct vqb_fused_outputs {
  const void* x_eff;   /* [N][D] dtype, the rows as searched (l2-normalised for cosine)      */
  const float* embed;  /* [K][D] fp32 codebook                                                 */
  void* q_out;         /* [N][D] dtype or NULL                                                 */
  int64_t* idx64_out;  /* written at idx64_out[row*idx_stride] or NULL                         */
  int64_t idx_stride;
  double* loss_sum;    /* f64[1] += sum((q-x)^2) or NULL                                       */
  const void* x_raw;   /* NULL = x_eff                                                         */
  void* resid_out;     /* [N][D] dtype = x_raw - q or NULL                                     */
  void* qsum;          /* [N][D] dtype += q or NULL                                            */
  float* stats_cnt;    /* [K] cluster_size += 1 per row, or NULL (caller zeroes)                 */
  float* stats_sum;    /* [K][D] embed_sum += x_eff row (vector RED), or NULL (caller zeroes)    */
  int dtype;           /* VQB_DTYPE_*                                                          */
  void* planes_out;    /* optional, fp32 rows with resid_out: the bf16 hi / lo split of the residual, [2][N][D] — the MMA
                          operand of the NEXT ResidualVQ stage, which then skips vqb_input_prepare (NULL to skip)          */
} vqb_fused_outputs;

int vqb_version(void);
const char* vqb_strerror(int code);

/* Codebook rows are padded to a multiple of the MMA N-tile; planes/bias are sized with this. */
int vqb_padded_codes(int K);

/* Derive the tensor-core operands of a codebook from its fp32 rows (embed, K x D):
 *   planes  bf16 [2][Kpad][D] : [0] hi = bf16(c), [1] lo = bf16(c - hi)  (rows >= K are zero)
 *   bext    bf16 [Kpad][16]   : -bias as three bf16 terms in columns 0..2 (rest 0); rows >= K hold -3e38.
 *                               A K=16 MMA against [1 1 1 0..] seeds the accumulator with -bias.
 *   bias    f32  [Kpad]       : euclid 0.5*||c||^2, cosine 0, rows >= K +inf (informational)
 *   cnorm2  f32  [K]          : ||c||^2 (f64-accumulated), used by the exact re-score
 *   cmax    f32  [3]          : [0] max_k ||c||, [1] max_k ||c - hi - lo||, [2] max_k ||lo||: the exact norms that size the
 *                               certification band of the search
 * Buffers sized for an older, larger layout (planes [3][Kpad][D], cmax [4]) still work: only the leading part is used.
 * Supported: D % 8 == 0, D <= 1024 (VQB_E_UNSUPPORTED otherwise, as for vqb_assign).
 * Replaces nothing in the reference (it searches the fp32 rows directly, :710-712, :743); this is
 * the layout change that lets the search run on the tensor cores.  Also done by vqb_ema_apply. */
int vqb_codebook_prepare(const float* embed, int K, int D, int metric, void* planes, void* bext, float* bias,
                         float* cnorm2, float* cmax, void* stream);

/* Input staging (only needed for fp32 inputs and/or the cosine metric):
 *   x_eff    [N][D] in `dtype`: l2norm(x) evaluated in the input dtype (:1159 -> :376); may be NULL for euclid
 *   a_planes bf16 [n_planes][N][D]: bf16 hi / lo split of the (normalised) input — fp32 inputs, n_planes = 2.
 *            (bf16 inputs need no planes: vqb_assign reads the bf16 rows in place)
 * For a bf16 euclid input nothing is needed: x itself is the single A plane. */
int vqb_input_prepare(const void* x, int dtype, int64_t N, int D, int metric, void* x_eff, void* a_planes,
                      int n_planes, void* stream);

/* Nearest-code search: replaces cdist/einsum + argmax (:58-62, :741-747, :130-145) without ever
 * materialising the (N x K) distance matrix.  wgmma over TMA-staged tiles, fp32 accumulate in
 * registers, fused running arg-max.  Scores are x.c - 0.5||c||^2 (euclid) or x.c (cosine).
 *   a_planes  n_a = 1: bf16 rows [N][D] (the input itself, read in place); n_a = 2: bf16 hi/lo planes [2][N][D] of an fp32
 *             input (vqb_input_prepare).
 *   n_passes  n_a + 1 : the "split" scheme, bf16 hi / lo codebook planes into ONE fp32 accumulator:
 *                       (x,c_hi)+(x,c_lo) for bf16 rows, +(x_lo,c_hi) for fp32 rows;
 *             0       : automatic (= n_a + 1).
 *             Anything else returns VQB_E_UNSUPPORTED.
 *   b_planes/bext/cmax           from vqb_codebook_prepare / vqb_ema_apply
 *   margin_rel                   m, the tensor-core accumulation share of the certification band
 *                                W = 2(||x|| cres + ||x_lo|| caux + m ||x|| cmax + 2^-21 cmax^2) + tag slack + sqrt-collapse
 *                                width (DESIGN.md 4.1): a row is certified when its best score leads every other code
 *                                by more than W; otherwise it is appended to `flagged`
 *   idx       i32 [N]            winner of the tensor-core pass (final for unflagged rows)
 *   flagged   [N] entries, flag_count i32[2] (caller zeroes both): [0] rows with 2 / 3 candidates, appended from the
 *             front; [1] rows with more (whole-row exact re-scan), appended from the back (flagged[N-1], [N-2], ...)  -> vqb_fix_flagged
 *   dbg_best  f32 [N] or NULL    best score per row (tests)
 * Supported: D % 8 == 0, 8 <= D <= 1024, 1 <= K, N >= 1, sm_90 device.  When n_a * ceil(D/64) > 8 (fp32 split input with
 * D > 256) the A tile does not stay resident in shared memory: its k-blocks are streamed with the codebook's. */
int vqb_assign(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
               const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx, vqb_flag_entry* flagged,
               int32_t* flag_count, float* dbg_best, const vqb_fused_outputs* fused /* NULL: search only */, void* stream);

/* vqb_assign + the metric / ||c||^2 (cnorm2 [K]) that the in-kernel commitment loss of the COSINE metric needs.
 * When the fused tail asks for neither residual, running sum nor fused statistics, the tail degenerates to a row copy
 * q <- codebook row (bf16 inputs: the bf16 hi plane) and the loss is read off the winning score. */
int vqb_assign_ex(const void* a_planes, int n_a, int64_t N, int D, const void* b_planes, const void* bext,
                  const float* cmax, int K, float margin_rel, int n_passes, int32_t* idx, vqb_flag_entry* flagged,
                  int32_t* flag_count, float* dbg_best, const vqb_fused_outputs* fused, int metric, const float* cnorm2,
                  void* stream);

/* Diagnostics: i64 [grid][16] per-role cycle counters written by subsequent vqb_assign calls (NULL disables). */
int vqb_debug_set_profile_buffer(void* device_buffer);
int vqb_debug_active(void);
int vqb_debug_set_mode(int mode); /* nonzero: diagnostics mode (the forward chains are enqueued one by one, never graph-captured) */
/* How vqb_vq_forward's CUDA-graph cache served the calls so far: out4 = {replayed, patched (cudaGraphExecUpdate),
 * instantiated, enqueued launch by launch after a capture / instantiate failure} (host array of 4 int64). */
int vqb_debug_graph_stats(long long* out4);
/* The shared-memory plan vqb_assign launches with for (n_a, D, n_passes) — host only, no device needed.  out6 (host int[6]) =
 * {stream_a (A k-blocks travel through the ring), ring stages, seed slots, ring items per code step, ceil(D/64), dynamic smem
 * bytes}.  Returns the code vqb_assign returns for that input (VQB_E_INVALID / VQB_E_UNSUPPORTED) when it is not supported. */
int vqb_debug_assign_plan(int n_a, int D, int n_passes, int* out6);
/* The counting-sort plan of the EMA statistics (vqb_ema_stats, vqb_vq_forward) for N rows and K codes on a device with `sms`
 * SMs — host only.  out3 (host int[3]) = {G: row slabs of the CTA-local sort, 0 when the global-atomic kernels run; shift: a
 * slab is 128 << shift rows (31 on the global path); the slab bound vqb_ema_stats_workspace sizes the histograms for}. */
int vqb_debug_stats_plan(int64_t N, int K, int sms, int* out3);

/* Exact re-score of the flagged rows with the reference's own fp32 formula and tie rule
 * (-(x2 + y2 - 2xy).clamp(1e-8).sqrt(), first maximal index; :58-62, :140).  Rewrites idx[row]. */
int vqb_fix_flagged(const void* x_eff, int dtype, int64_t N, int D, const float* embed, const float* cnorm2, int K,
                    int metric, vqb_flag_entry* flagged, const int32_t* flag_count, int32_t* idx,
                    const vqb_fused_outputs* fused /* NULL: indices only */, void* stream);

/* Gather + tail of VectorQuantize.forward / one ResidualVQ stage:
 *   q_out     [N][D] dtype : embed[idx] cast to the input dtype                       (:766/:779-781, :1178)
 *   idx64_out i64, written at idx64_out[row*idx_stride]  (NULL to skip)              (:140 int64 contract)
 *   loss_sum  f64[1] += sum((q - x)^2)  (bf16: each square rounded to bf16 as torch does) (:1327)
 *   x_raw     [N][D] dtype : the stage input before l2norm (cosine); NULL = x_eff
 *   resid_out [N][D] dtype = x_raw - q   (NULL to skip)                               (residual_vq.py:524)
 *   qsum      [N][D] dtype += q      (NULL to skip)                                   (residual_vq.py:525) */
int vqb_gather(const void* x_eff, int dtype, int64_t N, int D, const float* embed, const int32_t* idx, void* q_out,
               int64_t* idx64_out, int64_t idx_stride, double* loss_sum, const void* x_raw, void* resid_out, void* qsum,
               void* stream);

/* commit loss = weight * mean, rounded like F.mse_loss in `dtype` (:1282, :1327-1329). loss_out f32[1]. */
int vqb_loss_finalize(const double* loss_sum, int64_t numel, int dtype, float weight, float* loss_out, void* stream);

/* Batch statistics of the EMA update (:586-607), packed so that ONE all-reduce covers both tensors:
 *   stats f32 [vqb_stats_floats(K, D)] = [cluster_size (K, padded to a multiple of 4) | embed_sum (K x D)]
 * Counting sort by code + segmented row sums (no float atomics on the common path). */
int64_t vqb_stats_offset(int K);          /* float offset of embed_sum inside stats */
int64_t vqb_stats_floats(int K, int D);   /* total floats of stats */
size_t vqb_ema_stats_workspace(int64_t N, int K);
int vqb_ema_stats(const void* x_eff, int dtype, int64_t N, int D, const int32_t* idx, int K, float* stats,
                  void* workspace, size_t workspace_bytes, void* stream);

/* EMA apply (:76-97, :616-617) + Laplace-smoothed normalisation (:152-154, :576-584), then refresh
 * the tensor-core operands for the next search.
 *   decay, eps   : python floats of the reference (doubles), rounded to fp32 where torch rounds them
 *   do_lerp      : cluster_size.lerp_(stats[:K], 1-decay); embed_avg.lerp_(stats[off:], 1-decay)
 *   do_normalise : embed = embed_avg / (laplace(cluster_size) * sum(cluster_size)); l2norm if cosine;
 *                  planes / bext / bias / cnorm2 / cmax are regenerated (all five required then)
 *   scratch      : f32[2] used internally
 * Supported: D % 8 == 0, D <= 1024 (VQB_E_UNSUPPORTED otherwise). */
int vqb_ema_apply(float* cluster_size, float* embed_avg, float* embed, const float* stats, int K, int D, double decay,
                  double eps, int metric, int do_lerp, int do_normalise, void* planes, void* bext, float* bias,
                  float* cnorm2, float* cmax, float* scratch, void* stream);

/* vqb_ema_apply with the reference's per-code `ema_update_weight` (:86-97, :609-610): the lerp weight of code k is
 * (1 - decay) * code_weight[k] (fp32 product).  code_weight f32 [K] or NULL (= vqb_ema_apply). */
int vqb_ema_apply_weighted(float* cluster_size, float* embed_avg, float* embed, const float* stats, int K, int D,
                           double decay, double eps, int metric, int do_lerp, int do_normalise, const float* code_weight,
                           void* planes, void* bext, float* bias, float* cnorm2, float* cmax, float* scratch, void* stream);

/* ---- multi-GPU: the all-reduce of the statistics (:603, :607) fused into the EMA kernels over NVLink peer memory ----
 * Every rank keeps its packed statistics in SYMMETRIC memory (one allocation mapped into every peer's address space;
 * the Python glue obtains the peer pointers from torch.distributed._symmetric_memory).  After vqb_peer_barrier the EMA
 * kernels read all `world` copies with peer loads and add them in rank order 0..world-1 — identical fp32 additions on
 * every rank, so the replicas stay bit-identical.  Both calls only enqueue kernels (graph-capturable).
 *
 * vqb_peer_barrier: cross-GPU barrier.  peer_flags_host[r] = rank r's flag array u32[world] (symmetric memory, zeroed
 *   once), host array of `world` device pointers; epoch_dev u32[1] device memory owned by this rank (zeroed once).
 *   Everything this rank wrote before the barrier is visible to every peer's reads after it (release / acquire, system
 *   scope).  The caller double-buffers the statistics by step parity (a buffer may be rewritten two barriers later). */
int vqb_peer_barrier(void* const* peer_flags_host, int rank, int world, uint32_t* epoch_dev, void* stream);
/* vqb_ema_apply_weighted with `stats` replaced by the sum over ranks of peer_stats_host[r][slice_offset ...]
 * (host array of `world` device pointers to the ranks' packed buffers; slice_offset in floats, multiple of 4). */
int vqb_ema_apply_peers(float* cluster_size, float* embed_avg, float* embed, const void* const* peer_stats_host, int world,
                        int64_t slice_offset, int K, int D, double decay, double eps, int metric, int do_normalise,
                        const float* code_weight, void* planes, void* bext, float* bias, float* cnorm2, float* cmax,
                        float* scratch, void* stream);

/* One-call composite of VectorQuantize.forward's arithmetic (or one ResidualVQ stage): input staging ->
 * vqb_assign (+ fused tail) -> vqb_fix_flagged -> vqb_loss_finalize -> vqb_ema_stats -> vqb_ema_apply, all
 * enqueued from C++ (the Python glue pays one FFI call instead of ~20).  Replaces vqp:1159-1178 + :674-791.
 * Repeated calls with identical arguments are replayed from a cached CUDA graph (VQB_GRAPH=0 disables); besides the
 * launch gaps this removes the sensitivity of the step time to host-side scheduling jitter. */
typedef struct vqb_vq_forward_args {
  const void* x;            /* [N][D] dtype, BEFORE the cosine l2norm                                         */
  int dtype, metric;
  int64_t N;
  int D, K;
  int already_normalised;   /* cosine only: x is already unit-norm (Codebook.forward contract)                 */
  float* cluster_size;      /* [K]      state (update == 2)                                                    */
  float* embed_avg;         /* [K][D]   state (update == 2)                                                    */
  float* embed;             /* [K][D]   fp32 codebook (always)                                                 */
  void* planes; void* bext; float* bias; float* cnorm2; float* cmax; float* scratch; /* vqb_codebook_prepare     */
  void* q_out;              /* [N][D] dtype or NULL                                                            */
  int64_t* idx64_out; int64_t idx_stride;   /* int64 indices (NULL to skip)                                    */
  float* loss_out; float loss_weight;       /* f32[1] = weight * mse (NULL to skip)                            */
  void* resid_out; void* qsum;              /* ResidualVQ recurrence (NULL to skip)                            */
  int32_t* idx32;           /* [N] int32 indices (always written; input of the statistics)                     */
  int update;               /* 0: none; 1: statistics only (caller all-reduces, then vqb_ema_apply); 2: + apply;
                               3: + peer barrier + apply over every rank's statistics (see peer_* below)             */
  int stats_mode;           /* 0: statistics accumulated by the search kernel's store warps (vector RED into L2);
                               1: separate counting-sort + segmented-sum kernels (vqb_ema_stats)                 */
  int stats_accumulate;     /* stats_mode 0: do not zero `stats` first (chunked batches sum their statistics)   */
  int do_normalise;         /* update == 2: also embed = embed_avg / smoothed cluster_size                      */
  double decay, eps;
  float* stats;             /* [vqb_stats_floats(K, D)] (update != 0)                                          */
  float margin_rel;
  void* workspace; size_t workspace_bytes;  /* >= vqb_vq_forward_workspace(...), 256-byte aligned              */
  void* ev_search_begin; void* ev_search_end; /* optional cudaEvent_t recorded around the search kernel (profiling) */
  /* update == 3: statistics into `stats` (this rank's symmetric buffer slice) -> vqb_peer_barrier -> vqb_ema_apply_peers:
   * the whole multi-GPU step is one chain / one CUDA graph.  Unused (NULL / 0) otherwise. */
  const void* const* peer_stats; void* const* peer_flags; uint32_t* peer_epoch; int peer_rank, peer_world;
  int64_t peer_slice_offset;
  /* ResidualVQ stages on fp32 rows (Euclidean): a stage can take the bf16 hi / lo split of its input ([2][N][D], written by the
   * previous stage's tail through `planes_out`) instead of running vqb_input_prepare.  NULL = not used. */
  const void* a_planes_in; void* planes_out;
  /* Variable-length batches (mask / lens, vector_quantize_pytorch.py:1116-1119).  row_mask u8 [N], 0 = padding row: the row is
   * searched (the tiles stay dense) but gets index -1 in idx32, its q_out / idx64_out are NOT written (the caller pre-fills them:
   * zeros or the input, and -1, :1378-1396), it adds nothing to the loss (:1317-1325) or to the statistics (:599-600) and is
   * never re-scored.  n_live i64 [1] (device): the number of unmasked rows, the divisor of the loss (NULL: N).  VectorQuantize
   * chain only (resid_out / qsum / planes_out must be NULL, stats_mode 1).  NULL = no mask. */
  const uint8_t* row_mask; const int64_t* n_live;
} vqb_vq_forward_args;
size_t vqb_vq_forward_workspace(int64_t N, int D, int K, int dtype, int metric, int update);
int vqb_vq_forward(const vqb_vq_forward_args* args, void* stream);

/* Decode (next row of SURVEY 8f): out[row] = sum_q embed_q[idx[row, q]], index -1 contributes zeros
 * (vector_quantize_pytorch.py:998-1022, residual_vq.py:324-382).  embeds: Q codebooks stacked [Q][K][D] f32
 * (pass the same pointer stride 0 for a shared codebook via `embed_stride` in elements). */
int vqb_decode(const float* embeds, int64_t embed_stride, int Q, int K, int D, const int64_t* idx, int64_t N,
               void* out, int dtype, void* stream);

/* ResidualVQ's running sum rebuilt from the stage indices in one pass:
 *   out = (((q_0) + q_1) + ... + q_{Q-1}),  q_j = embed_j[idx[row, j]].type(dtype), every partial sum rounded to dtype
 * exactly like `quantized_out = quantized_out + quantized` (residual_vq.py:525, vector_quantize_pytorch.py:1178).
 * idx i64 [N][Q] (no -1 entries), embeds as for vqb_decode.  Replaces Q read-modify-write passes over (N x D). */
int vqb_rvq_accumulate(const float* embeds, int64_t embed_stride, int Q, int K, int D, const int64_t* idx, int64_t N,
                       void* out, int dtype, void* stream);
/* The slice plan vqb_decode / vqb_rvq_accumulate launch with — host only, no device needed.  nbooks codebooks (1 when
 * embed_stride is 0, Q otherwise) of K x D, staged as esz-byte elements (2: vqb_rvq_accumulate in bf16; 4 otherwise), N rows,
 * `sms` SMs.  out3 (host int[3]) = {W: column slice of every codebook in shared memory, 0 when the L2 kernel runs; slices =
 * D / W; CTAs per slice}. */
int vqb_debug_gather_sum_plan(int nbooks, int K, int D, int esz, int64_t N, int sms, int* out3);

/* A whole ResidualVQ / GroupedResidualVQ forward in ONE call (residual_vq.py:469-568 the stage loop, :593-601 the
 * deferred codebook updates, :676-724 the groups): the ops are enqueued in order and replayed together from one cached
 * CUDA graph, so the host pays one FFI call per forward instead of one per stage, and the chains of different lanes —
 * the independent groups of GroupedResidualVQ — run on parallel streams that fork from / join into `stream`.
 *   VQB_RVQ_STAGE       vqb_vq_forward(stage)             one quantizer (update = 1: its EMA is deferred to a later EMA op)
 *   VQB_RVQ_EMA         vqb_ema_apply_weighted(ema ...)   residual_vq.py:593-597 / vector_quantize_pytorch.py:616-617, :576-584
 *   VQB_RVQ_ACCUMULATE  vqb_rvq_accumulate(acc ...)       quantized_out from the indices (residual_vq.py:525)
 *   VQB_RVQ_BARRIER     vqb_peer_barrier(bar ...)         multi-GPU: every rank's statistics of this forward are in place
 *   VQB_RVQ_EMA_PEERS   vqb_ema_apply_peers(emap ...)     the EMA op with the sum over ranks taken inside (vqp:603, :607)
 * At most 62 ops, lanes 0..3; ops of one lane execute in list order. */
enum { VQB_RVQ_STAGE = 0, VQB_RVQ_EMA = 1, VQB_RVQ_ACCUMULATE = 2, VQB_RVQ_BARRIER = 3, VQB_RVQ_EMA_PEERS = 4 };
typedef struct vqb_rvq_op {
  int kind, lane;
  vqb_vq_forward_args stage;
  struct {
    float* cluster_size; float* embed_avg; float* embed; const float* stats; int K, D; double decay, eps;
    int metric, do_lerp, do_normalise; void* planes; void* bext; float* bias; float* cnorm2; float* cmax; float* scratch;
    int n_lerp; int64_t slice_stride;  /* n_lerp > 1: that many statistics slices, slice_stride floats apart, are lerped in order
                                          in one launch — the stages of a shared codebook (residual_vq.py:302-306) */
  } ema;
  struct {
    const float* embeds; int64_t embed_stride; int Q, K, D; const int64_t* idx; int64_t N; void* out; int dtype;
  } acc;
  struct { void* const* flags; uint32_t* epoch; int rank, world; } bar;
  struct {
    float* cluster_size; float* embed_avg; float* embed; const void* const* peer_stats; int64_t slice_offset; int world, K, D;
    double decay, eps; int metric, do_normalise; void* planes; void* bext; float* bias; float* cnorm2; float* cmax; float* scratch;
    int n_lerp; int64_t slice_stride;  /* as in `ema` */
  } emap;
} vqb_rvq_op;
int vqb_rvq_forward(const vqb_rvq_op* ops, int n_ops, void* stream);

/* Rotation-trick gradient estimator (vector_quantize_pytorch.py:287-318, default when x.requires_grad, :856, :1225-1228).
 *   grad_out == NULL: forward   out = rotate_to(src, tgt)        (numerically ~ tgt, carries d out / d src)
 *   grad_out != NULL: backward  out = d loss / d src given d loss / d rotate_to(src, tgt)
 * src, tgt, grad_out, out: [N][D] in `dtype` (arithmetic in fp32, rounded once on store). */
int vqb_rotate(const void* src, const void* tgt, const void* grad_out, int64_t N, int D, int dtype, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQB200_H */
