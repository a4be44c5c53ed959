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
  void* qsum;          /* reserved, must be NULL (VQB_E_UNSUPPORTED otherwise): ResidualVQ rebuilds */
                       /* its running sum from the indices (vqb_rvq_accumulate)                  */
  float* stats_cnt;    /* reserved, must be NULL (VQB_E_UNSUPPORTED otherwise): statistics come */
  float* stats_sum;    /* from vqb_ema_stats, the tail accumulates none                          */
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
 * When the fused tail asks for no residual, the tail degenerates to a row copy
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
 *   qsum      reserved, must be NULL (VQB_E_UNSUPPORTED otherwise): ResidualVQ's running sum (residual_vq.py:525)
 *             is rebuilt from the indices by vqb_rvq_accumulate */
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
  void* resid_out;                          /* ResidualVQ recurrence: x - q (NULL to skip)                     */
  void* qsum;                               /* reserved, must be NULL (VQB_E_UNSUPPORTED otherwise): the running
                                               sum is rebuilt from the indices (vqb_rvq_accumulate)             */
  int32_t* idx32;           /* [N] int32 indices (always written; input of the statistics)                     */
  int update;               /* 0: none; 1: statistics only (caller all-reduces, then vqb_ema_apply); 2: + apply;
                               3: + peer barrier + apply over every rank's statistics (see peer_* below)             */
  int stats_mode;           /* ignored: the statistics always come from the counting sort (vqb_ema_stats)         */
  int stats_accumulate;     /* must be 0 when update != 0 (VQB_E_UNSUPPORTED otherwise): `stats` is overwritten    */
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
   * chain only (resid_out / planes_out must be NULL).  NULL = no mask. */
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
 *   VQB_RVQ_SIMVQ_TAIL  vqb_rsimvq_tail(simvq ...)        one ResidualSimVQ stage tail, after that stage's search op
 * At most 62 ops, lanes 0..3; ops of one lane execute in list order. */
enum { VQB_RVQ_STAGE = 0, VQB_RVQ_EMA = 1, VQB_RVQ_ACCUMULATE = 2, VQB_RVQ_BARRIER = 3, VQB_RVQ_EMA_PEERS = 4,
       VQB_RVQ_SIMVQ_TAIL = 5 };
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
  struct {  /* the arguments of vqb_rsimvq_tail, in its order */
    const float* r; const float* codes; const int32_t* idx; int64_t N; int D, rotation; float* r_next; float* qsum; int first;
    int64_t* idx64_out; int64_t idx_stride; double* loss_sum; float* loss_out; float input_weight, weight;
  } simvq;
} vqb_rvq_op;
int vqb_rvq_forward(const vqb_rvq_op* ops, int n_ops, void* stream);

/* ResidualSimVQ (residual_sim_vq.py of the reference: a stack of SimVQ layers, rsv:182-203 over sim_vq.py:100-138).  A stage
 * is a search of the residual r (N x D fp32) against the stage's implicit codebook (vqb_codebook_prepare + a VQB_RVQ_STAGE op,
 * update = 1 when the codebook needs a gradient: its statistics [count | sum of r] per code are the codebook gradient's input),
 * then this tail, one warp per row (D <= 1024):
 *   c = codes[idx[row]] (codes [K][D] fp32, idx i32 [N] from the search)
 *   out = rotate_to(r, c) (rotation != 0, vector_quantize_pytorch.py:287-318) or (c - r) + r, in fp32
 *   r_next = r - out (NULL for the last stage)  — the estimator's forward value, as rsv:195 subtracts it
 *   qsum = 0 + out (first != 0) or qsum + out   — quantized_out, rsv:196
 *   idx64_out[row * idx_stride] = idx (NULL to skip)
 *   loss_out f32[1] = (mse + mse * input_weight) * weight with mse = mean((r - c)^2), sim_vq.py:121-124, :138; loss_sum f64[1]
 *   is its scratch (NULL loss_out: no loss) */
int vqb_rsimvq_tail(const float* r, const float* codes, const int32_t* idx, int64_t N, int D, int rotation, float* r_next,
                    float* qsum, int first, int64_t* idx64_out, int64_t idx_stride, double* loss_sum, float* loss_out,
                    float input_weight, float weight, void* stream);
/* Backward of a whole ResidualSimVQ forward, one warp per row.  The residuals r_0 = x, r_1, ... are recomputed with the tail's
 * own arithmetic (bit-identical to the forward's), so no residual is kept between forward and backward:
 *   grad_x = sum_{q < n_active} [ rotate_to backward of grad_q at (r_q, c_q) (or grad_q itself without the rotation trick)
 *                                 + grad_loss[q] * (r_q - c_q) ]
 *   codes [Q][K][D] fp32 (the codebooks the stages searched), idx i64 [N][Q], grad_q [N][D] or NULL (zero), grad_loss f32 [Q]
 *   or NULL (zero): dL/dloss_q already multiplied by 2 * weight * input_weight / (N * D).  Stages >= n_active were dropped.
 * The codebook gradient 2 weight dL/dloss_q / (N D) * (count * c - sum of r) comes from the stage statistics (caller). */
int vqb_rsimvq_backward(const float* x, const float* codes, int Q, int K, const int64_t* idx, int64_t N, int D, int n_active,
                        int rotation, const float* grad_q, const float* grad_loss, float* grad_x, void* stream);

/* Rotation-trick gradient estimator (vector_quantize_pytorch.py:287-318, default when x.requires_grad, :856, :1225-1228).
 *   grad_out == NULL: forward   out = rotate_to(src, tgt)        (numerically ~ tgt, carries d out / d src)
 *   grad_out != NULL: backward  out = d loss / d src given d loss / d rotate_to(src, tgt)
 * src, tgt, grad_out, out: [N][D] in `dtype` (arithmetic in fp32, rounded once on store). */
int vqb_rotate(const void* src, const void* tgt, const void* grad_out, int64_t N, int D, int dtype, void* out, void* stream);

/* The estimator of a masked training step (vector_quantize_pytorch.py:1225-1233, :1317-1325, :1378-1389), one warp per row.
 * row_mask u8 [N] (0: padding), n_live i64 [1] = the number of live rows, both on the device; src = x, tgt = the codes the
 * masked search wrote for the live rows (its padding rows are never read).
 *   grad_out == NULL: forward   live rows tgt, padding rows 0 (pad_zeros != 0) or src
 *   grad_out != NULL: backward  live rows  E(grad_out) + c (src - tgt),  c = 2 loss_weight grad_loss[0] / (n_live[0] D)
 *                               padding rows 0 (pad_zeros != 0) or grad_out
 * E = the rotate_to backward of vqb_rotate (VQB_ESTIMATOR_ROTATE), the identity (VQB_ESTIMATOR_STE) or 0 (VQB_ESTIMATOR_NONE);
 * grad_loss f32 [1] = d loss / d commitment loss, NULL: no commitment term.  Padding rows never reach the rotation.
 * src, tgt, grad_out, out: [N][D] in `dtype` (arithmetic in fp32, rounded once on store). */
#define VQB_ESTIMATOR_NONE 0
#define VQB_ESTIMATOR_STE 1
#define VQB_ESTIMATOR_ROTATE 2
int vqb_rotate_masked(const void* src, const void* tgt, const void* grad_out, const float* grad_loss, const uint8_t* row_mask,
                      const int64_t* n_live, float loss_weight, int estimator, int pad_zeros, int64_t N, int D, int dtype,
                      void* out, void* stream);

/* DiVeQ, the directional reparameterization estimator (vector_quantize_pytorch.py:323-330), one warp per row (D <= 1024):
 *   e = q - x,  u = l2norm(e + noise_scale * noise) (detached),  out = x + u * ||e||
 *   grad_out == NULL: forward   out = x + u ||e||                                  (dtype)
 *   grad_out != NULL: backward  out = dx = g - (g.u) e / ||e||, grad_q = (g.u) e / ||e||   (0 where ||e|| = 0)
 * x, q, noise (the raw N(0, 1) draw), grad_out, out: [N][D] in `dtype`; grad_q: f32 [N][D] (values rounded to `dtype`).
 * Every step is rounded to `dtype` where torch rounds the reference's expression; the backward recomputes e, u and ||e||. */
int vqb_diveq(const void* x, const void* q, const void* noise, const void* grad_out, int64_t N, int D, int dtype,
              float noise_scale, void* out, float* grad_q, void* stream);

/* Finite scalar quantization (finite_scalar_quantization.py "fsq", residual_fsq.py "rfsq"), one thread per (row, group) item.
 * z [N][G][D] (D = len(levels) <= 16, 16-byte aligned base) in in_dtype; work_dtype is the dtype of the reference's outer
 * chain and of `out` (the soft clamp, the stage scaling, the residual, the running sum): f32, or bf16 for bf16 inputs only.
 * consts f32 [7][D], computed by the caller with the reference's torch expressions:
 *   row 0  L - 1 (sym) | half_l = (L - 1) (1 + eps) / 2 (fsq:152)      row 1  2 / (L - 1) (sym) | offset (fsq:153)
 *   row 2  shift (fsq:154; unused when sym)                            row 3  L // 2 (fsq:156)     row 4  basis (fsq:92)
 *   row 5  1 / (2 / (L - 1))                                           row 6  1 / (L // 2)
 * (the reciprocals, rounded to nearest, turn every division by a constant into a correctly rounded product-and-fma).
 * sym: symmetry_preserving_bound (fsq:161-169), else bound (fsq:147-157); hard: the clamp replaces tanh (and atanh).
 * scales f32 [2][Q][D]: the W values of rfsq's `scales`, then their reciprocals (NULL for a plain FSQ: no scaling, Q = 1);
 * clampv f32 [2][D]: the soft-clamp value (rfsq:193-195) and its reciprocal (NULL: none).  Stages >= n_active (quantize
 * dropout) write index -1 and add nothing.  N * G < 2^31. */
int vqb_fsq_forward(const void* z, int in_dtype, int work_dtype, int64_t N, int G, int D, int Q, int n_active, int sym, int hard,
                    const float* consts, const float* scales, const float* clampv, void* out, void* idx, int idx64,
                    int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, void* stream);
/* d z of vqb_fsq_forward's `out` given grad_out [N][G][D] (work_dtype), the straight-through chain in autograd's order,
 * every stage recomputed from z (nothing kept from the forward).  grad_z [N][G][D] in in_dtype.  n_active * D <= 768. */
int vqb_fsq_backward(const void* z, int in_dtype, int work_dtype, int64_t N, int G, int D, int Q, int n_active, int sym, int hard,
                     const float* consts, const float* scales, const float* clampv, const void* grad_out, void* grad_z,
                     void* stream);
/* indices (element (row, g, q) at idx + row * idx_s_row + g * idx_s_g + q * idx_s_q, int32 or int64; -1 = dropped stage) ->
 * out [N][G][D] = sum_q code_q * scale_q (work_dtype) and/or codes [Q][N][G][D] (the scaled stage codes), each code from the
 * index digits (index // basis) % L.  levels_basis i32 [2][D]: levels, basis.  scales NULL: unscaled (fsq indices_to_codes). */
int vqb_fsq_decode(const void* idx, int idx64, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, int64_t N, int G, int D,
                   int Q, int work_dtype, int sym, const float* consts, const int32_t* levels_basis, const float* scales, void* out,
                   void* codes, void* stream);

/* Lookup-free quantization (lookup_free_quantization.py "lfq", residual_lfq.py "rlfq"), one thread per (row, group) item.
 * z [N][G][D] (D = log2(codebook_size) <= 20) in dtype (f32 or bf16; the chain runs in the input dtype, rounding after every
 * op).  params f32 [3][Q]: per stage the codebook_scale s, the code magnitude m (s, or the reference's l2norm(+-s) * s when
 * spherical) and the soft-clamp value (0: none).  Per stage q < n_active: soft clamp, spherical l2norm, q = x > 0 ? m : -m,
 * index bit j = 2^(D-1-j) (int64, element (row, g, q) at idx + row * idx_s_row + g * idx_s_g + q * idx_s_q; -1 for q >=
 * n_active), value x + (q - x) (training) or q, residual -= value, out += value (residual) or out = value (a plain LFQ).
 * ent f32 [n_active][N][G][D] or NULL: the entropy input x of every stage.  rowmask u8 [N] or NULL: rows that count in the
 * commitment sums.  commit f64 [n_active][commit_blocks] or NULL: per-block sums of (x - q)^2, commit_blocks =
 * vqb_lfq_forward_blocks(N, G).  N * G < 2^31, Q <= 64. */
int vqb_lfq_forward(const void* z, int dtype, int64_t N, int G, int D, int Q, int n_active, int residual, int training, int spherical,
                    const float* params, void* out, void* idx, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, float* ent,
                    const uint8_t* rowmask, double* commit, int commit_blocks, void* stream);
int vqb_lfq_forward_blocks(int64_t N, int G);
/* Entropy statistics of lfq:365-398 over K = 2^D codes without the (rows, K) matrix, every stage and group in one launch.
 * x f32 [S][N][G][D] (vqb_lfq_forward's ent); sg = s * G + g.  rows i32 [S * G][rows_stride] or NULL (rows 0..R-1): the R
 * rows of each sg (rows_stride 0: one list shared by all sg).  m f32 [S]; logits 2 tau m (x . sgn_k).  Writes
 * pse f64 [S * G][chunks][vqb_lfq_entropy_tiles(D)]: partial sums of h(p) = -p ln(max(p, 1e-5)) over the rows and codes, and
 * colsum f32 [chunks][S * G][K] (NULL: not needed) partial column sums of p; each chunk covers ceil(R / chunks) rows.  Sums run
 * in a fixed order: equal inputs give equal bits. */
int vqb_lfq_entropy(const float* x, int64_t N, int G, int D, int S, const int32_t* rows, int64_t R, int64_t rows_stride,
                    const float* m, float tau, int chunks, double* pse, float* colsum, void* stream);
int vqb_lfq_entropy_tiles(int D);
/* d/dx of the entropy outputs given dL/dp[sg][row][k] = cp[sg] h'(p) + V[sg][k] (cp f32 [S * G]; V f32 [S * G][K] or NULL),
 * h'(p) = -(ln p + 1) for p >= 1e-5, -ln 1e-5 below.  Writes grad (the layout of x) at the listed rows only.  ksplit: a power
 * of two dividing K into ranges of >= 16 codes; work f32 [ksplit][S * G][R][D + 1]. */
int vqb_lfq_entropy_backward(const float* x, int64_t N, int G, int D, int S, const int32_t* rows, int64_t R, int64_t rows_stride,
                             const float* m, float tau, const float* cp, const float* V, int ksplit, float* work, float* grad,
                             void* stream);
/* d z of vqb_lfq_forward's chain: grad_out [N][G][D] (dtype) through the straight-through value, plus grad_ent (f32, the
 * layout of ent, or NULL) and cc[q] * (x - q) for the rows of rowmask (cc f32 [Q] or NULL: the commitment gradient), through
 * the l2norm, the soft clamp and the residual chain; every stage recomputed from z.  grad_z [N][G][D] in dtype.  In eval
 * (training 0) the value is q, which does not depend on z: grad_out contributes nothing. */
int vqb_lfq_backward(const void* z, int dtype, int64_t N, int G, int D, int Q, int n_active, int residual, int training, int spherical,
                     const float* params, const void* grad_out, const float* grad_ent, const float* cc, const uint8_t* rowmask,
                     void* grad_z, void* stream);
/* indices (int32 / int64, strided as in vqb_lfq_forward; -1 = dropped stage: zeros) -> codes f32 [Q][N][G][D] (bit set: vals[q],
 * else -vals[q]) and / or out f32 [N][G][D], their fp32 sum over the stages in stage order. */
int vqb_lfq_decode(const void* idx, int idx64, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, int64_t N, int G, int D, int Q,
                   const float* vals, float* out, float* codes, void* stream);

/* Finite scalar perturbation (finite_scalar_perturbation.py "fsp"), one thread per row.  z [N][D] (D = len(levels) <= 16,
 * N < 2^31) in dtype (f32 or bf16), every pointer to an [N][D] plane 16-byte aligned; levels i32 [D] on the device
 * (prod(levels) < 2^31); act 0..4 = tanh, sigmoid, normal, laplace, cauchy; inv = need_inv_act.
 * vqb_fsp_blocks(N): the CTA count of every fsp launch over N rows (sizes accept and the stats work), or a VQB_E_* code. */
int vqb_fsp_blocks(int64_t N);
/* The row chain of fsp:323-351.  clamp_hi: 1 - eps cast to dtype (clamp_max before floor).  u1, u2: the two uniform draws
 * [N][D] in dtype (fsp:334, :340), or both NULL (eval, quantize_rate == 1: no perturbation); qrate: quantize_rate cast to dtype.
 * inv_lo, inv_hi: eps and 1 - eps cast to the output dtype (need_inv_act's clamp).  out [N][D]: f32 when perturbing, else dtype.
 * idx i32 [N]: the exact mixed-radix index; level_idx [N][D] in dtype or NULL; accept i32 [accept_blocks] (required when
 * perturbing): per-CTA counts of accepted proposals, accept_blocks = vqb_fsp_blocks(N). */
int vqb_fsp_forward(const void* z, int dtype, int64_t N, int D, int act, int inv, const int32_t* levels, float clamp_hi,
                    const void* u1, const void* u2, float qrate, float inv_lo, float inv_hi, void* out, int32_t* idx,
                    void* level_idx, int32_t* accept, int accept_blocks, void* stream);
/* Batch moments of z over the rows (fsp:93-99) and VectorNorm's loss (fsp:126-133), in fp64 with partials added in a fixed
 * order.  norm: host f64 [8] = l1_target, l1_weight, ..., l4_target, l4_weight.  work f64 [4 * blocks + 1][D], blocks =
 * vqb_fsp_blocks(N).  stats [4][D] (mean, unbiased variance, skewness, kurtosis - 3) and loss [1] in dtype; aux f64 [D][8]
 * (mean, clamped std, skewness, kurtosis, mean(t^2), clamp mask, variance, 0) for vqb_fsp_backward. */
int vqb_fsp_stats(const void* z, int dtype, int64_t N, int D, const double* norm, double* work, int blocks, void* stats,
                  void* loss, double* aux, void* stream);
/* d z of the FSP step: grad_q [N][D] (grad_dtype; NULL: zero) through the output map and the CDF (the identity with inv), plus
 * the statistics path from grad_stats f32 [4][D] and grad_loss f32 [1] (each NULL: zero), aux from vqb_fsp_stats.
 * grad_z [N][D] in dtype. */
int vqb_fsp_backward(const void* z, int dtype, int64_t N, int D, int act, int inv, const void* grad_q, int grad_dtype,
                     const double* aux, const float* grad_stats, const float* grad_loss, const double* norm, void* grad_z,
                     void* stream);
/* indices (contiguous [N], int32 or int64) -> act values (l + 1/2) / L (act_out f32 [N][D] or NULL) and codes f32 [N][D] (or
 * NULL): (act - 0.5) / 0.28867513459481287, or with inv the inverse CDF of act clamped to [lo, hi] (fsp:286-307). */
int vqb_fsp_decode(const void* idx, int idx64, int64_t N, int D, int act, int inv, const int32_t* levels, float lo, float hi,
                   float* act_out, float* codes, void* stream);


/* BinaryMapper (binary_mapper.py "bm"): the (rows, 2^bits) one-hot and its straight-through gradient, 1 <= bits <= 20.
 * vqb_binmap_hot: out f32 [rows][2^bits], zero-filled by the caller and 16-byte aligned; idx i64 [rows] (the sampled code).
 * Writes out[r][idx[r]]: 1 when logits is NULL (no straight-through), else fl(fl(1 + s) - s) with s the soft code of idx[r]
 * from logits f32 [rows][bits] (bit 0 least significant).  A row with a non-finite logit is written whole: NaN where the
 * reference's per-code log-probability is 0 * -inf or NaN, 0 elsewhere. */
int vqb_binmap_hot(const float* logits, const int64_t* idx, int64_t rows, int bits, float* out, void* stream);
/* The K split and segment width vqb_binmap_backward is run with for (rows, bits) on `sms` SMs: plan[0] = ksplit (a power of
 * two), plan[1] = codes per segment (min(32, 2^bits)).  Host-only. */
int vqb_binmap_backward_plan(int64_t rows, int bits, int sms, int* plan);
/* d logits [rows][bits] f32 of sum(out * g) through the straight-through soft codes: S1_j - sigmoid(l_j) S with
 * S = sum_k g_k s_k, S1_j = sum_{bit_j(k) = 1} g_k s_k, evaluated as sigmoid(-l_j) S1_j - sigmoid(l_j) S0_j.  g[r][k] at
 * g + r * g_row_stride + k * g_col_stride (floats, any 4-byte alignment, strides >= 0).  ksplit: a power of two dividing
 * the segment count; ksplit > 1 needs work f64 [rows][ksplit][2 bits].  Rows with a non-finite logit get NaN. */
int vqb_binmap_backward(const float* logits, int64_t rows, int bits, const float* g, int64_t g_row_stride,
                        int64_t g_col_stride, int ksplit, double* work, float* dlogits, void* stream);

/* HierarchicalVQ (hierarchical_vq.py "hvq"): the per-scale pool, upsample and residual update around the shared search, fp32,
 * no atomics (every backward is the gather-form adjoint, so reruns give the same bits).  Images are NCHW (B, D, H, W)
 * contiguous; rows are the channel-last (B, s, s, D) contiguous map the search reads and writes.  1 <= H, W, s <= 65536.
 * vqb_hvq_pool: rows = adaptive_avg_pool2d(x, (s, s)) with ATen's windows [floor(i H / s), ceil((i + 1) H / s)) (hvq:134). */
int vqb_hvq_pool(const float* x, int64_t B, int D, int H, int W, int s, float* rows, void* stream);
/* g_x (B, D, H, W) = the adjoint of vqb_hvq_pool applied to g_rows (B, s, s, D): each pixel sums g / kh / kw over its windows. */
int vqb_hvq_pool_backward(const float* g_rows, int64_t B, int D, int H, int W, int s, float* g_x, void* stream);
/* u = bilinear(rows (B, s, s, D), (H, W), align_corners = False) with ATen's source-index rule, or rows itself when
 * (s, s) == (H, W) (hvq:105-106).  Writes, each when non-NULL: q = u; recon_out = recon + u (recon NULL: 0 + u);
 * resid_out = resid - u (needs resid).  At least one output. */
int vqb_hvq_upsample(const float* rows, int64_t B, int D, int s, int H, int W, float* q, const float* recon,
                     const float* resid, float* recon_out, float* resid_out, void* stream);
/* g_rows (B, s, s, D) = the adjoint of vqb_hvq_upsample applied to g_a - g_b (each (B, D, H, W), NULL: zero; not both). */
int vqb_hvq_upsample_backward(const float* g_a, const float* g_b, int64_t B, int D, int s, int H, int W, float* g_rows,
                              void* stream);
/* q = (1 - r) up + r conv over n elements (hvq:25; both factors rounded to fp32, no fma), then recon_out = recon + q (recon
 * NULL: 0 + q) and resid_out = resid - q, each when non-NULL (at least one; resid_out needs resid). */
int vqb_hvq_blend_update(const float* up, const float* conv, int64_t n, double r, const float* recon, const float* resid,
                         float* recon_out, float* resid_out, void* stream);
/* g_q = g_recon - g_resid (each NULL: zero; not both), g_up = (1 - r) g_q, g_conv = r g_q. */
int vqb_hvq_blend_backward(const float* g_recon, const float* g_resid, int64_t n, double r, float* g_up, float* g_conv,
                           void* stream);

/* RandomProjectionQuantizer (random_projection_quantizer.py "rpq"): the rows its cosine search takes (rpq:49-53), in one fp32
 * pass over x (N, dim) contiguous:
 *   rows[r, h E + j] = sum_d LN(x[r])[d] proj[h, d, j]     (N, H E) contiguous; proj (H, dim, E) contiguous, as `rand_projs`
 * LN(v) = (v - mean) / sqrt(var + 1e-5) with the mean and the biased variance in fp32 (nn.LayerNorm(dim, elementwise_affine =
 * False)); norm = 0 skips it.  A full fp32 product (no TF32); the normalised x is never written.  1 <= dim <= 65536,
 * H E <= 1024, N dim and N H E below 2^40 (VQB_E_UNSUPPORTED otherwise); pointers 4-byte aligned (VQB_E_ALIGN). */
int vqb_rpq_norm_project(const float* x, int64_t N, int dim, const float* proj, int H, int E, int norm, float* rows,
                         void* stream);

/* LatentQuantize (latent_quantization.py "lq").  Tables: at most VQB_LQ_MAX_DIM latents and VQB_LQ_MAX_VALUES values in all,
 * staged in shared memory (VQB_E_UNSUPPORTED beyond). */
#define VQB_LQ_MAX_DIM 256
#define VQB_LQ_MAX_VALUES 8192
#define VQB_LQ_MAX_LOSS_BLOCKS 1024
/* z [N][C][D] contiguous in dtype (f32 or bf16), C codebooks sharing the D per-latent tables.  vals f32 [total]: the D tables
 * concatenated (any order, duplicates allowed); meta i32 [3][D] on the device: table lengths (summing to total), half widths
 * levels // 2, basis.  Per latent the first j minimising |z - vals_i[j]| in fp32 (a NaN distance is the minimum, as
 * torch.argmin), codes f32 [N][C][D] = z + (v - z), idx i32 [N][C] = int32(sum_i ((codes_i * 2) * hw_i + hw_i) * basis_i) in
 * fp32, each operation rounded separately, the sum left to right, truncated by cvt.rzi (NaN -> 0, saturating). */
int vqb_lq_quantize(const void* z, int dtype, int64_t N, int C, int D, const float* vals, int total, const int32_t* meta,
                    float* codes, int32_t* idx, void* stream);
/* The CTA count of vqb_lq_loss over n elements (the length of its partial array), or a VQB_E_* code.  Host-only. */
int vqb_lq_loss_blocks(int64_t n);
/* loss f32 [1] = w_c m_c + w_q m_q, m = mean over n of (x - out)^2 (x f32 or bf16, out f32, the same element order), a term's
 * m replaced by 0 unless its flag use_c / use_q (0 / 1) is set.  w_c, w_q: f32 [1] on the device.  partial f64 [blocks],
 * blocks = vqb_lq_loss_blocks(n).  Two launches, fp64 partials added in a fixed order, no atomics. */
int vqb_lq_loss(const void* x, int dtype, const float* out, int64_t n, const float* wc, const float* wq, int use_c, int use_q,
                double* partial, int blocks, float* loss, void* stream);
/* The loss's gradients for g_loss f32 [1] on the device: gx [n] in x's dtype = (2/n) (x - out) (w_q g) (0 without use_q) and
 * gout f32 [n] = (2/n) (out - x) (w_c g) (0 without use_c); either output may be NULL, not both.  One launch. */
int vqb_lq_loss_backward(const void* x, int dtype, const float* out, int64_t n, const float* g_loss, const float* wc,
                         const float* wq, int use_c, int use_q, void* gx, float* gout, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQB200_H */
