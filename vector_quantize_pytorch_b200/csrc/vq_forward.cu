// One-call composite of a VectorQuantize forward / one ResidualVQ stage.
//
// The Python glue used to issue ~10 ctypes calls + a dozen tiny torch ops per forward; at BASELINE config 2 the
// GPU work is ~0.5 ms and the host needed 1.6 ms to enqueue it.  vqb_vq_forward enqueues the whole chain
// (input staging -> tensor-core search with fused gather tail -> exact re-score -> EMA statistics -> EMA apply
// -> loss) from C++ in one call; the caller only provides outputs and one workspace.
#include "vqb_common.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>

using namespace vqb;

// Callers mirror these structs field for field (the ctypes stub of INTEGRATION.md, _C.py): their layout is part of the
// ABI and must not move.  Sizes on x86-64.
static_assert(sizeof(vqb_vq_forward_args) == 328, "vqb_vq_forward_args layout changed");
static_assert(sizeof(vqb_fused_outputs) == 104, "vqb_fused_outputs layout changed");
static_assert(sizeof(vqb_rvq_op) == 808, "vqb_rvq_op layout changed");

extern "C" int vqb_debug_active(void);  // vq_assign.cu: diagnostics (profile buffer / debug mode) are armed

namespace {
inline size_t up256(size_t v) { return (v + 255) / 256 * 256; }

struct FwdWs {
  size_t x_eff, a_planes, flagged, counters, stats_ws, idx_prov, total;
};

FwdWs carve_fwd(int64_t N, int D, int K, int dtype, int metric, int update) {
  FwdWs w;
  size_t off = 0;
  const size_t esz = dtype == VQB_DTYPE_BF16 ? 2 : 4;
  const bool cosine = metric == VQB_METRIC_COSINE;
  w.x_eff = off;
  if (cosine) off = up256(off + static_cast<size_t>(N) * D * esz);
  w.a_planes = off;
  if (dtype == VQB_DTYPE_F32) off = up256(off + static_cast<size_t>(2) * N * D * 2);
  w.flagged = off;
  off = up256(off + static_cast<size_t>(N) * sizeof(vqb_flag_entry));
  w.counters = off;  // [0..7] flag_count (int32) ; [8..15] loss_sum (double)
  off = up256(off + 16);
  w.stats_ws = off;
  if (update) off = up256(off + vqb_ema_stats_workspace(N, K));
  w.idx_prov = off;   // int32 [N]: search result with -1 for the rows that go through the exact re-score
  if (update) off = up256(off + static_cast<size_t>(N) * sizeof(int32_t));
  w.total = off;
  return w;
}
}  // namespace

extern "C" size_t vqb_vq_forward_workspace(int64_t N, int D, int K, int dtype, int metric, int update) {
  if (N <= 0 || D <= 0 || K <= 0) return 0;
  return carve_fwd(N, D, K, dtype, metric, update).total;
}

static int vq_forward_enqueue(const vqb_vq_forward_args* a, void* stream, int lane = 0);

// ---------------------------------------------------------------------------------------------
// CUDA-graph cache.  The chain is ~15 small launches around one big kernel; replaying it as a graph removes the
// launch gaps.  A call has a STRUCTURAL key (sizes, flags, which optional pointers are set, the stream: everything
// that decides the node topology) and a POINTER key.  Per structural key the cache keeps up to kVariants executable
// graphs, one per pointer set: torch's allocator cycles through a handful of blocks for the per-call outputs and the
// chunked host path uses one pointer set per chunk, so steady state is pure replay.  A pointer set that is not
// cached re-captures the chain (host-only, tens of microseconds) and patches the least recently used executable
// with cudaGraphExecUpdate instead of instantiating again — a miss never costs a GPU bubble, which is what made
// step times jump from 0.34 to 0.7+ ms whenever the allocator produced a new address combination mid-run.
// The first call of a structural key is enqueued directly (warms lazy module loading).  VQB_GRAPH=0 disables.
// Bypassed while profiling events are requested, or when the stream is already being captured
// (then the launches simply become part of the caller's graph).
// ---------------------------------------------------------------------------------------------
namespace {
constexpr int kKeyWords = 64;
constexpr int kVariants = 32;     // executable graphs per structural key
constexpr int kMaxStruct = 16;    // structural keys (LRU)
constexpr int kCaptureFailed = -2147483647;
struct Variant {
  uint64_t pkey[kKeyWords];
  cudaGraphExec_t exec;
  unsigned long long last_use;
};
struct StructEntry {
  uint64_t skey[kKeyWords];
  Variant var[kVariants];
  int n_var;
  unsigned long long last_use;
  bool used;
};
// ctypes releases the GIL around every call: two Python threads may enter vqb_vq_forward at once.  The cache (and the lazily
// created internal streams) are process-global, so one mutex serialises the cache lookup / capture / launch.
std::mutex g_cache_mutex;
StructEntry* g_struct = nullptr;  // [kMaxStruct], allocated on first use
unsigned long long g_tick = 0;
int g_graph_failures = 0;         // capture / instantiate / update failures: give up after a few
long long g_n_replay = 0, g_n_update = 0, g_n_instantiate = 0, g_n_direct = 0;  // vqb_debug_graph_stats
bool g_graph_disabled = false;

int graph_mode() {
  static int mode = -1;
  if (mode < 0) {
    const char* e = getenv("VQB_GRAPH");
    mode = (e && e[0] == '0') ? 0 : 1;
  }
  return mode;
}

void make_keys(const vqb_vq_forward_args* a, void* stream, uint64_t* sk, uint64_t* pk) {
  int si = 0, pi = 0;
  uint64_t present = 0;
  int nbit = 0;
  auto P = [&](const void* p) { pk[pi++] = reinterpret_cast<uint64_t>(p); present |= static_cast<uint64_t>(p != nullptr) << nbit++; };
  auto I = [&](long long v) { sk[si++] = static_cast<uint64_t>(v); };
  auto F = [&](double v) { uint64_t u; memcpy(&u, &v, 8); sk[si++] = u; };
  P(a->x); P(a->cluster_size); P(a->embed_avg); P(a->embed); P(a->planes); P(a->bext); P(a->bias); P(a->cnorm2); P(a->cmax);
  P(a->scratch); P(a->q_out); P(a->idx64_out); P(a->loss_out); P(a->resid_out); P(a->idx32); P(a->stats);
  P(a->workspace); P(a->a_planes_in); P(a->planes_out); P(a->row_mask); P(a->n_live);
  P(a->peer_epoch);
  for (int r = 0; r < a->peer_world && r < 16; ++r) { P(a->peer_stats ? a->peer_stats[r] : nullptr); P(a->peer_flags ? a->peer_flags[r] : nullptr); }
  I(a->dtype); I(a->metric); I(a->N); I(a->D); I(a->K); I(a->already_normalised); I(a->idx_stride); F(a->loss_weight);
  I(a->update); I(a->do_normalise); F(a->decay); F(a->eps); F(a->margin_rel);
  I(static_cast<long long>(a->workspace_bytes)); I(reinterpret_cast<long long>(stream)); I(static_cast<long long>(present));
  I(a->peer_rank); I(a->peer_world); I(a->peer_slice_offset);
  while (si < kKeyWords) sk[si++] = 0;
  while (pi < kKeyWords) pk[pi++] = 0;
}

// Side stream of the forward chain: the EMA sort runs on it, next to the exact re-score on the caller's stream.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork0 = nullptr, fork = nullptr, join = nullptr, counts = nullptr;
  bool ok = false;
};
constexpr int kLanes = 4;   // independent chains in flight inside one vqb_rvq_forward (the groups of GroupedResidualVQ)
SideStream* side_stream(int lane = 0) {
  static SideStream ss[kLanes];
  static bool tried[kLanes] = {false, false, false, false};
  static int dev = -1;
  if (lane < 0 || lane >= kLanes) return nullptr;
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (dev < 0) dev = cur;
  SideStream& s = ss[lane];
  if (!tried[lane]) {
    tried[lane] = true;
    s.ok = cur == dev && cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.fork0, cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&s.counts, cudaEventDisableTiming) == cudaSuccess;
    if (!s.ok) cudaGetLastError();
  }
  // one process drives one GPU (DESIGN.md section 5); a call on another device simply runs the chain in one stream
  return (s.ok && cur == dev) ? &s : nullptr;
}

// one line on stderr the first time the graph path is unavailable (the chain then runs launch by launch: same
// results, ~12 launches per forward instead of one)
void note_graph_error(const char* what, cudaError_t e) {
  static bool said = false;
  if (said) return;
  said = true;
  fprintf(stderr, "vqb200: %s failed (%s); vqb_vq_forward enqueues its kernels one by one on this stream\n", what,
          cudaGetErrorString(e));
}

// The chain is captured on an internal stream, never on the caller's: torch's default stream is the legacy stream,
// which CUDA refuses to capture ("operation not permitted when stream is capturing"), while an executable graph may
// be LAUNCHED into any stream.
cudaStream_t capture_stream() {
  static cudaStream_t cs = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    if (cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); cs = nullptr; }
  }
  return cs;
}

// A chain = a function that enqueues work on a stream (vq_forward_enqueue for one call, rvq_enqueue for a list of ops)
typedef int (*EnqueueFn)(const void* ctx, void* stream);

// capture the chain into a fresh graph (nothing executes)
int capture_chain(EnqueueFn fn, const void* ctx, cudaStream_t s, cudaGraph_t* out) {
  *out = nullptr;
  const cudaError_t be = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
  if (be != cudaSuccess) {  // e.g. the legacy default stream: CUDA does not capture it
    cudaGetLastError();
    note_graph_error("cudaStreamBeginCapture", be);
    return kCaptureFailed;
  }
  const int rc = fn(ctx, s);
  cudaGraph_t graph = nullptr;
  const cudaError_t ee = cudaStreamEndCapture(s, &graph);
  if (rc != VQB_OK || ee != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    if (rc == VQB_OK) note_graph_error("cudaStreamEndCapture", ee);
    return rc != VQB_OK ? rc : kCaptureFailed;
  }
  *out = graph;
  return VQB_OK;
}

// Serve one call of a chain from the cache (g_cache_mutex held).  sk / pk: structural and pointer key, kKeyWords each.
int run_cached(const uint64_t* sk, const uint64_t* pk, EnqueueFn fn, const void* ctx, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  constexpr size_t kKeyBytes = sizeof(uint64_t) * kKeyWords;
  if (!g_struct) {
    g_struct = static_cast<StructEntry*>(calloc(kMaxStruct, sizeof(StructEntry)));
    if (!g_struct) return fn(ctx, stream);
  }
  cudaStream_t cap_s = capture_stream();   // created here, outside any capture
  if (!cap_s) return fn(ctx, stream);
  ++g_tick;
  StructEntry* se = nullptr;
  for (int i = 0; i < kMaxStruct; ++i)
    if (g_struct[i].used && memcmp(g_struct[i].skey, sk, kKeyBytes) == 0) { se = &g_struct[i]; break; }
  if (!se) {  // first call of this structure: remember it, run directly
    int slot = 0;
    for (int i = 0; i < kMaxStruct; ++i) {
      if (!g_struct[i].used) { slot = i; break; }
      if (g_struct[i].last_use < g_struct[slot].last_use) slot = i;
    }
    se = &g_struct[slot];
    for (int v = 0; v < se->n_var; ++v)
      if (se->var[v].exec) cudaGraphExecDestroy(se->var[v].exec);
    memset(se, 0, sizeof(*se));
    memcpy(se->skey, sk, kKeyBytes);
    se->used = true;
    se->last_use = g_tick;
    return fn(ctx, stream);
  }
  se->last_use = g_tick;
  for (int v = 0; v < se->n_var; ++v)
    if (se->var[v].exec && memcmp(se->var[v].pkey, pk, kKeyBytes) == 0) {  // replay
      se->var[v].last_use = g_tick;
      ++g_n_replay;
      return static_cast<int>(cudaGraphLaunch(se->var[v].exec, s));
    }
  // New pointer set.  Instantiating an executable graph is the expensive step (it can synchronise with the device and
  // stall the whole launch queue), so a set earns its own executable only on its SECOND sighting ("pending" record);
  // until then the call is served by patching the least recently used executable in place.
  cudaGraph_t graph = nullptr;
  const int rc = capture_chain(fn, ctx, cap_s, &graph);
  if (rc != VQB_OK) {
    if (rc != kCaptureFailed) return rc;              // error reported by the chain itself (nothing ran)
    if (++g_graph_failures > 4) g_graph_disabled = true;
    ++g_n_direct;
    return fn(ctx, stream);                           // capture failed: nothing ran, enqueue directly
  }
  Variant* pend = nullptr;     // pending record of this pointer set
  Variant* donor = nullptr;    // least recently used executable
  Variant* spare = nullptr;    // free / least recently used pending record
  for (int v = 0; v < se->n_var; ++v) {
    Variant* q = &se->var[v];
    if (q->exec) { if (!donor || q->last_use < donor->last_use) donor = q; }
    else if (memcmp(q->pkey, pk, kKeyBytes) == 0) pend = q;
    else if (!spare || q->last_use < spare->last_use) spare = q;
  }
  if (se->n_var < kVariants) spare = &se->var[se->n_var];
  auto fail = [&]() {
    ++g_n_direct;
    cudaGetLastError();
    cudaGraphDestroy(graph);
    if (++g_graph_failures > 4) g_graph_disabled = true;
    return fn(ctx, stream);
  };
  Variant* use = nullptr;
  if (pend || !donor) {  // second sighting (or nothing to patch yet): instantiate
    use = pend ? pend : spare;
    if (!use) return fail();
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess || !exec) return fail();
    if (use == &se->var[se->n_var]) ++se->n_var;
    use->exec = exec;
    ++g_n_instantiate;
  } else {
    if (spare) {  // remember the sighting
      if (spare == &se->var[se->n_var]) ++se->n_var;
      memcpy(spare->pkey, pk, kKeyBytes);
      spare->exec = nullptr;
      spare->last_use = g_tick;
    }
    cudaGraphExecUpdateResultInfo info;
    if (cudaGraphExecUpdate(donor->exec, graph, &info) != cudaSuccess) {  // topology differs after all: rebuild it
      cudaGetLastError();
      cudaGraphExecDestroy(donor->exec);
      donor->exec = nullptr;
      if (cudaGraphInstantiate(&donor->exec, graph, 0) != cudaSuccess || !donor->exec) {
        donor->exec = nullptr;
        memset(donor->pkey, 0xFF, kKeyBytes);  // a pending record that matches nothing
        return fail();
      }
    }
    use = donor;
    ++g_n_update;
  }
  cudaGraphDestroy(graph);
  memcpy(use->pkey, pk, kKeyBytes);
  use->last_use = g_tick;
  return static_cast<int>(cudaGraphLaunch(use->exec, s));
}

bool graphs_usable(cudaStream_t s) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  return graph_mode() && !g_graph_disabled && !vqb_debug_active() && cudaStreamIsCapturing(s, &cap) == cudaSuccess &&
         cap == cudaStreamCaptureStatusNone;
}

int enqueue_one(const void* ctx, void* stream) { return vq_forward_enqueue(static_cast<const vqb_vq_forward_args*>(ctx), stream); }

// ---- a list of ops (vqb_rvq_forward) ----
struct RvqCtx { const vqb_rvq_op* ops; int n; };

struct LaneStreams {
  cudaStream_t stream[kLanes] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t begin = nullptr, done[kLanes] = {nullptr, nullptr, nullptr, nullptr};
  bool ok = false;
};
LaneStreams* lane_streams() {
  static LaneStreams ls;
  static bool tried = false;
  if (!tried) {
    tried = true;
    ls.ok = cudaEventCreateWithFlags(&ls.begin, cudaEventDisableTiming) == cudaSuccess;
    for (int l = 1; l < kLanes && ls.ok; ++l)
      ls.ok = cudaStreamCreateWithFlags(&ls.stream[l], cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&ls.done[l], cudaEventDisableTiming) == cudaSuccess;
    if (!ls.ok) cudaGetLastError();
  }
  return ls.ok ? &ls : nullptr;
}

int rvq_enqueue(const void* ctx, void* stream) {
  const RvqCtx* c = static_cast<const RvqCtx*>(ctx);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  bool used[kLanes] = {false, false, false, false};
  for (int i = 0; i < c->n; ++i) {
    if (c->ops[i].lane < 0 || c->ops[i].lane >= kLanes) return VQB_E_INVALID;
    used[c->ops[i].lane] = true;
  }
  LaneStreams* ls = (used[1] || used[2] || used[3]) ? lane_streams() : nullptr;
  cudaStream_t lane_s[kLanes] = {s, s, s, s};   // without lane streams everything runs in order on the caller's stream
  if (ls) {
    if (cudaEventRecord(ls->begin, s) != cudaSuccess) return static_cast<int>(cudaGetLastError());
    for (int l = 1; l < kLanes; ++l)
      if (used[l]) {
        if (cudaStreamWaitEvent(ls->stream[l], ls->begin, 0) != cudaSuccess) return static_cast<int>(cudaGetLastError());
        lane_s[l] = ls->stream[l];
      }
  }
  int rc = VQB_OK;
  for (int i = 0; i < c->n && rc == VQB_OK; ++i) {
    const vqb_rvq_op& op = c->ops[i];
    cudaStream_t os = lane_s[op.lane];
    if (op.kind == VQB_RVQ_STAGE) {
      rc = vq_forward_enqueue(&op.stage, os, ls ? op.lane : 0);
    } else if (op.kind == VQB_RVQ_EMA) {
      rc = ema_apply_part(3, local_stats(op.ema.stats), op.ema.cluster_size, op.ema.embed_avg, op.ema.embed, op.ema.K, op.ema.D,
                          op.ema.decay, op.ema.eps, op.ema.metric, op.ema.do_lerp ? (op.ema.n_lerp > 1 ? op.ema.n_lerp : 1) : 0,
                          op.ema.do_normalise, nullptr, op.ema.planes, op.ema.bext, op.ema.bias, op.ema.cnorm2, op.ema.cmax,
                          op.ema.scratch, os, op.ema.slice_stride);
    } else if (op.kind == VQB_RVQ_ACCUMULATE) {
      rc = vqb_rvq_accumulate(op.acc.embeds, op.acc.embed_stride, op.acc.Q, op.acc.K, op.acc.D, op.acc.idx, op.acc.N,
                              op.acc.out, op.acc.dtype, os);
    } else if (op.kind == VQB_RVQ_BARRIER) {
      rc = vqb_peer_barrier(op.bar.flags, op.bar.rank, op.bar.world, op.bar.epoch, os);
    } else if (op.kind == VQB_RVQ_EMA_PEERS) {
      EmaStats src;
      rc = peer_stats(&src, op.emap.peer_stats, op.emap.world, op.emap.slice_offset);
      if (rc == VQB_OK)
        rc = ema_apply_part(3, src, op.emap.cluster_size, op.emap.embed_avg, op.emap.embed, op.emap.K, op.emap.D, op.emap.decay,
                            op.emap.eps, op.emap.metric, op.emap.n_lerp > 1 ? op.emap.n_lerp : 1, op.emap.do_normalise, nullptr,
                            op.emap.planes, op.emap.bext, op.emap.bias, op.emap.cnorm2, op.emap.cmax, op.emap.scratch, os,
                            op.emap.slice_stride);
    } else if (op.kind == VQB_RVQ_SIMVQ_TAIL) {
      const auto& t = op.simvq;
      rc = vqb_rsimvq_tail(t.r, t.codes, t.idx, t.N, t.D, t.rotation, t.r_next, t.qsum, t.first, t.idx64_out, t.idx_stride,
                           t.loss_sum, t.loss_out, t.input_weight, t.weight, os);
    } else {
      rc = VQB_E_INVALID;
    }
  }
  if (ls) {  // join the lanes even after an error: a capture must not end with unjoined streams
    for (int l = 1; l < kLanes; ++l)
      if (used[l]) {
        if (cudaEventRecord(ls->done[l], ls->stream[l]) != cudaSuccess || cudaStreamWaitEvent(s, ls->done[l], 0) != cudaSuccess)
          if (rc == VQB_OK) rc = static_cast<int>(cudaGetLastError());
      }
  }
  return rc;
}

uint64_t hash_words(const uint64_t* w, int n, uint64_t seed) {
  uint64_t h = seed ^ 0x9E3779B97F4A7C15ull;
  for (int i = 0; i < n; ++i) {
    h ^= w[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h *= 0xFF51AFD7ED558CCDull;
    h ^= h >> 33;
  }
  return h;
}
}  // namespace

extern "C" int vqb_vq_forward(const vqb_vq_forward_args* a, void* stream) {
  if (!a) return VQB_E_INVALID;
  // the statistics always come from the counting sort, which writes `stats` whole: nothing accumulates onto it
  if (a->update && a->stats_accumulate) return VQB_E_UNSUPPORTED;
  // reserved: ResidualVQ rebuilds quantized_out from the indices (vqb_rvq_accumulate), the tail keeps no running sum
  if (a->qsum) return VQB_E_UNSUPPORTED;
  std::lock_guard<std::mutex> lock(g_cache_mutex);
  if (a->ev_search_begin || a->ev_search_end || !graphs_usable(static_cast<cudaStream_t>(stream)))
    return vq_forward_enqueue(a, stream);
  uint64_t sk[kKeyWords], pk[kKeyWords];
  make_keys(a, stream, sk, pk);
  return run_cached(sk, pk, enqueue_one, a, stream);
}

extern "C" int vqb_rvq_forward(const vqb_rvq_op* ops, int n_ops, void* stream) {
  if (!ops || n_ops <= 0 || n_ops > kKeyWords - 2) return VQB_E_INVALID;
  std::lock_guard<std::mutex> lock(g_cache_mutex);
  RvqCtx ctx{ops, n_ops};
  bool events = false;
  for (int i = 0; i < n_ops; ++i) {
    if (ops[i].kind != VQB_RVQ_STAGE) continue;
    if (ops[i].stage.update && ops[i].stage.stats_accumulate) return VQB_E_UNSUPPORTED;   // as in vqb_vq_forward
    if (ops[i].stage.qsum) return VQB_E_UNSUPPORTED;
    events |= ops[i].stage.ev_search_begin || ops[i].stage.ev_search_end;
  }
  if (events || !graphs_usable(static_cast<cudaStream_t>(stream))) return rvq_enqueue(&ctx, stream);
  // one key word per op: hashes of its structural words and of its pointers
  uint64_t sk[kKeyWords], pk[kKeyWords];
  memset(sk, 0, sizeof(sk));
  memset(pk, 0, sizeof(pk));
  for (int i = 0; i < n_ops; ++i) {
    const vqb_rvq_op& op = ops[i];
    uint64_t s1[kKeyWords], p1[kKeyWords];
    memset(s1, 0, sizeof(s1));
    memset(p1, 0, sizeof(p1));
    if (op.kind == VQB_RVQ_STAGE) {
      make_keys(&op.stage, nullptr, s1, p1);
    } else if (op.kind == VQB_RVQ_EMA) {
      const void* ptrs[] = {op.ema.cluster_size, op.ema.embed_avg, op.ema.embed, op.ema.stats, op.ema.planes, op.ema.bext,
                            op.ema.bias, op.ema.cnorm2, op.ema.cmax, op.ema.scratch};
      for (int j = 0; j < 10; ++j) p1[j] = reinterpret_cast<uint64_t>(ptrs[j]);
      s1[0] = op.ema.K; s1[1] = op.ema.D; s1[2] = op.ema.metric; s1[3] = op.ema.do_lerp; s1[4] = op.ema.do_normalise;
      memcpy(&s1[5], &op.ema.decay, 8); memcpy(&s1[6], &op.ema.eps, 8);
      s1[7] = static_cast<uint64_t>(op.ema.n_lerp); s1[8] = static_cast<uint64_t>(op.ema.slice_stride);
    } else if (op.kind == VQB_RVQ_BARRIER) {
      if (!op.bar.flags || op.bar.world < 1 || op.bar.world > 16) return VQB_E_INVALID;
      for (int r = 0; r < op.bar.world; ++r) p1[r] = reinterpret_cast<uint64_t>(op.bar.flags[r]);
      p1[16] = reinterpret_cast<uint64_t>(op.bar.epoch);
      s1[0] = op.bar.rank; s1[1] = op.bar.world;
    } else if (op.kind == VQB_RVQ_EMA_PEERS) {
      if (!op.emap.peer_stats || op.emap.world < 1 || op.emap.world > 16) return VQB_E_INVALID;
      const void* ptrs[] = {op.emap.cluster_size, op.emap.embed_avg, op.emap.embed, op.emap.planes, op.emap.bext,
                            op.emap.bias, op.emap.cnorm2, op.emap.cmax, op.emap.scratch};
      for (int j = 0; j < 9; ++j) p1[j] = reinterpret_cast<uint64_t>(ptrs[j]);
      for (int r = 0; r < op.emap.world; ++r) p1[16 + r] = reinterpret_cast<uint64_t>(op.emap.peer_stats[r]);
      s1[0] = op.emap.K; s1[1] = op.emap.D; s1[2] = op.emap.metric; s1[3] = op.emap.do_normalise; s1[4] = op.emap.world;
      s1[5] = static_cast<uint64_t>(op.emap.slice_offset);
      memcpy(&s1[6], &op.emap.decay, 8); memcpy(&s1[7], &op.emap.eps, 8);
      s1[8] = static_cast<uint64_t>(op.emap.n_lerp); s1[9] = static_cast<uint64_t>(op.emap.slice_stride);
    } else if (op.kind == VQB_RVQ_ACCUMULATE) {
      p1[0] = reinterpret_cast<uint64_t>(op.acc.embeds); p1[1] = reinterpret_cast<uint64_t>(op.acc.idx);
      p1[2] = reinterpret_cast<uint64_t>(op.acc.out);
      s1[0] = op.acc.embed_stride; s1[1] = op.acc.Q; s1[2] = op.acc.K; s1[3] = op.acc.D; s1[4] = op.acc.N; s1[5] = op.acc.dtype;
    } else if (op.kind == VQB_RVQ_SIMVQ_TAIL) {
      const auto& t = op.simvq;
      const void* ptrs[] = {t.r, t.codes, t.idx, t.r_next, t.qsum, t.idx64_out, t.loss_sum, t.loss_out};
      for (int j = 0; j < 8; ++j) p1[j] = reinterpret_cast<uint64_t>(ptrs[j]);
      s1[0] = static_cast<uint64_t>(t.N); s1[1] = t.D; s1[2] = t.rotation; s1[3] = t.first; s1[4] = static_cast<uint64_t>(t.idx_stride);
      s1[5] = t.loss_out != nullptr;   // the loss adds a memset and a kernel
      uint32_t wb[2];
      memcpy(&wb[0], &t.input_weight, 4); memcpy(&wb[1], &t.weight, 4);
      s1[6] = wb[0]; s1[7] = wb[1];
    } else {
      return VQB_E_INVALID;
    }
    sk[i] = hash_words(s1, kKeyWords, (static_cast<uint64_t>(op.kind) << 8) | static_cast<uint64_t>(op.lane));
    pk[i] = hash_words(p1, kKeyWords, 1);
  }
  sk[kKeyWords - 2] = static_cast<uint64_t>(n_ops) | (1ull << 40);   // never equal to a single-call key (word 62 is 0 there)
  sk[kKeyWords - 1] = reinterpret_cast<uint64_t>(stream);
  return run_cached(sk, pk, rvq_enqueue, &ctx, stream);
}

// diagnostics: how the graph cache served the calls so far {replayed, patched, instantiated, fell back after a failure}
extern "C" int vqb_debug_graph_stats(long long* out4) {
  if (!out4) return VQB_E_INVALID;
  out4[0] = g_n_replay; out4[1] = g_n_update; out4[2] = g_n_instantiate; out4[3] = g_n_direct;
  return VQB_OK;
}

static int vq_forward_enqueue(const vqb_vq_forward_args* a, void* stream, int lane) {
  if (!a || !a->x || !a->embed || !a->planes || !a->bext || !a->cnorm2 || !a->cmax || !a->idx32 || !a->workspace)
    return VQB_E_INVALID;
  if (a->N <= 0 || a->D <= 0 || a->K <= 0) return VQB_E_INVALID;
  if (a->dtype != VQB_DTYPE_F32 && a->dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if (a->update && (!a->stats)) return VQB_E_INVALID;
  if (a->update >= 2 && (!a->cluster_size || !a->embed_avg || !a->bias || !a->scratch)) return VQB_E_INVALID;
  if (a->update == 3 && (!a->peer_stats || !a->peer_flags || !a->peer_epoch || a->peer_world < 1 || a->peer_world > 16))
    return VQB_E_INVALID;
  if (a->update < 0 || a->update > 3) return VQB_E_INVALID;
  const FwdWs w = carve_fwd(a->N, a->D, a->K, a->dtype, a->metric, a->update);
  if (w.total > a->workspace_bytes) return VQB_E_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(a->workspace) & 255) return VQB_E_ALIGN;
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool cosine = a->metric == VQB_METRIC_COSINE;
  const bool l2 = cosine && !a->already_normalised;

  // ---- input staging (vqp:692, :1159 -> :376)
  const void* x_eff = a->x;
  const void* a_planes = a->x;
  int n_a = 1;
  int rc = VQB_OK;
  if (a->dtype == VQB_DTYPE_BF16) {
    if (l2) {
      rc = vqb_input_prepare(a->x, a->dtype, a->N, a->D, 1, ws + w.x_eff, nullptr, 0, stream);
      if (rc) return rc;
      x_eff = ws + w.x_eff;
      a_planes = x_eff;
    }
  } else if (a->a_planes_in && !l2) {
    // the previous ResidualVQ stage's tail already wrote the bf16 hi / lo split of these rows (planes_out)
    if (reinterpret_cast<uintptr_t>(a->a_planes_in) & 15) return VQB_E_ALIGN;
    a_planes = a->a_planes_in;
    n_a = 2;
  } else {
    rc = vqb_input_prepare(a->x, a->dtype, a->N, a->D, l2 ? 1 : 0, l2 ? ws + w.x_eff : nullptr, ws + w.a_planes, 2, stream);
    if (rc) return rc;
    if (l2) x_eff = ws + w.x_eff;
    a_planes = ws + w.a_planes;
    n_a = 2;
  }
  int32_t* flag_count = reinterpret_cast<int32_t*>(ws + w.counters);
  double* loss_sum = reinterpret_cast<double*>(ws + w.counters + 8);
  cudaError_t e = cudaSuccess;
  bool counters_zeroed = false;

  // ---- search with the fused gather / loss / residual tail (vqp:743-747, :766, :1178, :1327; rvq:524-525)
  vqb_fused_outputs f = {};
  f.x_eff = x_eff; f.embed = a->embed; f.q_out = a->q_out; f.idx64_out = a->idx64_out; f.idx_stride = a->idx_stride;
  f.loss_sum = a->loss_out ? loss_sum : nullptr;
  f.x_raw = (x_eff != a->x) ? a->x : nullptr;
  f.resid_out = a->resid_out; f.dtype = a->dtype;
  f.planes_out = (a->dtype == VQB_DTYPE_F32 && a->resid_out && !l2) ? a->planes_out : nullptr;
  if (a->planes_out && (a->dtype != VQB_DTYPE_F32 || !a->resid_out || l2)) return VQB_E_UNSUPPORTED;
  const bool want_tail = a->q_out || a->idx64_out || a->loss_out;
  // Masked batch (row_mask): padding rows keep their pre-filled outputs and leave loss and statistics alone (vq_assign.cu,
  // merge step).  Supported on the VectorQuantize chain: no ResidualVQ recurrence outputs.
  if (a->row_mask && (a->resid_out || a->planes_out)) return VQB_E_UNSUPPORTED;
  if (a->n_live && !a->row_mask) return VQB_E_INVALID;
  vqb_flag_entry* flagged = reinterpret_cast<vqb_flag_entry*>(ws + w.flagged);
  // The EMA sort (histogram -> scans -> scatter -> segmented sums) only needs the indices, and all but ~0.1 % of them
  // are final when the search kernel ends.  So the search also writes a provisional index array (-1 for the rows
  // it hands to the exact re-score) and counts the certified winners per slab of rows (the histogram of the counting
  // sort); the rest of the sort runs on a side stream NEXT TO the re-score; the few re-scored rows are added to the
  // (zero-initialised, accumulate-only) statistics by the main stream as soon as the code scan has written the cluster
  // sizes, and the cluster-size half of the EMA follows them there.  Only the row half of the EMA waits for the segmented
  // sums.  Critical path after the search: scan -> scatter -> sums -> EMA rows (was: hist -> colscan -> scan -> scatter ->
  // sums -> re-scored rows -> EMA sizes -> EMA rows).
  SideStream* side = a->update ? side_stream(lane) : nullptr;
  int32_t* idx_prov = side ? reinterpret_cast<int32_t*>(ws + w.idx_prov) : nullptr;
  const size_t stats_ws_bytes = a->update ? vqb_ema_stats_workspace(a->N, a->K) : 0;
  int32_t* hist = nullptr;
  int hist_shift = 0;
  if (side) {
    // ONE memset in front of the search: [flag / loss counters | sort ticket | slab histograms]; the statistics are zeroed
    // on the side stream, next to the search kernel (its CTAs leave room for a memset kernel on every SM)
    if (cudaEventRecord(side->fork0, s) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->fork0, 0) != cudaSuccess)
      return static_cast<int>(cudaGetLastError());
    static_assert(sizeof(vqb_flag_entry) == 32, "flag entry layout");
    rc = stats_begin(a->stats, a->dtype, a->N, a->D, a->K, ws + w.stats_ws, stats_ws_bytes, 1, w.stats_ws - w.counters, &hist,
                     &hist_shift, side->stream, stream);
    if (rc) return rc;
    counters_zeroed = true;
  }
  if (!counters_zeroed) {
    e = cudaMemsetAsync(ws + w.counters, 0, 16, s);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  if (a->ev_search_begin) cudaEventRecord(static_cast<cudaEvent_t>(a->ev_search_begin), s);
  rc = assign_launch(a_planes, n_a, a->N, a->D, a->planes, a->bext, a->cmax, a->K, a->margin_rel, 0, a->idx32, idx_prov,
                     hist, hist_shift, flagged, flag_count, nullptr, want_tail ? &f : nullptr, a->metric, a->cnorm2, stream,
                     a->row_mask);
  if (rc) return rc;
  if (a->ev_search_end) cudaEventRecord(static_cast<cudaEvent_t>(a->ev_search_end), s);
  if (side) {  // fork: certified rows -> statistics
    if (cudaEventRecord(side->fork, s) != cudaSuccess || cudaStreamWaitEvent(side->stream, side->fork, 0) != cudaSuccess)
      return static_cast<int>(cudaGetLastError());
    rc = stats_scan(idx_prov, a->dtype, a->N, a->D, a->K, a->stats, ws + w.stats_ws, stats_ws_bytes, 1, side->stream);
    const cudaError_t ce = cudaEventRecord(side->counts, side->stream);
    if (!rc) rc = stats_sum(x_eff, a->dtype, a->N, a->D, idx_prov, a->K, a->stats, ws + w.stats_ws, stats_ws_bytes, side->stream);
    const cudaError_t je = cudaEventRecord(side->join, side->stream);
    if (rc) return rc;
    if (ce != cudaSuccess || je != cudaSuccess) return static_cast<int>(cudaGetLastError());
  }
  rc = vqb_fix_flagged(x_eff, a->dtype, a->N, a->D, a->embed, a->cnorm2, a->K, a->metric, flagged, flag_count, a->idx32,
                       want_tail ? &f : nullptr, stream);
  if (rc) return rc;
  if (a->loss_out) {
    rc = loss_finalize_launch(loss_sum, a->N * a->D, a->row_mask ? a->n_live : nullptr, a->D, a->dtype, a->loss_weight, a->loss_out,
                              stream);
    if (rc) return rc;
  }
  // ---- EMA (vqp:586-617, :576-584).  update 3 (multi-GPU): every rank sums all ranks' statistics inside its EMA kernels, after a
  // barrier
  EmaStats src = local_stats(a->stats);
  if (a->update == 3) {
    rc = peer_stats(&src, a->peer_stats, a->peer_world, a->peer_slice_offset);
    if (rc) return rc;
  }
  auto ema = [&](int part) {
    return ema_apply_part(part, src, a->cluster_size, a->embed_avg, a->embed, a->K, a->D, a->decay, a->eps, a->metric, 1,
                          a->do_normalise, nullptr, a->planes, a->bext, a->bias, a->cnorm2, a->cmax, a->scratch, stream);
  };
  if (side) {  // the re-scored rows join the statistics of the certified ones (cluster sizes are in place after the scan)
    if (cudaStreamWaitEvent(s, side->counts, 0) != cudaSuccess) return static_cast<int>(cudaGetLastError());
    rc = stats_add_flagged(x_eff, a->dtype, a->N, a->D, flagged, flag_count, a->idx32, a->K, a->stats, stream);
    if (rc) return rc;
    if (a->update >= 2) {
      // cluster-size half of the EMA: does not need the row sums.  Multi-GPU: a first barrier as soon as this rank's COUNTS are
      // complete — it absorbs the skew between the ranks while the segmented sums still run
      if (a->update == 3) {
        rc = vqb_peer_barrier(a->peer_flags, a->peer_rank, a->peer_world, a->peer_epoch, stream);
        if (rc) return rc;
      }
      rc = ema(1);
      if (rc) return rc;
    }
    if (cudaStreamWaitEvent(s, side->join, 0) != cudaSuccess) return static_cast<int>(cudaGetLastError());
  } else if (a->update) {  // no side stream for this lane: the whole sort on the caller's stream
    rc = vqb_ema_stats(x_eff, a->dtype, a->N, a->D, a->idx32, a->K, a->stats, ws + w.stats_ws, stats_ws_bytes, stream);
    if (rc) return rc;
  }
  if (a->update < 2) return VQB_OK;
  if (a->update == 3) {
    rc = vqb_peer_barrier(a->peer_flags, a->peer_rank, a->peer_world, a->peer_epoch, stream);
    if (rc) return rc;
  }
  return ema(side ? 2 : 3);
}
