// Multi-GPU EMA update over NVLink peer memory — the all-reduce of the batch statistics FUSED into the EMA kernels.
//
// The reference all-reduces cluster_size and embed_sum separately, twice per codebook per stage
// (vector_quantize_pytorch.py:603, :607), then lerps.  Round 1 packed them into one buffer and called ncclAllReduce
// between the statistics kernels and the EMA kernel: a latency-bound 1 MiB collective that also split the step's CUDA
// graph in three.  Here every rank's packed statistics live in SYMMETRIC memory (same allocation mapped into every
// peer's address space over NVLink / NVSwitch); after one cross-GPU barrier (flag writes with system-scope
// release / acquire) the EMA kernels of every rank read all R copies directly with peer loads and add them in rank
// order 0..R-1 — every rank performs the identical fp32 additions, so the replicas' codebooks stay bit-identical, and
// the whole step (search -> statistics -> barrier -> reduce + lerp + normalise + operand refresh) is ONE graph.  This file
// holds the barrier and checks the peer pointers; the EMA kernels (vq_ema.cu) are the ones of the single-GPU update, with
// the sum over the ranks as their statistics source.
//
// Protocol (per step, per rank): statistics kernels write my buffer[parity] -> peer_barrier -> apply kernels read every
// peer's buffer[parity].  The buffers are double-buffered by step parity: a rank may only overwrite buffer[parity]
// two steps later, i.e. after it has passed the NEXT step's barrier, which every peer reaches only after its reads
// of this step have completed (stream order).
#include "vqb_common.cuh"

namespace vqb {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct PeerFlags { uint32_t* f[MAX_PEERS]; };

// One CTA, one thread per peer.  epoch lives in device memory (a CUDA graph replays the same arguments every step).
// flags.f[r] is rank r's flag array (uint32[world]) in symmetric memory; slot s of it is written by rank s.
__global__ void peer_barrier_kernel(const PeerFlags flags, int rank, int world, uint32_t* epoch) {
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) s_epoch = *epoch + 1u;
  __syncthreads();
  const uint32_t e = s_epoch;
  const int p = threadIdx.x;
  if (p < world) {
    __threadfence_system();                 // everything this rank wrote before (its statistics) is visible system-wide
    st_release_sys(flags.f[p] + rank, e);     // "rank has arrived at barrier e", posted into every peer (and itself)
    const uint32_t* mine = flags.f[rank] + p;
    const long long t0 = clock64();
    while (static_cast<int32_t>(ld_acquire_sys(mine) - e) < 0) {
      if (clock64() - t0 > 20000000000ll) {  // ~10 s: a peer died; fail loudly instead of hanging the box
        printf("vqb200: peer barrier timeout (rank %d waiting for rank %d, epoch %u)\n", rank, p, e);
        __trap();
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *epoch = e;
}

}  // namespace vqb

using namespace vqb;

extern "C" int vqb_peer_barrier(void* const* peer_flags_host, int rank, int world, uint32_t* epoch_dev, void* stream) {
  if (!peer_flags_host || !epoch_dev || world < 1 || world > MAX_PEERS || rank < 0 || rank >= world) return VQB_E_INVALID;
  PeerFlags fl;
  for (int r = 0; r < MAX_PEERS; ++r) fl.f[r] = r < world ? static_cast<uint32_t*>(peer_flags_host[r]) : nullptr;
  for (int r = 0; r < world; ++r) if (!fl.f[r]) return VQB_E_INVALID;
  peer_barrier_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(fl, rank, world, epoch_dev);
  return static_cast<int>(cudaGetLastError());
}

// peer_stats_host: host array of `world` device pointers to the ranks' packed statistics; slice_offset in floats
int vqb::peer_stats(EmaStats* src, const void* const* peer_stats_host, int world, int64_t slice_offset) {
  if (!peer_stats_host || world < 1 || world > MAX_PEERS || slice_offset < 0 || (slice_offset & 3)) return VQB_E_INVALID;
  *src = EmaStats{};
  src->world = world;
  for (int r = 0; r < world; ++r) {
    if (!peer_stats_host[r] || (reinterpret_cast<uintptr_t>(peer_stats_host[r]) & 15)) return VQB_E_ALIGN;
    src->p[r] = static_cast<const float*>(peer_stats_host[r]) + slice_offset;
  }
  return VQB_OK;
}
