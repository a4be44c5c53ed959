// Finite scalar quantization: FSQ (finite_scalar_quantization.py, "fsq"), ResidualFSQ and GroupedResidualFSQ
// (residual_fsq.py, "rfsq").  Three row kernels, one thread per (row, group) item with its d values in registers:
//
//   fsq_forward_kernel   soft clamp (rfsq:193-195), then per stage q < n_active (rfsq:228-241): u = r / scale_q, the bound
//                        (fsq:147-157 or fsq:161-169) with or without the hard clamp, codes_to_indices (fsq:220-224),
//                        quantized = code * scale_q, r -= quantized, out += quantized; stages >= n_active write index -1.
//   fsq_backward_kernel  d out -> d z through the same chain as autograd takes it, recomputing every stage from z.
//   fsq_decode_kernel    indices -> sum_q code_q * scale_q (rfsq:131-171, fsq:209-218), the codes from the index digits.
//
// Every per-dimension constant (half_l, offset, shift, 2 / (L - 1), levels // 2, the basis, the stage scales, the soft-clamp
// value) is computed by the module with the reference's own torch expressions and passed in; the kernels repeat only the
// reference's per-element operations, in its order, with explicitly rounded intrinsics (no contraction).  `W` is the dtype the
// reference runs its outer chain in (the soft clamp, the scaling, the residual and the running sum); W = bf16 rounds after
// every such operation, as torch does for a bf16 tensor op.  Inside a stage the reference always works in fp32 (fsq:282-283).
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int FSQ_THREADS = 256;
constexpr int FSQ_CTAS_PER_SM = 16;   // grid cap
constexpr int FSQ_MAX_D = 16;
constexpr int FSQ_MAX_Q = 64;
constexpr int FSQ_BWD_SMEM = 96 * 1024;   // per-thread stage gradients of the backward (see fsq_backward_kernel)

// Rows of the fp32 constant table [FSQ_NCONST][D] (include/vqb200.h).
enum { C_A = 0, C_B = 1, C_SHIFT = 2, C_HW = 3, C_BASIS = 4, C_RB = 5, C_RHW = 6, FSQ_NCONST = 7 };

__device__ __forceinline__ float clamp1(float v) { return v != v ? v : fminf(fmaxf(v, -1.f), 1.f); }   // torch.clamp keeps NaN

struct Consts {   // the shared-memory copy of the module's constants
  float c[FSQ_NCONST][FSQ_MAX_D];
  float clampv[FSQ_MAX_D], rclamp[FSQ_MAX_D];
  int lev[FSQ_MAX_D];
  int basis[FSQ_MAX_D];
};

// scales f32 [2][Q][D] (values, reciprocals), clampv f32 [2][D] (value, reciprocal).
__device__ __forceinline__ void load_consts(Consts& k, float2* sc, const float* consts, const int32_t* ilev, const float* scales,
                                           const float* clampv, int D, int Q, int nq) {
  for (int i = threadIdx.x; i < FSQ_NCONST * D; i += blockDim.x) k.c[i / D][i % D] = consts[i];
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    k.clampv[i] = clampv ? clampv[i] : 1.f;
    k.rclamp[i] = clampv ? clampv[D + i] : 1.f;
    if (ilev) { k.lev[i] = ilev[i]; k.basis[i] = ilev[D + i]; }
  }
  if (scales)
    for (int i = threadIdx.x; i < nq * D; i += blockDim.x) sc[i] = make_float2(scales[i], scales[Q * D + i]);
  __syncthreads();
}

// One element of one stage, fp32 (fsq:282-292): the code and the value codes_to_indices multiplies by the basis.  `pre` is the
// input of the clamp / tanh (kept for the backward's mask), `h` its output.
struct Elt {
  float pre, h, code;
};

__device__ __forceinline__ Elt quantize_elt(float z, bool sym, bool hard, float a, float b, float shift) {
  Elt e;
  if (sym) {   // fsq:161-169: a = L - 1, b = 2 / (L - 1)
    e.pre = z;
    e.h = hard ? clamp1(z) : tanhf(z);
    // x / 2 and x * 0.5 are the same real number, so they round alike; the product avoids the division's slow path
    const float br = __fadd_rn(__fmul_rn(__fmul_rn(a, __fadd_rn(e.h, 1.f)), 0.5f), 0.5f);
    const float fl = __fadd_rn(br, __fsub_rn(floorf(br), br));   // floor_ste (fsq:57-60)
    e.code = __fsub_rn(__fmul_rn(b, fl), 1.f);
  } else {     // fsq:147-157: a = half_l, b = offset, hw = levels // 2 (divides below)
    e.pre = __fadd_rn(z, shift);
    e.h = hard ? clamp1(e.pre) : tanhf(e.pre);
    const float v = __fsub_rn(__fmul_rn(e.h, a), b);
    e.code = __fadd_rn(v, __fsub_rn(rintf(v), v));                // round_ste (fsq:52-55), round half to even
  }
  return e;
}

// d (stage input z) from d code, fp32, in autograd's order: sym  g * b, / 2, * (L - 1), then the clamp mask or the tanh backward;
// non-sym  / hw, * half_l, then the mask or the tanh backward.  torch's clamp passes the gradient on the closed interval.
__device__ __forceinline__ float quantize_elt_bwd(float g, const Elt& e, bool sym, bool hard, float a, float b, float hw, float rhw) {
  float gh = sym ? __fmul_rn(__fmul_rn(__fmul_rn(g, b), 0.5f), a) : __fmul_rn(divc(g, hw, rhw), a);
  if (hard) return (e.pre >= -1.f && e.pre <= 1.f) ? gh : 0.f;
  return __fmul_rn(gh, __fsub_rn(1.f, __fmul_rn(e.h, e.h)));
}

// The soft clamp (rfsq:193-195): x / c, tanh, * c, each rounded to W.  Returns the tanh output for the backward.
template <bool BF>
__device__ __forceinline__ float soft_clamp(float& x, float c, float rc) {
  const float t = rw<BF>(tanhf(rw<BF>(divc(x, c, rc))));
  x = rw<BF>(__fmul_rn(t, c));
  return t;
}

// One stage of one element: u = r / scale (W), the fp32 stage, the code rounded to W (codes.to(orig_dtype), fsq:301), then
// quantized = code * scale (W).  `scaled` is false for a plain FSQ (no scales, the code is the output).
template <bool BF>
__device__ __forceinline__ float stage_elt(float r, float2 sc, bool scaled, bool sym, bool hard, const Consts& k, int j, Elt* e_out,
                                           float* idx_term) {
  const float u = scaled ? rw<BF>(divc(r, sc.x, sc.y)) : r;
  Elt e = quantize_elt(u, sym, hard, k.c[C_A][j], k.c[C_B][j], k.c[C_SHIFT][j]);
  if (!sym) e.code = divc(e.code, k.c[C_HW][j], k.c[C_RHW][j]);
  if (e_out) *e_out = e;
  if (idx_term) {   // _scale_and_shift (fsq:195-200) times the basis
    const float s = sym ? divc(__fadd_rn(e.code, 1.f), k.c[C_B][j], k.c[C_RB][j]) : __fadd_rn(__fmul_rn(e.code, k.c[C_HW][j]), k.c[C_HW][j]);
    *idx_term = __fmul_rn(s, k.c[C_BASIS][j]);
  }
  const float cw = rw<BF>(e.code);
  return scaled ? rw<BF>(__fmul_rn(cw, sc.x)) : cw;
}

struct FsqArgs {
  const void* z;
  int64_t items;   // N * G
  int G, Q, n_active, sym, hard;
  const float* consts;
  const float* scales;   // [Q][D] or null
  const float* clampv;   // [D] or null
};

template <int DT, bool BF, int D>
__global__ void __launch_bounds__(FSQ_THREADS, 1) fsq_forward_kernel(FsqArgs a, void* __restrict__ out, void* __restrict__ idx, int idx64,
                                                                  int64_t s_row, int64_t s_g, int64_t s_q) {
  __shared__ Consts k;
  __shared__ float2 sc[FSQ_MAX_Q * FSQ_MAX_D];
  load_consts(k, sc, a.consts, nullptr, a.scales, a.clampv, D, a.Q, a.n_active);
  const bool scaled = a.scales != nullptr, soft = a.clampv != nullptr, sym = a.sym, hard = a.hard;
  constexpr int WT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < a.items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float r[D], o[D];
    load_item<DT, D>(a.z, it, r);
    if (soft) {
#pragma unroll
      for (int j = 0; j < D; ++j) soft_clamp<BF>(r[j], k.clampv[j], k.rclamp[j]);
    }
    const int64_t row = static_cast<uint32_t>(it) / static_cast<uint32_t>(a.G), g = it - row * a.G;   // items < 2^31
    const int64_t ibase = row * s_row + g * s_g;
    for (int q = 0; q < a.n_active; ++q) {
      float isum = 0.f;
#pragma unroll
      for (int j = 0; j < D; ++j) {
        float term;
        const float qv = stage_elt<BF>(r[j], scaled ? sc[q * D + j] : make_float2(1.f, 1.f), scaled, sym, hard, k, j, nullptr, &term);
        isum = __fadd_rn(isum, term);
        r[j] = rw<BF>(__fsub_rn(r[j], qv));   // rfsq:238
        o[j] = q == 0 ? qv : rw<BF>(__fadd_rn(o[j], qv));   // rfsq:239
      }
      store_index(idx, idx64, ibase + q * s_q, static_cast<int64_t>(rintf(isum)));   // .round().to(int32)
    }
    for (int q = a.n_active; q < a.Q; ++q) store_index(idx, idx64, ibase + q * s_q, -1);   // rfsq:223, :230-232
    store_item<WT, D>(out, it, o);
  }
}

// d z of the whole chain.  The input of stage q's residual receives d u_q / scale_q from the stage and the whole gradient of
// r_{q+1} (rfsq:238 subtracts a detached value), and autograd adds the two: d r_q = A_q + d r_{q+1}, a sum nested from the LAST
// stage.  The A_q of one item are parked in shared memory ([q][j][thread], conflict-free) between the forward pass over the
// stages and that reverse sum.  r0_lowp: the input is bf16 but the chain is fp32 and nothing promoted it before stage 0 (no
// soft clamp): autograd rounds both of r_0's gradients to bf16 before it adds them.
template <int DT, bool BF, int D>
__global__ void __launch_bounds__(FSQ_THREADS, 1) fsq_backward_kernel(FsqArgs a, const void* __restrict__ gout, void* __restrict__ gz,
                                                                   int r0_lowp) {
  __shared__ Consts k;
  __shared__ float2 sc[FSQ_MAX_Q * FSQ_MAX_D];
  extern __shared__ float park[];
  load_consts(k, sc, a.consts, nullptr, a.scales, a.clampv, D, a.Q, a.n_active);
  const bool scaled = a.scales != nullptr, soft = a.clampv != nullptr, sym = a.sym, hard = a.hard;
  constexpr int WT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  const int nt = blockDim.x, t = threadIdx.x;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(nt) + t; it < a.items; it += static_cast<int64_t>(gridDim.x) * nt) {
    float r[D], g[D];
    load_item<DT, D>(a.z, it, r);
    load_item<WT, D>(gout, it, g);
    if (soft) {
#pragma unroll
      for (int j = 0; j < D; ++j) soft_clamp<BF>(r[j], k.clampv[j], k.rclamp[j]);
    }
    for (int q = 0; q < a.n_active; ++q) {
#pragma unroll
      for (int j = 0; j < D; ++j) {
        const float2 s = scaled ? sc[q * D + j] : make_float2(1.f, 1.f);
        Elt e;
        const float qv = stage_elt<BF>(r[j], s, scaled, sym, hard, k, j, &e, nullptr);
        const float gc = scaled ? rw<BF>(__fmul_rn(g[j], s.x)) : g[j];                             // quantized = code * scale
        const float gu = rw<BF>(quantize_elt_bwd(gc, e, sym, hard, k.c[C_A][j], k.c[C_B][j], k.c[C_HW][j], k.c[C_RHW][j]));   // z.float()
        park[(q * D + j) * nt + t] = scaled ? rw<BF>(divc(gu, s.x, s.y)) : gu;                     // u = r / scale
        r[j] = rw<BF>(__fsub_rn(r[j], qv));
      }
    }
    float d[D], tc[D];
    if (soft) {   // the soft clamp's tanh again, from z (fewer live registers than keeping it across the stages)
      load_item<DT, D>(a.z, it, tc);
#pragma unroll
      for (int j = 0; j < D; ++j) tc[j] = soft_clamp<BF>(tc[j], k.clampv[j], k.rclamp[j]);
    }
    const int last = a.n_active - 1;
#pragma unroll
    for (int j = 0; j < D; ++j) {
      d[j] = park[(last * D + j) * nt + t];
      for (int q = last - 1; q >= 1; --q) d[j] = rw<BF>(__fadd_rn(park[(q * D + j) * nt + t], d[j]));
      if (last >= 1) {
        const float a0 = park[j * nt + t];
        d[j] = r0_lowp ? bf16_round(__fadd_rn(bf16_round(a0), bf16_round(d[j]))) : rw<BF>(__fadd_rn(a0, d[j]));
      }
      if (soft) {   // x = tanh(x / c) * c backward: * c, tanh_backward (g (1 - t^2)), / c
        const float c = k.clampv[j];
        const float gt = rw<BF>(__fmul_rn(d[j], c));
        const float ga = rw<BF>(__fmul_rn(gt, __fsub_rn(1.f, __fmul_rn(tc[j], tc[j]))));
        d[j] = rw<BF>(divc(ga, c, k.rclamp[j]));
      }
    }
    store_item<DT, D>(gz, it, d);
  }
}

// indices -> codes: digit k_j = (index // basis_j) % L_j (fsq:214-218), code = k * (2 / (L - 1)) - 1 (sym) or
// (k - hw) / hw (fsq:202-207), rounded to W (the module's implicit codebook dtype), times scale_q (W); index -1 gives zeros
// (rfsq:148-155).  out = the fp32 sum over the stages in stage order, rounded once to W (torch's sum accumulates in fp32);
// codes [Q][items][D] the scaled stage codes.
template <bool BF, int D>
__global__ void __launch_bounds__(FSQ_THREADS, 1) fsq_decode_kernel(FsqArgs a, const int32_t* __restrict__ ilev, const void* __restrict__ idx,
                                                                 int idx64, int64_t s_row, int64_t s_g, int64_t s_q, void* __restrict__ out,
                                                                 void* __restrict__ codes) {
  __shared__ Consts k;
  __shared__ float2 sc[FSQ_MAX_Q * FSQ_MAX_D];
  load_consts(k, sc, a.consts, ilev, a.scales, nullptr, D, a.Q, a.Q);
  const bool scaled = a.scales != nullptr, sym = a.sym;
  constexpr int WT = BF ? VQB_DTYPE_BF16 : VQB_DTYPE_F32;
  for (int64_t it = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; it < a.items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = static_cast<uint32_t>(it) / static_cast<uint32_t>(a.G), g = it - row * a.G;   // items < 2^31
    float acc[D];
#pragma unroll
    for (int j = 0; j < D; ++j) acc[j] = 0.f;
    for (int q = 0; q < a.Q; ++q) {
      const int64_t ix = load_index(idx, idx64, row * s_row + g * s_g + q * s_q);
      float v[D];
#pragma unroll
      for (int j = 0; j < D; ++j) {
        float c = 0.f;
        if (ix != -1) {
          // non-negative indices below 2^32 (codes_to_indices makes int32): C and Python division agree, 32-bit is exact
          const int lv = static_cast<int>((static_cast<uint32_t>(ix) / static_cast<uint32_t>(k.basis[j])) % static_cast<uint32_t>(k.lev[j]));
          if (sym) {
            c = __fsub_rn(__fmul_rn(static_cast<float>(lv), k.c[C_B][j]), 1.f);
          } else {
            const int hw = static_cast<int>(k.c[C_HW][j]);
            c = divc(static_cast<float>(lv - hw), k.c[C_HW][j], k.c[C_RHW][j]);
          }
          c = rw<BF>(c);
          if (scaled) c = rw<BF>(__fmul_rn(c, sc[q * D + j].x));
        }
        v[j] = c;
        acc[j] = __fadd_rn(acc[j], c);
      }
      if (codes) store_item<WT, D>(codes, q * a.items + it, v);
    }
    if (out) {
#pragma unroll
      for (int j = 0; j < D; ++j) acc[j] = rw<BF>(acc[j]);
      store_item<WT, D>(out, it, acc);
    }
  }
}

int fsq_check(const FsqArgs& a, int D, int in_dtype, int work_dtype) {
  if (!a.z || !a.consts || a.items <= 0 || a.G <= 0 || a.Q <= 0 || a.n_active < 1 || a.n_active > a.Q) return VQB_E_INVALID;
  if (D < 1 || D > FSQ_MAX_D || a.Q > FSQ_MAX_Q || a.items >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if ((in_dtype != VQB_DTYPE_F32 && in_dtype != VQB_DTYPE_BF16) || (work_dtype != VQB_DTYPE_F32 && work_dtype != VQB_DTYPE_BF16))
    return VQB_E_INVALID;
  if (in_dtype == VQB_DTYPE_F32 && work_dtype == VQB_DTYPE_BF16) return VQB_E_UNSUPPORTED;   // torch promotes to fp32
  if (!aligned(a.z, 16)) return VQB_E_ALIGN;
  return check_device();
}

}  // namespace
}  // namespace vqb

// The launches below cover the (input dtype, W) pairs torch can produce: (f32, f32), (bf16, f32), (bf16, bf16).

extern "C" int vqb_fsq_forward(const void* z, int in_dtype, int work_dtype, int64_t N, int G, int D, int Q, int n_active, int sym,
                               int hard, const float* consts, const float* scales, const float* clampv, void* out, void* idx,
                               int idx64, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, void* stream) {
  using namespace vqb;
  const FsqArgs a{z, N * G, G, Q, n_active, sym, hard, consts, scales, clampv};
  if (!out || !idx || N <= 0) return VQB_E_INVALID;
  if (const int rc = fsq_check(a, D, in_dtype, work_dtype)) return rc;
  if (!aligned(out, 16)) return VQB_E_ALIGN;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid = capped_grid(a.items, FSQ_THREADS, FSQ_CTAS_PER_SM);
  const bool bf_in = in_dtype == VQB_DTYPE_BF16, bf_w = work_dtype == VQB_DTYPE_BF16;
#define VQB_FSQ_FWD(DD)                                                                                                         \
  if (!bf_in) fsq_forward_kernel<VQB_DTYPE_F32, false, DD><<<grid, FSQ_THREADS, 0, s>>>(a, out, idx, idx64, idx_s_row, idx_s_g, idx_s_q);  \
  else if (!bf_w) fsq_forward_kernel<VQB_DTYPE_BF16, false, DD><<<grid, FSQ_THREADS, 0, s>>>(a, out, idx, idx64, idx_s_row, idx_s_g, idx_s_q); \
  else fsq_forward_kernel<VQB_DTYPE_BF16, true, DD><<<grid, FSQ_THREADS, 0, s>>>(a, out, idx, idx64, idx_s_row, idx_s_g, idx_s_q);
  VQB_SWITCH_D(VQB_FSQ_FWD)
#undef VQB_FSQ_FWD
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fsq_backward(const void* z, int in_dtype, int work_dtype, int64_t N, int G, int D, int Q, int n_active, int sym,
                                int hard, const float* consts, const float* scales, const float* clampv, const void* grad_out,
                                void* grad_z, void* stream) {
  using namespace vqb;
  const FsqArgs a{z, N * G, G, Q, n_active, sym, hard, consts, scales, clampv};
  if (!grad_out || !grad_z || N <= 0) return VQB_E_INVALID;
  if (const int rc = fsq_check(a, D, in_dtype, work_dtype)) return rc;
  if (!aligned(grad_out, 16) || !aligned(grad_z, 16)) return VQB_E_ALIGN;
  const int per_thread = n_active * D * static_cast<int>(sizeof(float));
  int threads = FSQ_THREADS;
  while (threads > 32 && threads * per_thread > FSQ_BWD_SMEM) threads -= 32;
  if (threads * per_thread > FSQ_BWD_SMEM) return VQB_E_UNSUPPORTED;
  const size_t smem = static_cast<size_t>(threads) * per_thread;
  const int r0_lowp = in_dtype == VQB_DTYPE_BF16 && work_dtype == VQB_DTYPE_F32 && !clampv && scales;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid = capped_grid(a.items, threads, FSQ_CTAS_PER_SM);
  const bool bf_in = in_dtype == VQB_DTYPE_BF16, bf_w = work_dtype == VQB_DTYPE_BF16;
#define VQB_FSQ_BWD_LAUNCH(DT, BF, DD)                                                                                   \
  {                                                                                                                      \
    auto kern = fsq_backward_kernel<DT, BF, DD>;                                                                         \
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FSQ_BWD_SMEM);               \
    if (e != cudaSuccess) return static_cast<int>(e);                                                                    \
    kern<<<grid, threads, smem, s>>>(a, grad_out, grad_z, r0_lowp);                                                      \
  }
#define VQB_FSQ_BWD(DD)                                                  \
  if (!bf_in) VQB_FSQ_BWD_LAUNCH(VQB_DTYPE_F32, false, DD)               \
  else if (!bf_w) VQB_FSQ_BWD_LAUNCH(VQB_DTYPE_BF16, false, DD)          \
  else VQB_FSQ_BWD_LAUNCH(VQB_DTYPE_BF16, true, DD)
  VQB_SWITCH_D(VQB_FSQ_BWD)
#undef VQB_FSQ_BWD
#undef VQB_FSQ_BWD_LAUNCH
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_fsq_decode(const void* idx, int idx64, int64_t idx_s_row, int64_t idx_s_g, int64_t idx_s_q, int64_t N, int G,
                              int D, int Q, int work_dtype, int sym, const float* consts, const int32_t* levels_basis,
                              const float* scales, void* out, void* codes, void* stream) {
  using namespace vqb;
  if (!idx || !consts || !levels_basis || (!out && !codes) || N <= 0 || G <= 0 || Q <= 0) return VQB_E_INVALID;
  if (D < 1 || D > FSQ_MAX_D || Q > FSQ_MAX_Q || N * G >= (int64_t{1} << 31)) return VQB_E_UNSUPPORTED;
  if (work_dtype != VQB_DTYPE_F32 && work_dtype != VQB_DTYPE_BF16) return VQB_E_INVALID;
  if ((out && !aligned(out, 16)) || (codes && !aligned(codes, 16))) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const FsqArgs a{nullptr, N * G, G, Q, Q, sym, 0, consts, scales, nullptr};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid = capped_grid(a.items, FSQ_THREADS, FSQ_CTAS_PER_SM);
  const bool bf_w = work_dtype == VQB_DTYPE_BF16;
#define VQB_FSQ_DEC(DD)                                                                                                          \
  if (!bf_w) fsq_decode_kernel<false, DD><<<grid, FSQ_THREADS, 0, s>>>(a, levels_basis, idx, idx64, idx_s_row, idx_s_g, idx_s_q, out, codes); \
  else fsq_decode_kernel<true, DD><<<grid, FSQ_THREADS, 0, s>>>(a, levels_basis, idx, idx64, idx_s_row, idx_s_g, idx_s_q, out, codes);
  VQB_SWITCH_D(VQB_FSQ_DEC)
#undef VQB_FSQ_DEC
  return static_cast<int>(cudaGetLastError());
}
