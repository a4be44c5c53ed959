// HierarchicalVQ (hierarchical_vq.py, "hvq"): the per-scale work around the shared search (hvq:133-147).  Six kernels, all
// fp32, one thread per output element in a grid-stride loop, no atomics (every backward is the adjoint in gather form, so a
// rerun gives the same bits):
//
//   hvq_pool_kernel        residual (B, D, H, W) NCHW -> rows (B, s, s, D) channel-last: ATen's adaptive average,
//                          window [floor(i H / s), ceil((i + 1) H / s)), summed row by row, then / kh / kw.
//   hvq_pool_bwd_kernel    g rows -> g residual: each pixel sums g / kh / kw over every window that contains it.
//   hvq_up_kernel          rows (B, s, s, D) -> q (B, D, H, W): bilinear, align_corners = False, ATen's source-index rule;
//                          a plain copy when (s, s) == (H, W) (the reference skips the interpolate, hvq:105).  Optionally
//                          writes recon + q and residual - q in the same pass (the identity phi).
//   hvq_up_bwd_kernel      (g_a - g_b) -> g rows: each source element sums its taps' weights times g over the outputs it feeds.
//   hvq_blend_kernel       q = (1 - r) up + r conv (hvq:25, no fma contraction), then recon + q and residual - q.
//   hvq_blend_bwd_kernel   g_q = g_recon - g_resid, g_up = (1 - r) g_q, g_conv = r g_q.
#include "vqb_common.cuh"
#include "row_io.cuh"

namespace vqb {
namespace {

constexpr int HVQ_THREADS = 256;
constexpr int HVQ_CTAS_PER_SM = 8;
constexpr int HVQ_MAX_SIDE = 1 << 16;   // H, W, s: window and tap arithmetic stays in int32

// ATen's adaptive window of output cell i of s over n inputs: [start, end)
__device__ __forceinline__ int win_start(int i, int n, int s) { return static_cast<int>((static_cast<int64_t>(i) * n) / s); }
__device__ __forceinline__ int win_end(int i, int n, int s) {
  return static_cast<int>((static_cast<int64_t>(i + 1) * n + s - 1) / s);
}

// ATen's bilinear source index (align_corners = False): src = max(scale (dst + 0.5) - 0.5, 0) with scale = in / out in fp32,
// the lower tap i0 = (int) src, the upper tap i0 + p (p = 0 at the last input), and the upper tap's weight lam.
struct Tap {
  int i0, p;
  float lam;
};
__device__ __forceinline__ Tap source_tap(float scale, int dst, int in) {
  float src = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  Tap t;
  t.i0 = static_cast<int>(src);
  t.p = t.i0 < in - 1 ? 1 : 0;
  t.lam = src - static_cast<float>(t.i0);
  return t;
}

// The outputs [lo, hi) whose taps can reach input index y: i0(dst) is non-decreasing in dst, so this is every dst with
// i0(dst) in {y - 1, y}; lo starts two outputs early against the fp32 rounding of the inverse, and the caller checks each tap.
__device__ __forceinline__ void tap_range(float scale, int y, int out, int* lo, int* hi) {
  int a = static_cast<int>(floorf((static_cast<float>(y) - 0.5f) / scale - 0.5f)) - 2;
  a = a < 0 ? 0 : a;
  int b = static_cast<int>(floorf((static_cast<float>(y) + 1.5f) / scale - 0.5f)) + 3;
  *lo = a;
  *hi = b > out ? out : b;
}

// ---- pool ----

__global__ void __launch_bounds__(HVQ_THREADS) hvq_pool_kernel(const float* __restrict__ x, int64_t B, int D, int H, int W,
                                                                int s, float* __restrict__ rows) {
  const int64_t n = B * s * s * D;
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(e % D);
    const int64_t cell = e / D;
    const int j = static_cast<int>(cell % s), i = static_cast<int>((cell / s) % s);
    const int64_t b = cell / (static_cast<int64_t>(s) * s);
    const int h0 = win_start(i, H, s), h1 = win_end(i, H, s), w0 = win_start(j, W, s), w1 = win_end(j, W, s);
    const float* p = x + ((b * D + d) * H) * W;
    float sum = 0.f;
    for (int h = h0; h < h1; ++h)
      for (int w = w0; w < w1; ++w) sum += p[static_cast<int64_t>(h) * W + w];
    rows[e] = sum / static_cast<float>(h1 - h0) / static_cast<float>(w1 - w0);
  }
}

__global__ void __launch_bounds__(HVQ_THREADS) hvq_pool_bwd_kernel(const float* __restrict__ g, int64_t B, int D, int H, int W,
                                                                    int s, float* __restrict__ gx) {
  const int64_t n = B * D * H * W;
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(e % W), h = static_cast<int>((e / W) % H);
    const int64_t bd = e / (static_cast<int64_t>(H) * W);
    const int d = static_cast<int>(bd % D);
    const int64_t b = bd / D;
    // the windows holding pixel h: start(i) <= h < end(i)  <=>  floor(h s / H) <= i <= floor(((h + 1) s - 1) / H)
    const int i0 = static_cast<int>((static_cast<int64_t>(h) * s) / H);
    const int i1 = min(s - 1, static_cast<int>((static_cast<int64_t>(h + 1) * s - 1) / H));
    const int j0 = static_cast<int>((static_cast<int64_t>(w) * s) / W);
    const int j1 = min(s - 1, static_cast<int>((static_cast<int64_t>(w + 1) * s - 1) / W));
    float acc = 0.f;
    for (int i = i0; i <= i1; ++i) {
      const float kh = static_cast<float>(win_end(i, H, s) - win_start(i, H, s));
      for (int j = j0; j <= j1; ++j) {
        const float kw = static_cast<float>(win_end(j, W, s) - win_start(j, W, s));
        acc += g[((b * s + i) * s + j) * D + d] / kh / kw;
      }
    }
    gx[e] = acc;
  }
}

// ---- upsample (+ the identity phi's residual update) ----

__global__ void __launch_bounds__(HVQ_THREADS) hvq_up_kernel(const float* __restrict__ rows, int64_t B, int D, int s, int H, int W,
                                                              float* __restrict__ q_out, const float* __restrict__ recon,
                                                              const float* __restrict__ resid, float* __restrict__ recon_out,
                                                              float* __restrict__ resid_out) {
  const int64_t n = B * D * H * W;
  const bool same = s == H && s == W;
  const float sh = static_cast<float>(s) / static_cast<float>(H), sw = static_cast<float>(s) / static_cast<float>(W);
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(e % W), h = static_cast<int>((e / W) % H);
    const int64_t bd = e / (static_cast<int64_t>(H) * W);
    const int d = static_cast<int>(bd % D);
    const int64_t b = bd / D;
    const float* src = rows + b * s * s * D + d;   // src[(y s + x) D]
    float v;
    if (same) {
      v = src[(static_cast<int64_t>(h) * s + w) * D];
    } else {
      const Tap th = source_tap(sh, h, s), tw = source_tap(sw, w, s);
      const float* r0 = src + static_cast<int64_t>(th.i0) * s * D;
      const float* r1 = r0 + static_cast<int64_t>(th.p) * s * D;
      const int64_t c0 = static_cast<int64_t>(tw.i0) * D, c1 = c0 + static_cast<int64_t>(tw.p) * D;
      const float h0l = 1.f - th.lam, w0l = 1.f - tw.lam;
      v = h0l * (w0l * r0[c0] + tw.lam * r0[c1]) + th.lam * (w0l * r1[c0] + tw.lam * r1[c1]);
    }
    if (q_out) q_out[e] = v;
    if (recon_out) recon_out[e] = __fadd_rn(recon ? recon[e] : 0.f, v);
    if (resid_out) resid_out[e] = __fsub_rn(resid[e], v);
  }
}

__global__ void __launch_bounds__(HVQ_THREADS) hvq_up_bwd_kernel(const float* __restrict__ ga, const float* __restrict__ gb,
                                                                  int64_t B, int D, int s, int H, int W, float* __restrict__ g_rows) {
  const int64_t n = B * s * s * D;
  const bool same = s == H && s == W;
  const float sh = static_cast<float>(s) / static_cast<float>(H), sw = static_cast<float>(s) / static_cast<float>(W);
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(e % D);
    const int64_t cell = e / D;
    const int x = static_cast<int>(cell % s), y = static_cast<int>((cell / s) % s);
    const int64_t b = cell / (static_cast<int64_t>(s) * s);
    const int64_t plane = (b * D + d) * static_cast<int64_t>(H) * W;
    auto grad = [&](int h, int w) {
      const int64_t o = plane + static_cast<int64_t>(h) * W + w;
      return ga ? (gb ? __fsub_rn(ga[o], gb[o]) : ga[o]) : -gb[o];
    };
    if (same) {
      g_rows[e] = grad(y, x);
      continue;
    }
    int hlo, hhi, wlo, whi;
    tap_range(sh, y, H, &hlo, &hhi);
    tap_range(sw, x, W, &wlo, &whi);
    float acc = 0.f;
    for (int h = hlo; h < hhi; ++h) {
      const Tap th = source_tap(sh, h, s);
      if (th.i0 > y) break;
      if (th.i0 + th.p < y) continue;
      for (int a = 0; a < 2; ++a) {
        if (th.i0 + a * th.p != y) continue;
        const float lh = a ? th.lam : 1.f - th.lam;
        for (int w = wlo; w < whi; ++w) {
          const Tap tw = source_tap(sw, w, s);
          if (tw.i0 > x) break;
          if (tw.i0 + tw.p < x) continue;
          const float g = grad(h, w);
          for (int c = 0; c < 2; ++c) {
            if (tw.i0 + c * tw.p != x) continue;
            acc += (lh * (c ? tw.lam : 1.f - tw.lam)) * g;
          }
        }
      }
    }
    g_rows[e] = acc;
  }
}

// ---- the blended phi's residual update ----

__global__ void __launch_bounds__(HVQ_THREADS) hvq_blend_kernel(const float* __restrict__ up, const float* __restrict__ conv,
                                                                 int64_t n, float a, float r, const float* __restrict__ recon,
                                                                 const float* __restrict__ resid, float* __restrict__ recon_out,
                                                                 float* __restrict__ resid_out) {
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float q = __fadd_rn(__fmul_rn(up[e], a), __fmul_rn(conv[e], r));   // (1 - r) * x + r * conv(x), hvq:25
    if (recon_out) recon_out[e] = __fadd_rn(recon ? recon[e] : 0.f, q);
    if (resid_out) resid_out[e] = __fsub_rn(resid[e], q);
  }
}

__global__ void __launch_bounds__(HVQ_THREADS) hvq_blend_bwd_kernel(const float* __restrict__ g_recon, const float* __restrict__ g_resid,
                                                                     int64_t n, float a, float r, float* __restrict__ g_up,
                                                                     float* __restrict__ g_conv) {
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < n; e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float gq = g_recon ? (g_resid ? __fsub_rn(g_recon[e], g_resid[e]) : g_recon[e]) : -g_resid[e];
    g_up[e] = __fmul_rn(gq, a);
    g_conv[e] = __fmul_rn(gq, r);
  }
}

// Shape checks shared by the entry points: sizes positive, sides within HVQ_MAX_SIDE, element counts below 2^40.
int check_shape(int64_t B, int D, int H, int W, int s) {
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0 || s <= 0) return VQB_E_INVALID;
  if (H > HVQ_MAX_SIDE || W > HVQ_MAX_SIDE || s > HVQ_MAX_SIDE) return VQB_E_UNSUPPORTED;
  const int64_t lim = int64_t{1} << 40;
  if (B * D > lim / (static_cast<int64_t>(H) * W) || B * D > lim / (static_cast<int64_t>(s) * s)) return VQB_E_UNSUPPORTED;
  return VQB_OK;
}

bool aligned4(const void* p) { return !p || aligned(p, 4); }

}  // namespace
}  // namespace vqb

extern "C" int vqb_hvq_pool(const float* x, int64_t B, int D, int H, int W, int s, float* rows, void* stream) {
  using namespace vqb;
  if (!x || !rows) return VQB_E_INVALID;
  if (const int rc = check_shape(B, D, H, W, s)) return rc;
  if (!aligned4(x) || !aligned4(rows)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(B * s * s * D, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_pool_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(x, B, D, H, W, s, rows);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_hvq_pool_backward(const float* g_rows, int64_t B, int D, int H, int W, int s, float* g_x, void* stream) {
  using namespace vqb;
  if (!g_rows || !g_x) return VQB_E_INVALID;
  if (const int rc = check_shape(B, D, H, W, s)) return rc;
  if (!aligned4(g_rows) || !aligned4(g_x)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(B * D * H * W, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_pool_bwd_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(g_rows, B, D, H, W, s, g_x);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_hvq_upsample(const float* rows, int64_t B, int D, int s, int H, int W, float* q, const float* recon,
                                const float* resid, float* recon_out, float* resid_out, void* stream) {
  using namespace vqb;
  if (!rows || (!q && !recon_out && !resid_out) || (resid_out && !resid)) return VQB_E_INVALID;
  if (const int rc = check_shape(B, D, H, W, s)) return rc;
  if (!aligned4(rows) || !aligned4(q) || !aligned4(recon) || !aligned4(resid) || !aligned4(recon_out) || !aligned4(resid_out))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(B * D * H * W, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_up_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(rows, B, D, s, H, W, q, recon, resid, recon_out,
                                                                             resid_out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_hvq_upsample_backward(const float* g_a, const float* g_b, int64_t B, int D, int s, int H, int W,
                                         float* g_rows, void* stream) {
  using namespace vqb;
  if ((!g_a && !g_b) || !g_rows) return VQB_E_INVALID;
  if (const int rc = check_shape(B, D, H, W, s)) return rc;
  if (!aligned4(g_a) || !aligned4(g_b) || !aligned4(g_rows)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const int grid = capped_grid(B * s * s * D, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_up_bwd_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(g_a, g_b, B, D, s, H, W, g_rows);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_hvq_blend_update(const float* up, const float* conv, int64_t n, double r, const float* recon,
                                    const float* resid, float* recon_out, float* resid_out, void* stream) {
  using namespace vqb;
  if (!up || !conv || n <= 0 || (!recon_out && !resid_out) || (resid_out && !resid)) return VQB_E_INVALID;
  if (n >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  if (!aligned4(up) || !aligned4(conv) || !aligned4(recon) || !aligned4(resid) || !aligned4(recon_out) || !aligned4(resid_out))
    return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  // torch's `python_float * tensor` multiplies by the scalar rounded to fp32
  const float a = static_cast<float>(1.0 - r), rf = static_cast<float>(r);
  const int grid = capped_grid(n, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_blend_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(up, conv, n, a, rf, recon, resid, recon_out,
                                                                                resid_out);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int vqb_hvq_blend_backward(const float* g_recon, const float* g_resid, int64_t n, double r, float* g_up, float* g_conv,
                                      void* stream) {
  using namespace vqb;
  if ((!g_recon && !g_resid) || !g_up || !g_conv || n <= 0) return VQB_E_INVALID;
  if (n >= (int64_t{1} << 40)) return VQB_E_UNSUPPORTED;
  if (!aligned4(g_recon) || !aligned4(g_resid) || !aligned4(g_up) || !aligned4(g_conv)) return VQB_E_ALIGN;
  if (const int rc = check_device()) return rc;
  const float a = static_cast<float>(1.0 - r), rf = static_cast<float>(r);
  const int grid = capped_grid(n, HVQ_THREADS, HVQ_CTAS_PER_SM);
  hvq_blend_bwd_kernel<<<grid, HVQ_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(g_recon, g_resid, n, a, rf, g_up, g_conv);
  return static_cast<int>(cudaGetLastError());
}
