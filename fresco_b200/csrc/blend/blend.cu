// B1: the propagation stage's frame blending (video_blend.py:172-255 with blender/histogram_blend.py and
// blender/poisson_fusion.py): error masks and their nearest-warp propagation, the histogram blend in cv2's 8-bit Lab,
// and the Poisson gradient fusion solved to the exact least-squares solution by a Chebyshev iteration in fp64.
//
// Every kernel handles all frames of a sequence (and all three Lab channels) per launch; only the mask chain is
// launched once per frame, because frame k's propagated mask needs frame k-1's whole mask.  Colour conversion is a
// gather from 2^24-entry lookup tables the caller builds (cv2's own conversion on every triple), so it is cv2's bit for
// bit.  Where the reference's arithmetic is reproduced bit for bit (masks, histogram), every operation is an explicit
// _rn intrinsic, so nvcc cannot contract a multiply and an add into an FMA that numpy / torch do not use.
#include <cmath>

#include "../fresco_internal.h"

namespace fresco {
namespace {

constexpr int kStatBlocks = 64;    // partial sums per frame: a fixed grid, so the summation tree never changes
constexpr int kStatThreads = 256;
constexpr int kStatQ = 9;          // quantities per statistics pass (3 images x 3 channels at most)
constexpr int kStats = 24;         // per frame: mean a, b, e | std a, b, e | mean ab | std ab (3 channels each)
constexpr int kMaxCheby = 4096;

inline unsigned grid_1d(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

__global__ void blend_lut_gather_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ lut,
                                        uint8_t* __restrict__ out, long long pixels) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= pixels) return;
  const uint8_t* s = in + 3 * p;
  const uint8_t* t = lut + 3 * (((uint32_t)s[0] << 16) | ((uint32_t)s[1] << 8) | s[2]);
  const uint8_t c0 = t[0], c1 = t[1], c2 = t[2];
  out[3 * p] = c0;
  out[3 * p + 1] = c1;
  out[3 * p + 2] = c2;
}

// One step of the mask chain (video_blend.py:40-58, 223-228).  Step k: the error mask of frame k with
// weight1 = k / (interval - 1), OR (k > 0) the previous frame's final mask warped by frame k's backward flow with torch's
// CPU grid_sample (nearest, align_corners=True, zero padding): x = j + fx; xn = 2 x / (W-1) - 1;
// ix = rint((xn + 1) * ((W-1) / 2)), the vectorised kernel's unnormalize, in fp32 and torch's order.
__global__ void blend_mask_step_kernel(const float* __restrict__ dist1, const float* __restrict__ dist2,
                                       const float* __restrict__ flow, const uint8_t* __restrict__ prev,
                                       uint8_t* __restrict__ mask, int h, int w, double weight1, double weight2) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  uint8_t m = __dmul_rn(weight1, (double)dist1[p]) < __dmul_rn(weight2, (double)dist2[p]) ? 0 : 1;
  if (weight1 == 0.0) m = 0;
  else if (weight2 == 0.0) m = 1;
  if (prev != nullptr) {
    const int i = p / w, j = p - i * w;
    const float x = __fadd_rn((float)j, flow[p]);
    const float y = __fadd_rn((float)i, flow[h * w + p]);
    const float xn = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, x), (float)(w - 1)), 1.f);
    const float yn = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, y), (float)(h - 1)), 1.f);
    const float xs = rintf(__fmul_rn(__fadd_rn(xn, 1.f), (float)(w - 1) / 2.f));
    const float ys = rintf(__fmul_rn(__fadd_rn(yn, 1.f), (float)(h - 1) / 2.f));
    // comparisons in float: NaN and values past the int range fail them, as torch's int conversion sends them out of
    // bounds
    if (xs > -1.f && xs < (float)w && ys > -1.f && ys < (float)h) m |= prev[(int)ys * w + (int)xs];
  }
  mask[p] = m;
}

struct HistArgs {
  const uint8_t* a;       // Lab [F, hw, 3]
  const uint8_t* b;
  const uint8_t* e;       // min-error Lab image, or null: select a / b by mask
  const uint8_t* mask;    // [F, hw] (used when e is null)
  const double* weights;  // [F, 2]: the weights blend() multiplies a and b by
  double* partial;        // [F, kStatBlocks, kStatQ]
  double* stats;          // [F, kStats]
  uint8_t* out;           // Lab [F, hw, 3]
  int hw;
};

__device__ __forceinline__ uint8_t min_error_px(const HistArgs& A, long long f, int p, int c) {
  const long long o = f * A.hw + p;
  if (A.e) return A.e[3 * o + c];
  return A.mask[o] ? A.b[3 * o + c] : A.a[3 * o + c];
}

// histogram_transform of blend() for a and b: (x - mean) * fp32(256/36) / std + 128 in fp64, x an integer
__device__ __forceinline__ double to_target(uint8_t x, double mean, double std_) {
  const double t_std = (double)(float)((1.0 / 36.0) * 256.0);
  return __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn((double)x, mean), t_std), std_), 128.0);
}

// blend()'s ab before its final transform: ((a w1 + b w2) - 128) / 0.5 + 128
__device__ __forceinline__ double ab_px(const HistArgs& A, const double* st, double w1, double w2, long long f, int p,
                                        int c) {
  const long long o = 3 * (f * A.hw + p) + c;
  const double ta = to_target(A.a[o], st[c], st[9 + c]);
  const double tb = to_target(A.b[o], st[3 + c], st[12 + c]);
  return __dadd_rn(__ddiv_rn(__dsub_rn(__dadd_rn(__dmul_rn(ta, w1), __dmul_rn(tb, w2)), 128.0), 0.5), 128.0);
}

// One statistics pass over every frame: PASS 0 sums a, b, e; 1 sums (x - mean)^2 of a, b, e; 2 sums ab; 3 sums
// (ab - mean)^2.  Each thread walks a fixed pixel set, the block reduces by a fixed tree: deterministic.
template <int PASS>
__global__ void __launch_bounds__(kStatThreads) blend_hist_stats_kernel(HistArgs A) {
  constexpr int NQ = PASS < 2 ? 9 : 3;
  __shared__ double red[kStatThreads];
  const long long f = blockIdx.y;
  const double* st = A.stats + f * kStats;
  const double w1 = A.weights[2 * f], w2 = A.weights[2 * f + 1];
  double acc[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) acc[q] = 0.0;
  for (int p = blockIdx.x * kStatThreads + threadIdx.x; p < A.hw; p += kStatBlocks * kStatThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (PASS < 2) {
        const long long o = 3 * (f * A.hw + p) + c;
        const double v[3] = {(double)A.a[o], (double)A.b[o], (double)min_error_px(A, f, p, c)};
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          if (PASS == 0) {
            acc[3 * s + c] = __dadd_rn(acc[3 * s + c], v[s]);
          } else {
            const double d = __dsub_rn(v[s], st[3 * s + c]);
            acc[3 * s + c] = __dadd_rn(acc[3 * s + c], __dmul_rn(d, d));
          }
        }
      } else {
        const double ab = ab_px(A, st, w1, w2, f, p, c);
        if (PASS == 2) {
          acc[c] = __dadd_rn(acc[c], ab);
        } else {
          const double d = __dsub_rn(ab, st[18 + c]);
          acc[c] = __dadd_rn(acc[c], __dmul_rn(d, d));
        }
      }
    }
  }
  double* out = A.partial + (f * kStatBlocks + blockIdx.x) * kStatQ;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    red[threadIdx.x] = acc[q];
    __syncthreads();
    for (int s = kStatThreads / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x == 0) out[q] = red[0];
    __syncthreads();
  }
}

// Sums a pass's partials in block order and turns them into means (passes 0, 2) or stds (1, 3) as numpy does:
// mean = S / n, std = sqrt(S2 / n).  One block per frame, one thread per quantity.
template <int PASS>
__global__ void blend_hist_moments_kernel(HistArgs A) {
  constexpr int NQ = PASS < 2 ? 9 : 3;
  const int q = threadIdx.x;
  if (q >= NQ) return;
  const long long f = blockIdx.x;
  const double* part = A.partial + f * kStatBlocks * kStatQ;
  double s = 0.0;
  for (int b = 0; b < kStatBlocks; ++b) s = __dadd_rn(s, part[b * kStatQ + q]);
  s = __ddiv_rn(s, (double)A.hw);
  const int slot = PASS == 0 ? q : PASS == 1 ? 9 + q : PASS == 2 ? 18 + q : 21 + q;
  A.stats[f * kStats + slot] = (PASS & 1) ? __dsqrt_rn(s) : s;
}

// blend()'s last transform: ab cast to fp32, (x - mean_ab) * std_e / std_ab + mean_e in fp64, round half to even,
// clip to [0, 255]
__global__ void blend_hist_apply_kernel(HistArgs A, long long pixels) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= pixels) return;
  const long long f = g / A.hw;
  const int p = (int)(g - f * A.hw);
  const double* st = A.stats + f * kStats;
  const double w1 = A.weights[2 * f], w2 = A.weights[2 * f + 1];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double x = (double)(float)ab_px(A, st, w1, w2, f, p, c);
    const double y = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(x, st[18 + c]), st[15 + c]), st[21 + c]), st[6 + c]);
    A.out[3 * g + c] = (uint8_t)fmin(fmax(rint(y), 0.0), 255.0);
  }
}

// Right-hand side of the Poisson normal equations M u = b, M = w^2 (Gx^T Gx + Gy^T Gy) + I, per channel plane:
// b = im + w^2 (gx[i,j] - gx[i-1,j] + gy[i,j] - gy[i,j-1]), g the forward differences of a (mask 0) or b (mask 1),
// clipped to +-100, zero on the last row (gx) / column (gy).  Both iterate buffers start at im.
__global__ void blend_poisson_rhs_kernel(const uint8_t* __restrict__ tgt, const uint8_t* __restrict__ la,
                                         const uint8_t* __restrict__ lb, const uint8_t* __restrict__ mask,
                                         double* __restrict__ rhs, double* __restrict__ x0, double* __restrict__ x1,
                                         int h, int w, double w2_0, double w2_1, double w2_2, long long pixels) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= pixels) return;
  const int hw = h * w;
  const long long f = g / hw;
  const int p = (int)(g - f * hw);
  const int i = p / w, j = p - i * w;
  const long long base = f * hw;
  auto grad = [&](int q, int dq, int c) -> double {   // clip(I[q] - I[q + dq], +-100) from the image mask[q] picks
    const uint8_t* im = mask[base + q] ? lb : la;
    const double d = (double)im[3 * (base + q) + c] - (double)im[3 * (base + q + dq) + c];
    return fmin(fmax(d, -100.0), 100.0);
  };
  const double w2[3] = {w2_0, w2_1, w2_2};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double div = 0.0;
    if (i < h - 1) div += grad(p, w, c);
    if (i > 0) div -= grad(p - w, w, c);
    if (j < w - 1) div += grad(p, 1, c);
    if (j > 0) div -= grad(p - 1, 1, c);
    const double im = (double)tgt[3 * g + c];
    const long long o = (f * 3 + c) * hw + p;
    rhs[o] = im + w2[c] * div;
    x0[o] = im;
    x1[o] = im;
  }
}

struct ChebyStep {
  double omega[3];      // 2 sigma T_k(sigma) / T_{k+1}(sigma)  (1 on the first step)
  double inv_theta[3];  // 2 / (lambda_max + lambda_min)
  double w2[3];
  int active[3];        // this step is below the channel's iteration count
};

// One Chebyshev step on every (frame, channel) plane: y_next = omega (y - y_prev + (b - M y) / theta) + y_prev,
// written over y_prev.  M y = y + w^2 L y, L the 5-point Neumann Laplacian.
template <typename T>
__device__ __forceinline__ T pick3(const T (&v)[3], int c) {   // selects, not a local-memory index
  return c == 0 ? v[0] : c == 1 ? v[1] : v[2];
}

__global__ void blend_cheby_kernel(const double* __restrict__ cur, double* __restrict__ prev,
                                   const double* __restrict__ rhs, int h, int w, ChebyStep s) {
  const int c = blockIdx.y % 3;
  if (!pick3(s.active, c)) return;
  const int hw = h * w;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  const long long o = (long long)blockIdx.y * hw + p;
  const int i = p / w, j = p - i * w;
  const double y = cur[o];
  double lap = 0.0;
  if (i > 0) lap += y - cur[o - w];
  if (i < h - 1) lap += y - cur[o + w];
  if (j > 0) lap += y - cur[o - 1];
  if (j < w - 1) lap += y - cur[o + 1];
  const double r = rhs[o] - (y + pick3(s.w2, c) * lap);
  const double yp = prev[o];
  prev[o] = pick3(s.omega, c) * (y - yp + pick3(s.inv_theta, c) * r) + yp;
}

// clip(u, 0, 255) truncated to uint8 (poisson_fusion.py:91-93); the fp64 solution too when `solution` is given
__global__ void blend_poisson_finalize_kernel(const double* __restrict__ x0, const double* __restrict__ x1,
                                              uint8_t* __restrict__ out, double* __restrict__ solution, int hw,
                                              int odd0, int odd1, int odd2, long long pixels) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= pixels) return;
  const long long f = g / hw;
  const int p = (int)(g - f * hw);
  const int odd[3] = {odd0, odd1, odd2};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const long long o = (f * 3 + c) * hw + p;
    const double u = odd[c] ? x1[o] : x0[o];
    if (solution) solution[o] = u;
    out[3 * g + c] = (uint8_t)fmin(fmax(u, 0.0), 255.0);
  }
}

struct BlendWorkspace {
  double* partial;
  double* stats;
  double* rhs;
  double* x0;
  double* x1;
};

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

size_t hist_bytes(long long frames) {
  return align256(sizeof(double) * frames * kStatBlocks * kStatQ) + align256(sizeof(double) * frames * kStats);
}

size_t plane_bytes(long long frames, long long hw) { return align256(sizeof(double) * frames * 3 * hw); }

// spectrum of M = I + w^2 (L_h (x) I + I (x) L_w): [1, 1 + w^2 (4 sin^2(pi (h-1) / 2h) + 4 sin^2(pi (w-1) / 2w))]
double lambda_max(int h, int w, double weight) {
  const double sh = sin(M_PI * (h - 1) / (2.0 * h)), sw = sin(M_PI * (w - 1) / (2.0 * w));
  return 1.0 + weight * weight * (4.0 * sh * sh + 4.0 * sw * sw);
}

}  // namespace
}  // namespace fresco

using namespace fresco;

extern "C" size_t fresco_blend_workspace_bytes(int frames, int h, int w) {
  if (frames <= 0 || h <= 0 || w <= 0) return 0;
  return hist_bytes(frames) + 3 * plane_bytes(frames, (long long)h * w);
}

extern "C" int fresco_blend_cheby_iterations(int h, int w, double weight) {
  // oracle/blend_bound.py derives this count: the initial error u* - im = w^2 M^-1 G^T (g - G im) has 2-norm at most
  // (|w| / 2) 355 sqrt(edges) (|g| <= 100, |G im| <= 255, ||w^2 M^-1 G^T|| <= |w| / 2), and Chebyshev on
  // [1, lambda_max] divides the error by T_k(sigma); the count makes that at most 5e-4.
  if (h <= 0 || w <= 0) return -1;
  const double edges = (double)(h - 1) * w + (double)h * (w - 1);
  const double lmax = lambda_max(h, w, weight);
  if (edges == 0.0 || weight == 0.0 || lmax <= 1.0) return 0;
  const double e0 = 0.5 * fabs(weight) * 355.0 * sqrt(edges);
  const double sigma = (lmax + 1.0) / (lmax - 1.0);
  const double need = acosh(e0 / 5e-4);
  int k = (int)ceil(need / acosh(sigma));
  return k < 0 ? 0 : k;
}

extern "C" int fresco_blend_lut_gather(const uint8_t* in, const uint8_t* lut, uint8_t* out, long long pixels,
                                       void* stream) {
  if (!in || !lut || !out) return set_error(FRESCO_ERR_ARG, "fresco_blend_lut_gather: null pointer");
  if (pixels <= 0) return set_error(FRESCO_ERR_ARG, "fresco_blend_lut_gather: bad pixel count");
  blend_lut_gather_kernel<<<grid_1d(pixels, 256), 256, 0, (cudaStream_t)stream>>>(in, lut, out, pixels);
  return check_launch("blend_lut_gather_kernel");
}

extern "C" int fresco_blend_mask_chain(const float* dist1, const float* dist2, const float* flows, uint8_t* masks,
                                       int interval, int h, int w, void* stream) {
  if (!dist1 || !dist2 || !masks || (!flows && interval > 2))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_mask_chain: null pointer");
  if (interval < 2 || h <= 0 || w <= 0 || (long long)h * w > (1LL << 30))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_mask_chain: bad shape");
  const int hw = h * w;
  for (int k = 0; k < interval - 1; ++k) {
    const double w1 = (double)k / (double)(interval - 1);
    const double w2 = 1.0 - w1;
    blend_mask_step_kernel<<<grid_1d(hw, 256), 256, 0, (cudaStream_t)stream>>>(
        dist1 + (size_t)k * hw, dist2 + (size_t)k * hw, k ? flows + (size_t)k * 2 * hw : nullptr,
        k ? masks + (size_t)(k - 1) * hw : nullptr, masks + (size_t)k * hw, h, w, w1, w2);
    const int rc = check_launch("blend_mask_step_kernel");
    if (rc) return rc;
  }
  return FRESCO_OK;
}

extern "C" int fresco_blend_histogram(const uint8_t* lab_a, const uint8_t* lab_b, const uint8_t* lab_min_error,
                                      const uint8_t* masks, const double* weights, uint8_t* lab_out, int frames, int h,
                                      int w, void* workspace, size_t workspace_bytes, void* stream) {
  if (!lab_a || !lab_b || !weights || !lab_out || !workspace || (!lab_min_error && !masks))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_histogram: null pointer");
  if (frames <= 0 || frames > 65535 || h <= 0 || w <= 0 || (long long)h * w > (1LL << 30))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_histogram: bad shape");
  if (workspace_bytes < hist_bytes(frames))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_histogram: workspace too small");
  HistArgs A;
  A.a = lab_a;
  A.b = lab_b;
  A.e = lab_min_error;
  A.mask = masks;
  A.weights = weights;
  A.partial = (double*)workspace;
  A.stats = (double*)((char*)workspace + align256(sizeof(double) * frames * kStatBlocks * kStatQ));
  A.out = lab_out;
  A.hw = h * w;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 sg(kStatBlocks, frames);
  int rc;
  blend_hist_stats_kernel<0><<<sg, kStatThreads, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_stats_kernel<0>"))) return rc;
  blend_hist_moments_kernel<0><<<frames, 32, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_moments_kernel<0>"))) return rc;
  blend_hist_stats_kernel<1><<<sg, kStatThreads, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_stats_kernel<1>"))) return rc;
  blend_hist_moments_kernel<1><<<frames, 32, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_moments_kernel<1>"))) return rc;
  blend_hist_stats_kernel<2><<<sg, kStatThreads, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_stats_kernel<2>"))) return rc;
  blend_hist_moments_kernel<2><<<frames, 32, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_moments_kernel<2>"))) return rc;
  blend_hist_stats_kernel<3><<<sg, kStatThreads, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_stats_kernel<3>"))) return rc;
  blend_hist_moments_kernel<3><<<frames, 32, 0, s>>>(A);
  if ((rc = check_launch("blend_hist_moments_kernel<3>"))) return rc;
  const long long pixels = (long long)frames * A.hw;
  blend_hist_apply_kernel<<<grid_1d(pixels, 256), 256, 0, s>>>(A, pixels);
  return check_launch("blend_hist_apply_kernel");
}

extern "C" int fresco_blend_poisson(const uint8_t* lab_target, const uint8_t* lab_a, const uint8_t* lab_b,
                                    const uint8_t* masks, double weight0, double weight1, double weight2,
                                    uint8_t* lab_out, double* solution, int frames, int h, int w, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!lab_target || !lab_a || !lab_b || !masks || !lab_out || !workspace)
    return set_error(FRESCO_ERR_ARG, "fresco_blend_poisson: null pointer");
  if (frames <= 0 || 3LL * frames > 65535 || h <= 0 || w <= 0 || (long long)h * w > (1LL << 30))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_poisson: bad shape");
  if (workspace_bytes < fresco_blend_workspace_bytes(frames, h, w))
    return set_error(FRESCO_ERR_ARG, "fresco_blend_poisson: workspace too small");
  const double wt[3] = {weight0, weight1, weight2};
  int iters[3];
  ChebyStep st;
  double sigma[3], t_prev[3], t_cur[3];
  int total = 0;
  for (int c = 0; c < 3; ++c) {
    if (!std::isfinite(wt[c])) return set_error(FRESCO_ERR_ARG, "fresco_blend_poisson: weight not finite");
    iters[c] = fresco_blend_cheby_iterations(h, w, wt[c]);
    if (iters[c] > kMaxCheby) return set_error(FRESCO_ERR_UNSUPPORTED, "fresco_blend_poisson: weight too large");
    total = iters[c] > total ? iters[c] : total;
    const double lmax = lambda_max(h, w, wt[c]);
    st.inv_theta[c] = 2.0 / (lmax + 1.0);
    st.w2[c] = wt[c] * wt[c];
    sigma[c] = lmax > 1.0 ? (lmax + 1.0) / (lmax - 1.0) : 1.0;
    t_prev[c] = 1.0;          // T_0
    t_cur[c] = sigma[c];      // T_1
  }
  const long long hw = (long long)h * w;
  char* ws = (char*)workspace + hist_bytes(frames);
  double* rhs = (double*)ws;
  double* x[2] = {(double*)(ws + plane_bytes(frames, hw)), (double*)(ws + 2 * plane_bytes(frames, hw))};
  cudaStream_t s = (cudaStream_t)stream;
  const long long pixels = frames * hw;
  int rc;
  blend_poisson_rhs_kernel<<<grid_1d(pixels, 256), 256, 0, s>>>(lab_target, lab_a, lab_b, masks, rhs, x[0], x[1], h, w,
                                                               st.w2[0], st.w2[1], st.w2[2], pixels);
  if ((rc = check_launch("blend_poisson_rhs_kernel"))) return rc;
  const dim3 cg(grid_1d(hw, 256), 3 * frames);
  for (int k = 0; k < total; ++k) {
    for (int c = 0; c < 3; ++c) {
      st.active[c] = k < iters[c];
      if (k == 0) {
        st.omega[c] = 1.0;
      } else {     // omega_{k+1} = 2 sigma T_k / T_{k+1}, T_{k+1} = 2 sigma T_k - T_{k-1}
        const double t_next = 2.0 * sigma[c] * t_cur[c] - t_prev[c];
        st.omega[c] = 2.0 * sigma[c] * t_cur[c] / t_next;
        t_prev[c] = t_cur[c];
        t_cur[c] = t_next;
      }
    }
    blend_cheby_kernel<<<cg, 256, 0, s>>>(x[k & 1], x[(k & 1) ^ 1], rhs, h, w, st);
    if ((rc = check_launch("blend_cheby_kernel"))) return rc;
  }
  blend_poisson_finalize_kernel<<<grid_1d(pixels, 256), 256, 0, s>>>(x[0], x[1], lab_out, solution, (int)hw,
                                                                      iters[0] & 1, iters[1] & 1, iters[2] & 1, pixels);
  return check_launch("blend_poisson_finalize_kernel");
}
