// TMA + wgmma tile GEMM with fused epilogues, used by three entry points:
//
//   fresco_gram_sign            G = Xh Xh^T (per batch), epilogue T = sign(G-A) + sign(G-A^T), loss  (diffusion_hacked.py:473-475)
//   fresco_gram_grad  (step a)  Ghat = T Xh                                                         (backward of :473-475)
//   gmflow_global_corr_softmax  S = F0^T F1 / sqrt(C), online softmax over all key tiles, expected (x, y)  (matching.py:15-34)
//
// One CTA owns a 128-row tile and walks `n_iter` 128-column tiles; per column tile the K dimension is streamed in
// 64-element swizzle atoms through a 3-stage TMA/mbarrier ring (producer: warp 8) and accumulated by wgmma in the
// registers of two consumer warpgroups (64 rows each), which then run the epilogue on their own accumulators while the
// producer already streams the next column tile.
//
// RAGGED (EPI_STORE with an MN-major B, i.e. fresco_gram_grad's T Xh at tokens % 8 != 0): A = T [batch, M, M] fp16
// has a row stride of 2M bytes, which no tensor map can describe; the whole producer warp fills its atoms in the
// swizzled layout TMA would give them, B keeps its tensor map.  The consumers are the same code.
#include "common.cuh"
#include "fresco_internal.h"

namespace fresco {

constexpr int kGStages = 3;
constexpr int kGAtomA = 128 * 128;              // A atom: [128 rows x 64 fp16], 16 KB
constexpr int kGStageBytes = 2 * kGAtomA;       // + B atom(s), 16 KB
constexpr int kGThreads = 288;
constexpr int kGSmem = 1024 + kGStages * kGStageBytes + 256;

enum { EPI_STORE = 0, EPI_GRAM_SIGN = 1, EPI_GMFLOW = 2 };

struct GemmParams {
  int M, N, K;                // per-batch problem: C[M,N] = A[M,K] * B
  int n_iter;                 // column tiles walked by one CTA (gridDim.x * n_iter covers N)
  // EPI_STORE
  float* out;                 // [batch, M, N] fp32
  float alpha;
  // EPI_GRAM_SIGN
  const float* target;        // [batch, M, M] fp32
  __half* tsign;              // [batch, M, M] fp16
  float* loss_acc;
  float loss_scale;           // weight / (batch * M * M)
  // EPI_GMFLOW
  float* flow;                // [batch_total, 2, h, w]
  int w;
  int flow_batch_offset;      // forward flows at [0,B), backward at [B,2B)
  float scale_log2;
  const float2* vals;         // optional V [batch, N] (2 channels per key); null: V = the key's (x, y) pixel coordinate and
                              // the query's own coordinate is subtracted from the result (flow = correspondence - grid)
  const __half* a_ptr;        // RAGGED: A [batch, M, K], read without a tensor map
};

template <int EPI, bool B_MN, bool RAGGED = false>
__global__ void __launch_bounds__(kGThreads, 1)
tile_gemm_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                 const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kGStages * kGStageBytes);
  uint64_t* bar_full = bars;                     // [kGStages]
  uint64_t* bar_empty = bars + kGStages;         // [kGStages] one arrival per consumer warp

  if (EPI == EPI_GRAM_SIGN && blockIdx.x < blockIdx.y) return;   // symmetric output: tiles with J < I are mirrored
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * 128;
  const int batch = blockIdx.z;
  const int n_tile0 = blockIdx.x * p.n_iter;
  const int k_atoms = (p.K + 63) / 64;
  static_assert(!RAGGED || (EPI == EPI_STORE && B_MN), "the ragged A operand is T of fresco_gram_grad");

  if (threadIdx.x == 0) {
    for (int s = 0; s < kGStages; ++s) {
      mbar_init(bar_full + s, RAGGED ? 32 : 1);          // RAGGED: every lane of the producer warp arrives
      mbar_init(bar_empty + s, 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if constexpr (RAGGED) {
      // ---------------------------------------------------------------- producer: A by the warp, B by TMA
      int it = 0;
      for (int t = 0; t < p.n_iter; ++t) {
        const int n0 = (n_tile0 + t) * 128;
        for (int ka = 0; ka < k_atoms; ++ka, ++it) {
          const int st = it % kGStages;
          if (it >= kGStages) mbar_wait_mma_backoff(bar_empty + st, ((it / kGStages) - 1) & 1, 64);
          uint8_t* sa = smem + st * kGStageBytes;
          uint8_t* sb = sa + kGAtomA;
          fill_kmajor_atom_sw128(sa, p.a_ptr + (size_t)batch * p.M * p.K, p.K, m0, ka * 64, p.M, p.K, lane);
          fence_proxy_async_smem();                       // the generic stores, before wgmma reads them
          if (lane == 0) {
            mbar_expect_tx(bar_full + st, kGStageBytes - kGAtomA);
            tma_load_3d(sb, &tm_b, bar_full + st, n0, ka * 64, batch);
            tma_load_3d(sb + 8192, &tm_b, bar_full + st, n0 + 64, ka * 64, batch);
          } else {
            mbar_arrive(bar_full + st);
          }
        }
      }
      return;
    }
    // ------------------------------------------------------------------ TMA producer
    if (FRESCO_ISSUER_THREAD(lane)) {
      tma_prefetch_desc(&tm_a);
      tma_prefetch_desc(&tm_b);
      int it = 0;
      for (int t = 0; t < p.n_iter; ++t) {
        const int n0 = (n_tile0 + t) * 128;
        for (int ka = 0; ka < k_atoms; ++ka, ++it) {
          const int st = it % kGStages;
          if (it >= kGStages) mbar_wait_mma_backoff(bar_empty + st, ((it / kGStages) - 1) & 1, 64);
          uint8_t* sa = smem + st * kGStageBytes;
          uint8_t* sb = sa + kGAtomA;
          mbar_expect_tx(bar_full + st, kGStageBytes);
          tma_load_3d(sa, &tm_a, bar_full + st, ka * 64, m0, batch);
          if (B_MN) {
            // B is [K rows, N cols] row-major: two [64 k x 64 n] boxes cover the 128-wide column tile
            tma_load_3d(sb, &tm_b, bar_full + st, n0, ka * 64, batch);
            tma_load_3d(sb + 8192, &tm_b, bar_full + st, n0 + 64, ka * 64, batch);
          } else {
            tma_load_3d(sb, &tm_b, bar_full + st, ka * 64, n0, batch);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups: rows m0 + 64 wg + [0, 64)
  const int wg = warp >> 2;
  const int gm0 = m0 + wg * 64 + acc_row(0);       // this thread's two rows: gm0, gm0 + 8
  float loss = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, ax[2] = {0.f, 0.f}, ay[2] = {0.f, 0.f};  // EPI_GMFLOW
  int it = 0;
  for (int t = 0; t < p.n_iter; ++t) {
    const int n0 = (n_tile0 + t) * 128;
    float acc[64];
    for (int ka = 0; ka < k_atoms; ++ka, ++it) {
      const int st = it % kGStages;
      mbar_wait_mma(bar_full + st, (it / kGStages) & 1);
      const uint32_t a_addr = smem_u32(smem + st * kGStageBytes) + wg * 64 * 128;
      const uint32_t b_addr = smem_u32(smem + st * kGStageBytes + kGAtomA);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t accum = (ka > 0 || kk > 0) ? 1u : 0u;
        const uint64_t a_desc = make_smem_desc_sw128(a_addr + kk * 32, 16, 1024);
        if (B_MN)
          wgmma_ss<128, 1>(acc, a_desc, make_smem_desc_sw128(b_addr + kk * 2048, 8192, 1024), accum);
        else
          wgmma_ss<128>(acc, a_desc, make_smem_desc_sw128(b_addr + kk * 32, 16, 1024), accum);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + st);
    }

    if (EPI == EPI_STORE) {
#pragma unroll
      for (int i = 0; i < 64; i += 2) {
        const int gm = gm0 + 8 * ((i >> 1) & 1), gn = n0 + acc_col(i);
        if (gm < p.M && gn < p.N)
          *reinterpret_cast<float2*>(p.out + ((size_t)batch * p.M + gm) * p.N + gn) =
              make_float2(acc[i] * p.alpha, acc[i + 1] * p.alpha);
      }
    } else if (EPI == EPI_GRAM_SIGN) {
      // T is symmetric (T_ij = sign(G_ij - A_ij) + sign(G_ij - A_ji), G symmetric), so only tiles J >= I are
      // launched; this CTA also writes the mirrored tile T_JI and accounts for its share of the loss.
      const size_t plane = (size_t)batch * p.M * p.M;
      const bool diag_tile = (n0 == m0);
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int gm = gm0 + 8 * ((i >> 1) & 1), gn = n0 + acc_col(i);
        if (gm < p.M && gn < p.M) {
          const float d1 = acc[i] - __ldg(p.target + plane + (size_t)gm * p.M + gn);
          const float d2 = acc[i] - __ldg(p.target + plane + (size_t)gn * p.M + gm);
          loss += fabsf(d1) + (diag_tile ? 0.f : fabsf(d2));
          const __half tv = __float2half_rn(sgnf(d1) + sgnf(d2));
          p.tsign[plane + (size_t)gm * p.M + gn] = tv;
          if (!diag_tile) p.tsign[plane + (size_t)gn * p.M + gm] = tv;
        }
      }
    } else {  // EPI_GMFLOW: online softmax with V = (x, y) pixel coordinates of the key token (or p.vals)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (n0 + acc_col(i) < p.N) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], acc[i]);
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float m = mx[r];
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        const float m_new = fmaxf(m_run[r], m * p.scale_log2);
        alpha[r] = fast_exp2(m_run[r] - m_new);
        m_run[r] = m_new;
        l_run[r] *= alpha[r];
        ax[r] *= alpha[r];
        ay[r] *= alpha[r];
      }
      const float2* vrow = p.vals ? p.vals + (size_t)batch * p.N : nullptr;
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int gn = n0 + acc_col(i), r = (i >> 1) & 1;
        if (gn < p.N) {
          const float pe = fast_exp2(fmaf(acc[i], p.scale_log2, -m_run[r]));
          const float2 vv = vrow ? __ldg(vrow + gn) : make_float2((float)(gn % p.w), (float)(gn / p.w));
          l_run[r] += pe;
          ax[r] = fmaf(pe, vv.x, ax[r]);
          ay[r] = fmaf(pe, vv.y, ay[r]);
        }
      }
    }
  }
  if (EPI == EPI_GRAM_SIGN && p.loss_acc != nullptr) {
    loss = warp_sum(loss);
    if (lane == 0) atomicAdd(p.loss_acc, loss * p.loss_scale);
  }
  if (EPI == EPI_GMFLOW) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float l = l_run[r], sx = ax[r], sy = ay[r];
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        l += __shfl_xor_sync(0xffffffffu, l, o);
        sx += __shfl_xor_sync(0xffffffffu, sx, o);
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
      }
      const int gm = gm0 + 8 * r;
      if ((lane & 3) == 0 && gm < p.M) {
        const float inv = 1.f / l;
        const int qx = gm % p.w, qy = gm / p.w;
        float* f = p.flow + (size_t)(p.flow_batch_offset + batch) * 2 * p.M;
        f[gm] = sx * inv - (p.vals ? 0.f : (float)qx);
        f[p.M + gm] = sy * inv - (p.vals ? 0.f : (float)qy);
      }
    }
  }
}

template <int EPI, bool B_MN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid, cudaStream_t s) {
  if (int rc = allow_dynamic_smem((const void*)tile_gemm_kernel<EPI, B_MN>, kGSmem, "tile_gemm")) return rc;
  tile_gemm_kernel<EPI, B_MN><<<grid, kGThreads, kGSmem, s>>>(ta, tb, p);
  static const char* const kEpiNames[] = {"EPI_STORE", "EPI_GRAM_SIGN", "EPI_GMFLOW"};
  return check_launchf("tile_gemm_kernel<%s,%d>", kEpiNames[EPI], (int)B_MN);
}

static int launch_gemm_ragged_a(const CUtensorMap& tb, const GemmParams& p, dim3 grid, cudaStream_t s) {
  const void* k = (const void*)tile_gemm_kernel<EPI_STORE, true, true>;
  if (int rc = allow_dynamic_smem(k, kGSmem, "tile_gemm")) return rc;
  tile_gemm_kernel<EPI_STORE, true, true><<<grid, kGThreads, kGSmem, s>>>(tb, tb, p);
  return check_launch("tile_gemm_kernel<EPI_STORE,1,ragged>");
}

// ghat [batch, L, C] fp32 (token-major)  ->  grad [batch, C, L] += (ghat - (ghat . xhat) xhat) / norm
// one CTA per (batch, 32 tokens); the row dot needs the whole C extent, hence the separate pass
__global__ void gram_project_kernel(const float* __restrict__ ghat, const __half* __restrict__ xhat,
                                    const float* __restrict__ norms, float* __restrict__ grad, int channels,
                                    int tokens) {
  __shared__ float dot[32];
  __shared__ float tile[32][65];
  const int tiles = (tokens + 31) / 32;
  const int l0 = (blockIdx.x % tiles) * 32;
  const int b = blockIdx.x / tiles;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // row dots: warp w handles tokens w, w+8, ...
  for (int tk = warp; tk < 32; tk += 8) {
    const int l = l0 + tk;
    float acc = 0.f;
    if (l < tokens) {
      const float* g = ghat + ((size_t)b * tokens + l) * channels;
      const __half* x = xhat + ((size_t)b * tokens + l) * channels;
      for (int c = lane; c < channels; c += 32) acc = fmaf(g[c], __half2float(x[c]), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) dot[tk] = acc;
  }
  __syncthreads();
  for (int c0 = 0; c0 < channels; c0 += 64) {
    // read [32 tokens x 64 channels] (channel-contiguous), project, stage transposed
    for (int t = threadIdx.x; t < 32 * 64; t += blockDim.x) {
      const int tk = t / 64, cc = t % 64;
      const int l = l0 + tk, c = c0 + cc;
      float v = 0.f;
      if (l < tokens && c < channels) {
        const size_t off = ((size_t)b * tokens + l) * channels + c;
        const float xh = __half2float(xhat[off]);
        v = (ghat[off] - dot[tk] * xh) / norms[(size_t)b * tokens + l];
      }
      tile[tk][cc] = v;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 64 * 32; t += blockDim.x) {
      const int cc = t / 32, tk = t % 32;
      const int l = l0 + tk, c = c0 + cc;
      if (l < tokens && c < channels) grad[((size_t)b * channels + c) * tokens + l] += tile[tk][cc];
    }
    __syncthreads();
  }
}

// fp32 [batch, C, L] -> fp16 token-major [batch, L, C] (no normalisation); 32x32 smem transpose
__global__ void to_token_major_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, int channels,
                                          int tokens) {
  __shared__ float tile[32][33];
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + tx;
    tile[i][tx] = (c < channels && l < tokens) ? src[((size_t)b * channels + c) * tokens + l] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + tx;
    if (l < tokens && c < channels) dst[((size_t)b * tokens + l) * channels + c] = __float2half_rn(tile[tx][i]);
  }
}

}  // namespace fresco

using namespace fresco;

extern "C" int fresco_gram_sign_scaled(const void* xhat, const float* target, void* tsign, float* loss_acc, int batch,
                                       int tokens, int channels, double scale, void* stream) {
  if (!xhat || !target || !tsign) return set_error(FRESCO_ERR_ARG, "fresco_gram_sign: null pointer");
  // the target and T are read and written element by element in the epilogue, so any token count runs here
  if (batch <= 0 || tokens <= 0 || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_gram_sign: channels must be a multiple of 8");
  CUtensorMap ta;
  if (make_kmajor_map(&ta, xhat, tokens, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  GemmParams p = {};
  p.M = tokens;
  p.N = tokens;
  p.K = channels;
  p.n_iter = 1;
  p.target = target;
  p.tsign = static_cast<__half*>(tsign);
  p.loss_acc = loss_acc;
  p.loss_scale = (float)scale;
  const int tiles = (tokens + 127) / 128;
  return launch_gemm<EPI_GRAM_SIGN, false>(ta, ta, p, dim3(tiles, tiles, batch), (cudaStream_t)stream);
}

extern "C" int fresco_gram_sign(const void* xhat, const float* target, void* tsign, float* loss_acc, int batch,
                                int tokens, int channels, float weight, void* stream) {
  return fresco_gram_sign_scaled(xhat, target, tsign, loss_acc, batch, tokens, channels,
                                 (double)weight / ((double)batch * tokens * tokens), stream);
}

extern "C" size_t fresco_gram_grad_workspace_bytes(int batch, int tokens, int channels) {
  return (size_t)batch * tokens * channels * sizeof(float);
}

extern "C" int fresco_gram_grad_scaled(const void* tsign, const void* xhat, const float* norms, float* grad, int batch,
                                       int tokens, int channels, double scale, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  if (!tsign || !xhat || !norms || !grad || !workspace) return set_error(FRESCO_ERR_ARG, "fresco_gram_grad: null pointer");
  if (batch <= 0 || tokens <= 0 || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_gram_grad: channels must be a multiple of 8");
  if (workspace_bytes < fresco_gram_grad_workspace_bytes(batch, tokens, channels))
    return set_error(FRESCO_ERR_ARG, "fresco_gram_grad: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  const float alpha = (float)scale;
  int rc;
  if (option(OPT_GRAM_V, 2) == 2) {
    // persistent 128 x 256 tiles (gram_wgmma.cu)
    rc = fresco_gram_tx(tsign, xhat, static_cast<float*>(workspace), batch, tokens, channels, alpha, stream);
  } else {
    const bool ragged = tokens % 8 != 0;            // T's rows are not 16-byte aligned: no tensor map for it
    CUtensorMap ta, tb;
    if (!ragged && make_kmajor_map(&ta, tsign, tokens, tokens, batch, 128)) return FRESCO_ERR_TENSORMAP;
    if (make_mnmajor_map(&tb, xhat, tokens, channels, batch)) return FRESCO_ERR_TENSORMAP;
    GemmParams p = {};
    p.M = tokens;
    p.N = channels;
    p.K = tokens;
    p.n_iter = 1;
    p.out = static_cast<float*>(workspace);
    p.alpha = alpha;
    const dim3 grid((channels + 127) / 128, (tokens + 127) / 128, batch);
    if (ragged) {
      p.a_ptr = static_cast<const __half*>(tsign);
      rc = launch_gemm_ragged_a(tb, p, grid, s);
    } else {
      rc = launch_gemm<EPI_STORE, true>(ta, tb, p, grid, s);
    }
  }
  if (rc) return rc;
  const int tiles = (tokens + 31) / 32;
  gram_project_kernel<<<batch * tiles, 256, 0, s>>>(static_cast<const float*>(workspace), (const __half*)xhat, norms,
                                                    grad, channels, tokens);
  return check_launch("gram_project_kernel");
}

extern "C" int fresco_gram_grad(const void* tsign, const void* xhat, const float* norms, float* grad, int batch,
                                int tokens, int channels, float weight, void* workspace, size_t workspace_bytes,
                                void* stream) {
  return fresco_gram_grad_scaled(tsign, xhat, norms, grad, batch, tokens, channels,
                                 (double)weight / ((double)batch * tokens * tokens), workspace, workspace_bytes, stream);
}

extern "C" size_t fresco_gmflow_corr_workspace_bytes(int batch, int channels, int h, int w) {
  return (size_t)2 * batch * channels * h * w * sizeof(__half) + 256;
}

extern "C" int gmflow_global_corr_softmax(const float* feature0, const float* feature1, float* flow, int batch,
                                          int channels, int h, int w, int bidir, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  if (!feature0 || !feature1 || !flow || !workspace)
    return set_error(FRESCO_ERR_ARG, "gmflow_global_corr_softmax: null pointer");
  if (batch <= 0 || channels <= 0 || channels % 8 != 0 || h <= 0 || w <= 0)
    return set_error(FRESCO_ERR_ARG, "gmflow_global_corr_softmax: channels must be a multiple of 8");
  if (workspace_bytes < fresco_gmflow_corr_workspace_bytes(batch, channels, h, w))
    return set_error(FRESCO_ERR_ARG, "gmflow_global_corr_softmax: workspace too small");
  const int L = h * w;
  cudaStream_t s = (cudaStream_t)stream;
  __half* t0 = reinterpret_cast<__half*>((reinterpret_cast<uintptr_t>(workspace) + 127) & ~uintptr_t(127));
  __half* t1 = t0 + (size_t)batch * L * channels;
  dim3 tg((L + 31) / 32, (channels + 31) / 32, batch);
  to_token_major_f16_kernel<<<tg, 256, 0, s>>>(feature0, t0, channels, L);
  int rc = check_launch("to_token_major_f16_kernel");
  if (rc) return rc;
  to_token_major_f16_kernel<<<tg, 256, 0, s>>>(feature1, t1, channels, L);
  rc = check_launch("to_token_major_f16_kernel");
  if (rc) return rc;
  CUtensorMap m0, m1;
  if (make_kmajor_map(&m0, t0, L, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  if (make_kmajor_map(&m1, t1, L, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  GemmParams p = {};
  p.M = L;
  p.N = L;
  p.K = channels;
  p.n_iter = (L + 127) / 128;
  p.flow = flow;
  p.w = w;
  p.flow_batch_offset = 0;
  p.scale_log2 = (float)(1.4426950408889634 / sqrt((double)channels));
  dim3 grid(1, (L + 127) / 128, batch);
  rc = launch_gemm<EPI_GMFLOW, false>(m0, m1, p, grid, s);      // forward: rows = frame-0 tokens
  if (rc || !bidir) return rc;
  p.flow_batch_offset = batch;                                  // backward: softmax over the transposed volume
  return launch_gemm<EPI_GMFLOW, false>(m1, m0, p, grid, s);
}

// GMFlow's flow-propagation attention (gmflow/transformer.py:353-374): out = softmax(q k^T / sqrt(C)) flow, with the
// 2-channel flow field as V.  Same kernel as the global correlation (online softmax over all key tiles, the
// [B, L, L] probability volume never exists); q, k are token-major fp16 [batch, tokens, channels].
extern "C" int gmflow_flow_attention(const void* q, const void* k, const float* values, float* out, int batch, int tokens,
                                     int channels, float softmax_scale, void* stream) {
  if (!q || !k || !values || !out) return set_error(FRESCO_ERR_ARG, "gmflow_flow_attention: null pointer");
  if (batch <= 0 || tokens <= 0 || channels <= 0 || channels % 8 != 0 || softmax_scale <= 0.f)
    return set_error(FRESCO_ERR_ARG, "gmflow_flow_attention: bad shape (channels must be a multiple of 8)");
  CUtensorMap mq, mk;
  if (make_kmajor_map(&mq, q, tokens, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  if (make_kmajor_map(&mk, k, tokens, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  GemmParams p = {};
  p.M = tokens;
  p.N = tokens;
  p.K = channels;
  p.n_iter = (tokens + 127) / 128;
  p.flow = out;
  p.w = tokens;                    // unused with vals
  p.flow_batch_offset = 0;
  p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.vals = reinterpret_cast<const float2*>(values);
  return launch_gemm<EPI_GMFLOW, false>(mq, mk, p, dim3(1, (tokens + 127) / 128, batch), (cudaStream_t)stream);
}
