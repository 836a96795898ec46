// Persistent 128 x 256 wgmma GEMM for the spatial-consistency (normalised-Gram L1) loss of optimize_feature
// (src/diffusion_hacked.py:469-476 and its backward).  One CTA per SM walks a static list of tiles; every wgmma is
// M64 N256 K16, two consumer warpgroups own 64 rows each of a 128-row tile (128 fp32 accumulator registers per thread),
// and a producer warp keeps a 4-stage TMA ring ahead of them, across tile boundaries.
//
//   MODE_SIGN  D = Xh_I Xh_J^T - Yh_I Yh_J^T   (K = 2C: the second half of the K loop reads the normalised REFERENCE
//              features with the B operand negated by the instruction), T = 2 sign(D) as fp16 to [I, J] and
//              mirrored to [J, I], loss += sum |D|.  The fp32 [2N, L, L] Gram target of the reference (1.07 GB at layer
//              3, read every Adam iteration) is never materialised: what is stored per batch is Yh, [2N, L, C] fp16.
//              Only tiles that touch the upper triangle are computed (D is symmetric).
//   MODE_GRAD  Ghat = alpha * T Xh   (A = T, K-major; B = Xh read MN-major from its token-major layout), fp32 out.
//
// RAGGED (tokens % 8 != 0): T [batch, M, M] fp16 has a row stride of 2M bytes, which is not a multiple of 16, so no
// tensor map can describe it.  MODE_SIGN then stores T element by element (a pair store would straddle rows and lose
// its 4-byte alignment when M is odd); MODE_GRAD fills the A atom of every stage from the whole producer warp, in the
// swizzled layout TMA would give it, while B (Xh, row stride 2C bytes) keeps its tensor map.  The wgmma consumers are
// the same code.
#include "common.cuh"
#include "fresco_internal.h"

#include <type_traits>

namespace fresco {

constexpr int kG2Stages = 4;
constexpr int kG2AtomA = 128 * 128;                 // [128 rows x 64 fp16]
constexpr int kG2AtomB = 256 * 128;                 // [256 rows x 64 fp16] (K-major) or 4 x [64 k x 64 n] (MN-major)
constexpr int kG2StageBytes = kG2AtomA + kG2AtomB;  // 48 KB
constexpr int kG2Threads = 288;
constexpr int kG2Smem = 1024 + kG2Stages * kG2StageBytes + 256;

enum { G2_SIGN = 0, G2_GRAD = 1 };

struct Gram2Params {
  int M;                      // tokens
  int C;                      // channels
  int batch;
  int T;                      // 128-row tiles per side
  int P;                      // 256-column tile pairs per side
  int tiles_per_batch;
  int n_tiles;                // total
  // G2_SIGN
  __half* tsign;              // [batch, M, M]
  float* loss_acc;
  float loss_scale;           // weight / (batch * M * M), rounded once
  // G2_GRAD
  float* out;                 // [batch, M, C]
  float alpha;
  const __half* ta;           // G2_GRAD, RAGGED: T [batch, M, M], read without a tensor map
};

// tile id -> (batch, row tile I, column pair Jp) for G2_SIGN: row tile I needs the pairs that touch columns >= 128 I,
// i.e. Jp >= I / 2.  G2_GRAD: all pairs of ceil(C / 256).
template <int MODE>
__device__ __forceinline__ void decode_tile(const Gram2Params& p, int tile, int& b, int& I, int& Jp) {
  b = tile / p.tiles_per_batch;
  int r = tile - b * p.tiles_per_batch;
  if (MODE == G2_GRAD) {
    I = r / p.P;
    Jp = r - I * p.P;
    return;
  }
  I = 0;
  for (;;) {
    const int cnt = p.P - (I >> 1);
    if (r < cnt) break;
    r -= cnt;
    ++I;
  }
  Jp = (I >> 1) + r;
}

template <int MODE, bool RAGGED>
__global__ void __launch_bounds__(kG2Threads, 1)
gram2_kernel(const __grid_constant__ CUtensorMap tm_a0, const __grid_constant__ CUtensorMap tm_b0,
             const __grid_constant__ CUtensorMap tm_a1, const __grid_constant__ CUtensorMap tm_b1, const Gram2Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kG2Stages * kG2StageBytes);
  uint64_t* bar_full = bars;                       // [kG2Stages]
  uint64_t* bar_empty = bars + kG2Stages;          // [kG2Stages] one arrival per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // K atoms (64 elements) of one tile: SIGN walks the channels twice (current features, then reference features)
  const int c_atoms = (p.C + 63) / 64;
  const int k_atoms = MODE == G2_SIGN ? 2 * c_atoms : (p.M + 63) / 64;
  constexpr bool kWarpFill = RAGGED && MODE == G2_GRAD;    // the producer warp's 32 lanes each arrive on bar_full

  if (threadIdx.x == 0) {
    for (int s = 0; s < kG2Stages; ++s) {
      mbar_init(bar_full + s, kWarpFill ? 32 : 1);
      mbar_init(bar_empty + s, 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if constexpr (kWarpFill) {
      // ---------------------------------------------------------------- producer: A (T) by the warp, B (Xh) by TMA
      int it = 0;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        int b, I, Jp;
        decode_tile<MODE>(p, tile, b, I, Jp);
        for (int ka = 0; ka < k_atoms; ++ka, ++it) {
          const int st = it % kG2Stages;
          if (it >= kG2Stages) mbar_wait_mma_backoff(bar_empty + st, ((it / kG2Stages) - 1) & 1, 32);
          uint8_t* sa = smem + st * kG2StageBytes;
          uint8_t* sb = sa + kG2AtomA;
          fill_kmajor_atom_sw128(sa, p.ta + (size_t)b * p.M * p.M, p.M, I * 128, ka * 64, p.M, p.M, lane);
          fence_proxy_async_smem();                       // the generic stores, before wgmma reads them
          if (lane == 0) {
            mbar_expect_tx(bar_full + st, kG2AtomB);
#pragma unroll
            for (int q = 0; q < 4; ++q)
              tma_load_3d(sb + q * 8192, &tm_b0, bar_full + st, Jp * 256 + q * 64, ka * 64, b);
          } else {
            mbar_arrive(bar_full + st);
          }
        }
      }
      return;
    }
    // ------------------------------------------------------------------ TMA producer
    if (FRESCO_ISSUER_THREAD(lane)) {
      tma_prefetch_desc(&tm_a0);
      tma_prefetch_desc(&tm_b0);
      tma_prefetch_desc(&tm_a1);
      tma_prefetch_desc(&tm_b1);
      int it = 0;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        int b, I, Jp;
        decode_tile<MODE>(p, tile, b, I, Jp);
        for (int ka = 0; ka < k_atoms; ++ka, ++it) {
          const int st = it % kG2Stages;
          if (it >= kG2Stages) mbar_wait_mma_backoff(bar_empty + st, ((it / kG2Stages) - 1) & 1, 32);
          uint8_t* sa = smem + st * kG2StageBytes;
          uint8_t* sb = sa + kG2AtomA;
          mbar_expect_tx(bar_full + st, kG2StageBytes);
          if (MODE == G2_SIGN) {
            const bool ref = ka >= c_atoms;
            const int kc = (ref ? ka - c_atoms : ka) * 64;
            tma_load_3d(sa, ref ? &tm_a1 : &tm_a0, bar_full + st, kc, I * 128, b);
            tma_load_3d(sb, ref ? &tm_b1 : &tm_b0, bar_full + st, kc, Jp * 256, b);          // [256 rows x 64 k]
          } else {
            tma_load_3d(sa, &tm_a0, bar_full + st, ka * 64, I * 128, b);                       // T rows, K = tokens
#pragma unroll
            for (int q = 0; q < 4; ++q)                                                        // Xh [64 k x 64 n] x 4
              tma_load_3d(sb + q * 8192, &tm_b0, bar_full + st, Jp * 256 + q * 64, ka * 64, b);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  const int wg = warp >> 2;
  float loss = 0.f;
  int it = 0;
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    int b, I, Jp;
    decode_tile<MODE>(p, tile, b, I, Jp);
    float acc[128];
    // K atoms [ka0, ka1); NEG: B negated (the reference half of G2_SIGN).  A compile-time choice, as a branch between
    // wgmma forms would make ptxas serialise them.
    auto k_loop = [&](auto neg, int ka0, int ka1) {
      for (int ka = ka0; ka < ka1; ++ka, ++it) {
        const int st = it % kG2Stages;
        mbar_wait_mma(bar_full + st, (it / kG2Stages) & 1);
        const uint32_t a_addr = smem_u32(smem + st * kG2StageBytes) + wg * 64 * 128;
        const uint32_t b_addr = smem_u32(smem + st * kG2StageBytes + kG2AtomA);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint32_t accum = (ka > 0 || kk > 0) ? 1u : 0u;
          const uint64_t a_desc = make_smem_desc_sw128(a_addr + kk * 32, 16, 1024);
          if constexpr (MODE == G2_GRAD)
            wgmma_ss<256, 1>(acc, a_desc, make_smem_desc_sw128(b_addr + kk * 2048, 8192, 1024), accum);
          else
            wgmma_ss<256, 0, decltype(neg)::value ? -1 : 1>(acc, a_desc, make_smem_desc_sw128(b_addr + kk * 32, 16, 1024),
                                                            accum);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + st);
      }
    };
    if (MODE == G2_SIGN) {
      k_loop(std::false_type{}, 0, c_atoms);
      k_loop(std::true_type{}, c_atoms, k_atoms);
    } else {
      k_loop(std::false_type{}, 0, k_atoms);
    }

    const int gm0 = I * 128 + wg * 64 + acc_row(0);   // this thread's two rows: gm0, gm0 + 8
    if (MODE == G2_GRAD) {
#pragma unroll
      for (int i = 0; i < 128; i += 2) {
        const int gm = gm0 + 8 * ((i >> 1) & 1), c = Jp * 256 + acc_col(i);
        if (gm < p.M && c < p.C)
          *reinterpret_cast<float2*>(p.out + ((size_t)b * p.M + gm) * p.C + c) =
              make_float2(acc[i] * p.alpha, acc[i + 1] * p.alpha);
      }
    } else {
      const size_t plane = (size_t)b * p.M * p.M;
#pragma unroll
      for (int i = 0; i < 128; i += 2) {
        const int gm = gm0 + 8 * ((i >> 1) & 1), j = Jp * 256 + acc_col(i);
        const int J = j >> 7;                                   // 128-column block; j and j + 1 share it
        // below the diagonal: the mirror of tile (J, I) covers it; columns >= M are zero (TMA zero fill), never stored
        if (J < I || gm >= p.M || j >= p.M) continue;
        const bool diag = (J == I);
        const float d0 = acc[i], d1 = acc[i + 1];
        loss += (fabsf(d0) + fabsf(d1)) * (diag ? 1.f : 2.f);   // off-diagonal blocks stand for their mirror as well
        const float t0 = d0 > 0.f ? 2.f : (d0 < 0.f ? -2.f : 0.f);
        const float t1 = d1 > 0.f ? 2.f : (d1 < 0.f ? -2.f : 0.f);
        if constexpr (RAGGED) {                                 // j + 1 may be M; (gm, j) may be odd
          const bool pair = j + 1 < p.M;
          p.tsign[plane + (size_t)gm * p.M + j] = __float2half_rn(t0);
          if (pair) p.tsign[plane + (size_t)gm * p.M + j + 1] = __float2half_rn(t1);
          if (!diag) {
            p.tsign[plane + (size_t)j * p.M + gm] = __float2half_rn(t0);
            if (pair) p.tsign[plane + (size_t)(j + 1) * p.M + gm] = __float2half_rn(t1);
          }
        } else {
          *reinterpret_cast<uint32_t*>(p.tsign + plane + (size_t)gm * p.M + j) = pack_half2(t0, t1);   // M % 8 == 0
          if (!diag) {                                          // mirror T[j, i] = T[i, j]
            p.tsign[plane + (size_t)j * p.M + gm] = __float2half_rn(t0);
            p.tsign[plane + (size_t)(j + 1) * p.M + gm] = __float2half_rn(t1);
          }
        }
      }
    }
  }
  if (MODE == G2_SIGN && p.loss_acc != nullptr) {
    loss = warp_sum(loss);
    if (lane == 0) atomicAdd(p.loss_acc, loss * p.loss_scale);
  }
}

template <int MODE, bool RAGGED>
static int launch_gram2(const CUtensorMap& a0, const CUtensorMap& b0, const CUtensorMap& a1, const CUtensorMap& b1,
                        const Gram2Params& p, cudaStream_t s) {
  if (int rc = allow_dynamic_smem((const void*)gram2_kernel<MODE, RAGGED>, kG2Smem, "gram2")) return rc;
  int grid = sm_count();
  if (grid > p.n_tiles) grid = p.n_tiles;
  gram2_kernel<MODE, RAGGED><<<grid, kG2Threads, kG2Smem, s>>>(a0, b0, a1, b1, p);
  if (RAGGED) return check_launch(MODE == G2_SIGN ? "gram2_kernel<G2_SIGN,ragged>" : "gram2_kernel<G2_GRAD,ragged>");
  return check_launch(MODE == G2_SIGN ? "gram2_kernel<G2_SIGN>" : "gram2_kernel<G2_GRAD>");
}

}  // namespace fresco

using namespace fresco;

extern "C" int fresco_gram_sign_ref_scaled(const void* xhat, const void* yhat, void* tsign, float* loss_acc, int batch,
                                           int tokens, int channels, double scale, void* stream) {
  if (!xhat || !yhat || !tsign) return set_error(FRESCO_ERR_ARG, "fresco_gram_sign_ref: null pointer");
  if (batch <= 0 || tokens <= 0 || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_gram_sign_ref: channels must be a multiple of 8");
  CUtensorMap ax, bx, ay, by;
  if (make_kmajor_map(&ax, xhat, tokens, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  if (make_kmajor_map(&bx, xhat, tokens, channels, batch, 256)) return FRESCO_ERR_TENSORMAP;
  if (make_kmajor_map(&ay, yhat, tokens, channels, batch, 128)) return FRESCO_ERR_TENSORMAP;
  if (make_kmajor_map(&by, yhat, tokens, channels, batch, 256)) return FRESCO_ERR_TENSORMAP;
  Gram2Params p = {};
  p.M = tokens;
  p.C = channels;
  p.batch = batch;
  p.T = (tokens + 127) / 128;
  p.P = (p.T + 1) / 2;
  int per = 0;
  for (int I = 0; I < p.T; ++I) per += p.P - (I >> 1);
  p.tiles_per_batch = per;
  p.n_tiles = per * batch;
  p.tsign = static_cast<__half*>(tsign);
  p.loss_acc = loss_acc;
  p.loss_scale = (float)scale;
  if (tokens % 8 != 0) return launch_gram2<G2_SIGN, true>(ax, bx, ay, by, p, (cudaStream_t)stream);
  return launch_gram2<G2_SIGN, false>(ax, bx, ay, by, p, (cudaStream_t)stream);
}

extern "C" int fresco_gram_sign_ref(const void* xhat, const void* yhat, void* tsign, float* loss_acc, int batch,
                                    int tokens, int channels, float weight, void* stream) {
  return fresco_gram_sign_ref_scaled(xhat, yhat, tsign, loss_acc, batch, tokens, channels,
                                     (double)weight / ((double)batch * tokens * tokens), stream);
}

extern "C" int fresco_gram_tx(const void* tsign, const void* xhat, float* ghat, int batch, int tokens, int channels,
                              float alpha, void* stream) {
  if (!tsign || !xhat || !ghat) return set_error(FRESCO_ERR_ARG, "fresco_gram_tx: null pointer");
  if (batch <= 0 || tokens <= 0 || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_gram_tx: channels must be a multiple of 8");
  const bool ragged = tokens % 8 != 0;              // T's rows are not 16-byte aligned: no tensor map for it
  CUtensorMap ta, tb;
  if (!ragged && make_kmajor_map(&ta, tsign, tokens, tokens, batch, 128)) return FRESCO_ERR_TENSORMAP;
  if (make_mnmajor_map(&tb, xhat, tokens, channels, batch)) return FRESCO_ERR_TENSORMAP;
  if (ragged) ta = tb;                              // unused by the ragged kernel
  Gram2Params p = {};
  p.M = tokens;
  p.C = channels;
  p.batch = batch;
  p.T = (tokens + 127) / 128;
  p.P = (channels + 255) / 256;
  p.tiles_per_batch = p.T * p.P;
  p.n_tiles = p.tiles_per_batch * batch;
  p.out = ghat;
  p.alpha = alpha;
  p.ta = static_cast<const __half*>(tsign);
  if (ragged) return launch_gram2<G2_GRAD, true>(ta, tb, ta, tb, p, (cudaStream_t)stream);
  return launch_gram2<G2_GRAD, false>(ta, tb, ta, tb, p, (cudaStream_t)stream);
}
