// HBM-bound kernels of the FRESCO hot path: K/V compaction, temporal-guided (FLATTEN)
// attention, bilinear flow warp, the warp_tensor frame chain, the temporal-consistency
// loss forward+backward, Adam, AdaIN and the Gram-loss normalise/transposition.
// All are coalesced / vectorised streaming kernels; none is reshaped into a GEMM.
#include "common.cuh"
#include "fresco_internal.h"

namespace fresco {

// =============================================================================================
// A2  K/V compaction  (src/diffusion_hacked.py:234-247)
// =============================================================================================
__global__ void kv_compact_kernel(const uint4* __restrict__ k, const uint4* __restrict__ v,
                                  const int32_t* __restrict__ idx, uint4* __restrict__ k_out,
                                  uint4* __restrict__ v_out, int chunks, long long rows_per_chunk, int n_sel,
                                  int vec_per_row) {
  const long long total = (long long)chunks * n_sel * vec_per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int part = (int)(t % vec_per_row);
    const long long row = t / vec_per_row;
    const int i = (int)(row % n_sel);
    const int c = (int)(row / n_sel);
    const long long src = ((long long)c * rows_per_chunk + idx[i]) * vec_per_row + part;
    k_out[t] = __ldg(k + src);
    v_out[t] = __ldg(v + src);
  }
}

// K and V rows of the selected tokens side by side in one 2C-wide row: the send buffer of the cross-frame K/V exchange
// (fresco_b200/dist.py), [chunks, out_rows, 2C] with rows [0, n_sel) written
__global__ void kv_compact_packed_kernel(const uint4* __restrict__ k, const uint4* __restrict__ v,
                                         const int32_t* __restrict__ idx, uint4* __restrict__ kv_out, int chunks,
                                         long long rows_per_chunk, int n_sel, int out_rows, int vec_per_row) {
  const long long total = (long long)chunks * n_sel * vec_per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int part = (int)(t % vec_per_row);
    const long long row = t / vec_per_row;
    const int i = (int)(row % n_sel);
    const int c = (int)(row / n_sel);
    const long long src = ((long long)c * rows_per_chunk + idx[i]) * vec_per_row + part;
    const long long dst = ((long long)c * out_rows + i) * 2 * vec_per_row + part;
    kv_out[dst] = __ldg(k + src);
    kv_out[dst + vec_per_row] = __ldg(v + src);
  }
}

// dst row r (at byte offset dst_off inside a dst_stride-wide row) = src row idx[r]: 16-byte vectors, coalesced along rows
__global__ void rows_gather_kernel(const uint4* __restrict__ src, const int32_t* __restrict__ idx,
                                   uint4* __restrict__ dst, long long n_rows, int vec_per_row, int dst_stride_vec,
                                   int dst_off_vec) {
  const long long total = n_rows * vec_per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int part = (int)(t % vec_per_row);
    const long long r = t / vec_per_row;
    dst[r * dst_stride_vec + dst_off_vec + part] = __ldg(src + (long long)idx[r] * vec_per_row + part);
  }
}
// dst row idx[r] = src row r
__global__ void rows_scatter_kernel(const uint4* __restrict__ src, const int32_t* __restrict__ idx,
                                    uint4* __restrict__ dst, long long n_rows, int vec_per_row) {
  const long long total = n_rows * vec_per_row;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int part = (int)(t % vec_per_row);
    const long long r = t / vec_per_row;
    dst[(long long)idx[r] * vec_per_row + part] = __ldg(src + t);
  }
}

// =============================================================================================
// A5  temporal-guided attention  (src/diffusion_hacked.py:320-367)
// =============================================================================================
// The reference gathers q_raw / k_raw / attention-output rows along each flow trajectory into [2L, heads, N, d] tensors,
// runs an N x N masked SDPA per (trajectory, head) and gathers the result back -- about twelve full passes over
// [2N, L, C] tensors.  Here one CTA owns TPB trajectories of one CFG chunk: their 3 x N token rows (all heads, C halves
// each, contiguous in the token-major layout) are gathered into shared memory with fully coalesced 16-byte loads that
// are ALL in flight before anything is used (HBM-bound kernel: bytes in flight are what counts), every thread then
// computes ONE output row -- (trajectory, frame f, head h): N dot products of length d, a softmax over N held in
// registers, N x d accumulation -- and the rows go back through shared memory with coalesced 16-byte stores to the
// token the trajectory visits in frame f (fwd_map is a permutation, so every output row is written exactly once).
// The q row of a thread goes straight to registers (k and v rows are shared by the N x heads threads of a trajectory,
// q rows are not), which keeps shared memory at 2 N 2C bytes per trajectory and more CTAs on an SM.
// Algorithmic traffic: 3 reads + 1 write of [2N, L, C] fp16 + 8 B of index and N B of mask per (trajectory, frame).
template <int D, int NMAX>
__global__ void __launch_bounds__(256)
temporal_attn_rows_kernel(const __half* __restrict__ q_raw, const __half* __restrict__ k_raw,
                          const __half* __restrict__ v_src, __half* __restrict__ out,
                          const int64_t* __restrict__ fwd_map, const uint8_t* __restrict__ traj_mask, int frames,
                          int tokens, int heads, int tpb, float scale_log2, int in_row_vecs /* 16-byte vectors between
                          consecutive token rows of q/k/v (C/8 when dense) */) {
  extern __shared__ uint4 smem_rows[];
  constexpr int VPR = D / 8;                                   // 16-byte vectors per head row
  const int N = frames;
  const int C = heads * D;
  const int row_vecs = heads * VPR;                            // vectors per token row (all heads)
  const int traj_vecs = N * row_vecs;                          // vectors per trajectory per tensor
  const int blocks_per_chunk = (tokens + tpb - 1) / tpb;
  const int b = blockIdx.x / blocks_per_chunk;
  const int p0 = (blockIdx.x % blocks_per_chunk) * tpb;
  const int n_traj = min(tpb, tokens - p0);
  uint4* sk = smem_rows;                                       // [tpb][N][row_vecs]   (reused for the output rows)
  uint4* sv = sk + tpb * traj_vecs;
  int* spos = reinterpret_cast<int*>(sv + tpb * traj_vecs);    // [tpb][N] token visited in frame f

  for (int i = threadIdx.x; i < n_traj * N; i += blockDim.x) {
    const int tr = i / N, f = i % N;
    spos[tr * N + f] = (int)fwd_map[(long long)f * tokens + p0 + tr];
  }
  __syncthreads();
  // ---- this thread's output row (trajectory tr, frame f, head h): its q row goes straight to registers ...
  const int rows = n_traj * N * heads;                         // == blockDim.x rounded down (one row per thread)
  const int r = threadIdx.x;
  const bool active = r < rows;
  const int tr = active ? r / (N * heads) : 0, fh = active ? r % (N * heads) : 0;
  const int f = fh / heads, h = fh % heads;
  uint4 qraw[VPR];
  if (active) {
    const uint4* qrow = reinterpret_cast<const uint4*>(q_raw) +
                        (((long long)b * N + f) * tokens + spos[tr * N + f]) * in_row_vecs + h * VPR;
#pragma unroll
    for (int c = 0; c < VPR; ++c) qraw[c] = __ldg(qrow + c);
  }
  // ---- ... while the k and v rows of the CTA's trajectories are gathered cooperatively: consecutive threads read
  //      consecutive 16-byte pieces of a token row, all loads in flight before anything is used
  const int total_vecs = n_traj * traj_vecs;
  for (int i = threadIdx.x; i < total_vecs; i += blockDim.x) {
    const int t2 = i / traj_vecs, rem = i % traj_vecs;
    const int f2 = rem / row_vecs, part = rem % row_vecs;
    const long long src = (((long long)b * N + f2) * tokens + spos[t2 * N + f2]) * in_row_vecs + part;
    sk[i] = __ldg(reinterpret_cast<const uint4*>(k_raw) + src);
    sv[i] = __ldg(reinterpret_cast<const uint4*>(v_src) + src);
  }
  __syncthreads();
  uint4 orow[VPR];
  if (active) {
    float2 qv[D / 2];
#pragma unroll
    for (int c = 0; c < VPR; ++c) {
      const __half2* xh = reinterpret_cast<const __half2*>(&qraw[c]);
#pragma unroll
      for (int u = 0; u < 4; ++u) qv[c * 4 + u] = __half22float2(xh[u]);
    }
    const uint8_t* mrow = traj_mask + ((long long)(p0 + tr) * N + f) * N;
    float sc[NMAX];
    float mx = -INFINITY;
#pragma unroll
    for (int g = 0; g < NMAX; ++g) {
      sc[g] = -INFINITY;
      if (g < N) {
        const uint4* krow = sk + tr * traj_vecs + g * row_vecs + h * VPR;
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < VPR; ++c) {
          const uint4 y = krow[c];
          const __half2* yh = reinterpret_cast<const __half2*>(&y);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float2 yy = __half22float2(yh[u]);
            a0 = fmaf(qv[c * 4 + u].x, yy.x, a0);
            a1 = fmaf(qv[c * 4 + u].y, yy.y, a1);
          }
        }
        if (mrow[g]) sc[g] = (a0 + a1) * scale_log2;
        mx = fmaxf(mx, sc[g]);
      }
    }
    float l = 0.f;
#pragma unroll
    for (int g = 0; g < NMAX; ++g) {
      sc[g] = (g < N) ? fast_exp2(sc[g] - mx) : 0.f;             // (the diagonal is never masked: mx is finite)
      l += sc[g];
    }
    const float inv = 1.f / l;
    float2 acc[D / 2];
#pragma unroll
    for (int c = 0; c < D / 2; ++c) acc[c] = make_float2(0.f, 0.f);
#pragma unroll
    for (int g = 0; g < NMAX; ++g) {
      if (g < N) {
        const uint4* vrow = sv + tr * traj_vecs + g * row_vecs + h * VPR;
        const float pw = sc[g] * inv;
#pragma unroll
        for (int c = 0; c < VPR; ++c) {
          const uint4 y = vrow[c];
          const __half2* yh = reinterpret_cast<const __half2*>(&y);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float2 yy = __half22float2(yh[u]);
            acc[c * 4 + u].x = fmaf(pw, yy.x, acc[c * 4 + u].x);
            acc[c * 4 + u].y = fmaf(pw, yy.y, acc[c * 4 + u].y);
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < VPR; ++c) {
      orow[c].x = pack_half2(acc[c * 4 + 0].x, acc[c * 4 + 0].y);
      orow[c].y = pack_half2(acc[c * 4 + 1].x, acc[c * 4 + 1].y);
      orow[c].z = pack_half2(acc[c * 4 + 2].x, acc[c * 4 + 2].y);
      orow[c].w = pack_half2(acc[c * 4 + 3].x, acc[c * 4 + 3].y);
    }
  }
  __syncthreads();                                             // every k row has been read: stage the output rows there
  if (active) {
    uint4* dst = sk + tr * traj_vecs + f * row_vecs + h * VPR;
#pragma unroll
    for (int c = 0; c < VPR; ++c) dst[c] = orow[c];
  }
  __syncthreads();
  // ---- scatter back to the tokens the trajectories visit (coalesced 16-byte stores)
  for (int i = threadIdx.x; i < total_vecs; i += blockDim.x) {
    const int t2 = i / traj_vecs, rem = i % traj_vecs;
    const int f2 = rem / row_vecs, part = rem % row_vecs;
    const long long dst = (((long long)b * N + f2) * tokens + spos[t2 * N + f2]) * (C / 8) + part;
    reinterpret_cast<uint4*>(out)[dst] = sk[i];
  }
}

// any frames <= 64 / head_dim % 8 == 0: one CTA per (chunk, trajectory), one warp per head (round-1 kernel; kept for
// the shapes the row kernel is not instantiated for)
__global__ void temporal_attn_kernel(const __half* __restrict__ q_raw, const __half* __restrict__ k_raw,
                                     const __half* __restrict__ v_src, __half* __restrict__ out,
                                     const int64_t* __restrict__ fwd_map, const uint8_t* __restrict__ traj_mask,
                                     int frames, int tokens, int heads, int d, float scale) {
  extern __shared__ uint8_t smem_t[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = blockIdx.x % tokens;
  const int b = blockIdx.x / tokens;
  const int C = heads * d;
  const int N = frames;
  const int vpr = d / 8;                                       // 16-byte vectors per head row
  // per-warp shared: q,k,v as half [N][d], scores float [N][N]
  const size_t per_warp = (size_t)3 * N * d * sizeof(__half) + (size_t)N * N * sizeof(float);
  uint8_t* base = smem_t + warp * ((per_warp + 15) & ~size_t(15));
  __half* sq = reinterpret_cast<__half*>(base);
  __half* sk = sq + N * d;
  __half* sv = sk + N * d;
  float* sc = reinterpret_cast<float*>(sv + N * d);
  const int h = warp;

  const int nvec = N * vpr;
  for (int t = lane; t < 3 * nvec; t += 32) {
    const int which = t / nvec;
    const int rem = t % nvec;
    const int f = rem / vpr, part = rem % vpr;
    const long long pos = fwd_map[(long long)f * tokens + p];
    const __half* src = which == 0 ? q_raw : (which == 1 ? k_raw : v_src);
    const uint4 val = __ldg(reinterpret_cast<const uint4*>(src + (((long long)b * N + f) * tokens + pos) * C +
                                                           (long long)h * d) + part);
    reinterpret_cast<uint4*>(which == 0 ? sq : (which == 1 ? sk : sv))[rem] = val;
  }
  __syncwarp();
  const uint8_t* mrow = traj_mask + (long long)p * N * N;
  for (int pair = lane; pair < N * N; pair += 32) {
    const int f = pair / N, g = pair % N;
    const uint4* a = reinterpret_cast<const uint4*>(sq + f * d);      // 16-byte shared loads: 8 channels each
    const uint4* bb = reinterpret_cast<const uint4*>(sk + g * d);
    float acc = 0.f;
    for (int c = 0; c < vpr; ++c) {
      const uint4 xa = a[c], yb = bb[c];
      const __half2* xh = reinterpret_cast<const __half2*>(&xa);
      const __half2* yh = reinterpret_cast<const __half2*>(&yb);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float2 x = __half22float2(xh[u]);
        const float2 y = __half22float2(yh[u]);
        acc = fmaf(x.x, y.x, acc);
        acc = fmaf(x.y, y.y, acc);
      }
    }
    sc[pair] = mrow[pair] ? acc * scale : -INFINITY;
  }
  __syncwarp();
  for (int f = lane; f < N; f += 32) {                               // one softmax row per lane (frames may exceed 32)
    float* r = sc + f * N;
    float m = -INFINITY;
    for (int g = 0; g < N; ++g) m = fmaxf(m, r[g]);
    float s = 0.f;
    for (int g = 0; g < N; ++g) {
      const float e = __expf(r[g] - m);
      r[g] = e;
      s += e;
    }
    const float inv = 1.f / s;
    for (int g = 0; g < N; ++g) r[g] *= inv;
  }
  __syncwarp();
  for (int t = lane; t < nvec; t += 32) {                            // one (frame, 8-channel chunk) per lane
    const int f = t / vpr, part = t % vpr;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int g = 0; g < N; ++g) {
      const float pw = sc[f * N + g];
      const uint4 vv = reinterpret_cast<const uint4*>(sv + g * d)[part];
      const __half2* vh = reinterpret_cast<const __half2*>(&vv);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float2 y = __half22float2(vh[u]);
        acc[2 * u] = fmaf(pw, y.x, acc[2 * u]);
        acc[2 * u + 1] = fmaf(pw, y.y, acc[2 * u + 1]);
      }
    }
    uint4 o;
    o.x = pack_half2(acc[0], acc[1]);
    o.y = pack_half2(acc[2], acc[3]);
    o.z = pack_half2(acc[4], acc[5]);
    o.w = pack_half2(acc[6], acc[7]);
    reinterpret_cast<uint4*>(sq)[t] = o;                             // q is dead: reuse as the output staging
  }
  __syncwarp();
  for (int t = lane; t < nvec; t += 32) {
    const int f = t / vpr, part = t % vpr;
    const long long pos = fwd_map[(long long)f * tokens + p];
    reinterpret_cast<uint4*>(out + (((long long)b * N + f) * tokens + pos) * C + (long long)h * d)[part] =
        reinterpret_cast<const uint4*>(sq)[t];
  }
}

// =============================================================================================
// W3  bilinear flow warp  (gmflow/geometry.py:41-72)
// =============================================================================================
struct Taps {
  int i00, i01, i10, i11;        // plane offsets (clamped), -1 weight handled through w = 0
  float w00, w01, w10, w11;
};

__device__ __forceinline__ Taps make_taps(float x, float y, int h, int w) {
  Taps t;
  const float xf = floorf(x), yf = floorf(y);
  const float ax = x - xf, ay = y - yf;
  const int x0 = (int)xf, y0 = (int)yf, x1 = x0 + 1, y1 = y0 + 1;
  const bool vx0 = x0 >= 0 && x0 <= w - 1, vx1 = x1 >= 0 && x1 <= w - 1;
  const bool vy0 = y0 >= 0 && y0 <= h - 1, vy1 = y1 >= 0 && y1 <= h - 1;
  const int cx0 = min(max(x0, 0), w - 1), cx1 = min(max(x1, 0), w - 1);
  const int cy0 = min(max(y0, 0), h - 1), cy1 = min(max(y1, 0), h - 1);
  t.i00 = cy0 * w + cx0;
  t.i01 = cy0 * w + cx1;
  t.i10 = cy1 * w + cx0;
  t.i11 = cy1 * w + cx1;
  t.w00 = (vx0 && vy0) ? (1.f - ax) * (1.f - ay) : 0.f;
  t.w01 = (vx1 && vy0) ? ax * (1.f - ay) : 0.f;
  t.w10 = (vx0 && vy1) ? (1.f - ax) * ay : 0.f;
  t.w11 = (vx1 && vy1) ? ax * ay : 0.f;
  // NaN / inf coordinates (never produced by finite flows) sample nothing
  if (!(fabsf(x) < 1e9f) || !(fabsf(y) < 1e9f)) t.w00 = t.w01 = t.w10 = t.w11 = 0.f, t.i00 = t.i01 = t.i10 = t.i11 = 0;
  return t;
}

template <typename PlaneT>
__device__ __forceinline__ float sample_taps(const PlaneT* plane, const Taps& t) {
  return t.w00 * plane[t.i00] + t.w01 * plane[t.i01] + t.w10 * plane[t.i10] + t.w11 * plane[t.i11];
}

// four channels interleaved per pixel (the quad kernels' shared-memory planes)
struct __align__(8) half4 {
  __half2 lo, hi;
};
__device__ __forceinline__ float4 h4_to_f4(const half4& h) {
  const float2 a = __half22float2(h.lo), b = __half22float2(h.hi);
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 sample_taps4(const float4* plane, const Taps& t) {
  const float4 a0 = plane[t.i00], a1 = plane[t.i01], a2 = plane[t.i10], a3 = plane[t.i11];
  return make_float4(t.w00 * a0.x + t.w01 * a1.x + t.w10 * a2.x + t.w11 * a3.x,
                     t.w00 * a0.y + t.w01 * a1.y + t.w10 * a2.y + t.w11 * a3.y,
                     t.w00 * a0.z + t.w01 * a1.z + t.w10 * a2.z + t.w11 * a3.z,
                     t.w00 * a0.w + t.w01 * a1.w + t.w10 * a2.w + t.w11 * a3.w);
}
// fmaf(w, v, acc) for one channel or four
__device__ __forceinline__ float fma_acc(float w, float v, float acc) { return fmaf(w, v, acc); }
__device__ __forceinline__ float4 fma_acc(float w, const float4& v, const float4& acc) {
  return make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
}

// W1: one blend of the frame chain, z * (1 - m) + warp * m  (flow_utils.py:41-51); every chain kernel blends through
// these, so they agree element for element
__device__ __forceinline__ float chain_blend(float z, float warped, float m) { return z * (1.f - m) + warped * m; }
__device__ __forceinline__ float4 chain_blend(const float4& z, const float4& warped, float m) {
  return make_float4(chain_blend(z.x, warped.x, m), chain_blend(z.y, warped.y, m), chain_blend(z.z, warped.z, m),
                     chain_blend(z.w, warped.w, m));
}

// ---- O2 (temporal-consistency loss): the steps the three loss kernels share.  The frame-sharded optimize_feature is
//      bit-identical to the unsharded call only because every loss kernel sums in the fixed order written here.

// One row of a warp adjoint in ELL form, as ops._pack_adjoint / ops._pack_ell build it: 8 uint32 slots per destination
// pixel (two uint4), each (weight as unorm16) << 16 | (source pixel as u16).  A row's used slots come first, and a
// slot whose weight field is 0 ends the row; unused slots are all-zero (weight 0, source 0), so reading one adds 0.
struct EllRow {
  uint32_t e[8];
};
__device__ __forceinline__ EllRow ell_load_row(const uint4* __restrict__ ell, int q) {
  const uint4 e0 = __ldg(ell + 2 * q), e1 = __ldg(ell + 2 * q + 1);
  return {{e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w}};
}
__device__ __forceinline__ bool ell_used(uint32_t slot) { return (slot >> 16) != 0; }
__device__ __forceinline__ float ell_weight(uint32_t slot) { return (float)(slot >> 16) * (1.0f / 65535.0f); }
__device__ __forceinline__ int ell_source(uint32_t slot) { return slot & 0xffffu; }

// Overflow list of a warp adjoint: [n_ovf][3] int32 (destination, source, float bits of the weight) for the taps past
// the 8 ELL slots of their destination, sorted by destination; -1 pads the tail.  The thread that holds the head of a
// run sums the whole run in list order, with no atomics, so the result does not depend on scheduling.
// value(source) is the sign plane at a source pixel: a float, or a float4 for a channel quad.
__device__ __forceinline__ bool ovf_run_head(const int32_t* __restrict__ o, int e) {
  return o[3 * e] >= 0 && (e == 0 || o[3 * (e - 1)] != o[3 * e]);
}
template <typename Value>
__device__ __forceinline__ auto ovf_run_sum(const int32_t* __restrict__ o, int n_ovf, int e, Value value) {
  decltype(value(0)) acc{};
  for (int e2 = e; e2 < n_ovf && o[3 * e2] == o[3 * e]; ++e2)
    acc = fma_acc(-__int_as_float(o[3 * e2 + 2]), value(o[3 * e2 + 1]), acc);
  return acc;
}

// Frame f of the walk is paired with frame f + 1; after the last frame comes frame 0 (closed ring) or, in the open chain
// of a frame-sharded batch, index `frames`, which the kernels' loaders read as the halo plane.
__device__ __forceinline__ int next_frame(int f, int frames, bool open_chain) {
  return (f + 1 == frames) ? (open_chain ? frames : 0) : f + 1;
}

// The gradient of frame f is its term ga of pair f plus the carry, what it received as the "next" frame of pair f - 1,
// as two rounded products and one add: fl(fl(ga k) + fl(carry k)), never fl((ga + carry) k).  Frame 0 of the closed
// ring receives carry_term() of the last pair in a second pass (add_carry); the open chain writes carry_term() to
// halo_grad, and optimize_feature adds it to the next shard's first frame (`grad[:, 0] += from_prev`), which is the
// same add, so the sharded gradient has the unsharded bits.
__device__ __forceinline__ float carry_term(float carry, float k) { return __fmul_rn(carry, k); }
__device__ __forceinline__ float add_carry(float g, float carry, float k) { return __fadd_rn(g, carry_term(carry, k)); }
__device__ __forceinline__ float grad_term(float ga, float carry, float k) {
  return __fadd_rn(__fmul_rn(ga, k), carry_term(carry, k));
}

// *loss_acc += k * (sum of every thread's loss in the CTA): warp sums, then one float atomic per CTA.  Every thread of
// the CTA calls it.
__device__ __forceinline__ void cta_loss_add(float loss, float* loss_acc, float k) {
  __shared__ float red[32];
  loss = warp_sum(loss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = loss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < ((blockDim.x + 31) >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(loss_acc, v * k);
  }
}

__global__ void flow_warp_kernel(const float* __restrict__ src, const float* __restrict__ flow,
                                 float* __restrict__ dst, int batch, int channels, int h, int w, int flow_batch) {
  const int hw = h * w;
  const long long total = (long long)batch * hw;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int pix = (int)(t % hw);
    const int b = (int)(t / hw);
    const int x = pix % w, y = pix / w;
    const float* fl = flow + (long long)(b % flow_batch) * 2 * hw;
    const Taps tp = make_taps(x + fl[pix], y + fl[hw + pix], h, w);
    const float* s = src + (long long)b * channels * hw;
    float* d = dst + (long long)b * channels * hw;
    for (int c = 0; c < channels; ++c) d[(long long)c * hw + pix] = sample_taps(s + (long long)c * hw, tp);
  }
}

// =============================================================================================
// W1  warp_tensor frame chain  (src/flow_utils.py:41-51)
// =============================================================================================
template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ld_as_float<__half>(const __half* p) { return __half2float(*p); }
template <typename T>
__device__ __forceinline__ void st_from_float(T* p, float v);
template <>
__device__ __forceinline__ void st_from_float<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void st_from_float<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// K (chunk, channel) planes per CTA keep their running frames in shared memory (fp32, like the reference's
// `latent = sample.to(float32)`), so the N-1 dependent blends are block-local.  The per-pixel work that does not
// depend on the channel (two flow loads, the four bilinear taps, the blend weight) is done ONCE per pixel and applied
// to the K planes.
template <typename T, int K>
__global__ void __launch_bounds__(512)
warp_chain_group_kernel(const T* __restrict__ sample, T* __restrict__ out, const float* __restrict__ bwd_flow,
                        const float* __restrict__ fwd_flow_last, const float* __restrict__ blend, int frames,
                        int channels, int planes_total, int h, int w) {
  extern __shared__ float planes[];
  const int hw = h * w;
  float* cur = planes;                     // [K][hw]
  float* nxt = planes + K * hw;            // [K][hw]
  long long base[K];                       // offset of frame 0 of plane kk; frames are channels*hw apart
  bool live[K];
#pragma unroll
  for (int kk = 0; kk < K; ++kk) {
    const int pl = blockIdx.x * K + kk;
    live[kk] = pl < planes_total;
    const int j = live[kk] ? pl / channels : 0, c = live[kk] ? pl % channels : 0;
    base[kk] = ((long long)j * frames * channels + c) * hw;
  }
  const long long fstride = (long long)channels * hw;

  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
      if (!live[kk]) continue;
      const float v = ld_as_float(sample + base[kk] + i);
      cur[kk * hw + i] = v;
      st_from_float(out + base[kk] + i, v);
    }
  }
  __syncthreads();
  for (int ii = 0; ii + 1 < frames; ++ii) {
    const float* fl = bwd_flow + (long long)ii * 2 * hw;
    const float* mk = blend + (long long)ii * hw;
    const bool last = (ii + 2 == frames);
    const long long foff = (long long)(ii + 1) * fstride;
    for (int i = threadIdx.x; i < hw; i += blockDim.x) {
      const int x = i % w, y = i / w;
      const Taps tp = make_taps(x + fl[i], y + fl[hw + i], h, w);
      const float m = mk[i];
      float z[K];
#pragma unroll
      for (int kk = 0; kk < K; ++kk) z[kk] = live[kk] ? ld_as_float(sample + base[kk] + foff + i) : 0.f;
#pragma unroll
      for (int kk = 0; kk < K; ++kk) {
        const float v = chain_blend(z[kk], sample_taps(cur + kk * hw, tp), m);
        nxt[kk * hw + i] = v;
        if (!last && live[kk]) st_from_float(out + base[kk] + foff + i, v);
      }
    }
    __syncthreads();
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  // closing blend: frame N-1 <- warp(frame 0, fwd_flow[N-1])  (flow_utils.py:47-51)
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
#pragma unroll
    for (int kk = 0; kk < K; ++kk) nxt[kk * hw + i] = live[kk] ? ld_as_float(sample + base[kk] + i) : 0.f;
  }
  __syncthreads();
  const float* mk = blend + (long long)(frames - 1) * hw;
  const long long loff = (long long)(frames - 1) * fstride;
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
    const int x = i % w, y = i / w;
    const Taps tp = make_taps(x + fwd_flow_last[i], y + fwd_flow_last[hw + i], h, w);
    const float m = mk[i];
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
      const float c = cur[kk * hw + i];
      const float v = chain_blend(c, sample_taps(nxt + kk * hw, tp), m);
      if (live[kk]) st_from_float(out + base[kk] + loff + i, v);
    }
  }
}

// Channel-QUAD variant (the one warp_tensor runs on decoder features; see warp_loss_quad_kernel below for the
// measurement behind it): NQ quads of four (chunk, channel) planes per CTA, interleaved per pixel as float4 in shared
// memory, so the flows / blend weight of a pixel are fetched and its taps built once for 4 NQ channels and one 16-byte
// shared load serves a tap for four of them.  Same arithmetic per element as warp_chain_group_kernel (chain_blend).
template <typename T, int P, int NQ>
__global__ void __launch_bounds__(1024, 1)
warp_chain_quad_kernel(const T* __restrict__ sample, T* __restrict__ out, const float* __restrict__ bwd_flow,
                       const float* __restrict__ fwd_flow_last, const float* __restrict__ blend, int frames,
                       int channels, int h, int w) {
  extern __shared__ float4 chq[];
  const int hw = h * w;
  float4* cur = chq;                       // [NQ][hw]
  float4* nxt = chq + NQ * hw;             // [NQ][hw]
  const int T_ = blockDim.x, t = threadIdx.x;
  const int pl0 = blockIdx.x * 4 * NQ;
  const int j = pl0 / channels, c0 = pl0 % channels;
  const long long fstride = (long long)channels * hw;
  const long long base = ((long long)j * frames * channels + c0) * hw;
  auto ld4 = [&](const T* src, int q) {
    return make_float4(ld_as_float(src + q), ld_as_float(src + hw + q), ld_as_float(src + 2 * hw + q),
                       ld_as_float(src + 3 * hw + q));
  };
  auto st4 = [&](T* dst, int q, const float4& v) {
    st_from_float(dst + q, v.x), st_from_float(dst + hw + q, v.y), st_from_float(dst + 2 * hw + q, v.z),
        st_from_float(dst + 3 * hw + q, v.w);
  };
#pragma unroll
  for (int pp = 0; pp < P; ++pp) {
    const int q = t + pp * T_;
    if (q < hw) {
#pragma unroll
      for (int nq = 0; nq < NQ; ++nq) {
        const float4 v = ld4(sample + base + (long long)nq * 4 * hw, q);
        cur[nq * hw + q] = v;
        st4(out + base + (long long)nq * 4 * hw, q, v);
      }
    }
  }
  __syncthreads();
  for (int ii = 0; ii + 1 < frames; ++ii) {
    const float* fl = bwd_flow + (long long)ii * 2 * hw;
    const float* mk = blend + (long long)ii * hw;
    const bool last = (ii + 2 == frames);
    const long long foff = (long long)(ii + 1) * fstride;
#pragma unroll
    for (int pp = 0; pp < P; ++pp) {
      const int q = t + pp * T_;
      if (q >= hw) continue;
      const Taps tp = make_taps((q % w) + __ldg(fl + q), (q / w) + __ldg(fl + hw + q), h, w);
      const float m = __ldg(mk + q);
#pragma unroll
      for (int nq = 0; nq < NQ; ++nq) {
        const float4 z = ld4(sample + base + foff + (long long)nq * 4 * hw, q);
        const float4 v = chain_blend(z, sample_taps4(cur + nq * hw, tp), m);
        nxt[nq * hw + q] = v;
        if (!last) st4(out + base + foff + (long long)nq * 4 * hw, q, v);
      }
    }
    __syncthreads();
    float4* tmp = cur;
    cur = nxt;
    nxt = tmp;
  }
  // closing blend: frame N-1 <- warp(frame 0, fwd_flow[N-1])  (flow_utils.py:47-51)
#pragma unroll
  for (int pp = 0; pp < P; ++pp) {
    const int q = t + pp * T_;
    if (q < hw) {
#pragma unroll
      for (int nq = 0; nq < NQ; ++nq) nxt[nq * hw + q] = ld4(sample + base + (long long)nq * 4 * hw, q);
    }
  }
  __syncthreads();
  {
    const float* mk = blend + (long long)(frames - 1) * hw;
    const long long loff = (long long)(frames - 1) * fstride;
#pragma unroll
    for (int pp = 0; pp < P; ++pp) {
      const int q = t + pp * T_;
      if (q >= hw) continue;
      const Taps tp = make_taps((q % w) + __ldg(fwd_flow_last + q), (q / w) + __ldg(fwd_flow_last + hw + q), h, w);
      const float m = __ldg(mk + q);
#pragma unroll
      for (int nq = 0; nq < NQ; ++nq) {
        const float4 c = cur[nq * hw + q];
        st4(out + base + loff + (long long)nq * 4 * hw, q, chain_blend(c, sample_taps4(nxt + nq * hw, tp), m));
      }
    }
  }
}

// planes too large for shared memory (image resolution): one launch per chain step, fp32 scratch
__global__ void warp_blend_step_kernel(const float* __restrict__ src_frames, float* __restrict__ dst_frames,
                                       const float* __restrict__ flow, const float* __restrict__ mask, int chunks,
                                       int frames, int channels, int h, int w, int src_f, int dst_f) {
  const int hw = h * w;
  const long long total = (long long)chunks * channels * hw;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t % hw);
    const int c = (int)((t / hw) % channels);
    const int j = (int)(t / ((long long)hw * channels));
    const int x = i % w, y = i / w;
    const Taps tp = make_taps(x + flow[i], y + flow[hw + i], h, w);
    const float m = mask[i];
    const float* s = src_frames + ((long long)(j * frames + src_f) * channels + c) * hw;
    float* d = dst_frames + ((long long)(j * frames + dst_f) * channels + c) * hw;
    const float warped = sample_taps(s, tp);
    d[i] = chain_blend(d[i], warped, m);
  }
}

// =============================================================================================
// O2  temporal-consistency loss forward + backward  (src/diffusion_hacked.py:461-466)
// one CTA per (chunk, channel); frame pairs are walked sequentially with both planes in shared memory.
// The backward of the bilinear warp (the adjoint W^T, a scatter-add in autograd) is evaluated as a GATHER:
// W^T is the same sparse matrix for all chunks*channels planes of a frame pair, so it is built once per batch
// (warp_taps_kernel + a sort on the host) in ELL form (ell_load_row), and every plane just reads it: no atomics and
// no data-dependent loop in the per-iteration kernel.  Destinations hit by more than 8 taps go to a small overflow
// list (ovf_run_sum).
// =============================================================================================
__global__ void warp_taps_kernel(const float* __restrict__ flow, int32_t* __restrict__ dest,
                                 float* __restrict__ weight, int frames, int h, int w) {
  const int hw = h * w;
  const long long total = (long long)frames * hw;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(t % hw);
    const int f = (int)(t / hw);
    const float* fl = flow + (long long)f * 2 * hw;
    const Taps tp = make_taps((i % w) + fl[i], (i / w) + fl[hw + i], h, w);
    const int idx[4] = {tp.i00, tp.i01, tp.i10, tp.i11};
    const float wt[4] = {tp.w00, tp.w01, tp.w10, tp.w11};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      dest[t * 4 + k] = wt[k] != 0.f ? idx[k] : -1;
      weight[t * 4 + k] = wt[k];
    }
  }
}

__global__ void warp_loss_kernel(const float* __restrict__ cs, const float* __restrict__ fwd_flow,
                                 const float* __restrict__ bwd_flow, const float* __restrict__ fwd_keep,
                                 const float* __restrict__ bwd_keep, const uint4* __restrict__ bwd_ell,
                                 const uint4* __restrict__ fwd_ell, const int32_t* __restrict__ ovf /*[2][frames][n_ovf][3]*/,
                                 int n_ovf, float* __restrict__ grad, float* __restrict__ loss_acc, int accumulate,
                                 int frames, int channels, int h, int w, float k /* 2 / numel */,
                                 const float* __restrict__ halo_cs, float* __restrict__ halo_grad) {
  // halo_cs != null: OPEN chain (frame-sharded batch) -- the "next" frame of the last pair is the halo plane
  // [chunks, channels, h, w] (the following rank's first frame) and what it receives goes to halo_grad, overwritten
  extern __shared__ float sm[];
  const int hw = h * w;
  float* c1 = sm;
  float* c2 = sm + hw;
  float* s1 = sm + 2 * hw;          // sign(c2 - W_bf c1) * keep_b * k
  float* s2 = sm + 3 * hw;          // sign(c1 - W_ff c2) * keep_f * k
  const int c = blockIdx.x % channels;
  const int b = blockIdx.x / channels;
  auto plane_of = [&](int f) { return ((long long)(b * frames + f) * channels + c) * hw; };
  float loss = 0.f;

  for (int i = threadIdx.x; i < hw; i += blockDim.x) c2[i] = cs[plane_of(0) + i];
  for (int f = 0; f < frames; ++f) {
    const int fn = (f + 1) % frames;
    const bool to_halo = halo_cs != nullptr && f + 1 == frames;
    const long long halo_off = ((long long)b * channels + c) * hw;
    float* t = c1;
    c1 = c2;                                                    // previous "next" plane becomes c1
    c2 = t;
    __syncthreads();
    {
      const float* nsrc = to_halo ? halo_cs + halo_off : cs + plane_of(fn);
      for (int i = threadIdx.x; i < hw; i += blockDim.x) c2[i] = nsrc[i];
    }
    __syncthreads();
    const float* bf = bwd_flow + (long long)f * 2 * hw;
    const float* ff = fwd_flow + (long long)f * 2 * hw;
    const float* mb = bwd_keep + (long long)f * hw;
    const float* mf = fwd_keep + (long long)f * hw;
    // pixel coordinates advance incrementally (no integer division in the loop)
    const int dx = blockDim.x % w, dy = blockDim.x / w;
    int x = threadIdx.x % w, y = threadIdx.x / w;
#pragma unroll 2
    for (int i = threadIdx.x; i < hw; i += blockDim.x, x += dx, y += dy) {
      if (x >= w) {
        x -= w;
        ++y;
      }
      {  // r1 = c2 - W_bf(c1)
        const Taps tp = make_taps(x + bf[i], y + bf[hw + i], h, w);
        const float r = c2[i] - sample_taps(c1, tp);
        const float m = mb[i];
        loss += fabsf(r) * m;
        s1[i] = sgnf(r) * m * k;
      }
      {  // r2 = c1 - W_ff(c2)
        const Taps tp = make_taps(x + ff[i], y + ff[hw + i], h, w);
        const float r = c1[i] - sample_taps(c2, tp);
        const float m = mf[i];
        loss += fabsf(r) * m;
        s2[i] = sgnf(r) * m * k;
      }
    }
    __syncthreads();
    const bool a_add = accumulate || f > 0;                     // frame f   : first touched at f == 0
    const bool b_add = !to_halo && (accumulate || f == frames - 1);   // frame f+1 : first touched here, except the wrap to 0
    // adjoint as a gather through the ELL rows: all 8 slots of a row, unconditionally (an unused slot adds 0)
    const uint4* eb = bwd_ell + (long long)f * hw * 2;
    const uint4* ef = fwd_ell + (long long)f * hw * 2;
    float* ga = grad + plane_of(f);
    float* gb = to_halo ? halo_grad + halo_off : grad + plane_of(fn);
    auto gather8 = [&](const uint4* ell, int q, const float* sv) {
      const EllRow r = ell_load_row(ell, q);
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(ell_weight(r.e[j]), sv[ell_source(r.e[j])], acc);
      return acc;
    };
    // d/dc1 = s2 - W_bf^T s1      (frame f)
#pragma unroll 4
    for (int q = threadIdx.x; q < hw; q += blockDim.x) {
      const float acc = s2[q] - gather8(eb, q, s1);
      ga[q] = a_add ? ga[q] + acc : acc;
    }
    if (frames <= 2) __syncthreads();                           // ga / gb alias the same two planes
    // d/dc2 = s1 - W_ff^T s2      (frame f+1)
#pragma unroll 4
    for (int q = threadIdx.x; q < hw; q += blockDim.x) {
      const float acc = s1[q] - gather8(ef, q, s2);
      gb[q] = b_add ? gb[q] + acc : acc;
    }
    if (n_ovf > 0) {                                            // destinations hit by more than 8 taps (rare)
      __syncthreads();
      const int32_t* ob = ovf + ((long long)0 * frames + f) * n_ovf * 3;
      const int32_t* of = ovf + ((long long)1 * frames + f) * n_ovf * 3;
      for (int e = threadIdx.x; e < n_ovf; e += blockDim.x)
        if (ovf_run_head(ob, e)) ga[ob[3 * e]] += ovf_run_sum(ob, n_ovf, e, [&](int src) { return s1[src]; });
      __syncthreads();                                          // (frames <= 2: ga and gb may be the same plane)
      for (int e = threadIdx.x; e < n_ovf; e += blockDim.x)
        if (ovf_run_head(of, e)) gb[of[3 * e]] += ovf_run_sum(of, n_ovf, e, [&](int src) { return s2[src]; });
    }
  }
  if (loss_acc != nullptr) cta_loss_add(loss, loss_acc, k);
}

// ---------------------------------------------------------------------------------------------
// Channel-grouped temporal-consistency loss (the kernel optimize_feature runs).
// Everything that depends on the pixel but not on the channel -- two flows, eight bilinear taps, two keep masks and the
// two ELL rows of the warp adjoints (88 bytes per pixel and frame pair) -- is fetched and decoded ONCE per pixel and
// applied to KT planes held by the same thread; a CTA walks the N frame pairs of K = KT * G (chunk, channel) planes with
// four shared-memory planes per channel (frame f, frame f+1 in fp32; the two masked sign planes in fp16 -- exact for the
// {0,1} keep masks the reference produces, 2^-11 relative otherwise).  Every cs plane is read once and every grad plane
// is written once: the contribution a frame receives as the "next" frame of pair f is carried IN REGISTERS to pair f+1,
// where the same thread owns the same (pixel, plane) elements (frame 0 alone gets a second, read-modify-write pass for
// the wrap-around pair).  Algorithmic traffic: 8 bytes per element (read cs, write grad) + 1/N of that for frame 0.
//   thread mapping: hw >= blockDim: thread t owns pixels t + pp * blockDim (pp < P) of KT planes;
//                   hw <  blockDim: G = blockDim / hw sub-groups; thread (q = t % hw, g = t / hw) owns pixel q of planes
//                   kk * G + g (kk < KT).
// ---------------------------------------------------------------------------------------------
template <int P, int KT>
__global__ void __launch_bounds__(512, 2)
warp_loss_group_kernel(const float* __restrict__ cs, const float* __restrict__ fwd_flow,
                       const float* __restrict__ bwd_flow, const float* __restrict__ fwd_keep,
                       const float* __restrict__ bwd_keep, const uint4* __restrict__ bwd_ell,
                       const uint4* __restrict__ fwd_ell, const int32_t* __restrict__ ovf /*[2][frames][n_ovf][3]*/,
                       int n_ovf, float* __restrict__ grad, float* __restrict__ loss_acc, int accumulate, int frames,
                       int channels, int planes_total, int h, int w, int G, float k /* 2 / numel */,
                       const float* __restrict__ halo_cs, float* __restrict__ halo_grad /* open chain, see warp_loss_kernel */) {
  extern __shared__ float sm[];
  const int hw = h * w;
  const int K = KT * G;
  float* cur = sm;                                            // [K][hw] frame f
  float* nxt = sm + K * hw;                                   // [K][hw] frame f + 1
  __half* s1 = reinterpret_cast<__half*>(sm + 2 * K * hw);    // [K][hw] sign(c2 - W_bf c1) * keep_b
  __half* s2 = s1 + K * hw;                                   // [K][hw] sign(c1 - W_ff c2) * keep_f
  const int T = blockDim.x;
  const int t = threadIdx.x;
  const int g = (G > 1) ? t / hw : 0;
  const int q0 = (G > 1) ? t % hw : t;
  const bool active = g < G;
  const long long fstride = (long long)channels * hw;
  // global offset of frame 0 of the planes this thread owns, and of every plane of the CTA (for the cooperative loads)
  long long own_base[KT];
  bool own_live[KT];
#pragma unroll
  for (int kk = 0; kk < KT; ++kk) {
    const int slot = kk * G + g;
    const int pl = blockIdx.x * K + slot;
    own_live[kk] = active && pl < planes_total;
    const int b = own_live[kk] ? pl / channels : 0, c = own_live[kk] ? pl % channels : 0;
    own_base[kk] = ((long long)b * frames * channels + c) * hw;
  }
  auto load_plane = [&](float* dst, int f) {                  // frame f of all K planes -> dst (coalesced along pixels)
    for (int idx = t; idx < K * hw; idx += T) {                 // f == frames: the halo plane (open chain)
      const int slot = idx / hw, i = idx - slot * hw;
      const int pl = blockIdx.x * K + slot;
      float v = 0.f;
      if (pl < planes_total) {
        const int b = pl / channels, c = pl % channels;
        v = (f == frames) ? halo_cs[((long long)b * channels + c) * hw + i]
                          : cs[((long long)(b * frames + f) * channels + c) * hw + i];
      }
      dst[idx] = v;
    }
  };
  float carry[P * KT];
#pragma unroll
  for (int j = 0; j < P * KT; ++j) carry[j] = 0.f;
  float loss = 0.f;

  load_plane(cur, 0);
  for (int f = 0; f < frames; ++f) {
    const int fn = next_frame(f, frames, halo_cs != nullptr);
    load_plane(nxt, fn);
    __syncthreads();
    // ---- residuals of pair (f, fn): taps once per pixel, applied to the KT planes of this thread
    {
      const float* bf = bwd_flow + (long long)f * 2 * hw;
      const float* ff = fwd_flow + (long long)f * 2 * hw;
      const float* mbp = bwd_keep + (long long)f * hw;
      const float* mfp = fwd_keep + (long long)f * hw;
#pragma unroll
      for (int pp = 0; pp < P; ++pp) {
        const int q = q0 + pp * T;
        if (!active || q >= hw) continue;
        const int x = q % w, y = q / w;
        const Taps tb = make_taps(x + bf[q], y + bf[hw + q], h, w);
        const Taps tf = make_taps(x + ff[q], y + ff[hw + q], h, w);
        const float mb = mbp[q], mf = mfp[q];
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) {
          const int slot = kk * G + g;
          const float* c1 = cur + slot * hw;
          const float* c2 = nxt + slot * hw;
          const float r1 = c2[q] - sample_taps(c1, tb);       // c2 - W_bf(c1)
          const float r2 = c1[q] - sample_taps(c2, tf);       // c1 - W_ff(c2)
          loss += fabsf(r1) * mb + fabsf(r2) * mf;
          s1[slot * hw + q] = __float2half_rn(sgnf(r1) * mb);
          s2[slot * hw + q] = __float2half_rn(sgnf(r2) * mf);
        }
      }
    }
    __syncthreads();
    // ---- destinations hit by more than 8 taps of the backward-flow warp: their extra terms of d/dc1 (frame f) go
    //      through the dead frame-f planes and join ga BEFORE it meets the carry (grad_term)
    if (n_ovf > 0) {
      for (int idx = t; idx < K * hw; idx += T) cur[idx] = 0.f;
      __syncthreads();
      const int32_t* ob = ovf + ((long long)0 * frames + f) * n_ovf * 3;
      for (int e = t; e < n_ovf; e += T) {
        if (!ovf_run_head(ob, e)) continue;
        for (int slot = 0; slot < K; ++slot)
          cur[slot * hw + ob[3 * e]] = ovf_run_sum(ob, n_ovf, e, [&](int src) { return __half2float(s1[slot * hw + src]); });
      }
      __syncthreads();
    }
    // ---- adjoints as gathers through the ELL rows, each decoded once per pixel for the KT planes; unused slots skipped
    const uint4* ebp = bwd_ell + (long long)f * hw * 2;
    const uint4* efp = fwd_ell + (long long)f * hw * 2;
    const long long goff_a = (long long)f * fstride;
#pragma unroll
    for (int pp = 0; pp < P; ++pp) {
      const int q = q0 + pp * T;
      if (!active || q >= hw) continue;
      float ga[KT], gb[KT];
#pragma unroll
      for (int kk = 0; kk < KT; ++kk) {
        const int slot = kk * G + g;
        ga[kk] = __half2float(s2[slot * hw + q]);             // d/dc1 = s2 - W_bf^T s1   (frame f)
        gb[kk] = __half2float(s1[slot * hw + q]);             // d/dc2 = s1 - W_ff^T s2   (frame fn)
        if (n_ovf > 0) ga[kk] += cur[slot * hw + q];
      }
      const EllRow rb = ell_load_row(ebp, q);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (!ell_used(rb.e[j])) continue;
        const float wj = ell_weight(rb.e[j]);
        const int src = ell_source(rb.e[j]);
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) ga[kk] = fmaf(-wj, __half2float(s1[(kk * G + g) * hw + src]), ga[kk]);
      }
      const EllRow rf = ell_load_row(efp, q);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (!ell_used(rf.e[j])) continue;
        const float wj = ell_weight(rf.e[j]);
        const int src = ell_source(rf.e[j]);
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) gb[kk] = fmaf(-wj, __half2float(s2[(kk * G + g) * hw + src]), gb[kk]);
      }
#pragma unroll
      for (int kk = 0; kk < KT; ++kk) {
        if (own_live[kk]) {
          float* dst = grad + own_base[kk] + goff_a + q;
          const float val = grad_term(ga[kk], carry[pp * KT + kk], k);
          *dst = accumulate ? *dst + val : val;
        }
        carry[pp * KT + kk] = gb[kk];
      }
    }
    // ---- destinations with more than 8 taps of the forward-flow warp: extra terms of d/dc2, added to the carry
    if (n_ovf > 0) {
      __syncthreads();
      for (int idx = t; idx < K * hw; idx += T) cur[idx] = 0.f;
      __syncthreads();
      const int32_t* of = ovf + ((long long)1 * frames + f) * n_ovf * 3;
      for (int e = t; e < n_ovf; e += T) {
        if (!ovf_run_head(of, e)) continue;
        for (int slot = 0; slot < K; ++slot)
          cur[slot * hw + of[3 * e]] = ovf_run_sum(of, n_ovf, e, [&](int src) { return __half2float(s2[slot * hw + src]); });
      }
      __syncthreads();
#pragma unroll
      for (int pp = 0; pp < P; ++pp) {
        const int q = q0 + pp * T;
        if (!active || q >= hw) continue;
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) carry[pp * KT + kk] += cur[(kk * G + g) * hw + q];
      }
    }
    __syncthreads();                                           // s1 / s2 / cur are rewritten by the next pair
    float* tmp = cur;                                          // frame fn becomes frame f of the next pair
    cur = nxt;
    nxt = tmp;
  }
  // ---- wrap-around: what frame 0 receives as the "next" frame of pair N-1
#pragma unroll
  for (int pp = 0; pp < P; ++pp) {
    const int q = q0 + pp * T;
    if (!active || q >= hw) continue;
#pragma unroll
    for (int kk = 0; kk < KT; ++kk)
      if (own_live[kk]) {
        if (halo_grad != nullptr) {                            // open chain: the following rank's first frame receives it
          const int pl = blockIdx.x * K + kk * G + g;
          halo_grad[((long long)(pl / channels) * channels + pl % channels) * hw + q] = carry_term(carry[pp * KT + kk], k);
        } else {
          grad[own_base[kk] + q] = add_carry(grad[own_base[kk] + q], carry[pp * KT + kk], k);
        }
      }
  }
  if (loss_acc != nullptr) cta_loss_add(loss, loss_acc, k);
}

// ---------------------------------------------------------------------------------------------
// Channel-QUAD temporal-consistency loss: the kernel optimize_feature runs when the planes fit shared memory.
// Round-2 measurements: the two kernels above and a first quad kernel all moved ~3.4 TB/s from L2 whatever their
// structure -- the per-(pair, pixel) operands (two flows, two keep masks, two 32-byte ELL rows: 88 bytes) are re-read by
// every CTA for every frame pair and dwarf the 8 bytes per (pixel, channel) of payload.  So a CTA takes as many channels
// as shared memory allows -- NQ quads of four (chunk, channel) planes, interleaved per pixel: frame f and f+1 as float4,
// the two masked sign planes as 4 x fp16, 48 bytes per pixel and quad -- and everything that depends on the pixel only
// (taps from the flows, keep masks, ELL rows) is fetched and decoded once per pixel for all 4 NQ channels; a 16-byte
// (8-byte) shared load serves a tap for four channels.  Every thread owns P pixels for the whole walk over the frame
// pairs; what a frame receives as the "next" frame of pair f is carried in registers to pair f+1 (each cs plane read
// once, each grad plane written once, frame 0 once more for the wrap-around pair).
// ---------------------------------------------------------------------------------------------
template <int P, int NQ>
__global__ void __launch_bounds__(1024, 1)
warp_loss_quad_kernel(const float* __restrict__ cs, const float* __restrict__ fwd_flow,
                      const float* __restrict__ bwd_flow, const float* __restrict__ fwd_keep,
                      const float* __restrict__ bwd_keep, const uint4* __restrict__ bwd_ell,
                      const uint4* __restrict__ fwd_ell, const int32_t* __restrict__ ovf /*[2][frames][n_ovf][3]*/,
                      int n_ovf, float* __restrict__ grad, float* __restrict__ loss_acc, int accumulate, int frames,
                      int channels, int h, int w, float k, const float* __restrict__ halo_cs,
                      float* __restrict__ halo_grad /* open chain, see warp_loss_kernel */) {
  extern __shared__ float4 smq[];
  const int hw = h * w;
  float4* cur = smq;                                          // [NQ][hw] frame f,     4 channels per pixel
  float4* nxt = smq + NQ * hw;                                // [NQ][hw] frame f + 1
  half4* s1 = reinterpret_cast<half4*>(smq + 2 * NQ * hw);    // [NQ][hw] sign(c2 - W_bf c1) * keep_b
  half4* s2 = s1 + NQ * hw;                                   // [NQ][hw] sign(c1 - W_ff c2) * keep_f
  const int T = blockDim.x, t = threadIdx.x;
  const int pl0 = blockIdx.x * 4 * NQ;                        // first (chunk, channel) plane; channels % (4 NQ) == 0
  const int b = pl0 / channels, c0 = pl0 % channels;
  const long long fstride = (long long)channels * hw;
  const long long base = ((long long)b * frames * channels + c0) * hw;      // frame 0, channel c0
  const long long halo_base = ((long long)b * channels + c0) * hw;            // halo planes: [chunks, channels, h, w]
  auto load_frame = [&](float4* dst, int f) {                                 // f == frames: the halo plane (open chain)
    const float* src = (f == frames) ? halo_cs + halo_base : cs + base + (long long)f * fstride;
#pragma unroll
    for (int pp = 0; pp < P; ++pp) {
      const int q = t + pp * T;
      if (q < hw) {
#pragma unroll
        for (int nq = 0; nq < NQ; ++nq) {
          const float* s4 = src + (long long)nq * 4 * hw;
          dst[nq * hw + q] = make_float4(s4[q], s4[hw + q], s4[2 * hw + q], s4[3 * hw + q]);
        }
      }
    }
  };
  float4 carry[P][NQ];
#pragma unroll
  for (int pp = 0; pp < P; ++pp)
#pragma unroll
    for (int nq = 0; nq < NQ; ++nq) carry[pp][nq] = make_float4(0.f, 0.f, 0.f, 0.f);
  float loss = 0.f;

  load_frame(cur, 0);
  for (int f = 0; f < frames; ++f) {
    const int fn = next_frame(f, frames, halo_cs != nullptr);
    load_frame(nxt, fn);
    __syncthreads();
    // ---- residuals of pair (f, fn): taps and keep masks once per pixel, applied to the 4 NQ channels
    {
      const float* bf = bwd_flow + (long long)f * 2 * hw;
      const float* ff = fwd_flow + (long long)f * 2 * hw;
      const float* mbp = bwd_keep + (long long)f * hw;
      const float* mfp = fwd_keep + (long long)f * hw;
#pragma unroll
      for (int pp = 0; pp < P; ++pp) {
        const int q = t + pp * T;
        if (q >= hw) continue;
        const int x = q % w, y = q / w;
        const Taps tb = make_taps(x + __ldg(bf + q), y + __ldg(bf + hw + q), h, w);
        const Taps tf = make_taps(x + __ldg(ff + q), y + __ldg(ff + hw + q), h, w);
        const float mb = __ldg(mbp + q), mf = __ldg(mfp + q);
#pragma unroll
        for (int nq = 0; nq < NQ; ++nq) {
          const float4* c1p = cur + nq * hw;
          const float4* c2p = nxt + nq * hw;
          const float4 c1 = c1p[q], c2 = c2p[q];
          const float4 wb = sample_taps4(c1p, tb), wf = sample_taps4(c2p, tf);
          const float4 r1 = make_float4(c2.x - wb.x, c2.y - wb.y, c2.z - wb.z, c2.w - wb.w);     // c2 - W_bf(c1)
          const float4 r2 = make_float4(c1.x - wf.x, c1.y - wf.y, c1.z - wf.z, c1.w - wf.w);     // c1 - W_ff(c2)
          loss += (fabsf(r1.x) + fabsf(r1.y) + fabsf(r1.z) + fabsf(r1.w)) * mb +
                  (fabsf(r2.x) + fabsf(r2.y) + fabsf(r2.z) + fabsf(r2.w)) * mf;
          half4 hv;
          hv.lo = __floats2half2_rn(sgnf(r1.x) * mb, sgnf(r1.y) * mb);
          hv.hi = __floats2half2_rn(sgnf(r1.z) * mb, sgnf(r1.w) * mb);
          s1[nq * hw + q] = hv;
          hv.lo = __floats2half2_rn(sgnf(r2.x) * mf, sgnf(r2.y) * mf);
          hv.hi = __floats2half2_rn(sgnf(r2.z) * mf, sgnf(r2.w) * mf);
          s2[nq * hw + q] = hv;
        }
      }
    }
    __syncthreads();
    // ---- destinations hit by more than 8 taps of the backward-flow warp: extra terms of d/dc1 (frame f) through the
    //      dead frame-f planes; they join ga BEFORE it meets the carry (grad_term)
    if (n_ovf > 0) {
      for (int q = t; q < NQ * hw; q += T) cur[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      const int32_t* ob = ovf + ((long long)0 * frames + f) * n_ovf * 3;
      for (int e = t; e < n_ovf; e += T) {
        if (!ovf_run_head(ob, e)) continue;
        for (int nq = 0; nq < NQ; ++nq)
          cur[nq * hw + ob[3 * e]] = ovf_run_sum(ob, n_ovf, e, [&](int src) { return h4_to_f4(s1[nq * hw + src]); });
      }
      __syncthreads();
    }
    // ---- adjoints as gathers through the ELL rows: a warp stops at the first slot that is unused in all of its lanes
    {
      const uint4* ebp = bwd_ell + (long long)f * hw * 2;
      const uint4* efp = fwd_ell + (long long)f * hw * 2;
      float* gdst = grad + base + (long long)f * fstride;
#pragma unroll
      for (int pp = 0; pp < P; ++pp) {
        const int q = t + pp * T;
        const bool live = q < hw;
        const int qq = live ? q : 0;
        float4 ga[NQ], gb[NQ];
#pragma unroll
        for (int nq = 0; nq < NQ; ++nq) {
          ga[nq] = h4_to_f4(s2[nq * hw + qq]);                  // d/dc1 = s2 - W_bf^T s1   (frame f)
          gb[nq] = h4_to_f4(s1[nq * hw + qq]);                  // d/dc2 = s1 - W_ff^T s2   (frame fn)
          if (n_ovf > 0) {
            const float4 o = cur[nq * hw + qq];
            ga[nq].x += o.x, ga[nq].y += o.y, ga[nq].z += o.z, ga[nq].w += o.w;
          }
        }
        const EllRow rb = ell_load_row(ebp, qq);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (!__any_sync(0xffffffffu, live && ell_used(rb.e[j]))) break;
          const float wj = -ell_weight(rb.e[j]);
          const int src = ell_source(rb.e[j]);
#pragma unroll
          for (int nq = 0; nq < NQ; ++nq) ga[nq] = fma_acc(wj, h4_to_f4(s1[nq * hw + src]), ga[nq]);
        }
        const EllRow rf = ell_load_row(efp, qq);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (!__any_sync(0xffffffffu, live && ell_used(rf.e[j]))) break;
          const float wj = -ell_weight(rf.e[j]);
          const int src = ell_source(rf.e[j]);
#pragma unroll
          for (int nq = 0; nq < NQ; ++nq) gb[nq] = fma_acc(wj, h4_to_f4(s2[nq * hw + src]), gb[nq]);
        }
#pragma unroll
        for (int nq = 0; nq < NQ; ++nq) {
          if (live) {
            const float4 cr = carry[pp][nq];
            float* g4 = gdst + (long long)nq * 4 * hw;
            const float v0 = grad_term(ga[nq].x, cr.x, k), v1 = grad_term(ga[nq].y, cr.y, k);
            const float v2 = grad_term(ga[nq].z, cr.z, k), v3 = grad_term(ga[nq].w, cr.w, k);
            if (accumulate) {
              g4[q] += v0, g4[hw + q] += v1, g4[2 * hw + q] += v2, g4[3 * hw + q] += v3;
            } else {
              g4[q] = v0, g4[hw + q] = v1, g4[2 * hw + q] = v2, g4[3 * hw + q] = v3;
            }
          }
          carry[pp][nq] = gb[nq];
        }
      }
    }
    // ---- destinations with more than 8 taps of the forward-flow warp: extra terms of d/dc2, added to the carry
    if (n_ovf > 0) {
      __syncthreads();
      for (int q = t; q < NQ * hw; q += T) cur[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      const int32_t* of = ovf + ((long long)1 * frames + f) * n_ovf * 3;
      for (int e = t; e < n_ovf; e += T) {
        if (!ovf_run_head(of, e)) continue;
        for (int nq = 0; nq < NQ; ++nq)
          cur[nq * hw + of[3 * e]] = ovf_run_sum(of, n_ovf, e, [&](int src) { return h4_to_f4(s2[nq * hw + src]); });
      }
      __syncthreads();
#pragma unroll
      for (int pp = 0; pp < P; ++pp) {
        const int q = t + pp * T;
        if (q < hw) {
#pragma unroll
          for (int nq = 0; nq < NQ; ++nq) {
            const float4 o = cur[nq * hw + q];
            carry[pp][nq].x += o.x, carry[pp][nq].y += o.y, carry[pp][nq].z += o.z, carry[pp][nq].w += o.w;
          }
        }
      }
    }
    __syncthreads();                                           // s1 / s2 / cur are rewritten by the next pair
    float4* tmp = cur;                                          // frame fn becomes frame f of the next pair
    cur = nxt;
    nxt = tmp;
  }
  // ---- wrap-around: what frame 0 receives as the "next" frame of pair N-1
#pragma unroll
  for (int pp = 0; pp < P; ++pp) {
    const int q = t + pp * T;
    if (q < hw) {
#pragma unroll
      for (int nq = 0; nq < NQ; ++nq) {
        const float4 cr = carry[pp][nq];
        if (halo_grad != nullptr) {                              // open chain: the following rank's first frame receives it
          float* g0 = halo_grad + halo_base + (long long)nq * 4 * hw;
          g0[q] = carry_term(cr.x, k), g0[hw + q] = carry_term(cr.y, k);
          g0[2 * hw + q] = carry_term(cr.z, k), g0[3 * hw + q] = carry_term(cr.w, k);
        } else {
          float* g0 = grad + base + (long long)nq * 4 * hw;
          g0[q] = add_carry(g0[q], cr.x, k), g0[hw + q] = add_carry(g0[hw + q], cr.y, k);
          g0[2 * hw + q] = add_carry(g0[2 * hw + q], cr.z, k), g0[3 * hw + q] = add_carry(g0[3 * hw + q], cr.w, k);
        }
      }
    }
  }
  if (loss_acc != nullptr) cta_loss_add(loss, loss_acc, k);
}

// =============================================================================================
// O4  Adam  (torch.optim.Adam defaults; src/diffusion_hacked.py:433,485)
// =============================================================================================
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, float one_minus_b1, float b2, float one_minus_b2,
                            float step_size, float inv_sqrt_bc2, float eps) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i];
    const float mi = m[i] + (gi - m[i]) * one_minus_b1;
    const float vi = v[i] * b2 + gi * gi * one_minus_b2;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - step_size * (mi / (sqrtf(vi) * inv_sqrt_bc2 + eps));
  }
}

// =============================================================================================
// O5  AdaIN with the reference's eps quirk  (src/utils.py:58-78)
// one CTA per (sample, channel) plane
// =============================================================================================
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) t = warp_sum(t);
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  return red[0];
}

template <typename T>
__global__ void adain_kernel(const float* __restrict__ content, const T* __restrict__ style, T* __restrict__ out,
                             int hw, int content_rounds_to_half) {
  __shared__ float red[32];
  const long long off = (long long)blockIdx.x * hw;
  const float* cp = content + off;
  const T* sp = style + off;
  float cs = 0.f, ss = 0.f;
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
    float cv = cp[i];
    if (content_rounds_to_half) cv = __half2float(__float2half_rn(cv));   // `cs.data.to(sample.dtype)` (:488)
    cs += cv;
    ss += ld_as_float(sp + i);
  }
  const float c_mean = block_sum(cs, red) / hw;
  const float s_mean = block_sum(ss, red) / hw;
  float cq = 0.f, sq = 0.f;
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
    float cv = cp[i];
    if (content_rounds_to_half) cv = __half2float(__float2half_rn(cv));
    const float dc = cv - c_mean;
    const float ds = ld_as_float(sp + i) - s_mean;
    cq += dc * dc;
    sq += ds * ds;
  }
  const float c_var = block_sum(cq, red) / (hw - 1);            // unbiased, torch.var default
  const float s_var = block_sum(sq, red) / (hw - 1);
  const float c_std = sqrtf(c_var + 1e-5f);
  const float s_std = sqrtf(s_var + 1.0f);                      // eps slot receives `chunk` = 1 (utils.py:73)
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
    float cv = cp[i];
    if (content_rounds_to_half) cv = __half2float(__float2half_rn(cv));
    st_from_float(out + off + i, (cv - c_mean) / c_std * s_std + s_mean);
  }
}

// =============================================================================================
// O3 step 1: row-normalise and transpose to token-major fp16  (src/diffusion_hacked.py:470-473)
// cs [batch, C, L] fp32  ->  xhat [batch, L, C] fp16, norms [batch, L]
// one CTA per (batch, 32 tokens)
// =============================================================================================
__global__ void gram_normalize_kernel(const float* __restrict__ cs, __half* __restrict__ xhat,
                                      float* __restrict__ norms, int channels, int tokens) {
  __shared__ float part[8][33];
  __shared__ float inv_norm[32];
  __shared__ float tile[64][33];
  const int tiles = (tokens + 31) / 32;
  const int l0 = (blockIdx.x % tiles) * 32;
  const int b = blockIdx.x / tiles;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* src = cs + (long long)b * channels * tokens;
  const int l = l0 + lane;
  float ssq = 0.f;
  if (l < tokens)
    for (int c = warp; c < channels; c += 8) {
      const float v = src[(long long)c * tokens + l];
      ssq = fmaf(v, v, ssq);
    }
  part[warp][lane] = ssq;
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += part[i][lane];
    const float nrm = sqrtf(s);
    inv_norm[lane] = 1.f / nrm;
    if (l < tokens) norms[(long long)b * tokens + l] = nrm;
  }
  __syncthreads();
  for (int c0 = 0; c0 < channels; c0 += 64) {
    for (int cc = warp; cc < 64; cc += 8) {
      const int c = c0 + cc;
      tile[cc][lane] = (c < channels && l < tokens) ? src[(long long)c * tokens + l] * inv_norm[lane] : 0.f;
    }
    __syncthreads();
    // write 32 tokens x 64 channels, channel-contiguous
    for (int t = threadIdx.x; t < 32 * 32; t += blockDim.x) {
      const int tok = t / 32, cp = (t % 32) * 2;
      if (l0 + tok < tokens && c0 + cp < channels) {
        const __half2 hv = __floats2half2_rn(tile[cp][tok], tile[cp + 1][tok]);
        *reinterpret_cast<__half2*>(xhat + ((long long)b * tokens + l0 + tok) * channels + c0 + cp) = hv;
      }
    }
    __syncthreads();
  }
}

// =============================================================================================
// S1  classifier-free guidance + DDPM step arithmetic  (src/pipe_FRESCO.py:212-215, :22-35, :49-73)
// two elementwise passes because the background-smoothing VAE round trip sits between them (:44-47)
// =============================================================================================
// noise = uncond + g * (text - uncond);  x0 = (sample - sqrt(1 - a_t) * noise) / sqrt(a_t)
template <typename T>
__global__ void cfg_pred_x0_kernel(const T* __restrict__ uncond, const T* __restrict__ text, const T* __restrict__ sample,
                                   T* __restrict__ x0, long long n, float guidance, float sqrt_beta, float inv_sqrt_alpha) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float u = ld_as_float(uncond + i);
    const float e = text ? u + guidance * (ld_as_float(text + i) - u) : u;
    st_from_float(x0 + i, (ld_as_float(sample + i) - sqrt_beta * e) * inv_sqrt_alpha);
  }
}
// prev = c_x0 * x0 + c_xt * sample + sigma * noise   (noise of frame 0 for every frame when repeat_noise, :67-68)
template <typename T>
__global__ void ddpm_prev_kernel(const T* __restrict__ x0, const T* __restrict__ sample, const T* __restrict__ noise,
                                 T* __restrict__ prev, long long n, long long per_frame, int repeat_noise, float c_x0,
                                 float c_xt, float sigma) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float z = ld_as_float(noise + (repeat_noise ? i % per_frame : i));
    st_from_float(prev + i, c_x0 * ld_as_float(x0 + i) + c_xt * ld_as_float(sample + i) + sigma * z);
  }
}

// =============================================================================================
// W2  binary dilation with replicate padding  (src/utils.py:81-93: replicate-pad + conv2d(ones k x k) + clamp[0,1])
// for masks in [0, 1] the clamped box sum of a {0,1} mask is its k x k maximum; general inputs take the clamped sum
// =============================================================================================
__global__ void dilate_kernel(const float* __restrict__ in, float* __restrict__ out, int planes, int h, int w, int k) {
  const int r = (k - 1) / 2;
  const long long total = (long long)planes * h * w;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % w), y = (int)((t / w) % h);
    const float* pl = in + (t / ((long long)h * w)) * (long long)h * w;
    float acc = 0.f;
    for (int dy = -r; dy <= r; ++dy) {
      const int yy = min(max(y + dy, 0), h - 1);
      for (int dx = -r; dx <= r; ++dx) acc += pl[(long long)yy * w + min(max(x + dx, 0), w - 1)];
    }
    out[t] = fminf(fmaxf(acc, 0.f), 1.f);
  }
}

}  // namespace fresco

using namespace fresco;

static inline int grid_for(long long work, int block, int per_sm = 8) {
  long long g = (work + block - 1) / block;
  const long long cap = (long long)sm_count() * per_sm;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" int fresco_kv_compact(const void* k, const void* v, const int32_t* idx, void* k_out, void* v_out,
                                 int chunks, int rows_per_chunk, int n_sel, int channels, void* stream) {
  if (!k || !v || !idx || !k_out || !v_out) return set_error(FRESCO_ERR_ARG, "fresco_kv_compact: null pointer");
  if (chunks <= 0 || rows_per_chunk <= 0 || n_sel <= 0 || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_kv_compact: bad shape (channels must be a multiple of 8)");
  const int vpr = channels / 8;
  const long long total = (long long)chunks * n_sel * vpr;
  kv_compact_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)k, (const uint4*)v, idx, (uint4*)k_out, (uint4*)v_out, chunks, rows_per_chunk, n_sel, vpr);
  return check_launch("kv_compact_kernel");
}

extern "C" int fresco_kv_compact_packed(const void* k, const void* v, const int32_t* idx, void* kv_out, int chunks,
                                        int rows_per_chunk, int n_sel, int out_rows, int channels, void* stream) {
  if (!k || !v || !idx || !kv_out) return set_error(FRESCO_ERR_ARG, "fresco_kv_compact_packed: null pointer");
  if (chunks <= 0 || rows_per_chunk <= 0 || n_sel <= 0 || out_rows < n_sel || channels <= 0 || channels % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_kv_compact_packed: bad shape (channels must be a multiple of 8)");
  const int vpr = channels / 8;
  const long long total = (long long)chunks * n_sel * vpr;
  kv_compact_packed_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)k, (const uint4*)v, idx, (uint4*)kv_out, chunks, rows_per_chunk, n_sel, out_rows, vpr);
  return check_launch("kv_compact_packed_kernel");
}

extern "C" int fresco_rows_gather(const void* src, const int32_t* idx, void* dst, long long n_rows, int row_bytes,
                                  int dst_stride_bytes, int dst_offset_bytes, void* stream) {
  if (!src || !idx || !dst) return set_error(FRESCO_ERR_ARG, "fresco_rows_gather: null pointer");
  if (n_rows <= 0 || row_bytes <= 0 || row_bytes % 16 || dst_stride_bytes % 16 || dst_offset_bytes % 16 ||
      dst_offset_bytes + row_bytes > dst_stride_bytes)
    return set_error(FRESCO_ERR_ARG, "fresco_rows_gather: rows / strides / offsets must be multiples of 16 bytes");
  rows_gather_kernel<<<grid_for(n_rows * (row_bytes / 16), 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)src, idx, (uint4*)dst, n_rows, row_bytes / 16, dst_stride_bytes / 16, dst_offset_bytes / 16);
  return check_launch("rows_gather_kernel");
}

extern "C" int fresco_rows_scatter(const void* src, const int32_t* idx, void* dst, long long n_rows, int row_bytes,
                                   void* stream) {
  if (!src || !idx || !dst) return set_error(FRESCO_ERR_ARG, "fresco_rows_scatter: null pointer");
  if (n_rows <= 0 || row_bytes <= 0 || row_bytes % 16)
    return set_error(FRESCO_ERR_ARG, "fresco_rows_scatter: rows must be multiples of 16 bytes");
  rows_scatter_kernel<<<grid_for(n_rows * (row_bytes / 16), 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)src, idx, (uint4*)dst, n_rows, row_bytes / 16);
  return check_launch("rows_scatter_kernel");
}

template <int D, int NMAX>
static int launch_temporal_rows(const void* q_raw, const void* k_raw, const void* v_src, void* out, const int64_t* fwd_map,
                                const uint8_t* traj_mask, int chunks, int frames, int tokens, int heads, float scale,
                                int in_row_stride, cudaStream_t s) {
  // trajectories per CTA: exactly one thread per output row (trajectory, frame, head), up to 256 threads; shared memory
  // 2 * N * 2C bytes per trajectory (k and v rows; q rows go straight to registers)
  const int rows_per_traj = frames * heads;
  if (rows_per_traj > 256) return FRESCO_ERR_UNSUPPORTED;
  int tpb = 256 / rows_per_traj;
  const size_t per_traj = (size_t)2 * frames * heads * D * sizeof(__half) + (size_t)frames * sizeof(int);
  while (tpb > 1 && tpb * per_traj > 48 * 1024) --tpb;
  const size_t smem = tpb * per_traj;
  if (smem > 200 * 1024) return FRESCO_ERR_UNSUPPORTED;
  int threads = (tpb * rows_per_traj + 31) / 32 * 32;
  if (int rc = allow_dynamic_smem((const void*)temporal_attn_rows_kernel<D, NMAX>, smem, "temporal_attn_rows")) return rc;
  const int blocks = chunks * ((tokens + tpb - 1) / tpb);
  temporal_attn_rows_kernel<D, NMAX><<<blocks, threads, smem, s>>>(
      (const __half*)q_raw, (const __half*)k_raw, (const __half*)v_src, (__half*)out, fwd_map, traj_mask, frames, tokens,
      heads, tpb, scale * 1.4426950408889634f, in_row_stride / 8);
  return check_launchf("temporal_attn_rows_kernel<%d,%d>", D, NMAX);
}

extern "C" int fresco_temporal_attn_fwd(const void* q_raw, const void* k_raw, const void* v_src, void* out,
                                        const int64_t* fwd_map, const uint8_t* traj_mask, int chunks, int frames,
                                        int tokens, int heads, int head_dim, float scale, void* stream) {
  return fresco_temporal_attn_fwd_strided(q_raw, k_raw, v_src, out, fwd_map, traj_mask, chunks, frames, tokens, heads,
                                          head_dim, heads * head_dim, scale, stream);
}

extern "C" int fresco_temporal_attn_fwd_strided(const void* q_raw, const void* k_raw, const void* v_src, void* out,
                                                const int64_t* fwd_map, const uint8_t* traj_mask, int chunks,
                                                int frames, int tokens, int heads, int head_dim, int in_row_stride,
                                                float scale, void* stream) {
  if (!q_raw || !k_raw || !v_src || !out || !fwd_map || !traj_mask)
    return set_error(FRESCO_ERR_ARG, "fresco_temporal_attn_fwd: null pointer");
  if (chunks <= 0 || frames <= 0 || tokens <= 0 || heads <= 0 || heads > 32 || head_dim % 8 != 0 || frames > 64)
    return set_error(FRESCO_ERR_ARG, "fresco_temporal_attn_fwd: bad shape");
  if (out == v_src) return set_error(FRESCO_ERR_ARG, "fresco_temporal_attn_fwd: out must not alias v_src");
  if (in_row_stride < heads * head_dim || in_row_stride % 8 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_temporal_attn_fwd: bad input row stride");
  cudaStream_t s = (cudaStream_t)stream;
  // row kernel (one output row per thread) for the head dims / frame counts of the BASELINE configs
  const bool dense = in_row_stride == heads * head_dim;
  if (frames <= 16 && (option(OPT_TEMPORAL_V, 2) == 2 || !dense)) {
    int rc = FRESCO_ERR_UNSUPPORTED;
#define ROWS(DD)                                                                                                      \
  rc = frames <= 8 ? launch_temporal_rows<DD, 8>(q_raw, k_raw, v_src, out, fwd_map, traj_mask, chunks, frames, tokens, \
                                                 heads, scale, in_row_stride, s)                                       \
                   : launch_temporal_rows<DD, 16>(q_raw, k_raw, v_src, out, fwd_map, traj_mask, chunks, frames, tokens,\
                                                  heads, scale, in_row_stride, s)
    if (head_dim == 40) ROWS(40);
    else if (head_dim == 64) ROWS(64);
    else if (head_dim == 80) ROWS(80);
#undef ROWS
    if (rc != FRESCO_ERR_UNSUPPORTED) return rc;
  }
  if (!dense) return set_error(FRESCO_ERR_UNSUPPORTED, "fresco_temporal_attn_fwd: strided inputs need frames <= 16 and head_dim 40/64/80");
  const size_t per_warp =
      (((size_t)3 * frames * head_dim * sizeof(__half) + (size_t)frames * frames * sizeof(float)) + 15) & ~size_t(15);
  const size_t smem = per_warp * heads;
  if (smem > 200 * 1024) return set_error(FRESCO_ERR_UNSUPPORTED, "fresco_temporal_attn_fwd: frames*head_dim too large");
  if (int rc = allow_dynamic_smem((const void*)temporal_attn_kernel, smem, "temporal_attn")) return rc;
  temporal_attn_kernel<<<chunks * tokens, 32 * heads, smem, s>>>(
      (const __half*)q_raw, (const __half*)k_raw, (const __half*)v_src, (__half*)out, fwd_map, traj_mask, frames,
      tokens, heads, head_dim, scale);
  return check_launch("temporal_attn_kernel");
}

extern "C" int fresco_flow_warp(const float* src, const float* flow, float* dst, int batch, int channels, int h,
                                int w, int flow_batch, void* stream) {
  if (!src || !flow || !dst) return set_error(FRESCO_ERR_ARG, "fresco_flow_warp: null pointer");
  if (batch <= 0 || channels <= 0 || h <= 0 || w <= 0 || flow_batch <= 0)
    return set_error(FRESCO_ERR_ARG, "fresco_flow_warp: bad shape");
  flow_warp_kernel<<<grid_for((long long)batch * h * w, 256), 256, 0, (cudaStream_t)stream>>>(
      src, flow, dst, batch, channels, h, w, flow_batch);
  return check_launch("flow_warp_kernel");
}

template <typename T, int K>
static int launch_chain_group(const void* sample, void* out, const float* bwd_flow, const float* fwd_flow_last,
                              const float* blend, int chunks, int frames, int channels, int h, int w, cudaStream_t s) {
  const size_t smem = (size_t)2 * K * h * w * sizeof(float);
  if (int rc = allow_dynamic_smem((const void*)warp_chain_group_kernel<T, K>, 200 * 1024, "warp_chain_group")) return rc;
  const int planes = chunks * channels;
  warp_chain_group_kernel<T, K><<<(planes + K - 1) / K, 512, smem, s>>>((const T*)sample, (T*)out, bwd_flow, fwd_flow_last,
                                                                       blend, frames, channels, planes, h, w);
  return check_launchf("warp_chain_group_kernel<%s,%d>", sizeof(T) == 2 ? "half" : "float", K);
}

// (P pixels per thread, NQ channel quads per CTA) for a plane of hw pixels: as many quads as shared memory (bytes_per_px
// per quad, 200 KB) and the divisibility of the channel count allow, P * NQ == 4 carried float4 per thread, so one of
// (1,4), (2,2), (4,1).  False when that needs more than 1024 threads: the caller takes its channel-grouped kernel.
static bool quad_config(int hw, int channels, int planes, int bytes_per_px, int& P, int& NQ, int& T) {
  if (channels % 4 != 0) return false;
  for (NQ = 4; NQ >= 1; NQ >>= 1) {
    if (channels % (4 * NQ) != 0) continue;
    if ((size_t)NQ * hw * bytes_per_px > 200 * 1024) continue;
    if (NQ > 1 && planes / (4 * NQ) < sm_count()) continue;           // keep every SM busy
    P = 4 / NQ;
    T = ((hw + P - 1) / P + 31) / 32 * 32;
    if (T > 1024) return false;
    if (T < 32) T = 32;
    return true;
  }
  return false;
}

template <typename T, int P, int NQ>
static int launch_chain_quad(const void* sample, void* out, const float* bwd_flow, const float* fwd_flow_last,
                             const float* blend, int chunks, int frames, int channels, int h, int w, int threads,
                             cudaStream_t s) {
  const size_t smem = (size_t)NQ * h * w * 32;
  if (int rc = allow_dynamic_smem((const void*)warp_chain_quad_kernel<T, P, NQ>, 200 * 1024, "warp_chain_quad")) return rc;
  warp_chain_quad_kernel<T, P, NQ><<<chunks * channels / (4 * NQ), threads, smem, s>>>(
      (const T*)sample, (T*)out, bwd_flow, fwd_flow_last, blend, frames, channels, h, w);
  return check_launchf("warp_chain_quad_kernel<%s,%d,%d>", sizeof(T) == 2 ? "half" : "float", P, NQ);
}

template <typename T>
static int launch_chain(const void* sample, void* out, const float* bwd_flow, const float* fwd_flow_last,
                        const float* blend, int chunks, int frames, int channels, int h, int w, cudaStream_t s) {
  const int planes = chunks * channels;
  int P, NQ, threads;
  if (quad_config(h * w, channels, planes, 32, P, NQ, threads)) {
#define CQ(PP, QQ)                                                                                                     \
  if (P == PP && NQ == QQ)                                                                                             \
    return launch_chain_quad<T, PP, QQ>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w,   \
                                        threads, s);
    CQ(1, 4) CQ(2, 2) CQ(4, 1)
#undef CQ
  }
  // planes per CTA: as many as keep two CTAs on an SM (<= ~100 KB of shared memory each) and the grid above two waves
  const size_t plane2 = (size_t)2 * h * w * sizeof(float);
  if (8 * plane2 <= 100 * 1024 && planes / 8 >= 296)
    return launch_chain_group<T, 8>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w, s);
  if (3 * plane2 <= 100 * 1024 && planes / 3 >= 296)
    return launch_chain_group<T, 3>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w, s);
  return launch_chain_group<T, 1>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w, s);
}

extern "C" int fresco_warp_fuse_chain(const void* sample, void* out, int is_half, const float* bwd_flow,
                                      const float* fwd_flow_last, const float* blend, int chunks, int frames,
                                      int channels, int h, int w, void* stream) {
  if (!sample || !out || !bwd_flow || !fwd_flow_last || !blend)
    return set_error(FRESCO_ERR_ARG, "fresco_warp_fuse_chain: null pointer");
  if (chunks <= 0 || frames < 2 || channels <= 0 || h <= 0 || w <= 0)
    return set_error(FRESCO_ERR_ARG, "fresco_warp_fuse_chain: bad shape (frames >= 2)");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t plane_bytes = (size_t)h * w * sizeof(float);
  if (2 * plane_bytes <= 200 * 1024) {
    return is_half ? launch_chain<__half>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w, s)
                   : launch_chain<float>(sample, out, bwd_flow, fwd_flow_last, blend, chunks, frames, channels, h, w, s);
  }
  // large planes (image resolution): fp32 only, in place on `out`, one launch per chain step
  if (is_half) return set_error(FRESCO_ERR_UNSUPPORTED, "fresco_warp_fuse_chain: planes > 100 KB need float tensors");
  const long long hw = (long long)h * w;
  const long long total = (long long)chunks * frames * channels * hw;
  if (out != sample) {
    cudaError_t e = cudaMemcpyAsync(out, sample, total * sizeof(float), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return set_cuda_error(e, "cudaMemcpyAsync(warp chain)");
  }
  const int grid = grid_for((long long)chunks * channels * hw, 256);
  for (int ii = 0; ii + 1 < frames; ++ii) {
    warp_blend_step_kernel<<<grid, 256, 0, s>>>((const float*)out, (float*)out, bwd_flow + (long long)ii * 2 * hw,
                                                blend + (long long)ii * hw, chunks, frames, channels, h, w, ii, ii + 1);
    int rc = check_launch("warp_blend_step_kernel");
    if (rc) return rc;
  }
  warp_blend_step_kernel<<<grid, 256, 0, s>>>((const float*)out, (float*)out, fwd_flow_last,
                                              blend + (long long)(frames - 1) * hw, chunks, frames, channels, h, w, 0,
                                              frames - 1);
  return check_launch("warp_blend_step_kernel");
}

extern "C" int fresco_warp_taps(const float* flow, int32_t* dest, float* weight, int frames, int h, int w,
                                void* stream) {
  if (!flow || !dest || !weight) return set_error(FRESCO_ERR_ARG, "fresco_warp_taps: null pointer");
  if (frames <= 0 || h <= 0 || w <= 0) return set_error(FRESCO_ERR_ARG, "fresco_warp_taps: bad shape");
  warp_taps_kernel<<<grid_for((long long)frames * h * w, 256), 256, 0, (cudaStream_t)stream>>>(flow, dest, weight,
                                                                                              frames, h, w);
  return check_launch("warp_taps_kernel");
}

extern "C" int fresco_warp_loss_fwd_bwd(const float* cs, const float* fwd_flow, const float* bwd_flow,
                                        const float* fwd_keep, const float* bwd_keep, const void* bwd_ell,
                                        const void* fwd_ell, const int32_t* overflow, int n_overflow, float* grad,
                                        float* loss_acc, int accumulate, int chunks, int frames, int channels, int h,
                                        int w, void* stream) {
  return fresco_warp_loss_fwd_bwd_halo(cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, bwd_ell, fwd_ell, overflow, n_overflow,
                                       grad, loss_acc, accumulate, chunks, frames, channels, h, w, nullptr, nullptr,
                                       frames, stream);
}

extern "C" int fresco_warp_loss_fwd_bwd_halo(const float* cs, const float* fwd_flow, const float* bwd_flow,
                                             const float* fwd_keep, const float* bwd_keep, const void* bwd_ell,
                                             const void* fwd_ell, const int32_t* overflow, int n_overflow, float* grad,
                                             float* loss_acc, int accumulate, int chunks, int frames, int channels,
                                             int h, int w, const float* halo_cs, float* halo_grad, int total_frames,
                                             void* stream) {
  if (!cs || !fwd_flow || !bwd_flow || !fwd_keep || !bwd_keep || !grad || !bwd_ell || !fwd_ell)
    return set_error(FRESCO_ERR_ARG, "fresco_warp_loss_fwd_bwd: null pointer");
  if (n_overflow > 0 && !overflow) return set_error(FRESCO_ERR_ARG, "fresco_warp_loss_fwd_bwd: overflow list missing");
  if ((halo_cs == nullptr) != (halo_grad == nullptr))
    return set_error(FRESCO_ERR_ARG, "fresco_warp_loss_fwd_bwd_halo: halo_cs and halo_grad go together");
  const int min_frames = halo_cs != nullptr ? 1 : 2;
  if (chunks <= 0 || frames < min_frames || total_frames < frames || channels <= 0 || h <= 0 || w <= 0 || h * w > 65535)
    return set_error(FRESCO_ERR_ARG, "fresco_warp_loss_fwd_bwd: bad shape (frames >= 2, h*w <= 65535)");
  const double numel = (double)chunks * total_frames * channels * h * w;      // the mean runs over the WHOLE batch
  const float kk = (float)(2.0 / numel);
  cudaStream_t s = (cudaStream_t)stream;
  // ---- channel-quad kernel: 4 NQ planes per CTA interleaved in shared memory (48 bytes per pixel and quad)
  {
    int P, NQ, threads;
    if (quad_config(h * w, channels, chunks * channels, 48, P, NQ, threads)) {
      const size_t smem_q = (size_t)NQ * h * w * 48;
      const int grid_q = chunks * channels / (4 * NQ);
#define LQ(PP, QQ)                                                                                                      \
  if (P == PP && NQ == QQ) {                                                                                            \
    if (int rc = allow_dynamic_smem((const void*)warp_loss_quad_kernel<PP, QQ>, 200 * 1024, "warp_loss_quad"))         \
      return rc;                                                                                                        \
    warp_loss_quad_kernel<PP, QQ><<<grid_q, threads, smem_q, s>>>(                                                      \
        cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, (const uint4*)bwd_ell, (const uint4*)fwd_ell, overflow, n_overflow, \
        grad, loss_acc, accumulate, frames, channels, h, w, kk, halo_cs, halo_grad);                                    \
    return check_launchf("warp_loss_quad_kernel<%d,%d>", PP, QQ);                                                       \
  }
      LQ(1, 4) LQ(2, 2) LQ(4, 1)
#undef LQ
    }
  }
  // ---- channel-grouped kernel: 512 threads; P pixel slots x KT planes per thread (carried in registers)
  {
    const int T = 512, hw = h * w, planes = chunks * channels;
    const int P = hw > T ? (hw + T - 1) / T : 1;
    const int G = hw >= T ? 1 : T / hw;
    int KT = 0;
    for (int cand = 4; cand >= 1; cand >>= 1) {        // (8 planes per thread spill at 64 registers)
      const size_t smem_c = (size_t)cand * G * hw * 12;
      if (P * cand > 18 || smem_c > 100 * 1024) continue;
      if (cand > 1 && (planes + cand * G - 1) / (cand * G) < 296) continue;     // keep the grid above two waves
      KT = cand;
      break;
    }
    if (KT == 0 && P == 18 && (size_t)G * hw * 12 <= 200 * 1024) KT = 1;
    int rc = FRESCO_ERR_UNSUPPORTED;
    if (KT > 0) {
      const int K = KT * G;
      const size_t smem = (size_t)K * hw * 12;
      const int grid = (planes + K - 1) / K;
#define LOSS_CASE(PP, KK)                                                                                               \
  if (P == PP && KT == KK) {                                                                                            \
    rc = allow_dynamic_smem((const void*)warp_loss_group_kernel<PP, KK>, 200 * 1024, "warp_loss_group");               \
    if (rc) return rc;                                                                                                  \
    warp_loss_group_kernel<PP, KK><<<grid, T, smem, s>>>(cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep,                    \
                                                         (const uint4*)bwd_ell, (const uint4*)fwd_ell, overflow,        \
                                                         n_overflow, grad, loss_acc, accumulate, frames, channels,      \
                                                         planes, h, w, G, kk, halo_cs, halo_grad);                      \
    rc = check_launchf("warp_loss_group_kernel<%d,%d>", PP, KK);                                                        \
  }
      LOSS_CASE(1, 1) LOSS_CASE(1, 2) LOSS_CASE(1, 4)
      LOSS_CASE(2, 1) LOSS_CASE(2, 2) LOSS_CASE(2, 4)
      LOSS_CASE(3, 1) LOSS_CASE(3, 2) LOSS_CASE(3, 4)
      LOSS_CASE(4, 1) LOSS_CASE(4, 2) LOSS_CASE(4, 4)
      LOSS_CASE(5, 1) LOSS_CASE(5, 2)
      LOSS_CASE(8, 1) LOSS_CASE(8, 2)
      LOSS_CASE(18, 1)
#undef LOSS_CASE
    }
    if (rc != FRESCO_ERR_UNSUPPORTED) return rc;
  }
  // ---- any other plane size: one CTA per plane (round-1 kernel)
  const size_t smem = (size_t)4 * h * w * sizeof(float);
  if (smem > 200 * 1024) return set_error(FRESCO_ERR_UNSUPPORTED, "fresco_warp_loss_fwd_bwd: plane too large for shared memory");
  if (int rc = allow_dynamic_smem((const void*)warp_loss_kernel, 200 * 1024, "warp_loss")) return rc;
  warp_loss_kernel<<<chunks * channels, 256, smem, s>>>(
      cs, fwd_flow, bwd_flow, fwd_keep, bwd_keep, (const uint4*)bwd_ell, (const uint4*)fwd_ell, overflow, n_overflow,
      grad, loss_acc, accumulate, frames, channels, h, w, kk, halo_cs, halo_grad);
  return check_launch("warp_loss_kernel");
}

extern "C" int fresco_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n,
                                int step, double lr, double beta1, double beta2, double eps, void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq) return set_error(FRESCO_ERR_ARG, "fresco_adam_step: null pointer");
  if (n <= 0 || step <= 0) return set_error(FRESCO_ERR_ARG, "fresco_adam_step: bad n/step");
  double bc1 = 1.0, bc2 = 1.0, p1 = 1.0, p2 = 1.0;
  for (int i = 0; i < step; ++i) {
    p1 *= beta1;
    p2 *= beta2;
  }
  bc1 = 1.0 - p1;
  bc2 = 1.0 - p2;
  double sq = bc2 > 0 ? 1.0 / __builtin_sqrt(bc2) : 1.0;
  // hyper-parameters arrive as doubles (python floats) and are rounded to fp32 one by one, as torch.optim.Adam does
  // with its python scalars: (float)(1 - beta2) is NOT 1.f - (float)beta2
  adam_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n,
                                                                  (float)(1.0 - beta1), (float)beta2,
                                                                  (float)(1.0 - beta2), (float)(lr / bc1), (float)sq,
                                                                  (float)eps);
  return check_launch("adam_kernel");
}

extern "C" int fresco_adain(const float* content, const void* style, void* out, int is_half, int planes, int hw,
                            void* stream) {
  if (!content || !style || !out) return set_error(FRESCO_ERR_ARG, "fresco_adain: null pointer");
  if (planes <= 0 || hw <= 1) return set_error(FRESCO_ERR_ARG, "fresco_adain: bad shape");
  if (is_half)
    adain_kernel<__half><<<planes, 256, 0, (cudaStream_t)stream>>>(content, (const __half*)style, (__half*)out, hw, 1);
  else
    adain_kernel<float><<<planes, 256, 0, (cudaStream_t)stream>>>(content, (const float*)style, (float*)out, hw, 0);
  return check_launch(is_half ? "adain_kernel<half>" : "adain_kernel<float>");
}

extern "C" int fresco_gram_normalize(const float* cs, void* xhat, float* norms, int batch, int channels, int tokens,
                                     void* stream) {
  if (!cs || !xhat || !norms) return set_error(FRESCO_ERR_ARG, "fresco_gram_normalize: null pointer");
  if (batch <= 0 || channels <= 0 || tokens <= 0 || channels % 2 != 0)
    return set_error(FRESCO_ERR_ARG, "fresco_gram_normalize: bad shape");
  const int tiles = (tokens + 31) / 32;
  gram_normalize_kernel<<<batch * tiles, 256, 0, (cudaStream_t)stream>>>(cs, (__half*)xhat, norms, channels, tokens);
  return check_launch("gram_normalize_kernel");
}

extern "C" int fresco_cfg_pred_x0(const void* noise_uncond, const void* noise_text, const void* sample, void* x0,
                                  int is_half, long long n, float guidance_scale, float alpha_prod_t, void* stream) {
  if (!noise_uncond || !sample || !x0) return set_error(FRESCO_ERR_ARG, "fresco_cfg_pred_x0: null pointer");
  if (n <= 0 || !(alpha_prod_t > 0.f) || alpha_prod_t > 1.f) return set_error(FRESCO_ERR_ARG, "fresco_cfg_pred_x0: bad n / alpha");
  const float sb = sqrtf(1.f - alpha_prod_t), isa = 1.f / sqrtf(alpha_prod_t);
  const int grid = grid_for(n, 256);
  if (is_half)
    cfg_pred_x0_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)noise_uncond, (const __half*)noise_text,
                                                                       (const __half*)sample, (__half*)x0, n, guidance_scale, sb, isa);
  else
    cfg_pred_x0_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)noise_uncond, (const float*)noise_text,
                                                                      (const float*)sample, (float*)x0, n, guidance_scale, sb, isa);
  return check_launch(is_half ? "cfg_pred_x0_kernel<half>" : "cfg_pred_x0_kernel<float>");
}

extern "C" int fresco_ddpm_prev(const void* x0, const void* sample, const void* noise, void* prev, int is_half, long long n,
                                long long per_frame, int repeat_noise, float c_x0, float c_xt, float sigma, void* stream) {
  if (!x0 || !sample || !noise || !prev) return set_error(FRESCO_ERR_ARG, "fresco_ddpm_prev: null pointer");
  if (n <= 0 || per_frame <= 0 || n % per_frame != 0) return set_error(FRESCO_ERR_ARG, "fresco_ddpm_prev: bad n / per_frame");
  const int grid = grid_for(n, 256);
  if (is_half)
    ddpm_prev_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x0, (const __half*)sample, (const __half*)noise,
                                                                     (__half*)prev, n, per_frame, repeat_noise, c_x0, c_xt, sigma);
  else
    ddpm_prev_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)x0, (const float*)sample, (const float*)noise,
                                                                    (float*)prev, n, per_frame, repeat_noise, c_x0, c_xt, sigma);
  return check_launch(is_half ? "ddpm_prev_kernel<half>" : "ddpm_prev_kernel<float>");
}

extern "C" int fresco_dilate(const float* in, float* out, int planes, int h, int w, int kernel, void* stream) {
  if (!in || !out || in == out) return set_error(FRESCO_ERR_ARG, "fresco_dilate: null pointer / in-place");
  if (planes <= 0 || h <= 0 || w <= 0 || kernel <= 0 || kernel % 2 == 0)
    return set_error(FRESCO_ERR_ARG, "fresco_dilate: bad shape (odd kernel)");
  dilate_kernel<<<grid_for((long long)planes * h * w, 256), 256, 0, (cudaStream_t)stream>>>(in, out, planes, h, w, kernel);
  return check_launch("dilate_kernel");
}

