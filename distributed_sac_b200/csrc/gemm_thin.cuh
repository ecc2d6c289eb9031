// Thin backward GEMMs: the input-layer problems of the SAC step whose "N" is the observation/action width
// (8..16 columns), e.g. LunarLander's dW0 = dZ0^T [256 x B] * X [B x 10] and dQ/d(s,a) = dZ0 [B x 256] * W0 [256 x 10].
// The 32x32-tile engine of gemm_simt.cuh wastes 2/3 of every tile on them and leaves only M/32 CTAs with a serial
// 256..1280-long k loop that dominates the launch.  Here the
// narrow operand B[K][N<=16] is staged once in shared memory, the long dimension is spread over all 16 warps of a
// CTA and the partial sums are combined in a fixed order (bit-reproducible run to run / replica to replica):
//
//   WGRAD  C[m][n] = sum_k A[k][m] * B[k][n],  C2[m] = sum_k A[k][m]    32 m per CTA (lane = m), warp w takes k = w (mod 16)
//   DGRAD  C[m][n] = (sum_k A[m][k] * B[k][n]) * [mask[m][n] > 0]       16 m per CTA (warp = m),  lane takes k = lane (mod 32)
//
// Same GemmProb / GemmGroup descriptors as gemm_simt_kernel (blockIdx.z = replica x problem), so the plan builder only
// routes problems with mode != FWD and N <= 16 here.  Reference math: the autograd of nn.Linear at
// LunarLander_Distributed_SAC/src/model.py:41-44,119-125 (weight / input gradients of the first layer).
#pragma once
#include "gemm_simt.cuh"

namespace bsac {

constexpr int GT_THREADS = 512;
constexpr int GT_WARPS = GT_THREADS / 32;
constexpr int GT_NMAX = 16;              // widest "thin" N
constexpr int GT_KC = 512;               // k rows of B staged per pass
constexpr int GT_LDB = 20;               // staged row pitch: lanes of the DGRAD path read rows k = lane (mod 32) as float4 --
                                         // 20-float rows put a quarter-warp on 8 distinct 16-B bank groups (16 would 4-way conflict)
constexpr int GT_ROWS_WGRAD = 32, GT_ROWS_DGRAD = GT_WARPS;

B200_HD bool gemm_is_thin(const GemmProb& p) { return p.mode != GEMM_FWD && p.N <= GT_NMAX; }

__global__ void __launch_bounds__(GT_THREADS) gemm_thin_kernel(const __grid_constant__ GemmGroup grp) {
  const int sched = grp.sched ? sched_word(grp.sched + (int)(blockIdx.z / grp.G) * grp.sched_stride) : SCHED_ACTOR;
  KStamp ks_;
  const int G = grp.G;
  const int g = blockIdx.z % G, rep = blockIdx.z / G;
  const GemmProb& P = grp.p[g];
  const int M = P.M, N = P.N, K = P.K;
  const bool wgrad = P.mode == GEMM_WGRAD;
  const int m0 = blockIdx.y * (wgrad ? GT_ROWS_WGRAD : GT_ROWS_DGRAD);
  if (m0 >= M) return;
  if (!(sched & SCHED_ACTOR)) return;

  // B chunk [k][GT_LDB]; after the last pass the same storage holds the per-warp partial sums [16][32][17]
  __shared__ __align__(16) float sm[GT_KC * GT_LDB];
  static_assert(GT_KC * GT_LDB >= GT_WARPS * 32 * (GT_NMAX + 1), "the reduction buffer must fit the B chunk storage");

  const float* __restrict__ A = P.A + (long long)rep * P.rsA;
  const float* __restrict__ Bm = P.B + (long long)rep * P.rsB;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int lda = P.lda, ldb = P.ldb;
  const bool vecB = (ldb <= GT_NMAX) && ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(Bm) & 15) == 0);
  const int n4 = (N + 3) >> 2;

  float acc[GT_NMAX];
#pragma unroll
  for (int n = 0; n < GT_NMAX; ++n) acc[n] = 0.f;
  float asum = 0.f;                                   // WGRAD bias gradient

  for (int k0 = 0; k0 < K; k0 += GT_KC) {
    const int kc = (K - k0 < GT_KC) ? K - k0 : GT_KC;
    if (k0 > 0) __syncthreads();
    // ---- stage B[k0 .. k0+kc)[0 .. N) as [k][16] (columns >= N are never read into a stored result) ----
    if (vecB) {
      const int q4 = ldb >> 2;
      for (int e = tid; e < kc * q4; e += GT_THREADS) {
        const int k = e / q4, c = e - k * q4;
        *reinterpret_cast<float4*>(sm + k * GT_LDB + 4 * c) = __ldg(reinterpret_cast<const float4*>(Bm + (long long)(k0 + k) * ldb) + c);
      }
    } else {
      for (int e = tid; e < kc * N; e += GT_THREADS) {
        const int k = e / N, n = e - k * N;
        sm[k * GT_LDB + n] = __ldg(Bm + (long long)(k0 + k) * ldb + n);
      }
    }
    // ---- the long operand: issue this pass's loads before waiting for the staging barrier ----
    if (wgrad) {
      const int m = m0 + lane;
      constexpr int J = GT_KC / GT_WARPS;             // 32 k per warp per pass
      float a[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int k = w + GT_WARPS * j;
        a[j] = (k < kc && m < M) ? __ldg(A + (long long)(k0 + k) * lda + m) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int k = w + GT_WARPS * j;
        if (k < kc) {                                 // warp-uniform
          asum += a[j];
#pragma unroll
          for (int c = 0; c < GT_NMAX / 4; ++c)
            if (c < n4) {
              const float4 b = *reinterpret_cast<const float4*>(sm + k * GT_LDB + 4 * c);
              acc[4 * c + 0] = fmaf(a[j], b.x, acc[4 * c + 0]);
              acc[4 * c + 1] = fmaf(a[j], b.y, acc[4 * c + 1]);
              acc[4 * c + 2] = fmaf(a[j], b.z, acc[4 * c + 2]);
              acc[4 * c + 3] = fmaf(a[j], b.w, acc[4 * c + 3]);
            }
        }
      }
    } else {
      const int m = m0 + w;
      constexpr int J = GT_KC / 32;                   // 16 k per lane per pass
      float a[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int k = lane + 32 * j;
        a[j] = (k < kc && m < M) ? __ldg(A + (long long)m * lda + k0 + k) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int k = lane + 32 * j;
        if (k < kc) {
#pragma unroll
          for (int c = 0; c < GT_NMAX / 4; ++c)
            if (c < n4) {
              const float4 b = *reinterpret_cast<const float4*>(sm + k * GT_LDB + 4 * c);
              acc[4 * c + 0] = fmaf(a[j], b.x, acc[4 * c + 0]);
              acc[4 * c + 1] = fmaf(a[j], b.y, acc[4 * c + 1]);
              acc[4 * c + 2] = fmaf(a[j], b.z, acc[4 * c + 2]);
              acc[4 * c + 3] = fmaf(a[j], b.w, acc[4 * c + 3]);
            }
        }
      }
    }
  }

  float* __restrict__ C = P.C + (long long)rep * P.rsC;
  if (wgrad) {
    __syncthreads();                                  // everyone is done reading the B chunk
    float* red = sm + (w * 32 + lane) * (GT_NMAX + 1);
#pragma unroll
    for (int n = 0; n < GT_NMAX; ++n) red[n] = acc[n];
    red[GT_NMAX] = asum;
    __syncthreads();
    const bool want_c2 = P.C2 != nullptr;
    for (int e = tid; e < 32 * (N + 1); e += GT_THREADS) {
      const int mm = e & 31, n = e >> 5, m = m0 + mm;
      if (m >= M) continue;
      const int col = (n == N) ? GT_NMAX : n;
      float s = 0.f;
#pragma unroll
      for (int ww = 0; ww < GT_WARPS; ++ww) s += sm[(ww * 32 + mm) * (GT_NMAX + 1) + col];
      if (n < N) C[(long long)m * P.ldc + n] = s;
      else if (want_c2) (P.C2 + (long long)rep * P.rsC2)[m] = s;
    }
  } else {
    const int m = m0 + w;
    // 16 columns x 32 lanes -> one column per lane pair with a halving butterfly (16 shuffles instead of 80): at offset o
    // a lane keeps the half of its columns selected by bit o of its id and adds the partner's copy of that half; after
    // offsets 16, 8, 4, 2 lane l holds column l >> 1, offset 1 adds the two lanes of the pair.  Fixed tree -> reproducible.
#pragma unroll
    for (int o = 16, n = GT_NMAX; o >= 2; o >>= 1, n >>= 1) {
      const bool up = (lane & o) != 0;
#pragma unroll
      for (int i = 0; i < n / 2; ++i) {
        const float send = up ? acc[i] : acc[i + n / 2];
        const float keep = up ? acc[i + n / 2] : acc[i];
        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
    float v = acc[0] + __shfl_xor_sync(0xffffffffu, acc[0], 1);
    const int col = lane >> 1;
    if (m < M && col < N && (lane & 1) == 0) {
      if (P.mask != nullptr) {
        const float* __restrict__ mask = P.mask + (long long)rep * P.rsMask;
        if (!(mask[(long long)m * P.ldmask + col] > 0.f)) v = 0.f;
      }
      C[(long long)m * P.ldc + col] = v;
    }
  }
}

}  // namespace bsac
