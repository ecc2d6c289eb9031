// Grouped fp32 FFMA GEMM for the MLP layers of the SAC step (exact-fp32 path, and the thin
// first/last-layer problems of the wgmma path).
//
// One launch runs G independent problems x R replicas (blockIdx.z = rep * G + g), so the
// twin critics / target critics / the actor's 2B-row batch are a single grid.  Three
// problem kinds share one tile engine and differ only in how operand tiles are fetched:
//
//   FWD   C[m][n] = act( sum_k A[m][k] * W[n][k] + bias[n] )        nn.Linear forward
//                   (reference: LunarLander_Distributed_SAC/src/model.py:41-44,119-125)
//   DGRAD C[m][n] = ( sum_k dY[m][k] * W[k][n] ) * [mask[m][n] > 0]   input gradient, ReLU' fused
//   WGRAD C[m][n] = sum_k dY[k][m] * X[k][n] ;  C2[m] = sum_k dY[k][m]   weight + bias gradient
//
// The problems are tiny (256..1280 rows, 8..400 wide) and sit on the critical path of a
// strictly sequential step, so the kernel is built for LATENCY: 32x32 output tiles (many CTAs),
// 64-wide k chunks fetched as 128-bit loads with the next chunk's loads in flight (registers)
// while the current one is computed out of shared memory, operands kept in the orientation they
// have in global memory (row = m|n for K-contiguous operands, row = k for MN-contiguous ones) with
// paddings that make every shared-memory access conflict-free.
// Reductions run over the full K inside one CTA in a fixed order (no split-K, no atomics),
// so results are bit-reproducible run to run and replica to replica.
#pragma once
#include "common.cuh"

namespace bsac {

enum { GEMM_FWD = 0, GEMM_DGRAD = 1, GEMM_WGRAD = 2 };

struct GemmProb {
  const float* A;
  const float* B;
  const float* bias;   // FWD only (may be null)
  const float* mask;   // DGRAD only (may be null): activation whose >0 gates the gradient
  float* C;
  float* C2;           // WGRAD only (may be null): bias gradient
  long long rsA, rsB, rsBias, rsMask, rsC, rsC2;   // per-replica strides (floats)
  int M, N, K;
  int lda, ldb, ldc, ldmask;
  int mode;
  int relu;
};

constexpr int GS_T = 32;               // tile is GS_T x GS_T outputs
constexpr int GS_KC = 64;              // k chunk
constexpr int GS_LDK = GS_KC + 4;      // row pitch of a K-contiguous operand tile  [32][68]
constexpr int GS_LDM = GS_T + 4;       // row pitch of an MN-contiguous operand tile [64][36]
constexpr int GS_TILE_FLOATS = (GS_T * GS_LDK > GS_KC * GS_LDM) ? GS_T * GS_LDK : GS_KC * GS_LDM;   // 2304
constexpr int GS_THREADS = 256;
constexpr int GS_MAXG = 24;            // problems per launch (descriptors travel as kernel parameters)
constexpr int GS_INFLIGHT = 4;         // k chunks whose loads are issued before the first is consumed

struct GemmGroup {
  GemmProb p[GS_MAXG];
  int G;
  int sched_stride;    // ints between two replicas' schedule words
  const int* sched;    // actor-side launch: replica 0's schedule word (the launch is skipped on critic-only steps); null = always runs
};

// Fetch one operand chunk into registers (2 x float4 per thread).
//   kcontig: element (r, k) at P[r * ld + k], tile rows r0.., k range [k0, k0+64)
//   else   : element (r, k) at P[k * ld + r]
B200_D void gs_fetch(const float* __restrict__ P, int ld, bool kcontig, bool vec, int r0, int rlim, int k0, int klim,
                     int tid, float4 (&v)[2]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int e = tid + i * GS_THREADS;
    int row, col;          // row/col of the float4 in GLOBAL orientation: [row][col..col+3]
    int rbase, cbase, rmax, cmax;
    if (kcontig) { row = e >> 4; col = (e & 15) << 2; rbase = r0; cbase = k0; rmax = rlim; cmax = klim; }
    else         { row = e >> 3; col = (e & 7) << 2;  rbase = k0; cbase = r0; rmax = klim; cmax = rlim; }
    const int gr = rbase + row, gc = cbase + col;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gr < rmax) {
      const float* src = P + (long long)gr * ld + gc;
      if (vec && gc + 3 < cmax) {
        x = __ldg(reinterpret_cast<const float4*>(src));
      } else {
        if (gc < cmax) x.x = __ldg(src);
        if (gc + 1 < cmax) x.y = __ldg(src + 1);
        if (gc + 2 < cmax) x.z = __ldg(src + 2);
        if (gc + 3 < cmax) x.w = __ldg(src + 3);
      }
    }
    v[i] = x;
  }
}

B200_D void gs_stash(float* __restrict__ S, bool kcontig, int tid, const float4 (&v)[2]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int e = tid + i * GS_THREADS;
    if (kcontig) *reinterpret_cast<float4*>(S + (e >> 4) * GS_LDK + ((e & 15) << 2)) = v[i];
    else         *reinterpret_cast<float4*>(S + (e >> 3) * GS_LDM + ((e & 7) << 2)) = v[i];
  }
}

template <bool AK, bool BK>
B200_D void gs_compute(const float* __restrict__ As, const float* __restrict__ Bs, int tx, int ty, int kend, float (&acc)[2][2]) {
#pragma unroll 4
  for (int k4 = 0; k4 < kend; k4 += 4) {        // kend: valid k columns of this chunk rounded up to 4 (the tail is zero-filled)
    float a[2][4], b[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (AK) {
        const float4 t = *reinterpret_cast<const float4*>(As + (ty + 16 * i) * GS_LDK + k4);
        a[i][0] = t.x; a[i][1] = t.y; a[i][2] = t.z; a[i][3] = t.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) a[i][q] = As[(k4 + q) * GS_LDM + ty + 16 * i];
      }
      if (BK) {
        const float4 t = *reinterpret_cast<const float4*>(Bs + (tx + 16 * i) * GS_LDK + k4);
        b[i][0] = t.x; b[i][1] = t.y; b[i][2] = t.z; b[i][3] = t.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) b[i][q] = Bs[(k4 + q) * GS_LDM + tx + 16 * i];
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) acc[i][j] = fmaf(a[i][q], b[j][q], acc[i][j]);
  }
}

#ifdef GS_PROF   // scripts/micro/simt_lat.cu only: %globaltimer at four points of CTA (0,0,0)
__device__ unsigned long long g_gs_prof[4096];
__device__ int g_gs_prof_n = 0;
#define GS_MARK(i) do { if (prof_on) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(prof_t[i])); } while (0)
#else
#define GS_MARK(i) do { } while (0)
#endif

__global__ void __launch_bounds__(GS_THREADS) gemm_simt_kernel(const __grid_constant__ GemmGroup grp) {
  const int sched = grp.sched ? sched_word(grp.sched + (int)(blockIdx.z / grp.G) * grp.sched_stride) : SCHED_ACTOR;
  KStamp ks_;
#ifdef GS_PROF
  unsigned long long prof_t[4] = {0, 0, 0, 0};
  const bool prof_on = (threadIdx.x | blockIdx.x | blockIdx.y | blockIdx.z) == 0;
#endif
  GS_MARK(0);
  const int G = grp.G;
  const int g = blockIdx.z % G, rep = blockIdx.z / G;
  const GemmProb& P = grp.p[g];
  const int m0 = blockIdx.y * GS_T, n0 = blockIdx.x * GS_T;
  if (m0 >= P.M || n0 >= P.N) return;
  if (!(sched & SCHED_ACTOR)) return;

  const float* __restrict__ A = P.A + (long long)rep * P.rsA;
  const float* __restrict__ Bm = P.B + (long long)rep * P.rsB;
  const bool ak = (P.mode != GEMM_WGRAD);   // A element (m,k) at A[m*lda+k] else A[k*lda+m]
  const bool bk = (P.mode == GEMM_FWD);     // B element (n,k) at B[n*ldb+k] else B[k*ldb+n]
  const int M = P.M, N = P.N, K = P.K;
  const bool vecA = ((P.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool vecB = ((P.ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(Bm) & 15) == 0);

  __shared__ __align__(16) float As[2][GS_TILE_FLOATS];
  __shared__ __align__(16) float Bs[2][GS_TILE_FLOATS];

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float bsum = 0.f;   // WGRAD bias gradient, threads tid < 32 of the n-tile-0 CTAs
  const bool do_bsum = (P.mode == GEMM_WGRAD) && (P.C2 != nullptr) && (blockIdx.x == 0);

  // Epilogue operands (bias row / ReLU mask) are fetched NOW, together with the first operand tiles, so the
  // epilogue does not pay a second dependent L2 round trip.
  float ebias[2] = {0.f, 0.f};
  bool ekeep[2][2] = {{true, true}, {true, true}};
  if (P.mode == GEMM_FWD && P.bias != nullptr) {
    const float* __restrict__ bias = P.bias + (long long)rep * P.rsBias;
#pragma unroll
    for (int j = 0; j < 2; ++j) { const int n = n0 + tx + 16 * j; if (n < N) ebias[j] = __ldg(bias + n); }
  } else if (P.mode == GEMM_DGRAD && P.mask != nullptr) {
    const float* __restrict__ mask = P.mask + (long long)rep * P.rsMask;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
        if (m < M && n < N) ekeep[i][j] = __ldg(mask + (long long)m * P.ldmask + n) > 0.f;
      }
  }

  // Super-chunks of GS_INFLIGHT x 64 k columns: all loads of a super-chunk are issued before the first
  // is consumed, so a K <= 256 problem pays one global-memory round trip instead of one per chunk.
  for (int ks = 0; ks < K; ks += GS_KC * GS_INFLIGHT) {
    float4 ra[GS_INFLIGHT][2], rb[GS_INFLIGHT][2];
#pragma unroll
    for (int c = 0; c < GS_INFLIGHT; ++c) {
      const int k0 = ks + c * GS_KC;
      if (k0 < K) {
        gs_fetch(A, P.lda, ak, vecA, m0, M, k0, K, tid, ra[c]);
        gs_fetch(Bm, P.ldb, bk, vecB, n0, N, k0, K, tid, rb[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < GS_INFLIGHT; ++c) {
      const int k0 = ks + c * GS_KC;
      if (k0 < K) {                       // block-uniform
        const int buf = c & 1;            // double buffer: stash of chunk c+1 may overlap compute of chunk c
        gs_stash(As[buf], ak, tid, ra[c]);
        gs_stash(Bs[buf], bk, tid, rb[c]);
        __syncthreads();
        if (c == 0 && ks == 0) GS_MARK(1);
        const int kend = (K - k0 >= GS_KC) ? GS_KC : ((K - k0 + 3) & ~3);   // thin first layers: K = 8..53
        if (ak) {
          if (bk) gs_compute<true, true>(As[buf], Bs[buf], tx, ty, kend, acc);
          else gs_compute<true, false>(As[buf], Bs[buf], tx, ty, kend, acc);
        } else {
          gs_compute<false, false>(As[buf], Bs[buf], tx, ty, kend, acc);
        }
        if (do_bsum && tid < GS_T) {
#pragma unroll 8
          for (int kk = 0; kk < kend; ++kk) bsum += As[buf][kk * GS_LDM + tid];
        }
      }
    }
    __syncthreads();
  }

  GS_MARK(2);
  float* __restrict__ C = P.C + (long long)rep * P.rsC;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + ty + 16 * i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (P.mode == GEMM_FWD) {
        v += ebias[j];
        if (P.relu) v = fmaxf(v, 0.f);
      } else if (P.mode == GEMM_DGRAD) {
        if (!ekeep[i][j]) v = 0.f;
      }
      C[(long long)m * P.ldc + n] = v;
    }
  }
  if (do_bsum && tid < GS_T && (m0 + tid) < M) (P.C2 + (long long)rep * P.rsC2)[m0 + tid] = bsum;
#ifdef GS_PROF
  GS_MARK(3);
  if (prof_on) {
    const int i = atomicAdd(&g_gs_prof_n, 1);
    if (i < 1024) for (int q = 0; q < 4; ++q) g_gs_prof[i * 4 + q] = prof_t[q];
  }
#endif
}

}  // namespace bsac
