// Gradient-norm clipping (b200sac_cfg.grad_clip): torch.nn.utils.clip_grad_norm_(params, max_norm) over the parameters of
// one optimizer, evaluated inside the step between its last gradient and its first optimizer write.
//   g    = the gradient Adam reads: the split-K slices summed in index order (what b200sac_export(GRADS) returns)
//   norm = sqrt(sum g_i^2), the squares and sums in fp64, in an order that depends on the slice length alone
//   coef = (float) min(1, max_norm / (norm + 1e-6)), evaluated in fp64 and rounded once; adam_kernel<true> runs on g * coef
// A NaN quotient (an infinite threshold over an infinite norm, or a NaN gradient) gives coef = 1: no scaling.
#pragma once
#include "sac_kernels.cuh"

namespace bsac {

constexpr int kClipCols = 3;          // [R][3] per replica: 0 critic, 1 actor, 2 CARE(O) context encoder
constexpr int kGradNormMaxBlocks = 592;

// CTAs of an element-wise pass over n floats (grad_sqnorm_kernel and adam_kernel): 1024 floats per CTA, at most 592
B200_HD int elementwise_blocks(long long n) {
  long long nb = (n + 256 * 4 - 1) / (256 * 4);
  if (nb < 1) nb = 1;
  if (nb > kGradNormMaxBlocks) nb = kGradNormMaxBlocks;
  return (int)nb;
}

struct GradNormArgs {
  const float* g; const float* gx; long long xs; int nx;   // slice base (replica 0), extra split-K slices like AdamArgs
  long long rsM, n;
  int which;                  // Counters slot of the optimizer (0 critic, 1 actor, 4 context encoder)
  int col;                    // its column of the [R][3] tables
  const Counters* cnt;
  const double* thr;          // [R][3] thresholds (b200sac_set_grad_clip)
  float* coef;                // [R][3] clip coefficients of the step (adam_kernel<true> reads them)
  float* norms;               // [kLossSlots][R][3] mapped pinned ring of the pre-clip norms
  double* part;               // [R][gridDim.x] per-CTA partial sums
  unsigned* ticket;           // [R] CTAs done; the last one resets it
  int R;
};

B200_D double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// fixed-order block sum of 256 threads (shuffle trees, then the 8 warp sums in index order); valid in thread 0
B200_D double block_sum_d(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_d(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
#pragma unroll
    for (int q = 0; q < 8; ++q) s += red[q];
  return s;
}

// grid (nb, R), 256 threads.  Each CTA walks the slice exactly like adam_kernel (same float4 groups, same slice adds), writes
// its fp64 partial, and the last CTA of a replica (ticket counter behind a fence) sums the partials in index order and
// writes the norm, the coefficient and the ring entry.  The actor's launch returns at entry on a critic-only step and
// reports NaN.
__global__ void __launch_bounds__(256) grad_sqnorm_kernel(StepConst K, GradNormArgs P) {
  const int rep = blockIdx.y, tid = threadIdx.x;
  const bool skip = P.which == 1 && !(sched_of(P.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  __shared__ double red[8];
  __shared__ bool s_last;
  const long long cell = (long long)rep * kClipCols + P.col;
  if (skip) {
    if (blockIdx.x == 0 && tid == 0) {
      const long long slot = (P.cnt[rep].v[3] - 1) % kLossSlots;
      const float nan = __int_as_float(0x7fc00000);
      P.norms[slot * P.R * kClipCols + cell] = nan;
      P.coef[cell] = nan;
    }
    return;
  }
  const int nb = gridDim.x;
  const float4* __restrict__ g4 = reinterpret_cast<const float4*>(P.g + rep * P.rsM);
  const float4* __restrict__ gx4 = reinterpret_cast<const float4*>(P.gx + rep * P.rsM);
  const long long n4 = P.n >> 2, xs4 = P.xs >> 2;
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * 256 + tid; i < n4; i += (long long)nb * 256) {
    float4 gv = g4[i];
    for (int sx = 0; sx < P.nx; ++sx) {
      const float4 ge = gx4[(long long)sx * xs4 + i];
      gv.x += ge.x; gv.y += ge.y; gv.z += ge.z; gv.w += ge.w;
    }
    acc += (double)gv.x * (double)gv.x;      // (a float times a float is exact in fp64)
    acc += (double)gv.y * (double)gv.y;
    acc += (double)gv.z * (double)gv.z;
    acc += (double)gv.w * (double)gv.w;
  }
  const double s = block_sum_d(acc, red);
  if (tid == 0) {
    P.part[(long long)rep * nb + blockIdx.x] = s;
    __threadfence();
    s_last = atomicAdd(&P.ticket[rep], 1u) == (unsigned)(nb - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double t = 0.0;
  for (int j = tid; j < nb; j += 256) t += __ldcg(&P.part[(long long)rep * nb + j]);
  const double tot = block_sum_d(t, red);
  if (tid == 0) {
    P.ticket[rep] = 0;
    const double norm = sqrt(tot);
    const double q = P.thr[cell] / (norm + 1e-6);
    const long long slot = (P.cnt[rep].v[3] - 1) % kLossSlots;
    P.norms[slot * P.R * kClipCols + cell] = (float)norm;
    P.coef[cell] = (float)(q < 1.0 ? q : 1.0);
  }
}

}  // namespace bsac
