// Gradient surgery (b200sac_cfg.pcgrad): PCGrad (Yu et al., NeurIPS 2020) over the T per-task gradients of one optimizer,
// evaluated inside the step between its last gradient and its Adam launch.
//   g_t  = gradient slice t: the weight and bias gradients over the minibatch rows of task t (rows t*P .. t*P+P-1, P = B/T)
//   G_jk = sum_e g_j[e] g_k[e] in fp64, in an order that depends on the slice length and T alone
//   c^(i): for j in the permutation pi_i, dot = G_ij - sum_k c_k G_kj (k ascending); dot < 0 -> c_j += dot / G_jj
//   w_k  = (float)(1 - sum_i c^(i)_k) (i ascending); adam_kernel<false, true> runs on sum_k fp32(w_k g_k) in index order
// With the replica's switch off the permutations are still drawn and G still computed, but nothing projects: w = 1.
#pragma once
#include "clip_kernels.cuh"

namespace bsac {

constexpr int kPcMaxTasks = 64;
constexpr int kPcMaxPairSlots = 9;        // ceil(64 * 65 / 2 / 256) pair slots per thread

struct PcgArgs {
  const float* g; const float* gx; long long xs;   // slice 0 base (replica 0), slices 1..T-1 at gx + (t-1) * xs
  long long rsM, n;
  int T, opt;                  // opt: 0 critic (counter slot 0), 1 actor (slot 1)
  const Counters* cnt;
  const int* on;               // [R][2] switches (b200sac_set_pcgrad)
  double* part;                // [R][gridDim.x][T(T+1)/2] per-CTA partial products
  unsigned* ticket;            // [R] CTAs done; the last one resets it
  double* G;                   // [R][2][T][T] record: Gram matrix
  float* w;                    // [R][2][T] record and Adam's weights
  int* perm;                   // [R][2][T][T] record: permutation pi_i of row i
  unsigned long long* mask;    // [R][2][T] record: bit j of mask[i] = task i was projected onto task j
  const int* tid; long long rsR; int B;            // the critic launch counts the rows whose task id is not i / P ...
  int* bad;                    // ... into bad[rep]
  unsigned long long seed;
};

B200_HD int pcgrad_pairs(int T) { return T * (T + 1) / 2; }
// threads that share one pair of a 256-element chunk (interleaved elements): the largest power of two <= 256 / pairs, <= 32
B200_HD int pcgrad_tpp(int T) {
  int t = 1;
  while (t < 32 && 2 * t * pcgrad_pairs(T) <= 256) t *= 2;
  return t;
}
// chunk row pitch in floats.  The tpp lanes of a pair read columns x = sg (mod tpp) of rows j and k, and the lanes of
// neighbouring pairs usually share j and have k one apart: a pitch of 256 + tpp puts row k + 1's columns tpp banks
// after row k's, so the 32 lanes of a warp read 32 different banks.
B200_HD int pcgrad_pitch(int T) { return 256 + pcgrad_tpp(T); }
// dynamic shared memory: a chunk [T][pitch] floats, reused for G and the coefficients [2][T][T] doubles (T <= 64)
inline size_t pcgrad_smem(int T) { return (size_t)T * pcgrad_pitch(T) * sizeof(float); }

// Fisher-Yates over 0..T-1 for row i: Philox keyed by (seed, replica), counter (step, optimizer, i, draw)
B200_D void pcgrad_perm(unsigned long long seed, int rep, long long step, int opt, int i, int T, int* out) {
  for (int k = 0; k < T; ++k) out[k] = k;
  const Philox ph(seed ^ (0xD1B54A32D192ED03ull * (unsigned long long)(rep + 1)));
  uint32_t rnd[4];
  for (int m = T - 1, q = 0; m >= 1; --m, ++q) {
    if ((q & 3) == 0) ph((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)(opt * kPcMaxTasks + i), 0xC6A0u + (uint32_t)(q >> 2), rnd);
    const int j = (int)(((unsigned long long)rnd[q & 3] * (unsigned long long)(m + 1)) >> 32);
    const int t = out[m]; out[m] = out[j]; out[j] = t;
  }
}

// grid (nb, R), 256 threads, pcgrad_smem(T) bytes.  Every CTA walks 256-element chunks c = blockIdx.x, +nb, ... of the
// slices (nb = elementwise_blocks(n): the order depends on n alone), stages the T slices of a chunk in shared memory and
// accumulates each pair (j <= k) over it, tpp threads per pair on interleaved elements; it writes its fp64 partials and
// the last CTA of a replica (ticket behind a fence) sums them in an order fixed by nb and T, then solves for c and w, one
// thread per task.
// The actor's launch returns at entry on a critic-only step and records NaN weights.
__global__ void __launch_bounds__(256) pcgrad_kernel(StepConst K, PcgArgs P) {
  const int rep = blockIdx.y, tid = threadIdx.x, T = P.T;
  const long long cell = (long long)rep * 2 + P.opt;
  KStamp ks_;
  extern __shared__ __align__(16) float pc_sm[];
  __shared__ double red[8];
  __shared__ bool s_last;
  if (P.opt == 1 && !(sched_of(P.cnt, rep) & SCHED_ACTOR)) {
    if (blockIdx.x == 0) {
      const double dnan = __longlong_as_double(0x7ff8000000000000ll);
      for (int e = tid; e < T * T; e += 256) P.G[cell * T * T + e] = dnan;
      if (tid < T) { P.w[cell * T + tid] = __int_as_float(0x7fc00000); P.mask[cell * T + tid] = 0ull; }
    }
    return;
  }
  const int np = pcgrad_pairs(T), tpp = pcgrad_tpp(T), pitch = pcgrad_pitch(T), nb = gridDim.x;
  int pj[kPcMaxPairSlots], pk[kPcMaxPairSlots];
  double acc[kPcMaxPairSlots];
#pragma unroll
  for (int q = 0; q < kPcMaxPairSlots; ++q) {
    acc[q] = 0.0;
    int p = (tid + q * 256) / tpp, j = 0;
    if (p >= np) { pj[q] = -1; pk[q] = -1; continue; }
    while (p >= T - j) { p -= T - j; ++j; }
    pj[q] = j; pk[q] = j + p;
  }
  const float* g = P.g + rep * P.rsM;
  const float* gx = P.gx + rep * P.rsM;
  const long long nchunk = (P.n + 255) / 256;
  for (long long c = blockIdx.x; c < nchunk; c += nb) {
    const long long e = c * 256 + tid;
    for (int t0 = 0; t0 < T; t0 += 8) {     // eight slices' loads in flight before the first store
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int t = t0 + q;
        v[q] = (t < T && e < P.n) ? (t == 0 ? g[e] : gx[(long long)(t - 1) * P.xs + e]) : 0.f;
      }
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (t0 + q < T) pc_sm[(t0 + q) * pitch + tid] = v[q];
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kPcMaxPairSlots; ++q) {
      if (pj[q] < 0) continue;
      const float* a = pc_sm + pj[q] * pitch;
      const float* b = pc_sm + pk[q] * pitch;
      double s = acc[q];
      for (int x = (tid + q * 256) % tpp; x < 256; x += tpp) s += (double)a[x] * (double)b[x];   // (exact products)
      acc[q] = s;
    }
    __syncthreads();
  }
  // this CTA's partial of every pair: its tpp threads' sums in thread order
  double* sd = reinterpret_cast<double*>(pc_sm);      // [np * tpp] (<= the chunk's bytes for T <= 64)
#pragma unroll
  for (int q = 0; q < kPcMaxPairSlots; ++q)
    if (pj[q] >= 0) sd[tid + q * 256] = acc[q];
  __syncthreads();
  double* part = P.part + (long long)rep * nb * np + (long long)blockIdx.x * np;
  for (int p = tid; p < np; p += 256) {
    double s = 0.0;
    for (int u = 0; u < tpp; ++u) s += sd[p * tpp + u];
    part[p] = s;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&P.ticket[rep], 1u) == (unsigned)(nb - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid == 0) P.ticket[rep] = 0;
  // Gram matrix: the CTA partials summed in CTA order, in tpp contiguous segments per pair (eight loads in flight per
  // thread: one serial L2 round trip per partial would dominate the launch), the segments then summed in order
  const double* prt = P.part + (long long)rep * nb * np;
  for (int u = tid; u < np * tpp; u += 256) {
    const int p = u / tpp, sg = u % tpp;
    const int b1 = (int)((long long)nb * (sg + 1) / tpp);
    int b = (int)((long long)nb * sg / tpp);
    double s = 0.0;
    for (; b + 8 <= b1; b += 8) {
      double v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = __ldcg(&prt[(long long)(b + q) * np + p]);
#pragma unroll
      for (int q = 0; q < 8; ++q) s += v[q];
    }
    for (; b < b1; ++b) s += __ldcg(&prt[(long long)b * np + p]);
    sd[u] = s;
  }
  __syncthreads();
  double gp[kPcMaxPairSlots];
#pragma unroll
  for (int q = 0; q < kPcMaxPairSlots; ++q) {
    const int p = tid + q * 256;
    double s = 0.0;
    if (p < np)
      for (int sg = 0; sg < tpp; ++sg) s += sd[p * tpp + sg];
    gp[q] = s;
  }
  __syncthreads();
  double* Gs = sd;                    // [T][T]
  double* cs = sd + T * T;            // [T][T]: row i = c^(i)
  double* Gout = P.G + cell * T * T;
#pragma unroll
  for (int q = 0; q < kPcMaxPairSlots; ++q) {
    const int p = tid + q * 256;
    if (p >= np) continue;
    int j = 0, r = p;
    while (r >= T - j) { r -= T - j; ++j; }
    const int k = j + r;
    Gs[j * T + k] = gp[q]; Gs[k * T + j] = gp[q];
    Gout[j * T + k] = gp[q]; Gout[k * T + j] = gp[q];
  }
  if (P.bad) {                        // rows out of task-block order (b200sac_step: the caller's promise, checked here)
    const int per = P.B / T;
    double nbad = 0.0;
    for (int i = tid; i < P.B; i += 256) nbad += (P.tid + rep * P.rsR)[i] != i / per ? 1.0 : 0.0;
    const double tot = block_sum_d(nbad, red);
    if (tid == 0) P.bad[rep] = (int)tot;
  }
  __syncthreads();
  const bool on = P.on[cell] != 0;
  if (tid < T) {
    const int i = tid;
    int* pm = P.perm + (cell * T + i) * T;
    pcgrad_perm(P.seed, rep, P.cnt[rep].v[3], P.opt, i, T, pm);
    double* ci = cs + i * T;
    for (int k = 0; k < T; ++k) ci[k] = 0.0;
    unsigned long long m = 0ull;
    if (on)
      for (int pos = 0; pos < T; ++pos) {
        const int j = pm[pos];
        double s = 0.0;
        for (int k = 0; k < T; ++k) s += ci[k] * Gs[k * T + j];
        const double dot = Gs[i * T + j] - s;
        if (dot < 0.0) { ci[j] += dot / Gs[j * T + j]; m |= 1ull << j; }
      }
    P.mask[cell * T + i] = m;
  }
  __syncthreads();
  if (tid < T) {
    double s = 0.0;
    for (int i = 0; i < T; ++i) s += cs[i * T + tid];
    P.w[cell * T + tid] = (float)(1.0 - s);
  }
}

}  // namespace bsac
