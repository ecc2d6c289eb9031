// Gradient surgery (b200sac_cfg.pcgrad): PCGrad (Yu et al., NeurIPS 2020) over the T per-task gradients of one optimizer,
// evaluated inside the step between its last gradient and its Adam launch.
//   g_t  = gradient slice t: the weight and bias gradients over the minibatch rows of task t (rows t*P .. t*P+P-1, P = B/T)
//   G_jk = sum_e g_j[e] g_k[e] in fp64, in an order that depends on the slice length and T alone
//   c^(i): for j in the permutation pi_i, dot = G_ij - sum_k c_k G_kj (k ascending); dot < 0 -> c_j += dot / G_jj
//   w_k  = (float)(1 - sum_i c^(i)_k) (i ascending); adam_kernel<false, true> runs on sum_k fp32(w_k g_k) in index order
// With the replica's switch off the permutations are still drawn and G still computed, but nothing projects: w = 1.
//
// CAGrad (Liu et al., NeurIPS 2021) replaces the projections when the optimizer's coefficient c (b200sac_set_cagrad) is
// > 0: cagrad_solve below turns G into the weights of CAGrad's update (g_0 + lambda g_w) / (1 + c^2), in fp64, on one
// warp.  Lane l owns tasks l and l + 32.  No fused multiply-add (the library builds with -fmad=false).  Every sum over
// tasks, tsum(v), is one fixed tree: n = 32 for T <= 32, else 64, v padded with zeros to n; for n = 64 first
// s_l = v_l + v_{l+32} (l < 32), then s_l = s_l + s_{l xor o} for o = 16, 8, 4, 2, 1; every lane ends with s_0, so
// lanes without a task never divide by a zero sum (a slow path of the fp64 division).  tmax is the same tree with max and -inf padding.  Sums over k inside one task's value (the matrix-vector
// products, the row sums of A) are serial over k ascending from 0.0.
//   s  = tsum(sqrt(G_tt)) / T;  degenerate (w = 1, ibest = -2) if any G entry is not finite or s is 0 or not finite
//   A  = G / (s * s) in place of G;  a_j = (sum_k A_kj) / T;  abar = tsum(a) / T;  ce = c * sqrt(abar + 1e-4)
//   x = m = 0;  lr = 5 * c;  mu = 0.5;  best = +inf;  for it = 0 .. 20:
//     e = exp(x - tmax(x));  v_j = sum_k A_kj e_k;  Z = tsum(e);  ev = tsum(e v);  ea = tsum(e a)
//     p = e / Z;  u = v / Z;  q = ev / (Z * Z);  pa = ea / Z           (p = softmax(x), u = A p, q = p'Ap, pa = p.a)
//     r = sqrt(q + 1e-4);  F = pa + ce * r;  F < best: best = F, xbest = x, ibest = it
//     it < 20:  h_j = a_j + ce * u_j / r;  ph = pa + ce * q / r (= p.h);  d_j = p_j * (h_j - ph)
//               m = (it == 0 ? d : mu * m + d);  x = x - lr * m
//   p* and q* = p*'Ap* from xbest as in an iteration;  lambda = ce / (sqrt(q* + 1e-4) + 1e-4)
//   w_t = (float)((1 + T * lambda * p*_t) / (1 + c * c))          (oracle/cagrad_ref.py mirrors this order)
#pragma once
#include "clip_kernels.cuh"

namespace bsac {

constexpr int kPcMaxTasks = 64;
constexpr int kPcMaxPairSlots = 9;        // ceil(64 * 65 / 2 / 256) pair slots per thread
constexpr int kCagIters = 20;             // SGD steps of the CAGrad dual (21 evaluations of F)
constexpr int kCagScalars = 4;            // record per (replica, optimizer): lambda, best F, F at iteration 0, s
constexpr int kCagVecs = 4;               // T-long fp64 vectors of the solve in shared memory

// Where cagrad_solve writes one (replica, optimizer)'s result: w [T] (what Adam reads), p* [T], the kCagScalars
// scalars and ibest (-1: CAGrad did not run, -2: degenerate G, else the iteration of the best F).
struct CagOut { float* w; double* p; double* f; int* ibest; };

B200_D void cagrad_not_run(const CagOut& o, int T, int tid) {
  const double dnan = __longlong_as_double(0x7ff8000000000000ll);
  if (tid < T) o.p[tid] = dnan;
  if (tid < kCagScalars) o.f[tid] = dnan;
  if (tid == 0) *o.ibest = -1;
}

// One warp (all 32 lanes; lane l owns tasks l and l + 32).  A: [T][T] fp64 shared, G on entry (symmetric), A after.
// sv: kCagVecs * T doubles of shared scratch (e, xbest, a, m).  Reductions are register shuffles.
B200_D double cag_tsum(double v0, double v1, int n) {
  double s = n == 64 ? v0 + v1 : v0;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s = s + __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}
B200_D double cag_tmax(double v0, double v1, int n) {
  double s = n == 64 ? fmax(v0, v1) : v0;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s = fmax(s, __shfl_xor_sync(0xffffffffu, s, o));
  return s;
}

B200_D void cagrad_solve(double* A, double* sv, int T, double c, const CagOut& o) {
  const int lane = threadIdx.x & 31, j1 = lane + 32;
  const bool h0 = lane < T, h1 = j1 < T;         // the lane owns task lane / task lane + 32
  const int n = T > 32 ? 64 : 32;
  bool fin = true;
  for (int j = lane; j < T; j += 32)
    for (int k = 0; k < T; ++k) fin = fin && isfinite(A[j * T + k]);
  fin = __all_sync(0xffffffffu, fin);
  const double s = cag_tsum(h0 ? sqrt(A[lane * T + lane]) : 0.0, h1 ? sqrt(A[j1 * T + j1]) : 0.0, n) / T;
  if (!fin || !(s > 0.0) || isinf(s)) {
    const double dnan = __longlong_as_double(0x7ff8000000000000ll);
    for (int j = lane; j < T; j += 32) { o.w[j] = 1.0f; o.p[j] = dnan; }
    if (lane < kCagScalars) o.f[lane] = lane == 3 ? s : dnan;
    if (lane == 0) *o.ibest = -2;
    return;
  }
  __syncwarp();
  const double s2 = s * s;
  for (int j = lane; j < T; j += 32)
    for (int k = 0; k < T; ++k) A[j * T + k] = A[j * T + k] / s2;
  __syncwarp();
  double a0 = 0.0, a1 = 0.0;
  for (int k = 0; k < T; ++k) {
    if (h0) a0 += A[k * T + lane];
    if (h1) a1 += A[k * T + j1];
  }
  a0 = a0 / T; a1 = a1 / T;
  double* av = sv + 2 * T;     // [T] a (kept in shared memory: registers are the Gram pass's)
  if (h0) av[lane] = a0;
  if (h1) av[j1] = a1;
  const double abar = cag_tsum(a0, a1, n) / T;
  const double ce = c * sqrt(abar + 1e-4), lr = 5.0 * c, mu = 0.5;
  double* ev = sv;             // [T] e of the evaluation in flight
  double* bv = sv + T;         // [T] xbest
  // one evaluation at x: p, u = A p (the lane's tasks), q = p'Ap, pa = p.a
  double p0, p1, u0, u1, q, pa;
  auto evaluate = [&](double x0, double x1) {
    const double mx = cag_tmax(h0 ? x0 : -INFINITY, h1 ? x1 : -INFINITY, n);
    const double e0 = h0 ? exp(x0 - mx) : 0.0, e1 = h1 ? exp(x1 - mx) : 0.0;
    __syncwarp();                // the previous evaluation's reads of ev are done
    if (h0) ev[lane] = e0;
    if (h1) ev[j1] = e1;
    __syncwarp();
    double v0 = 0.0, v1 = 0.0;
#pragma unroll 2
    for (int k = 0; k < T; ++k) {
      const double ek = ev[k];
      if (h0) v0 += A[k * T + lane] * ek;
      if (h1) v1 += A[k * T + j1] * ek;
    }
    const double Z = cag_tsum(e0, e1, n);
    const double Ev = cag_tsum(e0 * v0, e1 * v1, n);
    const double Ea = cag_tsum(h0 ? e0 * av[lane] : 0.0, h1 ? e1 * av[j1] : 0.0, n);
    p0 = h0 ? e0 / Z : 0.0; p1 = h1 ? e1 / Z : 0.0;
    u0 = h0 ? v0 / Z : 0.0; u1 = h1 ? v1 / Z : 0.0;
    q = Ev / (Z * Z); pa = Ea / Z;
  };
  double* mv = sv + 3 * T;     // [T] momentum
  double x0 = 0.0, x1 = 0.0;
  double best = INFINITY;
  int ib = 0;
  for (int it = 0; it <= kCagIters; ++it) {
    evaluate(x0, x1);
    const double r = sqrt(q + 1e-4);
    const double F = pa + ce * r;
    if (it == 0 && lane == 0) o.f[2] = F;
    if (F < best) {
      best = F; ib = it;
      if (h0) bv[lane] = x0;
      if (h1) bv[j1] = x1;
    }
    if (it == kCagIters) break;
    const double ph = pa + ce * q / r;
    const double d0 = h0 ? p0 * ((av[lane] + ce * u0 / r) - ph) : 0.0;
    const double d1 = h1 ? p1 * ((av[j1] + ce * u1 / r) - ph) : 0.0;
    if (h0) { const double m = it == 0 ? d0 : mu * mv[lane] + d0; mv[lane] = m; x0 = x0 - lr * m; }
    if (h1) { const double m = it == 0 ? d1 : mu * mv[j1] + d1; mv[j1] = m; x1 = x1 - lr * m; }
  }
  __syncwarp();
  evaluate(h0 ? bv[lane] : 0.0, h1 ? bv[j1] : 0.0);
  const double lam = ce / (sqrt(q + 1e-4) + 1e-4);
  if (h0) { o.w[lane] = (float)((1.0 + T * lam * p0) / (1.0 + c * c)); o.p[lane] = p0; }
  if (h1) { o.w[j1] = (float)((1.0 + T * lam * p1) / (1.0 + c * c)); o.p[j1] = p1; }
  if (lane == 0) { o.f[0] = lam; o.f[1] = best; o.f[3] = s; *o.ibest = ib; }
}

// Stand-alone solve on a caller-given G [T][T] (b200sac_cagrad_solve_test): one CTA of 32 threads, (T + kCagVecs) * T
// doubles of dynamic shared memory.
__global__ void __launch_bounds__(32) cagrad_test_kernel(const double* G, int T, double c, CagOut o) {
  extern __shared__ __align__(16) double cg_sm[];
  for (int e = threadIdx.x; e < T * T; e += 32) cg_sm[e] = G[e];
  __syncwarp();
  cagrad_solve(cg_sm, cg_sm + T * T, T, c, o);
}

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
  const double* cac;           // [R][2] CAGrad coefficients c (b200sac_set_cagrad); c > 0 replaces the projections
  double* cgp;                 // [R][2][T] record: CAGrad's p*
  double* cgf;                 // [R][2][kCagScalars] record: lambda, best F, F at iteration 0, s
  int* cgi;                    // [R][2] record: ibest
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
// thread per task, or, with the optimizer's CAGrad coefficient > 0, runs cagrad_solve on warp 0 over the shared copy of G
// (overwritten with A; the coefficient region holds its vectors).
// The actor's launch returns at entry on a critic-only step and records NaN weights.
// Three CTAs per SM (80 registers) keep the Gram pass's occupancy; the CAGrad solve keeps its per-task vectors other than
// x in shared memory so that it fits that budget without spilling.
__global__ void __launch_bounds__(256, 3) pcgrad_kernel(StepConst K, PcgArgs P) {
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
      cagrad_not_run(CagOut{P.w + cell * T, P.cgp + cell * T, P.cgf + cell * kCagScalars, P.cgi + cell}, T, tid);
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
  const double cag = P.cac[cell];
  const bool on = P.on[cell] != 0 && !(cag > 0.0);
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
  const CagOut co{P.w + cell * T, P.cgp + cell * T, P.cgf + cell * kCagScalars, P.cgi + cell};
  if (cag > 0.0) {
    if (tid < 32) cagrad_solve(Gs, cs, T, cag, co);
    return;
  }
  if (tid < T) {
    double s = 0.0;
    for (int i = 0; i < T; ++i) s += cs[i * T + tid];
    P.w[cell * T + tid] = (float)(1.0 - s);
  }
  cagrad_not_run(co, T, tid);
}

}  // namespace bsac
