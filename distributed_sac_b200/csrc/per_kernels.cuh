// Prioritized experience replay on the device ring (Schaul et al. 2016, as used by Ape-X).
//
// Every (replica, task) sub-ring of a prioritized ring owns a sum-tree over its cap_per_task slots, padded to P = 2^levels
// leaves and stored as a heap: node 1 is the root, node n has the children 2n and 2n+1, leaf i is node P + i.
//   leaf      p_i = (prio_i + eps)^alpha in fp32 (the power is evaluated in fp64 and rounded once); empty slots hold 0
//   internal  the fp32 sum of its two children, always RECOMPUTED from them (never adjusted by a delta: the tree cannot drift)
// Sampling is stratified with replacement: slot j of a task's per = B/T rows draws u = (j + U(0,1)) S / per (S = root sum)
// and descends.  Importance weights w_i = (N_t p_i / S_t)^-beta (N_t = fill of the row's sub-ring) are divided by their
// maximum over the minibatch; both evaluated in fp64, rounded once.
// Priority update: prio_i = (|y - Q1| + |y - Q2|) / 2 from the step's own TD target and pre-update critic values; when an
// index appears more than once in a batch the HIGHEST batch slot wins.  A running max p per (replica, task) (initially 1)
// is the priority of newly written rows.
#pragma once
#include "sac_kernels.cuh"

namespace bsac {

struct PerTree {
  float* tree;                 // [R][T][2P]
  float* maxp;                 // [R][T] running maximum leaf value
  long long P;                 // leaves per tree (power of two >= cap)
  long long cap;               // cap_per_task
  int levels;                  // log2(P)
  int T;                       // sub-rings per replica, max(num_tasks, 1)
  double alpha, eps;
};

B200_D float* per_tree_of(const PerTree& Tr, int rep, int t) { return Tr.tree + ((long long)rep * Tr.T + t) * 2 * Tr.P; }

constexpr int kPerTopNodes = 4096;   // nodes of the top levels kept in shared memory, over all tasks of the replica (16 KB)
constexpr int kPerMaxB = 2048;       // batch <= 2048 (and set_priorities chunks)

B200_D double block_max_f64(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double m = red[0];
  for (int i = 1; i < nw; ++i) m = fmax(m, red[i]);
  return m;
}

// One CTA per replica (rep = rep0 + blockIdx.x): draws the replica's B rows, writes their ring indices and importance
// weights.  The Philox key is (seed, replica, draw counter, batch slot), the counter being the step index before this
// step's bump (cnt != nullptr, like sample_indices_kernel) or `fixed_step`.
__global__ void __launch_bounds__(512) per_sample_kernel(StepConst K, PerTree Tr, const Counters* __restrict__ cnt,
                                                         long long fixed_step, int rep0, const long long* __restrict__ fill,
                                                         const double* __restrict__ beta, int* __restrict__ idx_out,
                                                         float* __restrict__ w_out, long long rs_out, unsigned long long seed) {
  KStamp ks_;
  __shared__ float top[kPerTopNodes];
  __shared__ double wraw[kPerMaxB];
  __shared__ double red[32];
  const int rep = rep0 + blockIdx.x;
  const int B = K.B, T = Tr.T, per = B / T;
  // the top Lc levels of every task's tree (nodes 1 .. 2^Lc - 1) live in shared memory, the rest is read from L2
  int Lc = 12;
  while ((T << Lc) > kPerTopNodes) --Lc;
  if (Lc > Tr.levels + 1) Lc = Tr.levels + 1;
  const int topn = 1 << Lc;
  for (int e = threadIdx.x; e < T * topn; e += blockDim.x) {
    const int t = e >> Lc, n = e & (topn - 1);
    top[e] = n ? per_tree_of(Tr, rep, t)[n] : 0.f;
  }
  __syncthreads();
  const long long step = cnt ? cnt[rep].v[3] : fixed_step;
  const double b = beta[rep];
  Philox ph(seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(rep + 1));
  double mx = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const int t = i / per, j = i - t * per;
    const float* tree = per_tree_of(Tr, rep, t);
    const float* tt = top + t * topn;
    uint32_t rnd[4];
    ph((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)i, 0u, rnd);
    const double U = (double)((((unsigned long long)rnd[0] << 32) | rnd[1]) >> 11) * 0x1.0p-53;   // [0, 1)
    const float S = tt[1];
    double u = ((double)j + U) * (double)S / (double)per;
    long long node = 1;
    float p = S;
    for (int lv = 0; lv < Tr.levels; ++lv) {
      const long long l = 2 * node;
      const float Lv = l < topn ? tt[l] : tree[l];
      const float Rv = l + 1 < topn ? tt[l + 1] : tree[l + 1];
      // a zero-sum child is never entered, so rounding in u cannot reach an empty slot
      if (Lv > 0.f && (u < (double)Lv || !(Rv > 0.f))) { node = l; p = Lv; }
      else { u -= (double)Lv; node = l + 1; p = Rv; }
    }
    const long long leaf = node - Tr.P;
    (idx_out + (long long)blockIdx.x * rs_out)[i] = (int)((long long)t * Tr.cap + leaf);
    const double n_t = (double)fill[(long long)rep * T + t];
    const double wr = pow(n_t * (double)p / (double)S, -b);
    wraw[i] = wr;
    mx = fmax(mx, wr);
  }
  mx = block_max_f64(mx, red);
  for (int i = threadIdx.x; i < B; i += blockDim.x) (w_out + (long long)blockIdx.x * rs_out)[i] = (float)(wraw[i] / mx);
}

B200_D float per_leaf_value(const PerTree& Tr, double prio) { return (float)pow(prio + Tr.eps, Tr.alpha); }
// a row's priority from its TD target and both critics' values, in fp64
B200_D double td_priority(float y, float q1, float q2) {
  return 0.5 * (fabs((double)y - (double)q1) + fabs((double)y - (double)q2));
}

// One CTA per replica (rep = rep0 + blockIdx.x): n <= kPerMaxB priorities for the ring indices idx[0..n), either the raw
// values prio_in[i] or, when prio_in is null, the step's (|y - Q1| + |y - Q2|) / 2 (n = B, q = [2][B]).  Writes the leaves
// (highest slot wins a duplicated index), rebuilds their ancestors level by level and raises the running max p.  Optional
// outputs: the leaf value of every slot (p_out) and a copy of the indices (idx_copy).
__global__ void __launch_bounds__(512) per_update_kernel(PerTree Tr, int rep0, const int* __restrict__ idx, long long rs_idx, int n,
                                                         const float* __restrict__ y, const float* __restrict__ q, long long rsY,
                                                         const float* __restrict__ prio_in, float* __restrict__ p_out,
                                                         int* __restrict__ idx_copy, long long rs_out) {
  KStamp ks_;
  constexpr int kHash = 2 * kPerMaxB, kMaxPer = kPerMaxB / 256;
  __shared__ int keys[kHash];
  __shared__ int owner[kHash];
  __shared__ unsigned smax[64];
  const int rep = rep0 + blockIdx.x;
  for (int e = threadIdx.x; e < kHash; e += blockDim.x) { keys[e] = -1; owner[e] = -1; }
  if (threadIdx.x < 64) smax[threadIdx.x] = 0u;
  __syncthreads();
  const int* ix = idx + (long long)blockIdx.x * rs_idx;
  int key[kMaxPer], pos[kMaxPer];
  float pv[kMaxPer];
#pragma unroll
  for (int k = 0; k < kMaxPer; ++k) {
    const int i = threadIdx.x + k * blockDim.x;
    key[k] = -1; pos[k] = -1; pv[k] = 0.f;
    if (i >= n) continue;
    key[k] = ix[i];
    double prio;
    if (prio_in) {
      prio = (double)prio_in[i];
    } else {
      const float yv = (y + (long long)rep * rsY)[i];
      const float* Q = q + (long long)rep * 2 * rsY;
      prio = td_priority(yv, Q[i], Q[n + i]);
    }
    pv[k] = per_leaf_value(Tr, prio);
    unsigned hsh = ((unsigned)key[k] * 2654435761u) % (unsigned)kHash;
    for (int probe = 0; probe < kHash; ++probe) {       // n <= kHash / 2: a free or matching entry always exists
      const int prev = atomicCAS(&keys[hsh], -1, key[k]);
      if (prev == -1 || prev == key[k]) break;
      hsh = (hsh + 1) % (unsigned)kHash;
    }
    pos[k] = (int)hsh;
    atomicMax(&owner[hsh], i);
    atomicMax(&smax[key[k] / Tr.cap], __float_as_uint(pv[k]));     // p >= 0: its bits order like the value
    if (p_out) (p_out + (long long)blockIdx.x * rs_out)[i] = pv[k];
    if (idx_copy) (idx_copy + (long long)blockIdx.x * rs_out)[i] = key[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kMaxPer; ++k) {
    const int i = threadIdx.x + k * blockDim.x;
    if (key[k] >= 0 && owner[pos[k]] == i) per_tree_of(Tr, rep, key[k] / Tr.cap)[Tr.P + key[k] % Tr.cap] = pv[k];
  }
  if (threadIdx.x < Tr.T) {
    float* m = Tr.maxp + (long long)rep * Tr.T + threadIdx.x;
    *m = fmaxf(*m, __uint_as_float(smax[threadIdx.x]));
  }
  // ancestors: level by level, each slot recomputes its ancestor from that node's children (slots sharing an ancestor
  // write the same value)
  for (int lv = 1; lv <= Tr.levels; ++lv) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kMaxPer; ++k) {
      if (key[k] < 0) continue;
      float* tree = per_tree_of(Tr, rep, key[k] / Tr.cap);
      const long long node = (Tr.P + key[k] % Tr.cap) >> lv;
      tree[node] = tree[2 * node] + tree[2 * node + 1];
    }
  }
}

// One CTA per (task t0 + blockIdx.x, replica rep0 + blockIdx.y): leaves [lo, hi) of the task's tree become max p (below
// `lim`) or 0 (empty slots, at and above `lim`), then every ancestor of the range is rebuilt.  Pushes use lim = hi;
// fill_synthetic rewrites the whole tree.
__global__ void __launch_bounds__(1024) per_fill_kernel(PerTree Tr, int t0, int rep0, long long lo, long long hi, long long lim) {
  const int t = t0 + blockIdx.x, rep = rep0 + blockIdx.y;
  float* tree = per_tree_of(Tr, rep, t);
  const float mp = Tr.maxp[(long long)rep * Tr.T + t];
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) tree[Tr.P + i] = i < lim ? mp : 0.f;
  long long a = Tr.P + lo, b = Tr.P + hi - 1;
  for (int lv = 1; lv <= Tr.levels; ++lv) {
    __syncthreads();
    a >>= 1; b >>= 1;
    for (long long node = a + threadIdx.x; node <= b; node += blockDim.x) tree[node] = tree[2 * node] + tree[2 * node + 1];
  }
}

// Leaves (idx >= 0) or task roots (idx = -1 - t) of one replica's trees.
__global__ void per_read_kernel(PerTree Tr, int rep, const long long* __restrict__ idx, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long k = idx[i];
  out[i] = k >= 0 ? per_tree_of(Tr, rep, (int)(k / Tr.cap))[Tr.P + k % Tr.cap] : per_tree_of(Tr, rep, (int)(-1 - k))[1];
}

// rows[idx[i]] -> out[i] (b200sac_replay_sample_prioritized), one CTA per row
__global__ void per_gather_kernel(const float* __restrict__ rows, int row_stride, const int* __restrict__ idx, float* __restrict__ out) {
  const float* src = rows + (long long)idx[blockIdx.x] * row_stride;
  for (int j = threadIdx.x; j < row_stride; j += blockDim.x) out[(long long)blockIdx.x * row_stride + j] = src[j];
}

}  // namespace bsac
