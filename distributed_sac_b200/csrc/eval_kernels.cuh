// Critic evaluation outside the step (include/b200sac.h: b200sac_critic_values, b200sac_replay_refresh_priorities).
// The forwards themselves run on the engines b200sac_act uses (gemm_simt_kernel, policy_head_kernel, ln_fwd_kernel<false>);
// this file holds what the priority refresh adds around them, over one chunk of ring slots of one replica:
//   refresh_gather_kernel     one warp per slot: the row the step would train on (the n-step fold on a linked ring) into
//                             the critic inputs (s | a) and (s' | .), R, d, g and the task, plus the slot-keyed policy noise
//   refresh_td_kernel         one thread per slot: y = td_target(...) with critic_heads_kernel's operands, the priority and
//                             leaf of per_update_kernel, the leaf written and its task's maximum raised
//   per_rebuild_level_kernel  one level of a task's sum-tree recomputed from its children (launched level by level)
//   refresh_maxp_kernel       the running max p of the touched tasks
#pragma once
#include "per_kernels.cuh"
#include "nstep_kernels.cuh"

namespace bsac {

// Key multiplier of the refresh's policy noise: key = seed ^ (kRefreshKeyMul * (replica + 1)).  No other draw uses it.
constexpr unsigned long long kRefreshKeyMul = 0xC2B2AE3D27D4EB4Full;
constexpr unsigned kRefreshNoiseTag = 0x7E00u;   // counter word 3 of action k: kRefreshNoiseTag + k

struct RefreshGather {
  const float* rows;            // the replica's ring rows [cap][row_stride]
  const int* link;              // the replica's links [cap]; null: an unlinked ring
  const int* nstep;             // [R] horizons (linked ring)
  const HParams* hp;            // [R]
  const long long* idx;         // [n] ring slots
  float* XQ;                    // [n][ldx]: s | a
  float* XT;                    // [n][ldx]: s' (the policy head writes a' behind it)
  float *R, *d, *g, *eps;       // [n], [n], [n], [n][act]
  int* task;                    // [n]
  unsigned long long key;       // Philox key of the noise
  int row_stride, obs, act, ldx, cap_per_task, rep, n, stochastic;
};

__global__ void __launch_bounds__(256) refresh_gather_kernel(RefreshGather G) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (i >= G.n) return;
  const long long k = G.idx[i];
  const int off_r = G.obs + G.act, off_d = 2 * G.obs + G.act + 1;
  const float gamma = G.hp[G.rep].gamma;
  const float* row = G.rows + k * G.row_stride;
  NstepFold f;
  if (G.link) {
    f = nstep_fold(G.rows, G.row_stride, off_r, off_d, G.link, G.cap_per_task, k, G.nstep[G.rep], gamma);
  } else {
    f.R = row[off_r]; f.d = row[off_d]; f.disc = gamma; f.m = 1; f.last = k;
  }
  const float* last = G.rows + f.last * G.row_stride;
  float* xq = G.XQ + (long long)i * G.ldx;
  float* xt = G.XT + (long long)i * G.ldx;
  for (int j = lane; j < off_r; j += 32) xq[j] = row[j];
  for (int j = lane; j < G.obs; j += 32) xt[j] = last[off_r + 1 + j];
  const int t = (int)(k / G.cap_per_task);
  if (lane < G.act) {
    float e = 0.f;
    if (G.stochastic) {          // keyed by the slot, never by its place in the call
      const Philox ph(G.key);
      uint32_t rnd[4];
      ph((uint32_t)k, (uint32_t)((unsigned long long)k >> 32), (uint32_t)t, kRefreshNoiseTag + (uint32_t)lane, rnd);
      float z1;
      box_muller(rnd[0], rnd[1], e, z1);
    }
    G.eps[(long long)i * G.act + lane] = e;
  }
  if (lane == 0) { G.R[i] = f.R; G.d[i] = f.d; G.g[i] = f.disc; G.task[i] = t; }
}

struct RefreshTd {
  PerTree Tr;
  const long long* idx;         // [n] ring slots
  const float *R, *d, *g;       // [n]
  const int* task;              // [n]
  const float* logp;            // [n] log pi(a' | s')
  const float* q;               // [2][n] q1, q2 on (s, a)
  const float* qt;              // [2][n] q1_target, q2_target on (s', a')
  const float* log_alpha;       // the replica's log_alpha [T]
  const HParams* hp;            // [R]
  unsigned* tmax;               // [T] largest leaf written per task (fp32 bits; leaves are >= 0)
  int rep, n;
};

__global__ void __launch_bounds__(256) refresh_td_kernel(RefreshTd P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const int t = P.task[i];
  const float t1 = P.hp[P.rep].reward_scale * P.R[i];
  const float t2 = P.g[i] * (1.f - P.d[i]);
  const float alpha = (float)exp((double)P.log_alpha[t]);
  const float y = td_target(t1, t2, P.qt[i], P.qt[P.n + i], alpha, P.logp[i]);
  const float pv = per_leaf_value(P.Tr, td_priority(y, P.q[i], P.q[P.n + i]));
  per_tree_of(P.Tr, P.rep, t)[P.Tr.P + P.idx[i] % P.Tr.cap] = pv;     // a duplicated slot writes the same value
  atomicMax(&P.tmax[t], __float_as_uint(pv));
}

// grid (x, tasks): nodes [P >> lv, 2P >> lv) of task tasks[blockIdx.y]'s tree of replica rep
__global__ void __launch_bounds__(256) per_rebuild_level_kernel(PerTree Tr, int rep, const int* __restrict__ tasks, int lv) {
  float* tree = per_tree_of(Tr, rep, tasks[blockIdx.y]);
  const long long lo = Tr.P >> lv, hi = 2 * lo;
  for (long long node = lo + (long long)blockIdx.x * blockDim.x + threadIdx.x; node < hi; node += (long long)gridDim.x * blockDim.x)
    tree[node] = tree[2 * node] + tree[2 * node + 1];
}

// max p of the nt touched tasks: their largest refreshed leaf (full = 1) or the larger of that and the old value
__global__ void refresh_maxp_kernel(PerTree Tr, int rep, const int* __restrict__ tasks, int nt, const unsigned* __restrict__ tmax,
                                    int full) {
  for (int i = threadIdx.x; i < nt; i += blockDim.x) {
    const int t = tasks[i];
    float* m = Tr.maxp + (long long)rep * Tr.T + t;
    const float v = __uint_as_float(tmax[t]);
    *m = full ? v : fmaxf(*m, v);
  }
}

}  // namespace bsac
