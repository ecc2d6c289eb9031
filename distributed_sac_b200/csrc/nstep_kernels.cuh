// n-step returns on the device ring, folded at sample time (the way SB3 >= 2.x and TorchRL's MultiStep do it) from the
// 1-step transitions the ring holds plus a record of which slot follows which.
//
// A linked ring keeps link[R][cap] (int32): the sub-ring-local slot of the transition that followed this one in its
// trajectory, or -1.  The host maintains it at push time (b200sac.cu, push_links) under one invariant, valid at every
// point in stream order:  link[i] = j >= 0  =>  slot j currently holds the transition that followed slot i's.
// The fold of batch row i with horizon n = nstep[rep] and gamma = HParams[rep].gamma, all fp32, no fused multiply-add:
//   j = idx[i];  R = r_j;  g = gamma;  m = 1
//   while d_j == 0 and m < n and link[j] >= 0:
//     j = link[j];  R = R + g * r_j;  g = g * gamma;  m = m + 1
//   row = (s_i, a_i, R, s'_j, d_j),  disc = g
// so the horizon is simply shorter at a terminal, a time-limit cut (no link was made), a trajectory's current tail or an
// overwritten successor, and m = 1 is the ring's own row with disc = gamma, bit for bit.  The intermediate rows' actions
// are used uncorrected (Ape-X).  TD target of the step: y = rs R + disc (1 - d)(min(Qt1, Qt2) - alpha logpi').
#pragma once
#include "sac_kernels.cuh"

namespace bsac {

constexpr int kNstepMax = 16;        // horizon n in [1, 16]
constexpr int kNstepChunk = 2048;    // rows per launch of b200sac_replay_fold

struct NstepRing {
  const int* link;             // [R][cap]
  const int* nstep;            // [R] horizon per replica
  long long cap;               // slots per replica
  int cap_per_task;
};

struct NstepFold {
  float R, disc, d;
  int m;
  long long last;              // ring index of the last hop: its s' is the row's next state
};

// Every lane of the warp walks the same chain (the loads are broadcasts), so no lane waits for a shuffle.  The next hop's
// link, r and d are requested together as soon as j is known; only the last hop's s' needs the wide read (the caller's).
B200_D NstepFold nstep_fold(const float* __restrict__ rows, int row_stride, int off_r, int off_d, const int* __restrict__ link,
                            int cap_per_task, long long j, int n, float gamma) {
  const long long base = j - j % cap_per_task;
  const float* row = rows + j * row_stride;
  int nx = link[j];
  NstepFold f;
  f.R = row[off_r]; f.d = row[off_d]; f.disc = gamma; f.m = 1;
  while (f.d == 0.f && f.m < n && nx >= 0) {
    j = base + nx;
    row = rows + j * row_stride;
    nx = link[j];
    const float rj = row[off_r];
    f.d = row[off_d];
    f.R = f.R + f.disc * rj;
    f.disc = f.disc * gamma;
    f.m += 1;
  }
  f.last = j;
  return f;
}

// The gather of a step that samples from a linked ring: ingest_rows_kernel with the fold in front of the scatter.  out:
// [3][R][B] = disc (what K.disc points at), m and the ring index (int32 bit patterns), for b200sac_debug_read.
__global__ void ingest_nstep_kernel(StepConst K, IngestOut O, const float* __restrict__ rows, long long rs_rows, int row_stride,
                                    const int* __restrict__ idx, long long rs_idx, NstepRing N, float* __restrict__ out) {
  KStamp ks_;
  const int rep = blockIdx.y;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, wpb = blockDim.x / 32;
  const int B = K.B, R = gridDim.y;
  if (blockIdx.x == 0 && threadIdx.x == 0) bump_counters(O, rep, K.beta1, K.beta2);
  if (blockIdx.x == gridDim.x - 1) snapshot_alpha(K, O, rep, threadIdx.x);
  const float* base = rows + rep * rs_rows;
  const int n = N.nstep[rep];
  const float gamma = K.hp[rep].gamma;
  for (int i = blockIdx.x * wpb + warp; i < B; i += gridDim.x * wpb) {
    const long long src = (long long)idx[rep * rs_idx + i];
    const NstepFold f = nstep_fold(base, row_stride, K.obs + K.act, 2 * K.obs + K.act + 1, N.link + rep * N.cap, N.cap_per_task,
                                   src, n, gamma);
    const float* row = base + src * row_stride;
    ingest_row(K, O, rep, i, row, row + K.obs, f.R, base + f.last * row_stride + K.obs + K.act + 1, f.d, lane, 32);
    if (lane == 0) {
      const long long o = (long long)rep * B + i;
      out[o] = f.disc;
      out[(long long)R * B + o] = __int_as_float(f.m);
      out[(long long)2 * R * B + o] = __int_as_float((int)src);
    }
  }
}

// b200sac_replay_fold: the same fold for caller-given ring indices of one replica, as packed rows [s | a | R | s' | d].
__global__ void nstep_fold_kernel(const float* __restrict__ rows, int row_stride, int obs, int act, const int* __restrict__ link,
                                  int cap_per_task, const int* __restrict__ nstep, const HParams* __restrict__ hp, int rep,
                                  const long long* __restrict__ idx, int n_idx, float* __restrict__ out_rows,
                                  float* __restrict__ out_disc, int* __restrict__ out_m) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int i = blockIdx.x * (blockDim.x / 32) + warp;
  if (i >= n_idx) return;
  const int off_r = obs + act, off_d = 2 * obs + act + 1;
  const NstepFold f = nstep_fold(rows, row_stride, off_r, off_d, link, cap_per_task, idx[i], nstep[rep], hp[rep].gamma);
  const float* row = rows + idx[i] * row_stride;
  const float* last = rows + f.last * row_stride;
  float* o = out_rows + (long long)i * row_stride;
  for (int j = lane; j < off_r; j += 32) o[j] = row[j];
  for (int j = lane; j < obs; j += 32) o[off_r + 1 + j] = last[off_r + 1 + j];
  if (lane == 0) { o[off_r] = f.R; o[off_d] = f.d; out_disc[i] = f.disc; out_m[i] = f.m; }
}

// Link changes of one push: unique (ring index, value) pairs.
__global__ void nstep_scatter_links_kernel(int* __restrict__ link, const int* __restrict__ at, const int* __restrict__ val, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) link[at[i]] = val[i];
}

// fill_synthetic on a linked ring: slot i -> i + 1 of every sub-ring unless d_i != 0 or i is the last filled slot.
__global__ void nstep_fill_links_kernel(int* __restrict__ link, long long cap, int cap_per_task, const float* __restrict__ rows,
                                        long long rs_rows, int row_stride, int off_d, long long filled) {
  const int rep = blockIdx.y;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < cap; g += (long long)gridDim.x * blockDim.x) {
    const long long i = g % cap_per_task;
    const bool next = i + 1 < filled && (rows + rep * rs_rows + g * row_stride)[off_d] == 0.f;
    link[rep * cap + g] = next ? (int)(i + 1) : -1;
  }
}

}  // namespace bsac
