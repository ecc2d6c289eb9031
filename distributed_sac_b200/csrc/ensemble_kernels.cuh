// Critic ensembles (b200sac_cfg.critic_ensemble = E; REDQ, Chen et al. 2021; RLPD, Ball et al. 2023): the per-layer step's
// head, narrow-backward and LayerNorm launches over E critics instead of two.  Each kernel here is the twin kernel of the
// same role with the networks addressed as net k = net 0 + k * rsNet (the critics of one ensemble share one layout and sit
// back to back), the [2] buffers widened to [E], and the twin's arithmetic in the twin's order, so that E = 2 with the
// full subset and the min reduction computes what the twin kernels compute, bit for bit.
#pragma once
#include "sac_kernels.cuh"
#include "ln_kernels.cuh"

namespace bsac {

constexpr int kMaxEns = 10;
constexpr unsigned long long kEnsKeyMul = 0x8EBC6AF09C88C6E3ull;

// The step's target subset of replica rep as a bit set (bit k: critic k is in S): all E when m >= E; otherwise the m
// indices with the smallest (w_k, k), w_{4q..4q+3} = Philox(key = seed ^ (kEnsKeyMul * (rep + 1)), counter (step low,
// step high, 0, q)).
B200_D unsigned ens_subset(unsigned long long seed, int rep, long long step, int E, int m) {
  if (m >= E) return (1u << E) - 1u;
  const Philox ph(seed ^ (kEnsKeyMul * (unsigned long long)(rep + 1)));
  uint32_t w0[4], w1[4], w2[4];
  ph((uint32_t)step, (uint32_t)(step >> 32), 0u, 0u, w0);
  ph((uint32_t)step, (uint32_t)(step >> 32), 0u, 1u, w1);
  ph((uint32_t)step, (uint32_t)(step >> 32), 0u, 2u, w2);
  const uint32_t w[12] = {w0[0], w0[1], w0[2], w0[3], w1[0], w1[1], w1[2], w1[3], w2[0], w2[1], w2[2], w2[3]};
  unsigned s = 0;
#pragma unroll
  for (int k = 0; k < kMaxEns; ++k) {
    int rank = 0;
#pragma unroll
    for (int j = 0; j < kMaxEns; ++j)
      if (j < E && (w[j] < w[k] || (w[j] == w[k] && j < k))) ++rank;
    if (k < E && rank < m) s |= 1u << k;
  }
  return s;
}

// ------------------------------------------------------------------------------------------
// Critic heads of the critic update (critic_heads_kernel for E critics): Qt_k and Q_k, the TD target with the subset
// min, every dL/dQ_k and the row's squared errors; replica rep's subset to tsub from row 0.
// ------------------------------------------------------------------------------------------
struct CriticHeadEnsArgs {
  const float* hT; const float* hQ; long long rsHnet, rsHrep; int ldh;   // [E][B][Hc] per replica
  const float* Wt; const float* bt; const float* Wq; const float* bq;   // critic 0's heads; critic k at + k * rsNet
  long long rsNet, rsP;
  const float* r; const float* d; const int* tid; long long rsR;
  const float* logp; long long rsLogp;
  const float* log_alpha;
  float* y; float* q; float* dq; float* lq; long long rsY;   // y[B], q[E][B], dq[E][B] (replica stride E * rsY), lq[B]
  const int* ens;                                            // [R][2] (m, actor_mean)
  float* tsub; long long rsTsub;                             // [E] per replica
  int E;
};

__global__ void __launch_bounds__(256) critic_heads_ens_kernel(StepConst K, CriticHeadEnsArgs P) {
  KStamp ks_;
  const int rep = blockIdx.y;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int row = blockIdx.x * (blockDim.x / 32) + warp;
  const int B = K.B, H = K.Hc, E = P.E;
  if (row >= B) return;
  const float* hT = P.hT + rep * P.rsHrep + (long long)row * P.ldh;
  const float* hQ = P.hQ + rep * P.rsHrep + (long long)row * P.ldh;
  const long long po = rep * P.rsP;
  const int t = (P.tid + rep * P.rsR)[row];
  const float r = (P.r + rep * P.rsR)[row], d = (P.d + rep * P.rsR)[row];
  const float t1 = K.hp[rep].reward_scale * r;
  const float t2 = (K.disc ? K.disc[(long long)rep * B + row] : K.hp[rep].gamma) * (1.f - d);
  const float lp = (P.logp + rep * P.rsLogp)[row];
  const float la_t = (P.log_alpha + po)[t];
  const unsigned S = ens_subset(K.seed, rep, K.cnt[rep].v[3], E, P.ens[2 * rep]);
  float qv[kMaxEns], qt_min = 0.f;
  bool first = true;
#pragma unroll
  for (int k = 0; k < kMaxEns; ++k) {
    qv[k] = 0.f;
    if (k < E) {
      const long long pk = po + k * P.rsNet;
      const float b_t = (P.bt + pk)[0], b_q = (P.bq + pk)[0];
      const float p_t = warp_dot_partial(hT + k * P.rsHnet, P.Wt + pk, H, lane);
      const float p_q = warp_dot_partial(hQ + k * P.rsHnet, P.Wq + pk, H, lane);
      const float qt = warp_sum(p_t) + b_t;
      qv[k] = warp_sum(p_q) + b_q;
      if ((S >> k) & 1u) { qt_min = first ? qt : fminf(qt_min, qt); first = false; }
    }
  }
  if (lane == 0) {
    const float alpha = (float)exp((double)la_t);
    const float y = t1 + t2 * (qt_min - alpha * lp);
    (P.y + rep * P.rsY)[row] = y;
    float* Q = P.q + rep * E * P.rsY;
    float* DQ = P.dq + rep * E * P.rsY;
    const float w = K.isw ? K.isw[(long long)rep * B + row] : 1.f;
    float l = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxEns; ++k)
      if (k < E) {
        const float e = y - qv[k];
        l = k == 0 ? e * e : l + e * e;
        float g = 2.f * K.c_loss * (qv[k] - y);
        if (K.isw) g = g * w;
        Q[k * B + row] = qv[k];
        DQ[k * B + row] = g;
        if (row == 0) (P.tsub + rep * P.rsTsub)[k] = ((S >> k) & 1u) ? 1.f : 0.f;
      }
    if (K.isw) l = l * w;
    (P.lq + rep * P.rsY)[row] = l;
  }
}

// ------------------------------------------------------------------------------------------
// Actor-pass heads (actor_q_heads_kernel for E critics): Q_k at (s, a~) with the updated critics, the replica's mean or
// min reduction and its gradient routing, the per-row policy-loss term.
// ------------------------------------------------------------------------------------------
struct ActorQHeadEnsArgs {
  const float* hP; long long rsHnet, rsHrep; int ldh;
  const float* Wq; const float* bq; long long rsNet, rsP;
  const int* tid; long long rsR;
  const float* logp; long long rsLogp;    // +B offset applied by the host: current-state half
  const float* log_alpha;
  float* dqa; float* qp; float* la; float* qmin; long long rsY;   // dqa[E][B], qp[E][B] (replica stride E * rsY), la[B], qmin[B]
  const int* ens;                          // [R][2] (m, actor_mean)
  int E;
};

__global__ void __launch_bounds__(256) actor_q_heads_ens_kernel(StepConst K, ActorQHeadEnsArgs P) {
  const int rep = blockIdx.y;
  const int sched = sched_of(K.cnt, rep);
  KStamp ks_;
  if (!(sched & SCHED_ACTOR)) return;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int row = blockIdx.x * (blockDim.x / 32) + warp;
  const int B = K.B, H = K.Hc, E = P.E;
  if (row >= B) return;
  const float* hP = P.hP + rep * P.rsHrep + (long long)row * P.ldh;
  const long long po = rep * P.rsP;
  const int t = (P.tid + rep * P.rsR)[row];
  const float lp = (P.logp + rep * P.rsLogp)[row];
  const float la_t = (P.log_alpha + po)[t];
  const bool mean = P.ens[2 * rep + 1] != 0;
  float qv[kMaxEns], red = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxEns; ++k) {
    qv[k] = 0.f;
    if (k < E) {
      const long long pk = po + k * P.rsNet;
      const float b_q = (P.bq + pk)[0];
      qv[k] = warp_sum(warp_dot_partial(hP + k * P.rsHnet, P.Wq + pk, H, lane)) + b_q;
      red = k == 0 ? qv[k] : (mean ? red + qv[k] : fminf(red, qv[k]));
    }
  }
  if (lane == 0) {
    const float alpha = (float)exp((double)la_t);
    float g_all = 0.f;
    int ties = 0;
    if (mean) {
      red = red / (float)E;
      g_all = -K.c_loss / (float)E;
    } else {
#pragma unroll
      for (int k = 0; k < kMaxEns; ++k)
        if (k < E && qv[k] == red) ++ties;
      g_all = ties > 0 ? -K.c_loss / (float)ties : 0.f;
    }
    float* DQ = P.dqa + rep * E * P.rsY;
    float* QP = P.qp + rep * E * P.rsY;
#pragma unroll
    for (int k = 0; k < kMaxEns; ++k)
      if (k < E) {
        DQ[k * B + row] = (mean || qv[k] == red) ? g_all : 0.f;
        QP[k * B + row] = qv[k];
      }
    (P.la + rep * P.rsY)[row] = -(red - alpha * lp);
    (P.qmin + rep * P.rsY)[row] = red;
  }
}

// ------------------------------------------------------------------------------------------
// Narrow backward over E critics: head_bwd_kernel (critic heads; and the policy head, whose action gradient sums the E
// critics' input gradients in index order) and head_bwd4_kernel<1> (critic heads, 128-bit columns), with critic
// net = blockIdx.y at + net * rsNet in the parameter and gradient arenas.
// ------------------------------------------------------------------------------------------
struct HeadBwdEnsArgs {
  HeadBwdArgs a;       // W[0], dW[0], db[0], dWx[0], dbx[0]: critic 0's (the policy head's in policy mode)
  long long rsNet;
  int E;
};

// d(action) of row m, action j: the E critics' input gradients added in index order
B200_D float ens_dact(const HeadBwdArgs& P, int rep, int m, int j, int in_w, int E) {
  const float* __restrict__ dx0 = P.dx + rep * P.rsDxRep + (long long)m * P.lddx + in_w + j;
  float da = dx0[0];
  for (int k = 1; k < E; ++k) da = da + dx0[k * P.rsDxNet];
  return da;
}

// (256, 1): without the occupancy target ptxas keeps this kernel at 64 registers and spills
__global__ void __launch_bounds__(256, 1) head_bwd_ens_kernel(StepConst K, HeadBwdEnsArgs PE) {
  const HeadBwdArgs& P = PE.a;
  const int net = blockIdx.y, rep = blockIdx.z;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  extern __shared__ float sm[];
  if (skip) return;
  const int NO = P.NO, KD = P.Kdim;
  const int ncb = (KD + kHbCols - 1) / kHbCols;
  const int slice = blockIdx.x / ncb, cb = blockIdx.x - slice * ncb;
  const int rows_per = (P.M + P.row_slices - 1) / P.row_slices;
  const int r0 = slice * rows_per, r1 = (r0 + rows_per < P.M) ? r0 + rows_per : P.M;
  const int M = r1 - r0;
  if (M <= 0) return;
  float* sd = sm;                       // [M][NO]
  float* red = sm + (size_t)rows_per * NO;
  const int tid = threadIdx.x, tx = tid % kHbCols, ty = tid / kHbCols;
  const long long no = net * PE.rsNet;

  if (P.policy_mode) {
    const int A = K.act;
    __shared__ float s_alpha[64];
    const int Teff = K.T > 0 ? K.T : 1;
    if (tid < Teff) s_alpha[tid] = (float)exp((double)(P.log_alpha + rep * P.rsP)[tid]);
    __syncthreads();
    for (int e = tid; e < M * A; e += 256) {
      const int ml = e / A, j = e % A, m = r0 + ml;
      const float* __restrict__ sv = P.psave + rep * P.rsSave + ((long long)m * A + j) * kSaveW;
      const float da = ens_dact(P, rep, m, j, K.in_w, PE.E);
      const int tk = (P.tid + rep * P.rsR)[m];
      float dmu, dls;
      policy_dout_point(K, sv, da, s_alpha[tk], dmu, dls);
      sd[ml * NO + j] = dmu;
      sd[ml * NO + A + j] = dls;
      if (P.dout_dbg && cb == 0) {
        (P.dout_dbg + rep * P.rsDbg)[(long long)m * NO + j] = dmu;
        (P.dout_dbg + rep * P.rsDbg)[(long long)m * NO + A + j] = dls;
        (P.dact_dbg + rep * P.rsDbg)[(long long)m * A + j] = da;
      }
    }
  } else {
    const float* __restrict__ src = P.dout + rep * P.rsDoutRep + net * P.rsDoutNet + (long long)r0 * NO;
    for (int e = tid; e < M * NO; e += 256) sd[e] = src[e];
  }

  const int kcol = cb * kHbCols + tx;
  const bool kin = kcol < KD;
  const float* __restrict__ W = P.W[0] + no + rep * P.rsP;
  float w[kMaxHeadOut], gw[kMaxHeadOut];
#pragma unroll
  for (int j = 0; j < kMaxHeadOut; ++j) {
    w[j] = (j < NO && kin) ? W[(long long)j * KD + kcol] : 0.f;
    gw[j] = 0.f;
  }
  __syncthreads();
  const float* __restrict__ h = P.h + rep * P.rsHrep + net * P.rsHnet + (long long)r0 * P.ldh;
  float* __restrict__ dh = P.dh + rep * P.rsDhRep + net * P.rsDhNet + (long long)r0 * P.lddh;
  constexpr int U = 8;
  for (int mb = ty; mb < M; mb += kHbRows * U) {
    float hv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int m = mb + u * kHbRows;
      hv[u] = (kin && m < M) ? h[(long long)m * P.ldh + kcol] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int m = mb + u * kHbRows;
      if (m < M) {
        float ds = 0.f;
#pragma unroll
        for (int j = 0; j < kMaxHeadOut; ++j) {
          if (j < NO) {
            const float dv = sd[m * NO + j];
            ds = fmaf(dv, w[j], ds);
            gw[j] = fmaf(dv, hv[u], gw[j]);
          }
        }
        if (kin) dh[(long long)m * P.lddh + kcol] = hv[u] > 0.f ? ds : 0.f;
      }
    }
  }
  if (P.dW[0] != nullptr) {
    float* __restrict__ dWp = (slice == 0 ? P.dW[0] : P.dWx[0] + (long long)(slice - 1) * P.xs) + no + rep * P.rsG;
    float* __restrict__ dbp = (slice == 0 ? P.db[0] : P.dbx[0] + (long long)(slice - 1) * P.xs) + no + rep * P.rsG;
#pragma unroll
    for (int j = 0; j < kMaxHeadOut; ++j)
      if (j < NO) red[(ty * kHbCols + tx) * NO + j] = gw[j];
    __syncthreads();
    if (ty < NO && kin) {
      float ssum = 0.f;
      for (int q = 0; q < kHbRows; ++q) ssum += red[(q * kHbCols + tx) * NO + ty];
      dWp[(long long)ty * KD + kcol] = ssum;
    }
    if (cb == 0) {
      __syncthreads();
      float part[kMaxHeadOut];
#pragma unroll
      for (int j = 0; j < kMaxHeadOut; ++j) part[j] = 0.f;
      for (int m = tid; m < M; m += 256) {
#pragma unroll
        for (int j = 0; j < kMaxHeadOut; ++j)
          if (j < NO) part[j] += sd[m * NO + j];
      }
#pragma unroll
      for (int j = 0; j < kMaxHeadOut; ++j)
        if (j < NO) {
          const float v = warp_sum(part[j]);
          if ((tid & 31) == 0) red[(tid >> 5) * kMaxHeadOut + j] = v;
        }
      __syncthreads();
      if (tid < NO) {
        float ssum = 0.f;
#pragma unroll
        for (int wq = 0; wq < 8; ++wq) ssum += red[wq * kMaxHeadOut + tid];
        dbp[tid] = ssum;
      }
    }
  }
}

// the scalar critic heads' backward with 128-bit column accesses (head_bwd4_kernel<1> for E critics)
__global__ void __launch_bounds__(256, 1) head_bwd4_ens_kernel(StepConst K, HeadBwdEnsArgs PE) {
  const HeadBwdArgs& P = PE.a;
  const int net = blockIdx.y, rep = blockIdx.z;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  extern __shared__ float sm[];
  if (skip) return;
  const int KD = P.Kdim;
  const int ncb = (KD + kHb4Cols - 1) / kHb4Cols;
  const int slice = blockIdx.x / ncb, cb = blockIdx.x - slice * ncb;
  const int rows_per = (P.M + P.row_slices - 1) / P.row_slices;
  const int r0 = slice * rows_per, r1 = (r0 + rows_per < P.M) ? r0 + rows_per : P.M;
  const int M = r1 - r0;
  if (M <= 0) return;
  float* sd = sm;                                   // [M]
  float* red = sm + (((size_t)rows_per + 3) & ~(size_t)3);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long no = net * PE.rsNet;
  {
    const float* __restrict__ src = P.dout + rep * P.rsDoutRep + net * P.rsDoutNet + (long long)r0;
    for (int e = tid; e < M; e += 256) sd[e] = src[e];
  }
  const int kcol = cb * kHb4Cols + 4 * tx;
  const bool kin = kcol < KD;
  const float* __restrict__ W = P.W[0] + no + rep * P.rsP;
  const float4 w = kin ? *reinterpret_cast<const float4*>(W + kcol) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 gw = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  const float* __restrict__ h = P.h + rep * P.rsHrep + net * P.rsHnet + (long long)r0 * P.ldh;
  float* __restrict__ dh = P.dh + rep * P.rsDhRep + net * P.rsDhNet + (long long)r0 * P.lddh;
  constexpr int U = 8;
  for (int mb = ty; mb < M; mb += kHb4Rows * U) {
    float4 hv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int m = mb + u * kHb4Rows;
      hv[u] = (kin && m < M) ? *reinterpret_cast<const float4*>(h + (long long)m * P.ldh + kcol) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int m = mb + u * kHb4Rows;
      if (m < M) {
        float4 ds = make_float4(0.f, 0.f, 0.f, 0.f);
        const float dv = sd[m];
        ds.x = fmaf(dv, w.x, ds.x); ds.y = fmaf(dv, w.y, ds.y); ds.z = fmaf(dv, w.z, ds.z); ds.w = fmaf(dv, w.w, ds.w);
        gw.x = fmaf(dv, hv[u].x, gw.x); gw.y = fmaf(dv, hv[u].y, gw.y);
        gw.z = fmaf(dv, hv[u].z, gw.z); gw.w = fmaf(dv, hv[u].w, gw.w);
        if (kin)
          *reinterpret_cast<float4*>(dh + (long long)m * P.lddh + kcol) =
              make_float4(hv[u].x > 0.f ? ds.x : 0.f, hv[u].y > 0.f ? ds.y : 0.f, hv[u].z > 0.f ? ds.z : 0.f, hv[u].w > 0.f ? ds.w : 0.f);
      }
    }
  }
  if (P.dW[0] != nullptr) {
    float* __restrict__ dWp = (slice == 0 ? P.dW[0] : P.dWx[0] + (long long)(slice - 1) * P.xs) + no + rep * P.rsG;
    float* __restrict__ dbp = (slice == 0 ? P.db[0] : P.dbx[0] + (long long)(slice - 1) * P.xs) + no + rep * P.rsG;
    *reinterpret_cast<float4*>(red + (size_t)(ty * 16 + tx) * 4) = gw;
    __syncthreads();
    for (int cc = tid; cc < kHb4Cols; cc += 256) {
      const int col = cb * kHb4Cols + cc;
      if (col < KD) {
        float ssum = 0.f;
#pragma unroll
        for (int q = 0; q < kHb4Rows; ++q) ssum += red[(size_t)(q * 16 + (cc >> 2)) * 4 + (cc & 3)];
        dWp[col] = ssum;
      }
    }
    if (cb == 0) {
      __syncthreads();
      float part = 0.f;
      for (int m = tid; m < M; m += 256) part += sd[m];
      const float v = warp_sum(part);
      if ((tid & 31) == 0) red[(tid >> 5) * kMaxHeadOut] = v;
      __syncthreads();
      if (tid == 0) {
        float ssum = 0.f;
#pragma unroll
        for (int wq = 0; wq < 8; ++wq) ssum += red[wq * kMaxHeadOut];
        dbp[0] = ssum;
      }
    }
  }
}

// Large batches: the policy-head output gradient once per (row, action), from the E critics' summed action gradients
struct PolicyDoutEnsArgs {
  PolicyDoutArgs a;
  int E;
};

__global__ void __launch_bounds__(256) policy_dout_ens_kernel(StepConst K, PolicyDoutEnsArgs PE) {
  const PolicyDoutArgs& P = PE.a;
  const int rep = blockIdx.y, A = K.act;
  const int sched = sched_of(K.cnt, rep);
  KStamp ks_;
  if (!(sched & SCHED_ACTOR)) return;
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= P.M * A) return;
  const int m = e / A, j = e % A;
  const float* __restrict__ sv = P.psave + rep * P.rsSave + ((long long)m * A + j) * kSaveW;
  const float* __restrict__ dx0 = P.dx + rep * P.rsDxRep + (long long)m * P.lddx + K.in_w + j;
  float da = dx0[0];
  for (int k = 1; k < PE.E; ++k) da = da + dx0[k * P.rsDxNet];
  const float alpha = (float)exp((double)(P.log_alpha + rep * P.rsP)[(P.tid + rep * P.rsR)[m]]);
  float dmu, dls;
  policy_dout_point(K, sv, da, alpha, dmu, dls);
  float* o = P.dout + rep * P.rsDout + (long long)m * 2 * A;
  o[j] = dmu;
  o[A + j] = dls;
  (P.dact + rep * P.rsDout)[(long long)m * A + j] = da;
}

// ------------------------------------------------------------------------------------------
// LayerNorm (and dropout) over E critics: ln_fwd_kernel / ln_bwd_kernel with rows [E][B], critic k's g, c (and their
// gradient slots) at + k * rsNet, the backward's chunk sums [R][E][chunks][2][H] and tickets [R][E], and critic k's mask
// tag tag0 + k with tag0 = (pass * 8 + layer) * E.
// ------------------------------------------------------------------------------------------
struct LnEnsArgs {
  LnArgs a;            // g[0], c[0], dg[0], dc[0]: critic 0's
  long long rsNet;
  int E;
};

template <bool kDrop>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_ens_kernel(StepConst K, LnEnsArgs PE) {
  const LnArgs& P = PE.a;
  const int rep = blockIdx.y;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  if (skip) return;
  const int lane = threadIdx.x & 31, row = blockIdx.x * (kLnThreads / kWarp) + (threadIdx.x >> 5);
  if (row >= PE.E * P.B) return;
  const int net = row / P.B, H = P.H;
  const float* z = P.z + rep * P.rsZ + (long long)row * H;
  float* h = P.h + rep * P.rsH + (long long)row * H;
  const float* g = P.g[0] + net * PE.rsNet + rep * P.rsP;
  const float* c = P.c[0] + net * PE.rsNet + rep * P.rsP;
  if constexpr (kDrop) {
    const int words = (H + 31) / 32;
    const Philox ph(K.seed ^ (kDropKeyMul * (unsigned long long)(rep + 1)));
    drop_row(const_cast<float*>(z), P.mbits + rep * P.rsM + (long long)row * words, H, lane, ph, K.cnt[rep].v[3],
             row - net * P.B, (unsigned)(P.tag0 + net), P.drop[rep]);
  }
  double mu, rstd;
  ln_row_stats(z, H, lane, mu, rstd);
  for (int j = lane; j < H; j += kWarp) {
    const double y = (double)g[j] * (((double)z[j] - mu) * rstd) + (double)c[j];
    h[j] = y < 0.0 ? 0.f : (float)y;
  }
}

template <bool kDrop>
__global__ void __launch_bounds__(kLnThreads) ln_bwd_ens_kernel(StepConst K, LnEnsArgs PE) {
  const LnArgs& P = PE.a;
  const int rep = blockIdx.z, net = blockIdx.y, E = PE.E;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  __shared__ double st[kLnRows][4];
  __shared__ bool s_last;
  if (skip) return;
  const int H = P.H, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * kLnRows, nr = min(kLnRows, P.B - r0);
  const long long base = ((long long)net * P.B + r0) * H;
  const float* z = P.z + rep * P.rsZ + base;
  float* dh = P.dh + rep * P.rsH + base;
  const float* g = P.g[0] + net * PE.rsNet + rep * P.rsP;
  for (int r = warp; r < nr; r += kLnThreads / kWarp) {
    const float* zr = z + (long long)r * H;
    const float* dr = dh + (long long)r * H;
    double mu, rstd;
    ln_row_stats(zr, H, lane, mu, rstd);
    double sa = 0.0, sb = 0.0;
    for (int j = lane; j < H; j += kWarp) {
      const double gd = (double)g[j] * (double)dr[j];
      sa += gd;
      sb += gd * (((double)zr[j] - mu) * rstd);
    }
    sa = warp_sum_d(sa);
    sb = warp_sum_d(sb);
    if (lane == 0) { st[r][0] = mu; st[r][1] = rstd; st[r][2] = sa / (double)H; st[r][3] = sb / (double)H; }
  }
  __syncthreads();
  const bool wg = P.dg[0] != nullptr;
  const int chunks = gridDim.x;
  double* part = wg ? P.part + (((long long)rep * E + net) * chunks) * 2 * H : nullptr;
  const int words = (H + 31) / 32;
  const unsigned* mb = kDrop ? P.mbits + rep * P.rsM + ((long long)net * P.B + r0) * words : nullptr;
  const float ds = kDrop ? P.drop[rep].s : 0.f;
  for (int j = threadIdx.x; j < H; j += kLnThreads) {
    const double gj = (double)g[j];
    double sg = 0.0, sc = 0.0;
    for (int r = 0; r < nr; ++r) {
      const long long e = (long long)r * H + j;
      const double dy = (double)dh[e];
      const double xh = ((double)z[e] - st[r][0]) * st[r][1];
      sg += dy * xh;
      sc += dy;
      const float dz = (float)(st[r][1] * ((gj * dy - st[r][2]) - xh * st[r][3]));
      if constexpr (kDrop) {
        const unsigned m = mb[(long long)r * words + (j >> 5)] >> (j & 31);
        dh[e] = dz * ((m & 1u) ? ds : 0.f);
      } else {
        dh[e] = dz;
      }
    }
    if (wg) {
      part[((long long)blockIdx.x * 2 + 0) * H + j] = sg;
      part[((long long)blockIdx.x * 2 + 1) * H + j] = sc;
    }
  }
  if (!wg) return;
  __threadfence();
  __syncthreads();
  unsigned* ticket = P.ticket + rep * E + net;
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == (unsigned)(chunks - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  float* dg = P.dg[0] + net * PE.rsNet + rep * P.rsG;
  float* dc = P.dc[0] + net * PE.rsNet + rep * P.rsG;
  for (int j = threadIdx.x; j < H; j += kLnThreads) {
    double sg = 0.0, sc = 0.0;
    for (int k = 0; k < chunks; ++k) {
      sg += __ldcg(&part[((long long)k * 2 + 0) * H + j]);
      sc += __ldcg(&part[((long long)k * 2 + 1) * H + j]);
    }
    dg[j] = (float)sg;
    dc[j] = (float)sc;
  }
  if (threadIdx.x == 0) *ticket = 0;
}

}  // namespace bsac
