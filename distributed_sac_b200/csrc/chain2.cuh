// Twin-critic forward + backward in ONE kernel (LunarLander-class plan, see chain.cuh).
//
// Two places of the SAC step evaluate a critic forward and then differentiate a critic on the same rows, with only a
// per-row scalar in between that needs BOTH twins:
//   critic update   Qt1, Qt2 (s', a')  ->  y = rs r + gamma (1-d)(min(Qt1, Qt2) - alpha logpi')  ->  dQk = 2c (Qk - y)  -> backward of Qk
//                   (LunarLander_Distributed_SAC/src/learner.py:206-216, model.py:129-142)
//   actor pass      Q1, Q2 (s, a~)     ->  min(Q1, Q2): gradient to the smaller head             -> backward of Qk down to d(action)
//                   (learner.py:221-225, model.py:84-88)
// As two launches each pair paid a kernel boundary, a cold prologue and a restart of the weight pipeline.
// Here the CTA that owns rows [row0, row0+ROWS) of twin k walks the forward chain, the two CTAs of a thread-block CLUSTER
// (twin 0, twin 1 of the same rows) swap their ROWS head values through distributed shared memory (mapa + ld.shared::cluster
// between two barrier.cluster phases), and each goes on into the backward chain of its own twin -- the TMA weight pipeline
// never drains: the first backward chunks are requested while the forward head is still being computed.
#pragma once
#include <type_traits>
#include "chain.cuh"

namespace bsac {

constexpr int C2_MAXL = 4;                 // dense stages per direction
constexpr size_t C2_SMEM_BYTES = (size_t)(CH_NSTAGE * CH_CHUNK_FLOATS + CH_SM_BARS + 2 * CH_SM_ACT + 2 * CH_INP + 2 * CH_ROWS + CH_SM_W0A + CH_SM_PART) * sizeof(float) + 1024;
enum { C2_CRITIC = 0, C2_ACTORQ = 1 };

struct Chain2Job {
  int rows, nfwd, nbwd, net;
  const float* X; long long rsX; int ldx, K0;          // forward: input rows [rows][ldx]
  ChainStage fst[C2_MAXL];                             // forward stages (hidden layers)
  const float* Whf; const float* bhf; int Hhf;         // forward scalar head [1][Hhf] + bias (arena)
  float* qf_out; long long rsQf;                       // forward head output of this twin (row 0)
  const float* hlast; long long rsHlast; int ldh;      // backward: last hidden activation of the differentiated net [rows][Hhb]
  float* dylast; long long rsDy; int lddy;             // optional store of the generated dY
  const float* Whb; int Hhb;                           // the differentiated net's scalar head weights [1][Hhb]
  ChainStage bst[C2_MAXL];                             // backward stages
  const float* W0; int ldw0, col0, nact, H0;           // C2_ACTORQ: d(action) tail
  float* dx; long long rsDx; int lddx;
};

struct Chain2Args {
  int kind, early_weights;
  long long rsP;
  long long* dbg;
  Chain2Job job[2];
  ChainRows rw;
};

B200_D void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
B200_D float ld_peer_f32(const float* my_smem_addr, uint32_t peer_rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(my_smem_addr)), "r"(peer_rank));
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra) : "memory");
  return v;
}

template <int ROWS>
__global__ void __launch_bounds__(CH_BLOCK, 1) chain2_kernel(const __grid_constant__ Chain2Args A, StepConst K) {
  long long* const dbg = (A.dbg != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0 && threadIdx.x == 0) ? A.dbg : nullptr;
  int dbg_i = 0;
#define C2_STAMP() do { if (dbg != nullptr && dbg_i < CH_DBG_SLOTS) dbg[dbg_i++] = clock64(); } while (0)
  C2_STAMP();
  extern __shared__ __align__(1024) float sm2_raw[];
  float* sm = sm2_raw + (((1024u - (smem_u32(sm2_raw) & 1023u)) & 1023u) >> 2);
  const Chain2Job& J = A.job[blockIdx.y];
  const int rep = blockIdx.z;
  const int row0 = blockIdx.x * ROWS;
  if (row0 >= J.rows) return;              // (both CTAs of the cluster share row0 and rows: they leave together)
  const int nrows = (J.rows - row0 < ROWS) ? J.rows - row0 : ROWS;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const long long po = (long long)rep * A.rsP;
  uint32_t my_rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(my_rank));

  float* wst = sm;
  uint64_t* bars = reinterpret_cast<uint64_t*>(wst + CH_NSTAGE * CH_CHUNK_FLOATS);
  float* actA = wst + CH_NSTAGE * CH_CHUNK_FLOATS + CH_SM_BARS;
  float* actB = actA + CH_SM_ACT;
  float* headF = actB + CH_SM_ACT;         // [CH_INP] forward head row
  float* headB = headF + CH_INP;           // [CH_INP] backward (differentiated net's) head row
  float* sd = headB + CH_INP;              // [ROWS] d(head output) per row
  float* xch = sd + CH_ROWS;               // [ROWS] this twin's forward head values (read by the peer CTA)
  float* w0a = xch + CH_ROWS;
  float* part = w0a + CH_SM_W0A;

  // ---- weight pipeline over the flat stage list: forward stages (2-D TMA, swizzled [n][k]) then backward ([k][n] bulk) ----
  const int nst = J.nfwd + J.nbwd;
  const bool direct0 = J.nfwd > 1 && J.fst[0].K <= CH_KC;
  int is = direct0 ? 1 : 0, ic = 0, issued = 0;
  // (who / dry: see chain_kernel -- thread 0 requests the first two chunks before griddepcontrol.wait, the producer warp the rest)
  auto issue_next = [&](int who, bool dry) {
    const bool mine = who == 0 ? tid == 0 : tid >= CH_THREADS;        // thread 0 (early requests) | the whole producer warp
    if (mine && is < nst) {
      const bool f = is < J.nfwd;
      const ChainStage& S = f ? J.fst[is] : J.bst[is - J.nfwd];
      const int K4 = (S.K + 3) & ~3;
      const int k0 = ic * CH_KC;
      const int kc = (K4 - k0 < CH_KC) ? K4 - k0 : CH_KC;
      const int slot = issued % CH_NSTAGE;
      if (!dry) {
        if (issued >= CH_NSTAGE) ch_slot_acquire(slot);
        if (tid == who) {
          const uint32_t bar = smem_u32(bars + slot), dst = smem_u32(wst + slot * CH_CHUNK_FLOATS);
          if (f) {
            mbar_expect_tx(bar, (uint32_t)S.N * CH_KC * 4u);
            tma_load_2d(dst, S.tm + (long long)rep * S.rsTm, k0, 0, bar);
          } else {
            const uint32_t bytes = (uint32_t)kc * (uint32_t)S.N * 4u;
            mbar_expect_tx(bar, bytes);
            bulk_load_1d(dst, S.W + po + (long long)k0 * S.ldw, bytes, bar);
          }
        }
      }
      ++issued;
      if (k0 + CH_KC >= K4) { ic = 0; ++is; } else { ++ic; }
    }
  };
  int total_chunks = 0;
  for (int s_ = direct0 ? 1 : 0; s_ < nst; ++s_) {
    const ChainStage& S_ = s_ < J.nfwd ? J.fst[s_] : J.bst[s_ - J.nfwd];
    total_chunks += (((S_.K + 3) & ~3) + CH_KC - 1) / CH_KC;
  }
  float4 wr0[CH_KC / 4];
  float b00 = 0.f, bq = 0.f;
  auto request_weights = [&]() {
    bq = __ldg(J.bhf + po);
    for (int e = tid; e < (J.Hhf >> 2); e += CH_THREADS) cp_async16(headF + 4 * e, J.Whf + po + 4 * e);
    for (int e = tid; e < (J.Hhb >> 2); e += CH_THREADS) cp_async16(headB + 4 * e, J.Whb + po + 4 * e);
    if (direct0 && tid < J.fst[0].N) {
      const ChainStage& S = J.fst[0];
      const int K4 = (S.K + 3) & ~3;
      const float4* __restrict__ wp = reinterpret_cast<const float4*>(S.W + po + (long long)tid * S.ldw);
#pragma unroll
      for (int q = 0; q < CH_KC / 4; ++q) wr0[q] = (4 * q < K4) ? __ldg(wp + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      b00 = __ldg(S.bias + po + tid);
    }
  };
  if (tid == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(J.fst[direct0 ? 1 : 0].tm + (long long)rep * J.fst[direct0 ? 1 : 0].rsTm) : "memory");
#pragma unroll
    for (int i = 0; i < CH_NSTAGE; ++i) mbar_init(smem_u32(bars + i), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (A.early_weights) { issue_next(0, false); issue_next(0, false); }
  }
  if (A.early_weights && tid < CH_THREADS) request_weights();
  KStamp ks_;
  C2_STAMP();
  __syncthreads();                         // barriers initialised (all nine warps)
  if (tid >= CH_THREADS) {
    // ---- producer warp: every remaining weight chunk of the forward AND the backward part, in order.  It takes part in the
    // cluster barriers without ever blocking the twins' exchange: it arrives for the exchange phase right away (it needs
    // nothing from it) and collects that phase when its work is done.
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    if (A.early_weights) { issue_next(CH_THREADS, true); issue_next(CH_THREADS, true); }
    while (is < nst) issue_next(CH_THREADS, false);
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    cluster_sync_all();                    // the final one (nobody leaves while its twin may still read its shared memory)
    return;
  }
  if (!A.early_weights) request_weights();

  float* In = actA;
  float* Out = actB;
  {  // forward input rows
    const float* __restrict__ X = J.X + (long long)rep * J.rsX + (long long)row0 * J.ldx;
    const int k4 = (J.K0 + 3) >> 2;
    for (int e = tid; e < ROWS * k4; e += CH_THREADS) {
      const int m = e / k4, q = e - m * k4;
      if (m < nrows) cp_async16(In + m * CH_INP + 4 * q, X + (long long)m * J.ldx + 4 * q);
      else *reinterpret_cast<float4*>(In + m * CH_INP + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  cp_async_commit();
  // per-row scalars of the backward part (produced by earlier launches): requested now, consumed after the forward chain
  const ChainRows& R = A.rw;
  const int B = K.B;
  const int row = row0 + w;
  const bool owner = (w < nrows) && lane == 0;           // lane 0 of warp w owns row w
  int t_row = 0;
  float r_row = 0.f, d_row = 0.f, lp_row = 0.f, q1_row = 0.f, q2_row = 0.f, gamma = 0.f, reward_scale = 0.f;
  if (owner) {
    t_row = (R.tid + rep * R.rsR)[row];
    if (A.kind == C2_CRITIC) {
      r_row = (R.r + rep * R.rsR)[row]; d_row = (R.d + rep * R.rsR)[row];
      gamma = K.hp[rep].gamma; reward_scale = K.hp[rep].reward_scale;
      lp_row = (R.logp + rep * R.rsLogp)[row];
      const float* Q = R.q + rep * 2 * R.rsY;
      q1_row = Q[row]; q2_row = Q[B + row];
    } else {
      lp_row = (R.logp + rep * R.rsLogp)[B + row];
    }
  }
  const float alpha_lo = (R.alpha + rep * R.rsAlpha)[lane < (K.T > 0 ? K.T : 1) ? lane : 0];
  const float alpha_hi = (K.T > 32) ? (R.alpha + rep * R.rsAlpha)[lane + 32 < K.T ? lane + 32 : 0] : 0.f;
  // backward-part operands that do not depend on this kernel's forward part
  float w0r[CH_MAXW * kMaxAct / CH_THREADS];
  const bool want_w0a = A.kind == C2_ACTORQ && J.nact > 0;
  if (want_w0a) {
    const float* __restrict__ W0 = J.W0 + po;
#pragma unroll
    for (int i = 0; i < CH_MAXW * kMaxAct / CH_THREADS; ++i) {
      const int e = tid + i * CH_THREADS, k = e >> 3, j = e & 7;
      w0r[i] = (k < J.H0 && j < J.nact) ? __ldg(W0 + (long long)k * J.ldw0 + J.col0 + j) : 0.f;
    }
  }
  C2_STAMP();

  int g = 0;
  // ---- generic dense stage (forward or backward flavour), shared by both parts ----------------------------------------
  auto run_stage = [&](const ChainStage& S, auto fwd_tag) {
    constexpr bool fwd = decltype(fwd_tag)::value;
    const int N = S.N, K4 = (S.K + 3) & ~3;
    float ebias = 0.f, emask[ROWS];
    if constexpr (fwd) {
      if (tid < N) ebias = __ldg(S.bias + po + tid);
    } else {
      const float* __restrict__ mk = S.mask + (long long)rep * S.rsMask + (long long)row0 * S.ldmask;
#pragma unroll
      for (int m = 0; m < ROWS; ++m) emask[m] = (tid < N && m < nrows) ? mk[(long long)m * S.ldmask + tid] : 0.f;
    }
    float acc[ROWS][8];
#pragma unroll
    for (int m = 0; m < ROWS; ++m)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[m][i] = 0.f;
    for (int k0 = 0; k0 < K4; k0 += CH_KC, ++g) {
      if (g == 0) { cp_async_wait<0>(); ch_sync(); }
      mbar_wait(smem_u32(bars + g % CH_NSTAGE), (uint32_t)((g / CH_NSTAGE) & 1));
      C2_STAMP();
      const int kc = (K4 - k0 < CH_KC) ? K4 - k0 : CH_KC;
      const float* __restrict__ Wc = wst + (g % CH_NSTAGE) * CH_CHUNK_FLOATS;
      if (4 * w < kc) {
        float4 a[ROWS];
#pragma unroll
        for (int m = 0; m < ROWS; ++m) a[m] = *reinterpret_cast<const float4*>(In + m * CH_INP + k0 + 4 * w);
        if constexpr (fwd) {
          float4 wv[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) wv[i] = *reinterpret_cast<const float4*>(Wc + (lane + 32 * i) * CH_KC + 4 * (w ^ (lane & 7)));
#pragma unroll
          for (int q = 0; q < 4; ++q) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float wq = q == 0 ? wv[i].x : (q == 1 ? wv[i].y : (q == 2 ? wv[i].z : wv[i].w));
#pragma unroll
              for (int m = 0; m < ROWS; ++m) {
                const float av = q == 0 ? a[m].x : (q == 1 ? a[m].y : (q == 2 ? a[m].z : a[m].w));
                acc[m][i] = fmaf(av, wq, acc[m][i]);
              }
            }
          }
        } else {
          float4 w0[4], w1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float* __restrict__ wr = Wc + (4 * w + q) * N;
            w0[q] = *reinterpret_cast<const float4*>(wr + 4 * lane);
            w1[q] = *reinterpret_cast<const float4*>(wr + 128 + 4 * lane);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
#pragma unroll
            for (int m = 0; m < ROWS; ++m) {
              const float av = q == 0 ? a[m].x : (q == 1 ? a[m].y : (q == 2 ? a[m].z : a[m].w));
              acc[m][0] = fmaf(av, w0[q].x, acc[m][0]); acc[m][1] = fmaf(av, w0[q].y, acc[m][1]);
              acc[m][2] = fmaf(av, w0[q].z, acc[m][2]); acc[m][3] = fmaf(av, w0[q].w, acc[m][3]);
              acc[m][4] = fmaf(av, w1[q].x, acc[m][4]); acc[m][5] = fmaf(av, w1[q].y, acc[m][5]);
              acc[m][6] = fmaf(av, w1[q].z, acc[m][6]); acc[m][7] = fmaf(av, w1[q].w, acc[m][7]);
            }
          }
        }
      }
      if (g + CH_NSTAGE < total_chunks) ch_slot_release(g % CH_NSTAGE);
    }
    {
      float* __restrict__ pw = part + w * (ROWS * CH_MAXW);
      if constexpr (fwd) {
#pragma unroll
        for (int m = 0; m < ROWS; ++m)
#pragma unroll
          for (int i = 0; i < 8; ++i) pw[m * CH_MAXW + lane + 32 * i] = acc[m][i];
      } else {
#pragma unroll
        for (int m = 0; m < ROWS; ++m) {
          *reinterpret_cast<float4*>(pw + m * CH_MAXW + 4 * lane) = make_float4(acc[m][0], acc[m][1], acc[m][2], acc[m][3]);
          *reinterpret_cast<float4*>(pw + m * CH_MAXW + 128 + 4 * lane) = make_float4(acc[m][4], acc[m][5], acc[m][6], acc[m][7]);
        }
      }
    }
    ch_sync();      
    if (tid < N) {
      float* __restrict__ go = S.out ? S.out + (long long)rep * S.rsOut + (long long)row0 * S.ldo : nullptr;
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        float v = 0.f;
#pragma unroll
        for (int ww = 0; ww < CH_WARPS; ++ww) v += part[(ww * ROWS + m) * CH_MAXW + tid];
        if constexpr (fwd) v = fmaxf(v + ebias, 0.f);
        else if (!(emask[m] > 0.f)) v = 0.f;
        Out[m * CH_INP + tid] = v;
        if (go && m < nrows) go[(long long)m * S.ldo + tid] = v;
      }
    }
    ch_sync();      
    C2_STAMP();
    float* t_ = In; In = Out; Out = t_;
  };

  // ================================ forward part ================================
  if (direct0) {
    const ChainStage& S = J.fst[0];
    const int N = S.N, K4 = (S.K + 3) & ~3;
    cp_async_wait<0>();
    ch_sync();      
    if (tid < N) {
      float* __restrict__ go = S.out ? S.out + (long long)rep * S.rsOut + (long long)row0 * S.ldo : nullptr;
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < CH_KC / 4; ++q)
          if (4 * q < K4) {
            const float4 x = *reinterpret_cast<const float4*>(In + m * CH_INP + 4 * q);
            v = fmaf(x.x, wr0[q].x, v); v = fmaf(x.y, wr0[q].y, v); v = fmaf(x.z, wr0[q].z, v); v = fmaf(x.w, wr0[q].w, v);
          }
        v = fmaxf(v + b00, 0.f);
        Out[m * CH_INP + tid] = v;
        if (go && m < nrows) go[(long long)m * S.ldo + tid] = v;
      }
    }
    ch_sync();      
    C2_STAMP();
    float* t_ = In; In = Out; Out = t_;
  }
  for (int s = direct0 ? 1 : 0; s < J.nfwd; ++s) run_stage(J.fst[s], std::true_type{});
  cp_async_wait<0>();
  ch_sync();      
  // forward scalar head: warp w owns row w
  float q_own = 0.f;
  // gate activations of the backward part: requested before the head so that their latency hides behind it (critic
  // update: written by an earlier launch; actor pass: written by THIS thread in the forward epilogue above)
  float hv[ROWS];
  {
    const float* __restrict__ hl = J.hlast + (long long)rep * J.rsHlast + (long long)row0 * J.ldh;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) hv[m] = (tid < J.Hhb && m < nrows) ? hl[(long long)m * J.ldh + tid] : 0.f;
  }
  if (w < nrows) {
    const float* __restrict__ hr = In + w * CH_INP;
    float a = 0.f;
    for (int k = lane; k < J.Hhf; k += 32) a = fmaf(hr[k], headF[k], a);
    q_own = warp_sum(a) + bq;
    if (lane == 0) {
      xch[w] = q_own;
      (J.qf_out + (long long)rep * J.rsQf)[row] = q_own;
    }
  }
  // ================================ the twins swap their head values ================================
  cluster_sync_all();                      // (also a CTA-wide barrier: xch is complete in both CTAs)
  C2_STAMP();
  // alpha of the row's task: lanes hold alpha[lane] / alpha[lane + 32]; every lane of the warp takes part in the shuffle
  const int t_b = __shfl_sync(0xffffffffu, t_row, 0);
  const float a_lo = __shfl_sync(0xffffffffu, alpha_lo, t_b & 31), a_hi = __shfl_sync(0xffffffffu, alpha_hi, t_b & 31);
  const float alpha_row = t_b < 32 ? a_lo : a_hi;
  if (owner) {
    const float q_peer = ld_peer_f32(xch + w, my_rank ^ 1u);
    const float qa = J.net == 0 ? q_own : q_peer, qb = J.net == 0 ? q_peer : q_own;
    if (A.kind == C2_CRITIC) {             // qa, qb = Qt1, Qt2
      const float t1 = reward_scale * r_row;
      const float t2 = gamma * (1.f - d_row);
      const float t3 = fminf(qa, qb) - alpha_row * lp_row;
      const float y = t1 + t2 * t3;
      const float qn = J.net == 0 ? q1_row : q2_row;
      const float dqv = 2.f * K.c_loss * (qn - y);
      sd[w] = dqv;
      (R.dq + rep * 2 * R.rsY)[J.net * B + row] = dqv;
      if (J.net == 0) {
        const float e1 = y - q1_row, e2 = y - q2_row;
        (R.y + rep * R.rsY)[row] = y;
        (R.lq + rep * R.rsY)[row] = e1 * e1 + e2 * e2;
      }
    } else {                               // qa, qb = Q1, Q2 at (s, a~)
      float g1, g2;
      if (qa == qb) { g1 = g2 = -0.5f * K.c_loss; }
      else if (qa < qb) { g1 = -K.c_loss; g2 = 0.f; }
      else { g1 = 0.f; g2 = -K.c_loss; }
      const float gq = J.net == 0 ? g1 : g2;
      sd[w] = gq;
      (R.dqa + rep * 2 * R.rsY)[J.net * B + row] = gq;
      if (J.net == 0) {
        const float qm = fminf(qa, qb);
        (R.la + rep * R.rsY)[row] = -(qm - alpha_row * lp_row);
        (R.qmin + rep * R.rsY)[row] = qm;
      }
    }
  }
  // ================================ backward part ================================
  {
    ch_sync();                             // sd visible
    if (tid < J.Hhb) {
      float* __restrict__ dyl = J.dylast ? J.dylast + (long long)rep * J.rsDy + (long long)row0 * J.lddy : nullptr;
      const float wh = headB[tid];
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        float v = 0.f;
        if (m < nrows) {
          v = fmaf(sd[m], wh, 0.f);
          if (!(hv[m] > 0.f)) v = 0.f;
          if (dyl) dyl[(long long)m * J.lddy + tid] = v;
        }
        In[m * CH_INP + tid] = v;
      }
    }
    if (want_w0a) {
#pragma unroll
      for (int i = 0; i < CH_MAXW * kMaxAct / CH_THREADS; ++i) w0a[tid + i * CH_THREADS] = w0r[i];
    }
    ch_sync();      
    C2_STAMP();
  }
  for (int s = 0; s < J.nbwd; ++s) run_stage(J.bst[s], std::false_type{});
  if (A.kind == C2_ACTORQ && J.nact > 0 && w < nrows) {   // d(action) of this twin: warp w owns row w
    const float* __restrict__ hr = In + w * CH_INP;
    float acc[kMaxAct];
#pragma unroll
    for (int j = 0; j < kMaxAct; ++j) acc[j] = 0.f;
    for (int k = lane; k < J.H0; k += 32) {
      const float dv = hr[k];
      const float4 wa = *reinterpret_cast<const float4*>(w0a + k * kMaxAct);
      const float4 wb = *reinterpret_cast<const float4*>(w0a + k * kMaxAct + 4);
      acc[0] = fmaf(dv, wa.x, acc[0]); acc[1] = fmaf(dv, wa.y, acc[1]); acc[2] = fmaf(dv, wa.z, acc[2]); acc[3] = fmaf(dv, wa.w, acc[3]);
      acc[4] = fmaf(dv, wb.x, acc[4]); acc[5] = fmaf(dv, wb.y, acc[5]); acc[6] = fmaf(dv, wb.z, acc[6]); acc[7] = fmaf(dv, wb.w, acc[7]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int j = 0; j < kMaxAct; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    }
    if (lane == 0) {
      float* o_ = J.dx + (long long)rep * J.rsDx + (long long)row * J.lddx + J.col0;
#pragma unroll
      for (int j = 0; j < kMaxAct; ++j)
        if (j < J.nact) o_[j] = acc[j];
    }
  }
  C2_STAMP();
  if (dbg != nullptr) dbg[CH_DBG_SLOTS - 1] = dbg_i;
  cluster_sync_all();                      // nobody leaves while its twin may still read its shared memory
#undef C2_STAMP
}

}  // namespace bsac
