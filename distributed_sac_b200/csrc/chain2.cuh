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
// (twin 0, twin 1 of the same rows) swap their ROWS head values through distributed shared memory, and each goes on into the
// backward chain of its own twin -- the TMA weight pipeline never drains: the first backward chunks are requested while the
// forward head is still being computed.
// The swap is a remote st.async into the peer's xch, counted by the peer's exchange mbarrier (complete_tx), not a cluster
// barrier: barrier.cluster.arrive.release compiles to MEMBAR.ALL.GPU, which waits for every outstanding memory access of the
// thread while the producer warps of the whole grid keep the memory system full of weight requests -- 1 300 to 4 700 cycles
// of the critic update on the H100.  The one cluster barrier phase before the swap (relaxed arrive after the mbarrier
// initialisation, wait just before the first remote store) only guarantees that the peer's exchange mbarrier exists.
#pragma once
#include "chain.cuh"

namespace bsac {

// shared memory (floats) after the common part: forward / backward head rows [CH_INP] each, d(head output) [8], the
// exchanged head values [8], the action columns of W0 [256][8], the partial tiles
constexpr int C2_SM_W0A = CH_MAXW * kMaxAct;
constexpr size_t C2_SMEM_BYTES = (size_t)(CH_SM_COMMON + 2 * CH_INP + 2 * CH_ROWS + C2_SM_W0A + CH_SM_PART) * sizeof(float) + 1024;
enum { C2_CRITIC = 0, C2_ACTORQ = 1 };

struct Chain2Job {
  int rows, nfwd, nbwd, net;
  const float* X; long long rsX; int ldx, K0;          // forward: input rows [rows][ldx]
  const float* Whf; const float* bhf; int Hhf;         // forward scalar head [1][Hhf] + bias (arena)
  float* qf_out; long long rsQf;                       // forward head output of this twin (row 0)
  const float* hlast; long long rsHlast; int ldh;      // backward: last hidden activation of the differentiated net [rows][Hhb]
  float* dylast; long long rsDy; int lddy;             // optional store of the generated dY
  const float* Whb; int Hhb;                           // the differentiated net's scalar head weights [1][Hhb]
  const float* W0; int ldw0, col0, nact, H0;           // C2_ACTORQ: d(action) tail
  float* dx; long long rsDx; int lddx;
  ChainStage st[2 * CH_MAXL];                          // flat stage list: nfwd forward stages (hidden layers), then nbwd backward
};

struct Chain2Args {
  int kind, early_weights;
  long long rsP;
  long long* dbg;
  Chain2Job job[2];
  ChainRows rw;
};
static_assert(sizeof(Chain2Args) == 3424, "chain2_kernel argument layout changed");

B200_D void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
B200_D void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
// v -> the peer CTA's copy of *my_smem_addr, completing `bytes` of the transaction count of the peer's copy of *my_bar
B200_D void st_async_peer_f32(const float* my_smem_addr, const uint64_t* my_bar, uint32_t peer_rank, float v) {
  uint32_t ra, rb;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(my_smem_addr)), "r"(peer_rank));
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(smem_u32(my_bar)), "r"(peer_rank));
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra), "r"(__float_as_uint(v)), "r"(rb)
               : "memory");
}

// GATED: the actor pass (C2_ACTORQ), skipped on critic-only steps; its own instantiation, so that the critic update's
// launch carries no trace of the schedule.
template <int ROWS, bool GATED>
__global__ void __launch_bounds__(CH_BLOCK, 1) chain2_kernel(const __grid_constant__ Chain2Args A, StepConst K) {
  const Chain2Job& J = A.job[blockIdx.y];
  extern __shared__ __align__(1024) float sm2_raw[];
  ChainCta<ROWS> c(A.dbg, sm2_raw, J.rows, A.rsP);
  c.stamp();
  if (c.row0 >= J.rows) return;            // (both CTAs of the cluster share row0 and rows: they leave together)
  const int tid = c.tid, lane = c.lane, w = c.w, rep = c.rep, row0 = c.row0, nrows = c.nrows;
  const long long po = c.po;
  uint32_t my_rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(my_rank));

  float* headF = c.own_smem();             // [CH_INP] forward head row
  float* headB = headF + CH_INP;           // [CH_INP] backward (differentiated net's) head row
  float* sd = headB + CH_INP;              // [ROWS] d(head output) per row
  float* xch = sd + CH_ROWS;               // [ROWS] the PEER twin's forward head values (stored by the peer CTA)
  uint64_t* xbar = c.bars + CH_NSTAGE;     // exchange mbarrier: completes when the peer's nrows values have landed in xch
  float* w0a = xch + CH_ROWS;
  c.part = w0a + C2_SM_W0A;

  const int nst = J.nfwd + J.nbwd;
  const bool direct0 = J.nfwd > 1 && J.st[0].K <= CH_KC;
  c.set_stages(J.st, direct0 ? 1 : 0, J.nfwd, nst);
  DirectRow d0;
  float bq = 0.f;
  auto request_weights = [&]() {
    bq = __ldg(J.bhf + po);
    for (int e = tid; e < (J.Hhf >> 2); e += CH_THREADS) cp_async16(headF + 4 * e, J.Whf + po + 4 * e);
    for (int e = tid; e < (J.Hhb >> 2); e += CH_THREADS) cp_async16(headB + 4 * e, J.Whb + po + 4 * e);
    if (direct0) d0.load(J.st[0], po, tid);
  };
  // The actor pass on a critic-only step: both CTAs of a cluster belong to replica `rep` and read the same word, so they
  // leave together, before any cluster barrier.  The word is requested before griddepcontrol.wait (sched_word) and consumed
  // after it; a CTA that skips first drains what it requested early (no copy may outlive it).
  const int sched = GATED ? sched_of(K.cnt, rep) : SCHED_ACTOR;
  if (tid == 0) {
    mbar_init(smem_u32(xbar), 1);          // (start_pipeline's fence.mbarrier_init publishes it to the cluster)
    c.start_pipeline(A.early_weights);
  }
  if (A.early_weights && tid < CH_THREADS) request_weights();
  KStamp ks_;
  c.stamp();
  if (GATED && !(sched & SCHED_ACTOR)) {
    if (tid == 0)
      for (int i = 0; i < c.issued; ++i) mbar_wait(smem_u32(c.bars + i), 0u);
    asm volatile("cp.async.wait_all;" ::: "memory");
    return;
  }
  __syncthreads();                         // barriers initialised (all nine warps)
  cluster_arrive_relaxed();                // both CTAs' exchange mbarriers exist once this phase completes
  if (tid >= CH_THREADS) {
    // ---- producer warp: every remaining weight chunk of the forward AND the backward part, in order.  It collects the
    // initialisation phase when its work is done, so it never holds up the twins' exchange.
    c.produce(A.early_weights);
    cluster_wait();
    cluster_arrive_relaxed();              // the final phase (nobody leaves while its twin may still store into its shared memory)
    cluster_wait();
    return;
  }
  if (!A.early_weights) request_weights();
  c.load_input_rows(J.X, J.rsX, J.ldx, J.K0);
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
      gamma = K.disc ? K.disc[(long long)rep * B + row] : K.hp[rep].gamma; reward_scale = K.hp[rep].reward_scale;
      lp_row = (R.logp + rep * R.rsLogp)[row];
      const float* Q = R.q + rep * 2 * R.rsY;
      q1_row = Q[row]; q2_row = Q[B + row];
    } else {
      lp_row = (R.logp + rep * R.rsLogp)[B + row];
    }
  }
  const TaskAlpha alpha(R, K, rep, lane);
  // backward-part operands that do not depend on this kernel's forward part
  float w0r[C2_SM_W0A / CH_THREADS];
  const bool want_w0a = A.kind == C2_ACTORQ && J.nact > 0;
  if (want_w0a) {
    const float* __restrict__ W0 = J.W0 + po;
#pragma unroll
    for (int i = 0; i < C2_SM_W0A / CH_THREADS; ++i) {
      const int e = tid + i * CH_THREADS, k = e >> 3, j = e & 7;
      w0r[i] = (k < J.H0 && j < J.nact) ? __ldg(W0 + (long long)k * J.ldw0 + J.col0 + j) : 0.f;
    }
  }
  c.stamp();

  // ================================ forward part ================================
  if (direct0) direct_layer(c, J.st[0], d0);
  for (int s = c.first; s < J.nfwd; ++s) dense_stage<true>(c, J.st[s]);
  cp_async_wait<0>();
  ch_sync();
  // forward scalar head: warp w owns row w
  float q_own = 0.f;
  // gate activations of the backward part: requested before the head so that their latency hides behind it (critic
  // update: written by an earlier launch; actor pass: written by THIS thread in the forward epilogue above)
  float hv[ROWS];
  c.load_col(hv, J.hlast, J.rsHlast, J.ldh, J.Hhb);
  if (w < nrows) {
    const float* __restrict__ hr = c.In + w * CH_INP;
    float a = 0.f;
    for (int k = lane; k < J.Hhf; k += 32) a = fmaf(hr[k], headF[k], a);
    q_own = warp_sum(a) + bq;
  }
  // ================================ the twins swap their head values ================================
  cluster_wait();                          // the peer's exchange mbarrier is initialised
  if (w < nrows && lane == 0) {
    st_async_peer_f32(xch + w, xbar, my_rank ^ 1u, q_own);
    (J.qf_out + (long long)rep * J.rsQf)[row] = q_own;
  }
  if (tid == 0) mbar_expect_tx(smem_u32(xbar), (uint32_t)nrows * 4u);    // (the peer has the same rows)
  mbar_wait(smem_u32(xbar), 0u);
  c.stamp();
  const float alpha_row = alpha.of(__shfl_sync(0xffffffffu, t_row, 0));
  if (owner) {
    const float q_peer = xch[w];
    const float qa = J.net == 0 ? q_own : q_peer, qb = J.net == 0 ? q_peer : q_own;
    if (A.kind == C2_CRITIC) {             // qa, qb = Qt1, Qt2
      const float y = td_target(reward_scale * r_row, gamma * (1.f - d_row), qa, qb, alpha_row, lp_row);
      const float qn = J.net == 0 ? q1_row : q2_row;
      float dqv = 2.f * K.c_loss * (qn - y);
      const float iw = K.isw ? K.isw[(long long)rep * B + row] : 1.f;   // prioritized replay: importance weight
      if (K.isw) dqv = dqv * iw;
      sd[w] = dqv;
      (R.dq + rep * 2 * R.rsY)[J.net * B + row] = dqv;
      if (J.net == 0) {
        const float e1 = y - q1_row, e2 = y - q2_row;
        float l = e1 * e1 + e2 * e2;
        if (K.isw) l = l * iw;
        (R.y + rep * R.rsY)[row] = y;
        (R.lq + rep * R.rsY)[row] = l;
      }
    } else {                               // qa, qb = Q1, Q2 at (s, a~)
      float g1, g2;
      min_route(qa, qb, K.c_loss, g1, g2);
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
        c.In[m * CH_INP + tid] = v;
      }
    }
    if (want_w0a) {
#pragma unroll
      for (int i = 0; i < C2_SM_W0A / CH_THREADS; ++i) w0a[tid + i * CH_THREADS] = w0r[i];
    }
    ch_sync();
    c.stamp();
  }
  for (int s = J.nfwd; s < nst; ++s) dense_stage<false>(c, J.st[s]);
  if (A.kind == C2_ACTORQ && J.nact > 0 && w < nrows) {   // d(action) of this twin: warp w owns row w
    const float* __restrict__ hr = c.In + w * CH_INP;
    float acc[kMaxAct];
#pragma unroll
    for (int j = 0; j < kMaxAct; ++j) acc[j] = 0.f;
    for (int k = lane; k < J.H0; k += 32) {          // both float4 of the row's action weights are loaded before the FMAs
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
  c.stamp();
  c.stamp.done();
  cluster_arrive_relaxed();                // nobody leaves while its twin may still store into its shared memory
  cluster_wait();
}

}  // namespace bsac
