// Layer-chained MLP kernels for the "LunarLander-class" SAC step (every hidden width <= 256, exact-fp32 mode).
//
// The per-layer launches of the generic plan cost one kernel boundary + one cold operand round trip per layer; at
// 256-wide layers that costs more than the math of the layer.
// Here a CTA owns CH_ROWS = 8 rows of ONE network and walks the whole chain of that network with the activations in
// shared memory:
//
//   forward   X -> relu(W0 x + b0) -> relu(W1 . + b1) ... -> head         LunarLander_Distributed_SAC/src/model.py:38-48,117-127
//             head = scalar Q head, or the tanh-Gaussian policy head (rsample, squash, log-prob: model.py:50-65)
//   backward  d(head out) -> dY_last = (dout Wh) * [h_last > 0] -> (dY W_l) * [h_{l-1} > 0] ... -> dh_0 (-> d(action))
//             autograd of the same modules; d(head out) is produced in the kernel from per-row scalars:
//             critic update   dQ = 2c (Q - y), y = rs r + gamma (1-d)(min(Qt1,Qt2) - alpha logpi')   learner.py:210, model.py:139-140
//             actor pass      min(Q1,Q2) gradient routing                                            learner.py:222-223
//             policy          closed-form backward of rsample/tanh/log-prob (oracle/sac_manual.py)   model.py:50-60
//
// Two kernels are built from the blocks below: chain_kernel (the forward of the actor and the local critics, the policy
// backward) and chain2_kernel (chain2.cuh: a twin-critic forward, the per-row scalar that needs both twins, and the
// backward of one twin, in one launch).
//
// Rows are independent, so nothing is exchanged between CTAs (chain2_kernel's twin pair aside) and there is no barrier wider
// than the CTA.  Every CTA streams the full weight matrices of its network through a 3-stage TMA pipeline of 32-k chunks
// (32 KB each, landing on mbarriers): forward chunks [<=256 n][32 k] come through a 2-D tensor map with the 128-byte swizzle
// straight from the nn.Linear-layout matrix (cp.async.bulk.tensor.2d, out-of-range k zero-filled), backward chunks are 32
// consecutive rows of the same matrix = one contiguous cp.async.bulk.  One elected thread issues a chunk; nobody's registers
// or LSU slots are spent on the copy (per-thread cp.async staging costs as much issue as the chunk's math).  The pipeline runs
// ahead across layer boundaries (weights do not depend on activations); 128 CTAs x 256 KB per 256x256 layer = 32 MB of L2
// reads -- the bound of this design.  Inside a chunk the 8 warps split K (warp w takes k = 4w..4w+3 of the 32), each lane holds
// an 8-row x 8-column accumulator tile (40 shared-memory wavefronts per 256 FFMA), and the eight partial tiles are added in
// warp order in shared memory: a fixed summation order, bit-reproducible run to run and replica to replica.
// The chunk pipeline is warp-specialised: a ninth warp issues the TMA requests and refills a slot as soon as the eight compute
// warps have released it (a named hardware barrier per slot: bar.arrive by the compute threads, bar.sync by the producer); the
// compute warps neither issue copies (a cp.async.bulk issue stalls the issuing warp) nor meet at a CTA-wide barrier per chunk
// (both sat on the critical path of every chunk).
//
// Weight gradients (the reduction over the batch) are a separate kernel, wgrad_kernel below: 32x32 output tiles, the
// 8 warps split the batch rows, lanes hold 4x8 accumulators, fixed-order reduction.
#pragma once
#include "gemm_tc.cuh"        // mbarrier / TMA wrappers
#include "sac_kernels.cuh"

namespace bsac {

constexpr int CH_ROWS = 8;                 // rows per CTA (template parameter ROWS = 8, 4 or 2; buffers are sized for 8)
constexpr int CH_MAXW = 256;               // widest layer / widest reduction
constexpr int CH_KC = 32;                  // k rows per weight chunk
constexpr int CH_NSTAGE = 3;               // weight chunks in flight
constexpr int CH_MAXL = 8;                 // dense stages per direction (= B200SAC_MAX_HIDDEN)
constexpr int CH_THREADS = 256;             // compute threads (8 warps)
constexpr int CH_WARPS = CH_THREADS / 32;
constexpr int CH_BLOCK = CH_THREADS + 32;   // + one producer warp: issues every weight chunk, waits on the slots' "empty" barriers
constexpr int CH_INP = CH_MAXW + 4;        // row pitch of the activation buffers
constexpr int CH_CHUNK_FLOATS = CH_MAXW * CH_KC;                     // 8192 floats = 32 KB: [256 n][32 k] swizzled | [32 k][256 n]
constexpr int CH_MAXJOBS = 3;
// shared memory (floats) of every chain kernel: weight stages, mbarriers (64 B: full[3]), two activation buffers; then the
// kernel's own buffers, and the partial tiles [8 warps][8 rows][256] last
constexpr int CH_SM_ACT = CH_ROWS * CH_INP;
constexpr int CH_SM_BARS = 16;
constexpr int CH_SM_COMMON = CH_NSTAGE * CH_CHUNK_FLOATS + CH_SM_BARS + 2 * CH_SM_ACT;
constexpr int CH_SM_PART = CH_WARPS * CH_ROWS * CH_MAXW;
// chain_kernel's own: head weights [16][260], d(head out) [8][16]
constexpr int CH_SM_HEADW = kMaxHeadOut * CH_INP;
constexpr int CH_SM_SD = CH_ROWS * kMaxHeadOut;
constexpr size_t CH_SMEM_BYTES = (size_t)(CH_SM_COMMON + CH_SM_HEADW + CH_SM_SD + CH_SM_PART) * sizeof(float) + 1024;  // + slack to align the stage buffers to 1 KB

enum { CJ_FWD = 0, CJ_BWD_POLICY = 1 };
enum { CH_HEAD_NONE = 0, CH_HEAD_SCALAR = 1, CH_HEAD_POLICY = 2 };

struct ChainStage {
  const float* W;          // parameter arena (replica stride rsP). forward: W[n][k] (nn.Linear layout); backward: the same
                           // matrix read as W[k][n] (k = the layer's outputs, n = its inputs)
  const float* bias;       // forward only (arena)
  const float* mask;       // backward only: the forward activation [rows][N] whose > 0 gates the result (row 0 of the job)
  float* out;              // optional global store of the stage output (row 0 of the job)
  const CUtensorMap* tm;   // forward only: 2-D map of W [N][K] (box 32 k x N rows, SWIZZLE_128B), replica 0; replica r at tm + r * rsTm
  int reserved0, rsTm;     // reserved0: padding, keeps the argument layout
  long long rsMask, rsOut;
  int ldw, ldmask, ldo;
  int K, N;                // reduction width, output width
};

struct ChainJob {
  int kind, rows, nstages, head;
  const float* X; long long rsX; int ldx, K0;          // FWD: input rows [rows][ldx], K0 valid columns
  const float* hlast; long long rsHlast; int ldh;      // BWD: last hidden activation [rows][Hh] (gate of the generated dY)
  float* dylast; long long rsDy; int lddy;             // BWD: optional store of the generated dY (needed by the weight gradient)
  const float* Wh; const float* bh; int NO, Hh;        // head weights [NO][Hh], bias (arena)
  float* qout; long long rsQ;                          // scalar head: output (row 0 of this net)
  ChainStage st[CH_MAXL];
};

// per-row scalars the backward parts turn into d(head output)
struct ChainRows {
  const float* r; const float* d; const int* tid; long long rsR;
  const float* logp; long long rsLogp;                 // [0,B) next-state half, [B,2B) current-state half
  const float* alpha; long long rsAlpha;               // exp(log_alpha[t]) of this step, written once by the ingest kernel
  const float* q;                                      // [2][B] local (s,a) head outputs, replica stride 2*rsY
  float* y; float* dq; float* lq; float* dqa; float* la; float* qmin; long long rsY;   // dq, dqa: [2][B], replica stride 2*rsY
  const float* dxP; long long rsDxNet, rsDxRep; int lddx;   // critic input gradients [2][B][ldx] (policy job)
  const float* psave; long long rsSave;                // rows B.. (current-state half), pre-offset by the host
  float* dout_dbg; float* dact_dbg; long long rsDbg;   // d(mu|log_std) [B][2A] (also the head weight-gradient operand), d(action) [B][A]
};

constexpr int CH_DBG_SLOTS = 64;
struct ChainArgs {
  int njobs;
  int early_weights;                       // 1: the weight matrices were not written by the launch right before this one, so the
                                           // first chunks are requested BEFORE griddepcontrol.wait (they land while the predecessor drains)
  long long rsP;
  long long* dbg;                          // optional clock64() timeline of CTA (0,0,0), CH_DBG_SLOTS entries (B200SAC_CHAIN_DBG=1)
  ChainJob job[CH_MAXJOBS];
  PolicyHeadArgs pol;
  ChainRows rw;
};
// Kernel argument layout moves ptxas scheduling (see StepConst): these sizes stay put.
static_assert(sizeof(ChainStage) == 88 && sizeof(ChainArgs) == 2904, "chain_kernel argument layout changed");

B200_D void cp_async16(float* smem_dst, const float* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
B200_D void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> B200_D void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

B200_D void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

B200_D void ch_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }      // the eight compute warps (the producer warp is not part of it)
// slot hand-back: the 256 compute threads ARRIVE (non-blocking) on the slot's named barrier once their reads of the chunk are
// done, the producer warp SYNCs on it before the refill -- hardware barriers 2..4, one per slot, 288 participants
B200_D void ch_slot_release(int slot) { asm volatile("bar.arrive %0, 288;" ::"r"(2 + slot) : "memory"); }
B200_D void ch_slot_acquire(int slot) { asm volatile("bar.sync %0, 288;" ::"r"(2 + slot) : "memory"); }

// Optional clock64() timeline of thread 0 of CTA (0,0,0) (B200SAC_CHAIN_DBG=1, scripts/chain_timeline.py): one entry per
// call, at most CH_DBG_SLOTS - 1; the last slot holds the entry count.
struct DbgStamp {
  long long* p;
  int i;
  B200_D explicit DbgStamp(long long* dbg)
      : p((dbg != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0 && threadIdx.x == 0) ? dbg : nullptr), i(0) {}
  B200_D void operator()() { if (p != nullptr && i < CH_DBG_SLOTS) p[i++] = clock64(); }
  B200_D void done() const { if (p != nullptr) p[CH_DBG_SLOTS - 1] = i; }
};

// alpha[t] of the step's tasks (<= 64): the lanes request alpha[lane] and alpha[lane + 32] up front, so a row's alpha then
// comes from a shuffle instead of a second, dependent round trip behind its task-id load
struct TaskAlpha {
  float lo, hi;
  B200_D TaskAlpha(const ChainRows& R, const StepConst& K, int rep, int lane)
      : lo((R.alpha + rep * R.rsAlpha)[lane < (K.T > 0 ? K.T : 1) ? lane : 0]),
        hi((K.T > 32) ? (R.alpha + rep * R.rsAlpha)[lane + 32 < K.T ? lane + 32 : 0] : 0.f) {}
  B200_D float of(int t) const {           // every lane of the warp takes part
    const float a = __shfl_sync(0xffffffffu, lo, t & 31), b = __shfl_sync(0xffffffffu, hi, t & 31);
    return t < 32 ? a : b;
  }
};

// The state a chain kernel's CTA shares between the building blocks below: its rows, its replica, the common shared-memory
// buffers and the weight pipeline over a flat stage list st[first, nst).  Stages below nfwd are forward (the swizzled [n][k]
// chunk through the stage's 2-D tensor map), the others backward ([k][n] rows, one contiguous bulk copy).  Chunk g lands in
// slot g % 3 on bars[g % 3] (phase (g / 3) & 1).
template <int ROWS>
struct ChainCta {
  DbgStamp stamp;
  int tid, lane, w, rep, row0, nrows;
  long long po;                            // this replica's offset in the parameter arena
  float* wst; uint64_t* bars;              // weight stages, their "full" mbarriers
  float* In; float* Out;                   // activation buffers [ROWS][CH_INP]: the next stage's input, its output
  float* part;                             // partial tiles [CH_WARPS][ROWS][CH_MAXW] (set by the kernel: last in its layout)
  const ChainStage* st;
  int first, nfwd, nst;
  int is, ic, issued;                      // producer: next chunk to issue (stage, chunk within the stage), chunks issued
  int g, total;                            // compute warps: next chunk to consume, chunks of the whole list

  // sm_raw: the kernel's dynamic shared memory.  SWIZZLE_128B tiles want 1 KB alignment; the offset is applied as POINTER
  // arithmetic on the shared array: rounding the address through an integer makes every later access a generic LD/ST
  B200_D ChainCta(long long* dbg, float* sm_raw, int rows, long long rsP)
      : stamp(dbg), tid(threadIdx.x), lane(threadIdx.x & 31), w(threadIdx.x >> 5), rep(blockIdx.z), row0(blockIdx.x * ROWS),
        nrows((rows - (int)blockIdx.x * ROWS < ROWS) ? rows - (int)blockIdx.x * ROWS : ROWS), po((long long)blockIdx.z * rsP) {
    wst = sm_raw + (((1024u - (smem_u32(sm_raw) & 1023u)) & 1023u) >> 2);
    bars = reinterpret_cast<uint64_t*>(wst + CH_NSTAGE * CH_CHUNK_FLOATS);
    In = wst + CH_NSTAGE * CH_CHUNK_FLOATS + CH_SM_BARS;
    Out = In + CH_SM_ACT;
    part = nullptr;
  }
  B200_D float* own_smem() const { return Out + CH_SM_ACT; }     // start of the kernel's own buffers

  B200_D void set_stages(const ChainStage* st_, int first_, int nfwd_, int nst_) {
    st = st_; first = first_; nfwd = nfwd_; nst = nst_;
    is = first; ic = 0; issued = 0; g = 0; total = 0;
    for (int s = first; s < nst; ++s) total += (((st[s].K + 3) & ~3) + CH_KC - 1) / CH_KC;
  }
  // Issue the next chunk (if any).  Run by the whole producer warp (the slot hand-back is a warp-wide bar.sync) or by thread 0
  // alone for the requests before griddepcontrol.wait; `leader` issues the copy.  dry: only step past a chunk that thread 0
  // already requested.
  B200_D void issue_next(bool leader, bool dry) {
    if (is >= nst) return;
    const ChainStage& S = st[is];
    const int K4 = (S.K + 3) & ~3;
    const int k0 = ic * CH_KC;
    const int kc = (K4 - k0 < CH_KC) ? K4 - k0 : CH_KC;
    const int slot = issued % CH_NSTAGE;
    if (!dry) {
      if (issued >= CH_NSTAGE) ch_slot_acquire(slot);               // every compute thread is done with the slot's previous chunk
      if (leader) {
        const uint32_t bar = smem_u32(bars + slot), dst = smem_u32(wst + slot * CH_CHUNK_FLOATS);
        if (is < nfwd) {
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
  // thread 0, before griddepcontrol.wait: the barriers and, when the weights do not come from the launch right before this
  // one, the first two chunks
  B200_D void start_pipeline(bool early) {
    if (first < nfwd) asm volatile("prefetch.tensormap [%0];" ::"l"(st[first].tm + (long long)rep * st[first].rsTm) : "memory");
#pragma unroll
    for (int i = 0; i < CH_NSTAGE; ++i) mbar_init(smem_u32(bars + i), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (early) { issue_next(true, false); issue_next(true, false); }
  }
  // the producer warp: every chunk thread 0 did not request, in order
  B200_D void produce(bool early) {
    if (early) { issue_next(false, true); issue_next(false, true); }
    while (is < nst) issue_next(tid == CH_THREADS, false);
  }

  // v[m] = p[row0 + m][tid] of a [rows][ld] buffer (replica stride rs) for this thread's column, 0 outside it
  B200_D void load_col(float (&v)[ROWS], const float* p, long long rs, int ld, int ncols) const {
    const float* __restrict__ q = p + (long long)rep * rs + (long long)row0 * ld;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) v[m] = (tid < ncols && m < nrows) ? q[(long long)m * ld + tid] : 0.f;
  }
  // the CTA's input rows [ROWS][K0] -> In by cp.async (rows past the job's end read as zero); the caller commits the group
  B200_D void load_input_rows(const float* X, long long rsX, int ldx, int K0) {
    const float* __restrict__ Xr = X + (long long)rep * rsX + (long long)row0 * ldx;
    const int k4 = (K0 + 3) >> 2;
    for (int e = tid; e < ROWS * k4; e += CH_THREADS) {
      const int m = e / k4, q = e - m * k4;
      if (m < nrows) cp_async16(In + m * CH_INP + 4 * q, Xr + (long long)m * ldx + 4 * q);
      else *reinterpret_cast<float4*>(In + m * CH_INP + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  B200_D void swap() { float* t = In; In = Out; Out = t; }
};

// An input layer with K <= 32 (8 / 10 columns at LunarLander) is evaluated DIRECTLY: thread n holds row n of W0 in registers
// and does the K-long dot product for every row itself -- no weight chunk, no split-K partials, no reduction (a chunk wait +
// partial-tile epilogue would cost far more than the 80 FMAs per thread).  The row and bias do not depend on the launch
// before this one, so they are requested before griddepcontrol.wait when the kernel may.
struct DirectRow {
  float4 w[CH_KC / 4];
  float b = 0.f;
  B200_D void load(const ChainStage& S, long long po, int tid) {
    if (tid < S.N) {
      const int K4 = (S.K + 3) & ~3;
      const float4* __restrict__ wp = reinterpret_cast<const float4*>(S.W + po + (long long)tid * S.ldw);
#pragma unroll
      for (int q = 0; q < CH_KC / 4; ++q) w[q] = (4 * q < K4) ? __ldg(wp + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      b = __ldg(S.bias + po + tid);
    }
  }
};
template <int ROWS>
B200_D void direct_layer(ChainCta<ROWS>& c, const ChainStage& S, const DirectRow& r) {
  const int N = S.N, K4 = (S.K + 3) & ~3;
  cp_async_wait<0>();
  ch_sync();                               // the input rows are in shared memory
  if (c.tid < N) {
    float* __restrict__ go = S.out ? S.out + (long long)c.rep * S.rsOut + (long long)c.row0 * S.ldo : nullptr;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      float v = 0.f;
#pragma unroll
      for (int q = 0; q < CH_KC / 4; ++q)
        if (4 * q < K4) {
          const float4 x = *reinterpret_cast<const float4*>(c.In + m * CH_INP + 4 * q);
          v = fmaf(x.x, r.w[q].x, v); v = fmaf(x.y, r.w[q].y, v); v = fmaf(x.z, r.w[q].z, v); v = fmaf(x.w, r.w[q].w, v);
        }
      v = fmaxf(v + r.b, 0.f);
      c.Out[m * CH_INP + c.tid] = v;
      if (go && m < c.nrows) go[(long long)m * S.ldo + c.tid] = v;
    }
  }
  ch_sync();
  c.stamp();                               // input layer done (direct)
  c.swap();
}

// One dense stage on the next chunks of the pipeline: forward Out = relu(In W^T + b), backward Out = (In W) * [mask > 0].
// Widths are multiples of 4 (fused_eligible), so the next stage's K4 == this stage's N and no pad column is left to clear.
template <bool FWD, int ROWS>
B200_D void dense_stage(ChainCta<ROWS>& c, const ChainStage& S) {
  const int tid = c.tid, lane = c.lane, w = c.w;
  const int N = S.N, K4 = (S.K + 3) & ~3;
  // epilogue operands of this thread's column, requested now
  float ebias = 0.f, emask[ROWS];
  if constexpr (FWD) {
    if (tid < N) ebias = __ldg(S.bias + c.po + tid);
  } else {
    c.load_col(emask, S.mask, S.rsMask, S.ldmask, N);
  }
  float acc[ROWS][8];
#pragma unroll
  for (int m = 0; m < ROWS; ++m)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[m][i] = 0.f;

  for (int k0 = 0; k0 < K4; k0 += CH_KC, ++c.g) {
    const int g = c.g;
    if (g == 0) { cp_async_wait<0>(); ch_sync(); }   // the prologue's cp.async pieces (every thread's) are visible to all
    mbar_wait(smem_u32(c.bars + g % CH_NSTAGE), (uint32_t)((g / CH_NSTAGE) & 1));
    c.stamp();                             // per chunk: data landed
    const int kc = (K4 - k0 < CH_KC) ? K4 - k0 : CH_KC;
    const float* __restrict__ Wc = c.wst + (g % CH_NSTAGE) * CH_CHUNK_FLOATS;
    if (4 * w < kc) {
      // every operand of the chunk is requested before the first FMA (no branches in between: the loads of columns
      // >= N read stale shared memory into accumulators nobody reads)
      float4 a[ROWS];
#pragma unroll
      for (int m = 0; m < ROWS; ++m) a[m] = *reinterpret_cast<const float4*>(c.In + m * CH_INP + k0 + 4 * w);
      if constexpr (FWD) {
        float4 wv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) wv[i] = *reinterpret_cast<const float4*>(Wc + (lane + 32 * i) * CH_KC + 4 * (w ^ (lane & 7)));   // 128-B swizzle: chunk ^ (row & 7)
        // k component outermost: 64 independent FMAs between two uses of an accumulator (per accumulator the
        // summation order is still k ascending)
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
    if (g + CH_NSTAGE < c.total) ch_slot_release(g % CH_NSTAGE);         // this thread is done with the slot
  }
  // ---- stage epilogue: the 8 partial tiles -> fixed-order sum -> bias+ReLU | ReLU' gate -> next input -------------------
  {
    float* __restrict__ pw = c.part + w * (ROWS * CH_MAXW);
    if constexpr (FWD) {
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
    float* __restrict__ go = S.out ? S.out + (long long)c.rep * S.rsOut + (long long)c.row0 * S.ldo : nullptr;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      float v = 0.f;
#pragma unroll
      for (int ww = 0; ww < CH_WARPS; ++ww) v += c.part[(ww * ROWS + m) * CH_MAXW + tid];
      if constexpr (FWD) v = fmaxf(v + ebias, 0.f);
      else if (!(emask[m] > 0.f)) v = 0.f;
      c.Out[m * CH_INP + tid] = v;
      if (go && m < c.nrows) go[(long long)m * S.ldo + tid] = v;
    }
  }
  ch_sync();
  c.stamp();                               // per stage: epilogue done
  c.swap();
}

// The forward of the actor and the local critics (FWD: hidden layers, then the policy or scalar head of each job), and the
// policy backward (!FWD: d(mu|log_std) from the critics' d(action) and the saved policy values, then the input-gradient chain).
template <bool FWD, int ROWS>
__global__ void __launch_bounds__(CH_BLOCK, 1) chain_kernel(const __grid_constant__ ChainArgs A, StepConst K) {
  const ChainJob& J = A.job[blockIdx.y];
  extern __shared__ __align__(1024) float sm_raw[];
  ChainCta<ROWS> c(A.dbg, sm_raw, J.rows, A.rsP);
  c.stamp();                               // 0: kernel entry
  const int tid = c.tid, lane = c.lane, w = c.w, rep = c.rep, row0 = c.row0, nrows = c.nrows;
  const long long po = c.po;
  const bool live = row0 < J.rows;
  float* headW = c.own_smem();
  float* sd = headW + CH_SM_HEADW;
  c.part = sd + CH_SM_SD;

  const bool direct0 = FWD && J.nstages > 1 && J.st[0].K <= CH_KC;
  c.set_stages(J.st, direct0 ? 1 : 0, FWD ? J.nstages : 0, J.nstages);
  // weights that do not depend on the launch right before this one: the head matrix (cp.async) and, for a directly
  // evaluated input layer, this thread's row of W0 + its bias (registers)
  DirectRow d0;
  auto request_weights = [&]() {
    if (J.NO > 0) {
      const float* __restrict__ Wh = J.Wh + po;
      const int q4 = J.Hh >> 2;
      for (int e = tid; e < J.NO * q4; e += CH_THREADS) {
        const int j = e / q4, q = e - j * q4;
        cp_async16(headW + j * CH_INP + 4 * q, Wh + (long long)j * J.Hh + 4 * q);
      }
    }
    if (direct0) d0.load(J.st[0], po, tid);
  };
  if (live) {
    if (tid == 0) c.start_pipeline(A.early_weights);
    if (A.early_weights && tid < CH_THREADS) request_weights();
  }
  KStamp ks_;
  c.stamp();                               // 1: predecessor complete (griddepcontrol.wait)
  if (!live) return;
  __syncthreads();                         // barriers initialised (all nine warps)
  if (tid >= CH_THREADS) {                 // ---- producer warp ----
    c.produce(A.early_weights);
    return;
  }
  if (!A.early_weights) request_weights();
  if constexpr (FWD) c.load_input_rows(J.X, J.rsX, J.ldx, J.K0);   // (joins the head weights in the cp.async group)
  cp_async_commit();
  c.stamp();                               // 2: prologue loads issued

  // ---- policy backward: d(mu|log_std) of the CTA's rows, then dY_last = (dout Wh) * [h_last > 0] -----------------------
  if constexpr (!FWD) {
    const ChainRows& R = A.rw;
    const int Aa = K.act;
    const int row = row0 + w;                      // warp w owns row w
    float hv[ROWS];                                // gate activations of this thread's column (issued before anything is waited for)
    c.load_col(hv, J.hlast, J.rsHlast, J.ldh, J.Hh);
    const TaskAlpha alpha(R, K, rep, lane);
    if (w < nrows) {                               // lane j < A owns action j
      const float alpha_row = alpha.of(__shfl_sync(0xffffffffu, lane == 0 ? (R.tid + rep * R.rsR)[row] : 0, 0));
      if (lane < Aa) {
        const float* __restrict__ sv = R.psave + rep * R.rsSave + ((long long)row * Aa + lane) * kSaveW;
        const float* __restrict__ dx0 = R.dxP + rep * R.rsDxRep + (long long)row * R.lddx + K.in_w + lane;
        const float da = dx0[0] + dx0[R.rsDxNet];
        float dmu, dls;
        policy_dout_point(K, sv, da, alpha_row, dmu, dls);
        sd[w * kMaxHeadOut + lane] = dmu;
        sd[w * kMaxHeadOut + Aa + lane] = dls;
        float* o = R.dout_dbg + rep * R.rsDbg + (long long)row * 2 * Aa;
        o[lane] = dmu;
        o[Aa + lane] = dls;
        (R.dact_dbg + rep * R.rsDbg)[(long long)row * Aa + lane] = da;
      }
    }
    c.stamp();                                     // (bwd) per-row scalars -> d(head output) done by warp 0
    cp_async_wait<0>();                            // the head weights have landed
    ch_sync();
    c.stamp();                                     // (bwd) head weights landed, every warp's d(head output) visible
    if (tid < J.Hh) {
      float* __restrict__ dyl = J.dylast ? J.dylast + (long long)rep * J.rsDy + (long long)row0 * J.lddy : nullptr;
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        float v = 0.f;
        if (m < nrows) {
          for (int j = 0; j < J.NO; ++j) v = fmaf(sd[m * kMaxHeadOut + j], headW[j * CH_INP + tid], v);
          if (!(hv[m] > 0.f)) v = 0.f;
          if (dyl) dyl[(long long)m * J.lddy + tid] = v;
        }
        c.In[m * CH_INP + tid] = v;
      }
    }
    ch_sync();                                     // In visible to every warp
  }

  c.stamp();                               // 3: backward prologue done (forward: == 2)
  if (direct0) direct_layer(c, J.st[0], d0);
  for (int s = c.first; s < J.nstages; ++s) dense_stage<FWD>(c, J.st[s]);
  cp_async_wait<0>();
  ch_sync();                               // (jobs without dense stages: head weights / inputs visible)

  // ---- head: warp w owns row w ----------------------------------------------------------------------------------------
  const int row = row0 + w;
  const float* __restrict__ hr = c.In + w * CH_INP;
  if (FWD && J.head == CH_HEAD_SCALAR) {
    if (w < nrows) {
      const float bq = __ldg(J.bh + po);           // requested before the dot product, consumed after it
      float a = 0.f;
      for (int k = lane; k < J.Hh; k += 32) a = fmaf(hr[k], headW[k], a);
      a = warp_sum(a) + bq;
      if (lane == 0) (J.qout + (long long)rep * J.rsQ)[row] = a;
    }
  } else if (FWD && J.head == CH_HEAD_POLICY) {
    // (1) every warp: the head GEMV of its row -> sd[row][0..2A).  (2) ONE warp evaluates the tanh-Gaussian of all
    // ROWS x A (row, action) pairs in parallel lanes: the transcendentals are evaluated in fp64 (DESIGN.md 3), and a
    // warp-wide fp64 instruction costs the same with 2 or 32 active lanes -- eight warps with two active lanes each
    // queue eight times the FP64-pipe work of one warp with 16 lanes.
    const int NO = 2 * K.act, H = J.Hh, Aa = K.act;
    if (w < nrows) {
      const float* __restrict__ bias = J.bh + po;
      // head GEMV of this warp's row, compact on purpose (this code runs once per CTA, out of a cold instruction cache, where
      // unrolled straight-line code is slower).  The 32 lanes split into NOp groups of G lanes
      // (NOp = NO rounded up to a power of two): lane (j, part) sums h[k] * W[j][k] over k = part (mod G), then a
      // log2(G)-level butterfly inside the group; lane j * G holds output j.
      int NOp = 1;
      while (NOp < NO) NOp <<= 1;
      const int G = 32 / NOp, jj = lane / G, part_ = lane - jj * G;
      float accj = 0.f;
      if (jj < NO) {
        const float* __restrict__ wrow = headW + jj * CH_INP;
#pragma unroll 4
        for (int k = part_; k < H; k += G) accj = fmaf(hr[k], wrow[k], accj);
      }
      for (int o = G >> 1; o > 0; o >>= 1) accj += __shfl_xor_sync(0xffffffffu, accj, o);
      if (jj < NO && part_ == 0) sd[w * kMaxHeadOut + jj] = accj + __ldg(bias + jj);
    }
    ch_sync();
    c.stamp();                                     // (policy head) GEMVs done
    if (w == 0) {
      const PolicyHeadArgs& P = A.pol;
      float* lp_s = c.part;                        // [ROWS][A] log-prob terms, [ROWS][A] log-std terms (the partial tiles are free now)
      float* ls_s = c.part + ROWS * kMaxAct;
      for (int e0 = 0; e0 < nrows * Aa; e0 += 32) {
        const int e = e0 + lane;
        if (e < nrows * Aa) {
          const int m = e / Aa, j = e - m * Aa, r = row0 + m;
          const float mu = sd[m * kMaxHeadOut + j], raw = sd[m * kMaxHeadOut + Aa + j];
          const float eps = policy_noise(K, P, rep, r, j);
          const PolicyPoint pp = policy_point(mu, raw, eps, K.action_scale);
          lp_s[m * kMaxAct + j] = pp.logp_j;
          ls_s[m * kMaxAct + j] = pp.logstd;
          float* sv = P.psave + rep * P.rsSave + ((long long)r * Aa + j) * kSaveW;
          sv[0] = pp.std; sv[1] = pp.diff; sv[2] = pp.t; sv[3] = pp.act; sv[4] = pp.jac; sv[5] = pp.eps; sv[6] = pp.mask;
          sv[7] = pp.logp_j;
          (P.act_out + rep * P.rsAct)[(long long)r * Aa + j] = pp.act;
          float* pout = P.pout + rep * P.rsPout + (long long)r * NO;
          pout[j] = mu;
          pout[Aa + j] = raw;
          if (r < K.B) (P.XT + rep * P.rsX)[(long long)r * K.ldx + K.in_w + j] = pp.act;
          else (P.XP + rep * P.rsX)[(long long)(r - K.B) * K.ldx + K.in_w + j] = pp.act;
        }
      }
      __syncwarp();
      if (lane < nrows) {                          // sums over the actions in index order, like the per-row version
        float tot = 0.f, tls = 0.f;
        for (int j = 0; j < Aa; ++j) { tot += lp_s[lane * kMaxAct + j]; tls += ls_s[lane * kMaxAct + j]; }
        (P.logp + rep * P.rsLogp)[row0 + lane] = tot;
        (P.logstd_sum + rep * P.rsLogp)[row0 + lane] = tls;
      }
    }
  }
  c.stamp();                               // last: head done
  c.stamp.done();
}

// ------------------------------------------------------------------------------------------------------------------------
// Weight / bias gradients of one network group in a single launch:
//   C[k][n] = sum_m A[m][k] * B[m][n],   C2[k] = sum_m A[m][k]
// (autograd of nn.Linear: A = d(pre-activation) [M][out], B = the layer's input [M][in]; the scalar / policy head's
// weight gradient is the same form with A = d(head output) [M][NO]).  One CTA = one 32 x 32 tile of one job; the
// 8 warps split the batch rows (contiguous groups), each lane holds a 4 x 8 accumulator tile (3 shared-memory
// wavefronts per 32 FFMA), the partial tiles are added in warp order.
// ------------------------------------------------------------------------------------------------------------------------
constexpr int WG_T = 32;
constexpr int WG_ROWS = 256;               // batch rows staged per pass
constexpr int WG_MAXJOBS = 20;
constexpr int WG_THREADS = 256;
constexpr size_t WG_SMEM_BYTES = (size_t)(2 * WG_ROWS * WG_T + 8 * WG_T * WG_T + 8 * WG_T + 16) * sizeof(float) + 128;

// lane mappings of a tile: FULL 32 k x 32 n (4 x 8 per lane); NTHIN for Nin <= 16 (input-layer weights: 32 k x 16 n,
// 4 x 4 per lane -- half the FMAs); KTHIN for Kout <= 4 (head weights: 4 k x 32 n, 4 x 1 per lane -- an eighth)
enum { WG_FULL = 0, WG_NTHIN = 1, WG_KTHIN = 2 };

struct WgradJob {
  const float* A; const float* B;          // work-slab pointers (row 0)
  float* C; float* C2;                     // gradient arena (replica stride rsG); C2 may be null
  const CUtensorMap* tmA; const CUtensorMap* tmB;   // 2-D maps [M rows][cols], box 32 x 256, dense; null -> staged by the threads
  long long rsA, rsB;
  int lda, ldb, ldc;
  int Kout, Nin;
  int tile0, tn;                           // first blockIdx.x of the job, tiles along Nin
  int shape;
  int reserved0, reserved1, rsTm;          // reserved: padding, keeps the argument layout; replica r's maps at tm + r * rsTm
};
// Adam (+ Polyak) applied by the CTA that just reduced a gradient tile: the gradient value is final the moment the
// tile's fixed-order sum is done, so the separate optimizer launch (one more kernel boundary + a cold pass over p/m/v) is
// unnecessary.  Same element-wise math as adam_kernel (adam_one, torch _single_tensor_adam).
struct WgradAdam {
  int which;                               // Adam step-counter / learning-rate slot (0 critic, 1 actor)
  float* params; float* m; float* v;       // arenas; an element's index = its offset in the gradient arena
  const float* grads;                      // gradient arena base (to turn C pointers into offsets)
  long long rsP, rsM;
  long long target_delta;                  // != 0: params[i + target_delta] is the Polyak target of element i
  const Counters* cnt;
};
struct WgradArgs {
  int njobs, M;
  long long rsG;
  long long* dbg;                          // optional clock64() timeline of CTA (0,0) (B200SAC_CHAIN_DBG=1)
  WgradAdam adam;
  WgradJob job[WG_MAXJOBS];
};
static_assert(sizeof(WgradJob) == 112 && sizeof(WgradArgs) == 2336, "wgrad_kernel argument layout changed");

B200_D void wg_stage(float* __restrict__ dst, const float* __restrict__ src, int ld, int c0, int cmax, int m0, int M, int tid) {
  for (int e = tid; e < WG_ROWS * (WG_T / 4); e += WG_THREADS) {
    const int mm = e >> 3, q = (e & 7) << 2;
    const int m = m0 + mm, c = c0 + q;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) {
      const float* p = src + (long long)m * ld + c;
      if (c < cmax) x.x = __ldg(p);
      if (c + 1 < cmax) x.y = __ldg(p + 1);
      if (c + 2 < cmax) x.z = __ldg(p + 2);
      if (c + 3 < cmax) x.w = __ldg(p + 3);
    }
    *reinterpret_cast<float4*>(dst + mm * WG_T + q) = x;
  }
}

// STORE_ONLY (grad_clip plans): the reduced tiles go to the gradient arena and nothing else; adam_kernel<true> applies the
// optimizer once the whole gradient, and with it its norm, is known.
template <bool STORE_ONLY = false>
__global__ void __launch_bounds__(WG_THREADS, 2) wgrad_kernel(const __grid_constant__ WgradArgs A, StepConst K) {
  DbgStamp stamp(A.dbg);
  stamp();                                 // 0: entry
  const WgradAdam& O = A.adam;
  extern __shared__ __align__(128) float wsm_raw[];
  float* sm = wsm_raw + (((128u - (smem_u32(wsm_raw) & 127u)) & 127u) >> 2);      // (pointer arithmetic keeps the shared address space)
  int ji = 0;
  for (int j = 1; j < A.njobs; ++j)
    if ((int)blockIdx.x >= A.job[j].tile0) ji = j;
  const WgradJob& J = A.job[ji];
  const int rep = blockIdx.y;
  const int t = (int)blockIdx.x - J.tile0;
  const int bk = t / J.tn, bn = t - bk * J.tn;
  const int k0 = bk * WG_T, n0 = bn * WG_T;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int ky = lane >> 2, nx = lane & 3;

  float* As = sm;
  float* Bs = As + WG_ROWS * WG_T;
  float* part = Bs + WG_ROWS * WG_T;
  float* bpart = part + 8 * WG_T * WG_T;
  uint64_t* bar = reinterpret_cast<uint64_t*>(bpart + 8 * WG_T);
  const CUtensorMap* tmA = J.tmA ? J.tmA + (long long)rep * J.rsTm : nullptr;
  const CUtensorMap* tmB = J.tmB ? J.tmB + (long long)rep * J.rsTm : nullptr;
  if (tid == 0) {
    if (tmA) asm volatile("prefetch.tensormap [%0];" ::"l"(tmA) : "memory");
    if (tmB) asm volatile("prefetch.tensormap [%0];" ::"l"(tmB) : "memory");
    mbar_init(smem_u32(bar), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  KStamp ks_;                              // the operands come from the launch right before this one
  stamp();                                 // 1: predecessor complete
  __syncthreads();
  // bias corrections of the fused optimizer step (two counter loads, an fp64 division and square root): evaluated now, while
  // the operand tiles are in flight, instead of heading the epilogue
  float step_size = 0.f, bc2_sqrt = 1.f;
  const HParams& H = K.hp[rep];
  if constexpr (!STORE_ONLY) adam_scalars(H.lr[O.which], O.cnt[rep].b1p[O.which], O.cnt[rep].b2p[O.which], step_size, bc2_sqrt);
  // the step's schedule (same cache line as the counters just read); consumed once the first operand tiles have landed, so
  // that a full step never waits for it
  const int sched = sched_of(O.cnt, rep);
  const float tau = H.tau, one_minus_tau = H.one_minus_tau;
  const float* __restrict__ Ag = J.A + (long long)rep * J.rsA;
  const float* __restrict__ Bg = J.B + (long long)rep * J.rsB;
  const int M = A.M;

  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float asum[4] = {0.f, 0.f, 0.f, 0.f};

  int pass = 0;
  for (int m0 = 0; m0 < M; m0 += WG_ROWS, ++pass) {
    if (m0 > 0) __syncthreads();
    if (tid == 0 && (tmA || tmB)) {
      mbar_expect_tx(smem_u32(bar), (uint32_t)((tmA ? 1 : 0) + (tmB ? 1 : 0)) * WG_ROWS * WG_T * 4u);
      if (tmA) tma_load_2d(smem_u32(As), tmA, k0, m0, smem_u32(bar));
      if (tmB) tma_load_2d(smem_u32(Bs), tmB, n0, m0, smem_u32(bar));
    }
    if (!tmA) wg_stage(As, Ag, J.lda, k0, J.Kout, m0, M, tid);
    if (!tmB) wg_stage(Bs, Bg, J.ldb, n0, J.Nin, m0, M, tid);
    if (tmA || tmB) mbar_wait(smem_u32(bar), (uint32_t)(pass & 1));
    __syncthreads();
    if (pass == 0 && O.which == 1 && !(sched & SCHED_ACTOR)) return;   // the actor's gradients + Adam on a critic-only step
    stamp();                               // per pass: operands landed
    const int mcnt = (M - m0 < WG_ROWS) ? M - m0 : WG_ROWS;
    const int per = (mcnt + 7) >> 3;
    const int mb = w * per, me = (mb + per < mcnt) ? mb + per : mcnt;
    if (J.shape == WG_FULL) {
#pragma unroll 4
      for (int m = mb; m < me; ++m) {
        const float4 a = *reinterpret_cast<const float4*>(As + m * WG_T + 4 * ky);
        const float4 b0 = *reinterpret_cast<const float4*>(Bs + m * WG_T + 8 * nx);
        const float4 b1 = *reinterpret_cast<const float4*>(Bs + m * WG_T + 8 * nx + 4);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          asum[i] += av[i];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
      }
    } else if (J.shape == WG_NTHIN) {
#pragma unroll 4
      for (int m = mb; m < me; ++m) {
        const float4 a = *reinterpret_cast<const float4*>(As + m * WG_T + 4 * ky);
        const float4 b0 = *reinterpret_cast<const float4*>(Bs + m * WG_T + 4 * nx);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          asum[i] += av[i];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
      }
    } else {
#pragma unroll 4
      for (int m = mb; m < me; ++m) {
        const float4 a = *reinterpret_cast<const float4*>(As + m * WG_T);
        const float b = Bs[m * WG_T + lane];
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          asum[i] += av[i];
          acc[i][0] = fmaf(av[i], b, acc[i][0]);
        }
      }
    }
  }
  stamp();                                 // accumulation done
  // partial tiles -> fixed-order sum.  Every mapping fills the part of the [32 k][32 n] tile that holds its valid outputs.
  {
    float* pw = part + w * (WG_T * WG_T);
    if (J.shape == WG_FULL) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        *reinterpret_cast<float4*>(pw + (4 * ky + i) * WG_T + 8 * nx) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        *reinterpret_cast<float4*>(pw + (4 * ky + i) * WG_T + 8 * nx + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
      }
      if (nx == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) bpart[w * WG_T + 4 * ky + i] = asum[i];
      }
    } else if (J.shape == WG_NTHIN) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        *reinterpret_cast<float4*>(pw + (4 * ky + i) * WG_T + 4 * nx) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      if (nx == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) bpart[w * WG_T + 4 * ky + i] = asum[i];
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) pw[i * WG_T + lane] = acc[i][0];
      if (lane < 4) bpart[w * WG_T + lane] = lane == 0 ? asum[0] : (lane == 1 ? asum[1] : (lane == 2 ? asum[2] : asum[3]));
    }
  }
  __syncthreads();
  stamp();                                 // partial tiles visible
  float* __restrict__ C = J.C + (long long)rep * A.rsG;
  if constexpr (STORE_ONLY) {              // the same fixed-order sums as below, stored only
    const int kk = tid >> 3, nn4 = (tid & 7) << 2;
    if (k0 + kk < J.Kout && n0 + nn4 < J.Nin) {
      float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int ww = 0; ww < 8; ++ww) {
        const float4 q = *reinterpret_cast<const float4*>(part + ww * (WG_T * WG_T) + kk * WG_T + nn4);
        g4.x += q.x; g4.y += q.y; g4.z += q.z; g4.w += q.w;
      }
      *reinterpret_cast<float4*>(C + (long long)(k0 + kk) * J.ldc + n0 + nn4) = g4;
    }
    if (bn == 0 && J.C2 != nullptr && tid < WG_T && k0 + tid < J.Kout) {
      float v = 0.f;
#pragma unroll
      for (int ww = 0; ww < 8; ++ww) v += bpart[ww * WG_T + tid];
      (J.C2 + (long long)rep * A.rsG)[k0 + tid] = v;
    }
    stamp.done();
    return;
  }
  // fused optimizer step: adam_one per element like adam_kernel
  const float w1 = (float)(1.0 - K.beta1), b2 = (float)K.beta2, omb2 = (float)(1.0 - K.beta2), eps = (float)K.adam_eps;
  // One thread = four consecutive columns of one row of the tile (128-bit accesses; row pitches, tile origins and tensor
  // offsets are multiples of 4 floats by construction of the arena -- pad columns of a thin first layer see zero gradients
  // and stay zero).  Every operand of the optimizer step is REQUESTED before the first dependent instruction: the (p, m, v
  // [, target]) quadruples would otherwise be sequential global round trips between stores -- and the code is kept compact on
  // purpose: it runs once per CTA out of a cold instruction cache.
  const bool has_t = O.target_delta != 0 && (sched & SCHED_TARGET);   // targets untouched on a step without a target update
  const int kk = tid >> 3, nn4 = (tid & 7) << 2;
  const bool okq = k0 + kk < J.Kout && n0 + nn4 < J.Nin;
  const long long ci = (long long)(k0 + kk) * J.ldc + n0 + nn4;
  const long long gi = (J.C - O.grads) + ci;
  float4 p4 = make_float4(0.f, 0.f, 0.f, 0.f), m4 = p4, v4 = p4, t4 = p4;
  if (okq) {
    const float* pp = O.params + rep * O.rsP + gi;
    p4 = *reinterpret_cast<const float4*>(pp);
    m4 = *reinterpret_cast<const float4*>(O.m + rep * O.rsM + gi);
    v4 = *reinterpret_cast<const float4*>(O.v + rep * O.rsM + gi);
    if (has_t) t4 = *reinterpret_cast<const float4*>(pp + O.target_delta);
  }
  const bool bias_thread = bn == 0 && J.C2 != nullptr && tid < WG_T && k0 + tid < J.Kout;
  float bp = 0.f, bm = 0.f, bv_ = 0.f, bt = 0.f;
  const long long bgi = bias_thread ? (J.C2 - O.grads) + k0 + tid : 0;
  if (bias_thread) {
    const float* pp = O.params + rep * O.rsP + bgi;
    bp = *pp;
    bm = (O.m + rep * O.rsM)[bgi];
    bv_ = (O.v + rep * O.rsM)[bgi];
    if (has_t) bt = pp[O.target_delta];
  }
  float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int ww = 0; ww < 8; ++ww) {           // fixed order: warp 0's partial first
    const float4 q = *reinterpret_cast<const float4*>(part + ww * (WG_T * WG_T) + kk * WG_T + nn4);
    g4.x += q.x; g4.y += q.y; g4.z += q.z; g4.w += q.w;
  }
  stamp();                                 // partial tiles summed (optimizer operands still in flight)
  if (okq) {
    *reinterpret_cast<float4*>(C + ci) = g4;
    adam_one(p4.x, m4.x, v4.x, g4.x, w1, b2, omb2, step_size, bc2_sqrt, eps);
    adam_one(p4.y, m4.y, v4.y, g4.y, w1, b2, omb2, step_size, bc2_sqrt, eps);
    adam_one(p4.z, m4.z, v4.z, g4.z, w1, b2, omb2, step_size, bc2_sqrt, eps);
    adam_one(p4.w, m4.w, v4.w, g4.w, w1, b2, omb2, step_size, bc2_sqrt, eps);
    float* pp = O.params + rep * O.rsP + gi;
    *reinterpret_cast<float4*>(pp) = p4;
    *reinterpret_cast<float4*>(O.m + rep * O.rsM + gi) = m4;
    *reinterpret_cast<float4*>(O.v + rep * O.rsM + gi) = v4;
    if (has_t)
      *reinterpret_cast<float4*>(pp + O.target_delta) =
          make_float4(tau * p4.x + one_minus_tau * t4.x, tau * p4.y + one_minus_tau * t4.y,
                      tau * p4.z + one_minus_tau * t4.z, tau * p4.w + one_minus_tau * t4.w);
  }
  if (bias_thread) {
    float v = 0.f;
#pragma unroll
    for (int ww = 0; ww < 8; ++ww) v += bpart[ww * WG_T + tid];
    (J.C2 + (long long)rep * A.rsG)[k0 + tid] = v;
    adam_one(bp, bm, bv_, v, w1, b2, omb2, step_size, bc2_sqrt, eps);
    float* pp = O.params + rep * O.rsP + bgi;
    *pp = bp;
    (O.m + rep * O.rsM)[bgi] = bm;
    (O.v + rep * O.rsM)[bgi] = bv_;
    if (has_t) pp[O.target_delta] = tau * bp + one_minus_tau * bt;
  }
  stamp();                                 // reduction + optimizer step done
  stamp.done();
}

}  // namespace bsac
