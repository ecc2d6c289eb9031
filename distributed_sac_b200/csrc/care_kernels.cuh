// CARE(M) state-encoder stages that are not plain GEMMs (MT10_Distributed_CARE/src/state_encoder.py,
// context_encoder.py with use_modified_care = true):
//
//   care_tables_kernel       per TASK (not per sample): z = E[t] (frozen RoBERTa row), attention
//                            att = softmax(trunk(z)) and context code ctx = mlp_context(z).  The reference
//                            evaluates these 768-wide MLPs on all B rows (state_encoder.py:85-93); they only
//                            depend on the task id, so T rows suffice (SURVEY.md 8(a) a15).
//   care_mix_kernel          encoded state of a row: [ctx[t] | sum_k att[t][k] Zk[k][row] / sum_k att[t][k]]
//                            (state_encoder.py:88-94), written straight into the consumer MLP's input buffer(s).
//   care_mix_bwd_kernel      backward of the mix for the critic update: dZk, d(att) per row.
//   care_tab_reduce_kernel   per-task sums of d(att), d(ctx) (fixed order), softmax backward.
//   care_tab_wgrad_kernel    backward of trunk / mlp_context on the T task rows -> weight and bias gradients.
// The mixture-of-encoders layers themselves (einsum 'kio,bi->kbo', state_encoder.py:155-174) run as K grouped
// problems of the GEMM engines; the mixture weights are stored [k][out][in] here (the reference holds [k][in][out]).
#pragma once
#include "common.cuh"
#include "sac_kernels.cuh"

namespace bsac {

constexpr int kCareMaxLayers = 9;     // <= 8 hidden + output
constexpr int kCareMaxT = 64;

struct CareNet {                      // a small MLP given by offsets into one replica's parameter arena
  int n;                              // number of Linear layers
  int dims[kCareMaxLayers + 1];       // dims[0] = input width
  long long w[kCareMaxLayers], b[kCareMaxLayers];
  int act_off[kCareMaxLayers];        // where layer j's output lives inside a task row of the table
};

struct CareTabArgs {
  const float* params; long long rsP;
  long long inst_delta[2];            // parameter offset of the encoder instance (0 = critic's, target_delta = target's)
  float* tab[2]; long long rsTab;     // table block per instance: [T][row_w]
  long long emb_off;
  CareNet trunk, ctx;
  int T, K, row_w, off_att;
  int original;                       // CARE(O): ctx = the shared, trainable context encoder on relu(E[t]); the trunk reads its output
  int sched_stride; const int* sched; // actor-side launch: replica 0's schedule word (skipped on critic-only steps); null = always runs
};

// grid (T, n_inst, R), block 512: 16 warps, one output neuron per warp at a time, up to 24 independent
// loads in flight per lane (the 768-long dot products are pure latency otherwise)
__global__ void __launch_bounds__(512) care_tables_kernel(CareTabArgs P) {
  const int sched = P.sched ? sched_word(P.sched + (int)blockIdx.z * P.sched_stride) : SCHED_ACTOR;
  KStamp ks_;
  __shared__ float xe[2048];
  __shared__ float bufA[512], bufB[512];
  const int t = blockIdx.x, inst = blockIdx.y, rep = blockIdx.z;
  if (!(sched & SCHED_ACTOR)) return;
  const float* __restrict__ par = P.params + rep * P.rsP;
  const float* __restrict__ E = par + P.emb_off + (long long)t * P.ctx.dims[0];
  float* __restrict__ row = P.tab[inst] + rep * P.rsTab + (long long)t * P.row_w;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int cin = P.ctx.dims[0];       // embedding row; == trunk input for CARE(M), the header input for CARE(O)
  for (int i = threadIdx.x; i < cin; i += 512) xe[i] = E[i];
  __syncthreads();
  __shared__ float zc[512];                             // CARE(O): context code z = cenc(relu(E[t])), the trunk's input
  if (P.original) {
    for (int i = threadIdx.x; i < cin; i += 512) xe[i] = fmaxf(xe[i], 0.f);    // Embedding -> ReLU -> header (context_encoder.py:73-77)
    __syncthreads();
  }
  for (int pass = 0; pass < 2; ++pass) {
    const bool is_ctx = (pass == 0);                    // context net first: in CARE(O) the trunk consumes its output
    const CareNet& N = is_ctx ? P.ctx : P.trunk;
    const long long delta = (is_ctx && P.original) ? 0 : P.inst_delta[inst];    // the context encoder has no target copy
    const float* cur = (!is_ctx && P.original) ? zc : xe;
    float* nxt = bufA;
    for (int j = 0; j < N.n; ++j) {
      const int nin = N.dims[j], nout = N.dims[j + 1];
      const float* __restrict__ W = par + delta + N.w[j];
      const float* __restrict__ bb = par + delta + N.b[j];
      if (nin <= 64) {
        // narrow layer: a warp's (up to four) output neurons are evaluated together -- all their weights and biases are
        // requested before the first FMA, so the layer costs one memory round trip instead of one per neuron
        float a[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f}, w0[4], w1[4];
        const float x0 = lane < nin ? cur[lane] : 0.f, x1 = lane + 32 < nin ? cur[lane + 32] : 0.f;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int o = warp + 16 * g;
          const float* __restrict__ wr = W + (long long)o * nin;
          w0[g] = (o < nout && lane < nin) ? __ldg(wr + lane) : 0.f;
          w1[g] = (o < nout && lane + 32 < nin) ? __ldg(wr + lane + 32) : 0.f;
          bv[g] = o < nout ? __ldg(bb + o) : 0.f;
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int o = warp + 16 * g;
          if (o < nout) {                                  // warp-uniform
            a[g] = fmaf(x0, w0[g], a[g]);
            a[g] = fmaf(x1, w1[g], a[g]);
            float v = warp_sum(a[g]) + bv[g];
            if (j < N.n - 1) v = fmaxf(v, 0.f);
            if (lane == 0) { nxt[o] = v; row[N.act_off[j] + o] = v; }
          }
        }
        for (int o = warp + 64; o < nout; o += 16) {     // wider-than-64-output layers: remaining neurons one at a time
          const float* __restrict__ wr = W + (long long)o * nin;
          float acc = fmaf(x0, lane < nin ? __ldg(wr + lane) : 0.f, 0.f);
          acc = fmaf(x1, lane + 32 < nin ? __ldg(wr + lane + 32) : 0.f, acc);
          float v = warp_sum(acc) + bb[o];
          if (j < N.n - 1) v = fmaxf(v, 0.f);
          if (lane == 0) { nxt[o] = v; row[N.act_off[j] + o] = v; }
        }
      } else
      for (int o = warp; o < nout; o += 16) {
        const float* __restrict__ wr = W + (long long)o * nin;
        const float bo = __ldg(bb + o);                    // bias requested with the weights, not after the reduction
        float a = 0.f;
        int i = lane;
        for (; i + 23 * 32 < nin; i += 24 * 32) {        // 768-wide rows: the whole row in flight (one round trip, not three)
          float wv[24];
#pragma unroll
          for (int u = 0; u < 24; ++u) wv[u] = __ldg(wr + i + u * 32);
#pragma unroll
          for (int u = 0; u < 24; ++u) a = fmaf(cur[i + u * 32], wv[u], a);
        }
        for (; i + 7 * 32 < nin; i += 8 * 32) {
          float wv[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) wv[u] = __ldg(wr + i + u * 32);
#pragma unroll
          for (int u = 0; u < 8; ++u) a = fmaf(cur[i + u * 32], wv[u], a);
        }
        for (; i < nin; i += 32) a = fmaf(cur[i], __ldg(wr + i), a);
        a = warp_sum(a) + bo;
        if (j < N.n - 1) a = fmaxf(a, 0.f);
        if (lane == 0) { nxt[o] = a; row[N.act_off[j] + o] = a; }
      }
      __syncthreads();
      cur = nxt;
      nxt = (nxt == bufA) ? bufB : bufA;
    }
    if (is_ctx && P.original) {
      for (int i = threadIdx.x; i < N.dims[N.n]; i += 512) zc[i] = cur[i];
      __syncthreads();
    }
    if (!is_ctx && threadIdx.x == 0) {                  // softmax over the K logits (F.softmax, dim=-1)
      const float* lg = cur;
      float mx = lg[0];
      for (int k = 1; k < P.K; ++k) mx = fmaxf(mx, lg[k]);
      float s = 0.f, e[32];
      for (int k = 0; k < P.K; ++k) { e[k] = expf(lg[k] - mx); s += e[k]; }
      for (int k = 0; k < P.K; ++k) row[P.off_att + k] = e[k] / s;
    }
    __syncthreads();
  }
}

struct CareMixArgs {
  const float* Z; long long rsZ, kstride; int ldz;      // Zk[k] = Z + k*kstride, [rows][ldz]
  const float* tab; long long rsTab; int row_w, off_att, off_ctx;
  const int* tid; long long rsR;
  int rows, B, K, mo, co;
  float* dst1; long long rsD1; int ld1;                 // every row r -> dst1[r]
  float* dst2; long long rsD2; int ld2; int row_off2;   // rows r >= row_off2 -> dst2[r - row_off2]   (nullable)
  int sched_stride; const int* sched;                   // as in CareTabArgs
};

// one warp per row; grid (ceil(rows/8), R), block 256
__global__ void __launch_bounds__(256) care_mix_kernel(CareMixArgs P) {
  const int sched = P.sched ? sched_word(P.sched + (int)blockIdx.y * P.sched_stride) : SCHED_ACTOR;
  KStamp ks_;
  const int rep = blockIdx.y, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int r = blockIdx.x * 8 + warp;
  if (r >= P.rows) return;
  if (!(sched & SCHED_ACTOR)) return;
  const int t = (P.tid + rep * P.rsR)[r % P.B];        // the CURRENT observation's task, also for the s' rows
  const float* __restrict__ trow = P.tab + rep * P.rsTab + (long long)t * P.row_w;
  float den = 0.f;
  for (int k = 0; k < P.K; ++k) den += trow[P.off_att + k];       // alpha.sum(dim=1)
  float* d1 = P.dst1 + rep * P.rsD1 + (long long)r * P.ld1;
  float* d2 = (P.dst2 != nullptr && r >= P.row_off2) ? P.dst2 + rep * P.rsD2 + (long long)(r - P.row_off2) * P.ld2 : nullptr;
  for (int j = lane; j < P.co; j += 32) {
    const float v = trow[P.off_ctx + j];
    d1[j] = v;
    if (d2) d2[j] = v;
  }
  const float* __restrict__ Z = P.Z + rep * P.rsZ + (long long)r * P.ldz;
  for (int j = lane; j < P.mo; j += 32) {
    float num = 0.f;
    for (int k = 0; k < P.K; ++k) num += Z[k * P.kstride + j] * trow[P.off_att + k];    // (z_encs * alpha).sum(dim=1)
    const float v = num / den;
    d1[P.co + j] = v;
    if (d2) d2[P.co + j] = v;
  }
}

struct CareMixBwdArgs {
  const float* dx; long long rsDxNet, rsDxRep; int lddx;      // [2][B][xw] gradients wrt the critic input rows
  const float* Z; long long rsZ, kstride; int ldz; int z_row_off;   // Zk rows of the s half start at z_row_off
  const float* tab; long long rsTab; int row_w, off_att;
  const int* tid; long long rsR;
  float* dZ; long long rsDZ, dkstride; int lddz;               // [K][B][lddz]
  float* datt; long long rsDatt;                               // [B][K]
  int B, K, mo, co;
};

// one warp per row; grid (ceil(B/8), R)
__global__ void __launch_bounds__(256) care_mix_bwd_kernel(CareMixBwdArgs P) {
  KStamp ks_;
  const int rep = blockIdx.y, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int i = blockIdx.x * 8 + warp;
  if (i >= P.B) return;
  const int t = (P.tid + rep * P.rsR)[i];
  const float* __restrict__ trow = P.tab + rep * P.rsTab + (long long)t * P.row_w;
  const float* __restrict__ d0 = P.dx + rep * P.rsDxRep + (long long)i * P.lddx + P.co;   // d z_enc part
  const float* __restrict__ Z = P.Z + rep * P.rsZ + (long long)(P.z_row_off + i) * P.ldz;
  float att[32], den = 0.f;
  for (int k = 0; k < P.K; ++k) { att[k] = trow[P.off_att + k]; den += att[k]; }
  float dden = 0.f, dak[32];
  for (int k = 0; k < P.K; ++k) dak[k] = 0.f;
  float* dZ = P.dZ + rep * P.rsDZ + (long long)i * P.lddz;
  for (int j = lane; j < P.mo; j += 32) {
    const float dz = d0[j] + d0[P.rsDxNet + j];
    float num = 0.f;
    for (int k = 0; k < P.K; ++k) num += Z[k * P.kstride + j] * att[k];
    const float dnum = dz / den;                       // z_enc = num / den
    dden += -(dz * num) / (den * den);
    for (int k = 0; k < P.K; ++k) {
      dZ[k * P.dkstride + j] = dnum * att[k];
      dak[k] = fmaf(dnum, Z[k * P.kstride + j], dak[k]);
    }
  }
  dden = warp_sum(dden);
  for (int k = 0; k < P.K; ++k) {
    const float s = warp_sum(dak[k]);
    if (lane == 0) (P.datt + rep * P.rsDatt)[(long long)i * P.K + k] = s + dden;
  }
}

struct CareTabReduceArgs {
  const float* datt; long long rsDatt;                  // [B][K]
  const float* dx; long long rsDxNet, rsDxRep; int lddx; // d ctx = dx[net][i][0..co)
  const float* tab; long long rsTab; int row_w, off_att;
  const int* tid; long long rsR;
  float* dtab; long long rsDtab;                         // [T][K + co]: dlogits (after softmax backward) | dctx
  int B, K, co;
};

// grid (T, R), block 1024 = 16 row groups x 64 values; partial sums combined in a fixed order
__global__ void __launch_bounds__(1024) care_tab_reduce_kernel(CareTabReduceArgs P) {
  KStamp ks_;
  __shared__ float part[16][64];
  __shared__ float tot[64];
  const int t = blockIdx.x, rep = blockIdx.y;
  const int v = threadIdx.x % 64, g = threadIdx.x / 64;
  const int nv = P.K + P.co;
  const int* __restrict__ tid = P.tid + rep * P.rsR;
  for (int v0 = 0; v0 < nv; v0 += 64) {
    const int vv = v0 + v;
    float s = 0.f;
    if (vv < nv) {
      const float* __restrict__ src = vv < P.K ? P.datt + rep * P.rsDatt + vv : P.dx + rep * P.rsDxRep + (vv - P.K);
      const long long ld = vv < P.K ? P.K : P.lddx;
      const long long second = vv < P.K ? 0 : P.rsDxNet;
      for (int i = g; i < P.B; i += 16) {
        if (tid[i] != t) continue;
        const float* d = src + (long long)i * ld;
        s += second ? d[0] + d[second] : d[0];
      }
    }
    part[g][v] = s;
    __syncthreads();
    if (g == 0) {
      float a = 0.f;
#pragma unroll
      for (int q = 0; q < 16; ++q) a += part[q][v];
      tot[v] = a;
    }
    __syncthreads();
    float* out = P.dtab + rep * P.rsDtab + (long long)t * nv;
    if (g == 0 && vv < nv && vv >= P.K) out[vv] = tot[v];
    if (v0 == 0 && threadIdx.x == 0) {                 // softmax backward on the K attention gradients (K <= 32 < 64)
      const float* att = P.tab + rep * P.rsTab + (long long)t * P.row_w + P.off_att;
      float dot = 0.f;
      for (int k = 0; k < P.K; ++k) dot += att[k] * tot[k];
      for (int k = 0; k < P.K; ++k) out[k] = att[k] * (tot[k] - dot);
    }
    __syncthreads();
  }
}

struct CareTabWgradArgs {
  const float* params; long long rsP; long long emb_off;
  const float* tab; long long rsTab; int row_w;
  const float* dtab; long long rsDtab;                   // [T][K + co]
  float* grads; long long rsG;
  CareNet trunk, ctx;
  int T, K, co;
  int original, off_ctx;              // CARE(O): trunk layer-0 input = z (table, off_ctx); ctx layer-0 input = relu(E[t])
  int tchunk;                         // tasks whose backward chains are held in shared memory at once
  float* grads_x; long long xs;       // per-task instantiation: gradient slice t >= 1 at grads_x + (t-1) xs (+ rep rsG)
};

// Shared memory of care_tab_wgrad_kernel: the default 48 KiB (no opt-in).  One task's chains are at most
// 8 x 512 + 32 (trunk) + 9 x 512 (context net) = 8 736 floats, so every configuration check_cfg accepts fits one task at least.
constexpr int kCareTabWgradSmemFloats = 12288;

// gradient slice t of replica rep (per-task instantiation): slice 0 is G itself
__device__ __forceinline__ float* care_grad_slice(const CareTabWgradArgs& P, float* G, int rep, int t) {
  return t == 0 ? G : P.grads_x + (long long)(t - 1) * P.xs + rep * P.rsG;
}

// grid (nblk, R), block 256.  Every CTA re-derives the (tiny) per-task backward chains in shared memory, then
// takes a slice of the weight / bias gradient elements: dW_j[o][i] = sum_t dz_j[t][o] * a_{j-1}[t][i].
// The tasks are taken in chunks of P.tchunk (T x the chains of one task can reach 2.2 MB): every gradient element's sum over
// t continues from the value its thread stored after the previous chunk, so the summation order (t ascending) and with it
// the result do not depend on the chunk size.
// kPerTask (pcgrad handles): no sum over tasks -- task t's term goes to gradient slice t (slice 0 = grads, slice t >= 1 =
// grads_x + (t-1) xs), fmaf(dz, a, 0) for a weight and dz for a bias, so every element of every slice is written each step.
template <bool kPerTask>
__global__ void __launch_bounds__(256) care_tab_wgrad_kernel(CareTabWgradArgs P) {
  KStamp ks_;
  extern __shared__ float sm[];
  const int rep = blockIdx.y;
  const float* __restrict__ par = P.params + rep * P.rsP;
  const float* __restrict__ tab0 = P.tab + rep * P.rsTab;
  const float* __restrict__ dtab0 = P.dtab + rep * P.rsDtab;
  float* __restrict__ G = P.grads + rep * P.rsG;
  const long long gstart = (long long)blockIdx.x * 256 + threadIdx.x, gstride = (long long)gridDim.x * 256;
  for (int t0 = 0; t0 < P.T; t0 += P.tchunk) {
    const int T = P.T - t0 < P.tchunk ? P.T - t0 : P.tchunk;       // tasks t0 .. t0 + T - 1
    const float* __restrict__ tab = tab0 + (long long)t0 * P.row_w;
    const float* __restrict__ dtab = dtab0 + (long long)t0 * (P.K + P.co);
    const float* __restrict__ emb = par + P.emb_off + (long long)t0 * P.ctx.dims[0];
    if (t0 > 0) __syncthreads();                       // every thread is done with the previous chunk's chains
    // dz storage: for net n, layer j: dz[n][j] is [T][dims[j+1]]
    int dz_off[2][kCareMaxLayers];
    int cur = 0;
    for (int n = 0; n < 2; ++n) {
      const CareNet& N = n == 0 ? P.trunk : P.ctx;
      for (int j = 0; j < N.n; ++j) { dz_off[n][j] = cur; cur += T * N.dims[j + 1]; }
    }
    for (int n = 0; n < 2; ++n) {
      const CareNet& N = n == 0 ? P.trunk : P.ctx;
      const int last = N.n - 1, nlast = N.dims[N.n];
      for (int e = threadIdx.x; e < T * nlast; e += 256) {
        const int t = e / nlast, o = e % nlast;
        sm[dz_off[n][last] + e] = dtab[(long long)t * (P.K + P.co) + (n == 0 ? o : P.K + o)];
      }
      __syncthreads();
      for (int j = last; j >= 1; --j) {                // dz_{j-1} = (dz_j W_j) * [a_{j-1} > 0]
        const int nin = N.dims[j], nout = N.dims[j + 1];
        const float* __restrict__ W = par + N.w[j];
        for (int e = threadIdx.x; e < T * nin; e += 256) {
          const int t = e / nin, i = e % nin;
          float s = 0.f;
          for (int o = 0; o < nout; ++o) s = fmaf(sm[dz_off[n][j] + t * nout + o], __ldg(W + (long long)o * nin + i), s);
          const float a = tab[(long long)t * P.row_w + N.act_off[j - 1] + i];
          sm[dz_off[n][j - 1] + e] = a > 0.f ? s : 0.f;
        }
        __syncthreads();
      }
    }
    // gradient elements of every (net, layer): [weights | bias], grid-strided per layer
    for (int n = 0; n < 2; ++n) {
      const CareNet& N = n == 0 ? P.trunk : P.ctx;
      for (int j = 0; j < N.n; ++j) {
        const int nin = N.dims[j], nout = N.dims[j + 1];
        const long long nw = (long long)nin * nout, tot = nw + nout;
        for (long long q = gstart; q < tot; q += gstride) {
          if (q < nw) {
            const int o = (int)(q / nin), i = (int)(q % nin);
            float s = t0 > 0 ? G[N.w[j] + q] : 0.f;
            for (int t = 0; t < T; ++t) {
              float a;
              if (j > 0) a = tab[(long long)t * P.row_w + N.act_off[j - 1] + i];
              else if (P.original && n == 0) a = tab[(long long)t * P.row_w + P.off_ctx + i];        // trunk(z.detach())
              else {
                a = emb[(long long)t * nin + i];
                if (P.original) a = fmaxf(a, 0.f);                                                // header(relu(E))
              }
              if constexpr (kPerTask) care_grad_slice(P, G, rep, t0 + t)[N.w[j] + q] = fmaf(sm[dz_off[n][j] + t * nout + o], a, 0.f);
              else s = fmaf(sm[dz_off[n][j] + t * nout + o], a, s);
            }
            if constexpr (!kPerTask) G[N.w[j] + q] = s;
          } else {
            const int o = (int)(q - nw);
            if constexpr (kPerTask) {
              for (int t = 0; t < T; ++t) care_grad_slice(P, G, rep, t0 + t)[N.b[j] + o] = sm[dz_off[n][j] + t * nout + o];
            } else {
              float s = t0 > 0 ? G[N.b[j] + o] : 0.f;
              for (int t = 0; t < T; ++t) s += sm[dz_off[n][j] + t * nout + o];
              G[N.b[j] + o] = s;
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// Fused mixture-of-encoders forward (+ the attention mix): state_encoder.py:98-129 for up to three encoder instances in one
// launch.  As K grouped problems per layer on the GEMM engine the 39->50->50 encoders were 4 320 tiles of 32 x 32 whose
// launch cost dwarfed their 40 k FMAs each.
// Here a CTA keeps ALL mixture weights of its instance in shared memory (K * sum(in*out) floats = 107 KB at the reference's
// dims), owns CMF_ROWS rows, and warp k walks encoder k through its layers with the activations in shared memory (input rows
// transposed so that eight rows of one input column are two broadcast 128-bit loads; lane = output neuron, 8 x 2
// accumulators; one warp per (encoder, 8-row group)).  Every layer's output is also stored for the backward pass (mixH / mixZ, same layout as before); the mix
// [ctx[t] | sum_k att[t][k] Z_k / sum_k att[t][k]] is evaluated in k order exactly like care_mix_kernel and written
// straight into the consumer MLPs' input buffers.
// ------------------------------------------------------------------------------------------------------------------------
constexpr int CMF_ROWS = 32;               // rows per CTA
constexpr int CMF_RP = CMF_ROWS + 4;       // row pitch of the transposed activation tiles (conflict-free 128-bit stores)
constexpr int CMF_MAXL = 4;                // mixture layers
constexpr int CMF_MAXJOBS = 3;
constexpr int CMF_THREADS = 768;           // 24 warps: one (encoder, 8-row group) task each at K = 6 -- six warps per scheduler hide the
                                           // shared-memory latency of the inner loop (fewer busy warps leave it exposed)

struct CareMixFwdJob {
  long long inst_delta;                    // parameter offset of the encoder instance
  int rows, xs_row0, out_row0, rows_buf;   // rows of the job; first XS row; first row / row count of the instance's buffers
  int cta0;                                // first blockIdx.x of the job
  const float* tab; long long rsTab;
  float* H[CMF_MAXL]; long long rsH[CMF_MAXL];    // outputs of layers 0..nl-1 ([K][rows_buf][pitch4(out)]); the last one is Z
  float* dst1; long long rsD1; int ld1;
  float* dst2; long long rsD2; int ld2; int row_off2;
};
struct CareMixFwdArgs {
  int njobs, nl, K, B;
  const float* params; long long rsP;
  long long w_off[CMF_MAXL], b_off[CMF_MAXL];
  int in[CMF_MAXL], out[CMF_MAXL];
  const float* XS; long long rsXS; int ldx;
  const int* tid; long long rsR;
  int row_w, off_att, off_ctx, mo, co;
  int maxw;                                // widest hidden / output layer
  CareMixFwdJob job[CMF_MAXJOBS];
  int sched_stride; const int* sched;      // as in CareTabArgs
};

// shared memory (floats): weights + biases of every layer, xs [in0][RP], ha / hb [K][maxw][RP] (ping-pong hidden tiles),
// zs [K][ROWS][mo], att [ROWS][K + 1]
static inline size_t care_mixfwd_smem_floats(const CareMixFwdArgs& A) {
  size_t n = 0;
  for (int l = 0; l < A.nl; ++l) n += (((size_t)A.K * A.out[l] * A.in[l] + 3) & ~(size_t)3) + (((size_t)A.K * A.out[l] + 3) & ~(size_t)3);
  n += (size_t)A.in[0] * CMF_RP;
  n += (size_t)(A.nl > 2 ? 2 : 1) * A.K * A.maxw * CMF_RP;
  n += (size_t)A.K * CMF_ROWS * A.mo;
  n += (size_t)CMF_ROWS * (A.K + 1);
  return n + 8;
}

__global__ void __launch_bounds__(CMF_THREADS, 1) care_mixfwd_kernel(const __grid_constant__ CareMixFwdArgs A) {
  extern __shared__ __align__(16) float cmf_sm[];
  int ji = 0;
  for (int j = 1; j < A.njobs; ++j)
    if ((int)blockIdx.x >= A.job[j].cta0) ji = j;
  const CareMixFwdJob& J = A.job[ji];
  const int rep = blockIdx.y;
  const int r0 = ((int)blockIdx.x - J.cta0) * CMF_ROWS;
  const int nrows = J.rows - r0 < CMF_ROWS ? J.rows - r0 : CMF_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int K = A.K;
  // carve -- every region is addressed as cmf_sm + <integer offset>: a table of pointers (or a pointer rounded through an
  // integer) makes the compiler lose the shared address space and emit generic LD.E instead of LDS in the inner loop
  int wtot = 0, btot = 0;
  for (int l = 0; l < A.nl; ++l) { wtot += (K * A.out[l] * A.in[l] + 3) & ~3; btot += (K * A.out[l] + 3) & ~3; }
  const int xs_off = wtot + btot;
  const int ha_off = xs_off + A.in[0] * CMF_RP;
  const int hb_off = A.nl > 2 ? ha_off + K * A.maxw * CMF_RP : ha_off;
  const int zs_off = (A.nl > 2 ? hb_off : ha_off) + K * A.maxw * CMF_RP;
  const int att_off = zs_off + K * CMF_ROWS * A.mo;
  float* xs = cmf_sm + xs_off;
  float* zs = cmf_sm + zs_off;
  float* att = cmf_sm + att_off;
  // The encoder pass of the actor update on a critic-only step: decided before the weight requests below (the word may be
  // read before griddepcontrol.wait: sched_word), so that no copy is in flight when the CTA leaves.
  const bool skip = A.sched && !(sched_word(A.sched + rep * A.sched_stride) & SCHED_ACTOR);
  // ---- weights: do not depend on the launch before this one (the optimizer step that wrote them is further back) ----------
  const float* par = A.params + (long long)rep * A.rsP + J.inst_delta;
  if (!skip) {
    int wpos = 0, bpos = wtot;
    for (int l = 0; l < A.nl; ++l) {
      const int nW = K * A.out[l] * A.in[l], nb = K * A.out[l];
      const float* gW = par + A.w_off[l];
      const float* gb = par + A.b_off[l];
      float* Wl = cmf_sm + wpos;
      float* bl = cmf_sm + bpos;
      if ((nW & 3) == 0) {
        for (int e = tid; e < (nW >> 2); e += CMF_THREADS) {
          const unsigned d = (unsigned)__cvta_generic_to_shared(Wl + 4 * e);
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gW + 4 * e) : "memory");
        }
      } else {
        for (int e = tid; e < nW; e += CMF_THREADS) Wl[e] = __ldg(gW + e);
      }
      for (int e = tid; e < nb; e += CMF_THREADS) bl[e] = __ldg(gb + e);
      wpos += (nW + 3) & ~3; bpos += (nb + 3) & ~3;
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  KStamp ks_;                              // XS / the task tables come from the launches before this one
  if (skip) return;
  // ---- input rows, transposed: xs[i][r] ------------------------------------------------------------------------------
  {
    const float* X = A.XS + (long long)rep * A.rsXS + (long long)(J.xs_row0 + r0) * A.ldx;
    const int in0 = A.in[0];
    for (int e = tid; e < CMF_ROWS * in0; e += CMF_THREADS) {
      const int r = e / in0, i = e - r * in0;
      xs[i * CMF_RP + r] = r < nrows ? X[(long long)r * A.ldx + i] : 0.f;
    }
    // attention weights of the rows' tasks (+ their sum, in k order like care_mix_kernel)
    if (tid < CMF_ROWS) {
      float den = 0.f;
      if (tid < nrows) {
        const int t = (A.tid + rep * A.rsR)[(J.out_row0 + r0 + tid) % A.B];
        const float* trow = J.tab + rep * J.rsTab + (long long)t * A.row_w;
        for (int k = 0; k < K; ++k) { const float a = trow[A.off_att + k]; att[tid * (K + 1) + k] = a; den += a; }
      }
      att[tid * (K + 1) + K] = den;
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  // ---- one task = (encoder k, group of 8 rows): walks the encoder's layers for its rows; tasks are independent ------------
  for (int task = w; task < K * (CMF_ROWS / 8); task += CMF_THREADS / 32) {
    const int k = task / (CMF_ROWS / 8), g = (task - k * (CMF_ROWS / 8)) * 8;
    int in_off = xs_off;                   // layer 0 reads the shared input tile; later layers this encoder's own hidden tile
    int in_pitch_k = 0;                    // 0: shared tile; else per-encoder stride
    int out_off = ha_off;
    int wpos = 0, bpos = wtot;
    for (int l = 0; l < A.nl; ++l) {
      const int in = A.in[l], out = A.out[l];
      const bool last = l == A.nl - 1;
      const float* Wk = cmf_sm + wpos + k * out * in;
      const float* bk = cmf_sm + bpos + k * out;
      const float* Ik = cmf_sm + in_off + in_pitch_k * k;
      const int po = (out + 3) & ~3;
      float* Hg = J.H[l] + (long long)rep * J.rsH[l] + ((long long)k * J.rows_buf + J.out_row0 + r0) * po;
      for (int o0 = 0; o0 < out; o0 += 64) {
        const int oa = o0 + lane, ob = o0 + 32 + lane;
        const bool va = oa < out, vb = ob < out;
        const float* wa = Wk + (size_t)(va ? oa : 0) * in;
        const float* wb = Wk + (size_t)(vb ? ob : 0) * in;
        const float ba = va ? bk[oa] : 0.f, bb = vb ? bk[ob] : 0.f;
        float acc0[8], acc1[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) { acc0[q] = 0.f; acc1[q] = 0.f; }
#pragma unroll 2
        for (int i = 0; i < in; ++i) {
          const float4 x0 = *reinterpret_cast<const float4*>(Ik + i * CMF_RP + g);
          const float4 x1 = *reinterpret_cast<const float4*>(Ik + i * CMF_RP + g + 4);
          const float w0 = wa[i], w1 = wb[i];
          acc0[0] = fmaf(x0.x, w0, acc0[0]); acc0[1] = fmaf(x0.y, w0, acc0[1]); acc0[2] = fmaf(x0.z, w0, acc0[2]); acc0[3] = fmaf(x0.w, w0, acc0[3]);
          acc0[4] = fmaf(x1.x, w0, acc0[4]); acc0[5] = fmaf(x1.y, w0, acc0[5]); acc0[6] = fmaf(x1.z, w0, acc0[6]); acc0[7] = fmaf(x1.w, w0, acc0[7]);
          acc1[0] = fmaf(x0.x, w1, acc1[0]); acc1[1] = fmaf(x0.y, w1, acc1[1]); acc1[2] = fmaf(x0.z, w1, acc1[2]); acc1[3] = fmaf(x0.w, w1, acc1[3]);
          acc1[4] = fmaf(x1.x, w1, acc1[4]); acc1[5] = fmaf(x1.y, w1, acc1[5]); acc1[6] = fmaf(x1.z, w1, acc1[6]); acc1[7] = fmaf(x1.w, w1, acc1[7]);
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          float v0 = acc0[q] + ba, v1 = acc1[q] + bb;
          if (!last) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          acc0[q] = v0; acc1[q] = v1;
          const int r = g + q;
          if (r < nrows) {
            if (va) Hg[(long long)r * po + oa] = v0;
            if (vb) Hg[(long long)r * po + ob] = v1;
          }
        }
        if (last) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            if (va) zs[((size_t)k * CMF_ROWS + g + q) * A.mo + oa] = acc0[q];
            if (vb) zs[((size_t)k * CMF_ROWS + g + q) * A.mo + ob] = acc1[q];
          }
        } else {
          float* Ok = cmf_sm + out_off + k * A.maxw * CMF_RP;
          if (va) {
            *reinterpret_cast<float4*>(Ok + oa * CMF_RP + g) = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
            *reinterpret_cast<float4*>(Ok + oa * CMF_RP + g + 4) = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
          }
          if (vb) {
            *reinterpret_cast<float4*>(Ok + ob * CMF_RP + g) = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
            *reinterpret_cast<float4*>(Ok + ob * CMF_RP + g + 4) = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
          }
        }
      }
      __syncwarp();                        // this warp's columns of layer l are complete before it reads them as layer l+1's input
      in_off = out_off; in_pitch_k = A.maxw * CMF_RP;
      out_off = (out_off == ha_off) ? hb_off : ha_off;
      wpos += (K * out * in + 3) & ~3; bpos += (K * out + 3) & ~3;
    }
  }
  __syncthreads();
  // ---- mix: [ctx[t] | sum_k att_k Z_k / sum_k att_k], k ascending ------------------------------------------------------------
  for (int e = tid; e < nrows * A.co; e += CMF_THREADS) {
    const int r = e / A.co, j = e - r * A.co;
    const int rg = J.out_row0 + r0 + r;
    const int t = (A.tid + rep * A.rsR)[rg % A.B];
    const float v = (J.tab + rep * J.rsTab + (long long)t * A.row_w)[A.off_ctx + j];
    (J.dst1 + rep * J.rsD1 + (long long)rg * J.ld1)[j] = v;
    if (J.dst2 != nullptr && rg >= J.row_off2) (J.dst2 + rep * J.rsD2 + (long long)(rg - J.row_off2) * J.ld2)[j] = v;
  }
  for (int e = tid; e < nrows * A.mo; e += CMF_THREADS) {
    const int r = e / A.mo, j = e - r * A.mo;
    const int rg = J.out_row0 + r0 + r;
    float num = 0.f;
    for (int k = 0; k < K; ++k) num += zs[((size_t)k * CMF_ROWS + r) * A.mo + j] * att[r * (K + 1) + k];
    const float v = num / att[r * (K + 1) + K];
    (J.dst1 + rep * J.rsD1 + (long long)rg * J.ld1)[A.co + j] = v;
    if (J.dst2 != nullptr && rg >= J.row_off2) (J.dst2 + rep * J.rsD2 + (long long)(rg - J.row_off2) * J.ld2)[A.co + j] = v;
  }
}

}  // namespace bsac
