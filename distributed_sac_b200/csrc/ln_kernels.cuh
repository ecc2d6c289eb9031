// LayerNorm in the critics' hidden layers (b200sac_cfg.critic_ln): h = relu(g * (z - mu) * rstd + c) after each hidden
// Linear of the E critics (q1, q2 on a twin handle) and their targets, torch's nn.LayerNorm(H, eps=1e-5) between the
// Linear and its ReLU.  Critic k's g, c (and their gradient slots) sit at critic 0's + k * rsNet.
//   ln_fwd_kernel   one warp per row of the [E][B][H] pre-normalization buffer z (every critic): the row statistics, then
//                   h = relu(g * xhat + c), in fp64, rounded to fp32 once.
//   ln_bwd_kernel   one CTA per (chunk of kLnRows rows, critic, replica): the ReLU-masked gradient dy in dh becomes dz in
//                   place, dz = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)); with dg / dc set, each CTA leaves its
//                   chunk's column sums of dy*xhat and dy in a partial buffer, and the last CTA of the (critic, replica)
//                   (ticket counter behind a fence) adds the chunks in index order into the gradient arena.
// Every sum is fp64 in one fixed order that depends on H and B alone, never on the replica count; no floating-point
// atomics.  The library compiles without FMA contraction, so each product and sum is rounded on its own.
// Dropout Q-functions (b200sac_cfg.critic_dropout, the <true> instantiations): ln_fwd_kernel first draws the row's
// keep masks, writes z' = z * (m ? s : 0) over z in place and keeps the masks as bits; ln_bwd_kernel multiplies the dz it
// writes by the same m ? s : 0.  The <false> instantiations are the plain LayerNorm kernels.
#pragma once
#include "sac_kernels.cuh"
#include "clip_kernels.cuh"

namespace bsac {

constexpr int kLnThreads = 256;
constexpr int kLnRows = 16;                 // rows per ln_bwd_kernel CTA
constexpr double kLnEps = 1e-5;

// A replica's critic dropout rate p (b200sac_set_critic_dropout): an element is dropped iff its Philox word < t =
// floor(p * 2^32); a kept one is multiplied by s = (float)(1 / (1 - p)).  p = 0: t = 0, s = 1 (nothing changes).
struct DropRate { unsigned t; float s; };

struct LnArgs {
  const float* z;          // [R][E][B][H] pre-normalization activations, replica stride rsZ (the dropout forward
                           // writes z' over them)
  float* h;                // ln_fwd: [R][E][B][H] post-ReLU output, replica stride rsH
  float* dh;               // ln_bwd: [R][E][B][H] dy in, dz out, replica stride rsH
  const float* g;          // critic 0's LayerNorm weight and bias of the layer (replica 0; replica stride rsP)
  const float* c;
  float* dg;               // ln_bwd: gradient-arena slots of g and c (replica stride rsG); null: the input gradient only
  float* dc;
  double* part;            // ln_bwd with dg: [R][E][chunks][2][H] chunk column sums (dy*xhat, dy)
  unsigned* ticket;        // [R][E] CTAs done; the last one resets it
  long long rsZ, rsH, rsP, rsG;
  long long rsNet;         // from one critic's g, c, dg, dc to the next's
  int B, H, E;
  int actor_side;          // 1: the actor pass (returns at entry on a critic-only step)
  // critic_dropout only: the rate table [R], the pass's mask bits [R][E][B][ceil(H / 32)] (replica stride rsM) and
  // (pass * 8 + layer) * E, the tag of q1's masks in this launch (critic k's is k more)
  const DropRate* drop;
  unsigned* mbits;
  long long rsM;
  int tag0;
};

// The keep masks of one warp's row: Philox4x32-10 keyed by seed ^ (kDropKeyMul * (replica + 1)), counter (step low,
// step high, row, tag << 24 | j / 4); column j takes output word j % 4 and is kept iff that word >= t.  Lane k draws the
// groups of four columns g = k, k + 32, ...: it applies them to z in place and ORs its four bits into word g / 8, bit
// 4 (g % 8); the eight lanes of a word combine by xor shuffles and the first of them stores it.
constexpr unsigned long long kDropKeyMul = 0xE7037ED1A0B428DBull;
B200_D void drop_row(float* z, unsigned* bits, int H, int lane, const Philox& ph, long long step, int row, unsigned tag,
                     DropRate dr) {
  const int groups = (H + 3) / 4, words = (H + 31) / 32;
  for (int g0 = 0; g0 < groups; g0 += kWarp) {
    const int g = g0 + lane;
    unsigned nib = 0;
    if (g < groups) {
      uint32_t r[4];
      ph((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)row, (tag << 24) | (uint32_t)g, r);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int j = 4 * g + q;
        if (j < H) {
          const bool keep = r[q] >= dr.t;
          z[j] = z[j] * (keep ? dr.s : 0.f);
          nib |= (keep ? 1u : 0u) << q;
        }
      }
    }
    unsigned w = nib << (4 * (lane & 7));
    w |= __shfl_xor_sync(0xffffffffu, w, 1);
    w |= __shfl_xor_sync(0xffffffffu, w, 2);
    w |= __shfl_xor_sync(0xffffffffu, w, 4);
    const int word = g0 / 8 + (lane >> 3);
    if ((lane & 7) == 0 && word < words) bits[word] = w;
  }
  __syncwarp();         // the row statistics read columns other lanes wrote
}

// Row statistics of z[0, H) on one warp: s = sum_j z_j, lane l adding z_l, z_{l+32}, ... in increasing order and the 32
// lane sums combined by the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same bits); mu = s / H,
// var = (the same sum of (z_j - mu)^2) / H, rstd = 1 / sqrt(var + 1e-5).
B200_D void ln_row_stats(const float* z, int H, int lane, double& mu, double& rstd) {
  double s = 0.0;
  for (int j = lane; j < H; j += kWarp) s += (double)z[j];
  mu = warp_sum_d(s) / (double)H;
  double v = 0.0;
  for (int j = lane; j < H; j += kWarp) {
    const double d = (double)z[j] - mu;
    v += d * d;
  }
  rstd = 1.0 / sqrt(warp_sum_d(v) / (double)H + kLnEps);
}

// grid ((E B + 7) / 8, R), 256 threads: warp w of CTA x normalizes row 8x + w of [E][B] (critic row / B)
template <bool kDrop>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_kernel(StepConst K, LnArgs P) {
  const int rep = blockIdx.y;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  if (skip) return;
  const int lane = threadIdx.x & 31, row = blockIdx.x * (kLnThreads / kWarp) + (threadIdx.x >> 5);
  if (row >= P.E * P.B) return;
  const int net = row / P.B, H = P.H;
  const float* z = P.z + rep * P.rsZ + (long long)row * H;
  float* h = P.h + rep * P.rsH + (long long)row * H;
  const float* g = P.g + net * P.rsNet + rep * P.rsP;
  const float* c = P.c + net * P.rsNet + rep * P.rsP;
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
    h[j] = y < 0.0 ? 0.f : (float)y;                    // relu that keeps a NaN
  }
}

// grid (ceil(B / kLnRows), E, R), 256 threads.  Rows of one CTA: [blockIdx.x * kLnRows, +kLnRows) of critic blockIdx.y.
// Row sums (one warp per row, the order of ln_row_stats): a = (sum_j g_j dy_j) / H, b = (sum_j g_j dy_j xhat_j) / H,
// xhat_j = (z_j - mu) * rstd; then thread t owns columns t, t + 256, ...: dz = (float)(rstd * ((g dy - a) - xhat * b)) and,
// with dg, its chunk's sums of dy*xhat and dy over the rows in increasing order.  The last CTA adds the chunks' sums in
// chunk order and rounds once.
// Dropout: dz is then multiplied by m ? s : 0, m read from the forward's mask bits.
template <bool kDrop>
__global__ void __launch_bounds__(kLnThreads) ln_bwd_kernel(StepConst K, LnArgs P) {
  const int rep = blockIdx.z, net = blockIdx.y, E = P.E;
  const bool skip = P.actor_side && !(sched_of(K.cnt, rep) & SCHED_ACTOR);
  KStamp ks_;
  __shared__ double st[kLnRows][4];       // mu, rstd, a, b of each row
  __shared__ bool s_last;
  if (skip) return;
  const int H = P.H, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * kLnRows, nr = min(kLnRows, P.B - r0);
  const long long base = ((long long)net * P.B + r0) * H;
  const float* z = P.z + rep * P.rsZ + base;
  float* dh = P.dh + rep * P.rsH + base;
  const float* g = P.g + net * P.rsNet + rep * P.rsP;
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
  const bool wg = P.dg != nullptr;
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
  float* dg = P.dg + net * P.rsNet + rep * P.rsG;
  float* dc = P.dc + net * P.rsNet + rep * P.rsG;
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
