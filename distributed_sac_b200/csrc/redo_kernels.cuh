// Dormant-neuron recycling (ReDo; Sokar, Agarwal, Castro, Evci, ICML 2023), per replica: b200sac_redo.
//   redo_score_kernel    one CTA per (network, hidden layer): the layer's neuron scores s_i = a_i / mean_j a_j, with
//                        a_i = (1/n) sum_rows max(h_ri, 0), over the activations the call's forward left in hA / hQ, and
//                        the dormant flags s_i <= tau, into the replica's record.  fp64, one fixed order, no atomics.
//   redo_recycle_kernel  shaped like reset_kernel, one blockIdx.y per layer: for every flagged neuron i, row i of the
//                        layer's weight takes the create draw, b[i] = 0, column i of the next weight matrix = 0, and Adam
//                        m = v = 0 at those entries.
#pragma once
#include "sac_kernels.cuh"

namespace bsac {

constexpr int kRedoThreads = 256;
constexpr int kRedoMaxLayers = 3 * 8;           // actor, q1, q2 x B200SAC_MAX_HIDDEN hidden layers

struct RedoLayer {
  const float* h;                // the layer's activations, rows [0, n) with pitch H (hA / hQ)
  long long rec;                 // the layer's first neuron in the replica's record
  long long w, b, wn;            // arena offsets: this layer's weight [H][ld] and bias, the next layer's weight [next_out][H]
  long long next_rec;            // the next layer's first neuron in the record; -1 when the next layer is the head
  int H, in, ld, next_out, tag;  // tag: the weight's Philox tag (init_table)
  int critic;                    // 0 = actor (tau[0]), 1 = q1 / q2 (tau[1])
};
struct RedoArgs {
  float* params;                 // the replica's parameter arena
  float* m;                      // its Adam m and v (trainable floats, the parameters' offsets)
  float* v;
  double* score;                 // its record
  unsigned char* dormant;
  unsigned long long key;        // seed + replica
  double tau[2];
  int n, nl;
  RedoLayer l[kRedoMaxLayers];
};

__global__ void __launch_bounds__(kRedoThreads) redo_score_kernel(const __grid_constant__ RedoArgs A) {
  const RedoLayer& t = A.l[blockIdx.x];
  __shared__ double part[kRedoThreads];
  double* score = A.score + t.rec;
  double acc = 0.0;                                       // this thread's neurons, in increasing order
  for (int i = threadIdx.x; i < t.H; i += kRedoThreads) {
    double s = 0.0;
    for (int r = 0; r < A.n; ++r) {
      const double x = (double)t.h[(long long)r * t.H + i];
      s += x < 0.0 ? 0.0 : x;                             // max(x, 0) that keeps a NaN
    }
    s /= (double)A.n;
    score[i] = s;
    acc += s;
  }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int w = kRedoThreads / 2; w > 0; w >>= 1) {        // fixed pairwise tree
    if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
    __syncthreads();
  }
  const double mean = part[0] / (double)t.H;
  const double tau = A.tau[t.critic];
  for (int i = threadIdx.x; i < t.H; i += kRedoThreads) {     // the same thread re-reads its own a_i
    const double s = mean == 0.0 ? 0.0 : score[i] / mean;
    score[i] = s;
    A.dormant[t.rec + i] = s <= tau ? 1 : 0;                  // NaN: never dormant
  }
}

// Element e of layer blockIdx.y's work: [0, H*in) the incoming rows (element index as the create draw counts it),
// [H*in, H*in + H) the bias, then [next_out][H] the outgoing columns.  An entry of a flagged outgoing column that lies in a
// flagged row of the next hidden layer takes that row's draw (the next layer's block writes it): the neuron of that row has
// its own outgoing column zeroed, so its value does not reach the output either way.
__global__ void __launch_bounds__(kRedoThreads) redo_recycle_kernel(const __grid_constant__ RedoArgs A) {
  const RedoLayer& t = A.l[blockIdx.y];
  const unsigned char* flag = A.dormant + t.rec;
  const unsigned char* next_flag = t.next_rec >= 0 ? A.dormant + t.next_rec : nullptr;
  const Philox ph(A.key);
  const float bound = xavier_bound(t.H, t.in);
  const long long n_in = (long long)t.H * t.in, n_all = n_in + t.H + (long long)t.next_out * t.H;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n_all; e += (long long)gridDim.x * blockDim.x) {
    long long off;
    float val = 0.f;
    if (e < n_in) {
      const int row = (int)(e / t.in), col = (int)(e % t.in);
      if (!flag[row]) continue;
      off = t.w + (long long)row * t.ld + col;
      val = xavier_draw(ph, e, t.tag, bound);
    } else if (e < n_in + t.H) {
      const int i = (int)(e - n_in);
      if (!flag[i]) continue;
      off = t.b + i;
    } else {
      const long long k = e - n_in - t.H;
      const int row = (int)(k / t.H), col = (int)(k % t.H);
      if (!flag[col] || (next_flag && next_flag[row])) continue;
      off = t.wn + (long long)row * t.H + col;
    }
    A.params[off] = val;
    A.m[off] = 0.f;
    A.v[off] = 0.f;
  }
}

}  // namespace bsac
