// libb200sac: C-ABI implementation (see include/b200sac.h) -- host orchestration of the
// sm_90a SAC gradient step.  One handle = R independent learners of one shape stepped
// together; one step = a fixed list of grouped launches captured once into a CUDA graph.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <random>
#include <string>
#include <tuple>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <variant>
#include <vector>

#include "../../include/b200sac.h"
#include "gemm_simt.cuh"
#include "gemm_thin.cuh"
#include "gemm_tc.cuh"
#include "sac_kernels.cuh"
#include "care_kernels.cuh"
#include "chain.cuh"
#include "chain2.cuh"
#include "per_kernels.cuh"
#include "nstep_kernels.cuh"
#include "clip_kernels.cuh"
#include "pcgrad_kernels.cuh"
#include "redo_kernels.cuh"
#include "ln_kernels.cuh"
#include "eval_kernels.cuh"

using namespace bsac;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
// A failed call returns B200SAC_ERR_NOMEM when it ran out of memory, B200SAC_ERR_CUDA otherwise.  Its error is taken off
// cudaGetLastError, so that the launch check of a later call does not report it again.
#define CU(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e__ = (call);                                                                        \
    if (e__ != cudaSuccess) {                                                                        \
      cudaGetLastError();                                                                            \
      return fail(e__ == cudaErrorMemoryAllocation ? B200SAC_ERR_NOMEM : B200SAC_ERR_CUDA, "%s failed: %s (%s:%d)", #call, \
                  cudaGetErrorString(e__), __FILE__, __LINE__);                                      \
    }                                                                                                \
  } while (0)

extern "C" const char* b200sac_last_error(void) { return g_err; }
extern "C" const char* b200sac_version(void) { return "b200sac 0.1 (sm_90a)"; }

// Sole owner of one CUDA resource (memory, event, stream, graph): released by Release when the owner is destroyed or
// reset, and nowhere else.  put() hands the empty slot to the allocating call, e.g. CU(cudaMallocHost(buf.put(), bytes)).
template <class H, auto Release>
class Own {
 public:
  Own() = default;
  Own(Own&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Own& operator=(Own&& o) noexcept {
    if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); }
    return *this;
  }
  ~Own() { reset(); }
  H get() const { return h_; }
  operator H() const { return h_; }
  H* put() { reset(); return &h_; }
  void reset() { if (h_) Release(std::exchange(h_, nullptr)); }
 private:
  H h_ = nullptr;
};
template <class T> using DevMem = Own<T*, cudaFree>;
template <class T> using PinnedMem = Own<T*, cudaFreeHost>;
using Event = Own<cudaEvent_t, cudaEventDestroy>;
using Stream = Own<cudaStream_t, cudaStreamDestroy>;
using Graph = Own<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Own<cudaGraphExec_t, cudaGraphExecDestroy>;

// New device buffers, events and streams for the owners above.  Each returns the first failing CUDA call's error, so that
// a caller wraps it in CU like any CUDA call: CU(dev_fill(buf, n, 0.f)).
// n elements of T, uninitialised: scratch that is written before it is read
template <class T> cudaError_t dev_alloc(DevMem<T>& m, size_t n) { return cudaMalloc(m.put(), n * sizeof(T)); }
// n elements of T copied from the host array src
template <class T> cudaError_t dev_copy(DevMem<T>& m, const T* src, size_t n) {
  cudaError_t e = dev_alloc(m, n);
  return e != cudaSuccess ? e : cudaMemcpy(m, src, n * sizeof(T), cudaMemcpyHostToDevice);
}
// n elements of T, each v (T comes from m alone, so that v may be written 0, -1 or NAN): a value whose bytes are all equal
// (0, -1, an all-ones NaN) is set by cudaMemset, any other is copied from the host
template <class T> cudaError_t dev_fill(DevMem<T>& m, size_t n, std::common_type_t<T> v) {
  unsigned char b[sizeof(T)];
  memcpy(b, &v, sizeof(T));
  if (std::all_of(b, b + sizeof(T), [&](unsigned char x) { return x == b[0]; })) {
    cudaError_t e = dev_alloc(m, n);
    return e != cudaSuccess ? e : cudaMemset(m, b[0], n * sizeof(T));
  }
  const std::vector<T> host(n, v);
  return dev_copy(m, host.data(), n);
}
static cudaError_t new_event(Event& e) { return cudaEventCreateWithFlags(e.put(), cudaEventDisableTiming); }
static cudaError_t new_stream(Stream& s) { return cudaStreamCreateWithFlags(s.put(), cudaStreamNonBlocking); }

// ------------------------------------------------------------------------------------------
// layout
// ------------------------------------------------------------------------------------------
// ld = row pitch of the weight matrix (>= in); g, c = the LayerNorm weight and bias after a critic_ln critic's hidden
// Linear, -1 where there is none
struct LayerOff { int64_t w, b; int in, out; int ld; int64_t g = -1, c = -1; };
struct Layout {
  std::vector<b200sac_tensor_desc> descs;
  std::vector<LayerOff> actor, q[kMaxEns], qt[kMaxEns];   // critics q1 .. qE and their targets (E = 2 on twin handles)
  // CARE: the critic's state encoder (the target's sits at + target_delta with the same relative layout)
  std::vector<LayerOff> mix, trunk, ctx;      // mix: w = [K][out][in], b = [K][out]
  std::vector<LayerOff> cenc;                 // CARE(O): the trainable context encoder (header + mlp), no target copy
  int64_t cse_begin = 0, off_emb = 0, cenc_begin = 0, cenc_n = 0;
  int in_w = 0;                               // width of the state part of the MLP inputs
  int64_t off_alpha = 0, arena = 0, trainable = 0;
  int64_t actor_begin = 0, actor_n = 0, critic_begin = 0, critic_n = 0, target_delta = 0;
};

static int64_t pad4(int64_t x) { return (x + 3) & ~int64_t(3); }

static int check_cfg(const b200sac_cfg* c) {
  if (!c) return fail(B200SAC_ERR_INVALID, "cfg is NULL");
  if (c->state_dim < 1 || c->act_dim < 1 || c->act_dim > kMaxAct)
    return fail(B200SAC_ERR_INVALID, "state_dim >= 1 and 1 <= act_dim <= %d required", kMaxAct);
  if (c->num_tasks < 0 || c->num_tasks > 64) return fail(B200SAC_ERR_INVALID, "0 <= num_tasks <= 64 required");
  if (c->n_actor_hidden < 1 || c->n_actor_hidden > B200SAC_MAX_HIDDEN || c->n_critic_hidden < 1 ||
      c->n_critic_hidden > B200SAC_MAX_HIDDEN)
    return fail(B200SAC_ERR_INVALID, "1..%d hidden layers required", B200SAC_MAX_HIDDEN);
  for (int i = 0; i < c->n_actor_hidden; ++i)
    if (c->actor_hidden[i] < 1) return fail(B200SAC_ERR_INVALID, "actor_hidden[%d] < 1", i);
  for (int i = 0; i < c->n_critic_hidden; ++i)
    if (c->critic_hidden[i] < 1) return fail(B200SAC_ERR_INVALID, "critic_hidden[%d] < 1", i);
  if (c->batch < 1 || c->batch > 2048) return fail(B200SAC_ERR_INVALID, "1 <= batch <= 2048 required");
  if (c->num_tasks > 0 && c->batch % c->num_tasks != 0)
    return fail(B200SAC_ERR_INVALID, "batch must be a multiple of num_tasks");
  if (c->replicas < 1 || c->replicas > 4096) return fail(B200SAC_ERR_INVALID, "1 <= replicas <= 4096 required");
  if (c->precision != 0 && c->precision != 1) return fail(B200SAC_ERR_INVALID, "precision must be 0 (fp32 FFMA) or 1 (3xTF32 wgmma)");
  if (c->care != 0 && c->care != 1 && c->care != 2) return fail(B200SAC_ERR_INVALID, "care must be 0, 1 (CARE(M)) or 2 (CARE(O))");
  if (c->grad_clip != 0 && c->grad_clip != 1) return fail(B200SAC_ERR_INVALID, "grad_clip must be 0 or 1");
  if (c->pcgrad != 0 && c->pcgrad != 1) return fail(B200SAC_ERR_INVALID, "pcgrad must be 0 or 1");
  if (c->pcgrad && (c->num_tasks < 2 || c->grad_clip != 0))
    return fail(B200SAC_ERR_INVALID, "pcgrad needs num_tasks >= 2 and no grad_clip");
  if (c->critic_ln != 0 && c->critic_ln != 1) return fail(B200SAC_ERR_INVALID, "critic_ln must be 0 or 1");
  if (c->critic_ln && (c->care || c->pcgrad))
    return fail(B200SAC_ERR_INVALID, "critic_ln is for the plain-MLP critics without gradient surgery (care = 0, pcgrad = 0)");
  if (c->critic_dropout != 0 && c->critic_dropout != 1) return fail(B200SAC_ERR_INVALID, "critic_dropout must be 0 or 1");
  if (c->critic_dropout && !c->critic_ln)
    return fail(B200SAC_ERR_INVALID, "critic_dropout needs critic_ln = 1 (the dropout sits before each critic LayerNorm)");
  if (c->critic_ensemble != 0 && (c->critic_ensemble < 2 || c->critic_ensemble > B200SAC_MAX_ENSEMBLE))
    return fail(B200SAC_ERR_INVALID, "critic_ensemble must be 0 or in [2, %d], got %d", B200SAC_MAX_ENSEMBLE, c->critic_ensemble);
  if (c->critic_ensemble && (c->care || c->pcgrad))
    return fail(B200SAC_ERR_INVALID, "critic_ensemble is for the plain-MLP critics without gradient surgery (care = 0, pcgrad = 0)");
  if (c->care == 2) {
    if (c->emb_dim < 1 || c->emb_dim > 256) return fail(B200SAC_ERR_INVALID, "1 <= emb_dim <= 256 required for CARE(O)");
    if (c->emb_dim != c->ctx_out)
      return fail(B200SAC_ERR_INVALID, "CARE(O): the attention trunk reads the context code, so embedding_dim_contextEnc (%d) must equal output_dim_contextEnc (%d) (state_encoder.py:120-122)", c->emb_dim, c->ctx_out);
    if (c->n_ctx_hidden + 3 > kCareMaxLayers) return fail(B200SAC_ERR_INVALID, "too many context-encoder layers");
  }
  if (c->care) {
    if (c->num_tasks < 1) return fail(B200SAC_ERR_INVALID, "CARE needs num_tasks >= 1 (one-hot task id in the observation)");
    if (c->num_encoders < 1 || c->num_encoders > 32) return fail(B200SAC_ERR_INVALID, "1 <= num_encoders <= 32 required");
    if (c->n_mix_hidden < 1 || c->n_mix_hidden > B200SAC_MAX_HIDDEN || c->n_ctx_hidden < 0 || c->n_ctx_hidden > B200SAC_MAX_HIDDEN)
      return fail(B200SAC_ERR_INVALID, "bad number of encoder hidden layers");
    if (c->mix_out < 1 || c->mix_out > 512 || c->ctx_out < 1 || c->ctx_out > 512 || c->ctx_in < 1 || c->ctx_in > 2048)
      return fail(B200SAC_ERR_INVALID, "encoder widths out of range (mix_out, ctx_out <= 512, ctx_in <= 2048)");
    for (int i = 0; i < c->n_mix_hidden; ++i)
      if (c->mix_hidden[i] < 1 || c->mix_hidden[i] > 512) return fail(B200SAC_ERR_INVALID, "mix_hidden[%d] out of range", i);
    for (int i = 0; i < c->n_ctx_hidden; ++i)
      if (c->ctx_hidden[i] < 1 || c->ctx_hidden[i] > 512) return fail(B200SAC_ERR_INVALID, "ctx_hidden[%d] out of range", i);
    if (c->num_encoders + c->ctx_out > 64 * 8) return fail(B200SAC_ERR_INVALID, "num_encoders + ctx_out too large");
  }
  return 0;
}

static void build_layout(const b200sac_cfg* c, Layout& L) {
  const int obs = c->state_dim + c->num_tasks;
  L.in_w = c->care ? (c->ctx_out + c->mix_out) : obs;
  int64_t off = 0;
  auto add = [&](const char* name, int rows, int cols, int trainable, int opt, int pitch = 0) {
    b200sac_tensor_desc d;
    memset(&d, 0, sizeof(d));
    snprintf(d.name, sizeof(d.name), "%s", name);
    if (pitch < cols) pitch = cols;
    d.offset = off; d.rows = rows; d.cols = cols; d.trainable = trainable; d.opt = opt; d.pitch = pitch;
    L.descs.push_back(d);
    int64_t o = off;
    off = pad4(off + (int64_t)rows * pitch);
    return o;
  };
  char nm[48];
  // ln: a LayerNorm weight and bias (out, 1) right after every hidden layer's bias
  auto add_net = [&](const char* net, std::vector<LayerOff>* v, int in0, const int* hid, int nh, int out, int tr, int opt,
                     bool pad_first = false, bool ln = false) {
    int in = in0;
    for (int i = 0; i <= nh; ++i) {
      int o = (i < nh) ? hid[i] : out;
      LayerOff lo;
      lo.in = in; lo.out = o;
      lo.ld = (i == 0 && pad_first) ? (int)pad4(in) : in;     // first layer: TMA-addressable rows (16-B pitch)
      snprintf(nm, sizeof(nm), "%s.%d.weight", net, i);
      lo.w = add(nm, o, in, tr, opt, lo.ld);
      snprintf(nm, sizeof(nm), "%s.%d.bias", net, i);
      lo.b = add(nm, o, 1, tr, opt);
      if (ln && i < nh) {
        snprintf(nm, sizeof(nm), "%s.%d.ln.weight", net, i);
        lo.g = add(nm, o, 1, tr, opt);
        snprintf(nm, sizeof(nm), "%s.%d.ln.bias", net, i);
        lo.c = add(nm, o, 1, tr, opt);
      }
      if (v) v->push_back(lo);
      in = o;
    }
  };
  // state encoder block: mixture layers ([K][out][in] | [K][out]), attention trunk, context MLP
  auto add_encoder = [&](const char* pre, bool record, int tr, int opt) {
    int in = c->state_dim;
    for (int l = 0; l <= c->n_mix_hidden; ++l) {
      int o = (l < c->n_mix_hidden) ? c->mix_hidden[l] : c->mix_out;
      LayerOff lo;
      lo.in = in; lo.out = o; lo.ld = in;
      snprintf(nm, sizeof(nm), "%s.mix.%d.W", pre, l);
      lo.w = add(nm, c->num_encoders * o, in, tr, opt);
      snprintf(nm, sizeof(nm), "%s.mix.%d.b", pre, l);
      lo.b = add(nm, c->num_encoders * o, 1, tr, opt);
      if (record) L.mix.push_back(lo);
      in = o;
    }
    char pfx[24];
    snprintf(pfx, sizeof(pfx), "%s.trunk", pre);
    add_net(pfx, record ? &L.trunk : nullptr, c->care == 2 ? c->emb_dim : c->ctx_in, c->mix_hidden, c->n_mix_hidden,
            c->num_encoders, tr, opt);
    if (c->care == 1) {          // CARE(M): mlp_context lives inside every state encoder
      snprintf(pfx, sizeof(pfx), "%s.ctx", pre);
      add_net(pfx, record ? &L.ctx : nullptr, c->ctx_in, c->ctx_hidden, c->n_ctx_hidden, c->ctx_out, tr, opt);
    }
  };
  L.actor_begin = off;
  add_net("actor", &L.actor, L.in_w, c->actor_hidden, c->n_actor_hidden, 2 * c->act_dim, 1, 1, true);
  L.actor_n = off - L.actor_begin;
  L.critic_begin = off;
  const bool ln = c->critic_ln != 0;
  add_net("q1", &L.q[0], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 1, 0, true, ln);
  add_net("q2", &L.q[1], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 1, 0, true, ln);
  for (int k = 2; k < c->critic_ensemble; ++k) {
    snprintf(nm, sizeof(nm), "q%d", k + 1);
    const std::string net(nm);
    add_net(net.c_str(), &L.q[k], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 1, 0, true, ln);
  }
  L.cse_begin = off;
  if (c->care) add_encoder("cse", true, 1, 0);
  L.critic_n = off - L.critic_begin;
  L.off_alpha = add("log_alpha", c->num_tasks > 0 ? c->num_tasks : 1, 1, 1, 2);
  if (c->care == 2) {            // context encoder: Linear(ctx_in, 2e) ReLU Linear(2e, e) ReLU + mlp e -> ctx_hidden -> ctx_out
    L.cenc_begin = off;
    int hid[B200SAC_MAX_HIDDEN + 2];
    int nh = 0;
    hid[nh++] = 2 * c->emb_dim;
    hid[nh++] = c->emb_dim;
    for (int i = 0; i < c->n_ctx_hidden; ++i) hid[nh++] = c->ctx_hidden[i];
    add_net("cenc", &L.cenc, c->ctx_in, hid, nh, c->ctx_out, 1, 3);
    L.cenc_n = off - L.cenc_begin;
  }
  L.trainable = off;
  int64_t tb = off;
  add_net("q1_target", &L.qt[0], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 0, -1, true, ln);
  add_net("q2_target", &L.qt[1], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 0, -1, true, ln);
  for (int k = 2; k < c->critic_ensemble; ++k) {
    snprintf(nm, sizeof(nm), "q%d_target", k + 1);
    const std::string net(nm);
    add_net(net.c_str(), &L.qt[k], L.in_w + c->act_dim, c->critic_hidden, c->n_critic_hidden, 1, 0, -1, true, ln);
  }
  if (c->care) add_encoder("tse", false, 0, -1);
  L.target_delta = tb - L.critic_begin;
  if (c->care) L.off_emb = add("embedding", c->num_tasks, c->ctx_in, 0, -1);
  L.arena = off;
}

// How every parameter tensor is initialised, in the order b200sac_create draws them: the one source of the (init kind, tag)
// pairs that create and b200sac_reset both read.  Xavier weights and the CARE mixture's randn tensors take tags 0, 1, ...
// in this order; biases are zero; LayerNorm weights one and their biases zero (no tag); log_alpha is cfg.log_alpha_init; the frozen CARE embedding (part -1, never reset) is
// drawn under seed ^ 0x5EED.  depth: an actor or critic Linear layer's position counted from the network's output (1 = the
// head); 0 for the all-or-nothing parts.
struct InitTensor {
  int64_t off;
  int rows, cols, ld;
  int kind;                 // ResetInit
  int tag;
  int part;                 // B200SAC_RESET_*, -1 = the embedding
  int depth;                // 0 = reset with its part whatever the layer count
  bool target;              // has a target copy at + target_delta (q1, q2, cse)
  uint64_t seed_xor;
};

static std::vector<InitTensor> init_table(const b200sac_cfg* c, const Layout& L) {
  std::vector<InitTensor> v;
  int tag = 0;
  auto linear = [&](const std::vector<LayerOff>& net, int part, bool target) {
    const int n = (int)net.size();
    for (int i = 0; i < n; ++i) {
      const LayerOff& lo = net[i];
      const int depth = part == B200SAC_RESET_ACTOR || part == B200SAC_RESET_CRITIC ? n - i : 0;
      v.push_back({lo.w, lo.out, lo.in, lo.ld, RESET_XAVIER, tag++, part, depth, target, 0});
      v.push_back({lo.b, lo.out, 1, 1, RESET_ZERO, -1, part, depth, target, 0});
      if (lo.g >= 0) {
        v.push_back({lo.g, lo.out, 1, 1, RESET_ONES, -1, part, depth, target, 0});
        v.push_back({lo.c, lo.out, 1, 1, RESET_ZERO, -1, part, depth, target, 0});
      }
    }
  };
  linear(L.actor, B200SAC_RESET_ACTOR, false);
  linear(L.q[0], B200SAC_RESET_CRITIC, true);
  linear(L.q[1], B200SAC_RESET_CRITIC, true);
  for (int k = 2; k < c->critic_ensemble; ++k) linear(L.q[k], B200SAC_RESET_CRITIC, true);
  if (c->care) {
    for (const auto& lo : L.mix) {
      const int rows = c->num_encoders * lo.out;
      v.push_back({lo.w, rows, lo.in, lo.in, RESET_RANDN, tag++, B200SAC_RESET_ENCODER, 0, true, 0});
      v.push_back({lo.b, rows, 1, 1, RESET_RANDN, tag++, B200SAC_RESET_ENCODER, 0, true, 0});
    }
    linear(L.trunk, B200SAC_RESET_ENCODER, true);
    linear(L.ctx, B200SAC_RESET_ENCODER, true);
    linear(L.cenc, B200SAC_RESET_CONTEXT, false);
    v.push_back({L.off_emb, c->num_tasks, c->ctx_in, c->ctx_in, RESET_RANDN, tag++, -1, 0, false, 0x5EEDull});
  }
  v.push_back({L.off_alpha, c->num_tasks > 0 ? c->num_tasks : 1, 1, 1, RESET_CONST, -1, B200SAC_RESET_ALPHA, 0, false, 0});
  return v;
}

extern "C" int b200sac_layout(const b200sac_cfg* cfg, b200sac_tensor_desc* out, int32_t cap, int32_t* n,
                              int64_t* arena_floats, int64_t* trainable_floats) {
  if (int rc = check_cfg(cfg)) return rc;
  Layout L;
  build_layout(cfg, L);
  if (n) *n = (int32_t)L.descs.size();
  if (arena_floats) *arena_floats = L.arena;
  if (trainable_floats) *trainable_floats = L.trainable;
  if (out)
    for (int i = 0; i < (int)L.descs.size() && i < cap; ++i) out[i] = L.descs[i];
  return 0;
}

// ------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------
struct Buf {           // [R][n] fp32 (or int32) slab slice
  float* p = nullptr;
  long long rs = 0;    // replica stride in floats
};

// A plan launch's kernel, chosen by the builder that makes the launch, with its argument block.  The step kernels take
// (StepConst, args), (args, StepConst) or (args); the StepConst is the step's, handed over when the plan runs.
template <class P> struct StepFirst { void (*kern)(StepConst, P); P args; };
template <class P> struct StepLast { void (*kern)(P, StepConst); P args; };
template <class P> struct NoStep { void (*kern)(P); P args; };
// the wgmma GEMM: its problems [R][G] (replica-major) and, on an actor-side launch, replica 0's schedule word
typedef void (*TcKernel)(const TcProb*, const int*, int, int);
struct TcCall { TcKernel kern; const TcProb* probs; const int* sched; int G, sched_stride; };
using KernelCall = std::variant<StepFirst<PolicyDoutArgs>, StepFirst<PolicyHeadArgs>, StepFirst<CriticHeadArgs>,
                                StepFirst<ActorQHeadArgs>, StepFirst<HeadBwdArgs>, StepFirst<AdamArgs>, StepFirst<PcgArgs>,
                                StepFirst<GradNormArgs>, StepFirst<LnArgs>, StepLast<ChainArgs>, StepLast<Chain2Args>,
                                StepLast<WgradArgs>,
                                NoStep<CareTabArgs>, NoStep<CareMixArgs>, NoStep<CareMixFwdArgs>, NoStep<CareMixBwdArgs>,
                                NoStep<CareTabReduceArgs>, NoStep<CareTabWgradArgs>, NoStep<GemmGroup>, TcCall>;
template <class P> static KernelCall bind(void (*kern)(StepConst, P), const P& args) { return StepFirst<P>{kern, args}; }
template <class P> static KernelCall bind(void (*kern)(P, StepConst), const P& args) { return StepLast<P>{kern, args}; }
template <class P> static KernelCall bind(void (*kern)(P), const P& args) { return NoStep<P>{kern, args}; }
static KernelCall bind(TcKernel kern, const TcProb* probs, const int* sched, int G, int sched_stride) {
  return TcCall{kern, probs, sched, G, sched_stride};
}

struct Launch {
  // What b200sac_profile_step calls the launch, set by the builder that makes it.  The part before '(' and the "wgmma"
  // substring are what bench.py groups kernels by.
  std::string label;
  dim3 grid, block;
  size_t smem = 0;
  int cluster_y = 1;     // > 1: thread-block clusters of (1, cluster_y, 1)
  int branch = 0;        // 1: may run on the fork stream, concurrently with the launches that follow it on the main stream
  bool join = false;     // the main stream waits for the fork stream before this launch
  bool critic_loss = false;   // its rows carry the step's TD target and pre-update critic values (the PER priority update follows)
  KernelCall call;
};

struct b200sac_replay;

// What a step graph reads: the ring it samples (null: a step from rows already in `rows`), its rows buffer (a staging slot,
// b200sac_step's buffer or the ring's rows), the injected noise (null: drawn in the step; the handle's eps buffer: already
// in place), the steps it runs, and whether it was captured for the in-graph timeline (unforked).  Every pointer belongs to the handle or to a live ring, so the set of
// keys is bounded; a ring's graphs go with it (drop_ring_graphs).
struct GraphKey {
  b200sac_replay* ring;
  const float* rows;
  const float* eps;
  int nsteps;
  bool stamping;
  bool operator<(const GraphKey& o) const {
    return std::tie(ring, rows, eps, nsteps, stamping) < std::tie(o.ring, o.rows, o.eps, o.nsteps, o.stamping);
  }
};

// The environment switches that select a plan path or tile for tests and measurement scripts (none is needed in
// production).  env_switches() is the library's only reader of the environment: b200sac_create calls it once and the
// handle keeps the result, so a handle launches what it chose when it was built; the wgmma GEMM test entry points call
// it per call.
struct EnvSwitches {
  bool fuse = true;          // B200SAC_FUSE=0: the per-layer plan even where the layer-chained one is eligible
  int tc_bn = 0;             // B200SAC_TC_BN: every wgmma launch takes this tile width (128 or 160; any other value 64); 0: unset
  bool pair128 = false;      // B200SAC_TC_PAIR128=1: 128-wide wgmma tiles take the paired flavour
  bool chain_dbg = false;    // B200SAC_CHAIN_DBG set: clock64 timelines of the layer-chained kernels (scripts/chain_timeline.py)
};
static EnvSwitches env_switches() {
  EnvSwitches s;
  if (const char* e = getenv("B200SAC_FUSE")) s.fuse = e[0] != '0';
  if (const char* e = getenv("B200SAC_TC_BN")) { const int b = atoi(e); s.tc_bn = b == 128 ? 128 : (b == 160 ? 160 : 64); }
  if (const char* e = getenv("B200SAC_TC_PAIR128")) s.pair128 = e[0] == '1';
  s.chain_dbg = getenv("B200SAC_CHAIN_DBG") != nullptr;
  return s;
}

// A per-replica setting that may change between steps: a device table [R][N] of T that the step kernels read through a
// pointer captured in the graphs, and its host mirror [R][N] of the values as given (Mirror: the hyperparameters keep the
// caller's b200sac_hparams, the device gets hparams_row).  set() writes one row with a one-thread kernel in stream order
// (bridged off the legacy default stream like a step), so graphs already instantiated read the new value at their next
// launch, and updates the mirror once the write is enqueued, so a getter does not synchronise.
template <class T, int N> struct TableRow { T v[N]; };
template <class T, int N> __global__ void write_row_kernel(T* t, int r, TableRow<T, N> row) {
  for (int i = 0; i < N; ++i) t[r * N + i] = row.v[i];
}

template <class T, int N = 1, class Mirror = T>
struct ReplicaTable {
  DevMem<T> dev;
  std::vector<Mirror> host;
  // every replica's row <- v[0, N); all or nothing (a failed call leaves the table as it was)
  int init(int R, const Mirror* v);
  int check(int replica) const {
    if (replica < 0 || (size_t)replica >= host.size() / N) return fail(B200SAC_ERR_INVALID, "replica %d out of range", replica);
    return 0;
  }
  const Mirror* row(int replica) const { return host.data() + (size_t)replica * N; }
  // row `replica` <- v[0, N) behind the work on `stream`; `written` (if given) is recorded right after the write
  int set(b200sac* h, void* stream, int replica, const Mirror* v, cudaEvent_t written = nullptr);
};

// The twin critics are evaluated on three sets of rows per step, each a pass with its own buffers; the index of a pass is
// its Philox pass index (dropout masks).  Q: the local critics on (s, a) for the critic update (phase A, backward in C);
// T: the target critics on (s', a') for the TD target (phase B); P: the updated local critics on (s, a~) for the actor
// loss (phase D, forward and backward).  Every [2][B] / [2][B][H] buffer holds q1's rows, then q2's; on a critic_ensemble
// handle [E][B] / [E][B][H], the rows of q1 .. qE.
enum { PASS_Q = 0, PASS_T = 1, PASS_P = 2 };
struct CriticPass {
  const std::vector<LayerOff>* net;   // [2]: the networks the pass runs (L.q or L.qt)
  const Buf* X;                       // input rows [B][ldx] (XQ, XT, XP)
  const Buf* q;                       // head values [2][B] (q, qt, qp)
  const char* label;                  // in its LayerNorm launches' labels
  char letter;                        // in its debug names (b200sac_debug_read)
  // per critic hidden layer [2][B][H]: the post-ReLU activations; critic_ln: the pre-normalization activations (after the
  // dropout on critic_dropout handles); critic_dropout: the keep-mask bits [2][B][ceil(H / 32)] (uint32 words in float slots)
  std::vector<Buf> h, z, m;
};

// The evaluation scratch of b200sac_critic_values and b200sac_replay_refresh_priorities: one replica's rows, `rows` at a
// time, in an allocation of its own (at most kEvalScratchBytes, made by the first call), so that the step's slab and
// everything the next step reads stay untouched.  Each buffer holds `rows` rows:
//   XQ, XT [ldx]      critic inputs (s | a) and (s' | a')
//   hc[2] [2][Hc]     critic hidden activations, layer l in hc[l % 2]; z [2][Hc] pre-normalization (critic_ln); [E][Hc]
//                     on a critic_ensemble handle, like q and qt
//   ha[2] [Ha]        actor hidden activations, layer l in ha[l % 2]
//   q, qt [2]         q1 / q2 and their targets (row i of q1, then row i of q2)
//   pout [2A], psave [A][kSaveW], act [A], logp, logstd, eps [A]   the policy head's outputs and noise
//   R, d, g, task, idx                                             the refresh's folded rows and ring slots
// plus tmax [T] and tasks [T] for the refresh's per-task bookkeeping.
constexpr size_t kEvalScratchBytes = 64ull << 20;
struct EvalScratch {
  DevMem<float> mem;
  long long rows = 0;
  float *XQ, *XT, *hc[2], *z, *ha[2], *q, *qt, *pout, *psave, *act, *logp, *logstd, *eps, *R, *d, *g;
  int *task, *tasks;
  long long* idx;
  unsigned* tmax;
};

struct b200sac {
  b200sac_cfg cfg;
  EnvSwitches env;                // read at create
  int device = 0;
  Layout L;
  StepConst K;
  int R = 1;
  // arenas
  DevMem<float> params, adam_m, adam_v, grads;
  DevMem<Counters> cnt;
  ReplicaTable<HParams, 1, b200sac_hparams> hp;   // [R] per-replica hyperparameters (K.hp points here)
  ReplicaTable<int, 2> ivl;       // [R][2] update intervals (actor_every, target_every), read by the ingest
  DevMem<float> losses;           // [kLossSlots][R][4]
  long long host_steps = 0;       // steps enqueued so far
  // work slab
  DevMem<float> slab;
  Buf XA, XQ, XT, XP, r, d, tid, eps, pout, psave, act_out, logp, logstd, y, q, dq, lq, dqa, la, qmin, dxP,
      dout_dbg, dact_dbg, qt, qp, alpha;
  bool stamping = false;          // true while b200sac_graph_timeline runs on this handle (one unforked step per graph)
  bool fused = false;             // layer-chained plan (chain.cuh): every hidden width <= 256, exact-fp32 mode, no CARE
  PolicyHeadArgs pol;             // the policy head's arguments (also used by b200sac_act)
  // CARE
  Buf XS, careTab[3], careDtab, careDatt, mixZ[3], mixDZ;     // instances: 0 = critic's (old) on [s';s], 1 = target's on s', 2 = critic's (new) on s
  std::vector<Buf> mixH[3], mixDH;                             // per mixture hidden layer: [K][rows][pitch]
  CareNet care_trunk, care_ctx;
  int care_row_w = 0, care_off_att = 0, care_off_ctx = 0;
  std::vector<Buf> hA, dhA;       // per actor hidden layer
  CriticPass pass[3] = {{L.q, &XQ, &q, "critic", 'Q'}, {L.qt, &XT, &qt, "target", 'T'}, {L.q, &XP, &qp, "actor pass", 'P'}};
  std::vector<Buf> dhQ;           // per critic hidden layer [2][B][H]: the critic backward's gradients (passes Q and P)
  // cfg.critic_ln: the backward normalization's chunk column sums [R][2][chunks][2][max H] and tickets [R][2]
  DevMem<double> ln_part;
  DevMem<unsigned> ln_ticket;
  // cfg.critic_dropout: [R] dropout rates p (host mirror) and their DropRate
  ReplicaTable<DropRate, 1, double> drop;
  // critics per pass: cfg.critic_ensemble, or 2 (the twins).  [R][2] (target subset size m, actor reduction 1 = mean /
  // 0 = min; the twins' is fixed at (2, min)) and the last step's subset [R][E] as 0 / 1 (debug_read "tsub" on ensemble
  // handles)
  int E = 2;
  ReplicaTable<int, 2> ens;
  Buf tsub;
  std::vector<Launch> plan;
  // what the plan's launches read through their argument blocks: each wgmma launch's problems, each layer-chained launch's
  // tensor maps
  std::vector<DevMem<TcProb>> tprobs;
  std::vector<DevMem<CUtensorMap>> tmaps;
  IngestOut ing;
  // split-K weight gradients: slices 1..gslices-1 of the gradient arena, [slice-1][R][trainable] (slice 0 = grads)
  DevMem<float> grads_x;
  int gslices = 1;
  unsigned long long act_calls = 0;     // b200sac_act invocations (noise stream selector)
  // graphs
  std::map<GraphKey, GraphExec> graphs;
  // host staging for step_host / pinned replay
  PinnedMem<float> stage_h[2];
  DevMem<float> stage_d[2];
  size_t stage_floats = 0;
  int row_w = 0, row_stride = 0;
  Stream side;
  Stream fork;                    // capture-time fork for the next step's index sampling (multi-step graphs)
  Event ev_ingested, ev_sampled, ev_fork_src, ev_fork_done;
  Stream own;                     // used when the caller hands us the legacy default stream (not capturable)
  Event ev_in, ev_out;
  Event ev_copied[2], ev_consumed[2];
  int stage_slot = 0;
  bool stage_used[2] = {false, false};
  int prefetch_slot = -1;         // host-ring step_sampled: minibatch already drawn, gathered and in flight (H2D)
  b200sac_replay* prefetch_rb = nullptr;
  // blob publication (b200sac_blob_*): the published byte string is assembled ON THE DEVICE (constant bytes + float payloads
  // gathered from the arena by a kernel) and crosses PCIe as one copy on its own stream; the host never touches individual
  // tensors.  Two image slots: the caller may hand on blob k while blob k+1 (begun after the next step was enqueued) is
  // still landing
  Stream pub;
  DevMem<uint8_t> blob_d[2];
  PinnedMem<uint8_t> blob_h[2];
  DevMem<int> blob_src;                   // [blob_nf] arena index of payload float j
  DevMem<int> blob_dst;                   // [blob_nf] byte offset of payload float j inside the image
  int64_t blob_bytes = 0, blob_nf = 0;
  int blob_replica = 0, blob_head = 0, blob_pending = 0;
  Event ev_blob_snap[2], ev_blob_done[2];
  DevMem<long long> chain_dbg;    // env.chain_dbg: [plan launches][CH_DBG_SLOTS] clock64 timelines of the chain kernels
  DevMem<float> step_d;           // b200sac_step: the caller's minibatch as packed rows [R][B][row_stride] (stable graph pointers)
  PinnedMem<float> loss_h;        // mapped pinned loss ring [kLossSlots][R][4], written by the tail kernels
  float* loss_h_dev = nullptr;    // its device-side address
  // prioritized replay (allocated with the first prioritized ring): [3][R][B] importance weights of the step, leaf values
  // the step wrote, its ring indices (int32); a forked stream for the priority update
  DevMem<float> per_buf;
  Stream per_fork;
  Event ev_per_src, ev_per_done;
  // n-step returns (allocated with the first linked ring): [3][R][B] per-row discount of the step (K.disc), hops folded and
  // ring indices (int32), written by ingest_nstep_kernel
  DevMem<float> ns_buf;
  // gradient-norm clipping (cfg.grad_clip): [R][3] thresholds (critic, actor, context encoder), the step's clip
  // coefficients, the mapped pinned norm ring [kLossSlots][R][3], and the norm launches' partial sums
  // [3][R][kGradNormMaxBlocks] and tickets [3][R]
  ReplicaTable<double, kClipCols> clip_thr;
  DevMem<float> clip_coef;
  PinnedMem<float> gnorm_h;
  float* gnorm_h_dev = nullptr;
  DevMem<double> gn_part;
  DevMem<unsigned> gn_ticket;
  // dormant-neuron recycling (b200sac_redo): the last call's record per replica, [R][redo_n] neuron scores (NaN until a
  // call writes them) and dormant flags, redo_n = the hidden neurons of the actor, q1 and q2
  DevMem<double> redo_score;
  DevMem<uint8_t> redo_flag;
  int64_t redo_n = 0;
  // gradient surgery (cfg.pcgrad): [R][2] switches (critic, actor), the pcgrad launches' partial products
  // [2][R][kGradNormMaxBlocks][T(T+1)/2] and tickets [2][R], the last step's record per replica and optimizer
  // (G [R][2][T][T], w [R][2][T] -- also what Adam reads --, permutations [R][2][T][T], projection masks [R][2][T]) and
  // the rows of the last step whose task id was not i / P [R]
  ReplicaTable<int, 2> pc_on;
  DevMem<double> pc_part;
  DevMem<unsigned> pc_ticket;
  DevMem<double> pc_G;
  DevMem<float> pc_w;
  DevMem<int> pc_perm;
  DevMem<unsigned long long> pc_mask;
  DevMem<int> pc_bad;
  // CAGrad on the same handles: [R][2] coefficients c (0 = off) and the last step's solve per replica and optimizer
  // (p* [R][2][T], lambda / best F / first F / s [R][2][kCagScalars], ibest [R][2])
  ReplicaTable<double, 2> cg_c;
  DevMem<double> cg_p, cg_f;
  DevMem<int> cg_it;
  EvalScratch ev;                 // b200sac_critic_values / b200sac_replay_refresh_priorities (allocated by the first call)
  // prior-data rings (allocated with the first attach): [R][B] the encoded indices the last mixed gather read, and whether
  // the last sampled step from a device ring was a mixed one (debug_read "idx")
  DevMem<int> mix_idx;
  bool idx_mixed = false;

  // The members release their resources; the publication stream's last copy lands first.
  ~b200sac() {
    cudaSetDevice(device);
    if (pub) cudaStreamSynchronize(pub);
  }
};

// The argument checks the entry points share, each with its one error text.
static int check_replica(const b200sac* h, int replica) {
  if (replica < 0 || replica >= h->R) return fail(B200SAC_ERR_INVALID, "replica %d out of range", replica);
  return 0;
}
// on: the handle's cfg flag of the feature called `name`
static int need_feature(int on, const char* name) {
  if (!on) return fail(B200SAC_ERR_STATE, "the handle was created without %s", name);
  return 0;
}

struct b200sac_replay {
  b200sac* h = nullptr;
  int where = 0;
  long long cap = 0, cap_per_task = 0;
  int Teff = 1;
  float* rows = nullptr;          // [R][cap][row_stride]: rows_dev (device ring) or rows_pinned (pinned-host ring)
  DevMem<float> rows_dev;
  PinnedMem<float> rows_pinned;
  long long rs_rows = 0;
  std::vector<long long> fill, head;   // [R][Teff]
  DevMem<long long> d_fill;       // device copy (device ring)
  DevMem<int> d_idx;              // [R][B]
  unsigned long long seed = 0;
  std::mt19937_64 rng;
  std::mutex mu;
  Event ev_gather;                // device ring: recorded after the last enqueued gather (pushes wait for it under `mu`)
  bool gather_pending = false;
  // prioritized ring (per_kernels.cuh): sum-trees, per-replica beta, and what the synchronous calls work with
  bool per = false;
  PerTree tr;                     // (tr.tree and tr.maxp point into tree and maxp)
  DevMem<float> tree, maxp;
  ReplicaTable<double> beta;      // [R]
  std::vector<long long> draws;   // [R] b200sac_replay_sample_prioritized calls so far (its Philox counter)
  Stream st;                      // device ring: push (and prioritized set / get / sample) work, synchronised before those calls return
  DevMem<long long> s_lidx;       // scratch [kPerMaxB]
  DevMem<int> s_idx;              // scratch [kPerMaxB]
  DevMem<float> s_f;              // scratch [kPerMaxB]
  DevMem<float> s_rows;           // scratch [B][row_stride]
  // trajectory links (nstep_kernels.cuh; b200sac_replay_enable_trajectories)
  bool traj = false;
  DevMem<int> d_link;             // [R][cap] sub-ring-local slot of the successor, or -1
  ReplicaTable<int> nstep;        // [R] horizon
  std::vector<int> link_h, pred_h;   // [R][cap] host mirror of link, and its inverse (sub-ring-local slot of the predecessor)
  std::vector<std::unordered_map<int, long long>> tail;      // [R] stream id -> ring index of the stream's open tail
  std::vector<std::unordered_map<long long, int>> tail_at;   // [R] its inverse
  Event ev_nstep;                 // recorded after the last set_nstep (b200sac_replay_fold waits for it)
  DevMem<int> f_at;               // scratch [f_cap] x 2: link changes of one push (ring index, value)
  size_t f_cap = 0;
  DevMem<long long> f_idx;        // fold scratch [kNstepChunk], with f_rows [kNstepChunk][row_stride], f_disc, f_m
  DevMem<float> f_rows, f_disc;
  DevMem<int> f_m;
  // prior-data rings (b200sac_replay_attach_prior): the ring whose rows fill the first prior_rows rows of every task block
  // of this ring's steps, and the ring this one is the prior of; both are changed under both rings' locks
  b200sac_replay* prior = nullptr;
  b200sac_replay* prior_of = nullptr;
  ReplicaTable<int> prior_rows;   // [R] m, read by sample_mixed_kernel (made by the attach)
};

// Transition rows [s | a | r | s' | d], padded to row_stride floats: the format of the replay ring, the staging slots and
// b200sac_step's buffer (ingest_rows_kernel, ingest_nstep_kernel and nstep_fold_kernel read it on the device).  Field k of
// a row is w[k] floats at offset off[k]; a minibatch outside a row is five field arrays [n][w[k]].
enum { ROW_S, ROW_A, ROW_R, ROW_S2, ROW_D, ROW_FIELDS };
struct RowFields { int w[ROW_FIELDS], off[ROW_FIELDS]; };
static RowFields row_fields(const b200sac* h) {
  const int obs = h->K.obs, A = h->K.act;
  return {{obs, A, 1, obs, 1}, {0, obs, obs + A, obs + A + 1, 2 * obs + A + 1}};
}

// transition i of the field arrays f -> one row
static void pack_row(const b200sac* h, float* row, const float* const f[ROW_FIELDS], long long i) {
  const RowFields F = row_fields(h);
  for (int k = 0; k < ROW_FIELDS; ++k) memcpy(row + F.off[k], f[k] + i * F.w[k], F.w[k] * sizeof(float));
}

// n consecutive rows -> transitions i0 .. i0 + n - 1 of the field arrays f
static void unpack_rows(const b200sac* h, const float* rows, long long n, float* const f[ROW_FIELDS], long long i0) {
  const RowFields F = row_fields(h);
  for (long long i = 0; i < n; ++i)
    for (int k = 0; k < ROW_FIELDS; ++k)
      memcpy(f[k] + (i0 + i) * F.w[k], rows + i * h->row_stride + F.off[k], F.w[k] * sizeof(float));
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// The work slab: every [R][n] buffer of a step in one allocation.  request() gives a buffer its replica stride (n rounded up
// to 64 floats) and the next place in the slab; allocate() makes the slab, zeroed, and points every requested buffer into
// it.  The order of the requests fixes every buffer's offset, and with it the 16-byte alignment that the plan builder tests
// when it picks a GEMM engine or a tensor-mapped operand.
struct SlabCarver {
  int R;
  size_t floats = 0;
  std::vector<std::pair<Buf*, size_t>> at;     // requested buffer, its offset in floats
  void request(Buf& b, size_t n_per_rep) {
    b.rs = (long long)align_up(n_per_rep, 64);
    at.emplace_back(&b, floats);
    floats += (size_t)b.rs * R;
  }
  int allocate(DevMem<float>& slab) {
    CU(dev_fill(slab, floats, 0.f));
    for (auto& [b, off] : at) b->p = slab + off;
    return 0;
  }
};

// ---- TMA tensor maps (driver entry point resolved at run time: no link-time libcuda dependency) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D fp32 row-major [outer][inner] (pitch in floats), box {box_inner floats, box_outer rows}, zero OOB fill;
// SWIZZLE_128B (box_inner = 32: 128-B rows) unless dense
static int make_map(CUtensorMap* tm, const float* ptr, long long inner, long long outer, long long pitch, int box_outer,
                    bool dense = false, int box_inner = 32) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return fail(B200SAC_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   dense ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(B200SAC_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%lld outer=%lld pitch=%lld", (int)r, inner, outer, pitch);
  return 0;
}

// Streaming multiprocessors of the current device: one tensor-core GEMM tile or chained-layer CTA per SM is a "wave".
static int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
  return n;
}

static bool tc_eligible(const GemmProb& p) {
  auto al16 = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if (p.lda % 4 || p.ldb % 4 || !al16(p.A) || !al16(p.B) || (p.rsA % 4) || (p.rsB % 4)) return false;
  return p.M >= 32 && p.N >= 32 && p.K >= 32;
}

// Tile variants of the wgmma GEMM (gemm_tc.cuh): 128x64, 128x128 (EnvSwitches::pair128: the paired flavour), 128x160.
// A step plan binds the chosen instantiation to its launches.
static TcKernel tc_kernel(int bn, bool pair128) {
  if (bn == 160) return gemm_tc_kernel<160, false>;
  if (bn == 128) return pair128 ? (TcKernel)gemm_tc_kernel<128, true> : (TcKernel)gemm_tc_kernel<128, false>;
  return gemm_tc_kernel<64, false>;
}
static size_t tc_smem(int bn) {
  return bn == 160 ? TcCfg<160>::kSmemBytes : (bn == 128 ? TcCfg<128>::kSmemBytes : TcCfg<64>::kSmemBytes);
}
// Lets `kern` launch with `smem` bytes of dynamic shared memory.  The limit is one per kernel and device for the whole
// process, and every handle's plan launches the same kernels, so it is only ever raised.
static cudaError_t allow_smem(const void* kern, size_t smem) {
  if (smem == 0) return cudaSuccess;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, kern);
  if (e == cudaSuccess && (size_t)a.maxDynamicSharedSizeBytes < smem)
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  return e;
}
// Modelled cycles of one launch group with `bn`-wide tiles (constants from scripts/tc_timeline.py on an H100 SXM, 400 W
// power limit): a tile costs a ~3k-cycle prologue, 1.2k + 11.7 bn cycles per 32-wide k chunk (1.9k / 2.65k / 3.05k at
// bn = 64 / 128 / 160; 3.1k for the paired 128-wide tile) and an epilogue of ~38 bn cycles; tiles beyond one per SM wait for a second wave.  The plan
// builder takes the cheapest width.
static double tc_group_cost(const std::vector<GemmProb>& v, int bn, int R, bool pair128) {
  long long tiles = 0;
  int nk = 1;
  for (auto& p : v) {
    tiles += (long long)((p.M + TC_BM - 1) / TC_BM) * ((p.N + bn - 1) / bn);
    nk = std::max(nk, (p.K + TC_BK - 1) / TC_BK);
  }
  const double chunk = (bn == 128 && pair128) ? 3100.0 : 1200.0 + 11.7 * bn;
  const double tile = 3000.0 + nk * chunk + 38.0 * bn;
  const int sms = sm_count();
  const long long waves = (tiles * R + sms - 1) / sms;
  return (double)waves * tile;
}
static int tc_pick_bn(const std::vector<GemmProb>& v, int R, const EnvSwitches& sw) {
  if (sw.tc_bn) return sw.tc_bn;
  int maxN = 0;
  for (auto& p : v) maxN = std::max(maxN, p.N);
  int best = 64;
  double cost = tc_group_cost(v, 64, R, sw.pair128);
  for (int bn : {128, 160}) {
    if (maxN < 2 * bn - 64) continue;             // a lone, mostly empty wide tile is never better than 64-wide ones
    const double c = tc_group_cost(v, bn, R, sw.pair128);
    if (c < cost) { cost = c; best = bn; }
  }
  return best;
}

constexpr int kSplitK = 4, kSplitKMin = 512;     // weight gradients with K >= 512 rows are computed in 4 K slices

static int make_tc_prob(const GemmProb& p, int rep, TcProb& t, int bn = 64) {
  memset(&t, 0, sizeof(t));
  const float* A = p.A + (long long)rep * p.rsA;
  const float* B = p.B + (long long)rep * p.rsB;
  t.M = p.M; t.N = p.N; t.K = p.K; t.mode = p.mode; t.relu = p.relu; t.ldc = p.ldc; t.ldmask = p.ldmask;
  t.bias = p.bias ? p.bias + (long long)rep * p.rsBias : nullptr;
  t.mask = p.mask ? p.mask + (long long)rep * p.rsMask : nullptr;
  t.C = p.C + (long long)rep * p.rsC;
  t.C2 = p.C2 ? p.C2 + (long long)rep * p.rsC2 : nullptr;
  // K-major operands: box {32 k, rows}, SWIZZLE_128B (the wgmma K-major layout); MN-major ones: box {rows, 32 k}, unswizzled
  if (p.mode == GEMM_FWD) {            // A[M][K], B[N][K]: both K-major
    t.a_mn = 0; t.b_mn = 0;
    if (int rc = make_map(&t.tmA, A, p.K, p.M, p.lda, TC_BM)) return rc;
    if (int rc = make_map(&t.tmB, B, p.K, p.N, p.ldb, bn)) return rc;
  } else if (p.mode == GEMM_DGRAD) {   // A = dY[M][K] K-major, B = W[K][N] MN-major
    t.a_mn = 0; t.b_mn = 1;
    if (int rc = make_map(&t.tmA, A, p.K, p.M, p.lda, TC_BM)) return rc;
    if (int rc = make_map(&t.tmB, B, p.N, p.K, p.ldb, TC_BK, true, bn)) return rc;
  } else {                             // WGRAD: A = dY[K][M], B = X[K][N]: both MN-major
    t.a_mn = 1; t.b_mn = 1;
    if (int rc = make_map(&t.tmA, A, p.M, p.K, p.lda, TC_BK, true, TC_BM)) return rc;
    if (int rc = make_map(&t.tmB, B, p.N, p.K, p.ldb, TC_BK, true, bn)) return rc;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// Layer-chained plan (chain.cuh, chain2.cuh): 7 launches per step after the ingest, whatever the depth of the networks.
//   A   chain_kernel<FWD>  {actor on [s';s], Q1, Q2 on (s,a)}  -> policy head / scalar heads
//   BC  chain2_kernel      {Qt1, Qt2 on (s',a')} -> y, dQ -> input-gradient chain of {Q1, Q2}   -> wgrad + Adam + Polyak
//   D   chain2_kernel      {Q1, Q2 on (s,a~)} with the updated critics -> min routing -> input-gradient chain down to d(action)
//                          (forked beside E: actor loss, entropy, temperature gradient + its Adam)
//   E   chain_kernel<BWD>  {actor}: d(mu|log_std), input-gradient chain                          -> wgrad + Adam
// Eligible: exact-fp32 mode, no CARE, every hidden width a multiple of 4 and <= 256, obs+act <= 252.
// ------------------------------------------------------------------------------------------
static bool fused_eligible(const b200sac* h) {
  const b200sac_cfg& c = h->cfg;
  if (c.precision != 0 || c.care || c.pcgrad || c.critic_ln || c.critic_ensemble || !h->env.fuse) return false;
  for (int i = 0; i < c.n_actor_hidden; ++i) if (c.actor_hidden[i] % 4 || c.actor_hidden[i] > CH_MAXW) return false;
  for (int i = 0; i < c.n_critic_hidden; ++i) if (c.critic_hidden[i] % 4 || c.critic_hidden[i] > CH_MAXW) return false;
  if (c.state_dim + c.num_tasks + c.act_dim > CH_MAXW - 4) return false;
  return true;
}

// Rows per CTA (8, 4 or 2) of a chain launch of `groups` x ceil(rows / ROWS) CTAs per replica.  Every CTA streams the whole
// weight matrices whatever its row count, so fewer rows per CTA only pay while the launch still fits the GPU: the fewest
// rows whose launch stays within one wave (one CTA per SM).
static int chain_rows(long long rows, int groups, int R, int sms) {
  int bn = 8;
  for (int r = 4; r >= 2; r >>= 1)
    if (groups * ((rows + r - 1) / r) * R <= sms) bn = r;
  return bn;
}

// f(std::integral_constant<int, ROWS>) for the rows per CTA of a chain launch
template <typename F>
static auto with_chain_rows(int bn, F&& f) {
  if (bn == 8) return f(std::integral_constant<int, 8>{});
  if (bn == 4) return f(std::integral_constant<int, 4>{});
  return f(std::integral_constant<int, 2>{});
}

// ------------------------------------------------------------------------------------------
// Launch descriptions shared by the step plan and batched inference (b200sac_act).  The plan describes every replica at
// once (an operand and its replica stride); inference describes one replica: its base pointers and stride 0.
// ------------------------------------------------------------------------------------------
// the whole buffer (rep < 0) or replica rep of it alone
static Buf rep_view(const Buf& b, int rep) { return rep < 0 ? b : Buf{b.p + (long long)rep * b.rs, 0}; }
static int pitch(int w) { return (w + 3) & ~3; }   // row pitch of the CARE work buffers

// forward of one layer over M rows: out = relu(X W^T + b), W and b from the parameter arena `par`
static GemmProb fwd_prob(const Buf& par, const float* X, long long rsX, int M, const LayerOff& lo, float* out, long long rsOut) {
  GemmProb p;
  memset(&p, 0, sizeof(p));
  p.A = X; p.rsA = rsX; p.lda = lo.ld;
  p.B = par.p + lo.w; p.rsB = par.rs; p.ldb = lo.ld;
  p.bias = par.p + lo.b; p.rsBias = par.rs;
  p.C = out; p.rsC = rsOut; p.ldc = lo.out;
  p.M = M; p.N = lo.out; p.K = lo.in; p.mode = GEMM_FWD; p.relu = 1;
  return p;
}
// weight and bias gradient of one layer over K rows into the gradient arena `grd`: dW = dZ^T X, db = column sums of dZ
static GemmProb wgrad_prob(const Buf& grd, const float* dZ, long long rsdZ, const float* X, long long rsX, const LayerOff& lo, int K) {
  GemmProb p;
  memset(&p, 0, sizeof(p));
  p.A = dZ; p.rsA = rsdZ; p.lda = lo.out;
  p.B = X; p.rsB = rsX; p.ldb = lo.ld;
  p.C = grd.p + lo.w; p.rsC = grd.rs; p.ldc = lo.ld;
  p.C2 = grd.p + lo.b; p.rsC2 = grd.rs;
  p.M = lo.out; p.N = lo.in; p.K = K; p.mode = GEMM_WGRAD;
  return p;
}
// input gradient of one layer over M rows: out = (dZ W) * [mask > 0] (no mask: ungated)
static GemmProb dgrad_prob(const Buf& par, const float* dZ, long long rsdZ, const LayerOff& lo, const float* mask, long long rsMask,
                           float* out, long long rsOut, int M) {
  GemmProb p;
  memset(&p, 0, sizeof(p));
  p.A = dZ; p.rsA = rsdZ; p.lda = lo.out;
  p.B = par.p + lo.w; p.rsB = par.rs; p.ldb = lo.ld;
  p.mask = mask; p.rsMask = rsMask; p.ldmask = lo.ld;
  p.C = out; p.rsC = rsOut; p.ldc = lo.ld;
  p.M = M; p.N = lo.in; p.K = lo.out; p.mode = GEMM_DGRAD;
  return p;
}

// CARE encoder instances: 0 = critic's on [s';s] (2B rows), 1 = target's on s', 2 = critic's after its Adam step on s.
// The K problems of mixture layer l of instance `inst` on XS rows [row0, row0 + rows), appended to ps.  Instance 0 keeps
// the rows at the same place in its buffers, the others from row 0.
static void mix_fwd_probs(const b200sac* h, int rep, int inst, int l, int row0, int rows, std::vector<GemmProb>& ps) {
  const Layout& L = h->L;
  const int rows_buf = inst == 0 ? 2 * h->cfg.batch : h->cfg.batch;   // rows held by the instance's buffers
  const int out_row0 = inst == 0 ? row0 : 0;
  const LayerOff& lo = L.mix[l];
  const long long delta = inst == 1 ? L.target_delta : 0;
  const bool last = (l == (int)L.mix.size() - 1);
  const Buf par = rep_view(Buf{h->params, L.arena}, rep), xs = rep_view(h->XS, rep);
  const Buf ob = rep_view(last ? h->mixZ[inst] : h->mixH[inst][l], rep);
  for (int k = 0; k < h->cfg.num_encoders; ++k) {
    GemmProb p;
    memset(&p, 0, sizeof(p));
    if (l == 0) { p.A = xs.p + (long long)row0 * h->K.obs; p.rsA = xs.rs; p.lda = h->K.obs; }
    else {
      const Buf ib = rep_view(h->mixH[inst][l - 1], rep);
      p.A = ib.p + ((long long)k * rows_buf + out_row0) * pitch(lo.in); p.rsA = ib.rs; p.lda = pitch(lo.in);
    }
    p.B = par.p + delta + lo.w + (long long)k * lo.out * lo.in; p.rsB = par.rs; p.ldb = lo.in;
    p.bias = par.p + delta + lo.b + (long long)k * lo.out; p.rsBias = par.rs;
    p.C = ob.p + ((long long)k * rows_buf + out_row0) * pitch(lo.out); p.rsC = ob.rs; p.ldc = pitch(lo.out);
    p.M = rows; p.N = lo.out; p.K = lo.in; p.mode = GEMM_FWD; p.relu = last ? 0 : 1;
    ps.push_back(p);
  }
}

// per-task tables (trunk attention logits, context code) of the encoder instances insts, one per blockIdx.y
static CareTabArgs care_tab_args(const b200sac* h, int rep, const std::vector<int>& insts) {
  const b200sac_cfg& c = h->cfg;
  CareTabArgs P;
  memset(&P, 0, sizeof(P));
  const Buf par = rep_view(Buf{h->params, h->L.arena}, rep);
  P.params = par.p; P.rsP = par.rs; P.emb_off = h->L.off_emb;
  P.trunk = h->care_trunk; P.ctx = h->care_ctx;
  P.T = c.num_tasks; P.K = c.num_encoders; P.row_w = h->care_row_w; P.off_att = h->care_off_att;
  P.original = c.care == 2 ? 1 : 0;
  for (size_t i = 0; i < insts.size(); ++i) {
    P.inst_delta[i] = insts[i] == 1 ? h->L.target_delta : 0;
    P.tab[i] = rep_view(h->careTab[insts[i]], rep).p;
  }
  P.rsTab = rep_view(h->careTab[0], rep).rs;
  return P;
}

// Encoding of `rows` XS rows from xs_row0 by instance `inst`: [mixed state | context code] rows written to d1 and, from
// row off2 of the job on, to d2 (d2.p = nullptr: none).
struct EncJob { int inst, xs_row0, rows; Buf d1; int ld1; Buf d2; int ld2; int off2; };

// attention mix of the instance's K encoder outputs with its task tables
static CareMixArgs care_mix_args(const b200sac* h, int rep, const EncJob& e) {
  const b200sac_cfg& c = h->cfg;
  CareMixArgs P;
  memset(&P, 0, sizeof(P));
  const int rows_buf = e.inst == 0 ? 2 * c.batch : c.batch;
  const Buf Z = rep_view(h->mixZ[e.inst], rep), tab = rep_view(h->careTab[e.inst], rep), tid = rep_view(h->tid, rep);
  P.Z = Z.p; P.rsZ = Z.rs; P.kstride = (long long)rows_buf * pitch(c.mix_out); P.ldz = pitch(c.mix_out);
  P.tab = tab.p; P.rsTab = tab.rs; P.row_w = h->care_row_w; P.off_att = h->care_off_att;
  P.off_ctx = h->care_off_ctx;
  P.tid = (const int*)tid.p; P.rsR = tid.rs;
  P.rows = e.rows; P.B = c.batch; P.K = c.num_encoders; P.mo = c.mix_out; P.co = c.ctx_out;
  P.dst1 = e.d1.p; P.rsD1 = e.d1.rs; P.ld1 = e.ld1; P.dst2 = e.d2.p; P.rsD2 = e.d2.rs; P.ld2 = e.ld2; P.row_off2 = e.off2;
  return P;
}

// ------------------------------------------------------------------------------------------
// Step plan: build_plan sets the policy-head arguments, then build_plan_fused (the layer-chained plan) or
// build_plan_layered (the per-layer plan) appends the launches of one step to h->plan with the launch builders below.
// ------------------------------------------------------------------------------------------
struct PlanBuilder {
  b200sac* h;
  const b200sac_cfg& c;
  const Layout& L;
  const int B, R, A, La, Lc, sms;
  const long long rsP, rsG;
  const Buf par, grd;       // parameter and gradient arenas
  // critics per pass (2: the twins) and the distance from one critic to the next in the parameter and gradient arenas
  // (the critics share one layout and sit back to back)
  const int E;
  const long long rsNet;
  int branch = 0;           // branch tag given to the launches gemm_launch creates
  // per-layer plan, FFMA back-end, plain SAC nets: a layer's weight gradient only feeds Adam, while its input gradient heads
  // the rest of the backward chain.  The weight-gradient launch goes to the fork stream and the chain continues at once (the
  // kernels hold <= 2 CTAs per SM, so both fit); Adam joins.  (tensor-core tiles own a whole SM each: grouping is better there.)
  const bool use_fork;
  bool actor_side = false;  // the launches being built belong to the actor update: skipped on critic-only steps
  int rc = 0;               // error met by a builder that cannot return one; build_plan returns it

  explicit PlanBuilder(b200sac* hh)
      : h(hh), c(hh->cfg), L(hh->L), B(c.batch), R(hh->R), A(c.act_dim), La(c.n_actor_hidden), Lc(c.n_critic_hidden),
        sms(sm_count()), rsP(L.arena), rsG(L.trainable), par{hh->params, L.arena}, grd{hh->grads, L.trainable},
        E(hh->E), rsNet(L.q[1][0].w - L.q[0][0].w), use_fork(c.precision == 0 && !c.care) {}
  float* W(int64_t off) const { return h->params + off; }
  float* Gp(int64_t off) const { return h->grads + off; }
  // network net's rows of a [2][B][H] ([E][B][H]) buffer
  float* netp(const Buf& b, int net, int H) const { return b.p + (long long)net * B * H; }
  // network net's input rows at critic hidden layer l of pass cp: its input rows X, or layer l - 1's activations
  Buf critic_in(const CriticPass& cp, int net, int l) const {
    return l == 0 ? *cp.X : Buf{netp(cp.h[l - 1], net, cp.net[net][l].in), cp.h[l - 1].rs};
  }

  // appends launch l running kern(args), first letting kern take l.smem bytes of dynamic shared memory
  template <class F, class... P> void push(Launch l, F kern, const P&... args) {
    if (cudaError_t e = allow_smem((const void*)kern, l.smem)) {
      cudaGetLastError();
      rc = fail(B200SAC_ERR_CUDA, "%s: dynamic shared memory of %zu bytes refused: %s", l.label.c_str(), l.smem, cudaGetErrorString(e));
    }
    l.call = bind(kern, args...);
    h->plan.push_back(std::move(l));
  }
  // a copy of v on the device, owned by the handle (empty: null)
  template <class T> const T* upload(std::vector<DevMem<T>>& owner, const std::vector<T>& v) {
    if (v.empty()) return nullptr;
    DevMem<T> d;
    if (cudaError_t e = dev_copy(d, v.data(), v.size())) {
      cudaGetLastError();
      rc = fail(e == cudaErrorMemoryAllocation ? B200SAC_ERR_NOMEM : B200SAC_ERR_CUDA, "plan table upload failed: %s", cudaGetErrorString(e));
      return nullptr;
    }
    owner.push_back(std::move(d));
    return owner.back();
  }

  void gemm_launch(const std::vector<GemmProb>& ps_in);
  void care_tables(const std::vector<int>& insts);
  void care_encode(const std::vector<EncJob>& jobs);
  void head_bwd(bool policy, bool want_wgrad);
  void opt_slice(int which, int64_t& beg, int64_t& n) const;
  void adam(int which, bool tail_only, bool with_tail = true);
  void grad_norm(int which);
  void pcgrad(int which);
  void layer_norm(int pass, int l, bool fwd, bool want_grads);
  void critic_fwd(int pass, int l, std::vector<GemmProb> ps = {});
  void critic_bwd(int pass, int l, bool want_wgrad);
  int build_plan_fused();
  void build_plan_layered();
};

// Label of a grouped GEMM launch of the problems g: their kind (a thin launch is named after its first problem alone), the
// engine and wgmma tile (128x64 | 128x128 | 128x128 paired | 128x160) and, when the group holds weight gradients, their K
// slices ("split S")
static std::string gemm_label(const std::vector<GemmProb>& g, const std::string& engine, int split) {
  const GemmProb &p0 = g.front(), &pl = g.back();
  bool wg = false;
  for (auto& p : g) wg = wg || p.mode == GEMM_WGRAD;
  std::string s = p0.mode == GEMM_FWD ? "gemm_fwd(" : p0.mode == GEMM_DGRAD ? "gemm_dgrad(" :
                  (pl.mode == GEMM_DGRAD && engine != "thin") ? "gemm_wgrad+dgrad(" : "gemm_wgrad(";
  s += engine;
  if (wg) s += ", split " + std::to_string(split);
  return s + ")";
}

void PlanBuilder::gemm_launch(const std::vector<GemmProb>& ps_in) {
  // Split-K for the weight gradients: K = batch (1024 / 1280) is the long dimension and M x N = out x in gives only a
  // handful of tiles, so one CTA would walk 32-40 k chunks alone.
  // WGRAD operands are both [K][*] row-major, so a K slice is just a row offset: slice s of a problem becomes its own
  // problem writing gradient slice s; Adam adds the slices in index order (deterministic, no atomics).
  // pcgrad handles: every weight gradient is cut into the T task blocks of B / T rows, slice t = task t's gradient.
  auto sliced = [&](const GemmProb& p) { return p.mode == GEMM_WGRAD && (c.pcgrad || (p.K >= kSplitKMin && h->gslices > 1)); };
  auto expand = [&](int Smax, std::vector<GemmProb>& out) {
    for (auto& p : ps_in) {
      const int S = sliced(p) ? Smax : 1;
      if (S == 1) { out.push_back(p); continue; }
      const int len = c.pcgrad ? p.K / S : (((p.K + S - 1) / S) + 31) & ~31;
      const long long coff = p.C - h->grads, c2off = p.C2 ? p.C2 - h->grads : 0;
      if (coff < 0 || coff >= L.trainable) { rc = fail(B200SAC_ERR_INVALID, "internal: split-K output outside the gradient arena"); out.push_back(p); continue; }
      for (int sidx = 0; sidx < S; ++sidx) {
        const int kb = sidx * len;
        if (kb >= p.K) break;
        GemmProb q = p;
        q.A = p.A + (long long)kb * p.lda; q.B = p.B + (long long)kb * p.ldb;
        q.K = (p.K - kb < len) ? p.K - kb : len;
        if (sidx > 0) {
          float* base = h->grads_x + (long long)(sidx - 1) * R * L.trainable;
          q.C = base + coff;
          if (p.C2) q.C2 = base + c2off;
        }
        out.push_back(q);
      }
    }
  };
  // tensor-core tiles hold one CTA per SM: take the split factor (and with it the tile width) whose launch is cheapest under
  // tc_group_cost's model -- a finer split shortens the k loop but a second wave of CTAs costs a whole tile time; the FFMA
  // engine (several CTAs per SM) always takes the finest.
  auto tc_only = [&](const std::vector<GemmProb>& v) {
    std::vector<GemmProb> o;
    for (auto& p : v) if (tc_eligible(p)) o.push_back(p);
    return o;
  };
  std::vector<GemmProb> ps;
  int split = 1;                        // what expand did to this group's weight gradients (launch labels)
  {
    int S = c.pcgrad ? h->gslices : kSplitK;
    if (c.precision == 1 && !c.pcgrad) {
      double best = 1e300;
      for (int s_ = kSplitK; s_ >= 1; s_ >>= 1) {
        std::vector<GemmProb> trial;
        expand(s_, trial);
        const std::vector<GemmProb> o = tc_only(trial);
        if (o.empty()) { S = s_; break; }
        const double cost = tc_group_cost(o, tc_pick_bn(o, R, h->env), R, h->env.pair128);
        if (cost < best) { best = cost; S = s_; }
      }
    }
    expand(S, ps);
    for (auto& p : ps_in)
      if (sliced(p)) split = S;
  }
  if (c.precision == 1) {
    std::vector<GemmProb> tc, rest;
    for (auto& p : ps) (tc_eligible(p) ? tc : rest).push_back(p);
    if (!tc.empty()) {
      Launch l;
      int maxM = 0, maxN = 0;
      for (auto& p : tc) { maxM = p.M > maxM ? p.M : maxM; maxN = p.N > maxN ? p.N : maxN; }
      const int bn = tc_pick_bn(tc, R, h->env);  // tile width: the cheapest of 64 / 128 / 160 under tc_group_cost's model
      const bool pair128 = bn == 128 && h->env.pair128;
      l.branch = branch;
      l.label = gemm_label(tc, "wgmma 128x" + std::to_string(bn) + (pair128 ? " paired" : ""), split);
      l.grid = dim3((maxN + bn - 1) / bn, (maxM + TC_BM - 1) / TC_BM, (unsigned)(tc.size() * R));
      l.block = dim3(TC_THREADS);
      l.smem = tc_smem(bn);
      std::vector<TcProb> probs;
      for (int rep = 0; rep < R; ++rep)
        for (auto& p : tc) {
          TcProb t;
          if (int e = make_tc_prob(p, rep, t, bn)) rc = e;
          probs.push_back(t);
        }
      push(std::move(l), tc_kernel(bn, pair128), upload(h->tprobs, probs), actor_side ? &h->cnt[0].sched : nullptr,
           (int)tc.size(), kSchedStride);
    }
    ps = rest;
  }
  // More problems than one parameter block holds: one launch per GS_MAXG of them, each labelled as a group of its own
  // whose weight gradients need no further K slicing ("split 1").
  if (ps.size() > GS_MAXG) split = 1;
  for (size_t i0 = 0; i0 < ps.size(); i0 += GS_MAXG) {
    const std::vector<GemmProb> g(ps.begin() + i0, ps.begin() + std::min(ps.size(), i0 + GS_MAXG));
    Launch l;
    int maxM = 0, maxN = 0;
    bool thin = true;
    for (auto& p : g) { maxM = p.M > maxM ? p.M : maxM; maxN = p.N > maxN ? p.N : maxN; thin = thin && gemm_is_thin(p); }
    l.branch = branch;
    l.grid = dim3((maxN + GS_T - 1) / GS_T, (maxM + GS_T - 1) / GS_T, (unsigned)(g.size() * R));
    l.block = dim3(GS_THREADS);
    if (thin) {        // input-layer weight / input gradients (N = obs+act <= 16): gemm_thin.cuh
      int rows = 1;
      for (auto& p : g) {
        const int per = p.mode == GEMM_WGRAD ? GT_ROWS_WGRAD : GT_ROWS_DGRAD, r = (p.M + per - 1) / per;
        rows = r > rows ? r : rows;
      }
      l.grid = dim3(1, rows, (unsigned)(g.size() * R));
      l.block = dim3(GT_THREADS);
    }
    l.label = gemm_label(g, thin ? "thin" : "ffma", split);
    GemmGroup grp;
    memset(&grp, 0, sizeof(grp));
    grp.G = (int)g.size();
    grp.sched = actor_side ? &h->cnt[0].sched : nullptr; grp.sched_stride = kSchedStride;
    for (size_t i = 0; i < g.size(); ++i) grp.p[i] = g[i];
    push(std::move(l), thin ? gemm_thin_kernel : gemm_simt_kernel, grp);
  }
}

void PlanBuilder::care_tables(const std::vector<int>& insts) {
  Launch l;
  l.label = "care_tables";
  CareTabArgs P = care_tab_args(h, -1, insts);
  P.sched = actor_side ? &h->cnt[0].sched : nullptr; P.sched_stride = kSchedStride;
  l.grid = dim3(c.num_tasks, (unsigned)insts.size(), R);
  l.block = dim3(512);
  push(std::move(l), care_tables_kernel, P);
}

// mixture layers + attention mix of up to three encoder instances in ONE launch (care_mixfwd_kernel: all mixture weights of
// an instance resident in shared memory); falls back to grouped GEMMs and care_mix_kernel when the weights do not fit
void PlanBuilder::care_encode(const std::vector<EncJob>& jobs) {
  const int Kenc = c.num_encoders, nmix = (int)L.mix.size();
  CareMixFwdArgs A;
  memset(&A, 0, sizeof(A));
  A.njobs = (int)jobs.size(); A.nl = nmix; A.K = Kenc; A.B = B;
  A.params = h->params; A.rsP = rsP;
  A.XS = h->XS.p; A.rsXS = h->XS.rs; A.ldx = h->K.obs;
  A.tid = (const int*)h->tid.p; A.rsR = h->r.rs;
  A.row_w = h->care_row_w; A.off_att = h->care_off_att; A.off_ctx = h->care_off_ctx; A.mo = c.mix_out; A.co = c.ctx_out;
  A.sched = actor_side ? &h->cnt[0].sched : nullptr; A.sched_stride = kSchedStride;
  bool ok = nmix >= 1 && nmix <= CMF_MAXL && (int)jobs.size() <= CMF_MAXJOBS;
  for (int l = 0; ok && l < nmix; ++l) {
    A.w_off[l] = L.mix[l].w; A.b_off[l] = L.mix[l].b; A.in[l] = L.mix[l].in; A.out[l] = L.mix[l].out;
    A.maxw = std::max(A.maxw, L.mix[l].out);
  }
  int cta = 0;
  for (size_t i = 0; ok && i < jobs.size(); ++i) {
    const EncJob& e = jobs[i];
    CareMixFwdJob& J = A.job[i];
    const int rows_buf = e.inst == 0 ? 2 * B : B;
    J.inst_delta = e.inst == 1 ? L.target_delta : 0;
    J.rows = e.rows; J.xs_row0 = e.xs_row0; J.out_row0 = e.inst == 0 ? e.xs_row0 : 0; J.rows_buf = rows_buf;
    J.cta0 = cta; cta += (e.rows + CMF_ROWS - 1) / CMF_ROWS;
    J.tab = h->careTab[e.inst].p; J.rsTab = h->careTab[e.inst].rs;
    for (int l = 0; l < nmix; ++l) {
      const Buf& ob = (l == nmix - 1) ? h->mixZ[e.inst] : h->mixH[e.inst][l];
      J.H[l] = ob.p; J.rsH[l] = ob.rs;
    }
    J.dst1 = e.d1.p; J.rsD1 = e.d1.rs; J.ld1 = e.ld1; J.dst2 = e.d2.p; J.rsD2 = e.d2.rs; J.ld2 = e.ld2; J.row_off2 = e.off2;
  }
  const size_t smem = ok ? care_mixfwd_smem_floats(A) * sizeof(float) : 0;
  if (ok && smem <= 225 * 1024 && allow_smem((const void*)care_mixfwd_kernel, smem) == cudaSuccess) {
    Launch l;
    l.label = "care_mixture_fwd+mix";
    l.grid = dim3(cta, R);
    l.block = dim3(CMF_THREADS);
    l.smem = smem;
    push(std::move(l), care_mixfwd_kernel, A);
    return;
  }
  for (int l = 0; l < nmix; ++l) {
    std::vector<GemmProb> ps;
    for (const EncJob& e : jobs) mix_fwd_probs(h, -1, e.inst, l, e.xs_row0, e.rows, ps);
    gemm_launch(ps);
  }
  for (const EncJob& e : jobs) {
    Launch l;
    l.label = "care_mix";
    CareMixArgs P = care_mix_args(h, -1, e);
    P.sched = actor_side ? &h->cnt[0].sched : nullptr; P.sched_stride = kSchedStride;
    l.grid = dim3((e.rows + 7) / 8, R);
    l.block = dim3(256);
    push(std::move(l), care_mix_kernel, P);
  }
}

void PlanBuilder::head_bwd(bool policy, bool want_wgrad) {
  const int Hc = c.critic_hidden[Lc - 1], Ha = c.actor_hidden[La - 1];
  Launch l;
  HeadBwdArgs P;
  memset(&P, 0, sizeof(P));
  P.actor_side = (policy || !want_wgrad) ? 1 : 0;       // the actor pass / the policy backward, not the critic update
  P.M = B;
  P.rsP = rsP; P.rsG = rsG; P.rsNet = rsNet; P.E = E;
  if (!policy) {
    P.NO = 1; P.Kdim = Hc; P.nets = E;
    P.W = W(L.q[0][Lc].w);
    P.dW = want_wgrad ? Gp(L.q[0][Lc].w) : nullptr;
    P.db = want_wgrad ? Gp(L.q[0][Lc].b) : nullptr;
    const Buf& hb = h->pass[want_wgrad ? PASS_Q : PASS_P].h[Lc - 1];
    const Buf& dq = want_wgrad ? h->dq : h->dqa;
    P.dout = dq.p; P.rsDoutNet = B; P.rsDoutRep = E * h->y.rs;
    P.h = hb.p; P.rsHnet = (long long)B * Hc; P.rsHrep = hb.rs; P.ldh = Hc;
    P.dh = h->dhQ[Lc - 1].p; P.rsDhNet = (long long)B * Hc; P.rsDhRep = h->dhQ[Lc - 1].rs; P.lddh = Hc;
  } else {
    const bool split = (long long)B * A > 2048;      // large batch: one tiny kernel computes d(mu|log_std) for all rows
    if (split) {
      Launch pl;
      pl.label = "policy_dout";
      PolicyDoutArgs Q;
      memset(&Q, 0, sizeof(Q));
      Q.dx = h->dxP.p; Q.rsDxNet = (long long)B * h->K.ldx; Q.rsDxRep = h->dxP.rs; Q.lddx = h->K.ldx;
      Q.psave = h->psave.p + (long long)B * A * kSaveW; Q.rsSave = h->psave.rs;
      Q.tid = (const int*)h->tid.p; Q.rsR = h->r.rs;
      Q.log_alpha = W(L.off_alpha); Q.rsP = rsP;
      Q.dout = h->dout_dbg.p; Q.dact = h->dact_dbg.p; Q.rsDout = h->dout_dbg.rs;
      Q.M = B; Q.E = E;
      pl.grid = dim3((B * A + 255) / 256, R);
      pl.block = dim3(256);
      push(std::move(pl), policy_dout_kernel, Q);
    }
    P.NO = 2 * A; P.Kdim = Ha; P.nets = 1; P.policy_mode = split ? 0 : 1;
    if (split) { P.dout = h->dout_dbg.p; P.rsDoutNet = 0; P.rsDoutRep = h->dout_dbg.rs; }
    const LayerOff& lo = L.actor[La];
    P.W = W(lo.w); P.dW = Gp(lo.w); P.db = Gp(lo.b);
    P.h = h->hA[La - 1].p + (long long)B * Ha; P.rsHrep = h->hA[La - 1].rs; P.ldh = Ha;   // rows B..2B-1 (= s half)
    P.dh = h->dhA[La - 1].p; P.rsDhRep = h->dhA[La - 1].rs; P.lddh = Ha;
    P.dx = h->dxP.p; P.rsDxNet = (long long)B * h->K.ldx; P.rsDxRep = h->dxP.rs; P.lddx = h->K.ldx;
    P.psave = h->psave.p + (long long)B * A * kSaveW; P.rsSave = h->psave.rs;
    P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
    P.log_alpha = W(L.off_alpha);
    P.dout_dbg = h->dout_dbg.p; P.dact_dbg = h->dact_dbg.p; P.rsDbg = h->dout_dbg.rs;
  }
  // large batches: rows cut into slices (4x the CTAs, a quarter of the serial row loop each); slice s >= 1 leaves its
  // partial head-weight gradient in gradient slice s, exactly like the split-K GEMM weight gradients
  P.row_slices = h->gslices;
  P.xs = (long long)R * L.trainable;
  if (P.dW && h->grads_x) { P.dWx = h->grads_x + (P.dW - h->grads); P.dbx = h->grads_x + (P.db - h->grads); }
  const int rows_per = (B + P.row_slices - 1) / P.row_slices;
  // 128-bit column mapping (head_bwd4_kernel) when every row pitch / tensor offset involved is a multiple of 4 floats --
  // for the scalar critic heads; the policy head (NO = 2 x act outputs, one network) would be left with 28 CTAs, too
  // few to fill the GPU
  const bool wide = P.NO == 1 && (P.Kdim % 4) == 0 && (P.ldh % 4) == 0 && (P.lddh % 4) == 0;
  l.label = std::string(policy ? "head_bwd(policy, " : "head_bwd(q, ") + (wide ? "128-bit, " : "") + "row slices " +
            std::to_string(P.row_slices) + ")";
  const int cols = wide ? kHb4Cols : kHbCols;
  l.grid = dim3(((P.Kdim + cols - 1) / cols) * ((B + rows_per - 1) / rows_per), P.nets, R);
  l.block = dim3(256);
  l.smem = ((((size_t)rows_per * P.NO + 3) & ~(size_t)3) + (wide ? 1024 : 256) * (size_t)P.NO) * sizeof(float);   // head_bwd4: red 16-B aligned
  if (l.smem > 200 * 1024) {
    rc = fail(B200SAC_ERR_INVALID, "batch * head width too large for head_bwd smem");
    return;
  }
  push(std::move(l), wide ? head_bwd4_kernel : head_bwd_kernel, P);
}

// the trainable slice of optimizer `which` (0 critic, 1 actor, 2 CARE(O) context encoder)
void PlanBuilder::opt_slice(int which, int64_t& beg, int64_t& n) const {
  beg = which == 0 ? L.critic_begin : (which == 1 ? L.actor_begin : L.cenc_begin);
  n = which == 0 ? L.critic_n : (which == 1 ? L.actor_n : L.cenc_n);
}

// parameter update + the tail job (last CTA); tail_only: the tail job alone, on the fork stream, plus the critic-loss
// reduction (the layer-chained plan, whose parameter updates are fused into the weight-gradient launches).
// grad_clip handles: Adam runs on the clipped gradient and the grad_norm launch in front of it joins the fork stream;
// with_tail = false drops the tail job (the layer-chained plan's forked tail has it).
void PlanBuilder::adam(int which, bool tail_only, bool with_tail) {
  Launch l;
  l.label = which == 0 ? "adam_critic+polyak" : which == 2 ? "adam_context_encoder" :
            tail_only ? "alpha+losses(forked)" : with_tail ? "adam_actor+alpha" : "adam_actor";
  AdamArgs P;
  memset(&P, 0, sizeof(P));
  int64_t beg, n;
  opt_slice(which, beg, n);
  const bool clip = c.grad_clip && !tail_only;
  P.p = h->params + beg; P.m = h->adam_m + beg; P.v = h->adam_v + beg; P.g = h->grads + beg;
  P.rsP = rsP; P.rsM = rsG; P.n = n;
  P.gx = h->grads_x ? h->grads_x + beg : nullptr; P.xs = (long long)R * L.trainable; P.nx = h->gslices - 1;
  P.target_delta = which == 0 ? L.target_delta : 0;
  P.tau2_begin = (which == 0 && c.care) ? (L.cse_begin - L.critic_begin) : (long long)1 << 60;
  P.which = which == 2 ? 4 : which;                    // counter slot: 0 critic, 1 actor, 4 context encoder
  P.cnt = h->cnt;
  P.tail = which == 0 ? TAIL_CRITIC_LOSS : (which == 1 ? TAIL_ALPHA_AND_LOSSES : TAIL_NONE);
  if (tail_only) P.tail = TAIL_ALL;
  if (!with_tail) P.tail = TAIL_NONE;
  if (clip) {
    P.coef = h->clip_coef + which;
    if (h->fused) { P.gx = nullptr; P.nx = 0; }       // the chained weight-gradient launches write slice 0 only
  }
  const bool pcg = c.pcgrad && !tail_only && which < 2;
  if (pcg) P.pcw = h->pc_w + (size_t)which * c.num_tasks;
  P.lq = h->lq.p; P.la = h->la.p; P.rsY = h->y.rs;
  P.logp_cur = h->logp.p + B; P.logstd_sum = h->logstd.p + B; P.rsLogp = h->logp.rs;
  P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
  P.log_alpha = h->params + L.off_alpha;
  P.m_alpha = h->adam_m + L.off_alpha; P.v_alpha = h->adam_v + L.off_alpha; P.g_alpha = h->grads + L.off_alpha;
  P.losses = h->losses; P.losses_host = h->loss_h_dev; P.R = R;
  const int nb = elementwise_blocks(n);
  l.grid = dim3(nb + (P.tail != TAIL_NONE ? 1 : 0), R);
  l.block = dim3(256);
  l.join = !clip && !pcg;        // every gradient of the slice must have landed, including the forked weight gradients
  if (tail_only) { l.grid = dim3(1, R); l.join = false; l.branch = 1; }
  push(std::move(l), pcg ? adam_kernel<false, true> : clip ? adam_kernel<true> : adam_kernel<false>, P);
}

// grad_clip handles: the gradient norm of optimizer `which` and the clip coefficient its Adam launch (next) applies
void PlanBuilder::grad_norm(int which) {
  Launch l;
  l.label = which == 0 ? "grad_norm{critic}" : which == 1 ? "grad_norm{actor}" : "grad_norm{context_encoder}";
  GradNormArgs P;
  memset(&P, 0, sizeof(P));
  int64_t beg, n;
  opt_slice(which, beg, n);
  P.g = h->grads + beg; P.rsM = rsG; P.n = n;
  if (!h->fused && h->grads_x) { P.gx = h->grads_x + beg; P.xs = (long long)R * L.trainable; P.nx = h->gslices - 1; }
  P.which = which == 2 ? 4 : which;
  P.col = which;
  P.cnt = h->cnt;
  P.thr = h->clip_thr.dev; P.coef = h->clip_coef; P.norms = h->gnorm_h_dev;
  P.part = h->gn_part + (size_t)which * R * kGradNormMaxBlocks;
  P.ticket = h->gn_ticket + (size_t)which * R;
  P.R = R;
  l.grid = dim3(elementwise_blocks(n), R);
  l.block = dim3(256);
  l.join = true;                 // every gradient of the slice must have landed, including the forked weight gradients
  push(std::move(l), grad_sqnorm_kernel, P);
}

// pcgrad handles: the Gram matrix of optimizer `which`'s task slices, the surgery and the slice weights its Adam launch
// (next) applies
void PlanBuilder::pcgrad(int which) {
  Launch l;
  l.label = which == 0 ? "pcgrad{critic}" : "pcgrad{actor}";
  PcgArgs P;
  memset(&P, 0, sizeof(P));
  int64_t beg, n;
  opt_slice(which, beg, n);
  const int T = c.num_tasks;
  P.g = h->grads + beg; P.gx = h->grads_x + beg; P.xs = (long long)R * L.trainable; P.rsM = rsG; P.n = n;
  P.T = T; P.opt = which;
  P.cnt = h->cnt; P.on = h->pc_on.dev;
  P.part = h->pc_part + (size_t)which * R * kGradNormMaxBlocks * pcgrad_pairs(T);
  P.ticket = h->pc_ticket + (size_t)which * R;
  P.G = h->pc_G; P.w = h->pc_w; P.perm = h->pc_perm; P.mask = h->pc_mask;
  P.cac = h->cg_c.dev; P.cgp = h->cg_p; P.cgf = h->cg_f; P.cgi = h->cg_it;
  if (which == 0) { P.tid = (const int*)h->tid.p; P.rsR = h->r.rs; P.B = B; P.bad = h->pc_bad; }
  P.seed = h->K.seed;
  l.grid = dim3(elementwise_blocks(n), R);
  l.block = dim3(256);
  l.smem = pcgrad_smem(T);
  l.join = true;                 // every gradient of the slice must have landed, including the forked weight gradients
  push(std::move(l), pcgrad_kernel, P);
}

int PlanBuilder::build_plan_fused() {
  const bool clip = c.grad_clip != 0;
  ChainRows rw;
  memset(&rw, 0, sizeof(rw));
  rw.r = h->r.p; rw.d = h->d.p; rw.tid = (const int*)h->tid.p; rw.rsR = h->r.rs;
  rw.logp = h->logp.p; rw.rsLogp = h->logp.rs;
  rw.alpha = h->alpha.p; rw.rsAlpha = h->alpha.rs;
  rw.q = h->q.p;
  rw.y = h->y.p; rw.dq = h->dq.p; rw.lq = h->lq.p; rw.dqa = h->dqa.p; rw.la = h->la.p; rw.qmin = h->qmin.p; rw.rsY = h->y.rs;
  rw.dxP = h->dxP.p; rw.rsDxNet = (long long)B * h->K.ldx; rw.rsDxRep = h->dxP.rs; rw.lddx = h->K.ldx;
  rw.psave = h->psave.p + (long long)B * A * kSaveW; rw.rsSave = h->psave.rs;
  rw.dout_dbg = h->dout_dbg.p; rw.dact_dbg = h->dact_dbg.p; rw.rsDbg = h->dout_dbg.rs;

  if (h->env.chain_dbg) CU(dev_fill(h->chain_dbg, CH_DBG_SLOTS * 16, 0));
  auto dbg_slot = [&]() { return (h->chain_dbg && h->plan.size() < 16) ? h->chain_dbg + h->plan.size() * CH_DBG_SLOTS : nullptr; };

  // Stage tables of one MLP.  Forward: input rows X, hidden layers 0..nh-1, outputs stored to store[l] from row store_row.
  // Backward (input-gradient chain dh_{l-1} = (dh_l W_l) * [h_{l-1} > 0], l = nh-1 .. 1): gate activations acts[l] and
  // the gate of the generated dY from row act_row, stores dstore[l] (nullable) from row drow.  J is a ChainJob or a Chain2Job.
  auto fwd_stages = [&](auto& J, ChainStage* st, const std::vector<LayerOff>& net, int nh, const float* X, long long rsX, int ldx, int K0,
                        const std::vector<Buf>* store, long long store_row) {
    J.X = X; J.rsX = rsX; J.ldx = ldx; J.K0 = K0;
    for (int lyr = 0; lyr < nh; ++lyr) {
      const LayerOff& lo = net[lyr];
      ChainStage& S = st[lyr];
      S.W = W(lo.w); S.bias = W(lo.b); S.ldw = lo.ld; S.K = lo.in; S.N = lo.out;
      if (store) { S.out = (*store)[lyr].p + store_row * lo.out; S.rsOut = (*store)[lyr].rs; S.ldo = lo.out; }
    }
  };
  auto bwd_stages = [&](auto& J, ChainStage* st, const std::vector<LayerOff>& net, int nh, const std::vector<Buf>& acts, long long act_row,
                        const std::vector<Buf>* dstore, long long drow) {
    const int Hl = net[nh - 1].out;
    J.hlast = acts[nh - 1].p + act_row * Hl; J.rsHlast = acts[nh - 1].rs; J.ldh = Hl;
    if (dstore) { J.dylast = (*dstore)[nh - 1].p + drow * Hl; J.rsDy = (*dstore)[nh - 1].rs; J.lddy = Hl; }
    for (int s = 0; s + 1 < nh; ++s) {
      const int lyr = nh - 1 - s;
      const LayerOff& lo = net[lyr];
      ChainStage& S = st[s];
      S.W = W(lo.w); S.ldw = lo.ld; S.K = lo.out; S.N = lo.in;
      S.mask = acts[lyr - 1].p + act_row * lo.in; S.rsMask = acts[lyr - 1].rs; S.ldmask = lo.in;
      if (dstore) { S.out = (*dstore)[lyr - 1].p + drow * lo.in; S.rsOut = (*dstore)[lyr - 1].rs; S.ldo = lo.in; }
    }
  };
  // Tensor maps [R][n] of the forward stages fs (W [N][K] row-major, pitch ldw, box {32 k, N rows}, SWIZZLE_128B, OOB k
  // zero-filled), owned by the handle: stage i of replica r reads tm + r * n
  auto map_weights = [&](const std::vector<ChainStage*>& fs) {
    const int n = (int)fs.size();
    std::vector<CUtensorMap> maps((size_t)R * n);
    for (int rep = 0; rep < R; ++rep)
      for (int i = 0; i < n; ++i)
        if (int e = make_map(&maps[(size_t)rep * n + i], fs[i]->W + (long long)rep * rsP, fs[i]->K, fs[i]->N, fs[i]->ldw, fs[i]->N)) rc = e;
    const CUtensorMap* tm = upload(h->tmaps, maps);
    for (int i = 0; i < n; ++i) { fs[i]->tm = tm + i; fs[i]->rsTm = n; }
  };
  // chain_kernel launch; its jobs are filled by the caller, then finish_chain sizes the grid and appends it
  auto new_chain = [&](int njobs, int early_weights) {
    ChainArgs P;
    memset(&P, 0, sizeof(P));
    P.njobs = njobs;
    P.early_weights = early_weights;
    P.rsP = rsP;
    P.pol = h->pol;
    P.rw = rw;
    return P;
  };
  auto finish_chain = [&](const char* label, ChainArgs& P) {
    const bool fwd = P.job[0].kind == CJ_FWD;
    if (fwd) {
      std::vector<ChainStage*> fs;
      for (int j = 0; j < P.njobs; ++j)
        for (int s = 0; s < P.job[j].nstages; ++s) fs.push_back(&P.job[j].st[s]);
      map_weights(fs);
    }
    P.dbg = dbg_slot();
    long long total = 0;
    int maxrows = 0;
    for (int j = 0; j < P.njobs; ++j) {
      total += P.job[j].rows;
      maxrows = std::max(maxrows, P.job[j].rows);
    }
    const int rows = chain_rows(total, 1, R, sms);
    Launch l;
    l.label = label;
    l.grid = dim3(std::max(1, (maxrows + rows - 1) / rows), P.njobs, R);
    l.block = dim3(CH_BLOCK);
    l.smem = CH_SMEM_BYTES;
    push(std::move(l), with_chain_rows(rows, [&](auto r) {
           constexpr int ROWS = decltype(r)::value;
           return fwd ? chain_kernel<true, ROWS> : chain_kernel<false, ROWS>;
         }), P);
  };
  // chain2_kernel launch: forward of pass fwd's twins, their head values swapped, backward of pass bwd's (local) twins.
  // The forward's activations are stored only when the backward gates on them (fwd == bwd); the critic job stores its
  // input gradients for the weight gradients, the actor-pass job runs on to d(action).
  auto pair_launch = [&](const char* label, int kind, int early, int fwd, int bwd) {
    const CriticPass &f = h->pass[fwd], &b = h->pass[bwd];
    Chain2Args P;
    memset(&P, 0, sizeof(P));
    P.kind = kind; P.rsP = rsP; P.rw = rw;
    P.early_weights = early;
    std::vector<ChainStage*> fs;
    for (int net = 0; net < 2; ++net) {
      Chain2Job& J = P.job[net];
      J.rows = B; J.nfwd = Lc; J.nbwd = Lc - 1; J.net = net;
      fwd_stages(J, J.st, f.net[net], Lc, f.X->p, f.X->rs, h->K.ldx, h->K.xw, fwd == bwd ? &f.h : nullptr, (long long)net * B);
      for (int s = 0; s < Lc; ++s) fs.push_back(&J.st[s]);
      const LayerOff& fh = f.net[net][Lc];
      J.Whf = W(fh.w); J.bhf = W(fh.b); J.Hhf = fh.in;
      J.qf_out = f.q->p + (long long)net * B; J.rsQf = f.q->rs;
      const std::vector<LayerOff>& bn = b.net[net];
      bwd_stages(J, J.st + Lc, bn, Lc, b.h, (long long)net * B, kind == C2_CRITIC ? &h->dhQ : nullptr, (long long)net * B);
      J.Whb = W(bn[Lc].w); J.Hhb = bn[Lc].in;
      if (kind == C2_ACTORQ) {
        const LayerOff& lo = bn[0];
        J.W0 = W(lo.w); J.ldw0 = lo.ld; J.col0 = h->K.in_w; J.nact = A; J.H0 = lo.out;
        J.dx = h->dxP.p + (long long)net * B * h->K.ldx; J.rsDx = h->dxP.rs; J.lddx = h->K.ldx;
      }
    }
    map_weights(fs);
    P.dbg = dbg_slot();
    const int rows = chain_rows(B, 2, R, sms);
    Launch l;
    l.label = label;
    l.critic_loss = kind == C2_CRITIC;
    l.grid = dim3((B + rows - 1) / rows, 2, R);
    l.block = dim3(CH_BLOCK);
    l.smem = C2_SMEM_BYTES;
    l.cluster_y = 2;
    push(std::move(l), with_chain_rows(rows, [&](auto r) {
           constexpr int ROWS = decltype(r)::value;
           return kind == C2_ACTORQ ? chain2_kernel<ROWS, true> : chain2_kernel<ROWS, false>;
         }), P);
  };
  // weight-gradient launch of a group of networks; the CTA that reduces a gradient tile applies Adam (+ Polyak) to it,
  // unless store_only (the gradients alone, no optimizer step: grad_clip plans)
  struct WNet { const std::vector<LayerOff>* net; int nh; const std::vector<Buf>* dstore; const std::vector<Buf>* acts; long long act_row_off;
                const float* X; long long rsX; int ldx; const float* dout; long long rsDout; int lddout; int net_idx; };
  auto wgrad_launch = [&](const std::vector<WNet>& nets, const char* label, int which, bool store_only) -> int {
    WgradArgs P;
    memset(&P, 0, sizeof(P));
    P.M = B; P.rsG = rsG;
    WgradAdam& O = P.adam;
    O.which = which;
    O.params = h->params; O.m = h->adam_m; O.v = h->adam_v; O.grads = h->grads;
    O.rsP = rsP; O.rsM = rsG;
    O.target_delta = which == 0 ? L.target_delta : 0;
    O.cnt = h->cnt;
    int tiles = 0;
    // operands a tensor map can address (16-byte row pitch and base) arrive by TMA, the others are staged by the threads
    struct Operand { const CUtensorMap** tm; const float* p; long long rs; int ld, cols; };
    std::vector<Operand> ops;
    auto add = [&](const float* Ap, long long rsA, int lda, const float* Bp, long long rsB, int ldb, int64_t offW, int ldc, int64_t offB,
                   int Kout, int Nin) -> int {
      if (P.njobs >= WG_MAXJOBS) return fail(B200SAC_ERR_INVALID, "too many weight-gradient jobs in one launch");
      WgradJob& J = P.job[P.njobs++];
      J.A = Ap; J.rsA = rsA; J.lda = lda; J.B = Bp; J.rsB = rsB; J.ldb = ldb;
      J.C = Gp(offW); J.C2 = Gp(offB); J.ldc = ldc; J.Kout = Kout; J.Nin = Nin;
      J.tile0 = tiles; J.tn = (Nin + WG_T - 1) / WG_T;
      J.shape = Kout <= 4 ? WG_KTHIN : (Nin <= 16 ? WG_NTHIN : WG_FULL);
      tiles += J.tn * ((Kout + WG_T - 1) / WG_T);
      auto tmable = [&](const float* p_, long long rs_, int ld_) { return (ld_ % 4) == 0 && (((uintptr_t)p_) & 15) == 0 && (rs_ % 4) == 0; };
      if (tmable(Ap, rsA, lda)) ops.push_back(Operand{&J.tmA, Ap, rsA, lda, Kout});
      if (tmable(Bp, rsB, ldb)) ops.push_back(Operand{&J.tmB, Bp, rsB, ldb, Nin});
      return 0;
    };
    for (const WNet& n : nets) {
      const std::vector<LayerOff>& net = *n.net;
      for (int lyr = n.nh - 1; lyr >= 0; --lyr) {      // biggest layers first
        const LayerOff& lo = net[lyr];
        const Buf& db = (*n.dstore)[lyr];
        const float* Ap = db.p + (long long)n.net_idx * B * lo.out;
        const float* Bp; long long rsB; int ldb;
        if (lyr == 0) { Bp = n.X; rsB = n.rsX; ldb = n.ldx; }
        else {
          const Buf& ab = (*n.acts)[lyr - 1];
          Bp = ab.p + ((long long)n.net_idx * B + n.act_row_off) * lo.in; rsB = ab.rs; ldb = lo.in;   // (actor: [s';s], skip the s' half)
        }
        if (int rc = add(Ap, db.rs, lo.out, Bp, rsB, ldb, lo.w, lo.ld, lo.b, lo.out, lo.in)) return rc;
      }
      const LayerOff& hd = net[n.nh];
      const Buf& ab = (*n.acts)[n.nh - 1];
      const float* Bp = ab.p + ((long long)n.net_idx * B + n.act_row_off) * hd.in;
      if (int rc = add(n.dout, n.rsDout, n.lddout, Bp, ab.rs, hd.in, hd.w, hd.in, hd.b, hd.out, hd.in)) return rc;
    }
    // maps [R][n] of the operands, [B rows][cols] row-major, box {32 cols, 256 rows}, dense: operand i of replica r at tm + r * n
    const int n = (int)ops.size();
    std::vector<CUtensorMap> maps((size_t)R * n);
    for (int rep = 0; rep < R; ++rep)
      for (int i = 0; i < n; ++i)
        if (int rc = make_map(&maps[(size_t)rep * n + i], ops[i].p + (long long)rep * ops[i].rs, ops[i].cols, B, ops[i].ld, WG_ROWS, true))
          return rc;
    const CUtensorMap* tm = upload(h->tmaps, maps);
    for (int i = 0; i < n; ++i) *ops[i].tm = tm + i;
    for (int j = 0; j < P.njobs; ++j) P.job[j].rsTm = n;
    P.dbg = dbg_slot();
    Launch l;
    l.label = label;
    l.grid = dim3(tiles, R);
    l.block = dim3(WG_THREADS);
    l.smem = WG_SMEM_BYTES;
    push(std::move(l), store_only ? wgrad_kernel<true> : wgrad_kernel<false>, P);
    return 0;
  };

  const CriticPass& Q = h->pass[PASS_Q];
  // ---- A: actor over [s';s], Q1/Q2 over (s,a) ----------------------------------------------------------------------
  {
    ChainArgs P = new_chain(3, 1);
    for (int j = 0; j < 3; ++j) {
      ChainJob& J = P.job[j];
      const int net = j - 1;
      const std::vector<LayerOff>& mlp = j == 0 ? L.actor : Q.net[net];
      const int nh = j == 0 ? La : Lc;
      J.kind = CJ_FWD; J.nstages = nh;
      if (j == 0) {
        J.rows = 2 * B; J.head = CH_HEAD_POLICY;
        fwd_stages(J, J.st, mlp, nh, h->XA.p, h->XA.rs, h->K.ldxa, h->K.in_w, &h->hA, 0);
      } else {
        J.rows = B; J.head = CH_HEAD_SCALAR; J.qout = Q.q->p + (long long)net * B; J.rsQ = Q.q->rs;
        fwd_stages(J, J.st, mlp, nh, Q.X->p, Q.X->rs, h->K.ldx, h->K.xw, &Q.h, (long long)net * B);
      }
      const LayerOff& hd = mlp[nh];
      J.Wh = W(hd.w); J.bh = W(hd.b); J.NO = hd.out; J.Hh = hd.in;
    }
    finish_chain("chain_fwd{actor,q1,q2}", P);
  }
  // ---- B + C: target critics over (s', a'), TD target, critic backward (one clustered launch), weight gradients, Adam ----
  pair_launch("chain2{qt->y->bwd q}", C2_CRITIC, 1, PASS_T, PASS_Q);
  {
    std::vector<WNet> nets;
    for (int net = 0; net < 2; ++net)
      nets.push_back(WNet{&Q.net[net], Lc, &h->dhQ, &Q.h, 0, Q.X->p, Q.X->rs, h->K.ldx, h->dq.p + (long long)net * B, h->dq.rs, 1, net});
    if (int rc = wgrad_launch(nets, clip ? "wgrad{q1,q2}" : "wgrad+adam+polyak{q1,q2}", 0, clip)) return rc;
  }
  if (clip) {                    // the whole critic gradient first, then its norm, then Adam + Polyak on the clipped gradient
    grad_norm(0);
    adam(0, false, false);
  }
  // ---- D: actor pass through the updated critics ------------------------------------------------------------------------
  // (the launch right before this one is the critic Adam: no weight request before the dependency wait)
  pair_launch("chain2{q(s,a~)->min->bwd->d(action)}", C2_ACTORQ, 0, PASS_P, PASS_P);
  // actor loss / entropy / temperature gradient + its Adam step need only what D produced (the step's alpha is the
  // snapshot taken at ingest): they run on the fork stream beside the policy backward instead of trailing the actor Adam
  adam(1, true);
  // ---- E: policy backward, weight gradients, Adam ----------------------------------------------------------------------
  {
    ChainArgs P = new_chain(1, 1);
    ChainJob& J = P.job[0];
    J.kind = CJ_BWD_POLICY; J.rows = B; J.nstages = La - 1;
    const LayerOff& hd = L.actor[La];
    J.Wh = W(hd.w); J.bh = W(hd.b); J.NO = hd.out; J.Hh = hd.in;
    bwd_stages(J, J.st, L.actor, La, h->hA, (long long)B, &h->dhA, 0);
    finish_chain("chain_bwd{actor}", P);
    std::vector<WNet> nets;
    nets.push_back(WNet{&L.actor, La, &h->dhA, &h->hA, (long long)B, h->XA.p + (long long)B * h->K.ldxa, h->XA.rs, h->K.ldxa,
                        h->dout_dbg.p, h->dout_dbg.rs, 2 * A, 0});
    if (int rc = wgrad_launch(nets, clip ? "wgrad{actor}" : "wgrad+adam{actor}", 1, clip)) return rc;
  }
  if (clip) {
    grad_norm(1);
    adam(1, false, false);
  }
  return 0;
}

// critic_ln handles: the LayerNorm of hidden layer l of every network of pass `pass` over the [E][B][H]
// pre-normalization buffer z[l], every replica in one launch.  Forward: h[l] = relu(LN(z[l])).  Backward: dhQ[l] becomes
// the gradient at z[l] in place, and with want_grads the LayerNorm weight and bias gradients land in gradient slice 0 (the
// split-K slices hold zeros there, so Adam's slice sum reads them unchanged).  critic_dropout handles run the dropout
// instantiations on the same launches, with the pass's mask buffer and Philox tag.
void PlanBuilder::layer_norm(int pass, int l, bool fwd, bool want_grads) {
  const CriticPass& cp = h->pass[pass];
  const int H = c.critic_hidden[l];
  Launch ln;
  ln.label = std::string(fwd ? "ln_fwd{" : "ln_bwd{") + cp.label + " " + std::to_string(l) + "}";
  ln.branch = branch;
  LnArgs P;
  memset(&P, 0, sizeof(P));
  P.z = cp.z[l].p; P.rsZ = cp.z[l].rs;
  const Buf& out = fwd ? cp.h[l] : h->dhQ[l];
  (fwd ? P.h : P.dh) = out.p;
  P.rsH = out.rs;
  const LayerOff& lo = cp.net[0][l];
  P.g = W(lo.g); P.c = W(lo.c);
  if (want_grads) { P.dg = Gp(lo.g); P.dc = Gp(lo.c); }
  P.rsP = rsP; P.rsG = rsG; P.rsNet = rsNet;
  P.part = h->ln_part; P.ticket = h->ln_ticket;
  P.B = B; P.H = H; P.E = E;
  P.actor_side = actor_side ? 1 : 0;
  const bool drop = c.critic_dropout != 0;
  if (drop) {
    P.drop = h->drop.dev; P.mbits = (unsigned*)cp.m[l].p; P.rsM = cp.m[l].rs;
    P.tag0 = (pass * 8 + l) * E;
  }
  ln.block = dim3(kLnThreads);
  if (fwd) {
    ln.grid = dim3((E * B + kLnThreads / kWarp - 1) / (kLnThreads / kWarp), R);
    if (drop) push(std::move(ln), ln_fwd_kernel<true>, P);
    else push(std::move(ln), ln_fwd_kernel<false>, P);
  } else {
    ln.grid = dim3((B + kLnRows - 1) / kLnRows, E, R);
    if (drop) push(std::move(ln), ln_bwd_kernel<true>, P);
    else push(std::move(ln), ln_bwd_kernel<false>, P);
  }
}

// Forward of pass `pass`'s twins at critic hidden layer l, in one grouped launch after the problems ps already holds.
// critic_ln: the GEMMs write the pre-normalization buffer z (no ReLU), the layer_norm launch the post-ReLU h that the rest
// of the plan reads.
void PlanBuilder::critic_fwd(int pass, int l, std::vector<GemmProb> ps) {
  const CriticPass& cp = h->pass[pass];
  const bool ln = c.critic_ln != 0;
  const Buf& out = ln ? cp.z[l] : cp.h[l];
  for (int net = 0; net < E; ++net) {
    const LayerOff& lo = cp.net[net][l];
    const Buf x = critic_in(cp, net, l);
    GemmProb p = fwd_prob(par, x.p, x.rs, B, lo, netp(out, net, lo.out), out.rs);
    if (ln) p.relu = 0;
    ps.push_back(p);
  }
  gemm_launch(ps);
  if (ln) layer_norm(pass, l, true, false);
}

// Backward of pass `pass`'s twins at critic hidden layer l from dhQ[l]: with want_wgrad the weight gradients (the critic
// update), and the input gradients, gated by the layer's input activations, into dhQ[l - 1]; at layer 0 into dxP, which
// the actor pass needs and, on CARE handles, the critic update too (it trains the critic's state encoder).
void PlanBuilder::critic_bwd(int pass, int l, bool want_wgrad) {
  const CriticPass& cp = h->pass[pass];
  // (on the main stream: a forked weight gradient below waits for it like the input gradient does)
  if (c.critic_ln) layer_norm(pass, l, false, want_wgrad);
  std::vector<GemmProb> ps, dg;
  for (int net = 0; net < E; ++net) {
    const LayerOff& lo = cp.net[net][l];
    const Buf x = critic_in(cp, net, l), dz{netp(h->dhQ[l], net, lo.out), h->dhQ[l].rs};
    if (want_wgrad) ps.push_back(wgrad_prob(grd, dz.p, dz.rs, x.p, x.rs, lo, B));
    if (l > 0)
      dg.push_back(dgrad_prob(par, dz.p, dz.rs, lo, x.p, x.rs, netp(h->dhQ[l - 1], net, lo.in), h->dhQ[l - 1].rs, B));
    else if (!want_wgrad || c.care)
      dg.push_back(dgrad_prob(par, dz.p, dz.rs, lo, nullptr, 0, h->dxP.p + (long long)net * B * h->K.ldx, h->dxP.rs, B));
  }
  if (want_wgrad && use_fork && l > 0) {
    branch = 1; gemm_launch(ps); branch = 0;
    gemm_launch(dg);
  } else {
    ps.insert(ps.end(), dg.begin(), dg.end());      // {wgrad q1, wgrad q2, dgrad q1, dgrad q2}; ensembles: E of each
    gemm_launch(ps);
  }
}

// ---- per-layer plan: one grouped GEMM launch per layer (and kind) of the networks --------------------------------
void PlanBuilder::build_plan_layered() {
  const int Kenc = c.num_encoders, nmix = c.care ? (int)L.mix.size() : 0;
  if (c.care) {
    // encoded states of [s'; s] with the critic's (== actor's, tied) encoder and of s' with the target's
    care_tables({0, 1});
    care_encode({EncJob{0, 0, 2 * B, h->XA, h->K.ldxa, h->XQ, h->K.ldx, B}, EncJob{1, 0, B, h->XT, h->K.ldx, Buf{}, 0, 0}});
  }
  // ---- Phase A: actor over [s2; s] and Q1,Q2 over (s,a), layer by layer -----------------
  for (int l = 0; l < (La > Lc ? La : Lc); ++l) {
    std::vector<GemmProb> ps;
    if (l < La) {
      const LayerOff& lo = L.actor[l];
      ps.push_back(fwd_prob(par, l == 0 ? h->XA.p : h->hA[l - 1].p, l == 0 ? h->XA.rs : h->hA[l - 1].rs, 2 * B, lo,
                       h->hA[l].p, h->hA[l].rs));
    }
    if (use_fork && La == Lc) {
      // Q1,Q2 on (s,a) are not needed before critic_heads, while the actor's output heads the policy_head -> target-critic
      // chain: the critics' layer goes to the fork stream (joined at critic_heads), the actor's stays on the main stream.
      branch = 1;
      critic_fwd(PASS_Q, l);
      branch = 0;
      gemm_launch(ps);
    } else if (l < Lc) {
      critic_fwd(PASS_Q, l, ps);
    } else {
      gemm_launch(ps);
    }
  }
  {  // policy head
    Launch l;
    l.label = "policy_head";
    l.grid = dim3((2 * B + 7) / 8, R);
    l.block = dim3(256);
    push(std::move(l), policy_head_kernel, h->pol);
  }
  // ---- Phase B: target critics over (s2, a') ---------------------------------------------
  for (int l = 0; l < Lc; ++l) critic_fwd(PASS_T, l);
  const int Hc = c.critic_hidden[Lc - 1];
  {  // critic heads: y, Q1, Q2, dQ
    Launch l;
    l.label = "critic_heads";
    l.join = true;                 // needs Q1,Q2 on (s,a), which may have run on the fork stream
    l.critic_loss = true;
    l.grid = dim3((B + 7) / 8, R);
    l.block = dim3(256);
    CriticHeadArgs P;
    memset(&P, 0, sizeof(P));
    const Buf &hT = h->pass[PASS_T].h[Lc - 1], &hQ = h->pass[PASS_Q].h[Lc - 1];
    P.hT = hT.p; P.hQ = hQ.p; P.rsHnet = (long long)B * Hc; P.rsHrep = hT.rs; P.ldh = Hc;
    P.Wt = W(L.qt[0][Lc].w); P.bt = W(L.qt[0][Lc].b);
    P.Wq = W(L.q[0][Lc].w); P.bq = W(L.q[0][Lc].b);
    P.rsNet = rsNet; P.rsP = rsP;
    P.r = h->r.p; P.d = h->d.p; P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
    P.logp = h->logp.p; P.rsLogp = h->logp.rs;
    P.log_alpha = W(L.off_alpha);
    P.y = h->y.p; P.q = h->q.p; P.dq = h->dq.p; P.lq = h->lq.p; P.rsY = h->y.rs;
    P.ens = h->ens.dev; P.tsub = h->tsub.p; P.rsTsub = h->tsub.rs; P.E = E;
    push(std::move(l), critic_heads_kernel, P);
  }
  // ---- Phase C: critic backward + Adam/Polyak ----------------------------------------------
  head_bwd(false, true);
  for (int l = Lc - 1; l >= 0; --l) critic_bwd(PASS_Q, l, true);
  if (c.care) {
    {  // backward of the attention mix: dZk, d(att)
      Launch l;
      l.label = "care_mix_bwd";
      CareMixBwdArgs P;
      memset(&P, 0, sizeof(P));
      P.dx = h->dxP.p; P.rsDxNet = (long long)B * h->K.ldx; P.rsDxRep = h->dxP.rs; P.lddx = h->K.ldx;
      P.Z = h->mixZ[0].p; P.rsZ = h->mixZ[0].rs; P.kstride = (long long)2 * B * pitch(c.mix_out); P.ldz = pitch(c.mix_out);
      P.z_row_off = B;
      P.tab = h->careTab[0].p; P.rsTab = h->careTab[0].rs; P.row_w = h->care_row_w; P.off_att = h->care_off_att;
      P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
      P.dZ = h->mixDZ.p; P.rsDZ = h->mixDZ.rs; P.dkstride = (long long)B * pitch(c.mix_out); P.lddz = pitch(c.mix_out);
      P.datt = h->careDatt.p; P.rsDatt = h->careDatt.rs;
      P.B = B; P.K = Kenc; P.mo = c.mix_out; P.co = c.ctx_out;
      l.grid = dim3((B + 7) / 8, R);
      l.block = dim3(256);
      push(std::move(l), care_mix_bwd_kernel, P);
    }
    for (int l = nmix - 1; l >= 0; --l) {          // mixture-of-encoders backward, K problems per kind
      std::vector<GemmProb> ps;
      const LayerOff& lo = L.mix[l];
      const Buf& dzb = (l == nmix - 1) ? h->mixDZ : h->mixDH[l];
      for (int k = 0; k < Kenc; ++k) {
        GemmProb p;
        memset(&p, 0, sizeof(p));
        p.A = dzb.p + (long long)k * B * pitch(lo.out); p.rsA = dzb.rs; p.lda = pitch(lo.out);
        if (l == 0) { p.B = h->XS.p + (long long)B * h->K.obs; p.rsB = h->XS.rs; p.ldb = h->K.obs; }
        else {
          const Buf& ib = h->mixH[0][l - 1];
          p.B = ib.p + ((long long)k * 2 * B + B) * pitch(lo.in); p.rsB = ib.rs; p.ldb = pitch(lo.in);
        }
        p.C = Gp(lo.w + (long long)k * lo.out * lo.in); p.rsC = rsG; p.ldc = lo.in;
        p.C2 = Gp(lo.b + (long long)k * lo.out); p.rsC2 = rsG;
        p.M = lo.out; p.N = lo.in; p.K = B; p.mode = GEMM_WGRAD;
        ps.push_back(p);
      }
      if (l > 0)
        for (int k = 0; k < Kenc; ++k) {
          const Buf& ib = h->mixH[0][l - 1];
          GemmProb p;
          memset(&p, 0, sizeof(p));
          p.A = dzb.p + (long long)k * B * pitch(lo.out); p.rsA = dzb.rs; p.lda = pitch(lo.out);
          p.B = W(lo.w + (long long)k * lo.out * lo.in); p.rsB = rsP; p.ldb = lo.in;
          p.mask = ib.p + ((long long)k * 2 * B + B) * pitch(lo.in); p.rsMask = ib.rs; p.ldmask = pitch(lo.in);
          p.C = h->mixDH[l - 1].p + (long long)k * B * pitch(lo.in); p.rsC = h->mixDH[l - 1].rs; p.ldc = pitch(lo.in);
          p.M = B; p.N = lo.in; p.K = lo.out; p.mode = GEMM_DGRAD;
          ps.push_back(p);
        }
      gemm_launch(ps);
    }
    {  // per-task reduction + softmax backward, then the trunk / context-MLP weight gradients
      Launch l;
      l.label = "care_tab_reduce";
      CareTabReduceArgs P;
      memset(&P, 0, sizeof(P));
      P.datt = h->careDatt.p; P.rsDatt = h->careDatt.rs;
      P.dx = h->dxP.p; P.rsDxNet = (long long)B * h->K.ldx; P.rsDxRep = h->dxP.rs; P.lddx = h->K.ldx;
      P.tab = h->careTab[0].p; P.rsTab = h->careTab[0].rs; P.row_w = h->care_row_w; P.off_att = h->care_off_att;
      P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
      P.dtab = h->careDtab.p; P.rsDtab = h->careDtab.rs;
      P.B = B; P.K = Kenc; P.co = c.ctx_out;
      l.grid = dim3(c.num_tasks, R);
      l.block = dim3(1024);
      push(std::move(l), care_tab_reduce_kernel, P);
      Launch l2;
      l2.label = "care_tab_wgrad";
      CareTabWgradArgs Q;
      memset(&Q, 0, sizeof(Q));
      Q.params = h->params; Q.rsP = rsP; Q.emb_off = L.off_emb;
      Q.tab = h->careTab[0].p; Q.rsTab = h->careTab[0].rs; Q.row_w = h->care_row_w;
      Q.dtab = h->careDtab.p; Q.rsDtab = h->careDtab.rs;
      Q.grads = h->grads; Q.rsG = rsG;
      Q.trunk = h->care_trunk; Q.ctx = h->care_ctx;
      Q.T = c.num_tasks; Q.K = Kenc; Q.co = c.ctx_out;
      Q.original = c.care == 2 ? 1 : 0; Q.off_ctx = h->care_off_ctx;
      int fl = 0;                                   // backward-chain floats of one task
      for (int j = 0; j < Q.trunk.n; ++j) fl += Q.trunk.dims[j + 1];
      for (int j = 0; j < Q.ctx.n; ++j) fl += Q.ctx.dims[j + 1];
      if (fl > kCareTabWgradSmemFloats) rc = fail(B200SAC_ERR_INVALID, "internal: one task's CARE backward chains exceed %d floats", kCareTabWgradSmemFloats);
      Q.tchunk = std::max(1, std::min(c.num_tasks, kCareTabWgradSmemFloats / fl));
      l2.smem = (size_t)Q.tchunk * fl * sizeof(float);
      if (c.pcgrad) { Q.grads_x = h->grads_x; Q.xs = (long long)R * L.trainable; }   // one gradient slice per task
      l2.grid = dim3(sms, R);
      l2.block = dim3(256);
      push(std::move(l2), c.pcgrad ? care_tab_wgrad_kernel<true> : care_tab_wgrad_kernel<false>, Q);
    }
  }
  if (c.grad_clip) grad_norm(0);
  if (c.pcgrad) pcgrad(0);
  adam(0, false);
  // ---- the actor update (D, E): every launch below returns at entry on a critic-only step; adam(1) skips its own body and
  // its tail writes NaN for the actor-side losses.  adam(2) (CARE(O) context encoder, trained by the critic loss) always runs.
  actor_side = true;
  if (c.care) {          // encoded states of s with the UPDATED critic encoder for the actor pass (learner.py:336-341)
    care_tables({2});
    care_encode({EncJob{2, B, B, h->XP, h->K.ldx, Buf{}, 0, 0}});
  }
  // ---- Phase D: actor pass through the updated critics ---------------------------------------
  for (int l = 0; l < Lc; ++l) critic_fwd(PASS_P, l);
  {
    Launch l;
    l.label = "actor_q_heads";
    l.grid = dim3((B + 7) / 8, R);
    l.block = dim3(256);
    ActorQHeadArgs P;
    memset(&P, 0, sizeof(P));
    const Buf& hP = h->pass[PASS_P].h[Lc - 1];
    P.hP = hP.p; P.rsHnet = (long long)B * Hc; P.rsHrep = hP.rs; P.ldh = Hc;
    P.Wq = W(L.q[0][Lc].w); P.bq = W(L.q[0][Lc].b);
    P.rsNet = rsNet; P.rsP = rsP;
    P.tid = (const int*)h->tid.p; P.rsR = h->r.rs;
    P.logp = h->logp.p + B; P.rsLogp = h->logp.rs;
    P.log_alpha = W(L.off_alpha);
    P.dqa = h->dqa.p; P.qp = h->qp.p; P.la = h->la.p; P.qmin = h->qmin.p; P.rsY = h->y.rs;
    P.ens = h->ens.dev; P.E = E;
    push(std::move(l), actor_q_heads_kernel, P);
  }
  head_bwd(false, false);
  for (int l = Lc - 1; l >= 0; --l) critic_bwd(PASS_P, l, false);
  // ---- Phase E: policy backward + Adam + temperature -----------------------------------------
  head_bwd(true, true);
  for (int l = La - 1; l >= 0; --l) {
    std::vector<GemmProb> ps;
    const LayerOff& lo = L.actor[l];
    const float* X = l == 0 ? h->XA.p + (long long)B * lo.ld : h->hA[l - 1].p + (long long)B * lo.ld;
    const long long rsX = l == 0 ? h->XA.rs : h->hA[l - 1].rs;
    ps.push_back(wgrad_prob(grd, h->dhA[l].p, h->dhA[l].rs, X, rsX, lo, B));
    if (l > 0)
      ps.push_back(dgrad_prob(par, h->dhA[l].p, h->dhA[l].rs, lo, h->hA[l - 1].p + (long long)B * lo.ld, h->hA[l - 1].rs,
                         h->dhA[l - 1].p, h->dhA[l - 1].rs, B));
    if (use_fork && l > 0) {
      branch = 1; gemm_launch(std::vector<GemmProb>(ps.begin(), ps.begin() + 1)); branch = 0;
      gemm_launch(std::vector<GemmProb>(ps.begin() + 1, ps.end()));
    } else {
      gemm_launch(ps);
    }
  }
  actor_side = false;
  if (c.grad_clip) grad_norm(1);          // (returns at entry on a critic-only step, like the launches of D and E)
  if (c.pcgrad) pcgrad(1);                // (likewise)
  adam(1, false);
  if (c.care == 2) {                      // update(): context_encoder_optimizer.step() (learner.py:399), gradients from the critic loss
    if (c.grad_clip) grad_norm(2);
    adam(2, false);
  }
}

// Build the launch list of one gradient step (everything after the ingest kernel).
static int build_plan(b200sac* h) {
  PlanBuilder pb(h);
  {  // policy head arguments (the per-layer plan's policy_head launch, the chained forward kernel and b200sac_act share them)
    PolicyHeadArgs& P = h->pol;
    memset(&P, 0, sizeof(P));
    const int La = pb.La;
    const LayerOff& lo = h->L.actor[La];
    P.h = h->hA[La - 1].p; P.rsH = h->hA[La - 1].rs; P.ldh = lo.in;
    P.W = pb.W(lo.w); P.b = pb.W(lo.b); P.rsP = pb.rsP;
    P.eps = h->eps.p; P.rsEps = h->eps.rs; P.use_eps_buf = 0;
    P.pout = h->pout.p; P.rsPout = h->pout.rs;
    P.psave = h->psave.p; P.rsSave = h->psave.rs;
    P.XT = h->XT.p; P.XP = h->XP.p; P.rsX = h->XT.rs;
    P.act_out = h->act_out.p; P.rsAct = h->act_out.rs;
    P.logp = h->logp.p; P.rsLogp = h->logp.rs;
    P.logstd_sum = h->logstd.p;
    P.cnt = h->cnt;
  }
  if (h->fused) {
    if (int rc = pb.build_plan_fused()) return rc;
  } else {
    pb.build_plan_layered();
  }
  return pb.rc;
}

// Launch with programmatic stream serialization (PDL): the kernel may start while its predecessor
// drains; every kernel begins with griddepcontrol.wait (common.cuh::kstamp), so data dependencies hold.
// cluster_y > 1: thread-block clusters of (1, cluster_y, 1) -- the CTAs with equal blockIdx.x / z are co-scheduled and can
// read each other's shared memory.
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, int cluster_y, cudaStream_t st,
                            Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_y > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = 1; attr[n].val.clusterDim.y = cluster_y; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// Prioritized replay: the draw of one step (indices into rb->d_idx, importance weights into the handle's per_buf).
static cudaError_t per_sample_on(b200sac* h, b200sac_replay* rb, cudaStream_t s) {
  return launch_k(per_sample_kernel, dim3(h->R), dim3(h->cfg.batch > 256 ? 512 : 256), 0, 1, s, h->K, rb->tr, (const Counters*)h->cnt,
                  0LL, 0, (const long long*)rb->d_fill, (const double*)rb->beta.dev, rb->d_idx.get(), h->per_buf.get(), (long long)h->cfg.batch,
                  rb->seed);
}

// What a plan launch takes from the step when it runs: the StepConst, and the noise source (use_eps_buf) of the two
// argument blocks that carry it.  Every other argument block runs as its builder left it.
template <class P> static const P& with_noise(const P& a, int) { return a; }
static PolicyHeadArgs with_noise(PolicyHeadArgs a, int use_eps_buf) { a.use_eps_buf = use_eps_buf; return a; }
static ChainArgs with_noise(ChainArgs a, int use_eps_buf) { a.pol.use_eps_buf = use_eps_buf; return a; }
struct RunLaunch {
  const Launch& l;
  cudaStream_t s;
  const StepConst& K;
  int use_eps_buf;
  template <class P> cudaError_t operator()(const StepFirst<P>& c) const {
    return launch_k(c.kern, l.grid, l.block, l.smem, l.cluster_y, s, K, with_noise(c.args, use_eps_buf));
  }
  template <class P> cudaError_t operator()(const StepLast<P>& c) const {
    return launch_k(c.kern, l.grid, l.block, l.smem, l.cluster_y, s, with_noise(c.args, use_eps_buf), K);
  }
  template <class P> cudaError_t operator()(const NoStep<P>& c) const {
    return launch_k(c.kern, l.grid, l.block, l.smem, l.cluster_y, s, c.args);
  }
  cudaError_t operator()(const TcCall& c) const {
    return launch_k(c.kern, l.grid, l.block, l.smem, l.cluster_y, s, c.probs, c.sched, c.G, c.sched_stride);
  }
};

// rb: the device ring of a sampled step.  Prioritized ring -- the critic loss is importance-weighted and the priority update
// runs after the critic-loss launch (forked off the critical path when allow_fork, joined before the step ends); per_next:
// the next step's draw follows that update on the same stream (ev_sampled).  Linked ring -- the TD target discounts every
// row with what the gather folded for it.
static int run_plan(b200sac* h, cudaStream_t st, bool use_eps_buf, const Event* evs = nullptr, bool allow_fork = false,
                    b200sac_replay* rb = nullptr, bool per_next = false) {
  bool fork_pending = false, per_pending = false;
  b200sac_replay* per = rb && rb->per ? rb : nullptr;
  StepConst K = h->K;
  if (per) K.isw = h->per_buf;
  if (rb && rb->traj) K.disc = h->ns_buf;
  for (size_t i = 0; i < h->plan.size(); ++i) {
    Launch& l = h->plan[i];
    if (evs) CU(cudaEventRecord(evs[i], st));
    cudaStream_t s = st;
    if (l.join && fork_pending) {                       // e.g. Adam: wait for the forked weight gradients
      CU(cudaStreamWaitEvent(st, h->ev_fork_done, 0));
      fork_pending = false;
    }
    const bool forked = allow_fork && l.branch == 1;
    if (forked) {                                       // runs beside the launches that follow on `st`
      CU(cudaEventRecord(h->ev_fork_src, st));
      CU(cudaStreamWaitEvent(h->fork, h->ev_fork_src, 0));
      s = h->fork;
    }
    std::visit(RunLaunch{l, s, K, use_eps_buf ? 1 : 0}, l.call);
    if (forked) {
      CU(cudaEventRecord(h->ev_fork_done, h->fork));
      fork_pending = true;
    }
    if (per && l.critic_loss) {
      cudaStream_t ps = st;
      if (allow_fork) {
        CU(cudaEventRecord(h->ev_per_src, s));
        CU(cudaStreamWaitEvent(h->per_fork, h->ev_per_src, 0));
        ps = h->per_fork;
      }
      const int B = h->cfg.batch, R = h->R;
      launch_k(per_update_kernel, dim3(R), dim3(256), 0, 1, ps, per->tr, 0, (const int*)per->d_idx, (long long)B, B,
               (const float*)h->y.p, (const float*)h->q.p, h->y.rs, (const float*)nullptr, h->per_buf + (size_t)R * B,
               (int*)(h->per_buf + (size_t)2 * R * B), (long long)B);
      if (allow_fork) {
        CU(cudaEventRecord(h->ev_per_done, ps));
        per_pending = true;
      }
      if (per_next) {                                   // the next step's draw sees this step's priorities
        per_sample_on(h, per, ps);
        CU(cudaEventRecord(h->ev_sampled, ps));
      }
    }
  }
  if (fork_pending) CU(cudaStreamWaitEvent(st, h->ev_fork_done, 0));
  if (per_pending) CU(cudaStreamWaitEvent(st, h->ev_per_done, 0));
  if (evs) CU(cudaEventRecord(evs[h->plan.size()], st));
  CU(cudaGetLastError());
  return 0;
}

extern "C" int b200sac_launches_per_step(b200sac_t* h, int32_t* n) {
  if (!h || !n) return fail(B200SAC_ERR_INVALID, "null argument");
  *n = (int32_t)h->plan.size() + 1;   // + ingest (the sampled-device path adds one more: index sampling)
  return 0;
}

// The device row of a replica's hyperparameters, rounded the way the kernels consume them.
static HParams hparams_row(const b200sac_hparams& v) {
  HParams r;
  memset(&r, 0, sizeof(r));
  r.lr[0] = v.lr_critic; r.lr[1] = v.lr_actor; r.lr[2] = v.lr_alpha; r.lr[4] = v.lr_ctx;
  r.gamma = (float)v.gamma; r.reward_scale = (float)v.reward_scale;
  r.tau = (float)v.tau; r.one_minus_tau = (float)(1.0 - v.tau);
  r.tau_se = (float)v.tau_se; r.one_minus_tau_se = (float)(1.0 - v.tau_se);
  return r;
}

extern "C" int b200sac_create(const b200sac_cfg* cfg, int32_t device, uint64_t seed, b200sac_t** out) {
  if (!out) return fail(B200SAC_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (int rc = check_cfg(cfg)) return rc;
  int ndev = 0;
  CU(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(B200SAC_ERR_INVALID, "device %d out of range (%d visible)", device, ndev);
  CU(cudaSetDevice(device));
  std::unique_ptr<b200sac> owner(new (std::nothrow) b200sac());   // a failed create releases what it allocated
  b200sac* h = owner.get();
  if (!h) return fail(B200SAC_ERR_NOMEM, "out of host memory");
  h->cfg = *cfg;
  h->env = env_switches();
  h->device = device;
  h->R = cfg->replicas;

  build_layout(cfg, h->L);
  const Layout& L = h->L;
  const int B = cfg->batch, R = h->R, A = cfg->act_dim, obs = cfg->state_dim + cfg->num_tasks, xw = L.in_w + A;
  const int in_w = L.in_w;
  StepConst& K = h->K;
  memset(&K, 0, sizeof(K));
  K.B = B; K.obs = obs; K.act = A; K.T = cfg->num_tasks; K.xw = xw; K.in_w = in_w; K.care = cfg->care ? 1 : 0;
  K.ldxa = (int)pad4(in_w); K.ldx = (int)pad4(xw);
  const int ldxa = K.ldxa, ldx = K.ldx;
  K.Ha = cfg->actor_hidden[cfg->n_actor_hidden - 1];
  K.Hc = cfg->critic_hidden[cfg->n_critic_hidden - 1];
  K.action_scale = (float)cfg->action_scale;
  K.c_loss = (float)(1.0 / B / (cfg->weighted_loss ? (double)B : 1.0));
  K.inv_B = (float)(1.0 / B);
  K.hbar = -(float)A;
  K.beta1 = cfg->beta1; K.beta2 = cfg->beta2; K.adam_eps = cfg->adam_eps;
  K.seed = seed;

  Counters c0;
  memset(&c0, 0, sizeof(c0));
  for (int i = 0; i < 5; ++i) c0.b1p[i] = c0.b2p[i] = 1.0;
  CU(dev_fill(h->params, (size_t)L.arena * R, 0.f));
  CU(dev_fill(h->adam_m, (size_t)L.trainable * R, 0.f));
  CU(dev_fill(h->adam_v, (size_t)L.trainable * R, 0.f));
  CU(dev_fill(h->grads, (size_t)L.trainable * R, 0.f));
  CU(dev_fill(h->cnt, R, c0));
  CU(dev_fill(h->losses, (size_t)kLossSlots * R * 4, 0.f));
  h->gslices = cfg->batch >= kSplitKMin ? kSplitK : 1;   // K of every weight gradient = batch
  if (cfg->pcgrad) h->gslices = cfg->num_tasks;         // one slice per task
  if (h->gslices > 1)       // never-written entries of slices >= 1 must read as zero (Adam sums all slices)
    CU(dev_fill(h->grads_x, (size_t)L.trainable * R * (h->gslices - 1), 0.f));
  {
    b200sac_hparams hp0;
    hp0.gamma = cfg->gamma; hp0.reward_scale = cfg->reward_scale; hp0.tau = cfg->tau;
    hp0.lr_critic = cfg->lr_critic; hp0.lr_actor = cfg->lr_actor; hp0.lr_alpha = cfg->lr_alpha;
    hp0.tau_se = cfg->tau_se; hp0.lr_ctx = cfg->lr_ctx;
    if (int rc = h->hp.init(R, &hp0)) return rc;
    K.hp = h->hp.dev;
    const int every[2] = {1, 1};                   // every step updates the actor and the targets
    if (int rc = h->ivl.init(R, every)) return rc;
    K.cnt = h->cnt;
  }
  if (cfg->grad_clip) {       // thresholds +inf (no clipping), coefficients 1, every norm NaN until a step writes it
    const size_t n = (size_t)kClipCols * R;
    const double inf[kClipCols] = {INFINITY, INFINITY, INFINITY};
    if (int rc = h->clip_thr.init(R, inf)) return rc;
    CU(dev_fill(h->clip_coef, n, 1.f));
    CU(cudaHostAlloc(h->gnorm_h.put(), sizeof(float) * kLossSlots * n, cudaHostAllocMapped));
    std::fill(h->gnorm_h.get(), h->gnorm_h.get() + kLossSlots * n, NAN);
    CU(cudaHostGetDevicePointer((void**)&h->gnorm_h_dev, h->gnorm_h, 0));
    CU(dev_alloc(h->gn_part, kGradNormMaxBlocks * n));
    CU(dev_fill(h->gn_ticket, n, 0));
  }
  {                           // ReDo record: scores NaN (all-ones bytes), flags 0
    for (int l = 0; l < cfg->n_actor_hidden; ++l) h->redo_n += cfg->actor_hidden[l];
    for (int l = 0; l < cfg->n_critic_hidden; ++l) h->redo_n += 2 * cfg->critic_hidden[l];
    const size_t n = (size_t)h->redo_n * R;
    double nan_ones;
    memset(&nan_ones, 0xFF, sizeof(nan_ones));
    CU(dev_fill(h->redo_score, n, nan_ones));
    CU(dev_fill(h->redo_flag, n, 0));
  }
  if (cfg->pcgrad) {          // switches on, weights 1, record NaN until a step writes it
    const int T = cfg->num_tasks;
    const size_t n2 = (size_t)2 * R;
    const int on[2] = {1, 1};
    if (int rc = h->pc_on.init(R, on)) return rc;
    CU(dev_alloc(h->pc_part, n2 * kGradNormMaxBlocks * pcgrad_pairs(T)));
    CU(dev_fill(h->pc_ticket, n2, 0));
    CU(dev_fill(h->pc_G, n2 * T * T, NAN));
    CU(dev_fill(h->pc_w, n2 * T, 1.f));
    CU(dev_fill(h->pc_perm, n2 * T * T, 0));
    CU(dev_fill(h->pc_mask, n2 * T, 0));
    CU(dev_fill(h->pc_bad, R, 0));
    const double off[2] = {0.0, 0.0};      // CAGrad off, its record NaN / -1 until a step runs it
    if (int rc = h->cg_c.init(R, off)) return rc;
    CU(dev_fill(h->cg_p, n2 * T, NAN));
    CU(dev_fill(h->cg_f, n2 * kCagScalars, NAN));
    CU(dev_fill(h->cg_it, n2, -1));
  }

  // work slab.  Buffers that a kernel addresses with one replica stride get one length: rsX (XQ, XT, XP), rsR (r, d, tid),
  // rsY (y, lq, la, qmin; the [2][B] q, dq, dqa, qt, qp take 2 * rsY), rsLogp (logp, logstd), rsDbg (dout_dbg, dact_dbg).
  SlabCarver slab{R};
  const int La = cfg->n_actor_hidden, Lc = cfg->n_critic_hidden;
  const size_t nX = (size_t)B * ldx, rsB = align_up(B, 64), nLogp = (size_t)2 * B, nDbg = (size_t)B * 2 * A;
  slab.request(h->XA, (size_t)2 * B * ldxa);
  for (Buf* b : {&h->XQ, &h->XT, &h->XP}) slab.request(*b, nX);
  for (Buf* b : {&h->r, &h->d, &h->tid}) slab.request(*b, rsB);
  slab.request(h->eps, (size_t)2 * B * A);
  slab.request(h->pout, (size_t)2 * B * 2 * A);
  slab.request(h->psave, (size_t)2 * B * A * kSaveW);
  slab.request(h->act_out, (size_t)2 * B * A);
  for (Buf* b : {&h->logp, &h->logstd}) slab.request(*b, nLogp);
  for (Buf* b : {&h->y, &h->lq, &h->la, &h->qmin}) slab.request(*b, rsB);
  const int E = h->E = cfg->critic_ensemble ? cfg->critic_ensemble : 2;
  for (Buf* b : {&h->q, &h->dq, &h->dqa, &h->qt, &h->qp}) slab.request(*b, E * rsB);
  slab.request(h->alpha, 64);
  slab.request(h->dxP, (size_t)E * B * ldx);
  for (Buf* b : {&h->dout_dbg, &h->dact_dbg}) slab.request(*b, nDbg);
  h->hA.resize(La); h->dhA.resize(La);
  for (int l = 0; l < La; ++l) {
    slab.request(h->hA[l], (size_t)2 * B * cfg->actor_hidden[l]);
    slab.request(h->dhA[l], (size_t)B * cfg->actor_hidden[l]);
  }
  for (CriticPass& p : h->pass) p.h.resize(Lc);
  h->dhQ.resize(Lc);
  for (int l = 0; l < Lc; ++l) {
    for (CriticPass& p : h->pass) slab.request(p.h[l], (size_t)E * B * cfg->critic_hidden[l]);
    slab.request(h->dhQ[l], (size_t)E * B * cfg->critic_hidden[l]);
  }
  if (cfg->care) {
    const int Kenc = cfg->num_encoders, T = cfg->num_tasks;
    auto pitch = [](int w) { return (w + 3) & ~3; };
    slab.request(h->XS, (size_t)2 * B * obs);
    // per-task table row: trunk activations per layer, attention, context-MLP activations per layer
    int off = 0;
    CareNet& tr = h->care_trunk;
    CareNet& cx = h->care_ctx;
    memset(&tr, 0, sizeof(tr)); memset(&cx, 0, sizeof(cx));
    const std::vector<LayerOff>& cxl = cfg->care == 2 ? L.cenc : L.ctx;      // CARE(O): the context net is the shared encoder
    tr.n = (int)L.trunk.size(); cx.n = (int)cxl.size();
    tr.dims[0] = cfg->care == 2 ? cfg->emb_dim : cfg->ctx_in;
    cx.dims[0] = cfg->ctx_in;
    for (int j = 0; j < tr.n; ++j) { tr.dims[j + 1] = L.trunk[j].out; tr.w[j] = L.trunk[j].w; tr.b[j] = L.trunk[j].b; tr.act_off[j] = off; off += L.trunk[j].out; }
    h->care_off_att = off; off += Kenc;
    for (int j = 0; j < cx.n; ++j) { cx.dims[j + 1] = cxl[j].out; cx.w[j] = cxl[j].w; cx.b[j] = cxl[j].b; cx.act_off[j] = off; off += cxl[j].out; }
    h->care_off_ctx = cx.act_off[cx.n - 1];
    h->care_row_w = off;
    for (int i = 0; i < 3; ++i) slab.request(h->careTab[i], (size_t)T * off);
    slab.request(h->careDtab, (size_t)T * (Kenc + cfg->ctx_out));
    slab.request(h->careDatt, (size_t)B * Kenc);
    const int rows_of[3] = {2 * B, B, B};
    for (int i = 0; i < 3; ++i) {
      h->mixH[i].resize(cfg->n_mix_hidden);
      for (int l = 0; l < cfg->n_mix_hidden; ++l) slab.request(h->mixH[i][l], (size_t)Kenc * rows_of[i] * pitch(cfg->mix_hidden[l]));
      slab.request(h->mixZ[i], (size_t)Kenc * rows_of[i] * pitch(cfg->mix_out));
    }
    h->mixDH.resize(cfg->n_mix_hidden);
    for (int l = 0; l < cfg->n_mix_hidden; ++l) slab.request(h->mixDH[l], (size_t)Kenc * B * pitch(cfg->mix_hidden[l]));
    slab.request(h->mixDZ, (size_t)Kenc * B * pitch(cfg->mix_out));
  }
  if (cfg->critic_ln) {
    for (CriticPass& p : h->pass) p.z.resize(Lc);
    int maxH = 0;
    for (int l = 0; l < Lc; ++l) {
      for (CriticPass& p : h->pass) slab.request(p.z[l], (size_t)E * B * cfg->critic_hidden[l]);
      maxH = std::max(maxH, cfg->critic_hidden[l]);
    }
    const size_t chunks = (size_t)(B + kLnRows - 1) / kLnRows;
    CU(dev_alloc(h->ln_part, R * E * chunks * 2 * maxH));
    CU(dev_fill(h->ln_ticket, (size_t)R * E, 0));
  }
  if (cfg->critic_dropout) {  // rate 0 on every replica; masks all zero until a step draws them
    for (CriticPass& p : h->pass) {
      p.m.resize(Lc);
      for (int l = 0; l < Lc; ++l) slab.request(p.m[l], (size_t)E * B * ((cfg->critic_hidden[l] + 31) / 32));
    }
    const double p0 = 0.0;
    if (int rc = h->drop.init(R, &p0)) return rc;
  }
  {  // ensembles: REDQ's and RLPD's defaults, a subset of 2 and the mean over the ensemble for the actor; twins: both
     // critics and the min, which the head kernels then compute as the twin step does
    slab.request(h->tsub, E);
    const int e0[2] = {2, cfg->critic_ensemble ? 1 : 0};
    if (int rc = h->ens.init(R, e0)) return rc;
  }
  if (int rc = slab.allocate(h->slab)) return rc;

  IngestOut& O = h->ing;
  O.XA = h->XA.p; O.XQ = h->XQ.p; O.XT = h->XT.p; O.XP = h->XP.p; O.r = h->r.p; O.d = h->d.p; O.eps = h->eps.p;
  O.tid = (int*)h->tid.p; O.cnt = h->cnt; O.ivl = h->ivl.dev;
  O.rsXA = h->XA.rs; O.rsXQ = h->XQ.rs; O.rsR = h->r.rs; O.rsEps = h->eps.rs;
  O.XS = cfg->care ? h->XS.p : nullptr; O.rsXS = cfg->care ? h->XS.rs : 0;
  O.log_alpha = h->params + L.off_alpha; O.rsP = L.arena; O.alpha = h->alpha.p; O.rsAlpha = h->alpha.rs;

  // parameter init: Xavier-uniform weights, zero biases (the memset above), LayerNorm weights 1, log_alpha = cfg;
  // targets = locals
  {
    for (const InitTensor& t : init_table(cfg, L)) {
      const uint64_t key = seed ^ t.seed_xor;
      if (t.kind == RESET_XAVIER) {
        xavier_kernel<<<dim3(64, R), 256>>>(h->params + t.off, L.arena, t.rows, t.cols, t.ld, key, t.tag);
      } else if (t.kind == RESET_RANDN) {
        randn_kernel<<<dim3(t.cols > 1 ? 64 : 8, R), 256>>>(h->params + t.off, L.arena, (long long)t.rows * t.cols, key, t.tag);
      } else if (t.kind == RESET_CONST || t.kind == RESET_ONES) {
        std::vector<float> la((size_t)t.rows, t.kind == RESET_ONES ? 1.0f : (float)cfg->log_alpha_init);
        for (int rep = 0; rep < R; ++rep)
          CU(cudaMemcpy(h->params + (size_t)rep * L.arena + t.off, la.data(), la.size() * sizeof(float), cudaMemcpyHostToDevice));
      }
    }
    polyak_kernel<<<dim3(128, R), 256>>>(h->params + L.critic_begin, L.arena, L.critic_n, L.target_delta, 1.0f, 0.0f);
    CU(cudaGetLastError());
  }

  // staging (pinned host <-> device), side stream
  h->row_w = row_fields(h).off[ROW_D] + 1;
  h->row_stride = (h->row_w + 31) / 32 * 32;   // 128-byte aligned transition rows
  h->stage_floats = (size_t)R * B * h->row_stride + (size_t)2 * R * B * A;   // rows + eps_next/eps_cur
  for (int i = 0; i < 2; ++i) {
    CU(cudaMallocHost(h->stage_h[i].put(), h->stage_floats * sizeof(float)));
    CU(dev_alloc(h->stage_d[i], h->stage_floats));
    CU(new_event(h->ev_copied[i]));
    CU(new_event(h->ev_consumed[i]));
  }
  CU(cudaHostAlloc(h->loss_h.put(), sizeof(float) * R * 4 * kLossSlots, cudaHostAllocMapped));
  memset(h->loss_h, 0, sizeof(float) * R * 4 * kLossSlots);
  CU(cudaHostGetDevicePointer((void**)&h->loss_h_dev, h->loss_h, 0));
  for (Stream* s : {&h->side, &h->own, &h->fork}) CU(new_stream(*s));
  for (Event* e : {&h->ev_ingested, &h->ev_sampled, &h->ev_fork_src, &h->ev_fork_done, &h->ev_in, &h->ev_out}) CU(new_event(*e));

  h->fused = fused_eligible(h);
  if (int rc = build_plan(h)) return rc;
  CU(cudaDeviceSynchronize());
  *out = owner.release();
  return 0;
}

extern "C" int b200sac_destroy(b200sac_t* h) {
  delete h;
  return 0;
}

static int arena_of(b200sac* h, int which, float** p, int64_t* n) {
  switch (which) {
    case B200SAC_PARAMS: *p = h->params; *n = h->L.arena; return 0;
    case B200SAC_ADAM_M: *p = h->adam_m; *n = h->L.trainable; return 0;
    case B200SAC_ADAM_V: *p = h->adam_v; *n = h->L.trainable; return 0;
    case B200SAC_GRADS: *p = h->grads; *n = h->L.trainable; return 0;
  }
  return fail(B200SAC_ERR_INVALID, "unknown arena %d", which);
}

extern "C" int b200sac_arena_ptr(b200sac_t* h, int32_t which, float** dev_ptr, int64_t* floats_per_replica) {
  if (!h || !dev_ptr || !floats_per_replica) return fail(B200SAC_ERR_INVALID, "null argument");
  return arena_of(h, which, dev_ptr, floats_per_replica);
}

extern "C" int b200sac_export(b200sac_t* h, int32_t which, int32_t replica, float* buf, int64_t n_floats, void* stream) {
  if (!h || !buf) return fail(B200SAC_ERR_INVALID, "null argument");
  float* p; int64_t n;
  if (int rc = arena_of(h, which, &p, &n)) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  if (n_floats != n) return fail(B200SAC_ERR_INVALID, "arena %d holds %lld floats per replica, got %lld", which, (long long)n, (long long)n_floats);
  CU(cudaSetDevice(h->device));
  CU(cudaMemcpyAsync(buf, p + (size_t)replica * n, n * sizeof(float), cudaMemcpyDefault, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  if (which == B200SAC_GRADS && h->gslices > 1) {       // split-K slices: the gradient is their sum (same order as Adam's)
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, buf) != cudaSuccess || at.type == cudaMemoryTypeDevice) {
      cudaGetLastError();
      return fail(B200SAC_ERR_INVALID, "exporting split-K gradients needs a host buffer");
    }
    std::vector<float> tmp((size_t)n);
    for (int sidx = 1; sidx < h->gslices; ++sidx) {
      CU(cudaMemcpy(tmp.data(), h->grads_x + ((size_t)(sidx - 1) * h->R + replica) * n, n * sizeof(float), cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; ++i) buf[i] += tmp[(size_t)i];
    }
  }
  return 0;
}

// A few floats of one arena (e.g. log_alpha for the logger) without exporting the whole arena.
extern "C" int b200sac_read_range(b200sac_t* h, int32_t which, int32_t replica, int64_t offset, int64_t n_floats, float* out_host,
                                  void* stream) {
  if (!h || !out_host) return fail(B200SAC_ERR_INVALID, "null argument");
  float* p; int64_t n;
  if (int rc = arena_of(h, which, &p, &n)) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  if (offset < 0 || n_floats < 1 || offset + n_floats > n) return fail(B200SAC_ERR_INVALID, "range [%lld, +%lld) outside the arena", (long long)offset, (long long)n_floats);
  CU(cudaSetDevice(h->device));
  CU(cudaMemcpyAsync(out_host, p + (size_t)replica * n + offset, (size_t)n_floats * sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int b200sac_import(b200sac_t* h, int32_t which, int32_t replica, const float* buf, int64_t n_floats, void* stream) {
  if (!h || !buf) return fail(B200SAC_ERR_INVALID, "null argument");
  float* p; int64_t n;
  if (int rc = arena_of(h, which, &p, &n)) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  if (n_floats != n) return fail(B200SAC_ERR_INVALID, "arena %d holds %lld floats per replica, got %lld", which, (long long)n, (long long)n_floats);
  CU(cudaSetDevice(h->device));
  CU(cudaMemcpyAsync(p + (size_t)replica * n, buf, n * sizeof(float), cudaMemcpyDefault, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int b200sac_get_steps(b200sac_t* h, int32_t replica, int64_t steps[4]) {
  if (!h || !steps) return fail(B200SAC_ERR_INVALID, "bad argument");
  if (int rc = check_replica(h, replica)) return rc;
  CU(cudaSetDevice(h->device));
  Counters c;
  CU(cudaMemcpy(&c, h->cnt + replica, sizeof(c), cudaMemcpyDeviceToHost));
  steps[0] = c.v[0]; steps[1] = c.v[1]; steps[2] = c.v[2]; steps[3] = c.v[4];
  return 0;
}

extern "C" int b200sac_set_steps(b200sac_t* h, int32_t replica, const int64_t steps[4]) {
  if (!h || !steps) return fail(B200SAC_ERR_INVALID, "bad argument");
  if (int rc = check_replica(h, replica)) return rc;
  CU(cudaSetDevice(h->device));
  Counters c;
  CU(cudaMemcpy(&c, h->cnt + replica, sizeof(c), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 4; ++i) {
    const int slot = i == 3 ? 4 : i;
    c.v[slot] = steps[i];
    c.b1p[slot] = pow(h->cfg.beta1, (double)steps[i]);
    c.b2p[slot] = pow(h->cfg.beta2, (double)steps[i]);
  }
  CU(cudaMemcpy(h->cnt + replica, &c, sizeof(c), cudaMemcpyHostToDevice));
  return 0;
}

// The legacy default stream cannot be captured into a graph.  When the caller passes it (NULL,
// which is also torch's default current stream) the step runs on the handle's own stream,
// ordered after everything already queued on the caller's stream, and the caller's stream is
// made to wait for it afterwards -- same ordering semantics, capturable.
struct StreamBridge {
  b200sac* h;
  cudaStream_t user, run;
  bool bridged;
  StreamBridge(b200sac* h_, void* s) : h(h_), user((cudaStream_t)s) {
    bridged = (user == nullptr || user == cudaStreamLegacy || user == cudaStreamPerThread);
    run = bridged ? h->own : user;
  }
  int begin() {
    if (!bridged) return 0;
    CU(cudaEventRecord(h->ev_in, user));
    CU(cudaStreamWaitEvent(run, h->ev_in, 0));
    return 0;
  }
  int end() {
    if (!bridged) return 0;
    CU(cudaEventRecord(h->ev_out, run));
    CU(cudaStreamWaitEvent(user, h->ev_out, 0));
    return 0;
  }
};

// ------------------------------------------------------------------------------------------
// Per-replica settings (ReplicaTable): replicas of one handle can train with different values, and a value can change
// between steps.  Each entry point checks its own arguments and leaves the write, its ordering and the mirror to the table.
// ------------------------------------------------------------------------------------------
// t = floor(p * 2^32) and s = 1 / (1 - p), both in fp64, s rounded to fp32 once
static DropRate drop_rate(double p) { return DropRate{(unsigned)floor(p * 4294967296.0), (float)(1.0 / (1.0 - p))}; }

template <class T, class Mirror> static T device_value(const Mirror& v) {
  if constexpr (std::is_same_v<T, Mirror>) return v;
  else if constexpr (std::is_same_v<T, DropRate>) return drop_rate(v);
  else return hparams_row(v);
}

template <class T, int N, class Mirror>
int ReplicaTable<T, N, Mirror>::init(int R, const Mirror* v) {
  ReplicaTable t;
  std::vector<T> rows((size_t)R * N);
  for (size_t i = 0; i < rows.size(); ++i) {
    t.host.push_back(v[i % N]);
    rows[i] = device_value<T>(v[i % N]);
  }
  CU(dev_copy(t.dev, rows.data(), rows.size()));
  *this = std::move(t);
  return 0;
}

template <class T, int N, class Mirror>
int ReplicaTable<T, N, Mirror>::set(b200sac* h, void* stream, int replica, const Mirror* v, cudaEvent_t written) {
  TableRow<T, N> row;
  for (int i = 0; i < N; ++i) row.v[i] = device_value<T>(v[i]);
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  write_row_kernel<<<1, 1, 0, sb.run>>>(dev.get(), replica, row);
  CU(cudaGetLastError());
  if (written) CU(cudaEventRecord(written, sb.run));
  if (int rc = sb.end()) return rc;
  std::copy(v, v + N, host.begin() + (size_t)replica * N);
  return 0;
}

extern "C" int b200sac_get_hparams(b200sac_t* h, int32_t replica, b200sac_hparams* out) {
  if (!h || !out) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = h->hp.check(replica)) return rc;
  *out = *h->hp.row(replica);
  return 0;
}

extern "C" int b200sac_set_hparams(b200sac_t* h, int32_t replica, const b200sac_hparams* hp, void* stream) {
  if (!h || !hp) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = h->hp.check(replica)) return rc;
  const double all[8] = {hp->gamma, hp->reward_scale, hp->tau, hp->lr_critic, hp->lr_actor, hp->lr_alpha, hp->tau_se, hp->lr_ctx};
  for (double x : all)
    if (!std::isfinite(x)) return fail(B200SAC_ERR_INVALID, "hyperparameters must be finite");
  if (hp->tau < 0.0 || hp->tau > 1.0 || hp->tau_se < 0.0 || hp->tau_se > 1.0)
    return fail(B200SAC_ERR_INVALID, "0 <= tau, tau_se <= 1 required (got %g, %g)", hp->tau, hp->tau_se);
  if (hp->lr_critic < 0.0 || hp->lr_actor < 0.0 || hp->lr_alpha < 0.0 || hp->lr_ctx < 0.0)
    return fail(B200SAC_ERR_INVALID, "learning rates must be >= 0");
  return h->hp.set(h, stream, replica, hp);
}

// Per-replica update intervals: the ingest of each step turns them and the critic's step count into the step's schedule
// (Counters::sched).
extern "C" int b200sac_get_update_intervals(b200sac_t* h, int32_t replica, int32_t* actor_every, int32_t* target_every) {
  if (!h || !actor_every || !target_every) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = h->ivl.check(replica)) return rc;
  *actor_every = h->ivl.row(replica)[0];
  *target_every = h->ivl.row(replica)[1];
  return 0;
}

extern "C" int b200sac_set_update_intervals(b200sac_t* h, int32_t replica, int32_t actor_every, int32_t target_every, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = h->ivl.check(replica)) return rc;
  constexpr int32_t kMaxEvery = 1 << 30;
  if (actor_every < 1 || actor_every > kMaxEvery || target_every < 1 || target_every > kMaxEvery)
    return fail(B200SAC_ERR_INVALID, "update intervals must be in [1, 2^30] (got actor %d, target %d)", actor_every, target_every);
  const int v[2] = {actor_every, target_every};
  return h->ivl.set(h, stream, replica, v);
}

// Gradient-norm clipping thresholds, read by the grad_norm launches of the step graphs.
extern "C" int b200sac_get_grad_clip(b200sac_t* h, int32_t replica, double* critic, double* actor, double* ctx) {
  if (!h || !critic || !actor || !ctx) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.grad_clip, "grad_clip")) return rc;
  if (int rc = h->clip_thr.check(replica)) return rc;
  const double* t = h->clip_thr.row(replica);
  *critic = t[0]; *actor = t[1]; *ctx = t[2];
  return 0;
}

extern "C" int b200sac_set_grad_clip(b200sac_t* h, int32_t replica, double critic, double actor, double ctx, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.grad_clip, "grad_clip")) return rc;
  if (int rc = h->clip_thr.check(replica)) return rc;
  if (!(critic > 0.0) || !(actor > 0.0) || !(ctx > 0.0))       // (NaN fails every comparison)
    return fail(B200SAC_ERR_INVALID, "gradient-norm thresholds must be > 0 (+inf: no clipping), got %g, %g, %g", critic, actor, ctx);
  const double v[kClipCols] = {critic, actor, ctx};
  return h->clip_thr.set(h, stream, replica, v);
}

// Critic dropout rates, read by the dropout LayerNorm launches of the step graphs.
extern "C" int b200sac_get_critic_dropout(b200sac_t* h, int32_t replica, double* p) {
  if (!h || !p) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.critic_dropout, "critic_dropout")) return rc;
  if (int rc = h->drop.check(replica)) return rc;
  *p = *h->drop.row(replica);
  return 0;
}

extern "C" int b200sac_set_critic_dropout(b200sac_t* h, int32_t replica, double p, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.critic_dropout, "critic_dropout")) return rc;
  if (int rc = h->drop.check(replica)) return rc;
  if (!(p >= 0.0 && p < 1.0))                                   // (NaN fails every comparison)
    return fail(B200SAC_ERR_INVALID, "the critic dropout rate must be in [0, 1), got %g", p);
  return h->drop.set(h, stream, replica, &p);
}

// Target subset size and actor reduction of an ensemble handle, read by its head launches.
extern "C" int b200sac_get_ensemble(b200sac_t* h, int32_t replica, int32_t* m, int32_t* actor_mean) {
  if (!h || !m || !actor_mean) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.critic_ensemble, "critic_ensemble")) return rc;
  if (int rc = h->ens.check(replica)) return rc;
  *m = h->ens.row(replica)[0]; *actor_mean = h->ens.row(replica)[1];
  return 0;
}

extern "C" int b200sac_set_ensemble(b200sac_t* h, int32_t replica, int32_t m, int32_t actor_mean, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.critic_ensemble, "critic_ensemble")) return rc;
  if (int rc = h->ens.check(replica)) return rc;
  if (m < 1 || m > h->E) return fail(B200SAC_ERR_INVALID, "the target subset size must be in [1, %d], got %d", h->E, m);
  if (actor_mean != 0 && actor_mean != 1) return fail(B200SAC_ERR_INVALID, "actor_mean must be 0 (min) or 1 (mean), got %d", actor_mean);
  const int row[2] = {m, actor_mean};
  return h->ens.set(h, stream, replica, row);
}

// Gradient-surgery switches, read by the pcgrad launches of the step graphs.
extern "C" int b200sac_get_pcgrad(b200sac_t* h, int32_t replica, int32_t* critic_on, int32_t* actor_on) {
  if (!h || !critic_on || !actor_on) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = h->pc_on.check(replica)) return rc;
  *critic_on = h->pc_on.row(replica)[0]; *actor_on = h->pc_on.row(replica)[1];
  return 0;
}

extern "C" int b200sac_set_pcgrad(b200sac_t* h, int32_t replica, int32_t critic_on, int32_t actor_on, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = h->pc_on.check(replica)) return rc;
  if ((critic_on != 0 && critic_on != 1) || (actor_on != 0 && actor_on != 1))
    return fail(B200SAC_ERR_INVALID, "pcgrad switches must be 0 or 1, got %d, %d", critic_on, actor_on);
  const int v[2] = {critic_on, actor_on};
  return h->pc_on.set(h, stream, replica, v);
}

extern "C" int b200sac_read_pcgrad(b200sac_t* h, int32_t replica, double* gram, float* w, int32_t* perm, uint64_t* mask,
                                   int32_t* task_mismatch, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  const size_t T = (size_t)h->cfg.num_tasks, r2 = (size_t)replica * 2;
  CU(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  CU(cudaStreamSynchronize(st));
  if (gram) CU(cudaMemcpy(gram, h->pc_G + r2 * T * T, sizeof(double) * 2 * T * T, cudaMemcpyDeviceToHost));
  if (w) CU(cudaMemcpy(w, h->pc_w + r2 * T, sizeof(float) * 2 * T, cudaMemcpyDeviceToHost));
  if (perm) CU(cudaMemcpy(perm, h->pc_perm + r2 * T * T, sizeof(int) * 2 * T * T, cudaMemcpyDeviceToHost));
  if (mask) CU(cudaMemcpy(mask, h->pc_mask + r2 * T, sizeof(uint64_t) * 2 * T, cudaMemcpyDeviceToHost));
  if (task_mismatch) CU(cudaMemcpy(task_mismatch, h->pc_bad + replica, sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}

// CAGrad coefficients, read by the pcgrad launches of the step graphs.
extern "C" int b200sac_get_cagrad(b200sac_t* h, int32_t replica, double* c_critic, double* c_actor) {
  if (!h || !c_critic || !c_actor) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = h->cg_c.check(replica)) return rc;
  *c_critic = h->cg_c.row(replica)[0]; *c_actor = h->cg_c.row(replica)[1];
  return 0;
}

extern "C" int b200sac_set_cagrad(b200sac_t* h, int32_t replica, double c_critic, double c_actor, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = h->cg_c.check(replica)) return rc;
  if (!(c_critic >= 0.0) || !(c_actor >= 0.0) || std::isinf(c_critic) || std::isinf(c_actor))   // (NaN fails >=)
    return fail(B200SAC_ERR_INVALID, "CAGrad coefficients must be finite and >= 0, got %g, %g", c_critic, c_actor);
  const double v[2] = {c_critic, c_actor};
  return h->cg_c.set(h, stream, replica, v);
}

extern "C" int b200sac_read_cagrad(b200sac_t* h, int32_t replica, double* p, double* lambda, double* best, double* first,
                                   double* scale, int32_t* ibest, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  const size_t T = (size_t)h->cfg.num_tasks, r2 = (size_t)replica * 2;
  CU(cudaSetDevice(h->device));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  double f[2][kCagScalars];
  CU(cudaMemcpy(f, h->cg_f + r2 * kCagScalars, sizeof(f), cudaMemcpyDeviceToHost));
  if (p) CU(cudaMemcpy(p, h->cg_p + r2 * T, sizeof(double) * 2 * T, cudaMemcpyDeviceToHost));
  if (ibest) CU(cudaMemcpy(ibest, h->cg_it + r2, sizeof(int) * 2, cudaMemcpyDeviceToHost));
  double* outs[kCagScalars] = {lambda, best, first, scale};
  for (int k = 0; k < kCagScalars; ++k)
    if (outs[k]) for (int o = 0; o < 2; ++o) outs[k][o] = f[o][k];
  return 0;
}

// Stand-alone CAGrad solve (cagrad_test_kernel) on a HOST G [T][T] on the current device, like b200sac_gemm_test; outputs
// as in b200sac_read_cagrad for one optimizer.
extern "C" int b200sac_cagrad_solve_test(int32_t T, const double* G, double c, float* w, double* p, double* lambda,
                                         double* best, double* first, double* scale, int32_t* ibest) {
  if (!G || !w || T < 1 || T > kPcMaxTasks) return fail(B200SAC_ERR_INVALID, "bad argument (T in [1, %d], G and w non-null)", kPcMaxTasks);
  if (!(c > 0.0) || std::isinf(c)) return fail(B200SAC_ERR_INVALID, "c must be finite and > 0, got %g", c);
  const size_t nG = (size_t)T * T;
  DevMem<double> dG, dp, df;
  DevMem<float> dw;
  DevMem<int> di;
  CU(dev_copy(dG, G, nG)); CU(dev_alloc(dp, T)); CU(dev_alloc(df, kCagScalars)); CU(dev_alloc(dw, T)); CU(dev_alloc(di, 1));
  cagrad_test_kernel<<<1, 32, sizeof(double) * (nG + kCagVecs * T), cudaStreamLegacy>>>(dG, T, c, CagOut{dw, dp, df, di});
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(cudaStreamLegacy));
  double f[kCagScalars];
  CU(cudaMemcpy(w, dw, sizeof(float) * T, cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(f, df, sizeof(f), cudaMemcpyDeviceToHost));
  if (p) CU(cudaMemcpy(p, dp, sizeof(double) * T, cudaMemcpyDeviceToHost));
  if (ibest) CU(cudaMemcpy(ibest, di, sizeof(int), cudaMemcpyDeviceToHost));
  double* outs[kCagScalars] = {lambda, best, first, scale};
  for (int k = 0; k < kCagScalars; ++k)
    if (outs[k]) *outs[k] = f[k];
  return 0;
}

extern "C" int b200sac_export_task_grad(b200sac_t* h, int32_t replica, int32_t task, float* buf, int64_t n_floats, void* stream) {
  if (!h || !buf) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.pcgrad, "pcgrad")) return rc;
  if (int rc = check_replica(h, replica)) return rc;
  if (task < 0 || task >= h->cfg.num_tasks) return fail(B200SAC_ERR_INVALID, "task %d out of range", task);
  const int64_t n = h->L.trainable;
  if (n_floats != n) return fail(B200SAC_ERR_INVALID, "the gradient arena holds %lld floats per replica, got %lld", (long long)n, (long long)n_floats);
  const float* src = task == 0 ? h->grads.get() : h->grads_x + (size_t)(task - 1) * h->R * n;
  CU(cudaSetDevice(h->device));
  CU(cudaMemcpyAsync(buf, src + (size_t)replica * n, n * sizeof(float), cudaMemcpyDefault, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int b200sac_copy_replica(b200sac_t* h, int32_t src, int32_t dst, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (src < 0 || src >= h->R || dst < 0 || dst >= h->R)
    return fail(B200SAC_ERR_INVALID, "replicas %d -> %d out of range (%d in the handle)", src, dst, h->R);
  if (src == dst) return 0;
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  const size_t na = (size_t)h->L.arena, nt = (size_t)h->L.trainable;
  CU(cudaMemcpyAsync(h->params + dst * na, h->params + src * na, na * sizeof(float), cudaMemcpyDeviceToDevice, sb.run));
  CU(cudaMemcpyAsync(h->adam_m + dst * nt, h->adam_m + src * nt, nt * sizeof(float), cudaMemcpyDeviceToDevice, sb.run));
  CU(cudaMemcpyAsync(h->adam_v + dst * nt, h->adam_v + src * nt, nt * sizeof(float), cudaMemcpyDeviceToDevice, sb.run));
  CU(cudaMemcpyAsync(h->cnt + dst, h->cnt + src, sizeof(Counters), cudaMemcpyDeviceToDevice, sb.run));
  return sb.end();
}

extern "C" int b200sac_reset(b200sac_t* h, int32_t replica, const b200sac_reset_spec* spec, uint64_t seed, void* stream) {
  if (!h || !spec) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = check_replica(h, replica)) return rc;
  static const char* const kPart[B200SAC_RESET_PARTS] = {"actor", "critic", "alpha", "encoder", "context"};
  for (int p = 0; p < B200SAC_RESET_PARTS; ++p) {
    const b200sac_reset_part& q = spec->part[p];
    if (q.layers < 0 || (p >= B200SAC_RESET_ALPHA && q.layers > 1))
      return fail(B200SAC_ERR_INVALID, "%s: layers %d out of range", kPart[p], q.layers);
    if (!(q.shrink >= 0.0 && q.shrink <= 1.0))       // (NaN fails both)
      return fail(B200SAC_ERR_INVALID, "%s: shrink must be in [0, 1], got %g", kPart[p], q.shrink);
  }
  const b200sac_cfg& c = h->cfg;
  if (spec->part[B200SAC_RESET_ENCODER].layers && !c.care) return fail(B200SAC_ERR_INVALID, "encoder reset on a handle without CARE");
  if (spec->part[B200SAC_RESET_CONTEXT].layers && c.care != 2)
    return fail(B200SAC_ERR_INVALID, "context reset on a handle that is not CARE(O)");

  const Layout& L = h->L;
  ResetArgs A;
  memset(&A, 0, sizeof(A));
  A.params = h->params + (size_t)replica * L.arena;
  A.target_delta = L.target_delta;
  A.key = seed + (uint64_t)replica;
  for (int p = 0; p < B200SAC_RESET_PARTS; ++p) A.shrink[p] = spec->part[p].shrink;
  // the touched tensors, kResetMaxTensors per launch (critic ensembles can have more)
  std::vector<ResetTensor> ts;
  long long widest = 0;
  for (const InitTensor& t : init_table(&c, L)) {
    if (t.part < 0) continue;
    const int layers = spec->part[t.part].layers;
    if (layers == 0 || t.depth > layers) continue;
    ResetTensor r;
    memset(&r, 0, sizeof(r));
    r.off = t.off; r.rows = t.rows; r.cols = t.cols; r.ld = t.ld;
    r.kind = (unsigned char)t.kind; r.part = (unsigned char)t.part; r.target = t.target ? 1 : 0;
    r.tag = t.tag; r.c0 = t.kind == RESET_ONES ? 1.0f : (float)c.log_alpha_init;
    widest = std::max(widest, (long long)t.rows * t.cols);
    ts.push_back(r);
  }
  const int n = (int)ts.size();
  // optimizers that own a touched tensor: {counter slot, first trainable float, floats}
  struct Owner { int slot; int64_t begin, n; };
  std::vector<Owner> owners;
  if (spec->part[B200SAC_RESET_CRITIC].layers || spec->part[B200SAC_RESET_ENCODER].layers)
    owners.push_back({0, L.critic_begin, L.critic_n});
  if (spec->part[B200SAC_RESET_ACTOR].layers) owners.push_back({1, L.actor_begin, L.actor_n});
  if (spec->part[B200SAC_RESET_ALPHA].layers) owners.push_back({2, L.off_alpha, c.num_tasks > 0 ? c.num_tasks : 1});
  if (spec->part[B200SAC_RESET_CONTEXT].layers) owners.push_back({4, L.cenc_begin, L.cenc_n});
  if (n == 0) return 0;

  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  const unsigned bx = (unsigned)std::min<long long>(64, (widest + 255) / 256);
  for (int i0 = 0; i0 < n; i0 += kResetMaxTensors) {
    const int k = std::min(n - i0, kResetMaxTensors);
    std::copy(ts.begin() + i0, ts.begin() + i0 + k, A.t);
    reset_kernel<<<dim3(bx, k), 256, 0, sb.run>>>(A);
    CU(cudaGetLastError());
  }
  int slots = 0;
  const size_t nt = (size_t)L.trainable;
  for (const Owner& o : owners) {
    CU(cudaMemsetAsync(h->adam_m + replica * nt + o.begin, 0, o.n * sizeof(float), sb.run));
    CU(cudaMemsetAsync(h->adam_v + replica * nt + o.begin, 0, o.n * sizeof(float), sb.run));
    slots |= 1 << o.slot;
  }
  reset_counters_kernel<<<1, 1, 0, sb.run>>>(h->cnt + replica, slots);
  CU(cudaGetLastError());
  return sb.end();
}

// ------------------------------------------------------------------------------------------
// Blob publication.  What Learner.run() stores in Redis after every update is ONE byte string: _pickle.dumps of
// {'actor': state_dict} (LunarLander_Distributed_SAC/src/learner.py:272-276,298-299).  Its shape never changes, so the
// caller hands over the byte image once (b200sac_blob_template: constant pickle bytes + where every payload float sits and
// which arena element it is -- pitch padding and the CARE [k][out][in] -> [k][in][out] transposition are just index maps);
// per publication a kernel, in stream order between two steps, gathers the floats into a device copy of the image, one
// D2H copy on the private stream brings it to pinned memory, and the host's only work is handing the bytes on.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) blob_pack_kernel(const float* __restrict__ params, const int* __restrict__ src,
                                                        const int* __restrict__ dst, uint8_t* __restrict__ img, int n) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= n) return;
  const uint32_t v = __float_as_uint(params[src[j]]);
  uint8_t* o = img + dst[j];
  if ((reinterpret_cast<uintptr_t>(o) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(o) = v;
  } else {                                  // pickle payloads start at arbitrary byte offsets
    o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); o[2] = (uint8_t)(v >> 16); o[3] = (uint8_t)(v >> 24);
  }
}

extern "C" int b200sac_blob_template(b200sac_t* h, int32_t replica, const uint8_t* image, int64_t image_bytes, int64_t n_floats,
                                     const int32_t* src_index, const int32_t* dst_byte) {
  if (!h || !image || image_bytes <= 0 || n_floats <= 0 || !src_index || !dst_byte) return fail(B200SAC_ERR_INVALID, "bad argument");
  if (int rc = check_replica(h, replica)) return rc;
  if (n_floats > 0x7fffffffLL || image_bytes > 0x7fffffffLL) return fail(B200SAC_ERR_INVALID, "image too large");
  for (int64_t j = 0; j < n_floats; ++j) {
    if (src_index[j] < 0 || src_index[j] >= h->L.arena) return fail(B200SAC_ERR_INVALID, "payload float %lld reads arena index %d outside [0, %lld)", (long long)j, src_index[j], (long long)h->L.arena);
    if (dst_byte[j] < 0 || (int64_t)dst_byte[j] + 4 > image_bytes) return fail(B200SAC_ERR_INVALID, "payload float %lld lands outside the image", (long long)j);
  }
  CU(cudaSetDevice(h->device));
  // All or nothing: the stream and events are created once, together; the new images and index maps are built aside and
  // replace the old ones only when all of them exist, so a failed call leaves the previous template working.
  if (!h->pub) {
    Stream pub;
    Event snap[2], done[2];
    CU(new_stream(pub));
    for (int i = 0; i < 2; ++i) {
      CU(new_event(snap[i]));
      CU(new_event(done[i]));
    }
    h->pub = std::move(pub);
    for (int i = 0; i < 2; ++i) { h->ev_blob_snap[i] = std::move(snap[i]); h->ev_blob_done[i] = std::move(done[i]); }
  }
  DevMem<uint8_t> img_d[2];
  PinnedMem<uint8_t> img_h[2];
  DevMem<int> src, dst;
  for (int i = 0; i < 2; ++i) {
    CU(dev_copy(img_d[i], image, (size_t)image_bytes));
    CU(cudaHostAlloc(img_h[i].put(), (size_t)image_bytes, cudaHostAllocDefault));
  }
  CU(dev_copy(src, src_index, (size_t)n_floats));
  CU(dev_copy(dst, dst_byte, (size_t)n_floats));
  CU(cudaStreamSynchronize(h->pub));             // no copy of the old images is in flight
  for (int i = 0; i < 2; ++i) { std::swap(h->blob_d[i], img_d[i]); std::swap(h->blob_h[i], img_h[i]); }
  std::swap(h->blob_src, src);
  std::swap(h->blob_dst, dst);
  h->blob_bytes = image_bytes; h->blob_nf = n_floats; h->blob_replica = replica;
  h->blob_head = 0; h->blob_pending = 0;
  return 0;
}

extern "C" int b200sac_blob_begin(b200sac_t* h, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (h->blob_nf <= 0) return fail(B200SAC_ERR_STATE, "blob_begin without blob_template");
  CU(cudaSetDevice(h->device));
  if (h->blob_pending == 2) {           // both images hold uncollected blobs: the older one is superseded
    CU(cudaEventSynchronize(h->ev_blob_done[h->blob_head]));
    h->blob_pending = 1;
  }
  const int slot = h->blob_head;
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  // (slot reuse: the D2H of the blob begun two calls ago was collected or superseded above, so image `slot` is idle)
  const float* base = h->params + (size_t)h->blob_replica * h->L.arena;
  blob_pack_kernel<<<(unsigned)((h->blob_nf + 255) / 256), 256, 0, sb.run>>>(base, h->blob_src, h->blob_dst, h->blob_d[slot], (int)h->blob_nf);
  CU(cudaGetLastError());
  CU(cudaEventRecord(h->ev_blob_snap[slot], sb.run));
  if (int rc = sb.end()) return rc;
  CU(cudaStreamWaitEvent(h->pub, h->ev_blob_snap[slot], 0));
  CU(cudaMemcpyAsync(h->blob_h[slot], h->blob_d[slot], (size_t)h->blob_bytes, cudaMemcpyDeviceToHost, h->pub));
  CU(cudaEventRecord(h->ev_blob_done[slot], h->pub));
  h->blob_head ^= 1;
  h->blob_pending += 1;
  return 0;
}

extern "C" int b200sac_blob_wait(b200sac_t* h, const uint8_t** host_ptr, int64_t* n_bytes) {
  if (!h || !host_ptr || !n_bytes) return fail(B200SAC_ERR_INVALID, "null argument");
  if (h->blob_pending <= 0) return fail(B200SAC_ERR_STATE, "blob_wait without blob_begin");
  CU(cudaSetDevice(h->device));
  const int slot = (h->blob_head + 2 - h->blob_pending) & 1;    // the oldest blob not collected yet
  CU(cudaEventSynchronize(h->ev_blob_done[slot]));
  h->blob_pending -= 1;
  *host_ptr = h->blob_h[slot];
  *n_bytes = h->blob_bytes;
  return 0;
}

static int ring_ready(const b200sac_replay* rb, int replica, int batches);

// A ring's lock and, while it has a prior, the prior's as well, for the entry points that enqueue steps from the ring.  The
// two are taken together (std::lock), never one while waiting for the other, and the prior is read again under both: an
// attach or detach may have run in between.
struct RingLocks {
  std::unique_lock<std::mutex> own, pri;
  explicit RingLocks(b200sac_replay* rb) : own(rb->mu) {
    while (b200sac_replay* p = rb->prior) {
      own.unlock();
      pri = std::unique_lock<std::mutex>(p->mu, std::defer_lock);
      std::lock(own, pri);
      if (rb->prior == p) return;
      pri.unlock();
    }
  }
};

// (under RingLocks) Every replica that draws prior rows finds every task sub-ring of the prior ready (ring_ready's rule).
static int prior_ready(const b200sac_replay* rb) {
  if (!rb->prior) return 0;
  for (int rep = 0; rep < rb->h->R; ++rep)
    if (*rb->prior_rows.row(rep) > 0)
      if (int rc = ring_ready(rb->prior, rep, 4)) return rc;
  return 0;
}

// (under RingLocks) The steps just enqueued on `st` read the ring and its prior: a writer of either waits for them.
static int record_gather(b200sac_replay* rb, cudaStream_t st) {
  for (b200sac_replay* x : {rb, rb->prior}) {
    if (!x) continue;
    CU(cudaEventRecord(x->ev_gather, st));
    x->gather_pending = true;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// the step: from packed rows (a staging slot or b200sac_step's buffer) or sampled from a device ring
// ------------------------------------------------------------------------------------------
// ring sampling modes (multi-step graphs): SAMPLE_INLINE = sample on `st` right before the gather (one step per graph);
// SAMPLE_DONE = the indices of this step were already drawn on the fork stream (wait for them); `fork_next` = once this
// step's gather has consumed the index buffer and bumped the step counter, draw the NEXT step's indices on the fork stream
// -- that kernel then overlaps the whole step instead of heading its critical path.
enum { SAMPLE_INLINE = 0, SAMPLE_DONE = 1 };
static NstepRing nstep_ring(const b200sac_replay* rb) {
  NstepRing N;
  N.link = rb->d_link; N.nstep = rb->nstep.dev; N.cap = rb->cap; N.cap_per_task = (int)rb->cap_per_task;
  return N;
}

static int enqueue_body(b200sac* h, cudaStream_t st, const GraphKey& key, const Event* evs = nullptr,
                        int sample_mode = SAMPLE_INLINE, bool fork_next = false) {
  if (evs) CU(cudaEventRecord(evs[0], st));
  const int B = h->cfg.batch, R = h->R;
  dim3 grid((B + 7) / 8, R), block(256);
  if (grid.x > 64) grid.x = 64;
  b200sac_replay* rb = key.ring;
  if (!rb) {
    launch_k(ingest_rows_kernel, grid, block, 0, 1, st, h->K, h->ing, key.rows, (long long)B * h->row_stride, h->row_stride,
             (const int*)nullptr, (long long)0);
    if (key.eps && key.eps != h->eps.p) {      // staged eps, [R][B][A] next, then [R][B][A] cur: into the step's buffer
      const float* e = key.eps;
      const size_t n = (size_t)B * h->cfg.act_dim * sizeof(float);
      for (int rep = 0; rep < R; ++rep) {
        CU(cudaMemcpyAsync(h->eps.p + rep * h->eps.rs, e + (size_t)rep * B * h->cfg.act_dim, n, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(h->eps.p + rep * h->eps.rs + (size_t)B * h->cfg.act_dim,
                           e + (size_t)(R + rep) * B * h->cfg.act_dim, n, cudaMemcpyDeviceToDevice, st));
      }
    }
  } else {
    auto sample_on = [&](cudaStream_t s2) {
      if (rb->per) return per_sample_on(h, rb, s2);
      if (rb->prior)
        return launch_k(sample_mixed_kernel, dim3(R), dim3(B > 256 ? 512 : 256), 0, 1, s2, h->K, (const Counters*)h->cnt,
                        (const long long*)rb->d_fill, rb->cap_per_task, rb->d_idx.get(), (long long)B, rb->seed,
                        PriorDraw{rb->prior_rows.dev, rb->prior->d_fill, rb->prior->cap_per_task, rb->prior->seed});
      return launch_k(sample_indices_kernel, dim3(R), dim3(B > 256 ? 512 : 256), 0, 1, s2, h->K,   // __launch_bounds__(512): 512 threads fit
                      (const Counters*)h->cnt, (const long long*)rb->d_fill, rb->cap_per_task, rb->d_idx.get(), (long long)B, rb->seed);
    };
    if (sample_mode == SAMPLE_INLINE) sample_on(st);
    else CU(cudaStreamWaitEvent(st, h->ev_sampled, 0));
    if (rb->traj)                               // linked ring: the same gather with the n-step fold in front of the scatter
      launch_k(ingest_nstep_kernel, grid, block, 0, 1, st, h->K, h->ing, (const float*)rb->rows, rb->rs_rows, h->row_stride,
               (const int*)rb->d_idx, (long long)B, nstep_ring(rb), h->ns_buf.get());
    else if (rb->prior)                         // ring with a prior: online and prior rows through one encoded index
      launch_k(ingest_mixed_kernel, grid, block, 0, 1, st, h->K, h->ing, (const float*)rb->rows, rb->rs_rows,
               (const float*)rb->prior->rows, rb->prior->rs_rows, h->row_stride, (const int*)rb->d_idx, (long long)B,
               h->mix_idx.get());
    else
      launch_k(ingest_rows_kernel, grid, block, 0, 1, st, h->K, h->ing, (const float*)rb->rows, rb->rs_rows, h->row_stride,
               (const int*)rb->d_idx, (long long)B);
    if (fork_next && !rb->per) {                // (prioritized: the next draw follows this step's priority update)
      CU(cudaEventRecord(h->ev_ingested, st));
      CU(cudaStreamWaitEvent(h->fork, h->ev_ingested, 0));
      sample_on(h->fork);
      CU(cudaEventRecord(h->ev_sampled, h->fork));
    }
  }
  CU(cudaGetLastError());
  return run_plan(h, st, key.eps != nullptr, evs ? evs + 1 : nullptr, evs == nullptr && !key.stamping, rb,
                  rb && rb->per && fork_next);
}

// nsteps > 1 (device-ring sampling only): that many consecutive gradient steps captured in ONE graph, so a pipelined
// run pays the graph-launch gap (a few us between two graph launches) once per graph.  A run of n steps is cut
// greedily into graphs of 8, 4, 2 and 1 steps.
constexpr int kGraphSteps = 8;
static int get_graph(b200sac* h, cudaStream_t st, const GraphKey& key, cudaGraphExec_t* out) {
  auto it = h->graphs.find(key);
  if (it == h->graphs.end()) {
    const int nsteps = key.nsteps;
    Graph g;
    CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = 0;
    for (int k = 0; k < nsteps && rc == 0; ++k)
      rc = enqueue_body(h, st, key, nullptr, (nsteps > 1 && k > 0) ? SAMPLE_DONE : SAMPLE_INLINE, nsteps > 1 && k + 1 < nsteps);
    cudaError_t e = cudaStreamEndCapture(st, g.put());
    if (rc) return rc;
    if (e != cudaSuccess) return fail(B200SAC_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    GraphExec ge;
    e = cudaGraphInstantiate(ge.put(), g, 0);
    if (e != cudaSuccess) return fail(B200SAC_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    if (cudaGraphUpload(ge, st) != cudaSuccess) cudaGetLastError();    // best effort: first launch does not pay the upload
    it = h->graphs.emplace(key, std::move(ge)).first;
  }
  *out = it->second;
  return 0;
}

static int launch_step(b200sac* h, cudaStream_t st, const GraphKey& key) {
  cudaGraphExec_t ge = nullptr;
  if (int rc = get_graph(h, st, key, &ge)) return rc;
  CU(cudaGraphLaunch(ge, st));
  h->host_steps += key.nsteps;
  return 0;
}

// Capture + instantiate every graph the sampled path can launch (device ring: the 8/4/2/1-step graphs; host ring: the
// staged one-step graphs of both staging slots) without running a step, so that no later call pays graph construction.
extern "C" int b200sac_prepare(b200sac_t* h, b200sac_replay_t* rb, void* stream) {
  if (!h || !rb || rb->h != h) return fail(B200SAC_ERR_INVALID, "bad handle");
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaGraphExec_t ge = nullptr;
  if (rb->where == 0) {
    RingLocks lk(rb);                           // the graphs capture the prior's rows and fill (capture enqueues no work)
    for (int n = kGraphSteps; n >= 1; n >>= 1)
      if (int rc = get_graph(h, sb.run, GraphKey{rb, rb->rows, nullptr, n, h->stamping}, &ge)) return rc;
  } else {
    for (int slot = 0; slot < 2; ++slot)
      if (int rc = get_graph(h, sb.run, GraphKey{nullptr, h->stage_d[slot], nullptr, 1, h->stamping}, &ge)) return rc;
  }
  if (int rc = sb.end()) return rc;
  CU(cudaStreamSynchronize(sb.run));
  return 0;
}

extern "C" int b200sac_step(b200sac_t* h, const float* s, const float* a, const float* r, const float* s2, const float* d,
                            const float* eps_next, const float* eps_cur, void* stream) {
  if (!h || !s || !a || !r || !s2 || !d) return fail(B200SAC_ERR_INVALID, "null minibatch pointer");
  if ((eps_next == nullptr) != (eps_cur == nullptr)) return fail(B200SAC_ERR_INVALID, "eps_next and eps_cur must both be given or both NULL");
  CU(cudaSetDevice(h->device));
  // The caller's arrays are copied (in stream order) into handle-owned buffers, so the captured graph sees the same
  // pointers whatever tensors the caller passes: one graph per (with / without injected noise), never a re-capture per
  // call.  The transitions become rows laid out like a staging slot's (the staged step's graph body), the noise goes
  // straight into the step's noise buffer.
  const size_t RB = (size_t)h->R * h->cfg.batch, nA = (size_t)h->cfg.batch * h->cfg.act_dim;
  if (!h->step_d) CU(dev_alloc(h->step_d, RB * h->row_stride));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  const RowFields F = row_fields(h);
  const float* f[ROW_FIELDS] = {s, a, r, s2, d};
  for (int k = 0; k < ROW_FIELDS; ++k)
    CU(cudaMemcpy2DAsync(h->step_d + F.off[k], h->row_stride * sizeof(float), f[k], F.w[k] * sizeof(float),
                         F.w[k] * sizeof(float), RB, cudaMemcpyDefault, sb.run));
  if (eps_next)           // [R][B][A] next and cur -> per replica [B][A] next, then [B][A] cur
    for (int k = 0; k < 2; ++k)
      CU(cudaMemcpy2DAsync(h->eps.p + k * nA, h->eps.rs * sizeof(float), k ? eps_cur : eps_next, nA * sizeof(float),
                           nA * sizeof(float), h->R, cudaMemcpyDefault, sb.run));
  if (int rc = launch_step(h, sb.run, GraphKey{nullptr, h->step_d, eps_next ? h->eps.p : nullptr, 1, h->stamping})) return rc;
  return sb.end();
}

// stage slot -> device on the side stream, make `st` wait for it, run the step from the staged rows
static int staged_step(b200sac* h, cudaStream_t st, int slot, bool with_eps) {
  const size_t rows_f = (size_t)h->R * h->cfg.batch * h->row_stride;
  const size_t eps_f = (size_t)2 * h->R * h->cfg.batch * h->cfg.act_dim;
  CU(cudaMemcpyAsync(h->stage_d[slot], h->stage_h[slot], (rows_f + (with_eps ? eps_f : 0)) * sizeof(float),
                     cudaMemcpyHostToDevice, h->side));
  CU(cudaEventRecord(h->ev_copied[slot], h->side));
  CU(cudaStreamWaitEvent(st, h->ev_copied[slot], 0));
  const float* eps = with_eps ? h->stage_d[slot] + rows_f : nullptr;
  if (int rc = launch_step(h, st, GraphKey{nullptr, h->stage_d[slot], eps, 1, h->stamping})) return rc;
  CU(cudaEventRecord(h->ev_consumed[slot], st));
  h->stage_used[slot] = true;
  return 0;
}

static int acquire_slot(b200sac* h, int* slot) {
  int s = h->stage_slot;
  if (s == h->prefetch_slot) h->prefetch_slot = -1;          // the slot is being reused: its prefetched batch is void
  h->stage_slot ^= 1;
  if (h->stage_used[s]) {
    CU(cudaEventSynchronize(h->ev_consumed[s]));          // host may overwrite the pinned slot
    CU(cudaStreamWaitEvent(h->side, h->ev_consumed[s], 0));   // and the side stream the device slot
  }
  *slot = s;
  return 0;
}

// the last n_last entries of a mapped pinned per-step ring [kLossSlots][R][width] (losses: width 4, gradient norms: 3)
static int fetch_ring(b200sac* h, cudaStream_t st, int n_last, const float* ring, int width, float* out) {
  if (n_last < 1 || n_last > kLossSlots || n_last > h->host_steps)
    return fail(B200SAC_ERR_INVALID, "n_last=%d out of range (steps so far %lld, ring %d)", n_last, h->host_steps, kLossSlots);
  const size_t per = (size_t)h->R * width;
  CU(cudaStreamSynchronize(st));       // the kernels wrote the mapped host ring directly
  for (int i = 0; i < n_last; ++i) {
    const long long step = h->host_steps - n_last + i;
    const long long slot = step % kLossSlots;
    memcpy(out + (size_t)i * per, ring + (size_t)slot * per, per * sizeof(float));
  }
  return 0;
}
static int fetch_losses(b200sac* h, cudaStream_t st, int n_last, float* out) { return fetch_ring(h, st, n_last, h->loss_h, 4, out); }

extern "C" int b200sac_step_host(b200sac_t* h, const float* s, const float* a, const float* r, const float* s2,
                                 const float* d, const float* eps_next, const float* eps_cur, float* out_losses, void* stream) {
  if (!h || !s || !a || !r || !s2 || !d) return fail(B200SAC_ERR_INVALID, "null minibatch pointer");
  if ((eps_next == nullptr) != (eps_cur == nullptr)) return fail(B200SAC_ERR_INVALID, "eps_next and eps_cur must both be given or both NULL");
  if (h->cfg.pcgrad) {          // row i must belong to task i / P (the first maximum of its one-hot, as the ingest reads it)
    const int B = h->cfg.batch, T = h->cfg.num_tasks, obs = h->K.obs;
    for (long long i = 0; i < (long long)h->R * B; ++i) {
      const float* oh = s + i * obs + (obs - T);
      int t = 0;
      for (int q = 1; q < T; ++q) if (oh[q] > oh[t]) t = q;
      if (t != (int)(i % B) / (B / T))
        return fail(B200SAC_ERR_INVALID, "pcgrad: replica %lld row %lld belongs to task %d, not to task %d (rows in task blocks of batch / num_tasks)",
                    i / B, i % B, t, (int)(i % B) / (B / T));
    }
  }
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  int slot;
  if (int rc = acquire_slot(h, &slot)) return rc;
  const float* f[ROW_FIELDS] = {s, a, r, s2, d};
  for (long long i = 0; i < (long long)h->R * h->cfg.batch; ++i) pack_row(h, h->stage_h[slot] + i * h->row_stride, f, i);
  if (eps_next) {
    const size_t rows_f = (size_t)h->R * h->cfg.batch * h->row_stride;
    const size_t n = (size_t)h->R * h->cfg.batch * h->cfg.act_dim;
    memcpy(h->stage_h[slot] + rows_f, eps_next, n * sizeof(float));
    memcpy(h->stage_h[slot] + rows_f + n, eps_cur, n * sizeof(float));
  }
  if (int rc = staged_step(h, st, slot, eps_next != nullptr)) return rc;
  if (out_losses)
    if (int rc = fetch_losses(h, st, 1, out_losses)) return rc;
  return sb.end();
}

// Eager (non-graph) run of `iters` sampled steps with a CUDA event between every launch.
// out_ms[i] = mean device time of launch i (i = 0 is sampling + ingest); names are returned as a
// ';'-separated list.  This is what bench.py uses for the per-kernel roofline numbers.
extern "C" int b200sac_profile_step(b200sac_t* h, b200sac_replay_t* rb, int32_t iters, float* out_ms, int32_t cap,
                                    int32_t* n_out, char* names, int32_t names_cap, void* stream) {
  if (!h || !rb || rb->h != h || rb->where != 0 || !out_ms || !n_out) return fail(B200SAC_ERR_INVALID, "profile_step needs a device ring");
  CU(cudaSetDevice(h->device));
  const int n = (int)h->plan.size() + 1;
  *n_out = n;
  if (cap < n) return fail(B200SAC_ERR_INVALID, "need room for %d launches", n);
  RingLocks lk(rb);
  if (int rc = prior_ready(rb)) return rc;
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  std::vector<Event> evs((size_t)n + 1);
  for (auto& e : evs) CU(cudaEventCreate(e.put()));
  std::vector<double> acc((size_t)n, 0.0);
  for (int it = 0; it < iters; ++it) {
    if (int rc = enqueue_body(h, sb.run, GraphKey{rb, rb->rows, nullptr, 1, h->stamping}, evs.data())) return rc;
    h->host_steps += 1;
    h->idx_mixed = rb->prior != nullptr;
    if (int rc = record_gather(rb, sb.run)) return rc;
    CU(cudaStreamSynchronize(sb.run));
    for (int i = 0; i < n; ++i) {
      float ms = 0.f;
      CU(cudaEventElapsedTime(&ms, evs[i], evs[i + 1]));
      acc[i] += ms;
    }
  }
  for (int i = 0; i < n; ++i) out_ms[i] = (float)(acc[i] / iters);
  if (names && names_cap > 0) {
    std::string s = rb->prior ? "sample_mixed+ingest_mixed" : "sample+ingest";
    for (auto& l : h->plan) s += ";" + l.label;
    snprintf(names, names_cap, "%s", s.c_str());
  }
  return sb.end();
}

// Stand-alone run of one GEMM engine on caller-provided DEVICE arrays (parity tests):
// engine 0 = 32x32-tile FFMA (gemm_simt.cuh), 1 = wgmma 3xTF32 (gemm_tc.cuh), 2 = thin backward (gemm_thin.cuh).
static int tc_gemm_test_impl(int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B, int32_t ldb,
                             const float* bias, const float* mask, int32_t ldmask, float* C, int32_t ldc, float* C2, int32_t relu,
                             void* stream);
extern "C" int b200sac_gemm_test(int32_t engine, int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda,
                                 const float* B, int32_t ldb, const float* bias, const float* mask, int32_t ldmask, float* C,
                                 int32_t ldc, float* C2, int32_t relu, void* stream) {
  if (engine == 1) return tc_gemm_test_impl(mode, M, N, K, A, lda, B, ldb, bias, mask, ldmask, C, ldc, C2, relu, stream);
  if (!A || !B || !C || M < 1 || N < 1 || K < 1 || mode < 0 || mode > 2) return fail(B200SAC_ERR_INVALID, "bad argument");
  GemmGroup grp;
  memset(&grp, 0, sizeof(grp));
  grp.G = 1;
  GemmProb& p = grp.p[0];
  p.A = A; p.B = B; p.bias = bias; p.mask = mask; p.C = C; p.C2 = C2;
  p.M = M; p.N = N; p.K = K; p.lda = lda; p.ldb = ldb; p.ldc = ldc; p.ldmask = ldmask; p.mode = mode; p.relu = relu;
  if (engine == 0) {
    gemm_simt_kernel<<<dim3((N + GS_T - 1) / GS_T, (M + GS_T - 1) / GS_T, 1), GS_THREADS, 0, (cudaStream_t)stream>>>(grp);
  } else if (engine == 2) {
    if (!gemm_is_thin(p)) return fail(B200SAC_ERR_INVALID, "thin engine needs a backward problem with N <= %d", GT_NMAX);
    const int per = mode == GEMM_WGRAD ? GT_ROWS_WGRAD : GT_ROWS_DGRAD;
    gemm_thin_kernel<<<dim3(1, (M + per - 1) / per, 1), GT_THREADS, 0, (cudaStream_t)stream>>>(grp);
  } else {
    return fail(B200SAC_ERR_INVALID, "unknown GEMM engine %d", engine);
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
  if (e != cudaSuccess) return fail(B200SAC_ERR_CUDA, "GEMM engine %d failed: %s", engine, cudaGetErrorString(e));
  return 0;
}

extern "C" int b200sac_tc_gemm_test(int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda,
                                    const float* B, int32_t ldb, const float* bias, const float* mask, int32_t ldmask,
                                    float* C, int32_t ldc, float* C2, int32_t relu, void* stream) {
  return tc_gemm_test_impl(mode, M, N, K, A, lda, B, ldb, bias, mask, ldmask, C, ldc, C2, relu, stream);
}

static int tc_gemm_test_impl(int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda,
                                    const float* B, int32_t ldb, const float* bias, const float* mask, int32_t ldmask,
                                    float* C, int32_t ldc, float* C2, int32_t relu, void* stream) {
  if (!A || !B || !C) return fail(B200SAC_ERR_INVALID, "null argument");
  GemmProb p;
  memset(&p, 0, sizeof(p));
  p.A = A; p.B = B; p.bias = bias; p.mask = mask; p.C = C; p.C2 = C2;
  p.M = M; p.N = N; p.K = K; p.lda = lda; p.ldb = ldb; p.ldc = ldc; p.ldmask = ldmask; p.mode = mode; p.relu = relu;
  if (!tc_eligible(p)) return fail(B200SAC_ERR_INVALID, "problem not eligible for the wgmma path (need 16-B aligned operands, lda/ldb %% 4 == 0, M,N,K >= 32)");
  const EnvSwitches sw = env_switches();
  const int bn = sw.tc_bn ? sw.tc_bn : 64;
  TcProb t;
  if (int rc = make_tc_prob(p, 0, t, bn)) return rc;
  DevMem<TcProb> d;
  CU(dev_copy(d, &t, 1));
  CU(allow_smem((const void*)tc_kernel(bn, sw.pair128), tc_smem(bn)));
  dim3 grid((N + bn - 1) / bn, (M + TC_BM - 1) / TC_BM, 1);
  tc_kernel(bn, sw.pair128)<<<grid, TC_THREADS, tc_smem(bn), (cudaStream_t)stream>>>(d, nullptr, 1, 0);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
  if (e != cudaSuccess) return fail(B200SAC_ERR_CUDA, "gemm_tc_kernel failed: %s", cudaGetErrorString(e));
  return 0;
}

// clock64() timeline of CTA (0,0) of one warm wgmma GEMM launch (see TC_STAMP indices in gemm_tc.cuh).
extern "C" int b200sac_tc_gemm_timeline(int32_t mode, int32_t M, int32_t N, int32_t K, long long* out96) {
  DevMem<float> A, B, C;
  DevMem<long long> dbg;
  const size_t na = (size_t)(mode == GEMM_WGRAD ? K * M : M * K), nb = (size_t)(mode == GEMM_FWD ? N * K : K * N);
  CU(dev_fill(A, na, 0.f)); CU(dev_fill(B, nb, 0.f)); CU(dev_alloc(C, (size_t)M * N)); CU(dev_fill(dbg, 96, 0));
  GemmProb p;
  memset(&p, 0, sizeof(p));
  p.A = A; p.B = B; p.C = C; p.M = M; p.N = N; p.K = K; p.mode = mode;
  p.lda = mode == GEMM_WGRAD ? M : K; p.ldb = mode == GEMM_FWD ? K : N; p.ldc = N;
  const EnvSwitches sw = env_switches();
  const int bn = sw.tc_bn ? sw.tc_bn : 64;
  TcProb t;
  if (int rc = make_tc_prob(p, 0, t, bn)) return rc;
  t.dbg = dbg;
  DevMem<TcProb> d;
  CU(dev_copy(d, &t, 1));
  CU(allow_smem((const void*)tc_kernel(bn, sw.pair128), tc_smem(bn)));
  dim3 grid((N + bn - 1) / bn, (M + TC_BM - 1) / TC_BM, 1);
  for (int it = 0; it < 3; ++it) tc_kernel(bn, sw.pair128)<<<grid, TC_THREADS, tc_smem(bn)>>>(d, nullptr, 1, 0);
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out96, dbg, 96 * 8, cudaMemcpyDeviceToHost));
  return 0;
}

// In-graph timeline: run `iters` sampled steps (graph launches) with kernel-start stamping enabled and
// return the mean start-to-start time (us) of each launch of the step: out_us[0] = sampling kernel, ...,
// out_us[n-1] = last kernel (measured to the next step's first kernel).
extern "C" int b200sac_graph_timeline(b200sac_t* h, b200sac_replay_t* rb, int32_t iters, float* out_us, int32_t cap,
                                      int32_t* n_out, void* stream) {
  if (!h || !rb || rb->h != h || rb->where != 0 || !out_us || !n_out) return fail(B200SAC_ERR_INVALID, "graph_timeline needs a device ring");
  CU(cudaSetDevice(h->device));
  const int n = (int)h->plan.size() + 2 + (rb->per ? 1 : 0);   // sample + ingest + plan (+ the priority update)
  *n_out = n;
  if (cap < n) return fail(B200SAC_ERR_INVALID, "need room for %d launches", n);
  const int total = n * (iters + 1);
  DevMem<unsigned long long> dt;
  DevMem<int> di;
  CU(dev_alloc(dt, total));
  CU(dev_fill(di, 1, 0));
  StampBuf sb_on = {dt, di, total}, sb_off = {nullptr, nullptr, 0};
  if (int rc = b200sac_step_sampled(h, rb, 5, stream)) return rc;     // warm (graph instantiated)
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpyToSymbol(g_stamp, &sb_on, sizeof(StampBuf)));
  h->stamping = true;
  int rc = b200sac_step_sampled(h, rb, iters + 1, stream);
  h->stamping = false;
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpyToSymbol(g_stamp, &sb_off, sizeof(StampBuf)));
  if (rc) return rc;
  std::vector<unsigned long long> t((size_t)total);
  CU(cudaMemcpy(t.data(), dt, sizeof(unsigned long long) * total, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; ++i) {
    double acc = 0;
    for (int it = 0; it < iters; ++it) acc += (double)(t[(size_t)it * n + i + 1] - t[(size_t)it * n + i]);
    out_us[i] = (float)(acc / iters * 1e-3);
  }
  return 0;
}

// Learner.update() in one call: sample + one gradient step + the losses of that step (LL/learner.py:246-264).
extern "C" int b200sac_update(b200sac_t* h, b200sac_replay_t* rb, float* losses_host, void* stream) {
  if (!h || !rb || !losses_host) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = b200sac_step_sampled(h, rb, 1, stream)) return rc;
  CU(cudaSetDevice(h->device));
  return fetch_losses(h, (cudaStream_t)stream, 1, losses_host);
}

extern "C" int b200sac_read_losses(b200sac_t* h, int32_t n_last, float* out_host, void* stream) {
  if (!h || !out_host) return fail(B200SAC_ERR_INVALID, "null argument");
  CU(cudaSetDevice(h->device));
  return fetch_losses(h, (cudaStream_t)stream, n_last, out_host);
}

extern "C" int b200sac_read_grad_norms(b200sac_t* h, int32_t n_last, float* out_host, void* stream) {
  if (!h || !out_host) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = need_feature(h->cfg.grad_clip, "grad_clip")) return rc;
  CU(cudaSetDevice(h->device));
  return fetch_ring(h, (cudaStream_t)stream, n_last, h->gnorm_h, kClipCols, out_host);
}

// ------------------------------------------------------------------------------------------
// Batched policy inference (SURVEY 8(f) rank 4): the actor forward + tanh-Gaussian head the step uses, on n <= 2B
// caller-provided observation rows -- Actor.get_action (LunarLander_Distributed_SAC/src/model.py:67-82; MT: mtobs rows,
// MT10_Distributed_MTSAC/src/model.py:58-73) for many environments at once.  stochastic = 0 gives k*tanh(mu).
// Uses the actor's own work buffers, so it is ordered with the steps on `stream` like any other call of the handle.
// ------------------------------------------------------------------------------------------
// LunarLander's deterministic action: k * mu, no tanh (LunarLander_Distributed_SAC/src/model.py:78-80)
__global__ void act_scaled_mu_kernel(const float* __restrict__ pout, int A, int n, float k, float* __restrict__ act) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * A) return;
  act[e] = k * pout[(long long)(e / A) * 2 * A + (e % A)];
}

// task id of n observation rows: argmax of the trailing one-hot (context_encoder.py:101-106), first maximum like torch.argmax
__global__ void act_task_ids_kernel(const float* __restrict__ X, int obs, int T, int n, int* __restrict__ tid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* row = X + (long long)i * obs + (obs - T);
  int t = 0;
  float best = row[0];
  for (int q = 1; q < T; ++q)
    if (row[q] > best) { best = row[q]; t = q; }
  tid[i] = t;
}

// one replica's problems of equal M and N on gemm_simt_kernel, GS_MAXG per launch
static void act_gemm(const std::vector<GemmProb>& ps, cudaStream_t st) {
  for (size_t i0 = 0; i0 < ps.size(); i0 += GS_MAXG) {
    GemmGroup grp;
    memset(&grp, 0, sizeof(grp));
    grp.G = (int)std::min(ps.size() - i0, (size_t)GS_MAXG);
    for (int q = 0; q < grp.G; ++q) grp.p[q] = ps[i0 + q];
    const GemmProb& p = grp.p[0];
    gemm_simt_kernel<<<dim3((p.N + GS_T - 1) / GS_T, (p.M + GS_T - 1) / GS_T, grp.G), GS_THREADS, 0, st>>>(grp);
  }
}

// CARE actors (MT10_Distributed_CARE/src/player.py:199-209: z = context_encoder(mtobs); actor.get_action(mtobs, z)):
// encode the n observation rows sitting in XS[0..n) of `replica` with the critic's state encoder -- the actor's is its
// hard copy (learner.py:402) -- into XA[0..n) and, when d2.p is set, into d2's rows [0, n) too (pitch ld2; b200sac_redo's
// critic input XQ): per-task tables, K mixture encoders, attention mix.
static int care_encode_rows(b200sac* h, cudaStream_t st, int replica, int n, Buf d2 = Buf{}, int ld2 = 0) {
  act_task_ids_kernel<<<(n + 255) / 256, 256, 0, st>>>(rep_view(h->XS, replica).p, h->K.obs, h->cfg.num_tasks, n,
                                                       (int*)rep_view(h->tid, replica).p);
  care_tables_kernel<<<dim3(h->cfg.num_tasks, 1, 1), 512, 0, st>>>(care_tab_args(h, replica, {0}));
  for (int l = 0; l < (int)h->L.mix.size(); ++l) {
    std::vector<GemmProb> ps;
    mix_fwd_probs(h, replica, 0, l, 0, n, ps);
    act_gemm(ps, st);
  }
  const EncJob job{0, 0, n, rep_view(h->XA, replica), h->K.ldxa, d2, ld2, 0};
  care_mix_kernel<<<dim3((n + 7) / 8, 1), 256, 0, st>>>(care_mix_args(h, replica, job));
  CU(cudaGetLastError());
  return 0;
}

extern "C" int b200sac_act(b200sac_t* h, int32_t replica, int32_t n, const float* obs, const float* eps, int32_t stochastic,
                           float* actions_out, void* stream) {
  if (!h || !obs || !actions_out) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = check_replica(h, replica)) return rc;
  const b200sac_cfg& c = h->cfg;
  const int B = c.batch, A = c.act_dim, La = c.n_actor_hidden;
  const int nmax = c.care ? B : 2 * B;           // CARE: one task id per row lives in the [batch] task-id buffer
  if (n < 1 || n > nmax) return fail(B200SAC_ERR_INVALID, "n must be in [1, %d] (2*batch; batch for CARE handles), got %d", nmax, n);
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  const Layout& L = h->L;
  const int obs_w = h->K.obs;
  float* XA = h->XA.p + (long long)replica * h->XA.rs;
  if (c.care) {
    CU(cudaMemcpyAsync(h->XS.p + (long long)replica * h->XS.rs, obs, (size_t)n * obs_w * sizeof(float), cudaMemcpyDefault, st));
    if (int rc = care_encode_rows(h, st, replica, n)) return rc;
  } else {
    CU(cudaMemcpy2DAsync(XA, (size_t)h->K.ldxa * sizeof(float), obs, (size_t)obs_w * sizeof(float), (size_t)obs_w * sizeof(float),
                         (size_t)n, cudaMemcpyDefault, st));
  }
  const Buf par = rep_view(Buf{h->params, L.arena}, replica);
  for (int l = 0; l < La; ++l) {
    const Buf X = rep_view(l == 0 ? h->XA : h->hA[l - 1], replica), out = rep_view(h->hA[l], replica);
    act_gemm({fwd_prob(par, X.p, X.rs, n, L.actor[l], out.p, out.rs)}, st);
  }
  PolicyHeadArgs P = h->pol;
  P.h += replica * P.rsH; P.W += replica * P.rsP; P.b += replica * P.rsP; P.eps += replica * P.rsEps;
  P.pout += replica * P.rsPout; P.psave += replica * P.rsSave; P.XT += replica * P.rsX; P.XP += replica * P.rsX;
  P.act_out += replica * P.rsAct; P.logp += replica * P.rsLogp; P.logstd_sum += replica * P.rsLogp; P.cnt += replica;
  P.rows = n;
  float* epsb = h->eps.p + (long long)replica * h->eps.rs;
  if (eps != nullptr) {
    CU(cudaMemcpyAsync(epsb, eps, (size_t)n * A * sizeof(float), cudaMemcpyDefault, st));
    P.use_eps_buf = 1;
  } else if (stochastic <= 0) {
    CU(cudaMemsetAsync(epsb, 0, (size_t)n * A * sizeof(float), st));       // u = mu: Actor.get_action(stochastic=False)
    P.use_eps_buf = 1;
  } else {
    P.use_eps_buf = 0;
  }
  StepConst K = h->K;
  K.seed ^= 0x5851F42D4C957F2Dull * (unsigned long long)(++h->act_calls);    // fresh noise per call, not per training step
  policy_head_kernel<<<dim3((n + 7) / 8, 1), 256, 0, st>>>(K, P);
  if (stochastic < 0 && eps == nullptr)          // k * mu instead of k * tanh(mu)
    act_scaled_mu_kernel<<<(n * A + 255) / 256, 256, 0, st>>>(P.pout, A, n, (float)c.action_scale, P.act_out);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(actions_out, h->act_out.p + (long long)replica * h->act_out.rs, (size_t)n * A * sizeof(float), cudaMemcpyDefault, st));
  if (int rc = sb.end()) return rc;
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

// Dormant-neuron recycling (include/b200sac.h): the forward of b200sac_act's engine over (obs, act) into the step's XA / XQ /
// hA / hQ rows [0, n), then redo_score_kernel and, unless both thresholds are negative, redo_recycle_kernel.
extern "C" int b200sac_redo(b200sac_t* h, int32_t replica, int32_t n, const float* obs, const float* act, double tau_actor,
                            double tau_critic, uint64_t seed, void* stream) {
  if (!h || !obs || !act) return fail(B200SAC_ERR_INVALID, "null argument");
  if (h->cfg.critic_ln)     // its forward has no LayerNorm, and one recycled unit would move its whole row's statistics
    return fail(B200SAC_ERR_STATE, "ReDo does not run on a handle created with critic_ln");
  if (h->cfg.critic_ensemble) return fail(B200SAC_ERR_STATE, "ReDo does not run on a handle created with critic_ensemble");
  if (int rc = check_replica(h, replica)) return rc;
  const b200sac_cfg& c = h->cfg;
  const int B = c.batch, A = c.act_dim, La = c.n_actor_hidden, Lc = c.n_critic_hidden;
  if (n < 1 || n > B) return fail(B200SAC_ERR_INVALID, "n must be in [1, batch = %d], got %d", B, n);
  if (std::isnan(tau_actor) || std::isnan(tau_critic)) return fail(B200SAC_ERR_INVALID, "tau must not be NaN");
  const Layout& L = h->L;
  RedoArgs RA;
  memset(&RA, 0, sizeof(RA));
  const size_t nt = (size_t)L.trainable;
  RA.params = h->params + (size_t)replica * L.arena;
  RA.m = h->adam_m + replica * nt; RA.v = h->adam_v + replica * nt;
  RA.score = h->redo_score + replica * h->redo_n; RA.dormant = h->redo_flag + replica * h->redo_n;
  RA.key = seed + (uint64_t)replica;
  RA.tau[0] = tau_actor; RA.tau[1] = tau_critic;
  RA.n = n;
  std::unordered_map<int64_t, int> tag;                  // weight offset -> its Philox tag, as create drew it
  for (const InitTensor& t : init_table(&c, L))
    if (t.kind == RESET_XAVIER) tag[t.off] = t.tag;
  long long rec = 0, widest = 0;
  auto layers = [&](const std::vector<LayerOff>& net, int nh, const std::vector<Buf>& hb, int net_idx, int critic) {
    for (int l = 0; l < nh; ++l) {
      const LayerOff &lo = net[l], &nx = net[l + 1];
      RedoLayer& t = RA.l[RA.nl++];
      t.h = rep_view(hb[l], replica).p + (long long)net_idx * B * lo.out;
      t.rec = rec; t.w = lo.w; t.b = lo.b; t.wn = nx.w; t.next_rec = l + 1 < nh ? rec + lo.out : -1;
      t.H = lo.out; t.in = lo.in; t.ld = lo.ld; t.next_out = nx.out; t.tag = tag.at(lo.w); t.critic = critic;
      rec += lo.out;
      widest = std::max(widest, (long long)lo.out * (lo.in + 1 + nx.out));
    }
  };
  const CriticPass& Q = h->pass[PASS_Q];
  layers(L.actor, La, h->hA, 0, 0);
  layers(Q.net[0], Lc, Q.h, 0, 1);
  layers(Q.net[1], Lc, Q.h, 1, 1);

  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  const int obs_w = h->K.obs, ldx = h->K.ldx;
  const Buf XA = rep_view(h->XA, replica), XQ = rep_view(*Q.X, replica);
  if (c.care) {
    CU(cudaMemcpyAsync(rep_view(h->XS, replica).p, obs, (size_t)n * obs_w * sizeof(float), cudaMemcpyDefault, st));
    if (int rc = care_encode_rows(h, st, replica, n, XQ, ldx)) return rc;
  } else {
    for (const auto& [X, ld] : {std::make_pair(XA.p, h->K.ldxa), std::make_pair(XQ.p, ldx)})
      CU(cudaMemcpy2DAsync(X, (size_t)ld * sizeof(float), obs, (size_t)obs_w * sizeof(float), (size_t)obs_w * sizeof(float),
                           (size_t)n, cudaMemcpyDefault, st));
  }
  CU(cudaMemcpy2DAsync(XQ.p + L.in_w, (size_t)ldx * sizeof(float), act, (size_t)A * sizeof(float), (size_t)A * sizeof(float),
                       (size_t)n, cudaMemcpyDefault, st));
  const Buf par = rep_view(Buf{h->params, L.arena}, replica);
  for (int l = 0; l < La; ++l) {
    const Buf X = rep_view(l == 0 ? h->XA : h->hA[l - 1], replica), out = rep_view(h->hA[l], replica);
    act_gemm({fwd_prob(par, X.p, X.rs, n, L.actor[l], out.p, out.rs)}, st);
  }
  for (int l = 0; l < Lc; ++l) {           // q1 and q2 in one launch: equal shapes
    std::vector<GemmProb> ps;
    for (int net = 0; net < 2; ++net) {
      const LayerOff& lo = Q.net[net][l];
      const float* X = l == 0 ? XQ.p : rep_view(Q.h[l - 1], replica).p + (long long)net * B * lo.in;
      ps.push_back(fwd_prob(par, X, 0, n, lo, rep_view(Q.h[l], replica).p + (long long)net * B * lo.out, 0));
    }
    act_gemm(ps, st);
  }
  redo_score_kernel<<<RA.nl, kRedoThreads, 0, st>>>(RA);
  if (tau_actor >= 0.0 || tau_critic >= 0.0) {
    const unsigned bx = (unsigned)std::min<long long>(64, (widest + kRedoThreads - 1) / kRedoThreads);
    redo_recycle_kernel<<<dim3(bx, RA.nl), kRedoThreads, 0, st>>>(RA);
  }
  CU(cudaGetLastError());
  return sb.end();
}

extern "C" int b200sac_read_redo(b200sac_t* h, int32_t replica, double* scores, uint8_t* dormant, int64_t cap,
                                 int64_t* n_neurons, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (int rc = check_replica(h, replica)) return rc;
  if (n_neurons) *n_neurons = h->redo_n;
  if ((scores || dormant) && cap < h->redo_n) return fail(B200SAC_ERR_INVALID, "buffer too small: need %lld", (long long)h->redo_n);
  CU(cudaSetDevice(h->device));
  const size_t n = (size_t)h->redo_n;
  if (scores) CU(cudaMemcpyAsync(scores, h->redo_score + replica * n, n * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  if (dormant) CU(cudaMemcpyAsync(dormant, h->redo_flag + replica * n, n, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

// ------------------------------------------------------------------------------------------
// Critic evaluation outside the step (eval_kernels.cuh): b200sac_critic_values and the priority refresh
// ------------------------------------------------------------------------------------------
// The evaluation scratch's buffers in carving order: the pointer each sets and its floats per row.  With n = 0 nothing
// is set and the sum is the floats of one row, alignment padding excluded.
static long long eval_carve(const b200sac* h, long long n, float* base) {
  const b200sac_cfg& c = h->cfg;
  const int A = c.act_dim, T = h->K.T > 0 ? h->K.T : 1;
  int Hc = 0, Ha = 0;
  for (int l = 0; l < c.n_critic_hidden; ++l) Hc = std::max(Hc, c.critic_hidden[l]);
  for (int l = 0; l < c.n_actor_hidden; ++l) Ha = std::max(Ha, c.actor_hidden[l]);
  EvalScratch& E = const_cast<b200sac*>(h)->ev;
  const int nets = h->E;
  const std::pair<void**, long long> rowbufs[] = {
      {(void**)&E.XQ, h->K.ldx}, {(void**)&E.XT, h->K.ldx}, {(void**)&E.hc[0], nets * Hc}, {(void**)&E.hc[1], nets * Hc},
      {(void**)&E.z, c.critic_ln ? nets * Hc : 0}, {(void**)&E.ha[0], Ha}, {(void**)&E.ha[1], Ha}, {(void**)&E.q, nets},
      {(void**)&E.qt, nets}, {(void**)&E.pout, 2 * A}, {(void**)&E.psave, A * kSaveW}, {(void**)&E.act, A},
      {(void**)&E.logp, 1}, {(void**)&E.logstd, 1}, {(void**)&E.eps, A}, {(void**)&E.R, 1}, {(void**)&E.d, 1},
      {(void**)&E.g, 1}, {(void**)&E.task, 1}, {(void**)&E.idx, 2}};
  if (n == 0) {
    long long w = 0;
    for (const auto& b : rowbufs) w += b.second;
    return w;
  }
  long long off = 0;
  auto take = [&](void** p, long long floats) {     // every buffer starts 256-byte aligned
    if (base) *p = base + off;
    off += (floats + 63) / 64 * 64;
  };
  for (const auto& b : rowbufs) take(b.first, n * b.second);
  take((void**)&E.tmax, T);
  take((void**)&E.tasks, T);
  return off;
}

// Rows per chunk: as many as fit kEvalScratchBytes, a multiple of 32, at most 65536 (the GEMM grid's row dimension).
static long long eval_rows(const b200sac* h) {
  const long long slack = 64 * 24 + 2 * (h->K.T + 64);    // alignment padding and the per-task buffers
  const long long n = ((long long)(kEvalScratchBytes / sizeof(float)) - slack) / eval_carve(h, 0, nullptr) / 32 * 32;
  return std::min<long long>(65536, n);
}

static int eval_alloc(b200sac* h) {
  EvalScratch& E = h->ev;
  if (E.mem) return 0;
  const long long n = eval_rows(h);
  const long long floats = eval_carve(h, n, nullptr);
  DevMem<float> mem;
  CU(dev_fill(mem, (size_t)floats, 0.f));
  eval_carve(h, n, mem);
  E.rows = n;
  E.mem = std::move(mem);
  return 0;
}

// Q of nets[0] and nets[1] (L.q: q1 and q2; L.qt: their targets; nets[0 .. E) on a critic_ensemble handle) of replica
// `rep` on n <= E.rows rows X [n][ldx] into out [2][n] ([E][n]), in eval mode: b200sac_act's per-layer gemm_simt_kernel and, on critic_ln handles, ln_fwd_kernel<false> between
// each hidden GEMM and its ReLU (no dropout, whatever the replica's rate).  Each output row depends on its input row alone.
static void eval_critics(b200sac* h, cudaStream_t st, int rep, const std::vector<LayerOff>* nets, const float* X, int n, float* out) {
  const EvalScratch& E = h->ev;
  const Buf par = rep_view(Buf{h->params, h->L.arena}, rep);
  const int Lc = h->cfg.n_critic_hidden;
  const bool ln = h->cfg.critic_ln != 0;
  for (int l = 0; l <= Lc; ++l) {
    std::vector<GemmProb> ps;
    for (int net = 0; net < h->E; ++net) {
      const LayerOff& lo = nets[net][l];
      const float* in = l == 0 ? X : E.hc[(l - 1) & 1] + (long long)net * n * lo.in;
      float* o = l == Lc ? out + (long long)net * n : (ln ? E.z : E.hc[l & 1]) + (long long)net * n * lo.out;
      GemmProb p = fwd_prob(par, in, 0, n, lo, o, 0);
      if (l == 0) p.lda = h->K.ldx;
      p.relu = l < Lc && !ln;
      ps.push_back(p);
    }
    act_gemm(ps, st);
    if (ln && l < Lc) {
      LnArgs P;
      memset(&P, 0, sizeof(P));
      P.z = E.z; P.h = E.hc[l & 1];
      P.g = par.p + nets[0][l].g; P.c = par.p + nets[0][l].c; P.rsNet = nets[1][l].g - nets[0][l].g;
      P.B = n; P.H = nets[0][l].out; P.E = h->E;
      ln_fwd_kernel<false><<<dim3((h->E * n + kLnThreads / kWarp - 1) / (kLnThreads / kWarp), 1), kLnThreads, 0, st>>>(h->K, P);
    }
  }
}

extern "C" int b200sac_critic_values_chunk(b200sac_t* h, int64_t* rows) {
  if (!h || !rows) return fail(B200SAC_ERR_INVALID, "null argument");
  *rows = eval_rows(h);
  return 0;
}

extern "C" int b200sac_critic_values(b200sac_t* h, int32_t replica, int64_t n, const float* obs, const float* act, int32_t which,
                                     float* q_out, void* stream) {
  if (!h || !obs || !act || !q_out) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = check_replica(h, replica)) return rc;
  if (n < 1) return fail(B200SAC_ERR_INVALID, "n must be >= 1, got %lld", (long long)n);
  if (which != 0 && which != 1) return fail(B200SAC_ERR_INVALID, "which must be 0 (q1, q2) or 1 (their targets), got %d", which);
  if (h->cfg.care) return fail(B200SAC_ERR_STATE, "critic_values does not run on a CARE handle");
  CU(cudaSetDevice(h->device));
  if (int rc = eval_alloc(h)) return rc;
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  const EvalScratch& E = h->ev;
  const int obs_w = h->K.obs, A = h->K.act;
  const size_t ldx = (size_t)h->K.ldx * sizeof(float);
  for (int64_t i0 = 0; i0 < n; i0 += E.rows) {
    const int m = (int)std::min<int64_t>(E.rows, n - i0);
    CU(cudaMemcpy2DAsync(E.XQ, ldx, obs + i0 * obs_w, (size_t)obs_w * sizeof(float), (size_t)obs_w * sizeof(float), (size_t)m,
                         cudaMemcpyDefault, st));
    CU(cudaMemcpy2DAsync(E.XQ + h->K.in_w, ldx, act + i0 * A, (size_t)A * sizeof(float), (size_t)A * sizeof(float), (size_t)m,
                         cudaMemcpyDefault, st));
    eval_critics(h, st, replica, which ? h->L.qt : h->L.q, E.XQ, m, E.q);
    CU(cudaGetLastError());
    for (int net = 0; net < h->E; ++net)
      CU(cudaMemcpyAsync(q_out + net * n + i0, E.q + (long long)net * m, (size_t)m * sizeof(float), cudaMemcpyDefault, st));
  }
  if (int rc = sb.end()) return rc;
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

extern "C" int b200sac_soft_update(b200sac_t* h, double tau, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  CU(cudaSetDevice(h->device));
  // CARE: Learner.soft_update is called per module with its own tau; this entry point applies `tau` to the Q
  // functions and, unless tau == 1 (hard copy of everything), the replica's state_encoder_tau to the state encoder.
  const bool hard = (tau == 1.0);
  polyak_kernel<<<dim3(128, h->R), 256, 0, (cudaStream_t)stream>>>(
      h->params + h->L.critic_begin, h->L.arena, h->L.critic_n, h->L.target_delta, (float)tau, (float)(1.0 - tau),
      (h->cfg.care && !hard) ? (long long)(h->L.cse_begin - h->L.critic_begin) : -1LL, h->hp.dev);
  CU(cudaGetLastError());
  return 0;
}

extern "C" int b200sac_soft_update_critic(b200sac_t* h, int32_t critic, double tau, void* stream) {
  if (!h) return fail(B200SAC_ERR_INVALID, "null handle");
  if (critic < 1 || critic > h->E) return fail(B200SAC_ERR_INVALID, "critic must be in [1, %d], got %d", h->E, critic);
  CU(cudaSetDevice(h->device));
  // q1, q2 (.. qE) are each contiguous in [critic_begin, cse_begin), each right behind the one before; their targets sit at
  // + target_delta
  const Layout& L = h->L;
  const int64_t beg = L.q[critic - 1][0].w, end = critic < h->E ? L.q[critic][0].w : L.cse_begin;
  polyak_kernel<<<dim3(128, h->R), 256, 0, (cudaStream_t)stream>>>(h->params + beg, L.arena, end - beg, L.target_delta,
                                                                  (float)tau, (float)(1.0 - tau));
  CU(cudaGetLastError());
  return 0;
}

extern "C" int b200sac_debug_read(b200sac_t* h, const char* name, int32_t replica, float* out_host, int64_t cap_floats,
                                  int64_t* n_floats, void* stream) {
  if (!h || !name || !out_host) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = check_replica(h, replica)) return rc;
  CU(cudaSetDevice(h->device));
  const int B = h->cfg.batch, A = h->cfg.act_dim;
  const float* src = nullptr;
  int64_t n = 0;
  std::string nm(name);
  if (nm == "y") { src = h->y.p + replica * h->y.rs; n = B; }
  else if (nm == "q1") { src = h->q.p + replica * h->q.rs; n = B; }
  else if (nm == "q2") { src = h->q.p + replica * h->q.rs + B; n = B; }
  else if (int k = 0; h->cfg.critic_ensemble && sscanf(name, "q%d", &k) == 1 && nm == "q" + std::to_string(k) && k >= 1 && k <= h->E) {
    src = h->q.p + replica * h->q.rs + (int64_t)(k - 1) * B; n = B;
  }
  else if (nm == "a_next") { src = h->act_out.p + replica * h->act_out.rs; n = (int64_t)B * A; }
  else if (nm == "a_cur") { src = h->act_out.p + replica * h->act_out.rs + (int64_t)B * A; n = (int64_t)B * A; }
  else if (nm == "logp_next") { src = h->logp.p + replica * h->logp.rs; n = B; }
  else if (nm == "logp_cur") { src = h->logp.p + replica * h->logp.rs + B; n = B; }
  else if (nm == "r") { src = h->r.p + replica * h->r.rs; n = B; }
  else if (nm == "d") { src = h->d.p + replica * h->d.rs; n = B; }
  else if (nm == "qmin") { src = h->qmin.p + replica * h->qmin.rs; n = B; }
  else if (nm == "q_pi") { src = h->qp.p + replica * h->E * h->y.rs; n = h->E * B; }        // [2][B]: Q1, Q2 at (s, a~) (actor pass); [E][B]
  else if (nm == "dq_pi") { src = h->dqa.p + replica * h->E * h->y.rs; n = h->E * B; }      // [2][B]: d(actor loss)/dQk -- the min routing; [E][B]
  else if (nm == "tsub") {                                  // critic_ensemble: [E] the last step's target subset as 0 / 1
    if (!h->cfg.critic_ensemble) return fail(B200SAC_ERR_INVALID, "'tsub' needs a handle created with critic_ensemble");
    src = h->tsub.p + replica * h->tsub.rs; n = h->E;
  }
  else if (nm == "d_action") { src = h->dact_dbg.p + replica * h->dact_dbg.rs; n = (int64_t)B * A; }
  else if (nm == "d_head") { src = h->dout_dbg.p + replica * h->dout_dbg.rs; n = (int64_t)B * 2 * A; }
  else if (nm == "head") { src = h->pout.p + replica * h->pout.rs; n = (int64_t)2 * B * 2 * A; }      // [2B][2A]: mu | raw log-std
  else if (nm == "psave") { src = h->psave.p + replica * h->psave.rs; n = (int64_t)2 * B * A * kSaveW; }   // [2B][A][8]: std, diff, tanh, act, jac, EPS, mask, logp_j
  else if (nm == "isw" || nm == "prio" || nm == "idx") {   // prioritized replay: [B] weights, leaf values, ring indices (int32 bits)
    if (nm == "idx" && h->idx_mixed) {                      // a ring with a prior: online k as k, prior k as -1 - k
      src = reinterpret_cast<const float*>(h->mix_idx.get()) + (size_t)replica * B; n = B;
    } else if (nm == "idx" && !h->per_buf && h->ns_buf) {   // a uniform linked ring: the indices its gather folded from
      src = h->ns_buf + ((size_t)2 * h->R + replica) * B; n = B;
    } else {
      if (!h->per_buf) return fail(B200SAC_ERR_INVALID, "'%s' needs a prioritized replay ring", name);
      src = h->per_buf + ((nm == "isw" ? 0 : nm == "prio" ? 1 : 2) * (size_t)h->R + replica) * B; n = B;
    }
  }
  else if (nm == "disc" || nm == "nstep_m") {               // n-step returns: [B] per-row discount, hops folded (int32 bits)
    if (!h->ns_buf) return fail(B200SAC_ERR_INVALID, "'%s' needs a replay ring with trajectory links", name);
    src = h->ns_buf + ((nm == "disc" ? 0 : 1) * (size_t)h->R + replica) * B; n = B;
  }
  else if (nm == "clip") {                                  // [3] clip coefficients of the last step
    if (!h->cfg.grad_clip) return fail(B200SAC_ERR_INVALID, "'clip' needs a handle created with grad_clip");
    src = h->clip_coef + (size_t)replica * kClipCols; n = kClipCols;
  }
  else if (nm == "chain_dbg") {
    if (!h->chain_dbg) return fail(B200SAC_ERR_INVALID, "chain_dbg needs B200SAC_CHAIN_DBG=1 at create time");
    src = reinterpret_cast<const float*>(h->chain_dbg.get()); n = 2 * CH_DBG_SLOTS * 16;     // int64 stamps viewed as float pairs
  }
  else {
    // hidden activations (the ReLU masks of the step): "hA.<l>" [2B][H] rows [s';s]; per critic pass (letter Q, T or P)
    // "h<pass>.<l>" [2][B][H] (the target pass's are not kept by the layer-chained plan), on critic_ln handles
    // "z<pass>.<l>", the pre-normalization activations (critic_dropout: after the dropout), on critic_dropout handles
    // "m<pass>.<l>", the keep masks as 0.0 / 1.0; CARE mixture encoders "mixH.<inst>.<l>" [K][rows][pitch4(H)], inst 0 =
    // critic's on [s';s] (rows 2B), 1 = target's on s', 2 = updated critic's on s
    int l = -1, inst = -1;
    char kind[2] = "", letter[2] = "";
    const Buf* b = nullptr;
    if (sscanf(name, "mixH.%d.%d", &inst, &l) == 2) {
      if (!h->cfg.care || inst < 0 || inst > 2 || l < 0 || l >= (int)h->mixH[inst].size()) return fail(B200SAC_ERR_INVALID, "no such tensor '%s'", name);
      b = &h->mixH[inst][l];
      const int rows = inst == 0 ? 2 * B : B, pw = (h->cfg.mix_hidden[l] + 3) & ~3;
      n = (int64_t)h->cfg.num_encoders * rows * pw;
    } else if (sscanf(name, "hA.%d", &l) == 1) {
      if (l < 0 || l >= (int)h->hA.size()) return fail(B200SAC_ERR_INVALID, "no such tensor '%s'", name);
      b = &h->hA[l];
      n = (int64_t)2 * B * h->cfg.actor_hidden[l];
    } else if (sscanf(name, "%1[hzm]%1[QTP].%d", kind, letter, &l) == 3) {
      const CriticPass* cp = nullptr;
      for (const CriticPass& p : h->pass)
        if (p.letter == letter[0]) cp = &p;
      const std::vector<Buf>& v = kind[0] == 'h' ? cp->h : (kind[0] == 'z' ? cp->z : cp->m);
      if (l < 0 || l >= (int)v.size()) return fail(B200SAC_ERR_INVALID, "no such tensor '%s'", name);
      const int H = h->cfg.critic_hidden[l];
      n = (int64_t)h->E * B * H;
      if (kind[0] == 'm') {
        if (n_floats) *n_floats = n;
        if (cap_floats < n) return fail(B200SAC_ERR_INVALID, "buffer too small: need %lld floats", (long long)n);
        const int words = (H + 31) / 32;
        std::vector<uint32_t> bits((size_t)h->E * B * words);
        CU(cudaMemcpyAsync(bits.data(), v[l].p + replica * v[l].rs, bits.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                           (cudaStream_t)stream));
        CU(cudaStreamSynchronize((cudaStream_t)stream));
        for (int64_t row = 0; row < (int64_t)h->E * B; ++row)
          for (int j = 0; j < H; ++j) out_host[row * H + j] = (float)((bits[row * words + j / 32] >> (j % 32)) & 1u);
        return 0;
      }
      b = &v[l];
    } else {
      return fail(B200SAC_ERR_INVALID, "unknown debug tensor '%s'", name);
    }
    src = b->p + replica * b->rs;
  }
  if (n_floats) *n_floats = n;
  if (cap_floats < n) return fail(B200SAC_ERR_INVALID, "buffer too small: need %lld floats", (long long)n);
  CU(cudaMemcpyAsync(out_host, src, n * sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

// ------------------------------------------------------------------------------------------
// replay ring
// ------------------------------------------------------------------------------------------
// The ring's rules, each written once:
//   arguments    ring_check: a ring, a replica of its handle, and the kind of ring the call needs;
//   writers      rows, fill, tree leaves and links are written under rb->mu after ring_quiesce, so no gather already
//                enqueued by a step reads a torn row and no concurrent writer interleaves;
//   samplers     ring_ready: every sub-ring a draw reads holds enough transitions;
//   indices      filled_slot: a ring index the caller names holds a transition;
//   allocation   all pieces or none: each goes into a local owner, and they move into the ring / handle only when every
//                one exists.
enum { RING_ANY, RING_PER, RING_TRAJ };
static int ring_check(const b200sac_replay* rb, int32_t replica, int kind = RING_ANY) {
  if (!rb) return fail(B200SAC_ERR_INVALID, "null ring");
  if (kind == RING_PER && !rb->per) return fail(B200SAC_ERR_INVALID, "not a prioritized ring (b200sac_replay_create_prioritized)");
  if (kind == RING_TRAJ && !rb->traj)
    return fail(B200SAC_ERR_STATE, "the ring has no trajectory links (b200sac_replay_enable_trajectories)");
  return check_replica(rb->h, replica);
}

// Waits (under rb->mu) until every step enqueued so far has gathered its rows and updated its priorities.
static int ring_quiesce(b200sac_replay* rb) {
  if (rb->gather_pending) { CU(cudaEventSynchronize(rb->ev_gather)); rb->gather_pending = false; }
  return 0;
}

// (under rb->mu) Every task sub-ring of `replica` (kAllReplicas: of every replica) holds at least `batches` per-task
// batches: 4 for the step's samplers, 1 for a draw without replacement, which would not end with fewer.
constexpr int kAllReplicas = -1;
static int ring_ready(const b200sac_replay* rb, int replica, int batches) {
  const long long need = (long long)batches * (rb->h->cfg.batch / rb->Teff);
  const int r0 = replica == kAllReplicas ? 0 : replica, r1 = replica == kAllReplicas ? rb->h->R : replica + 1;
  for (int rep = r0; rep < r1; ++rep)
    for (int t = 0; t < rb->Teff; ++t)
      if (rb->fill[(size_t)rep * rb->Teff + t] < need)
        return fail(B200SAC_ERR_STATE, "replay not ready: replica %d task %d holds %lld transitions, need >= %lld (%d x per-task batch)",
                    rep, t, rb->fill[(size_t)rep * rb->Teff + t], need, batches);
  return 0;
}

// (under rb->mu) ring index k of `replica` holds a transition
static int filled_slot(const b200sac_replay* rb, int replica, long long k) {
  if (k < 0 || k >= rb->cap) return fail(B200SAC_ERR_INVALID, "index %lld outside the ring [0, %lld)", k, rb->cap);
  if (k % rb->cap_per_task >= rb->fill[(size_t)replica * rb->Teff + k / rb->cap_per_task])
    return fail(B200SAC_ERR_INVALID, "index %lld is an empty slot", k);
  return 0;
}

// Graphs that captured a ring's pointers (its gather) go when the ring goes or its gather changes.
static void drop_ring_graphs(b200sac* h, const b200sac_replay* rb) {
  for (auto it = h->graphs.begin(); it != h->graphs.end();) {
    if (it->first.ring == rb) it = h->graphs.erase(it);
    else ++it;
  }
}

extern "C" int b200sac_replay_create(b200sac_t* h, int64_t capacity, int32_t where, uint64_t seed, b200sac_replay_t** out) {
  if (!h || !out) return fail(B200SAC_ERR_INVALID, "null argument");
  *out = nullptr;
  if (where != 0 && where != 1) return fail(B200SAC_ERR_INVALID, "where must be 0 (device) or 1 (pinned host)");
  const int Teff = h->cfg.num_tasks > 0 ? h->cfg.num_tasks : 1;
  if (capacity / Teff < 4LL * (h->cfg.batch / Teff))
    return fail(B200SAC_ERR_INVALID, "capacity %lld too small for batch %d", (long long)capacity, h->cfg.batch);
  if ((long long)capacity > 0x7fffffffLL) return fail(B200SAC_ERR_INVALID, "capacity must fit in int32");
  CU(cudaSetDevice(h->device));
  std::unique_ptr<b200sac_replay> owner(new (std::nothrow) b200sac_replay());   // a failed create releases what it allocated
  b200sac_replay* rb = owner.get();
  if (!rb) return fail(B200SAC_ERR_NOMEM, "out of host memory");
  rb->h = h; rb->where = where; rb->Teff = Teff;
  rb->cap_per_task = capacity / Teff;
  rb->cap = rb->cap_per_task * Teff;
  rb->rs_rows = rb->cap * h->row_stride;
  rb->seed = seed;
  rb->rng.seed(seed);
  rb->fill.assign((size_t)h->R * Teff, 0);
  rb->head.assign((size_t)h->R * Teff, 0);
  const size_t n = (size_t)h->R * rb->rs_rows;
  if (where == 0) {
    CU(dev_alloc(rb->rows_dev, n));
    rb->rows = rb->rows_dev;
    CU(dev_fill(rb->d_fill, (size_t)h->R * Teff, 0));
    CU(dev_alloc(rb->d_idx, (size_t)h->R * h->cfg.batch));
    CU(new_event(rb->ev_gather));
    CU(new_stream(rb->st));
  } else {
    CU(cudaMallocHost(rb->rows_pinned.put(), n * sizeof(float)));
    rb->rows = rb->rows_pinned;
  }
  *out = owner.release();
  return 0;
}

extern "C" int b200sac_replay_destroy(b200sac_replay_t* rb) {
  if (!rb) return 0;
  cudaSetDevice(rb->h->device);
  if (rb->h->prefetch_rb == rb) { rb->h->prefetch_slot = -1; rb->h->prefetch_rb = nullptr; }
  if (rb->prior) b200sac_replay_attach_prior(rb, nullptr);
  if (rb->prior_of) b200sac_replay_attach_prior(rb->prior_of, nullptr);
  drop_ring_graphs(rb->h, rb);
  delete rb;
  return 0;
}

// Trajectory links of one push (linked ring; under rb->mu).  Row i of the push went to sub-ring task[i], slot slot[i]
// (slot -1: a push larger than the sub-ring dropped it).  Rows are replayed in push order, as if appended one by one:
//   overwrite rule   the new occupant of slot j cuts the link that pointed to j (only if link[pred[j]] is still j), clears
//                    pred of the slot j pointed to (a stale pred must never cut the new occupant's link later), and a
//                    stream whose tail was j forgets it;
//   stream rule      row x becomes the successor of its stream's tail t iff t exists (d_t = 0, cut_t = 0: a closed tail is
//                    not kept) and both lie in the same task sub-ring.
// The host mirrors are updated here; `touched` collects the ring indices whose link changed.
static void push_links(b200sac_replay* rb, int replica, int64_t n, const std::vector<int>& task, const std::vector<long long>& slot,
                       const float* d, const int32_t* stream, const uint8_t* cut, std::vector<int>& touched) {
  const long long cpt = rb->cap_per_task;
  int* link = rb->link_h.data() + (size_t)replica * rb->cap;
  int* pred = rb->pred_h.data() + (size_t)replica * rb->cap;
  auto& tail = rb->tail[(size_t)replica];
  auto& tail_at = rb->tail_at[(size_t)replica];
  for (int64_t i = 0; i < n; ++i) {
    const int sid = stream ? stream[i] : -1;
    if (slot[(size_t)i] < 0) {                     // written and overwritten inside this push: its stream loses its tail
      if (sid >= 0) {
        auto it = tail.find(sid);
        if (it != tail.end()) { tail_at.erase(it->second); tail.erase(it); }
      }
      continue;
    }
    const long long tb = (long long)task[(size_t)i] * cpt, j = slot[(size_t)i], g = tb + j;
    const int p = pred[g], nx = link[g];
    if (p >= 0 && link[tb + p] == (int)j) { link[tb + p] = -1; touched.push_back((int)(tb + p)); }
    if (nx >= 0 && pred[tb + nx] == (int)j) pred[tb + nx] = -1;
    auto at = tail_at.find(g);
    if (at != tail_at.end()) { tail.erase(at->second); tail_at.erase(at); }
    link[g] = -1; pred[g] = -1;
    touched.push_back((int)g);
    if (sid < 0) continue;
    auto it = tail.find(sid);
    if (it != tail.end()) {
      const long long t = it->second;
      if (t / cpt == task[(size_t)i]) { link[t] = (int)j; pred[g] = (int)(t - tb); touched.push_back((int)t); }
      tail_at.erase(t);
      tail.erase(it);
    }
    if (d[i] == 0.f && !(cut && cut[i])) { tail[sid] = g; tail_at[g] = sid; }
  }
  std::sort(touched.begin(), touched.end());
  touched.erase(std::unique(touched.begin(), touched.end()), touched.end());
}

static int push_impl(b200sac_replay_t* rb, int32_t replica, int64_t n, const float* s, const float* a, const float* r,
                     const float* s2, const float* d, const int32_t* stream, const uint8_t* cut) {
  if (int rc = ring_check(rb, replica)) return rc;
  if (!s || !a || !r || !s2 || !d) return fail(B200SAC_ERR_INVALID, "null argument");
  b200sac* h = rb->h;
  if (n < 0) return fail(B200SAC_ERR_INVALID, "n < 0");
  if (stream)
    for (int64_t i = 0; i < n; ++i)
      if (stream[i] < 0 || stream[i] >= 65536)
        return fail(B200SAC_ERR_INVALID, "row %lld: stream id %d outside [0, 65536)", (long long)i, stream[i]);
  CU(cudaSetDevice(h->device));
  std::vector<int> row_task;
  std::vector<long long> row_slot;                 // first the row's position in its task bucket, then its slot
  if (rb->traj) { row_task.resize((size_t)n); row_slot.resize((size_t)n); }
  const int obs = h->K.obs, T = h->cfg.num_tasks, rs = h->row_stride;
  // pack the rows, bucketed by task, then copy each bucket as at most two contiguous runs (ring wrap)
  std::vector<std::vector<float>> bucket((size_t)rb->Teff);
  std::vector<float> row((size_t)rs, 0.f);
  const float* f[ROW_FIELDS] = {s, a, r, s2, d};
  for (int64_t i = 0; i < n; ++i) {
    pack_row(h, row.data(), f, i);
    int task = 0;
    if (T > 0) {
      float best = row[obs - T];
      for (int q = 1; q < T; ++q)
        if (row[obs - T + q] > best) { best = row[obs - T + q]; task = q; }
    }
    if (rb->traj) { row_task[(size_t)i] = task; row_slot[(size_t)i] = (long long)(bucket[(size_t)task].size() / (size_t)rs); }
    bucket[(size_t)task].insert(bucket[(size_t)task].end(), row.begin(), row.end());
  }
  std::lock_guard<std::mutex> lk(rb->mu);
  if (rb->traj) {                                  // bucket position -> slot, with the heads as they are before the copy
    for (int64_t i = 0; i < n; ++i) {
      const int task = row_task[(size_t)i];
      const long long cnt = (long long)(bucket[(size_t)task].size() / (size_t)rs);
      const long long skip = std::max(0LL, cnt - rb->cap_per_task), k = row_slot[(size_t)i];
      row_slot[(size_t)i] = k < skip ? -1 : (rb->head[(size_t)replica * rb->Teff + task] + (k - skip)) % rb->cap_per_task;
    }
  }
  // step_sampled enqueues under the same mutex, so no gather can slip in while we copy
  if (int rc = ring_quiesce(rb)) return rc;
  for (int task = 0; task < rb->Teff; ++task) {
    const float* src = bucket[(size_t)task].data();
    long long cnt = (long long)(bucket[(size_t)task].size() / (size_t)rs);
    if (cnt > rb->cap_per_task) {                  // more than a full ring: only the newest cap rows survive (deque maxlen)
      src += (size_t)(cnt - rb->cap_per_task) * rs;
      cnt = rb->cap_per_task;
    }
    long long& hd = rb->head[(size_t)replica * rb->Teff + task];
    long long& fl = rb->fill[(size_t)replica * rb->Teff + task];
    long long done = 0;
    while (done < cnt) {
      const long long run = std::min(cnt - done, rb->cap_per_task - hd);
      float* dst = rb->rows + (size_t)replica * rb->rs_rows + ((size_t)task * rb->cap_per_task + hd) * rs;
      if (rb->where == 0)
        CU(cudaMemcpyAsync(dst, src + (size_t)done * rs, (size_t)run * rs * sizeof(float), cudaMemcpyHostToDevice, rb->st));
      else memcpy(dst, src + (size_t)done * rs, (size_t)run * rs * sizeof(float));
      if (rb->per)                                 // the new rows get the current max p
        per_fill_kernel<<<dim3(1, 1), 1024, 0, rb->st>>>(rb->tr, task, replica, hd, hd + run, hd + run);
      hd = (hd + run) % rb->cap_per_task;
      fl = std::min(fl + run, rb->cap_per_task);
      done += run;
    }
  }
  if (rb->per) CU(cudaGetLastError());
  std::vector<int> touched, vals;
  if (rb->traj) {                                  // the link changes travel with the rows
    push_links(rb, replica, n, row_task, row_slot, d, stream, cut, touched);
    const size_t m = touched.size();
    if (m > rb->f_cap) {
      rb->f_at.reset(); rb->f_cap = 0;
      CU(dev_alloc(rb->f_at, 2 * m));
      rb->f_cap = m;
    }
    vals.resize(m);
    for (size_t i = 0; i < m; ++i) vals[i] = rb->link_h[(size_t)replica * rb->cap + touched[i]];
    if (m > 0) {
      CU(cudaMemcpyAsync(rb->f_at, touched.data(), m * sizeof(int), cudaMemcpyHostToDevice, rb->st));
      CU(cudaMemcpyAsync(rb->f_at + rb->f_cap, vals.data(), m * sizeof(int), cudaMemcpyHostToDevice, rb->st));
      nstep_scatter_links_kernel<<<(unsigned)((m + 255) / 256), 256, 0, rb->st>>>(rb->d_link + (size_t)replica * rb->cap, rb->f_at,
                                                                                 rb->f_at + rb->f_cap, (int)m);
      CU(cudaGetLastError());
    }
  }
  // A copy from pageable memory may return before its DMA has landed, and a step enqueued on a non-blocking stream is not
  // ordered after the legacy stream: the rows and the fill go on the ring's own stream, which is drained before the mutex
  // is released, so every step enqueued after this call gathers the new rows.
  if (rb->where == 0) {
    CU(cudaMemcpyAsync(rb->d_fill + (size_t)replica * rb->Teff, rb->fill.data() + (size_t)replica * rb->Teff,
                       sizeof(long long) * rb->Teff, cudaMemcpyHostToDevice, rb->st));
    CU(cudaStreamSynchronize(rb->st));
  }
  return 0;
}

extern "C" int b200sac_replay_push(b200sac_replay_t* rb, int32_t replica, int64_t n, const float* s, const float* a,
                                   const float* r, const float* s2, const float* d) {
  return push_impl(rb, replica, n, s, a, r, s2, d, nullptr, nullptr);
}

extern "C" int b200sac_replay_push_traj(b200sac_replay_t* rb, int32_t replica, int64_t n, const float* s, const float* a,
                                        const float* r, const float* s2, const float* d, const int32_t* stream,
                                        const uint8_t* cut) {
  if (!stream) return fail(B200SAC_ERR_INVALID, "null argument");
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  return push_impl(rb, replica, n, s, a, r, s2, d, stream, cut);
}

extern "C" int b200sac_replay_fill_synthetic(b200sac_replay_t* rb, int64_t n, uint64_t seed, void* stream) {
  if (!rb) return fail(B200SAC_ERR_INVALID, "null argument");
  b200sac* h = rb->h;
  CU(cudaSetDevice(h->device));
  long long per = n / rb->Teff;
  if (per > rb->cap_per_task) per = rb->cap_per_task;
  if (per < 1) return fail(B200SAC_ERR_INVALID, "n too small");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(rb->mu);
  if (int rc = ring_quiesce(rb)) return rc;
  float* dev_rows = rb->rows;
  DevMem<float> tmp;
  if (rb->where == 1) {   // generate on the device, copy down into the pinned ring
    CU(dev_alloc(tmp, (size_t)h->R * rb->rs_rows));
    dev_rows = tmp;
  }
  CU(cudaMemsetAsync(dev_rows, 0, (size_t)h->R * rb->rs_rows * sizeof(float), st));
  fill_synthetic_kernel<<<dim3(592, h->R), 256, 0, st>>>(dev_rows, rb->rs_rows, h->row_stride, per, rb->cap_per_task,
                                                        h->cfg.state_dim, h->cfg.act_dim, h->cfg.num_tasks, seed);
  CU(cudaGetLastError());
  if (rb->where == 1) {
    CU(cudaMemcpyAsync(rb->rows, tmp, (size_t)h->R * rb->rs_rows * sizeof(float), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  if (rb->per) {                                   // rows [0, per) of every sub-ring get the current max p, the rest are empty
    per_fill_kernel<<<dim3(rb->Teff, h->R), 1024, 0, st>>>(rb->tr, 0, 0, 0, rb->tr.P, per);
    CU(cudaGetLastError());
  }
  for (auto& f : rb->fill) f = per;
  for (auto& hd : rb->head) hd = per % rb->cap_per_task;
  if (rb->where == 0)
    CU(cudaMemcpyAsync(rb->d_fill, rb->fill.data(), sizeof(long long) * rb->fill.size(), cudaMemcpyHostToDevice, st));
  if (rb->traj) {                                  // slot i -> i + 1 unless d_i != 0 or i is the last filled slot; no open streams
    nstep_fill_links_kernel<<<dim3(256, h->R), 256, 0, st>>>(rb->d_link, rb->cap, (int)rb->cap_per_task, rb->rows, rb->rs_rows,
                                                            h->row_stride, row_fields(h).off[ROW_D], per);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(rb->link_h.data(), rb->d_link, rb->link_h.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::fill(rb->pred_h.begin(), rb->pred_h.end(), -1);
    for (size_t g = 0; g < rb->link_h.size(); ++g)
      if (rb->link_h[g] >= 0) rb->pred_h[g + 1] = (int)(g % (size_t)rb->cap_per_task);
    for (auto& t : rb->tail) t.clear();
    for (auto& t : rb->tail_at) t.clear();
  }
  CU(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int b200sac_replay_size(b200sac_replay_t* rb, int32_t replica, int64_t* n) {
  if (int rc = ring_check(rb, replica)) return rc;
  if (!n) return fail(B200SAC_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(rb->mu);
  long long mn = rb->fill[(size_t)replica * rb->Teff];
  for (int t = 1; t < rb->Teff; ++t) mn = std::min(mn, rb->fill[(size_t)replica * rb->Teff + t]);
  *n = rb->Teff > 1 ? mn : rb->fill[(size_t)replica * rb->Teff];
  return 0;
}

// host-side index draw (under rb->mu): uniform without replacement, per task (random.sample semantics)
static int host_draw(b200sac_replay* rb, int replica, std::vector<long long>& idx) {
  if (int rc = ring_ready(rb, replica, 1)) return rc;
  const int B = rb->h->cfg.batch, per = B / rb->Teff;
  idx.clear();
  for (int t = 0; t < rb->Teff; ++t) {
    const long long n = rb->fill[(size_t)replica * rb->Teff + t];
    std::unordered_set<long long> seen;
    while ((int)seen.size() < per) {
      const long long v = (long long)(rb->rng() % (unsigned long long)n);
      if (seen.insert(v).second) idx.push_back((long long)t * rb->cap_per_task + v);
    }
  }
  // MS/replay_buffers.py:83-84.  A pcgrad handle keeps the task blocks: its plan cuts the minibatch into tasks at rows
  // i / (B/T), and the losses are row sums, so the row order does not change what a step computes.
  if (rb->Teff > 1 && !rb->h->cfg.pcgrad) std::shuffle(idx.begin(), idx.end(), rb->rng);
  return 0;
}

extern "C" int b200sac_replay_sample(b200sac_replay_t* rb, int32_t replica, float* s, float* a, float* r, float* s2,
                                     float* d, int64_t* idx_out) {
  if (int rc = ring_check(rb, replica)) return rc;
  if (!s || !a || !r || !s2 || !d) return fail(B200SAC_ERR_INVALID, "null argument");
  b200sac* h = rb->h;
  if (rb->per) return fail(B200SAC_ERR_INVALID, "prioritized ring: sample with b200sac_replay_sample_prioritized (rows, indices, weights)");
  CU(cudaSetDevice(h->device));
  const int B = h->cfg.batch, rs = h->row_stride;
  std::vector<long long> idx;
  std::vector<float> row((size_t)rs);
  float* const f[ROW_FIELDS] = {s, a, r, s2, d};
  std::lock_guard<std::mutex> lk(rb->mu);
  if (int rc = host_draw(rb, replica, idx)) return rc;
  for (int i = 0; i < B; ++i) {
    const float* src = rb->rows + (size_t)replica * rb->rs_rows + (size_t)idx[i] * rs;
    if (rb->where == 0) { CU(cudaMemcpy(row.data(), src, rs * sizeof(float), cudaMemcpyDeviceToHost)); src = row.data(); }
    unpack_rows(h, src, 1, f, i);
    if (idx_out) idx_out[i] = idx[i];
  }
  return 0;
}

extern "C" int b200sac_step_sampled(b200sac_t* h, b200sac_replay_t* rb, int32_t n_steps, void* stream) {
  if (!h || !rb || rb->h != h) return fail(B200SAC_ERR_INVALID, "bad handle");
  if (n_steps < 1) return fail(B200SAC_ERR_INVALID, "n_steps < 1");
  CU(cudaSetDevice(h->device));
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  const int B = h->cfg.batch;
  if (rb->where == 0) {
    RingLocks lk(rb);                           // ordered against the writers of the ring and its prior (ring_quiesce)
    if (int rc = ring_ready(rb, kAllReplicas, 4)) return rc;
    if (int rc = prior_ready(rb)) return rc;
    int i = 0;
    if (!h->stamping)                           // (the in-graph timeline wants one step per graph)
      for (int n = kGraphSteps; n > 1; n >>= 1)
        for (; i + n <= n_steps; i += n)
          if (int rc = launch_step(h, st, GraphKey{rb, rb->rows, nullptr, n, h->stamping})) return rc;
    for (; i < n_steps; ++i)
      if (int rc = launch_step(h, st, GraphKey{rb, rb->rows, nullptr, 1, h->stamping})) return rc;
    if (int rc = record_gather(rb, st)) return rc;
    h->idx_mixed = rb->prior != nullptr;
    return sb.end();
  }
  {
    std::lock_guard<std::mutex> lk(rb->mu);
    if (int rc = ring_ready(rb, kAllReplicas, 4)) return rc;
  }
  // pinned-host ring: draw + gather on the host into the pinned slot, H2D on the side stream.  The NEXT
  // minibatch is prepared right after the current step has been launched, so host sampling, the gather and
  // the copy overlap the GPU step (the reference samples at the start of update(); here the draw for step k+1
  // happens while step k runs -- the same RNG sequence, the ring contents as of that moment).
  std::vector<long long> idx;
  const int rs = h->row_stride;
  const size_t rows_bytes = (size_t)h->R * B * rs * sizeof(float);
  auto prepare = [&](int* slot_out) -> int {
    int slot;
    if (int rc = acquire_slot(h, &slot)) return rc;
    {
      std::lock_guard<std::mutex> lk(rb->mu);
      for (int rep = 0; rep < h->R; ++rep) {
        if (int rc = host_draw(rb, rep, idx)) return rc;
        float* dst = h->stage_h[slot] + (size_t)rep * B * rs;
        const float* base = rb->rows + (size_t)rep * rb->rs_rows;
        for (int j = 0; j < B; ++j) memcpy(dst + (size_t)j * rs, base + (size_t)idx[j] * rs, rs * sizeof(float));
      }
    }
    CU(cudaMemcpyAsync(h->stage_d[slot], h->stage_h[slot], rows_bytes, cudaMemcpyHostToDevice, h->side));
    CU(cudaEventRecord(h->ev_copied[slot], h->side));
    *slot_out = slot;
    return 0;
  };
  if (h->prefetch_slot >= 0 && h->prefetch_rb != rb) h->prefetch_slot = -1;     // belongs to another ring: drop it
  for (int i = 0; i < n_steps; ++i) {
    int slot = h->prefetch_slot;
    if (slot < 0)
      if (int rc = prepare(&slot)) return rc;
    h->prefetch_slot = -1;
    CU(cudaStreamWaitEvent(st, h->ev_copied[slot], 0));
    if (int rc = launch_step(h, st, GraphKey{nullptr, h->stage_d[slot], nullptr, 1, h->stamping})) return rc;
    CU(cudaEventRecord(h->ev_consumed[slot], st));
    h->stage_used[slot] = true;
    int next;
    if (int rc = prepare(&next)) return rc;      // overlaps the step just launched
    h->prefetch_slot = next;
    h->prefetch_rb = rb;
  }
  return sb.end();
}

// ------------------------------------------------------------------------------------------
// prioritized replay (per_kernels.cuh): a device ring with one sum-tree per (replica, task) sub-ring
// ------------------------------------------------------------------------------------------
extern "C" int b200sac_replay_create_prioritized(b200sac_t* h, int64_t capacity, uint64_t seed, double alpha, double beta,
                                                 double eps, b200sac_replay_t** out) {
  if (!h || !out) return fail(B200SAC_ERR_INVALID, "null argument");
  *out = nullptr;
  if (h->cfg.critic_ensemble)
    return fail(B200SAC_ERR_INVALID, "prioritized replay is not available on a handle created with critic_ensemble");
  if (!(alpha >= 0.0) || !std::isfinite(alpha)) return fail(B200SAC_ERR_INVALID, "prioritized replay: alpha must be finite and >= 0 (got %g)", alpha);
  if (!(beta >= 0.0 && beta <= 1.0)) return fail(B200SAC_ERR_INVALID, "prioritized replay: beta must be in [0, 1] (got %g)", beta);
  if (!(eps > 0.0) || !std::isfinite(eps)) return fail(B200SAC_ERR_INVALID, "prioritized replay: eps must be finite and > 0 (got %g)", eps);
  // The smallest leaf a filled slot can hold is (0 + eps)^alpha, rounded to fp32 as per_leaf_value does.  It must be > 0:
  // then every sub-ring the sampler visits has a root > 0 and the descent, which never enters a zero-sum child, ends on a
  // filled slot.  (With a zero root it would end on leaf P - 1, past the sub-ring's filled slots or past the sub-ring.)
  const float min_leaf = (float)std::pow(eps, alpha);
  if (!(min_leaf > 0.f) || !std::isfinite(min_leaf))
    return fail(B200SAC_ERR_INVALID, "prioritized replay: the leaf of a zero priority, (0 + eps)^alpha = %g, must be > 0 and finite in fp32 "
                "(alpha %g, eps %g)", std::pow(eps, alpha), alpha, eps);
  b200sac_replay_t* rb = nullptr;
  if (int rc = b200sac_replay_create(h, capacity, 0, seed, &rb)) return rc;
  std::unique_ptr<b200sac_replay> owner(rb);       // not handed out yet: a failure below releases the whole ring
  rb->per = true;
  PerTree& tr = rb->tr;
  tr.cap = rb->cap_per_task; tr.T = rb->Teff; tr.alpha = alpha; tr.eps = eps;
  tr.P = 1; tr.levels = 0;
  while (tr.P < tr.cap) { tr.P <<= 1; ++tr.levels; }
  rb->draws.assign((size_t)h->R, 0);
  const size_t nt = (size_t)h->R * tr.T;
  CU(dev_fill(rb->tree, nt * 2 * (size_t)tr.P, 0.f));
  CU(dev_fill(rb->maxp, nt, 1.f));
  if (int rc = rb->beta.init(h->R, &beta)) return rc;
  CU(dev_alloc(rb->s_lidx, kPerMaxB));
  CU(dev_alloc(rb->s_idx, kPerMaxB));
  CU(dev_alloc(rb->s_f, kPerMaxB));
  CU(dev_alloc(rb->s_rows, (size_t)h->cfg.batch * h->row_stride));
  tr.tree = rb->tree; tr.maxp = rb->maxp;
  if (!h->per_buf) {                               // the handle's step buffers, with its first prioritized ring
    DevMem<float> per_buf;
    Stream per_fork;
    Event ev_src, ev_done;
    CU(dev_fill(per_buf, (size_t)3 * h->R * h->cfg.batch, 0.f));
    CU(new_stream(per_fork));
    CU(new_event(ev_src));
    CU(new_event(ev_done));
    h->per_buf = std::move(per_buf); h->per_fork = std::move(per_fork);
    h->ev_per_src = std::move(ev_src); h->ev_per_done = std::move(ev_done);
  }
  *out = owner.release();
  return 0;
}

extern "C" int b200sac_replay_set_beta(b200sac_replay_t* rb, int32_t replica, double beta, void* stream) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  if (!(beta >= 0.0 && beta <= 1.0)) return fail(B200SAC_ERR_INVALID, "beta must be in [0, 1] (got %g)", beta);
  return rb->beta.set(rb->h, stream, replica, &beta);
}

extern "C" int b200sac_replay_set_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, const float* prio) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  if (n < 0 || (n > 0 && (!idx || !prio))) return fail(B200SAC_ERR_INVALID, "bad argument");
  CU(cudaSetDevice(rb->h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  std::vector<int> ix((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    if (int rc = filled_slot(rb, replica, idx[i])) return rc;
    if (!(prio[i] >= 0.f) || !std::isfinite(prio[i])) return fail(B200SAC_ERR_INVALID, "priority %lld is not a finite value >= 0", (long long)i);
    if (!std::isfinite((float)std::pow((double)prio[i] + rb->tr.eps, rb->tr.alpha)))     // (alpha > 1) an inf leaf: NaN weights
      return fail(B200SAC_ERR_INVALID, "priority %lld: (%g + eps)^alpha overflows fp32", (long long)i, (double)prio[i]);
    ix[(size_t)i] = (int)idx[i];
  }
  if (int rc = ring_quiesce(rb)) return rc;
  for (int64_t i0 = 0; i0 < n; i0 += kPerMaxB) {          // chunks in order: a later index wins, as inside one chunk
    const int m = (int)std::min<int64_t>(kPerMaxB, n - i0);
    CU(cudaMemcpyAsync(rb->s_idx, ix.data() + i0, m * sizeof(int), cudaMemcpyHostToDevice, rb->st));
    CU(cudaMemcpyAsync(rb->s_f, prio + i0, m * sizeof(float), cudaMemcpyHostToDevice, rb->st));
    per_update_kernel<<<1, 256, 0, rb->st>>>(rb->tr, replica, rb->s_idx, 0, m, nullptr, nullptr, 0, rb->s_f, nullptr, nullptr, 0);
    CU(cudaGetLastError());
  }
  CU(cudaStreamSynchronize(rb->st));
  return 0;
}

extern "C" int b200sac_replay_get_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, float* p_out) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  if (n < 0 || (n > 0 && (!idx || !p_out))) return fail(B200SAC_ERR_INVALID, "bad argument");
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] >= rb->cap || idx[i] < -(long long)rb->Teff)
      return fail(B200SAC_ERR_INVALID, "index %lld: neither a ring slot [0, %lld) nor a task root [-%d, -1]", (long long)idx[i], rb->cap, rb->Teff);
  CU(cudaSetDevice(rb->h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  if (int rc = ring_quiesce(rb)) return rc;
  for (int64_t i0 = 0; i0 < n; i0 += kPerMaxB) {
    const int m = (int)std::min<int64_t>(kPerMaxB, n - i0);
    CU(cudaMemcpyAsync(rb->s_lidx, idx + i0, m * sizeof(long long), cudaMemcpyHostToDevice, rb->st));
    per_read_kernel<<<(m + 255) / 256, 256, 0, rb->st>>>(rb->tr, replica, rb->s_lidx, m, rb->s_f);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(p_out + i0, rb->s_f, m * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
    CU(cudaStreamSynchronize(rb->st));
  }
  return 0;
}

extern "C" int b200sac_replay_get_tree(b200sac_replay_t* rb, int32_t replica, int32_t task, int64_t n, float* out) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  if (task < 0 || task >= rb->Teff) return fail(B200SAC_ERR_INVALID, "task %d out of range", task);
  if (!out || n != 2 * rb->tr.P) return fail(B200SAC_ERR_INVALID, "a tree is 2P = %lld floats (got n = %lld)", 2 * rb->tr.P, (long long)n);
  CU(cudaSetDevice(rb->h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  if (int rc = ring_quiesce(rb)) return rc;
  const float* src = rb->tr.tree + ((size_t)replica * rb->tr.T + task) * 2 * rb->tr.P;
  CU(cudaMemcpyAsync(out, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
  CU(cudaStreamSynchronize(rb->st));
  return 0;
}

extern "C" int b200sac_replay_sample_prioritized(b200sac_replay_t* rb, int32_t replica, float* s, float* a, float* r, float* s2,
                                                 float* d, int64_t* idx_out, float* w_out) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  if (!s || !a || !r || !s2 || !d) return fail(B200SAC_ERR_INVALID, "null argument");
  b200sac* h = rb->h;
  const int B = h->cfg.batch, rs = h->row_stride;
  CU(cudaSetDevice(h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  if (int rc = ring_ready(rb, replica, 4)) return rc;
  if (int rc = ring_quiesce(rb)) return rc;
  per_sample_kernel<<<1, B > 256 ? 512 : 256, 0, rb->st>>>(h->K, rb->tr, nullptr, rb->draws[(size_t)replica]++, replica,
                                                           rb->d_fill, rb->beta.dev, rb->s_idx, rb->s_f, (long long)B, rb->seed);
  per_gather_kernel<<<B, 128, 0, rb->st>>>(rb->rows + (size_t)replica * rb->rs_rows, rs, rb->s_idx, rb->s_rows);
  CU(cudaGetLastError());
  std::vector<int> ix((size_t)B);
  std::vector<float> rows((size_t)B * rs), w((size_t)B);
  CU(cudaMemcpyAsync(ix.data(), rb->s_idx, B * sizeof(int), cudaMemcpyDeviceToHost, rb->st));
  CU(cudaMemcpyAsync(w.data(), rb->s_f, B * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
  CU(cudaMemcpyAsync(rows.data(), rb->s_rows, rows.size() * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
  CU(cudaStreamSynchronize(rb->st));
  float* const f[ROW_FIELDS] = {s, a, r, s2, d};
  unpack_rows(h, rows.data(), B, f, 0);
  for (int i = 0; i < B; ++i) {
    if (idx_out) idx_out[i] = ix[(size_t)i];
    if (w_out) w_out[i] = w[(size_t)i];
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// n-step returns (nstep_kernels.cuh): trajectory links on a device ring, folded by the step's gather
// ------------------------------------------------------------------------------------------
extern "C" int b200sac_replay_enable_trajectories(b200sac_replay_t* rb) {
  if (!rb) return fail(B200SAC_ERR_INVALID, "null ring");
  if (rb->where != 0) return fail(B200SAC_ERR_INVALID, "trajectory links need the device ring");
  b200sac* h = rb->h;
  std::lock_guard<std::mutex> lk(rb->mu);
  if (rb->traj) return fail(B200SAC_ERR_STATE, "the ring already has trajectory links");
  if (rb->prior || rb->prior_of) return fail(B200SAC_ERR_STATE, "the ring takes part in a prior-data attachment");
  for (auto f : rb->fill)
    if (f != 0) return fail(B200SAC_ERR_STATE, "trajectory links can only be enabled on an empty ring");
  CU(cudaSetDevice(h->device));
  if (int rc = ring_quiesce(rb)) return rc;
  const size_t nl = (size_t)h->R * rb->cap;
  DevMem<int> link, f_m;
  DevMem<long long> f_idx;
  DevMem<float> f_rows, f_disc;
  Event ev;
  CU(dev_fill(link, nl, -1));
  ReplicaTable<int> nstep;
  const int one = 1;
  if (int rc = nstep.init(h->R, &one)) return rc;
  CU(dev_alloc(f_idx, kNstepChunk));
  CU(dev_alloc(f_rows, kNstepChunk * (size_t)h->row_stride));
  CU(dev_alloc(f_disc, kNstepChunk));
  CU(dev_alloc(f_m, kNstepChunk));
  CU(new_event(ev));
  if (!h->ns_buf) {                                // the handle's step buffer, with its first linked ring
    DevMem<float> ns_buf;
    CU(dev_fill(ns_buf, (size_t)3 * h->R * h->cfg.batch, 0.f));
    h->ns_buf = std::move(ns_buf);
  }
  drop_ring_graphs(h, rb);                         // they hold the unlinked gather
  rb->d_link = std::move(link); rb->nstep = std::move(nstep); rb->f_idx = std::move(f_idx); rb->f_rows = std::move(f_rows);
  rb->f_disc = std::move(f_disc); rb->f_m = std::move(f_m); rb->ev_nstep = std::move(ev);
  rb->link_h.assign(nl, -1);
  rb->pred_h.assign(nl, -1);
  rb->tail.assign((size_t)h->R, {});
  rb->tail_at.assign((size_t)h->R, {});
  rb->traj = true;
  return 0;
}

extern "C" int b200sac_replay_close_streams(b200sac_replay_t* rb, int32_t replica, int64_t n, const int32_t* stream) {
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  if (n < 0 || (n > 0 && !stream)) return fail(B200SAC_ERR_INVALID, "bad argument");
  for (int64_t i = 0; i < n; ++i)
    if (stream[i] < 0 || stream[i] >= 65536) return fail(B200SAC_ERR_INVALID, "stream id %d outside [0, 65536)", stream[i]);
  std::lock_guard<std::mutex> lk(rb->mu);
  for (int64_t i = 0; i < n; ++i) {
    auto it = rb->tail[(size_t)replica].find(stream[i]);
    if (it != rb->tail[(size_t)replica].end()) { rb->tail_at[(size_t)replica].erase(it->second); rb->tail[(size_t)replica].erase(it); }
  }
  return 0;
}

extern "C" int b200sac_replay_set_nstep(b200sac_replay_t* rb, int32_t replica, int32_t n, void* stream) {
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  if (n < 1 || n > kNstepMax) return fail(B200SAC_ERR_INVALID, "n-step horizon must be in [1, %d] (got %d)", kNstepMax, n);
  return rb->nstep.set(rb->h, stream, replica, &n, rb->ev_nstep);
}

extern "C" int b200sac_replay_get_nstep(b200sac_replay_t* rb, int32_t replica, int32_t* n) {
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  if (!n) return fail(B200SAC_ERR_INVALID, "null argument");
  *n = *rb->nstep.row(replica);
  return 0;
}

extern "C" int b200sac_replay_get_links(b200sac_replay_t* rb, int32_t replica, int32_t task, int64_t n, int32_t* out) {
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  if (task < 0 || task >= rb->Teff) return fail(B200SAC_ERR_INVALID, "task %d out of range", task);
  if (!out || n != rb->cap_per_task) return fail(B200SAC_ERR_INVALID, "a sub-ring has %lld slots (got n = %lld)", rb->cap_per_task, (long long)n);
  CU(cudaSetDevice(rb->h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  CU(cudaMemcpyAsync(out, rb->d_link + (size_t)replica * rb->cap + (size_t)task * rb->cap_per_task, (size_t)n * sizeof(int),
                     cudaMemcpyDeviceToHost, rb->st));
  CU(cudaStreamSynchronize(rb->st));
  return 0;
}

extern "C" int b200sac_replay_fold(b200sac_replay_t* rb, int32_t replica, int64_t n_idx, const int64_t* idx, float* s, float* a,
                                   float* R, float* s2, float* d, float* disc, int32_t* m) {
  if (int rc = ring_check(rb, replica, RING_TRAJ)) return rc;
  if (n_idx < 0 || (n_idx > 0 && (!idx || !s || !a || !R || !s2 || !d || !disc || !m))) return fail(B200SAC_ERR_INVALID, "bad argument");
  b200sac* h = rb->h;
  const int obs = h->K.obs, A = h->K.act, rs = h->row_stride;
  CU(cudaSetDevice(h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  for (int64_t i = 0; i < n_idx; ++i)
    if (int rc = filled_slot(rb, replica, idx[i])) return rc;
  CU(cudaStreamWaitEvent(rb->st, rb->ev_nstep, 0));
  std::vector<float> rows((size_t)kNstepChunk * rs);
  float* const f[ROW_FIELDS] = {s, a, R, s2, d};
  for (int64_t i0 = 0; i0 < n_idx; i0 += kNstepChunk) {
    const int c = (int)std::min<int64_t>(kNstepChunk, n_idx - i0);
    CU(cudaMemcpyAsync(rb->f_idx, idx + i0, c * sizeof(long long), cudaMemcpyHostToDevice, rb->st));
    nstep_fold_kernel<<<(c + 7) / 8, 256, 0, rb->st>>>(rb->rows + (size_t)replica * rb->rs_rows, rs, obs, A,
                                                       rb->d_link + (size_t)replica * rb->cap, (int)rb->cap_per_task, rb->nstep.dev, h->hp.dev,
                                                       replica, rb->f_idx, c, rb->f_rows, rb->f_disc, rb->f_m);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(rows.data(), rb->f_rows, (size_t)c * rs * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
    CU(cudaMemcpyAsync(disc + i0, rb->f_disc, c * sizeof(float), cudaMemcpyDeviceToHost, rb->st));
    CU(cudaMemcpyAsync(m + i0, rb->f_m, c * sizeof(int), cudaMemcpyDeviceToHost, rb->st));
    CU(cudaStreamSynchronize(rb->st));
    unpack_rows(h, rows.data(), c, f, i0);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// prior-data rings (sample_mixed_kernel, ingest_mixed_kernel): a second uniform device ring whose rows fill the first m rows
// of every task block of the online ring's steps
// ------------------------------------------------------------------------------------------
// (under both rings' locks) rb goes back to a plain ring; its steps no longer read the prior once they have gathered.
static int detach_prior(b200sac_replay* rb) {
  b200sac_replay* p = rb->prior;
  if (int rc = ring_quiesce(rb)) return rc;
  if (int rc = ring_quiesce(p)) return rc;
  drop_ring_graphs(rb->h, rb);
  rb->prior = nullptr;
  p->prior_of = nullptr;
  std::fill(rb->prior_rows.host.begin(), rb->prior_rows.host.end(), 0);
  return 0;
}

extern "C" int b200sac_replay_attach_prior(b200sac_replay_t* rb, b200sac_replay_t* prior) {
  if (!rb) return fail(B200SAC_ERR_INVALID, "null ring");
  b200sac* h = rb->h;
  CU(cudaSetDevice(h->device));
  if (!prior) {
    RingLocks lk(rb);
    return rb->prior ? detach_prior(rb) : 0;
  }
  if (prior == rb) return fail(B200SAC_ERR_INVALID, "a ring cannot be its own prior");
  if (prior->h != h) return fail(B200SAC_ERR_INVALID, "the prior belongs to another handle");
  std::scoped_lock lk(rb->mu, prior->mu);
  for (const b200sac_replay* x : {rb, prior}) {
    if (x->where != 0) return fail(B200SAC_ERR_INVALID, "prior-data rings are device rings (not pinned-host)");
    if (x->per) return fail(B200SAC_ERR_INVALID, "prior-data rings are uniform (not prioritized)");
    if (x->traj) return fail(B200SAC_ERR_INVALID, "prior-data rings are unlinked (no trajectory links)");
  }
  if (rb->prior) return fail(B200SAC_ERR_STATE, "the ring already has a prior");
  if (prior->prior_of) return fail(B200SAC_ERR_STATE, "the prior is already the prior of a ring");
  if (prior->prior) return fail(B200SAC_ERR_STATE, "the prior has a prior itself");
  ReplicaTable<int> m;
  const int zero = 0;
  if (int rc = m.init(h->R, &zero)) return rc;
  if (!h->mix_idx) {                               // the handle's step buffer, with its first attachment
    DevMem<int> mix_idx;
    CU(dev_fill(mix_idx, (size_t)h->R * h->cfg.batch, 0));
    h->mix_idx = std::move(mix_idx);
  }
  if (int rc = ring_quiesce(rb)) return rc;
  if (int rc = ring_quiesce(prior)) return rc;
  drop_ring_graphs(h, rb);                         // they hold the plain draw and gather
  rb->prior_rows = std::move(m);
  rb->prior = prior;
  prior->prior_of = rb;
  return 0;
}

extern "C" int b200sac_replay_set_prior_rows(b200sac_replay_t* rb, int32_t replica, int32_t m, void* stream) {
  if (int rc = ring_check(rb, replica)) return rc;
  const int P = rb->h->cfg.batch / rb->Teff;
  if (m < 0 || m > P) return fail(B200SAC_ERR_INVALID, "prior rows must be in [0, %d] (got %d)", P, m);
  std::lock_guard<std::mutex> lk(rb->mu);
  if (!rb->prior) return fail(B200SAC_ERR_STATE, "the ring has no prior (b200sac_replay_attach_prior)");
  return rb->prior_rows.set(rb->h, stream, replica, &m);
}

extern "C" int b200sac_replay_get_prior_rows(b200sac_replay_t* rb, int32_t replica, int32_t* m) {
  if (int rc = ring_check(rb, replica)) return rc;
  if (!m) return fail(B200SAC_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(rb->mu);
  *m = rb->prior_rows.host.empty() ? 0 : *rb->prior_rows.row(replica);
  return 0;
}

// ------------------------------------------------------------------------------------------
// priority refresh (eval_kernels.cuh): a prioritized ring's leaves re-scored by the replica's current networks
// ------------------------------------------------------------------------------------------
extern "C" int b200sac_replay_refresh_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, uint64_t seed,
                                                 int32_t stochastic, void* stream) {
  if (int rc = ring_check(rb, replica, RING_PER)) return rc;
  b200sac* h = rb->h;
  if (h->cfg.care) return fail(B200SAC_ERR_STATE, "the priority refresh does not run on a CARE handle");
  if (n < 0 || (n > 0 && !idx)) return fail(B200SAC_ERR_INVALID, "bad argument");
  if (stochastic != 0 && stochastic != 1) return fail(B200SAC_ERR_INVALID, "stochastic must be 0 or 1, got %d", stochastic);
  CU(cudaSetDevice(h->device));
  std::lock_guard<std::mutex> lk(rb->mu);
  const long long cpt = rb->cap_per_task;
  const int T = rb->Teff;
  const bool full = idx == nullptr;
  std::vector<long long> slots;          // the slots to refresh: every filled one, or the caller's
  std::vector<char> touched((size_t)T, 0);
  if (full) {
    for (int t = 0; t < T; ++t) {
      const long long f = rb->fill[(size_t)replica * T + t];
      touched[(size_t)t] = f > 0;
      for (long long k = 0; k < f; ++k) slots.push_back(t * cpt + k);
    }
  } else {
    slots.resize((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      if (int rc = filled_slot(rb, replica, idx[i])) return rc;
      slots[(size_t)i] = idx[i];
      touched[(size_t)(idx[i] / cpt)] = 1;
    }
  }
  std::vector<int> tasks;
  for (int t = 0; t < T; ++t)
    if (touched[(size_t)t]) tasks.push_back(t);
  if (tasks.empty()) return 0;
  if (int rc = eval_alloc(h)) return rc;
  if (int rc = ring_quiesce(rb)) return rc;
  StreamBridge sb(h, stream);
  if (int rc = sb.begin()) return rc;
  cudaStream_t st = sb.run;
  if (rb->traj) CU(cudaStreamWaitEvent(st, rb->ev_nstep, 0));
  const EvalScratch& E = h->ev;
  const Layout& L = h->L;
  const int La = h->cfg.n_actor_hidden;
  const Buf par = rep_view(Buf{h->params, L.arena}, replica);
  CU(cudaMemcpyAsync(E.tasks, tasks.data(), tasks.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(E.tmax, 0, (size_t)T * sizeof(unsigned), st));

  RefreshGather G;
  memset(&G, 0, sizeof(G));
  G.rows = rb->rows + (size_t)replica * rb->rs_rows;
  if (rb->traj) { G.link = rb->d_link + (size_t)replica * rb->cap; G.nstep = rb->nstep.dev; }
  G.hp = h->hp.dev; G.idx = E.idx; G.XQ = E.XQ; G.XT = E.XT;
  G.R = E.R; G.d = E.d; G.g = E.g; G.eps = E.eps; G.task = E.task;
  G.key = seed ^ (kRefreshKeyMul * (unsigned long long)(replica + 1));
  G.row_stride = h->row_stride; G.obs = h->K.obs; G.act = h->K.act; G.ldx = h->K.ldx; G.cap_per_task = (int)cpt;
  G.rep = replica; G.stochastic = stochastic;
  PolicyHeadArgs P;                      // one replica's head over the chunk's rows; every row is below K.B, so a' lands in XT
  memset(&P, 0, sizeof(P));
  const LayerOff& head = L.actor[La];
  P.h = E.ha[(La - 1) & 1]; P.ldh = head.in;
  P.W = par.p + head.w; P.b = par.p + head.b;
  P.eps = E.eps; P.use_eps_buf = 1;
  P.pout = E.pout; P.psave = E.psave; P.XT = E.XT; P.XP = E.XT; P.act_out = E.act; P.logp = E.logp; P.logstd_sum = E.logstd;
  P.cnt = h->cnt;
  StepConst K = h->K;
  K.B = (int)E.rows;
  RefreshTd D;
  memset(&D, 0, sizeof(D));
  D.Tr = rb->tr; D.idx = E.idx; D.R = E.R; D.d = E.d; D.g = E.g; D.task = E.task; D.logp = E.logp; D.q = E.q; D.qt = E.qt;
  D.log_alpha = par.p + L.off_alpha; D.hp = h->hp.dev; D.tmax = E.tmax; D.rep = replica;

  const long long total = (long long)slots.size();
  for (long long i0 = 0; i0 < total; i0 += E.rows) {
    const int m = (int)std::min<long long>(E.rows, total - i0);
    CU(cudaMemcpyAsync(E.idx, slots.data() + i0, (size_t)m * sizeof(long long), cudaMemcpyHostToDevice, st));
    G.n = m;
    refresh_gather_kernel<<<(m + 7) / 8, 256, 0, st>>>(G);
    for (int l = 0; l < La; ++l) {
      GemmProb p = fwd_prob(par, l == 0 ? E.XT : E.ha[(l - 1) & 1], 0, m, L.actor[l], E.ha[l & 1], 0);
      if (l == 0) p.lda = h->K.ldx;
      act_gemm({p}, st);
    }
    P.rows = m;
    policy_head_kernel<<<dim3((m + 7) / 8, 1), 256, 0, st>>>(K, P);
    eval_critics(h, st, replica, L.qt, E.XT, m, E.qt);
    eval_critics(h, st, replica, L.q, E.XQ, m, E.q);
    D.n = m;
    refresh_td_kernel<<<(m + 255) / 256, 256, 0, st>>>(D);
    CU(cudaGetLastError());
  }
  for (int lv = 1; lv <= rb->tr.levels; ++lv) {
    const long long nodes = rb->tr.P >> lv;
    per_rebuild_level_kernel<<<dim3((unsigned)std::min<long long>(1024, (nodes + 255) / 256), (unsigned)tasks.size()), 256, 0, st>>>(
        rb->tr, replica, E.tasks, lv);
  }
  refresh_maxp_kernel<<<1, 256, 0, st>>>(rb->tr, replica, E.tasks, (int)tasks.size(), E.tmax, full ? 1 : 0);
  CU(cudaGetLastError());
  if (int rc = sb.end()) return rc;
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}
