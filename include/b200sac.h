/*
 * b200sac.h -- C ABI of the H100-native (sm_90a) SAC learner hot path.
 *
 * The reference (SKSKSK94/Distributed_SAC) is pure Python and has no FFI; the seam
 * this library sits behind is the Python method surface of `Learner` /
 * `ReplayBuffer`.  Each entry point below names the reference code it replaces
 * (paths relative to the reference checkout):
 *
 *   b200sac_step*, b200sac_update
 *                            Learner.update() -> update_SAC()
 *                            LunarLander_Distributed_SAC/src/learner.py:246-264,203-239
 *                            MT1_Distributed_VSAC/src/learner.py:205-244,251-269
 *                            MT10_Distributed_MTSAC/src/learner.py:253-325,332-352
 *                            MT10_Distributed_CARE/src/learner.py:281-404 (care = 1 | 2), MT1_Distributed_CARE/src/learner.py:247-348
 *   b200sac_replay_*         ReplayBuffer.sample()/__len__ and the append in run()
 *                            LunarLander_Distributed_SAC/src/replay_buffer.py:43-77
 *                            MT10_Distributed_MTSAC/src/replay_buffers.py:47-107
 *   b200sac_layout/export/import
 *                            build_model/build_optimizer/save_checkpoint
 *                            LunarLander_Distributed_SAC/src/learner.py:100-124,144-163
 *   b200sac_soft_update      Learner.soft_update()            learner.py:126-137
 *   b200sac_get/set_hparams, b200sac_copy_replica
 *                            the hyperparameters build_optimizer / update_SAC / soft_update fix per learner, made per replica
 *   b200sac_reset            build_model + build_optimizer again for some networks of one replica (periodic resets,
 *                            shrink-and-perturb), keeping the replay ring
 *                            LunarLander_Distributed_SAC/src/learner.py:115-137,210; MT10_Distributed_CARE/src/learner.py:136-158,361-367
 *   b200sac_redo, b200sac_read_redo
 *                            dormant-neuron recycling (ReDo) of one replica and its record of neuron scores
 *   b200sac_get/set_update_intervals
 *                            actor / target update intervals (TD3 policy_delay, pytorch_sac actor_update_frequency and
 *                            critic_target_update_frequency, SB3 target_update_interval), per replica
 *   b200sac_set/get_grad_clip, b200sac_read_grad_norms
 *                            torch.nn.utils.clip_grad_norm_ before each optimizer.step() (Ape-X's max-norm 40, the
 *                            max_grad_norm of SAC / TD3 code bases) and the norms it returns, per replica and optimizer
 *   b200sac_set/get/read_pcgrad, b200sac_export_task_grad
 *                            PCGrad gradient surgery (Yu et al., NeurIPS 2020) for the multi-task learners' optimizers,
 *                            per replica and optimizer, with the step's Gram matrix and surgery decisions reported
 *   b200sac_set/get_critic_dropout
 *                            Dropout Q-functions (DroQ, Hiraoka et al., ICLR 2022): dropout before every critic LayerNorm,
 *                            with a rate per replica
 *   b200sac_set/get/read_cagrad, b200sac_cagrad_solve_test
 *                            CAGrad (Liu et al., NeurIPS 2021) on the same handles, per replica and optimizer, with the
 *                            step's dual solution reported
 *   b200sac_blob_*           Learner.get_parameters() and server.set('parameters', _pickle.dumps(get_parameters())) in
 *                            Learner.run(), learner.py:272-276,298-299 (MT10_Distributed_CARE/src/learner.py:412-417,442-443):
 *                            the byte string, device-assembled
 *   b200sac_act              Actor.get_action() for a batch of environments
 *                            LunarLander_Distributed_SAC/src/model.py:67-82; MT10_Distributed_CARE/src/player.py:199-209 (CARE handles)
 *   b200sac_critic_values    Critic.forward() (q1, q2 or their targets) for any number of rows, in eval mode
 *                            LunarLander_Distributed_SAC/src/model.py (Critic); not on CARE handles
 *   b200sac_replay_refresh_priorities
 *                            PER priorities of a ring's slots recomputed with the current networks (after resets, ReDo)
 *
 * Conventions: plain pointers and sizes only (no torch types).  Every function
 * returns 0 on success or a negative b200sac_status; a message for the calling
 * thread is available from b200sac_last_error().  No exceptions cross the
 * boundary.  All device work is enqueued on the caller's stream (a
 * cudaStream_t passed as void*; NULL = legacy default stream).  A handle is
 * single-caller (not re-entrant); distinct handles are independent.
 * `replicas` independent learners of the same shape can live in one handle and
 * are stepped together (grouped launches); every per-learner array then has a
 * leading replica dimension.
 */
#ifndef B200SAC_H_
#define B200SAC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SAC_MAX_HIDDEN 8

typedef enum b200sac_status {
  B200SAC_OK = 0,
  B200SAC_ERR_INVALID = -1,   /* bad argument / unsupported shape */
  B200SAC_ERR_CUDA = -2,      /* a CUDA runtime call failed for any other reason */
  B200SAC_ERR_NOMEM = -3,     /* out of host memory, or a CUDA runtime call failed with cudaErrorMemoryAllocation */
  B200SAC_ERR_STATE = -4      /* call not valid in this state (e.g. replay too small) */
} b200sac_status;

/* Mirrors the cfg JSON + hard-coded dims of the reference learners
 * (cfg/*.json; LL/learner.py:62-81; MS/learner.py:62-98). */
typedef struct b200sac_cfg {
  int32_t state_dim;                 /* raw state width (8 / 39) */
  int32_t act_dim;                   /* 2 / 4 */
  int32_t num_tasks;                 /* 0 = single task; T>0 = one-hot appended to the state (mtobs) */
  int32_t n_actor_hidden;            /* number of hidden layers */
  int32_t n_critic_hidden;
  int32_t actor_hidden[B200SAC_MAX_HIDDEN];
  int32_t critic_hidden[B200SAC_MAX_HIDDEN];
  int32_t batch;                     /* minibatch per learner */
  int32_t weighted_loss;             /* MTSAC use_weighted_loss (== extra 1/batch, SURVEY 0.6) */
  int32_t replicas;                  /* independent learners in this handle (>= 1) */
  int32_t precision;                 /* 0 = fp32 FFMA; 1 = 3xTF32 on wgmma for hidden layers */
  int32_t care;                      /* CARE state encoders (MT10_Distributed_CARE/src/{context,state}_encoder.py):
                                        1 = CARE(M) use_modified_care=true: frozen embedding, per-encoder mlp_context;
                                        2 = CARE(O) use_modified_care=false (= MT1_Distributed_CARE): trainable context
                                            encoder z = mlp(header(relu(E[t]))) with its own Adam (lr_ctx) */
  double gamma, tau, reward_scale;
  double lr_actor, lr_critic, lr_alpha;
  double action_scale;               /* k = (hi - lo) / 2 */
  double beta1, beta2, adam_eps;
  double log_alpha_init;
  /* CARE only (cfg "encoder" block): */
  int32_t num_encoders;              /* K (num_encoders) */
  int32_t n_mix_hidden;              /* hidden_dims_mixtureEnc (also the attention trunk's hidden dims) */
  int32_t mix_hidden[B200SAC_MAX_HIDDEN];
  int32_t mix_out;                   /* output_dim_mixtureEnc */
  int32_t ctx_in;                    /* RoBERTa_embedding_dim (768) */
  int32_t n_ctx_hidden;              /* hidden_dims_contextEnc */
  int32_t ctx_hidden[B200SAC_MAX_HIDDEN];
  int32_t ctx_out;                   /* output_dim_contextEnc */
  int32_t emb_dim;                   /* embedding_dim_contextEnc: CARE(O) header = Linear(ctx_in, 2e), Linear(2e, e) */
  double tau_se;                     /* state_encoder_tau */
  double lr_ctx;                     /* lr_contextEnc (CARE(O) context-encoder Adam) */
  int32_t grad_clip;                 /* 0 = the default plan; 1 = the plan with gradient-norm clipping and gradient norms
                                        (b200sac_set_grad_clip), every threshold +inf at create.  Fixed at create. */
  int32_t pcgrad;                    /* 0 = the default plan; 1 = the per-layer plan with PCGrad gradient surgery
                                        (b200sac_set_pcgrad), both switches on at create.  Needs num_tasks >= 2 and
                                        grad_clip = 0; MTSAC and CARE (care = 1 | 2) alike.  Fixed at create. */
  int32_t critic_ensemble;           /* 0 = the twin critics q1, q2; E in [2, B200SAC_MAX_ENSEMBLE] = E critics q1 .. qE with
                                        a per-replica target subset (b200sac_set_ensemble).  Fixed at create.  See "Critic
                                        ensembles" below. */
  int32_t critic_ln;                 /* 0 = the default plan; 1 = LayerNorm in the critics' hidden layers.  Fixed at create.
                                        See "Layer-normalized critics" below. */
  int32_t critic_dropout;            /* 0 = the critic_ln plan; 1 = dropout before every critic LayerNorm (DroQ), the rate
                                        set per replica by b200sac_set_critic_dropout.  Needs critic_ln = 1.  Fixed at
                                        create.  See "Dropout Q-functions" below. */
} b200sac_cfg;

#define B200SAC_MAX_ENSEMBLE 10

/* Layer-normalized critics (cfg.critic_ln = 1; Ba et al. 2016, as high-replay-ratio SAC uses it: DroQ, Lyle et al. 2023,
 * BRO).  Every hidden layer l of q1, q2, q1_target and q2_target, width H, is nn.Sequential(Linear, nn.LayerNorm(H,
 * eps=1e-5), ReLU):
 *   z = W_l x + b_l;  mu = (1/H) sum_j z_j;  var = (1/H) sum_j (z_j - mu)^2 (biased);  rstd = 1 / sqrt(var + 1e-5);
 *   xhat = (z - mu) * rstd;  h = relu(g_l * xhat + c_l).
 * The heads and the actor are unchanged.  Numerics (fp64 throughout, no fused multiply-add, one rounding to fp32 at the
 * end of each output):
 *   - a row sum over j: lane k of one warp adds j = k, k + 32, ... in increasing order from 0.0, then the 32 lane sums are
 *     combined by the xor butterfly with offsets 16, 8, 4, 2, 1.  mu and var are such sums divided by H; h is
 *     (float)(g * xhat + c) with a negative value replaced by 0 (a NaN stays NaN);
 *   - backward, dy = the ReLU-masked gradient at h: a = (row sum of g*dy) / H, b = (row sum of g*dy*xhat) / H, and
 *     dz = (float)(rstd * ((g*dy - a) - xhat * b));
 *   - dg_l = sum over the batch of dy*xhat and dc_l = sum of dy, per critic: rows cut into chunks of 16 in row order, each
 *     chunk's sum over its rows in increasing order from 0.0, then the chunk sums added in chunk order and rounded once.
 *     No floating-point atomics: the result is bit-reproducible and does not depend on the replica count.
 * Parameters: <net>.<l>.ln.weight and <net>.<l>.ln.bias, shape (H, 1), right after <net>.<l>.bias; trainable with opt 0
 * in q1 / q2, trainable 0 and opt -1 in the targets (at + target_delta, like every target tensor).  q1, q2 and their
 * targets stay contiguous, so the critic Adam, the Polyak updates, b200sac_soft_update(_critic), b200sac_copy_replica,
 * export / import and the gradient-clipping norm cover them.  Create: g = 1, c = 0, targets = locals; they take no Philox
 * tag, so every Linear tensor is bit-identical to the same cfg with critic_ln = 0.  b200sac_reset: the LayerNorm of
 * hidden Linear i goes with that Linear's depth; its fresh draw is g = 1, c = 0.
 * Plan: always the per-layer plan (never the layer-chained one), at precision 0 and 1.  Each of the passes A (critics
 * on (s, a)), B (targets on (s', a')) and D (critics on (s, a~), the actor pass) runs its hidden GEMMs without ReLU into
 * the pre-normalization buffers and one forward LayerNorm launch per layer for both critics and every replica; the
 * critic backward (C) and the actor pass's input gradient (D) run one backward launch per layer before that layer's
 * weight and input gradients.  A step has 5 * n_critic_hidden launches more than the same cfg's per-layer plan
 * without critic_ln; they are labelled "ln_fwd{critic|target|actor pass <l>}" and "ln_bwd{critic|actor pass <l>}".
 * The actor-pass launches return at entry on a critic-only step.
 * Refused with B200SAC_ERR_INVALID by b200sac_layout and b200sac_create: critic_ln outside {0, 1}, or together with
 * care != 0 or pcgrad = 1.  b200sac_redo on such a handle gives B200SAC_ERR_STATE (see there). */

/* Dropout Q-functions (cfg.critic_dropout = 1; DroQ, Hiraoka et al., ICLR 2022).  On a critic_ln handle, every hidden
 * layer l of q1, q2, q1_target and q2_target becomes nn.Sequential(Linear, Dropout(p), LayerNorm, ReLU), in training
 * mode on every critic evaluation of the step: pass A (critics on (s, a)), pass B (targets on (s', a')) and pass D
 * (critics on (s, a~), the actor pass).  With p the replica's rate (b200sac_set_critic_dropout; 0 at create):
 *   z' = z * (m ? s : 0) with z = W_l x + b_l, then h = relu(LN(z')) as under "Layer-normalized critics";
 *   s = (float)(1 / (1 - p)), evaluated in fp64 and rounded once; the product is one fp32 multiply;
 *   m in {0, 1}: an element is dropped iff its 32-bit Philox word is below t = floor(p * 2^32) (fp64, on the host).
 * p = 0 drops nothing and multiplies by 1: the step is bit-identical to the same handle with critic_dropout = 0.
 * Random stream: Philox4x32-10 with key = seed ^ (0xE7037ED1A0B428DB * (replica + 1)) (mod 2^64; seed = b200sac_create's,
 * the policy noise's; key[0] = its low 32 bits, key[1] = its high 32 bits), a multiplier no other draw of the library uses;
 * counter (c0, c1, c2, c3) = (step & 0xFFFFFFFF, step >> 32, b, (tag << 24) | (j / 4)) where step = the replica's step
 * index the policy noise uses (the number of steps the replica has run, this one included; 1 on the first), b the row of
 * the minibatch (0..batch-1), j the column (0..H-1) and tag = (pass * 8 + l) * 2 + net with pass A = 0, B = 1, D = 2 and
 * net = 0 for q1 / q1_target, 1 for q2 / q2_target.  Column j takes output word j % 4.  Masks therefore do not depend on
 * the replica count, and differ per step, pass, layer, net and replica.
 * Backward: dz = dz' * (m ? s : 0), dz' the LayerNorm backward's output as without dropout; the weight and input
 * gradients and the LayerNorm weight / bias gradients follow unchanged.  On a critic-only step the pass-D launches return
 * at entry: no pass-D masks are drawn.
 * Plan: the same launches and labels as the critic_ln plan; the LayerNorm launches draw, apply and keep the masks (bits
 * [2][batch][ceil(H / 32)] per replica, pass and layer; column j is bit j % 32 of word j / 32).  No parameters: the layout
 * is that of the same cfg with critic_dropout = 0.  The rate is not copied by b200sac_copy_replica and not part of the
 * parameter arenas.  b200sac_critic_values and b200sac_replay_refresh_priorities evaluate the critics in eval mode: no
 * dropout, whatever the rate.
 * Refused with B200SAC_ERR_INVALID by b200sac_layout and b200sac_create: critic_dropout outside {0, 1}, or 1 with
 * critic_ln = 0. */

/* Critic ensembles (cfg.critic_ensemble = E in [2, 10]; REDQ, Chen et al., ICLR 2021; RLPD, Ball et al., ICML 2023).
 * Networks: q1 .. qE and q1_target .. qE_target, all of the shape of q1.  q3 .. qE follow q2 in the trainable critic block
 * and q3_target .. follow q2_target, so every critic k has its target at + target_delta and the critic Adam, the Polyak
 * updates, b200sac_copy_replica, export / import and the critic gradient-clipping norm cover all E.  The Xavier tags of
 * q3 .. qE come after q2's: actor, q1, q2, their targets and log_alpha are bit-identical to a twin handle created with
 * the same seed.  critic_ln / critic_dropout parameters and masks follow per critic as for the twins.
 * Per replica (b200sac_set_ensemble; m = 2 and MEAN at create): the subset size m in [1, E] and the actor reduction.
 *   Critic loss: sum over k of the mean((y - Q_k)^2) terms with the twin plan's weighting; dL/dQ_k = 2 c (Q_k - y), with
 *     the squared errors added in index order.
 *   TD target: y = rs r + gamma (1 - d)(min_{k in S} Qt_k - alpha logpi'), the min folded with fminf in increasing index
 *     order.  All E targets are evaluated; S holds m of them.
 *   Subset S, one per replica and step (every row of the minibatch): m = E takes all E without a draw.  Otherwise
 *     Philox4x32-10 with key = seed ^ (0x8EBC6AF09C88C6E3 * (replica + 1)) (mod 2^64; seed = b200sac_create's; a multiplier
 *     no other draw uses) and counter (step & 0xFFFFFFFF, step >> 32, 0, q) gives words w_{4q} .. w_{4q+3}; S is the m
 *     indices k with the smallest pairs (w_k, k).  step = the replica's step index the policy noise uses.  The draw does
 *     not depend on the replica count and runs on critic-only steps too.  debug_read "tsub" [E] holds the last step's S
 *     as 0.0 / 1.0.
 *   Actor loss (the actor pass): MEAN: Q = (sum_k Q_k) / E, the sum in index order, each critic gets -c / E.  MIN: Q =
 *     the fminf fold over all E; the gradient -c is split evenly among the critics equal to the minimum (torch.amin's
 *     backward).  The action's input gradient adds the E critics' contributions in index order.
 *   critic_dropout: the tag of critic k's masks is (pass * 8 + l) * E + k (the twin formula at E = 2).
 * A twin handle runs the same kernels with its table fixed at m = 2 and MIN (b200sac_get/set_ensemble still refuse it), so
 * E = 2 with m = 2 and MIN computes exactly what the twin per-layer plan computes, bit for bit.
 * Plan: always the per-layer plan (never the layer-chained one), at precision 0 and 1.  The extra critics are extra problems
 * in the same grouped launches; a step has the launches and labels of the same cfg with critic_ensemble = 0 on the
 * per-layer plan, plus any launch a grouped GEMM's GS_MAXG split adds.
 * Entry points: b200sac_critic_values writes q_out[E][n]; b200sac_soft_update_critic takes critic in [1, E];
 * b200sac_debug_read gains "q<k>" (k <= E) and "tsub", and "q_pi", "dq_pi" and the per-pass "h/z/m<pass>.<l>" hold E
 * critics; b200sac_reset's CRITIC part re-draws all E with the same depth rule.
 * Refused with B200SAC_ERR_INVALID by b200sac_layout and b200sac_create: critic_ensemble outside {0} and [2, 10], or with
 * care != 0 or pcgrad = 1.  b200sac_redo gives B200SAC_ERR_STATE and b200sac_replay_create_prioritized B200SAC_ERR_INVALID
 * on an ensemble handle. */

typedef struct b200sac_tensor_desc {
  char name[48];                     /* canonical name, e.g. "q1_target.2.weight" */
  int64_t offset;                    /* in floats, inside one replica's parameter arena */
  int32_t rows, cols;                /* weight: (out, in) row-major; bias/log_alpha: (n, 1) */
  int32_t trainable;                 /* 1 -> has Adam m/v at the same offset in the m/v arenas */
  int32_t opt;                       /* 0 critic, 1 actor, 2 alpha, 3 context encoder, -1 none (targets, embedding) */
  int32_t pitch;                     /* floats between consecutive rows (>= cols): first-layer weights are padded to a
                                        multiple of 4 so that TMA can address them; pad columns are and stay zero */
  int32_t reserved;
} b200sac_tensor_desc;

typedef struct b200sac b200sac_t;               /* learner handle */
typedef struct b200sac_replay b200sac_replay_t; /* replay ring handle */

/* arenas addressable through export/import */
enum { B200SAC_PARAMS = 0, B200SAC_ADAM_M = 1, B200SAC_ADAM_V = 2, B200SAC_GRADS = 3 };

const char* b200sac_last_error(void);
const char* b200sac_version(void);

/* Pure host function (no GPU needed): parameter layout for a cfg.
 * Writes up to `cap` descriptors, returns the total count in *n and the arena
 * size (floats per replica; trainable prefix length) in *arena_floats / *trainable_floats. */
int b200sac_layout(const b200sac_cfg* cfg, b200sac_tensor_desc* out, int32_t cap, int32_t* n,
                   int64_t* arena_floats, int64_t* trainable_floats);

/* Create a learner on CUDA device `device`.  Parameters are Xavier-uniform /
 * zero-bias initialised from `seed` (replica r uses seed + r); targets = locals. */
int b200sac_create(const b200sac_cfg* cfg, int32_t device, uint64_t seed, b200sac_t** out);
int b200sac_destroy(b200sac_t* h);

/* Copy one replica's arena out / in.  `buf` may be a host or a device pointer. */
int b200sac_export(b200sac_t* h, int32_t which, int32_t replica, float* buf, int64_t n_floats, void* stream);
int b200sac_import(b200sac_t* h, int32_t which, int32_t replica, const float* buf, int64_t n_floats, void* stream);
/* n_floats floats at `offset` of one replica's arena into HOST memory (the logger's read of log_alpha, learner.py:199:
 * a handful of floats instead of the whole arena).  Synchronises the stream. */
int b200sac_read_range(b200sac_t* h, int32_t which, int32_t replica, int64_t offset, int64_t n_floats, float* out_host,
                       void* stream);
/* Device address of an arena (replica 0; replicas are contiguous, stride = arena floats).  For
 * zero-copy views and for the one-time NCCL broadcast of initial weights done by the host shim. */
int b200sac_arena_ptr(b200sac_t* h, int32_t which, float** dev_ptr, int64_t* floats_per_replica);
/* Adam step counters {critic, actor, alpha, context encoder (CARE(O), else unused)} of one replica. */
int b200sac_get_steps(b200sac_t* h, int32_t replica, int64_t steps[4]);
int b200sac_set_steps(b200sac_t* h, int32_t replica, const int64_t steps[4]);

/* Per-replica hyperparameters.  The reference fixes them when it builds a learner: the TD target and the Polyak rate
 * (LunarLander_Distributed_SAC/src/learner.py:126-137,210; MT10_Distributed_CARE/src/learner.py:361-367 with
 * state_encoder_tau) and the Adam learning rates (LunarLander_Distributed_SAC/src/learner.py:115-124;
 * MT10_Distributed_CARE/src/learner.py:136-158).  Here every replica of a handle has its own row, initialised from the
 * cfg by b200sac_create, so co-scheduled learners can sweep them (e.g. population-based training) and a schedule can
 * change them between steps.  action_scale, the Adam betas / eps and the target entropy stay per handle. */
typedef struct b200sac_hparams {
  double gamma, reward_scale, tau;          /* TD target; Polyak rate of the target critics */
  double lr_critic, lr_actor, lr_alpha;     /* Adam learning rates */
  double tau_se, lr_ctx;                    /* CARE: state-encoder Polyak rate; CARE(O) context-encoder lr (ignored otherwise) */
} b200sac_hparams;

/* The values last set for `replica` (host mirror: does not synchronise). */
int b200sac_get_hparams(b200sac_t* h, int32_t replica, b200sac_hparams* out);
/* Enqueued on `stream`: applies to every step enqueued after it and to none enqueued before it, including between
 * launches of the graphs b200sac_prepare instantiated (no graph is rebuilt).  Every value must be finite,
 * 0 <= tau, tau_se <= 1 and learning rates >= 0; otherwise B200SAC_ERR_INVALID and nothing changes.  b200sac_soft_update
 * uses the replica's tau_se for the CARE state encoder. */
int b200sac_set_hparams(b200sac_t* h, int32_t replica, const b200sac_hparams* hp, void* stream);
/* Enqueued on `stream`: replica `dst`'s learner state becomes a copy of `src`'s -- the whole parameter arena (targets,
 * log_alpha and the CARE embedding included), Adam m and v and the step counters -- device to device, without a host
 * round trip (the exploit step of population-based training).  Hyperparameters, update intervals, gradient-clipping
 * thresholds, gradients and replay rings are not copied. */
int b200sac_copy_replica(b200sac_t* h, int32_t src, int32_t dst, void* stream);

/* Network resets and shrink-and-perturb, per replica (Nikishin et al. 2022; D'Oro et al. 2023; Ash & Adams 2020).
 * Parts a reset can touch, index of b200sac_reset_spec.part[]:
 *   ACTOR    the actor MLP (actor.*);
 *   CRITIC   q1 and q2, the same depth for both; their targets follow;
 *   ALPHA    log_alpha, every task;
 *   ENCODER  the CARE critic state encoder cse.* (mixture, attention trunk and, CARE(M), the context MLP); its target tse
 *            follows, and so does the actor's state encoder, which is its tied copy.  Not on a non-CARE handle;
 *   CONTEXT  the CARE(O) context encoder cenc.*.  Only on CARE(O) handles.
 * The frozen CARE embedding is never touched. */
enum { B200SAC_RESET_ACTOR = 0, B200SAC_RESET_CRITIC = 1, B200SAC_RESET_ALPHA = 2,
       B200SAC_RESET_ENCODER = 3, B200SAC_RESET_CONTEXT = 4, B200SAC_RESET_PARTS = 5 };
typedef struct b200sac_reset_part {
  int32_t layers;   /* ACTOR / CRITIC: Linear layers counted from the output layer (1 = the head only); 0 = untouched;
                       >= the network's Linear count = all.  ALPHA / ENCODER / CONTEXT: 0 or 1 (all or nothing). */
  int32_t reserved;
  double shrink;    /* lambda in [0, 1]: 0 = fresh draw, 1 = keep the values (the optimizer state is still reset) */
} b200sac_reset_part;
typedef struct b200sac_reset_spec { b200sac_reset_part part[B200SAC_RESET_PARTS]; } b200sac_reset_spec;

/* Enqueued on `stream`: re-initialise the parts `spec` names of replica `replica`.
 * Fresh draw theta0 of every touched tensor: what b200sac_create(seed) gives replica `replica` -- the same Philox key
 * (seed + replica) and per-tensor tag, Xavier-uniform weights, zero biases, N(0,1) CARE mixture weights and biases,
 * cfg.log_alpha_init for log_alpha.  A reset with the create seed and shrink 0 therefore reproduces the created
 * parameters bit for bit.
 * Blend, per element, lambda = the part's shrink:
 *   lambda = 0: theta' = theta0 (a select: a reset also recovers a NaN or inf network);
 *   otherwise:  theta' = (float)(lambda * theta + (1 - lambda) * theta0), evaluated in fp64 with 1 - lambda in fp64 and
 *               rounded once, no fused multiply-add.
 * A touched critic or state-encoder tensor's target gets the same blend of its own value with the same theta0, so at
 * lambda = 0 the targets equal the new locals, as after create.  Pad columns of first-layer weights stay zero.
 * Optimizer state: every optimizer that owns a touched tensor starts afresh, as if the torch optimizer were re-created:
 * Adam m = v = 0 over its whole slice, its step count 0 and its beta-power products 1 (the values create writes).  The
 * owners are the critic (counter slot 0: q1, q2 and cse) for CRITIC or ENCODER, the actor (slot 1) for ACTOR, the
 * temperature (slot 2) for ALPHA and the context encoder (slot 4) for CONTEXT.  This is all or nothing per optimizer,
 * because the counters are per optimizer, not per tensor: a head-only critic reset restarts Adam for all of q1, q2 and cse.
 * Left alone: the step index (the Philox noise stream and the loss-ring slots continue), gradient arenas and PCGrad
 * slices, every per-replica setting (hyperparameters, update intervals, clip thresholds, PCGrad / CAGrad), replay rings,
 * PER priorities and n-step links, and the other replicas.  The update-interval phase follows the critic count, as after
 * b200sac_set_steps: a critic reset restarts it.
 * Stream order as b200sac_set_hparams: steps enqueued before the call are unaffected and steps enqueued after it see the
 * reset, including launches of the graphs b200sac_prepare instantiated (no graph is rebuilt); b200sac_act and the next
 * b200sac_blob_begin see the new actor.
 * A NULL spec, a bad replica, layers < 0, an all-or-nothing part with layers > 1, shrink outside [0, 1] or NaN, ENCODER on
 * a non-CARE handle or CONTEXT on a handle that is not CARE(O) give B200SAC_ERR_INVALID, and nothing is enqueued. */
int b200sac_reset(b200sac_t* h, int32_t replica, const b200sac_reset_spec* spec, uint64_t seed, void* stream);

/* Dormant-neuron recycling, ReDo (Sokar, Agarwal, Castro, Evci, ICML 2023), per replica.  Enqueued on `stream`:
 * 1. Forward.  With replica `replica`'s current parameters, the actor's hidden layers on obs[n][state_dim + num_tasks]
 *    and q1's and q2's on (obs, act[n][act_dim]), 1 <= n <= batch rows in host or device memory, on the per-layer fp32
 *    FFMA engine b200sac_act uses, whatever the handle's plan or precision.  CARE handles first encode the rows as
 *    b200sac_act does (the critic's state encoder cse, of which the actor's is the tied copy); the critic input is that
 *    encoding with act appended, laid out as the step's XQ.  The results land in the step's own XA / XQ / hA / hQ
 *    buffers, rows [0, n) of each network (the next step recomputes all of them), so debug_read("hA.<l>") and
 *    debug_read("hQ.<l>") show them afterwards: hA rows [0, n), hQ rows [0, n) of q1 and [batch, batch + n) of q2.
 * 2. Scores.  For every hidden layer of N in {actor, q1, q2} with H neurons: a_i = (1/n) sum_rows max(h_ri, 0),
 *    mean = (1/H) sum_j a_j, s_i = a_i / mean (every s_i = 0 when mean = 0).  Both sums in fp64 in one fixed order that
 *    does not depend on the replica count, no floating-point atomics.  Neuron i is dormant iff s_i <= tau, tau =
 *    tau_actor for the actor and tau_critic for q1 and q2 (each critic scored on its own neurons); a NaN score is never
 *    dormant, and a negative tau (-inf included) recycles nothing: the measure-only call.
 * 3. Recycle, for every dormant neuron i of hidden layer l:
 *    - row i of W_l becomes what b200sac_create(seed) draws for those elements: the same Philox key (seed + replica),
 *      tag and element index as b200sac_reset's theta0; pad columns stay zero;
 *    - b_l[i] = 0;
 *    - column i of the next weight matrix (the next hidden layer's, or for the last hidden layer the head's: the Q head,
 *      or the policy head's mu and log-std rows) = 0, except where that entry lies in a recycled row of the next hidden
 *      layer, which takes the draw (that neuron's own outgoing column is zero, so the function is the same either way);
 *    - Adam m = v = 0 at exactly those entries.  Step counters and beta-power products are unchanged: ReDo resets
 *      moments, not optimizers.
 *    Left alone: targets (the network's function is unchanged, so the Polyak average stays valid), log_alpha, the CARE
 *    encoders, gradients and PCGrad slices, per-replica settings, replay rings and the other replicas.
 * 4. Record.  Per replica, each hidden neuron's score (fp64) and dormant flag, actor layers, then q1's, then q2's, in
 *    layer order; NaN scores and 0 flags before the first call.  b200sac_read_redo reads it.
 * Stream order as b200sac_reset: steps enqueued before the call are unaffected, steps enqueued after it (launches of
 * graphs b200sac_prepare instantiated included; no graph is rebuilt) see the recycled networks.  Does not synchronise.
 * A bad replica, n outside [1, batch], a NULL obs or act, or a NaN tau give B200SAC_ERR_INVALID, and nothing is
 * enqueued.  A handle created with critic_ln gives B200SAC_ERR_STATE and nothing is enqueued: this forward has no
 * LayerNorm, and recycling one unit would change its whole row's statistics, so the recycle would not preserve the
 * network's function. */
int b200sac_redo(b200sac_t* h, int32_t replica, int32_t n, const float* obs, const float* act, double tau_actor,
                 double tau_critic, uint64_t seed, void* stream);

/* The last b200sac_redo record of replica `replica`: scores[*n_neurons] and dormant[*n_neurons] (either may be NULL), in
 * the order b200sac_redo states; cap = the capacity of each.  Synchronises the stream. */
int b200sac_read_redo(b200sac_t* h, int32_t replica, double* scores, uint8_t* dormant, int64_t cap, int64_t* n_neurons,
                      void* stream);

/* Per-replica update intervals, both 1 (every step is a full step) after b200sac_create.  Let n be the replica's critic
 * Adam step count after a step (steps[0] of b200sac_get_steps).  The step is
 *   - an ACTOR step iff n % actor_every == 0: it updates the actor and the temperature log_alpha (Adam), as always.  On any
 *     other step (a critic-only step) the actor parameters, log_alpha, their Adam m / v and the actor and temperature step
 *     counters are left bit for bit as they were: exactly as if the reference skipped actor_optimizer.step() and
 *     alpha_optimizer.step(), so Adam's bias correction counts only the updates that happened;
 *   - a TARGET step iff n % target_every == 0: the target critics get their Polyak update (tau) and, with CARE, the target
 *     state encoder its update (tau_se).  On other steps the targets are not written at all.
 * Everything else runs on every step: the critic update (TD target with the current actor and the temperature of the
 * step), prioritized-replay weights and priority updates, the CARE(O) context encoder's Adam, the step index.
 * The phase follows the counters, so it carries over b200sac_set_steps, checkpoint restores and b200sac_copy_replica
 * (which copies the counters but, like the hyperparameters, not the intervals).
 * Set: enqueued on `stream` like b200sac_set_hparams -- applies to every step enqueued after it and to none enqueued before
 * it, including between launches of the graphs b200sac_prepare instantiated.  Both values must be in [1, 2^30]; otherwise
 * B200SAC_ERR_INVALID and nothing changes.  Get: the values last set (host mirror: does not synchronise). */
int b200sac_set_update_intervals(b200sac_t* h, int32_t replica, int32_t actor_every, int32_t target_every, void* stream);
int b200sac_get_update_intervals(b200sac_t* h, int32_t replica, int32_t* actor_every, int32_t* target_every);

/* Gradient-norm clipping, per replica and optimizer (handles created with cfg.grad_clip = 1; others: B200SAC_ERR_STATE).
 * torch.nn.utils.clip_grad_norm_(params, max_norm) right before each optimizer's step(), for the critic (counter slot 0: q1,
 * q2 and, with CARE, the critic state encoder), the actor (slot 1) and the CARE(O) context encoder (slot 4); the temperature
 * log_alpha is not clipped.  Per step and optimizer, with g = the gradient Adam reads (what b200sac_export(GRADS) returns;
 * pad columns and gaps are zero):
 *   norm = sqrt(sum g_i^2), accumulated in fp64 over the whole slice in a fixed order (bit-reproducible, independent of the
 *          replica count, no floating-point atomics);
 *   coef = (float) min(1, max_norm / (norm + 1e-6)), in fp64 and rounded once (a NaN quotient gives 1);
 *   Adam runs on g * coef (one fp32 multiply: m and v see the clipped gradient, as with torch); GRADS keeps g.
 * A critic-only step (b200sac_set_update_intervals) leaves the actor untouched and reports its norm as NaN.
 * Set: enqueued on `stream` like b200sac_set_hparams (applies to the steps enqueued after it, including launches of graphs
 * already instantiated).  Every value must be > 0; +inf = no clipping (the norms are still reported); NaN, a value <= 0 or
 * a bad replica give B200SAC_ERR_INVALID and nothing changes.  The thresholds are not copied by b200sac_copy_replica and not
 * part of a checkpoint.  Get: the values last set (host mirror: does not synchronise). */
int b200sac_set_grad_clip(b200sac_t* h, int32_t replica, double critic, double actor, double ctx, void* stream);
int b200sac_get_grad_clip(b200sac_t* h, int32_t replica, double* critic, double* actor, double* ctx);

/* Critic dropout rate p of one replica ("Dropout Q-functions" above).  Set: stream-ordered like b200sac_set_grad_clip --
 * steps enqueued after the call (launches of graphs b200sac_prepare instantiated included; no graph is rebuilt) use the
 * new rate, steps enqueued before it do not.  p in [0, 1); NaN, p < 0, p >= 1 or a bad replica give B200SAC_ERR_INVALID
 * and change nothing.  A handle created without critic_dropout gives B200SAC_ERR_STATE.  Get reads the host mirror of
 * the last accepted value (no synchronisation). */
int b200sac_set_critic_dropout(b200sac_t* h, int32_t replica, double p, void* stream);
int b200sac_get_critic_dropout(b200sac_t* h, int32_t replica, double* p);
/* Target subset size m and actor reduction of one replica ("Critic ensembles" above): actor_mean = 1 takes the mean of the
 * E critics, 0 their minimum.  Set: stream-ordered like b200sac_set_critic_dropout (prepared graphs read the new values
 * without a rebuild; steps enqueued before the call do not).  m outside [1, E] or actor_mean outside {0, 1} give
 * B200SAC_ERR_INVALID and change nothing; a handle created without critic_ensemble gives B200SAC_ERR_STATE.  Get reads the
 * host mirror (no synchronisation).  Not copied by b200sac_copy_replica. */
int b200sac_set_ensemble(b200sac_t* h, int32_t replica, int32_t m, int32_t actor_mean, void* stream);
int b200sac_get_ensemble(b200sac_t* h, int32_t replica, int32_t* m, int32_t* actor_mean);
/* Pre-clip gradient norms of the most recent `n_last` steps (<= 1024 kept, slots aligned with b200sac_read_losses):
 * out[n_last][replicas][3] = {critic, actor, context encoder}; NaN where that optimizer did not step (the actor on a
 * critic-only step, the context encoder outside CARE(O)).  Synchronises the stream. */
int b200sac_read_grad_norms(b200sac_t* h, int32_t n_last, float* out_host, void* stream);

/* PCGrad gradient surgery, per replica and optimizer (handles created with cfg.pcgrad = 1; others: B200SAC_ERR_STATE).
 * T = num_tasks, P = batch / T; row i of a step's minibatch belongs to task t(i) = i / P.  On a pcgrad handle
 * b200sac_step_sampled, b200sac_update and b200sac_replay_sample draw P rows per task in this order, on the device and the
 * pinned-host ring alike (the pinned-host ring skips its shuffle of the rows; the losses are row sums, so the order does
 * not change what a step computes).  For each optimizer o (the critic: q1, q2 and, on CARE handles, the critic state
 * encoder cse together, counter slot 0; the actor: its MLP, slot 1 -- the actor's state encoder is the tied copy of cse
 * and has no optimizer), with l_i = row i's term of o's loss exactly as the step defines it (the 1/B mean,
 * weighted_loss's extra 1/B, importance weights and the per-task temperature included):
 *   g_t  = the gradient of L_{o,t} = sum over the rows i of task t of l_i, so sum_t g_t is the ordinary step gradient.  The
 *          published implementations use per-task means, T times this: the projections do not depend on the scale, Adam
 *          only through its eps;
 *   G_jk = sum_e g_j[e] g_k[e] over the optimizer's slice, in fp64 in a fixed order (bit-reproducible, independent of the
 *          replica count, no floating-point atomics);
 *   for every task i: a permutation pi_i of all T tasks (i included), Fisher-Yates from Philox keyed by (handle seed,
 *          replica, step index, optimizer, i); c = 0 (fp64); for each j in pi_i: dot = G_ij - sum_k c_k G_kj (k ascending),
 *          and if dot < 0, c_j += dot / G_jj.  This is "if g_i^PC . g_j < 0: g_i^PC -= (g_i^PC . g_j) / |g_j|^2 g_j" with
 *          g_i^PC = g_i - sum_k c_k g_k; a zero or NaN g_j never projects (dot is 0 or NaN);
 *   w_k  = (float)(1 - sum_i c^(i)_k), the sum in fp64 over i ascending;
 *   Adam runs on w_0 g_0 + w_1 g_1 + ... + w_{T-1} g_{T-1}: each product rounded to fp32, added in index order, no FMA.
 *          The Adam math and the Polyak update fused after it are unchanged.
 * The temperature keeps its own per-task Adam and takes no part; so does the CARE(O) context encoder (slot 4), whose Adam
 * reads the plain sum of its T slices in index order (trained by the critic loss, it has slices like every optimizer).
 * Rows out of task order (b200sac_step only, counted in task_mismatch): the weight-gradient GEMM and head parts of slice t
 * come from the rows i with i / P = t, the CARE trunk and context-net parts (per-task table rows) from the rows whose
 * one-hot task is t; the sum over the slices is the ordinary gradient either way.  A critic-only step leaves the actor untouched and records
 * NaN actor weights.  b200sac_export(GRADS) still returns the slices summed in index order: the unprojected gradient.
 * Set: enqueued on `stream` like b200sac_set_hparams (applies to the steps enqueued after it, including launches of graphs
 * already instantiated).  Each switch is 0 or 1, both 1 at create; off means w = 1 (Adam reads the plain slice sum) while
 * G is still computed and reported.  The switches are not copied by b200sac_copy_replica and not part of a checkpoint.
 * Get: the values last set (host mirror: does not synchronise). */
int b200sac_set_pcgrad(b200sac_t* h, int32_t replica, int32_t critic_on, int32_t actor_on, void* stream);
int b200sac_get_pcgrad(b200sac_t* h, int32_t replica, int32_t* critic_on, int32_t* actor_on);
/* The last step's record of one replica, for both optimizers (index 0 critic, 1 actor); any output may be NULL:
 * gram [2][T][T] (fp64), w [2][T], perm [2][T][T] (row i = pi_i), mask [2][T] (bit j of mask[o][i] set iff task i was
 * projected onto task j), task_mismatch = the rows of the step whose one-hot task (its first maximum) was not t(i).
 * Before the first step: gram NaN, w 1, perm and mask 0, task_mismatch 0.  After a critic-only step the actor's entries
 * hold gram NaN, w NaN and mask 0, and its perm keeps the permutations of the last actor step.  Synchronises the stream. */
int b200sac_read_pcgrad(b200sac_t* h, int32_t replica, double* gram, float* w, int32_t* perm, uint64_t* mask,
                        int32_t* task_mismatch, void* stream);
/* Gradient slice of task `task` (rows t(i) = task) of one replica, the whole trainable arena (n_floats = trainable floats;
 * on CARE handles the critic state encoder and the CARE(O) context encoder included) into host or device memory.
 * Synchronises the stream. */
int b200sac_export_task_grad(b200sac_t* h, int32_t replica, int32_t task, float* buf, int64_t n_floats, void* stream);

/* CAGrad, conflict-averse gradient descent (Liu et al., NeurIPS 2021), on the same handles (cfg.pcgrad = 1; others:
 * B200SAC_ERR_STATE) over the same slices g_t and Gram matrix G.  Each replica and optimizer (critic = counter slot 0,
 * actor = slot 1) has a coefficient c, 0 at create.  c = 0: CAGrad is off and the PCGrad switch decides, as above.
 * c > 0: the optimizer's Adam reads the CAGrad combination whatever its PCGrad switch says; the permutations are still
 * drawn and G still computed and reported, the projection mask is 0 and b200sac_read_pcgrad's w holds the CAGrad weights.
 * Per step, in fp64, on one warp, every sum over tasks in one fixed shuffle tree (pcgrad_kernels.cuh has the exact order
 * of operations; p, A p, p.a and p.h are evaluated there through the unnormalised softmax numerators):
 *   s  = (1/T) sum_t sqrt(G_tt); if s is 0 or not finite, or any G entry is not finite: w = 1 (plain sum), "degenerate"
 *   A  = G / s^2 (the solve does not depend on the loss scale: the 1/B mean, weighted_loss's 1/B, T)
 *   a_j = (1/T) sum_k A_jk;  abar = (1/T) sum_j a_j;  ce = c sqrt(abar + 1e-4)
 *   x = 0, m = 0 (length T);  lr = 5c;  mu = 0.5;  best = +inf;  for it = 0 .. 20:
 *     p = softmax(x) (max subtracted);  u = A p;  q = p.u;  r = sqrt(q + 1e-4);  F = p.a + ce r
 *     if F < best: best = F, xbest = x, ibest = it
 *     if it < 20: h = a + ce u / r;  d_j = p_j (h_j - p.h);  m = (it == 0 ? d : mu m + d);  x = x - lr m
 *   p* = softmax(xbest);  lambda = ce / (sqrt(p*' A p* + 1e-4) + 1e-4);  w_t = (float)((1 + T lambda p*_t) / (1 + c^2))
 *   Adam runs on sum_t fp32(w_t g_t) exactly as with PCGrad.
 * This is CAGrad's update (g_0 + lambda g_w) / (1 + c^2) with g_0 the mean of the per-task mean gradients T g_t.  Its dual,
 * min over the simplex of p' A b + ce sqrt(p' A p) (b uniform), is solved at a fixed cost as the authors' Metaworld code
 * does, as far as that code is recalled here (softmax weights, 20 SGD steps with momentum 0.5, the best iterate); this
 * definition, not that code, is the contract.  One deliberate difference: s has no epsilon, so the weights do not depend
 * on the loss's absolute scale.
 * Set: enqueued on `stream` like b200sac_set_hparams (applies to the steps enqueued after it, including launches of graphs
 * already instantiated).  A negative, NaN or infinite c gives B200SAC_ERR_INVALID and nothing changes.  Not copied by
 * b200sac_copy_replica and not part of a checkpoint.  Get: the values last set (host mirror: does not synchronise).
 * The launch count of a step does not change. */
int b200sac_set_cagrad(b200sac_t* h, int32_t replica, double c_critic, double c_actor, void* stream);
int b200sac_get_cagrad(b200sac_t* h, int32_t replica, double* c_critic, double* c_actor);
/* The last step's CAGrad record of one replica, index 0 critic and 1 actor; any output may be NULL: p [2][T] (p*),
 * lambda [2], best [2] (best F), first [2] (F at iteration 0: uniform weights), scale [2] (s), ibest [2] (the iteration
 * of the best F; -1 = CAGrad did not run for that optimizer on the last step, -2 = degenerate G).  Where ibest = -1 every
 * fp64 entry is NaN; where it is -2, p, lambda, best and first are NaN and scale holds s.  Before the first step and for
 * the actor of a critic-only step: ibest -1.  Synchronises the stream. */
int b200sac_read_cagrad(b200sac_t* h, int32_t replica, double* p, double* lambda, double* best, double* first,
                        double* scale, int32_t* ibest, void* stream);
/* The same solve run stand-alone by one warp of the current device on a caller-given HOST G [T][T] (1 <= T <= 64,
 * symmetric) with c > 0 (finite), outputs to HOST memory (w [T]; p [T] and the scalars nullable).  Enqueued on the legacy
 * default stream, which it synchronises. */
int b200sac_cagrad_solve_test(int32_t T, const double* G, double c, float* w, double* p, double* lambda, double* best,
                              double* first, double* scale, int32_t* ibest);

/* One gradient step from caller-provided DEVICE minibatches, each
 * [replicas][batch][width] fp32: s,s2 width obs(=state_dim+num_tasks), a width act, r,d width 1.
 * eps_next / eps_cur: [replicas][batch][act] standard-normal noise for the two
 * rsample() calls (next-state actor first), or NULL to draw in-kernel (Philox).
 * Losses land in an internal device ring; fetch with b200sac_read_losses.
 * Every step entry point (b200sac_step, _step_host, _step_sampled, _update) follows each replica's update intervals
 * (b200sac_set_update_intervals): a critic-only step updates the critics only. */
/* pcgrad handles: row i of every replica's minibatch must belong to task i / (batch / num_tasks); b200sac_read_pcgrad
 * reports how many rows of the last step did not. */
int b200sac_step(b200sac_t* h, const float* s, const float* a, const float* r, const float* s2,
                 const float* d, const float* eps_next, const float* eps_cur, void* stream);

/* Same, from HOST buffers (any host memory; staged through the handle's pinned
 * double buffer with cudaMemcpyAsync on a side stream).  out_losses (host,
 * [replicas][4] = critic, actor, alpha-loss, entropy) may be NULL; if given the call
 * synchronises and fills it -- this is the reference's `update()` contract. */
/* pcgrad handles: a minibatch with a row i whose one-hot task is not i / (batch / num_tasks) gives B200SAC_ERR_INVALID and
 * enqueues nothing. */
int b200sac_step_host(b200sac_t* h, const float* s, const float* a, const float* r, const float* s2,
                      const float* d, const float* eps_next, const float* eps_cur, float* out_losses,
                      void* stream);

/* n_steps gradient steps, each sampling its own minibatch from the replay ring
 * (uniform without replacement; per-task B/T when num_tasks > 0) with in-kernel noise.
 * Device-resident ring: everything is enqueued asynchronously (one CUDA graph per step).
 * Pinned-host ring: indices drawn on the host, rows gathered into pinned staging and
 * copied on a side stream, overlapped with the previous step. */
int b200sac_step_sampled(b200sac_t* h, b200sac_replay_t* rb, int32_t n_steps, void* stream);

/* Capture and instantiate every CUDA graph b200sac_step_sampled / b200sac_update can launch for this ring (device ring:
 * the 8-, 4-, 2- and 1-step graphs a run is cut into; host ring: the staged one-step graph of both staging slots) without
 * running a step, so that no later call pays graph construction (milliseconds).  Synchronises the stream. */
int b200sac_prepare(b200sac_t* h, b200sac_replay_t* rb, void* stream);

/* Learner.update() (learner.py:246-264) in one call: b200sac_step_sampled(h, rb, 1) followed by the losses of that
 * step, out[replicas][4] = {critic, actor, alpha loss, entropy}.  Synchronises the stream. */
int b200sac_update(b200sac_t* h, b200sac_replay_t* rb, float* losses_host, void* stream);

/* Losses of the most recent `n_last` steps (<= 1024 kept): out[n_last][replicas][4].
 * On a replica's critic-only step (b200sac_set_update_intervals) the actor loss, alpha loss and entropy entries are NaN
 * (the same holds for b200sac_step_host and b200sac_update).  Synchronises the stream. */
int b200sac_read_losses(b200sac_t* h, int32_t n_last, float* out_host, void* stream);

/* Polyak update of the target critics outside a step (Learner.soft_update; tau = 1 is
 * the hard copy Learner.run() does before training, learner.py:287-288). */
int b200sac_soft_update(b200sac_t* h, double tau, void* stream);
/* The same for one critic pair only: critic = 1 updates q1_target from q1, critic = 2 q2_target from q2, with `tau`
 * (Learner.soft_update(local_critic_k, target_critic_k, tau), LunarLander_Distributed_SAC/src/learner.py:126-137,236-237).
 * Every other target, the CARE target state encoder included, is left as it is. */
int b200sac_soft_update_critic(b200sac_t* h, int32_t critic, double tau, void* stream);

/* Batched policy inference for n <= 2*batch observation rows obs[n][obs_dim] (obs_dim = state_dim + num_tasks), host or
 * device memory: actions[n][act_dim] = k * tanh(mu + std * eps) -- Actor.get_action
 * (LunarLander_Distributed_SAC/src/model.py:67-82, MT10_Distributed_MTSAC/src/model.py:58-73) vectorised over environments.
 * CARE handles (n <= batch): the rows are first encoded like the player does it, z = context_encoder(mtobs) then the
 * actor's state encoder -- the hard copy of the critic's -- (MT10_Distributed_CARE/src/player.py:199-209, model.py:90-114).
 * eps (nullable, [n][act_dim]) injects the noise; eps == NULL: stochastic = 1 draws fresh Philox noise; stochastic = 0
 * returns the deterministic action k * tanh(mu) of the VSAC / MTSAC / CARE actors (MT1_Distributed_VSAC/src/model.py:63,80);
 * stochastic = -1 returns k * mu, no squashing, which is what the LunarLander actor's get_action(stochastic=False) does
 * (LunarLander_Distributed_SAC/src/model.py:67-82).  Synchronises the stream. */
int b200sac_act(b200sac_t* h, int32_t replica, int32_t n, const float* obs, const float* eps, int32_t stochastic,
                float* actions_out, void* stream);

/* Critic inference: Q1 and Q2 of replica `replica` on n >= 1 rows obs[n][state_dim + num_tasks] and act[n][act_dim] (host
 * or device memory).  which = 0: q1 and q2; which = 1: q1_target and q2_target.  q_out[2][n] (host or device): row i of
 * q1 at q_out[i], row i of q2 at q_out[n + i] -- Critic.forward (LunarLander_Distributed_SAC/src/model.py) vectorised over
 * rows, e.g. for Q against Monte-Carlo returns (overestimation bias) or for priorities of fresh rows.
 *   Engine: b200sac_act's per-layer fp32 FFMA engine, whatever the handle's plan or precision.  critic_ln handles apply
 *     the LayerNorm forward with the numerics of "Layer-normalized critics" (the step's own row routine).  Eval mode, as
 *     torch's .eval(): no dropout, whatever the replica's critic_dropout rate, so a rate of 0.5 gives the values of 0.
 *   Chunk independence: row i's values depend only on the parameters and row i -- bit-identical whatever n is, wherever
 *     the row sits in the call and whatever the handle's replica count.
 *   Scratch: the rows are evaluated b200sac_critic_values_chunk rows at a time in an evaluation scratch of the handle's
 *     own (at most 64 MiB, allocated by the first call of this function or of b200sac_replay_refresh_priorities; a handle
 *     that calls neither pays nothing).  The step's buffers are not touched: the next step is bit-identical whether or
 *     not this call ran in between.
 *   Stream order and synchronisation as b200sac_act: it sees every reset, recycle and step enqueued before it.
 * A bad replica, n < 1, a NULL pointer or which outside {0, 1} give B200SAC_ERR_INVALID; a CARE handle gives
 * B200SAC_ERR_STATE (no per-task encoding of arbitrary rows yet). */
int b200sac_critic_values(b200sac_t* h, int32_t replica, int64_t n, const float* obs, const float* act, int32_t which,
                          float* q_out, void* stream);
/* Rows per chunk of the evaluation scratch (pure host function): the most rows of this handle's shapes that fit 64 MiB, a
 * multiple of 32, at most 65536. */
int b200sac_critic_values_chunk(b200sac_t* h, int64_t* rows);

/* Blob publication: the byte string Learner.run() stores under the Redis key 'parameters' after every update
 * (LunarLander_Distributed_SAC/src/learner.py:298-299: _pickle.dumps({'actor': state_dict}); read back by
 * Player.pull_parameters, player.py:75-85) assembled on the device.  blob_template: `image` = the constant bytes of the
 * string (any values in the payload positions); payload float j (j < n_floats) is the 4 bytes at dst_byte[j] and holds
 * element src_index[j] of replica `replica`'s parameter arena (b200sac_layout offsets; pitch padding / transposed views
 * are expressed through the index map).  blob_begin enqueues, in stream order, the gather of all payload floats into a
 * device copy of the image and starts ONE D2H copy of it on a private stream; it does not block and later steps overlap
 * the copy.  blob_wait blocks until the OLDEST uncollected blob has landed in pinned memory and returns it (valid until
 * the second blob_begin after the one that produced it).  Two image slots: blob_begin may be called again before the
 * previous blob is collected; a third begin without a wait supersedes the oldest. */
int b200sac_blob_template(b200sac_t* h, int32_t replica, const uint8_t* image, int64_t image_bytes, int64_t n_floats,
                          const int32_t* src_index, const int32_t* dst_byte);
int b200sac_blob_begin(b200sac_t* h, void* stream);
int b200sac_blob_wait(b200sac_t* h, const uint8_t** host_ptr, int64_t* n_bytes);

/* Debug / parity access to per-step intermediates of replica `replica`:
 * name in {"y","q1","q2","a_next","logp_next","a_cur","logp_cur","qmin","d_action","d_head","r","d"}, "dq_pi" ([2][B]: d(actor loss)/dQ1, dQ2 -- which twin
 * min(Q1,Q2) routed the gradient to), "q_pi" ([2][B]: Q1, Q2 at (s, a~)), "psave" ([2B][act][8]:
 * what the policy head saved per (row, action) -- std, u-mu, tanh(u), action, Jacobian term, the NOISE it used, clamp mask,
 * log-prob term), "head" ([2B][2*act]: the policy head's output as the head computed it, mu | log-std before the clamp;
 * after b200sac_act its first n rows), or a hidden (after b200sac_redo: its forward's rows, see there)
 * activation whose sign pattern is the ReLU mask the step used: "hA.<l>" [2B][H] (rows [s';s]), "hQ.<l>" / "hP.<l>" /
 * "hT.<l>" [2][B][H] (critic-update pass / actor pass / target pass; the layer-chained plan does not keep hT); with
 * cfg.critic_ln, "zQ.<l>" / "zP.<l>" / "zT.<l>" [2][B][H], the same passes' pre-normalization activations W x + b (with
 * cfg.critic_dropout: z', after the dropout); with cfg.critic_dropout, "mQ.<l>" / "mP.<l>" / "mT.<l>" [2][B][H], the same
 * passes' keep masks as 0.0 / 1.0;
 * "mixH.<inst>.<l>" [K][rows][pitch4(H)] (CARE mixture encoders).  After a step from a prioritized ring: "isw" [B] (the
 * importance weights of its critic loss), "prio" [B] (the leaf values p it wrote) and "idx" [B] (its ring indices, int32
 * bit patterns).  After a step from a linked ring (n-step returns): "disc" [B] (the per-row discount of its TD target),
 * "nstep_m" [B] (hops folded, int32 bit patterns), "idx" as above, and "r" / "d" hold the folded values.  With
 * cfg.grad_clip: "clip" [3] (the clip coefficients of the last step: critic, actor, context encoder; NaN for an actor that
 * did not step; the context encoder's entry is meaningful for CARE(O) only). */
int b200sac_debug_read(b200sac_t* h, const char* name, int32_t replica, float* out_host, int64_t cap_floats,
                       int64_t* n_floats, void* stream);

/* Eager (no graph) run of `iters` sampled steps from a DEVICE ring with a CUDA event between all
 * launches: out_ms[i] = mean device time of launch i of the step (0 = sampling + ingest).
 * names (nullable): ';'-separated kernel labels.  Measurement helper for bench.py's roofline. */
int b200sac_profile_step(b200sac_t* h, b200sac_replay_t* rb, int32_t iters, float* out_ms, int32_t cap,
                         int32_t* n_out, char* names, int32_t names_cap, void* stream);

/* In-graph timeline: `iters` sampled steps from a DEVICE ring as normal graph launches, with every
 * kernel stamping %globaltimer at entry; out_us[i] = mean start-to-start time of launch i
 * (0 = index sampling, 1 = ingest, then the step's launches in order, as b200sac_profile_step names them). */
int b200sac_graph_timeline(b200sac_t* h, b200sac_replay_t* rb, int32_t iters, float* out_us, int32_t cap,
                           int32_t* n_out, void* stream);

/* Stand-alone run of the wgmma 3xTF32 GEMM kernel on DEVICE arrays (parity tests of the tensor-core
 * path): mode 0 FWD C[M][N] = act(A[M][K] B[N][K]^T + bias), 1 DGRAD C[M][N] = (A[M][K] B[K][N]) * [mask > 0],
 * 2 WGRAD C[M][N] = A[K][M]^T B[K][N], C2[M] = column sums of A.  Synchronises. */
int b200sac_tc_gemm_test(int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda, const float* B,
                         int32_t ldb, const float* bias, const float* mask, int32_t ldmask, float* C, int32_t ldc,
                         float* C2, int32_t relu, void* stream);

/* The same for any GEMM engine of the step: engine 0 = 32x32-tile fp32 FFMA, 1 = wgmma 3xTF32,
 * 2 = thin backward kernel (modes 1/2 with N <= 16: the input-layer weight / input gradients). */
int b200sac_gemm_test(int32_t engine, int32_t mode, int32_t M, int32_t N, int32_t K, const float* A, int32_t lda,
                      const float* B, int32_t ldb, const float* bias, const float* mask, int32_t ldmask, float* C,
                      int32_t ldc, float* C2, int32_t relu, void* stream);

/* Number of kernels one step launches (for bench.py's gpu_launches accounting). */
int b200sac_launches_per_step(b200sac_t* h, int32_t* n);

/* ---- replay ring ---------------------------------------------------------------- */
/* where: 0 = device-resident ring (HBM), 1 = pinned host DRAM ring.
 * capacity = transitions per replica (per task: capacity / num_tasks when num_tasks > 0). */
int b200sac_replay_create(b200sac_t* h, int64_t capacity, int32_t where, uint64_t seed, b200sac_replay_t** out);
int b200sac_replay_destroy(b200sac_replay_t* rb);
/* Append n transitions (HOST arrays, fp32, same widths as b200sac_step) to one replica's ring.
 * Thread-safe against one concurrent sampler. */
int b200sac_replay_push(b200sac_replay_t* rb, int32_t replica, int64_t n, const float* s, const float* a,
                        const float* r, const float* s2, const float* d);
/* Fill every replica's ring with `n` synthetic transitions generated on the device
 * (s,s'~N(0,1), a~U(-1,1), r~N(0,1), d~Bernoulli(0.01), task = i mod T). Benchmark helper.
 * Like push, it waits for the gathers of the steps already enqueued before it rewrites the ring, and is thread-safe
 * against one concurrent sampler.  Synchronises the stream. */
int b200sac_replay_fill_synthetic(b200sac_replay_t* rb, int64_t n, uint64_t seed, void* stream);
/* min over tasks of the per-task fill, like ReplayBuffer.__len__ in the MT variant. */
int b200sac_replay_size(b200sac_replay_t* rb, int32_t replica, int64_t* n);
/* Draw one minibatch the way step_sampled would and return it in HOST arrays
 * (reference-shaped ReplayBuffer.sample()); idx_out (nullable) gets the ring indices. */
int b200sac_replay_sample(b200sac_replay_t* rb, int32_t replica, float* s, float* a, float* r, float* s2,
                          float* d, int64_t* idx_out);

/* ---- prioritized replay (device ring only) ------------------------------------------
 * Each (replica, task) sub-ring has a sum-tree over its slots.  Leaf i holds p_i = (prio_i + eps)^alpha (fp32, the power in
 * fp64 rounded once); internal nodes are recomputed sums of their children; empty slots hold 0 and are never drawn.
 * A step draws, per task, B/T rows (B when num_tasks = 0) stratified with replacement: slot j draws u = (j + U(0,1)) S / (B/T)
 * (S = the task's root sum) and descends; the Philox key is (seed, replica, step counter, slot).  Importance weights
 * w_i = (N_t p_i / S_t)^-beta (N_t = fill of the sub-ring), divided by their maximum over the minibatch (fp64, rounded once),
 * multiply the per-row critic gradient and loss term: dQk = (2c (Qk - y)) w, lq = (e1^2 + e2^2) w.  After the critic loss, in
 * the step's graph, the sampled leaves get prio_i = (|y - Q1| + |y - Q2|) / 2 (the highest batch slot wins a duplicated
 * index) and a running max p per (replica, task), initially 1, is raised; rows written by push / fill_synthetic get it.
 * b200sac_step_sampled, b200sac_update and b200sac_prepare accept a prioritized ring; b200sac_replay_sample does not.
 * alpha >= 0, 0 <= beta <= 1, eps > 0, and (0 + eps)^alpha > 0 and finite in fp32, else B200SAC_ERR_INVALID: a filled
 * slot's leaf is then always > 0, so every sub-ring the sampler visits has a root > 0 and every draw lands on a filled slot.
 * With alpha > 1 a large priority can still give an inf leaf: set_priorities refuses one; in the step's own update it can
 * only come from a TD error near 1e38^(1/alpha), i.e. a critic that has already diverged, and the weights are then NaN. */
int b200sac_replay_create_prioritized(b200sac_t* h, int64_t capacity, uint64_t seed, double alpha, double beta, double eps,
                                      b200sac_replay_t** out);
/* beta of one replica, in stream order on `stream`: steps enqueued afterwards use it (no graph is rebuilt). */
int b200sac_replay_set_beta(b200sac_replay_t* rb, int32_t replica, double beta, void* stream);
/* Raw priorities (|delta|-like, >= 0; the exponent is applied inside) of n filled ring slots, e.g. actor-computed initial
 * priorities; a later entry wins a duplicated index.  Raises max p.  Synchronous; ordered after every enqueued step. */
int b200sac_replay_set_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, const float* prio);
/* Leaf values p of n ring slots; an index -1 - t reads task t's root sum instead.  Synchronous, like set_priorities. */
int b200sac_replay_get_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, float* p_out);
/* The whole sum-tree of one (replica, task) sub-ring, n = 2P floats in heap order (out[1] = root, leaf i = out[P + i],
 * out[0] unused), P = the power of two >= cap_per_task.  Synchronous, like set_priorities. */
int b200sac_replay_get_tree(b200sac_replay_t* rb, int32_t replica, int32_t task, int64_t n, float* out);
/* Reference-shaped PER sample(): one draw of the device sampler with its own draw counter (0, 1, ... per replica) in place
 * of the step counter; rows, ring indices (nullable) and importance weights (nullable) to HOST arrays. */
int b200sac_replay_sample_prioritized(b200sac_replay_t* rb, int32_t replica, float* s, float* a, float* r, float* s2,
                                      float* d, int64_t* idx_out, float* w_out);
/* Priority refresh: recompute the priorities of n filled slots idx[n] of replica `replica`'s sub-rings (ring indices as
 * b200sac_replay_set_priorities takes them; idx == NULL with n = 0: every filled slot of every task) with the replica's
 * current networks -- after b200sac_reset or b200sac_redo every leaf still holds the TD error of the discarded network
 * until its slot is sampled again.  Per slot i with task t:
 *   1. Row: what the step would train on.  Linked ring: the n-step fold with the replica's current horizon and gamma
 *      ("n-step returns"), (s_i, a_i, R, s'_j, d_j, g); otherwise (s, a, r, s', d) with g = gamma.
 *   2. Next action: a' and log pi' from the actor on s'_j through the step's policy head, with noise eps per action k:
 *      stochastic = 0: eps = 0 (the mean action); stochastic = 1: eps = z0 of box_muller(w0, w1), (w0, w1) the first two
 *      words of Philox4x32-10 with key = seed ^ (0xC2B2AE3D27D4EB4F * (replica + 1)) (mod 2^64; a multiplier no other draw
 *      of the library uses) and counter (i & 0xFFFFFFFF, i >> 32, t, 0x7E00 + k).  The noise depends on the slot only, not
 *      on n, the chunking or the order of idx.
 *   3. Critic values: Qt1, Qt2 (targets) on (s'_j, a') and Q1, Q2 (locals) on (s_i, a_i) as b200sac_critic_values computes
 *      them (eval mode).
 *   4. TD target: y = rs R + g (1 - d_j)(min(Qt1, Qt2) - alpha log pi'), alpha = (float)exp((double)log_alpha[t]), formed
 *      as the step forms it.
 *   5. Leaf: prio = (|y - Q1| + |y - Q2|) / 2 in fp64, p = (prio + eps)^alpha as the step's priority update writes it.
 *   6. Tree: every internal node of each touched (replica, task) tree is recomputed from its children; slots not refreshed
 *      keep their leaves bit for bit.  A duplicated index is harmless: every copy computes the same value.
 *   7. Max p: idx == NULL: each task's running max p becomes the largest of its refreshed leaves (rows pushed later get
 *      it); otherwise max p is only raised, as by set_priorities.  A task with no filled slots is untouched.
 * Synchronous, like set_priorities: ordered after everything enqueued on `stream` (a b200sac_reset / b200sac_redo enqueued
 * just before it included), after every enqueued step, push and set_nstep, and done under the ring's lock.  Runs through
 * the handle's evaluation scratch (b200sac_critic_values); the step's buffers and plan are untouched.
 * A ring that is not prioritized, a bad replica, n < 0, n > 0 with a NULL idx, an idx that is not a filled slot or
 * stochastic outside {0, 1} give B200SAC_ERR_INVALID; a CARE handle gives B200SAC_ERR_STATE; nothing changes then. */
int b200sac_replay_refresh_priorities(b200sac_replay_t* rb, int32_t replica, int64_t n, const int64_t* idx, uint64_t seed,
                                      int32_t stochastic, void* stream);

/* ---- n-step returns (device ring only) --------------------------------------------------
 * A linked ring records, next to its 1-step transitions, which slot follows which: link[replica][slot] (int32) is the
 * sub-ring-local slot of the transition that followed this one in its trajectory, or -1.  The n-step return is folded at
 * sample time, in the gather of the step's graph, so the horizon n and gamma stay per replica and settable between steps.
 * Fold of a sampled slot i with n = the replica's horizon and gamma = its b200sac_hparams.gamma (fp32, no fused multiply-add):
 *     j = i;  R = r_j;  g = gamma;  m = 1
 *     while d_j == 0 and m < n and link[j] >= 0:   j = link[j];  R = R + g * r_j;  g = g * gamma;  m = m + 1
 * The step trains on the row (s_i, a_i, R, s'_j, d_j) with the TD target y = rs R + g (1 - d_j)(min(Qt1, Qt2) - alpha logpi'):
 * the horizon is shorter at a terminal, a time-limit cut, a trajectory's current tail (successor not pushed yet) or an
 * overwritten successor; with m = 1 the row and the target are the unlinked ring's, bit for bit.  On a prioritized ring the
 * priorities become n-step TD errors by themselves.  The intermediate rows' actions are used uncorrected, as in Ape-X.
 * Links are made by b200sac_replay_push_traj: every row carries a stream id (one per player / environment); the library
 * keeps the tail of every (replica, stream), and row x becomes the successor of its stream's tail t iff t exists, d_t == 0,
 * cut_t == 0 and both lie in the same task sub-ring.  Overwrite rule: when a push overwrites slot j, the link that pointed
 * to j is reset to -1, and a stream whose tail was j forgets it.  Invariant, at every point in stream order:
 * link[i] = j >= 0 implies that slot j currently holds the transition that followed slot i's.
 * b200sac_step_sampled, b200sac_update and b200sac_prepare accept a linked ring (uniform or prioritized); the launch count
 * of a step does not change.  Links are not part of a checkpoint. */
/* Valid once, on an empty device ring: B200SAC_ERR_INVALID for a pinned-host ring, B200SAC_ERR_STATE for a ring that holds
 * rows or is linked already; nothing changes then.  4 bytes per slot; every replica's horizon starts at 1. */
int b200sac_replay_enable_trajectories(b200sac_replay_t* rb);
/* b200sac_replay_push (same order, bucketing by task, wrap, "only the newest rows survive", max-p leaf on a prioritized ring)
 * plus, per row, a stream id in [0, 65536) and a nullable cut flag (time-limit truncation: the episode ended but d = 0, so
 * the row bootstraps from its own s').  The link changes land with the rows, before the call returns.  Plain
 * b200sac_replay_push stays legal on a linked ring: its rows get link = -1, obey the overwrite rule and join no stream.
 * b200sac_replay_fill_synthetic on a linked ring links slot i -> i + 1 of a sub-ring unless d_i != 0 or i is the last
 * filled slot. */
int b200sac_replay_push_traj(b200sac_replay_t* rb, int32_t replica, int64_t n, const float* s, const float* a, const float* r,
                             const float* s2, const float* d, const int32_t* stream, const uint8_t* cut);
/* Forget the open tails of n streams of one replica (host bookkeeping only, no link changes): the next row of each starts a
 * new trajectory.  For callers that recycle stream ids of trajectories that ended without a terminal or cut row. */
int b200sac_replay_close_streams(b200sac_replay_t* rb, int32_t replica, int64_t n, const int32_t* stream);
/* Horizon of one replica, n in [1, 16], in stream order on `stream` like b200sac_replay_set_beta: steps enqueued afterwards
 * use it, including launches of graphs b200sac_prepare instantiated.  Get: the value last set (host mirror). */
int b200sac_replay_set_nstep(b200sac_replay_t* rb, int32_t replica, int32_t n, void* stream);
int b200sac_replay_get_nstep(b200sac_replay_t* rb, int32_t replica, int32_t* n);
/* The link table of one (replica, task) sub-ring, n = its slot count.  Synchronous. */
int b200sac_replay_get_links(b200sac_replay_t* rb, int32_t replica, int32_t task, int64_t n, int32_t* out);
/* Reference-shaped sample() of a linked ring: the device fold of n_idx caller-given filled ring slots with the replica's
 * current horizon and gamma, to HOST arrays (s, a, R, s2, d as in b200sac_replay_sample; disc[n_idx] = g; m[n_idx] = hops).
 * Synchronous; ordered after every b200sac_replay_set_nstep.  A b200sac_set_hparams still in flight on another stream is
 * not waited for. */
int b200sac_replay_fold(b200sac_replay_t* rb, int32_t replica, int64_t n_idx, const int64_t* idx, float* s, float* a, float* R,
                        float* s2, float* d, float* disc, int32_t* m);

/* ---- prior-data rings (device rings only) ----------------------------------------------
 * Symmetric sampling (RLPD, Ball et al. 2023): every minibatch takes a fixed number of its rows from a fixed prior dataset
 * (demonstrations, scripted rollouts, an earlier run's buffer) and the rest from the online ring, drawn and gathered inside
 * the step's graph.  The prior is an ordinary ring of the same handle, filled by push / fill_synthetic.
 * Split: with P = batch / num_tasks (batch when num_tasks = 0) and m = the replica's prior-row count, rows [tP, tP + m) of
 * every task block t come from task t's sub-ring of the prior and rows [tP + m, (t + 1)P) from the online ring, so the
 * minibatch keeps its task blocks (pcgrad handles see task_mismatch = 0).
 * Draw: batch slot i of replica r draws exactly as the online ring's plain draw does -- Philox4x32-10 key
 * seed + 0x9E3779B97F4A7C15 * (r + 1), counter (step, step >> 32, i, attempt), index (w0 << 32 | w1) % fill_t -- with the
 * prior's seed and per-task fill for a prior slot.  Slots are distinct within each (task block, part): the lowest slot keeps
 * a contested index and the others redraw with attempt + 1.  An online index and a prior index never compete.  So m = 0 is
 * the plain ring's minibatch and step bit for bit, and m = P is that of a plain ring with the prior's seed and rows.
 * Gather: the step trains on the drawn rows.  After a step from a ring with a prior, b200sac_debug_read "idx" [B] holds the
 * encoded indices (int32 bit patterns): online ring index k as k, prior ring index k as -1 - k.  The launch count of a step
 * is unchanged (b200sac_profile_step labels the launch "sample_mixed+ingest_mixed").
 * Readiness: a step needs the online ring ready as before and, for every replica with m > 0, every task sub-ring of the
 * prior holding >= 4 per-task batches; else B200SAC_ERR_STATE and nothing is enqueued.  b200sac_step_sampled, b200sac_update,
 * b200sac_prepare, b200sac_profile_step and b200sac_graph_timeline hold both rings' locks while they enqueue, and a push into
 * either ring waits for the steps that read it.  b200sac_replay_sample still draws from the online ring only. */
/* Make `prior` the prior ring of `rb`; prior == NULL detaches (every replica's m back to 0: rb is a plain ring again).  Both
 * must be uniform, unlinked device rings of one handle, prior != rb, else B200SAC_ERR_INVALID; rb already having a prior,
 * prior already being a ring's prior or having a prior itself give B200SAC_ERR_STATE; nothing changes then.  Waits for the
 * gathers both rings have pending and drops rb's graphs (rebuilt on next use).  b200sac_replay_destroy of either ring
 * detaches first; b200sac_replay_enable_trajectories on an attached ring gives B200SAC_ERR_STATE. */
int b200sac_replay_attach_prior(b200sac_replay_t* rb, b200sac_replay_t* prior);
/* m of one replica, in [0, P], in stream order on `stream` like b200sac_replay_set_beta: steps enqueued afterwards use it,
 * including launches of graphs b200sac_prepare instantiated (no graph is rebuilt).  m outside [0, P] or a bad replica:
 * B200SAC_ERR_INVALID; a ring without a prior: B200SAC_ERR_STATE.  Get: the value last set (host mirror; 0 by default). */
int b200sac_replay_set_prior_rows(b200sac_replay_t* rb, int32_t replica, int32_t m, void* stream);
int b200sac_replay_get_prior_rows(b200sac_replay_t* rb, int32_t replica, int32_t* m);

#ifdef __cplusplus
}
#endif
#endif /* B200SAC_H_ */
