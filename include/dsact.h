/*
 * dsact.h — C ABI of the H100-native DSAC-T update engine (libdsact.so).
 *
 * Drop-in boundary for ONE path of Jingliang-Duan/DSAC-v2: the per-step
 * critic/actor/temperature update over a replay minibatch,
 *     DSAC_V2.local_update(data, iteration)             reference dsac_v2.py:102-105
 * plus the replay minibatch gather that feeds it,
 *     ReplayBuffer.sample_batch(batch_size)             reference training/replay_buffer.py:85-90
 * called from OffSerialTrainer.step                      reference training/trainer.py:69,82.
 *
 * Conventions
 *  - plain C types only; every function returns 0 on success or a negative
 *    DSACT_E* code, and `dsact_last_error()` holds a message for the caller's thread;
 *  - the CALLER (PyTorch) owns every device allocation; the library borrows
 *    pointers handed over in `dsact_bind*` and never frees them;
 *  - all work is enqueued on the caller's CUDA stream (`cudaStream_t` passed as
 *    `void*`) and is asynchronous with respect to the host;
 *  - one handle per device and per trainer thread (not thread safe);
 *  - all tensors are fp32, row-major, contiguous unless a leading dimension is given.
 *
 * Flat parameter layout (`dsact_layout`): params = [ q1 | q2 | policy | log_alpha ],
 * targets = [ q1_target | q2_target | policy_target ]; each network is the
 * concatenation, in `state_dict` order (reference SURVEY §4 schema), of
 * weight_j [out_j, in_j] then bias_j [out_j].  grads / adam_m / adam_v mirror params.
 */
#ifndef DSACT_H
#define DSACT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSACT_ABI_VERSION 4
#define DSACT_MAX_HIDDEN 6
#define DSACT_NUM_STATS 16

enum {
  DSACT_OK = 0,
  DSACT_EINVAL = -1,   /* bad argument / unsupported configuration */
  DSACT_ECUDA = -2,    /* a CUDA runtime call failed */
  DSACT_ESTATE = -3,   /* call sequence error (e.g. step before bind) */
  DSACT_EARCH = -4     /* device is not sm_90 */
};

/* hidden activations, reference utils/common_utils.py:16-45 */
enum {
  DSACT_ACT_LINEAR = 0, DSACT_ACT_RELU = 1, DSACT_ACT_GELU = 2, DSACT_ACT_TANH = 3,
  DSACT_ACT_SIGMOID = 4, DSACT_ACT_ELU = 5, DSACT_ACT_SELU = 6
};

/* arithmetic of the dense layers */
enum {
  DSACT_GEMM_FP32 = 0,     /* fp32 FFMA, bit-comparable with the reference's fp32 path */
  DSACT_GEMM_BF16X3 = 1,   /* wgmma bf16 split-precision (hi*hi + hi*lo + lo*hi), fp32 accumulate */
  DSACT_GEMM_BF16 = 2      /* wgmma single-pass bf16, fp32 accumulate (throughput mode) */
};

/* The policy's std_type (reference networks/mlp.py:43-72) and the flat layout of the policy span it implies:
 *  DSACT_STD_SHARED    "mlp_shared":    one MLP [O, hidden_pi.., 2A] (mean | log_std);
 *  DSACT_STD_SEPARATED "mlp_separated": [ mean.* | log_std.* ], two MLPs [O, hidden_pi.., A];
 *  DSACT_STD_PARAMETER "parameter":     [ log_std row (A floats) | mean.* ], the row a learnable [1, A] parameter.
 * The last two are the layouts dsact_cnn_query_layout reports for the same networks (n_conv = 0, q_heads = 1). */
enum { DSACT_STD_SHARED = 0, DSACT_STD_SEPARATED = 1, DSACT_STD_PARAMETER = 2 };

/* What ApproxContainer.__init__ + DSAC_V2.__init__ read from kwargs
 * (reference dsac_v2.py:25-59,79-90; utils/common_utils.py:48-89). */
typedef struct dsact_config {
  int32_t abi_version;           /* = DSACT_ABI_VERSION */
  int32_t obs_dim;               /* obsv_dim */
  int32_t act_dim;               /* action_dim */
  int32_t n_hidden_q;            /* len(value_hidden_sizes) */
  int32_t n_hidden_pi;           /* len(policy_hidden_sizes) */
  int32_t hidden_q[DSACT_MAX_HIDDEN];
  int32_t hidden_pi[DSACT_MAX_HIDDEN];
  int32_t act_q;                 /* value_hidden_activation  */
  int32_t act_pi;                /* policy_hidden_activation */
  int32_t max_batch;             /* largest minibatch a step will see */
  int32_t auto_alpha;            /* dsac_v2.py:85 */
  int32_t delay_update;          /* dsac_v2.py:87 */
  int32_t gemm_mode;             /* DSACT_GEMM_* */
  int32_t use_graph;             /* replay captured CUDA graphs for repeated identical calls */
  int32_t act_dist;              /* policy_act_distribution: 0 TanhGaussDistribution, 1 GaussDistribution
                                    (utils/act_distribution_cls.py:20-79, 82-116) */
  int32_t policy_std;            /* DSACT_STD_*: the policy's std_type (networks/mlp.py:43-72); DSAC-T handles only */
  /* scalars are doubles because the reference holds them as Python floats and forms
   * 1-beta, lr/(1-beta^t) ... in double before they touch an fp32 tensor */
  double gamma, tau, tau_b;       /* dsac_v2.py:82,83,90 */
  double alpha_fixed;             /* dsac_v2.py:86 (used when auto_alpha == 0) */
  double lr_q, lr_pi, lr_alpha;   /* dsac_v2.py:54-59 */
  double min_log_std, max_log_std;/* networks/mlp.py:73-74 */
  double adam_beta1, adam_beta2, adam_eps; /* torch.optim.Adam defaults 0.9 / 0.999 / 1e-8 */
} dsact_config;

typedef struct dsact_layout {
  int64_t n_q;          /* floats in one Q network */
  int64_t n_pi;         /* floats in the policy span (see DSACT_STD_*) */
  int64_t n_params;     /* 2*n_q + n_pi + 1 (log_alpha last) */
  int64_t n_targets;    /* 2*n_q + n_pi */
  int64_t workspace_bytes; /* activation / scratch arena the caller must provide */
  int64_t state_floats; /* persistent device state (EMA, counters, accumulators, stats) */
  int64_t max_batch;
  /* workspace slots, in floats from the workspace base: the replay indices the last index-drawing gather recorded
   * (int64 [max_batch]); the noise eps1 / eps2 [max_batch, act_dim], z3 / z4 [max_batch] (device noise, or host noise a
   * caller stages there); the weight-gradient split slabs of the tensor-core modes, the last region, `slab_floats` long
   * (0 in fp32 mode and on the head-wise engine) and zeroed by dsact_bind */
  int64_t off_idx, off_eps1, off_eps2, off_z3, off_z4, off_slabs, slab_floats;
} dsact_layout;

/* Device pointers of caller-owned tensors. */
typedef struct dsact_buffers {
  float *params, *targets, *grads, *adam_m, *adam_v;
  const float *act_high, *act_low;   /* [act_dim], policy.act_high_lim / act_low_lim */
  float *state;                      /* [state_floats], zero-initialised by the caller */
  void *workspace;                   /* [workspace_bytes], 256-byte aligned */
} dsact_buffers;

/* One replay minibatch, device pointers (the dict `data`, dsac_v2.py:219-225). */
typedef struct dsact_batch {
  const float *obs, *act, *rew, *obs2, *done;
  int32_t batch;
  const float *logp;  /* behaviour log-prob; stored and gathered like the reference does, never read by the update */
} dsact_batch;

/* The normal draws that affect an update (SURVEY Appendix B): eps1/eps2 [B,A]
 * for the two rsample() calls, z3/z4 [B] for the two target __q_evaluate calls.
 * Pass NULL instead of the struct to draw them on the device (Philox4x32-10). */
typedef struct dsact_noise {
  const float *eps1, *eps2, *z3, *z4;
} dsact_noise;

typedef struct dsact_handle dsact_handle;

const char *dsact_last_error(void);
int dsact_abi_version(void);

/* sizes implied by a configuration; no device needed */
int dsact_query_layout(const dsact_config *cfg, dsact_layout *out);

/* replaces ApproxContainer/DSAC_V2 construction (dsac_v2.py:25-59,79-90) */
int dsact_create(const dsact_config *cfg, int device, dsact_handle **out);
void dsact_destroy(dsact_handle *h);
int dsact_bind(dsact_handle *h, const dsact_buffers *bufs);

/* The networks' output activations (the reference's value_output_activation / policy_output_activation: the
 * `output_activation` of every network's last layer, networks/mlp.py and networks/cnn.py), as DSACT_ACT_* codes.
 * value_act applies to every critic output (mean and raw std, before the softplus).  policy_act applies to the policy's
 * outputs: all 2A of "mlp_shared", both networks of "mlp_separated", the mean network only of "parameter" (its log_std
 * row is not activated), and every head of the CNN approximators.  Works on a handle of any create call; call it
 * between create and dsact_bind (DSACT_ESTATE after bind).  DSACT_EINVAL for an unknown code.  Default: both linear. */
int dsact_set_output_activations(dsact_handle *h, int32_t value_act, int32_t policy_act);

/* seed / counter of the device noise generator and of replay index sampling */
int dsact_seed(dsact_handle *h, uint64_t seed);

/* overwrite the carried scalars: mean_std1/2 (< 0 = "unset", dsac_v2.py:88-89),
 * Adam step counters of the critics and of policy/alpha */
int dsact_set_carry(dsact_handle *h, float mean_std1, float mean_std2,
                    int64_t adam_steps_q, int64_t adam_steps_pi, void *stream);

/* DSAC_V2.local_update (dsac_v2.py:102-105): gradients + Adam + delayed Polyak */
int dsact_step(dsact_handle *h, const dsact_batch *batch, const dsact_noise *noise,
               int64_t iteration, void *stream);

/* The same call with a HOST minibatch — what the reference's trainer hands to local_update (training/trainer.py:69,82:
 * `replay_samples` are CPU tensors): `host` holds host pointers (pinned for full PCIe rate; pageable works).  The five
 * arrays are copied into one of two internal device staging sets on a private copy stream (the copy of call k+1 runs
 * under the kernels of call k), then dsact_step runs on that set.  dsact_stage_host / dsact_stage_release are the two
 * halves for callers that want another entry point (dsact_dp_step, dsact_compute_grads ...) on a host minibatch:
 * stage -> device pointers in `dev` (valid until the second next stage call) -> any step call(s) on `dev` ->
 * release (marks the set reusable once the work enqueued on `stream` so far has finished). */
int dsact_step_host(dsact_handle *h, const dsact_batch *host, const dsact_noise *noise, int64_t iteration, void *stream);
int dsact_stage_host(dsact_handle *h, const dsact_batch *host, dsact_batch *dev, void *stream);
int dsact_stage_release(dsact_handle *h, void *stream);

/* split form = get_remote_update_info / remote_update (dsac_v2.py:107-138).
 * phase1: all forwards up to the per-critic sum of std over the local shard
 *         (state[DSACT_STATE_STDSUM..+1]); phase2: EMA, losses, all backward passes
 *         with loss means taken over `global_batch` rows.  A data-parallel caller
 *         all-reduces the two std sums between the phases and `grads` after phase2. */
int dsact_grad_phase1(dsact_handle *h, const dsact_batch *batch, const dsact_noise *noise, void *stream);
int dsact_grad_phase2(dsact_handle *h, int64_t global_batch, void *stream);
int dsact_compute_grads(dsact_handle *h, const dsact_batch *batch, const dsact_noise *noise, void *stream);
/* DSAC_V2.__update (dsac_v2.py:320-347) on whatever is in `grads` */
int dsact_apply(dsact_handle *h, int64_t iteration, void *stream);

/* tb_info (dsac_v2.py:188-202) of the last step, in this order:
 *  0 q1 mean, 1 q2 mean, 2 std1 mean, 3 std2 mean, 4 min std1, 5 min std2,
 *  6 actor loss, 7 critic loss, 8 mean tanh(policy mean), 9 mean policy std,
 * 10 entropy, 11 alpha (pre-update), 12 mean_std1, 13 mean_std2,
 * 14 data-parallel exchange status (0 = ok, 1 + r = rank r never arrived, see dsact_dp_step), 15 reserved.
 * Finalises the accumulators over `global_batch` rows and copies 16 floats to `host_out`
 * (pinned or pageable) asynchronously on `stream`. */
int dsact_read_stats(dsact_handle *h, int64_t global_batch, float *host_out, void *stream);

/* ---- device replay ring buffer (ReplayBuffer, training/replay_buffer.py:15-90) ---- */
typedef struct dsact_replay {
  float *obs, *obs2, *act, *rew, *done, *logp; /* [capacity, O], [capacity, O], [capacity, A], 3x [capacity] */
  int64_t capacity;
} dsact_replay;

int dsact_replay_bind(dsact_handle *h, const dsact_replay *rb);
/* store(): copy n transitions (rows of the staging arrays; host-pinned, pageable or device)
 * into rows (ptr + i) % capacity */
int dsact_replay_add(dsact_handle *h, const float *obs, const float *obs2, const float *act,
                     const float *rew, const float *done, const float *logp,
                     int64_t n, int64_t ptr, void *stream);
/* ---- frame replay ring: each observation frame stored once ----
 * The flat ring above stores obs and obs2 of every row as separate copies, although obs2 of row t is usually obs of row
 * t + 1 (and, with stacked frames, obs2 is obs shifted by one frame).  This ring stores frames instead: an observation
 * of O = obs_elems floats is K = frames_per_obs frames of F = O / K floats, frame k being floats [k*F, (k+1)*F) (for an
 * NCHW image and K = C, one channel).  Row r's obs is frames[obs_frames[r*K + k]], k = 0..K-1; obs2 likewise through
 * obs2_frames.  Which frames rows share is the caller's decision; every gather reads the ring that is bound, and yields
 * bit for bit the rows a flat ring holding the same observations would.
 * dsact_replay_bind_frames: DSACT_EINVAL unless frames_per_obs is in [1, 64] and divides obs_elems, frame_capacity is in
 * [frames_per_obs, 2^31 - 1], capacity >= 1 and no pointer is null.  Binding either ring kind replaces the other. */
typedef struct dsact_frame_replay {
  float *frames;                      /* [frame_capacity, obs_elems / frames_per_obs] */
  int32_t *obs_frames, *obs2_frames;  /* [capacity, frames_per_obs]: frame slots of each row */
  float *act, *rew, *done, *logp;     /* as in dsact_replay */
  int64_t capacity, frame_capacity;
  int32_t frames_per_obs;             /* K: 1 = the whole observation is one frame */
} dsact_frame_replay;

int dsact_replay_bind_frames(dsact_handle *h, const dsact_frame_replay *rb);
/* copy n_frames frames (host or device) into frame slots (frame_ptr + i) % frame_capacity, and n rows into rows
 * (ptr + i) % capacity: their frame ids (HOST int32 [n, frames_per_obs] each), act, rew, done, logp (host or device).
 * Every id is checked against [0, frame_capacity) before anything is copied (DSACT_EINVAL otherwise).  A handle with a
 * frame ring bound refuses dsact_replay_add (DSACT_ESTATE), and one with a flat ring refuses this call. */
int dsact_replay_add_frames(dsact_handle *h, const float *frames, int64_t n_frames, int64_t frame_ptr,
                            const int32_t *obs_frames, const int32_t *obs2_frames, const float *act, const float *rew,
                            const float *done, const float *logp, int64_t n, int64_t ptr, void *stream);
/* ---- coded frame replay ring: frames of 8-bit codes ----
 * A frame ring whose frame store holds one uint8 code per value (rb->frames points to uint8 [frame_capacity,
 * obs_elems / frames_per_obs]) and a device table of 256 floats: code c stands for table[c], bit for bit.  For sources
 * with at most 256 distinct values (8-bit images scaled to floats) it stores a quarter of the fp32 frame ring's bytes,
 * and every gather yields bit for bit what the fp32 frame ring holding the decoded frames would.
 * dsact_replay_bind_coded_frames: the checks of dsact_replay_bind_frames, and DSACT_EINVAL for a null table.  Binding
 * any ring kind replaces the others. */
int dsact_replay_bind_coded_frames(dsact_handle *h, const dsact_frame_replay *rb, const float *table);
/* dsact_replay_add_frames for a coded ring: n_frames frames of codes (HOST uint8) and table[0, n_codes) (host or device)
 * copied into the device table's first n_codes entries.  Every code is checked against n_codes, and n_codes against
 * [0, 256], before anything is copied (DSACT_EINVAL otherwise).  A coded ring refuses dsact_replay_add_frames
 * (DSACT_ESTATE), and every other ring kind refuses this call. */
int dsact_replay_add_coded_frames(dsact_handle *h, const uint8_t *codes, int64_t n_frames, int64_t frame_ptr,
                                  const float *table, int32_t n_codes, const int32_t *obs_frames,
                                  const int32_t *obs2_frames, const float *act, const float *rew, const float *done,
                                  const float *logp, int64_t n, int64_t ptr, void *stream);
/* ---- coded frame replay ring: frames of 16-bit codes ----
 * The coded ring with one uint16 code per value (rb->frames points to uint16 [frame_capacity, obs_elems /
 * frames_per_obs]) and a device table of 65 536 floats: half the fp32 frame ring's bytes, for sources with at most 65 536
 * distinct values, such as CarRacing's stacked grey frames (dot(rgb, [0.299, 0.587, 0.114]) / 128 - 1 take up to
 * 247 024 float32 values over all RGB triples; a stream that uses at most 65 536 of them fits).  Every gather yields bit
 * for bit what the fp32 frame ring holding the decoded frames would, and never reads how many table entries are in use,
 * so a captured replay step stays valid while the table grows.
 * dsact_replay_bind_coded16_frames: the checks of dsact_replay_bind_coded_frames. */
int dsact_replay_bind_coded16_frames(dsact_handle *h, const dsact_frame_replay *rb, const float *table);
/* dsact_replay_add_coded_frames for a 16-bit coded ring: HOST uint16 codes, n_codes in [0, 65 536], the same checks
 * before anything is copied.  Each ring kind's add call refuses every other ring kind (DSACT_ESTATE): the 8-bit and the
 * 16-bit coded rings refuse each other's calls. */
int dsact_replay_add_coded16_frames(dsact_handle *h, const uint16_t *codes, int64_t n_frames, int64_t frame_ptr,
                                    const float *table, int32_t n_codes, const int32_t *obs_frames,
                                    const int32_t *obs2_frames, const float *act, const float *rew, const float *done,
                                    const float *logp, int64_t n, int64_t ptr, void *stream);
/* sample_batch(): gather rows idx[i] (device int64, or NULL = draw uniformly in [0,size) on
 * the device) into the engine's batch arena; `out` receives the arena's device pointers */
int dsact_replay_sample(dsact_handle *h, int32_t batch, int64_t size, const int64_t *idx,
                        dsact_batch *out, void *stream);
/* sample_batch + local_update in one submission (no host round trip in between) */
int dsact_replay_step(dsact_handle *h, int32_t batch, int64_t size, const int64_t *idx,
                      const dsact_noise *noise, int64_t iteration, void *stream);
/* n_steps consecutive dsact_replay_step calls in one submission (one graph launch with use_graph): updates for iterations
 * iteration .. iteration+n_steps-1, each drawing from the ring of `size` rows, with the same generator counters, delayed-
 * update phases and resulting device state as the n single calls (the off_idx slot holds the last update's indices,
 * dsact_read_stats returns the last update's statistics).  The gather of update k+1 runs beside update k's backward, into
 * a second minibatch input set the library allocates on the first call, or in dsact_dp_connect (for max_batch rows; freed
 * by dsact_destroy).
 *   idx:       NULL (each update draws its own indices on the device) or device int64 [n_steps, batch].
 *   noise:     NULL (device draws) or arrays with a leading n_steps dimension: eps1/eps2 [n_steps, batch, act_dim],
 *              z3/z4 [n_steps, batch].
 *   stats_out: NULL or device float [n_steps, DSACT_NUM_STATS]. Row k holds update k's finalised tb_info over `batch`
 *              rows: the 16 floats dsact_read_stats(h, batch, ...) would return after the k-th single call.
 * MLP-engine handles only (DSAC-T and DSAC_V1); 1 <= n_steps <= DSACT_MAX_REPLAY_STEPS. */
#define DSACT_MAX_REPLAY_STEPS 64
int dsact_replay_steps(dsact_handle *h, int32_t n_steps, int32_t batch, int64_t size, const int64_t *idx,
                       const dsact_noise *noise, float *stats_out, int64_t iteration, void *stream);

/* ---- data-parallel replicas over NVLink peer memory (one process per GPU) ---------------------------------------
 * Replaces, for the same path, what `dsac-v2_b200/dp.py` does with three graph launches and four NCCL all-reduces
 * (reference: the reduction semantics of DSAC_V2.__compute_gradient, dsac_v2.py:150-206/233-241, under data
 * parallelism; the reference itself has no multi-GPU path, SURVEY.md 8e).  Set-up, once, on every rank:
 *   dsact_dp_export  -> allocate this rank's exchange buffer, return its CUDA IPC handle (DSACT_IPC_HANDLE_BYTES);
 *   (exchange the handles between the processes: any host transport, e.g. torch.distributed.all_gather_object)
 *   dsact_dp_connect -> map every peer's buffer (`handles` = world x DSACT_IPC_HANDLE_BYTES, rank order), reset epochs;
 *   (host barrier between the ranks).
 * Then dsact_dp_step / dsact_dp_replay_step = dsact_step / dsact_replay_step on this rank's shard, with the critic-std
 * sums, the gradients and the logged sums reduced over all ranks inside the step's own kernels (rank-ordered sums: the
 * replicas stay bit-identical).  `global_batch` = sum of the ranks' batch sizes.  A peer that never arrives makes
 * tb_info slot 14 non-zero (1 + its rank) after DSACT_DP_TIMEOUT_MS (default 10 s) instead of hanging the GPU.
 * MLP-engine handles with policy_std != DSACT_STD_SHARED return DSACT_EINVAL from all five calls (reduce between the split
 * calls dsact_grad_phase1/2 and dsact_apply instead). */
#define DSACT_IPC_HANDLE_BYTES 64
#define DSACT_DP_MAX_RANKS 8
int dsact_dp_export(dsact_handle *h, void *handle_out, int64_t *bytes_out);
int dsact_dp_connect(dsact_handle *h, int32_t rank, int32_t world, const void *handles);
int dsact_dp_step(dsact_handle *h, const dsact_batch *batch, const dsact_noise *noise, int64_t global_batch,
                  int64_t iteration, void *stream);
int dsact_dp_replay_step(dsact_handle *h, int32_t batch, int64_t size, const int64_t *idx, const dsact_noise *noise,
                         int64_t global_batch, int64_t iteration, void *stream);
/* n_steps consecutive dsact_dp_replay_step calls in one submission: dsact_replay_steps with every update data-parallel.
 * Updates for iterations iteration .. iteration+n_steps-1, each with its exchanges inside its kernels, in the order and
 * with the exchange epochs, generator counters and device state of the n single calls.  idx and noise as in
 * dsact_replay_steps ([n_steps, batch] and n_steps draws back to back; NULL: device draws, one generator counter per
 * update).  stats_out: NULL or device float [n_steps, DSACT_NUM_STATS]; row k holds update k's finalised tb_info over
 * `global_batch` rows, slot 14 included: what dsact_read_stats(h, global_batch, ...) returns after the k-th single call.
 * Every rank must make the same call (n_steps, iteration, global_batch).  Refused as its siblings refuse: head-wise and
 * DSAC_V1 handles, policy_std != DSACT_STD_SHARED, no dsact_dp_connect (DSACT_ESTATE), n_steps outside
 * [1, DSACT_MAX_REPLAY_STEPS], global_batch below batch. */
int dsact_dp_replay_steps(dsact_handle *h, int32_t n_steps, int32_t batch, int64_t size, const int64_t *idx,
                          const dsact_noise *noise, int64_t global_batch, float *stats_out, int64_t iteration, void *stream);

/* ---- DSAC_V1 on the MLP engine ---------------------------------------------------------------------------------------
 * DSAC_V1 (reference dsac_v1.py:56-273: ONE distributional critic, fixed TD bound) with MLP approximators and the policy's
 * "mlp_shared" std type (policy_std = DSACT_STD_SHARED; any other value is DSACT_EINVAL), on the tensor-core / SIMT engine of
 * dsact_create: the same dsact_config, in which critic and policy
 * may differ in depth, width and activation, in all three gemm_modes, with use_graph on or off, plus the two settings
 * DSAC-T lacks.
 * Flat layout: params = [ q | policy | log_alpha ], targets = [ q_target | policy_target ] (n_params = n_q + n_pi + 1,
 * n_targets = n_q + n_pi).  The handle takes dsact_step, dsact_step_host, dsact_stage_host / _release, dsact_replay_*,
 * dsact_read_stats (DSAC_V1's tb_info in slots 0, 2, 6, 8, 9, 10, 11) and dsact_profile_step with the semantics they
 * have for a DSAC-T handle; the split and data-parallel calls (dsact_grad_phase1/2, dsact_compute_grads, dsact_apply,
 * dsact_dp_*) return DSACT_EINVAL. */
typedef struct dsact_v1_options {
  int32_t abi_version;   /* = DSACT_ABI_VERSION */
  int32_t bound;         /* dsac_v1.py `bound` (:80): 1 = bounded loss (:219-229), 0 = Gaussian NLL (:231) */
  double td_bound;       /* dsac_v1.py `TD_bound` (:79, default 20): finite, > 0 */
} dsact_v1_options;
int dsact_v1_query_layout(const dsact_config *cfg, const dsact_v1_options *v1, dsact_layout *out);
int dsact_v1_create(const dsact_config *cfg, const dsact_v1_options *v1, int device, dsact_handle **out);

/* ---- head-wise fp32 engine: CNN approximators and the variants the MLP engine does not implement ---------------------
 * CNN approximators (BASELINE config 5, reference networks/cnn.py:30-53,151-240,383-461), value_func_type /
 * policy_func_type = "CNN": every network is a private conv encoder (Conv2d + ReLU per layer, no padding) followed by two
 * separate MLP heads `mean` and `log_std` on the flattened feature (the critics append the action to it).  Flat layout per
 * network, in state_dict order: conv.{0,2,..}.weight [Cout,Cin,k,k] / .bias, mean.{0,2,..}.weight / .bias,
 * log_std.{0,2,..}.weight / .bias; params = [q1|q2|policy|log_alpha].  fp32 direct convolutions + the fp32 grouped GEMMs
 * for the heads, eager launches.  data["obs"] / ["obs2"] are [B, C, H, W] (contiguous); replay rows are the flattened
 * [C*H*W] images (fp32, like the reference's CarRacing data, env_gym/gym_carracing_data.py:19-21).
 * The same engine also carries the variants of the reference that keep network outputs in separate heads or need another
 * loss, all in fp32: no encoder (n_conv = 0: the observation vector feeds the heads), one two-output head per critic
 * (q_heads = 1, networks/mlp.py), the policy's std types (pi_std), the plain Gaussian action distribution (act_dist) and
 * DSAC_V1 (algo = 1: ONE critic, flat layout [q | policy | log_alpha], dsac_v1.py).  DSAC_V1 with MLP approximators and
 * the "mlp_shared" policy also runs on the MLP engine (dsact_v1_create above), with its tensor-core modes, captured steps,
 * host staging and replay-fused steps.
 * dsact_cnn_create returns a dsact_handle that every dsact_* entry point above takes, with the same semantics, except:
 *  - dsact_step_host, dsact_stage_host / _release, dsact_replay_step(s), dsact_dp_replay_step(s), dsact_profile_step and
 *    dsact_test_gemm / dsact_test_chain return DSACT_EINVAL (the MLP engine implements them);
 *  - a DSAC_V1 handle (algo = 1) returns DSACT_EINVAL from the split and data-parallel calls (dsact_grad_phase1/2,
 *    dsact_compute_grads, dsact_apply, dsact_dp_export / _connect / _step);
 *  - phase 2's log_alpha gradient is this shard's additive share, and dsact_dp_step runs eagerly on `stream`. */
#define DSACT_MAX_CONV 8
typedef struct dsact_cnn_config {
  int32_t abi_version;
  int32_t channels, height, width;   /* obsv_dim = (C, H, W) */
  int32_t act_dim;
  int32_t n_conv;                    /* 0: no encoder, the observation (channels = obs_dim, height = width = 1) feeds the heads */
  int32_t conv_kernel[DSACT_MAX_CONV], conv_channels[DSACT_MAX_CONV], conv_stride[DSACT_MAX_CONV];
  int32_t n_hidden;                  /* hidden layers of every head MLP (networks/cnn.py:204 mlp_hidden_layers) */
  int32_t hidden[DSACT_MAX_HIDDEN];
  int32_t act_hidden;                /* DSACT_ACT_* of the head MLPs (the conv stack is ReLU) */
  int32_t max_batch, auto_alpha, delay_update;
  int32_t q_heads;                   /* 2: separate mean and std heads (networks/cnn.py:383-461); 1: one head with both outputs
                                        (networks/mlp.py:113-127, with n_conv = 0) */
  int32_t act_dist;                  /* 0 TanhGaussDistribution, 1 GaussDistribution (as in dsact_config) */
  int32_t pi_std;                    /* 0: log_std from its own head (networks/cnn.py, mlp.py std_type "mlp_separated");
                                        1: learnable row [1, act_dim] (mlp.py std_type "parameter"), laid out BEFORE the mean head;
                                        2: ONE head with 2 * act_dim outputs (mlp.py std_type "mlp_shared") */
  int32_t algo;                      /* 0: DSAC_V2 / DSAC-T (dsac_v2.py); 1: DSAC_V1 (dsac_v1.py:56-273): ONE critic, flat layout
                                        [q | policy | log_alpha], fixed TD bound */
  int32_t v1_bound;                  /* DSAC_V1 `bound` (dsac_v1.py:80): 1 = bounded loss (:219-229), 0 = Gaussian NLL (:231) */
  double gamma, tau, tau_b, alpha_fixed, lr_q, lr_pi, lr_alpha, min_log_std, max_log_std;
  double adam_beta1, adam_beta2, adam_eps;
  double td_bound;                   /* DSAC_V1 `TD_bound` (dsac_v1.py:79, default 20) */
} dsact_cnn_config;
int dsact_cnn_query_layout(const dsact_cnn_config *cfg, dsact_layout *out);
int dsact_cnn_create(const dsact_cnn_config *cfg, int device, dsact_handle **out);

/* introspection for tests/bench: number of kernel launches (graph nodes included)
 * submitted by this handle so far, and by the most recent entry-point call */
int64_t dsact_launch_count(const dsact_handle *h);
int32_t dsact_last_call_launches(const dsact_handle *h);

/* One eager (un-graphed) dsact_step with a CUDA event after every launch; per kernel class
 * [0 elementwise/other, 1 forward GEMM, 2 dgrad GEMM, 3 wgrad GEMM]: device milliseconds,
 * algorithmic FLOPs (2*M*N*K of every problem) and launch count.  Synchronises the stream. */
typedef struct dsact_profile {
  double ms[4], flops[4];
  int32_t launches[4];
  double total_ms;
} dsact_profile;
int dsact_profile_step(dsact_handle *h, const dsact_batch *batch, const dsact_noise *noise, int64_t iteration,
                       void *stream, dsact_profile *out);

/* Test hooks of the dense-layer kernels, in the handle's gemm_mode, on caller buffers (scratch images and weight-gradient
 * slabs come from cudaMalloc; the call synchronises `stream`).
 *
 * dsact_test_gemm: one group of problems of one variant, lowered and launched as a step lowers and launches its GEMM
 * groups (up to 16 problems; in fp32 mode a group of more than 8 is issued as two launches).
 *  variant 0 (forward): C[M,N]  = epi(A0[M,K0] * B[N,K0]^T + A1[M,K1] * B[N,K0:K0+K1]^T)
 *  variant 1 (dgrad)  : C[M,N]  = epi(A0[M,K0] * B[K0,N])
 *  variant 2 (wgrad)  : C[M,N] += A0[K0,M]^T * B[K0,N]   (batch split into slabs, summed into C)
 * epi (forward / dgrad): 0 store (+ bias[N]); 1 (forward) y = act(z), z = the product + bias, with Zout[M,ldc] (optional) = z (fp32
 * mode) or act'(z) (tensor-core modes); 2 (dgrad) y = the product * act'(z) with act'(z) from Zin[M,ldz] (tensor-core
 * modes; fp32 mode: z, the derivative taken in the epilogue), colsum[N] += column sums of y.
 * kB1: column of the second segment inside B's image (K0 rounded up to 64 in the step).  img (tensor-core modes): the bf16
 * hi/lo image of y ([M, img_pitch] per plane, planes img_plane elements apart, img_pitch % 8 == 0) is also stored; with
 * epi 1 or 2 C is then not written.  max_ctas > 0: issue the group in launches of at most that many CTAs. */
typedef struct dsact_test_layer {
  int32_t M, N, K0, K1, kB1;
  const float *A0, *A1, *B;
  int32_t lda0, lda1, ldb;
  int32_t epi, act;
  const float *bias;
  float *Zout;
  const float *Zin;
  int32_t ldz;
  float *colsum;
  float *C;
  int32_t ldc;
  void *img;            /* bf16 */
  int32_t img_pitch;
  int64_t img_plane;
} dsact_test_layer;
int dsact_test_gemm(dsact_handle *h, int32_t variant, const dsact_test_layer *probs, int32_t n, int32_t max_ctas, void *stream);

/* dsact_test_chain (tensor-core modes): one launch of the fused layer-chain kernel with 1-4 passes of one MLP, built by
 * the step's own chain code.  sizes[0..L+1]: input, L hidden widths, output; params: the flat fp32 [W_0 | b_0 | ... |
 * W_L | b_L] (W_j [sizes[j+1], sizes[j]]); act: hidden activation.  Layer 0 reads cat(x0[M,K0], x1[M,K1]) (K0 + K1 =
 * sizes[0]) with the x1 block at column kB1 of W_0's image.
 *  dgrad 0 (forward): out[M, sizes[L+1]] = the MLP's output; per hidden layer j (0-based), optional Zout[j] [M, sizes[j+1]]
 *                     = act'(z_j) and img[j] = the bf16 image of act(z_j).
 *  dgrad 1          : x0 = dOut[M, sizes[L+1]]; dz_j = (dz_{j+1} W_{j+1}) * act'(z_j) with Zin[j] = act'(z_j) [M, sizes[j+1]];
 *                     optional img[j] = the image of dz_j, colsum[j] += column sums of dz_j; out (optional) = dz_0 W_0
 *                     restricted to the x1 columns, [M, K1].
 * Images: pitch = sizes[j+1] rounded up to 8, planes pitch * M elements apart. */
typedef struct dsact_test_chain_pass {
  int32_t M;
  const float *x0, *x1;
  float *Zout[DSACT_MAX_HIDDEN];
  const float *Zin[DSACT_MAX_HIDDEN];
  void *img[DSACT_MAX_HIDDEN];
  float *colsum[DSACT_MAX_HIDDEN];
  float *out;
  int32_t out_ld;   /* forward: row pitch of `out` in floats, >= sizes[L+1] (0: contiguous): the head writes its columns of wider rows */
} dsact_test_chain_pass;
int dsact_test_chain(dsact_handle *h, int32_t dgrad, int32_t L, const int32_t *sizes, int32_t K0, int32_t K1, int32_t kB1,
                     int32_t act, const float *params, const dsact_test_chain_pass *passes, int32_t n_passes, void *stream);
/* dsact_test_chain_tiling: the same launch on a chosen layer-chain kernel instead of the one the launch shape selects:
 * tiling 0 = the column split (one 64-row tile per CTA), 1 = the ping-pong kernel (two 64-row tiles per CTA). */
int dsact_test_chain_tiling(dsact_handle *h, int32_t tiling, int32_t dgrad, int32_t L, const int32_t *sizes, int32_t K0,
                            int32_t K1, int32_t kB1, int32_t act, const float *params, const dsact_test_chain_pass *passes,
                            int32_t n_passes, void *stream);

/* Test hooks of the step kernels between the networks, on both engines: the step's own launch code (grid sizing and
 * argument construction) with the per-row arrays taken from caller buffers instead of the workspace.  Hyperparameters
 * come from the handle's configuration, the carried state (mean_std, counters, accumulators, iteration) from its bound
 * `state` and log_alpha from its bound `params`: set them there first.  Both calls synchronise `stream` and return
 * DSACT_EINVAL with a message, before any launch, for an unknown kernel or part, a batch outside [1, max_batch], a null
 * pointer the kernel needs, or an image on a handle without tensor-core images.
 *
 * dsact_test_rows runs one kernel over `batch` rows (A = act_dim):
 *  DSACT_TEST_SAMPLE: sample_kernel.  logits[0|1] [batch, 2A] (mean | log_std of pi(s), pi'(s')), eps[0|1] [batch, A] ->
 *    act[0|1] [batch, A], logp[0|1] [batch]; reads out_q[0] (and out_q[1] on DSAC-T) for the critic-std sums
 *    (state[DSACT_STATE_STDSUM..+1]) and adds the logged policy sums to the accumulators.  advance_rng: also step the
 *    generator counter.
 *  DSACT_TEST_LOSS: loss_kernel (DSAC-T) or loss_v1_kernel (DSAC_V1), chosen by the handle.  rew, done, z3 (DSAC-T: and
 *    z4), logp[0] (logp_new), logp[1] (logp2) [batch], out_q[p] [batch, 2] (mean, raw std) of Q_k(s,a) (p = k),
 *    Q'_k(s',a') (p = 2 + k), Q_k(s,a~) (p = 4 + k) -> d_out_q[k], d_out_qa[k] [batch, 2]; gbias_q[k] += the mean's
 *    bias gradient, gbias_q_raw[k] += the std output's (null: gbias_q[k] + 1).  DSAC_V1 uses k = 0 only.
 *  DSACT_TEST_POLICY_GRAD: policy_grad_kernel (one critic: DSAC_V1 on the MLP engine, which ignores d_act[1]).
 *    logits[0], eps[0], d_act[k] [batch, A] -> d_logits [batch, 2A]; gbias_pi += the bias gradient of the mean half
 *    (of the whole row when gbias_ls is null), gbias_ls += that of the log_std half.
 *  DSACT_TEST_STATS: finalize_stats_kernel over global_batch rows into stats_out (16 floats; null: the state's slots).
 * global_batch: the denominator of every batch mean (>= batch).  max_blocks > 0 caps the grid's blocks, so that a small
 * batch takes several grid-stride trips.  img_* (tensor-core modes of the MLP engine; may be null): bf16 hi / lo images
 * [2][batch][pitch] of act[k] (width A), d_out_q[k] / d_out_qa[k] (width 2) and d_logits (width 2A), pitch = width
 * rounded up to 8; the second plane only in bf16x3. */
enum { DSACT_TEST_SAMPLE = 0, DSACT_TEST_LOSS = 1, DSACT_TEST_POLICY_GRAD = 2, DSACT_TEST_STATS = 3 };
typedef struct dsact_test_row_io {
  int32_t kernel, batch;
  int64_t global_batch;
  int32_t max_blocks, advance_rng;
  const float *logits[2], *eps[2];
  float *act[2], *logp[2];
  const float *rew, *done, *z3, *z4;
  const float *out_q[6];
  float *d_out_q[2], *d_out_qa[2];
  const float *d_act[2];
  float *d_logits;
  float *gbias_q[2], *gbias_q_raw[2], *gbias_pi, *gbias_ls;
  void *img_act[2], *img_q[2], *img_qa[2], *img_dlogits;
  float *stats_out;
  /* DSACT_TEST_POLICY_GRAD with split_dlogits != 0 (two policy heads, or a log_std row): img_dlogits is the image of the
   * mean half alone (width A) and img_dlogits_ls that of the log_std half (width A; null: not written) */
  void *img_dlogits_ls;
  int32_t split_dlogits;
} dsact_test_row_io;
int dsact_test_rows(dsact_handle *h, const dsact_test_row_io *rows, void *stream);

/* dsact_test_apply: one launch of the Adam / Polyak kernel on the handle's bound buffers, built as a single-call step
 * builds it.  part: 0 the whole flat buffer, 1 the critics' span without closing the step, 2 the rest and the closing
 * (a 4-element group straddling the boundary goes with part 2).  fold_slabs (tensor-core modes of the MLP engine, 0 to
 * the number of slabs the workspace holds): fold that many weight-gradient split slabs into `grads` first.
 * scalars_ready: the Adam step sizes are 0 formed in the kernel, 1 read from state[DSACT_STATE_ADAM..+4], 2 read there
 * only if stamped with the current counters.  tail_rows > 0: also form the log_alpha gradient over tail_rows rows (of
 * global_batch) and, when closing, commit the mean_std EMA and stamp the next step's scalars as the step does.
 * max_blocks > 0 caps the grid's blocks. */
int dsact_test_apply(dsact_handle *h, int32_t part, int32_t fold_slabs, int32_t scalars_ready, int32_t tail_rows,
                     int64_t global_batch, int32_t max_blocks, void *stream);

/* Test hooks of the peer-memory data-parallel exchange, with every rank of a world on one device.
 *
 * dsact_test_dp_attach: make h rank `rank` of the `world` handles peers[0..world-1] (rank order, peers[rank] == h), all
 * of one process, one device and one engine with the same parameter count, each after dsact_dp_export.  The peers'
 * exchange buffers are used directly (no CUDA IPC).  Like dsact_dp_connect it resets h's flags, epoch and error slot and
 * drops the MLP engine's captured graphs.  buffer / floats (may be null): h's exchange buffer and its length in floats
 * (header, gradient block, reduced block; layout in csrc/dp_peer.cuh).
 *
 * dsact_test_dp: one operation on an attached handle, through the data-parallel step's own launch code; synchronises
 * `stream`.
 *  DSACT_TEST_DP_EXCHANGE: the exchange of kind io->kind (0 critic-std sums, 1 logged sums) for every rank of the world
 *    at once: io->ranks holds the world's attached handles in rank order.
 *  DSACT_TEST_DP_FOLD: io->grads plus io->nslabs slabs at io->slabs (io->slab_stride floats apart) over elements
 *    [0, io->n) into h's gradient block; io->tail_rows > 0: element n - 1 is the log_alpha gradient of tail_rows rows of
 *    io->global_batch formed from the logged sum in h's state (the MLP engine's step), 0: a plain sum (the head-wise one).
 *  DSACT_TEST_DP_REDUCE_SCATTER: h's slice of the two-shot reduction (worlds of 6 and more ranks in the step).
 *  DSACT_TEST_DP_APPLY: Adam / Polyak on the rank-ordered gradient sum, as the engine's step builds it (one-shot below
 *    6 ranks, the reduced block from 6 up); the MLP engine's with the end-of-backward bookkeeping over io->tail_rows
 *    (>= 1) rows of io->global_batch.
 * Both calls return DSACT_EINVAL or DSACT_ESTATE with a message, before any launch, for an unknown op, a rank or world
 * outside [2, 8], a handle that is not exported or attached, a DSAC_V1 handle or an MLP handle whose policy_std is not
 * mlp_shared. */
int dsact_test_dp_attach(dsact_handle *h, int32_t rank, int32_t world, dsact_handle *const *peers, void **buffer,
                         int64_t *floats);
enum { DSACT_TEST_DP_EXCHANGE = 0, DSACT_TEST_DP_FOLD = 1, DSACT_TEST_DP_REDUCE_SCATTER = 2, DSACT_TEST_DP_APPLY = 3 };
typedef struct dsact_test_dp_io {
  int32_t kind;
  dsact_handle *const *ranks;
  const float *grads, *slabs;
  int32_t nslabs;
  int64_t slab_stride, n;
  int32_t tail_rows;
  int64_t global_batch;
} dsact_test_dp_io;
int dsact_test_dp(dsact_handle *h, int32_t op, const dsact_test_dp_io *io, void *stream);

/* Test hook of the head-wise engine's convolution kernels: one layer (NCHW, square k x k window, stride, no padding) on
 * caller buffers, enqueued on `stream` of the current device.
 *  op 0 (forward)        : out[B,cout,hout,wout] = relu(conv(x, w) + b)
 *  op 1 (weight gradient): dw[cout,cin,k,k] += corr(x, dy), db[cout] += sum(dy)   (dy: gradient of the pre-activation)
 *  op 2 (dgrad)          : out[B,cin,hin,win] = convT(dy, w) (.) [x > 0]
 * r, cob, slabs, channels: 0 = the engine's choice; otherwise positions per thread of the forward (1, 2, 4), output
 * channels per weight-gradient block (1, 4, 8), row slabs of the weight gradient, and channels per thread of the forward /
 * dgrad kernels (8 or 1).  DSACT_EINVAL for a combination that has no kernel. */
int dsact_cnn_test_conv(int32_t op, int32_t batch, int32_t cin, int32_t hin, int32_t win, int32_t cout, int32_t k, int32_t stride,
                        const float *x, const float *w, const float *b, const float *dy, float *out, float *dw, float *db,
                        int32_t r, int32_t cob, int32_t slabs, int32_t channels, void *stream);

#define DSACT_STATE_STDSUM 4   /* state[4], state[5]: local sums of critic std (phase1 -> phase2) */
#define DSACT_STATE_ACC 16     /* state[16..47]: per-step accumulators (sums first, then mins) */
#define DSACT_STATE_STATS 48   /* state[48..63]: finalised tb_info */
#define DSACT_STATE_ADAM 64    /* state[64..68]: Adam step sizes / bias corrections of the running step (internal) */
#define DSACT_STATE_DP_ERR 7    /* int32: 0, or 1 + rank of the peer a dsact_dp_step exchange timed out on */
#define DSACT_STATE_DP_EPOCH 15 /* int32: exchanges opened by dsact_dp_step so far (reset by dsact_dp_connect) */

#ifdef __cplusplus
}
#endif
#endif /* DSACT_H */
