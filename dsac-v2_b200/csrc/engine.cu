// libdsact.so — host side of the H100-native (sm_90a) DSAC-T update engine (C ABI in include/dsact.h).
//
// Orchestrates one `DSAC_V2.local_update` (reference dsac_v2.py:102-105,150-347) as a fixed sequence of
// kernel launches on caller-owned flat fp32 buffers, optionally captured once into a CUDA graph and
// replayed.  No CPU fallback: every entry point needs a CUDA device.
//
// Two engines sit behind one handle: the MLP engine of this file (wgmma / SIMT GEMMs) and the head-wise fp32 engine of
// cnn_engine.cuh (CNN approximators, the policy's other std types, DSAC_V1).  This file holds the shell they share, the
// launches of the step kernels they share (noise, begin_step, sample, loss, policy gradient, apply, gather) and the
// C entry points, which dispatch once on the handle's engine.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <tuple>

#include <vector>

#include "../../include/dsact.h"
#include "gemm_simt.cuh"
#include "kernels.cuh"
#include "tc_host.cuh"
#include "chain_pp.cuh"
#include "wgrad_tc.cuh"
#include "dp_peer.cuh"

using namespace dsact;

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CUDA_TRY(x)                                                                       \
  do {                                                                                    \
    cudaError_t e_ = (x);                                                                 \
    if (e_ != cudaSuccess) return fail(DSACT_ECUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
  } while (0)

// ---- network geometry -------------------------------------------------------
struct Net {
  int L;                                   // hidden layers
  int s[DSACT_MAX_HIDDEN + 2];             // s[0] input, s[1..L] hidden, s[L+1] output
  int64_t w[DSACT_MAX_HIDDEN + 1], b[DSACT_MAX_HIDDEN + 1], n;  // offsets inside the net, total floats
  void build(int in, const int32_t* hidden, int L_, int out) {
    L = L_;
    s[0] = in;
    for (int j = 0; j < L; ++j) s[j + 1] = hidden[j];
    s[L + 1] = out;
    n = 0;
    for (int j = 0; j <= L; ++j) {
      w[j] = n; n += (int64_t)s[j + 1] * s[j];
      b[j] = n; n += s[j + 1];
    }
  }
};

static int64_t round64(int64_t x) { return (x + 63) / 64 * 64; }

// The policy span of the flat layout (DSACT_STD_*): `pi` is the network that produces the mean (mlp_shared: mean | log_std).
// mean / ls: where that network and the log_std network or row start inside the span (ls -1: none), n: floats in the span.
struct PiSpan { int64_t mean, ls, n; };
static PiSpan pi_span(int policy_std, const Net& pi, int A) {
  if (policy_std == DSACT_STD_SEPARATED) return PiSpan{0, pi.n, 2 * pi.n};
  if (policy_std == DSACT_STD_PARAMETER) return PiSpan{A, 0, A + pi.n};   // a module's own parameter precedes its children's
  return PiSpan{0, -1, pi.n};
}
static int pi_outputs(const dsact_config& c) { return c.policy_std == DSACT_STD_SHARED ? 2 * c.act_dim : c.act_dim; }

// bf16 image slot inside the arena (TC modes only)
struct ImgSlot {
  int64_t off = -1;  // floats from the workspace base
  int rows = 0, width = 0, pitch = 0;
  int64_t plane = 0;
};

// The arena slots both engines have and the step kernels they share read (floats from the workspace base).  Each engine
// places them in its own arena order.
struct StepSlots {
  int64_t obs, obs2, act, rew, done, logp, idx;    // gathered minibatch + int64 indices
  int64_t eps1, eps2, z3, z4;                      // device-generated noise
  int64_t logitsP, logitsT, dlogits;               // policy outputs (mean | log_std) of pi(s), pi'(s'); their gradient
  int64_t new_act, act2, logp_new, logp2;          // a~ ~ pi(s), a' ~ pi'(s') and their log-probs
  int64_t outQ[6], dOut[6], dAct[2];               // Q_k(s,a), Q'_k(s',a'), Q_k(s,a~) [B,2] and gradients; dL/da~ per critic
                                                   // (pass p belongs to critic p & 1; -1: a slot of a critic the handle lacks)
};

// The hyperparameters both configuration structs name alike
struct StepHyper {
  int auto_alpha, delay_update, act_dist;
  double gamma, tau, tau_b, alpha_fixed, lr_q, lr_pi, lr_alpha, min_log_std, max_log_std, adam_beta1, adam_beta2, adam_eps;
  template <typename Cfg> static StepHyper of(const Cfg& c) {
    return StepHyper{c.auto_alpha, c.delay_update, c.act_dist, c.gamma, c.tau, c.tau_b, c.alpha_fixed, c.lr_q, c.lr_pi,
                     c.lr_alpha, c.min_log_std, c.max_log_std, c.adam_beta1, c.adam_beta2, c.adam_eps};
  }
};

// activation arena of the MLP engine, all offsets in floats from the workspace base
struct Arena : StepSlots {
  int64_t zP[DSACT_MAX_HIDDEN], hP[DSACT_MAX_HIDDEN], hT[DSACT_MAX_HIDDEN];
  int64_t zQ[6][DSACT_MAX_HIDDEN], hQ[6][DSACT_MAX_HIDDEN];
  int64_t dzQ[6][DSACT_MAX_HIDDEN], dzP[DSACT_MAX_HIDDEN];
  int64_t zL[DSACT_MAX_HIDDEN], hL[DSACT_MAX_HIDDEN], hLT[DSACT_MAX_HIDDEN], dzL[DSACT_MAX_HIDDEN];   // log_std network (mlp_separated)
  // ---- tensor-core modes: bf16 hi/lo images of every GEMM operand + wgrad split slabs
  bool tc;
  // i_dlogits: dL/d(mean | log_std) [B, 2A] of mlp_shared; with two policy heads, or a log_std row, dL/d(mean) [B, A], and
  // i_dlogits_ls dL/d(log_std) [B, A] of the log_std network: a TMA operand starts 16-byte aligned, column A of a row does not
  ImgSlot i_obs, i_obs2, i_act, i_new_act, i_act2, i_dlogits, i_dlogits_ls;
  ImgSlot i_hP[DSACT_MAX_HIDDEN], i_hT[DSACT_MAX_HIDDEN], i_dzP[DSACT_MAX_HIDDEN];
  ImgSlot i_hL[DSACT_MAX_HIDDEN], i_hLT[DSACT_MAX_HIDDEN], i_dzL[DSACT_MAX_HIDDEN];
  ImgSlot i_hQ[6][DSACT_MAX_HIDDEN], i_dzQ[6][DSACT_MAX_HIDDEN], i_dOut[6];
  ImgSlot i_wq[4][DSACT_MAX_HIDDEN + 1], i_wpi[4][DSACT_MAX_HIDDEN + 1];  // q1,q2,q1',q2' (DSAC_V1: q, -, q', -) / pi,pi',
                                                                          // log_std network of pi, of pi' (mlp_separated)
  int kpad_q0;        // column of the act block inside the Q layer-0 weight image
  int64_t slabs;      // [nslabs][n_params] fp32 wgrad partials, the arena's last region
  int nslabs;
  int64_t slab_stride;   // floats between slabs: n_params rounded up to 4 (float4 access to every slab)
  int64_t total;
  // nq critics (DSAC-T 2, DSAC_V1 1): the passes and weight images of critic 1 exist only with two
  void build(const dsact_config& c, const Net& q, const Net& pi, int nq = 2) {
    int64_t B = c.max_batch, O = c.obs_dim, A = c.act_dim, off = 0;
    auto take = [&](int64_t n) { int64_t o = off; off += round64(n); return o; };
    auto img = [&](int rows, int width) {
      ImgSlot s;
      s.rows = rows; s.width = width; s.pitch = (width + 7) / 8 * 8;
      s.plane = round64((int64_t)rows * s.pitch);  // elements per plane, multiple of 64
      s.off = take(s.plane);  // 2 planes of bf16 = plane floats
      return s;
    };
    obs = take(B * O); obs2 = take(B * O); act = take(B * A); rew = take(B); done = take(B); logp = take(B); idx = take(2 * B);
    eps1 = take(B * A); eps2 = take(B * A); z3 = take(B); z4 = take(B);
    for (int j = 0; j < pi.L; ++j) { zP[j] = take(B * pi.s[j + 1]); hP[j] = take(B * pi.s[j + 1]); hT[j] = take(B * pi.s[j + 1]); dzP[j] = take(B * pi.s[j + 1]); }
    const bool two_heads = c.policy_std == DSACT_STD_SEPARATED;
    for (int j = 0; j < pi.L && two_heads; ++j) { zL[j] = take(B * pi.s[j + 1]); hL[j] = take(B * pi.s[j + 1]); hLT[j] = take(B * pi.s[j + 1]); dzL[j] = take(B * pi.s[j + 1]); }
    logitsP = take(B * 2 * A); logitsT = take(B * 2 * A); dlogits = take(B * 2 * A);
    new_act = take(B * A); act2 = take(B * A); logp_new = take(B); logp2 = take(B);
    for (int p = 0; p < 6; ++p) {
      outQ[p] = dOut[p] = -1;
      if ((p & 1) >= nq) continue;
      for (int j = 0; j < q.L; ++j) { zQ[p][j] = take(B * q.s[j + 1]); hQ[p][j] = take(B * q.s[j + 1]); dzQ[p][j] = take(B * q.s[j + 1]); }
      outQ[p] = take(B * 2); dOut[p] = take(B * 2);
    }
    dAct[0] = take(B * A); dAct[1] = nq == 2 ? take(B * A) : -1;
    tc = c.gemm_mode != DSACT_GEMM_FP32;
    nslabs = 0; slabs = 0; slab_stride = 0; kpad_q0 = (int)((O + 63) / 64 * 64);
    if (tc) {
      const int Bi = (int)B;
      i_obs = img(Bi, (int)O); i_obs2 = img(Bi, (int)O); i_act = img(Bi, (int)A); i_new_act = img(Bi, (int)A); i_act2 = img(Bi, (int)A);
      i_dlogits = img(Bi, pi.s[pi.L + 1]);
      if (two_heads) i_dlogits_ls = img(Bi, (int)A);
      for (int j = 0; j < pi.L; ++j) { i_hP[j] = img(Bi, pi.s[j + 1]); i_hT[j] = img(Bi, pi.s[j + 1]); i_dzP[j] = img(Bi, pi.s[j + 1]); }
      for (int j = 0; j < pi.L && two_heads; ++j) { i_hL[j] = img(Bi, pi.s[j + 1]); i_hLT[j] = img(Bi, pi.s[j + 1]); i_dzL[j] = img(Bi, pi.s[j + 1]); }
      for (int p = 0; p < 6; ++p) {
        if ((p & 1) >= nq) continue;
        for (int j = 0; j < q.L; ++j) { i_hQ[p][j] = img(Bi, q.s[j + 1]); i_dzQ[p][j] = img(Bi, q.s[j + 1]); }
        i_dOut[p] = img(Bi, 2);
      }
      for (int n = 0; n < 4; ++n)
        for (int j = 0; j <= q.L && (n & 1) < nq; ++j) i_wq[n][j] = img(q.s[j + 1], j == 0 ? kpad_q0 + (int)A : q.s[j]);
      for (int n = 0; n < (two_heads ? 4 : 2); ++n)
        for (int j = 0; j <= pi.L; ++j) i_wpi[n][j] = img(pi.s[j + 1], pi.s[j]);
      // batch split of the weight-gradient GEMMs: at most 4 slabs of >= 256 rows (more slabs mean more partial tiles to
      // write and to fold in apply)
      nslabs = (int)(B / 256); if (nslabs > 4) nslabs = 4; if (nslabs < 1) nslabs = 1;
      slab_stride = (nq * q.n + pi_span(c.policy_std, pi, (int)A).n + 1 + 3) / 4 * 4;
      slabs = take((int64_t)nslabs * slab_stride);
    } else {
      slabs = off;   // the (empty) last region
    }
    total = off;
  }
};

// Everything the work captured for an update call depends on that is not read from device memory when the graph runs
// (graph_key derives it from the call)
struct GraphKey {
  int run; bool replay, dp;                              // what the call runs (UpdateCall)
  const float *obs, *act, *rew, *obs2, *done; int32_t batch;   // its rows
  const float *eps1, *eps2, *z3, *z4;                    // its noise (null: device noise)
  int64_t global_batch;
  bool imaged;                                           // the inputs' images were already written (not by the prologue)
  const int64_t* idx;                                    // replay indices (null: drawn on the device)
  int32_t n_steps; const float* stats_out;
  auto tie() const {
    return std::tie(run, replay, dp, obs, act, rew, obs2, done, batch, eps1, eps2, z3, z4, global_batch, imaged, idx,
                    n_steps, stats_out);
  }
  bool operator==(const GraphKey& o) const { return tie() == o.tie(); }
};
struct GraphEntry { GraphKey key; cudaGraphExec_t exec; int launches; uint64_t stamp; };

// The shell both engines share: device, bound buffers, generator seed, replay ring, peer exchange, what the last phase 1
// ran on, launch counts, the few sizes the shell's entry points check against, and the arena slots and hyperparameters
// of the step kernels both engines launch.  `engine` says which of MlpHandle (the wgmma / SIMT MLP engine, this file)
// and HeadsHandle (the head-wise fp32 engine, cnn_engine.cuh) it is.
enum { ENGINE_MLP = 0, ENGINE_HEADS = 1 };
struct dsact_handle {
  int engine;
  int device = 0, num_sms = 0;
  int64_t obs_elems = 0;     // floats of one observation row
  int act_dim = 0, max_batch = 0;
  int64_t n_params = 0;      // flat parameter count (log_alpha included)
  bool v1 = false;           // DSAC_V1: one critic, local steps only, its own policy-statistic denominator
  int v1_bound = 1;          // DSAC_V1's critic loss: 1 bounded (dsac_v1.py:219-229), 0 Gaussian NLL (:231)
  double td_bound = 20.0;    // DSAC_V1's TD bound (dsac_v1.py:79)
  StepSlots slot = {};
  StepHyper hyper = {};
  // output activations (dsact_set_output_activations; fixed at bind): ACT_* codes of the critics' outputs and of the
  // policy's mean / log_std halves
  OutActs oa = {ACT_LINEAR, ACT_LINEAR, ACT_LINEAR};
  bool outact() const { return oa.q != ACT_LINEAR || oa.mean != ACT_LINEAR || oa.ls != ACT_LINEAR; }
  dsact_buffers buf = {};
  bool bound = false, rb_bound = false;
  uint64_t seed = 0x5DEECE66Dull;
  int64_t dev_iter = -1;     // what state[ST_ITER] will hold when the next enqueued work runs (-1 unknown)
  int64_t dev_rb_size = -1;  // what state[ST_RB_SIZE] holds
  dsact_replay rb = {};
  dsact_frame_replay fr = {};   // the frame ring, when rb_frames (binding either ring kind replaces the other)
  bool rb_frames = false;
  int rb_code_bytes = 0;        // rb_frames: fr.frames holds fp32 values (0), or uint8 (1) / uint16 (2) codes decoded
                                // through fr_table
  float* fr_table = nullptr;    // a coded ring's device table [256 or 65 536]
  DpPeer dp;                 // peer-memory data parallelism (dp_peer.cuh)
  dsact_batch pending = {};  // the rows the last phase 1 ran on (batch 0: none); dsact_grad_phase2 runs on them
  dsact_noise pending_noise = {};   // ... and its noise (the arena's slots for device noise)
  int64_t launches = 0;
  int32_t last_launches = 0;
  explicit dsact_handle(int e) : engine(e) {}
  float* W() const { return reinterpret_cast<float*>(buf.workspace); }
  int64_t rb_rows() const { return rb_frames ? fr.capacity : rb.capacity; }
};

struct MlpHandle : dsact_handle {
  dsact_config cfg;
  Net q, pi;
  Arena ar;
  bool arena_imaged;         // the last dsact_replay_sample left bf16 images of obs/obs2/act beside the arena batch
  cudaStream_t cap_stream;   // capture-only stream
  cudaStream_t side_stream;  // second branch inside a step (critic weight gradients || policy backward chain)
  cudaEvent_t ev_fork, ev_join;
  cudaEvent_t ev_pro_fork, ev_pro_join;   // prologue branch (weight images, noise, clears) beside the replay gather
  cudaEvent_t ev_dp_fork, ev_dp_join;     // std-sum exchange of the data-parallel step beside the second forward chain
  // host-minibatch staging (dsact_stage_host): two device sets + a private copy stream
  float* stage_buf[2] = {nullptr, nullptr};
  int64_t stage_floats = 0;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_stage_ready[2] = {nullptr, nullptr}, ev_stage_done[2] = {nullptr, nullptr};
  bool stage_done_valid[2] = {false, false};
  int stage_turn = 0, stage_held = -1;
  // second minibatch input set of dsact_replay_steps (library-owned, allocated on its first call for max_batch rows):
  // consecutive updates of one call alternate between the arena's set (0) and this one (1), so that the gather of update
  // k + 1 runs beside update k's backward.  Offsets in floats from in2: fp32 obs / obs2 / act / rew / done / logp, and
  // (tensor-core modes) the bf16 images of obs / obs2 / act.
  float* in2 = nullptr;
  int64_t in2_obs = 0, in2_obs2 = 0, in2_act = 0, in2_rew = 0, in2_done = 0, in2_logp = 0;
  ImgSlot in2_img[3];
  cudaStream_t gather_stream = nullptr;   // the next update's gather, forked beside a captured update's backward
  cudaEvent_t ev_gather_fork = nullptr, ev_gather_join = nullptr;
  bool tc_attr_done = false, chain_attr_done = false, wgrad_attr_done = false;   // cudaFuncSetAttribute is per device:
                                                                                 // tracked per handle
  TcGroup tc_scratch;                                   // host-side lowering scratch of launch_tc (~5 KiB)
  std::vector<GraphEntry> graphs;
  uint64_t stamp = 0;
  MlpHandle() : dsact_handle(ENGINE_MLP) {}
  int nq() const { return v1 ? 1 : 2; }   // critics: DSAC_V1 has one (flat layout [q | policy | log_alpha])
  PiSpan span() const { return pi_span(cfg.policy_std, pi, cfg.act_dim); }
  bool tc() const { return cfg.gemm_mode != DSACT_GEMM_FP32; }
  bool fused() const {  // layer-chain kernel: every layer must fit one 256-column wgmma accumulator / A operand
    if (!tc()) return false;
    for (int j = 1; j <= q.L + 1; ++j) if (q.s[j] > 256) return false;
    for (int j = 1; j <= pi.L + 1; ++j) if (pi.s[j] > 256) return false;
    for (int j = 1; j <= q.L; ++j) if (q.s[j] % 8) return false;    // hidden widths: multiples of 8 (the validated shapes)
    for (int j = 1; j <= pi.L; ++j) if (pi.s[j] % 8) return false;
    return cfg.act_dim <= 256;
  }
  int passes() const { return cfg.gemm_mode == DSACT_GEMM_BF16X3 ? 3 : 1; }
  Img img(const ImgSlot& s, int rows) const {  // image handle with the live row count
    Img i;
    if (s.off < 0) return i;
    i.p = reinterpret_cast<__nv_bfloat16*>(W() + s.off);
    i.rows = rows; i.width = s.width; i.pitch = s.pitch; i.plane = s.plane;
    return i;
  }
  // image of input `which` (0 obs, 1 obs2, 2 act) of input set `set`
  Img input_img(int set, int which, int rows) const {
    if (set == 0) return img(which == 0 ? ar.i_obs : which == 1 ? ar.i_obs2 : ar.i_act, rows);
    Img i;
    const ImgSlot& s = in2_img[which];
    if (s.off < 0) return i;
    i.p = reinterpret_cast<__nv_bfloat16*>(in2 + s.off);
    i.rows = rows; i.width = s.width; i.pitch = s.pitch; i.plane = s.plane;
    return i;
  }
};

enum { CLS_OTHER = 0, CLS_GEMM_FWD = 1, CLS_GEMM_DGRAD = 2, CLS_GEMM_WGRAD = 3, CLS_COUNT = 4 };
struct Prof {  // dsact_profile_step: an event after every launch
  std::vector<cudaEvent_t> ev;
  std::vector<int> cls;
  std::vector<double> flops;
};
struct Ctx {
  cudaStream_t s;
  int launches;
  cudaError_t err;
  Prof* prof = nullptr;
  cudaStream_t side = nullptr;   // optional second stream for an independent branch (null: serialise on `s`)
  bool pdl = true;               // programmatic dependent launch for this enqueue (off in fp32 mode, see launch_k)
  void check() { cudaError_t e = cudaGetLastError(); if (e != cudaSuccess && err == cudaSuccess) err = e; }
  void done(int cls = CLS_OTHER, double flops = 0.0) {
    launches++;
    if (prof) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      cudaEventRecord(e, s);
      prof->ev.push_back(e);
      prof->cls.push_back(cls);
      prof->flops.push_back(flops);
    }
  }
};

// Every kernel goes out with the programmatic-dependent-launch attribute (each kernel begins with griddepcontrol.wait),
// so that inside the captured graph a kernel's launch and prologue overlap its predecessor's tail.  The fp32 SIMT mode
// launches without it: its multi-wave GEMM grids would lose SM slots to early-launched dependents.
template <typename... KArgs, typename... Args>
static void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Ctx& c, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = c.s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = c.pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
  if (e != cudaSuccess && c.err == cudaSuccess) c.err = e;
}

// ---- GEMM group launch -------------------------------------------------------
enum { V_FWD = 0, V_DGRAD = 1, V_WGRAD = 2 };

// A group of independent problems in both lowerings: fp32 pointers (GemmGroup) and bf16 images (TcExtra).
struct Group {
  GemmGroup g;               // SIMT lowering holds at most MAXG problems per launch; wgmma up to TC_MAXG
  GemmProb more[TC_MAXG - MAXG];
  TcExtra x[TC_MAXG];
  int n = 0;
  GemmProb& prob(int i) { return i < MAXG ? g.p[i] : more[i - MAXG]; }
  const GemmProb& prob(int i) const { return i < MAXG ? g.p[i] : more[i - MAXG]; }
  float* wg_slab = nullptr;   // wgrad split slabs (default: the arena's, addressed like the gradient buffer)
  long long wg_stride = 0;
  long long wg_off[TC_MAXG] = {};   // with wg_slab: where problem i's partial tiles start inside each slab
  int wg_nslabs = 0;
  Group() { g.n = 0; }
  void push(const GemmProb& p, const TcExtra& e) { x[n] = e; prob(n) = p; ++n; g.n = n < MAXG ? n : MAXG; }
};

template <int BM, int BN>
static void launch_variant(const GemmGroup& g, int variant, int grid, Ctx& c) {
  if (variant == V_FWD) launch_k(gemm_kernel<BM, BN, true, true>, grid, 256, 0, c, g);
  else if (variant == V_DGRAD) launch_k(gemm_kernel<BM, BN, true, false>, grid, 256, 0, c, g);
  else launch_k(gemm_kernel<BM, BN, false, false>, grid, 256, 0, c, g);
}

static void launch_simt(int num_sms, GemmGroup& g, int variant, Ctx& c) {
  auto count = [&](int T) {
    int total = 0;
    for (int i = 0; i < g.n; ++i) total += ((g.p[i].M + T - 1) / T) * ((g.p[i].N + T - 1) / T);
    return total;
  };
  const bool big = variant != V_WGRAD && count(128) >= num_sms;
  const int T = big ? 128 : 64;
  const int base = count(T);
  int grid = 0;
  for (int i = 0; i < g.n; ++i) {
    GemmProb& p = g.p[i];
    p.tiles_m = (p.M + T - 1) / T;
    p.tiles_n = (p.N + T - 1) / T;
    p.ksplit = 1;
    if (variant == V_WGRAD) {  // reduction over the batch: split it until ~2 CTAs per SM, >= 4 k-tiles each
      const int nt = (p.K[0] + KT - 1) / KT;
      int want = (2 * num_sms + base - 1) / base;
      int maxs = nt / 4 > 0 ? nt / 4 : 1;
      p.ksplit = want < maxs ? want : maxs;
      if (p.ksplit < 1) p.ksplit = 1;
      const int per = (nt + p.ksplit - 1) / p.ksplit;
      p.ksplit = (nt + per - 1) / per;  // no empty splits
    }
    p.tile_start = grid;
    grid += p.tiles_m * p.tiles_n * p.ksplit;
  }
  if (big) launch_variant<128, 128>(g, variant, grid, c);
  else launch_variant<64, 64>(g, variant, grid, c);
}

// Weight gradients: the persistent two-warpgroup kernel (wgrad_tc.cuh), one launch of at most `max_ctas` CTAs (0: one
// per SM; a bound leaves the remaining SMs to a concurrent branch of the step graph for the whole duration).  Every
// problem is split over the batch into the fixed slab count; empty splits store zeros, so the reduction is always valid.
static void launch_tc_wgrad(MlpHandle* h, Group& G, Ctx& c, int max_ctas) {
  TcGroup& t = h->tc_scratch;
  memset(&t, 0, sizeof(t));
  t.n = G.n;
  t.passes = h->passes();
  const int nslabs = G.wg_slab ? G.wg_nslabs : h->ar.nslabs;
  const int budget = max_ctas > 0 && max_ctas < h->num_sms ? max_ctas : h->num_sms;
  // 128-wide tiles, unless they would leave more than half of the CTAs idle
  int bn_cap = 128, tiles128 = 0;
  for (int i = 0; i < G.n; ++i) tiles128 += ((G.prob(i).M + WG_BM - 1) / WG_BM) * ((G.prob(i).N + 127) / 128) * nslabs;
  if (tiles128 * 2 <= budget) bn_cap = 64;
  // the list holds the problems by the cost of their tiles (rows x MMA width), largest first: see wgrad_tc.cuh
  int order[TC_MAXG], cost[TC_MAXG];
  for (int i = 0; i < G.n; ++i) {
    const int bn = std::min((G.prob(i).N + 15) / 16 * 16, bn_cap);
    cost[i] = (G.prob(i).M > TC_BM ? 2 : 1) * ((bn + 63) / 64);
    order[i] = i;
  }
  std::stable_sort(order, order + G.n, [&](int a, int b) { return cost[a] > cost[b]; });
  int total = 0, bn_max = 16;
  for (int o = 0; o < G.n; ++o) {
    const int i = order[o];
    const GemmProb& s = G.prob(i);
    const TcExtra& x = G.x[i];
    TcProb& p = t.p[o];
    p.M = s.M; p.N = s.N;
    p.bn = std::min((s.N + 15) / 16 * 16, bn_cap);
    if (p.bn > bn_max) bn_max = p.bn;
    p.tiles_m = (s.M + WG_BM - 1) / WG_BM;
    p.tiles_n = (s.N + p.bn - 1) / p.bn;
    p.kblocks[0] = (s.K[0] + TC_BK - 1) / TC_BK;
    p.kB0[0] = x.kB0[0];
    if (!make_map(&p.mapA[0], x.a[0], 64) || !make_map(&p.mapB, x.b, 64)) { c.err = cudaErrorInvalidValue; return; }
    p.ksplit = nslabs;
    p.epi = EPI_PARTIAL;
    if (G.wg_slab) { p.C = G.wg_slab + G.wg_off[i]; p.split_stride = G.wg_stride; }
    else { p.C = h->W() + h->ar.slabs + (s.C - h->buf.grads); p.split_stride = h->ar.slab_stride; }
    p.ldc = s.ldc;
    p.tile_start = total;
    total += p.tiles_m * p.tiles_n * p.ksplit;
  }
  const int planes = t.passes == 3 ? 2 : 1;
  const int stage_b = (bn_max + 63) / 64 * 8192;   // bytes of one B plane per stage: 64-column boxes
  const int stage_bytes = planes * (2 * TC_STAGE_A + stage_b);
  const int stages = std::min(8, (200 * 1024) / stage_bytes);
  const int smem = stages * stage_bytes + 2 * stages * 8 + 1024;
  if (!h->wgrad_attr_done) {
    cudaFuncSetAttribute(tc_gemm_kernel_wgrad<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_gemm_kernel_wgrad<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    h->wgrad_attr_done = true;
  }
  const int grid = std::min(total, budget);
  if (planes == 2) launch_k(tc_gemm_kernel_wgrad<true>, grid, WG_THREADS, smem, c, t, total, stages, stage_b);
  else launch_k(tc_gemm_kernel_wgrad<false>, grid, WG_THREADS, smem, c, t, total, stages, stage_b);
}

// Lower a forward or dgrad group onto wgmma: images instead of fp32 operands, TMA tensor maps, 64 x bn tiles.
// `max_ctas` > 0: issue the group as several launches of at most that many CTAs (one CTA occupies an SM).
static void launch_tc(MlpHandle* h, Group& G, int variant, Ctx& c, int max_ctas = 0) {
  if (variant == V_WGRAD) { launch_tc_wgrad(h, G, c, max_ctas); return; }
  TcGroup& t = h->tc_scratch;
  memset(&t, 0, sizeof(t));
  t.n = G.n;
  t.passes = h->passes();
  const bool b_mn = variant != V_FWD;
  int grid = 0;
  int bn_max = 16;
  for (int i = 0; i < G.n; ++i) {
    const GemmProb& s = G.prob(i);
    const TcExtra& x = G.x[i];
    TcProb& p = t.p[i];
    p.M = s.M; p.N = s.N;
    int bn = (s.N + 15) / 16 * 16;
    if (bn > 256) bn = 256;
    p.bn = bn;
    if (bn > bn_max) bn_max = bn;
    p.tiles_m = (s.M + TC_BM - 1) / TC_BM;
    p.tiles_n = (s.N + bn - 1) / bn;
    for (int sgm = 0; sgm < 2; ++sgm) {
      p.kblocks[sgm] = (s.K[sgm] + TC_BK - 1) / TC_BK;
      p.kB0[sgm] = x.kB0[sgm];
      if (s.K[sgm] > 0 && !make_map(&p.mapA[sgm], x.a[sgm], TC_BM)) { c.err = cudaErrorInvalidValue; return; }
    }
    if (!make_map(&p.mapB, x.b, b_mn ? 64 : bn)) { c.err = cudaErrorInvalidValue; return; }
    p.ksplit = 1;
    p.C = s.C; p.ldc = s.ldc; p.bias = s.bias; p.Zout = s.Zout; p.Zin = s.Zin; p.ldz = s.ldz; p.colsum = s.colsum;
    p.epi = s.epi; p.act = s.act;
    if (x.out.p) {
      p.img = x.out.p; p.img_pitch = x.out.pitch; p.img_plane = x.out.plane;
      if (p.epi == EPI_BIAS_ACT || p.epi == EPI_DACT) p.C = nullptr;  // the next GEMM reads the image; no fp32 copy
    }
    p.tile_start = grid;
    grid += p.tiles_m * p.tiles_n * p.ksplit;
  }
  static unsigned long long* dbg = nullptr;
  const bool debug = getenv("DSACT_TC_DEBUG") != nullptr;
  if (debug && !dbg) cudaMalloc(&dbg, sizeof(unsigned long long) * TC_DBG_SLOTS * 4096);
  if (debug && grid <= 4096) { cudaMemsetAsync(dbg, 0, sizeof(unsigned long long) * TC_DBG_SLOTS * grid, c.s); t.dbg = dbg; }
  const int planes = t.passes == 3 ? 2 : 1;
  const int stage_b = (bn_max + 63) / 64 * 64 * 128;   // bytes of one B plane per stage: the wgmma N (64 multiple) reads that many rows
  int stages = (200 * 1024) / (planes * (TC_STAGE_A + stage_b));
  if (stages > 8) stages = 8;
  const int smem = tc_smem_bytes(stages, planes, stage_b);
  if (!h->tc_attr_done) {
    cudaFuncSetAttribute(tc_gemm_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_gemm_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_gemm_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_gemm_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    h->tc_attr_done = true;
  }
  const int total = grid;
  if (max_ctas > 0 && !debug && total > max_ctas) {  // equal slices, none above the bound
    const int parts = (total + max_ctas - 1) / max_ctas;
    grid = (total + parts - 1) / parts;
  }
  for (int t0 = 0; t0 < total; t0 += grid) {
    t.tile0 = t0;
    const int n = total - t0 < grid ? total - t0 : grid;
    if (t0 > 0) c.launches++;
    if (planes == 2) {
      if (variant == V_FWD) launch_k(tc_gemm_kernel<false, false, true>, n, TC_THREADS, smem, c, t, stages, stage_b);
      else launch_k(tc_gemm_kernel<false, true, true>, n, TC_THREADS, smem, c, t, stages, stage_b);
    } else {
      if (variant == V_FWD) launch_k(tc_gemm_kernel<false, false, false>, n, TC_THREADS, smem, c, t, stages, stage_b);
      else launch_k(tc_gemm_kernel<false, true, false>, n, TC_THREADS, smem, c, t, stages, stage_b);
    }
  }
  grid = total;
  if (debug && t.dbg) {  // per-CTA phase breakdown (ns): setup | first TMA landed | MMA issue done | accumulator ready | epilogue | teardown
    cudaStreamSynchronize(c.s);
    std::vector<unsigned long long> hbuf(TC_DBG_SLOTS * (size_t)grid);
    cudaMemcpy(hbuf.data(), dbg, sizeof(unsigned long long) * TC_DBG_SLOTS * grid, cudaMemcpyDeviceToHost);
    unsigned long long tmin = ~0ull, tmax = 0;
    double ph[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < grid; ++i) {
      const unsigned long long* d = &hbuf[TC_DBG_SLOTS * (size_t)i];
      if (d[0] < tmin) tmin = d[0];
      if (d[6] > tmax) tmax = d[6];
      ph[0] += (double)(d[1] - d[0]); ph[1] += (double)(d[2] - d[1]); ph[2] += (double)(d[3] - d[2]);
      ph[3] += (double)(d[4] - d[3]); ph[4] += (double)(d[5] - d[4]); ph[5] += (double)(d[6] - d[5]);
    }
    fprintf(stderr, "[tc_debug] variant %d grid %d span %.1f us | per-CTA avg ns: setup %.0f, first-load %.0f, mma-issue %.0f, acc-wait %.0f, epilogue %.0f, teardown %.0f\n",
            variant, grid, (tmax - tmin) / 1000.0, ph[0] / grid, ph[1] / grid, ph[2] / grid, ph[3] / grid, ph[4] / grid, ph[5] / grid);
  }
}

static void launch_group(MlpHandle* h, Group& G, int variant, Ctx& c, int max_ctas = 0) {
  if (G.n == 0) return;
  double flops = 0.0;
  for (int i = 0; i < G.n; ++i) flops += 2.0 * G.prob(i).M * G.prob(i).N * ((double)G.prob(i).K[0] + G.prob(i).K[1]);
  if (h->tc()) {
    launch_tc(h, G, variant, c, max_ctas);
    c.done(CLS_GEMM_FWD + variant, flops);
  } else {
    G.g.n = G.n < MAXG ? G.n : MAXG;
    launch_simt(h->num_sms, G.g, variant, c);
    c.done(CLS_GEMM_FWD + variant, flops);
    if (G.n > MAXG) {  // second launch for the overflow
      GemmGroup g2;
      g2.n = G.n - MAXG;
      for (int i = 0; i < g2.n; ++i) g2.p[i] = G.more[i];
      launch_simt(h->num_sms, g2, variant, c);
      c.done(CLS_GEMM_FWD + variant, 0.0);
    }
  }
  c.check();
}

static GemmProb prob_zero() {
  GemmProb p;
  memset(&p, 0, sizeof(p));
  return p;
}

// a [rows, ld] tensor as both lowerings see it
struct Ten {
  float* f = nullptr;
  Img im;
  int ld = 0;   // fp32 row pitch when the tensor is a column range of wider rows (0: contiguous)
};
struct Wt {       // one layer's weights: fp32 [out, in] + image
  const float* f = nullptr;
  const float* bias = nullptr;
  Img im;
};

// forward layer j: out = act(in0 * W[:, :k0]^T + in1 * W[:, k0:k0+k1]^T + b)
static void add_fwd(Group& G, const Net& net, int j, const Wt& w, const Ten& in0, int k0, const Ten& in1, int k1, int kB1,
                    const Ten& out, float* zout, int B, int act) {
  GemmProb p = prob_zero();
  TcExtra x;
  const int in_dim = net.s[j];
  p.A[0] = in0.f; p.lda[0] = k0; p.K[0] = k0; p.B[0] = w.f; p.ldb[0] = in_dim;
  x.a[0] = in0.im;
  if (k1 > 0) {
    p.A[1] = in1.f; p.lda[1] = k1; p.K[1] = k1; p.B[1] = w.f + k0; p.ldb[1] = in_dim;
    x.a[1] = in1.im; x.kB0[1] = kB1;
  }
  x.b = w.im;
  p.M = B; p.N = net.s[j + 1]; p.C = out.f; p.ldc = out.ld ? out.ld : net.s[j + 1];
  p.bias = w.bias;
  const bool last = j == net.L;
  p.epi = last ? EPI_STORE : EPI_BIAS_ACT;
  p.act = act;
  p.Zout = last ? nullptr : zout;
  x.out = last ? Img() : out.im;
  G.push(p, x);
}

// dgrad through layer j, weight columns [col0, col0+ncols): dX = dY * W[:, cols]   (* act'(Zprev), bias-grad colsum)
static void add_dgrad(Group& G, const Net& net, int j, const Wt& w, int col0, int img_col0, int ncols, const Ten& dY,
                      const Ten& dX, const float* Zprev, float* gbias_prev, int B, int act) {
  GemmProb p = prob_zero();
  TcExtra x;
  p.A[0] = dY.f; p.lda[0] = dY.ld ? dY.ld : net.s[j + 1]; p.K[0] = net.s[j + 1];
  p.B[0] = w.f + col0; p.ldb[0] = net.s[j];
  x.a[0] = dY.im;
  x.b = w.im.cols(img_col0, ncols);
  p.M = B; p.N = ncols; p.C = dX.f; p.ldc = ncols;
  if (Zprev) { p.epi = EPI_DACT; p.Zin = Zprev; p.ldz = ncols; p.colsum = gbias_prev; p.act = act; }
  else p.epi = EPI_STORE;
  x.out = dX.im;
  G.push(p, x);
}

// wgrad of layer j, weight columns [col0, col0+ncols): gW[:, cols] += dY^T X
static void add_wgrad(Group& G, const Net& net, int j, float* Gw, int col0, int ncols, const Ten& dY, const Ten& X, int B) {
  GemmProb p = prob_zero();
  TcExtra x;
  p.A[0] = dY.f; p.lda[0] = dY.ld ? dY.ld : net.s[j + 1]; p.K[0] = B;
  p.B[0] = X.f; p.ldb[0] = ncols;
  x.a[0] = dY.im; x.b = X.im;
  p.M = net.s[j + 1]; p.N = ncols; p.C = Gw + col0; p.ldc = net.s[j];
  p.epi = EPI_ATOMIC;
  G.push(p, x);
}

// fp32 -> image conversions (TC modes)
struct ImgBatch {
  ImgGroup g;
  bool overflow = false;
  ImgBatch() { g.n = 0; }
  void add(const float* src, int ld_src, const Img& dst, int rows, int w0, int w1 = 0, int dst1 = 0) {
    if (g.n >= IMG_MAXJ) { overflow = true; return; }
    ImgJob& j = g.j[g.n++];
    memset(&j, 0, sizeof(j));
    j.src = src; j.dst = dst.p; j.rows = rows; j.ld_src = ld_src;
    j.seg_w[0] = w0; j.seg_src0[0] = 0; j.seg_dst0[0] = 0;
    j.seg_w[1] = w1; j.seg_src0[1] = w0; j.seg_dst0[1] = dst1;
    j.pitch = dst.pitch; j.fill_w = w1 > 0 ? dst1 + w1 : w0; j.plane = dst.plane;
  }
  void reserve(const MlpHandle* h, Ctx& c, int jobs) { if (g.n + jobs > IMG_MAXJ) launch(h, c); }   // flush when full
  // `pro` != null: the clears and the device noise ride in the same launch (step_prologue_kernel)
  void launch(const MlpHandle* h, Ctx& c, PrologueArgs* pro = nullptr) {
    if (overflow) { c.err = cudaErrorInvalidValue; return; }
    if (g.n == 0 && !pro) return;
    g.planes = h->passes() == 3 ? 2 : 1;
    int grid = 0;
    for (int i = 0; i < g.n; ++i) {
      g.j[i].block_start = grid;
      long long total = (long long)g.j[i].rows * (g.j[i].pitch / 8);
      int blocks = (int)((total + 255) / 256);
      if (blocks < 1) blocks = 1;
      if (blocks > 2 * h->num_sms) blocks = 2 * h->num_sms;
      grid += blocks;
    }
    if (pro) {
      pro->img_blocks = grid;
      launch_k(step_prologue_kernel, grid + pro->zero_blocks + pro->noise_blocks, 256, 0, c, g, *pro);
    } else {
      launch_k(image_kernel, grid, 256, 0, c, g);
    }
    c.done();
    g.n = 0;
  }
};

static ImgOut img_out(const MlpHandle* h, const ImgSlot& s) {
  ImgOut o;
  o.p = nullptr; o.pitch = 0; o.planes = h->passes() == 3 ? 2 : 1; o.plane = 0;
  if (h->tc() && s.off >= 0) { o.p = reinterpret_cast<__nv_bfloat16*>(h->W() + s.off); o.pitch = s.pitch; o.plane = s.plane; }
  return o;
}
static ImgOut img_out_of(const MlpHandle* h, const Img& i) {
  ImgOut o;
  o.p = i.p; o.pitch = i.p ? i.pitch : 0; o.planes = h->passes() == 3 ? 2 : 1; o.plane = i.p ? i.plane : 0;
  return o;
}


// ---- layer-chain launches (tensor-core modes) -------------------------------------------------------
struct ChainBuild {
  ChainGroup g;
  int grid = 0, stage_b = 16 * 128;
  int b_mn = -1;   // B orientation, one per launch: forward chains K-major, dgrad chains MN-major
  Img w[CH_MAX_PASSES][CH_MAX_LAYERS];   // each layer's weight image (the ping-pong kernel's K-major maps differ)
  double flops = 0.0;
  bool ok = true;
  explicit ChainBuild(int passes) { memset(&g, 0, sizeof(g)); g.passes = passes; }
  ChainPass& begin(const Img& a0, const Img& a1, int M) {
    ChainPass& P = g.p[g.n++];
    P.n_layers = 0; P.M = M; P.tile_start = grid;
    grid += (M + TC_BM - 1) / TC_BM;
    ok = ok && make_map(&P.mapA[0], a0, TC_BM);
    if (a1.p) ok = ok && make_map(&P.mapA[1], a1, TC_BM);
    return P;
  }
  ChainLayer& layer(ChainPass& P, const Img& wimg, bool b_mn, int N, int K0, int K1, int kB1) {
    ChainLayer& L = P.L[P.n_layers++];
    L.N = N; L.ldc = N; L.bn = (N + 15) / 16 * 16;
    const int o = b_mn ? 1 : 0;
    if (this->b_mn >= 0 && this->b_mn != o) ok = false;   // the kernel takes one B orientation per launch
    this->b_mn = o;
    L.kblocks[0] = (K0 + TC_BK - 1) / TC_BK; L.kblocks[1] = (K1 + TC_BK - 1) / TC_BK;
    L.kB0[0] = 0; L.kB0[1] = kB1;
    ok = ok && make_map(&L.mapB, wimg, b_mn ? 64 : L.bn);
    w[&P - g.p][P.n_layers - 1] = wimg;
    const int sb = (L.bn + 63) / 64 * 8192;   // the wgmma N (64 multiple) reads that many rows of a K-major tile
    if (sb > stage_b) stage_b = sb;
    flops += 2.0 * P.M * N * ((double)K0 + K1);
    return L;
  }
  // the bf16 image of layer L's result (p null: none), stored by TMA up to column (N + 7) / 8 * 8 and row im.rows
  void image(ChainLayer& L, Img im) {
    if (!im.p) return;
    im.width = (L.N + 7) / 8 * 8;
    L.img = 1;
    ok = ok && make_map(&L.mapImg, im, TC_BM);
  }
};

// The layer-chain kernel of a launch: the column split (tc_chain_kernel, one 64-row tile per CTA) when its grid fits one
// wave, the ping-pong kernel (tc_pingpong_kernel, two tiles per CTA) when it needs more.  `tiling` (tests): 0 / 1 forces
// the column split / the ping-pong kernel, -1 selects by shape.
enum { CHAIN_BY_SHAPE = -1, CHAIN_COLUMN_SPLIT = 0, CHAIN_PINGPONG = 1 };

// The epilogue kind of a layer's full tiles in the ping-pong kernel (gemm_tc.cuh): a forward hidden layer (bias, GELU or
// ReLU, with or without Zout) or a dgrad hidden layer (with or without column sums), N a multiple of 64 (every column
// of the accumulator is an output) and 8-byte aligned inputs and act' stores.  Anything else (heads, C stores, the other
// activations) keeps the runtime body.
static int chain_epi_kind(const ChainLayer& L) {
  const auto al8 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; };
  if (L.N % 64 != 0 || L.C) return EK_RUNTIME;
  if (L.epi == EPI_BIAS_ACT && L.bias && al8(L.bias) && (L.act == ACT_GELU || L.act == ACT_RELU) &&
      (!L.Zout || (al8(L.Zout) && L.ldc == L.N))) {
    if (L.act == ACT_GELU) return L.Zout ? EK_GELU_Z : EK_GELU;
    return L.Zout ? EK_RELU_Z : EK_RELU;
  }
  if (L.epi == EPI_DACT && L.Zin && al8(L.Zin)) return L.colsum ? EK_DACT_SUM : EK_DACT;
  return EK_RUNTIME;
}

static void launch_chain(MlpHandle* h, ChainBuild& cb, int cls, Ctx& c, int tiling = CHAIN_BY_SHAPE) {
  if (cb.g.n == 0) return;
  for (int i = 0; i < cb.g.n; ++i)
    for (int j = 0; j < cb.g.p[i].n_layers; ++j) {
      ChainLayer& L = cb.g.p[i].L[j];
      if (L.ldc != L.N && L.Zout) cb.ok = false;   // Zout rows are N apart
      L.kind = chain_epi_kind(L);
    }
  if (!cb.ok) { c.err = cudaErrorInvalidValue; return; }
  static unsigned long long* dbg = nullptr;
  const bool debug = getenv("DSACT_TC_DEBUG") != nullptr;
  if (debug && !dbg) cudaMalloc(&dbg, sizeof(unsigned long long) * TC_DBG_SLOTS * 4096);
  if (debug && cb.grid <= 4096) { cudaMemsetAsync(dbg, 0, sizeof(unsigned long long) * TC_DBG_SLOTS * cb.grid, c.s); cb.g.dbg = dbg; }
  const int planes = cb.g.passes == 3 ? 2 : 1;
  const int stages = planes == 2 ? 2 : 4;   // layer 0's A ring lives in the 4-k-block operand buffer
  const int smem = chain_smem_bytes(stages, planes, cb.stage_b);
  const int pp_smem = pp_smem_bytes(stages, planes);
  if (!h->chain_attr_done) {
    cudaFuncSetAttribute(tc_chain_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_chain_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_chain_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_chain_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(tc_pingpong_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    cudaFuncSetAttribute(tc_pingpong_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    cudaFuncSetAttribute(tc_pingpong_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    cudaFuncSetAttribute(tc_pingpong_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    h->chain_attr_done = true;
  }
  if (tiling == CHAIN_BY_SHAPE) {   // the column split's resident CTAs on the device
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tc_chain_kernel<true, false>, CH_THREADS, smem);
    if (e != cudaSuccess) { c.err = e; return; }
    tiling = cb.grid > std::max(per_sm, 1) * h->num_sms ? CHAIN_PINGPONG : CHAIN_COLUMN_SPLIT;
  }
  if (tiling == CHAIN_PINGPONG) {
    // K-major weight maps load one column half (min(bn, 128) weight rows) per ring stage
    for (int i = 0; i < cb.g.n && !cb.b_mn; ++i)
      for (int j = 0; j < cb.g.p[i].n_layers; ++j)
        if (cb.g.p[i].L[j].bn > PP_HALF && !make_map(&cb.g.p[i].L[j].mapB, cb.w[i][j], PP_HALF)) { c.err = cudaErrorInvalidValue; return; }
    int ctas = 0;
    for (int i = 0; i < cb.g.n; ++i) ctas += (cb.g.p[i].M + 2 * TC_BM - 1) / (2 * TC_BM);
    if (planes == 2) {
      if (cb.b_mn) launch_k(tc_pingpong_kernel<true, true>, ctas, PP_THREADS, pp_smem, c, cb.g, stages);
      else launch_k(tc_pingpong_kernel<true, false>, ctas, PP_THREADS, pp_smem, c, cb.g, stages);
    } else {
      if (cb.b_mn) launch_k(tc_pingpong_kernel<false, true>, ctas, PP_THREADS, pp_smem, c, cb.g, stages);
      else launch_k(tc_pingpong_kernel<false, false>, ctas, PP_THREADS, pp_smem, c, cb.g, stages);
    }
  } else if (planes == 2) {
    if (cb.b_mn) launch_k(tc_chain_kernel<true, true>, cb.grid, CH_THREADS, smem, c, cb.g, stages, cb.stage_b);
    else launch_k(tc_chain_kernel<true, false>, cb.grid, CH_THREADS, smem, c, cb.g, stages, cb.stage_b);
  } else {
    if (cb.b_mn) launch_k(tc_chain_kernel<false, true>, cb.grid, CH_THREADS, smem, c, cb.g, stages, cb.stage_b);
    else launch_k(tc_chain_kernel<false, false>, cb.grid, CH_THREADS, smem, c, cb.g, stages, cb.stage_b);
  }
  c.done(cls, cb.flops);
  c.check();
  if (debug && cb.g.dbg) {
    cudaStreamSynchronize(c.s);
    std::vector<unsigned long long> hbuf(TC_DBG_SLOTS * (size_t)cb.grid);
    cudaMemcpy(hbuf.data(), dbg, sizeof(unsigned long long) * TC_DBG_SLOTS * cb.grid, cudaMemcpyDeviceToHost);
    unsigned long long tmin = ~0ull, tmax = 0;
    for (int i = 0; i < cb.grid; ++i) {
      const unsigned long long* d = &hbuf[TC_DBG_SLOTS * (size_t)i];
      if (d[0] < tmin) tmin = d[0];
      if (d[6] > tmax) tmax = d[6];
    }
    fprintf(stderr, "[chain_debug] class %d passes %d grid %d span %.1f us %s\n", cls, cb.g.n, cb.grid, (tmax - tmin) / 1000.0,
            tiling == CHAIN_PINGPONG ? "ping-pong" : "column split");
    // first CTA of every pass (ping-pong: both of its tiles, one per warpgroup): per-layer timeline relative to the CTA's
    // start (us)
    for (int pi = 0; pi < cb.g.n; ++pi) {
      const int t0 = cb.g.p[pi].tile_start, tend = pi + 1 < cb.g.n ? cb.g.p[pi + 1].tile_start : cb.grid;
      const unsigned long long* d0 = &hbuf[TC_DBG_SLOTS * (size_t)t0];
      for (int t = t0; t < (tiling == CHAIN_PINGPONG ? std::min(t0 + 2, tend) : t0 + 1); ++t) {
        const unsigned long long* d = &hbuf[TC_DBG_SLOTS * (size_t)t];
        fprintf(stderr, "  pass %d tile %d: setup %.1f first-load %.1f |", pi, t - t0, (d[1] - d0[0]) / 1e3, (d[2] - d0[0]) / 1e3);
        for (int j = 0; j < cb.g.p[pi].n_layers; ++j)
          fprintf(stderr, " L%d mma-done %.1f epilogue %.1f operand %.1f |", j, (d[8 + 3 * j] - d0[0]) / 1e3,
                  (d[9 + 3 * j] - d0[0]) / 1e3, (d[10 + 3 * j] - d0[0]) / 1e3);
        fprintf(stderr, " end %.1f\n", (d[6] - d0[0]) / 1e3);
      }
    }
  }
}

// Where one pass of a chain reads and writes, resolved to pointers and images: per layer j the weight image, and per hidden
// layer j the act'(z_j) store / load (null: none), the image of its output (p null: none) and, in dgrad, its bias
// gradient (null: none).
struct ChainIo {
  Img w[DSACT_MAX_HIDDEN + 1];
  float* z[DSACT_MAX_HIDDEN] = {};
  Img img[DSACT_MAX_HIDDEN];
  float* colsum[DSACT_MAX_HIDDEN] = {};
};

// forward chain of one pass: out = head(act(...act(in W_0^T + b_0)...))
static ChainPass& chain_fwd_layers(ChainBuild& cb, const Net& net, const float* Wbase, const ChainIo& io, const Img& in0, int k0,
                                   const Img& in1, int k1, int kB1, int B, int act, float* out, int out_ld = 0) {
  ChainPass& P = cb.begin(in0, in1, B);
  for (int j = 0; j <= net.L; ++j) {
    ChainLayer& L = j == 0 ? cb.layer(P, io.w[0], false, net.s[1], k0, k1, kB1) : cb.layer(P, io.w[j], false, net.s[j + 1], net.s[j], 0, 0);
    const bool last = j == net.L;
    L.epi = last ? EPI_STORE : EPI_BIAS_ACT;
    L.act = act;
    L.bias = Wbase + net.b[j];
    if (last) { L.C = out; if (out_ld) L.ldc = out_ld; }   // only a head layer takes a pitch: the epilogue indexes Zout with
                                                           // ldc as well, and a head layer has no Zout
    else {
      L.Zout = io.z[j];
      cb.image(L, io.img[j]);
    }
  }
  return P;
}

// dgrad chain of one pass: dz_{j-1} = (dz_j W_j) (.) act'(z_{j-1}) for j = L..1 (+ dAct = dz_0 W_0[:, act columns])
static ChainPass& chain_dgrad_layers(ChainBuild& cb, const Net& net, const ChainIo& io, const Img& dout, int B, int act,
                                     float* dact_out, int act_col_img, int act_cols) {
  const Img none;
  ChainPass& P = cb.begin(dout, none, B);
  for (int j = net.L; j >= 1; --j) {
    ChainLayer& L = cb.layer(P, io.w[j], true, net.s[j], net.s[j + 1], 0, 0);   // image rows = reduction, width = inputs
    L.epi = EPI_DACT; L.act = act;
    L.Zin = io.z[j - 1];
    L.colsum = io.colsum[j - 1];
    cb.image(L, io.img[j - 1]);
  }
  if (dact_out) {
    ChainLayer& L = cb.layer(P, io.w[0].cols(act_col_img, act_cols), true, act_cols, net.s[1], 0, 0);
    L.epi = EPI_STORE; L.C = dact_out;
  }
  return P;
}

// ---- the network passes of a step and their two lowerings ----------------------------------------------------------
// A network instance of the step (q_k and q'_k for k < nq, pi, pi'): its fp32 parameters (in params; in targets for q'_k
// and pi'), gradients (null: a target network), the weight-image slot of every layer and the hidden activation
struct NetInst { const Net* net; const float* P; float* G; const ImgSlot* wimg; int act; };
struct NetInsts { NetInst q[2], qt[2], pi, pit, pi_ls, pit_ls; };   // pi_ls / pit_ls: the log_std networks (mlp_separated)

static NetInsts net_insts(const MlpHandle* h) {
  const Net &q = h->q, &pi = h->pi;
  const int nq = h->nq();
  float *P = h->buf.params, *T = h->buf.targets, *G = h->buf.grads;   // flat layout [q_0 .. q_{nq-1} | pi | log_alpha]
  NetInsts I = {};
  for (int k = 0; k < nq; ++k) {
    I.q[k] = NetInst{&q, P + k * q.n, G + k * q.n, h->ar.i_wq[k], h->cfg.act_q};
    I.qt[k] = NetInst{&q, T + k * q.n, nullptr, h->ar.i_wq[2 + k], h->cfg.act_q};
  }
  const PiSpan sp = h->span();
  const int64_t mean = nq * q.n + sp.mean, ls = nq * q.n + sp.ls;
  I.pi = NetInst{&pi, P + mean, G + mean, h->ar.i_wpi[0], h->cfg.act_pi};
  I.pit = NetInst{&pi, T + mean, nullptr, h->ar.i_wpi[1], h->cfg.act_pi};
  if (h->cfg.policy_std == DSACT_STD_SEPARATED) {
    I.pi_ls = NetInst{&pi, P + ls, G + ls, h->ar.i_wpi[2], h->cfg.act_pi};
    I.pit_ls = NetInst{&pi, T + ls, nullptr, h->ar.i_wpi[3], h->cfg.act_pi};
  }
  return I;
}

// A forward pass.  Layer 0 reads in0 (k0 columns) and, for a critic, the action segment in1 (k1 columns, at column kB1 of
// the weight image).  Per hidden layer j, act'(z_j) goes to slot z[j] (z null: nowhere) and the activation to slots hf[j]
// (fp32) / hi[j] (image); a layer chain writes the activations only if they must outlive the pass (`keep`: the weight
// gradients read them).
struct FwdPass {
  NetInst n;
  Ten in0, in1;
  int k0, k1, kB1;
  const int64_t *z, *hf;
  const ImgSlot* hi;
  bool keep;
  float* out;
  int out_ld;   // row pitch of `out` when the pass writes its columns of wider rows (0: contiguous)
};

// The backward of forward pass f: dL/d(output) in slots dout / dout_img, dL/dz_j in slots dz[j] / dz_img[j].  `grads`: it
// adds the bias gradients and, from f's layer inputs, the weight gradients of f's network (a layer chain writes the dz
// images only then).  dact != null: dL/d(f's action segment) goes there.
struct BwdPass {
  FwdPass f;
  int64_t dout;
  int dout_ld;   // row pitch of the fp32 dL/d(output) when it is a column range of wider rows (0: contiguous)
  ImgSlot dout_img;
  const int64_t* dz;
  const ImgSlot* dz_img;
  bool grads;
  float* dact;
};

// The passes of one step in launch order.  Wave A: pi(s), pi'(s'), Q_k(s,a); wave B (it reads a~ ~ pi(s), a' ~ pi'(s')):
// Q'_k(s',a'), Q_k(s,a~); the critics' backward: Q_k(s,a) with gradients, Q_k(s,a~) with dL/da~; the policy's: pi(s).
// mlp_separated: pi and pi' are two passes each, the mean network into columns [0, A) of the [B, 2A] logits and the
// log_std network into [A, 2A), and the policy's backward two.  parameter: the mean network alone, into columns [0, A).
struct StepPasses {
  NetInsts I;
  FwdPass a[6], b[4];
  BwdPass q[4], pi[2];
  int na = 0, nb = 0, nqb = 0, npb = 0;
};

static Ten ten(const MlpHandle* h, const float* f, const ImgSlot& s, int B) { return Ten{const_cast<float*>(f), h->img(s, B)}; }
static Wt weight(const MlpHandle* h, const NetInst& n, int j) {   // layer j of instance n
  return Wt{n.P + n.net->w[j], n.P + n.net->b[j], h->img(n.wimg[j], n.net->s[j + 1])};
}

// the passes of one update on the rows `bt`, whose images are those of input set `set`
static StepPasses step_passes(const MlpHandle* h, const dsact_batch& bt, int set) {
  const Arena& ar = h->ar;
  float* W = h->W();
  const int B = bt.batch, O = h->cfg.obs_dim, A = h->cfg.act_dim;
  StepPasses s;
  s.I = net_insts(h);
  const Ten obs{const_cast<float*>(bt.obs), h->input_img(set, 0, B)}, obs2{const_cast<float*>(bt.obs2), h->input_img(set, 1, B)};
  const Ten act{const_cast<float*>(bt.act), h->input_img(set, 2, B)};
  const Ten new_act = ten(h, W + ar.new_act, ar.i_new_act, B), act2 = ten(h, W + ar.act2, ar.i_act2, B);
  // the arena holds critic pass Q_k(s,a) at slot k, Q'_k(s',a') at 2 + k and Q_k(s,a~) at 4 + k
  auto critic = [&](const NetInst& n, int p, const Ten& in, const Ten& a, bool store_z, bool keep) {
    return FwdPass{n, in, a, O, A, ar.kpad_q0, store_z ? ar.zQ[p] : nullptr, ar.hQ[p], ar.i_hQ[p], keep, W + ar.outQ[p], 0};
  };
  auto critic_bwd = [&](const FwdPass& f, int p, bool grads, float* dact) {
    return BwdPass{f, ar.dOut[p], 0, ar.i_dOut[p], ar.dzQ[p], ar.i_dzQ[p], grads, dact};
  };
  const int pstd = h->cfg.policy_std;
  const int ld = pstd == DSACT_STD_SHARED ? 0 : 2 * A;   // an A-wide head writes its columns of the [B, 2A] logits
  const FwdPass pi{s.I.pi, obs, Ten(), O, 0, 0, ar.zP, ar.hP, ar.i_hP, true, W + ar.logitsP, ld};
  const FwdPass pit{s.I.pit, obs2, Ten(), O, 0, 0, nullptr, ar.hT, ar.i_hT, false, W + ar.logitsT, ld};
  s.pi[s.npb++] = BwdPass{pi, ar.dlogits, ld, ar.i_dlogits, ar.dzP, ar.i_dzP, true, nullptr};
  if (pstd == DSACT_STD_SEPARATED) {
    const FwdPass pi_ls{s.I.pi_ls, obs, Ten(), O, 0, 0, ar.zL, ar.hL, ar.i_hL, true, W + ar.logitsP + A, ld};
    s.a[s.na++] = pi;
    s.a[s.na++] = pi_ls;
    s.a[s.na++] = pit;
    s.a[s.na++] = FwdPass{s.I.pit_ls, obs2, Ten(), O, 0, 0, nullptr, ar.hLT, ar.i_hLT, false, W + ar.logitsT + A, ld};
    s.pi[s.npb++] = BwdPass{pi_ls, ar.dlogits + A, ld, ar.i_dlogits_ls, ar.dzL, ar.i_dzL, true, nullptr};
  } else {
    s.a[s.na++] = pi;
    s.a[s.na++] = pit;
  }
  const int nq = h->nq();
  for (int k = 0; k < nq; ++k) {
    const FwdPass f = critic(s.I.q[k], k, obs, act, true, true);
    s.a[s.na++] = f;
    s.q[s.nqb++] = critic_bwd(f, k, true, nullptr);
  }
  for (int k = 0; k < nq; ++k) s.b[s.nb++] = critic(s.I.qt[k], 2 + k, obs2, act2, false, false);
  for (int k = 0; k < nq; ++k) {
    const FwdPass f = critic(s.I.q[k], 4 + k, obs, new_act, true, false);
    s.b[s.nb++] = f;
    s.q[s.nqb++] = critic_bwd(f, 4 + k, false, W + ar.dAct[k]);
  }
  return s;
}

// a pass's weight images and, per hidden layer, its act'(z) slot and output image (null slots: none)
static ChainIo chain_io(const MlpHandle* h, const NetInst& n, int B, const int64_t* z_off, const ImgSlot* himg) {
  ChainIo io;
  float* W = h->W();
  const Net& net = *n.net;
  for (int j = 0; j <= net.L; ++j) io.w[j] = h->img(n.wimg[j], net.s[j + 1]);
  for (int j = 0; j < net.L; ++j) {
    if (z_off) io.z[j] = W + z_off[j];
    if (himg) io.img[j] = h->img(himg[j], B);
  }
  return io;
}

// One wave of forward passes: one layer-chain launch (each CTA runs a 64-row block through every layer of its pass), or
// one GEMM group per layer depth
static void enqueue_fwd(MlpHandle* h, const FwdPass* ps, int n, int B, Ctx& c) {
  float* W = h->W();
  if (h->fused()) {   // a launch carries CH_MAX_PASSES passes: the six of mlp_separated's wave A go out as the four of the
                      // policies, then the critics'
    for (int i0 = 0; i0 < n; i0 += CH_MAX_PASSES) {
      ChainBuild cb(h->passes());
      for (int i = i0; i < n && i < i0 + CH_MAX_PASSES; ++i) {
        const FwdPass& p = ps[i];
        chain_fwd_layers(cb, *p.n.net, p.n.P, chain_io(h, p.n, B, p.z, p.keep ? p.hi : nullptr), p.in0.im, p.k0, p.in1.im, p.k1,
                         p.kB1, B, p.n.act, p.out, p.out_ld);
      }
      launch_chain(h, cb, CLS_GEMM_FWD, c);
    }
    return;
  }
  for (int j = 0; j <= DSACT_MAX_HIDDEN; ++j) {
    Group G;
    for (int i = 0; i < n; ++i) {
      const FwdPass& p = ps[i];
      const Net& net = *p.n.net;
      if (j > net.L) continue;
      const bool last = j == net.L;
      const Ten out = last ? Ten{p.out, Img(), p.out_ld} : ten(h, W + p.hf[j], p.hi[j], B);
      float* z = last || !p.z ? nullptr : W + p.z[j];
      const Wt w = weight(h, p.n, j);
      if (j == 0) add_fwd(G, net, 0, w, p.in0, p.k0, p.in1, p.k1, p.kB1, out, z, B, p.n.act);
      else add_fwd(G, net, j, w, ten(h, W + p.hf[j - 1], p.hi[j - 1], B), net.s[j], Ten(), 0, 0, out, z, B, p.n.act);
    }
    launch_group(h, G, V_FWD, c);
  }
}

// dL/d(output of layer j) of a backward pass
static Ten bwd_dy(const MlpHandle* h, const BwdPass& p, int j, int B) {
  if (j < p.f.n.net->L) return ten(h, h->W() + p.dz[j], p.dz_img[j], B);
  Ten t = ten(h, h->W() + p.dout, p.dout_img, B);
  t.ld = p.dout_ld;
  return t;
}

// The dgrad of a list of backward passes, top layer down: one layer-chain launch (dz stays on chip between layers), or one
// GEMM group per layer.  Returns true for the chain.  The chain also computes dL/d(action); the per-layer lowering leaves
// those problems in `act_cols` for the caller to launch.
static bool enqueue_dgrad(MlpHandle* h, const BwdPass* ps, int n, int B, Ctx& c, Group& act_cols) {
  float* W = h->W();
  if (h->fused()) {
    ChainBuild cb(h->passes());
    for (int i = 0; i < n; ++i) {
      const BwdPass& p = ps[i];
      const NetInst& ni = p.f.n;
      ChainIo io = chain_io(h, ni, B, p.f.z, p.grads ? p.dz_img : nullptr);
      for (int j = 0; j < ni.net->L && p.grads; ++j) io.colsum[j] = ni.G + ni.net->b[j];
      chain_dgrad_layers(cb, *ni.net, io, h->img(p.dout_img, B), B, ni.act, p.dact, p.f.kB1, p.f.k1);
    }
    launch_chain(h, cb, CLS_GEMM_DGRAD, c);
    return true;
  }
  for (int j = DSACT_MAX_HIDDEN; j >= 0; --j) {
    Group gd;   // (stays empty at j = 0)
    for (int i = 0; i < n; ++i) {
      const BwdPass& p = ps[i];
      const NetInst& ni = p.f.n;
      const Net& net = *ni.net;
      if (j > net.L) continue;
      const Wt w = weight(h, ni, j);
      if (j > 0)
        add_dgrad(gd, net, j, w, 0, 0, net.s[j], bwd_dy(h, p, j, B), ten(h, W + p.dz[j - 1], p.dz_img[j - 1], B), W + p.f.z[j - 1],
                  p.grads ? ni.G + net.b[j - 1] : nullptr, B, ni.act);
      else if (p.dact)
        add_dgrad(act_cols, net, 0, w, p.f.k0, p.f.kB1, p.f.k1, bwd_dy(h, p, 0, B), Ten{p.dact}, nullptr, nullptr, B, 0);
    }
    launch_group(h, gd, V_DGRAD, c);
  }
  return false;
}

// The weight-gradient problems of the backward passes with `grads`, layers top down (layer 0: one per input segment)
static void add_wgrads(Group& gw, const MlpHandle* h, const BwdPass* ps, int n, int B) {
  for (int j = DSACT_MAX_HIDDEN; j >= 0; --j)
    for (int i = 0; i < n; ++i) {
      const BwdPass& p = ps[i];
      const Net& net = *p.f.n.net;
      if (!p.grads || j > net.L) continue;
      float* g = p.f.n.G + net.w[j];
      const Ten dy = bwd_dy(h, p, j, B);
      if (j > 0) add_wgrad(gw, net, j, g, 0, net.s[j], dy, ten(h, h->W() + p.f.hf[j - 1], p.f.hi[j - 1], B), B);
      else add_wgrad(gw, net, 0, g, 0, p.f.k0, dy, p.f.in0, B);
      if (j == 0 && p.f.k1 > 0) add_wgrad(gw, net, 0, g, p.f.k0, p.f.k1, dy, p.f.in1, B);
    }
}

// `branch` on the side stream (or on `on`), after all that c.s holds so far; the caller joins it by waiting on `join`
template <typename F>
static void fork_branch(Ctx& c, cudaEvent_t fork, cudaEvent_t join, F branch, cudaStream_t on = nullptr) {
  if (!on) on = c.side;
  cudaEventRecord(fork, c.s);
  cudaStreamWaitEvent(on, fork, 0);
  Ctx cs{on, 0, cudaSuccess};
  cs.pdl = c.pdl;
  branch(cs);
  cudaEventRecord(join, on);
  c.launches += cs.launches;
  if (cs.err != cudaSuccess && c.err == cudaSuccess) c.err = cs.err;
}

static unsigned long long dp_timeout_ns() {
  static const unsigned long long t =
      (unsigned long long)(getenv("DSACT_DP_TIMEOUT_MS") ? atoll(getenv("DSACT_DP_TIMEOUT_MS")) : 10000) * 1000000ull;
  return t;
}
// two-shot gradient exchange (dp_peer.cuh) from 6 ranks up, one-shot below (fewer barriers).  Replicas stay bit-identical
// in both variants.
static bool dp_two_shot(const DpPeer& dp) { return dp.comm.world >= 6; }

// apply_kernel<2>'s view of the exchange: the reduced block in this rank's own memory once every rank's kind-2 flag is
// here (two-shot), or every rank's block, summed in rank order (one-shot)
static void dp_apply_args(const DpPeer& dp, ApplyArgs& a) {
  if (dp_two_shot(dp)) {
    a.dp_world = 1;
    a.dp_grads[0] = dp.buf + DP_GRADS_OFF + dp.npad();
    a.dp_own = dp.buf; a.dp_wait_world = dp.comm.world;
  } else {
    a.dp_world = dp.comm.world;
    for (int r = 0; r < dp.comm.world; ++r) a.dp_grads[r] = dp.comm.peer[r] + DP_GRADS_OFF;
  }
}

// ---- the step kernels both engines launch ---------------------------------------------------------------------------
// They read the shell's arena slots and hyperparameters.  What only the MLP engine has (the bf16 images its tensor-core
// GEMMs read) comes in as ImgOut arguments; the head-wise engine passes NO_IMG.
static const ImgOut NO_IMG{nullptr, 0, 1, 0};

static AdamHyper adam_hyper(const dsact_handle* h) {
  const StepHyper& p = h->hyper;
  return AdamHyper{p.lr_q, p.lr_pi, p.lr_alpha, p.adam_beta1, p.adam_beta2};
}
static StepScalars step_scalars(const dsact_handle* h, int64_t global_batch) {
  StepScalars sc;
  sc.tau_b = (float)h->hyper.tau_b; sc.alpha_fixed = (float)h->hyper.alpha_fixed;
  sc.inv_global_batch = (float)(1.0 / (double)global_batch);
  sc.auto_alpha = h->hyper.auto_alpha; sc.log_alpha = h->buf.params + h->n_params - 1;   // log_alpha is the last parameter
  return sc;
}
// the caller's noise, or the arena's device-noise slots
static dsact_noise step_noise(const dsact_handle* h, const dsact_noise* nz) {
  const float* W = h->W();
  return nz ? *nz : dsact_noise{W + h->slot.eps1, W + h->slot.eps2, W + h->slot.z3, W + h->slot.z4};
}

static int begin_step_blocks(const dsact_handle* h) {
  int blocks = (int)((h->n_params / 4 + 255) / 256); if (blocks > 2 * h->num_sms) blocks = 2 * h->num_sms; if (blocks < 1) blocks = 1;
  return blocks;
}
// accumulator clears and the flat gradient memset
static void enqueue_begin_step(const dsact_handle* h, Ctx& c) {
  launch_k(begin_step_kernel, begin_step_blocks(h), 256, 0, c, h->buf.state, h->buf.grads, (long long)h->n_params);
  c.done();
}

static int noise_blocks(int B, int A) {   // one thread per pair of draws
  const int total = (B * A + 1) / 2 * 2 + (B + 1) / 2 * 2;
  const int blocks = (total / 2 + 255) / 256;
  return blocks < 1 ? 1 : blocks;
}
// device noise into the arena; the counter it reads is stepped by sample_kernel, once every reader of this step has run
static void enqueue_noise(const dsact_handle* h, int B, Ctx& c) {
  const StepSlots& s = h->slot;
  float* W = h->W();
  launch_k(noise_kernel, noise_blocks(B, h->act_dim), 256, 0, c, W + s.eps1, W + s.eps2, W + s.z3, W + s.z4, B, h->act_dim, h->seed,
           h->buf.state);
  c.done();
}

// The per-row arrays the sampling, loss and policy-gradient kernels read and write, and where they add their output-bias
// gradients.  The steps fill it from the arena slots (step_rows); dsact_test_rows from caller buffers.  Indices follow
// StepSlots: out_q[p] is pass p (Q_k(s,a) = k, Q'_k(s',a') = 2 + k, Q_k(s,a~) = 4 + k; DSAC_V1: k = 0 only).
struct RowIo {
  const float *logits[2], *eps[2];   // pi(s), pi'(s') outputs (mean | log_std) [B,2A]; their noise [B,A]
  float *act[2], *logp[2];           // a~, a' [B,A]; logp_new, logp2 [B] (written by sample, read by the losses)
  const float *rew, *done, *z3, *z4;
  const float* out_q[6];             // [B,2] (mean, raw std)
  float *d_out_q[2], *d_out_qa[2];   // dL/d(mean, raw std) of Q_k(s,a) and of Q_k(s,a~)
  const float* d_act[2];             // dL/da~ through critic k [B,A]; d_act[1] null: one critic (policy_grad_kernel<1>)
  float* d_logits;                   // [B,2A]
  // output-bias gradients (+=): gbias_q[k] critic k's mean; gbias_q_raw[k] its std output, or null for the element after
  // gbias_q[k] (one two-output layer); gbias_pi the policy's mean (the whole (mean | log_std) row when gbias_ls is null)
  float *gbias_q[2], *gbias_q_raw[2], *gbias_pi, *gbias_ls;
  ImgOut img_act[2], img_q[2], img_qa[2], img_dlogits;   // bf16 images (NO_IMG: none)
  // split_dlogits: img_dlogits is [B, A], the mean half alone, and the log_std half goes to img_dlogits_ls [B, A] (NO_IMG: a
  // log_std row, which no GEMM reads); otherwise img_dlogits is [B, 2A]
  bool split_dlogits;
  ImgOut img_dlogits_ls;
};
// the step's row arrays: the arena slots, the minibatch `bt` and the noise `nz`; no bias-gradient targets and no images
static RowIo step_rows(const dsact_handle* h, const dsact_batch& bt, const dsact_noise& nz) {
  const StepSlots& s = h->slot;
  float* W = h->W();
  RowIo io;
  memset(&io, 0, sizeof(io));
  io.logits[0] = W + s.logitsP; io.logits[1] = W + s.logitsT;
  io.eps[0] = nz.eps1; io.eps[1] = nz.eps2;
  io.act[0] = W + s.new_act; io.act[1] = W + s.act2;
  io.logp[0] = W + s.logp_new; io.logp[1] = W + s.logp2;
  io.rew = bt.rew; io.done = bt.done; io.z3 = nz.z3; io.z4 = nz.z4;
  for (int p = 0; p < 6; ++p) io.out_q[p] = s.outQ[p] < 0 ? nullptr : W + s.outQ[p];
  for (int k = 0; k < 2; ++k) {
    io.d_out_q[k] = s.dOut[k] < 0 ? nullptr : W + s.dOut[k];
    io.d_out_qa[k] = s.dOut[4 + k] < 0 ? nullptr : W + s.dOut[4 + k];
    io.d_act[k] = s.dAct[k] < 0 ? nullptr : W + s.dAct[k];   // DSAC_V1 on the MLP engine: no second action-gradient slot
  }
  io.d_logits = W + s.dlogits;
  io.img_act[0] = io.img_act[1] = io.img_q[0] = io.img_q[1] = io.img_qa[0] = io.img_qa[1] = io.img_dlogits = io.img_dlogits_ls = NO_IMG;
  return io;
}
// a launch's blocks: the step's count `natural`, or at most `max_blocks` (> 0, dsact_test_rows / dsact_test_apply) so that
// few rows take several grid-stride trips
static int capped(int natural, int max_blocks) { return max_blocks > 0 && natural > max_blocks ? max_blocks : natural; }

// rsample of both policies (utils/act_distribution_cls.py:44-54); also sums the critics' std over the rows (DSAC_V1: of
// its one critic, and its own logged policy statistics)
static void enqueue_sample(const dsact_handle* h, const RowIo& io, int B, bool advance_rng, Ctx& c, int max_blocks = 0) {
  const StepHyper& p = h->hyper;
  SampleArgs a;
  for (int k = 0; k < 2; ++k) {
    a.logits[k] = io.logits[k]; a.eps[k] = io.eps[k]; a.act[k] = io.act[k]; a.logp[k] = io.logp[k]; a.img[k] = io.img_act[k];
  }
  a.hi = h->buf.act_high; a.lo = h->buf.act_low; a.state = h->buf.state;
  a.B = B; a.A = h->act_dim; a.min_log_std = (float)p.min_log_std; a.max_log_std = (float)p.max_log_std; a.gauss = p.act_dist;
  a.out_q[0] = io.out_q[0]; a.out_q[1] = io.out_q[h->v1 ? 0 : 1];
  a.advance_rng = advance_rng ? 1 : 0;
  a.v1_stats = h->v1 ? 1 : 0;
  a.oa = h->oa;
  int blocks = (B + 7) / 8; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
  launch_k(h->outact() ? sample_kernel<true> : sample_kernel<false>, dim3(capped(blocks, max_blocks), 2), 256, 0, c, a);
  c.done();
}

// the DSAC-T losses and the gradients of the critics' outputs
static void enqueue_loss(const dsact_handle* h, const RowIo& io, int B, const StepScalars& sc, Ctx& c, int max_blocks = 0) {
  LossArgs a;
  a.sc = sc;
  a.rew = io.rew; a.done = io.done; a.z3 = io.z3; a.z4 = io.z4;
  a.logp2 = io.logp[1]; a.logp_new = io.logp[0];
  for (int k = 0; k < 2; ++k) {
    a.out_q[k] = io.out_q[k]; a.out_qt[k] = io.out_q[2 + k]; a.out_qa[k] = io.out_q[4 + k];
    a.d_out_q[k] = io.d_out_q[k]; a.d_out_qa[k] = io.d_out_qa[k];
    a.gbias_q[k] = io.gbias_q[k]; a.gbias_q_raw[k] = io.gbias_q_raw[k];
    a.img_q[k] = io.img_q[k]; a.img_qa[k] = io.img_qa[k];
  }
  a.state = h->buf.state; a.B = B; a.gamma = (float)h->hyper.gamma; a.inv_global_batch = sc.inv_global_batch;
  a.act_q = h->oa.q;
  int blocks = (B + 63) / 64; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;   // latency bound: spread over the SMs
  launch_k(h->outact() ? loss_kernel<true> : loss_kernel<false>, capped(blocks, max_blocks), 64, 0, c, a);
  c.done();
}

// DSAC_V1's losses (one critic, fixed TD bound) and the gradients of the critic's outputs (critic 0 of `io`)
static void enqueue_loss_v1(const dsact_handle* h, const RowIo& io, int B, const StepScalars& sc, Ctx& c, int max_blocks = 0) {
  LossV1Args a;
  a.rew = io.rew; a.done = io.done; a.z = io.z3; a.logp2 = io.logp[1]; a.logp_new = io.logp[0];
  a.out_q = io.out_q[0]; a.out_qt = io.out_q[2]; a.out_qa = io.out_q[4];
  a.d_out_q = io.d_out_q[0]; a.d_out_qa = io.d_out_qa[0];
  a.gbias_q = io.gbias_q[0]; a.gbias_q_raw = io.gbias_q_raw[0];
  a.state = h->buf.state; a.B = B; a.bound = h->v1_bound; a.gamma = (float)h->hyper.gamma; a.inv_global_batch = sc.inv_global_batch;
  a.td_bound = (float)h->td_bound; a.sc = sc;
  a.img_q = io.img_q[0]; a.img_qa = io.img_qa[0];
  a.act_q = h->oa.q;
  int blocks = (B + 63) / 64; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
  launch_k(h->outact() ? loss_v1_kernel<true> : loss_v1_kernel<false>, capped(blocks, max_blocks), 64, 0, c, a);
  c.done();
}

// the actor loss's gradient w.r.t. the policy outputs of pi(s)
static void enqueue_policy_grad(const dsact_handle* h, const RowIo& io, int B, const StepScalars& sc, Ctx& c, int max_blocks = 0) {
  const StepHyper& p = h->hyper;
  const int A = h->act_dim;
  PolicyGradArgs a;
  const bool one_critic = io.d_act[1] == nullptr;
  a.logits = io.logits[0]; a.eps = io.eps[0]; a.d_act1 = io.d_act[0]; a.d_act2 = io.d_act[1];
  a.hi = h->buf.act_high; a.lo = h->buf.act_low;
  a.d_logits = io.d_logits; a.gbias = io.gbias_pi; a.gbias_ls = io.gbias_ls; a.state = h->buf.state;
  a.B = B; a.A = A; a.min_log_std = (float)p.min_log_std; a.max_log_std = (float)p.max_log_std; a.gauss = p.act_dist;
  a.inv_global_batch = sc.inv_global_batch;
  a.img = io.img_dlogits;
  a.img_ls = io.split_dlogits ? io.img_dlogits_ls : io.img_dlogits;
  a.ls_col = io.split_dlogits ? 0 : A;
  a.sc = sc;
  a.oa = h->oa;
  int blocks = (B + 7) / 8; if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms; if (blocks < 1) blocks = 1;   // a warp per row
  auto* k = h->outact() ? (one_critic ? policy_grad_kernel<1, true> : policy_grad_kernel<2, true>)
                        : (one_critic ? policy_grad_kernel<1, false> : policy_grad_kernel<2, false>);
  launch_k(k, capped(blocks, max_blocks), 256, sizeof(float) * 2 * A, c, a);
  c.done();
}

// Adam / Polyak over the whole flat buffers, on `grads` or (dp) on the rank-ordered sum of every rank's exchange block.
// n_q2: the critics' span (Adam every iteration).  scalars_ready: see ApplyArgs
static ApplyArgs apply_args(const dsact_handle* h, int64_t n_q2, int scalars_ready, bool dp) {
  const StepHyper& p = h->hyper;
  ApplyArgs a;
  memset(&a, 0, sizeof(a));
  a.params = h->buf.params; a.targets = h->buf.targets; a.grads = h->buf.grads; a.m = h->buf.adam_m; a.v = h->buf.adam_v;
  a.state = h->buf.state;
  a.n_q2 = n_q2; a.n_all = h->n_params;
  a.delay_update = p.delay_update; a.auto_alpha = p.auto_alpha;
  a.hy = adam_hyper(h); a.scalars_ready = scalars_ready;
  a.eps = (float)p.adam_eps; a.tau = (float)p.tau;
  a.omb1 = (float)(1.0 - p.adam_beta1); a.b2f = (float)p.adam_beta2; a.omb2 = (float)(1.0 - p.adam_beta2);
  a.dp_timeout_ns = dp_timeout_ns();
  if (dp) dp_apply_args(h->dp, a);
  a.g_lo = 0; a.g_hi = (a.n_all + 3) / 4; a.finish = 1;
  return a;
}
// `part` of the flat buffers: 0 = all of it; 1 = the critics' span only, without closing the step (launched beside the
// policy backward, see enqueue_phase2); 2 = everything after that span + the end-of-step bookkeeping.  A group straddling
// the critic / policy boundary goes with part 2.
static void apply_part(ApplyArgs& a, int part) {
  const int64_t g_q = a.n_q2 / 4;
  if (part == 2) a.g_lo = g_q;
  if (part == 1) { a.g_hi = g_q; a.finish = 0; }
}
static void launch_apply(const dsact_handle* h, const ApplyArgs& a, Ctx& c, int max_blocks = 0) {
  int blocks = (int)((a.g_hi - a.g_lo + 255) / 256);   // one 4-element group per thread
  if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms;
  if (blocks < 1) blocks = 1;
  blocks = capped(blocks, max_blocks);
  // (its last block also advances the step counters)
  if (a.dp_world > 0) launch_k(apply_kernel<2>, blocks, 256, 0, c, a);
  else if (a.nslabs > 0) launch_k(apply_kernel<1>, blocks, 256, 0, c, a);
  else launch_k(apply_kernel<0>, blocks, 256, 0, c, a);
  c.done();
  c.check();
}

// the replay gather: ring rows idx[i] (null: drawn on the device and recorded in the arena) -> the arena minibatch (or
// the fp32 rows of `dst`).  img: bf16 images of obs / obs2 / act to write as well; write_f32 = false leaves out their
// fp32 rows
static void enqueue_gather(const dsact_handle* h, int B, const int64_t* idx, const ImgOut img[3], bool write_f32, Ctx& c,
                           const dsact_batch* dst = nullptr) {
  const StepSlots& s = h->slot;
  float* W = h->W();
  // no index list: every warp of the gather draws its row's index itself (the sequence index_kernel defines) and records it
  int64_t* draw = idx ? nullptr : reinterpret_cast<int64_t*>(W + s.idx);
  float* d[6] = {W + s.obs, W + s.obs2, W + s.act, W + s.rew, W + s.done, W + s.logp};
  if (dst) {
    const float* o[6] = {dst->obs, dst->obs2, dst->act, dst->rew, dst->done, dst->logp};
    for (int i = 0; i < 6; ++i) d[i] = const_cast<float*>(o[i]);
  }
  int blocks = (B + 7) / 8; if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms;
  if (h->rb_frames) {
    const dsact_frame_replay& r = h->fr;
    launch_k(h->rb_code_bytes == 2 ? gather_kernel<true, 2> : h->rb_code_bytes == 1 ? gather_kernel<true, 1> : gather_kernel<true>,
             blocks, 256, 0, c, (const float*)r.frames,
             (const float*)r.frames, r.act, r.rew, r.done,
             r.logp, idx, d[0], d[1], d[2], d[3], d[4], d[5], B, (int)h->obs_elems, h->act_dim,
             img[0], img[1], img[2], draw, (unsigned long long)h->seed, (const float*)h->buf.state, write_f32 ? 1 : 0,
             (const int32_t*)r.obs_frames, (const int32_t*)r.obs2_frames, (int)r.frames_per_obs, (const float*)h->fr_table);
  } else {
    launch_k(gather_kernel<false>, blocks, 256, 0, c, h->rb.obs, h->rb.obs2, h->rb.act, h->rb.rew, h->rb.done, h->rb.logp, idx,
             d[0], d[1], d[2], d[3], d[4], d[5], B, (int)h->obs_elems, h->act_dim,
             img[0], img[1], img[2], draw, (unsigned long long)h->seed, (const float*)h->buf.state, write_f32 ? 1 : 0,
             (const int32_t*)nullptr, (const int32_t*)nullptr, 1, (const float*)nullptr);
  }
  c.done();
  c.check();
}

static dsact_batch arena_batch(const dsact_handle* h, int32_t batch) {
  const StepSlots& s = h->slot;
  float* W = h->W();
  dsact_batch b;
  b.obs = W + s.obs; b.act = W + s.act; b.rew = W + s.rew; b.obs2 = W + s.obs2; b.done = W + s.done;
  b.logp = W + s.logp;
  b.batch = batch;
  return b;
}

// ---- enqueue: pieces of one MLP update -------------------------------------------
// Where an update's prologue is enqueued: by its phase 1, forked beside the replay gather (phase 1 joins it), or on c.s
// before phase 1
enum { PRO_HERE = 0, PRO_FORKED = 1, PRO_DONE = 2 };
// One MLP update as the enqueue pieces see it
struct UpdatePlan {
  dsact_batch bt;            // its rows
  const dsact_noise* nz;     // its noise (null: device noise)
  int64_t global_batch;      // rows of the whole update (every rank's, dp)
  bool dp;                   // gradients and statistics reduced over the peers (dsact_dp_connect) instead of locally
  bool imaged;               // the bf16 images of obs / obs2 / act are in place (the prologue does not write them)
  int set;                   // the input set whose images the passes read (dsact_replay_steps)
  int prologue;              // PRO_*
};

// Everything of a step that depends on neither the minibatch gather nor a forward pass: accumulator clears, the
// gradient memset, the bf16 images of all weights (and of a caller-supplied batch), the device noise.
static void enqueue_prologue(MlpHandle* h, const UpdatePlan& u, Ctx& c) {
  const dsact_config& cf = h->cfg;
  const Net &q = h->q, &pi = h->pi;
  const Arena& ar = h->ar;
  float* W = h->W();
  const dsact_batch& bt = u.bt;
  const dsact_noise* nz = u.nz;
  const int B = bt.batch, O = cf.obs_dim, A = cf.act_dim;
  const bool tc = h->tc();
  const int nq = h->nq();
  const NetInsts I = net_insts(h);

  const bool want_noise = !nz;
  if (!tc) enqueue_begin_step(h, c);

  if (tc) {  // refresh the weight images (the caller may have written params/targets through its views) + inputs; the clears
             // and the device noise ride in the same launch
    ImgBatch ib;
    // one job per layer (a critic's layer 0: its obs and act columns, the act block at column kpad_q0 of the image)
    auto add_weights = [&](const NetInst& n) {
      const Net& net = *n.net;
      for (int j = 0; j <= net.L; ++j) {
        ib.reserve(h, c, 1);
        const Img im = h->img(n.wimg[j], net.s[j + 1]);
        if (j == 0 && &net == &q) ib.add(n.P + q.w[0], O + A, im, q.s[1], O, A, ar.kpad_q0);
        else ib.add(n.P + net.w[j], net.s[j], im, net.s[j + 1], net.s[j]);
      }
    };
    for (int k = 0; k < nq; ++k) add_weights(I.q[k]);
    const bool two_heads = cf.policy_std == DSACT_STD_SEPARATED;
    ib.reserve(h, c, pi.L + 2);
    add_weights(I.pi);
    if (!u.imaged) ib.add(bt.obs, O, h->img(ar.i_obs, B), B, O);
    if (two_heads) add_weights(I.pi_ls);
    for (int k = 0; k < nq; ++k) add_weights(I.qt[k]);
    if (two_heads) add_weights(I.pit_ls);
    ib.reserve(h, c, pi.L + 3);
    add_weights(I.pit);
    if (!u.imaged) {
      ib.add(bt.obs2, O, h->img(ar.i_obs2, B), B, O);
      ib.add(bt.act, A, h->img(ar.i_act, B), B, A);
    }
    PrologueArgs pa;
    memset(&pa, 0, sizeof(pa));
    pa.zero_blocks = begin_step_blocks(h);
    pa.state = h->buf.state; pa.grads = h->buf.grads; pa.n_grads = h->n_params;
    pa.hy = adam_hyper(h);
    if (want_noise) {
      pa.noise_blocks = noise_blocks(B, A);
      pa.eps1 = W + ar.eps1; pa.eps2 = W + ar.eps2; pa.z3 = W + ar.z3; pa.z4 = W + ar.z4;
      pa.B = B; pa.A = A; pa.seed = h->seed;
    }
    ib.launch(h, c, &pa);
  }

  if (want_noise && !tc) enqueue_noise(h, B, c);
  if (cf.policy_std == DSACT_STD_PARAMETER) {   // the log_std rows of pi and pi' (the head of the policy span) -> their logits
    const int64_t row = nq * q.n + h->span().ls;
    int blocks = (B * A + 255) / 256; if (blocks > 2 * h->num_sms) blocks = 2 * h->num_sms;
    launch_k(log_std_rows_kernel, blocks, 256, 0, c, W + ar.logitsP, W + ar.logitsT, (const float*)(h->buf.params + row),
             (const float*)(h->buf.targets + row), B, A);
    c.done();
  }
  c.check();
}

// In a captured step the prologue runs as its own branch next to whatever the main stream does first (the replay
// gather); returns PRO_FORKED if it was forked and must be joined (enqueue_phase1 does) before the first forward pass.
static int fork_prologue(MlpHandle* h, const UpdatePlan& u, Ctx& c) {
  if (!c.side) return PRO_HERE;
  fork_branch(c, h->ev_pro_fork, h->ev_pro_join, [&](Ctx& cs) { enqueue_prologue(h, u, cs); });
  return PRO_FORKED;
}

static void enqueue_dp_reduce_scatter(const DpPeer& dp, const float* state, int num_sms, Ctx& c) {
  const long long groups = dp.npad() / 4, per = (groups + dp.comm.world - 1) / dp.comm.world;
  DpSlice sl;
  sl.g_lo = per * dp.comm.rank;
  sl.g_hi = sl.g_lo + per < groups ? sl.g_lo + per : groups;
  if (sl.g_lo > groups) sl.g_lo = groups;
  sl.red_off = DP_GRADS_OFF + dp.npad();
  sl.ticket = reinterpret_cast<int*>(dp.buf) + DP_TICKET;
  int blocks = (int)((per + 255) / 256); if (blocks < 1) blocks = 1; if (blocks > 2 * num_sms) blocks = 2 * num_sms;
  launch_k(dp_reduce_scatter_kernel, blocks, 256, 0, c, dp.comm, sl, state);
  c.done();
}

// One exchange of the peer-memory data-parallel path (dp_peer.cuh): kind 0 = critic-std sums, 1 = logged sums.
static void enqueue_dp_exchange(const DpPeer& dp, float* state, int kind, Ctx& c) {
  launch_k(dp_exchange_kernel, 1, 32 * dp.comm.world, 0, c, dp.comm, state, kind, dp_timeout_ns());
  c.done();
}
static void enqueue_dp_exchange(MlpHandle* h, int kind, Ctx& c) { enqueue_dp_exchange(h->dp, h->buf.state, kind, c); }

// This rank's local gradient total into its exchange block: elements [0, n) of `grads` plus the first `nslabs`
// weight-gradient slabs (`slab_stride` floats apart); `tail`.enabled: the log_alpha element formed from the logged sum
static void enqueue_dp_fold(const dsact_handle* h, const float* grads, const float* slabs, int nslabs, long long slab_stride,
                            long long n, const TailArgs& tail, Ctx& c) {
  int blocks = (int)((n / 4 + 255) / 256); if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms; if (blocks < 1) blocks = 1;
  launch_k(dp_grad_fold_kernel, blocks, 256, 0, c, h->dp.buf + DP_GRADS_OFF, grads, slabs, n, nslabs, slab_stride,
           (const float*)h->buf.state, tail);
  c.done();
}

// ---- exchange-buffer setup (dsact_dp_export / dsact_dp_connect, both engines) ---------------------------------------
static int dp_peer_export(DpPeer& dp, int device, long long n_params, void* handle_out, int64_t* bytes_out) {
  CUDA_TRY(cudaSetDevice(device));
  dp.n_params = n_params;
  // header + this rank's gradient block + the reduced block of the two-shot exchange
  const size_t bytes = sizeof(float) * (size_t)(DP_GRADS_OFF + 2 * dp.npad());
  if (!dp.buf) {
    CUDA_TRY(cudaMalloc(&dp.buf, bytes));
    CUDA_TRY(cudaMemset(dp.buf, 0, bytes));
  }
  cudaIpcMemHandle_t ipc;
  CUDA_TRY(cudaIpcGetMemHandle(&ipc, dp.buf));
  static_assert(sizeof(ipc) == DSACT_IPC_HANDLE_BYTES, "IPC handle size");
  memcpy(handle_out, &ipc, sizeof(ipc));
  if (bytes_out) *bytes_out = (int64_t)bytes;
  return DSACT_OK;
}

// the peers' buffers this rank had opened are closed and the map is not ready until dp_peer_start
static int dp_peer_reset(DpPeer& dp, int device, int32_t rank, int32_t world) {
  if (!dp.buf) return fail(DSACT_ESTATE, "the exchange buffer has not been exported (dp_export)");
  if (world < 2 || world > DP_MAX_RANKS || rank < 0 || rank >= world) return fail(DSACT_EINVAL, "rank %d / world %d outside [2, %d]", rank, world, DP_MAX_RANKS);
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(cudaDeviceSynchronize());
  dp.ready = false;
  for (int r = 0; r < DP_MAX_RANKS; ++r)
    if (dp.opened[r]) { cudaIpcCloseMemHandle(dp.opened[r]); dp.opened[r] = nullptr; }
  dp.comm = DpComm();
  dp.comm.rank = rank; dp.comm.world = world;
  return DSACT_OK;
}

// once every peer's buffer is in dp.comm: every rank starts at epoch 0 with clear flags (the caller synchronises the
// ranks after this call)
static int dp_peer_start(DpPeer& dp, float* state) {
  CUDA_TRY(cudaMemset(dp.buf, 0, sizeof(float) * DP_GRADS_OFF));
  CUDA_TRY(cudaMemset(state + ST_DP_EPOCH, 0, sizeof(float)));
  CUDA_TRY(cudaMemset(state + ST_DP_ERR, 0, sizeof(float)));
  CUDA_TRY(cudaDeviceSynchronize());
  dp.ready = true;
  return DSACT_OK;
}

static int dp_peer_connect(DpPeer& dp, int device, float* state, int32_t rank, int32_t world, const void* handles) {
  int rc = dp_peer_reset(dp, device, rank, world);
  if (rc) return rc;
  for (int r = 0; r < world; ++r) {
    if (r == rank) { dp.comm.peer[r] = dp.buf; continue; }
    cudaIpcMemHandle_t ipc;
    memcpy(&ipc, static_cast<const char*>(handles) + (size_t)r * sizeof(ipc), sizeof(ipc));
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(DSACT_ECUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e)); }
    dp.opened[r] = p;
    dp.comm.peer[r] = static_cast<float*>(p);
  }
  return dp_peer_start(dp, state);
}

static void dp_peer_release(DpPeer& dp) {
  for (int r = 0; r < DP_MAX_RANKS; ++r) if (dp.opened[r]) cudaIpcCloseMemHandle(dp.opened[r]);
  if (dp.buf) cudaFree(dp.buf);
  dp = DpPeer();
}

// Forward passes and sampling of update `u`.  With `u.dp` the std sums are complete once sample_kernel has run, one whole
// forward chain before the loss needs them: in a captured step their exchange (kernel + NVLink flag round trip + whatever
// the ranks are skewed by) runs as a side branch under that chain.
static void enqueue_phase1(MlpHandle* h, const UpdatePlan& u, Ctx& c) {
  const dsact_batch& bt = u.bt;
  const int B = bt.batch;
  if (u.prologue == PRO_FORKED) cudaStreamWaitEvent(c.s, h->ev_pro_join, 0);
  else if (u.prologue == PRO_HERE) enqueue_prologue(h, u, c);

  const dsact_noise noise = step_noise(h, u.nz);   // device noise: sample_kernel steps the counter
  const StepPasses sp = step_passes(h, bt, u.set);
  enqueue_fwd(h, sp.a, sp.na, B, c);
  RowIo io = step_rows(h, bt, noise);
  io.img_act[0] = img_out(h, h->ar.i_new_act); io.img_act[1] = img_out(h, h->ar.i_act2);
  enqueue_sample(h, io, B, !u.nz, c);
  const bool dp_forked = u.dp && c.side != nullptr;
  if (dp_forked) fork_branch(c, h->ev_dp_fork, h->ev_dp_join, [&](Ctx& cs) { enqueue_dp_exchange(h, 0, cs); });
  else if (u.dp) enqueue_dp_exchange(h, 0, c);
  enqueue_fwd(h, sp.b, sp.nb, B, c);
  if (dp_forked) cudaStreamWaitEvent(c.s, h->ev_dp_join, 0);
  c.check();
}

// the apply of a single-call step can fold the weight-gradient split slabs itself (apply_kernel<1>)
static bool slabs_foldable(const MlpHandle* h) {
  return h->tc() && ((uintptr_t)(h->W() + h->ar.slabs) & 15) == 0 && ((uintptr_t)h->buf.grads & 15) == 0;
}
static TailArgs tail_args(const dsact_handle* h, int64_t global_batch, int rows) {
  TailArgs t;
  t.sc = step_scalars(h, global_batch);
  t.target_entropy = -(float)h->act_dim; t.rows = rows; t.enabled = 1;
  return t;
}
static void enqueue_apply(MlpHandle* h, Ctx& c, const TailArgs* tail, bool dp, int part);
// Losses and backward of update `u`.  `tail` == null (split API): the weight-gradient slabs are folded into the gradient
// buffer here and phase2_tail_kernel closes the backward.  Otherwise (single-call steps) the kernels that follow do both:
// enqueue_apply (u.dp = false), or dp_grad_fold into this rank's exchange block (u.dp = true).  Single-GPU fused steps
// also update the critics on the side branch as soon as their weight gradients are complete, beside the policy backward;
// returns true when it did, and the caller's enqueue_apply then does the rest (part 2).
static bool enqueue_phase2(MlpHandle* h, const UpdatePlan& u, Ctx& c, const TailArgs* tail) {
  const dsact_batch& bt = u.bt;
  const int64_t global_batch = u.global_batch;
  const bool dp = u.dp;
  const dsact_config& cf = h->cfg;
  const Net &q = h->q, &pi = h->pi;
  const Arena& ar = h->ar;
  float* W = h->W();
  const int B = bt.batch;
  const bool tc = h->tc();
  float* G_ = h->buf.grads;
  const long long n_flat = h->n_params;
  const StepPasses sp = step_passes(h, bt, u.set);
  const NetInsts& I = sp.I;

  const StepScalars sc = step_scalars(h, global_batch);
  RowIo io = step_rows(h, bt, step_noise(h, u.nz));
  for (int k = 0; k < h->nq(); ++k) {   // one two-output layer per critic: the std output's bias follows the mean's
    io.gbias_q[k] = I.q[k].G + q.b[q.L];
    io.img_q[k] = img_out(h, ar.i_dOut[k]); io.img_qa[k] = img_out(h, ar.i_dOut[4 + k]);
  }
  io.gbias_pi = I.pi.G + pi.b[pi.L];
  io.img_dlogits = img_out(h, ar.i_dlogits);
  if (cf.policy_std != DSACT_STD_SHARED) {   // the log_std half's gradient: the log_std network's output bias, or the row itself
    io.gbias_ls = cf.policy_std == DSACT_STD_SEPARATED ? I.pi_ls.G + pi.b[pi.L] : G_ + h->nq() * q.n + h->span().ls;
    io.split_dlogits = true;
    io.img_dlogits_ls = cf.policy_std == DSACT_STD_SEPARATED ? img_out(h, ar.i_dlogits_ls) : NO_IMG;
  }
  if (h->v1) enqueue_loss_v1(h, io, B, sc, c);
  else enqueue_loss(h, io, B, sc, c);
  // The freeze trick of the reference (dsac_v2.py:166-181) makes the critics' and the policy's backward independent: the
  // critics' dgrad, then, beside a policy backward chain, their weight gradients as a side branch.
  Group gw, ga;   // the critics' weight gradients; the per-layer lowering's dL/da~
  const bool chained = enqueue_dgrad(h, sp.q, sp.nqb, B, c, ga);
  add_wgrads(gw, h, sp.q, sp.nqb, B);
  const bool forked = chained && c.side != nullptr;
  bool applied = false;
  if (forked) {
    fork_branch(c, h->ev_fork, h->ev_join, [&](Ctx& cs) {
      // the policy backward chain needs ceil(B/64) whole SMs: keep them free of weight-gradient CTAs
      const int chain_ctas = (B + TC_BM - 1) / TC_BM;
      const int cap = h->num_sms - chain_ctas;
      launch_group(h, gw, V_WGRAD, cs, cap >= h->num_sms / 2 ? cap : 0);
      if (tail && !dp && slabs_foldable(h)) {   // Adam + Polyak of the critics beside the policy backward: every critic gradient is final here
        enqueue_apply(h, cs, tail, false, 1);
        applied = true;
      }
    });
  } else {
    launch_group(h, gw, V_WGRAD, c);
  }
  launch_group(h, ga, V_DGRAD, c);

  enqueue_policy_grad(h, io, B, sc, c);
  Group gwp, no_act;   // (the policy passes have no action segment)
  enqueue_dgrad(h, sp.pi, sp.npb, B, c, no_act);
  add_wgrads(gwp, h, sp.pi, sp.npb, B);
  launch_group(h, gwp, V_WGRAD, c);

  if (forked) cudaStreamWaitEvent(c.s, h->ev_join, 0);
  if (tc && !dp && !(tail && slabs_foldable(h))) {  // fold the weight-gradient split slabs into the flat gradient buffer
    const long long n = n_flat;
    int blocks = (int)((n + 255) / 256); if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
    launch_k(grad_reduce_kernel, blocks, 256, 0, c, G_, W + ar.slabs, n, ar.nslabs, (long long)ar.slab_stride); c.done();
  }
  if (!tail) {
    launch_k(phase2_tail_kernel, 1, 32, 0, c, G_ + n_flat - 1, h->buf.state, sc, -(float)cf.act_dim, B, adam_hyper(h), 0);
    c.done();
  }
  if (dp)  // local total (bias gradients + slabs + log_alpha) -> this rank's block of the exchange buffer
    enqueue_dp_fold(h, G_, tc ? W + ar.slabs : G_, tc ? ar.nslabs : 0, tc ? ar.slab_stride : 4, n_flat, *tail, c);
  c.check();
  return applied;
}

// The MLP engine's apply of `part` (see apply_part) with the Adam scalars `scalars_ready` (see ApplyArgs), the step's
// end-of-backward bookkeeping `tail` (null: none) and the first `nslabs` weight-gradient split slabs folded in
static ApplyArgs mlp_apply_args(const MlpHandle* h, int scalars_ready, const TailArgs* tail, bool dp, int part, int nslabs) {
  ApplyArgs a = apply_args(h, h->nq() * h->q.n, scalars_ready, dp);
  if (tail) a.tail = *tail;
  if (nslabs > 0) { a.slabs = h->W() + h->ar.slabs; a.nslabs = nslabs; a.slab_stride = h->ar.slab_stride; }
  apply_part(a, part);
  a.next_scalars = h->tc() ? 0 : 1;   // the tensor-core modes' prologue (step_prologue_kernel) forms them itself
  return a;
}
// `tail` != null: this apply also does the end-of-backward bookkeeping of the step (see TailArgs) and, single-GPU, folds
// the weight-gradient split slabs.  `dp`: the gradients are the rank-ordered sum of the exchange blocks.
static void enqueue_apply(MlpHandle* h, Ctx& c, const TailArgs* tail = nullptr, bool dp = false, int part = 0) {
  // split API: the Adam scalars are formed here; single-call steps: precomputed by the previous apply / prologue if stamped
  const int nslabs = tail && !dp && slabs_foldable(h) ? h->ar.nslabs : 0;
  launch_apply(h, mlp_apply_args(h, tail ? 2 : 0, tail, dp, part, nslabs), c);
}

// The rest of a single-call update after its phase 1: phase 2 over `u.global_batch` rows, then (u.dp) the logged-sum
// exchange (also the "every rank's block is complete" barrier) and the reduce-scatter from 6 ranks up, then Adam / Polyak.
static void enqueue_phase2_apply(MlpHandle* h, const UpdatePlan& u, Ctx& c) {
  const TailArgs ta = tail_args(h, u.global_batch, u.bt.batch);
  const bool critics_applied = enqueue_phase2(h, u, c, &ta);
  if (u.dp) {
    enqueue_dp_exchange(h, 1, c);
    if (dp_two_shot(h->dp)) enqueue_dp_reduce_scatter(h->dp, h->buf.state, h->num_sms, c);
  }
  enqueue_apply(h, c, &ta, u.dp, critics_applied ? 2 : 0);
}

// One whole update of the single-call steps
static void enqueue_update(MlpHandle* h, const UpdatePlan& u, Ctx& c) {
  enqueue_phase1(h, u, c);
  enqueue_phase2_apply(h, u, c);
}

// the generator counter step of a call whose last draw is the gather's (no sample_kernel after it steps it)
static void enqueue_rng_advance(const dsact_handle* h, Ctx& c) {
  launch_k(rng_advance_kernel, 1, 32, 0, c, h->buf.state);
  c.done();
}

// the replay gather with the bf16 images of obs / obs2 / act.  `images_only`: the caller is a fused tensor-core step,
// which reads them through their images alone
static void enqueue_gather_imaged(MlpHandle* h, int B, const int64_t* idx, Ctx& c, bool images_only) {
  const ImgOut img[3] = {img_out(h, h->ar.i_obs), img_out(h, h->ar.i_obs2), img_out(h, h->ar.i_act)};
  enqueue_gather(h, B, idx, img, !images_only, c);
}

// ---- n replay-fed updates in one submission (dsact_replay_steps, dsact_dp_replay_steps) ------------------------------
// the minibatch of input set `set` (0: the arena's, 1: the library-owned second set)
static dsact_batch input_batch(const MlpHandle* h, int set, int32_t batch) {
  if (set == 0) return arena_batch(h, batch);
  const float* b = h->in2;
  dsact_batch o;
  o.obs = b + h->in2_obs; o.obs2 = b + h->in2_obs2; o.act = b + h->in2_act; o.rew = b + h->in2_rew; o.done = b + h->in2_done;
  o.logp = b + h->in2_logp; o.batch = batch;
  return o;
}

// allocate the second input set on the first call, laid out like the arena's (Arena::build)
static int ensure_input_set2(MlpHandle* h) {
  if (h->in2) return DSACT_OK;
  const int64_t B = h->cfg.max_batch, O = h->cfg.obs_dim, A = h->cfg.act_dim;
  int64_t off = 0;
  auto take = [&](int64_t n) { int64_t o = off; off += round64(n); return o; };
  h->in2_obs = take(B * O); h->in2_obs2 = take(B * O); h->in2_act = take(B * A);
  h->in2_rew = take(B); h->in2_done = take(B); h->in2_logp = take(B);
  const int widths[3] = {(int)O, (int)O, (int)A};
  for (int i = 0; i < 3; ++i) {
    ImgSlot& s = h->in2_img[i];
    if (!h->tc()) { s = ImgSlot(); continue; }
    s.rows = (int)B; s.width = widths[i]; s.pitch = (widths[i] + 7) / 8 * 8;
    s.plane = round64(B * s.pitch);
    s.off = take(s.plane);   // 2 planes of bf16 = plane floats
  }
  CUDA_TRY(cudaMalloc(&h->in2, sizeof(float) * (size_t)off));
  CUDA_TRY(cudaMemset(h->in2, 0, sizeof(float) * (size_t)off));
  CUDA_TRY(cudaStreamCreateWithFlags(&h->gather_stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&h->ev_gather_fork, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&h->ev_gather_join, cudaEventDisableTiming));
  return DSACT_OK;
}

// tb_info denominators (dsact_read_stats): DSAC_V1 logs one entry of the logits row per sample (dsac_v1.py:142-143),
// DSAC-T the mean over all action dimensions
static void stats_scales(const dsact_handle* h, int64_t global_batch, float* inv_batch, float* inv_policy) {
  const double pol = h->v1 ? (double)global_batch : (double)global_batch * h->act_dim;
  *inv_batch = (float)(1.0 / (double)global_batch);
  *inv_policy = (float)(1.0 / pol);
}

// noise of update k of a call whose caller noise `np` holds n updates' draws back to back
static dsact_noise update_noise(const dsact_noise& np, int k, int B, int A) {
  return dsact_noise{np.eps1 + (size_t)k * B * A, np.eps2 + (size_t)k * B * A, np.z3 + (size_t)k * B, np.z4 + (size_t)k * B};
}

// Updates k = 0 .. n-1, each one dsact_replay_step on its slice of idx / noise.  Update k reads input set k & 1; the gather
// of update k + 1 into the other set needs only the generator counter update k's sample_kernel leaves, so it is forked
// (captured: onto its own stream) once update k's forward passes are enqueued and runs beside update k's backward; the
// set it overwrites was last read by update k - 1.  The prologue of update k + 1 (weight images, noise, clears, Adam
// scalars) reads what update k's apply writes and follows it on the main stream with programmatic dependent launch.
// stats_out: row k = update k's finalised tb_info over `global_batch` rows, written before update k + 1 clears the
// accumulators (slot 14: the peer-timeout flag as update k left it).
// `dp`: every update is dsact_dp_replay_step's, the data-parallel body of enqueue_update: the std-sum exchange on the side
// branch under phase 1's second forward chain, phase 2 over `global_batch` rows ending in dp_grad_fold, the logged-sum
// exchange, the reduce-scatter from 6 ranks up, the apply on the exchanged sums.  Each update bumps the exchange epoch as
// its single call does.  The exchange branch is joined inside phase 1, before the gather branch is forked, and the
// gather branch is joined before the next update's phase 1 forks the exchange again: neither pair of fork / join events
// is recorded again while the branch it bounds is open.
static void enqueue_replay_steps(MlpHandle* h, int n, int B, const int64_t* idx, const dsact_noise* np, int64_t global_batch,
                                 bool dp, float* stats_out, Ctx& c) {
  const int A = h->cfg.act_dim;
  const bool fused = h->fused();
  const bool fork = c.side != nullptr;
  auto idx_of = [&](int k) { return idx ? idx + (size_t)k * B : nullptr; };
  // gather of update k into input set k & 1 (+ the counter step a drawn-index, caller-noise update takes after it)
  auto gather = [&](int k, Ctx& cg) {
    const int set = k & 1;
    const dsact_batch dst = input_batch(h, set, B);
    const ImgOut img[3] = {img_out_of(h, h->input_img(set, 0, B)), img_out_of(h, h->input_img(set, 1, B)),
                           img_out_of(h, h->input_img(set, 2, B))};
    enqueue_gather(h, B, idx_of(k), img, !fused, cg, &dst);
    if (!idx && np) enqueue_rng_advance(h, cg);
  };
  float inv_b, inv_pol;
  stats_scales(h, global_batch, &inv_b, &inv_pol);
  bool gather_forked = false;
  for (int k = 0; k < n; ++k) {
    const int set = k & 1;
    dsact_noise nk;
    if (np) nk = update_noise(*np, k, B, A);
    UpdatePlan u{input_batch(h, set, B), np ? &nk : nullptr, global_batch, dp, true, set, PRO_DONE};
    if (k == 0) {   // as dsact_replay_step: the prologue beside the gather
      u.prologue = fork_prologue(h, u, c);
      gather(0, c);
    } else {
      enqueue_prologue(h, u, c);
      if (gather_forked) cudaStreamWaitEvent(c.s, h->ev_gather_join, 0);
    }
    enqueue_phase1(h, u, c);
    gather_forked = false;
    if (k + 1 < n) {
      if (fork) {
        fork_branch(c, h->ev_gather_fork, h->ev_gather_join, [&](Ctx& cg) { gather(k + 1, cg); }, h->gather_stream);
        gather_forked = true;
      } else {
        gather(k + 1, c);
      }
    }
    enqueue_phase2_apply(h, u, c);
    if (stats_out) {
      launch_k(finalize_stats_kernel, 1, 32, 0, c, h->buf.state, inv_b, inv_pol, stats_out + (size_t)k * DSACT_NUM_STATS);
      c.done();
    }
  }
  c.check();
}

// ---- graph cache -------------------------------------------------------------
static void drop_graphs(MlpHandle* h) {
  for (auto& e : h->graphs) cudaGraphExecDestroy(e.exec);
  h->graphs.clear();
}

// one eager enqueue on `s` and its launch bookkeeping (both engines)
template <typename F>
static int run_eager(dsact_handle* h, cudaStream_t s, bool pdl, F enqueue) {
  Ctx c{s, 0, cudaSuccess};
  c.pdl = pdl;
  enqueue(c);
  if (c.err != cudaSuccess) return fail(DSACT_ECUDA, "kernel launch failed: %s", cudaGetErrorString(c.err));
  h->launches += c.launches;
  h->last_launches = c.launches;
  return DSACT_OK;
}

template <typename F>
static int run(MlpHandle* h, cudaStream_t user, const GraphKey& key, F enqueue) {
  if (!h->cfg.use_graph) return run_eager(h, user, h->tc(), enqueue);
  GraphEntry* hit = nullptr;
  for (auto& e : h->graphs)
    if (e.key == key) { hit = &e; break; }
  if (!hit) {
    CUDA_TRY(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeRelaxed));
    Ctx c{h->cap_stream, 0, cudaSuccess};
    c.pdl = h->tc();
    c.side = h->side_stream;
    enqueue(c);
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(h->cap_stream, &graph);
    if (c.err != cudaSuccess || e != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return fail(DSACT_ECUDA, "graph capture failed: %s", cudaGetErrorString(c.err != cudaSuccess ? c.err : e));
    }
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail(DSACT_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
    if (h->graphs.size() >= 16) {  // evict the least recently used
      size_t victim = 0;
      for (size_t i = 1; i < h->graphs.size(); ++i)
        if (h->graphs[i].stamp < h->graphs[victim].stamp) victim = i;
      cudaGraphExecDestroy(h->graphs[victim].exec);
      h->graphs.erase(h->graphs.begin() + victim);
    }
    h->graphs.push_back(GraphEntry{key, exec, c.launches, 0});
    hit = &h->graphs.back();
  }
  hit->stamp = ++h->stamp;
  CUDA_TRY(cudaGraphLaunch(hit->exec, user));
  h->launches += hit->launches;
  h->last_launches = hit->launches;
  return DSACT_OK;
}

// dsact_profile_step: one eager enqueue on `s` with an event after every launch (no side stream: the critics' update is
// not split off), synchronised, and the time, FLOPs and launches per class into `out`
template <typename F>
static int run_profiled(MlpHandle* h, cudaStream_t s, dsact_profile* out, F enqueue) {
  Prof prof;
  Ctx c{s, 0, cudaSuccess};
  c.pdl = h->tc();
  c.prof = &prof;
  cudaEvent_t e0;
  CUDA_TRY(cudaEventCreate(&e0));
  CUDA_TRY(cudaEventRecord(e0, s));
  enqueue(c);
  cudaError_t e = cudaStreamSynchronize(s);
  memset(out, 0, sizeof(*out));
  cudaEvent_t prev = e0;
  for (size_t i = 0; i < prof.ev.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, prev, prof.ev[i]);
    out->ms[prof.cls[i]] += ms;
    out->flops[prof.cls[i]] += prof.flops[i];
    out->launches[prof.cls[i]] += 1;
    out->total_ms += ms;
    prev = prof.ev[i];
  }
  cudaEventDestroy(e0);
  for (auto ev : prof.ev) cudaEventDestroy(ev);
  if (c.err != cudaSuccess || e != cudaSuccess)
    return fail(DSACT_ECUDA, "profile step failed: %s", cudaGetErrorString(c.err != cudaSuccess ? c.err : e));
  h->launches += c.launches;
  h->last_launches = c.launches;
  return DSACT_OK;
}

// true when `bt` is the arena minibatch that the preceding dsact_replay_sample gathered (images already there)
static bool take_arena_images(MlpHandle* h, const dsact_batch& bt) {
  const bool yes = h->tc() && h->arena_imaged && bt.obs == h->W() + h->ar.obs && bt.obs2 == h->W() + h->ar.obs2 &&
                   bt.act == h->W() + h->ar.act;
  // any other batch is imaged into the same shared slots by the call that asked: the arena's images are gone after it.
  // (The arena views handed out by dsact_replay_sample are read-only for the same reason: edits are not re-imaged.)
  if (!yes) h->arena_imaged = false;
  return yes;
}

static MlpHandle* mlp(dsact_handle* h) { return static_cast<MlpHandle*>(h); }

// ---- checks and device-state syncs of the shell (both engines) ---------------------------------------------------
static int check_batch(const dsact_handle* h, const dsact_batch* b) {
  if (!h) return fail(DSACT_EINVAL, "null handle");
  if (!h->bound) return fail(DSACT_ESTATE, "dsact_bind has not been called");
  if (!b || !b->obs || !b->act || !b->rew || !b->obs2 || !b->done) return fail(DSACT_EINVAL, "null batch pointer");
  if (b->batch < 1 || b->batch > h->max_batch)
    return fail(DSACT_EINVAL, "batch %d outside [1, max_batch=%d]", b->batch, h->max_batch);
  return DSACT_OK;
}
static int check_noise(const dsact_noise* n) {
  if (n && (!n->eps1 || !n->eps2 || !n->z3 || !n->z4)) return fail(DSACT_EINVAL, "null noise pointer");
  return DSACT_OK;
}
// the split and data-parallel entry points implement DSAC_V2 (DSAC-T); DSAC_V1 has local steps only
static int check_v2(const dsact_handle* h) {
  return h->v1 ? fail(DSACT_EINVAL, "DSAC_V1 handles have no split or data-parallel update") : DSACT_OK;
}
// the peer-memory data-parallel step has not run with two policy heads or a log_std row: refused until it has
static int check_dp(const dsact_handle* h) {
  int rc = check_v2(h);
  if (rc) return rc;
  if (h->engine == ENGINE_MLP && static_cast<const MlpHandle*>(h)->cfg.policy_std != DSACT_STD_SHARED)
    return fail(DSACT_EINVAL, "the MLP engine's data-parallel step runs the mlp_shared policy only (policy_std %d): use the split "
                              "calls (dsact_grad_phase1/2, dsact_apply) with an all-reduce between them",
                static_cast<const MlpHandle*>(h)->cfg.policy_std);
  return DSACT_OK;
}
// host staging, the replay-fused steps, the profiler and the GEMM test hook exist on the MLP engine only
static int check_mlp(const dsact_handle* h, const char* fn) {
  return h && h->engine != ENGINE_MLP ? fail(DSACT_EINVAL, "%s: the head-wise engine does not implement this call", fn) : DSACT_OK;
}

static int sync_iteration(dsact_handle* h, int64_t iteration, cudaStream_t s) {
  if (iteration < 0 || iteration > 0x7fffffff) return fail(DSACT_EINVAL, "iteration out of range");
  if (h->dev_iter != iteration) {
    set_iter_kernel<<<1, 32, 0, s>>>(h->buf.state, (int)iteration);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
  }
  return DSACT_OK;
}

static int sync_rb_size(dsact_handle* h, int64_t size, cudaStream_t s) {
  if (size < 1 || size > h->rb_rows()) return fail(DSACT_EINVAL, "size %lld outside [1, capacity]", (long long)size);
  if (h->dev_rb_size != size) {
    set_rb_size_kernel<<<1, 32, 0, s>>>(h->buf.state, size);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    h->dev_rb_size = size;
  }
  return DSACT_OK;
}

// the SM count of `device`, which must be an sm_90 part
static int check_sm90(int device, int* num_sms) {
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(DSACT_EARCH, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  *num_sms = prop.multiProcessorCount;
  return DSACT_OK;
}

#include "cnn_engine.cuh"

// ---- one path for every update entry point (both engines) -----------------------------------------------------------
// What an update call runs: phase 1, phase 2, both, Adam / Polyak, a whole update, n_steps replay-fed updates, or the
// replay gather alone
enum { RUN_PHASE1, RUN_PHASE2, RUN_GRADS, RUN_APPLY, RUN_STEP, RUN_STEPS, RUN_GATHER };

// One update call as its entry point describes it
struct UpdateCall {
  const char* fn;                       // the entry point (refusals name it)
  int run;                              // RUN_*
  const dsact_batch* batch = nullptr;   // the caller's rows; null: the replay gather's (replay), or (phase 2) the last phase 1's
  bool replay = false;                  // rows gathered from the replay ring: `rows` of them, ring rows idx[i] (null: drawn on
  int32_t rows = 0;                     // the device) among the first `size`
  int64_t size = 0;
  const int64_t* idx = nullptr;
  const dsact_noise* noise = nullptr;   // null: device noise
  int64_t iteration = 0;                // RUN_APPLY, RUN_STEP, RUN_STEPS: the iteration of the (first) update
  int64_t global_batch = 0;             // rows of the whole update (0: its own rows)
  bool dp = false;                      // the data-parallel step over the peers (dsact_dp_connect)
  int32_t n_steps = 1;                  // updates (RUN_STEPS)
  float* stats_out = nullptr;           // RUN_STEPS: row k = update k's statistics (null: none)
  bool profiled = false;                // dsact_profile_step: eager, an event after every launch, timings into `prof`
  dsact_profile* prof = nullptr;
  dsact_batch* out = nullptr;           // RUN_GATHER: the arena views of the gathered rows (null: none)
  UpdateCall(const char* f, int r) : fn(f), run(r) {}
  bool split() const { return run <= RUN_APPLY; }   // the split calls (DSAC-T only)
  bool iterates() const { return run == RUN_APPLY || run == RUN_STEP || run == RUN_STEPS; }
};

// the refusals of call `u`, each with the code its entry point has always returned for it
static int check_call(const dsact_handle* h, const UpdateCall& u) {
  int rc = u.profiled || (u.replay && u.run != RUN_GATHER) ? check_mlp(h, u.fn) : DSACT_OK;
  if (rc) return rc;
  if (u.batch) {
    if ((rc = check_batch(h, u.batch))) return rc;
  } else if (!h || !h->bound || (u.replay && !h->rb_bound)) {
    return fail(DSACT_ESTATE, "not bound");
  }
  if (u.run == RUN_STEPS && (u.n_steps < 1 || u.n_steps > DSACT_MAX_REPLAY_STEPS))
    return fail(DSACT_EINVAL, "n_steps %d outside [1, %d]", u.n_steps, DSACT_MAX_REPLAY_STEPS);
  if (u.replay && (u.rows < 1 || u.rows > h->max_batch)) return fail(DSACT_EINVAL, "batch outside [1, max_batch]");
  if (u.run == RUN_STEPS && u.iteration + u.n_steps - 1 > 0x7fffffff) return fail(DSACT_EINVAL, "iteration out of range");
  if ((rc = check_noise(u.noise))) return rc;
  if (u.split() && (rc = check_v2(h))) return rc;
  if (u.dp) {
    if ((rc = check_dp(h))) return rc;
    if (!h->dp.ready) return fail(DSACT_ESTATE, "dsact_dp_connect has not been called");
  }
  if (u.run == RUN_PHASE2 && h->pending.batch < 1)
    return fail(DSACT_ESTATE, "dsact_grad_phase2 without a preceding dsact_grad_phase1");
  const int32_t local = u.run == RUN_PHASE2 ? h->pending.batch : u.batch ? u.batch->batch : u.rows;
  if ((u.dp || u.run == RUN_PHASE2) && u.global_batch < local)
    return fail(DSACT_EINVAL, "global_batch %lld < local batch %d", (long long)u.global_batch, local);
  if (u.profiled && !u.prof) return fail(DSACT_EINVAL, "null out");
  return DSACT_OK;
}

// The captured graph of call `u` on plan `p`: the call's kind, and every input of its work that is not device state
static GraphKey graph_key(const UpdateCall& u, const UpdatePlan& p) {
  const dsact_noise n = p.nz ? *p.nz : dsact_noise{};
  return GraphKey{u.run, u.replay, u.dp, p.bt.obs, p.bt.act, p.bt.rew, p.bt.obs2, p.bt.done, p.bt.batch,
                  n.eps1, n.eps2, n.z3, n.z4, p.global_batch, p.imaged, u.idx, u.n_steps, u.stats_out};
}

// The MLP engine's enqueue of call `u`, whose (first) update is `p`
static void enqueue_call(MlpHandle* h, const UpdateCall& u, UpdatePlan p, Ctx& c) {
  const int B = p.bt.batch;
  switch (u.run) {
    case RUN_PHASE1: enqueue_phase1(h, p, c); break;
    case RUN_PHASE2: enqueue_phase2(h, p, c, nullptr); break;
    case RUN_GRADS: enqueue_phase1(h, p, c); enqueue_phase2(h, p, c, nullptr); break;
    case RUN_APPLY: enqueue_apply(h, c); break;
    case RUN_STEPS: enqueue_replay_steps(h, u.n_steps, B, u.idx, p.nz, p.global_batch, p.dp, u.stats_out, c); break;
    case RUN_GATHER:
      enqueue_gather_imaged(h, B, u.idx, c, false);
      if (!u.idx) enqueue_rng_advance(h, c);
      break;
    case RUN_STEP:
      if (u.replay) {   // weight images, noise, clears: beside the gather
        p.prologue = fork_prologue(h, p, c);
        enqueue_gather_imaged(h, B, u.idx, c, h->fused());
        if (!u.idx && p.nz) enqueue_rng_advance(h, c);   // device noise: phase 1 advances the counter after the join
      }
      enqueue_update(h, p, c);
      break;
  }
}

// Every update entry point: the checks, the device, the ring-size and iteration syncs, the rows and noise, the engine's
// enqueue (captured, eager or profiled), then what the handle records about it
static int update(dsact_handle* h, const UpdateCall& u, void* stream) {
  int rc = check_call(h, u);
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  const cudaStream_t s = (cudaStream_t)stream;
  MlpHandle* m = h->engine == ENGINE_MLP ? mlp(h) : nullptr;
  if (u.run == RUN_STEPS && (rc = ensure_input_set2(m))) return rc;
  if (u.replay && (rc = sync_rb_size(h, u.size, s))) return rc;
  if (u.iterates() && (rc = sync_iteration(h, u.iteration, s))) return rc;

  // the rows and noise: the caller's, the arena's (replay), or (phase 2) those of the last phase 1
  dsact_batch bt = {};
  dsact_noise nz = u.noise ? *u.noise : dsact_noise{};
  const dsact_noise* np = u.noise ? &nz : nullptr;
  if (u.batch) bt = *u.batch;
  else if (u.replay) bt = arena_batch(h, u.rows);
  else if (u.run == RUN_PHASE2) { bt = h->pending; nz = h->pending_noise; np = &nz; }
  const int64_t gb = u.global_batch > 0 ? u.global_batch : bt.batch;

  if (!m) {
    HeadsHandle* hh = heads(h);
    rc = run_eager(h, s, false, [&](Ctx& c) {
      switch (u.run) {
        case RUN_PHASE1: cnn_enqueue_phase1(hh, bt, np, c); break;
        case RUN_PHASE2: cnn_enqueue_phase2(hh, bt, nz, gb, c); break;
        case RUN_GRADS: cnn_enqueue_phase1(hh, bt, np, c); cnn_enqueue_phase2(hh, bt, step_noise(h, np), gb, c); break;
        case RUN_APPLY: cnn_enqueue_apply(hh, c, 0, false); break;
        case RUN_STEP:
          if (u.dp) cnn_enqueue_dp_step(hh, bt, np, gb, c);
          else cnn_enqueue_step(hh, bt, np, c);
          break;
        case RUN_GATHER: {
          const ImgOut none[3] = {NO_IMG, NO_IMG, NO_IMG};
          enqueue_gather(h, u.rows, u.idx, none, true, c);
          if (!u.idx) enqueue_rng_advance(h, c);
          break;
        }
      }
    });
  } else {
    // the inputs' images: written by this call's gather, left by the preceding dsact_replay_sample, or written by the
    // prologue (take_arena_images, the one place that tracks what the arena's images hold)
    const UpdatePlan p{bt, np, gb, u.dp, u.replay || (u.batch && take_arena_images(m, bt)), 0, PRO_HERE};
    auto enqueue = [&](Ctx& c) { enqueue_call(m, u, p, c); };
    rc = u.profiled ? run_profiled(m, s, u.prof, enqueue) : run(m, s, graph_key(u, p), enqueue);
  }
  if (rc) return rc;

  // the arena's images (and, in the fused modes, only they) now belong to this call's gather
  if (m && u.replay) m->arena_imaged = u.run == RUN_GATHER;
  if (u.run == RUN_GATHER) {
    if (u.out) *u.out = bt;
  } else if (u.run != RUN_PHASE2 && u.run != RUN_APPLY) {   // the rows and noise of the (last) phase 1, for dsact_grad_phase2
    const int k = u.n_steps - 1;   // (dsact_replay_steps: update k read input set k & 1)
    h->pending = u.run == RUN_STEPS ? input_batch(m, k & 1, bt.batch) : bt;
    h->pending_noise = np ? update_noise(nz, k, bt.batch, h->act_dim) : step_noise(h, nullptr);
  }
  if (u.iterates()) h->dev_iter = u.iteration + u.n_steps;
  return DSACT_OK;
}

// ---- C ABI ---------------------------------------------------------------------
extern "C" {

const char* dsact_last_error(void) { return g_err; }
int dsact_abi_version(void) { return DSACT_ABI_VERSION; }

static int validate(const dsact_config* c) {
  if (!c) return fail(DSACT_EINVAL, "null config");
  if (c->abi_version != DSACT_ABI_VERSION) return fail(DSACT_EINVAL, "abi_version %d != %d", c->abi_version, DSACT_ABI_VERSION);
  if (c->obs_dim < 1 || c->act_dim < 1) return fail(DSACT_EINVAL, "obs_dim/act_dim must be positive");
  if (c->n_hidden_q < 1 || c->n_hidden_q > DSACT_MAX_HIDDEN || c->n_hidden_pi < 1 || c->n_hidden_pi > DSACT_MAX_HIDDEN)
    return fail(DSACT_EINVAL, "1..%d hidden layers supported", DSACT_MAX_HIDDEN);
  for (int j = 0; j < c->n_hidden_q; ++j) if (c->hidden_q[j] < 1) return fail(DSACT_EINVAL, "bad value hidden size");
  for (int j = 0; j < c->n_hidden_pi; ++j) if (c->hidden_pi[j] < 1) return fail(DSACT_EINVAL, "bad policy hidden size");
  if (c->act_q < 0 || c->act_q > DSACT_ACT_SELU || c->act_pi < 0 || c->act_pi > DSACT_ACT_SELU)
    return fail(DSACT_EINVAL, "unknown activation");
  if (c->max_batch < 1) return fail(DSACT_EINVAL, "max_batch must be positive");
  if (c->delay_update < 1) return fail(DSACT_EINVAL, "delay_update must be >= 1");
  if (c->gemm_mode < DSACT_GEMM_FP32 || c->gemm_mode > DSACT_GEMM_BF16) return fail(DSACT_EINVAL, "unknown gemm_mode %d", c->gemm_mode);
  if (c->act_dist != 0 && c->act_dist != 1) return fail(DSACT_EINVAL, "act_dist must be 0 (TanhGaussDistribution) or 1 (GaussDistribution)");
  if (c->policy_std < DSACT_STD_SHARED || c->policy_std > DSACT_STD_PARAMETER)
    return fail(DSACT_EINVAL, "policy_std must be 0 (mlp_shared), 1 (mlp_separated) or 2 (parameter), got %d", c->policy_std);
  return DSACT_OK;
}

static int validate_v1(const dsact_config* c, const dsact_v1_options* v) {
  if (!v) return fail(DSACT_EINVAL, "null DSAC_V1 options");
  if (c->policy_std != DSACT_STD_SHARED)
    return fail(DSACT_EINVAL, "DSAC_V1 on the MLP engine runs the mlp_shared policy only (policy_std %d)", c->policy_std);
  if (v->abi_version != DSACT_ABI_VERSION) return fail(DSACT_EINVAL, "dsact_v1_options.abi_version %d != %d", v->abi_version, DSACT_ABI_VERSION);
  if (v->bound != 0 && v->bound != 1) return fail(DSACT_EINVAL, "DSAC_V1 bound must be 0 (Gaussian NLL) or 1 (bounded loss), got %d", v->bound);
  if (!(v->td_bound > 0.0) || !std::isfinite(v->td_bound)) return fail(DSACT_EINVAL, "DSAC_V1 TD_bound must be finite and > 0, got %g", v->td_bound);
  return DSACT_OK;
}

// the layout of an MLP-engine handle with nq critics (DSAC-T 2, DSAC_V1 1)
static int mlp_query_layout(const dsact_config* cfg, int nq, dsact_layout* out) {
  if (!out) return fail(DSACT_EINVAL, "null out");
  Net q, pi;
  q.build(cfg->obs_dim + cfg->act_dim, cfg->hidden_q, cfg->n_hidden_q, 2);
  pi.build(cfg->obs_dim, cfg->hidden_pi, cfg->n_hidden_pi, pi_outputs(*cfg));
  Arena ar;
  ar.build(*cfg, q, pi, nq);
  out->n_q = q.n; out->n_pi = pi_span(cfg->policy_std, pi, cfg->act_dim).n;
  out->n_params = nq * q.n + out->n_pi + 1;
  out->n_targets = nq * q.n + out->n_pi;
  out->workspace_bytes = ar.total * (int64_t)sizeof(float);
  out->state_floats = ST_FLOATS;
  out->max_batch = cfg->max_batch;
  out->off_idx = ar.idx; out->off_eps1 = ar.eps1; out->off_eps2 = ar.eps2; out->off_z3 = ar.z3; out->off_z4 = ar.z4;
  out->off_slabs = ar.slabs; out->slab_floats = ar.total - ar.slabs;
  return DSACT_OK;
}

int dsact_query_layout(const dsact_config* cfg, dsact_layout* out) {
  int rc = validate(cfg);
  return rc ? rc : mlp_query_layout(cfg, 2, out);
}

int dsact_v1_query_layout(const dsact_config* cfg, const dsact_v1_options* v1, dsact_layout* out) {
  int rc = validate(cfg);
  if (rc || (rc = validate_v1(cfg, v1))) return rc;
  return mlp_query_layout(cfg, 1, out);
}

// an MLP-engine handle: DSAC-T (v1 == null) or DSAC_V1
static int mlp_create(const dsact_config* cfg, const dsact_v1_options* v1, int device, dsact_handle** out) {
  if (!out) return fail(DSACT_EINVAL, "null out");
  CUDA_TRY(cudaSetDevice(device));
  int num_sms = 0;
  int rc = check_sm90(device, &num_sms);
  if (rc) return rc;
  MlpHandle* h = new MlpHandle();
  h->cfg = *cfg;
  h->device = device;
  h->num_sms = num_sms;
  if (v1) { h->v1 = true; h->v1_bound = v1->bound; h->td_bound = v1->td_bound; }
  h->q.build(cfg->obs_dim + cfg->act_dim, cfg->hidden_q, cfg->n_hidden_q, 2);
  h->pi.build(cfg->obs_dim, cfg->hidden_pi, cfg->n_hidden_pi, pi_outputs(*cfg));
  h->ar.build(*cfg, h->q, h->pi, h->nq());
  h->slot = h->ar;
  h->hyper = StepHyper::of(*cfg);
  h->obs_elems = cfg->obs_dim; h->act_dim = cfg->act_dim; h->max_batch = cfg->max_batch;
  h->n_params = h->nq() * h->q.n + h->span().n + 1;
  h->arena_imaged = false;
  cudaError_t e = cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_pro_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_pro_join, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_dp_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_dp_join, cudaEventDisableTiming);
  if (e != cudaSuccess) { delete h; return fail(DSACT_ECUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e)); }
  *out = h;
  return DSACT_OK;
}

int dsact_create(const dsact_config* cfg, int device, dsact_handle** out) {
  int rc = validate(cfg);
  return rc ? rc : mlp_create(cfg, nullptr, device, out);
}

int dsact_v1_create(const dsact_config* cfg, const dsact_v1_options* v1, int device, dsact_handle** out) {
  int rc = validate(cfg);
  if (rc || (rc = validate_v1(cfg, v1))) return rc;
  return mlp_create(cfg, v1, device, out);
}

void dsact_destroy(dsact_handle* hh) {
  if (!hh) return;
  cudaSetDevice(hh->device);
  dp_peer_release(hh->dp);
  if (hh->engine == ENGINE_HEADS) { delete heads(hh); return; }
  MlpHandle* h = mlp(hh);
  drop_graphs(h);
  cudaStreamDestroy(h->cap_stream);
  cudaStreamDestroy(h->side_stream);
  cudaEventDestroy(h->ev_fork);
  cudaEventDestroy(h->ev_join);
  cudaEventDestroy(h->ev_pro_fork);
  cudaEventDestroy(h->ev_pro_join);
  cudaEventDestroy(h->ev_dp_fork);
  cudaEventDestroy(h->ev_dp_join);
  for (int t = 0; t < 2; ++t) {
    if (h->stage_buf[t]) cudaFree(h->stage_buf[t]);
    if (h->ev_stage_ready[t]) cudaEventDestroy(h->ev_stage_ready[t]);
    if (h->ev_stage_done[t]) cudaEventDestroy(h->ev_stage_done[t]);
  }
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  if (h->in2) cudaFree(h->in2);
  if (h->gather_stream) cudaStreamDestroy(h->gather_stream);
  if (h->ev_gather_fork) cudaEventDestroy(h->ev_gather_fork);
  if (h->ev_gather_join) cudaEventDestroy(h->ev_gather_join);
  delete h;
}

int dsact_bind(dsact_handle* h, const dsact_buffers* b) {
  if (!h || !b) return fail(DSACT_EINVAL, "null argument");
  if (!b->params || !b->targets || !b->grads || !b->adam_m || !b->adam_v || !b->act_high || !b->act_low || !b->state || !b->workspace)
    return fail(DSACT_EINVAL, "null buffer pointer");
  if ((reinterpret_cast<uintptr_t>(b->workspace) & 255) != 0) return fail(DSACT_EINVAL, "workspace must be 256-byte aligned");
  h->buf = *b;
  h->bound = true;
  h->dev_iter = -1;
  h->dev_rb_size = -1;
  if (h->engine != ENGINE_MLP) return DSACT_OK;
  MlpHandle* m = mlp(h);
  m->arena_imaged = false;
  drop_graphs(m);
  if (m->tc()) {  // bias regions of the wgrad slabs are never written by a kernel: they must read as zero
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaMemset(m->W() + m->ar.slabs, 0, sizeof(float) * (size_t)m->ar.nslabs * m->ar.slab_stride));
  }
  return DSACT_OK;
}

int dsact_set_output_activations(dsact_handle* h, int32_t value_act, int32_t policy_act) {
  if (!h) return fail(DSACT_EINVAL, "null handle");
  if (h->bound) return fail(DSACT_ESTATE, "dsact_set_output_activations: call it before dsact_bind");
  for (int32_t a : {value_act, policy_act})
    if (a < DSACT_ACT_LINEAR || a > DSACT_ACT_SELU) return fail(DSACT_EINVAL, "unknown output activation %d", a);
  // std_type "parameter": the log_std half is the learnable row, which the reference does not activate
  const bool ls_row = h->engine == ENGINE_MLP ? mlp(h)->cfg.policy_std == DSACT_STD_PARAMETER
                                              : static_cast<HeadsHandle*>(h)->pi.ls_row >= 0;
  h->oa = OutActs{value_act, policy_act, ls_row ? (int)DSACT_ACT_LINEAR : policy_act};
  return DSACT_OK;
}

int dsact_seed(dsact_handle* h, uint64_t seed) {
  if (!h) return fail(DSACT_EINVAL, "null handle");
  h->seed = seed;
  if (h->engine == ENGINE_MLP) drop_graphs(mlp(h));  // the seed is a baked kernel argument
  return DSACT_OK;
}

int dsact_set_carry(dsact_handle* h, float m1, float m2, int64_t tq, int64_t tp, void* stream) {
  if (!h || !h->bound) return fail(DSACT_ESTATE, "not bound");
  CUDA_TRY(cudaSetDevice(h->device));
  set_carry_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(h->buf.state, m1, m2, (int)tq, (int)tp);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return DSACT_OK;
}

int dsact_grad_phase1(dsact_handle* h, const dsact_batch* batch, const dsact_noise* noise, void* stream) {
  UpdateCall u("dsact_grad_phase1", RUN_PHASE1);
  u.batch = batch; u.noise = noise;
  return update(h, u, stream);
}

int dsact_grad_phase2(dsact_handle* h, int64_t global_batch, void* stream) {
  UpdateCall u("dsact_grad_phase2", RUN_PHASE2);
  u.global_batch = global_batch;
  return update(h, u, stream);
}

int dsact_compute_grads(dsact_handle* h, const dsact_batch* batch, const dsact_noise* noise, void* stream) {
  UpdateCall u("dsact_compute_grads", RUN_GRADS);
  u.batch = batch; u.noise = noise;
  return update(h, u, stream);
}

int dsact_apply(dsact_handle* h, int64_t iteration, void* stream) {
  UpdateCall u("dsact_apply", RUN_APPLY);
  u.iteration = iteration;
  return update(h, u, stream);
}

int dsact_step(dsact_handle* h, const dsact_batch* batch, const dsact_noise* noise, int64_t iteration, void* stream) {
  UpdateCall u("dsact_step", RUN_STEP);
  u.batch = batch; u.noise = noise; u.iteration = iteration;
  return update(h, u, stream);
}

// ---- host minibatches: staging on a private copy stream -------------------------------------------------------
int dsact_stage_host(dsact_handle* hh, const dsact_batch* host, dsact_batch* dev, void* stream) {
  int rc = check_mlp(hh, "dsact_stage_host");
  if (rc || (rc = check_batch(hh, host))) return rc;
  if (!dev) return fail(DSACT_EINVAL, "null out");
  MlpHandle* h = mlp(hh);
  CUDA_TRY(cudaSetDevice(h->device));
  const int64_t O = h->cfg.obs_dim, A = h->cfg.act_dim, Bm = h->cfg.max_batch;
  const int64_t seg[5] = {round64(Bm * O), round64(Bm * A), round64(Bm), round64(Bm * O), round64(Bm)};   // obs act rew obs2 done
  if (!h->copy_stream) {
    h->stage_floats = seg[0] + seg[1] + seg[2] + seg[3] + seg[4];
    CUDA_TRY(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int t = 0; t < 2; ++t) {
      CUDA_TRY(cudaMalloc(&h->stage_buf[t], sizeof(float) * (size_t)h->stage_floats));
      CUDA_TRY(cudaEventCreateWithFlags(&h->ev_stage_ready[t], cudaEventDisableTiming));
      CUDA_TRY(cudaEventCreateWithFlags(&h->ev_stage_done[t], cudaEventDisableTiming));
    }
  }
  const int t = h->stage_turn;
  const int64_t B = host->batch;
  float* base = h->stage_buf[t];
  float* d_obs = base; float* d_act = d_obs + seg[0]; float* d_rew = d_act + seg[1]; float* d_obs2 = d_rew + seg[2]; float* d_done = d_obs2 + seg[3];
  if (h->stage_done_valid[t]) CUDA_TRY(cudaStreamWaitEvent(h->copy_stream, h->ev_stage_done[t], 0));   // last reader of this set
  CUDA_TRY(cudaMemcpyAsync(d_obs, host->obs, sizeof(float) * B * O, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(cudaMemcpyAsync(d_obs2, host->obs2, sizeof(float) * B * O, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(cudaMemcpyAsync(d_act, host->act, sizeof(float) * B * A, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(cudaMemcpyAsync(d_rew, host->rew, sizeof(float) * B, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(cudaMemcpyAsync(d_done, host->done, sizeof(float) * B, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(cudaEventRecord(h->ev_stage_ready[t], h->copy_stream));
  CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)stream, h->ev_stage_ready[t], 0));
  dev->obs = d_obs; dev->act = d_act; dev->rew = d_rew; dev->obs2 = d_obs2; dev->done = d_done; dev->logp = nullptr;
  dev->batch = host->batch;
  h->stage_held = t;
  h->stage_turn = t ^ 1;
  return DSACT_OK;
}

int dsact_stage_release(dsact_handle* hh, void* stream) {
  if (!hh) return fail(DSACT_EINVAL, "null handle");
  int rc = check_mlp(hh, "dsact_stage_release");
  if (rc) return rc;
  MlpHandle* h = mlp(hh);
  if (h->stage_held < 0) return DSACT_OK;
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaEventRecord(h->ev_stage_done[h->stage_held], (cudaStream_t)stream));
  h->stage_done_valid[h->stage_held] = true;
  h->stage_held = -1;
  return DSACT_OK;
}

int dsact_step_host(dsact_handle* h, const dsact_batch* host, const dsact_noise* noise, int64_t iteration, void* stream) {
  int rc = check_mlp(h, "dsact_step_host");
  if (rc) return rc;
  dsact_batch dev;
  rc = dsact_stage_host(h, host, &dev, stream);
  if (rc) return rc;
  rc = dsact_step(h, &dev, noise, iteration, stream);
  const int rc2 = dsact_stage_release(h, stream);
  return rc ? rc : rc2;
}

int dsact_read_stats(dsact_handle* h, int64_t global_batch, float* host_out, void* stream) {
  if (!h || !h->bound) return fail(DSACT_ESTATE, "not bound");
  if (!host_out || global_batch < 1) return fail(DSACT_EINVAL, "bad argument");
  CUDA_TRY(cudaSetDevice(h->device));
  float inv_b, inv_pol;
  stats_scales(h, global_batch, &inv_b, &inv_pol);
  finalize_stats_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(h->buf.state, inv_b, inv_pol, nullptr);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  CUDA_TRY(cudaMemcpyAsync(host_out, h->buf.state + ST_STATS, DSACT_NUM_STATS * sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return DSACT_OK;
}

// ---- replay ring buffer ----------------------------------------------------------
int dsact_replay_bind(dsact_handle* h, const dsact_replay* rb) {
  if (!h || !rb) return fail(DSACT_EINVAL, "null argument");
  if (!rb->obs || !rb->obs2 || !rb->act || !rb->rew || !rb->done || !rb->logp || rb->capacity < 1)
    return fail(DSACT_EINVAL, "bad replay buffers");
  h->rb = *rb;
  h->rb_bound = true;
  h->rb_frames = false;
  h->rb_code_bytes = 0;
  if (h->engine == ENGINE_MLP) drop_graphs(mlp(h));
  return DSACT_OK;
}

// the shape and pointers of a frame ring of either kind (DSACT_OK, or DSACT_EINVAL with the reason)
static int check_frame_ring(const dsact_handle* h, const dsact_frame_replay* rb) {
  const int64_t K = rb->frames_per_obs;
  if (K < 1 || K > 64 || h->obs_elems % K != 0)
    return fail(DSACT_EINVAL, "frames_per_obs %lld must be in [1, 64] and divide obs_elems %lld", (long long)K,
                (long long)h->obs_elems);
  if (rb->frame_capacity < K || rb->frame_capacity > 0x7fffffff)
    return fail(DSACT_EINVAL, "frame_capacity %lld outside [frames_per_obs, 2^31 - 1]", (long long)rb->frame_capacity);
  if (rb->capacity < 1) return fail(DSACT_EINVAL, "capacity %lld < 1", (long long)rb->capacity);
  if (!rb->frames || !rb->obs_frames || !rb->obs2_frames || !rb->act || !rb->rew || !rb->done || !rb->logp)
    return fail(DSACT_EINVAL, "null frame-ring pointer");
  return DSACT_OK;
}

static int bind_frame_ring(dsact_handle* h, const dsact_frame_replay* rb, const float* table, int code_bytes) {
  h->fr = *rb;
  h->fr_table = const_cast<float*>(table);
  h->rb_bound = true;
  h->rb_frames = true;
  h->rb_code_bytes = code_bytes;
  if (h->engine == ENGINE_MLP) drop_graphs(mlp(h));
  return DSACT_OK;
}

int dsact_replay_bind_frames(dsact_handle* h, const dsact_frame_replay* rb) {
  if (!h || !rb) return fail(DSACT_EINVAL, "null argument");
  if (int rc = check_frame_ring(h, rb)) return rc;
  return bind_frame_ring(h, rb, nullptr, 0);
}

static int bind_coded_ring(dsact_handle* h, const dsact_frame_replay* rb, const float* table, int code_bytes) {
  if (!h || !rb) return fail(DSACT_EINVAL, "null argument");
  if (int rc = check_frame_ring(h, rb)) return rc;
  if (!table) return fail(DSACT_EINVAL, "null table");
  return bind_frame_ring(h, rb, table, code_bytes);
}

int dsact_replay_bind_coded_frames(dsact_handle* h, const dsact_frame_replay* rb, const float* table) {
  return bind_coded_ring(h, rb, table, 1);
}

int dsact_replay_bind_coded16_frames(dsact_handle* h, const dsact_frame_replay* rb, const float* table) {
  return bind_coded_ring(h, rb, table, 2);
}

// the first n entries of a HOST frame-id table (nullptr: not host memory, or an id outside [0, frame_capacity))
static const char* check_frame_ids(const int32_t* ids, int64_t n, int64_t frame_capacity) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, ids) != cudaSuccess) { cudaGetLastError(); return "not a valid pointer"; }
  if (at.type == cudaMemoryTypeDevice) return "device memory (frame-id tables must be host memory)";
  for (int64_t i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= frame_capacity) return "an id outside [0, frame_capacity)";
  return nullptr;
}

// the arguments of an add to a frame ring of either kind, every frame id included (DSACT_OK: nothing has been copied yet)
static int check_frame_rows(dsact_handle* h, const void* frames, int64_t n_frames, int64_t frame_ptr,
                            const int32_t* obs_frames, const int32_t* obs2_frames, const float* act, const float* rew,
                            const float* done, const float* logp, int64_t n, int64_t ptr) {
  const dsact_frame_replay& r = h->fr;
  if (n < 0 || n > r.capacity || ptr < 0 || ptr >= r.capacity) return fail(DSACT_EINVAL, "bad n/ptr");
  if (n_frames < 0 || n_frames > r.frame_capacity || frame_ptr < 0 || frame_ptr >= r.frame_capacity)
    return fail(DSACT_EINVAL, "bad n_frames/frame_ptr");
  if (n_frames > 0 && !frames) return fail(DSACT_EINVAL, "null frame staging pointer");
  if (n > 0 && (!obs_frames || !obs2_frames || !act || !rew || !done || !logp)) return fail(DSACT_EINVAL, "null staging pointer");
  const int64_t K = r.frames_per_obs;
  CUDA_TRY(cudaSetDevice(h->device));
  if (n > 0) {   // the gather follows these ids: every one is checked before anything is copied
    const char* bad = check_frame_ids(obs_frames, n * K, r.frame_capacity);
    if (!bad) bad = check_frame_ids(obs2_frames, n * K, r.frame_capacity);
    if (bad) return fail(DSACT_EINVAL, "frame-id table: %s", bad);
  }
  return DSACT_OK;
}

// the copies of a checked add: frames of F elements of `elem_bytes` each, and the rows
static int put_frame_rows(dsact_handle* h, const void* frames, size_t elem_bytes, int64_t n_frames, int64_t frame_ptr,
                          const int32_t* obs_frames, const int32_t* obs2_frames, const float* act, const float* rew,
                          const float* done, const float* logp, int64_t n, int64_t ptr, cudaStream_t s) {
  const dsact_frame_replay& r = h->fr;
  const int64_t K = r.frames_per_obs;
  // n items of w elements of `bytes` each from src into ring dst of `cap` items, starting at item p
  auto put = [&](void* dst, const void* src, int64_t cnt, int64_t p, int64_t cap, int64_t w, size_t bytes) -> cudaError_t {
    const int64_t first = (p + cnt <= cap) ? cnt : cap - p;
    cudaError_t e = cudaMemcpyAsync((char*)dst + p * w * bytes, src, first * w * bytes, cudaMemcpyDefault, s);
    if (e == cudaSuccess && first < cnt)
      e = cudaMemcpyAsync(dst, (const char*)src + first * w * bytes, (cnt - first) * w * bytes, cudaMemcpyDefault, s);
    return e;
  };
  if (n_frames > 0) CUDA_TRY(put(r.frames, frames, n_frames, frame_ptr, r.frame_capacity, h->obs_elems / K, elem_bytes));
  if (n > 0) {
    CUDA_TRY(put(r.obs_frames, obs_frames, n, ptr, r.capacity, K, sizeof(int32_t)));
    CUDA_TRY(put(r.obs2_frames, obs2_frames, n, ptr, r.capacity, K, sizeof(int32_t)));
    CUDA_TRY(put(r.act, act, n, ptr, r.capacity, h->act_dim, sizeof(float)));
    CUDA_TRY(put(r.rew, rew, n, ptr, r.capacity, 1, sizeof(float)));
    CUDA_TRY(put(r.done, done, n, ptr, r.capacity, 1, sizeof(float)));
    CUDA_TRY(put(r.logp, logp, n, ptr, r.capacity, 1, sizeof(float)));
  }
  return DSACT_OK;
}

int dsact_replay_add_frames(dsact_handle* h, const float* frames, int64_t n_frames, int64_t frame_ptr,
                            const int32_t* obs_frames, const int32_t* obs2_frames, const float* act, const float* rew,
                            const float* done, const float* logp, int64_t n, int64_t ptr, void* stream) {
  if (!h || !h->rb_bound || !h->rb_frames) return fail(DSACT_ESTATE, "frame replay ring not bound");
  if (h->rb_code_bytes)
    return fail(DSACT_ESTATE, "a coded frame ring is bound: frames go in through dsact_replay_add_coded%s_frames",
                h->rb_code_bytes == 2 ? "16" : "");
  if (int rc = check_frame_rows(h, frames, n_frames, frame_ptr, obs_frames, obs2_frames, act, rew, done, logp, n, ptr)) return rc;
  return put_frame_rows(h, frames, sizeof(float), n_frames, frame_ptr, obs_frames, obs2_frames, act, rew, done, logp, n, ptr,
                        (cudaStream_t)stream);
}

// an add to a coded ring of `Code` codes (uint8_t: dsact_replay_add_coded_frames, uint16_t: ..._coded16_frames)
extern "C++" template <typename Code>
int add_coded_frames(dsact_handle* h, const Code* codes, int64_t n_frames, int64_t frame_ptr, const float* table,
                     int32_t n_codes, const int32_t* obs_frames, const int32_t* obs2_frames, const float* act,
                     const float* rew, const float* done, const float* logp, int64_t n, int64_t ptr, void* stream) {
  constexpr int bytes = (int)sizeof(Code), max_codes = 1 << (8 * bytes);
  if (!h || !h->rb_bound || h->rb_code_bytes != bytes)
    return fail(DSACT_ESTATE, "%scoded frame replay ring not bound", bytes == 2 ? "16-bit " : "");
  if (n_codes < 0 || n_codes > max_codes) return fail(DSACT_EINVAL, "n_codes %d outside [0, %d]", (int)n_codes, max_codes);
  if (n_codes > 0 && !table) return fail(DSACT_EINVAL, "null table");
  if (int rc = check_frame_rows(h, codes, n_frames, frame_ptr, obs_frames, obs2_frames, act, rew, done, logp, n, ptr)) return rc;
  if (n_frames > 0) {   // the gather decodes through these codes: every one is checked before anything is copied
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, codes) != cudaSuccess) { cudaGetLastError(); return fail(DSACT_EINVAL, "codes: not a valid pointer"); }
    if (at.type == cudaMemoryTypeDevice) return fail(DSACT_EINVAL, "codes: device memory (staged codes must be host memory)");
    const int64_t m = n_frames * (h->obs_elems / h->fr.frames_per_obs);
    for (int64_t i = 0; i < m; ++i)
      if (codes[i] >= n_codes) return fail(DSACT_EINVAL, "codes: code %d at %lld is not below n_codes %d", (int)codes[i], (long long)i, (int)n_codes);
  }
  const cudaStream_t s = (cudaStream_t)stream;
  if (n_codes > 0) CUDA_TRY(cudaMemcpyAsync(h->fr_table, table, n_codes * sizeof(float), cudaMemcpyDefault, s));
  return put_frame_rows(h, codes, bytes, n_frames, frame_ptr, obs_frames, obs2_frames, act, rew, done, logp, n, ptr, s);
}

int dsact_replay_add_coded_frames(dsact_handle* h, const uint8_t* codes, int64_t n_frames, int64_t frame_ptr,
                                  const float* table, int32_t n_codes, const int32_t* obs_frames, const int32_t* obs2_frames,
                                  const float* act, const float* rew, const float* done, const float* logp, int64_t n,
                                  int64_t ptr, void* stream) {
  return add_coded_frames(h, codes, n_frames, frame_ptr, table, n_codes, obs_frames, obs2_frames, act, rew, done, logp, n,
                          ptr, stream);
}

int dsact_replay_add_coded16_frames(dsact_handle* h, const uint16_t* codes, int64_t n_frames, int64_t frame_ptr,
                                    const float* table, int32_t n_codes, const int32_t* obs_frames,
                                    const int32_t* obs2_frames, const float* act, const float* rew, const float* done,
                                    const float* logp, int64_t n, int64_t ptr, void* stream) {
  return add_coded_frames(h, codes, n_frames, frame_ptr, table, n_codes, obs_frames, obs2_frames, act, rew, done, logp, n,
                          ptr, stream);
}

int dsact_replay_add(dsact_handle* h, const float* obs, const float* obs2, const float* act, const float* rew,
                     const float* done, const float* logp, int64_t n, int64_t ptr, void* stream) {
  if (!h || !h->rb_bound) return fail(DSACT_ESTATE, "replay buffer not bound");
  if (h->rb_frames) return fail(DSACT_ESTATE, "a frame replay ring is bound: rows go in through dsact_replay_add_frames");
  if (n < 0 || n > h->rb.capacity || ptr < 0 || ptr >= h->rb.capacity) return fail(DSACT_EINVAL, "bad n/ptr");
  if (n == 0) return DSACT_OK;
  if (!obs || !obs2 || !act || !rew || !done || !logp) return fail(DSACT_EINVAL, "null staging pointer");
  CUDA_TRY(cudaSetDevice(h->device));
  const int64_t first = (ptr + n <= h->rb.capacity) ? n : h->rb.capacity - ptr;
  const int64_t O = h->obs_elems, A = h->act_dim;
  struct { float* dst; const float* src; int64_t w; } cols[6] = {
      {h->rb.obs, obs, O}, {h->rb.obs2, obs2, O}, {h->rb.act, act, A}, {h->rb.rew, rew, 1}, {h->rb.done, done, 1}, {h->rb.logp, logp, 1}};
  for (auto& c : cols) {
    CUDA_TRY(cudaMemcpyAsync(c.dst + ptr * c.w, c.src, first * c.w * sizeof(float), cudaMemcpyDefault, (cudaStream_t)stream));
    if (first < n)
      CUDA_TRY(cudaMemcpyAsync(c.dst, c.src + first * c.w, (n - first) * c.w * sizeof(float), cudaMemcpyDefault, (cudaStream_t)stream));
  }
  return DSACT_OK;
}

int dsact_replay_sample(dsact_handle* h, int32_t batch, int64_t size, const int64_t* idx, dsact_batch* out, void* stream) {
  UpdateCall u("dsact_replay_sample", RUN_GATHER);
  u.replay = true; u.rows = batch; u.size = size; u.idx = idx; u.out = out;
  return update(h, u, stream);
}

int dsact_replay_step(dsact_handle* h, int32_t batch, int64_t size, const int64_t* idx, const dsact_noise* noise,
                      int64_t iteration, void* stream) {
  UpdateCall u("dsact_replay_step", RUN_STEP);
  u.replay = true; u.rows = batch; u.size = size; u.idx = idx; u.noise = noise; u.iteration = iteration;
  return update(h, u, stream);
}

int dsact_replay_steps(dsact_handle* h, int32_t n_steps, int32_t batch, int64_t size, const int64_t* idx,
                       const dsact_noise* noise, float* stats_out, int64_t iteration, void* stream) {
  UpdateCall u("dsact_replay_steps", RUN_STEPS);
  u.replay = true; u.rows = batch; u.size = size; u.idx = idx; u.noise = noise; u.iteration = iteration;
  u.n_steps = n_steps; u.stats_out = stats_out;
  return update(h, u, stream);
}

// ---- data parallelism over peer memory (dp_peer.cuh) ------------------------------------------------------------
// After a (re)connect: captured data-parallel steps hold the previous peer map, and the MLP engine allocates the second
// input set of dsact_dp_replay_steps here rather than in the first call.  There its cudaMalloc and cudaMemset would sit
// between the ranks' enqueues, and CUDA does not run work issued before such calls beside work issued after them: ranks
// that share a device would wait on each other until their exchanges timed out.
static int dp_connected(dsact_handle* h) {
  if (h->engine != ENGINE_MLP) return DSACT_OK;
  drop_graphs(mlp(h));
  return ensure_input_set2(mlp(h));
}

int dsact_dp_export(dsact_handle* h, void* handle_out, int64_t* bytes_out) {
  if (!h || !handle_out) return fail(DSACT_EINVAL, "null argument");
  int rc = check_dp(h);
  if (rc) return rc;
  return dp_peer_export(h->dp, h->device, h->n_params, handle_out, bytes_out);
}

int dsact_dp_connect(dsact_handle* h, int32_t rank, int32_t world, const void* handles) {
  if (!h || !handles) return fail(DSACT_EINVAL, "null argument");
  if (!h->bound) return fail(DSACT_ESTATE, "dsact_bind has not been called");
  int rc = check_dp(h);
  if (rc) return rc;
  if (!h->dp.buf) return fail(DSACT_ESTATE, "dsact_dp_export has not been called");
  rc = dp_peer_connect(h->dp, h->device, h->buf.state, rank, world, handles);
  return rc ? rc : dp_connected(h);
}

// One data-parallel update as one submission: forward, std-sum exchange, losses + backward scaled by 1/global_batch,
// gradient + statistics exchange, Adam on the rank-ordered global sum.  Every rank must call it for the same iteration.
int dsact_dp_step(dsact_handle* h, const dsact_batch* batch, const dsact_noise* noise, int64_t global_batch, int64_t iteration,
                  void* stream) {
  UpdateCall u("dsact_dp_step", RUN_STEP);
  u.batch = batch; u.noise = noise; u.iteration = iteration; u.global_batch = global_batch; u.dp = true;
  return update(h, u, stream);
}

int dsact_dp_replay_step(dsact_handle* h, int32_t batch, int64_t size, const int64_t* idx, const dsact_noise* noise,
                         int64_t global_batch, int64_t iteration, void* stream) {
  UpdateCall u("dsact_dp_replay_step", RUN_STEP);
  u.replay = true; u.rows = batch; u.size = size; u.idx = idx; u.noise = noise; u.iteration = iteration;
  u.global_batch = global_batch; u.dp = true;
  return update(h, u, stream);
}

int dsact_dp_replay_steps(dsact_handle* h, int32_t n_steps, int32_t batch, int64_t size, const int64_t* idx,
                          const dsact_noise* noise, int64_t global_batch, float* stats_out, int64_t iteration, void* stream) {
  UpdateCall u("dsact_dp_replay_steps", RUN_STEPS);
  u.replay = true; u.rows = batch; u.size = size; u.idx = idx; u.noise = noise; u.iteration = iteration;
  u.n_steps = n_steps; u.stats_out = stats_out; u.global_batch = global_batch; u.dp = true;
  return update(h, u, stream);
}

int dsact_profile_step(dsact_handle* h, const dsact_batch* batch, const dsact_noise* noise, int64_t iteration,
                       void* stream, dsact_profile* out) {
  UpdateCall u("dsact_profile_step", RUN_STEP);
  u.batch = batch; u.noise = noise; u.iteration = iteration; u.profiled = true; u.prof = out;
  return update(h, u, stream);
}

int64_t dsact_launch_count(const dsact_handle* h) { return h ? h->launches : 0; }
int32_t dsact_last_call_launches(const dsact_handle* h) { return h ? h->last_launches : 0; }

// Scratch of the test hooks: one cudaMalloc per image or slab region, freed when the hook returns (after its stream has
// been synchronised).
struct HookScratch {
  std::vector<void*> mem;
  cudaError_t err = cudaSuccess;
  void* get(size_t bytes) {
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) { if (err == cudaSuccess) err = e; return nullptr; }
    mem.push_back(p);
    return p;
  }
  Img img(int rows, int width) {   // the arena's image geometry
    Img i;
    i.rows = rows; i.width = width; i.pitch = (width + 7) / 8 * 8; i.plane = round64((int64_t)rows * i.pitch);
    i.p = static_cast<__nv_bfloat16*>(get((size_t)i.plane * 4));
    return i;
  }
  ~HookScratch() { for (void* p : mem) cudaFree(p); }
};

static int finish_hook(MlpHandle* h, Ctx& c, const HookScratch& mem) {
  const cudaError_t e = cudaStreamSynchronize(c.s);
  const cudaError_t err = mem.err != cudaSuccess ? mem.err : (c.err != cudaSuccess ? c.err : e);
  if (err != cudaSuccess) return fail(DSACT_ECUDA, "launch failed: %s", cudaGetErrorString(err));
  h->launches += c.launches;
  return DSACT_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int dsact_test_gemm(dsact_handle* hh, int32_t variant, const dsact_test_layer* probs, int32_t n, int32_t max_ctas, void* stream) {
  if (!hh) return fail(DSACT_EINVAL, "null handle");
  int rc = check_mlp(hh, "dsact_test_gemm");
  if (rc) return rc;
  MlpHandle* h = mlp(hh);
  if (variant < 0 || variant > 2 || !probs || n < 1 || n > TC_MAXG || max_ctas < 0) return fail(DSACT_EINVAL, "bad argument");
  const bool tc = h->tc();
  for (int i = 0; i < n; ++i) {
    const dsact_test_layer& t = probs[i];
    const int epi_ok = variant == V_FWD ? EPI_BIAS_ACT : (variant == V_DGRAD ? EPI_DACT : EPI_STORE);
    if (t.M < 1 || t.N < 1 || t.K0 < 1 || t.K1 < 0 || !t.A0 || !t.B || (!t.C && !t.img) || t.act < 0 || t.act > ACT_SELU ||
        (t.epi != EPI_STORE && t.epi != epi_ok))
      return fail(DSACT_EINVAL, "problem %d: bad argument", i);
    if (t.K1 > 0 && (variant != V_FWD || !t.A1 || t.kB1 < t.K0 || t.kB1 % 8))
      return fail(DSACT_EINVAL, "problem %d: a second K segment needs the forward variant, A1 and kB1 >= K0, kB1 %% 8 == 0", i);
    if (t.epi == EPI_DACT && !t.Zin) return fail(DSACT_EINVAL, "problem %d: the derivative epilogue needs Zin", i);
    if (t.img && (!tc || variant == V_WGRAD || t.img_pitch < (t.N + 7) / 8 * 8 || t.img_pitch % 8 || t.img_plane < (int64_t)t.M * t.img_pitch))
      return fail(DSACT_EINVAL, "problem %d: bad output image", i);
    if (tc && variant == V_WGRAD && (t.ldc != t.N || !aligned16(t.C)))
      return fail(DSACT_EINVAL, "problem %d: the tensor-core weight gradient needs a contiguous, 16-byte aligned C", i);
  }
  CUDA_TRY(cudaSetDevice(h->device));
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  c.pdl = tc;
  HookScratch mem;
  ImgBatch ibt;
  Group G;
  long long slab_floats = 0;
  for (int i = 0; i < n; ++i) {
    const dsact_test_layer& t = probs[i];
    GemmProb p = prob_zero();
    TcExtra x;
    p.A[0] = t.A0; p.lda[0] = t.lda0; p.K[0] = t.K0;
    p.B[0] = t.B; p.ldb[0] = t.ldb;
    if (t.K1 > 0) { p.A[1] = t.A1; p.lda[1] = t.lda1; p.K[1] = t.K1; p.B[1] = t.B + t.K0; p.ldb[1] = t.ldb; x.kB0[1] = t.kB1; }
    p.M = t.M; p.N = t.N; p.C = t.C; p.ldc = t.ldc;
    p.epi = variant == V_WGRAD ? EPI_ATOMIC : t.epi; p.act = t.act;
    if (variant != V_WGRAD) { p.bias = t.bias; p.Zout = t.Zout; p.Zin = t.Zin; p.ldz = t.ldz; p.colsum = t.colsum; }
    if (tc) {   // images as the step forms them: operands by image_kernel, the B segments at their image columns
      const int a_rows = variant == V_WGRAD ? t.K0 : t.M, a_w = variant == V_WGRAD ? t.M : t.K0;
      ibt.reserve(h, c, 3);
      x.a[0] = mem.img(a_rows, a_w);
      ibt.add(t.A0, t.lda0, x.a[0], a_rows, a_w);
      if (t.K1 > 0) { x.a[1] = mem.img(t.M, t.K1); ibt.add(t.A1, t.lda1, x.a[1], t.M, t.K1); }
      if (variant == V_FWD) {
        x.b = mem.img(t.N, t.K1 > 0 ? t.kB1 + t.K1 : t.K0);
        ibt.add(t.B, t.ldb, x.b, t.N, t.K0, t.K1, t.kB1);
      } else {
        x.b = mem.img(t.K0, t.N);
        ibt.add(t.B, t.ldb, x.b, t.K0, t.N);
      }
      if (t.img) {
        x.out.p = static_cast<__nv_bfloat16*>(t.img); x.out.rows = t.M; x.out.width = t.N;
        x.out.pitch = t.img_pitch; x.out.plane = t.img_plane;
      }
      G.wg_off[i] = slab_floats;
      if (variant == V_WGRAD) slab_floats += ((long long)t.M * t.N + 3) / 4 * 4;
    }
    G.push(p, x);
  }
  const int nslabs = 4;
  if (tc) {
    ibt.launch(h, c);
    if (variant == V_WGRAD) {
      G.wg_slab = static_cast<float*>(mem.get(sizeof(float) * (size_t)nslabs * slab_floats));
      G.wg_stride = slab_floats; G.wg_nslabs = nslabs;
      // NaN: a slab element the kernel leaves unwritten reaches C
      if (G.wg_slab) c.err = cudaMemsetAsync(G.wg_slab, 0xff, sizeof(float) * (size_t)nslabs * slab_floats, c.s);
    }
  }
  if (mem.err == cudaSuccess) launch_group(h, G, variant, c, max_ctas);
  if (tc && variant == V_WGRAD && c.err == cudaSuccess && mem.err == cudaSuccess) {
    for (int i = 0; i < n; ++i) {
      grad_reduce_kernel<<<64, 256, 0, c.s>>>(probs[i].C, G.wg_slab + G.wg_off[i], (long long)probs[i].M * probs[i].N, nslabs,
                                               G.wg_stride);
      c.done();
    }
    c.check();
  }
  return finish_hook(h, c, mem);
}

static int test_chain(dsact_handle* hh, int tiling, int32_t dgrad, int32_t L, const int32_t* sizes, int32_t K0, int32_t K1,
                      int32_t kB1, int32_t act, const float* params, const dsact_test_chain_pass* passes, int32_t n_passes,
                      void* stream) {
  if (!hh) return fail(DSACT_EINVAL, "null handle");
  int rc = check_mlp(hh, "dsact_test_chain");
  if (rc) return rc;
  MlpHandle* h = mlp(hh);
  if (!h->tc()) return fail(DSACT_EINVAL, "dsact_test_chain: the layer-chain kernel runs in the tensor-core modes only");
  if (!sizes || !params || !passes || L < 0 || L > DSACT_MAX_HIDDEN || n_passes < 1 || n_passes > CH_MAX_PASSES ||
      act < 0 || act > ACT_SELU || (dgrad != 0 && dgrad != 1) || (dgrad && L < 1))
    return fail(DSACT_EINVAL, "bad argument");
  for (int j = 0; j <= L + 1; ++j)
    if (sizes[j] < 1 || (j > 0 && sizes[j] > 256) || (j > 0 && j <= L && sizes[j] % 8))
      return fail(DSACT_EINVAL, "sizes[%d] = %d: widths are >= 1, layer outputs <= 256, hidden widths multiples of 8", j, sizes[j]);
  if (K0 < 1 || K1 < 0 || K0 + K1 != sizes[0] || (K1 > 0 && (kB1 < K0 || kB1 % 8)))
    return fail(DSACT_EINVAL, "layer-0 segments: K0 + K1 == sizes[0], kB1 >= K0, kB1 %% 8 == 0");
  for (int i = 0; i < n_passes; ++i) {
    const dsact_test_chain_pass& q = passes[i];
    if (q.M < 1 || !q.x0 || (!dgrad && (!q.out || (K1 > 0 && !q.x1))) || (dgrad && q.out && K1 == 0) ||
        (q.out_ld != 0 && (dgrad || q.out_ld < sizes[L + 1])))
      return fail(DSACT_EINVAL, "pass %d: bad argument", i);
    for (int j = 0; j < L && dgrad; ++j)
      if (!q.Zin[j]) return fail(DSACT_EINVAL, "pass %d: Zin[%d] is null", i, j);
  }
  CUDA_TRY(cudaSetDevice(h->device));
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  HookScratch mem;
  ImgBatch ibt;
  Net net;
  net.build(sizes[0], sizes + 1, L, sizes[L + 1]);
  ChainIo io;
  for (int j = 0; j <= L; ++j) {   // weight images: layer 0's second segment at column kB1, as the critics' in the step
    io.w[j] = mem.img(sizes[j + 1], j == 0 && K1 > 0 ? kB1 + K1 : sizes[j]);
    ibt.reserve(h, c, 1);
    if (j == 0) ibt.add(params + net.w[0], sizes[0], io.w[0], sizes[1], K0, K1, kB1);
    else ibt.add(params + net.w[j], sizes[j], io.w[j], sizes[j + 1], sizes[j]);
  }
  ChainBuild cb(h->passes());
  for (int i = 0; i < n_passes; ++i) {
    const dsact_test_chain_pass& q = passes[i];
    ChainIo pio = io;
    for (int j = 0; j < L; ++j) {
      pio.z[j] = dgrad ? const_cast<float*>(q.Zin[j]) : q.Zout[j];
      pio.colsum[j] = dgrad ? q.colsum[j] : nullptr;
      if (q.img[j]) {
        Img& o = pio.img[j];
        o.p = static_cast<__nv_bfloat16*>(q.img[j]); o.rows = q.M; o.width = sizes[j + 1];
        o.pitch = (sizes[j + 1] + 7) / 8 * 8; o.plane = (long long)o.pitch * q.M;
      }
    }
    const int w0 = dgrad ? sizes[L + 1] : K0;
    ibt.reserve(h, c, 2);
    const Img in0 = mem.img(q.M, w0);
    ibt.add(q.x0, w0, in0, q.M, w0);
    if (dgrad) {
      chain_dgrad_layers(cb, net, pio, in0, q.M, act, q.out, kB1, K1);
    } else {
      Img in1;
      if (K1 > 0) { in1 = mem.img(q.M, K1); ibt.add(q.x1, K1, in1, q.M, K1); }
      chain_fwd_layers(cb, net, params, pio, in0, K0, in1, K1, kB1, q.M, act, q.out, q.out_ld);
    }
  }
  if (mem.err == cudaSuccess) {
    ibt.launch(h, c);
    launch_chain(h, cb, dgrad ? CLS_GEMM_DGRAD : CLS_GEMM_FWD, c, tiling);
  }
  return finish_hook(h, c, mem);
}

int dsact_test_chain(dsact_handle* h, int32_t dgrad, int32_t L, const int32_t* sizes, int32_t K0, int32_t K1, int32_t kB1,
                     int32_t act, const float* params, const dsact_test_chain_pass* passes, int32_t n_passes, void* stream) {
  return test_chain(h, CHAIN_BY_SHAPE, dgrad, L, sizes, K0, K1, kB1, act, params, passes, n_passes, stream);
}

int dsact_test_chain_tiling(dsact_handle* h, int32_t tiling, int32_t dgrad, int32_t L, const int32_t* sizes, int32_t K0,
                            int32_t K1, int32_t kB1, int32_t act, const float* params, const dsact_test_chain_pass* passes,
                            int32_t n_passes, void* stream) {
  if (tiling != CHAIN_COLUMN_SPLIT && tiling != CHAIN_PINGPONG)
    return fail(DSACT_EINVAL, "dsact_test_chain_tiling: tiling %d is neither 0 (column split) nor 1 (ping-pong)", tiling);
  return test_chain(h, tiling, dgrad, L, sizes, K0, K1, kB1, act, params, passes, n_passes, stream);
}

static int sync_hook(dsact_handle* h, Ctx& c) {
  const cudaError_t e = cudaStreamSynchronize(c.s);
  const cudaError_t err = c.err != cudaSuccess ? c.err : e;
  if (err != cudaSuccess) return fail(DSACT_ECUDA, "launch failed: %s", cudaGetErrorString(err));
  h->launches += c.launches;
  return DSACT_OK;
}

int dsact_test_rows(dsact_handle* h, const dsact_test_row_io* t, void* stream) {
  if (!h || !h->bound) return fail(DSACT_ESTATE, "not bound");
  if (!t) return fail(DSACT_EINVAL, "null rows");
  if (t->kernel < DSACT_TEST_SAMPLE || t->kernel > DSACT_TEST_STATS) return fail(DSACT_EINVAL, "unknown kernel %d", t->kernel);
  const int B = t->batch;
  if (t->kernel != DSACT_TEST_STATS && (B < 1 || B > h->max_batch)) return fail(DSACT_EINVAL, "batch %d outside [1, max_batch]", B);
  if (t->global_batch < (t->kernel == DSACT_TEST_STATS ? 1 : B)) return fail(DSACT_EINVAL, "global_batch < batch");
  if (t->max_blocks < 0) return fail(DSACT_EINVAL, "max_blocks < 0");
  const bool v1 = h->v1, mlp_eng = h->engine == ENGINE_MLP;
  const bool tc = mlp_eng && mlp(h)->tc();
  const int A = h->act_dim, nq = v1 ? 1 : 2;
  const void* imgs[8] = {t->img_act[0], t->img_act[1], t->img_q[0], t->img_q[1], t->img_qa[0], t->img_qa[1], t->img_dlogits,
                         t->img_dlogits_ls};
  for (const void* p : imgs)
    if (p && !tc) return fail(DSACT_EINVAL, "images need a tensor-core mode of the MLP engine");
  auto need = [&](const void* p, const char* what) { return p ? DSACT_OK : fail(DSACT_EINVAL, "%s is null", what); };
  int rc = DSACT_OK;
  RowIo io;
  memset(&io, 0, sizeof(io));
  auto img = [&](void* p, int width) {
    if (!p) return NO_IMG;
    ImgOut o;
    o.p = static_cast<__nv_bfloat16*>(p); o.pitch = (width + 7) / 8 * 8; o.planes = mlp(h)->passes() == 3 ? 2 : 1;
    o.plane = (long long)B * o.pitch;
    return o;
  };
  for (int k = 0; k < 2; ++k) {
    io.logits[k] = t->logits[k]; io.eps[k] = t->eps[k]; io.act[k] = t->act[k]; io.logp[k] = t->logp[k];
    io.d_out_q[k] = t->d_out_q[k]; io.d_out_qa[k] = t->d_out_qa[k];
    io.gbias_q[k] = t->gbias_q[k]; io.gbias_q_raw[k] = t->gbias_q_raw[k];
    io.img_act[k] = img(t->img_act[k], A); io.img_q[k] = img(t->img_q[k], 2); io.img_qa[k] = img(t->img_qa[k], 2);
  }
  for (int p = 0; p < 6; ++p) io.out_q[p] = t->out_q[p];
  io.rew = t->rew; io.done = t->done; io.z3 = t->z3; io.z4 = t->z4;
  // the step's choice of policy_grad_kernel<1 | 2>: one critic only where the handle has no second action-gradient slot
  io.d_act[0] = t->d_act[0]; io.d_act[1] = h->slot.dAct[1] < 0 ? nullptr : t->d_act[1];
  io.d_logits = t->d_logits; io.gbias_pi = t->gbias_pi; io.gbias_ls = t->gbias_ls;
  io.split_dlogits = t->split_dlogits != 0;
  io.img_dlogits = img(t->img_dlogits, io.split_dlogits ? A : 2 * A);
  io.img_dlogits_ls = io.split_dlogits ? img(t->img_dlogits_ls, A) : NO_IMG;
  if (t->kernel == DSACT_TEST_SAMPLE) {
    for (int k = 0; k < 2 && !rc; ++k)
      if (!(rc = need(io.logits[k], "logits")) && !(rc = need(io.eps[k], "eps")) && !(rc = need(io.act[k], "act")))
        rc = need(io.logp[k], "logp");
    for (int k = 0; k < nq && !rc; ++k) rc = need(io.out_q[k], "out_q");
  } else if (t->kernel == DSACT_TEST_LOSS) {
    const void* in[5] = {io.rew, io.done, io.z3, io.logp[0], io.logp[1]};
    for (const void* p : in) if (!rc) rc = need(p, "a row input");
    if (!rc && !v1) rc = need(io.z4, "z4");
    for (int k = 0; k < nq && !rc; ++k)
      if (!(rc = need(io.out_q[k], "out_q")) && !(rc = need(io.out_q[2 + k], "out_q")) && !(rc = need(io.out_q[4 + k], "out_q")) &&
          !(rc = need(io.d_out_q[k], "d_out_q")) && !(rc = need(io.d_out_qa[k], "d_out_qa")))
        rc = need(io.gbias_q[k], "gbias_q");
  } else if (t->kernel == DSACT_TEST_POLICY_GRAD) {
    if (!(rc = need(io.logits[0], "logits")) && !(rc = need(io.eps[0], "eps")) && !(rc = need(io.d_act[0], "d_act")) &&
        !(rc = need(io.d_logits, "d_logits")) && !(rc = need(io.gbias_pi, "gbias_pi")) && h->slot.dAct[1] >= 0)
      rc = need(io.d_act[1], "d_act[1]");
  }
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(h->device));
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  c.pdl = tc;
  const StepScalars sc = step_scalars(h, t->global_batch);
  if (t->kernel == DSACT_TEST_SAMPLE) {
    enqueue_sample(h, io, B, t->advance_rng != 0, c, t->max_blocks);
  } else if (t->kernel == DSACT_TEST_LOSS) {
    if (v1) enqueue_loss_v1(h, io, B, sc, c, t->max_blocks);
    else enqueue_loss(h, io, B, sc, c, t->max_blocks);
  } else if (t->kernel == DSACT_TEST_POLICY_GRAD) {
    enqueue_policy_grad(h, io, B, sc, c, t->max_blocks);
  } else {
    float inv_b, inv_pol;
    stats_scales(h, t->global_batch, &inv_b, &inv_pol);
    launch_k(finalize_stats_kernel, 1, 32, 0, c, h->buf.state, inv_b, inv_pol, t->stats_out);
    c.done();
  }
  c.check();
  return sync_hook(h, c);
}

int dsact_test_apply(dsact_handle* h, int32_t part, int32_t fold_slabs, int32_t scalars_ready, int32_t tail_rows,
                     int64_t global_batch, int32_t max_blocks, void* stream) {
  if (!h || !h->bound) return fail(DSACT_ESTATE, "not bound");
  if (part < 0 || part > 2) return fail(DSACT_EINVAL, "part %d outside 0..2", part);
  if (scalars_ready < 0 || scalars_ready > 2) return fail(DSACT_EINVAL, "scalars_ready %d outside 0..2", scalars_ready);
  if (max_blocks < 0 || tail_rows < 0 || (tail_rows > 0 && global_batch < tail_rows)) return fail(DSACT_EINVAL, "bad argument");
  const bool mlp_eng = h->engine == ENGINE_MLP;
  const int max_slabs = mlp_eng && slabs_foldable(mlp(h)) ? mlp(h)->ar.nslabs : 0;
  if (fold_slabs < 0 || fold_slabs > max_slabs)
    return fail(DSACT_EINVAL, "fold_slabs %d outside [0, %d] (the weight-gradient slabs of this handle)", fold_slabs, max_slabs);
  CUDA_TRY(cudaSetDevice(h->device));
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  c.pdl = mlp_eng && mlp(h)->tc();
  const TailArgs ta = tail_args(h, tail_rows > 0 ? global_batch : 1, tail_rows);
  const TailArgs* tail = tail_rows > 0 ? &ta : nullptr;
  ApplyArgs a;
  if (mlp_eng) {
    a = mlp_apply_args(mlp(h), scalars_ready, tail, false, part, fold_slabs);
  } else {
    a = apply_args(h, heads(h)->nq() * heads(h)->q.n, scalars_ready, false);
    if (tail) a.tail = *tail;
    apply_part(a, part);
  }
  launch_apply(h, a, c, max_blocks);
  return sync_hook(h, c);
}

// ---- test hooks of the peer-memory exchange: every rank of a world on one device -------------------------------------
static int check_dp_hook(const dsact_handle* h) {
  if (!h || !h->bound) return fail(DSACT_ESTATE, "not bound");
  return check_dp(h);
}

int dsact_test_dp_attach(dsact_handle* h, int32_t rank, int32_t world, dsact_handle* const* peers, void** buffer, int64_t* floats) {
  if (world < 2 || world > DP_MAX_RANKS || rank < 0 || rank >= world)
    return fail(DSACT_EINVAL, "rank %d / world %d outside [2, %d]", rank, world, DP_MAX_RANKS);
  if (!peers) return fail(DSACT_EINVAL, "null peers");
  int rc = check_dp_hook(h);
  if (rc) return rc;
  if (peers[rank] != h) return fail(DSACT_EINVAL, "peers[%d] is not the handle being attached", rank);
  for (int r = 0; r < world; ++r) {
    const dsact_handle* p = peers[r];
    if (!p || !p->dp.buf) return fail(DSACT_ESTATE, "peer %d has not called dsact_dp_export", r);
    if (p->device != h->device || p->engine != h->engine || p->dp.n_params != h->dp.n_params)
      return fail(DSACT_EINVAL, "peer %d is on another device or engine, or has another parameter count", r);
  }
  if ((rc = dp_peer_reset(h->dp, h->device, rank, world))) return rc;
  for (int r = 0; r < world; ++r) h->dp.comm.peer[r] = peers[r]->dp.buf;
  if ((rc = dp_peer_start(h->dp, h->buf.state)) || (rc = dp_connected(h))) return rc;
  if (buffer) *buffer = h->dp.buf;
  if (floats) *floats = DP_GRADS_OFF + 2 * h->dp.npad();
  return DSACT_OK;
}

int dsact_test_dp(dsact_handle* h, int32_t op, const dsact_test_dp_io* io, void* stream) {
  if (op < DSACT_TEST_DP_EXCHANGE || op > DSACT_TEST_DP_APPLY) return fail(DSACT_EINVAL, "unknown op %d", op);
  if (!io) return fail(DSACT_EINVAL, "null io");
  int rc = check_dp_hook(h);
  if (rc) return rc;
  if (!h->dp.ready) return fail(DSACT_ESTATE, "not attached (dsact_test_dp_attach)");
  const DpPeer& dp = h->dp;
  const int world = dp.comm.world;
  const bool mlp_eng = h->engine == ENGINE_MLP;
  DpTestWorld w;
  memset(&w, 0, sizeof(w));
  if (op == DSACT_TEST_DP_EXCHANGE) {
    if (io->kind != 0 && io->kind != 1) return fail(DSACT_EINVAL, "exchange kind %d is not 0 or 1", io->kind);
    if (!io->ranks) return fail(DSACT_EINVAL, "null ranks");
    for (int r = 0; r < world; ++r) {
      const dsact_handle* p = io->ranks[r];
      if (!p || !p->dp.ready || p->dp.comm.rank != r || p->dp.comm.world != world ||
          memcmp(p->dp.comm.peer, dp.comm.peer, sizeof(dp.comm.peer)) != 0)
        return fail(DSACT_EINVAL, "ranks[%d] is not rank %d of this handle's world", r, r);
      w.comm[r] = p->dp.comm; w.state[r] = p->buf.state;
    }
  } else if (op == DSACT_TEST_DP_FOLD) {
    if (!io->grads || io->n < 1 || io->n > h->n_params || io->nslabs < 0 || io->nslabs > 16 ||
        (io->nslabs > 0 && (!io->slabs || io->slab_stride < io->n)) || io->tail_rows < 0 ||
        (io->tail_rows > 0 && io->global_batch < io->tail_rows))
      return fail(DSACT_EINVAL, "bad fold argument");
  } else if (op == DSACT_TEST_DP_APPLY && mlp_eng) {
    if (io->tail_rows < 1 || io->global_batch < io->tail_rows) return fail(DSACT_EINVAL, "tail_rows / global_batch");
  }
  CUDA_TRY(cudaSetDevice(h->device));
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  c.pdl = mlp_eng && mlp(h)->tc();
  if (op == DSACT_TEST_DP_EXCHANGE) {
    int kind = io->kind;
    unsigned long long timeout = dp_timeout_ns();
    void* args[] = {&w, &kind, &timeout};
    c.err = cudaLaunchCooperativeKernel((const void*)dp_exchange_world_kernel, dim3(world), dim3(32 * world), args, 0, c.s);
    c.done();
  } else if (op == DSACT_TEST_DP_FOLD) {
    TailArgs ta;
    memset(&ta, 0, sizeof(ta));
    if (io->tail_rows > 0) ta = tail_args(h, io->global_batch, io->tail_rows);
    const bool slabs = io->nslabs > 0;   // (none: the steps' arguments, grads and a stride of 4)
    enqueue_dp_fold(h, io->grads, slabs ? io->slabs : io->grads, io->nslabs, slabs ? io->slab_stride : 4, io->n, ta, c);
  } else if (op == DSACT_TEST_DP_REDUCE_SCATTER) {
    enqueue_dp_reduce_scatter(dp, h->buf.state, h->num_sms, c);
  } else if (mlp_eng) {
    const TailArgs ta = tail_args(h, io->global_batch, io->tail_rows);
    enqueue_apply(mlp(h), c, &ta, true);
  } else {
    cnn_enqueue_apply(heads(h), c, 1, true);
  }
  c.check();
  return sync_hook(h, c);
}

}  // extern "C"
