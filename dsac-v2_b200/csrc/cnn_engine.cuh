// DSAC-T update with the reference's CNN approximators (BASELINE config 5; reference networks/cnn.py:30-53 conv stack,
// :151-240 StochaPolicy, :383-461 ActionValueDistri).  Included by engine.cu before its C ABI: it reuses the grouped fp32 GEMM
// launcher and the step launches both engines share (noise, sample, loss, policy gradient, apply, gather); what is new here
// is the conv stack (conv.cuh) and the two-head wiring (separate `mean` and `log_std` MLPs per network, their outputs
// packed into the [B,2] / [B,2A] arrays the loss kernels read, by strided GEMM outputs).
//
// The same wiring without an encoder (n_conv = 0), with one two-output head per critic (q_heads = 1), with the policy as one
// head / two heads / mean head + learnable log_std row (pi_std) serves the MLP approximators whose variants the wgmma
// engine does not implement (policy std_type mlp_separated / parameter).  DSAC_V1 (algo = 1) runs the same phases with
// one critic instead of two (flat layout [q | policy | log_alpha]) and its own critic loss, loss_v1_kernel.
//
// One eager sequence of launches per step (no graph capture yet), for critics k = 0 .. nq-1:
//   conv forwards: pi(s), pi'(s'), Q_k features of s (shared by the (s,a) and (s,a~) passes), Q'_k features of s'
//   heads: pi, pi' -> sample -> Q_k(s,a), Q'_k(s',a'), mean head of Q_k(s,a~) -> loss -> head backward (critics: both
//   heads; actor path: mean head, input gradient only) -> policy_grad -> policy heads backward -> conv backward -> Adam.
#pragma once
#include "conv.cuh"

namespace dsact {
__global__ void relu_mask_kernel(float* __restrict__ g, const float* __restrict__ a, long long n) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (!(a[i] > 0.f)) g[i] = 0.f;
}
// logits[b][col0 + j] = row[j]: the learnable log_std row of policy std_type "parameter" broadcast over the batch
// (reference networks/mlp.py:95-96)
__global__ void bcast_row_kernel(float* __restrict__ out, int ld, int col0, const float* __restrict__ row, int B, int A) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)B * A; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / A), j = (int)(i - (long long)b * A);
    out[(size_t)b * ld + col0 + j] = row[j];
  }
}
__global__ void zero_kernel(float* __restrict__ p, long long n) {
  pdl_sync();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = 0.f;
}
}  // namespace dsact

struct CnnGeom {   // one network: conv encoder (possibly empty) + 1 or 2 identical head MLPs (+ a learnable log_std row)
  int nconv;
  int nheads;            // 2: separate mean / log_std (std) heads; 1: one head (both outputs, or the mean with a log_std row)
  int64_t ls_row;        // offset of the learnable log_std row [out] (policy std_type "parameter"), or -1
  int C[DSACT_MAX_CONV + 1], H[DSACT_MAX_CONV + 1], W[DSACT_MAX_CONV + 1];   // [0] = input image
  int K[DSACT_MAX_CONV], S[DSACT_MAX_CONV];
  int64_t cw[DSACT_MAX_CONV], cb[DSACT_MAX_CONV];
  int F;                 // flattened feature size
  Net head;              // s[0] = F (+ act_dim), hidden..., s[L+1] = outputs of ONE head
  int64_t head_off[2];   // mean, log_std
  int64_t n;
  bool build(const dsact_cnn_config& c, int extra_in, int out, int heads, bool std_row) {
    nconv = c.n_conv; nheads = heads; ls_row = -1;
    C[0] = c.channels; H[0] = c.height; W[0] = c.width;
    n = 0;
    for (int j = 0; j < nconv; ++j) {
      K[j] = c.conv_kernel[j]; S[j] = c.conv_stride[j];
      C[j + 1] = c.conv_channels[j];
      H[j + 1] = (H[j] - K[j]) / S[j] + 1;
      W[j + 1] = (W[j] - K[j]) / S[j] + 1;
      if (H[j + 1] < 1 || W[j + 1] < 1) return false;
      cw[j] = n; n += (int64_t)C[j + 1] * C[j] * K[j] * K[j];
      cb[j] = n; n += C[j + 1];
    }
    F = C[nconv] * H[nconv] * W[nconv];
    head.build(F + extra_in, c.hidden, c.n_hidden, out);
    if (std_row) { ls_row = n; n += out; }   // nn.Module.parameters() yields a module's own parameters before its children's
    head_off[1] = -1;
    for (int hd = 0; hd < nheads; ++hd) { head_off[hd] = n; n += head.n; }
    return true;
  }
  ConvShape shape(int j, int B) const { return ConvShape{B, C[j], H[j], W[j], C[j + 1], K[j], S[j], H[j + 1], W[j + 1]}; }
  int64_t act_elems(int j) const { return (int64_t)C[j] * H[j] * W[j]; }   // per sample, activation j (0 = image)
};

constexpr int CNN_DGRAD_SMEM = 96 * 1024;   // opt-in dynamic shared memory of conv_dgrad8_kernel

struct CnnHeadBuf { int64_t z[DSACT_MAX_HIDDEN], h[DSACT_MAX_HIDDEN], dz[DSACT_MAX_HIDDEN]; };

struct HeadsHandle : dsact_handle {
  dsact_cnn_config cfg;
  CnnGeom q, pi;
  // arena (floats from the workspace base), besides the shell's slots
  int64_t convP[DSACT_MAX_CONV + 1], convT[DSACT_MAX_CONV + 1], convQ[4][DSACT_MAX_CONV + 1];   // activations 1..nconv
  CnnHeadBuf hb[14];   // 0,1 pi mean/ls; 2,3 pi'; 4..7 Q1,Q2 (s,a) mean/ls; 8..11 Q1',Q2'; 12,13 mean head of Q1,Q2 on (s,a~)
  int64_t dfeat[3], dfa[2];   // dL/dfeature of pi, Q1, Q2; dL/d(feature|act) scratch of the actor path
  int64_t ga, gb;             // conv-backward ping-pong buffers (largest activation)
  int64_t total;
  HeadsHandle() : dsact_handle(ENGINE_HEADS) {}
  int nq() const { return v1 ? 1 : 2; }   // critics: DSAC_V1 has one
  void layout() {
    const int64_t B = cfg.max_batch, A = cfg.act_dim;
    StepSlots& s = slot;
    int64_t off = 0;
    auto take = [&](int64_t n) { int64_t o = off; off += round64(n); return o; };
    auto conv_acts = [&](const CnnGeom& g, int64_t* a) { a[0] = -1; for (int j = 1; j <= g.nconv; ++j) a[j] = take(B * g.act_elems(j)); };
    conv_acts(pi, convP); conv_acts(pi, convT);
    for (int k = 0; k < 4; ++k) conv_acts(q, convQ[k]);
    for (int p = 0; p < 14; ++p) {
      const Net& net = p < 4 ? pi.head : q.head;
      for (int j = 0; j < net.L; ++j) { hb[p].z[j] = take(B * net.s[j + 1]); hb[p].h[j] = take(B * net.s[j + 1]); hb[p].dz[j] = take(B * net.s[j + 1]); }
    }
    s.logitsP = take(B * 2 * A); s.logitsT = take(B * 2 * A); s.dlogits = take(B * 2 * A);
    s.new_act = take(B * A); s.act2 = take(B * A); s.logp_new = take(B); s.logp2 = take(B);
    s.eps1 = take(B * A); s.eps2 = take(B * A); s.z3 = take(B); s.z4 = take(B);
    for (int p = 0; p < 6; ++p) { s.outQ[p] = take(B * 2); s.dOut[p] = take(B * 2); }
    s.dAct[0] = take(B * A); s.dAct[1] = take(B * A);
    dfeat[0] = take(B * pi.F); dfeat[1] = take(B * q.F); dfeat[2] = take(B * q.F);
    dfa[0] = take(B * (q.F + A)); dfa[1] = take(B * (q.F + A));
    int64_t big = 0;
    for (int j = 1; j <= q.nconv; ++j) big = big > q.act_elems(j) ? big : q.act_elems(j);
    for (int j = 1; j <= pi.nconv; ++j) big = big > pi.act_elems(j) ? big : pi.act_elems(j);
    ga = take(B * big); gb = take(B * big);
    const int64_t O = (int64_t)cfg.channels * cfg.height * cfg.width;
    s.obs = take(B * O); s.obs2 = take(B * O); s.act = take(B * A); s.rew = take(B); s.done = take(B); s.logp = take(B); s.idx = take(2 * B);
    total = off;
  }
};

// critics: two heads of one output (networks/cnn.py) or one head of two (networks/mlp.py:113-127); policy: mean and
// log_std heads (networks/cnn.py, mlp.py std_type "mlp_separated") or a mean head + learnable row (std_type "parameter").
// Also lays out the arena and sets the shell's sizes.
static void cnn_setup(HeadsHandle* h, const dsact_cnn_config& c) {
  const bool q1 = c.q_heads == 1, row = c.pi_std == 1, shared = c.pi_std == 2;
  h->cfg = c;
  h->hyper = StepHyper::of(c);
  h->q.build(c, c.act_dim, q1 ? 2 : 1, q1 ? 1 : 2, false);
  h->pi.build(c, 0, shared ? 2 * c.act_dim : c.act_dim, (row || shared) ? 1 : 2, row);
  h->layout();
  h->obs_elems = (int64_t)c.channels * c.height * c.width;
  h->act_dim = c.act_dim;
  h->max_batch = c.max_batch;
  h->v1 = c.algo == 1;
  h->v1_bound = c.v1_bound; h->td_bound = c.td_bound;
  h->n_params = h->nq() * h->q.n + h->pi.n + 1;
}

static int cnn_validate(const dsact_cnn_config* c) {
  if (!c) return fail(DSACT_EINVAL, "null config");
  if (c->abi_version != DSACT_ABI_VERSION) return fail(DSACT_EINVAL, "abi_version %d != %d", c->abi_version, DSACT_ABI_VERSION);
  if (c->channels < 1 || c->height < 1 || c->width < 1 || c->act_dim < 1) return fail(DSACT_EINVAL, "bad observation / action shape");
  if (c->n_conv < 0 || c->n_conv > DSACT_MAX_CONV) return fail(DSACT_EINVAL, "0..%d conv layers supported", DSACT_MAX_CONV);
  if (c->q_heads != 1 && c->q_heads != 2) return fail(DSACT_EINVAL, "q_heads must be 1 (one head, two outputs) or 2 (mean and std heads)");
  if (c->pi_std < 0 || c->pi_std > 2) return fail(DSACT_EINVAL, "pi_std must be 0 (log_std head), 1 (learnable row) or 2 (one head, 2*act_dim outputs)");
  if (c->algo != 0 && c->algo != 1) return fail(DSACT_EINVAL, "algo must be 0 (DSAC_V2 / DSAC-T) or 1 (DSAC_V1)");
  if (c->algo == 1 && !(c->td_bound > 0.0)) return fail(DSACT_EINVAL, "DSAC_V1 needs TD_bound > 0");
  if (c->act_dist != 0 && c->act_dist != 1) return fail(DSACT_EINVAL, "act_dist must be 0 (TanhGaussDistribution) or 1 (GaussDistribution)");
  for (int j = 0; j < c->n_conv; ++j)
    if (c->conv_kernel[j] < 1 || (c->conv_kernel[j] > 4 && c->conv_kernel[j] != 8) || c->conv_stride[j] < 1 || c->conv_channels[j] < 1)
      return fail(DSACT_EINVAL, "conv layer %d: kernel sizes 1..4 and 8 are implemented (the reference's type_1 / type_2 encoders)", j);
  if (c->n_hidden < 1 || c->n_hidden > DSACT_MAX_HIDDEN) return fail(DSACT_EINVAL, "1..%d hidden layers per head", DSACT_MAX_HIDDEN);
  if (c->act_hidden < 0 || c->act_hidden > DSACT_ACT_SELU) return fail(DSACT_EINVAL, "unknown activation");
  if (c->max_batch < 1 || c->delay_update < 1) return fail(DSACT_EINVAL, "bad max_batch / delay_update");
  CnnGeom g;
  if (!g.build(*c, 0, 1, 2, false)) return fail(DSACT_EINVAL, "the conv stack consumes the whole image");
  return DSACT_OK;
}

// ---- head MLPs through the grouped fp32 GEMM -------------------------------------------------------------------------
struct CnnHeadFwd {
  const float* base;     // parameters of this head
  const float* in0; int k0;
  const float* in1; int k1;     // second input segment (the action) or null
  CnnHeadBuf* hbuf;
  bool keep_z;
  float* out; int out_ld;       // head output column(s) inside a packed array
};
static void cnn_heads_forward(HeadsHandle* h, const Net& net, std::vector<CnnHeadFwd>& P, int B, Ctx& c) {
  float* W = h->W();
  for (int j = 0; j <= net.L; ++j) {
    size_t i0 = 0;
    while (i0 < P.size()) {
      GemmGroup G;
      G.n = 0;
      for (; i0 < P.size() && G.n < MAXG; ++i0) {
        const CnnHeadFwd& f = P[i0];
        GemmProb p = prob_zero();
        const int in_dim = net.s[j];
        if (j == 0) {
          p.A[0] = f.in0; p.lda[0] = f.k0; p.K[0] = f.k0; p.B[0] = f.base + net.w[0]; p.ldb[0] = in_dim;
          if (f.k1 > 0) { p.A[1] = f.in1; p.lda[1] = f.k1; p.K[1] = f.k1; p.B[1] = f.base + net.w[0] + f.k0; p.ldb[1] = in_dim; }
        } else {
          p.A[0] = W + f.hbuf->h[j - 1]; p.lda[0] = in_dim; p.K[0] = in_dim; p.B[0] = f.base + net.w[j]; p.ldb[0] = in_dim;
        }
        p.M = B; p.N = net.s[j + 1]; p.bias = f.base + net.b[j]; p.act = h->cfg.act_hidden;
        if (j == net.L) { p.C = f.out; p.ldc = f.out_ld; p.epi = EPI_STORE; }
        else { p.C = W + f.hbuf->h[j]; p.ldc = net.s[j + 1]; p.epi = EPI_BIAS_ACT; p.Zout = f.keep_z ? W + f.hbuf->z[j] : nullptr; }
        G.p[G.n++] = p;
      }
      launch_simt(h->num_sms, G, V_FWD, c);
      c.done();
    }
  }
  c.check();
}

struct CnnHeadBwd {
  const float* base;     // parameters of this head
  float* gbase;          // its gradients, or null (actor path through a critic: input gradient only)
  const float* in0; int k0; const float* in1; int k1;   // layer-0 inputs (for the weight gradient)
  CnnHeadBuf* hbuf;
  const float* dout; int dout_ld;   // dL/d(head output) inside a packed array
  float* din;            // [B, k0 + k1] dL/d(layer-0 input), accumulated (+=), or null
};
static void cnn_heads_backward(HeadsHandle* h, const Net& net, std::vector<CnnHeadBwd>& P, int B, Ctx& c) {
  float* W = h->W();
  for (int j = net.L; j >= 0; --j) {
    GemmGroup gw, gd;
    gw.n = gd.n = 0;
    auto flush = [&](GemmGroup& G, int variant) { if (G.n) { launch_simt(h->num_sms, G, variant, c); c.done(); G.n = 0; } };
    for (const CnnHeadBwd& f : P) {
      const float* dY = j == net.L ? f.dout : W + f.hbuf->dz[j];
      const int ldy = j == net.L ? f.dout_ld : net.s[j + 1];
      if (f.gbase) {   // dW_j += dY^T X
        auto wgrad = [&](const float* X, int ldx, int col0, int ncols) {
          GemmProb p = prob_zero();
          p.A[0] = dY; p.lda[0] = ldy; p.K[0] = B; p.B[0] = X; p.ldb[0] = ldx;
          p.M = net.s[j + 1]; p.N = ncols; p.C = f.gbase + net.w[j] + col0; p.ldc = net.s[j]; p.epi = EPI_ATOMIC;
          if (gw.n == MAXG) flush(gw, V_WGRAD);
          gw.p[gw.n++] = p;
        };
        if (j == 0) { wgrad(f.in0, f.k0, 0, f.k0); if (f.k1 > 0) wgrad(f.in1, f.k1, f.k0, f.k1); }
        else wgrad(W + f.hbuf->h[j - 1], net.s[j], 0, net.s[j]);
      }
      GemmProb p = prob_zero();   // dX = dY W_j (.) act'(z_{j-1})
      p.A[0] = dY; p.lda[0] = ldy; p.K[0] = net.s[j + 1]; p.B[0] = f.base + net.w[j]; p.ldb[0] = net.s[j];
      p.M = B; p.N = net.s[j];
      if (j >= 1) {
        p.C = W + f.hbuf->dz[j - 1]; p.ldc = net.s[j];
        p.epi = EPI_DACT; p.Zin = W + f.hbuf->z[j - 1]; p.ldz = net.s[j]; p.act = h->cfg.act_hidden;
        p.colsum = f.gbase ? f.gbase + net.b[j - 1] : nullptr;
      } else {
        if (!f.din) continue;
        p.C = f.din; p.ldc = net.s[0]; p.epi = EPI_ATOMIC;   // several heads add into the same input gradient
      }
      if (gd.n == MAXG) flush(gd, V_DGRAD);
      gd.p[gd.n++] = p;
    }
    flush(gw, V_WGRAD);
    flush(gd, V_DGRAD);
  }
  c.check();
}

// The kernel variant one convolution layer runs with; 0 in a field = the engine's choice (conv_layer_*).  `r`: output
// positions per thread of conv_fwd8_kernel (1, 2, 4); `cob`: output channels per conv_wgrad_kernel block (1, 4, 8);
// `slabs`: row slabs of the weight gradient; `channels`: 8 (conv_fwd8 / conv_dgrad8) or 1 (conv_fwd / conv_dgrad)
// channels per thread.  With a field set, a layer whose window is its whole input runs the direct kernels too.
struct ConvPick { int r = 0, cob = 0, slabs = 0, channels = 0; };

template <int R>
static int launch_conv_fwd8(const ConvShape& s, long long rows, size_t smem, Ctx& c, const float* x, const float* w, const float* b, float* y) {
  const dim3 grid((unsigned)((rows + 128 * R - 1) / (128 * R)), s.Cout / 8);
  switch (s.K) {
    case 1: launch_k(conv_fwd8_kernel<1, R>, grid, 128, smem, c, x, w, b, y, s); return DSACT_OK;
    case 2: launch_k(conv_fwd8_kernel<2, R>, grid, 128, smem, c, x, w, b, y, s); return DSACT_OK;
    case 3: launch_k(conv_fwd8_kernel<3, R>, grid, 128, smem, c, x, w, b, y, s); return DSACT_OK;
    case 4: launch_k(conv_fwd8_kernel<4, R>, grid, 128, smem, c, x, w, b, y, s); return DSACT_OK;
    case 8:   // 8x8 window (type_1's first layer): one position per thread (64 taps in registers)
      if constexpr (R == 1) { launch_k(conv_fwd8_kernel<8, 1>, grid, 128, smem, c, x, w, b, y, s); return DSACT_OK; }
      return fail(DSACT_EINVAL, "conv forward: the 8x8 window runs one position per thread (R = %d requested)", R);
    default: return fail(DSACT_EINVAL, "conv forward: no kernel for a %dx%d window", s.K, s.K);
  }
}

// a layer whose window is its whole input is a linear layer over the flattened [Cin*K*K] sample (its NCHW order)
static bool conv_is_linear(const ConvShape& s) { return s.Hin == s.K && s.Win == s.K; }
static bool conv_pick_default(const ConvPick& pk) { return !pk.r && !pk.cob && !pk.slabs && !pk.channels; }

// y = relu(conv(x, w) + b) of one layer
static int conv_layer_fwd(int num_sms, const ConvShape& s, const float* x, const float* w, const float* b, float* y, const ConvPick& pk, Ctx& c) {
  const long long rows = (long long)s.B * s.Hout * s.Wout;
  const size_t smem8 = sizeof(float) * 8 * s.Cin * s.K * s.K;
  if (pk.cob || pk.slabs) return fail(DSACT_EINVAL, "conv forward: cob / slabs are weight-gradient choices");
  if (conv_pick_default(pk) && conv_is_linear(s)) {
    GemmGroup G; G.n = 0;
    GemmProb p = prob_zero();
    const int kin = s.Cin * s.K * s.K;
    p.A[0] = x; p.lda[0] = kin; p.K[0] = kin; p.B[0] = w; p.ldb[0] = kin;
    p.M = s.B; p.N = s.Cout; p.C = y; p.ldc = s.Cout; p.bias = b; p.act = ACT_RELU; p.epi = EPI_BIAS_ACT;
    G.p[G.n++] = p;
    launch_simt(num_sms, G, V_FWD, c);
    return DSACT_OK;
  }
  const bool fits8 = s.Cout % 8 == 0 && smem8 <= 48 * 1024;   // eight output channels per thread, 1 / 2 / 4 positions
  const int channels = pk.channels ? pk.channels : fits8 ? 8 : 1;
  if (channels == 8) {
    if (!fits8) return fail(DSACT_EINVAL, "conv forward: 8 channels per thread needs Cout %% 8 == 0 and Cin*K*K*32 B <= 48 KiB");
    const long long wave = 2LL * num_sms * 128;
    const int r = pk.r ? pk.r : s.K > 4 ? 1 : rows >= 4 * wave ? 4 : rows >= 2 * wave ? 2 : 1;
    if (r == 4) return launch_conv_fwd8<4>(s, rows, smem8, c, x, w, b, y);
    if (r == 2) return launch_conv_fwd8<2>(s, rows, smem8, c, x, w, b, y);
    if (r == 1) return launch_conv_fwd8<1>(s, rows, smem8, c, x, w, b, y);
    return fail(DSACT_EINVAL, "conv forward: R must be 1, 2 or 4");
  }
  if (channels != 1 || pk.r > 1) return fail(DSACT_EINVAL, "conv forward: channels per thread 8 or 1 (one position per thread)");
  const size_t smem1 = sizeof(float) * s.Cin * s.K * s.K;
  if (smem1 > 48 * 1024) return fail(DSACT_EINVAL, "conv forward: Cin*K*K*4 B above 48 KiB");
  dim3 grid((unsigned)((rows + 127) / 128), s.Cout);
  launch_k(conv_fwd_kernel, grid, 128, smem1, c, x, w, b, y, s);
  return DSACT_OK;
}

template <int COB>
static int launch_conv_wgrad(const ConvShape& s, int slabs, Ctx& c, const float* dy, const float* x, float* dw, float* db) {
  const dim3 grid(s.Cin, s.Cout / COB, slabs);
  switch (s.K) {
    case 1: launch_k(conv_wgrad_kernel<1, COB>, grid, 256, 0, c, dy, x, dw, db, s); return DSACT_OK;
    case 2: launch_k(conv_wgrad_kernel<2, COB>, grid, 256, 0, c, dy, x, dw, db, s); return DSACT_OK;
    case 3: launch_k(conv_wgrad_kernel<3, COB>, grid, 256, 0, c, dy, x, dw, db, s); return DSACT_OK;
    case 4:
      if constexpr (COB <= 4) { launch_k(conv_wgrad_kernel<4, COB>, grid, 256, 0, c, dy, x, dw, db, s); return DSACT_OK; }
      return fail(DSACT_EINVAL, "conv weight gradient: a 4x4 window takes at most 4 output channels per block (COB = %d)", COB);
    case 8:   // 64 taps x 1 channel
      if constexpr (COB == 1) { launch_k(conv_wgrad_kernel<8, 1>, grid, 256, 0, c, dy, x, dw, db, s); return DSACT_OK; }
      return fail(DSACT_EINVAL, "conv weight gradient: an 8x8 window takes 1 output channel per block (COB = %d)", COB);
    default: return fail(DSACT_EINVAL, "conv weight gradient: no kernel for a %dx%d window", s.K, s.K);
  }
}

// dw += corr(x, dy), db += sum(dy) of one layer (dy: gradient of its pre-activation)
static int conv_layer_wgrad(int num_sms, const ConvShape& s, const float* dy, const float* x, float* dw, float* db, const ConvPick& pk, Ctx& c) {
  const long long rows = (long long)s.B * s.Hout * s.Wout;
  if (pk.r || pk.channels) return fail(DSACT_EINVAL, "conv weight gradient: R / channels are forward and dgrad choices");
  if (conv_pick_default(pk) && conv_is_linear(s)) {   // dW = dz^T x through the GEMM
    GemmGroup gw; gw.n = 0;
    GemmProb p = prob_zero();
    const int kin = s.Cin * s.K * s.K;
    p.A[0] = dy; p.lda[0] = s.Cout; p.K[0] = s.B; p.B[0] = x; p.ldb[0] = kin;
    p.M = s.Cout; p.N = kin; p.C = dw; p.ldc = kin; p.epi = EPI_ATOMIC;
    gw.p[gw.n++] = p;
    launch_simt(num_sms, gw, V_WGRAD, c); c.done();
    launch_k(colsum_rows_kernel, (s.Cout + 31) / 32, dim3(32, 8), 0, c, dy, s.B, s.Cout, db);
    return DSACT_OK;
  }
  // K*K*cob accumulators per thread; slabs: >= 32 rows per thread, enough blocks for ~4 per SM
  const int cob = pk.cob ? pk.cob : s.K > 4 ? 1 : (s.Cout % 8 == 0 && s.K <= 3) ? 8 : s.Cout % 4 == 0 ? 4 : 1;
  if (s.Cout % cob != 0) return fail(DSACT_EINVAL, "conv weight gradient: Cout %d is no multiple of COB %d", s.Cout, cob);
  long long slabs = pk.slabs;
  if (!slabs) {
    const int base = s.Cin * (s.Cout / cob);
    slabs = (4LL * num_sms + base - 1) / base;
    const long long cap = (rows + 256 * 32 - 1) / (256 * 32);
    if (slabs > cap) slabs = cap;
    if (slabs < 1) slabs = 1;
  }
  if (slabs < 1 || slabs > 65535) return fail(DSACT_EINVAL, "conv weight gradient: 1..65535 slabs");
  if (cob == 8) return launch_conv_wgrad<8>(s, (int)slabs, c, dy, x, dw, db);
  if (cob == 4) return launch_conv_wgrad<4>(s, (int)slabs, c, dy, x, dw, db);
  if (cob == 1) return launch_conv_wgrad<1>(s, (int)slabs, c, dy, x, dw, db);
  return fail(DSACT_EINVAL, "conv weight gradient: COB must be 1, 4 or 8");
}

// dx = convT(dy, w) (.) [x > 0] of one layer (x: its input, the ReLU output of the layer below).  conv_dgrad8_kernel needs
// the CNN_DGRAD_SMEM opt-in of dsact_cnn_create / dsact_cnn_test_conv.
static int conv_layer_dgrad(int num_sms, const ConvShape& s, const float* dy, const float* w, const float* x, float* dx, const ConvPick& pk, Ctx& c) {
  const long long rin = (long long)s.B * s.Hin * s.Win;
  const size_t smem8 = sizeof(float) * 8 * s.Cout * s.K * s.K;
  if (pk.r > 1 || pk.cob || pk.slabs) return fail(DSACT_EINVAL, "conv dgrad: one input position per thread; cob / slabs are weight-gradient choices");
  if (conv_pick_default(pk) && conv_is_linear(s)) {   // dx = dz W (.) [x > 0]
    GemmGroup G; G.n = 0;
    GemmProb p = prob_zero();
    const int kin = s.Cin * s.K * s.K;
    p.A[0] = dy; p.lda[0] = s.Cout; p.K[0] = s.Cout; p.B[0] = w; p.ldb[0] = kin;
    p.M = s.B; p.N = kin; p.C = dx; p.ldc = kin; p.epi = EPI_DACT; p.Zin = x; p.ldz = kin; p.act = ACT_RELU;
    G.p[G.n++] = p;
    launch_simt(num_sms, G, V_DGRAD, c);
    return DSACT_OK;
  }
  const bool fits8 = s.Cin % 8 == 0 && smem8 <= (size_t)CNN_DGRAD_SMEM;
  const int channels = pk.channels ? pk.channels : fits8 ? 8 : 1;
  if (channels == 8) {
    if (!fits8) return fail(DSACT_EINVAL, "conv dgrad: 8 channels per thread needs Cin %% 8 == 0 and Cout*K*K*32 B <= 96 KiB");
    dim3 grid((unsigned)((rin + 127) / 128), s.Cin / 8);
    launch_k(conv_dgrad8_kernel, grid, 128, smem8, c, dy, w, x, dx, s, 1);
    return DSACT_OK;
  }
  if (channels != 1) return fail(DSACT_EINVAL, "conv dgrad: channels per thread 8 or 1");
  dim3 grid((unsigned)((rin + 127) / 128), s.Cin);
  launch_k(conv_dgrad_kernel, grid, 128, 0, c, dy, w, x, dx, s, 1);
  return DSACT_OK;
}

static void conv_note(int rc, Ctx& c) { if (rc != DSACT_OK && c.err == cudaSuccess) c.err = cudaErrorInvalidValue; }

static void cnn_conv_forward(HeadsHandle* h, const CnnGeom& g, const float* params, const float* img, const int64_t* acts, int B, Ctx& c) {
  float* W = h->W();
  const float* x = img;
  for (int j = 0; j < g.nconv; ++j) {
    conv_note(conv_layer_fwd(h->num_sms, g.shape(j, B), x, params + g.cw[j], params + g.cb[j], W + acts[j + 1], ConvPick(), c), c);
    c.done();
    x = W + acts[j + 1];
  }
  c.check();
}

// backward through one encoder: `gtop` = dL/d(feature) [B, F] (consumed); gparams was cleared by begin_step_kernel
static void cnn_conv_backward(HeadsHandle* h, const CnnGeom& g, const float* params, float* gparams, const float* img,
                              const int64_t* acts, float* gtop, int B, Ctx& c) {
  float* W = h->W();
  float* gcur = gtop;
  float* bufs[2] = {W + h->ga, W + h->gb};
  int flip = 0;
  {   // dz of the top layer = g (.) [feature > 0]; the layers below are masked by the dgrad kernel that produces them
    const long long n_out = (long long)B * g.act_elems(g.nconv);
    int blocks = (int)((n_out + 255) / 256); if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms;
    launch_k(relu_mask_kernel, blocks, 256, 0, c, gcur, (const float*)(W + acts[g.nconv]), n_out); c.done();
  }
  for (int j = g.nconv - 1; j >= 0; --j) {
    const ConvShape s = g.shape(j, B);
    const float* x = j == 0 ? img : W + acts[j];
    conv_note(conv_layer_wgrad(h->num_sms, s, gcur, x, gparams + g.cw[j], gparams + g.cb[j], ConvPick(), c), c);
    c.done();
    if (j > 0) {
      float* gnext = bufs[flip]; flip ^= 1;
      conv_note(conv_layer_dgrad(h->num_sms, s, gcur, params + g.cw[j], x, gnext, ConvPick(), c), c);
      c.done();
      gcur = gnext;
    }
  }
  c.check();
}

// ---- the step in three phases ---------------------------------------------------------------------------------------
// dsact_step runs them back to back on its own rows; the data-parallel step (dsact_dp_step) runs the critic-std
// exchange between phases 1 and 2 and the gradient exchange between phase 2 and the update.  DSAC_V1 runs them with one
// critic: every "for k < nq" loop below then stops after k = 0.
struct CnnFeats { const float *P, *T, *Q[4]; };   // head inputs: pi(s), pi'(s'), Q1/Q2 features of s, Q1'/Q2' features of s'
static CnnFeats cnn_feats(const HeadsHandle* h, const dsact_batch& bt) {
  // without a conv stack (the MLP approximators with separate heads) the feature is the observation itself
  float* W = h->W();
  const bool enc = h->pi.nconv > 0;
  const int qL = h->q.nconv;
  CnnFeats f;
  f.P = enc ? W + h->convP[h->pi.nconv] : bt.obs;
  f.T = enc ? W + h->convT[h->pi.nconv] : bt.obs2;
  for (int k = 0; k < 2; ++k) {
    f.Q[k] = enc ? W + h->convQ[k][qL] : bt.obs;
    f.Q[2 + k] = enc ? W + h->convQ[2 + k][qL] : bt.obs2;
  }
  return f;
}

// phase 1: clear the step's accumulators and gradients, noise, the encoder forwards, the policy heads, the critics on
// (s, a), sample_kernel (whose y = 1 half leaves the local critic-std sums in state[ST_STDSUM..+1]), the targets and the
// mean heads of the critics on (s, a~)
static void cnn_enqueue_phase1(HeadsHandle* h, const dsact_batch& bt, const dsact_noise* noise, Ctx& c) {
  const CnnGeom &q = h->q, &pi = h->pi;
  const StepSlots& s = h->slot;
  const int B = bt.batch, A = h->act_dim, nq = h->nq();
  float* W = h->W();
  float* P = h->buf.params; float* T = h->buf.targets;
  float* Pq[2] = {P, P + q.n}; float* Ppi = P + nq * q.n;
  float* Tq[2] = {T, T + q.n}; float* Tpi = T + nq * q.n;
  enqueue_begin_step(h, c);
  if (!noise) enqueue_noise(h, B, c);
  const dsact_noise nz = step_noise(h, noise);

  // ---- encoders: pi(s), pi'(s'), Q_k features of s, Q'_k features of s'
  cnn_conv_forward(h, pi, Ppi, bt.obs, h->convP, B, c);
  cnn_conv_forward(h, pi, Tpi, bt.obs2, h->convT, B, c);
  for (int k = 0; k < nq; ++k) {
    cnn_conv_forward(h, q, Pq[k], bt.obs, h->convQ[k], B, c);
    cnn_conv_forward(h, q, Tq[k], bt.obs2, h->convQ[2 + k], B, c);
  }
  const CnnFeats f = cnn_feats(h, bt);

  // ---- policy heads: logits = (mean | log_std), the layout sample_kernel reads (networks/cnn.py:233-240)
  {
    std::vector<CnnHeadFwd> v;
    for (int hd = 0; hd < pi.nheads; ++hd) {
      v.push_back({Ppi + pi.head_off[hd], f.P, pi.F, nullptr, 0, &h->hb[hd], true, W + s.logitsP + hd * A, 2 * A});
      v.push_back({Tpi + pi.head_off[hd], f.T, pi.F, nullptr, 0, &h->hb[2 + hd], false, W + s.logitsT + hd * A, 2 * A});
    }
    cnn_heads_forward(h, pi.head, v, B, c);
    if (pi.ls_row >= 0) {   // std_type "parameter": log_std columns = the learnable row
      int blocks = (B * A + 255) / 256; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
      launch_k(bcast_row_kernel, blocks, 256, 0, c, W + s.logitsP, 2 * A, A, (const float*)(Ppi + pi.ls_row), B, A); c.done();
      launch_k(bcast_row_kernel, blocks, 256, 0, c, W + s.logitsT, 2 * A, A, (const float*)(Tpi + pi.ls_row), B, A); c.done();
    }
  }
  // ---- critics on (s, a): out = (mean, raw std) packed [B,2] (networks/cnn.py:454-461; softplus is applied by the loss kernels)
  {
    std::vector<CnnHeadFwd> v;
    for (int k = 0; k < nq; ++k)
      for (int hd = 0; hd < q.nheads; ++hd)
        v.push_back({Pq[k] + q.head_off[hd], f.Q[k], q.F, bt.act, A, &h->hb[4 + 2 * k + hd], true, W + s.outQ[k] + hd, 2});
    cnn_heads_forward(h, q.head, v, B, c);
  }
  enqueue_sample(h, step_rows(h, bt, nz), B, !noise, c);
  // ---- targets on (s', a') and the mean heads of the critics on (s, a~)
  {
    std::vector<CnnHeadFwd> v;
    for (int k = 0; k < nq; ++k)
      for (int hd = 0; hd < q.nheads; ++hd)
        v.push_back({Tq[k] + q.head_off[hd], f.Q[2 + k], q.F, W + s.act2, A, &h->hb[8 + 2 * k + hd], false, W + s.outQ[2 + k] + hd, 2});
    for (int k = 0; k < nq; ++k)
      v.push_back({Pq[k] + q.head_off[0], f.Q[k], q.F, W + s.new_act, A, &h->hb[12 + k], true, W + s.outQ[4 + k], 2});
    cnn_heads_forward(h, q.head, v, B, c);
  }
  c.check();
}

// phase 2: losses, the head and encoder backward passes, and phase2_tail_kernel, on the rows `bt` and noise `nz` phase 1
// ran.  Every batch mean is a sum over these rows times 1/global_batch; phase2_tail_kernel keeps rows = B (this shard), so
// that the log_alpha gradient it writes is this rank's additive share -(sum_local logp + B * H) / global_batch (see
// tail_grad_log_alpha).
static void cnn_enqueue_phase2(HeadsHandle* h, const dsact_batch& bt, const dsact_noise& nz, int64_t global_batch, Ctx& c) {
  const CnnGeom &q = h->q, &pi = h->pi;
  const StepSlots& s = h->slot;
  const int B = bt.batch, A = h->act_dim, nq = h->nq();
  float* W = h->W();
  float* P = h->buf.params; float* G = h->buf.grads;
  float* Pq[2] = {P, P + q.n}; float* Ppi = P + nq * q.n;
  float* Gq[2] = {G, G + q.n}; float* Gpi = G + nq * q.n;
  const bool enc = pi.nconv > 0;
  const CnnFeats f = cnn_feats(h, bt);

  // ---- losses and head-output gradients
  const StepScalars sc = step_scalars(h, global_batch);
  RowIo io = step_rows(h, bt, nz);
  for (int k = 0; k < 2; ++k) {
    io.gbias_q[k] = Gq[k] + q.head_off[0] + q.head.b[q.head.L];                                       // output bias of the mean head
    io.gbias_q_raw[k] = q.nheads == 2 ? Gq[k] + q.head_off[1] + q.head.b[q.head.L] : nullptr;   // ... of the std head (one head: the next element)
  }
  io.gbias_pi = Gpi + pi.head_off[0] + pi.head.b[pi.head.L];   // output bias of the mean head [A]
  io.gbias_ls = pi.ls_row >= 0 ? Gpi + pi.ls_row : (pi.nheads == 2 ? Gpi + pi.head_off[1] + pi.head.b[pi.head.L] : nullptr);   // log_std head / row [A]
  if (h->v1) enqueue_loss_v1(h, io, B, sc, c);
  else enqueue_loss(h, io, B, sc, c);
  auto zero = [&](float* p, long long n) {
    int blocks = (int)((n + 255) / 256); if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms; if (blocks < 1) blocks = 1;
    launch_k(zero_kernel, blocks, 256, 0, c, p, n); c.done();
  };
  if (enc) {   // feature gradients (read only by the encoders' backward)
    zero(W + h->dfeat[0], (long long)B * pi.F);
    for (int k = 0; k < nq; ++k) zero(W + h->dfeat[1 + k], (long long)B * q.F);
  }
  for (int k = 0; k < nq; ++k) zero(W + h->dfa[k], (long long)B * (q.F + A));
  if (h->v1) zero(W + s.dAct[1], (long long)B * A);   // policy_grad_kernel adds the action gradients of two critics: the second is absent
  // ---- critic backward through both heads (feature gradient accumulated over the heads), actor path through the mean head
  {
    std::vector<CnnHeadBwd> v;
    for (int k = 0; k < nq; ++k)
      for (int hd = 0; hd < q.nheads; ++hd)   // d(feature|act): only the feature part is used (replayed actions carry no gradient)
        v.push_back({Pq[k] + q.head_off[hd], Gq[k] + q.head_off[hd], f.Q[k], q.F, bt.act, A, &h->hb[4 + 2 * k + hd],
                     W + s.dOut[k] + hd, 2, nullptr});
    for (int k = 0; k < nq; ++k)
      v.push_back({Pq[k] + q.head_off[0], nullptr, f.Q[k], q.F, W + s.new_act, A, &h->hb[12 + k], W + s.dOut[4 + k], 2, W + h->dfa[k]});
    cnn_heads_backward(h, q.head, v, B, c);
  }
  // feature gradients of the critics: the layer-0 input gradient of both heads, feature columns only.  The generic
  // backward above skipped it for the critic passes (din = null): do it here with the feature-width problem
  for (int k = 0; k < nq && enc; ++k) {
    GemmGroup gd;
    gd.n = 0;
    for (int hd = 0; hd < q.nheads; ++hd) {
      GemmProb p = prob_zero();
      const Net& net = q.head;
      p.A[0] = W + h->hb[4 + 2 * k + hd].dz[0]; p.lda[0] = net.s[1]; p.K[0] = net.s[1];
      p.B[0] = Pq[k] + q.head_off[hd] + net.w[0]; p.ldb[0] = net.s[0];
      p.M = B; p.N = q.F; p.C = W + h->dfeat[1 + k]; p.ldc = q.F; p.epi = EPI_ATOMIC;
      gd.p[gd.n++] = p;
    }
    launch_simt(h->num_sms, gd, V_DGRAD, c); c.done();
  }
  // dL/da~ through critic k = the action columns of dfa[k]: compact them for policy_grad_kernel
  for (int k = 0; k < nq; ++k) {
    const cudaError_t e = cudaMemcpy2DAsync(W + s.dAct[k], sizeof(float) * A, W + h->dfa[k] + q.F, sizeof(float) * (q.F + A),
                                            sizeof(float) * A, B, cudaMemcpyDeviceToDevice, c.s);
    if (e != cudaSuccess && c.err == cudaSuccess) c.err = e;
  }
  enqueue_policy_grad(h, io, B, sc, c);
  {
    std::vector<CnnHeadBwd> v;
    for (int hd = 0; hd < pi.nheads; ++hd)
      v.push_back({Ppi + pi.head_off[hd], Gpi + pi.head_off[hd], f.P, pi.F, nullptr, 0, &h->hb[hd], W + s.dlogits + hd * A, 2 * A,
                   enc ? W + h->dfeat[0] : nullptr});
    cnn_heads_backward(h, pi.head, v, B, c);
  }
  // ---- encoders backward
  if (enc) {
    cnn_conv_backward(h, pi, Ppi, Gpi, bt.obs, h->convP, W + h->dfeat[0], B, c);
    for (int k = 0; k < nq; ++k) cnn_conv_backward(h, q, Pq[k], Gq[k], bt.obs, h->convQ[k], W + h->dfeat[1 + k], B, c);
  }

  // ---- end of backward bookkeeping: log_alpha gradient (this shard's share), mean_std EMA commit, the Adam scalars
  launch_k(phase2_tail_kernel, 1, 32, 0, c, G + h->n_params - 1, h->buf.state, sc, -(float)A, B, adam_hyper(h), 1); c.done();
  c.check();
}

// Adam / Polyak on `grads` (dp = false), or on the rank-ordered sum of every rank's exchange block (dp = true).  The
// critics' span is nq networks: DSAC_V1's q_optimizer also steps every iteration (dsac_v1.py:259).
// scalars_ready: 1 = phase 2 of this step wrote the Adam scalars; 0 = apply_kernel forms them (a handle that only receives
// gradients never runs phase 2)
static void cnn_enqueue_apply(HeadsHandle* h, Ctx& c, int scalars_ready, bool dp) {
  launch_apply(h, apply_args(h, h->nq() * h->q.n, scalars_ready, dp), c);
}

static HeadsHandle* heads(dsact_handle* h) { return static_cast<HeadsHandle*>(h); }

// dsact_step: phase 1, phase 2 and the update on its own rows
static void cnn_enqueue_step(HeadsHandle* h, const dsact_batch& bt, const dsact_noise* noise, Ctx& c) {
  cnn_enqueue_phase1(h, bt, noise, c);
  cnn_enqueue_phase2(h, bt, step_noise(h, noise), bt.batch, c);
  cnn_enqueue_apply(h, c, 1, false);
}

// One data-parallel update on this rank's shard (dsact_dp_step), eager on the caller's stream: phase 1, critic-std sums
// exchanged, phase 2 scaled by 1/global_batch, the local gradients into this rank's exchange block, logged sums exchanged
// (also the "every block is complete" barrier), [reduce-scatter from 6 ranks up], Adam on the rank-ordered global sum.
static void cnn_enqueue_dp_step(HeadsHandle* h, const dsact_batch& bt, const dsact_noise* noise, int64_t global_batch, Ctx& c) {
  float* state = h->buf.state;
  cnn_enqueue_phase1(h, bt, noise, c);
  enqueue_dp_exchange(h->dp, state, 0, c);
  cnn_enqueue_phase2(h, bt, step_noise(h, noise), global_batch, c);
  {   // phase 2 already wrote the log_alpha share: a plain copy of the flat gradients into this rank's block
    TailArgs none;
    memset(&none, 0, sizeof(none));
    enqueue_dp_fold(h, h->buf.grads, h->buf.grads, 0, 4, h->n_params, none, c);
  }
  enqueue_dp_exchange(h->dp, state, 1, c);
  if (dp_two_shot(h->dp)) enqueue_dp_reduce_scatter(h->dp, state, h->num_sms, c);
  cnn_enqueue_apply(h, c, 1, true);
}

extern "C" {

int dsact_cnn_query_layout(const dsact_cnn_config* cfg, dsact_layout* out) {
  int rc = cnn_validate(cfg);
  if (rc) return rc;
  if (!out) return fail(DSACT_EINVAL, "null out");
  HeadsHandle h;
  cnn_setup(&h, *cfg);
  out->n_q = h.q.n; out->n_pi = h.pi.n;
  out->n_params = h.n_params;
  out->n_targets = h.n_params - 1;
  out->workspace_bytes = h.total * (int64_t)sizeof(float);
  out->state_floats = ST_FLOATS;
  out->max_batch = cfg->max_batch;
  const StepSlots& s = h.slot;
  out->off_idx = s.idx; out->off_eps1 = s.eps1; out->off_eps2 = s.eps2; out->off_z3 = s.z3; out->off_z4 = s.z4;
  out->off_slabs = h.total; out->slab_floats = 0;
  return DSACT_OK;
}

int dsact_cnn_create(const dsact_cnn_config* cfg, int device, dsact_handle** out) {
  int rc = cnn_validate(cfg);
  if (rc) return rc;
  if (!out) return fail(DSACT_EINVAL, "null out");
  CUDA_TRY(cudaSetDevice(device));
  int num_sms = 0;
  if ((rc = check_sm90(device, &num_sms))) return rc;
  CUDA_TRY(cudaFuncSetAttribute(conv_dgrad8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CNN_DGRAD_SMEM));
  HeadsHandle* h = new HeadsHandle();
  h->device = device;
  h->num_sms = num_sms;
  cnn_setup(h, *cfg);
  *out = h;
  return DSACT_OK;
}

int dsact_cnn_test_conv(int32_t op, int32_t batch, int32_t cin, int32_t hin, int32_t win, int32_t cout, int32_t k, int32_t stride,
                        const float* x, const float* w, const float* b, const float* dy, float* out, float* dw, float* db,
                        int32_t r, int32_t cob, int32_t slabs, int32_t channels, void* stream) {
  if (op < 0 || op > 2) return fail(DSACT_EINVAL, "op must be 0 (forward), 1 (weight gradient) or 2 (dgrad)");
  if (batch < 1 || cin < 1 || cout < 1 || k < 1 || stride < 1 || hin < k || win < k) return fail(DSACT_EINVAL, "bad layer shape");
  if (r < 0 || cob < 0 || slabs < 0 || channels < 0) return fail(DSACT_EINVAL, "negative kernel choice");
  int dev = 0, num_sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  int rc = check_sm90(dev, &num_sms);
  if (rc) return rc;
  CUDA_TRY(cudaFuncSetAttribute(conv_dgrad8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CNN_DGRAD_SMEM));
  ConvShape s;
  s.B = batch; s.Cin = cin; s.Hin = hin; s.Win = win; s.Cout = cout; s.K = k; s.S = stride;
  s.Hout = (hin - k) / stride + 1; s.Wout = (win - k) / stride + 1;
  ConvPick pk; pk.r = r; pk.cob = cob; pk.slabs = slabs; pk.channels = channels;
  Ctx c{(cudaStream_t)stream, 0, cudaSuccess};
  if (op == 0) {
    if (!x || !w || !b || !out) return fail(DSACT_EINVAL, "forward needs x, w, b, out");
    rc = conv_layer_fwd(num_sms, s, x, w, b, out, pk, c);
  } else if (op == 1) {
    if (!x || !dy || !dw || !db) return fail(DSACT_EINVAL, "weight gradient needs x, dy, dw, db");
    rc = conv_layer_wgrad(num_sms, s, dy, x, dw, db, pk, c);
  } else {
    if (!x || !w || !dy || !out) return fail(DSACT_EINVAL, "dgrad needs x, w, dy, out");
    rc = conv_layer_dgrad(num_sms, s, dy, w, x, out, pk, c);
  }
  if (rc) return rc;
  c.check();
  if (c.err != cudaSuccess) return fail(DSACT_ECUDA, "kernel launch failed: %s", cudaGetErrorString(c.err));
  return DSACT_OK;
}

}  // extern "C"
