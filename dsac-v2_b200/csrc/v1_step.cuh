// DSAC_V1 (reference dsac_v1.py:56-273; SURVEY.md §8f rank 4): the older algorithm with ONE distributional critic and a fixed
// TD bound, on the head-wise fp32 engine of cnn_engine.cuh (`dsact_cnn_config.algo = 1`).  Same networks, sampling, policy
// gradient, Adam / Polyak kernels as DSAC-T; what differs is the critic loss (this file) and the network set
// (q, q_target, policy, policy_target: flat layout [q | policy | log_alpha]).
#pragma once

namespace dsact {

struct LossV1Args {
  const float *rew, *done, *z, *logp2, *logp_new;
  const float *out_q, *out_qt, *out_qa;   // Q(s,a), Q'(s',a'), Q(s,a~): [B,2] (mean, raw std)
  float *d_out_q, *d_out_qa;              // dL/d(mean, raw std)
  float *gbias_q, *gbias_q_raw;           // output-bias gradient (+=); raw: null = gbias_q + 1 (one two-output head)
  float* state;
  int B, bound;
  float gamma, inv_global_batch, td_bound;
  StepScalars sc;
};

// __compute_loss_q / __compute_target_q / __compute_loss_policy of dsac_v1.py:195-248, one thread per sample:
//   target = r + (1-d) gamma (q' + clamp(z,-3,3) sigma' - alpha logp'),  target_b = q + clamp(target - q, -TD, TD)
//   bound:  L = mean( -(target - q)/(sigma^2 + 0.1) q - ((q - target_b)^2 - sigma^2)/(sigma^3 + 0.1) sigma )   (coefficients detached)
//   else:   L = mean( -log N(target; q, sigma) )
//   actor:  L_pi = mean( alpha logp - q(s,a~) )
__global__ void loss_v1_kernel(const __grid_constant__ LossV1Args a) {
  pdl_sync();
  __shared__ float red[6 * 32];
  const float alpha = step_alpha(a.sc);
  const float invB = a.inv_global_batch;
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // q, sigma, loss_pi, logp, gb_mean, gb_raw
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.B; i += gridDim.x * blockDim.x) {
    const float qn = a.out_qt[2 * i], sn = softplus_f(a.out_qt[2 * i + 1]);
    const float zc = fminf(fmaxf(a.z[i], -3.f), 3.f);
    const float target = a.rew[i] + (1.f - a.done[i]) * a.gamma * ((qn + zc * sn) - alpha * a.logp2[i]);
    const float q = a.out_q[2 * i], raw = a.out_q[2 * i + 1];
    const float sd = softplus_f(raw);
    float g_mean, g_sd;
    if (a.bound) {
      const float sdd = fmaxf(sd, 0.f);
      const float tb = q + fminf(fmaxf(target - q, -a.td_bound), a.td_bound);
      g_mean = -(target - q) / (sdd * sdd + 0.1f) * invB;
      g_sd = -((q - tb) * (q - tb) - sdd * sdd) / (sdd * sdd * sdd + 0.1f) * invB;
    } else {
      const float d = target - q;
      g_mean = -d / (sd * sd) * invB;
      g_sd = (1.f / sd - d * d / (sd * sd * sd)) * invB;
    }
    const float dsoft = raw > 20.f ? 1.f : 1.f / (1.f + expf(-raw));
    const float g_raw = g_sd * dsoft;
    a.d_out_q[2 * i] = g_mean;
    a.d_out_q[2 * i + 1] = g_raw;
    const float lp = a.logp_new[i];
    a.d_out_qa[2 * i] = -invB;
    a.d_out_qa[2 * i + 1] = 0.f;
    s[0] += q; s[1] += sd; s[2] += alpha * lp - a.out_qa[2 * i]; s[3] += lp; s[4] += g_mean; s[5] += g_raw;
  }
  block_sum<6>(s, red);
  if (threadIdx.x == 0) {
    float* acc = a.state + ST_ACC;
    atomicAdd(acc + ACC_Q1, s[0]);
    atomicAdd(acc + ACC_S1, s[1]);
    atomicAdd(acc + ACC_LOSS_PI, s[2]);
    atomicAdd(acc + ACC_LOGP, s[3]);
    atomicAdd(a.gbias_q, s[4]);
    atomicAdd(a.gbias_q_raw ? a.gbias_q_raw : a.gbias_q + 1, s[5]);
  }
}

}  // namespace dsact

// One DSAC_V1 update (local_update, dsac_v1.py:95-98).  `noise`: eps1, eps2 as for DSAC-T; z3 = the draw of the target
// critic's sample (the reference's second of three z draws; the other two do not enter the arithmetic); z4 unused.
static void cnn_enqueue_v1(HeadsHandle* h, const dsact_batch* batch, const dsact_noise* noise, Ctx& c) {
  const dsact_cnn_config& cf = h->cfg;
  const CnnGeom &q = h->q, &pi = h->pi;
  const int B = batch->batch, A = cf.act_dim;
  float* W = h->W();
  float* P = h->buf.params; float* T = h->buf.targets; float* G = h->buf.grads;
  float* Pq = P; float* Ppi = P + q.n;
  float* Tq = T; float* Tpi = T + q.n;
  float* Gq = G; float* Gpi = G + q.n;
  const long long n_all = q.n + pi.n + 1;
  {
    int blocks = (int)((n_all / 4 + 255) / 256); if (blocks > 2 * h->num_sms) blocks = 2 * h->num_sms; if (blocks < 1) blocks = 1;
    launch_k(begin_step_kernel, blocks, 256, 0, c, h->buf.state, G, n_all); c.done();
  }
  const float *eps1, *eps2, *zn;
  if (noise) { eps1 = noise->eps1; eps2 = noise->eps2; zn = noise->z3; }
  else {
    const int total = (B * A + 1) / 2 * 2 + (B + 1) / 2 * 2;
    int blocks = (total / 2 + 255) / 256; if (blocks < 1) blocks = 1;
    launch_k(noise_kernel, blocks, 256, 0, c, W + h->eps1, W + h->eps2, W + h->z3, W + h->z4, B, A, h->seed, (const float*)h->buf.state); c.done();
    eps1 = W + h->eps1; eps2 = W + h->eps2; zn = W + h->z3;
  }
  // ---- encoders (if any): pi(s), pi'(s'), Q features of s, Q' features of s'
  cnn_conv_forward(h, pi, Ppi, batch->obs, h->convP, B, c);
  cnn_conv_forward(h, pi, Tpi, batch->obs2, h->convT, B, c);
  cnn_conv_forward(h, q, Pq, batch->obs, h->convQ[0], B, c);
  cnn_conv_forward(h, q, Tq, batch->obs2, h->convQ[2], B, c);
  const bool enc = pi.nconv > 0;
  const float* featP = enc ? W + h->convP[pi.nconv] : batch->obs;
  const float* featT = enc ? W + h->convT[pi.nconv] : batch->obs2;
  const float* featQ = enc ? W + h->convQ[0][q.nconv] : batch->obs;
  const float* featQt = enc ? W + h->convQ[2][q.nconv] : batch->obs2;
  const int pw = pi.head.s[pi.head.L + 1];   // outputs of one policy head: A, or 2A for the one-head (mlp_shared) policy
  {
    std::vector<CnnHeadFwd> v;
    for (int hd = 0; hd < pi.nheads; ++hd) {
      v.push_back({Ppi + pi.head_off[hd], featP, pi.F, nullptr, 0, &h->hb[hd], true, W + h->logitsP + hd * pw, 2 * A});
      v.push_back({Tpi + pi.head_off[hd], featT, pi.F, nullptr, 0, &h->hb[2 + hd], false, W + h->logitsT + hd * pw, 2 * A});
    }
    cnn_heads_forward(h, pi.head, v, B, c);
    if (pi.ls_row >= 0) {
      int blocks = (B * A + 255) / 256; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
      launch_k(bcast_row_kernel, blocks, 256, 0, c, W + h->logitsP, 2 * A, A, (const float*)(Ppi + pi.ls_row), B, A); c.done();
      launch_k(bcast_row_kernel, blocks, 256, 0, c, W + h->logitsT, 2 * A, A, (const float*)(Tpi + pi.ls_row), B, A); c.done();
    }
  }
  {
    std::vector<CnnHeadFwd> v;
    for (int hd = 0; hd < q.nheads; ++hd)
      v.push_back({Pq + q.head_off[hd], featQ, q.F, batch->act, A, &h->hb[4 + hd], true, W + h->outQ[0] + hd, 2});
    cnn_heads_forward(h, q.head, v, B, c);
  }
  {
    SampleArgs a;
    a.logits[0] = W + h->logitsP; a.logits[1] = W + h->logitsT;
    a.eps[0] = eps1; a.eps[1] = eps2;
    a.act[0] = W + h->new_act; a.act[1] = W + h->act2;
    a.logp[0] = W + h->logp_new; a.logp[1] = W + h->logp2;
    a.hi = h->buf.act_high; a.lo = h->buf.act_low; a.state = h->buf.state;
    a.B = B; a.A = A; a.min_log_std = (float)cf.min_log_std; a.max_log_std = (float)cf.max_log_std; a.gauss = cf.act_dist;
    a.img[0] = ImgOut{nullptr, 0, 1, 0}; a.img[1] = ImgOut{nullptr, 0, 1, 0};
    a.out_q[0] = W + h->outQ[0]; a.out_q[1] = W + h->outQ[0];
    a.advance_rng = noise ? 0 : 1;
    a.v1_stats = 1;
    int blocks = (B + 7) / 8; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
    launch_k(sample_kernel, dim3(blocks, 2), 256, 0, c, a); c.done();
  }
  {
    std::vector<CnnHeadFwd> v;
    for (int hd = 0; hd < q.nheads; ++hd)
      v.push_back({Tq + q.head_off[hd], featQt, q.F, W + h->act2, A, &h->hb[8 + hd], false, W + h->outQ[2] + hd, 2});
    v.push_back({Pq + q.head_off[0], featQ, q.F, W + h->new_act, A, &h->hb[12], true, W + h->outQ[4], 2});
    cnn_heads_forward(h, q.head, v, B, c);
  }
  const float invB = (float)(1.0 / (double)B);
  StepScalars sc;
  sc.tau_b = (float)cf.tau_b; sc.alpha_fixed = (float)cf.alpha_fixed; sc.inv_global_batch = invB;
  sc.auto_alpha = cf.auto_alpha; sc.log_alpha = P + q.n + pi.n;
  {
    LossV1Args a;
    a.rew = batch->rew; a.done = batch->done; a.z = zn; a.logp2 = W + h->logp2; a.logp_new = W + h->logp_new;
    a.out_q = W + h->outQ[0]; a.out_qt = W + h->outQ[2]; a.out_qa = W + h->outQ[4];
    a.d_out_q = W + h->dOut[0]; a.d_out_qa = W + h->dOut[4];
    a.gbias_q = Gq + q.head_off[0] + q.head.b[q.head.L];
    a.gbias_q_raw = q.nheads == 2 ? Gq + q.head_off[1] + q.head.b[q.head.L] : nullptr;
    a.state = h->buf.state; a.B = B; a.bound = cf.v1_bound; a.gamma = (float)cf.gamma; a.inv_global_batch = invB;
    a.td_bound = (float)cf.td_bound; a.sc = sc;
    int blocks = (B + 63) / 64; if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms;
    launch_k(loss_v1_kernel, blocks, 64, 0, c, a); c.done();
  }
  auto zero = [&](float* p, long long n) {
    int blocks = (int)((n + 255) / 256); if (blocks > 4 * h->num_sms) blocks = 4 * h->num_sms; if (blocks < 1) blocks = 1;
    launch_k(zero_kernel, blocks, 256, 0, c, p, n); c.done();
  };
  if (enc) { zero(W + h->dfeat[0], (long long)B * pi.F); zero(W + h->dfeat[1], (long long)B * q.F); }
  zero(W + h->dfa[0], (long long)B * (q.F + A));
  zero(W + h->dAct[1], (long long)B * A);   // policy_grad_kernel adds the action gradients of two critics: the second is absent
  {
    std::vector<CnnHeadBwd> v;
    for (int hd = 0; hd < q.nheads; ++hd)
      v.push_back({Pq + q.head_off[hd], Gq + q.head_off[hd], featQ, q.F, batch->act, A, &h->hb[4 + hd], W + h->dOut[0] + hd, 2, nullptr});
    v.push_back({Pq + q.head_off[0], nullptr, featQ, q.F, W + h->new_act, A, &h->hb[12], W + h->dOut[4], 2, W + h->dfa[0]});
    cnn_heads_backward(h, q.head, v, B, c);
  }
  if (enc) {   // feature gradient of the critic: layer-0 input gradient of its head(s), feature columns only
    GemmGroup gd;
    gd.n = 0;
    for (int hd = 0; hd < q.nheads; ++hd) {
      GemmProb p = prob_zero();
      const Net& net = q.head;
      p.A[0] = W + h->hb[4 + hd].dz[0]; p.lda[0] = net.s[1]; p.K[0] = net.s[1];
      p.B[0] = Pq + q.head_off[hd] + net.w[0]; p.ldb[0] = net.s[0];
      p.M = B; p.N = q.F; p.C = W + h->dfeat[1]; p.ldc = q.F; p.epi = EPI_ATOMIC;
      gd.p[gd.n++] = p;
    }
    launch_simt(h->num_sms, gd, V_DGRAD, c); c.done();
  }
  {
    const cudaError_t e = cudaMemcpy2DAsync(W + h->dAct[0], sizeof(float) * A, W + h->dfa[0] + q.F, sizeof(float) * (q.F + A),
                                            sizeof(float) * A, B, cudaMemcpyDeviceToDevice, c.s);
    if (e != cudaSuccess && c.err == cudaSuccess) c.err = e;
  }
  {
    PolicyGradArgs a;
    a.logits = W + h->logitsP; a.eps = eps1; a.d_act1 = W + h->dAct[0]; a.d_act2 = W + h->dAct[1];
    a.hi = h->buf.act_high; a.lo = h->buf.act_low;
    a.d_logits = W + h->dlogits; a.state = h->buf.state;
    a.gbias = Gpi + pi.head_off[0] + pi.head.b[pi.head.L];
    a.gbias_ls = pi.ls_row >= 0 ? Gpi + pi.ls_row : (pi.nheads == 2 ? Gpi + pi.head_off[1] + pi.head.b[pi.head.L] : nullptr);
    a.B = B; a.A = A; a.min_log_std = (float)cf.min_log_std; a.max_log_std = (float)cf.max_log_std; a.gauss = cf.act_dist;
    a.inv_global_batch = invB;
    a.img = ImgOut{nullptr, 0, 1, 0};
    a.sc = sc;
    int blocks = (B + 7) / 8; if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms; if (blocks < 1) blocks = 1;
    launch_k(policy_grad_kernel, blocks, 256, sizeof(float) * 2 * A, c, a); c.done();
  }
  {
    std::vector<CnnHeadBwd> v;
    for (int hd = 0; hd < pi.nheads; ++hd)
      v.push_back({Ppi + pi.head_off[hd], Gpi + pi.head_off[hd], featP, pi.F, nullptr, 0, &h->hb[hd], W + h->dlogits + hd * pw, 2 * A,
                   enc ? W + h->dfeat[0] : nullptr});
    cnn_heads_backward(h, pi.head, v, B, c);
  }
  if (enc) {
    cnn_conv_backward(h, pi, Ppi, Gpi, batch->obs, h->convP, W + h->dfeat[0], B, c);
    cnn_conv_backward(h, q, Pq, Gq, batch->obs, h->convQ[0], W + h->dfeat[1], B, c);
  }
  AdamHyper hy{cf.lr_q, cf.lr_pi, cf.lr_alpha, cf.adam_beta1, cf.adam_beta2};
  launch_k(phase2_tail_kernel, 1, 32, 0, c, G + q.n + pi.n, h->buf.state, sc, -(float)cf.act_dim, B, hy, 1); c.done();
  {
    ApplyArgs a;
    memset(&a, 0, sizeof(a));
    a.params = P; a.targets = T; a.grads = G; a.m = h->buf.adam_m; a.v = h->buf.adam_v; a.state = h->buf.state;
    a.n_q2 = q.n; a.n_all = n_all;   // the critic span is ONE network (q_optimizer every iteration, dsac_v1.py:259)
    a.delay_update = cf.delay_update; a.auto_alpha = cf.auto_alpha;
    a.hy = hy; a.scalars_ready = 1;
    a.eps = (float)cf.adam_eps; a.tau = (float)cf.tau;
    a.omb1 = (float)(1.0 - cf.adam_beta1); a.b2f = (float)cf.adam_beta2; a.omb2 = (float)(1.0 - cf.adam_beta2);
    a.g_lo = 0; a.g_hi = (n_all + 3) / 4; a.finish = 1;
    int blocks = (int)(((n_all + 3) / 4 + 255) / 256); if (blocks > 8 * h->num_sms) blocks = 8 * h->num_sms;
    launch_k(apply_kernel<0>, blocks, 256, 0, c, a); c.done();
  }
  c.check();
}
