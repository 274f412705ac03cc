// Non-GEMM kernels of the DSAC-T update: tanh-Gaussian sampling, the fused
// target/loss/gradient kernel (and DSAC_V1's), the policy-head gradient, Adam +
// Polyak, noise and index generation, replay gather.  Formulas follow SURVEY.md Appendix A;
// reference line numbers are given per kernel.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "gemm_simt.cuh"   // act_fwd / act_bwd

namespace dsact {

constexpr float TG_EPS = 1e-6f;          // utils/act_distribution_cls.py:3
constexpr float HUBER_DELTA = 50.0f;     // dsac_v2.py:282-287
constexpr float STD_BIAS = 0.1f;         // dsac_v2.py:277
constexpr float HALF_LOG_2PI = 0.91893853320467274f;  // log(sqrt(2*pi))

// ---- persistent state (float slots; see include/dsact.h) ------------------
enum {
  ST_MEAN_STD1 = 0, ST_MEAN_STD2 = 1, ST_ALPHA_USED = 2,
  ST_STDSUM = 4,                       // [4],[5] local sums of softplus std (phase1 -> phase2)
  ST_ADAM_Q = 8, ST_ADAM_PI = 9,       // int32 step counters
  ST_RNG_CTR = 10,                     // uint32 step counter of the device generator
  ST_ITER = 11,                        // int32 iteration the next apply will use (dsac_v2.py:324)
  ST_RB_SIZE = 12,                     // [12],[13] int64 number of valid replay rows
  ST_DP_ERR = 7,                       // int32: nonzero = a peer did not arrive in time (1 + its rank), dp_peer.cuh
  ST_TICKET = 14,                      // int32: blocks of apply_kernel that have finished (the last one advances the counters)
  ST_DP_EPOCH = 15,                    // int32: exchanges completed by the peer-memory data-parallel path
  ST_ACC = 16,                         // 16 sums then 16 mins
  ST_STATS = 48,
  ST_ADAM_SC = 64,                     // [64..68] Adam step sizes / bias corrections of this step (phase2 tail -> apply)
  ST_FLOATS = 80,
};
enum {  // accumulator slots (sums)
  ACC_Q1 = 0, ACC_Q2, ACC_S1, ACC_S2, ACC_LOSS_PI, ACC_LOSS_Q, ACC_TANH_MEAN, ACC_PI_STD, ACC_LOGP,
  ACC_MIN = 16  // [16] min std1, [17] min std2 (float bits, positive values only)
};

// Programmatic dependent launch: every kernel of the step is launched with the PDL attribute, waits here for its
// predecessors' memory, and immediately lets its successors begin launching (their prologue overlaps our tail).
__device__ __forceinline__ void pdl_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// Optional bf16 hi/lo image of a kernel's fp32 output (tensor-core modes; p == nullptr otherwise): the next GEMM
// reads the image by TMA, so producing it here saves a conversion launch.
struct ImgOut {
  __nv_bfloat16* p;
  int pitch, planes;
  long long plane;
};
__device__ __forceinline__ void img_put(const ImgOut& o, size_t row, int col, float x) {
  if (!o.p) return;
  const __nv_bfloat16 hi = __float2bfloat16_rn(x);
  o.p[row * o.pitch + col] = hi;
  if (o.planes == 2) o.p[o.plane + row * o.pitch + col] = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// four consecutive columns (col % 4 == 0, pitch % 8 == 0): one 8-byte store per plane
__device__ __forceinline__ void img_put4(const ImgOut& o, size_t row, int col, float4 x) {
  if (!o.p) return;
  const __nv_bfloat16 h0 = __float2bfloat16_rn(x.x), h1 = __float2bfloat16_rn(x.y), h2 = __float2bfloat16_rn(x.z), h3 = __float2bfloat16_rn(x.w);
  uint2 hv;
  hv.x = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
  hv.y = (uint32_t)__bfloat16_as_ushort(h2) | ((uint32_t)__bfloat16_as_ushort(h3) << 16);
  *reinterpret_cast<uint2*>(o.p + row * o.pitch + col) = hv;
  if (o.planes == 2) {
    const __nv_bfloat16 l0 = __float2bfloat16_rn(x.x - __bfloat162float(h0)), l1 = __float2bfloat16_rn(x.y - __bfloat162float(h1));
    const __nv_bfloat16 l2 = __float2bfloat16_rn(x.z - __bfloat162float(h2)), l3 = __float2bfloat16_rn(x.w - __bfloat162float(h3));
    uint2 lv;
    lv.x = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    lv.y = (uint32_t)__bfloat16_as_ushort(l2) | ((uint32_t)__bfloat16_as_ushort(l3) << 16);
    *reinterpret_cast<uint2*>(o.p + o.plane + row * o.pitch + col) = lv;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum of NV values per thread; result valid in thread 0. blockDim.x multiple of 32, <= 1024.
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float* smem /* >= NV*32 floats */) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < NV; ++i) smem[i * 32 + w] = v[i];
  __syncthreads();
  if (w == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float x = lane < nw ? smem[i * 32 + lane] : 0.f;
      v[i] = warp_sum(x);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float softplus_f(float x) {  // F.softplus, beta=1, threshold=20
  return x > 20.f ? x : log1pf(expf(x));
}
__device__ __forceinline__ float huber_f(float d) {
  const float a = fabsf(d);
  return a <= HUBER_DELTA ? 0.5f * d * d : HUBER_DELTA * (a - 0.5f * HUBER_DELTA);
}

// ---- Philox4x32-10 ---------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
__device__ __forceinline__ float u01(uint32_t x) { return (x + 0.5f) * 2.3283064365386963e-10f; }  // (0,1]
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& n0, float& n1) {
  const float r = sqrtf(-2.0f * logf(u01(a)));
  float s, c;
  sincospif(2.0f * u01(b), &s, &c);
  n0 = r * c;
  n1 = r * s;
}

// Start of every step: clear the accumulators (and the std sums of phase1) and zero the flat gradient buffer
// (bias gradients and column sums accumulate into it with atomics).
__device__ __forceinline__ void begin_step_body(float* __restrict__ state, float* __restrict__ grads, long long n, int block, int nblocks) {
  const int t = threadIdx.x;
  if (block == 0) {
    if (t < 16) state[ST_ACC + t] = 0.f;
    else if (t < 32) state[ST_ACC + t] = __int_as_float(0x7f800000);
    if (t < 2) state[ST_STDSUM + t] = 0.f;
    if (t == 2) reinterpret_cast<int*>(state)[ST_TICKET] = 0;
  }
  const bool vec = (reinterpret_cast<uintptr_t>(grads) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = block * (long long)blockDim.x + t; i < n4; i += (long long)nblocks * blockDim.x)
    reinterpret_cast<float4*>(grads)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = n4 * 4 + block * (long long)blockDim.x + t; i < n; i += (long long)nblocks * blockDim.x) grads[i] = 0.f;
}
__global__ void begin_step_kernel(float* __restrict__ state, float* __restrict__ grads, long long n) {
  pdl_sync();
  begin_step_body(state, grads, n, (int)blockIdx.x, (int)gridDim.x);
}

// Device noise: eps1, eps2 [B,A] and z3, z4 [B] (SURVEY Appendix B keeps only the draws that matter).
__device__ __forceinline__ void noise_body(float* __restrict__ eps1, float* __restrict__ eps2, float* __restrict__ z3,
                                           float* __restrict__ z4, int B, int A, uint64_t seed, const float* __restrict__ state,
                                           int block, int nblocks) {
  const uint32_t step = reinterpret_cast<const uint32_t*>(state)[ST_RNG_CTR];
  const int n_pairs_ea = (B * A + 1) / 2, n_pairs_z = (B + 1) / 2;
  const int total = 2 * n_pairs_ea + 2 * n_pairs_z;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  for (int i = block * blockDim.x + threadIdx.x; i < (total + 1) / 2; i += nblocks * blockDim.x) {
    const uint4 r = philox4x32(make_uint4((uint32_t)i, step, 0x4e4f4953u, 0u), key);
    float n[4];
    box_muller(r.x, r.y, n[0], n[1]);
    box_muller(r.z, r.w, n[2], n[3]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int p = 2 * i + h;  // pair index
      if (p >= total) break;
      float* dst; int len, off;
      if (p < n_pairs_ea) { dst = eps1; len = B * A; off = p; }
      else if (p < 2 * n_pairs_ea) { dst = eps2; len = B * A; off = p - n_pairs_ea; }
      else if (p < 2 * n_pairs_ea + n_pairs_z) { dst = z3; len = B; off = p - 2 * n_pairs_ea; }
      else { dst = z4; len = B; off = p - 2 * n_pairs_ea - n_pairs_z; }
      if (2 * off < len) dst[2 * off] = n[2 * h];
      if (2 * off + 1 < len) dst[2 * off + 1] = n[2 * h + 1];
    }
  }
}

__global__ void noise_kernel(float* __restrict__ eps1, float* __restrict__ eps2, float* __restrict__ z3,
                             float* __restrict__ z4, int B, int A, uint64_t seed, const float* __restrict__ state) {
  pdl_sync();
  noise_body(eps1, eps2, z3, z4, B, A, seed, state, (int)blockIdx.x, (int)gridDim.x);
}

// Uniform replay indices in [0, size) (np.random.randint, training/replay_buffer.py:86).
// rows 2i and 2i+1 share one Philox block
__device__ __forceinline__ int64_t replay_index(int row, uint32_t step, int64_t size, uint2 key) {
  const uint4 r = philox4x32(make_uint4((uint32_t)(row >> 1), step, 0x49445853u, 0u), key);
  const uint64_t a = (row & 1) ? (((uint64_t)r.z << 32) | r.w) : (((uint64_t)r.x << 32) | r.y);
  return (int64_t)__umul64hi(a, (uint64_t)size);
}
// Replay gather (training/replay_buffer.py:87-90): one warp per sampled row, vectorised over obs columns.
// FRAMES = false: the flat ring (dsact_replay), rows r_obs / r_obs2 [capacity, O].
// FRAMES = true: the frame ring (dsact_frame_replay): r_obs = r_obs2 = the frame store [frame_capacity, F = O / K]; frame
// k of row src's obs is frame f_obs[src * K + k] (obs2: f_obs2), i.e. floats [k * F, (k + 1) * F) of the observation.
// CODE = 1 or 2 (with FRAMES): a coded frame ring: the frame store holds CODE-byte codes [frame_capacity, F] (r_obs points
// to them) and value c decodes to table[c]; every other read and every write is the fp32 frame ring's.  CODE = 1: uint8
// codes, the 256 table floats staged in shared memory.  CODE = 2: uint16 codes, 65 536 table floats (256 KiB, more than
// shared memory holds), every lookup through the read-only path from L1 / L2 (faster on every measured stream than
// staging the table's first 4096 entries in shared memory, DESIGN §7).  The kernel never reads how many table entries
// are in use: a captured graph stays valid while the table grows.
template <bool FRAMES, int CODE = 0>
__global__ void gather_kernel(const float* __restrict__ r_obs, const float* __restrict__ r_obs2,
                              const float* __restrict__ r_act, const float* __restrict__ r_rew,
                              const float* __restrict__ r_done, const float* __restrict__ r_logp,
                              const int64_t* __restrict__ idx, float* __restrict__ obs, float* __restrict__ obs2,
                              float* __restrict__ act, float* __restrict__ rew, float* __restrict__ done,
                              float* __restrict__ logp, int B, int O, int A, ImgOut i_obs, ImgOut i_obs2, ImgOut i_act,
                              int64_t* __restrict__ draw_idx, uint64_t seed, const float* __restrict__ state, int write_f32,
                              const int32_t* __restrict__ f_obs, const int32_t* __restrict__ f_obs2, int K,
                              const float* __restrict__ table) {
  static_assert(FRAMES || CODE == 0, "codes index frames");
  static_assert(CODE >= 0 && CODE <= 2, "codes are 1 or 2 bytes");
  using Code = typename std::conditional<CODE == 2, uint16_t, uint8_t>::type;
  constexpr int PER = CODE == 2 ? 8 : 16;   // codes per 16-byte load
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int F = FRAMES ? O / K : O;   // floats of one frame (a float4 never straddles two frames when F % 4 == 0)
  const bool v4 = (F & 3) == 0;
  // address of float e of row src's observation in the frame store (row slots `fs`)
  auto frame_at = [&](const int32_t* fs, int e) {
    const int k = e / F;
    return r_obs + (int64_t)__ldg(fs + k) * F + (e - k * F);
  };
  const float* tab = nullptr;   // CODE = 1: the decode table, staged in shared memory
  if constexpr (CODE == 1) {
    __shared__ float s_table[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_table[i] = __ldg(table + i);
    __syncthreads();
    tab = s_table;
  }
  // the value of code c
  auto dec = [&](auto c) -> float {
    if constexpr (CODE == 1) return tab[c];
    else return __ldg(table + c);
  };
  // address of code e of row src's observation in the coded frame store
  auto code_at = [&](const int32_t* fs, int e) {
    const int k = e / F;
    return reinterpret_cast<const Code*>(r_obs) + (int64_t)__ldg(fs + k) * F + (e - k * F);
  };
  // PER codes (one 16-byte load) -> floats [e, e + PER) of a destination row and its images
  auto put16 = [&](const uint4 q, float* dst, const ImgOut& img, size_t row, int e) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    if constexpr (CODE == 1) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 v = make_float4(tab[w[j] & 0xff], tab[(w[j] >> 8) & 0xff], tab[(w[j] >> 16) & 0xff], tab[w[j] >> 24]);
        if (write_f32) reinterpret_cast<float4*>(dst + e)[j] = v;
        img_put4(img, row, e + 4 * j, v);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float4 v = make_float4(dec(w[2 * j] & 0xffff), dec(w[2 * j] >> 16), dec(w[2 * j + 1] & 0xffff),
                                     dec(w[2 * j + 1] >> 16));
        if (write_f32) reinterpret_cast<float4*>(dst + e)[j] = v;
        img_put4(img, row, e + 4 * j, v);
      }
    }
  };
  // draw_idx != null: no index list was given; every warp draws its row's index itself  and records it in draw_idx
  uint32_t step = 0;
  int64_t size = 1;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  if (draw_idx) {
    step = reinterpret_cast<const uint32_t*>(state)[ST_RNG_CTR];
    size = *reinterpret_cast<const int64_t*>(state + ST_RB_SIZE);
  }
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < B; row += gridDim.x * wpb) {
    int64_t src;
    if (draw_idx) {
      src = replay_index(row, step, size, key);
      if (lane == 0) draw_idx[row] = src;
    } else {
      src = idx[row];
    }
    const float* so = r_obs + src * O;
    const float* so2 = r_obs2 + src * O;
    const int32_t* fo = FRAMES ? f_obs + src * K : nullptr;
    const int32_t* fo2 = FRAMES ? f_obs2 + src * K : nullptr;
    float* dobs = obs + (size_t)row * O;
    float* dobs2 = obs2 + (size_t)row * O;
    if constexpr (CODE > 0) {
      if ((F & (PER - 1)) == 0) {
        // PER codes per 16-byte load (a load never straddles two frames); three of obs and of obs2 in flight per lane, as
        // the fp32 path keeps
        for (int c0 = lane; c0 < O / PER; c0 += 96) {
          uint4 a[3], b[3];
#pragma unroll
          for (int u = 0; u < 3; ++u) {
            const int c = c0 + 32 * u;
            if (c < O / PER) {
              a[u] = __ldg(reinterpret_cast<const uint4*>(code_at(fo, PER * c)));
              b[u] = __ldg(reinterpret_cast<const uint4*>(code_at(fo2, PER * c)));
            }
          }
#pragma unroll
          for (int u = 0; u < 3; ++u) {
            const int c = c0 + 32 * u;
            if (c < O / PER) { put16(a[u], dobs, i_obs, row, PER * c); put16(b[u], dobs2, i_obs2, row, PER * c); }
          }
        }
      } else {
        for (int c = lane; c < O; c += 32) {
          const float a = dec(__ldg(code_at(fo, c))), b = dec(__ldg(code_at(fo2, c)));
          if (write_f32) { dobs[c] = a; dobs2[c] = b; }
          img_put(i_obs, row, c, a); img_put(i_obs2, row, c, b);
        }
      }
    } else if (v4) {
      // three 16-byte columns of obs and of obs2 per lane and trip: six independent loads in flight per lane (the gather is
      // bound by DRAM latency on 1.5 KB random rows, not by bandwidth)
      for (int c0 = lane; c0 < O / 4; c0 += 96) {
        float4 a[3], b[3];
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          const int c = c0 + 32 * u;
          if (c < O / 4) {
            if constexpr (FRAMES) {
              a[u] = __ldg(reinterpret_cast<const float4*>(frame_at(fo, 4 * c)));
              b[u] = __ldg(reinterpret_cast<const float4*>(frame_at(fo2, 4 * c)));
            } else {
              a[u] = __ldg(reinterpret_cast<const float4*>(so) + c); b[u] = __ldg(reinterpret_cast<const float4*>(so2) + c);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          const int c = c0 + 32 * u;
          if (c < O / 4) {
            if (write_f32) {   // (fused tensor-core steps read only the images of obs / obs2 / act)
              reinterpret_cast<float4*>(dobs)[c] = a[u];
              reinterpret_cast<float4*>(dobs2)[c] = b[u];
            }
            img_put4(i_obs, row, 4 * c, a[u]);
            img_put4(i_obs2, row, 4 * c, b[u]);
          }
        }
      }
    } else {
      for (int c = lane; c < O; c += 32) {
        float a, b;
        if constexpr (FRAMES) { a = __ldg(frame_at(fo, c)); b = __ldg(frame_at(fo2, c)); }
        else { a = __ldg(so + c); b = __ldg(so2 + c); }
        if (write_f32) { dobs[c] = a; dobs2[c] = b; }
        img_put(i_obs, row, c, a); img_put(i_obs2, row, c, b);
      }
    }
    for (int c = lane; c < A; c += 32) {
      const float a = __ldg(r_act + src * A + c);
      if (write_f32) act[(size_t)row * A + c] = a;
      img_put(i_act, row, c, a);
    }
    if (lane == 0) { rew[row] = __ldg(r_rew + src); done[row] = __ldg(r_done + src); logp[row] = __ldg(r_logp + src); }
  }
}

// Output activations of the networks (networks/mlp.py, networks/cnn.py: `output_activation` of the last layer), as
// ACT_* codes: the output GEMMs stay linear and write z; the row kernels read y = act(z) and multiply every output
// gradient they write by act'(z).  q: every critic output; mean / ls: the two halves of the policy's (mean | log_std)
// row (ls is linear for std_type "parameter", whose log_std row the reference does not activate).  The row kernels
// take a compile-time OUTACT switch: the linear instantiation never reads these codes.
struct OutActs { int q, mean, ls; };

// TanhGaussDistribution.rsample (utils/act_distribution_cls.py:44-54) on the raw policy-head output
// (mean | log_std), with StochaPolicy's std = exp(clamp(log_std)) (networks/mlp.py:89-92) folded in.
// blockIdx.y = 0: online policy on obs with eps1 (+ the two logged means, dsac_v2.py:155-157);
// blockIdx.y = 1: target policy on obs2 with eps2.  One warp per row.
struct SampleArgs {
  const float* logits[2];
  const float* eps[2];
  float* act[2];
  float* logp[2];
  const float *hi, *lo;
  float* state;
  int B, A;
  float min_log_std, max_log_std;
  ImgOut img[2];
  const float* out_q[2];   // Q_k(s,a) [B,2]: the blockIdx.y = 1 half also sums softplus(raw std) into ST_STDSUM, the
                           // input of the mean_std EMA (dsac_v2.py:233-241)
  int advance_rng;         // device noise/indices were drawn with the current counter: step it (all readers are done)
  int gauss;               // 1: GaussDistribution (utils/act_distribution_cls.py:82-116): no squashing, no action limits
  int v1_stats = 0;        // 1: DSAC_V1's logged policy_mean / policy_std (dsac_v1.py:142-143): tanh(logits[..., 0]) and
                           // logits[..., 1] of cat(mean, std), i.e. the first mean and the SECOND entry of the 2A-wide row
  OutActs oa;              // output activations (read by the OUTACT instantiation only)
};
// One action component of TanhGaussDistribution.rsample: the squashed, scaled action and its log-prob term
// (gauss: GaussDistribution.rsample, the raw Gaussian sample and Normal.log_prob).
__device__ __forceinline__ void sample_elem(float mean, float ls, float eps, float hi, float lo, float min_ls, float max_ls,
                                            float& act, float& lp, float& tanh_mean, float& sd_out, bool gauss = false) {
  const float sd = expf(fminf(fmaxf(ls, min_ls), max_ls));
  const float u = mean + sd * eps;
  if (gauss) {
    const float d = u - mean;
    act = u;
    lp = -(d * d) / (2.f * sd * sd) - logf(sd) - HALF_LOG_2PI;
    tanh_mean = tanhf(mean);
    sd_out = sd;
    return;
  }
  const float th = tanhf(u);
  const float scale = 0.5f * (hi - lo), shift = 0.5f * (hi + lo);
  act = scale * th + shift;
  const float d = u - mean;
  lp = -(d * d) / (2.f * sd * sd) - logf(sd) - HALF_LOG_2PI - logf(1.f + TG_EPS - th * th) - logf(scale);
  tanh_mean = tanhf(mean);
  sd_out = sd;
}
// OUTACT: the (mean | log_std) row and the critics' raw std go through the output activations `a.oa` first
template <bool OUTACT>
__global__ void sample_kernel(const __grid_constant__ SampleArgs a) {
  pdl_sync();
  __shared__ float red[2 * 32];
  const int which = blockIdx.y;
  if (a.advance_rng && blockIdx.x == 0 && which == 0 && threadIdx.x == 0) reinterpret_cast<uint32_t*>(a.state)[ST_RNG_CTR] += 1u;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int A = a.A;
  const float* __restrict__ logits = a.logits[which];
  const float* __restrict__ eps = a.eps[which];
  float sums[2] = {0.f, 0.f};
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < a.B; row += gridDim.x * wpb) {
    float lp = 0.f;
    for (int j = lane; j < A; j += 32) {
      float act, lpj, tm, sd;
      float mean = logits[(size_t)row * 2 * A + j], ls = logits[(size_t)row * 2 * A + A + j];
      if constexpr (OUTACT) { mean = act_fwd(mean, a.oa.mean); ls = act_fwd(ls, a.oa.ls); }
      sample_elem(mean, ls, eps[(size_t)row * A + j], a.hi[j], a.lo[j], a.min_log_std, a.max_log_std, act, lpj, tm, sd, a.gauss != 0);
      a.act[which][(size_t)row * A + j] = act;
      img_put(a.img[which], row, j, act);
      lp += lpj;
      if (!a.v1_stats) { sums[0] += tm; sums[1] += sd; }
      else {
        if (j == 0) sums[0] += tm;
        // (j == 1 < A: the mean of action component 1)
        if (A == 1 ? j == 0 : j == 1) sums[1] += A == 1 ? sd : (OUTACT ? mean : logits[(size_t)row * 2 * A + j]);
      }
    }
    lp = warp_sum(lp);
    if (lane == 0) a.logp[which][row] = lp;
  }
  if (which == 0) {
    block_sum<2>(sums, red);
    if (threadIdx.x == 0) {
      atomicAdd(a.state + ST_ACC + ACC_TANH_MEAN, sums[0]);
      atomicAdd(a.state + ST_ACC + ACC_PI_STD, sums[1]);
    }
  } else {
    float sd[2] = {0.f, 0.f};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.B; i += gridDim.x * blockDim.x) {
      if constexpr (OUTACT) {
        sd[0] += softplus_f(act_fwd(a.out_q[0][2 * i + 1], a.oa.q));
        sd[1] += softplus_f(act_fwd(a.out_q[1][2 * i + 1], a.oa.q));
      } else {
        sd[0] += softplus_f(a.out_q[0][2 * i + 1]);
        sd[1] += softplus_f(a.out_q[1][2 * i + 1]);
      }
    }
    block_sum<2>(sd, red);
    if (threadIdx.x == 0) {
      atomicAdd(a.state + ST_STDSUM, sd[0]);
      atomicAdd(a.state + ST_STDSUM + 1, sd[1]);
    }
  }
}

// mean_std EMA (dsac_v2.py:233-241) and the temperature this step uses (dsac_v2.py:140-148), from the carried state
// and the (all-reduced) std sums of phase 1.  Every block of the loss / policy-gradient kernels evaluates these three
// scalars itself; phase2_tail_kernel commits them to the state at the end of the backward pass.
struct StepScalars {
  float tau_b, alpha_fixed, inv_global_batch;
  int auto_alpha;
  const float* log_alpha;
};
__device__ __forceinline__ float step_mean_std(const float* state, const StepScalars& p, int k) {
  const float mean = state[ST_STDSUM + k] * p.inv_global_batch;
  const float old = state[ST_MEAN_STD1 + k];
  // each operation rounded, as the reference's float32 arithmetic rounds it.  Left to contraction, nvcc fused a different
  // product into the add in different kernels, and the split API (phase2_tail_kernel) committed an EMA one ulp away from
  // the one the single-call and data-parallel steps commit (apply_kernel).
  return old < 0.f ? mean : __fadd_rn(__fmul_rn(1.f - p.tau_b, old), __fmul_rn(p.tau_b, mean));
}
__device__ __forceinline__ float step_alpha(const StepScalars& p) { return p.auto_alpha ? expf(*p.log_alpha) : p.alpha_fixed; }

// Fused clipped-Gaussian distributional TD target + three-refinement critic loss + actor/alpha loss terms
// and all output-layer gradients (dsac_v2.py:218-318, SURVEY Appendix A steps 5-8).  One thread per sample.
struct LossArgs {
  const float *rew, *done, *z3, *z4, *logp2, *logp_new;
  const float* out_q[2];    // Q_k(s,a)    [B,2] (mean, raw std)
  const float* out_qt[2];   // Q'_k(s',a') [B,2]
  const float* out_qa[2];   // Q_k(s,a~)   [B,2]
  float* d_out_q[2];        // dL/d(mean, raw std) of Q_k(s,a)
  float* d_out_qa[2];       // dL/d(mean, raw std) of Q_k(s,a~)
  float* gbias_q[2];        // bias gradient of the critics' output layer [2] (+=)
  float* gbias_q_raw[2];    // null: the raw-std component goes to gbias_q[k] + 1; else its own address (separate log_std head)
  float* state;
  int B;
  float gamma, inv_global_batch;
  ImgOut img_q[2], img_qa[2];
  StepScalars sc;
  int act_q;                // output activation of the critics (OUTACT instantiation)
};
// Everything the loss needs of ONE sample (dsac_v2.py:218-318): gradients w.r.t. the critics' outputs on (s,a) and on
// (s,a~), the per-sample loss terms and the logged values.  m[k] = mean_std of critic k, alpha = temperature in use.
struct LossRow {
  float g_mean[2], g_raw[2];   // dL/d(mean, raw std) of Q_k(s,a)
  float g_pa[2];               // dL/d mean of Q_k(s,a~) (the raw-std component is zero)
  float q[2], sd[2];           // Q_k(s,a) mean and softplus std
  float loss_q, loss_pi, logp_new;
};
// OUTACT: every critic output is read as y = act(z) (a.act_q), and every gradient w.r.t. one is multiplied by act'(z)
template <bool OUTACT>
__device__ __forceinline__ LossRow loss_row(const LossArgs& a, int i, const float (&m)[2], float alpha) {
  LossRow R;
  const float invB = a.inv_global_batch;
  auto outq = [&](float z) { if constexpr (OUTACT) return act_fwd(z, a.act_q); else return z; };
  const float q1n = outq(a.out_qt[0][2 * i]), s1n = softplus_f(outq(a.out_qt[0][2 * i + 1]));
  const float q2n = outq(a.out_qt[1][2 * i]), s2n = softplus_f(outq(a.out_qt[1][2 * i + 1]));
  const float zc3 = fminf(fmaxf(a.z3[i], -3.f), 3.f), zc4 = fminf(fmaxf(a.z4[i], -3.f), 3.f);
  const float qn = fminf(q1n, q2n);
  const float qn_s = q1n < q2n ? q1n + zc3 * s1n : q2n + zc4 * s2n;  // dsac_v2.py:252-253
  const float nd = (1.f - a.done[i]) * a.gamma, lp2 = a.logp2[i], r = a.rew[i];
  const float y = r + nd * (qn - alpha * lp2);      // dsac_v2.py:293-295
  const float ys = r + nd * (qn_s - alpha * lp2);   // dsac_v2.py:296-298
  R.loss_q = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float zq = a.out_q[k][2 * i], zraw = a.out_q[k][2 * i + 1];
    const float q = outq(zq), raw = outq(zraw);
    const float sd = softplus_f(raw);
    const float b3 = 3.f * m[k];
    const float yb = q + fminf(fmaxf(ys - q, -b3), b3);  // dsac_v2.py:299-301
    const float w = fminf(fmaxf(m[k] * m[k] / (sd * sd + STD_BIAS), 0.1f), 10.f);  // dsac_v2.py:279-280
    const float dq = q - y;
    const float sterm = (sd * sd - huber_f(q - yb)) / (sd + STD_BIAS);
    R.loss_q += w * (huber_f(dq) + sd * sterm);
    R.g_mean[k] = w * fminf(fmaxf(dq, -HUBER_DELTA), HUBER_DELTA) * invB;
    const float dsoft = raw > 20.f ? 1.f : 1.f / (1.f + expf(-raw));
    R.g_raw[k] = w * sterm * invB * dsoft;
    if constexpr (OUTACT) { R.g_mean[k] *= act_bwd(zq, a.act_q); R.g_raw[k] *= act_bwd(zraw, a.act_q); }
    R.q[k] = q;
    R.sd[k] = sd;
  }
  // actor: L_pi = mean(alpha*logp - min(q1pi, q2pi)), dsac_v2.py:304-310; ties split like torch.min
  const float q1p = outq(a.out_qa[0][2 * i]), q2p = outq(a.out_qa[1][2 * i]);
  R.logp_new = a.logp_new[i];
  R.loss_pi = alpha * R.logp_new - fminf(q1p, q2p);
  R.g_pa[0] = q1p < q2p ? -invB : (q1p == q2p ? -0.5f * invB : 0.f);
  R.g_pa[1] = q2p < q1p ? -invB : (q1p == q2p ? -0.5f * invB : 0.f);
  if constexpr (OUTACT) {
    R.g_pa[0] *= act_bwd(a.out_qa[0][2 * i], a.act_q);
    R.g_pa[1] *= act_bwd(a.out_qa[1][2 * i], a.act_q);
  }
  return R;
}
template <bool OUTACT>
__global__ void loss_kernel(const __grid_constant__ LossArgs a) {
  pdl_sync();
  __shared__ float red[10 * 32];
  const float m[2] = {step_mean_std(a.state, a.sc, 0), step_mean_std(a.state, a.sc, 1)};
  const float alpha = step_alpha(a.sc);
  // sums: q1 q2 s1 s2 loss_pi loss_q logp | gb(q1 mean, q1 raw, q2 mean) ; q2 raw handled separately below
  float s[10] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gb_q2_raw = 0.f;
  float mn[2] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000)};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.B; i += gridDim.x * blockDim.x) {
    const LossRow R = loss_row<OUTACT>(a, i, m, alpha);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      a.d_out_q[k][2 * i] = R.g_mean[k];
      a.d_out_q[k][2 * i + 1] = R.g_raw[k];
      img_put(a.img_q[k], i, 0, R.g_mean[k]);
      img_put(a.img_q[k], i, 1, R.g_raw[k]);
      s[k] += R.q[k];
      s[2 + k] += R.sd[k];
      mn[k] = fminf(mn[k], R.sd[k]);
      if (k == 0) { s[7] += R.g_mean[k]; s[8] += R.g_raw[k]; } else { s[9] += R.g_mean[k]; gb_q2_raw += R.g_raw[k]; }
    }
    s[ACC_LOSS_Q] += R.loss_q;
    s[ACC_LOSS_PI] += R.loss_pi;
    s[6] += R.logp_new;
    a.d_out_qa[0][2 * i] = R.g_pa[0]; a.d_out_qa[0][2 * i + 1] = 0.f;
    a.d_out_qa[1][2 * i] = R.g_pa[1]; a.d_out_qa[1][2 * i + 1] = 0.f;
    img_put(a.img_qa[0], i, 0, R.g_pa[0]); img_put(a.img_qa[0], i, 1, 0.f);
    img_put(a.img_qa[1], i, 0, R.g_pa[1]); img_put(a.img_qa[1], i, 1, 0.f);
  }
  block_sum<10>(s, red);
  float one[1] = {gb_q2_raw};
  block_sum<1>(one, red);
  mn[0] = warp_min(mn[0]);
  mn[1] = warp_min(mn[1]);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(reinterpret_cast<int*>(a.state + ST_ACC + ACC_MIN), __float_as_int(mn[0]));
    atomicMin(reinterpret_cast<int*>(a.state + ST_ACC + ACC_MIN + 1), __float_as_int(mn[1]));
  }
  if (threadIdx.x == 0) {
    float* acc = a.state + ST_ACC;
    atomicAdd(acc + ACC_Q1, s[0]); atomicAdd(acc + ACC_Q2, s[1]);
    atomicAdd(acc + ACC_S1, s[2]); atomicAdd(acc + ACC_S2, s[3]);
    atomicAdd(acc + ACC_LOSS_PI, s[4]); atomicAdd(acc + ACC_LOSS_Q, s[5]);
    atomicAdd(acc + ACC_LOGP, s[6]);
    atomicAdd(a.gbias_q[0], s[7]); atomicAdd(a.gbias_q_raw[0] ? a.gbias_q_raw[0] : a.gbias_q[0] + 1, s[8]);
    atomicAdd(a.gbias_q[1], s[9]); atomicAdd(a.gbias_q_raw[1] ? a.gbias_q_raw[1] : a.gbias_q[1] + 1, one[0]);
  }
}

// The critic loss of DSAC_V1 (reference dsac_v1.py:56-273; SURVEY.md §8f rank 4), which has ONE distributional critic
// and a fixed TD bound; it takes the place of loss_kernel in the head-wise engine's phase 2 (`dsact_cnn_config.algo = 1`).
struct LossV1Args {
  const float *rew, *done, *z, *logp2, *logp_new;
  const float *out_q, *out_qt, *out_qa;   // Q(s,a), Q'(s',a'), Q(s,a~): [B,2] (mean, raw std)
  float *d_out_q, *d_out_qa;              // dL/d(mean, raw std)
  float *gbias_q, *gbias_q_raw;           // output-bias gradient (+=); raw: null = gbias_q + 1 (one two-output head)
  float* state;
  int B, bound;
  float gamma, inv_global_batch, td_bound;
  StepScalars sc;
  ImgOut img_q, img_qa;                   // bf16 images of d_out_q / d_out_qa (the MLP engine's dgrad chain reads them)
  int act_q;                              // output activation of the critic (OUTACT instantiation)
};

// __compute_loss_q / __compute_target_q / __compute_loss_policy of dsac_v1.py:195-248, one thread per sample:
//   target = r + (1-d) gamma (q' + clamp(z,-3,3) sigma' - alpha logp'),  target_b = q + clamp(target - q, -TD, TD)
//   bound:  L = mean( -(target - q)/(sigma^2 + 0.1) q - ((q - target_b)^2 - sigma^2)/(sigma^3 + 0.1) sigma )   (coefficients detached)
//   else:   L = mean( -log N(target; q, sigma) )
//   actor:  L_pi = mean( alpha logp - q(s,a~) )
// OUTACT: the critic's outputs are read as y = act(z) (a.act_q), and every gradient w.r.t. one is multiplied by act'(z)
template <bool OUTACT>
__global__ void loss_v1_kernel(const __grid_constant__ LossV1Args a) {
  pdl_sync();
  __shared__ float red[6 * 32];
  const float alpha = step_alpha(a.sc);
  const float invB = a.inv_global_batch;
  auto outq = [&](float z) { if constexpr (OUTACT) return act_fwd(z, a.act_q); else return z; };
  float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // q, sigma, loss_pi, logp, gb_mean, gb_raw
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.B; i += gridDim.x * blockDim.x) {
    const float qn = outq(a.out_qt[2 * i]), sn = softplus_f(outq(a.out_qt[2 * i + 1]));
    const float zc = fminf(fmaxf(a.z[i], -3.f), 3.f);
    const float target = a.rew[i] + (1.f - a.done[i]) * a.gamma * ((qn + zc * sn) - alpha * a.logp2[i]);
    const float q = outq(a.out_q[2 * i]), raw = outq(a.out_q[2 * i + 1]);
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
    float g_raw = g_sd * dsoft;
    float g_qa = -invB;
    if constexpr (OUTACT) {
      g_mean *= act_bwd(a.out_q[2 * i], a.act_q);
      g_raw *= act_bwd(a.out_q[2 * i + 1], a.act_q);
      g_qa *= act_bwd(a.out_qa[2 * i], a.act_q);
    }
    a.d_out_q[2 * i] = g_mean;
    a.d_out_q[2 * i + 1] = g_raw;
    img_put(a.img_q, i, 0, g_mean); img_put(a.img_q, i, 1, g_raw);
    const float lp = a.logp_new[i];
    a.d_out_qa[2 * i] = g_qa;
    a.d_out_qa[2 * i + 1] = 0.f;
    img_put(a.img_qa, i, 0, g_qa); img_put(a.img_qa, i, 1, 0.f);
    s[0] += q; s[1] += sd; s[2] += alpha * lp - outq(a.out_qa[2 * i]); s[3] += lp; s[4] += g_mean; s[5] += g_raw;
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

// Gradient of the actor loss w.r.t. the raw policy-head output (mean | log_std): chain rule through
// a~ = scale*tanh(u)+shift, u = mean + std*eps, and log-prob (SURVEY Appendix A step 1 and 7).
// Also accumulates the output-layer bias gradient.  One warp per row.
struct PolicyGradArgs {
  const float *logits, *eps, *d_act1, *d_act2;  // d_act_k: dL/da~ through critic k  [B,A] (d_act2 unused with one critic)
  const float *hi, *lo;
  float* d_logits;   // [B,2A]
  float* gbias;      // [2A] (+=), or [A] for the mean half when gbias_ls is given
  float* gbias_ls;   // null, or [A]: bias gradient of a separate log_std head
  const float* state;
  int B, A;
  float min_log_std, max_log_std, inv_global_batch;
  ImgOut img;        // bf16 image of the mean half (columns [0, A))
  ImgOut img_ls;     // and of the log_std half, at columns [ls_col, ls_col + A): the same image at column A (one 2A-wide
  int ls_col;        // head), an image of its own at column 0 (a separate log_std head), or none (a log_std row)
  StepScalars sc;
  int gauss;         // 1: GaussDistribution (a~ = u, log-prob of the Normal only)
  OutActs oa;        // output activations of the two halves (OUTACT instantiation)
};
// d(actor loss)/d(mean_j, log_std_j) of one row (chain rule through a~ = scale tanh(u) + shift and the log-prob).
// NQ: critics whose action gradients add up (DSAC-T 2, DSAC_V1 on the MLP engine 1).  OUTACT: the row holds z, the
// distribution reads act(z) (a.oa.mean / a.oa.ls), and the gradients are taken w.r.t. z.
template <int NQ, bool OUTACT>
__device__ __forceinline__ void pgrad_elem(const PolicyGradArgs& a, int row, int j, float coef, float& gu, float& gls) {
  const int A = a.A;
  const float scale = 0.5f * (a.hi[j] - a.lo[j]);
  const float zm = a.logits[(size_t)row * 2 * A + j];
  const float zl = a.logits[(size_t)row * 2 * A + A + j];
  float mean = zm, ls = zl;
  if constexpr (OUTACT) { mean = act_fwd(zm, a.oa.mean); ls = act_fwd(zl, a.oa.ls); }
  const bool inside = ls >= a.min_log_std && ls <= a.max_log_std;
  const float sd = expf(fminf(fmaxf(ls, a.min_log_std), a.max_log_std));
  const float e = a.eps[(size_t)row * A + j];
  const float da = NQ == 2 ? a.d_act1[(size_t)row * A + j] + a.d_act2[(size_t)row * A + j] : a.d_act1[(size_t)row * A + j];
  if (a.gauss) {   // a~ = u; d logp / d mean = 0, d logp / d sd = -1/sd
    gu = da;
    gls = inside ? (gu * e - coef / sd) * sd : 0.f;
  } else {
    const float th = tanhf(mean + sd * e);
    const float om = 1.f - th * th;
    gu = da * scale * om + coef * (2.f * th * om / (1.f + TG_EPS - th * th));
    const float gsd = gu * e - coef / sd;
    gls = inside ? gsd * sd : 0.f;
  }
  if constexpr (OUTACT) { gu *= act_bwd(zm, a.oa.mean); gls *= act_bwd(zl, a.oa.ls); }
}
template <int NQ, bool OUTACT>
__global__ void policy_grad_kernel(const __grid_constant__ PolicyGradArgs a) {
  pdl_sync();
  extern __shared__ float gb[];   // [2A] block-local bias-gradient sums
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5, warp = threadIdx.x >> 5;
  const int A = a.A;
  for (int i = threadIdx.x; i < 2 * A; i += blockDim.x) gb[i] = 0.f;
  __syncthreads();
  const float coef = step_alpha(a.sc) * a.inv_global_batch;  // dL/dlogp
  for (int j0 = 0; j0 < A; j0 += 32) {   // block-uniform loop (barriers inside)
    const int j = j0 + lane;
    float gb_mean = 0.f, gb_ls = 0.f;
    for (int row = blockIdx.x * wpb + warp; j < A && row < a.B; row += gridDim.x * wpb) {
      float gu, gls;
      pgrad_elem<NQ, OUTACT>(a, row, j, coef, gu, gls);
      a.d_logits[(size_t)row * 2 * A + j] = gu;
      a.d_logits[(size_t)row * 2 * A + A + j] = gls;
      img_put(a.img, row, j, gu);
      img_put(a.img_ls, row, a.ls_col + j, gls);
      gb_mean += gu;
      gb_ls += gls;
    }
    // the warps add their partial sums in warp order, so the block's sum does not depend on warp timing (with at most
    // two blocks, as for batches up to 16 rows, the bias gradient is then the same bits on every run)
    for (int w = 0; w < wpb; ++w) {
      if (warp == w && j < A) { gb[j] += gb_mean; gb[A + j] += gb_ls; }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < 2 * A; i += blockDim.x) atomicAdd((a.gbias_ls && i >= A) ? a.gbias_ls + (i - A) : a.gbias + i, gb[i]);
}

// std_type "parameter" (networks/mlp.py:63-64,94-96): log_std is a learnable [1, A] row, the same for every sample.  Writes
// the rows of pi and pi' into the log_std half of their [B, 2A] logits, where sample_kernel and policy_grad_kernel read
// any other policy's log_std.
__global__ void log_std_rows_kernel(float* __restrict__ logitsP, float* __restrict__ logitsT, const float* __restrict__ rowP,
                                    const float* __restrict__ rowT, int B, int A) {
  pdl_sync();
  const int total = B * A;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / A, j = i - r * A;
    logitsP[(size_t)r * 2 * A + A + j] = rowP[j];
    logitsT[(size_t)r * 2 * A + A + j] = rowT[j];
  }
}

// __update (dsac_v2.py:320-347): Adam on q1|q2 every step; on policy|log_alpha plus Polyak of all three
// targets when iteration % delay_update == 0.  One pass over the flat buffers; also writes the gradient
// of log_alpha (dsac_v2.py:312-318) from the accumulated sum of log-probs.
// Step sizes lr/(1-beta1^t) and sqrt(1-beta2^t) in double, like the Python scalars of torch's Adam:
// out = {lr_q/bc1q, sqrt(bc2q), lr_pi/bc1p, lr_alpha/bc1p, sqrt(bc2p)}.  A few hundred dependent FP64 instructions: done
// once per step by the phase-2 tail (single-call steps) instead of by thread 0 of every apply block.
struct AdamHyper { double lr_q, lr_pi, lr_alpha, b1, b2; };
__device__ __forceinline__ void adam_scalars(const int* sti, const AdamHyper& a, float* out) {
  const double tq = sti[ST_ADAM_Q] + 1, tp = sti[ST_ADAM_PI] + 1;
  const double bc1q = 1.0 - pow(a.b1, tq), bc1p = 1.0 - pow(a.b1, tp);
  out[0] = (float)(a.lr_q / bc1q);
  out[1] = (float)sqrt(1.0 - pow(a.b2, tq));
  out[2] = (float)(a.lr_pi / bc1p);
  out[3] = (float)(a.lr_alpha / bc1p);
  out[4] = (float)sqrt(1.0 - pow(a.b2, tp));
}
constexpr int ADAM_SC_MAGIC = 0x5ca1ab1e;   // state[ST_ADAM_SC + 7]: slots +0..4 hold the scalars for the counters in +5, +6
// The same five scalars by four lanes of one warp (one double-precision pow each: a single thread needs ~5 us for them),
// stamped with the counters they belong to.  Called by the step prologue: off the critical path, the counters are final
// there (the previous step's apply advanced them), and apply_kernel finds the stamp.
__device__ __forceinline__ void adam_scalars_stamp(float* state, const AdamHyper& a) {
  const int t = threadIdx.x;
  int* sti = reinterpret_cast<int*>(state);
  if (t < 4) {
    const double step = ((t & 1) ? sti[ST_ADAM_PI] : sti[ST_ADAM_Q]) + 1;
    const double pw = pow(t < 2 ? a.b1 : a.b2, step);
    if (t == 0) state[ST_ADAM_SC + 0] = (float)(a.lr_q / (1.0 - pw));
    else if (t == 1) { state[ST_ADAM_SC + 2] = (float)(a.lr_pi / (1.0 - pw)); state[ST_ADAM_SC + 3] = (float)(a.lr_alpha / (1.0 - pw)); }
    else if (t == 2) state[ST_ADAM_SC + 1] = (float)sqrt(1.0 - pw);
    else state[ST_ADAM_SC + 4] = (float)sqrt(1.0 - pw);
    if (t == 0) { sti[ST_ADAM_SC + 5] = sti[ST_ADAM_Q]; sti[ST_ADAM_SC + 6] = sti[ST_ADAM_PI]; sti[ST_ADAM_SC + 7] = ADAM_SC_MAGIC; }
  }
}
// The end-of-backward bookkeeping of a step (phase2_tail_kernel below) folded into the kernels that follow it in the
// single-call steps: the log_alpha gradient is formed where the gradient element is consumed, the EMA / temperature
// commit and the NEXT step's Adam scalars are written by the last block of apply_kernel.
struct TailArgs {
  StepScalars sc;
  float target_entropy;
  int rows;       // local shard size
  int enabled;
};
__device__ __forceinline__ float tail_grad_log_alpha(const float* state, const TailArgs& t) {
  return -(state[ST_ACC + ACC_LOGP] + (float)t.rows * t.target_entropy) * t.sc.inv_global_batch;
}
struct ApplyArgs {
  float *params, *targets, *grads, *m, *v;
  TailArgs tail;
  float* state;
  int64_t n_q2;      // 2*n_q  (critic span)
  int64_t n_all;     // 2*n_q + n_pi + 1
  int delay_update, auto_alpha;
  AdamHyper hy;
  int scalars_ready;   // the Adam scalars: 0 = formed here, 1 = phase2_tail_kernel of this step wrote them, 2 = stamped (see below)
  float omb1, b2f, omb2, eps, tau;  // (float)(1-beta1), (float)beta2, (float)(1-beta2) formed in double on the host
  // tensor-core modes, single-call steps: the weight-gradient split slabs are folded in here (grads += sum of slabs, stored
  // back so that the caller's .grad views hold the totals) instead of by a separate grad_reduce launch
  const float* slabs;
  int nslabs;
  long long slab_stride;
  // peer-memory data parallelism (dp_peer.cuh): the global gradient is the rank-ordered sum of every rank's block
  const float* dp_grads[8];
  int dp_world;
  // two-shot exchange (dp_peer.cuh): dp_world == 1, dp_grads[0] = this rank's reduced block; wait for `dp_wait_world`
  // kind-2 flags in `dp_own` first
  const float* dp_own;
  int dp_wait_world;
  unsigned long long dp_timeout_ns;
  // 4-element groups [g_lo, g_hi) of the flat buffers this launch updates; `finish`: its last block closes the step
  // (counters, EMA commit, next Adam scalars).  A step may update the critics' span early, beside the policy backward,
  // with finish = 0, and the rest afterwards with finish = 1.
  int64_t g_lo, g_hi;
  int finish;
  int next_scalars;   // the finishing block also precomputes the NEXT step's Adam scalars (steps whose prologue does not)
};
__device__ __forceinline__ bool dp_wait_reduced(const float* own_buf, int world, uint32_t epoch, unsigned long long timeout_ns);
// torch.optim.Adam single-tensor step (amsgrad / weight decay off)
__device__ __forceinline__ float adam_update(float w, float g, float& m, float& v, float step_size, float bc2_sqrt,
                                             float omb1, float b2, float omb2, float eps) {
  m = m + (g - m) * omb1;                  // exp_avg.lerp_(grad, 1-beta1)
  v = v * b2 + omb2 * g * g;               // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2)
  const float denom = sqrtf(v) / bc2_sqrt + eps;
  return w - step_size * (m / denom);      // param.addcdiv_(exp_avg, denom, value=-lr/bias_correction1)
}
// MODE 0: gradients as they are in `grads`; 1: + the weight-gradient split slabs; 2: rank-ordered sum of the peers' blocks.
// Four blocks per SM (<= 64 registers): the pass is a single sweep of ~13 independent 16-byte streams per thread and is
// bound by how many loads the SM keeps in flight (the 88-register version ran at 2 blocks per SM and 1 TB/s).
template <int MODE>
__global__ void __launch_bounds__(256, 4) apply_kernel(const __grid_constant__ ApplyArgs a) {
  pdl_sync();
  __shared__ float sh[6];
  const int* sti = reinterpret_cast<const int*>(a.state);
  const bool delayed = (sti[ST_ITER] % a.delay_update) == 0;
  // scalars_ready: 1 = written by phase2_tail_kernel of this step; 2 = possibly precomputed by the previous apply (or
  // set_carry): valid if stamped with the current counters; 0 = compute here
  const bool stamped = a.scalars_ready == 2 && sti[ST_ADAM_SC + 7] == ADAM_SC_MAGIC && sti[ST_ADAM_SC + 5] == sti[ST_ADAM_Q] &&
                       sti[ST_ADAM_SC + 6] == sti[ST_ADAM_PI];
  if (a.scalars_ready == 1 || stamped) {
    if (threadIdx.x < 5) sh[threadIdx.x] = a.state[ST_ADAM_SC + threadIdx.x];
  } else if (threadIdx.x == 0) {
    adam_scalars(sti, a.hy, sh);
  }
  if (MODE == 2 && a.dp_wait_world > 0 && threadIdx.x == 32) {   // two-shot exchange: the reduced block is complete
    if (!dp_wait_reduced(a.dp_own, a.dp_wait_world, (uint32_t)sti[ST_DP_EPOCH], a.dp_timeout_ns))
      reinterpret_cast<int*>(a.state)[ST_DP_ERR] = 1 + a.dp_wait_world;   // (no single rank to name)
  }
  __syncthreads();
  const int64_t n_targets = a.n_all - 1;
  const float polyak = 1.f - a.tau;
  // 4 consecutive elements per thread (float4 traffic); a group is uniform unless it straddles the critic/policy
  // boundary or holds log_alpha, so the per-element logic below stays cheap
  for (int64_t gi = a.g_lo + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gi < a.g_hi; gi += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i0 = gi * 4;
    const bool full = i0 + 3 < n_targets;
    float w[4], g[4], m[4], v[4], t[4];
    if (full) {
      const float4 W4 = reinterpret_cast<const float4*>(a.params)[gi], G4 = reinterpret_cast<const float4*>(a.grads)[gi];
      const float4 M4 = reinterpret_cast<const float4*>(a.m)[gi], V4 = reinterpret_cast<const float4*>(a.v)[gi];
      w[0] = W4.x; w[1] = W4.y; w[2] = W4.z; w[3] = W4.w; g[0] = G4.x; g[1] = G4.y; g[2] = G4.z; g[3] = G4.w;
      m[0] = M4.x; m[1] = M4.y; m[2] = M4.z; m[3] = M4.w; v[0] = V4.x; v[1] = V4.y; v[2] = V4.z; v[3] = V4.w;
      if (delayed) {
        const float4 T4 = reinterpret_cast<const float4*>(a.targets)[gi];
        t[0] = T4.x; t[1] = T4.y; t[2] = T4.z; t[3] = T4.w;
      }
      if (MODE == 2) {
#pragma unroll 1
        for (int r0 = 0; r0 < a.dp_world; r0 += 4) {   // four peers' loads in flight at a time, summed in rank order
          float4 p[4];
#pragma unroll
          for (int r = 0; r < 4; ++r)
            if (r0 + r < a.dp_world) {
              asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];"
                           : "=f"(p[r].x), "=f"(p[r].y), "=f"(p[r].z), "=f"(p[r].w) : "l"(a.dp_grads[r0 + r] + 4 * gi) : "memory");
            }
#pragma unroll
          for (int r = 0; r < 4; ++r)
            if (r0 + r < a.dp_world) {
              if (r0 + r == 0) { g[0] = p[0].x; g[1] = p[0].y; g[2] = p[0].z; g[3] = p[0].w; }
              else { g[0] += p[r].x; g[1] += p[r].y; g[2] += p[r].z; g[3] += p[r].w; }
            }
        }
        reinterpret_cast<float4*>(a.grads)[gi] = make_float4(g[0], g[1], g[2], g[3]);
      } else if (MODE == 1) {
#pragma unroll 1
        for (int k0 = 0; k0 < a.nslabs; k0 += 4) {   // independent loads first, then the sum in slab order
          float4 p[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            p[k] = k0 + k < a.nslabs ? __ldg(reinterpret_cast<const float4*>(a.slabs + (size_t)(k0 + k) * a.slab_stride) + gi)
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < 4; ++k) { g[0] += p[k].x; g[1] += p[k].y; g[2] += p[k].z; g[3] += p[k].w; }
        }
        reinterpret_cast<float4*>(a.grads)[gi] = make_float4(g[0], g[1], g[2], g[3]);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + e;
        const bool in = i < a.n_all;
        w[e] = in ? a.params[i] : 0.f; g[e] = in ? a.grads[i] : 0.f; m[e] = in ? a.m[i] : 0.f; v[e] = in ? a.v[i] : 0.f;
        t[e] = (in && i < n_targets) ? a.targets[i] : 0.f;
        if (in && MODE == 2) {
          float acc = 0.f;
          for (int r = 0; r < a.dp_world; ++r) {
            float v;
            asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(a.dp_grads[r] + i) : "memory");
            acc = r == 0 ? v : acc + v;
          }
          g[e] = acc;
          a.grads[i] = acc;
        } else if (in && MODE == 1) {
          for (int k = 0; k < a.nslabs; ++k) g[e] += a.slabs[(size_t)k * a.slab_stride + i];
          a.grads[i] = g[e];
        }
        if (a.tail.enabled && i == a.n_all - 1) {   // log_alpha: dsac_v2.py:312-318 (data parallel: dp_grad_fold_kernel formed it)
          if (MODE != 2) { g[e] = tail_grad_log_alpha(a.state, a.tail); a.grads[i] = g[e]; }
          a.state[ST_ALPHA_USED] = a.tail.sc.auto_alpha ? expf(w[e]) : a.tail.sc.alpha_fixed;   // temperature this step used
        }
      }
    }
    bool touched = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t i = i0 + e;
      if (i >= a.n_all) continue;
      const bool critic = i < a.n_q2;
      if (critic || delayed) {
        const bool is_alpha = i == a.n_all - 1;
        if (!(is_alpha && !a.auto_alpha)) {
          const float step = critic ? sh[0] : (is_alpha ? sh[3] : sh[2]);
          w[e] = adam_update(w[e], g[e], m[e], v[e], step, critic ? sh[1] : sh[4], a.omb1, a.b2f, a.omb2, a.eps);
          touched = true;
        }
      }
      if (delayed && i < n_targets) t[e] = t[e] * polyak + (1.f - polyak) * w[e];  // p_targ.mul_(polyak).add_((1-polyak)*p)
    }
    if (full) {
      if (touched) {
        reinterpret_cast<float4*>(a.params)[gi] = make_float4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<float4*>(a.m)[gi] = make_float4(m[0], m[1], m[2], m[3]);
        reinterpret_cast<float4*>(a.v)[gi] = make_float4(v[0], v[1], v[2], v[3]);
      }
      if (delayed) reinterpret_cast<float4*>(a.targets)[gi] = make_float4(t[0], t[1], t[2], t[3]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + e;
        if (i >= a.n_all) continue;
        if (touched) { a.params[i] = w[e]; a.m[i] = m[e]; a.v[i] = v[e]; }
        if (delayed && i < n_targets) a.targets[i] = t[e];
      }
    }
  }
  // the block that finishes last advances the counters every block read at its start
  if (!a.finish) return;
  __syncthreads();
  if (threadIdx.x == 0) {
    int* stw = reinterpret_cast<int*>(a.state);
    __threadfence();
    if (atomicAdd(stw + ST_TICKET, 1) == (int)gridDim.x - 1) {
      if (a.tail.enabled) {   // commit of the mean_std EMA (every reader of this step used the carried values)
        const float m0 = step_mean_std(a.state, a.tail.sc, 0), m1 = step_mean_std(a.state, a.tail.sc, 1);
        a.state[ST_MEAN_STD1] = m0;
        a.state[ST_MEAN_STD2] = m1;
      }
      stw[ST_ADAM_Q] += 1;
      if (delayed) stw[ST_ADAM_PI] += 1;
      stw[ST_ITER] += 1;
      stw[ST_TICKET] = 0;
      if (a.tail.enabled && a.next_scalars) {   // the next step's Adam scalars, stamped with the counters they belong to
        adam_scalars(stw, a.hy, a.state + ST_ADAM_SC);
        stw[ST_ADAM_SC + 5] = stw[ST_ADAM_Q];
        stw[ST_ADAM_SC + 6] = stw[ST_ADAM_PI];
        stw[ST_ADAM_SC + 7] = ADAM_SC_MAGIC;
      }
    }
  }
}
__global__ void set_iter_kernel(float* __restrict__ state, int iteration) {
  pdl_sync();
  if (threadIdx.x == 0) reinterpret_cast<int*>(state)[ST_ITER] = iteration;
}
__global__ void set_rb_size_kernel(float* __restrict__ state, int64_t size) {
  pdl_sync();
  if (threadIdx.x == 0) *reinterpret_cast<int64_t*>(state + ST_RB_SIZE) = size;
}
__global__ void rng_advance_kernel(float* __restrict__ state) {
  pdl_sync();
  if (threadIdx.x == 0) reinterpret_cast<uint32_t*>(state)[ST_RNG_CTR] += 1u;
}

// End of the backward pass: gradient of log_alpha (dsac_v2.py:312-318) = -(mean(logp_new) + target_entropy), and the
// commit of this step's mean_std EMA and temperature to the state (every earlier reader used the carried values).
// `rows` = local shard size, so that per-rank values sum to the global gradient under data parallelism.
__global__ void phase2_tail_kernel(float* __restrict__ grad_log_alpha, float* __restrict__ state, const StepScalars sc,
                                   float target_entropy, int rows, const AdamHyper hy, int with_adam) {
  pdl_sync();
  const int t = threadIdx.x;
  if (with_adam && t == 4) adam_scalars(reinterpret_cast<const int*>(state), hy, state + ST_ADAM_SC);
  float val = 0.f;
  if (t < 2) val = step_mean_std(state, sc, t);
  else if (t == 2) val = step_alpha(sc);
  else if (t == 3) *grad_log_alpha = -(state[ST_ACC + ACC_LOGP] + (float)rows * target_entropy) * sc.inv_global_batch;
  __syncwarp();
  if (t < 2) state[ST_MEAN_STD1 + t] = val;
  else if (t == 2) state[ST_ALPHA_USED] = val;
}

// tb_info (dsac_v2.py:188-202) from the accumulators, into `out` (16 floats; null: the state's ST_STATS slots).
__global__ void finalize_stats_kernel(float* __restrict__ state, float inv_global_batch, float inv_policy_elems,
                                      float* __restrict__ out) {
  pdl_sync();
  if (threadIdx.x != 0) return;
  const float* acc = state + ST_ACC;
  float* o = out ? out : state + ST_STATS;
  o[0] = acc[ACC_Q1] * inv_global_batch;
  o[1] = acc[ACC_Q2] * inv_global_batch;
  o[2] = acc[ACC_S1] * inv_global_batch;
  o[3] = acc[ACC_S2] * inv_global_batch;
  o[4] = acc[ACC_MIN];
  o[5] = acc[ACC_MIN + 1];
  o[6] = acc[ACC_LOSS_PI] * inv_global_batch;
  o[7] = acc[ACC_LOSS_Q] * inv_global_batch;
  o[8] = acc[ACC_TANH_MEAN] * inv_policy_elems;
  o[9] = acc[ACC_PI_STD] * inv_policy_elems;
  o[10] = -acc[ACC_LOGP] * inv_global_batch;
  o[11] = state[ST_ALPHA_USED];
  o[12] = state[ST_MEAN_STD1];
  o[13] = state[ST_MEAN_STD2];
  o[14] = (float)reinterpret_cast<const int*>(state)[ST_DP_ERR];   // 0, or 1 + rank of the peer that timed out
  o[15] = 0.f;
}

__global__ void set_carry_kernel(float* __restrict__ state, float m1, float m2, int tq, int tp) {
  pdl_sync();
  if (threadIdx.x == 0) {
    state[ST_MEAN_STD1] = m1;
    state[ST_MEAN_STD2] = m2;
    reinterpret_cast<int*>(state)[ST_ADAM_Q] = tq;
    reinterpret_cast<int*>(state)[ST_ADAM_PI] = tp;
  }
}

}  // namespace dsact
