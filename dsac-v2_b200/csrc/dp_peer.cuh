// Data-parallel replicas over NVLink peer memory (SURVEY.md §8e): the two exchanges of a data-parallel DSAC-T step
// (critic-std sums before the loss; gradients + logged sums before Adam) done by the step's own kernels on buffers
// that every rank maps with CUDA IPC, so that the whole step stays ONE captured graph per rank: no host round trip,
// no NCCL launch between the phases.
//
// Per rank one cudaMalloc'd exchange buffer (floats):
//   [0, 128)                      arrival flags (uint32 epochs): flag[kind * 16 + source_rank]; word 96: block ticket
//   [128, 128 + 2*2*R*32)         small payloads: small[kind][parity][source_rank][32]
//   [DP_GRADS_OFF, + n_params)    this rank's local gradient sum of the running step
//   [DP_GRADS_OFF + n_pad, + n_params)  the global gradient sum ("reduced" block; two-shot exchange only, see below)
// kind 0 = after the forward passes (2 std sums, SUM), kind 1 = before Adam (16 logged sums SUM + 2 minima MIN; it is
// also the "local gradients are complete" barrier), kind 2 = the reduced slices of the two-shot exchange have arrived
// (no payload).  Every rank pushes its payload into every peer's buffer, raises its flag there (release, system scope)
// and polls only its own memory.  Reductions run in rank order on every rank, so the replicas stay bit-identical.
// Reuse is safe without further barriers: a rank overwrites its gradient block in phase 2 of step t+1, i.e. after the
// kind-0 barrier of t+1, which every peer reaches only after its apply of t.
//
// Gradient exchange, two variants.  ONE-SHOT (world < 6): apply_kernel reads every rank's block through NVLink and sums
// in rank order — (N-1) x n floats cross the links per rank.  TWO-SHOT (world >= 6, dp_reduce_scatter_kernel): rank r
// sums slice r of every rank's block in rank order (reads (N-1)/N x n), writes the sum into slice r of EVERY rank's
// reduced block (writes (N-1)/N x n), raises its kind-2 flag everywhere; apply_kernel waits for all kind-2 flags and then
// reads only local memory.  At N = 8 that is 2 x 2.46 MB per rank instead of 19.7 MB.  Sums run in rank order on the
// one rank that owns the slice, so the replicas still hold bit-identical gradients.
#pragma once
#include <stdint.h>

#include "kernels.cuh"

namespace dsact {

constexpr int DP_MAX_RANKS = 8;
constexpr int DP_FLAGS = 128;   // kinds 0-2 x 16 ranks of arrival flags, then the block ticket of the reduce-scatter launch
constexpr int DP_TICKET = 96;   // header word 96
constexpr int DP_SMALL = 32;
constexpr int DP_SMALL_OFF = DP_FLAGS;
constexpr int DP_GRADS_OFF = 2048;   // floats; 8 KiB header

struct DpComm {
  float* peer[DP_MAX_RANKS];   // peer[rank] = this rank's own buffer
  int rank, world;
};

// Host-side exchange state of one handle (MLP or head-wise engine): the buffer it exports, the peers' buffers as opened
// here, and the rank map the kernels take.  Export / connect / release are in engine.cu (dp_peer_*).
struct DpPeer {
  float* buf = nullptr;                   // this rank's exchange buffer (cudaMalloc, exported with CUDA IPC)
  void* opened[DP_MAX_RANKS] = {};        // peers' buffers as opened here
  DpComm comm = {};
  bool ready = false;                     // dp_peer_connect succeeded
  long long n_params = 0;                 // length of the flat gradient buffer the blocks mirror
  long long npad() const { return (n_params + 3) / 4 * 4; }   // a block, padded to whole float4 groups
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_sys_f4(const float* p) {   // coherent at the owner's L2, never the read-only path
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_sys_f(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long dp_time_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// One block of 32 * world threads.  kind 0: all-reduce state[ST_STDSUM..+1] (SUM) and open epoch e = epoch + 1;
// kind 1: all-reduce the 16 sums (SUM) and 2 minima (MIN) of state[ST_ACC..] at the epoch kind 0 opened.
// A peer that does not arrive within `timeout_ns` sets state[ST_DP_ERR] instead of hanging the GPU.
__device__ __forceinline__ void dp_exchange(const DpComm& c, float* __restrict__ state, int kind, unsigned long long timeout_ns) {
  int* sti = reinterpret_cast<int*>(state);
  const uint32_t e = (uint32_t)sti[ST_DP_EPOCH] + (kind == 0 ? 1u : 0u);
  const int par = (int)(e & 1u);
  const int n = kind == 0 ? 2 : 18;
  float* src = kind == 0 ? state + ST_STDSUM : state + ST_ACC;   // (the 2 minima sit at ST_ACC + 16, 17)
  const int t = threadIdx.x, p = t >> 5, i = t & 31;
  // 1. push my payload into every rank's small[kind][par][my rank][...]
  if (p < c.world && i < n) {
    float* dst = c.peer[p] + DP_SMALL_OFF + ((kind * 2 + par) * DP_MAX_RANKS + c.rank) * DP_SMALL;
    dst[i] = src[i];
    __threadfence_system();
  }
  __syncthreads();
  // 2. raise my flag at every rank, then wait for every rank's flag here
  if (t < c.world) {
    st_release_sys(reinterpret_cast<uint32_t*>(c.peer[t]) + kind * 16 + c.rank, e);
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(c.peer[c.rank]) + kind * 16 + t;
    const unsigned long long t0 = dp_time_ns();
    while ((int32_t)(ld_acquire_sys(mine) - e) < 0) {
      if (dp_time_ns() - t0 > timeout_ns) { sti[ST_DP_ERR] = 1 + t; break; }
      __nanosleep(64);
    }
  }
  __syncthreads();
  // 3. reduce in rank order (identical on every rank)
  if (t < n) {
    const float* base = c.peer[c.rank] + DP_SMALL_OFF + (kind * 2 + par) * DP_MAX_RANKS * DP_SMALL;
    float acc = ld_sys_f(base + t);
    for (int r = 1; r < c.world; ++r) {
      const float v = ld_sys_f(base + r * DP_SMALL + t);
      acc = (kind == 1 && t >= 16) ? fminf(acc, v) : acc + v;
    }
    src[t] = acc;
  }
  if (kind == 0 && t == 0) sti[ST_DP_EPOCH] = (int)e;
}
__global__ void dp_exchange_kernel(const DpComm c, float* __restrict__ state, int kind, unsigned long long timeout_ns) {
  pdl_sync();
  dp_exchange(c, state, kind, timeout_ns);
}

// Test hook only (dsact_test_dp): the exchange of a whole world of ranks on one device in one cooperative launch, block r
// being rank r.  Cooperative launch keeps the W blocks resident together, so every flag wait can resolve.
struct DpTestWorld {
  DpComm comm[DP_MAX_RANKS];
  float* state[DP_MAX_RANKS];
};
__global__ void dp_exchange_world_kernel(const __grid_constant__ DpTestWorld w, int kind, unsigned long long timeout_ns) {
  dp_exchange(w.comm[blockIdx.x], w.state[blockIdx.x], kind, timeout_ns);
}

// grads_out[i] = grads[i] + sum of the weight-gradient slabs (the local total, into the exchange buffer)
// `tail`.enabled: the log_alpha element (index n - 1) is formed here from the logged sum (phase2_tail_kernel folded in)
__global__ void dp_grad_fold_kernel(float* __restrict__ out, const float* __restrict__ grads, const float* __restrict__ slabs,
                                    long long n, int nslabs, long long slab_stride, const float* __restrict__ state, const TailArgs tail) {
  pdl_sync();
  const bool vec = (slab_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(grads) & 15) == 0 && (reinterpret_cast<uintptr_t>(slabs) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  const long long n4 = vec ? (tail.enabled ? n - 1 : n) / 4 : 0;   // the log_alpha element always takes the scalar path
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = reinterpret_cast<const float4*>(grads)[i];
    for (int k = 0; k < nslabs; ++k) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(slabs + (size_t)k * slab_stride) + i);
      s.x += q.x; s.y += q.y; s.z += q.z; s.w += q.w;
    }
    reinterpret_cast<float4*>(out)[i] = s;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = grads[i];
    for (int k = 0; k < nslabs; ++k) s += slabs[(size_t)k * slab_stride + i];
    if (tail.enabled && i == n - 1) s = tail_grad_log_alpha(state, tail);
    out[i] = s;
  }
}

// Two-shot exchange, first half + broadcast: this rank owns slice [lo, hi) (in float4 groups).  Launched after the
// kind-1 exchange (every rank's block is complete).  The block that finishes last raises this rank's kind-2 flag at every
// peer (release, system scope) after the slice has been written everywhere.
struct DpSlice {
  long long g_lo, g_hi;      // float4 groups of this rank's slice
  long long red_off;         // floats from a rank's buffer base to its reduced block
  int* ticket;               // zero-initialised int in this rank's buffer header
};
__global__ void __launch_bounds__(256) dp_reduce_scatter_kernel(const DpComm c, const DpSlice sl, const float* __restrict__ state) {
  pdl_sync();
  const uint32_t e = (uint32_t)reinterpret_cast<const int*>(state)[ST_DP_EPOCH];
  for (long long gi = sl.g_lo + blockIdx.x * (long long)blockDim.x + threadIdx.x; gi < sl.g_hi; gi += (long long)gridDim.x * blockDim.x) {
    float4 acc = ld_sys_f4(c.peer[0] + DP_GRADS_OFF + 4 * gi);
    for (int r0 = 1; r0 < c.world; r0 += 4) {   // up to four peers' loads in flight, summed in rank order
      float4 p[4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (r0 + r < c.world) p[r] = ld_sys_f4(c.peer[r0 + r] + DP_GRADS_OFF + 4 * gi);
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (r0 + r < c.world) { acc.x += p[r].x; acc.y += p[r].y; acc.z += p[r].z; acc.w += p[r].w; }
    }
    for (int r = 0; r < c.world; ++r)
      asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(c.peer[r] + sl.red_off + 4 * gi), "f"(acc.x), "f"(acc.y),
                   "f"(acc.z), "f"(acc.w) : "memory");
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(sl.ticket, 1) == (int)gridDim.x - 1) {
      *sl.ticket = 0;
      __threadfence_system();
      for (int r = 0; r < c.world; ++r) st_release_sys(reinterpret_cast<uint32_t*>(c.peer[r]) + 2 * 16 + c.rank, e);
    }
  }
}

// apply_kernel's side of the two-shot exchange: one thread per block waits until every rank's kind-2 flag of this epoch
// has arrived in this rank's own memory (the reduced block is then complete).  Returns false on timeout.
__device__ __forceinline__ bool dp_wait_reduced(const float* own_buf, int world, uint32_t epoch, unsigned long long timeout_ns) {
  const uint32_t* flags = reinterpret_cast<const uint32_t*>(own_buf) + 2 * 16;
  const unsigned long long t0 = dp_time_ns();
  for (int r = 0; r < world; ++r)
    while ((int32_t)(ld_acquire_sys(flags + r) - epoch) < 0) {
      if (dp_time_ns() - t0 > timeout_ns) return false;
      __nanosleep(32);
    }
  return true;
}

}  // namespace dsact
