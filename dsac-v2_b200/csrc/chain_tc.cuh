// Fused MLP layer-chain kernel on wgmma (DSACT_GEMM_BF16X3 / DSACT_GEMM_BF16), sm_90a.
//
// One CTA carries one 64-row block of one "pass" (an MLP applied to one input) through ALL of its layers:
//   forward chain : x -> [Linear + act] x L -> Linear            (reference networks/mlp.py:15-20)
//   dgrad chain   : dOut -> [dY W_j (.) act'(z_{j-1})] x L (-> dY W_0[:, act columns] for the actor path)
// Layer 0 takes its A operand from global memory by TMA (the bf16 hi/lo images of obs / act / dOut); every later
// layer takes A from SHARED MEMORY: the epilogue of layer j writes act(z_j) (or dz_j) as bf16 hi/lo pairs, in the
// 128-byte-swizzled K-major layout wgmma reads, into the operand buffer, so hidden activations never leave the SM
// unless the backward pass needs them (act' for the dgrad chain, images for wgrad).
// The weight tiles of layer j+1 are prefetched by the TMA warp while the epilogue of layer j runs.  The MMAs of a k-block
// issue back to back and one k-block stays in flight while the next is issued; the layer width (64, 128, 192 or 256) is
// a compile-time parameter of each layer's body, dispatched once per layer.
//
// Shared memory: [ B ring: stages x planes x stage_b ][ operand buffer: planes x 4 k-blocks x 8 KiB (layer 0: its A
// ring) ][ 16-float scratch row per MMA thread ][ barriers ].
// Roles: warps 0..3 the MMA warpgroup (wgmma, accumulator in registers, epilogue), warp 4 TMA producer.
#pragma once
#include "gemm_tc.cuh"

namespace dsact {

constexpr int CH_MAX_LAYERS = DSACT_MAX_HIDDEN + 1;
constexpr int CH_MAX_PASSES = 4;
constexpr int CH_KB_MAX = 4;                              // 256 columns of operand = 4 k-blocks of 64
constexpr int CH_OPND_PLANE = CH_KB_MAX * TC_STAGE_A;     // 32 KiB

struct ChainLayer {
  CUtensorMap mapB;          // weight image; forward: K-major (box = bn rows), dgrad: MN-major (box = 64 x 64)
  int kblocks[2];            // k-blocks of 64; layer 0 may have two A segments, later layers use [0] only
  int kB0[2];                // offset of each segment along B's reduction dimension
  int N, bn;                 // outputs; tile width (multiple of 16, <= 256)
  int epi, act;             // EPI_BIAS_ACT | EPI_DACT | EPI_STORE
  const float* bias;
  float* Zout;               // forward: act'(pre-activation) store, ld = N (null: not needed by a backward pass)
  const float* Zin;          // dgrad: act'(pre-activation) of the layer below, ld = N
  float* colsum;             // dgrad: bias gradient (+=)
  float* C;                  // fp32 result, ld = N (head layers)
  __nv_bfloat16* img;        // bf16 hi/lo image of the result for the weight-gradient GEMM (null: not needed)
  int img_pitch;
  long long img_plane;
};

struct ChainPass {
  CUtensorMap mapA[2];       // layer-0 A operand segments (K-major images, box = 64 rows)
  int n_layers, M, tile_start;
  ChainLayer L[CH_MAX_LAYERS];
};

struct ChainGroup {
  int n, passes;
  unsigned long long* dbg;
  ChainPass p[CH_MAX_PASSES];
};

inline int chain_smem_bytes(int stages, int planes, int stage_b) {
  return stages * planes * stage_b + planes * CH_OPND_PLANE + TC_SCRATCH + 2 * stages * 8 + 1024;
}

// One layer on the MMA warpgroup, 64 x (64 NB) outputs: the MMAs with one k-block in flight (the ring slot of k-block kb is
// released once kb + 1 has been issued and kb has retired), the epilogue on the accumulator registers, and the next
// layer's A operand.  (stage, phase) is the consumer's position in the B ring, carried from layer to layer.
template <bool PLANES2, bool B_MN, int NB>
__device__ __forceinline__ void chain_layer(const ChainGroup& g, const ChainPass& P, int j, uint8_t* ringB, uint8_t* opnd,
                                            float* row, int stages, int stage_b, uint64_t* full, uint64_t* empty, int m0,
                                            int& stage, uint32_t& phase) {
  constexpr int planes = PLANES2 ? 2 : 1;
  const ChainLayer& Lj = P.L[j];
  const int lane = threadIdx.x & 31, r_lo = (threadIdx.x >> 5) * 16 + (lane >> 2);   // this thread's rows r_lo, r_lo + 8
  const int nkb = Lj.kblocks[0] + Lj.kblocks[1];
  float acc[128];
#pragma unroll
  for (int i = 0; i < 32 * NB; ++i) acc[i] = 0.f;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full[stage], phase);
    if (j == 0 && kb == 0 && threadIdx.x == 0) TC_STAMP(2);
    const uint32_t sB = smem_u32(ringB + (size_t)stage * planes * stage_b);
    // layer 0: the ring slot of this stage; later layers: k-block kb of the operand buffer
    const uint32_t sA = smem_u32(opnd) + (uint32_t)(j == 0 ? stage * planes * TC_STAGE_A : kb * TC_STAGE_A);
    const uint32_t a_plane = j == 0 ? TC_STAGE_A : CH_OPND_PLANE;
    wg_fence();
    // All four k16 steps, also in a partial last k-block: past K the operand buffer holds the zeros the previous
    // epilogue wrote and TMA zero-fills B, so the extra products add exact zeros.
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) {
      const uint32_t b_off = B_MN ? k * 2048 : k * 32;
      const uint64_t b_hi = make_desc(sB + b_off, B_MN ? 8192 : 16, 1024);
      const uint64_t b_lo = make_desc(sB + stage_b + b_off, B_MN ? 8192 : 16, 1024);
      const uint64_t a_hi = make_desc(sA + k * 32, 16, 1024);
      const uint64_t a_lo = make_desc(sA + a_plane + k * 32, 16, 1024);
      wgmma_step<NB, 0, B_MN, PLANES2>(acc, a_hi, b_hi, a_lo, b_lo);
    }
    wg_commit();
    wg_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);   // this warp's share of k-block kb - 1 retired
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
  if (threadIdx.x == 0) TC_STAMP(8 + 3 * j);   // MMAs of layer j retired
  EpiArgs E;
  E.epi = Lj.epi; E.act = Lj.act; E.M = P.M; E.N = Lj.N; E.ldc = Lj.N; E.ldz = Lj.N;
  E.bias = Lj.bias; E.Zout = Lj.Zout; E.Zin = Lj.Zin; E.colsum = Lj.colsum; E.C = Lj.C;
  E.img = Lj.img; E.img_pitch = Lj.img_pitch; E.img_plane = Lj.img_plane;
  epi_frag<PLANES2, NB>(acc, E, m0, 0, row);
  if (threadIdx.x == 0) TC_STAMP(9 + 3 * j);
  if (j + 1 < P.n_layers) {
    // next layer's A operand: bf16 hi/lo pairs at (row, column) of the swizzled K-major k-block tiles
    // (16-byte chunk index ^= row & 7).  Every warp's MMAs of this layer have retired before anyone overwrites.
    wg_bar();
#pragma unroll
    for (int i = 0; i < 8 * NB; ++i) {
      const int c = 8 * i + 2 * (lane & 3), cc = c & 63;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h;
        uint32_t whi, wlo;
        split_pack2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], whi, wlo);
        const uint32_t off = (uint32_t)((c >> 6) * TC_STAGE_A + r * 128 + ((((cc >> 3) ^ (r & 7)) << 4) | ((cc & 7) * 2)));
        *reinterpret_cast<uint32_t*>(opnd + off) = whi;
        if (PLANES2) *reinterpret_cast<uint32_t*>(opnd + CH_OPND_PLANE + off) = wlo;
      }
    }
    fence_async_smem();   // generic-proxy stores -> visible to wgmma's operand reads
    wg_bar();
  }
  if (threadIdx.x == 0) TC_STAMP(10 + 3 * j);
}

// B_MN: the weight tiles are MN-major (dgrad chains); forward chains read them K-major.
template <bool PLANES2, bool B_MN>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_chain_kernel(const __grid_constant__ ChainGroup g, int stages, int stage_b) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // keeps the shared address space (LDS/STS)
  constexpr int planes = PLANES2 ? 2 : 1;
  uint8_t* ringB = smem;
  uint8_t* opnd = smem + (size_t)stages * planes * stage_b;   // stages * planes <= 4 * planes: layer 0's A ring fits
  float* scratch = reinterpret_cast<float*>(opnd + planes * CH_OPND_PLANE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scratch) + TC_SCRATCH);
  uint64_t* full = bars;               // [stages] TMA -> MMA
  uint64_t* empty = bars + stages;     // [stages] MMA -> TMA (one arrival per MMA warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) TC_STAMP(0);

  int pi = 0;
#pragma unroll
  for (int i = 1; i < CH_MAX_PASSES; ++i)
    if (i < g.n && (int)blockIdx.x >= g.p[i].tile_start) pi = i;
  const ChainPass& P = g.p[pi];
  const int m0 = (blockIdx.x - P.tile_start) * TC_BM;
  const int nl = P.n_layers;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_MMA_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 4) {   // descriptor prefetch: every tensor map this CTA will use (kernel parameters: no dependency on the
                     // preceding kernel)
    for (int i = lane; i < 2 + nl; i += 32) {
      const CUtensorMap* m = nullptr;
      if (i == 0) m = &P.mapA[0];
      else if (i == 1) { if (P.L[0].kblocks[1] > 0) m = &P.mapA[1]; }
      else m = &P.L[i - 2].mapB;
      if (m) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
    }
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");            // programmatic dependent launch, see gemm_tc.cuh
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) TC_STAMP(1);

  if (warp == 4) {
    // ===== TMA producer: runs ahead of the epilogues, bounded only by free ring slots =====
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nl; ++j) {
        const ChainLayer& Lj = P.L[j];
        const int nkb = Lj.kblocks[0] + Lj.kblocks[1];
        const int b_boxes = B_MN ? (Lj.bn + 63) / 64 : 1;
        const uint32_t b_bytes = B_MN ? (uint32_t)b_boxes * 8192 : (uint32_t)Lj.bn * 128;
        const uint32_t tx = planes * (b_bytes + (j == 0 ? (uint32_t)TC_STAGE_A : 0u));
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], tx);
          const int seg = kb >= Lj.kblocks[0] ? 1 : 0;
          const int kloc = (seg ? kb - Lj.kblocks[0] : kb) * TC_BK;
          const int kB = Lj.kB0[seg] + kloc;
          uint8_t* sB = ringB + (size_t)stage * planes * stage_b;
          for (int pl = 0; pl < planes; ++pl) {
            if (j == 0)  // A ring slot = B ring slot: reuse is ordered by the same empty barrier
              tma_load_3d(opnd + (size_t)(stage * planes + pl) * TC_STAGE_A, &P.mapA[seg], &full[stage], kloc, m0, pl);
            if (B_MN) {
              for (int i = 0; i < b_boxes; ++i) tma_load_3d(sB + pl * stage_b + i * 8192, &Lj.mapB, &full[stage], 64 * i, kB, pl);
            } else {
              tma_load_3d(sB + pl * stage_b, &Lj.mapB, &full[stage], kB, 0, pl);
            }
          }
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===== MMA warpgroup: per layer the MMAs, then the epilogue on the accumulator registers, which also writes the
    // next layer's operand; the tile width is dispatched once per layer =====
    float* row = scratch + threadIdx.x * 16;
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < nl; ++j) {
      switch ((P.L[j].bn + 63) / 64) {
        case 1: chain_layer<PLANES2, B_MN, 1>(g, P, j, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
        case 2: chain_layer<PLANES2, B_MN, 2>(g, P, j, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
        case 3: chain_layer<PLANES2, B_MN, 3>(g, P, j, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
        default: chain_layer<PLANES2, B_MN, 4>(g, P, j, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
      }
    }
  }

  if (lane == 0 && warp < 4) { if (g.dbg) atomicMax(&g.dbg[(size_t)blockIdx.x * TC_DBG_SLOTS + 5], gtime()); }
  __syncthreads();
  if (threadIdx.x == 0) TC_STAMP(6);
}

}  // namespace dsact
