// Fused MLP layer-chain kernel on wgmma (DSACT_GEMM_BF16X3 / DSACT_GEMM_BF16), sm_90a.
//
// One CTA carries one 64-row block of one "pass" (an MLP applied to one input) through ALL of its layers:
//   forward chain : x -> [Linear + act] x L -> Linear            (reference networks/mlp.py:15-20)
//   dgrad chain   : dOut -> [dY W_j (.) act'(z_{j-1})] x L (-> dY W_0[:, act columns] for the actor path)
// Layer 0 takes its A operand from global memory by TMA (the bf16 hi/lo images of obs / act / dOut); every later
// layer takes A from SHARED MEMORY: the epilogue of layer j writes act(z_j) (or dz_j) as bf16 hi/lo pairs, in the
// 128-byte-swizzled K-major layout wgmma reads, into the operand buffer (stmatrix), so hidden activations never leave the SM
// unless the backward pass needs them (act' for the dgrad chain, images for wgrad).  The bf16 image a weight gradient
// needs is that same tile: it leaves as a TMA store of the operand buffer's k-blocks (a layer with an image and no next
// layer stages it there all the same).
// The weight tiles of layer j+1 are prefetched by the TMA warp while the epilogue of layer j runs.  The MMAs of a k-block
// issue back to back and one k-block stays in flight while the next is issued; each warpgroup's share of the layer width
// (64 or 128 columns) is a compile-time parameter of its layer body, dispatched once per layer.
//
// Shared memory: [ B ring: stages x planes x stage_b ][ operand buffer: planes x 4 k-blocks x 8 KiB (layer 0: its A
// ring) ][ 16-float scratch row per MMA thread ][ barriers ].
// Roles: warps 0..7 two MMA warpgroups (wgmma, accumulator in registers, epilogue), warp 8 TMA producer (warps 9..11
// only complete its warpgroup, see CH_MMA_REGS).  Of a layer's nb = ceil(bn / 64) column blocks, warpgroup 0 takes the
// first ceil(nb / 2) and warpgroup 1 the rest (256 = 128 + 128, 192 = 128 + 64, 64 = 64 + 0): both read the same A
// operand and their own columns of the same B stage.  The epilogue is bound by instruction issue and latency, so two
// warps per scheduler with half the values each finish it sooner than one warp with all of them.
#pragma once
#include "gemm_tc.cuh"

namespace dsact {

constexpr int CH_MAX_LAYERS = DSACT_MAX_HIDDEN + 1;
constexpr int CH_MAX_PASSES = 4;
constexpr int CH_KB_MAX = 4;                              // 256 columns of operand = 4 k-blocks of 64
constexpr int CH_OPND_PLANE = CH_KB_MAX * TC_STAGE_A;     // 32 KiB
constexpr int CH_MMA_THREADS = 2 * TC_MMA_THREADS;        // two MMA / epilogue warpgroups
constexpr int CH_THREADS = CH_MMA_THREADS + TC_MMA_THREADS;   // + the producer warpgroup (warp 8 issues the TMA)
constexpr int CH_SCRATCH = CH_MMA_THREADS * 16 * 4;       // per-thread 16-float rows for the generic activations
// Registers per thread after the role split (setmaxnreg works on whole warpgroups, hence a whole producer warpgroup).
// At launch 384 threads get 168 each (each SM sub-partition holds one warp of each warpgroup: 3 x 168 <= 512); the
// epilogue of a 128-column accumulator spills at 168, so the producer gives its registers to the MMA warpgroups:
// 40 + 232 + 232 = 504.
constexpr int CH_PRODUCER_REGS = 40;
constexpr int CH_MMA_REGS = 232;

struct ChainLayer {
  CUtensorMap mapB;          // weight image; forward: K-major (box = bn rows), dgrad: MN-major (box = 64 x 64)
  CUtensorMap mapImg;        // bf16 hi/lo image of the result for the weight-gradient GEMM, [M, (N + 7) / 8 * 8] (box =
                             // 64 x 64): stored by TMA from the operand buffer (valid when `img`)
  int kblocks[2];            // k-blocks of 64; layer 0 may have two A segments, later layers use [0] only
  int kB0[2];                // offset of each segment along B's reduction dimension
  int N, bn;                 // outputs; tile width (multiple of 16, <= 256)
  int epi, act;             // EPI_BIAS_ACT | EPI_DACT | EPI_STORE
  const float* bias;
  float* Zout;               // forward: act'(pre-activation) store, ld = N (null: not needed by a backward pass)
  const float* Zin;          // dgrad: act'(pre-activation) of the layer below, ld = N
  float* colsum;             // dgrad: bias gradient (+=)
  float* C;                  // fp32 result, ld = ldc (head layers)
  int ldc;                   // >= N: a head may write its columns of a wider row (the policy's mean | log_std logits)
  int img;                   // nonzero: the image is needed (mapImg)
  int kind;                  // epilogue kind of the ping-pong kernel's full tiles (EK_*, gemm_tc.cuh), set by the host
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
// the kernel's parameters (the group, stages, stage_b) within the 32764 bytes a launch may pass (CUDA 12.1+, sm_70+)
static_assert(sizeof(ChainGroup) + 2 * sizeof(int) <= 32764, "ChainGroup exceeds the kernel-parameter limit");

inline int chain_smem_bytes(int stages, int planes, int stage_b) {
  return stages * planes * stage_b + planes * CH_OPND_PLANE + CH_SCRATCH + 2 * stages * 8 + 1024;
}

// Both MMA warpgroups: the operand buffer is read by all of them and rewritten between layers.
__device__ __forceinline__ void ch_bar() { asm volatile("bar.sync 1, %0;" ::"n"(CH_MMA_THREADS) : "memory"); }

// One layer on one MMA warpgroup, 64 x (64 NB) outputs from column n0: the loads of the epilogue's global inputs, the MMAs
// with one k-block in flight (the ring slot of k-block kb is released once kb + 1 has been issued and kb has retired), the
// epilogue on the accumulator registers, and this warpgroup's columns of the next layer's A operand.  (stage, phase) is
// the consumer's position in the B ring, carried from layer to layer.
template <bool PLANES2, bool B_MN, int NB>
__device__ __forceinline__ void chain_layer(const ChainGroup& g, const ChainPass& P, int j, int n0, uint8_t* ringB,
                                            uint8_t* opnd, float* row, int stages, int stage_b, uint64_t* full,
                                            uint64_t* empty, int m0, int& stage, uint32_t& phase) {
  constexpr int planes = PLANES2 ? 2 : 1;
  const ChainLayer& Lj = P.L[j];
  const int lane = threadIdx.x & 31;
  const int nkb = Lj.kblocks[0] + Lj.kblocks[1];
  EpiArgs E;
  E.epi = Lj.epi; E.act = Lj.act; E.M = P.M; E.N = Lj.N; E.ldc = Lj.ldc; E.ldz = Lj.N;
  E.bias = Lj.bias; E.Zout = Lj.Zout; E.Zin = Lj.Zin; E.colsum = Lj.colsum; E.C = Lj.C;
  E.img = nullptr;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 32 * NB; ++i) acc[i] = 0.f;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    // When k-block kb has not landed yet, the MMAs of kb - 1 retire before it does: drain them and release kb - 1's slot
    // now, so that the producer loads kb + 1 while kb is still in flight.  With two stages, releasing only after kb is
    // issued leaves one load in flight, and the layer's MMA phase is set by the load latency.  The four-stage ring of
    // one plane already has three loads in flight; draining there only loses the MMA overlap.
    if (stages == 2 && prev >= 0 && !__all_sync(0xffffffffu, mbar_test(&full[stage], phase))) {
      wg_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev]);
      prev = -1;
    }
    mbar_wait(&full[stage], phase);
    if (j == 0 && kb == 0 && threadIdx.x == 0) TC_STAMP(2);
    // this warpgroup's columns of the stage: K-major rows of 128 B, MN-major 64-column boxes of 8 KiB (1024-byte aligned)
    const uint32_t sB = smem_u32(ringB + (size_t)stage * planes * stage_b) + (uint32_t)(B_MN ? n0 / 64 * 8192 : n0 * 128);
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
  // The epilogue is a rolled loop over the 16-value groups, each group's global inputs loaded two groups ahead (the first
  // two under the last k-block's MMAs).  Unrolled, every layer body carried its own copy of the whole epilogue (all
  // activation variants and stores per group), and each layer ran its epilogue from a cold instruction cache.
  float nx0[16], nx1[16];
  epi_in(nx0, E, m0, n0, 0);
  epi_in(nx1, E, m0, n0, 1);   // 2 NB >= 2 groups
  wg_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
  if (threadIdx.x == 0) TC_STAMP(8 + 3 * j);   // MMAs of layer j retired
  // The result is written group by group into the operand buffer as the epilogue computes it, as the next layer's A
  // operand and as the source of the image's TMA store: both warpgroups' MMAs of this layer must have retired first
  // (each reads all of A), and so must the previous layer's image store (thread 0 issued it).
  const bool opw = j + 1 < P.n_layers || Lj.img;
  if (opw) {
    if (threadIdx.x == 0) bulk_wait_read();
    ch_bar();
  }
  // Lane l addresses row l & 7 of 8 x 8 matrix l >> 3 of a stmatrix: matrix m of stmatrix s holds rows 8 (m & 1) .. + 7
  // of the warp's 16 and the 8 columns ii = 2 s + (m >> 1) of the group (fragment words v[4 ii + 2 h], + 1, h = m & 1).
  // In the 128-byte-swizzled K-major k-block tiles, the 16-byte chunk of that row and column block is chunk ^ (row & 7).
  const int m_row = ((threadIdx.x & (TC_MMA_THREADS - 1)) >> 5) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  const uint32_t s_row = smem_u32(opnd) + (uint32_t)((n0 >> 6) * TC_STAGE_A + m_row * 128);
#pragma unroll 1
  for (int q = 0; q < 2 * NB; ++q) {
    float x[16], v[16];
#pragma unroll
    for (int t = 0; t < 16; ++t) { x[t] = nx0[t]; nx0[t] = nx1[t]; }
    if (q + 2 < 2 * NB) epi_in(nx1, E, m0, n0, q + 2);
#pragma unroll
    for (int c = 0; c < 2 * NB; ++c)   // group q of the accumulator (registers: compile-time indices)
      if (q == c) {
#pragma unroll
        for (int t = 0; t < 16; ++t) v[t] = acc[16 * c + t];
      }
    epi_group<PLANES2>(v, x, E, m0, n0, q, row);
    if (opw) {
      // bf16 hi/lo pairs, split once: word i = matrix (ii, h) = (i >> 1, i & 1)
      uint32_t whi[8], wlo[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (PLANES2) split_pack2(v[2 * i], v[2 * i + 1], whi[i], wlo[i]);
        else whi[i] = cvt_bf16x2(v[2 * i], v[2 * i + 1]);
      }
      const uint32_t s_q = s_row + (uint32_t)((q >> 1) * TC_STAGE_A);
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const uint32_t a = s_q + (uint32_t)((((4 * (q & 1) + 2 * s + (lane >> 4)) ^ (lane & 7))) << 4);
        stsm_x4(a, whi[4 * s], whi[4 * s + 1], whi[4 * s + 2], whi[4 * s + 3]);
        if (PLANES2) stsm_x4(a + CH_OPND_PLANE, wlo[4 * s], wlo[4 * s + 1], wlo[4 * s + 2], wlo[4 * s + 3]);
      }
    }
  }
  if (threadIdx.x == 0) TC_STAMP(9 + 3 * j);
  if (opw) {
    fence_async_smem();   // generic-proxy stores -> visible to wgmma's operand reads and the TMA store
    ch_bar();
    // The image: k-block tiles of the layer's columns, clipped by the tensor map to rows < M and columns < (N + 7) / 8 * 8
    if (Lj.img && threadIdx.x == 0) {
      for (int kb = 0; kb < (Lj.N + 63) / 64; ++kb)
        for (int pl = 0; pl < planes; ++pl) tma_store_3d(&Lj.mapImg, opnd + pl * CH_OPND_PLANE + kb * TC_STAGE_A, kb * TC_BK, m0, pl);
      bulk_commit();
    }
  }
  if (threadIdx.x == 0) TC_STAMP(10 + 3 * j);
}

// A warpgroup with no columns in layer j (a layer of 64 columns) still consumes the layer's ring slots, so that the ring
// protocol does not depend on the layer width, and meets the other warpgroup at the operand barriers.
__device__ __forceinline__ void chain_idle(const ChainPass& P, int j, int stages, uint64_t* full, uint64_t* empty, int& stage,
                                           uint32_t& phase) {
  const int nkb = P.L[j].kblocks[0] + P.L[j].kblocks[1];
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full[stage], phase);
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage]);
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  if (j + 1 < P.n_layers || P.L[j].img) { ch_bar(); ch_bar(); }
}

// B_MN: the weight tiles are MN-major (dgrad chains); forward chains read them K-major.
template <bool PLANES2, bool B_MN>
__global__ void __launch_bounds__(CH_THREADS, 1) tc_chain_kernel(const __grid_constant__ ChainGroup g, int stages, int stage_b) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // keeps the shared address space (LDS/STS)
  constexpr int planes = PLANES2 ? 2 : 1;
  uint8_t* ringB = smem;
  uint8_t* opnd = smem + (size_t)stages * planes * stage_b;   // stages * planes <= 4 * planes: layer 0's A ring fits
  float* scratch = reinterpret_cast<float*>(opnd + planes * CH_OPND_PLANE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scratch) + CH_SCRATCH);
  uint64_t* full = bars;               // [stages] TMA -> MMA
  uint64_t* empty = bars + stages;     // [stages] MMA -> TMA (one arrival per MMA warp of both warpgroups)

  constexpr int PRODUCER = CH_MMA_THREADS / 32;   // warp 8
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
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CH_MMA_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == PRODUCER) {   // descriptor prefetch: every tensor map this CTA will use (kernel parameters: no dependency on the
                     // preceding kernel)
    for (int i = lane; i < 2 + 2 * nl; i += 32) {
      const CUtensorMap* m = nullptr;
      if (i == 0) m = &P.mapA[0];
      else if (i == 1) { if (P.L[0].kblocks[1] > 0) m = &P.mapA[1]; }
      else if (i < 2 + nl) m = &P.L[i - 2].mapB;
      else if (P.L[i - 2 - nl].img) m = &P.L[i - 2 - nl].mapImg;
      if (m) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
    }
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");            // programmatic dependent launch, see gemm_tc.cuh
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) TC_STAMP(1);

  if (threadIdx.x >= CH_MMA_THREADS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(CH_PRODUCER_REGS));
    // ===== TMA producer: runs ahead of the epilogues, bounded only by free ring slots =====
    if (warp == PRODUCER && lane == 0) {
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
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CH_MMA_REGS));
    // ===== MMA warpgroups: per layer the MMAs, then the epilogue on the accumulator registers, which also writes the
    // next layer's operand; each warpgroup's share of the columns is dispatched once per layer =====
    float* row = scratch + threadIdx.x * 16;
    const int wg = threadIdx.x / TC_MMA_THREADS;
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < nl; ++j) {
      const int nb = (P.L[j].bn + 63) / 64, nb0 = (nb + 1) / 2;
      const int n0 = wg == 0 ? 0 : 64 * nb0;
      switch (wg == 0 ? nb0 : nb - nb0) {
        case 0: chain_idle(P, j, stages, full, empty, stage, phase); break;
        case 1: chain_layer<PLANES2, B_MN, 1>(g, P, j, n0, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
        default: chain_layer<PLANES2, B_MN, 2>(g, P, j, n0, ringB, opnd, row, stages, stage_b, full, empty, m0, stage, phase); break;
      }
    }
    if (threadIdx.x == 0) bulk_wait();   // the image stores this thread issued have completed
  }

  if (lane == 0 && warp < PRODUCER) { if (g.dbg) atomicMax(&g.dbg[(size_t)blockIdx.x * TC_DBG_SLOTS + 5], gtime()); }
  __syncthreads();
  if (threadIdx.x == 0) TC_STAMP(6);
}

}  // namespace dsact
