// Weight-gradient GEMM dW = dy^T x of a group of problems on wgmma (DSACT_GEMM_BF16X3 / DSACT_GEMM_BF16), sm_90a:
// a persistent grid of two-MMA-warpgroup CTAs that walk a static list of 128-row tiles.
//
// A tile is 128 output rows x bn columns (bn = 64 NB <= 128) of one problem over one batch split ("slab"), stored with
// plain stores into that slab (no atomics; reduced later).  Both operands are MN-major bf16 hi/lo images (dy image, x
// image), read with the tensor maps of tc_gemm_kernel.  Warpgroup w computes rows [64 w, 64 w + 64) of the tile; both read
// their own 64-row A box and the same B stage, so one B load feeds 128 rows.  The k-blocks of a slab, the k16 steps of a
// k-block and the planes of a k16 step are issued in tc_gemm_kernel's order: every partial tile is the same float sum.
//
// Roles (384 threads): warps 0..7 two MMA warpgroups, warp 8 the TMA producer (warps 9..11 only complete its warpgroup,
// see WG_MMA_REGS).  CTA b takes tiles b, 2G - 1 - b, 2G + b, ... of the list (G = grid): the host orders the problems by
// the cost of their tiles, largest first, so that the serpentine pairs the heaviest tiles with the lightest.  The ring of
// stages runs across tile boundaries: each k-block's slot is released once the next one has been issued and it has
// retired, the last one as soon as the tile's MMAs have retired, so the producer loads the next tile's first k-blocks
// while the MMA warpgroups store the finished tile.
#pragma once
#include "gemm_tc.cuh"

namespace dsact {

constexpr int WG_BM = 2 * TC_BM;                         // rows of a CTA tile
constexpr int WG_MMA_THREADS = 2 * TC_MMA_THREADS;
constexpr int WG_THREADS = WG_MMA_THREADS + TC_MMA_THREADS;
// Registers per thread after the role split, as in the layer-chain kernel: 168 each at launch (384 threads), the producer
// warpgroup gives its share to the MMA warpgroups, 40 + 232 + 232 = 504 per SM sub-partition.
constexpr int WG_PRODUCER_REGS = 40;
constexpr int WG_MMA_REGS = 232;

// Where tile `t` of the group lies: problem, slab, first row / column, k-block range (empty for a slab past the end of a
// short reduction: the tile then stores zeros, so the reduction over slabs always reads written values).
struct WgTile {
  int pi, ks, m0, n0, kb_begin, kb_end;
};
__device__ __forceinline__ WgTile wg_tile(const TcGroup& g, int t) {
  WgTile w;
  w.pi = 0;
#pragma unroll
  for (int i = 1; i < TC_MAXG; ++i)
    if (i < g.n && t >= g.p[i].tile_start) w.pi = i;
  const TcProb& P = g.p[w.pi];
  int local = t - P.tile_start;
  const int tiles_mn = P.tiles_m * P.tiles_n;
  w.ks = local / tiles_mn;
  local -= w.ks * tiles_mn;
  w.m0 = (local / P.tiles_n) * WG_BM;
  w.n0 = (local % P.tiles_n) * P.bn;
  const int nkb = P.kblocks[0];
  const int per = (nkb + P.ksplit - 1) / P.ksplit;
  w.kb_begin = w.ks * per;
  w.kb_end = min(nkb, w.kb_begin + per);
  return w;
}
// the list of CTA b: round r takes tile r G + b (r even) or r G + G - 1 - b (r odd)
__device__ __forceinline__ int wg_tile_id(int r) {
  return r * (int)gridDim.x + ((r & 1) ? (int)gridDim.x - 1 - (int)blockIdx.x : (int)blockIdx.x);
}

// A warpgroup whose rows of the tile all lie past M: the ring protocol alone (it waits on each slot and arrives on its
// release), no MMAs, no stores.
__device__ __forceinline__ void wg_tile_idle(const WgTile& w, uint64_t* full, uint64_t* empty, int stages, int& stage,
                                             uint32_t& phase) {
  for (int kb = w.kb_begin; kb < w.kb_end; ++kb) {
    mbar_wait(&full[stage], phase);
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage]);
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
}

// One warpgroup's 64 x (64 NB) share of a tile: the MMAs (one k-block kept in flight; each slot released once the next
// k-block has been issued and it has retired, the last one once the tile's MMAs have), then the stores into the slab.
template <bool PLANES2, int NB>
__device__ __forceinline__ void wg_tile_mma(const TcProb& P, const WgTile& w, uint8_t* smem, int stage_bytes, int stage_b,
                                            uint64_t* full, uint64_t* empty, int stages, int& stage, uint32_t& phase) {
  constexpr int planes = PLANES2 ? 2 : 1;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x / TC_MMA_THREADS;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 32 * NB; ++i) acc[i] = 0.f;
  int prev = -1;
  for (int kb = w.kb_begin; kb < w.kb_end; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint32_t sA = smem_u32(smem + (size_t)stage * stage_bytes) + wg * planes * TC_STAGE_A;
    const uint32_t sB = smem_u32(smem + (size_t)stage * stage_bytes) + 2 * planes * TC_STAGE_A;
    wg_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) {
      const uint64_t a_hi = make_desc(sA + k * 2048, 8192, 1024);
      const uint64_t b_hi = make_desc(sB + k * 2048, 8192, 1024);
      const uint64_t a_lo = make_desc(sA + TC_STAGE_A + k * 2048, 8192, 1024);
      const uint64_t b_lo = make_desc(sB + stage_b + k * 2048, 8192, 1024);
      wgmma_step<NB, true, true, PLANES2>(acc, a_hi, b_hi, a_lo, b_lo);
    }
    wg_commit();
    wg_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);   // the ring moves on to the next tile under these stores
  // acc[16 g + t]: row ra (t & 2 == 0) or ra + 8, column cq + 32 g + 8 (t >> 2) + (t & 1)
  float* C = P.C + (size_t)w.ks * P.split_stride;
  const int ra = w.m0 + 64 * wg + ((threadIdx.x & (TC_MMA_THREADS - 1)) >> 5) * 16 + (lane >> 2);
  const int cq = w.n0 + 2 * (lane & 3);
  const int N = P.N;
  const bool pair = pairs_ok(C, P.ldc);
#pragma unroll
  for (int g = 0; g < 2 * NB; ++g)
#pragma unroll
    for (int t = 0; t < 16; t += 2) {
      const int r = ra + ((t & 2) ? 8 : 0);
      if (r < P.M) st_pair(C + (size_t)r * P.ldc, cq + 32 * g + 8 * (t >> 2), N, pair, acc[16 * g + t], acc[16 * g + t + 1]);
    }
}

template <bool PLANES2>
__global__ void __launch_bounds__(WG_THREADS, 1) tc_gemm_kernel_wgrad(const __grid_constant__ TcGroup g, int total, int stages,
                                                                      int stage_b) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // keeps the shared address space (LDS/STS)
  constexpr int planes = PLANES2 ? 2 : 1;
  const int stage_bytes = planes * (2 * TC_STAGE_A + stage_b);   // [A rows 0..63: planes][A rows 64..127: planes][B: planes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)stages * stage_bytes);
  uint64_t* full = bars;             // [stages]  TMA -> MMA
  uint64_t* empty = bars + stages;   // [stages]  MMA -> TMA (one arrival per MMA warp of both warpgroups)
  constexpr int PRODUCER = WG_MMA_THREADS / 32;   // warp 8
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], WG_MMA_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == PRODUCER) {   // descriptor prefetch (kernel parameters: independent of the preceding kernel)
    for (int i = lane; i < 2 * g.n; i += 32) {
      const CUtensorMap* m = (i & 1) ? &g.p[i >> 1].mapB : &g.p[i >> 1].mapA[0];
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
    }
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");   // programmatic dependent launch, see gemm_tc.cuh
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  int stage = 0;
  uint32_t phase = 0;
  if (threadIdx.x >= WG_MMA_THREADS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(WG_PRODUCER_REGS));
    // ===== TMA producer: runs ahead across tiles, bounded only by free ring slots =====
    if (warp == PRODUCER && lane == 0) {
      for (int r = 0;; ++r) {
        const int t = wg_tile_id(r);
        if (t >= total) break;
        const WgTile w = wg_tile(g, t);
        const TcProb& P = g.p[w.pi];
        const int a_boxes = w.m0 + TC_BM < P.M ? 2 : 1;   // no load for a warpgroup whose rows all lie past M
        const int b_boxes = (P.bn + 63) / 64;
        const uint32_t tx = planes * (uint32_t)(a_boxes + b_boxes) * 8192u;
        for (int kb = w.kb_begin; kb < w.kb_end; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], tx);
          const int k0 = kb * TC_BK;
          uint8_t* s = smem + (size_t)stage * stage_bytes;
          for (int pl = 0; pl < planes; ++pl) {
            for (int i = 0; i < a_boxes; ++i)
              tma_load_3d(s + (i * planes + pl) * TC_STAGE_A, &P.mapA[0], &full[stage], w.m0 + TC_BM * i, k0, pl);
            for (int i = 0; i < b_boxes; ++i)
              tma_load_3d(s + 2 * planes * TC_STAGE_A + pl * stage_b + i * 8192, &P.mapB, &full[stage], w.n0 + 64 * i, P.kB0[0] + k0, pl);
          }
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WG_MMA_REGS));
    // ===== MMA warpgroups: the tile width is dispatched once per tile =====
    const int wg = threadIdx.x / TC_MMA_THREADS;
    for (int r = 0;; ++r) {
      const int t = wg_tile_id(r);
      if (t >= total) break;
      const WgTile w = wg_tile(g, t);
      const TcProb& P = g.p[w.pi];
      if (w.m0 + TC_BM * wg >= P.M) wg_tile_idle(w, full, empty, stages, stage, phase);
      else if (P.bn > 64) wg_tile_mma<PLANES2, 2>(P, w, smem, stage_bytes, stage_b, full, empty, stages, stage, phase);
      else wg_tile_mma<PLANES2, 1>(P, w, smem, stage_bytes, stage_b, full, empty, stages, stage, phase);
    }
  }
  __syncthreads();
}

}  // namespace dsact
