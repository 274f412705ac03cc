// Ping-pong layer-chain kernel (DSACT_GEMM_BF16X3 / DSACT_GEMM_BF16), sm_90a: two 64-row tiles of one pass per CTA, for
// launches whose column-split grid (tc_chain_kernel, one 64-row tile per CTA) needs more than one wave.
//
// MMA warpgroup w owns tile w (rows m0 + 64 w ... + 63) and ALL columns of a layer: its accumulator is 64 x (64 NB), NB <=
// 4, and its layer-to-layer dependency stays inside its own tile (its own operand buffer, its own named barrier).  Warp 8
// is the TMA producer as in the column split.  The producer streams the weight tiles in consumption order: warpgroup 0's
// k-blocks of layer j, then warpgroup 1's of layer j, then layer j + 1, so each weight tile is loaded once per 64 rows (the
// L2 bytes per row of the column split).  The ring's order is the schedule: warpgroup 1 runs layer j's MMAs once
// warpgroup 0 has released its ring slots of layer j, that is while warpgroup 0 runs layer j's epilogue, and warpgroup 0's
// MMAs of layer j + 1 run under warpgroup 1's epilogue of layer j.  A ring stage holds one k-block of one column half
// (128 columns; K-major: 128 weight rows, MN-major: two 64 x 64 boxes), so a layer wider than 128 columns takes two ring
// items per k-block, and two 32 KiB bf16x3 stages fit beside the two operand buffers.
//
// Shared memory: [ B ring: stages x planes x 16 KiB ][ operand buffer of tile 0 | of tile 1: planes x 4 k-blocks x 8 KiB
// each (layer 0: the tile's A ring, k-block kb in slot kb & 3) ][ 16-float scratch row per MMA thread ][ barriers ].
//
// Every output element accumulates over the same k16 steps, in the same order and with the same planes, as in the column
// split, so the outputs, act', images and column sums are the same bits (the column sums' float atomics aside).
//
// Epilogue bodies: a full tile (64 rows < M) of a layer whose kind the host set (ChainLayer::kind: forward hidden GELU /
// ReLU with or without act', dgrad hidden with or without column sums) runs a straight-line body templated on (NB, kind):
// one activation, no row or column checks, unconditional 8-byte loads and stores.  Every other tile and layer runs the
// runtime body.  The per-value arithmetic is the same in both.
#pragma once
#include "chain_tc.cuh"

namespace dsact {

constexpr int PP_HALF = 128;                   // columns of one ring stage
constexpr int PP_STAGE_B = PP_HALF * 128;      // bytes of one plane of a stage
constexpr int PP_THREADS = CH_THREADS;         // two MMA warpgroups + the producer warpgroup

inline int pp_smem_bytes(int stages, int planes) {
  return stages * planes * PP_STAGE_B + 2 * planes * CH_OPND_PLANE + CH_SCRATCH + 2 * stages * 8 + 1024;
}

// The thread index read afresh (volatile: not kept in a register across the layer bodies, where a 256-column accumulator
// leaves none to spare), its warpgroup, and whether it leads the warpgroup (stamps, TMA stores).
__device__ __forceinline__ uint32_t pp_tid() {
  uint32_t t;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
  return t;
}
__device__ __forceinline__ int pp_wg() { return (int)(pp_tid() / TC_MMA_THREADS); }
__device__ __forceinline__ bool pp_lead() { return (pp_tid() & (TC_MMA_THREADS - 1)) == 0; }
// The 128 threads of the calling MMA warpgroup (named barriers 2 and 3; ch_bar is 1).
__device__ __forceinline__ void pp_bar() { asm volatile("bar.sync %0, %1;" ::"r"(2 + pp_wg()), "n"(TC_MMA_THREADS) : "memory"); }
// The turn of the calling warpgroup on the ring (named barriers 4 and 5, 256 threads): it waits for it before its first
// ring wait of a layer, and the other warpgroup gives it once it has waited for its last item of its own layer.  An
// mbarrier wait tells phases apart by parity only, so a warpgroup must not wait for an item while the ring is still two
// or more phases behind it: with its turn given, every item before its first one has landed.
__device__ __forceinline__ void pp_wait_turn() {
  asm volatile("bar.sync %0, %1;" ::"r"(4 + pp_wg()), "n"(2 * TC_MMA_THREADS) : "memory");
}
__device__ __forceinline__ void pp_give_turn() {
  asm volatile("bar.arrive %0, %1;" ::"r"(5 - pp_wg()), "n"(2 * TC_MMA_THREADS) : "memory");
}

// wgmma into the upper half of the accumulator (columns 128 ... of the warpgroup: d[64 ...]); A is K-major.
template <int TB>
__device__ __forceinline__ void wgmma_n64_hi(float (&d)[128], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %34;\n\t}"
      : "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(a), "l"(b), "n"(TB));
}

template <int TB>
__device__ __forceinline__ void wgmma_n128_hi(float (&d)[128], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %66;\n\t}"
      : "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "n"(TB));
}

// One k16 step of column half 1 (64 NBH columns from column 128) into d[64 ...], planes as wgmma_step.
template <int NBH, int TB, bool PLANES2>
__device__ __forceinline__ void pp_step_hi(float (&d)[128], uint64_t a_hi, uint64_t b_hi, uint64_t a_lo, uint64_t b_lo) {
  if constexpr (NBH == 1) {
    wgmma_n64_hi<TB>(d, a_hi, b_hi);
    if constexpr (PLANES2) { wgmma_n64_hi<TB>(d, a_hi, b_lo); wgmma_n64_hi<TB>(d, a_lo, b_hi); }
  } else {
    wgmma_n128_hi<TB>(d, a_hi, b_hi);
    if constexpr (PLANES2) { wgmma_n128_hi<TB>(d, a_hi, b_lo); wgmma_n128_hi<TB>(d, a_lo, b_hi); }
  }
}

// Debug stamps per 64-row tile, at the tile's index in the column split's grid (its row of slots there): kept in shared
// memory, not in a register of the MMA warpgroups.
__shared__ int pp_dbg_tile[2];
#define PP_STAMP(slot) do { if (g.dbg) g.dbg[(size_t)pp_dbg_tile[pp_wg()] * TC_DBG_SLOTS + (slot)] = gtime(); } while (0)

// The epilogue of one layer of one tile: the rolled loop of the column split over all 2 NB groups, each group's global
// inputs loaded one group ahead (the first under the last item's MMAs).  A group's inputs (bias or act') are applied
// (epi_apply) before the next group's loads go into the same registers: a 256-column accumulator leaves no room for a
// second 16-value input buffer.  `prev`: the ring slot of the layer's last item, released once its MMAs retire.
template <bool PLANES2, int NB, int KIND>
__device__ __forceinline__ void pp_epilogue(const ChainGroup& g, const ChainPass& P, int j, const EpiArgs& E,
                                            float (&acc)[128], uint8_t* opnd, float* row, uint64_t* empty, int prev, int m0) {
  constexpr int planes = PLANES2 ? 2 : 1;
  const ChainLayer& Lj = P.L[j];
  const int lane = threadIdx.x & 31;
  float nx[16];
  epi_in<KIND>(nx, E, m0, 0, 0);
  wg_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
  if (pp_lead()) PP_STAMP(8 + 3 * j);   // MMAs of layer j retired
  // The operand buffer is this tile's alone: its warpgroup's MMAs of this layer must have retired (each warp reads all of
  // A), and so must the previous layer's image store (the lead thread issued it).
  const bool opw = j + 1 < P.n_layers || Lj.img;
  if (opw) {
    if (pp_lead()) bulk_wait_read();
    pp_bar();
  }
  const int m_row = ((threadIdx.x & (TC_MMA_THREADS - 1)) >> 5) * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
  const uint32_t s_row = smem_u32(opnd) + (uint32_t)(m_row * 128);
#pragma unroll 1
  for (int q = 0; q < 2 * NB; ++q) {
    float v[16];
#pragma unroll
    for (int c = 0; c < 2 * NB; ++c)
      if (q == c) {
#pragma unroll
        for (int t = 0; t < 16; ++t) v[t] = acc[16 * c + t];
      }
    epi_apply<KIND>(v, nx, E);
    if (q + 1 < 2 * NB) epi_in<KIND>(nx, E, m0, 0, q + 1);
    epi_group<PLANES2, KIND, true>(v, nx, E, m0, 0, q, row);
    if (opw) {   // as chain_layer: bf16 hi/lo pairs split once, two stmatrix per plane
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
  if (pp_lead()) PP_STAMP(9 + 3 * j);
  if (opw) {
    fence_async_smem();   // generic-proxy stores -> visible to wgmma's operand reads and the TMA store
    pp_bar();
    if (Lj.img && pp_lead()) {
      for (int kb = 0; kb < (Lj.N + 63) / 64; ++kb)
        for (int pl = 0; pl < planes; ++pl) tma_store_3d(&Lj.mapImg, opnd + pl * CH_OPND_PLANE + kb * TC_STAGE_A, kb * TC_BK, m0, pl);
      bulk_commit();
    }
  }
  if (pp_lead()) PP_STAMP(10 + 3 * j);
}

// One layer of one tile on its warpgroup: 64 x (64 NB) outputs.  The MMAs of each ring item (one k-block of one column
// half) issue back to back and one item stays in flight while the next is issued; then the epilogue on the accumulator,
// which writes the next layer's A operand into this tile's operand buffer.  `pos`: the ring position of the warpgroup's
// first item of the layer; `wait_turn` / `give_turn`: the layer starts on the turn the other warpgroup gives, and gives
// the other warpgroup its turn once its last item has landed (both false when the CTA has one tile).
template <bool PLANES2, bool B_MN, int NB>
__device__ __forceinline__ void pp_layer(const ChainGroup& g, const ChainPass& P, int j, uint8_t* ringB,
                                         uint8_t* opnd, float* row, int stages, uint64_t* full, uint64_t* empty, int m0,
                                         int pos, bool wait_turn, bool give_turn) {
  constexpr int planes = PLANES2 ? 2 : 1;
  constexpr int NH = NB > 2 ? 2 : 1;      // ring items per k-block
  constexpr int NB0 = NB > 2 ? 2 : NB;    // 64-column blocks of half 0
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
  int stage = pos % stages, prev = -1;
  uint32_t phase = (uint32_t)(pos / stages) & 1u;
  if (wait_turn) pp_wait_turn();
  for (int kb = 0; kb < nkb; ++kb) {
    // layer 0: slot kb & 3 of this tile's A ring; later layers: k-block kb of the operand buffer
    const uint32_t sA = smem_u32(opnd) + (uint32_t)(j == 0 ? (kb & 3) * planes * TC_STAGE_A : kb * TC_STAGE_A);
    const uint32_t a_plane = j == 0 ? TC_STAGE_A : CH_OPND_PLANE;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      // the early release of the column split (chain_layer): with two stages, drain and release the previous item when
      // the next one has not landed yet
      if (stages == 2 && prev >= 0 && !__all_sync(0xffffffffu, mbar_test(&full[stage], phase))) {
        wg_wait<0>();
        if (lane == 0) mbar_arrive(&empty[prev]);
        prev = -1;
      }
      mbar_wait(&full[stage], phase);
      if (j == 0 && kb == 0 && h == 0 && pp_lead()) PP_STAMP(2);
      const uint32_t sB = smem_u32(ringB + (size_t)stage * planes * PP_STAGE_B);
      wg_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) {
        const uint32_t b_off = B_MN ? k * 2048 : k * 32;
        const uint64_t b_hi = make_desc(sB + b_off, B_MN ? 8192 : 16, 1024);
        const uint64_t b_lo = make_desc(sB + PP_STAGE_B + b_off, B_MN ? 8192 : 16, 1024);
        const uint64_t a_hi = make_desc(sA + k * 32, 16, 1024);
        const uint64_t a_lo = make_desc(sA + a_plane + k * 32, 16, 1024);
        if (h == 0) wgmma_step<NB0, 0, B_MN, PLANES2>(acc, a_hi, b_hi, a_lo, b_lo);
        else pp_step_hi<NB - 2, B_MN, PLANES2>(acc, a_hi, b_hi, a_lo, b_lo);
      }
      wg_commit();
      wg_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);   // this warp's share of the previous item retired
      prev = stage;
      if (++stage == stages) { stage = 0; phase ^= 1; }
    }
  }
  if (give_turn) pp_give_turn();
  // The epilogue body, chosen once per layer: a full tile of a layer with an epilogue kind (ChainLayer::kind) runs that
  // kind's straight-line body, anything else the runtime body with its row and column checks.  Each kernel holds only the
  // kinds of its direction.
  const int kind = m0 + TC_BM <= P.M ? Lj.kind : EK_RUNTIME;
#define PP_EPI(K) pp_epilogue<PLANES2, NB, K>(g, P, j, E, acc, opnd, row, empty, prev, m0)
  if constexpr (B_MN) {
    switch (kind) {
      case EK_DACT: PP_EPI(EK_DACT); break;
      case EK_DACT_SUM: PP_EPI(EK_DACT_SUM); break;
      default: PP_EPI(EK_RUNTIME); break;
    }
  } else {
    switch (kind) {
      case EK_GELU: PP_EPI(EK_GELU); break;
      case EK_GELU_Z: PP_EPI(EK_GELU_Z); break;
      case EK_RELU: PP_EPI(EK_RELU); break;
      case EK_RELU_Z: PP_EPI(EK_RELU_Z); break;
      default: PP_EPI(EK_RUNTIME); break;
    }
  }
#undef PP_EPI
}

// Ring items of layer j for one tile: k-blocks x column halves.
__device__ __forceinline__ int pp_items(const ChainLayer& L) { return (L.kblocks[0] + L.kblocks[1]) * (L.bn > PP_HALF ? 2 : 1); }

// B_MN: the weight tiles are MN-major (dgrad chains); forward chains read them K-major, through maps whose box is
// min(bn, 128) weight rows (one column half).  Pass i covers ceil(M_i / 128) CTAs.
template <bool PLANES2, bool B_MN>
__global__ void __launch_bounds__(PP_THREADS, 1) tc_pingpong_kernel(const __grid_constant__ ChainGroup g, int stages) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // keeps the shared address space (LDS/STS)
  constexpr int planes = PLANES2 ? 2 : 1;
  uint8_t* ringB = smem;
  uint8_t* opnd0 = smem + (size_t)stages * planes * PP_STAGE_B;
  float* scratch = reinterpret_cast<float*>(opnd0 + 2 * planes * CH_OPND_PLANE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(scratch) + CH_SCRATCH);
  uint64_t* full = bars;               // [stages] TMA -> MMA
  uint64_t* empty = bars + stages;     // [stages] MMA -> TMA (one arrival per MMA warp of the item's warpgroup)

  constexpr int PRODUCER = CH_MMA_THREADS / 32;   // warp 8
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  int pi = 0, cta0 = 0;
  for (int i = 0; i + 1 < g.n; ++i) {
    const int c = (g.p[i].M + 2 * TC_BM - 1) / (2 * TC_BM);
    if ((int)blockIdx.x < cta0 + c) break;
    cta0 += c;
    pi = i + 1;
  }
  const ChainPass& P = g.p[pi];
  const int tile0 = 2 * ((int)blockIdx.x - cta0);                          // first 64-row tile of the pass
  const int ntiles = min(2, (P.M + TC_BM - 1) / TC_BM - tile0);            // 1: the pass's last tile is alone
  const int nl = P.n_layers;
  const int w = threadIdx.x / TC_MMA_THREADS;                              // 2: the producer warpgroup
  if (w < ntiles && (threadIdx.x & (TC_MMA_THREADS - 1)) == 0) {
    pp_dbg_tile[w] = P.tile_start + tile0 + w;
    PP_STAMP(0);
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_MMA_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == PRODUCER) {   // descriptor prefetch, as in tc_chain_kernel
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
  if (w < ntiles && (threadIdx.x & (TC_MMA_THREADS - 1)) == 0) PP_STAMP(1);

  if (threadIdx.x >= CH_MMA_THREADS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(CH_PRODUCER_REGS));
    // ===== TMA producer: per layer, tile 0's items, then tile 1's (a missing tile has none) =====
    if (warp == PRODUCER && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nl; ++j) {
        const ChainLayer& Lj = P.L[j];
        const int nkb = Lj.kblocks[0] + Lj.kblocks[1];
        const int nb = (Lj.bn + 63) / 64, nh = nb > 2 ? 2 : 1;
        for (int t = 0; t < ntiles; ++t) {
          const int m0 = (tile0 + t) * TC_BM;
          uint8_t* opnd = opnd0 + (size_t)t * planes * CH_OPND_PLANE;
          for (int kb = 0; kb < nkb; ++kb) {
            const int seg = kb >= Lj.kblocks[0] ? 1 : 0;
            const int kloc = (seg ? kb - Lj.kblocks[0] : kb) * TC_BK;
            const int kB = Lj.kB0[seg] + kloc;
            for (int h = 0; h < nh; ++h) {
              const int boxes = min(2, nb - 2 * h);   // MN-major 64-column boxes of this half
              const uint32_t b_bytes = B_MN ? (uint32_t)boxes * 8192 : (uint32_t)min(Lj.bn, PP_HALF) * 128;
              const bool a = j == 0 && h == 0;
              mbar_wait(&empty[stage], phase ^ 1);
              mbar_expect_tx(&full[stage], planes * (b_bytes + (a ? (uint32_t)TC_STAGE_A : 0u)));
              uint8_t* sB = ringB + (size_t)stage * planes * PP_STAGE_B;
              for (int pl = 0; pl < planes; ++pl) {
                if (a) tma_load_3d(opnd + (size_t)((kb & 3) * planes + pl) * TC_STAGE_A, &P.mapA[seg], &full[stage], kloc, m0, pl);
                if (B_MN) {
                  for (int i = 0; i < boxes; ++i)
                    tma_load_3d(sB + pl * PP_STAGE_B + i * 8192, &Lj.mapB, &full[stage], 64 * (2 * h + i), kB, pl);
                } else {
                  tma_load_3d(sB + pl * PP_STAGE_B, &Lj.mapB, &full[stage], kB, PP_HALF * h, pl);
                }
              }
              if (++stage == stages) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CH_MMA_REGS));
    // ===== MMA warpgroup w: tile w through every layer; a missing tile's warpgroup has nothing to do =====
    if (w < ntiles) {
      float* row = scratch + threadIdx.x * 16;
      uint8_t* opnd = opnd0 + (size_t)w * planes * CH_OPND_PLANE;
      const int m0 = (tile0 + w) * TC_BM;
      int pos = 0;   // ring position of tile 0's first item of layer j
      for (int j = 0; j < nl; ++j) {
        const int items = pp_items(P.L[j]);
        const int wg = pp_wg();   // read afresh: not kept in a register through the layer bodies
        const int mine = pos + wg * items;
        // turns: warpgroup 0's layer j, warpgroup 1's layer j, warpgroup 0's layer j + 1, ...
        const bool wait = ntiles == 2 && (wg == 1 || j > 0), give = ntiles == 2 && (wg == 0 || j + 1 < nl);
        switch ((P.L[j].bn + 63) / 64) {
          case 1: pp_layer<PLANES2, B_MN, 1>(g, P, j, ringB, opnd, row, stages, full, empty, m0, mine, wait, give); break;
          case 2: pp_layer<PLANES2, B_MN, 2>(g, P, j, ringB, opnd, row, stages, full, empty, m0, mine, wait, give); break;
          case 3: pp_layer<PLANES2, B_MN, 3>(g, P, j, ringB, opnd, row, stages, full, empty, m0, mine, wait, give); break;
          default: pp_layer<PLANES2, B_MN, 4>(g, P, j, ringB, opnd, row, stages, full, empty, m0, mine, wait, give); break;
        }
        pos += items * ntiles;
      }
      if ((threadIdx.x & (TC_MMA_THREADS - 1)) == 0) bulk_wait();   // the image stores this thread issued have completed
    }
  }

  if ((pp_tid() & 31) == 0 && pp_wg() < ntiles) { if (g.dbg) atomicMax(&g.dbg[(size_t)pp_dbg_tile[pp_wg()] * TC_DBG_SLOTS + 5], gtime()); }
  __syncthreads();
  if (pp_wg() < ntiles && pp_lead()) PP_STAMP(6);
}

#undef PP_STAMP

}  // namespace dsact
