// wgmma grouped GEMM for the dense layers of the DSAC-T update (DSACT_GEMM_BF16X3 / DSACT_GEMM_BF16), sm_90a.
//
// Operands are bf16 "images" of the fp32 tensors: plane 0 = hi = bf16(x), plane 1 = lo = bf16(x - hi).
// BF16X3 accumulates hi*hi + hi*lo + lo*hi in fp32 (relative product error ~2^-16, enough for the 1e-4
// parity gate, SURVEY.md §7 "Parity vs speed"); BF16 uses plane 0 only.
//
// One CTA computes one 64 x BN output tile (BN <= 256) of one problem of the group:
//   warps 0..3 : one warpgroup: wgmma.mma_async (accumulator in registers, fp32), then the epilogue straight from the
//                accumulator fragment (bias / activation / derivative / fp32 / bf16-image stores)
//   warp 4     : TMA producer (cp.async.bulk.tensor.3d, 128B swizzle, mbarrier complete_tx)
// The three orientations of a linear layer never need a transposed copy: the wgmma descriptors read
// K-major or MN-major shared-memory tiles as the reduction dimension requires
//   forward  y  = x W^T   : A K-major (x image),   B K-major  (W image)
//   dgrad    dx = dy W    : A K-major (dy image),  B MN-major (W image)
//   wgrad    dW = dy^T x  : A MN-major (dy image), B MN-major (x image); split over the batch, each split
//                           stores its partial tile to a workspace slab (no atomics), reduced later.  The step's
//                           weight gradients run on the persistent 128-row kernel of wgrad_tc.cuh, which reads the
//                           same images with the same tensor maps.
#pragma once
#include <stdio.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm_simt.cuh"  // activations, EPI_* enums
#include "kernels.cuh"    // begin_step / noise bodies of the merged prologue launch
#include "wgmma.cuh"

namespace dsact {

constexpr int TC_BM = 64;        // rows of a tile: the M of one warpgroup's wgmma
constexpr int TC_BK = 64;        // bf16 elements per k-block = one 128-byte swizzle row
constexpr int TC_MAXG = 16;
constexpr int TC_STAGE_A = TC_BM * TC_BK * 2;   // 8 KiB per plane
constexpr int TC_MMA_THREADS = 128;             // the MMA / epilogue warpgroup
constexpr int TC_THREADS = TC_MMA_THREADS + 32; // + the TMA producer warp
constexpr int TC_SCRATCH = TC_MMA_THREADS * 16 * 4;   // per-thread 16-float rows for the generic activations

enum { EPI_PARTIAL = 4 };  // wgrad: plain store into slab `ks`

struct TcProb {
  CUtensorMap mapA[2];      // A operand; a second K segment for cat(obs, act)
  CUtensorMap mapB;
  int kblocks[2];           // k-blocks (of 64) per A segment
  int kB0[2];               // element offset of each segment along B's reduction dimension
  int M, N, bn;             // output extents; N-tile width (multiple of 16, <= 256)
  int tiles_m, tiles_n, ksplit, tile_start;
  float* C;                 // fp32 output or null
  int ldc;
  long long split_stride;   // floats between consecutive split slabs (EPI_PARTIAL)
  const float* bias;
  float* Zout;              // act'(pre-activation) store (ld = ldc)
  const float* Zin;         // act'(pre-activation) input of the derivative
  int ldz;
  float* colsum;            // bias gradient accumulation (EPI_DACT)
  __nv_bfloat16* img;       // bf16 hi/lo image of the result, or null
  int img_pitch;
  long long img_plane;      // elements between the hi and lo planes
  int epi, act;
};

struct TcGroup {
  int n;
  int passes;               // 3 = hi*hi + hi*lo + lo*hi, 1 = hi*hi
  unsigned long long* dbg;  // optional per-CTA phase timestamps (DSACT_TC_DEBUG), 8 slots per CTA
  int tile0;                // first tile of this launch (a group may be issued as several launches of bounded size)
  TcProb p[TC_MAXG];
};

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Build with -DDSACT_MBAR_GUARD to turn a barrier that never completes (a protocol bug in a kernel under development)
// into a trap after ~2 s instead of a hung GPU: DSACT_NVCC_FLAGS="-DDSACT_MBAR_GUARD" python -c "import __graft_entry__ ..."
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#ifdef DSACT_MBAR_GUARD
  unsigned long long t0;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
  for (;;) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, P1;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680) : "memory");
    if (ok) return;
    unsigned long long t1;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
    if (t1 - t0 > 2000000000ull) {
      printf("mbar_wait timeout: block %d thread %d barrier smem+%u parity %u\n", (int)blockIdx.x, (int)threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
#else
  asm volatile(
      "{\n\t.reg .pred P1;\n\tWAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra WAIT_DONE;\n\tbra WAIT_LOOP;\n\tWAIT_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity), "r"(0x989680)
      : "memory");
#endif
}
// Non-blocking: has the phase of `parity` completed?
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.u32 %0, 1, 0, P1;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" ::"r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>   // at most N committed wgmma groups of this warp still in flight
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wg_bar() { asm volatile("bar.sync 1, %0;" ::"n"(TC_MMA_THREADS) : "memory"); }   // the MMA warpgroup only
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// TMA store of one box from shared memory (elements outside the tensor are not written), as part of this thread's next
// bulk async-group; wait_read: the source of every committed group has been read (shared memory may be rewritten).
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// Four 8 x 8 b16 matrices: lane l passes the shared address of row l & 7 of matrix l >> 3 (16 bytes), and word i of every
// lane is its fragment of matrix i (row lane >> 2, columns 2 (lane & 3), + 1).
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(w0), "r"(w1), "r"(w2), "r"(w3)
               : "memory");
}

// Shared-memory matrix descriptor of wgmma, 128-byte swizzle (bits 62-63 = 1).
//   K-major : rows of 128 B (64 bf16 of K), 8-row groups SBO = 1024 B apart; advance K by 32 B per k16 step.
//   MN-major: k-rows of 128 B (64 bf16 of M/N), 8-k groups SBO = 1024 B apart, 64-wide M/N blocks LBO apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// One m64 x (64 NB) x k16 wgmma.
template <int NB, int TA, int TB>
__device__ __forceinline__ void wgmma_nb(float (&d)[128], uint64_t a, uint64_t b) {
  if constexpr (NB == 1) wgmma_n64<TA, TB>(d, a, b);
  else if constexpr (NB == 2) wgmma_n128<TA, TB>(d, a, b);
  else if constexpr (NB == 3) wgmma_n192<TA, TB>(d, a, b);
  else wgmma_n256<TA, TB>(d, a, b);
}

// One k16 step of a 64 x (64 NB) tile: hi*hi, and with two planes also hi*lo + lo*hi.
// The tile width is a compile-time constant of the whole MMA loop and epilogue: with a runtime width the accumulator
// is read and written on paths ptxas cannot prove uniform, and it then waits for every wgmma before issuing the next.
template <int NB, int TA, int TB, bool PLANES2>
__device__ __forceinline__ void wgmma_step(float (&d)[128], uint64_t a_hi, uint64_t b_hi, uint64_t a_lo, uint64_t b_lo) {
  wgmma_nb<NB, TA, TB>(d, a_hi, b_hi);
  if constexpr (PLANES2) { wgmma_nb<NB, TA, TB>(d, a_hi, b_lo); wgmma_nb<NB, TA, TB>(d, a_lo, b_hi); }
}

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define TC_DBG_SLOTS 48
#define TC_STAMP(slot) do { if (g.dbg) g.dbg[(size_t)blockIdx.x * TC_DBG_SLOTS + (slot)] = gtime(); } while (0)

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// ---- epilogue math ---------------------------------------------------------------------------------------
// The activation arithmetic is written on pairs of neighbouring columns (two independent dependency chains per call).
struct f2 { float x, y; };
__device__ __forceinline__ f2 pk2(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ void upk2(f2 a, float& lo, float& hi) { lo = a.x; hi = a.y; }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return f2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return f2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ f2 bc2(float c) { return pk2(c, c); }

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcpf(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// Exact-erf GELU (nn.GELU(), reference networks/mlp.py:15-20) and its derivative for a pair of pre-activations:
//   Phi(z) = 0.5 erfc(-z / sqrt 2),  erfc(x) = t P(t) exp(-x^2),  t = 1 / (1 + p x)  for x = |z| / sqrt 2 >= 0
// (Abramowitz & Stegun 7.1.26, |error of erf| <= 1.5e-7; 3.0e-7 on Phi as evaluated here in fp32 — the bf16 split
// products of this mode carry 1.5e-5).  exp(-x^2) = exp(-z^2 / 2) is also the Gaussian density up to a constant, so
// one ex2 serves Phi and phi.
template <bool WANT_D>
__device__ __forceinline__ void gelu_pair(float& z0, float& z1, float& d0, float& d1) {
  const f2 z = pk2(z0, z1);
  const f2 az = pk2(fabsf(z0), fabsf(z1));
  const f2 den = fma2(az, bc2(0.23164189f), bc2(1.0f));          // 1 + p |z| / sqrt 2, p = 0.3275911
  float n0, n1;
  upk2(den, n0, n1);
  const f2 t = pk2(rcpf(n0), rcpf(n1));
  const f2 se = mul2(mul2(z, bc2(-0.72134752044448170f)), z);     // -z^2 / 2 * log2 e
  float s0, s1;
  upk2(se, s0, s1);
  const f2 e = pk2(ex2f(s0), ex2f(s1));                            // exp(-z^2 / 2)
  f2 pl = fma2(bc2(0.5f * 1.061405429f), t, bc2(0.5f * -1.453152027f));
  pl = fma2(pl, t, bc2(0.5f * 1.421413741f));
  pl = fma2(pl, t, bc2(0.5f * -0.284496736f));
  pl = fma2(pl, t, bc2(0.5f * 0.254829592f));
  const f2 hu = mul2(mul2(pl, t), e);                              // 0.5 erfc(|z| / sqrt 2) = Phi(-|z|)
  const f2 omh = fma2(hu, bc2(-1.0f), bc2(1.0f));
  float h0, h1, o0, o1;
  upk2(hu, h0, h1);
  upk2(omh, o0, o1);
  const f2 cdf = pk2(z0 < 0.f ? h0 : o0, z1 < 0.f ? h1 : o1);
  const f2 a = mul2(z, cdf);
  if (WANT_D) {
    const f2 dd = fma2(mul2(z, bc2(0.3989422804014327f)), e, cdf);   // Phi + z phi
    upk2(dd, d0, d1);
  }
  upk2(a, z0, z1);
}

// v[i] = act(z_i) with z_i = v[i] on entry; if WANT_D also d[i] = act'(z_i).  The dispatch is hoisted out of the
// unrolled loops (inlining the 7-way switch per element makes the kernels several times larger): GELU (the
// reference's default) and ReLU get unrolled bodies, the rest a compact loop over a private shared-memory row.
template <bool WANT_D, int NV>
__device__ __forceinline__ void act_fwdN(float (&v)[NV], float (&d)[NV], int act, float* row) {
  if (act == ACT_GELU) {
#pragma unroll
    for (int i = 0; i < NV; i += 2) gelu_pair<WANT_D>(v[i], v[i + 1], d[i], d[i + 1]);
  } else if (act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (WANT_D) d[i] = v[i] > 0.f ? 1.f : 0.f;
      v[i] = fmaxf(v[i], 0.f);
    }
  } else if (act != ACT_LINEAR) {
#pragma unroll
    for (int i = 0; i < NV; ++i) row[i] = v[i];
    if (WANT_D) {
#pragma unroll 1
      for (int i = 0; i < NV; ++i) row[i] = act_bwd(row[i], act);
#pragma unroll
      for (int i = 0; i < NV; ++i) { d[i] = row[i]; row[i] = v[i]; }
    }
#pragma unroll 1
    for (int i = 0; i < NV; ++i) row[i] = act_fwd(row[i], act);
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = row[i];
  } else if (WANT_D) {
#pragma unroll
    for (int i = 0; i < NV; ++i) d[i] = 1.f;
  }
}

// hi/lo split of two neighbouring K elements straight into packed words (x0 = lower k -> low half)
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo_k, float hi_k) {
  uint32_t w;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w) : "f"(hi_k), "f"(lo_k));
  return w;
}
__device__ __forceinline__ void split_pack2(float x0, float x1, uint32_t& whi, uint32_t& wlo) {
  whi = cvt_bf16x2(x0, x1);
  wlo = cvt_bf16x2(x0 - __uint_as_float(whi << 16), x1 - __uint_as_float(whi & 0xffff0000u));
}

// What the epilogue of a tile needs.  In the tensor-core modes `Zout`/`Zin` carry act'(z) (computed where erf is
// already at hand) instead of z, so the backward epilogue is a load and a multiply.
struct EpiArgs {
  int epi, act, M, N, ldc, ldz;
  const float* bias;
  float* Zout;
  const float* Zin;
  float* colsum;
  float* C;
  __nv_bfloat16* img;
  int img_pitch;
  long long img_plane;
};

// Predicated read-only loads (0 where `pred` is false), kept by the compiler where they are written: it would otherwise
// hoist every load of an epilogue (__ldg reads invariant memory) to the top, where the results wait in registers through
// the arithmetic of the groups before them, and a branch per load leaves a merge of values to allocate per load.
__device__ __forceinline__ float ldg_if(const float* p, bool pred) {
  float v = 0.f;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p ld.global.nc.f32 %0, [%1];\n\t}"
               : "+f"(v) : "l"(p), "r"((int)pred));
  return v;
}
__device__ __forceinline__ float2 ldg2_if(const float* p, bool pred) {
  float2 v = make_float2(0.f, 0.f);
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p ld.global.nc.v2.f32 {%0, %1}, [%2];\n\t}"
               : "+f"(v.x), "+f"(v.y) : "l"(p), "r"((int)pred));
  return v;
}

// Columns (c, c + 1) of one row, c even; columns >= n are not touched (loads return 0).  `pair`: the row pitch is even and
// the base 8-byte aligned, so the two columns are one 8-byte access (the last column of an odd n a 4-byte one).
__device__ __forceinline__ void ld_pair(const float* p, int c, int n, bool pair, float& a, float& b) {
  if (pair) {
    const float2 x = ldg2_if(p + c, c + 1 < n);
    const float s = ldg_if(p + c, c + 1 == n);
    a = c + 1 < n ? x.x : s;
    b = x.y;
  } else {
    a = ldg_if(p + c, c < n);
    b = ldg_if(p + c + 1, c + 1 < n);
  }
}
__device__ __forceinline__ void st_pair(float* p, int c, int n, bool pair, float a, float b) {
  if (pair && c + 1 < n) {
    *reinterpret_cast<float2*>(p + c) = make_float2(a, b);
  } else {
    if (c < n) p[c] = a;
    if (c + 1 < n) p[c + 1] = b;
  }
}
__device__ __forceinline__ bool pairs_ok(const float* p, int ld) { return ((ld | (int)(reinterpret_cast<uintptr_t>(p) >> 2)) & 1) == 0; }
// An unconditional 8-byte read-only load, kept where it is written as ldg2_if is.
__device__ __forceinline__ void ldg2(const float* p, float& a, float& b) {
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(a), "=f"(b) : "l"(p));
}

// Epilogue kinds.  EK_RUNTIME reads the variant (epi, act, which optional pointers are set) from EpiArgs and checks every
// value's row against M and column against N.  The others fix the variant at compile time for a FULL tile: all rows of the
// 64-row tile are < M, every column of the accumulator is < N, the bias / act' / Zout pointers are 8-byte aligned with
// rows N floats apart, and there is no fp32 C store.  Each kind body then holds one activation and no masking.  The layer
// chain decides a layer's kind on the host (ChainLayer::kind) and checks the rows per tile.
//   EK_GELU / EK_RELU     : EPI_BIAS_ACT with a bias, without Zout;  EK_GELU_Z / EK_RELU_Z: with Zout
//   EK_DACT / EK_DACT_SUM : EPI_DACT without / with colsum
enum { EK_RUNTIME = 0, EK_GELU, EK_GELU_Z, EK_RELU, EK_RELU_Z, EK_DACT, EK_DACT_SUM };
__host__ __device__ constexpr bool ek_fwd(int k) { return k >= EK_GELU && k <= EK_RELU_Z; }
__host__ __device__ constexpr int ek_epi(int k) { return ek_fwd(k) ? EPI_BIAS_ACT : EPI_DACT; }
__host__ __device__ constexpr int ek_act(int k) { return k == EK_GELU || k == EK_GELU_Z ? ACT_GELU : ACT_RELU; }
__host__ __device__ constexpr bool ek_zout(int k) { return k == EK_GELU_Z || k == EK_RELU_Z; }

// Epilogue of the warpgroup's 64 x (64 NB) accumulator, element (0, 0) = output (m0, n0), straight from the wgmma
// fragment: acc[16 g + t] sits in row ra (t & 2 == 0) or ra + 8, column n0 + 32 g + 8 (t >> 2) + 2 (lane & 3) + (t & 1).
// Group g (16 values) is split into the loads of its global inputs (epi_in) and the arithmetic and stores (epi_group),
// so that a caller can issue the loads early.
#define COL(t) (cq + 32 * g + 8 * ((t) >> 2) + ((t) & 1))
#define ROW(t) (ra + (((t) & 2) ? 8 : 0))
#define ROW_OK(t) (((t) & 2) ? ok1 : ok0)
#define EPI_FRAG_COORDS                                                         \
  const int lane = threadIdx.x & 31;                                            \
  const int ra = m0 + (((threadIdx.x & (TC_MMA_THREADS - 1)) >> 5) * 16) + (lane >> 2); \
  const bool ok0 = ra < E.M, ok1 = ra + 8 < E.M;                                \
  const int cq = n0 + 2 * (lane & 3);

// The global inputs of group g: x[t] = act'(z) of value t (EPI_DACT), or x[2 (t >> 2) + (t & 1)] = the bias of value t's
// column (EPI_STORE / EPI_BIAS_ACT with a bias).
template <int KIND = EK_RUNTIME>
__device__ __forceinline__ void epi_in(float (&x)[16], const EpiArgs& E, int m0, int n0, int g) {
  EPI_FRAG_COORDS
  if constexpr (KIND != EK_RUNTIME) {   // full tile: unconditional 8-byte loads
    if constexpr (ek_epi(KIND) == EPI_DACT) {
#pragma unroll
      for (int t = 0; t < 16; t += 2) ldg2(E.Zin + (size_t)ROW(t) * E.ldz + COL(t), x[t], x[t + 1]);
    } else {
#pragma unroll
      for (int t = 0; t < 16; t += 4) ldg2(E.bias + COL(t), x[t / 2], x[t / 2 + 1]);
    }
    return;
  }
  // one loop body per access width, so that `pair` is a constant inside it
#define EPI_IN_ZIN(pair) \
  _Pragma("unroll") for (int t = 0; t < 16; t += 2) ld_pair(E.Zin + (size_t)ROW(t) * E.ldz, COL(t), ROW_OK(t) ? E.N : 0, pair, x[t], x[t + 1]);
#define EPI_IN_BIAS(pair) \
  _Pragma("unroll") for (int t = 0; t < 16; t += 4) ld_pair(E.bias, COL(t), E.N, pair, x[t / 2], x[t / 2 + 1]);
  if (E.epi == EPI_DACT) {
    if (pairs_ok(E.Zin, E.ldz)) { EPI_IN_ZIN(true) } else { EPI_IN_ZIN(false) }
  } else if ((E.epi == EPI_STORE || E.epi == EPI_BIAS_ACT) && E.bias) {
    if (pairs_ok(E.bias, 0)) { EPI_IN_BIAS(true) } else { EPI_IN_BIAS(false) }
  }
#undef EPI_IN_ZIN
#undef EPI_IN_BIAS
}

// Group g's global inputs x (epi_in) applied to its values v as epi_group applies them: the bias added or act'
// multiplied.  A caller that loads the next group's inputs into the same registers applies them first (APPLIED).
template <int KIND = EK_RUNTIME>
__device__ __forceinline__ void epi_apply(float (&v)[16], const float (&x)[16], const EpiArgs& E) {
  const int epi = KIND == EK_RUNTIME ? E.epi : ek_epi(KIND);
  if ((epi == EPI_STORE || epi == EPI_BIAS_ACT) && (KIND != EK_RUNTIME || E.bias)) {
#pragma unroll
    for (int t = 0; t < 16; ++t) v[t] += x[2 * (t >> 2) + (t & 1)];
  } else if (epi == EPI_DACT) {
#pragma unroll
    for (int t = 0; t < 16; ++t) v[t] *= x[t];
  }
}

// Arithmetic and stores of group g: v = the accumulator values on entry, the result on return; x = its inputs (epi_in),
// unused when the caller has APPLIED them.  Columns >= N leave as zeros (they are the next layer's K padding and the image
// padding).  `row`: this thread's 16-float shared-memory row (generic activations).
template <bool PLANES2, int KIND = EK_RUNTIME, bool APPLIED = false>
__device__ __forceinline__ void epi_group(float (&v)[16], const float (&x)[16], const EpiArgs& E, int m0, int n0, int g,
                                          float* row) {
  EPI_FRAG_COORDS
  constexpr bool RT = KIND == EK_RUNTIME;
  const int epi = RT ? E.epi : ek_epi(KIND);
  const int act = RT ? E.act : ek_act(KIND);
  float d[16];
  if (epi == EPI_STORE || epi == EPI_BIAS_ACT) {
    if (!APPLIED && (!RT || E.bias)) {
#pragma unroll
      for (int t = 0; t < 16; ++t) v[t] += x[2 * (t >> 2) + (t & 1)];
    }
    if (epi == EPI_BIAS_ACT) {
      if (RT ? E.Zout != nullptr : ek_zout(KIND)) {
        act_fwdN<true, 16>(v, d, act, row);
        if constexpr (RT) {
          const bool pair = pairs_ok(E.Zout, E.ldc);
#pragma unroll
          for (int t = 0; t < 16; t += 2) st_pair(E.Zout + (size_t)ROW(t) * E.ldc, COL(t), ROW_OK(t) ? E.N : 0, pair, d[t], d[t + 1]);
        } else {   // full tile: unconditional 8-byte stores
#pragma unroll
          for (int t = 0; t < 16; t += 2) *reinterpret_cast<float2*>(E.Zout + (size_t)ROW(t) * E.ldc + COL(t)) = make_float2(d[t], d[t + 1]);
        }
      } else {
        act_fwdN<false, 16>(v, d, act, row);
      }
    }
  } else if (epi == EPI_DACT) {
    if (!APPLIED) {
#pragma unroll
      for (int t = 0; t < 16; ++t) v[t] *= x[t];
    }
    if (RT ? E.colsum != nullptr : KIND == EK_DACT_SUM) {  // bias gradient: both rows of the thread, then the eight lanes that share its columns
      // s[k]: column k = 2 (t >> 2) + (t & 1) of the thread's eight.  A transposing butterfly over lane bits 2, 3, 4: at
      // each step a lane keeps half of its columns (the upper half if its bit is set), adds the partner's partial sums of
      // them and sends the other half, so each lane ends with one column's sum over the eight lanes, added in the same
      // tree (own + partner at every step) as a full xor reduction per column.
      float s[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) s[k] = v[4 * (k >> 1) + (k & 1)] + v[4 * (k >> 1) + 2 + (k & 1)];
#pragma unroll
      for (int h = 4; h >= 1; h >>= 1) {
        const bool up = lane & (16 / h);
#pragma unroll
        for (int i = 0; i < h; ++i) {
          const float send = up ? s[i] : s[i + h], keep = up ? s[i + h] : s[i];
          s[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16 / h);
        }
      }
      const int k = ((lane >> 2) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 4) & 1);
      const int c = cq + 32 * g + 8 * (k >> 1) + (k & 1);
      if (!RT || c < E.N) atomicAdd(E.colsum + c, s[0]);
    }
  }
  if constexpr (RT) {
#pragma unroll
    for (int t = 0; t < 16; ++t) v[t] = COL(t) < E.N ? v[t] : 0.f;
    if (E.C) {   // scalar: head outputs have odd widths (e.g. the action columns)
#pragma unroll
      for (int t = 0; t < 16; ++t)
        if (ROW_OK(t) && COL(t) < E.N) E.C[(size_t)ROW(t) * E.ldc + COL(t)] = v[t];
    }
  }
}

// The bf16 hi/lo image of group g's results v (columns >= N are zeros) up to column (N + 7) / 8 * 8.  The layer chain
// stores its images by TMA from its operand buffer instead.
template <bool PLANES2>
__device__ __forceinline__ void epi_img(const float (&v)[16], const EpiArgs& E, int m0, int n0, int g) {
  EPI_FRAG_COORDS
  const int img_w = (E.N + 7) / 8 * 8;
  if (E.img) {  // packed bf16 pairs (pitch % 8 == 0, even column): one 4-byte store per plane
#pragma unroll
    for (int t = 0; t < 16; t += 2) {
      if (ROW_OK(t) && COL(t) < img_w) {
        uint32_t whi, wlo;
        split_pack2(v[t], v[t + 1], whi, wlo);
        __nv_bfloat16* hp = E.img + (size_t)ROW(t) * E.img_pitch + COL(t);
        *reinterpret_cast<uint32_t*>(hp) = whi;
        if (PLANES2) *reinterpret_cast<uint32_t*>(hp + E.img_plane) = wlo;
      }
    }
  }
}
#undef COL
#undef ROW
#undef ROW_OK
#undef EPI_FRAG_COORDS

// The whole epilogue, group by group (loads, then arithmetic).  On return acc holds the result.
template <bool PLANES2, int NB>
__device__ __forceinline__ void epi_frag(float (&acc)[128], const EpiArgs& E, int m0, int n0, float* row) {
#pragma unroll
  for (int g = 0; g < 2 * NB; ++g) {
    float x[16], v[16];
    epi_in(x, E, m0, n0, g);
#pragma unroll
    for (int t = 0; t < 16; ++t) v[t] = acc[16 * g + t];
    epi_group<PLANES2>(v, x, E, m0, n0, g, row);
    epi_img<PLANES2>(v, E, m0, n0, g);
#pragma unroll
    for (int t = 0; t < 16; ++t) acc[16 * g + t] = v[t];
  }
}

// MMA warpgroup of one 64 x (64 NB) tile: the MMAs, one k-block of them kept in flight (the slot of k-block kb is
// released once kb + 1 has been issued and kb has retired), then the epilogue on the accumulator registers.
template <bool A_MN, bool B_MN, bool PLANES2, int NB>
__device__ __forceinline__ void gemm_tile_mma(const TcGroup& g, const TcProb& P, uint8_t* smem, int stages, int stage_b,
                                              uint64_t* full, uint64_t* empty, int kb_begin, int kb_end, int ks, int m0, int n0) {
  constexpr int planes = PLANES2 ? 2 : 1;
  const int stage_bytes = planes * (TC_STAGE_A + stage_b);
  const int lane = threadIdx.x & 31;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 32 * NB; ++i) acc[i] = 0.f;
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kb = kb_begin; kb < kb_end; ++kb) {
    mbar_wait(&full[stage], phase);
    if (kb == kb_begin && threadIdx.x == 0) TC_STAMP(2);
    const uint32_t sA = smem_u32(smem + (size_t)stage * stage_bytes);
    const uint32_t sB = sA + planes * TC_STAGE_A;
    wg_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) {
      const uint32_t a_off = A_MN ? k * 2048 : k * 32;
      const uint32_t b_off = B_MN ? k * 2048 : k * 32;
      const uint64_t a_hi = make_desc(sA + a_off, A_MN ? 8192 : 16, 1024);
      const uint64_t b_hi = make_desc(sB + b_off, B_MN ? 8192 : 16, 1024);
      const uint64_t a_lo = make_desc(sA + TC_STAGE_A + a_off, A_MN ? 8192 : 16, 1024);
      const uint64_t b_lo = make_desc(sB + stage_b + b_off, B_MN ? 8192 : 16, 1024);
      wgmma_step<NB, A_MN, B_MN, PLANES2>(acc, a_hi, b_hi, a_lo, b_lo);
    }
    wg_commit();
    wg_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);  // this warp's share of k-block kb - 1 retired
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
  if (threadIdx.x == 0) TC_STAMP(3);
  wg_bar();   // every MMA of the tile retired: the pipeline smem is dead and serves as the activation scratch
  if (threadIdx.x == 0) TC_STAMP(4);
  EpiArgs E;
  E.epi = P.epi; E.act = P.act; E.M = P.M; E.N = P.N; E.ldc = P.ldc; E.ldz = P.ldz;
  E.bias = P.bias; E.Zout = P.Zout; E.Zin = P.Zin; E.colsum = P.colsum;
  E.C = P.C ? P.C + (P.epi == EPI_PARTIAL ? (size_t)ks * P.split_stride : 0) : nullptr;
  E.img = P.img; E.img_pitch = P.img_pitch; E.img_plane = P.img_plane;
  epi_frag<PLANES2, NB>(acc, E, m0, n0, reinterpret_cast<float*>(smem) + threadIdx.x * 16);
}

// A_MN / B_MN: operand is MN-major (reduction dimension strided in global memory).
template <bool A_MN, bool B_MN, bool PLANES2>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_gemm_kernel(const __grid_constant__ TcGroup g, int stages, int stage_b) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzle atoms
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // pointer arithmetic on the __shared__ array keeps LDS/STS
  constexpr int planes = PLANES2 ? 2 : 1;
  const int stage_bytes = planes * (TC_STAGE_A + stage_b);  // stage_b: bytes of one B plane (widest tile of the launch)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)stages * stage_bytes);
  uint64_t* full = bars;             // [stages]  TMA -> MMA
  uint64_t* empty = bars + stages;   // [stages]  MMA -> TMA (one arrival per MMA warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) TC_STAMP(0);

  const int tile_id = (int)blockIdx.x + g.tile0;
  int pi = 0;
#pragma unroll
  for (int i = 1; i < TC_MAXG; ++i)
    if (i < g.n && tile_id >= g.p[i].tile_start) pi = i;
  const TcProb& P = g.p[pi];
  int local = tile_id - P.tile_start;
  const int tiles_mn = P.tiles_m * P.tiles_n;
  const int ks = local / tiles_mn;
  local -= ks * tiles_mn;
  const int m0 = (local / P.tiles_n) * TC_BM, n0 = (local % P.tiles_n) * P.bn;
  const int bn = P.bn;

  // k-block range of this CTA (split only ever applies to single-segment problems)
  const int nkb = P.kblocks[0] + P.kblocks[1];
  int kb_begin = 0, kb_end = nkb;
  if (P.ksplit > 1) {
    const int per = (nkb + P.ksplit - 1) / P.ksplit;
    kb_begin = ks * per;
    kb_end = min(nkb, kb_begin + per);
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_MMA_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 4 && lane < 3) {   // descriptor prefetch (kernel parameters: independent of the preceding kernel)
    const CUtensorMap* m = lane == 0 ? &P.mapA[0] : (lane == 1 ? (P.kblocks[1] > 0 ? &P.mapA[1] : nullptr) : &P.mapB);
    if (m) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
  }
  __syncthreads();
  // programmatic dependent launch: everything above overlapped the predecessor's tail; its memory is needed from here on
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) TC_STAMP(1);

  if (warp == 4) {
    // ===== TMA producer =====
    if (lane == 0) {
      const int b_boxes = B_MN ? (bn + 63) / 64 : 1;
      const uint32_t b_bytes = B_MN ? (uint32_t)b_boxes * 64 * 128 : (uint32_t)bn * 128;
      const uint32_t tx = planes * ((uint32_t)TC_STAGE_A + b_bytes);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], tx);
        const int seg = kb >= P.kblocks[0] ? 1 : 0;
        const int kloc = (seg ? kb - P.kblocks[0] : kb) * TC_BK;   // offset inside the A segment
        const int kB = P.kB0[seg] + kloc;                         // offset along B's reduction dimension
        uint8_t* sA = smem + (size_t)stage * stage_bytes;
        uint8_t* sB = sA + planes * TC_STAGE_A;
        for (int pl = 0; pl < planes; ++pl) {
          if (A_MN) tma_load_3d(sA + pl * TC_STAGE_A, &P.mapA[seg], &full[stage], m0, kloc, pl);
          else tma_load_3d(sA + pl * TC_STAGE_A, &P.mapA[seg], &full[stage], kloc, m0, pl);
          if (B_MN) {
            for (int i = 0; i < b_boxes; ++i)
              tma_load_3d(sB + pl * stage_b + i * 8192, &P.mapB, &full[stage], n0 + 64 * i, kB, pl);
          } else {
            tma_load_3d(sB + pl * stage_b, &P.mapB, &full[stage], kB, n0, pl);
          }
        }
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===== MMA warpgroup: wgmma N = 64 nb; columns >= bn are never stored =====
    switch ((bn + 63) / 64) {
      case 1: gemm_tile_mma<A_MN, B_MN, PLANES2, 1>(g, P, smem, stages, stage_b, full, empty, kb_begin, kb_end, ks, m0, n0); break;
      case 2: gemm_tile_mma<A_MN, B_MN, PLANES2, 2>(g, P, smem, stages, stage_b, full, empty, kb_begin, kb_end, ks, m0, n0); break;
      case 3: gemm_tile_mma<A_MN, B_MN, PLANES2, 3>(g, P, smem, stages, stage_b, full, empty, kb_begin, kb_end, ks, m0, n0); break;
      default: gemm_tile_mma<A_MN, B_MN, PLANES2, 4>(g, P, smem, stages, stage_b, full, empty, kb_begin, kb_end, ks, m0, n0); break;
    }
  }

  if (lane == 0 && warp < 4) { if (g.dbg) atomicMax(&g.dbg[(size_t)blockIdx.x * TC_DBG_SLOTS + 5], gtime()); }
  __syncthreads();
  if (threadIdx.x == 0) TC_STAMP(6);
}

// fp32 -> bf16 hi/lo image conversion for tensors that elementwise kernels (or the optimiser) produce.
// Up to two column segments let cat(obs, act)-shaped weights land with the act block on a 64-column boundary.
struct ImgJob {
  const float* src;
  __nv_bfloat16* dst;
  int rows, ld_src;
  int seg_w[2], seg_src0[2], seg_dst0[2];
  int pitch;            // image row pitch (elements); columns not covered by a segment are zero-filled up to `fill_w`
  int fill_w;
  long long plane;
  int block_start;
};
constexpr int IMG_MAXJ = 32;   // every weight of the six networks + a caller-supplied batch in one launch
struct ImgGroup {
  int n, planes;
  ImgJob j[IMG_MAXJ];
};
// One thread converts 8 consecutive columns of one row (one 16-byte store per plane).
__device__ __forceinline__ void image_body(const ImgGroup& g, int block, int img_blocks) {
  int ji = 0;
#pragma unroll
  for (int i = 1; i < IMG_MAXJ; ++i)
    if (i < g.n && block >= g.j[i].block_start) ji = i;
  const ImgJob& J = g.j[ji];
  const int vec_per_row = J.pitch >> 3;
  const int total = J.rows * vec_per_row;
  const int nblocks = (ji + 1 < g.n ? g.j[ji + 1].block_start : img_blocks) - J.block_start;
  for (int i = (block - J.block_start) * blockDim.x + threadIdx.x; i < total; i += nblocks * blockDim.x) {
    const int r = i / vec_per_row, c0 = (i - r * vec_per_row) * 8;
    const float* src = J.src + (size_t)r * J.ld_src;
    uint32_t whi[4], wlo[4];
    float x[8];
    const uintptr_t addr = reinterpret_cast<uintptr_t>(src + c0);
    if (c0 + 8 <= J.seg_w[0] && (addr & 7) == 0) {   // the common case: eight columns of the first segment, vector loads
      if ((addr & 15) == 0) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(src + c0)), b = __ldg(reinterpret_cast<const float4*>(src + c0) + 1);
        x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = __ldg(reinterpret_cast<const float2*>(src + c0) + k);
          x[2 * k] = a.x; x[2 * k + 1] = a.y;
        }
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int c = c0 + e;
        float v = 0.f;
        if (c < J.seg_w[0]) v = __ldg(src + c);
        else if (c >= J.seg_dst0[1] && c < J.seg_dst0[1] + J.seg_w[1]) v = __ldg(src + J.seg_src0[1] + (c - J.seg_dst0[1]));
        x[e] = v;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) split_pack2(x[2 * k], x[2 * k + 1], whi[k], wlo[k]);
    __nv_bfloat16* dst = J.dst + (size_t)r * J.pitch + c0;
    *reinterpret_cast<uint4*>(dst) = make_uint4(whi[0], whi[1], whi[2], whi[3]);
    if (g.planes == 2) *reinterpret_cast<uint4*>(dst + J.plane) = make_uint4(wlo[0], wlo[1], wlo[2], wlo[3]);
  }
}

__global__ void image_kernel(const __grid_constant__ ImgGroup g) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  image_body(g, (int)blockIdx.x, (int)gridDim.x);
}

// Start-of-step work that depends on nothing of the step itself, as ONE launch: weight (and caller-batch) images, the
// accumulator / gradient clears (begin_step_kernel) and the device noise (noise_kernel), each on its own range of blocks.
struct PrologueArgs {
  int img_blocks, zero_blocks, noise_blocks;
  float *state, *grads;
  long long n_grads;
  float *eps1, *eps2, *z3, *z4;
  int B, A;
  unsigned long long seed;
  AdamHyper hy;   // this step's Adam scalars are formed here (last block of the clear range), see adam_scalars_stamp
};
__global__ void step_prologue_kernel(const __grid_constant__ ImgGroup g, const __grid_constant__ PrologueArgs p) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int b = (int)blockIdx.x;
  if (b < p.img_blocks) image_body(g, b, p.img_blocks);
  else if (b < p.img_blocks + p.zero_blocks) {
    if (b == p.img_blocks + p.zero_blocks - 1) adam_scalars_stamp(p.state, p.hy);
    begin_step_body(p.state, p.grads, p.n_grads, b - p.img_blocks, p.zero_blocks);
  }
  else noise_body(p.eps1, p.eps2, p.z3, p.z4, p.B, p.A, p.seed, p.state, b - p.img_blocks - p.zero_blocks, p.noise_blocks);
}

// Sum the wgrad split slabs into the flat gradient buffer (which already holds the bias gradients).
__global__ void grad_reduce_kernel(float* __restrict__ grads, const float* __restrict__ slabs, long long n, int nslabs,
                                   long long slab_stride) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const bool vec = (slab_stride & 3) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = reinterpret_cast<const float4*>(grads)[i];
    for (int k = 0; k < nslabs; ++k) {
      const float4 p = __ldg(reinterpret_cast<const float4*>(slabs + (size_t)k * slab_stride) + i);
      s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
    }
    reinterpret_cast<float4*>(grads)[i] = s;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = grads[i];
    for (int k = 0; k < nslabs; ++k) s += slabs[(size_t)k * slab_stride + i];
    grads[i] = s;
  }
}

}  // namespace dsact
