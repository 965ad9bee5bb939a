// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA, wgmma / mma.sync wrappers (inline PTX),
// wgmma descriptor builders, Philox dropout, small math helpers.
//
// Everything in csrc/ is written for sm_90a only (H100); there is no other code path.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace mmfb {

typedef __nv_bfloat16 bf16;

// --------------------------------------------------------------------------------------
// misc
// --------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// First 1024-byte aligned address of the dynamic shared-memory window (SW128 tiles need it).  Pure pointer arithmetic
// on the __shared__ array - an integer round trip would make every later access a generic LD.E/ST.E with 64-bit
// address arithmetic instead of LDS/STS.
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* raw) {
  return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
}

// --------------------------------------------------------------------------------------
// programmatic dependent launch: every kernel of the library lets the NEXT kernel of the stream start launching as soon
// as all of its own CTAs have started (griddep_launch at the top), and waits for the PREVIOUS kernel to have completed and
// flushed its memory before it touches global data (griddep_wait after its own set-up: barrier init,
// descriptor prefetch).  The launch latency and the prologue of kernel n+1 overlap the tail of kernel n.  launch_k
// (mmfb_internal.h) sets the launch attribute that enables this on every kernel of the library.
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// --------------------------------------------------------------------------------------
// mbarrier
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA stores / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Wait with a watchdog: a protocol bug must abort the kernel (trap) instead of hanging the GPU.
// The spin loop is kept to three instructions per failed probe (try_wait itself suspends the warp in hardware for a
// while before it returns false): the clock is read only every 2^16 probes, so that a waiting warp takes few issue
// slots from the other warps of its SM.  No function call (printf) in it: the GEMM consumers wait between wgmma commit
// and wgmma wait, and a call there makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try_wait(bar, parity)) return;
    if ((spins & 0xFFFFu) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
    }
  }
}

// --------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), loads signal an mbarrier with complete_tx::bytes
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// TMA stores: shared -> global, tracked per thread in bulk async-groups.  The smem source must be made visible to the
// async proxy first (fence_proxy_async by every writing thread, then a barrier); elements outside the tensor map are
// not written.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's committed store groups may still be reading their shared-memory source
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// every store group of this thread has completed its global writes
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// named barrier over `count` threads (a multiple of 32); id 0 is __syncthreads'
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// --------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): D[64 x N] (+)= A[64 x 16] * B[16 x N]^T, bf16 operands from shared memory,
// fp32 accumulators in registers, issued by all 128 threads of a warpgroup.
//
// Shared-memory matrix descriptors, SWIZZLE_128B canonical layouts (bf16):
// K-major operand tile  [rows][64 k]  : each row is one 128-byte line (64 bf16 along K), lines of 8
//   consecutive rows form a 1024-byte swizzle atom (exactly what a TMA box {64, rows} with
//   CU_TENSOR_MAP_SWIZZLE_128B writes).  SBO = 1024 B (next 8 rows).  One wgmma (K=16) reads 32 bytes
//   of each line, so the k-th wgmma of the tile starts 32*k bytes further.
// MN-major operand tile [64 k][64 mn] per 8 KB panel: each line is one k, 64 bf16 along M/N (TMA box
//   {64 mn, 64 k}); SBO = 1024 B (next 8 k), LBO = bytes between 64-wide mn panels.  One wgmma (K=16)
//   reads 16 lines = 2048 bytes.
// Descriptor bits: [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, [62,64) layout (1 = 128-byte swizzle).
//
// Accumulator layout of m64nNk16 (f32): thread t of warp w of the warpgroup holds d[i], i < N/2, at
//   row 16 w + t/4 + 8 ((i/2) & 1), column 8 (i/4) + 2 (t%4) + (i & 1).
// --------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// TA / TB = 1: the A / B operand is MN-major (transposed) in shared memory
#define MMFB_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                   "+f"(d[i + 6]), "+f"(d[i + 7])
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : MMFB_F8(0), MMFB_F8(8), MMFB_F8(16), MMFB_F8(24),
        MMFB_F8(32), MMFB_F8(40), MMFB_F8(48), MMFB_F8(56)
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : MMFB_F8(0), MMFB_F8(8), MMFB_F8(16), MMFB_F8(24),
        MMFB_F8(32), MMFB_F8(40), MMFB_F8(48), MMFB_F8(56),
        MMFB_F8(64), MMFB_F8(72), MMFB_F8(80), MMFB_F8(88),
        MMFB_F8(96), MMFB_F8(104), MMFB_F8(112), MMFB_F8(120)
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));
}
#undef MMFB_F8

// The attention kernels' shapes.  Their accumulators are d[N/8][4], one row of four per n8 tile: flattened, that is the
// d[N/2] layout above, and per warp it is the mma.sync m16n8k16 accumulator (rows t/4 and t/4 + 8, columns 2 (t%4) and
// 2 (t%4) + 1 of every n8 tile).
// wgmma_ss: both operands K-major in shared memory.
// wgmma_rs: A from registers - a[4] of thread t of warp w is rows 16 w + t/4 (+ 8 for a[1], a[3]), k columns 2 (t%4),
//   2 (t%4) + 1 (+ 8 for a[2], a[3]), the m16n8k16 A fragment - and B MN-major in shared memory (transpose bit set).
#define MMFB_F4(i) "+f"(d[i][0]), "+f"(d[i][1]), "+f"(d[i][2]), "+f"(d[i][3])
#define MMFB_F16(i) MMFB_F4(i), MMFB_F4(i + 1), MMFB_F4(i + 2), MMFB_F4(i + 3)
#define MMFB_R10(n) "%" #n "0, %" #n "1, %" #n "2, %" #n "3, %" #n "4, %" #n "5, %" #n "6, %" #n "7, %" #n "8, %" #n "9, "
__device__ __forceinline__ void wgmma_ss(float (&d)[4][4], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : MMFB_F16(0)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_ss(float (&d)[8][4], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, " MMFB_R10(1) MMFB_R10(2)
      "%30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : MMFB_F16(0), MMFB_F16(4)
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[8][4], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, " MMFB_R10(1) MMFB_R10(2)
      "%30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
      : MMFB_F16(0), MMFB_F16(4)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_rs(float (&d)[16][4], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, " MMFB_R10(1) MMFB_R10(2)
      MMFB_R10(3) MMFB_R10(4) MMFB_R10(5) "%60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}\n"
      : MMFB_F16(0), MMFB_F16(4), MMFB_F16(8), MMFB_F16(12)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
#undef MMFB_F4
#undef MMFB_F16
#undef MMFB_R10

// --------------------------------------------------------------------------------------
// mma.sync (m16n8k16, bf16 -> fp32) and ldmatrix, for the kernels whose operands are small register tiles (the
// attention-probabilities kernel, optimal transport)
// --------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}

// --------------------------------------------------------------------------------------
// Philox4x32-7 counter RNG (7 rounds: the smallest variant that passes BigCrush) for the dropout keep-bits
// --------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t ctr) {
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  uint32_t c0 = static_cast<uint32_t>(ctr), c1 = static_cast<uint32_t>(ctr >> 32), c2 = 0x243F6A88u,
           c3 = 0x85A308D3u;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
    c0 = n0; c1 = l1; c2 = n2; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// --------------------------------------------------------------------------------------
// math
// --------------------------------------------------------------------------------------
// exact (erf) GELU, branch-free: erf(z) = sign(z) (1 - P(t) exp(-z^2)), t = 1/(1 + 0.3275911 |z|)  (Abramowitz-Stegun
// 7.1.26, |error| <= 1.5e-7, i.e. fp32 rounding level).  With z = x/sqrt(2), exp(-z^2) = exp(-x^2/2) is also the
// Gaussian density needed by the derivative, so forward and backward cost one ex2 + one rcp (both MUFU approx,
// no IEEE slow paths -> no branches) and ~15 FMA-pipe instructions per element.
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float gelu_phi_parts(float x, float& e) {
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752f, fabsf(x), 1.0f));
  e = ex2_approx(x * x * (-0.5f * 1.4426950408889634f));          // exp(-x^2/2)
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float erf_abs = fmaf(-poly * t, e, 1.0f);                  // erf(|x|/sqrt(2))
  return fmaf(0.5f, copysignf(erf_abs, x), 0.5f);                  // Phi(x)
}
__device__ __forceinline__ float gelu_erf(float x) {
  float e;
  return x * gelu_phi_parts(x, e);
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float e;
  const float cdf = gelu_phi_parts(x, e);
  return fmaf(x * 0.3989422804014327f, e, cdf);
}
// ---- fp32 pairs carried in one 64-bit value ----
// The row kernels keep pairs of fp32 lanes together (two bf16 of a packed word).  Hopper has no packed fp32 arithmetic,
// so each helper is two scalar IEEE operations (round-to-nearest, no ftz): the results equal fmaf / * / + per lane.
__device__ __forceinline__ uint64_t pk2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void upk2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace mmfb
