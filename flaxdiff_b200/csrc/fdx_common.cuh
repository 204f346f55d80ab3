// fdx_common.cuh -- shared device helpers for the libfdx sm_90a kernels.
//
// Thin inline-PTX wrappers for the Hopper primitives the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors),
// plus error plumbing for the C-ABI.  No torch, no CUTLASS types.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

// ---------------------------------------------------------------------------
// status codes of the C-ABI (mirrored in include/fdx.h)
// ---------------------------------------------------------------------------
#define FDX_OK 0
#define FDX_ERR_INVALID_ARG (-1)
#define FDX_ERR_UNSUPPORTED (-2)
#define FDX_ERR_CUDA (-3)
#define FDX_ERR_NO_DEVICE (-4)

void fdx_set_error(const char* fmt, ...);
int fdx_check_cuda(cudaError_t e, const char* what);

#define FDX_CUDA(call)                                        \
  do {                                                        \
    int _s = fdx_check_cuda((call), #call);                   \
    if (_s != FDX_OK) return _s;                              \
  } while (0)

#define FDX_REQUIRE(cond, ...)                                \
  do {                                                        \
    if (!(cond)) {                                            \
      fdx_set_error(__VA_ARGS__);                             \
      return FDX_ERR_INVALID_ARG;                             \
    }                                                         \
  } while (0)

void fdx_count_launch();
// which tensor-core kernel family the most recent launch belonged to (bench.py attributes event times)
void fdx_note_kernel(int kind);
#define FDX_LAUNCH_CHECK()                 \
  do {                                     \
    fdx_count_launch();                    \
    FDX_CUDA(cudaPeekAtLastError());       \
  } while (0)

// Encode a tiled TMA descriptor (bf16) through the driver entry point.
// rank <= 5, dims/strides innermost first; strides in BYTES for dims 1..rank-1.
int fdx_make_tmap_bf16(CUtensorMap* map, const void* base, int rank,
                       const uint64_t* dims, const uint64_t* strides_bytes,
                       const uint32_t* box, const uint32_t* elem_strides,
                       int swizzle_128b);

int fdx_num_sms();

// ---------------------------------------------------------------------------
// device-side helpers
// ---------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----- mbarrier -------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(addr),
      "r"(parity)
      : "memory");
}

// ----- TMA ------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// L2 policy for data touched once (evict first): it does not push out lines that other CTAs still read
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void tma_load_4d_hint(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                 int c2, int c3, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(policy)
      : "memory");
}
// Bulk tensor store shared -> global.  The writing threads issue fence_proxy_async_smem() before the barrier
// that precedes it; the source may be rewritten once bulk_wait_group_read shows the store's group has read it.
__device__ __forceinline__ void tma_store_4d_hint(const CUtensorMap* m, const void* src, int c0, int c1, int c2,
                                                  int c3, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group.L2::cache_hint"
      " [%0, {%2, %3, %4, %5}], [%1], %6;" ::"l"(reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(policy)
      : "memory");
}
// bulk async-groups belong to the thread that committed them: only it can wait on them
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----- wgmma ----------------------------------------------------------------------
// One warpgroup (four consecutive warps, the first a multiple of four) computes D(64 x N, f32 registers)
// += A(64 x 16) * B(16 x N), both operands read from shared memory through matrix descriptors.  TA / TB = 1
// selects an MN-major (transposed) operand, 0 a K-major one.  scale_d = 0 ignores D's old contents (D = A * B),
// so the first K step of a product needs no zeroed registers.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t da, uint64_t db, int scale_d = 1) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %20, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, %18, %19;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "n"(TA), "n"(TB), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, int scale_d = 1) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %36, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, %34, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(TA), "n"(TB), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int scale_d = 1) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %68, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, %66, %67;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "n"(TA), "n"(TB), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n192k16(float (&d)[96], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %100, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
      "}, %96, %97, p, 1, 1, %98, %99;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(da), "l"(db), "n"(TA), "n"(TB), "r"(1));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %132, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, %130, %131;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "n"(TA), "n"(TB), "r"(1));
}

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 32 || N == 64 || N == 128 || N == 192 || N == 256, "wgmma_bf16: unsupported N");
  if constexpr (N == 32) wgmma_m64n32k16<TA, TB>(d, da, db);
  else if constexpr (N == 64) wgmma_m64n64k16<TA, TB>(d, da, db);
  else if constexpr (N == 128) wgmma_m64n128k16<TA, TB>(d, da, db);
  else if constexpr (N == 192) wgmma_m64n192k16<TA, TB>(d, da, db);
  else wgmma_m64n256k16<TA, TB>(d, da, db);
}

// ----- GMMA shared-memory descriptors --------------------------------------------
//  [0,14) start>>4  [16,30) LBO>>4  [32,46) SBO>>4  [49,52) base_offset  [62,64) layout (1 = SWIZZLE_128B)
//  K-major, 128B swizzle: rows of 64 bf16 (128 B), SBO = 1024 (8 rows); K advances 16 elements = +32 B.
//  MN-major, 128B swizzle: 64-element MN runs per K row; LBO = byte stride between 64-wide MN blocks,
//  SBO = 1024 (8 K rows); K advances 16 rows = +2048 B.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Warp-specialised kernels with two consumer warpgroups and one producer warpgroup (384 threads): the
// register file is budgeted per warpgroup, so the producer hands its registers to the consumers.
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// arrive without waiting: the other `count` - 32 * (arriving warps) threads wait with named_bar_sync
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ----- warpgroup accumulator ---------------------------------------------------------
// A 128 x WN f32 tile held by one warpgroup as two m64 wgmma fragments (rows 0..63 and 64..127).
// row32() hands each thread one accumulator row (by default row 32 w + l for warp w of the warpgroup, lane l),
// columns [c, c + 32): the one-row-per-thread layout the epilogues work in.  The fragments cross through a 128 x 32 f32 tile
// in shared memory (kAccXchgBytes per warpgroup, 16-byte aligned); every thread of the warpgroup must call
// it with the same c.  Named barrier `bar` (one per warpgroup) orders the exchange.
constexpr int kAccXchgLd = 36;                 // padded row: conflict-free 16-byte row reads
constexpr int kAccXchgBytes = 128 * kAccXchgLd * 4;

template <int WN>
struct WgAcc {
  static_assert(WN == 32 || WN == 64 || WN == 128, "WgAcc: N = 32, 64 or 128");
  float d[2][WN / 2];

  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < WN / 2; ++i) d[h][i] = 0.f;
  }
  // rows 0..63 from da_lo, rows 64..127 from da_hi, all WN columns from db (one K = 16 step)
  template <int TA, int TB>
  __device__ __forceinline__ void mma(uint64_t da_lo, uint64_t da_hi, uint64_t db) {
    wgmma_bf16<WN, TA, TB>(d[0], da_lo, db);
    wgmma_bf16<WN, TA, TB>(d[1], da_hi, db);
  }
  // row < 0: row 32 w + l of the calling thread (warp w of the warpgroup, lane l)
  __device__ __forceinline__ void row32(float* xs, int bar, int c, float (&f)[32], int row = -1) const {
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    if (row < 0) row = w * 32 + l;
    named_bar_sync(bar, 128);                  // the previous chunk's reads of xs are done
#pragma unroll
    for (int cc = 0; cc < WN / 32; ++cc) {
      if (cc == (c >> 5)) {                     // compile-time register indices, run-time chunk
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int r = h * 64 + w * 16 + (l >> 2), col = j * 8 + 2 * (l & 3);
            const float* s = &d[h][(cc * 4 + j) * 4];
            *reinterpret_cast<float2*>(xs + r * kAccXchgLd + col) = make_float2(s[0], s[1]);
            *reinterpret_cast<float2*>(xs + (r + 8) * kAccXchgLd + col) = make_float2(s[2], s[3]);
          }
      }
    }
    named_bar_sync(bar, 128);
    const float4* src = reinterpret_cast<const float4*>(xs + row * kAccXchgLd);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 v = src[j];
      f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
    }
  }
};

// ----- ldmatrix / stmatrix --------------------------------------------------------------
// Four 8 x 8 b16 matrices; lane l gives the shared address of row l % 8 of matrix l / 8.  With .trans, register i
// of lane l holds (or receives) elements (2 (l % 4), l / 4) and (2 (l % 4) + 1, l / 4) of matrix i as stored, so a
// row-major [pixel][channel] tile maps onto the (channel row, pixel pair) layout of a wgmma accumulator fragment.
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// ----- misc ------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(h);
}
// sigmoid(z) = 0.5 * tanh(z / 2) + 0.5 : ONE MUFU op (tanh.approx.f32, rel. error ~2^-11) instead of
// ex2 + rcp; the GroupNorm kernels are MUFU / issue bound, and their outputs are rounded to bf16.
__device__ __forceinline__ float sigmoid_fast(float z) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
  return fmaf(t, 0.5f, 0.5f);
}
__device__ __forceinline__ float silu_f(float z) { return z * sigmoid_fast(z); }

// ---- f32 pairs ---------------------------------------------------------------------------------------
// The streaming GroupNorm kernels work on channel pairs; sm_90 has no packed f32x2 instructions, so each
// pair operation is two scalar f32 operations.
typedef float2 f32x2_t;
__device__ __forceinline__ f32x2_t f2_pack(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void f2_unpack(f32x2_t v, float& lo, float& hi) { lo = v.x; hi = v.y; }
__device__ __forceinline__ f32x2_t f2_fma(f32x2_t a, f32x2_t b, f32x2_t c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ f32x2_t f2_mul(f32x2_t a, f32x2_t b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ f32x2_t f2_add(f32x2_t a, f32x2_t b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ f32x2_t f2_sub(f32x2_t a, f32x2_t b) { return make_float2(a.x - b.x, a.y - b.y); }
// bf16x2 word -> (lo, hi): a shift and a mask
__device__ __forceinline__ f32x2_t f2_from_bf16x2(uint32_t u) {
  return f2_pack(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(f32x2_t v) { return pack_bf16x2(v.x, v.y); }
__device__ __forceinline__ f32x2_t f2_tanh(f32x2_t v) {
  asm("tanh.approx.f32 %0, %0;" : "+f"(v.x));
  asm("tanh.approx.f32 %0, %0;" : "+f"(v.y));
  return v;
}

#endif  // __CUDACC__
