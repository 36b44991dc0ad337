// b200q_gemm.cu — prefill (n_batch > 8) path: wgmma / TMA GEMM for sm_90a (Hopper).
//
//   dst[n][m] (f32, ggml layout dst[n*M + m]) = sum_k W[m][k] * X[n][k]
//
// replaces the reference's quantize_mmq_q8_1 + mul_mat_q<type> (mma.sync m16n8k32 s8, ggml-cuda/mmq.cuh:3849-4173)
// and its dequantize + cublasGemmEx fallback (ggml-cuda.cu:1723-1894).
//
// Every kernel here computes one 128 x BN output tile per CTA (BN = 128 or 256 tokens) with 288 threads:
//   warps 0..7  two consumer warpgroups; warpgroup g owns rows 64g..64g+63 of the tile and accumulates them in registers with
//               wgmma.mma_async m64nBNk16 (bf16) / m64nBNk32 (u8 x s8), both operands K-major in 128-byte-swizzled shared memory
//   warp 8      TMA producer: cp.async.bulk.tensor 2-D loads into STAGES-deep shared-memory rings guarded by full/empty mbarriers
// A comes either from the bf16 scratch written by k_dequant_bf16 (generic types) or is decoded inside the kernel (k_gemm_q, k_gemm_bn_i8).
// With 288 threads and one CTA per SM a thread may hold up to 224 registers: the m64n256 f32 accumulator takes 128 of them.
#include "b200q_internal.h"
#include "b200q_decode_plan.h"
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <mutex>

namespace {

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// warp index broadcast from lane 0: ptxas can then prove that the producer / consumer split is warp-uniform.  With the plain
// threadIdx.x >> 5 it cannot, inserts its own warpgroup arrive on a divergent path and serialises every wgmma (ptxas C7520).
__device__ __forceinline__ int warp_uniform_id() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }
// barrier of the 128 threads of one consumer warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__device__ __forceinline__ void tma_load_2d(void * smem_dst, const CUtensorMap * tm, uint64_t * bar, int x, int y) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tm), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}
// 3-D map (bytes or elements along the row, row, matrix): one map covers all experts of a MoE weight tensor
__device__ __forceinline__ void tma_load_3d(void * smem_dst, const CUtensorMap * tm, uint64_t * bar, int x, int y, int z) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tm), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap * tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)tm) : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator registers across the asynchronous wgmma window
template <typename T, int R> __device__ __forceinline__ void wg_fence_acc(T (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(reinterpret_cast<uint32_t &>(d[i])) :: "memory");
}

// K-major operand tile in smem, rows of 128 bytes, SWIZZLE_128B, 8-row groups 1024 bytes apart
// (sm_90 matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base offset [49,52) = 0 | layout [62,64) = SWIZZLE_128B (1))
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;                 // LBO (ignored for swizzled K-major), canonical value 1
    d |= (uint64_t)(1024 >> 4) << 32;       // SBO: 8 rows * 128 B
    d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
    return d;
}

// D (+)= A[smem desc] * B[smem desc]; m64 x N, the accumulator in registers (fragment layout of the PTX ISA, "wgmma .m64nNk16 D")
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
        ", %64, %65, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
        ", %128, %129, p, 1, 1, 0, 0;\n}\n"
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
        : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_u8s8_n128(uint32_t (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
        ", %64, %65, p;\n}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_u8s8_n256(uint32_t (&d)[128], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k32.s32.u8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
        ", %128, %129, p;\n}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
          "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
          "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
          "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
          "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]),
          "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]),
          "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
          "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]),
          "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(1));
}

// the accumulator type selects the instruction: f32 <- bf16 x bf16 (k16) or s32 <- u8 x s8 (k32); either one reads 32 bytes of K
template <int BN> struct wgmma_op;
template <> struct wgmma_op<128> {
    __device__ __forceinline__ static void mma(float (&d)[64], uint64_t a, uint64_t b) { wgmma_bf16_n128(d, a, b); }
    __device__ __forceinline__ static void mma(uint32_t (&d)[64], uint64_t a, uint64_t b) { wgmma_u8s8_n128(d, a, b); }
};
template <> struct wgmma_op<256> {
    __device__ __forceinline__ static void mma(float (&d)[128], uint64_t a, uint64_t b) { wgmma_bf16_n256(d, a, b); }
    __device__ __forceinline__ static void mma(uint32_t (&d)[128], uint64_t a, uint64_t b) { wgmma_u8s8_n256(d, a, b); }
};

// accumulator element j of thread (warp w of its warpgroup, lane) -> (row, column) of the m64 x N warpgroup tile
__device__ __forceinline__ int acc_row(int w, int lane, int j) { return 16 * w + (lane >> 2) + 8 * ((j >> 1) & 1); }
__device__ __forceinline__ int acc_col(int lane, int j) { return 8 * (j >> 2) + 2 * (lane & 3) + (j & 1); }

constexpr int BM = 128, BK = 64;
constexpr int CONSUMER_WARPS = 8;                 // two warpgroups
constexpr int GEMM_THREADS = 32 * CONSUMER_WARPS + 32;
constexpr int PRODUCER_WARP = CONSUMER_WARPS;

// use i of a STAGES-deep ring of mbarrier-guarded stages: its stage and the parity of that stage's (i / STAGES)-th phase
struct ring_pos { int s; uint32_t ph; };
template <int STAGES> __device__ __forceinline__ ring_pos ring(int i) { return {i % STAGES, (uint32_t)(i / STAGES) & 1u}; }

template <bool GROUPED> __device__ __forceinline__ void tma_load(void * smem_dst, const CUtensorMap * tm, uint64_t * bar, int x, int y, int z) {
    if constexpr (GROUPED) tma_load_3d(smem_dst, tm, bar, x, y, z); else tma_load_2d(smem_dst, tm, bar, x, y);
}

// k-block i of a warpgroup: 4 wgmmas over one 128-byte row of K, each advancing both descriptors by 32 bytes (+2 in 16-byte units) inside the
// swizzle row.  The wait_group<1> completes k-block i - 1, whose B stage (use i - 1 of the `empty` ring) the leader thread then releases.
template <int BN, int STAGES, typename Acc>
__device__ __forceinline__ void mma_kblock(Acc (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr, uint64_t * empty, int i, bool leader) {
    const uint64_t a_desc = make_kmajor_sw128_desc(a_addr), b_desc = make_kmajor_sw128_desc(b_addr);
    wg_fence_acc(acc);
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_op<BN>::mma(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k));
    wg_commit();
    wg_wait<1>();
    wg_fence_acc(acc);
    if (i > 0 && leader) mbar_arrive(&empty[ring<STAGES>(i - 1).s]);
}

// epilogue of a warpgroup's 64 x BN tile (rows from m0): dst[n][m] = value(j, m, n) for m < M, n < n_end, a store or (split-K) an f32 atomic add;
// GROUPED: row n of the expert-sorted operand belongs to slot slot[n], dst[slot[n]][m]
template <int BN, bool GROUPED, typename F>
__device__ __forceinline__ void store_tile(float * __restrict__ dst, int M, int m0, int n0, int n_end, bool atomic, const int * slot, int wl, int lane, F value) {
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) {
        const int m = m0 + acc_row(wl, lane, j), n = n0 + acc_col(lane, j);
        if (m >= M || n >= n_end) continue;
        if constexpr (GROUPED) {
            dst[(size_t)__ldg(slot + n) * M + m] = value(j, m, n);
        } else {
            float * p = dst + (size_t)n * M + m;
            if (atomic) atomicAdd(p, value(j, m, n)); else *p = value(j, m, n);
        }
    }
}

template <int BN> struct gemm_cfg {
    static constexpr int STAGES = BN == 256 ? 4 : 6;
    static constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr size_t SMEM = 1024 /*align slack*/ + (size_t)STAGES * STAGE_BYTES + 256 /*barriers*/;
    static_assert(SMEM <= 227 * 1024, "k_gemm_bf16: shared memory");
};

// MoE prefill (GROUPED): blockIdx.y indexes the tile table of the expert-sorted activation rows (k_moe_route); a tile covers the rows
// [n0, n0 + BN) of ONE expert e, the columns at or past bounds[e + 1] belong to the next expert and are dropped in the epilogue, which stores
// each kept column straight to its slot: dst[slot[n]][m].  CTAs past the device-side tile count return at once.
__device__ __forceinline__ bool moe_tile(const b200q_moe_route & rt, int & e, int & n0, int & n_end) {
    const int tile = __ldg(rt.tile_start + rt.e0) + (int)blockIdx.y;
    if (tile >= __ldg(rt.tile_start + rt.e1)) return false;
    const int2 te = __ldg(rt.tiles + tile);
    e = te.x; n0 = te.y; n_end = __ldg(rt.bounds + e + 1);
    return true;
}

// GROUPED: A is the bf16 scratch of experts e0 .. e1-1 through a 3-D map (k, row, expert - e0)
template <int BN, bool GROUPED = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_bf16(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            float * __restrict__ dst, int M, int N, int K, int k_split, const b200q_moe_route rt) {
    using cfg = gemm_cfg<BN>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char * smem = reinterpret_cast<unsigned char *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t * full_bar  = reinterpret_cast<uint64_t *>(smem + (size_t)cfg::STAGES * cfg::STAGE_BYTES);
    uint64_t * empty_bar = full_bar + cfg::STAGES;

    const int warp = warp_uniform_id(), lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM;
    int n0 = blockIdx.y * BN, e = 0, n_end = N;
    if constexpr (GROUPED) { if (!moe_tile(rt, e, n0, n_end)) return; }
    const int nk_total = (K + BK - 1) / BK;
    const int nk_per = (nk_total + k_split - 1) / k_split;
    const int kb0 = blockIdx.z * nk_per;
    const int kb1 = min(nk_total, kb0 + nk_per);
    const int nk = kb1 - kb0;                                   // may be <= 0 for trailing splits

    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
        tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            for (int i = 0; i < nk; ++i) {
                const auto [s, ph] = ring<cfg::STAGES>(i);
                mbar_wait(&empty_bar[s], ph ^ 1);
                unsigned char * sa = smem + (size_t)s * cfg::STAGE_BYTES; unsigned char * sb = sa + cfg::A_BYTES;
                mbar_expect_tx(&full_bar[s], cfg::STAGE_BYTES);
                tma_load<GROUPED>(sa, &tmA, &full_bar[s], (kb0 + i) * BK, m0, e - rt.e0);
                tma_load_2d(sb, &tmB, &full_bar[s], (kb0 + i) * BK, n0);
            }
        }
        return;
    }
    const int wg = warp >> 2, wl = warp & 3, t = threadIdx.x & 127;
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.0f;
    for (int i = 0; i < nk; ++i) {
        const auto [s, ph] = ring<cfg::STAGES>(i);
        mbar_wait(&full_bar[s], ph);
        const uint32_t stage = smem_u32(smem + (size_t)s * cfg::STAGE_BYTES);
        mma_kblock<BN, cfg::STAGES>(acc, stage + wg * 64 * 128, stage + cfg::A_BYTES, empty_bar, i, t == 0);
    }
    wg_wait<0>();
    wg_fence_acc(acc);
    if (nk <= 0) return;
    store_tile<BN, GROUPED>(dst, M, m0 + 64 * wg, n0, n_end, k_split > 1, rt.slot, wl, lane, [&](int j, int, int) { return acc[j]; });
}

// ---------------------------------------------------------------------------------------------------------------
// Decode GEMMs: the A operand is decoded INSIDE the kernel from the packed weight planes (no bf16 weight scratch in HBM).
//   warp 8      TMA producer: (a) the weight planes of a 128-row raw block (low-bit plane 128 B/row with SWIZZLE_128B, optional
//               scale/meta planes of 16 or 32 B/row) into a 2-deep RAW ring, (b) activation tiles of 128-byte rows into the B ring
//   warps 0..7  thread = (weight row, half of a 128-byte k-block): decode its raw bytes into its 64 bytes of the 128-byte K-major
//               SWIZZLE_128B row of the A stage; the warpgroup that owns the rows then issues the wgmma of that k-block and decodes
//               the next one while it runs
// Pipelines: raw_full/raw_empty (TMA <-> decode), b_full/b_empty (TMA <-> wgmma); the A stages are private to a warpgroup and reused
// after wgmma.wait_group.  Generic-proxy smem writes of the decode are published to the tensor core with fence.proxy.async + bar.sync.
// A raw block is 4 MMA k-blocks; split-K (blockIdx.z) is in units of raw blocks.
//   k_gemm_q      the nine fused types (gemmq_planes), bf16 A = dl*q - ml, 64 k per k-block, split-K and GROUPED (MoE)
//   k_gemm_bn_i8  IQ2_BN on the int8 tensor pipe, u8 A = the 2-bit fields, 128 k per k-block (see gemmbn_policy)
// ---------------------------------------------------------------------------------------------------------------
constexpr int GEMMQ_MAX_SEGS = 3;

// the layout of a decode GEMM's shared memory: A | B | RAW | barriers, all rows 128 bytes; raw planes 0..2 take 128, P1, P2 bytes per row
template <int NB, int B_STAGES_, int P1_, int P2_> struct decode_cfg {
    static constexpr int BN = NB == 0 ? 128 : 256;      // NB = 1: 256 tokens per CTA, NB = 0: 128
    static constexpr int A_STAGES = 2, B_STAGES = B_STAGES_, RAW_STAGES = 2;
    static constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128;
    static constexpr int P1 = P1_, P2 = P2_, N_PLANES = P2 ? 3 : P1 ? 2 : 1;
    static constexpr int RAW_P0 = BM * 128, RAW_P1 = BM * P1, RAW_P2 = BM * P2, RAW_BYTES = RAW_P0 + RAW_P1 + RAW_P2;
    static constexpr size_t SMEM = 1024 + (size_t)A_STAGES * A_BYTES + (size_t)B_STAGES * B_BYTES + (size_t)RAW_STAGES * RAW_BYTES + 256;
    static_assert(SMEM <= 227 * 1024, "decode GEMM: shared memory");
};

// Up to GEMMQ_MAX_SEGS weight tensors that share the activation tile (Q,K,V: the reference's look-ahead fusion,
// ggml-cuda.cu:2573-2601) are covered by ONE launch: blockIdx.x walks the concatenated 128-row tiles of all segments.
struct gemm_decode_seg { float * dst; const float * rs; int M; int tile0; };     // rs: IQ2_BN row scales
// (only the maps of the N_PLANES planes a kernel reads: the arguments are copied at every launch)
template <int N_PLANES> struct gemm_decode_args {
    CUtensorMap tmP[N_PLANES][GEMMQ_MAX_SEGS], tmB;
    gemm_decode_seg seg[GEMMQ_MAX_SEGS];
    int n_seg, N, K, k_split;
    const float * ts; const int * sx;            // IQ2_BN: per-token scale and integer sum of the quantised activations
    b200q_moe_route rt;                          // GROUPED only: the plane maps are 3-D (bytes along the row, row, expert)
};

// The pipeline of both decode GEMMs.  The policy P supplies the shared-memory layout (P::cfg), the k per k-block (P::KB), whether
// split-K and grouping apply (P::SPLIT, P::GROUPED), the accumulator type, the decode of a thread's raw bytes into the 16 words of its
// half A row (a_row) and the epilogue value (value).
template <class P>
__device__ __forceinline__ void gemm_decode(const gemm_decode_args<P::cfg::N_PLANES> & a) {
    using cfg = typename P::cfg;
    constexpr int BN = cfg::BN, KB_PER_RAW = 4;
    int sg = 0;
#pragma unroll
    for (int s = 1; s < GEMMQ_MAX_SEGS; ++s) if (s < a.n_seg && (int)blockIdx.x >= a.seg[s].tile0) sg = s;
    const CUtensorMap * tmB = &a.tmB;
    const gemm_decode_seg seg = a.seg[sg];
    const int M = seg.M, N = a.N, K = a.K, k_split = P::SPLIT ? a.k_split : 1;
    extern __shared__ unsigned char smem_raw[];
    unsigned char * smem = reinterpret_cast<unsigned char *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    unsigned char * sA = smem;
    unsigned char * sB = sA + (size_t)cfg::A_STAGES * cfg::A_BYTES;
    unsigned char * sR = sB + (size_t)cfg::B_STAGES * cfg::B_BYTES;
    uint64_t * bars = reinterpret_cast<uint64_t *>(sR + (size_t)cfg::RAW_STAGES * cfg::RAW_BYTES);
    uint64_t * b_full = bars, * b_empty = b_full + cfg::B_STAGES;
    uint64_t * raw_full = b_empty + cfg::B_STAGES, * raw_empty = raw_full + cfg::RAW_STAGES;

    const int warp = warp_uniform_id(), lane = threadIdx.x & 31;
    const int m0 = ((int)blockIdx.x - seg.tile0) * BM;
    int n0 = blockIdx.y * BN, e = 0, n_end = N;
    if constexpr (P::GROUPED) { if (!moe_tile(a.rt, e, n0, n_end)) return; }
    const int nr_total = (K + KB_PER_RAW * P::KB - 1) / (KB_PER_RAW * P::KB);
    const int nr_per = (nr_total + k_split - 1) / k_split;
    const int rb0 = (P::SPLIT ? (int)blockIdx.z : 0) * nr_per, rb1 = min(nr_total, rb0 + nr_per);
    const int nr = rb1 - rb0;                                   // raw blocks of this CTA (may be <= 0)
    const int kb_begin = rb0 * KB_PER_RAW;
    const int kb_end = min((K + P::KB - 1) / P::KB, rb1 * KB_PER_RAW);
    const int nk = kb_end - kb_begin;                           // MMA k-blocks of this CTA

    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg::B_STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 2); }
        for (int s = 0; s < cfg::RAW_STAGES; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 2); }
        fence_barrier_init();
#pragma unroll
        for (int p = 0; p < cfg::N_PLANES; ++p) tma_prefetch_desc(&a.tmP[p][sg]);
        tma_prefetch_desc(tmB);
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            int ib = 0;
            for (int r = 0; r < nr; ++r) {
                const auto [rs, rph] = ring<cfg::RAW_STAGES>(r);
                mbar_wait(&raw_empty[rs], rph ^ 1);
                unsigned char * raw = sR + (size_t)rs * cfg::RAW_BYTES;
                mbar_expect_tx(&raw_full[rs], cfg::RAW_BYTES);
                tma_load<P::GROUPED>(raw, &a.tmP[0][sg], &raw_full[rs], (rb0 + r) * 128, m0, e);            // bytes along the row
                if constexpr (cfg::N_PLANES > 1) tma_load<P::GROUPED>(raw + cfg::RAW_P0, &a.tmP[1][sg], &raw_full[rs], (rb0 + r) * cfg::P1, m0, e);
                if constexpr (cfg::N_PLANES > 2) tma_load<P::GROUPED>(raw + cfg::RAW_P0 + cfg::RAW_P1, &a.tmP[2][sg], &raw_full[rs], (rb0 + r) * cfg::P2, m0, e);
                for (int q = 0; q < KB_PER_RAW && ib < nk; ++q, ++ib) {
                    const auto [s, ph] = ring<cfg::B_STAGES>(ib);
                    mbar_wait(&b_empty[s], ph ^ 1);
                    mbar_expect_tx(&b_full[s], cfg::B_BYTES);
                    tma_load_2d(sB + (size_t)s * cfg::B_BYTES, tmB, &b_full[s], (kb_begin + ib) * P::KB, n0);
                }
            }
        }
        return;
    }
    // ---------------- consumer warpgroups: decode (thread = row, half of the k-block), then wgmma over the warpgroup's 64 rows ----------------
    const int wg = warp >> 2, wl = warp & 3, t = threadIdx.x & 127;
    const int half = wl >> 1;
    const int row = 64 * wg + 32 * (wl & 1) + lane;              // row of the tile owned by this thread
    const P pol;
    typename P::acc_t acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0;
    int ia = 0;
    for (int r = 0; r < nr; ++r) {
        const auto [rs, rph] = ring<cfg::RAW_STAGES>(r);
        mbar_wait(&raw_full[rs], rph);
        const unsigned char * raw = sR + (size_t)rs * cfg::RAW_BYTES;
        for (int q = 0; q < KB_PER_RAW && ia < nk; ++q, ++ia) {
            unsigned char * sa = sA + (size_t)(ia % cfg::A_STAGES) * cfg::A_BYTES;
            const auto [sb, pb] = ring<cfg::B_STAGES>(ia);
            uint32_t o[16];
            pol.a_row(raw, row, half, q, o);
            // A stage sa was last read by the wgmma of k-block ia - 2, which the wait_group<1> of the previous iteration completed
            unsigned char * arow = sa + (size_t)(row >> 3) * 1024 + (size_t)(row & 7) * 128;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int chunk = (4 * half + c) ^ (row & 7);
                *reinterpret_cast<uint4 *>(arow + chunk * 16) = make_uint4(o[4 * c], o[4 * c + 1], o[4 * c + 2], o[4 * c + 3]);
            }
            fence_proxy_async();                              // make the generic-proxy writes visible to the tensor core
            wg_bar_sync(wg);
            mbar_wait(&b_full[sb], pb);
            mma_kblock<BN, cfg::B_STAGES>(acc, smem_u32(sa) + wg * 64 * 128, smem_u32(sB + (size_t)sb * cfg::B_BYTES), b_empty, ia, t == 0);
        }
        if (t == 0) mbar_arrive(&raw_empty[rs]);              // every thread of the warpgroup has passed the bar.sync after its last read
    }
    wg_wait<0>();
    wg_fence_acc(acc);
    if (nk <= 0) return;
    store_tile<BN, P::GROUPED>(seg.dst, M, m0 + 64 * wg, n0, n_end, k_split > 1, a.rt.slot, wl, lane,
                               [&](int j, int m, int n) { return P::value(a, seg, acc[j], m, n); });
}

// bytes per 256 weights of the planes after the 128-byte low-bit plane (every one a multiple of 16: the inner box of a TMA map)
template <int TYPE> struct gemmq_planes { static constexpr int P1 = 16, P2 = 0; };                    // IQ4_NL / Q4_0 (8 halfs), Q4_K, IQ4_K
template <> struct gemmq_planes<B200Q_TYPE_Q4_1>  { static constexpr int P1 = 32, P2 = 0; };          // {d,m} per item
template <> struct gemmq_planes<B200Q_TYPE_Q5_0>  { static constexpr int P1 = 32, P2 = 16; };         // qh | d
template <> struct gemmq_planes<B200Q_TYPE_Q5_1>  { static constexpr int P1 = 32, P2 = 32; };         // qh | {d,m}
template <> struct gemmq_planes<B200Q_TYPE_Q5_K>  { static constexpr int P1 = 32, P2 = 16; };         // qh | {d,dmin,scales}
template <> struct gemmq_planes<B200Q_TYPE_IQ5_K> { static constexpr int P1 = 32, P2 = 16; };         // qh | {d,extra,scales}

// carry-less per-byte add of two packed int8x4 (the A/B halves of the sign-fill LUT)
__device__ __forceinline__ uint32_t vadd4_wrap(uint32_t a, uint32_t b) {
    return ((a & 0x7f7f7f7fu) + (b & 0x7f7f7f7fu)) ^ ((a ^ b) & 0x80808080u);
}
// signed int8 lane J of a word already XOR-ed with 0x80808080 (biased by +128) -> float(v), exact:
// place the byte under the exponent of 2^23 and subtract 2^23 + 128
template <int J> __device__ __forceinline__ float biased_byte_to_float(uint32_t wb) {
    const uint32_t bits = __byte_perm(wb, 0x4B000000u, 0x7650 + J);       // {byte J, 0x00, 0x00, 0x4B}
    return __uint_as_float(bits) - 8388736.0f;
}

// k_gemm_q: a raw block is 256 weights per row; thread (row, half) decodes 32-weight item 2q + half (PRMT-LUT / mask canonical decode ->
// exact int8->f32 via the 2^23 exponent trick -> bf16(dl*q - ml)).
template <int TYPE, int NB, bool GROUPED_> struct gemmq_policy {
    using cfg = decode_cfg<NB, NB == 0 ? 4 : 3, gemmq_planes<TYPE>::P1, gemmq_planes<TYPE>::P2>;
    using acc_t = float;
    static constexpr int KB = BK;
    static constexpr bool SPLIT = true, GROUPED = GROUPED_;
    const b200q_kv4 T = b200q_kv4_init();
    __device__ __forceinline__ void a_row(const unsigned char * raw, int row, int half, int q, uint32_t (&o)[16]) const {
        b200q_planes SP; SP.p[0] = raw; SP.p[1] = raw + cfg::RAW_P0; SP.p[2] = raw + cfg::RAW_P0 + cfg::RAW_P1; SP.p[3] = SP.p[4] = nullptr; SP.n32 = 8; SP.nb = 1;
        const int it = 2 * q + half;
        b200q_item I; b200q_canon C;
        b200q_load_item<TYPE, b200q_ld_plain, false, int, true>(I, SP, row, it);
        b200q_decode_item<TYPE>(I, it, C, T);
#pragma unroll
        for (int w = 0; w < 8; ++w) {                     // word w = weights 4w..4w+3
            uint32_t v = (uint32_t)C.va[w];
            if (b200q_traits<TYPE>::HAS_B) v = vadd4_wrap(v, (uint32_t)C.vb[w]);
            v ^= 0x80808080u;                             // bias +128 -> unsigned bytes
            const float dl = C.dl[w / 4], ml = C.ml[w / 4];
            const float f0 = fmaf(biased_byte_to_float<0>(v), dl, -ml), f1 = fmaf(biased_byte_to_float<1>(v), dl, -ml);
            const float f2 = fmaf(biased_byte_to_float<2>(v), dl, -ml), f3 = fmaf(biased_byte_to_float<3>(v), dl, -ml);
            __nv_bfloat162 b01 = __floats2bfloat162_rn(f0, f1), b23 = __floats2bfloat162_rn(f2, f3);
            o[2 * w] = *reinterpret_cast<uint32_t *>(&b01); o[2 * w + 1] = *reinterpret_cast<uint32_t *>(&b23);
        }
    }
    template <class A> __device__ __forceinline__ static float value(const A &, const gemm_decode_seg &, float acc, int, int) { return acc; }
};

// ---------------------------------------------------------------------------------------------------------------
// Ternary prefill on the INT8 tensor pipe: IQ2_BN (bitnet b1.58) weights x per-token int8 activations -> s32 accumulators.
// (The reference has no integer tensor-core path for this type: its prefill is dequantize_block_iq2_bn + cublasGemmEx in f16 with
//  f16 accumulation, ggml-cuda.cu:1723-1894, SURVEY §8 a13.)
//   A: the 2-bit fields q in {0,1,2} of the wire blocks are expanded to UNSIGNED int8 in the K-major SWIZZLE_128B A stage (128 rows x 128 k
//      = 128 bytes per row: one shift + mask per 4 weights, no table, no scale); w = rs * (q - 1) is applied in the epilogue:
//      dst[n][m] = rs[m] * ts[n] * (acc[m][n] - S[n]),  acc = sum_k q[m][k] * xq[n][k]  (wgmma m64nNk32 u8 x s8 -> s32, exact),
//      S[n] = sum_k xq[n][k] and ts[n] = amax_n / 127 come from the activation quantiser (k_quantize_rows_i8).
//   B: int8 activations [N][K], TMA (SWIZZLE_128B, 128 k = 128 bytes per row), one per-TOKEN scale: the whole K reduction is integer.
//   Zero-filled TMA tails make any K % 64 == 0 work (bitnet: K = 3200, 8640): q = 0 and xq = 0 beyond K contribute nothing, S[n] covers real k only.
// A raw block is 512 weights per row (128 bytes of 2-bit fields); no split-K, no grouping.
// Accuracy: activations rounded to 8 bits per token (NMSE ~1e-4 for Gaussian activations; the reference's own q8_1 decode path: ~2e-5, its f16-accumulate
// prefill: ~1e-6 + f16 overflow risk); weights exact.  Tolerance in tests/test_gpu_parity.py: NMSE <= 5e-4 (the reference's test bar).
// ---------------------------------------------------------------------------------------------------------------
template <int NB> struct gemmbn_policy {
    using cfg = decode_cfg<NB, 3, 0, 0>;
    using acc_t = uint32_t;
    static constexpr int KB = 128;
    static constexpr bool SPLIT = false, GROUPED = false;
    __device__ __forceinline__ void a_row(const unsigned char * raw, int row, int half, int q, uint32_t (&o)[16]) const {
        // wire block (64 weights, 16 bytes) number 2q + half of this raw row; SWIZZLE_128B: 16-byte chunk c sits at c ^ (row & 7)
        const uint4 wv = *reinterpret_cast<const uint4 *>(raw + (size_t)row * 128 + (((2 * q + half) ^ (row & 7)) << 4));
        const uint32_t w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
        for (int f = 0; f < 4; ++f)                       // field f of byte j = weight 16 f + j of the block: one 16-byte chunk of 16 consecutive k
#pragma unroll
            for (int i = 0; i < 4; ++i) o[4 * f + i] = (w[i] >> (2 * f)) & 0x03030303u;
    }
    template <class A> __device__ __forceinline__ static float value(const A & a, const gemm_decode_seg & seg, uint32_t acc, int m, int n) {
        return __ldg(seg.rs + m) * __ldg(a.ts + n) * (float)((int)acc - __ldg(a.sx + n));
    }
};

template <int TYPE, int NB, bool GROUPED = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_q(const __grid_constant__ gemm_decode_args<gemmq_policy<TYPE, NB, GROUPED>::cfg::N_PLANES> a) { gemm_decode<gemmq_policy<TYPE, NB, GROUPED>>(a); }

template <int NB>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_bn_i8(const __grid_constant__ gemm_decode_args<1> a) { gemm_decode<gemmbn_policy<NB>>(a); }

// f32 [N][K] (row stride xs) -> int8 [N][K] with ONE scale per token: q = rint(x * 127 / amax_n); ts[n] = amax_n / 127; sx[n] = sum_k q
__global__ void __launch_bounds__(256) k_quantize_rows_i8(const float * __restrict__ x, int64_t xs, int8_t * __restrict__ q, float * __restrict__ ts, int * __restrict__ sx, int64_t K) {
    const int64_t n = blockIdx.x; const float * xr = x + n * xs; int8_t * qr = q + n * K;
    __shared__ float s_amax[8]; __shared__ int s_sum[8];
    float amax = 0.0f;
    for (int64_t k = threadIdx.x * 4; k < K; k += blockDim.x * 4) { const float4 v = *reinterpret_cast<const float4 *>(xr + k); amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)))); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) s_amax[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = s_amax[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, s_amax[i]);
    const float d = __fdiv_rn(amax, 127.0f), inv = d > 0.0f ? __frcp_rn(d) : 0.0f;
    int sum = 0;
    for (int64_t k = threadIdx.x * 4; k < K; k += blockDim.x * 4) {
        const float4 v = *reinterpret_cast<const float4 *>(xr + k);
        const int a = max(-127, min(127, __float2int_rn(v.x * inv))), b = max(-127, min(127, __float2int_rn(v.y * inv)));
        const int c = max(-127, min(127, __float2int_rn(v.z * inv))), e = max(-127, min(127, __float2int_rn(v.w * inv)));
        sum += a + b + c + e;
        *reinterpret_cast<uint32_t *>(qr + k) = (uint32_t)(a & 0xff) | ((uint32_t)(b & 0xff) << 8) | ((uint32_t)(c & 0xff) << 16) | ((uint32_t)(e & 0xff) << 24);
    }
    sum = __reduce_add_sync(0xffffffffu, sum);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) { int t = 0; for (int i = 0; i < 8; ++i) t += s_sum[i]; sx[n] = t; ts[n] = d; }
}

// dst = act(clamp(gate)) * clamp(up) elementwise (the reference's ggml_fused_mul_unary after two MMQs, ggml-cuda.cu:3588-3618);
// gate may alias dst; optional bf16 copy for the following MUL_MAT
__global__ void k_mul_unary(const float * gate /* may alias dst: no __restrict__ */, const float * __restrict__ up, float * dst, __nv_bfloat16 * __restrict__ dst_bf,
                            int64_t total4, int act, float lim) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 g = reinterpret_cast<const float4 *>(gate)[i]; float4 u = reinterpret_cast<const float4 *>(up)[i];
        float4 r; r.x = b200q_glu<true>(act, g.x, u.x, lim); r.y = b200q_glu<true>(act, g.y, u.y, lim); r.z = b200q_glu<true>(act, g.z, u.z, lim); r.w = b200q_glu<true>(act, g.w, u.w, lim);
        reinterpret_cast<float4 *>(dst)[i] = r;
        if (dst_bf != nullptr) {
            __nv_bfloat162 b0 = __floats2bfloat162_rn(r.x, r.y), b1 = __floats2bfloat162_rn(r.z, r.w);
            uint2 o; o.x = *reinterpret_cast<uint32_t *>(&b0); o.y = *reinterpret_cast<uint32_t *>(&b1);
            reinterpret_cast<uint2 *>(dst_bf)[i] = o;
        }
    }
}

// f32 [N][K] (row stride xs) -> bf16 [N][K].  HBM-bound glue between the GEMMs (12 MB per 512 x 4096 activation): a thread converts 8 consecutive
// values (two LDG.128 -> one STG.128) and keeps U such groups in flight, so that enough loads are outstanding to approach HBM bandwidth.
// MAP (MoE gather): output row n reads activation column c = row_map[n] = t * nb1 + j, at x + t * xs + j * xs_col; a negative entry (past the
// routed rows) gives a zero row.
template <bool MAP = false>
__global__ void __launch_bounds__(256) k_f32_to_bf16(const float * __restrict__ x, int64_t xs, __nv_bfloat16 * __restrict__ out, int64_t K, int64_t N,
                                                     const int * __restrict__ row_map = nullptr, int nb1 = 1, int64_t xs_col = 0) {
    constexpr int U = 4;
    const int64_t k8 = K / 8, total8 = N * k8, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < total8; i0 += U * stride) {
        float4 a[U], b[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int64_t i = i0 + u * stride;
            if (i < total8) {
                const int64_t n = i / k8, c = i % k8;
                const int64_t src = MAP ? (int64_t)__ldg(row_map + n) : n;
                if (MAP && src < 0) { a[u] = b[u] = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
                const int64_t off = MAP ? (src / nb1) * xs + (src % nb1) * xs_col : src * xs;
                const float4 * p = reinterpret_cast<const float4 *>(x + off + 8 * c); a[u] = __ldg(p); b[u] = __ldg(p + 1);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int64_t i = i0 + u * stride;
            if (i < total8) {
                __nv_bfloat162 p0 = __floats2bfloat162_rn(a[u].x, a[u].y), p1 = __floats2bfloat162_rn(a[u].z, a[u].w), p2 = __floats2bfloat162_rn(b[u].x, b[u].y), p3 = __floats2bfloat162_rn(b[u].z, b[u].w);
                uint4 o; o.x = *reinterpret_cast<uint32_t *>(&p0); o.y = *reinterpret_cast<uint32_t *>(&p1); o.z = *reinterpret_cast<uint32_t *>(&p2); o.w = *reinterpret_cast<uint32_t *>(&p3);
                const int64_t n = i / k8, c = i % k8;
                *reinterpret_cast<uint4 *>(out + n * K + 8 * c) = o;
            }
        }
    }
}
// K % 8 != 0 (K % 4 == 0): the simple version
__global__ void k_f32_to_bf16_k4(const float * __restrict__ x, int64_t xs, __nv_bfloat16 * __restrict__ out, int64_t K, int64_t N) {
    const int64_t total4 = N * (K / 4);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = i / (K / 4), k4 = i % (K / 4);
        const float4 v = *reinterpret_cast<const float4 *>(x + n * xs + 4 * k4);
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 u; u.x = *reinterpret_cast<uint32_t *>(&a); u.y = *reinterpret_cast<uint32_t *>(&b);
        *reinterpret_cast<uint2 *>(out + n * K + 4 * k4) = u;
    }
}

// f16 [N][K] (row stride xs halves) -> OUT [N][K] (bf16, or f32 to widen), E = 8 halves per item (one 16-byte load, one 16-byte bf16 store or two
// f32 ones) or, for K % 8 != 0, 4.  Both outputs are exact images of float(x): widening f16 is exact, and bf16(f16) rounds the same real value as
// bf16(f32(f16)), so the products that follow give the bits of the same call over f32 activations holding float(x).
template <typename OUT, int E>
__global__ void __launch_bounds__(256) k_f16_convert(const __half * __restrict__ x, int64_t xs, OUT * __restrict__ out, int64_t K, int64_t N) {
    using V = typename std::conditional<E == 8, uint4, uint2>::type;
    const int64_t ke = K / E, total = N * ke;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = i / ke, c = i % ke;
        const V v = __ldg(reinterpret_cast<const V *>(x + n * xs + E * c));
        const uint32_t * w = reinterpret_cast<const uint32_t *>(&v);
        float f[E];
#pragma unroll
        for (int j = 0; j < E / 2; ++j) { const float2 t = __half22float2(*reinterpret_cast<const __half2 *>(w + j)); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
        OUT * o = out + n * K + E * c;
        if constexpr (std::is_same<OUT, float>::value) {
#pragma unroll
            for (int q = 0; q < E / 4; ++q) reinterpret_cast<float4 *>(o)[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
        } else {
            V r; uint32_t * rw = reinterpret_cast<uint32_t *>(&r);
#pragma unroll
            for (int j = 0; j < E / 2; ++j) { const __nv_bfloat162 b = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]); rw[j] = *reinterpret_cast<const uint32_t *>(&b); }
            *reinterpret_cast<V *>(o) = r;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side: tensor maps
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
encode_tiled_fn get_encode() {
    static encode_tiled_fn fn = nullptr; static std::once_flag once;
    std::call_once(once, [] {
        void * p = nullptr; cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (encode_tiled_fn)p;
    });
    return fn;
}
// row-major tensor of rank 2 or 3: dims innermost first (elements), byte strides of the outer dimensions, box (elements); 128B swizzle or none.
// Out-of-range elements of a box are zero-filled.
int make_tmap(CUtensorMap * tm, CUtensorMapDataType type, int rank, const void * ptr, const int64_t (&dims)[3], const int64_t (&strides)[2],
              const int (&box)[3], bool swizzle128) {
    encode_tiled_fn enc = get_encode(); if (!enc) return -1;
    cuuint64_t gd[3], gs[2]; cuuint32_t bx[3], estr[3] = {1, 1, 1};
    for (int i = 0; i < 3; ++i) { gd[i] = (cuuint64_t)dims[i]; bx[i] = (cuuint32_t)box[i]; }
    for (int i = 0; i < 2; ++i) gs[i] = (cuuint64_t)strides[i];
    CUresult r = enc(tm, type, (cuuint32_t)rank, const_cast<void *>(ptr), gd, gs, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}
constexpr CUtensorMapDataType TM_BF16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, TM_U8 = CU_TENSOR_MAP_DATA_TYPE_UINT8;

// activation row tiles on blockIdx.y; GROUPED: an upper bound of the tiles of n_mat experts, each expert's last tile may be partial
template <int BN, bool GROUPED> unsigned row_tiles(int64_t N, int64_t n_mat) {
    return (unsigned)((N + BN - 1) / BN + (GROUPED ? std::min<int64_t>(n_mat, N) : 0));
}

// dst f32 [N][M] = A bf16 [M][K] x B bf16 [N][K]; GROUPED: A holds n_mat experts [n_mat][a_rows][K], those of rt.e0 .. rt.e1-1, and the product
// reads the first M rows of each (A_bf16 may point at a later row of expert 0: a row range of every expert)
template <int BN, bool GROUPED>
int launch_gemm_bf16(const void * A_bf16, int64_t n_mat, int64_t a_rows, const void * B_bf16, float * dst, int64_t M, int64_t N, int64_t K, int k_split,
                     const b200q_moe_route & rt, cudaStream_t st) {
    using cfg = gemm_cfg<BN>;
    CUtensorMap tmA, tmB;
    if (make_tmap(&tmA, TM_BF16, GROUPED ? 3 : 2, A_bf16, {K, M, n_mat}, {K * 2, a_rows * K * 2}, {64, BM, 1}, true)) return -10;
    if (make_tmap(&tmB, TM_BF16, 2, B_bf16, {K, N}, {K * 2}, {64, BN}, true)) return -11;
    if (!b200q_opt_in_smem((const void *)k_gemm_bf16<BN, GROUPED>, cfg::SMEM)) return -12;
    dim3 grid((unsigned)((M + BM - 1) / BM), row_tiles<BN, GROUPED>(N, n_mat), (unsigned)k_split);
    k_gemm_bf16<BN, GROUPED><<<grid, GEMM_THREADS, cfg::SMEM, st>>>(tmA, tmB, dst, (int)M, (int)N, (int)K, k_split, rt);
    return (int)cudaGetLastError();
}

// types whose plane 0 is 16 B / item of low bits and whose other planes are 16 or 32 B per 256 weights (gemmq_planes): the weight slab is decoded
// inside the GEMM.  (Q6_K / Q6_0 / Q8_0 would not fit the shared memory next to a 256-token B tile, Q3_K / IQ2_K / *_KS have planes that are not a
// multiple of 16 bytes per 256 weights: those keep the bf16 scratch.)
#define GEMMQ_TYPES(X) X(B200Q_TYPE_IQ4_NL) X(B200Q_TYPE_Q4_0) X(B200Q_TYPE_Q4_K) X(B200Q_TYPE_IQ4_K) \
                       X(B200Q_TYPE_Q4_1) X(B200Q_TYPE_Q5_0) X(B200Q_TYPE_Q5_1) X(B200Q_TYPE_Q5_K) X(B200Q_TYPE_IQ5_K)
constexpr bool gemmq_supported(int type) {
#define X(T) type == T ||
    return GEMMQ_TYPES(X) false;
#undef X
}

// k_gemm_q over the segments of d.  GROUPED: d.W[i] holds n_mat expert matrices (one 3-D map per plane covers them all) and blockIdx.y walks
// the tile table of rt.  Segment i is the row range [d.row0[i], d.row0[i] + d.M[i]) of matrices of d.rows_layout rows (merged up/gate experts, a
// row slice of a dense weight): its maps start at that row and end after d.M[i] rows, so a partial last tile is zero-filled, not the next range
template <int TYPE, int NB, bool GROUPED>
int launch_gemm_q(const b200q_gemm_multi & d, int k_split, int64_t n_mat, const b200q_moe_route & rt, cudaStream_t st) {
    using cfg = typename gemmq_policy<TYPE, NB, GROUPED>::cfg;
    gemm_decode_args<cfg::N_PLANES> a; memset(&a, 0, sizeof a);
    const int box[3] = {128, cfg::P1, cfg::P2};                   // bytes per row of each plane per 256 weights
    int tiles = 0;
    for (int i = 0; i < d.n_seg; ++i) {
        b200q_layout L; if (b200q_make_layout(TYPE, d.rows_layout ? d.rows_layout : d.M[i], d.K, &L)) return -1;
        for (int p = 0; p < cfg::N_PLANES; ++p) {
            const int64_t row_bytes = (d.K / 256) * box[p];
            const char * base = (const char *)d.W[i] + L.plane_off[p] + b200q_row_offset(L, p, d.row0[i]);
            if (make_tmap(&a.tmP[p][i], TM_U8, GROUPED ? 3 : 2, base, {row_bytes, d.M[i], n_mat},
                                    {row_bytes, L.total_bytes}, {box[p], BM, 1}, p == 0)) return p == 0 ? -10 : -13;
        }
        a.seg[i].dst = d.dst[i]; a.seg[i].M = (int)d.M[i]; a.seg[i].tile0 = tiles;
        tiles += (int)((d.M[i] + BM - 1) / BM);
    }
    if (make_tmap(&a.tmB, TM_BF16, 2, d.xb, {d.K, d.N}, {d.K * 2}, {64, cfg::BN}, true)) return -11;
    a.n_seg = d.n_seg; a.N = (int)d.N; a.K = (int)d.K; a.k_split = k_split; a.rt = rt;
    if (!b200q_opt_in_smem((const void *)k_gemm_q<TYPE, NB, GROUPED>, cfg::SMEM)) return -12;
    dim3 grid((unsigned)tiles, row_tiles<cfg::BN, GROUPED>(d.N, n_mat), (unsigned)k_split);
    k_gemm_q<TYPE, NB, GROUPED><<<grid, GEMM_THREADS, cfg::SMEM, st>>>(a);
    return (int)cudaGetLastError();
}
template <bool GROUPED>
int launch_gemm_q(int type, bool bn256, const b200q_gemm_multi & d, int k_split, int64_t n_mat, const b200q_moe_route & rt, cudaStream_t st) {
    switch (type) {
#define X(T) case T: return bn256 ? launch_gemm_q<T, 1, GROUPED>(d, k_split, n_mat, rt, st) : launch_gemm_q<T, 0, GROUPED>(d, k_split, n_mat, rt, st);
        GEMMQ_TYPES(X)
#undef X
        default: return -1;
    }
}

// IQ2_BN planes of d x int8 activations xq [N][K] (per-token scale ts, sum sx)
template <int NB>
int launch_gemm_bn_i8(const b200q_gemm_multi & d, const int8_t * xq, const float * ts, const int * sx, cudaStream_t st) {
    using cfg = typename gemmbn_policy<NB>::cfg;
    gemm_decode_args<1> a; memset(&a, 0, sizeof a);
    int tiles = 0;
    for (int i = 0; i < d.n_seg; ++i) {
        b200q_layout L; if (b200q_slice_layout(B200Q_TYPE_IQ2_BN, d.rows_layout ? d.rows_layout : d.M[i], d.row0[i], d.M[i], d.K, &L)) return -1;
        if (make_tmap(&a.tmP[0][i], TM_U8, 2, (const char *)d.W[i] + L.plane_off[0], {d.K / 4, d.M[i]}, {d.K / 4}, {128, BM}, true)) return -10;
        a.seg[i].dst = d.dst[i]; a.seg[i].rs = reinterpret_cast<const float *>((const char *)d.W[i] + L.plane_off[1]); a.seg[i].M = (int)d.M[i]; a.seg[i].tile0 = tiles;
        tiles += (int)((d.M[i] + BM - 1) / BM);
    }
    if (make_tmap(&a.tmB, TM_U8, 2, xq, {d.K, d.N}, {d.K}, {128, cfg::BN}, true)) return -11;
    a.ts = ts; a.sx = sx; a.n_seg = d.n_seg; a.N = (int)d.N; a.K = (int)d.K; a.k_split = 1;
    if (!b200q_opt_in_smem((const void *)k_gemm_bn_i8<NB>, cfg::SMEM)) return -12;
    dim3 grid((unsigned)tiles, row_tiles<cfg::BN, false>(d.N, 1), 1);
    k_gemm_bn_i8<NB><<<grid, GEMM_THREADS, cfg::SMEM, st>>>(a);
    return (int)cudaGetLastError();
}

// split-K factor of the fused kernel: minimise waves x (raw blocks per CTA + fixed cost), the fixed cost (pipeline fill,
// epilogue) being worth ~4 raw blocks; split-K pays memset + f32 atomics
int gemmq_choose_split(int64_t tiles, int64_t nr, int sm_count) {
    static const int forced = [] { const char * e = getenv("B200Q_GEMM_SPLIT"); return e ? atoi(e) : 0; }();      // experiments only
    if (forced > 0) return forced <= nr ? forced : (int)nr;
    int best = 1; int64_t best_cost = INT64_MAX;
    for (int ks = 1; ks <= 16 && ks <= nr; ++ks) {
        const int64_t per = (nr + ks - 1) / ks;
        if (ks > 1 && per * (ks - 1) >= nr) continue;                 // an empty split
        const int64_t waves = (tiles * ks + sm_count - 1) / sm_count;
        const int64_t cost = waves * (per + 4) + (ks > 1 ? 2 : 0);
        if (cost < best_cost) { best_cost = cost; best = ks; }
    }
    return best;
}

}  // namespace


// IQ2_BN prefill on the int8 tensor pipe.  X f32 [N][K] is quantised per token into `ws` (int8 [N][K] | ts[N] | sx[N]); up to 3 tensors share it.
// Eligible shapes (b200q_gemm_bn_i8_ok): K % 64 == 0 (16-byte TMA strides), 16-byte aligned rows of x; callers take the bf16 path for the others.
size_t b200q_gemm_i8_workspace_bytes(int64_t K, int64_t N) { return (size_t)b200q_align_up(N * K, 256) + (size_t)b200q_align_up(N * 8, 256); }
bool b200q_gemm_bn_i8_ok(int type, int64_t K, int64_t N, const float * x, int64_t x_stride, size_t ws_bytes) {
    const int64_t xs = x_stride ? x_stride : K;
    return type == B200Q_TYPE_IQ2_BN && K % 64 == 0 && N >= 1 && !((uintptr_t)x & 15) && !(xs & 3) && ws_bytes >= b200q_gemm_i8_workspace_bytes(K, N);
}
int b200q_launch_gemm_bn_i8(const b200q_gemm_multi & d, const float * x, int64_t x_stride, void * ws, size_t ws_bytes, cudaStream_t st) {
    if (!b200q_gemm_bn_i8_ok(d.type, d.K, d.N, x, x_stride, ws_bytes) || d.n_seg < 1 || d.n_seg > GEMMQ_MAX_SEGS) return -2;
    const int64_t xs = x_stride ? x_stride : d.K;
    int8_t * xq = (int8_t *)ws; float * ts = (float *)((char *)ws + b200q_align_up(d.N * d.K, 256)); int * sx = (int *)(ts + d.N);
    k_quantize_rows_i8<<<(unsigned)d.N, 256, 0, st>>>(x, xs, xq, ts, sx, d.K);
    cudaError_t e = cudaGetLastError(); if (e != cudaSuccess) return (int)e;
    return d.N > 128 ? launch_gemm_bn_i8<1>(d, xq, ts, sx, st) : launch_gemm_bn_i8<0>(d, xq, ts, sx, st);
}

// dst[j][i] = a[j][i] + b[j % nb][i]  (GGML_OP_ADD of a mat-mul result with a bias row / a same-shape tensor, when it is NOT fused into the mat-vec).
// dst may be a or b (an in-place ADD of ggml's allocator): no __restrict__ on the operands
__global__ void k_add_rows(const float * a, const float * b, float * dst, int64_t m, int64_t n, int64_t nb) {
    const int64_t total = m * n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) dst[i] = a[i] + b[((i / m) % nb) * m + i % m];
}
int b200q_launch_add_rows(const float * a, const float * b, float * dst, int64_t m, int64_t n, int64_t nb, cudaStream_t st) {
    if (m < 1 || n < 1 || nb < 1) return -2;
    int64_t g = (m * n + 255) / 256; if (g > 132 * 16) g = 132 * 16;
    k_add_rows<<<(unsigned)g, 256, 0, st>>>(a, b, dst, m, n, nb);
    return (int)cudaGetLastError();
}

// elementwise tail of GGML_OP_FUSED_UP_GATE for n > 8
int b200q_launch_mul_unary(const float * gate, const float * up, float * dst, void * dst_bf16, int64_t total, int act, float limit, cudaStream_t st) {
    if (total % 4) return -2;
    int64_t nb = (total / 4 + 255) / 256; if (nb > 132 * 16) nb = 132 * 16; if (nb < 1) nb = 1;
    k_mul_unary<<<(unsigned)nb, 256, 0, st>>>(gate, up, dst, (__nv_bfloat16 *)dst_bf16, total / 4, act, limit);
    return (int)cudaGetLastError();
}

b200q_dense_ws b200q_dense_layout(int kind, int64_t M, int64_t K, int64_t N) {
    b200q_dense_ws L{}; size_t off = 0;
    auto take = [&](int64_t bytes) { const size_t o = off; off += (size_t)b200q_align_up(bytes, 256); return o; };
    if (kind == B200Q_DENSE_GEMM_WIDEN) L.xf = take(N * K * 4);
    if (kind == B200Q_DENSE_GEMM || kind == B200Q_DENSE_GEMM_WIDEN || kind == B200Q_DENSE_UP_GATE) L.x = take(N * K * 2);
    if (kind >= B200Q_DENSE_UP_GATE) L.up = take(M * N * 4);
    if (kind == B200Q_DENSE_UP_GATE_I8) L.x = take((int64_t)b200q_gemm_i8_workspace_bytes(K, N));
    else L.wsc = take(M * K * 2);
    L.total = off;
    return L;
}
size_t b200q_gemm_workspace_bytes(int type, int64_t M, int64_t K, int64_t N) {
    (void)type;
    return b200q_dense_layout(B200Q_DENSE_GEMM, M, K, N).total;
}

// f32 [N][K] -> bf16 [N][K] (shared by the mat-muls that consume the same activation)
int b200q_launch_f32_to_bf16(const float * x, int64_t x_stride, void * out, int64_t K, int64_t N, cudaStream_t st) {
    if (K % 4) return -2;
    const int64_t xs = x_stride ? x_stride : K;
    if (K % 8 == 0 && xs % 4 == 0 && !((uintptr_t)x & 15) && !((uintptr_t)out & 15)) {
        const int64_t total8 = N * (K / 8); int64_t nb = (total8 + 256 * 4 - 1) / (256 * 4); if (nb > 132 * 8) nb = 132 * 8; if (nb < 1) nb = 1;
        k_f32_to_bf16<false><<<(unsigned)nb, 256, 0, st>>>(x, xs, (__nv_bfloat16 *)out, K, N);
    } else {
        const int64_t total4 = N * (K / 4); int64_t nb = (total4 + 255) / 256; if (nb > 132 * 32) nb = 132 * 32; if (nb < 1) nb = 1;
        k_f32_to_bf16_k4<<<(unsigned)nb, 256, 0, st>>>(x, xs, (__nv_bfloat16 *)out, K, N);
    }
    return (int)cudaGetLastError();
}

int b200q_launch_f16_convert(const void * x, int64_t x_stride, void * out, int to_bf16, int64_t K, int64_t N, cudaStream_t st) {
    const int64_t xs = x_stride ? x_stride : K;
    if (K % 4 || xs % 4 || ((uintptr_t)x & 7) || ((uintptr_t)out & 7)) return -2;
    const bool e8 = K % 8 == 0 && xs % 8 == 0 && !((uintptr_t)x & 15) && !((uintptr_t)out & 15);
    const int64_t total = N * (K / (e8 ? 8 : 4)); int64_t nb = (total + 255) / 256; if (nb > 132 * 32) nb = 132 * 32; if (nb < 1) nb = 1;
    const __half * h = (const __half *)x;
    if (to_bf16) {
        if (e8) k_f16_convert<__nv_bfloat16, 8><<<(unsigned)nb, 256, 0, st>>>(h, xs, (__nv_bfloat16 *)out, K, N);
        else k_f16_convert<__nv_bfloat16, 4><<<(unsigned)nb, 256, 0, st>>>(h, xs, (__nv_bfloat16 *)out, K, N);
    } else {
        if (e8) k_f16_convert<float, 8><<<(unsigned)nb, 256, 0, st>>>(h, xs, (float *)out, K, N);
        else k_f16_convert<float, 4><<<(unsigned)nb, 256, 0, st>>>(h, xs, (float *)out, K, N);
    }
    return (int)cudaGetLastError();
}

// n_seg weight tensors of one type and K sharing X = bf16 [N][K] (already converted); dst[i] f32 [N][M_i].
// wscratch: bf16 W scratch (max M_i x K) for the unfused path.
int b200q_launch_gemm_multi_bf16x(const b200q_gemm_multi & d, void * wscratch, size_t ws_bytes, int sm_count, int fused, cudaStream_t st) {
    if (d.K % 8) return -2;
    if (d.n_seg < 1 || d.n_seg > GEMMQ_MAX_SEGS) return -2;
    const int type = d.type; const int64_t K = d.K, N = d.N;
    const bool use_fused = fused && gemmq_supported(type) && K % 256 == 0;
    if (use_fused) {
        // one CTA dequantises a 128-row block once for up to 256 tokens (the register accumulators of two m64n256 warpgroups);
        // split-K (f32 atomics) fills the SMs when there are few row blocks
        const bool bn256 = N > 128;
        const int bn = bn256 ? 256 : 128;
        int64_t mt = 0; for (int i = 0; i < d.n_seg; ++i) mt += (d.M[i] + BM - 1) / BM;
        const int64_t tiles = mt * ((N + bn - 1) / bn);
        const int k_split = gemmq_choose_split(tiles, K / 256, sm_count);
        if (k_split > 1) for (int i = 0; i < d.n_seg; ++i) { cudaError_t e = cudaMemsetAsync(d.dst[i], 0, (size_t)d.M[i] * N * sizeof(float), st); if (e != cudaSuccess) return -3; }
        return launch_gemm_q<false>(type, bn256, d, k_split, 1, b200q_moe_route{}, st);
    }
    // unfused: bf16 weight scratch + plain bf16 GEMM per tensor; tile / split selection: fill ~1 wave of the SMs.
    // Every segment's type and scratch size is checked before the first memset or launch: an error return leaves every dst untouched.
    // (a row slice dequantises only its own rows: its layout's plane offsets start at row0)
    b200q_layout Ls[GEMMQ_MAX_SEGS];
    for (int i = 0; i < d.n_seg; ++i) {
        if (b200q_slice_layout(type, d.rows_layout ? d.rows_layout : d.M[i], d.row0[i], d.M[i], K, &Ls[i])) return -1;
        if (ws_bytes < b200q_dense_layout(B200Q_DENSE_GEMM_BF16, d.M[i], K, N).total) return -5;
    }
    for (int i = 0; i < d.n_seg; ++i) {
        const int64_t M = d.M[i];
        const b200q_layout & L = Ls[i];
        const int64_t mt = (M + BM - 1) / BM;
        const bool bn256 = N >= 256 && mt * ((N + 255) / 256) >= sm_count / 2;
        const int64_t tiles = bn256 ? mt * ((N + 255) / 256) : mt * ((N + 127) / 128);
        int k_split = 1;
        const int64_t nk = (K + BK - 1) / BK;
        while (tiles * k_split * 2 <= sm_count && k_split * 2 <= 8 && nk / (k_split * 2) >= 8) k_split *= 2;
        if (k_split > 1) { cudaError_t e = cudaMemsetAsync(d.dst[i], 0, (size_t)M * N * sizeof(float), st); if (e != cudaSuccess) return -3; }
        int rc = b200q_launch_dequant_bf16(d.W[i], L, wscratch, st); if (rc) return rc;
        rc = bn256 ? launch_gemm_bf16<256, false>(wscratch, 1, M, d.xb, d.dst[i], M, N, K, k_split, b200q_moe_route{}, st)
                   : launch_gemm_bf16<128, false>(wscratch, 1, M, d.xb, d.dst[i], M, N, K, k_split, b200q_moe_route{}, st);
        if (rc) return rc;
    }
    return 0;
}

int b200q_gemm_fused_type(int type) { return gemmq_supported(type) ? 1 : 0; }

// MoE gather: bf16 [N][K] whose row n is activation column row_map[n] of x (see b200q_internal.h); a negative entry gives a zero row
int b200q_launch_f32_to_bf16_rows(const float * x, const int * row_map, int nb1, int64_t x_tok_stride, int64_t x_col_stride, void * out, int64_t K, int64_t N,
                                  cudaStream_t st) {
    if (K % 8 || nb1 < 1 || (x_tok_stride | x_col_stride) & 3 || ((uintptr_t)x & 15) || ((uintptr_t)out & 15)) return -2;
    const int64_t total8 = N * (K / 8); int64_t nb = (total8 + 256 * 4 - 1) / (256 * 4); if (nb > 132 * 8) nb = 132 * 8; if (nb < 1) nb = 1;
    k_f32_to_bf16<true><<<(unsigned)nb, 256, 0, st>>>(x, x_tok_stride, (__nv_bfloat16 *)out, K, N, row_map, nb1, x_col_stride);
    return (int)cudaGetLastError();
}

// MoE grouped GEMM over the expert-sorted rows g.xb.  Types of the fused kernel: ONE launch over the row tiles of the segments, the weights
// decoded inside the kernel.  Every other type: the experts are walked in groups whose bf16 copies fit `wscratch` (a contiguous range of the
// sorted rows each); per group and segment the experts that received rows are dequantised, then one grouped bf16 GEMM.  Segment i reads the rows
// [g.row0[i], g.row0[i] + g.M) of matrices of g.rows_layout rows; segments of one tensor (merged up/gate experts) share one dequantised copy.
int b200q_launch_gemm_grouped(const b200q_moe_gemm & g, void * wscratch, size_t ws_bytes, cudaStream_t st) {
    if (g.K % 256 || g.n_seg < 1 || g.n_seg > 2 || g.n_rows < 1 || (g.bn != 128 && g.bn != 256)) return -2;
    for (int i = 0; i < g.n_seg; ++i) if (g.row0[i] < 0 || g.row0[i] + g.M > g.rows_layout) return -2;
    const bool bn256 = g.bn == 256;
    if (gemmq_supported(g.type)) {
        b200q_gemm_multi d; memset(&d, 0, sizeof d);
        d.type = g.type; d.n_seg = g.n_seg; d.K = g.K; d.N = g.n_rows; d.xb = g.xb; d.rows_layout = g.rows_layout;
        for (int i = 0; i < g.n_seg; ++i) { d.W[i] = g.W[i]; d.dst[i] = g.dst[i]; d.M[i] = g.M; d.row0[i] = g.row0[i]; }
        return launch_gemm_q<true>(g.type, bn256, d, 1, g.n_expert, g.rt, st);
    }
    b200q_layout L; if (b200q_make_layout(g.type, g.rows_layout, g.K, &L)) return -1;
    const int64_t ebytes = g.rows_layout * g.K * 2;
    const int64_t per = std::min<int64_t>(g.n_expert, (int64_t)(ws_bytes / (size_t)ebytes));
    if (per < 1) return -5;
    for (int e0 = 0; e0 < g.n_expert; e0 += (int)per) {
        b200q_moe_route rt = g.rt; rt.e0 = e0; rt.e1 = (int)std::min<int64_t>(g.n_expert, e0 + per);
        for (int i = 0; i < g.n_seg; ++i) {
            int rc = 0;
            if (i == 0 || g.W[i] != g.W[i - 1]) { rc = b200q_launch_dequant_bf16_experts(g.W[i], L, wscratch, rt.e0, rt.e1 - rt.e0, g.rt.bounds, st); if (rc) return rc; }
            const char * A = (const char *)wscratch + g.row0[i] * g.K * 2;
            rc = bn256 ? launch_gemm_bf16<256, true>(A, rt.e1 - rt.e0, g.rows_layout, g.xb, g.dst[i], g.M, g.n_rows, g.K, 1, rt, st)
                       : launch_gemm_bf16<128, true>(A, rt.e1 - rt.e0, g.rows_layout, g.xb, g.dst[i], g.M, g.n_rows, g.K, 1, rt, st);
            if (rc) return rc;
        }
    }
    return 0;
}

int b200q_launch_gemm_bf16x(int type, const void * W, const void * xb, float * dst, int64_t M, int64_t K, int64_t N,
                            void * wscratch, size_t ws_bytes, int sm_count, int fused, cudaStream_t st) {
    b200q_gemm_multi d; memset(&d, 0, sizeof d);
    d.type = type; d.n_seg = 1; d.W[0] = W; d.dst[0] = dst; d.M[0] = M; d.K = K; d.N = N; d.xb = xb;
    return b200q_launch_gemm_multi_bf16x(d, wscratch, ws_bytes, sm_count, fused, st);
}

// A = planes of `type` [M][K]; X = f32 [N][K]; dst f32 [N][M].  Workspace: B200Q_DENSE_GEMM.
int b200q_launch_gemm(int type, const void * W, const float * x, int64_t x_stride, float * dst, int64_t M, int64_t K, int64_t N,
                      void * ws, size_t ws_bytes, int sm_count, int fused, cudaStream_t st) {
    return b200q_launch_gemm_rows(type, W, M, 0, x, 0, x_stride, dst, M, K, N, ws, ws_bytes, sm_count, fused, st);
}
// A = rows [row0, row0 + M) of the planes of `type` [rows_layout][K]: the activations become bf16 once (f16 ones by k_f16_convert, which replaces
// k_f32_to_bf16), or, for IQ2_BN on the int8 pipe, are quantised from f32 (f16 ones widened first)
int b200q_launch_gemm_rows(int type, const void * W, int64_t rows_layout, int64_t row0, const void * x, int x_f16, int64_t x_stride, float * dst,
                           int64_t M, int64_t K, int64_t N, void * ws, size_t ws_bytes, int sm_count, int fused, cudaStream_t st) {
    const bool widen = x_f16 && fused && b200q_gemm_bn_i8_ok(type, K, N, nullptr, K, SIZE_MAX);
    const b200q_dense_ws L = b200q_dense_layout(widen ? B200Q_DENSE_GEMM_WIDEN : B200Q_DENSE_GEMM, M, K, N);
    if (ws_bytes < L.total) return -5;
    char * w = (char *)ws;
    b200q_gemm_multi d; memset(&d, 0, sizeof d);
    d.type = type; d.n_seg = 1; d.W[0] = W; d.dst[0] = dst; d.M[0] = M; d.K = K; d.N = N; d.rows_layout = rows_layout; d.row0[0] = row0;
    const float * xf = (const float *)x; int64_t xs = x_stride;
    if (widen) {
        if (const int rc = b200q_launch_f16_convert(x, x_stride, w + L.xf, 0, K, N, st)) return rc;
        xf = (const float *)(w + L.xf); xs = K;
    }
    if (fused && (!x_f16 || widen) && b200q_gemm_bn_i8_ok(type, K, N, xf, xs, ws_bytes - L.x))     // ternary weights: int8 tensor pipe (u8 x s8 wgmma), exact integer accumulation
        return b200q_launch_gemm_bn_i8(d, xf, xs, w + L.x, ws_bytes - L.x, st);
    d.xb = w + L.x;
    const int rc = x_f16 ? b200q_launch_f16_convert(x, x_stride, w + L.x, 1, K, N, st) : b200q_launch_f32_to_bf16(xf, x_stride, w + L.x, K, N, st);
    if (rc) return rc;
    return b200q_launch_gemm_multi_bf16x(d, w + L.wsc, ws_bytes - L.wsc, sm_count, fused, st);
}
