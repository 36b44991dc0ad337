// b200q_reduce.cu — GGML_OP_REDUCE (sum) over NVLink/NVSwitch for the row-parallel mat-muls of "split mode graph".
// Replaces ggml_cuda_op_reduce (ggml/src/ggml-cuda/reduce.cu:125-598: ncclAllReduce / copy-engine ring / k_reduce_add_T).
//
// One kernel per all-reduce, one process per GPU, buffers in symmetric memory with an NVLS multicast mapping:
//   (1) zero the dirty part of the OTHER parity buffer (it is used by the next all-reduce; peers may only start adding to it after they have
//       seen this rank's flag increment below, which is ordered after the zeroing);
//   (2) multimem.red.add.f32 of the local partial into the multicast address: the switch adds it into EVERY rank's copy;
//   (3) last CTA: multimem.red.add.u32 on the multicast flag (release.sys) -> every rank's flag += 1;
//   (4) every CTA spins (ld.acquire.sys) until the local flag reaches world * use_count, then copies its slice of the
//       local (now fully reduced) buffer to `out`.
// tg: n = n_embd floats (16 KiB) -> 1 CTA, pure latency (~2 NVLink hops); pp512: 8 MiB -> up to one CTA per SM (132).
// f32 adds are performed by the switch in arrival order (like NCCL's NVLS algorithm): run-to-run LSB differences are possible.
#include "b200q_internal.h"
#include <cuda_runtime.h>

namespace {
__device__ __forceinline__ void mm_red_add_f32x4(float * mc, float4 v) {
    asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void mm_red_add_f32(float * mc, float v) {
    asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(mc), "f"(v) : "memory");
}
__device__ __forceinline__ void mm_red_add_u32_release(uint32_t * mc, uint32_t v) {
    asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t * p) {
    uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}

// `seq` (device-local counter of reduces issued on this communicator) selects the parity buffer and the flag target inside the
// kernel, so the launch parameters are constant and the kernel can be replayed from a CUDA graph.
__global__ void __launch_bounds__(512) k_allreduce_nvls(const float * __restrict__ in, float * __restrict__ out, int64_t n,
                                                         float * mc_base, float * local_base, int64_t stride,
                                                         uint32_t * mc_flag, const uint32_t * local_flag, uint32_t world,
                                                         uint32_t * seq, uint32_t * cta_counter) {
    const uint32_t s = *reinterpret_cast<volatile uint32_t *>(seq);      // read before this CTA's counter increment (see below)
    // seq[1 + p] = number of floats of parity buffer p that may be non-zero (left there by its last use): reduces of different
    // lengths share the buffers (tg: n_embd floats, pp512: 512 x n_embd), so the zeroing covers what was actually dirtied
    const int64_t n_dirty = (int64_t)reinterpret_cast<volatile uint32_t *>(seq)[1 + ((s & 1) ^ 1)];
    const uint32_t target = world * (s + 1);
    float * mc_buf = mc_base + (int64_t)(s & 1) * stride;
    const float * local_buf = local_base + (int64_t)(s & 1) * stride;
    float * local_zero = local_base + (int64_t)((s & 1) ^ 1) * stride;
    const int64_t n4 = n / 4;
    const int64_t per = (n4 + gridDim.x - 1) / gridDim.x;
    const int64_t i0 = (int64_t)blockIdx.x * per, i1 = min(n4, i0 + per);
    // (1)
    {
        const int64_t d4 = (n_dirty + 3) / 4, dper = (d4 + gridDim.x - 1) / gridDim.x;
        const int64_t z0 = (int64_t)blockIdx.x * dper, z1 = min(d4, z0 + dper);
        for (int64_t i = z0 + threadIdx.x; i < z1; i += blockDim.x) reinterpret_cast<float4 *>(local_zero)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // (2)
    for (int64_t i = i0 + threadIdx.x; i < i1; i += blockDim.x)
        mm_red_add_f32x4(mc_buf + 4 * i, __ldg(reinterpret_cast<const float4 *>(in) + i));
    if (blockIdx.x == gridDim.x - 1)
        for (int64_t i = 4 * n4 + threadIdx.x; i < n; i += blockDim.x) mm_red_add_f32(mc_buf + i, in[i]);
    __threadfence_system();
    __syncthreads();
    // (3)
    if (threadIdx.x == 0) {
        const uint32_t done = atomicAdd(cta_counter, 1u);
        if (done == gridDim.x - 1) {                 // every CTA has read `seq` (it does so before its atomicAdd)
            *cta_counter = 0;
            reinterpret_cast<volatile uint32_t *>(seq)[1 + ((s & 1) ^ 1)] = 0; reinterpret_cast<volatile uint32_t *>(seq)[1 + (s & 1)] = (uint32_t)n;
            *reinterpret_cast<volatile uint32_t *>(seq) = s + 1; __threadfence();
            mm_red_add_u32_release(mc_flag, 1u);
        }
        // (4)
        while ((int32_t)(ld_acquire_sys(local_flag) - target) < 0) { __nanosleep(32); }
    }
    __syncthreads();
    for (int64_t i = i0 + threadIdx.x; i < i1; i += blockDim.x)
        reinterpret_cast<float4 *>(out)[i] = __ldcv(reinterpret_cast<const float4 *>(local_buf) + i);
    if (blockIdx.x == gridDim.x - 1)
        for (int64_t i = 4 * n4 + threadIdx.x; i < n; i += blockDim.x) out[i] = __ldcv(local_buf + i);
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Two-shot bf16 all-reduce for the prefill-sized REDUCE (the reference casts the partial to bf16/f16 when ne[1] > 32,
// src/llama-build-context.cpp:1198-1200, and runs reduce-scatter + all-gather, ggml-cuda/reduce.cu:306-372).  One kernel:
//   (a) f32 partial -> bf16 into this rank's slice-addressable STAGING buffer in symmetric memory (local stores);
//       barrier A (multicast flag): every rank's staging is complete;
//   (b) reduce-scatter + all-gather in the switch: rank r owns slice r: multimem.ld_reduce (f32 accumulation of the world's bf16
//       values inside the NVSwitch) and multimem.st of the sum back into EVERY rank's staging (16 bytes per instruction);
//       barrier B: every slice has been broadcast;
//   (c) the fully reduced bf16 vector is copied out of the local staging (bf16 for the next GEMM's activation operand and / or f32).
// Per GPU and reduce the NVLink carries ~2 x n x 2 bytes (one-shot f32: world x n x 4 inbound); the payload of pp512 is 4 MiB.
// state: rank-local u32[4] {reduces done, CTA counter a, CTA counter b, pad}; the flag counts 2 x world per reduce.
// Safe with ONE staging buffer: (a) of reduce k+1 follows this rank's (c) of reduce k in stream order, and no peer touches this
// rank's staging outside its own phase (b), which lies between the two barriers.
// ---------------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 mm_ld_reduce_bf16x8(const void * mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mm_st_b128(void * mc, uint4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    uint32_t r; asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a)); return r;      // low half = a
}
__device__ __forceinline__ void grid_rendezvous(uint32_t * cta_counter, uint32_t * mc_flag, const uint32_t * local_flag, uint32_t target,
                                                uint32_t * seq_to_bump, uint32_t seq_next) {
    __threadfence_system();                     // this thread's staging stores / multimem stores are performed system-wide
    __syncthreads();
    if (threadIdx.x == 0) {
        if (atomicAdd(cta_counter, 1u) == gridDim.x - 1) {
            *cta_counter = 0;
            if (seq_to_bump) *reinterpret_cast<volatile uint32_t *>(seq_to_bump) = seq_next;
            __threadfence();
            mm_red_add_u32_release(mc_flag, 1u);
        }
        while ((int32_t)(ld_acquire_sys(local_flag) - target) < 0) __nanosleep(32);
    }
    __syncthreads();
}
__global__ void __launch_bounds__(512) k_allreduce_nvls_2shot(const float * __restrict__ in, float * __restrict__ out_f32, uint4 * __restrict__ out_bf16, int64_t n8,
                                                              uint4 * mc_stage, uint4 * local_stage, uint32_t * mc_flag, const uint32_t * local_flag,
                                                              uint32_t world, uint32_t rank, uint32_t * state) {
    const uint32_t s = *reinterpret_cast<volatile uint32_t *>(state);
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    // (a)
    for (int64_t i = tid; i < n8; i += nth) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(in) + 2 * i), b = __ldg(reinterpret_cast<const float4 *>(in) + 2 * i + 1);
        local_stage[i] = make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
    }
    grid_rendezvous(state + 1, mc_flag, local_flag, world * (2 * s + 1), nullptr, 0);
    // (b)
    {
        const int64_t per = (n8 + world - 1) / world, b0 = per * rank, b1 = min(n8, b0 + per);
        for (int64_t i = b0 + tid; i < b1; i += nth) mm_st_b128(mc_stage + i, mm_ld_reduce_bf16x8(mc_stage + i));
    }
    grid_rendezvous(state + 2, mc_flag, local_flag, world * (2 * s + 2), state, s + 1);
    // (c)
    for (int64_t i = tid; i < n8; i += nth) {
        const uint4 v = __ldcv(local_stage + i);
        if (out_bf16) out_bf16[i] = v;
        if (out_f32) {
            float4 a, b;
            a.x = __uint_as_float(v.x << 16); a.y = __uint_as_float(v.x & 0xFFFF0000u); a.z = __uint_as_float(v.y << 16); a.w = __uint_as_float(v.y & 0xFFFF0000u);
            b.x = __uint_as_float(v.z << 16); b.y = __uint_as_float(v.z & 0xFFFF0000u); b.z = __uint_as_float(v.w << 16); b.w = __uint_as_float(v.w & 0xFFFF0000u);
            reinterpret_cast<float4 *>(out_f32)[2 * i] = a; reinterpret_cast<float4 *>(out_f32)[2 * i + 1] = b;
        }
    }
}
}  // namespace

int b200q_launch_allreduce_nvls_2shot(const float * in, float * out_f32, void * out_bf16, int64_t n, void * mc_stage, void * local_stage,
                                      void * mc_flag, const void * local_flag, uint32_t world, uint32_t rank, void * state, int sm_count, cudaStream_t st) {
    if (n <= 0 || (n & 7) || ((uintptr_t)in & 15) || ((uintptr_t)out_f32 & 15) || ((uintptr_t)out_bf16 & 15) || ((uintptr_t)mc_stage & 15) || ((uintptr_t)local_stage & 15)) return -2;
    int64_t grid = (n / 8 + 2047) / 2048;          // >= 4 vectors per thread
    if (grid > sm_count) grid = sm_count;          // all CTAs must be co-resident: they spin on the flag
    if (grid < 1) grid = 1;
    k_allreduce_nvls_2shot<<<(unsigned)grid, 512, 0, st>>>(in, out_f32, (uint4 *)out_bf16, n / 8, (uint4 *)mc_stage, (uint4 *)local_stage,
                                                          (uint32_t *)mc_flag, (const uint32_t *)local_flag, world, rank, (uint32_t *)state);
    return (int)cudaGetLastError();
}

int b200q_launch_allreduce_nvls(const float * in, float * out, int64_t n, void * mc_base, void * local_base, int64_t stride,
                                void * mc_flag, const void * local_flag, uint32_t world, void * seq, void * cta_counter, int sm_count, cudaStream_t st) {
    if (n <= 0 || n > stride || ((uintptr_t)in & 15) || ((uintptr_t)out & 15) || ((uintptr_t)mc_base & 15) || (stride & 3)) return -2;
    int64_t grid = (n + 16383) / 16384;            // >= 64 KiB per CTA
    if (grid > sm_count) grid = sm_count;          // all CTAs must be co-resident: they spin on the flag
    if (grid < 1) grid = 1;
    k_allreduce_nvls<<<(unsigned)grid, 512, 0, st>>>(in, out, n, (float *)mc_base, (float *)local_base, stride,
                                                    (uint32_t *)mc_flag, (const uint32_t *)local_flag, world, (uint32_t *)seq, (uint32_t *)cta_counter);
    return (int)cudaGetLastError();
}
