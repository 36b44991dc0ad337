// b200q_wire.cu — kernels for the wire-layout types (b200q_wire.cuh): the types the reference's CUDA back-end serves through
// vec_dot_<type>_q8_1 / iqk_mul_mat_vec_q (ggml-cuda/vecdotq.cuh:852-1127, iqk_mmvq.cu, template-instances/mmvq-instance-iq*_kt.cu,
// -iq*_r4.cu) and through dequantize_block_* + GEMM for prefill (ggml-cuda/convert.cu, iqk_mmvq / mmq loaders mmq.cuh:2149-2445).
//   * k_wire_dequant_bf16   wire bytes -> bf16 [M][K]: feeder of the wgmma GEMM (same path as the unfused plane types)
//   * k_wire_mmvq           decode mat-vec, n <= 8: activations quantised to q8_1 in shared memory exactly like the plane kernels, one
//                           warp per row, lanes stride the 32-weight items, f32 dot of the decoded weights with the q8 values:
//                           the result is the quantity the reference's MMVQ kernels compute, up to f32 summation order.
// The weights stay in their GGUF byte layout (2-byte aligned blocks, no 16-byte loads): this is the COMPLETE-coverage path, not the fast
// one; the bandwidth-critical types live in the plane layout (b200q_types.cuh).
#include "b200q_wire.cuh"
#include "b200q_internal.h"
#include "b200q_decode_common.cuh"
#include "b200q_decode_plan.h"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <string.h>

namespace {

// blockIdx.y = expert e0 + y of an expert tensor (experts estride bytes apart) -> out[y][M][K], skipped when `bounds` says it received no rows
template <int TYPE>
__global__ void k_wire_dequant_bf16(const uint8_t * __restrict__ W, int64_t M, int64_t K, __nv_bfloat16 * __restrict__ out,
                                    int64_t estride, int e0, const int * __restrict__ bounds) {
    const int e = e0 + (int)blockIdx.y;
    if (bounds != nullptr && __ldg(bounds + e + 1) == __ldg(bounds + e)) return;
    W += (int64_t)e * estride; out += (int64_t)blockIdx.y * M * K;
    const int64_t n32 = K / 32, total = M * n32;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / n32, it = i % n32;
        float f[32];
        b200q_wire_decode32<TYPE>(W, K, row, it, f);
        uint4 * o = reinterpret_cast<uint4 *>(out + row * K + it * 32);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            __nv_bfloat162 p0 = __floats2bfloat162_rn(f[8 * v + 0], f[8 * v + 1]), p1 = __floats2bfloat162_rn(f[8 * v + 2], f[8 * v + 3]);
            __nv_bfloat162 p2 = __floats2bfloat162_rn(f[8 * v + 4], f[8 * v + 5]), p3 = __floats2bfloat162_rn(f[8 * v + 6], f[8 * v + 7]);
            uint4 u; u.x = *reinterpret_cast<uint32_t *>(&p0); u.y = *reinterpret_cast<uint32_t *>(&p1); u.z = *reinterpret_cast<uint32_t *>(&p2); u.w = *reinterpret_cast<uint32_t *>(&p3);
            o[v] = u;
        }
    }
}

struct wire_mmvq_args {
    const uint8_t * W[B200Q_MAX_SEGS]; const uint8_t * W2; float * dst[B200Q_MAX_SEGS]; const float * bias[B200Q_MAX_SEGS];
    int64_t M[B200Q_MAX_SEGS], row0[B200Q_MAX_SEGS];
    int n_seg; int64_t M_total, K; const float * x; int64_t x_stride; int act; float limit;
};

template <int TYPE, int NCOLS, bool UPGATE>
__global__ void __launch_bounds__(256) k_wire_mmvq(const wire_mmvq_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int64_t K = a.K; const int n32 = (int)(K / 32);
    int8_t * sq = reinterpret_cast<int8_t *>(smem_raw);
    float *  sd = reinterpret_cast<float *>(smem_raw + (size_t)NCOLS * K);
    int *    sis = reinterpret_cast<int *>(sd + NCOLS * n32);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    pdl_trigger();
    pdl_wait();
    quantize_x_to_smem<NCOLS>(a.x, a.x_stride, K, sq, sd, sis, threadIdx.x, blockDim.x);
    __syncthreads();
    for (int64_t grow = (int64_t)blockIdx.x * nwarps + warp; grow < a.M_total; grow += (int64_t)gridDim.x * nwarps) {
        int s = 0;
#pragma unroll
        for (int i = 1; i < B200Q_MAX_SEGS; ++i) if (i < a.n_seg && grow >= a.row0[i]) s = i;
        const int64_t row = grow - a.row0[s];
        float acc[NCOLS], acc2[NCOLS];
#pragma unroll
        for (int c = 0; c < NCOLS; ++c) { acc[c] = 0.0f; acc2[c] = 0.0f; }
        for (int it = lane; it < n32; it += 32) {
            float w[32];
            b200q_wire_decode32<TYPE>(a.W[s], K, row, it, w);
#pragma unroll
            for (int c = 0; c < NCOLS; ++c) {
                const int8_t * q = sq + (size_t)c * K + (size_t)it * 32;
                float t = 0.0f;
#pragma unroll
                for (int e = 0; e < 32; ++e) t = fmaf(w[e], (float)q[e], t);
                acc[c] = fmaf(sd[c * n32 + it], t, acc[c]);
            }
            if (UPGATE) {
                b200q_wire_decode32<TYPE>(a.W2, K, row, it, w);
#pragma unroll
                for (int c = 0; c < NCOLS; ++c) {
                    const int8_t * q = sq + (size_t)c * K + (size_t)it * 32;
                    float t = 0.0f;
#pragma unroll
                    for (int e = 0; e < 32; ++e) t = fmaf(w[e], (float)q[e], t);
                    acc2[c] = fmaf(sd[c * n32 + it], t, acc2[c]);
                }
            }
        }
#pragma unroll
        for (int c = 0; c < NCOLS; ++c) {
            float v = warp_sum(acc[c]);
            if (UPGATE) { const float g = warp_sum(acc2[c]); v = b200q_glu<false>(a.act, g, v, a.limit); }     // acc = up . x, acc2 = gate . x
            else if (a.bias[s]) v += a.bias[s][row];
            if (lane == 0) a.dst[s][(int64_t)c * a.M[s] + row] = v;
        }
    }
}

// the kernel a plan (plan_mmvq) launches for this type
template <int TYPE>
const void * wire_mmvq_kernel(const b200q_mmvq_plan & p) {
#define CASE(N) case N: return p.upgate ? (const void *)k_wire_mmvq<TYPE, N, true> : (const void *)k_wire_mmvq<TYPE, N, false>;
    switch (p.ncols) { CASE(1) CASE(2) CASE(4) CASE(8) default: return nullptr; }
#undef CASE
}

// MoE decode for wire-layout experts (DeepSeek-style IQ2_XXS / IQ1_S expert tensors): same contract as k_mmvq_id (b200q_decode_ring.cuh)
struct wire_id_args {
    const uint8_t * W; const uint8_t * W2; int64_t estride; const int32_t * ids; int n_expert, n_slots, n_used, nb1, ncx;
    int64_t M, K; const float * x; float * dst; int act; float limit;
    int64_t xs_tok, xs_col;
};
template <int TYPE, bool UPGATE>
__global__ void __launch_bounds__(256) k_wire_mmvq_id(const wire_id_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int64_t K = a.K; const int n32 = (int)(K / 32);
    int8_t * sq = reinterpret_cast<int8_t *>(smem_raw);
    float *  sd = reinterpret_cast<float *>(smem_raw + (size_t)a.ncx * K);
    int *    sis = reinterpret_cast<int *>(sd + a.ncx * n32);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    pdl_trigger();
    pdl_wait();
    // the columns are quantised concurrently, each by a group of whole warps with a thread per 8 floats (the whole CTA once K >= 8 x blockDim)
    const int gs = min((int)blockDim.x, (int)((K / 8 + 31) / 32 * 32)), ng = blockDim.x / gs, grp = threadIdx.x / gs;
    if (grp < ng)
        for (int c = grp; c < a.ncx; c += ng)
            quantize_x_to_smem<1>(a.x + (int64_t)(c / a.nb1) * a.xs_tok + (int64_t)(c % a.nb1) * a.xs_col, K, K, sq + (size_t)c * K, sd + c * n32,
                                  sis + c * n32, threadIdx.x - grp * gs, gs);
    __syncthreads();
    const int64_t total = (int64_t)a.n_slots * a.M;
    for (int64_t g = (int64_t)blockIdx.x * nwarps + warp; g < total; g += (int64_t)gridDim.x * nwarps) {
        const int s = (int)(g / a.M); const int64_t row = g - (int64_t)s * a.M;
        const int e = __ldg(a.ids + s);
        if (e < 0 || e >= a.n_expert) {             // skipped slot: a zero row, no weights read (s is warp-uniform)
            if (lane == 0) a.dst[(int64_t)s * a.M + row] = 0.0f;
            continue;
        }
        const int col = (s / a.n_used) * a.nb1 + (s % a.n_used) % a.nb1;
        const int8_t * xq = sq + (size_t)col * K; const float * xd = sd + col * n32;
        float acc = 0.0f, acc2 = 0.0f;
        for (int it = lane; it < n32; it += 32) {
            float w[32]; float t = 0.0f;
            b200q_wire_decode32<TYPE>(a.W + (int64_t)e * a.estride, K, row, it, w);
#pragma unroll
            for (int j = 0; j < 32; ++j) t = fmaf(w[j], (float)xq[(size_t)it * 32 + j], t);
            acc = fmaf(xd[it], t, acc);
            if (UPGATE) {
                b200q_wire_decode32<TYPE>(a.W2 + (int64_t)e * a.estride, K, row, it, w); t = 0.0f;
#pragma unroll
                for (int j = 0; j < 32; ++j) t = fmaf(w[j], (float)xq[(size_t)it * 32 + j], t);
                acc2 = fmaf(xd[it], t, acc2);
            }
        }
        float v = warp_sum(acc);
        if (UPGATE) { const float gt = warp_sum(acc2); v = b200q_glu<false>(a.act, gt, v, a.limit); }
        if (lane == 0) a.dst[(int64_t)s * a.M + row] = v;
    }
}
}  // namespace

int b200q_launch_wire_mmvq_id(const b200q_mmvq_id_desc & d, cudaStream_t st) {
    const int rc = b200q_wire_check(d.type, d.M, d.K); if (rc) return rc;
    b200q_layout L; if (const int lr = b200q_make_layout(d.type, d.rows_layout, d.K, &L)) return lr;
    if (d.W_row0 % L.wire || d.W2_row0 % L.wire) return -2;          // a row origin inside a group of interleaved rows
    wire_id_args a; memset(&a, 0, sizeof a);
    a.W = (const uint8_t *)d.W + b200q_row_offset(L, 0, d.W_row0); a.W2 = d.W2 ? (const uint8_t *)d.W2 + b200q_row_offset(L, 0, d.W2_row0) : nullptr;
    a.estride = L.total_bytes; a.ids = d.ids; a.n_expert = d.n_expert; a.n_slots = d.n_tokens * d.n_used;
    a.n_used = d.n_used; a.nb1 = d.nb1; a.ncx = d.n_tokens * d.nb1; a.M = d.M; a.K = d.K; a.x = d.x; a.dst = d.dst; a.act = d.act; a.limit = d.limit;
    a.xs_tok = d.x_tok_stride; a.xs_col = d.x_col_stride;
    b200q_mmvq_plan p; if (const int prc = b200q_plan_mmvq_id(d, p)) return prc;
    const void * k = nullptr;
    switch (d.type) {
#define X(T) case T: k = p.upgate ? (const void *)k_wire_mmvq_id<T, true> : (const void *)k_wire_mmvq_id<T, false>; break;
        B200Q_FOR_WIRE_TYPES(X)
#undef X
        default: return -1;
    }
    if (!b200q_opt_in_smem(k, p.smem)) return -3;
    return b200q_launch_pdl(k, p.grid, p.block, p.smem, &a, d.pdl != 0, st);
}

// wire "layout": the tensor is stored verbatim; M must be a multiple of the row interleave
int b200q_wire_check(int type, int64_t M, int64_t K) {
    b200q_wire_geom g; if (!b200q_wire_geom_of(type, g)) return -1;
    if (K <= 0 || K % g.qk || K % 32 || M % g.interleave) return -2;
    return 0;
}

int b200q_launch_wire_dequant_bf16(int type, const void * W, int64_t M, int64_t K, void * out, cudaStream_t st) {
    return b200q_launch_wire_dequant_bf16_experts(type, W, M, K, 0, out, 0, 1, nullptr, st);
}
int b200q_launch_wire_dequant_bf16_experts(int type, const void * W, int64_t M, int64_t K, int64_t estride, void * out, int e0, int n_e, const int * bounds, cudaStream_t st) {
    const int rc = b200q_wire_check(type, M, K); if (rc) return rc;
    if (n_e < 1 || n_e > 65535) return -2;
    const int64_t total = M * (K / 32);
    const int bs = 128; int64_t nb = (total + bs - 1) / bs; const int64_t cap = 132 * 64 / n_e > 1 ? 132 * 64 / n_e : 1; if (nb > cap) nb = cap; if (nb < 1) nb = 1;
    const dim3 grid((unsigned)nb, (unsigned)n_e);
    switch (type) {
#define X(T) case T: k_wire_dequant_bf16<T><<<grid, bs, 0, st>>>((const uint8_t *)W, M, K, (__nv_bfloat16 *)out, estride, e0, bounds); break;
        B200Q_FOR_WIRE_TYPES(X)
#undef X
        default: return -1;
    }
    return (int)cudaGetLastError();
}

int b200q_launch_wire_mmvq(const b200q_mmvq_desc & d, const b200q_mmvq_plan & p, cudaStream_t st) {
    wire_mmvq_args a; memset(&a, 0, sizeof a);
    int64_t r0 = 0;
    for (int i = 0; i < d.n_seg; ++i) {
        a.W[i] = (const uint8_t *)d.seg[i].W; a.dst[i] = d.seg[i].dst; a.bias[i] = d.seg[i].bias; a.M[i] = d.seg[i].M; a.row0[i] = r0; r0 += d.seg[i].M;
    }
    a.W2 = (const uint8_t *)d.seg[0].W2;
    a.n_seg = d.n_seg; a.M_total = r0; a.K = d.K; a.x = d.x; a.x_stride = d.x_stride ? d.x_stride : d.K; a.act = d.act; a.limit = d.limit;
    const void * k = nullptr;
    switch (d.type) {
#define X(T) case T: k = wire_mmvq_kernel<T>(p); break;
        B200Q_FOR_WIRE_TYPES(X)
#undef X
        default: return -1;
    }
    if (!b200q_opt_in_smem(k, p.smem)) return -3;
    return b200q_launch_pdl(k, p.grid, p.block, p.smem, &a, d.pdl != 0, st);
}
