// b200q_decode.cu — HBM-bound kernels of the hot path for sm_90a:
//   * k_repack / k_unrepack   wire (GGUF) blocks <-> plane layout (b200q_types.cuh), run once per tensor upload/download
//   * k_mmvq                  decode mat-vec  dst[n][m] = sum_k W[m][k] x[n][k],  n <= 8   (replaces the reference's
//                             quantize_q8_1 + mul_mat_vec_q / iqk_mul_mat_vec_q / fused_mul_mat_vec_q:
//                             ggml/src/ggml-cuda/quantize.cu:13-47, mmvq-templates.cuh:68-330, iqk_mmvq_templates.cuh:21-300)
//   * k_dequant_bf16          planes -> bf16 [M][K] (generic feeder of the wgmma GEMM for types without a fused prefill kernel)
//
// Decode design (one launch per GGML_OP_MUL_MAT / FUSED_UP_GATE node, no tensor cores):
//   - prologue: every CTA quantises the activation column(s) to q8_1 semantics straight into shared memory
//     (int8 values in natural k order, d rounded to half like block_q8_1.ds.x, integer sums per 16) — no separate
//     quantize launch, no q8_1 round trip through HBM;
//   - main loop: one warp per output row; lane l owns items l, l+32, ... (item = 32 weights = one 16-byte LDG.128 of the
//     low-bit plane, perfectly coalesced: 512 contiguous bytes per warp-load), UNROLL independent loads in flight
//     before the first use; PRMT-LUT / mask decode into int8x4 lanes; dp4a against the smem activations;
//   - epilogue: warp-shuffle reduce, optional bias, optional act(gate)*up fusion, one 4-byte store per row.
#include "b200q_types.cuh"
#include "b200q_internal.h"
#include "b200q_decode_common.cuh"
#include "b200q_decode_ring.cuh"
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdlib.h>

// ------------------------------------------------------------------------------------------------
// repack
// ------------------------------------------------------------------------------------------------
__global__ void k_repack(const uint8_t * __restrict__ wire, uint8_t * __restrict__ planes, b200q_layout L, int inverse) {
    const int64_t rs = (int64_t)L.row_meta + L.nb * L.wire_block;
    const int64_t total = L.M * L.nb;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / L.nb, blk = i % L.nb;
        const uint8_t * w = wire + row * rs + L.row_meta + blk * L.wire_block;
        b200q_repack_block(L, w, planes, row, blk, inverse != 0);
        if (blk == 0) b200q_repack_row_meta(L, wire + row * rs, planes, row, inverse != 0);
    }
}

// ------------------------------------------------------------------------------------------------
// dequantise planes -> bf16 [M][K]; blockIdx.y = expert e0 + y of an expert tensor (experts L.total_bytes apart) -> out[y][M][K],
// skipped when `bounds` says that it received no rows (MoE prefill)
// ------------------------------------------------------------------------------------------------
template <int TYPE>
__global__ void k_dequant_bf16(const uint8_t * __restrict__ W, b200q_layout L, __nv_bfloat16 * __restrict__ out, int e0, const int * __restrict__ bounds) {
    const int e = e0 + (int)blockIdx.y;
    if (bounds != nullptr && __ldg(bounds + e + 1) == __ldg(bounds + e)) return;
    W += (int64_t)e * L.total_bytes; out += (int64_t)blockIdx.y * L.M * L.K;
    const int64_t n32 = L.K / 32, total = L.M * n32;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / n32, it = i % n32;
        b200q_item I; b200q_canon C;
        b200q_load_item<TYPE>(I, b200q_planes_from(W, L), row, it);
        b200q_decode_item<TYPE>(I, it, C);
        float f[32];
        b200q_canon_to_float<b200q_traits<TYPE>::HAS_B>(C, f);
        uint4 * o = reinterpret_cast<uint4 *>(out + row * L.K + it * 32);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            __nv_bfloat162 p0 = __floats2bfloat162_rn(f[8 * v + 0], f[8 * v + 1]), p1 = __floats2bfloat162_rn(f[8 * v + 2], f[8 * v + 3]);
            __nv_bfloat162 p2 = __floats2bfloat162_rn(f[8 * v + 4], f[8 * v + 5]), p3 = __floats2bfloat162_rn(f[8 * v + 6], f[8 * v + 7]);
            uint4 u; u.x = *reinterpret_cast<uint32_t *>(&p0); u.y = *reinterpret_cast<uint32_t *>(&p1); u.z = *reinterpret_cast<uint32_t *>(&p2); u.w = *reinterpret_cast<uint32_t *>(&p3);
            o[v] = u;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
#ifdef B200Q_BENCH_TYPES_ONLY      // tuning variants (scripts/build_variant.sh): only the benchmarked type, small and quick to build
#define B200Q_FOR_TYPES(X) X(B200Q_TYPE_IQ4_NL)
#else
#define B200Q_FOR_TYPES(X) X(B200Q_TYPE_IQ4_NL) X(B200Q_TYPE_Q4_0) X(B200Q_TYPE_Q8_0) X(B200Q_TYPE_Q4_K) X(B200Q_TYPE_Q5_K) \
    X(B200Q_TYPE_Q6_K) X(B200Q_TYPE_IQ4_XS) X(B200Q_TYPE_IQ4_K) X(B200Q_TYPE_IQ4_KS) X(B200Q_TYPE_IQ5_K) X(B200Q_TYPE_IQ2_BN) \
    X(B200Q_TYPE_Q4_1) X(B200Q_TYPE_Q5_0) X(B200Q_TYPE_Q5_1) X(B200Q_TYPE_Q6_0) X(B200Q_TYPE_Q2_K) X(B200Q_TYPE_Q3_K) \
    X(B200Q_TYPE_IQ2_K) X(B200Q_TYPE_IQ3_K) X(B200Q_TYPE_MXFP4) X(B200Q_TYPE_IQ5_KS) \
    X(B200Q_TYPE_IQ2_KS) X(B200Q_TYPE_IQ3_KS)
#endif

// the per-type mat-vec launchers are instantiated in b200q_decode_i<N>.cu (parallel compilation)
#define X(T) extern template int launch_mmvq_type<T>(const mmvq_args &, int, bool, int, bool, bool, cudaStream_t); \
             extern template int launch_mmvq_id_type<T>(const mmvq_id_args &, bool, int, bool, cudaStream_t);
B200Q_FOR_TYPES(X)
#undef X

int b200q_launch_repack(const void * wire, void * planes, const b200q_layout & L, int inverse, cudaStream_t st) {
    if (L.wire) {       // wire-layout type: the device copy IS the GGUF payload
        const size_t nbytes = (size_t)(L.M * b200q_wire_row_size(L));
        return (int)(inverse ? cudaMemcpyAsync(const_cast<void *>(wire), planes, nbytes, cudaMemcpyDeviceToDevice, st) : cudaMemcpyAsync(planes, wire, nbytes, cudaMemcpyDeviceToDevice, st));
    }
    const int64_t total = L.M * L.nb;
    const int bs = 128; const int64_t nb = (total + bs - 1) / bs;
    k_repack<<<(unsigned)(nb > 65535 * 16 ? 65535 * 16 : (nb < 1 ? 1 : nb)), bs, 0, st>>>((const uint8_t *)wire, (uint8_t *)planes, L, inverse);
    return (int)cudaGetLastError();
}

int b200q_launch_dequant_bf16(const void * W, const b200q_layout & L, void * out, cudaStream_t st) {
    return b200q_launch_dequant_bf16_experts(W, L, out, 0, 1, nullptr, st);
}
int b200q_launch_dequant_bf16_experts(const void * W, const b200q_layout & L, void * out, int e0, int n_e, const int * bounds, cudaStream_t st) {
    if (n_e < 1 || n_e > 65535) return -2;
    if (L.wire) return b200q_launch_wire_dequant_bf16_experts(L.type, W, L.M, L.K, L.total_bytes, out, e0, n_e, bounds, st);
    const int64_t total = L.M * (L.K / 32);
    const int bs = 256; int64_t nb = (total + bs - 1) / bs; const int64_t cap = 132 * 64 / n_e > 1 ? 132 * 64 / n_e : 1; if (nb > cap) nb = cap; if (nb < 1) nb = 1;
    const dim3 grid((unsigned)nb, (unsigned)n_e);
    switch (L.type) {
#define X(T) case T: k_dequant_bf16<T><<<grid, bs, 0, st>>>((const uint8_t *)W, L, (__nv_bfloat16 *)out, e0, bounds); break;
        B200Q_FOR_TYPES(X)
#undef X
        default: return -1;
    }
    return (int)cudaGetLastError();
}

// per-launch phase timestamps (debug aid for the PDL pipeline; see scripts/trace_decode.py)
static unsigned long long * g_trace = nullptr; static int g_trace_slot = 0;
static unsigned long long * g_trace_cta = nullptr;      // [512 launches][512 CTAs][4]
extern "C" __attribute__((visibility("default"))) int b200q_debug_trace(int enable, unsigned long long * host_out, int max_slots) {
    if (enable == 4 && host_out && g_trace_cta) {           // per-CTA timeline of launch slot `max_slots`
        cudaMemcpy(host_out, g_trace_cta + (size_t)max_slots * 2048, 2048 * sizeof(unsigned long long), cudaMemcpyDeviceToHost); return 0;
    }
    if ((enable == 1 || enable == 3) && !g_trace_cta) cudaMalloc(&g_trace_cta, (size_t)512 * 2048 * sizeof(unsigned long long));
    if ((enable == 1 || enable == 3) && g_trace_cta) cudaMemset(g_trace_cta, 0, (size_t)512 * 2048 * sizeof(unsigned long long));
    if (enable == 1) { if (!g_trace) { cudaMalloc(&g_trace, 4096 * 8 * sizeof(unsigned long long)); } cudaMemset(g_trace, 0, 4096 * 8 * sizeof(unsigned long long)); g_trace_slot = 0; return 0; }
    if (enable == 2) { g_trace_slot = 0; return 0; }                               // rewind (start of a step)
    if (enable == 3 && g_trace) { cudaDeviceSynchronize(); cudaMemset(g_trace, 0, 4096 * 8 * sizeof(unsigned long long)); return 0; }   // clear, keep the slot assignment
    if (enable == 0 && host_out && g_trace) { cudaMemcpy(host_out, g_trace, (size_t)max_slots * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost); return g_trace_slot; }
    return -1;
}
int b200q_launch_mmvq(const b200q_mmvq_desc & d, cudaStream_t st) {
    if (b200q_is_wire_type(d.type)) return b200q_launch_wire_mmvq(d, st);
    mmvq_args a; memset(&a, 0, sizeof a);
    if (g_trace && g_trace_slot < 4096) { if (g_trace_cta && g_trace_slot < 512) a.trace_cta = g_trace_cta + (size_t)g_trace_slot * 2048; a.trace = g_trace + 8 * (g_trace_slot++); }
    if (d.n_seg < 1 || d.n_seg > B200Q_MAX_SEGS || d.ncols < 1 || d.ncols > 8) return -2;
    int64_t r0 = 0;
    for (int i = 0; i < d.n_seg; ++i) {
        b200q_layout L; const int rc = b200q_make_layout(d.type, d.seg[i].M, d.K, &L); if (rc) return rc;
        a.seg[i].P = b200q_planes_from((const uint8_t *)d.seg[i].W, L);
        if (d.seg[i].W2) a.seg[i].P2 = b200q_planes_from((const uint8_t *)d.seg[i].W2, L);
        a.seg[i].dst = d.seg[i].dst; a.seg[i].bias = d.seg[i].bias; a.seg[i].M = d.seg[i].M; a.seg[i].row0 = r0; r0 += d.seg[i].M;
    }
    a.n_seg = d.n_seg; a.M_total = r0; a.K = d.K; a.x = d.x; a.x_stride = d.x_stride ? d.x_stride : d.K; a.act = d.act; a.limit = d.limit;
    a.tp = d.tp;
    if (d.next) {
        static const int cps = [] { const char * e = getenv("B200Q_CTAS_PER_SM"); return e ? atoi(e) : B200Q_MIN_CTAS; }();
        make_next_prefetch(*d.next, d.sm_count, cps, a.pf);
    }
    const bool upgate = d.seg[0].W2 != nullptr;
    if (d.q8_in || d.q8_out) {          // q8 hand-off: n = 1, single tensor, ring kernel, bulk-copyable image
        if (d.ncols != 1 || d.n_seg != 1 || !d.ring || a.tp.in || a.tp.out) return -8;
        if (d.q8_in && (d.K % 64 || ((uintptr_t)d.q8_in & 15))) return -8;
        if (d.q8_out && (!upgate || d.seg[0].M % 64 || ((uintptr_t)d.q8_out & 15))) return -8;
        a.q8_in = d.q8_in; a.q8_out = d.q8_out;
    }
    if (a.tp.in || a.tp.out) {          // only the TMA-ring kernel implements the fused reduce
        if (d.ncols != 1 || !d.ring || d.K % 256 || (a.tp.out && r0 > a.tp.ll_stride) || (a.tp.in && d.K > a.tp.ll_stride)) return -7;
    }
    switch (d.type) {
#define X(T) case T: return launch_mmvq_type<T>(a, d.ncols, upgate, d.sm_count, d.pdl != 0, d.ring != 0, st);
        B200Q_FOR_TYPES(X)
#undef X
        default: return -1;
    }
}

// MoE decode (GGML_OP_MUL_MAT_ID / MOE_FUSED_UP_GATE, small batches): see k_mmvq_id / k_wire_mmvq_id.  The operands' row origins are folded into
// the plane pointers here (b200q_planes_at): the kernels see the rows [row0, row0 + M) of each expert as an [M x K] matrix, estride bytes apart.
int b200q_launch_mmvq_id(const b200q_mmvq_id_desc & d, cudaStream_t st) {
    if (d.n_tokens < 1 || d.n_used < 1 || d.nb1 < 1 || d.n_used % d.nb1 || d.n_expert < 1 || !d.W || !d.ids || !d.x || !d.dst) return -2;
    if (d.M < 1 || d.W_row0 < 0 || d.W2_row0 < 0 || d.W_row0 + d.M > d.rows_layout || (d.W2 && d.W2_row0 + d.M > d.rows_layout)) return -2;
    if (b200q_is_wire_type(d.type)) return b200q_launch_wire_mmvq_id(d, st);
    b200q_layout L; const int rc = b200q_make_layout(d.type, d.rows_layout, d.K, &L); if (rc) return rc;
    mmvq_id_args a; memset(&a, 0, sizeof a);
    a.P = b200q_planes_at((const uint8_t *)d.W, L, d.W_row0); if (d.W2) a.P2 = b200q_planes_at((const uint8_t *)d.W2, L, d.W2_row0);
    a.estride = L.total_bytes; a.ids = d.ids; a.n_expert = d.n_expert; a.n_slots = d.n_tokens * d.n_used; a.n_used = d.n_used; a.nb1 = d.nb1; a.ncx = d.n_tokens * d.nb1;
    a.M = d.M; a.K = d.K; a.x = d.x; a.dst = d.dst; a.act = d.act; a.limit = d.limit;
    switch (d.type) {
#define X(T) case T: return launch_mmvq_id_type<T>(a, d.W2 != nullptr, d.sm_count, d.pdl != 0, st);
        B200Q_FOR_TYPES(X)
#undef X
        default: return -1;
    }
}
