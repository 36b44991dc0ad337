// b200q_moe.cu — MoE prefill: GGML_OP_MUL_MAT_ID / GGML_OP_MOE_FUSED_UP_GATE as a grouped wgmma GEMM over expert-sorted slots.
//
//   dst[t][u][m] = W[ids[t][u]][m] . x[t][u % nb1]        (up/gate: unary(W_gate[id] . x) * (W[id] . x))
//
// One launch sequence per op, with no host round trip, so the whole path can be captured in a CUDA graph:
//   1. k_moe_route (one CTA): per-expert counts -> bounds (exclusive scan), the slots sorted by expert, the tile table {expert, first sorted row}
//      of the BN-row tiles of every expert, the activation column of each sorted row.  Slots whose id is out of range (the -1 of
//      ggml_top_k_thresh) are not routed; their dst rows are zeroed here.
//   2. k_f32_to_bf16 with a row map: the bf16 B operand [slot][K] in sorted order.
//   3. the grouped GEMM (b200q_launch_gemm_grouped): k_gemm_q<.., GROUPED> for the fused types, dequantise-the-active-experts + k_gemm_bf16<.., GROUPED>
//      for the others; the epilogue stores each column straight to dst[slot].
//   4. up/gate: up and gate are two segments of that launch (up -> workspace, gate -> dst), then k_mul_unary over n_slots x M.  Merged up/gate
//      experts ([gate; up] in one [2 M x K] matrix per expert) are the same two segments over row ranges of one tensor (b200q_moe_gemm::row0).
// The reference's generic path (ggml_cuda_mul_mat_id, ggml-cuda.cu:2836-2950) copies ids to the host and synchronises to build its row mapping.
//
// k_moe_combine: GGML_OP_MUL_MULTI_ADD, the routing-weighted sum over the n_used slots of a token that ends every MoE FFN (and, under tensor
// parallelism, produces a rank's partial of it).
#include "b200q_internal.h"
#include <cuda_runtime.h>
#include <algorithm>

namespace {

constexpr int ROUTE_THREADS = 1024;                        // one thread per expert in the scans: n_expert <= 1024
constexpr int64_t MOE_MAX_SLOTS = (int64_t)1 << 22;        // keeps the tile-table grid below 65535 CTAs in y
// bf16 copies of the experts of a generic-type group: the experts are walked in groups that fit this budget
constexpr int64_t MOE_SCRATCH_BUDGET = (int64_t)256 << 20;

__global__ void __launch_bounds__(ROUTE_THREADS)
k_moe_route(const int32_t * __restrict__ ids, int n_slots, int n_used, int nb1, int n_expert, int bn,
            int * __restrict__ bounds, int * __restrict__ tile_start, int2 * __restrict__ tiles, int * __restrict__ slot, int * __restrict__ col,
            float * __restrict__ zero0, float * __restrict__ zero1, int64_t M) {
    __shared__ int s_cnt[ROUTE_THREADS], s_tl[ROUTE_THREADS], s_pos[ROUTE_THREADS];
    const int t = threadIdx.x;
    s_cnt[t] = 0;
    __syncthreads();
    for (int s = t; s < n_slots; s += ROUTE_THREADS) { const int e = __ldg(ids + s); if (e >= 0 && e < n_expert) atomicAdd(&s_cnt[e], 1); }
    __syncthreads();
    const int c = s_cnt[t], tl = (c + bn - 1) / bn;
    s_tl[t] = tl;
    __syncthreads();
    for (int off = 1; off < ROUTE_THREADS; off <<= 1) {       // inclusive scans of the row and tile counts
        const int a = t >= off ? s_cnt[t - off] : 0, b = t >= off ? s_tl[t - off] : 0;
        __syncthreads();
        s_cnt[t] += a; s_tl[t] += b;
        __syncthreads();
    }
    const int r0 = s_cnt[t] - c, tile0 = s_tl[t] - tl, n_routed = s_cnt[ROUTE_THREADS - 1];
    if (t < n_expert) {
        bounds[t] = r0; tile_start[t] = tile0;
        for (int j = 0; j < tl; ++j) tiles[tile0 + j] = make_int2(t, r0 + j * bn);
        if (t == n_expert - 1) { bounds[n_expert] = s_cnt[t]; tile_start[n_expert] = s_tl[t]; }
    }
    s_pos[t] = r0;
    __syncthreads();
    // the order of the slots inside an expert follows the atomics; a column's result does not depend on its position in the tile
    for (int s = t; s < n_slots; s += ROUTE_THREADS) {
        const int e = __ldg(ids + s);
        if (e >= 0 && e < n_expert) { const int r = atomicAdd(&s_pos[e], 1); slot[r] = s; col[r] = (s / n_used) * nb1 + (s % n_used) % nb1; }
    }
    for (int r = n_routed + t; r < n_slots; r += ROUTE_THREADS) col[r] = -1;        // gathered as zero rows
    // skipped slots: zero rows (one warp per slot, coalesced)
    const int warp = t >> 5, lane = t & 31;
    for (int s = warp; s < n_slots; s += ROUTE_THREADS / 32) {
        const int e = __ldg(ids + s);
        if (e >= 0 && e < n_expert) continue;
        for (int64_t m = lane; m < M; m += 32) { zero0[(int64_t)s * M + m] = 0.0f; if (zero1) zero1[(int64_t)s * M + m] = 0.0f; }
    }
}

// the tile width: BN = 256 once an average expert has that many rows
int moe_tile_rows(int64_t n_slots, int n_expert) { return n_slots >= (int64_t)256 * n_expert ? 256 : 128; }

struct moe_ws_layout { size_t bounds, tile_start, tiles, slot, col, xb, up, wsc, wsc_bytes, total; };
// rows_layout: rows of one expert matrix (M, or 2 M for merged up/gate experts, whose generic-type scratch holds both halves)
moe_ws_layout moe_layout(int type, int64_t M, int64_t K, int64_t n_slots, int n_expert, int up_gate, int64_t rows_layout) {
    moe_ws_layout L; size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (size_t)b200q_align_up((int64_t)bytes, 256); return o; };
    const int64_t max_tiles = (n_slots + 127) / 128 + std::min<int64_t>(n_expert, n_slots);
    L.bounds = take(sizeof(int) * (n_expert + 1)); L.tile_start = take(sizeof(int) * (n_expert + 1)); L.tiles = take(sizeof(int2) * max_tiles);
    L.slot = take(sizeof(int) * n_slots); L.col = take(sizeof(int) * n_slots);
    L.xb = take((size_t)n_slots * K * 2);
    L.up = up_gate ? take((size_t)n_slots * M * 4) : 0;
    const int64_t ebytes = rows_layout * K * 2;
    L.wsc_bytes = b200q_gemm_fused_type(type) ? 0 : (size_t)(std::min<int64_t>(n_expert, std::max<int64_t>(1, MOE_SCRATCH_BUDGET / ebytes)) * ebytes);
    L.wsc = take(L.wsc_bytes);
    L.total = off;
    return L;
}

// dst[t][i] = sum_u w[t][u] * rows[t][u][i] in slot order with the association of the reference CPU op (iqk_mul_multi_add: y = x0 w0, then
// y = y + x_u w_u), every product and sum rounded on its own (no FMA contraction): bit-equal to the same loop in f32 on the host.
// T = float4: m % 4 == 0 and 16-byte aligned rows / dst, one 16-byte load per slot and one 16-byte store; T = float otherwise.
__device__ __forceinline__ float comb_mul(float a, float s) { return __fmul_rn(a, s); }
__device__ __forceinline__ float4 comb_mul(float4 a, float s) { return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s), __fmul_rn(a.w, s)); }
__device__ __forceinline__ float comb_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float4 comb_add(float4 a, float4 b) { return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w)); }

template <typename T>
__global__ void __launch_bounds__(256)
k_moe_combine(const T * __restrict__ rows, const float * __restrict__ w, T * __restrict__ dst, int64_t mv, int n_used, int64_t total) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i / mv, c = i - t * mv;
        const T * r = rows + t * n_used * mv + c;
        const float * wt = w + t * n_used;
        T y = comb_mul(__ldg(r), __ldg(wt));
#pragma unroll 8
        for (int u = 1; u < n_used; ++u) y = comb_add(y, comb_mul(__ldg(r + u * mv), __ldg(wt + u)));
        dst[i] = y;
    }
}

__global__ void k_batch_ids(int32_t * __restrict__ ids, int n, int64_t total, int per_entry) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) ids[i] = per_entry ? (int32_t)(i / n) : 0;
}

}  // namespace

int b200q_launch_batch_ids(int32_t * ids, int n_batch, int n, int per_entry, cudaStream_t st) {
    const int64_t total = (int64_t)n_batch * n;
    const int64_t g = std::min<int64_t>((total + 255) / 256, 132 * 4);
    k_batch_ids<<<(unsigned)g, 256, 0, st>>>(ids, n, total, per_entry);
    return (int)cudaGetLastError();
}

int b200q_launch_moe_combine(const float * rows, const float * w, float * dst, int64_t m, int n_used, int n_tokens, cudaStream_t st) {
    const bool v4 = m % 4 == 0 && !((uintptr_t)rows & 15) && !((uintptr_t)dst & 15);
    const int64_t mv = v4 ? m / 4 : m, total = mv * n_tokens;
    const int64_t g = std::min<int64_t>((total + 255) / 256, 132 * 16);
    if (v4) k_moe_combine<float4><<<(unsigned)g, 256, 0, st>>>((const float4 *)rows, w, (float4 *)dst, mv, n_used, total);
    else k_moe_combine<float><<<(unsigned)g, 256, 0, st>>>(rows, w, dst, mv, n_used, total);
    return (int)cudaGetLastError();
}

// shapes the grouped path takes: K a multiple of 256 (the fused kernel's raw blocks, 16-byte TMA strides), a type the layout supports, at most
// 1024 experts (one routing thread each); for up/gate n_slots * M a multiple of 4 (the vectorised unary-mul tail)
int b200q_moe_gemm_shape_ok(int type, int64_t M, int64_t K, int n_used, int nb1, int n_tokens, int n_expert, int up_gate) {
    if (M < 1 || M > INT32_MAX / 2 || K < 256 || K % 256 || n_used < 1 || nb1 < 1 || n_used % nb1 || n_tokens < 1 || n_expert < 1 || n_expert > ROUTE_THREADS) return 0;
    const int64_t n_slots = (int64_t)n_tokens * n_used;
    if (n_slots > MOE_MAX_SLOTS || (up_gate && (n_slots * M) % 4)) return 0;
    b200q_layout L; return b200q_make_layout(type, M, K, &L) == 0 ? 1 : 0;
}

size_t b200q_moe_gemm_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_slots, int n_expert, int up_gate, int64_t rows_layout) {
    return moe_layout(type, M, K, n_slots, n_expert, up_gate, rows_layout).total;
}

int b200q_launch_moe_gemm(const b200q_mmvq_id_desc & d, void * ws, size_t ws_bytes, cudaStream_t st) {
    const bool ug = d.W2 != nullptr;
    if (!b200q_moe_gemm_shape_ok(d.type, d.M, d.K, d.n_used, d.nb1, d.n_tokens, d.n_expert, ug)) return -2;
    if (((uintptr_t)d.x & 15) || ((uintptr_t)ws & 255)) return -2;
    const int64_t n_slots = (int64_t)d.n_tokens * d.n_used;
    const moe_ws_layout L = moe_layout(d.type, d.M, d.K, n_slots, d.n_expert, ug, d.rows_layout);
    if (ws_bytes < L.total) return -5;
    char * b = (char *)ws;
    int * bounds = (int *)(b + L.bounds), * tile_start = (int *)(b + L.tile_start), * slot = (int *)(b + L.slot), * col = (int *)(b + L.col);
    int2 * tiles = (int2 *)(b + L.tiles);
    float * up = ug ? (float *)(b + L.up) : nullptr;
    const int bn = moe_tile_rows(n_slots, d.n_expert);
    k_moe_route<<<1, ROUTE_THREADS, 0, st>>>(d.ids, (int)n_slots, d.n_used, d.nb1, d.n_expert, bn, bounds, tile_start, tiles, slot, col, d.dst, up, d.M);
    int rc = (int)cudaGetLastError(); if (rc) return rc;
    if ((rc = b200q_launch_f32_to_bf16_rows(d.x, col, d.nb1, d.x_tok_stride, d.x_col_stride, b + L.xb, d.K, n_slots, st))) return rc;
    b200q_moe_gemm g{};
    g.type = d.type; g.n_seg = ug ? 2 : 1; g.W[0] = d.W; g.dst[0] = ug ? up : d.dst; g.W[1] = d.W2; g.dst[1] = d.dst;
    g.row0[0] = d.W_row0; g.row0[1] = d.W2_row0; g.rows_layout = d.rows_layout;
    g.M = d.M; g.K = d.K; g.n_expert = d.n_expert; g.n_rows = n_slots; g.xb = b + L.xb; g.bn = bn;
    g.rt = b200q_moe_route{bounds, tile_start, tiles, slot, 0, d.n_expert};
    if ((rc = b200q_launch_gemm_grouped(g, b + L.wsc, L.wsc_bytes, st))) return rc;
    if (ug) return b200q_launch_mul_unary(d.dst, up, d.dst, nullptr, n_slots * d.M, d.act, d.limit, st);
    return 0;
}
