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
#include <string.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>

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

// the per-type kernel selections are instantiated in b200q_decode_i<N>.cu (parallel compilation)
#define X(T) extern template const void * mmvq_kernel<T>(const b200q_mmvq_plan &); \
             extern template const void * mmvq_id_kernel<T>(bool);
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

// ------------------------------------------------------------------------------------------------
// decode launch planning: which kernel serves a launch, with which template arguments, grid, block and shared memory
// ------------------------------------------------------------------------------------------------
// ring geometry for a type; returns false if the planes cannot be bulk-copied (alignment) -> LDG kernel
// long_rows: K > 4096: a stage holds up to 2 x B200Q_SEG_ITEMS items of ONE row (plane-major), else a pair of single-segment rows
static bool make_ring_geom(int type, int64_t K, ring_geom & g, bool long_rows) {
    b200q_layout L; if (b200q_make_layout(type, 1, K, &L)) return false;
    if (K % 32) return false;
    // K % 256 != 0 (32- / 64-weight block types only: bitnet's IQ2_BN rows of 3200 / 8640): fine as long as every plane row is a whole number of
    // bytes and stays 16-byte aligned (checked per plane below)
    const int64_t n32 = K / 32;
    memset(&g, 0, sizeof g); g.row_plane = -1;
    int off = 0, np = 0;
    for (int p = 0; p < L.n_planes; ++p) {
        if (L.plane_per_row[p]) { g.row_plane = p; continue; }
        if (p != np) return false;                       // block planes must come first (they do for every type)
        const int b8 = L.plane_bytes[p] * 256 / L.qk;
        if (b8 <= 0 || (n32 * b8) % 128) return false;   // every row/segment start must be 16-byte aligned: row bytes = n32 * b8 / 8
        g.b8[np] = b8; g.seg_off[np] = off; off += (int)b200q_align_up((B200Q_SEG_ITEMS / 8) * b8, 16); ++np;
    }
    g.n_planes = np; g.stage_bytes = (int)b200q_align_up(off, 128);
    for (int p = 0; p < np; ++p) g.row1[p] = g.stage_bytes;          // row-major stage: [row 0: planes][row 1: planes]
    // one segment per row: merge the two rows of a pair into one copy per plane (B200Q_MERGE_PAIR=0 restores the round-1 scheme)
    static const int merge = [] { const char * e = getenv("B200Q_MERGE_PAIR"); return e ? atoi(e) : 1; }();
    if (long_rows) {
        int o = 0;
        for (int p = 0; p < np; ++p) { const int hb = (B200Q_SEG_ITEMS / 8) * g.b8[p]; g.seg_off[p] = o; g.row1[p] = hb; o += (int)b200q_align_up(2 * hb, 16); }
        g.merged = 1;
    } else if (merge && K / 32 <= B200Q_SEG_ITEMS && np > 0 && np <= 4) {
        int o = 0;
        for (int p = 0; p < np; ++p) { const int rb = (int)((n32 * g.b8[p]) >> 3); g.seg_off[p] = o; g.row1[p] = rb; o += (int)b200q_align_up(2 * rb, 16); }
        if (o <= 2 * g.stage_bytes) g.merged = 1;
        else { int o2 = 0; for (int p = 0; p < np; ++p) { g.seg_off[p] = o2; o2 += (int)b200q_align_up((B200Q_SEG_ITEMS / 8) * g.b8[p], 16); g.row1[p] = g.stage_bytes; } }
    }
    return np > 0 && np <= 4;
}

// consumer warps / stages of a ring launch
static inline size_t ring_xbytes(int ncols, int64_t K) { return b200q_mmvq_x_bytes(ncols, K) + 512 + 512 + 256 + 128; }
static inline bool ring_shape(int ncols, int64_t K, size_t pair_stage, int64_t n_units, int sm_count, int & ncw, int & S) {
    const size_t xbytes = ring_xbytes(ncols, K), budget = B200Q_SMEM_BUDGET;
    ncw = B200Q_RING_CONSUMERS; S = 0;                   // consumer warps (+1 producer warp)
    for (;;) {
        const size_t per_stage = (size_t)ncw * (pair_stage + 16);
        S = xbytes + 64 < budget ? (int)((budget - xbytes - 64) / per_stage) : 0;
        if (S >= 2 || ncw == 3) break;
        ncw = ncw > 19 ? 19 : ncw > 15 ? 15 : ncw > 11 ? 11 : ncw > 7 ? 7 : 3;      // (10 warps would still fit two stages for K = 14336 but measured slower: 13.8 vs 11.3 us)
    }
    if (S < 2) return false;
    if (S > B200Q_MAX_STAGES) S = B200Q_MAX_STAGES;
    while (ncw > 3 && n_units <= (int64_t)sm_count * (ncw > 7 ? 7 : 3)) ncw = ncw > 7 ? 7 : 3;
    while (ncw * S > B200Q_PAIR_SLOTS) --S;
    return true;
}

// ceil(work / per_cta) CTAs, at least one, at most cap
static dim3 grid_for(int64_t work, int per_cta, int64_t cap) {
    int64_t grid = (work + per_cta - 1) / per_cta;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    return dim3((unsigned)grid);
}
// the wire-layout kernels run as many CTAs per SM as their shared memory allows
static int64_t wire_grid_cap(int sm_count, size_t smem) { return (int64_t)sm_count * (smem > 100 * 1024 ? 1 : smem > 48 * 1024 ? 2 : 4); }

// the TMA-ring launch of d (p.multi, p.tp and p.q8 already set), or false when the ring cannot serve it -> LDG kernel
static bool plan_ring(const b200q_mmvq_desc & d, int64_t M_total, b200q_mmvq_plan & p) {
    // row pairs amortise the activation loads; single rows give more, shorter units when the matrix is small
    const bool pair = d.K / 32 <= B200Q_SEG_ITEMS;         // K <= 4096: row pairs; longer rows: one row, up to 256 items per stage
    ring_geom g;
    if (!make_ring_geom(d.type, d.K, g, !pair)) return false;
    if (pair) for (int i = 0; i + 1 < d.n_seg; ++i) if (d.seg[i].M & 1) return false;     // row pairs must not straddle tensors
    if (M_total >= (int64_t)1 << 30) return false;
    const size_t pair_stage = 2 * (size_t)g.stage_bytes;
    const int64_t n_units = pair ? (M_total + 1) / 2 : M_total;
    int ncw, S;
    if (!ring_shape(d.ncols, d.K, pair_stage, n_units, d.sm_count, ncw, S)) return false;
    g.n_stages = S;
    size_t smem = (size_t)ncw * S * (pair_stage + 16) + ring_xbytes(d.ncols, d.K) + 64;
    static const int cps = [] { const char * e = getenv("B200Q_CTAS_PER_SM"); return e ? atoi(e) : B200Q_MIN_CTAS; }();
    // B200Q_GRID_FULL=1 (experiment): always spread over every SM, even when a CTA then has fewer units than consumer warps
    static const int grid_full = [] { const char * e = getenv("B200Q_GRID_FULL"); return e ? atoi(e) : 0; }();
    const dim3 grid = grid_for(n_units, grid_full ? 1 : ncw, (int64_t)d.sm_count * cps);
    if (d.tp.out && !p.multi) {
        // row buffer of a reduce_out launch: the rows of one CTA (a contiguous range, +-1 unit) are sent in one coalesced burst at the end
        const int64_t rows = (pair ? 2 : 1) * ((n_units + grid.x - 1) / grid.x + 1) + 2;
        // (measured at 2 GPUs: no gain, the extra CTA barrier costs more than the coalescing saves -> off by default, B200Q_TP_ROWBUF=1 enables it)
        static const int on_env = [] { const char * e = getenv("B200Q_TP_ROWBUF"); return e ? atoi(e) : -1; }();
        const bool on = on_env >= 0 ? on_env != 0 : d.tp.ll_peer[0] != nullptr;       // the coalescing only exists for the unicast stores
        if (on && rows <= 2048 && smem + rows * 4 + 16 <= B200Q_SMEM_BUDGET) {
            p.tp_rowbuf_off = (int)((smem + 15) & ~(size_t)15); p.tp_rowbuf_rows = (int)rows;
            smem = (size_t)p.tp_rowbuf_off + rows * 4;
        }
    }
    p.kernel = B200Q_MMVQ_RING; p.pair = pair; p.g = g; p.ncw = ncw;
    p.grid = grid; p.block = dim3((ncw + 1) * 32); p.smem = smem;
    return true;
}

// 0, or the error the launch of d returns
static int plan_mmvq(const b200q_mmvq_desc & d, b200q_mmvq_plan & p) {
    p = b200q_mmvq_plan{};
    if (d.n_seg < 1 || d.n_seg > B200Q_MAX_SEGS || d.ncols < 1 || d.ncols > 8) return -2;
    const bool tp = d.tp.in || d.tp.out, upgate = d.seg[0].W2 != nullptr;
    const bool ldg_cols = d.ncols == 1 || d.ncols == 2 || d.ncols == 4 || d.ncols == 8;      // the LDG kernels are instantiated for 1/2/4/8 columns
    int64_t M_total = 0;
    for (int i = 0; i < d.n_seg; ++i) M_total += d.seg[i].M;
    p.ncols = d.ncols; p.upgate = upgate;
    if (b200q_is_wire_type(d.type)) {                       // k_wire_mmvq: 8 warps, a warp per row
        if (tp) return -1;                                  // the fused reduce exists only in the ring kernel of the plane types
        for (int i = 0; i < d.n_seg; ++i) if (const int rc = b200q_wire_check(d.type, d.seg[i].M, d.K)) return rc;
        if ((upgate && d.n_seg != 1) || !ldg_cols) return -2;
        p.kernel = B200Q_MMVQ_WIRE; p.smem = b200q_mmvq_x_bytes(d.ncols, d.K);
        p.block = dim3(8 * 32); p.grid = grid_for(M_total, 8, wire_grid_cap(d.sm_count, p.smem));
        return 0;
    }
    for (int i = 0; i < d.n_seg; ++i) { b200q_layout L; if (const int rc = b200q_make_layout(d.type, d.seg[i].M, d.K, &L)) return rc; }
    // only the TMA-ring kernel implements the fused reduce: every other case is a shape error
    if (tp && (d.ncols != 1 || !d.ring || d.K % 256 || (d.tp.out && M_total > d.tp.ll_stride) || (d.tp.in && d.K > d.tp.ll_stride))) return -2;
    // q8 hand-off: n = 1, single tensor, ring kernel, bulk-copyable image; the up/gate launch emits it (q8 = 2), a plain launch consumes it (q8 = 1)
    const bool q8_ok = d.ncols == 1 && d.n_seg == 1 && d.ring && !tp
                    && (!d.q8_in || (d.K % 64 == 0 && !((uintptr_t)d.q8_in & 15)))
                    && (!d.q8_out || (upgate && d.seg[0].M % 64 == 0 && !((uintptr_t)d.q8_out & 15)));
    p.q8 = !q8_ok ? 0 : d.q8_out ? 2 : d.q8_in && !upgate ? 1 : 0;
    p.multi = !upgate && d.n_seg > 1; p.tp = tp;
    if (d.ring && d.ncols <= 2 && plan_ring(d, M_total, p)) return 0;
    if (tp) return -2;                                      // no ring geometry for this (type, K) or ring layout for this shape
    p.multi = p.tp = false; p.q8 = 0;
    if (!ldg_cols) return -2;
    // k_mmvq: one warp per row, one CTA per SM; shrink the CTA when there are fewer rows than warps
    int nwarps = 16;
    while (nwarps > 2 && M_total <= (int64_t)d.sm_count * (nwarps / 2)) nwarps >>= 1;
    p.kernel = B200Q_MMVQ_LDG; p.smem = b200q_mmvq_x_bytes(d.ncols, d.K);
    p.block = dim3(nwarps * 32); p.grid = grid_for(M_total, nwarps, d.sm_count);
    return 0;
}

// MoE decode: every activation column of the launch is quantised into shared memory; k_mmvq_id: 16 warps, at most one CTA per SM,
// k_wire_mmvq_id: 8 warps, as many CTAs per SM as the shared memory allows.  A warp owns one (slot, row) at a time.
int b200q_plan_mmvq_id(const b200q_mmvq_id_desc & d, b200q_mmvq_plan & p) {
    p = b200q_mmvq_plan{};
    const int64_t ncx = (int64_t)d.n_tokens * d.nb1;
    if (ncx > b200q_mmvq_max_cols(d.K)) return -2;
    const bool wire = b200q_is_wire_type(d.type);
    const int nwarps = wire ? 8 : 16;
    p.kernel = wire ? B200Q_MMVQ_WIRE : B200Q_MMVQ_LDG; p.upgate = d.W2 != nullptr;
    p.smem = b200q_mmvq_x_bytes(ncx, d.K); p.block = dim3(nwarps * 32);
    p.grid = grid_for((int64_t)(d.n_tokens * d.n_used) * d.M, nwarps, wire ? wire_grid_cap(d.sm_count, p.smem) : d.sm_count);
    return 0;
}

bool b200q_opt_in_smem(const void * kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return true;
    // function attributes are per device, and several host threads (one per GPU) may launch at once
    static std::mutex mu; static std::map<std::pair<const void *, int>, size_t> done;
    const int dev = b200q_current_device();
    std::lock_guard<std::mutex> lk(mu);
    size_t & cur = done[{kernel, dev}];
    if (bytes <= cur) return true;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) return false;
    cur = bytes;
    return true;
}

int b200q_launch_pdl(const void * kernel, dim3 grid, dim3 block, size_t smem, void * arg, bool pdl, cudaStream_t st) {
    cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof cfg);
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    void * args[1] = {arg};
    return (int)cudaLaunchKernelExC(&cfg, kernel, args);
}

// what the next decode launch (descriptor nx) will request first -> mmvq_pf (see struct mmvq_pf)
static void make_next_prefetch(const b200q_mmvq_desc & nx, mmvq_pf & pf) {
    memset(&pf, 0, sizeof pf);
    if (nx.n_seg < 1 || nx.ncols > 2 || nx.tp.in || nx.tp.out) return;
    const bool upgate = nx.seg[0].W2 != nullptr;
    int64_t M_total = 0; for (int i = 0; i < nx.n_seg; ++i) M_total += nx.seg[i].M;
    if (b200q_is_wire_type(nx.type)) {                   // wire-layout tensors: whole (or the head of) each tensor
        b200q_layout L;
        for (int i = 0; i < nx.n_seg && pf.n < 8; ++i) for (int t = 0; t < (upgate ? 2 : 1) && pf.n < 8; ++t) {
            if (b200q_make_layout(nx.type, nx.seg[i].M, nx.K, &L)) return;
            pf.ptr[pf.n] = (const uint8_t *)(t ? nx.seg[i].W2 : nx.seg[i].W); pf.bytes[pf.n] = std::min<long long>(L.M * b200q_wire_row_size(L), 24ll << 20); ++pf.n;
        }
        pf.mode = 0; return;
    }
    b200q_mmvq_plan np;
    if (plan_mmvq(nx, np) || np.kernel != B200Q_MMVQ_RING || nx.K % 256) return;
    const ring_geom & g = np.g;
    const int64_t n8 = nx.K / 256;
    const int64_t n_units = np.pair ? (M_total + 1) / 2 : M_total;
    long long total = 0;
    for (int i = 0; i < nx.n_seg; ++i) for (int p = 0; p < g.n_planes; ++p) total += (long long)nx.seg[i].M * n8 * g.b8[p] * (upgate ? 2 : 1);
    if (nx.n_seg > 1 || total <= (24ll << 20)) {         // small: everything, split evenly over our CTAs
        for (int i = 0; i < nx.n_seg; ++i) for (int t = 0; t < (upgate ? 2 : 1); ++t) {
            b200q_layout L; if (b200q_make_layout(nx.type, nx.seg[i].M, nx.K, &L)) return;
            const b200q_planes P = b200q_planes_from((const uint8_t *)(t ? nx.seg[i].W2 : nx.seg[i].W), L);
            for (int p = 0; p < g.n_planes && pf.n < 8; ++p) { pf.ptr[pf.n] = P.p[p]; pf.bytes[pf.n] = (long long)nx.seg[i].M * n8 * g.b8[p]; ++pf.n; }
        }
        pf.mode = 0; return;
    }
    // one (or up + gate) large tensor: the first stages of every CTA of the next grid
    const int nseg = np.pair ? 1 : (int)((nx.K / 32 + 2 * B200Q_SEG_ITEMS - 1) / (2 * B200Q_SEG_ITEMS)), nt = upgate ? 2 : 1;
    for (int t = 0; t < nt; ++t) {
        b200q_layout L; if (b200q_make_layout(nx.type, nx.seg[0].M, nx.K, &L)) return;
        const b200q_planes P = b200q_planes_from((const uint8_t *)(t ? nx.seg[0].W2 : nx.seg[0].W), L);
        for (int p = 0; p < g.n_planes && pf.n < 8; ++p) { pf.ptr[pf.n] = P.p[p]; pf.rowb[pf.n] = (int)(n8 * g.b8[p]); ++pf.n; }
    }
    pf.mode = 1; pf.n_units = (int)n_units; pf.rpu = np.pair ? 2 : 1; pf.grid = (int)np.grid.x;
    pf.per_cta = (np.ncw * g.n_stages + nseg * nt - 1) / (nseg * nt);
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
int b200q_launch_mmvq(const b200q_mmvq_desc & d, cudaStream_t st, b200q_mmvq_plan * plan) {
    b200q_mmvq_plan p;
    if (const int rc = plan_mmvq(d, p)) return rc;
    if (plan) *plan = p;
    if (p.kernel == B200Q_MMVQ_WIRE) return b200q_launch_wire_mmvq(d, p, st);
    mmvq_ring_args ra; memset(&ra, 0, sizeof ra);
    mmvq_args & a = ra.a;
    if (g_trace && g_trace_slot < 4096) { if (g_trace_cta && g_trace_slot < 512) a.trace_cta = g_trace_cta + (size_t)g_trace_slot * 2048; a.trace = g_trace + 8 * (g_trace_slot++); }
    int64_t r0 = 0;
    for (int i = 0; i < d.n_seg; ++i) {
        b200q_layout L; b200q_make_layout(d.type, d.seg[i].M, d.K, &L);
        a.seg[i].P = b200q_planes_from((const uint8_t *)d.seg[i].W, L);
        if (d.seg[i].W2) a.seg[i].P2 = b200q_planes_from((const uint8_t *)d.seg[i].W2, L);
        a.seg[i].dst = d.seg[i].dst; a.seg[i].bias = d.seg[i].bias; a.seg[i].M = d.seg[i].M; a.seg[i].row0 = r0; r0 += d.seg[i].M;
    }
    a.n_seg = d.n_seg; a.M_total = r0; a.K = d.K; a.x = d.x; a.x_stride = d.x_stride ? d.x_stride : d.K; a.act = d.act; a.limit = d.limit;
    a.tp = d.tp; a.tp_rowbuf_off = p.tp_rowbuf_off; a.tp_rowbuf_rows = p.tp_rowbuf_rows;
    if (p.q8 == 1) a.q8_in = d.q8_in;
    if (p.q8 == 2) a.q8_out = d.q8_out;
    if (d.next) make_next_prefetch(*d.next, a.pf);
    ra.g = p.g;
    const void * k = nullptr;
    switch (d.type) {
#define X(T) case T: k = mmvq_kernel<T>(p); break;
        B200Q_FOR_TYPES(X)
#undef X
        default: return -1;
    }
    if (!b200q_opt_in_smem(k, p.kernel == B200Q_MMVQ_RING ? B200Q_SMEM_BUDGET : p.smem)) return -3;
    return b200q_launch_pdl(k, p.grid, p.block, p.smem, p.kernel == B200Q_MMVQ_RING ? (void *)&ra : (void *)&a, d.pdl != 0, st);
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
    a.M = d.M; a.K = d.K; a.x = d.x; a.dst = d.dst; a.act = d.act; a.limit = d.limit; a.xs_tok = d.x_tok_stride; a.xs_col = d.x_col_stride;
    b200q_mmvq_plan p; if (const int prc = b200q_plan_mmvq_id(d, p)) return prc;
    const void * k = nullptr;
    switch (d.type) {
#define X(T) case T: k = mmvq_id_kernel<T>(p.upgate); break;
        B200Q_FOR_TYPES(X)
#undef X
        default: return -1;
    }
    if (!b200q_opt_in_smem(k, p.smem)) return -3;
    return b200q_launch_pdl(k, p.grid, p.block, p.smem, &a, d.pdl != 0, st);
}
