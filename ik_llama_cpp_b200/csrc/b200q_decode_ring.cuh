// b200q_decode_ring.cuh — the decode mat-vec kernels (k_mmvq, k_mmvq_ring, k_mmvq_id) and, per type, the kernel each launch plan selects.
// Included by b200q_decode.cu (planner and launcher; declares the per-type selections extern) and by the b200q_decode_i<N>.cu instantiation units,
// which split the 23 x 17 kernel instantiations over several translation units so that they compile in parallel.
#pragma once
#include "b200q_types.cuh"
#include "b200q_internal.h"
#include "b200q_decode_common.cuh"
#include "b200q_decode_plan.h"
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

// ------------------------------------------------------------------------------------------------
// decode mat-vec
// ------------------------------------------------------------------------------------------------
// L2 warm-up of the NEXT mat-vec's weights.  While this kernel runs, the next one cannot stream yet: its CTAs only become resident when ours leave
// (shared memory), and then need a full HBM round trip for their first stages before the first useful instruction.  The producer warp therefore issues cp.async.bulk.prefetch.L2 for exactly the bytes the next kernel's CTAs will
// request first; HBM works on them during OUR prologue / main loop, the next kernel's ring then fills from L2.
//   mode 0: whole ranges ptr[q] .. +bytes[q], split evenly over this grid (small tensors: Q,K,V / wo)
//   mode 1: plane q of a tensor whose units (rpu rows each, rowb[q] bytes per row) are split over `grid` CTAs like k_mmvq_ring does: the first
//           per_cta units of every next-CTA chunk
struct mmvq_pf { const uint8_t * ptr[8]; long long bytes[8]; int rowb[8]; int n; int mode; int n_units; int rpu; int grid; int per_cta; };
struct mmvq_seg {               // one weight tensor of a multi-tensor launch (Q,K,V share the activation)
    b200q_planes    P;          // resolved plane pointers
    b200q_planes    P2;         // second tensor (gate) for the fused up/gate mode
    float *         dst;        // [ncols][M] f32 (ggml: dst[j*M + i])
    const float *   bias;       // optional [M]
    int64_t         M;
    int64_t         row0;       // first global row index of this segment
};
struct mmvq_args {
    mmvq_seg     seg[B200Q_MAX_SEGS];
    int          n_seg;
    int64_t      M_total;
    int64_t      K;
    const float * x;            // [ncols][K] f32, row stride x_stride floats
    int64_t      x_stride;
    int          act;           // B200Q_ACT_* for the up/gate mode
    float        limit;         // clamp for swiglu variants (0 = none)
    int tp_rowbuf_off, tp_rowbuf_rows;   // reduce_out: byte offset (in dynamic smem) / capacity of the CTA's row buffer (0 rows: send every row pair on its own)
    unsigned long long * trace_cta;   // tuning builds (B200Q_TRACE_FINE): per-CTA timeline, 4 words per CTA
    b200q_tp_comm tp;           // tensor-parallel decode: GGML_OP_REDUCE fused into the mat-vec (tp.in / tp.out), see k_mmvq_ring
    unsigned long long * trace; // optional phase timestamps (b200q_debug_trace): [slot][8] = entry, after griddepcontrol.wait, prologue done, last consumer done,
                                //   activation loads landed, quantised (before the barrier), 2^62 - first consumer done, first unit of CTA 0 / warp 1 done
    mmvq_pf pf;                 // weights of the NEXT decode launch to warm in L2 (b200q_decode_prefetch_next), pf.n == 0: none
    const void * q8_in;         // activations already quantised by the producing kernel (b200q_q8 layout, n = 1): bulk-copied instead of re-quantised
    void *       q8_out;        // fused up/gate, n = 1: also emit dst quantised to q8_1 for the following MUL_MAT (ffn_down), see q8_emit_block
};
// ---- q8 hand-off between two mat-vec launches (n = 1) -------------------------------------------------------------
// Layout of a b200q_q8 scratch for a vector of K floats (K % 64 == 0): [K int8 q][K/32 f32 d][K/32 i32 packed int16 sums]
// = exactly the shared-memory image (sq | sd | sis) the mat-vec consumes, followed by [K/32 u32 arrival counters].
// Producer side (fused up/gate epilogue): the warp that completes the LAST rows of a 32-block (arrival counter) quantises that
// block from the f32 results in L2 with the arithmetic of quantize_x_to_smem; consumer side: one bulk copy instead of
// 296 CTAs re-reading and re-quantising K floats (reference: quantize_q8_1 runs once per activation, quantize.cu:13-47).
__device__ __forceinline__ void q8_emit_block(void * q8, int64_t K, const float * dst, int64_t M, int blk, int lane) {
    int8_t * q8q = reinterpret_cast<int8_t *>(q8);
    float * q8d = reinterpret_cast<float *>(q8q + K);
    int * q8s = reinterpret_cast<int *>(q8d + K / 32);
    const int64_t r = (int64_t)blk * 32 + lane;
    const float v = r < M ? __ldcg(dst + r) : 0.0f;
    float amax = fabsf(v);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = __fdiv_rn(amax, 127.0f);
    const float inv = d > 0.0f ? __frcp_rn(d) : 0.0f;
    const int q = max(-127, min(127, __float2int_rn(__fmul_rn(v, inv))));
    q8q[r] = (int8_t)q;
    const int s_lo = __reduce_add_sync(0xffffffffu, lane < 16 ? q : 0), s_hi = __reduce_add_sync(0xffffffffu, lane < 16 ? 0 : q);
    if (lane == 0) { q8d[blk] = __half2float(__float2half_rn(d)); q8s[blk] = (s_lo & 0xFFFF) | (s_hi << 16); }
}

template <int TYPE, int NCOLS>
__device__ __forceinline__ void item_dot(const b200q_canon & C, const int8_t * sq, const float * sd, const int * sis,
                                         int64_t K, int n32, int it, float acc[NCOLS]) {
    constexpr bool HAS_B = b200q_traits<TYPE>::HAS_B;
#pragma unroll
    for (int c = 0; c < NCOLS; ++c) {
        const int4 * xp = reinterpret_cast<const int4 *>(sq + (size_t)c * K + (size_t)it * 32);
        const int4 x0 = xp[0], x1 = xp[1];
        int s0 = 0, s1 = 0;
        s0 = b200q_dp4a(C.va[0], x0.x, s0); s0 = b200q_dp4a(C.va[1], x0.y, s0); s0 = b200q_dp4a(C.va[2], x0.z, s0); s0 = b200q_dp4a(C.va[3], x0.w, s0);
        s1 = b200q_dp4a(C.va[4], x1.x, s1); s1 = b200q_dp4a(C.va[5], x1.y, s1); s1 = b200q_dp4a(C.va[6], x1.z, s1); s1 = b200q_dp4a(C.va[7], x1.w, s1);
        if (HAS_B) {
            s0 = b200q_dp4a(C.vb[0], x0.x, s0); s0 = b200q_dp4a(C.vb[1], x0.y, s0); s0 = b200q_dp4a(C.vb[2], x0.z, s0); s0 = b200q_dp4a(C.vb[3], x0.w, s0);
            s1 = b200q_dp4a(C.vb[4], x1.x, s1); s1 = b200q_dp4a(C.vb[5], x1.y, s1); s1 = b200q_dp4a(C.vb[6], x1.z, s1); s1 = b200q_dp4a(C.vb[7], x1.w, s1);
        }
        const float d8 = sd[c * n32 + it];
        float t;
        if (b200q_split16(TYPE)) t = C.dl[0] * (float)s0 + C.dl[1] * (float)s1;
        else                     t = C.dl[0] * (float)(s0 + s1);
        if (b200q_mmvq_has_ml(TYPE)) {
            const int is = sis[c * n32 + it];
            if (b200q_split16(TYPE)) t -= C.ml[0] * (float)(int)(short)(is & 0xFFFF) + C.ml[1] * (float)(is >> 16);
            else                     t -= C.ml[0] * (float)((int)(short)(is & 0xFFFF) + (is >> 16));
        }
        acc[c] = fmaf(d8, t, acc[c]);
    }
}

// One CTA per SM (512 threads = 16 warps, <= 64 registers): leaves half of the SM for the NEXT kernel of the graph,
// which under programmatic dependent launch is already resident, has its first weight batch in flight and is parked
// in griddepcontrol.wait while this one drains.
template <int TYPE, int NCOLS, bool UPGATE>
__global__ void __launch_bounds__(512, (NCOLS == 1 ? 2 : 1)) k_mmvq(const mmvq_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int64_t K = a.K; const int n32 = (int)(K / 32);
    int8_t * sq = reinterpret_cast<int8_t *>(smem_raw);
    float *  sd = reinterpret_cast<float *>(smem_raw + (size_t)NCOLS * K);
    int *    sis = reinterpret_cast<int *>(sd + NCOLS * n32);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * nwarps + warp, tw = (int64_t)gridDim.x * nwarps;
    constexpr int U = UPGATE ? 2 : 4;

    auto locate = [&](int64_t grow, int & s, int64_t & row) {
        s = 0;
#pragma unroll
        for (int i = 1; i < B200Q_MAX_SEGS; ++i) if (i < a.n_seg && grow >= a.seg[i].row0) s = i;
        row = grow - a.seg[s].row0;
    };

    // (1) weights do not depend on the previous kernel: get the first batch of this warp's first row in flight now
    b200q_item I[U], J[U];
    int64_t grow = gw;
    if (grow < a.M_total) {
        int s; int64_t row; locate(grow, s, row);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int it = lane + 32 * u;
            if (it < n32) { b200q_load_item<TYPE>(I[u], a.seg[s].P, row, it); if (UPGATE) b200q_load_item<TYPE>(J[u], a.seg[s].P2, row, it); }
        }
    }
    pdl_trigger();                       // let the next kernel of the stream/graph become resident
    // (2) the activations are produced by the previous kernel
    pdl_wait();
    quantize_x_to_smem<NCOLS>(a.x, a.x_stride, K, sq, sd, sis, threadIdx.x, blockDim.x);
    __shared__ uint32_t kv_slot[128];
    const b200q_kv4 T = b200q_kv4_init_via_smem(kv_slot);     // includes the __syncthreads() that publishes the activations
    for (; grow < a.M_total; grow += tw) {
        int s; int64_t row; locate(grow, s, row);
        const mmvq_seg & sg = a.seg[s];
        float acc[NCOLS], acc2[NCOLS];
#pragma unroll
        for (int c = 0; c < NCOLS; ++c) { acc[c] = 0.0f; acc2[c] = 0.0f; }

        for (int it0 = lane; it0 < n32; it0 += 32 * U) {
            if (it0 != lane || grow != gw) {          // the very first batch is already in registers
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int it = it0 + 32 * u;
                    if (it < n32) { b200q_load_item<TYPE>(I[u], sg.P, row, it); if (UPGATE) b200q_load_item<TYPE>(J[u], sg.P2, row, it); }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int it = it0 + 32 * u;
                if (it < n32) {
                    b200q_canon C;
                    b200q_decode_item<TYPE>(I[u], it, C, T);
                    item_dot<TYPE, NCOLS>(C, sq, sd, sis, K, n32, it, acc);
                    if (UPGATE) { b200q_decode_item<TYPE>(J[u], it, C, T); item_dot<TYPE, NCOLS>(C, sq, sd, sis, K, n32, it, acc2); }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < NCOLS; ++c) {
            float v = warp_sum(acc[c]);
            if (UPGATE) {
                float g = warp_sum(acc2[c]);      // acc = up . x, acc2 = gate . x
                v = b200q_glu<false>(a.act, g, v, a.limit);
            } else if (sg.bias) v += sg.bias[row];
            if (lane == 0) sg.dst[(int64_t)c * sg.M + row] = v;
        }
    }
}


// ------------------------------------------------------------------------------------------------
// MoE decode: GGML_OP_MUL_MAT_ID / GGML_OP_MOE_FUSED_UP_GATE for small batches (reference: mul_mat_vec_q with `ids`, blockIdx.y = expert slot,
// mmvq-templates.cuh:293-302; ggml_cuda_mul_mat_id / ggml_cuda_moe_up_gate_unary, ggml-cuda.cu:2836-3540).  Slot s = (token t, used expert e):
//     dst[s][:] = W[ids[s]] . x[col(s)][:]          (W2 != nullptr: unary(W2[ids[s]] . x) * (W[ids[s]] . x))
// One launch over all slots: the expert index is read on the DEVICE (no host round trip), every distinct activation column is quantised once
// per CTA, a warp owns one (slot, row) at a time.  LDG kernel (same inner loop as k_mmvq).
// ------------------------------------------------------------------------------------------------
struct mmvq_id_args {
    b200q_planes P, P2;             // planes of expert 0 of W (and of the gate tensor)
    int64_t estride;                // bytes between consecutive experts (same in every plane)
    const int32_t * ids;            // [n_slots] expert per slot
    int n_expert, n_slots, n_used, nb1, ncx;   // slots = n_tokens * n_used; x columns = n_tokens * nb1, column of slot s = (s / n_used) * nb1 + (s % n_used) % nb1
    int64_t M, K; const float * x; float * dst; int act; float limit;
    int64_t xs_tok, xs_col;         // column c = t * nb1 + j starts at x + t * xs_tok + j * xs_col
};
template <int TYPE, bool UPGATE>
__global__ void __launch_bounds__(512, 1) k_mmvq_id(const mmvq_id_args a) {
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
    __shared__ uint32_t kv_slot[128];
    const b200q_kv4 T = b200q_kv4_init_via_smem(kv_slot);     // includes the __syncthreads() that publishes the activations
    constexpr int U = UPGATE ? 2 : 4;
    const int64_t total = (int64_t)a.n_slots * a.M;
    for (int64_t g = (int64_t)blockIdx.x * nwarps + warp; g < total; g += (int64_t)gridDim.x * nwarps) {
        const int s = (int)(g / a.M); const int64_t row = g - (int64_t)s * a.M;
        const int e = __ldg(a.ids + s);
        if (e < 0 || e >= a.n_expert) {             // skipped slot (the -1 of ggml_top_k_thresh): a zero row, no weights read; s is warp-uniform
            if (lane == 0) a.dst[(int64_t)s * a.M + row] = 0.0f;
            continue;
        }
        const int col = (s / a.n_used) * a.nb1 + (s % a.n_used) % a.nb1;
        b200q_planes P = a.P, P2 = a.P2;
#pragma unroll
        for (int p = 0; p < B200Q_MAX_PLANES; ++p) { P.p[p] += (int64_t)e * a.estride; P2.p[p] += (int64_t)e * a.estride; }
        float acc[1] = {0.0f}, acc2[1] = {0.0f};
        for (int it0 = lane; it0 < n32; it0 += 32 * U) {
            b200q_item I[U], J[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int it = it0 + 32 * u;
                if (it < n32) { b200q_load_item<TYPE>(I[u], P, row, it); if (UPGATE) b200q_load_item<TYPE>(J[u], P2, row, it); }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int it = it0 + 32 * u;
                if (it < n32) {
                    b200q_canon C;
                    b200q_decode_item<TYPE>(I[u], it, C, T);
                    item_dot<TYPE, 1>(C, sq + (size_t)col * K, sd + col * n32, sis + col * n32, K, n32, it, acc);
                    if (UPGATE) { b200q_decode_item<TYPE>(J[u], it, C, T); item_dot<TYPE, 1>(C, sq + (size_t)col * K, sd + col * n32, sis + col * n32, K, n32, it, acc2); }
                }
            }
        }
        float v = warp_sum(acc[0]);
        if (UPGATE) { const float gt = warp_sum(acc2[0]); v = b200q_glu<false>(a.act, gt, v, a.limit); }
        if (lane == 0) a.dst[(int64_t)s * a.M + row] = v;
    }
}
template <int TYPE>
const void * mmvq_id_kernel(bool upgate) { return upgate ? (const void *)k_mmvq_id<TYPE, true> : (const void *)k_mmvq_id<TYPE, false>; }

// ------------------------------------------------------------------------------------------------
// decode mat-vec, TMA-ring variant (the default): weights are streamed HBM -> shared memory by cp.async.bulk (1-D TMA)
// into warp-private rings, decoupled from registers and from the data dependency on the previous kernel.
//   * every warp owns S stages; a stage holds one SEGMENT (<= 128 items = 4096 weights) of one row of one tensor:
//     one bulk copy per plane (rows are contiguous inside a plane), completion on a per-stage mbarrier (expect_tx);
//   * lane 0 refills a stage as soon as the warp has consumed it, so W*S*stage bytes (~74 KB/SM) stay in flight
//     (tools/membench.cu compares bulk-copy rings with LDG streams at several depths);
//   * the first S units of every warp are issued BEFORE griddepcontrol.wait: under programmatic dependent launch the
//     next mat-vec of the graph is already resident (one 512-thread CTA per SM leaves room for a second) and has its
//     ring full when the previous kernel finishes; only the activation quantisation is on the dependent path.
// ------------------------------------------------------------------------------------------------
#ifndef B200Q_SEG_ITEMS
#define B200Q_SEG_ITEMS 128          // items (of 32 weights) per row per ring stage; tuning knob (scripts/build_variant.sh)
#endif
#ifndef B200Q_MAX_STAGES
#define B200Q_MAX_STAGES 4
#endif
#ifndef B200Q_RING_CONSUMERS
#define B200Q_RING_CONSUMERS 11      // consumer warps per CTA (+1 producer): 12 warps x 2 CTAs per SM at <= 80 registers.  Round-2 knob: 15 with
#endif                               // -maxrregcount 64 gives 32 warps per SM (more latency hiding) if the ring stages are shrunk to fit
#ifndef B200Q_TRACE_FINE
#define B200Q_TRACE_FINE 0           // 1: extra phase timestamps (slots 4..7 of b200q_debug_trace); costs registers / branches, tuning builds only
#endif
#ifndef B200Q_PRODUCER_LAST
#define B200Q_PRODUCER_LAST 0        // 1: the producer is the LAST warp of the CTA (the warp scheduler prefers high warp ids: B300_MICROARCH.md)
#endif
#ifndef B200Q_EXP_PREFILL_AFTER_WAIT
#define B200Q_EXP_PREFILL_AFTER_WAIT 0
#endif
#ifndef B200Q_EXP_LATE_TRIGGER
#define B200Q_EXP_LATE_TRIGGER 0
#endif
#ifndef B200Q_MIN_CTAS
#define B200Q_MIN_CTAS 2             // resident CTAs per SM the ring kernel is compiled for (register cap = 65536 / (MIN_CTAS * threads))
#endif
#ifndef B200Q_SMEM_BUDGET
#define B200Q_SMEM_BUDGET (112 * 1024)   // dynamic shared memory per CTA: two CTAs per SM (same kernel, or this one + the next under PDL)
#endif
#define B200Q_PAIR_SLOTS 124         // ncw * S stage descriptors (+ the claim counter) fit the 128-int slot table
struct mmvq_ring_args {
    mmvq_args  a;
    ring_geom  g;
};

__device__ __forceinline__ uint32_t smem_addr(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void rb_init(uint64_t * bar) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(bar))); }
__device__ __forceinline__ void rb_expect(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void rb_wait(uint64_t * bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tRW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra RD_%=;\n\tbra RW_%=;\n\tRD_%=:\n\t}"
                 ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ bool rb_test(uint64_t * bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void * dst, const void * src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}

// ---- tensor-parallel fusion (split-mode-graph): the partial rows of a row-parallel mat-vec are broadcast to every rank by the switch ----
// one multimem.st = one NVLink write that the NVSwitch replicates into every rank's copy of the slot; {value, tag} travel together (8 bytes)
__device__ __forceinline__ void tp_bcast1(float2 * mc, float v, uint32_t id) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(mc), "f"(v), "f"(__uint_as_float(id)) : "memory");
}
__device__ __forceinline__ void tp_bcast2(float2 * mc, float v0, float v1, uint32_t id) {       // two adjacent rows: 16 bytes, 16-byte aligned
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v0), "f"(__uint_as_float(id)), "f"(v1), "f"(__uint_as_float(id)) : "memory");
}
// the same entries as ordinary stores into ONE rank's copy (peer memory): lanes that write consecutive 16-byte entries are coalesced by the LSU into
// 128-byte NVLink packets, which the multicast stores above are not (one packet per lane)
__device__ __forceinline__ void tp_ucast1(float2 * p, float v, uint32_t id) {
    asm volatile("st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(v), "f"(__uint_as_float(id)) : "memory");
}
__device__ __forceinline__ void tp_ucast2(float2 * p, float v0, float v1, uint32_t id) {
    asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v0), "f"(__uint_as_float(id)), "f"(v1), "f"(__uint_as_float(id)) : "memory");
}

__device__ __forceinline__ void rb_arrive(uint64_t * bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory"); }

__device__ __forceinline__ void bulk_prefetch_l2(const uint8_t * p, long long bytes) {
    for (long long o = 0; o < bytes; o += 32768) {
        const uint32_t n = (uint32_t)min(32768ll, bytes - o);
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p + o), "r"(n) : "memory");
    }
}
__device__ __forceinline__ void issue_next_prefetch(const mmvq_pf & pf, int lane) {
    if (lane >= pf.n) return;
    if (pf.mode == 0) {
        const long long per = ((pf.bytes[lane] / 16 + gridDim.x - 1) / gridDim.x) * 16, o = per * blockIdx.x;
        if (o < pf.bytes[lane]) bulk_prefetch_l2(pf.ptr[lane] + o, min(per, pf.bytes[lane] - o));
    } else {
        for (int j = blockIdx.x; j < pf.grid; j += gridDim.x) {
            const long long c0 = (long long)pf.n_units * j / pf.grid, c1 = (long long)pf.n_units * (j + 1) / pf.grid;
            const long long cnt = min((long long)pf.per_cta, c1 - c0);
            if (cnt > 0) bulk_prefetch_l2(pf.ptr[lane] + c0 * pf.rpu * pf.rowb[lane], cnt * pf.rpu * pf.rowb[lane]);
        }
    }
}

// Warp 0 = producer (lane l streams the units of consumer warp l), warps 1..NCW = consumers.
// A stage holds 2 x B200Q_SEG_ITEMS items (8192 weights) and is filled by ONE bulk copy per plane (fewer, larger bulk copies in flight per SM
// stream faster; tools/membench.cu measures it):
//   PAIR = true  (K <= 4096, the row is one segment): a unit is a PAIR of adjacent output rows: inside every plane the two rows are adjacent, so they
//                travel together; they share every activation load and all loop bookkeeping and give two independent dependency chains;
//   PAIR = false (K > 4096, "long rows"): a unit is a segment of up to 256 items of ONE row (contiguous inside every plane); lane l owns items
//                l + 32 i of both halves of the segment, the two halves are the two dependency chains.
// TP: tensor-parallel instantiation (fused GGML_OP_REDUCE); a separate instantiation so that the single-GPU kernels carry none of it
// (as runtime branches the extra code slowed the plain path down)
// Q8: 0 = none, 1 = activations arrive as a b200q_q8 image (a.q8_in), 2 = fused up/gate also emits its result as one (a.q8_out)
template <int TYPE, int NCOLS, bool UPGATE, bool MULTI, bool PAIR, bool TP, int Q8 = 0>
__global__ void __launch_bounds__(32 * (B200Q_RING_CONSUMERS + 1), B200Q_MIN_CTAS) k_mmvq_ring(const mmvq_ring_args ra) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const mmvq_args & a = ra.a; const ring_geom & g = ra.g;
    const int K = (int)a.K, n32 = K / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ncw = (blockDim.x >> 5) - 1;     // consumer warps
    const bool is_prod = B200Q_PRODUCER_LAST ? warp == ncw : warp == 0;
    const int cw = B200Q_PRODUCER_LAST ? warp : warp - 1;                                         // consumer index (producer: out of range)
    const int ctid = cw * 32 + lane, cthreads = ncw * 32;                                         // thread index among the consumers
    const bool lead = cw == 0 && lane == 0;                                                       // first consumer thread (flag waits, trace)
    const int S = g.n_stages;
    const int row_stage = g.stage_bytes, pair_stage = 2 * row_stage;
    // smem carve-up: [ring: ncw*S pair-stages][full barriers ncw*S][empty barriers ncw*S][kv table 128 words][x: sq | sd | sis]
    unsigned char * ring0 = smem_raw;
    uint64_t * full0  = reinterpret_cast<uint64_t *>(smem_raw + (size_t)ncw * S * pair_stage);
    uint64_t * empty0 = full0 + ncw * S;
    uint32_t * kv_slot = reinterpret_cast<uint32_t *>(empty0 + ncw * S);
    int * pair_id = reinterpret_cast<int *>(kv_slot + 128);       // [ncw*S] pair index streamed into each stage (-1 = end)
    int * next_pair = pair_id + B200Q_PAIR_SLOTS;                 // CTA-wide claim counter ([1]: finished consumer warps (tp.out))
    uint64_t * xbar = reinterpret_cast<uint64_t *>(next_pair + 2); // completion of the q8_in bulk copy
    uint32_t * k16tab = reinterpret_cast<uint32_t *>(kv_slot + 128 + 128 + 64);   // 32 x 65536 at lane-dependent addresses (B200Q_SHR_VIA_IMAD)
    unsigned char * xbase = reinterpret_cast<unsigned char *>(kv_slot + 128 + 128 + 64 + 32);
    int8_t * sq = reinterpret_cast<int8_t *>(xbase);
    float *  sd = reinterpret_cast<float *>(xbase + (size_t)NCOLS * K);
    int *    sis = reinterpret_cast<int *>(sd + NCOLS * n32);

    constexpr int SEGI = PAIR ? B200Q_SEG_ITEMS : 2 * B200Q_SEG_ITEMS;   // items of one row per stage
    const int nseg = (n32 + SEGI - 1) / SEGI;
    constexpr int NT = UPGATE ? 2 : 1;                            // tensors per row (up, gate)
    constexpr int RPU = PAIR ? 2 : 1;                             // rows per unit
    const int n_pairs = (int)((a.M_total + RPU - 1) / RPU);       // unit p = rows RPU*p (.. +1) (segments have even row counts)
    // static split of the pairs over CTAs (+-1 pair), dynamic claiming inside the CTA: the producer lane of a consumer
    // warp takes the next pair from a shared counter whenever that warp's ring has room, so warps never idle on a
    // coarse static remainder (2.2 pairs/warp for the FFN up/gate shape would otherwise mean 3 for some, 2 for others)
    const int c0 = (int)(((int64_t)n_pairs * blockIdx.x) / gridDim.x), c1 = (int)(((int64_t)n_pairs * (blockIdx.x + 1)) / gridDim.x);
    auto locate = [&](int grow, int & s, int & row) {
        s = 0; row = grow;
        if (MULTI) {
#pragma unroll
            for (int i = 1; i < B200Q_MAX_SEGS; ++i) if (i < a.n_seg && grow >= (int)a.seg[i].row0) s = i;
            row = grow - (int)a.seg[s].row0;
        }
    };

    if (a.trace && blockIdx.x == 0 && threadIdx.x == 0) a.trace[0] = gtime();
    if (is_prod) {
        for (int i = lane; i < ncw * S; i += 32) { rb_init(&full0[i]); rb_init(&empty0[i]); }
        if (Q8 == 1 && lane == 0) rb_init(xbar);
        kv_slot[lane * 4 + 0] = B200Q_KV4_A0; kv_slot[lane * 4 + 1] = B200Q_KV4_A1; kv_slot[lane * 4 + 2] = B200Q_KV4_B0; kv_slot[lane * 4 + 3] = B200Q_KV4_B1;
        if (lane == 0) { *next_pair = c0; next_pair[1] = 0; }    // [1]: consumer warps that have finished (tp.out)
        k16tab[lane] = 65536u;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        __syncwarp();
    }

    // ---------------- producer state (warp 0, lane = consumer warp index) ----------------
    int pcur = -1, pt = 0, psg = 0, pst = 0, pu = 0; bool pdone = !(is_prod && lane < ncw);
    auto produce_one = [&]() {                                    // issue the next unit of consumer warp `lane` into stage pst
        uint64_t * fb = &full0[lane * S + pst];
        if (pt == 0 && psg == 0) { pcur = atomicAdd(next_pair, 1); if (pcur >= c1) pcur = -1; }
        pair_id[lane * S + pst] = pcur;
        if (pcur < 0) { rb_arrive(fb); pdone = true; return; }   // sentinel: nothing left for this consumer
        int s, row; locate(RPU * pcur, s, row);
        const mmvq_seg & sgm = a.seg[MULTI ? s : 0];
        const b200q_planes & P = (UPGATE && pt == 1) ? sgm.P2 : sgm.P;
        const int gi = min(SEGI, n32 - psg * SEGI);               // items of this segment; bytes of plane p = gi * b8[p] / 8 (exact: make_ring_geom)
        const bool two = PAIR && row + 1 < (int)sgm.M;
        unsigned char * dstb = ring0 + ((size_t)lane * S + pst) * pair_stage;
        uint32_t bytes = 0;
#pragma unroll
        for (int p = 0; p < 4; ++p) if (p < g.n_planes) bytes += (uint32_t)((gi * g.b8[p]) >> 3);
        rb_expect(fb, two ? 2 * bytes : bytes);
#pragma unroll
        for (int p = 0; p < 4; ++p) if (p < g.n_planes) {
            const int64_t rowb = ((int64_t)n32 * g.b8[p]) >> 3;
            const uint32_t sb = (uint32_t)((gi * g.b8[p]) >> 3);
            const uint8_t * src = P.p[p] + (int64_t)row * rowb + (int64_t)psg * (SEGI / 8) * g.b8[p];
            if (!PAIR || g.merged) bulk_g2s(dstb + g.seg_off[p], src, (two ? 2 : 1) * sb, fb);
            else {
                bulk_g2s(dstb + g.seg_off[p], src, sb, fb);
                if (two) bulk_g2s(dstb + g.row1[p] + g.seg_off[p], src + rowb, sb, fb);
            }
        }
        ++pu; if (++pst == S) pst = 0;
        if (++psg == nseg) { psg = 0; if (++pt == NT) pt = 0; }
    };
    // (1) weights do not depend on the previous kernel: fill the ring before waiting for it
#if B200Q_EXP_PREFILL_AFTER_WAIT          // experiment: no memory traffic of this grid before the previous one has completed
    pdl_trigger();
    pdl_wait();
    if (is_prod) { for (int s = 0; s < S; ++s) if (!pdone) produce_one(); }
#else
    if (is_prod) {
        for (int s = 0; s < S; ++s) if (!pdone) produce_one();
        if (a.pf.n) issue_next_prefetch(a.pf, lane);       // after our own first stages: the next kernel's first stages -> L2
    }
#if !B200Q_EXP_LATE_TRIGGER
    pdl_trigger();                       // the next kernel of the stream/graph may become resident and fill ITS ring
#endif
    pdl_wait();                          // (2) the activations are produced by the previous kernel
#endif
    if (a.trace && blockIdx.x == 0 && lead) a.trace[1] = gtime();
    // Tensor-parallel mode.  seq[0] = fused reduces this rank has issued (device counter, so the launch arguments are constant under CUDA-graph
    // replay); it cannot change while this grid runs before its own last CTA bumps it.  A reduce_out launch issues reduce number tps + 1 into
    // parity tps & 1; a reduce_in launch consumes reduce number tps (parity (tps - 1) & 1).  Entries carry the number as their tag, so nothing is
    // ever zeroed and stale data of the reduce two steps back (same parity) can never be mistaken for the current one.
    uint32_t tps = 0;
    if (TP && (a.tp.in || a.tp.out)) tps = *reinterpret_cast<volatile uint32_t *>(a.tp.seq);
    if (!is_prod) {
        if (TP && a.tp.in) {
            const int64_t par = (tps - 1) & 1;
            ll_source src; src.slots = a.tp.ll_local + par * a.tp.world * a.tp.ll_stride; src.red = a.tp.ll_red + par * a.tp.ll_stride;
            src.stride = a.tp.ll_stride; src.world = a.tp.world; src.id = tps;
            // (1) this CTA sums its slice of the vector over the ranks (waiting for the peers' rows to arrive) and publishes it for its siblings,
            // (2) every CTA quantises the whole vector from the published sums (falling back to the slots for entries that are not there yet)
            const int e0 = (int)(((int64_t)K * blockIdx.x) / gridDim.x), e1 = (int)(((int64_t)K * (blockIdx.x + 1)) / gridDim.x);
            if (a.tp.world > 2) for (int e = e0 + ctid; e < e1; e += cthreads) {
                const float sum = ll_sum_slots(src.slots, src.stride, src.world, e, src.id);
                asm volatile("st.volatile.global.v2.f32 [%0], {%1,%2};" ::"l"(a.tp.ll_red + par * a.tp.ll_stride + e), "f"(sum), "f"(__uint_as_float(src.id)) : "memory");
#if B200Q_TRACE_FINE
                if (a.trace && blockIdx.x == 0 && e == e0) a.trace[4] = gtime();      // every rank's entry for this CTA's first element has arrived
#endif
            }
            quantize_x_to_smem<NCOLS, true>(nullptr, 0, K, sq, sd, sis, ctid, cthreads, nullptr, &src);
        } else if (Q8 == 1) {
            // quantised once by the producing kernel: nothing to do here, the producer warp bulk-copies the image (below)
        } else {
#if B200Q_TRACE_FINE
            quantize_x_to_smem<NCOLS>(a.x, a.x_stride, K, sq, sd, sis, ctid, cthreads, a.trace && blockIdx.x == 0 && lead ? a.trace + 4 : nullptr);
#else
            quantize_x_to_smem<NCOLS>(a.x, a.x_stride, K, sq, sd, sis, ctid, cthreads);
#endif
        }
#if B200Q_TRACE_FINE
        if (a.trace && blockIdx.x == 0 && lead) a.trace[5] = gtime();
#endif
    } else if (Q8 == 1 && lane == 0) {
        const uint32_t bytes = (uint32_t)(K + 8 * n32);
        rb_expect(xbar, bytes);
        bulk_g2s(sq, a.q8_in, bytes, xbar);
    }
    __syncthreads();                     // publishes barriers, kv table and activations
    if (Q8 == 1 && !is_prod) rb_wait(xbar, 0);
    if (a.trace && blockIdx.x == 0 && lead) a.trace[2] = gtime();

    if (is_prod) {
        // ---------------- producer: refill a stage as soon as its consumer has released it ----------------
        // All lanes poll their consumer's empty barrier with a NON-blocking test_wait and stay converged: a lane parked in a
        // blocking try_wait would stall the refills of the other ten consumers that share this warp.
        uint32_t epar = 1;               // first pass over the ring: the S initial units are already issued
        int k = 0;
        while (__any_sync(0xffffffffu, !pdone)) {
            bool ready = false;
            if (!pdone) ready = rb_test(&empty0[lane * S + pst], epar ^ 1);
            if (ready) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                produce_one();
                if (++k == S) { k = 0; epar ^= 1; }
            }
            if (!__any_sync(0xffffffffu, ready)) __nanosleep(64);
        }
#if B200Q_EXP_LATE_TRIGGER
        pdl_trigger();                   // experiment: the next grid is launched only when this CTA has issued its last weight copy
#endif
        return;
    }

    // ---------------- consumers ----------------
    b200q_kv4 T; T.a0 = kv_slot[lane * 4 + 0]; T.a1 = kv_slot[lane * 4 + 1]; T.b0 = kv_slot[lane * 4 + 2]; T.b1 = kv_slot[lane * 4 + 3];
    T.k16 = k16tab[lane];
    unsigned char * ring = ring0 + (size_t)cw * S * pair_stage;
    uint64_t * fullb = full0 + cw * S, * emptyb = empty0 + cw * S;
    float acc0[NCOLS], acc1[NCOLS], up0[NCOLS], up1[NCOLS];
    int t = 0, sg = 0;
    int cs = 0, crow = 0; float rs[2][2] = {{0.0f, 0.0f}, {0.0f, 0.0f}};
    int st = 0; uint32_t parity = 0;
    for (;;) {
        rb_wait(&fullb[st], parity);
        const int pid = pair_id[cw * S + st];
        if (pid < 0) break;
        if (sg == 0) {
#pragma unroll
            for (int c = 0; c < NCOLS; ++c) { acc0[c] = 0.0f; acc1[c] = 0.0f; }
            if (t == 0) {
                locate(RPU * pid, cs, crow);
                if (b200q_row_plane(TYPE) >= 0) {              // per-row scales straight from global memory
                    const mmvq_seg & sgm = a.seg[MULTI ? cs : 0];
                    const int r1 = min(crow + 1, (int)sgm.M - 1);
                    rs[0][0] = __ldg(reinterpret_cast<const float *>(sgm.P.p[b200q_row_plane(TYPE)]) + crow);
                    rs[0][1] = __ldg(reinterpret_cast<const float *>(sgm.P.p[b200q_row_plane(TYPE)]) + r1);
                    if (UPGATE) { rs[1][0] = __ldg(reinterpret_cast<const float *>(sgm.P2.p[b200q_row_plane(TYPE)]) + crow);
                                  rs[1][1] = __ldg(reinterpret_cast<const float *>(sgm.P2.p[b200q_row_plane(TYPE)]) + r1); }
                }
            }
        }
        const int items = min(SEGI, n32 - sg * SEGI);                 // items of this row in the stage (LONG: both halves together)
        b200q_planes SP0, SP1;
#pragma unroll
        for (int p = 0; p < 4; ++p) { SP0.p[p] = ring + (size_t)st * pair_stage + g.seg_off[p < g.n_planes ? p : 0]; SP1.p[p] = SP0.p[p] + g.row1[p < g.n_planes ? p : 0]; }
        SP0.p[4] = SP1.p[4] = nullptr; SP0.nb = SP1.nb = 0; SP0.n32 = SP1.n32 = 0;
        const float rsa = rs[UPGATE ? t : 0][0], rsb = rs[UPGATE ? t : 0][1];
        // PAIR: item itl of row 0 (SP0) and of row 1 (SP1) against the same activations; LONG: items itl and itl + 128 of the same row (SP1 = SP0 + 128
        // items in every plane) against their own activations; acc1 is the second dependency chain either way
        auto do_item = [&](int itl, bool second) {
            b200q_item I0, I1; b200q_canon C;
            b200q_load_item<TYPE, b200q_ld_plain, false, int>(I0, SP0, 0, itl);
            if (second) b200q_load_item<TYPE, b200q_ld_plain, false, int>(I1, SP1, 0, itl);
            I0.rs = rsa; I1.rs = PAIR ? rsb : rsa;
            const int it = sg * SEGI + itl;
            b200q_decode_item<TYPE>(I0, itl, C, T);
            item_dot<TYPE, NCOLS>(C, sq, sd, sis, K, n32, it, acc0);
            if (second) { b200q_decode_item<TYPE>(I1, itl, C, T); item_dot<TYPE, NCOLS>(C, sq, sd, sis, K, n32, PAIR ? it : it + B200Q_SEG_ITEMS, acc1); }
        };
        if (items == SEGI) {
#pragma unroll
            for (int i = 0; i < B200Q_SEG_ITEMS / 32; ++i) do_item(lane + 32 * i, true);
        } else if (PAIR) {
            for (int itl = lane; itl < items; itl += 32) do_item(itl, true);
        } else {
            for (int itl = lane; itl < min(items, B200Q_SEG_ITEMS); itl += 32) do_item(itl, itl + B200Q_SEG_ITEMS < items);
        }
        __syncwarp();
        if (lane == 0) rb_arrive(&emptyb[st]);                  // stage may be overwritten by the producer
        if (++st == S) { st = 0; parity ^= 1; }
        if (++sg == nseg) {
            sg = 0;
            const mmvq_seg & sgm = a.seg[MULTI ? cs : 0];
            if (UPGATE && t == 0) {
#pragma unroll
                for (int c = 0; c < NCOLS; ++c) { up0[c] = acc0[c]; up1[c] = acc1[c]; }      // up . x (still per-lane partials)
                t = 1;
            } else {
                const bool two = PAIR && crow + 1 < (int)sgm.M;
#pragma unroll
                for (int c = 0; c < NCOLS; ++c) {
                    // four (two) independent butterfly chains interleave in the pipeline
                    float v0 = acc0[c], v1 = acc1[c], u0 = UPGATE ? up0[c] : 0.0f, u1 = UPGATE ? up1[c] : 0.0f;
                    if (!PAIR) { v0 += v1; u0 += u1; }                            // long rows: the two chains belong to the same row
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        v0 += __shfl_xor_sync(0xffffffffu, v0, o); if (PAIR) v1 += __shfl_xor_sync(0xffffffffu, v1, o);
                        if (UPGATE) { u0 += __shfl_xor_sync(0xffffffffu, u0, o); if (PAIR) u1 += __shfl_xor_sync(0xffffffffu, u1, o); }
                    }
                    if (UPGATE) {                                                 // v = gate . x, u = up . x
                        v0 = b200q_glu<false>(a.act, v0, u0, a.limit); if (PAIR) v1 = b200q_glu<false>(a.act, v1, u1, a.limit);
                    } else if (sgm.bias) { v0 += sgm.bias[crow]; if (two) v1 += sgm.bias[crow + 1]; }
                    if (lane == 0) {
                        if (TP && a.tp.out) {
                            // partial rows of a row-parallel mat-vec.  Optional (B200Q_TP_ROWBUF=1): collect the rows of this CTA (a contiguous range) in
                            // shared memory and send them as contiguous 16-byte lanes of one warp at the end (fewer, larger packets)
                            const int rel = (int)sgm.row0 + crow - RPU * c0;
                            if (a.tp_rowbuf_rows > 0 && rel >= 0 && rel + 1 < a.tp_rowbuf_rows) {
                                float * rb = reinterpret_cast<float *>(smem_raw + a.tp_rowbuf_off);
                                rb[rel] = v0; if (two) rb[rel + 1] = v1;
                            } else {
                                const int64_t off = ((int64_t)(tps & 1) * a.tp.world + a.tp.rank) * a.tp.ll_stride + (int64_t)sgm.row0 + crow;
                                const bool al = two && !(((int64_t)sgm.row0 + crow) & 1);
                                if (a.tp.ll_peer[0]) {
                                    for (uint32_t r = 0; r < a.tp.world; ++r) {
                                        if (al) tp_ucast2(a.tp.ll_peer[r] + off, v0, v1, tps + 1);
                                        else { tp_ucast1(a.tp.ll_peer[r] + off, v0, tps + 1); if (two) tp_ucast1(a.tp.ll_peer[r] + off + 1, v1, tps + 1); }
                                    }
                                } else {
                                    float2 * mc = a.tp.ll_mc + off;
                                    if (al) tp_bcast2(mc, v0, v1, tps + 1);
                                    else { tp_bcast1(mc, v0, tps + 1); if (two) tp_bcast1(mc + 1, v1, tps + 1); }
                                }
                            }
                        } else { sgm.dst[(int64_t)c * sgm.M + crow] = v0; if (two) sgm.dst[(int64_t)c * sgm.M + crow + 1] = v1; }
                    }
                }
#if B200Q_TRACE_FINE
                if (a.trace && blockIdx.x == 0 && lead && a.trace[7] == 0) a.trace[7] = gtime();
#endif
                t = 0;
            }
        }
    }
    if (Q8 == 2) {
        // q8 hand-off, producer side: once every consumer warp of this CTA has stored its rows (bar.sync: their stores are performed with respect to
        // the whole CTA), the CTA quantises the 32-row blocks of its static row range [RPU c0, RPU c1): blocks that lie inside the range directly,
        // the (at most two) blocks shared with a neighbouring CTA through an arrival counter: the CTA whose rows complete the block quantises it.
        // One fence + atomic per SHARED block per CTA (a __threadfence per row pair costs far more).
        asm volatile("bar.sync 1, %0;" ::"r"(cthreads) : "memory");
        const mmvq_seg & sgm = a.seg[0];
        const int M = (int)sgm.M, r0 = min(RPU * c0, M), r1 = min(RPU * c1, M);
        uint32_t * cnt0 = reinterpret_cast<uint32_t *>(reinterpret_cast<int8_t *>(a.q8_out) + sgm.M + 8 * (sgm.M / 32));
        if (r1 > r0) for (int blk = (r0 >> 5) + cw; blk <= ((r1 - 1) >> 5); blk += ncw) {
            const int lo = max(r0, 32 * blk), hi = min(r1, 32 * blk + 32), need = min(32, M - 32 * blk), own = hi - lo;
            bool mine = own == need;
            if (!mine) {
                int old = 0;
                if (lane == 0) { __threadfence(); old = (int)atomicAdd(cnt0 + blk, (uint32_t)own); }
                old = __shfl_sync(0xffffffffu, old, 0);
                mine = old + own == need;
                if (mine) { __threadfence(); if (lane == 0) cnt0[blk] = 0; }
            }
            if (mine) q8_emit_block(a.q8_out, sgm.M, sgm.dst, sgm.M, blk, lane);
        }
    }
    if (TP && a.tp.out && a.tp_rowbuf_rows > 0) {
        asm volatile("bar.sync 1, %0;" ::"r"(cthreads) : "memory");           // every consumer warp of the CTA has deposited its rows
        const int r0 = RPU * c0, r1 = min(RPU * c1, (int)a.M_total), n = min(r1 - r0, a.tp_rowbuf_rows - 1);
        const float * rb = reinterpret_cast<const float *>(smem_raw + a.tp_rowbuf_off);
        const int64_t off = ((int64_t)(tps & 1) * a.tp.world + a.tp.rank) * a.tp.ll_stride + r0;
        if (a.tp.ll_peer[0]) {
            // unicast: consumer warp w serves ranks w, w + ncw, ...; one warp-wide store of consecutive 16-byte entries per 64 rows
            for (uint32_t r = (uint32_t)cw; r < a.tp.world; r += (uint32_t)ncw) {
                float2 * p = a.tp.ll_peer[(r + a.tp.rank) % a.tp.world] + off;          // start with the own copy, then the peers in ring order
                if (!(r0 & 1)) {
                    for (int i = 2 * lane; i + 1 < n; i += 64) tp_ucast2(p + i, rb[i], rb[i + 1], tps + 1);
                    if ((n & 1) && lane == 0) tp_ucast1(p + n - 1, rb[n - 1], tps + 1);
                } else for (int i = lane; i < n; i += 32) tp_ucast1(p + i, rb[i], tps + 1);
            }
        } else if (cw == 0) {
            float2 * mc = a.tp.ll_mc + off;
            if (!(r0 & 1)) {                                                   // 16-byte lanes: {v, tag, v', tag}
                for (int i = 2 * lane; i + 1 < n; i += 64) tp_bcast2(mc + i, rb[i], rb[i + 1], tps + 1);
                if ((n & 1) && lane == 0) tp_bcast1(mc + n - 1, rb[n - 1], tps + 1);
            } else for (int i = lane; i < n; i += 32) tp_bcast1(mc + i, rb[i], tps + 1);
        }
    }
    if (TP && a.tp.out) {
        // bookkeeping only (the data needs no completion signal: every entry carries its tag): the last warp of the last CTA advances the
        // rank-local count of issued reduces, which the next launch of this stream reads after its griddepcontrol.wait
        if (lane == 0) {
            if (atomicAdd(next_pair + 1, 1) == ncw - 1) {
                if (atomicAdd(a.tp.seq + 1, 1u) == gridDim.x - 1) {
                    a.tp.seq[1] = 0;
                    *reinterpret_cast<volatile uint32_t *>(a.tp.seq) = tps + 1;
                }
            }
        }
    }
#if B200Q_TRACE_FINE
    if (a.trace && lane == 0) {
        const unsigned long long tt = gtime(); atomicMax(a.trace + 3, tt); atomicMax(a.trace + 6, (1ull << 62) - tt);
        if (a.trace_cta && blockIdx.x < 512) {                       // per-CTA timeline: [end of last warp, SM id, units of the CTA, end of first warp]
            unsigned long long * tc = a.trace_cta + 4 * blockIdx.x; unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            atomicMax(tc, tt); tc[1] = smid; tc[2] = (unsigned long long)(c1 - c0); atomicMax(tc + 3, (1ull << 62) - tt);
        }
    }
#else
    if (a.trace && lane == 0) atomicMax(a.trace + 3, gtime());
#endif
}

// the kernel a plan (plan_mmvq) launches for this type.  The kernels are referenced (and so emitted) in the order of the instantiations
// they had before, which keeps ptxas' output for them unchanged.
template <int TYPE, int NCOLS, bool UPGATE, bool MULTI, bool PAIR, bool TP = false, int Q8 = 0>
static const void * ring_kernel() { return (const void *)k_mmvq_ring<TYPE, NCOLS, UPGATE, MULTI, PAIR, TP, Q8>; }
template <int TYPE, int NCOLS, bool UPGATE, bool MULTI>
static const void * ring_kernel(const b200q_mmvq_plan & p) {
    if (p.tp) return p.pair ? ring_kernel<TYPE, 1, UPGATE, MULTI, true, true>() : ring_kernel<TYPE, 1, UPGATE, MULTI, false, true>();
    if (p.q8 == 2) return p.pair ? ring_kernel<TYPE, 1, true, false, true, false, 2>() : ring_kernel<TYPE, 1, true, false, false, false, 2>();
    if (p.q8 == 1) return p.pair ? ring_kernel<TYPE, 1, false, false, true, false, 1>() : ring_kernel<TYPE, 1, false, false, false, false, 1>();
    return p.pair ? ring_kernel<TYPE, NCOLS, UPGATE, MULTI, true>() : ring_kernel<TYPE, NCOLS, UPGATE, MULTI, false>();
}
template <int TYPE>
const void * mmvq_kernel(const b200q_mmvq_plan & p) {
    if (p.kernel == B200Q_MMVQ_RING) {
        if (p.upgate) return p.ncols == 1 ? ring_kernel<TYPE, 1, true, false>(p) : ring_kernel<TYPE, 2, true, false>(p);
        if (p.multi) return p.ncols == 1 ? ring_kernel<TYPE, 1, false, true>(p) : ring_kernel<TYPE, 2, false, true>(p);
        return p.ncols == 1 ? ring_kernel<TYPE, 1, false, false>(p) : ring_kernel<TYPE, 2, false, false>(p);
    }
#define CASE(N) case N: return p.upgate ? (const void *)k_mmvq<TYPE, N, true> : (const void *)k_mmvq<TYPE, N, false>;
    switch (p.ncols) { CASE(1) CASE(2) CASE(4) CASE(8) default: return nullptr; }
#undef CASE
}
