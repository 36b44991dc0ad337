// b200q_decode_common.cuh — device helpers shared by the decode mat-vec kernels (b200q_decode.cu: plane-layout types, b200q_wire.cu: wire-layout types)
#pragma once
#include "b200q_internal.h"
#include <cuda_fp16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// programmatic dependent launch (no-ops unless the launch carries the PDL attribute)
__device__ __forceinline__ void pdl_wait()    { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- tagged-slot exchange (fused tensor-parallel decode reduce) ----
// An entry {value, id} is written with ONE 8-byte store (locally, or by a peer GPU through the NVLS multicast mapping), so a reader that sees the id
// of the reduce it waits for also sees the value: no fences, no separate flag, no acknowledgement round trip.
__device__ __forceinline__ float2 ll_load(const float2 * p) {
    float2 v; asm volatile("ld.volatile.global.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory"); return v;
}
// element e of reduce `id`: the sum over ranks in rank order (every rank and every CTA gets the same bits), waiting for the peers' entries.
// All ranks' entries are requested at once (one L2 round trip when the data is already there), then only the missing ones are polled again.
static __device__ __noinline__ float ll_sum_slots(const float2 * slots, int64_t stride, uint32_t world, int e, uint32_t id) {
    float2 v[8];
#pragma unroll
    for (uint32_t r = 0; r < 8; ++r) if (r < world) v[r] = ll_load(slots + (int64_t)r * stride + e);
    float acc = 0.0f;
#pragma unroll
    for (uint32_t r = 0; r < 8; ++r) if (r < world) {
        while (__float_as_uint(v[r].y) != id) v[r] = ll_load(slots + (int64_t)r * stride + e);
        acc += v[r].x;
    }
    for (uint32_t r = 8; r < world; ++r) {                       // (worlds beyond 8: one at a time)
        float2 w = ll_load(slots + (int64_t)r * stride + e);
        while (__float_as_uint(w.y) != id) w = ll_load(slots + (int64_t)r * stride + e);
        acc += w.x;
    }
    return acc;
}
struct ll_source { const float2 * red; const float2 * slots; int64_t stride; uint32_t world, id; };

// Quantise ncols activation columns into shared memory (q8_1 semantics of ggml-cuda/quantize.cu:13-47):
//   d = amax/127 ; q = amax == 0 ? 0 : roundf(x/d) ; d kept as float(half(d)) ; isum = packed int16 sums of q over each 16.
// Cooperative and vectorised: a thread owns 8 consecutive floats (two LDG.128), 4 adjacent lanes own one 32-block.
// LL = true (NCOLS = 1): the column is the result of a fused tensor-parallel reduce: entries of ll->red (summed by the CTA that owns the slice, see
// k_mmvq_ring); an entry whose tag is still old is summed here from the per-rank slots instead, so no CTA ever waits for a sibling CTA.
template <int NCOLS, bool LL = false>
__device__ __forceinline__ void quantize_x_to_smem(const float * __restrict__ x, int64_t x_stride, int64_t K,
                                                   int8_t * sq, float * sd, int * sis, int tid, int nthreads, unsigned long long * tr = nullptr,
                                                   const ll_source * ll = nullptr) {
    const int nch = (int)(K / 8), total = nch * NCOLS, n32 = (int)(K / 32);
    constexpr int B = 4;                                   // chunks per thread per batch: 8 independent LDG.128 in flight, so the
                                                           // activation vector costs 1 (K=4096) .. 2 (K=14336) L2 round trips, not 2 .. 6
    for (int base = 0; base < total; base += nthreads * B) {
        float4 va[B], vb[B];
#pragma unroll
        for (int u = 0; u < B; ++u) {
            const int c = base + u * nthreads + tid;
            int col = 0, ch = c < total ? c : 0;
            if (NCOLS > 1) { col = ch / nch; ch -= col * nch; }
            if (c < total && LL) {
                // All loads of a batch are issued together and the WHOLE batch is re-requested until every tag matches: one L2 round trip after the
                // data has arrived, however long the wait was (a per-entry wait would serialise eight round trips behind it).
                float t[8];
                const float4 * p0 = reinterpret_cast<const float4 *>((ll->world == 2 ? ll->slots : ll->red) + (int64_t)ch * 8);
                const float4 * p1 = reinterpret_cast<const float4 *>(ll->slots + ll->stride + (int64_t)ch * 8);
                bool ok = false;
                for (int spin = 0; spin < 64 && !ok; ++spin) {          // bounded: progress must not depend on a sibling CTA that is not resident
                    float4 w0[4], w1[4];
                    ok = true;
#pragma unroll
                    for (int j = 0; j < 4; ++j) { w0[j] = __ldcv(p0 + j); if (ll->world == 2) w1[j] = __ldcv(p1 + j); }
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        ok = ok && __float_as_uint(w0[j].y) == ll->id && __float_as_uint(w0[j].w) == ll->id;
                        if (ll->world == 2) {                           // two ranks: sum the two slots directly (no publish -> poll hop)
                            ok = ok && __float_as_uint(w1[j].y) == ll->id && __float_as_uint(w1[j].w) == ll->id;
                            t[2 * j] = w0[j].x + w1[j].x; t[2 * j + 1] = w0[j].z + w1[j].z;
                        } else { t[2 * j] = w0[j].x; t[2 * j + 1] = w0[j].z; }
                    }
                }
                if (!ok) {
#pragma unroll 1
                    for (int j = 0; j < 8; ++j) t[j] = ll_sum_slots(ll->slots, ll->stride, ll->world, ch * 8 + j, ll->id);
                }
                va[u] = make_float4(t[0], t[1], t[2], t[3]); vb[u] = make_float4(t[4], t[5], t[6], t[7]);
            } else if (c < total) {
                va[u] = __ldg(reinterpret_cast<const float4 *>(x + col * x_stride + (int64_t)ch * 8));
                vb[u] = __ldg(reinterpret_cast<const float4 *>(x + col * x_stride + (int64_t)ch * 8 + 4));
            } else { va[u] = make_float4(0.f, 0.f, 0.f, 0.f); vb[u] = va[u]; }
        }
        if (tr && base == 0 && va[0].x != 123456.789f) *tr = gtime();       // (debug trace) first batch of loads has landed
#pragma unroll
        for (int u = 0; u < B; ++u) {
            const int c = base + u * nthreads + tid;
            if (base + u * nthreads >= total) break;       // warp-uniform: the whole batch slot is past the end
            const bool valid = c < total;
            int col = 0, ch = valid ? c : 0;
            if (NCOLS > 1) { col = ch / nch; ch -= col * nch; }
            const float v[8] = {va[u].x, va[u].y, va[u].z, va[u].w, vb[u].x, vb[u].y, vb[u].z, vb[u].w};
            float amax = 0.0f;
#pragma unroll
            for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            // d = amax/127 exactly as the reference; q = rint(x * (1/d)) with a correctly rounded reciprocal: one division and one
            // reciprocal per block instead of one division per element.  Differs from the reference's roundf(x / d) only for
            // products within 1 ulp of a rounding tie (p ~ 1e-5 per element, 1 LSB); the oracle restates exactly this arithmetic
            // (oracle_quantize_q8_1_b200) next to the reference's (oracle_quantize_q8_1).
            const float d = __fdiv_rn(amax, 127.0f);
            const float inv = d > 0.0f ? __frcp_rn(d) : 0.0f;
            int q[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) q[j] = max(-127, min(127, __float2int_rn(__fmul_rn(v[j], inv))));
            int2 pk;
            pk.x = (int)__byte_perm(__byte_perm(q[0], q[1], 0x0040), __byte_perm(q[2], q[3], 0x0040), 0x5410);
            pk.y = (int)__byte_perm(__byte_perm(q[4], q[5], 0x0040), __byte_perm(q[6], q[7], 0x0040), 0x5410);
            int s = __dp4a(pk.x, 0x01010101, __dp4a(pk.y, 0x01010101, 0));
            s += __shfl_xor_sync(0xffffffffu, s, 1);                       // sum over 16 weights (2 lanes)
            const int s_hi = __shfl_down_sync(0xffffffffu, s, 2);          // the second 16 of the 32-block
            if (valid) {
                // natural order.  (Tried: two half planes [K/2 | K/2] so that the LDS.128 pairs of item_dot are conflict-free across the
                // warp -> slower; kept simple.)
                *reinterpret_cast<int2 *>(sq + (size_t)col * K + (size_t)ch * 8) = pk;
                if ((ch & 3) == 0) {
                    sd[col * n32 + (ch >> 2)]  = __half2float(__float2half_rn(d));
                    sis[col * n32 + (ch >> 2)] = (s & 0xFFFF) | (s_hi << 16);
                }
            }
        }
    }
}


