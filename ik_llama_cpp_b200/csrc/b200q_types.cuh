// b200q_types.cuh — wire formats -> device layout ("planes") -> canonical decode.
//
// The wire format of every type is the reference's GGUF payload, consumed verbatim
// (reference: ggml/src/ggml-common.h:166-775 block_* structs; value tables :2212-2250).
// Those AoS blocks (18 B, 210 B, 4-byte row headers, ...) are only 2-byte aligned, which
// rules out 16-byte vector loads and TMA boxes.  On upload (set_tensor) each tensor is
// therefore re-laid-out ONCE into structure-of-planes form with identical total size:
//
//     plane p of a tensor [M rows x K cols]:  base + plane_off[p] + (row*nb + blk)*BYTES[p]
//
// where nb = K/QK is the number of wire blocks per row and plane_off[] are 256-byte aligned.
// Inside a plane the bit order is chosen so that the decode kernels need no cross-lane
// shuffles: every 32 weights ("item") own 16 contiguous bytes of low bits whose nibble order
// makes `(w & 0x0F0F0F0F)` / PRMT-lookups produce int8 lanes in NATURAL k order, matching
// a q8_1-quantised activation vector stored in natural order.
// The mapping is a bijection (b200q_unrepack restores the wire bytes bit-for-bit), so
// get_tensor / state save stay exact — same contract as the reference's run-time repack (-rtr).
//
// Canonical decode of one item (32 consecutive weights of one row), shared by the decode
// mat-vec (b200q_mmvq.cu), the bf16 dequantiser and the wgmma prefill kernel (b200q_gemm.cu):
//
//     w[e] = dl[e/16] * q[e] - ml[e/16],    q[e] = int8(va byte e) (+ int8(vb byte e) if HAS_B)
//
// Everything here is __host__ __device__ so that tests/test_host_emulation.py can run the
// exact same bit manipulation on the CPU (compiled with g++) against the oracle.
#pragma once
#include <stdint.h>
#include <string.h>
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif

#if defined(__CUDACC__)
#define B200Q_HD __host__ __device__ __forceinline__
#else
#define B200Q_HD inline
#endif

// ggml_type ids (reference ggml/include/ggml.h:391-492)
enum b200q_type : int {
    B200Q_TYPE_Q4_0 = 2, B200Q_TYPE_Q4_1 = 3, B200Q_TYPE_Q5_0 = 6, B200Q_TYPE_Q5_1 = 7, B200Q_TYPE_Q6_0 = 133, B200Q_TYPE_Q8_0 = 8, B200Q_TYPE_Q2_K = 10, B200Q_TYPE_Q3_K = 11, B200Q_TYPE_Q4_K = 12, B200Q_TYPE_Q5_K = 13, B200Q_TYPE_Q6_K = 14,
    B200Q_TYPE_IQ4_NL = 20, B200Q_TYPE_IQ4_XS = 23, B200Q_TYPE_MXFP4 = 39, B200Q_TYPE_IQ5_KS = 152, B200Q_TYPE_IQ2_KS = 145, B200Q_TYPE_IQ3_KS = 156, B200Q_TYPE_IQ2_BN = 135, B200Q_TYPE_IQ2_K = 137, B200Q_TYPE_IQ3_K = 138, B200Q_TYPE_IQ4_K = 139,
    B200Q_TYPE_IQ5_K = 140, B200Q_TYPE_IQ4_KS = 144,
};

// ---------------------------------------------------------------------------------------------
// small portable intrinsics
// ---------------------------------------------------------------------------------------------
B200Q_HD int b200q_dp4a(int a, int b, int c) {
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, c);
#else
    for (int i = 0; i < 4; ++i) c += (int)(int8_t)(a >> (8 * i)) * (int)(int8_t)(b >> (8 * i));
    return c;
#endif
}
// PTX prmt.b32 (default mode): selector nibble = {bit3: replicate sign of the selected byte, bits0-2: byte index in {a,b}}
B200Q_HD uint32_t b200q_prmt(uint32_t a, uint32_t b, uint32_t s) {
#if defined(__CUDA_ARCH__)
    // NOT __byte_perm(): the intrinsic masks the selector with 0x7777, which removes the sign-replicate mode we rely on
    uint32_t r; asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(s)); return r;
#else
    uint64_t ab = ((uint64_t)b << 32) | a; uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        uint32_t sel = (s >> (4 * i)) & 0xF; uint32_t byte = (uint32_t)(ab >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) byte = (byte & 0x80) ? 0xFF : 0x00;
        r |= byte << (8 * i);
    }
    return r;
#endif
}
B200Q_HD float b200q_u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
B200Q_HD float b200q_h2f(uint16_t h) {
#if defined(__CUDA_ARCH__)
    return __half2float(__ushort_as_half(h));
#else
    uint32_t s = (uint32_t)(h & 0x8000) << 16, e = (h >> 10) & 0x1f, m = h & 0x3ff, u;
    if (e == 0) { if (m == 0) u = s; else { int sh = 0; while (!(m & 0x400)) { m <<= 1; ++sh; } m &= 0x3ff; u = s | ((uint32_t)(113 - sh) << 23) | (m << 13); } }
    else if (e == 31) u = s | 0x7f800000u | (m << 13);
    else u = s | ((e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &u, 4); return f;
#endif
}

// f32 -> f16 for values that are exactly representable in f16 (used to restore a half row scale from its f32 plane copy)
B200Q_HD uint16_t b200q_f2h_exact(float f) {
    uint32_t u; memcpy(&u, &f, 4);
    const uint32_t s = (u >> 16) & 0x8000u, e = (u >> 23) & 0xFF, m = u & 0x7FFFFFu;
    if (e == 0xFF) return (uint16_t)(s | 0x7C00u | (m ? (0x200u | (m >> 13)) : 0));      // inf / NaN (payload top bits)
    if (e == 0) return (uint16_t)s;                                                      // +-0 (f32 subnormals cannot come from a half)
    const int eh = (int)e - 127 + 15;
    if (eh >= 31) return (uint16_t)(s | 0x7C00u);
    if (eh <= 0) { if (eh < -10) return (uint16_t)s; return (uint16_t)(s | ((m | 0x800000u) >> (14 - eh))); }   // f16 subnormal
    return (uint16_t)(s | ((uint32_t)eh << 10) | (m >> 13));
}

// ---------------------------------------------------------------------------------------------
// wire-layout types (decoded by b200q_wire.cuh): kept in their GGUF byte layout, no plane repack
// ---------------------------------------------------------------------------------------------
enum b200q_wire_type : int {
    B200Q_TYPE_IQ2_XXS = 16, B200Q_TYPE_IQ2_XS = 17, B200Q_TYPE_IQ3_XXS = 18, B200Q_TYPE_IQ1_S = 19, B200Q_TYPE_IQ3_S = 21, B200Q_TYPE_IQ2_S = 22, B200Q_TYPE_IQ1_M = 29,
    B200Q_TYPE_IQ1_BN = 134, B200Q_TYPE_IQ6_K = 141, B200Q_TYPE_IQ4_KSS = 146, B200Q_TYPE_IQ2_KT = 153, B200Q_TYPE_IQ3_KT = 154, B200Q_TYPE_IQ4_KT = 155,
    B200Q_TYPE_IQ2_KL = 157, B200Q_TYPE_IQ1_KT = 158,
    B200Q_TYPE_IQ1_S_R4 = 219, B200Q_TYPE_IQ1_M_R4 = 229, B200Q_TYPE_IQ2_K_R4 = 337, B200Q_TYPE_IQ3_K_R4 = 338, B200Q_TYPE_IQ4_K_R4 = 339, B200Q_TYPE_IQ5_K_R4 = 340,
    B200Q_TYPE_IQ4_KS_R4 = 344, B200Q_TYPE_IQ5_KS_R4 = 352,
};

// per-ROW wire geometry: weights per block, bytes per block, bytes of row header, rows interleaved on the wire (1 or 4)
struct b200q_wire_geom { int qk, block_bytes, row_meta, interleave; };
B200Q_HD bool b200q_wire_geom_of(int type, b200q_wire_geom & g) {
    switch (type) {
        case B200Q_TYPE_IQ2_XXS: g = {256, 66, 0, 1}; return true;
        case B200Q_TYPE_IQ2_XS:  g = {256, 74, 0, 1}; return true;
        case B200Q_TYPE_IQ3_XXS: g = {256, 98, 0, 1}; return true;
        case B200Q_TYPE_IQ2_S:   g = {256, 82, 0, 1}; return true;
        case B200Q_TYPE_IQ3_S:   g = {256, 110, 0, 1}; return true;
        case B200Q_TYPE_IQ1_S:   g = {256, 50, 0, 1}; return true;
        case B200Q_TYPE_IQ1_M:   g = {256, 56, 0, 1}; return true;
        case B200Q_TYPE_IQ6_K:   g = {256, 212, 0, 1}; return true;
        case B200Q_TYPE_IQ4_KSS: g = {256, 128, 4, 1}; return true;
        case B200Q_TYPE_IQ2_KL:  g = {256, 86, 2, 1}; return true;
        case B200Q_TYPE_IQ1_BN:  g = {64, 13, 2, 1}; return true;
        case B200Q_TYPE_IQ1_KT:  g = {256, 56, 4, 1}; return true;
        case B200Q_TYPE_IQ2_KT:  g = {256, 68, 4, 1}; return true;
        case B200Q_TYPE_IQ3_KT:  g = {256, 100, 4, 1}; return true;
        case B200Q_TYPE_IQ4_KT:  g = {256, 128, 4, 1}; return true;
        case B200Q_TYPE_IQ1_S_R4: g = {32, 6, 2, 4}; return true;
        case B200Q_TYPE_IQ1_M_R4: g = {32, 7, 2, 4}; return true;
        case B200Q_TYPE_IQ2_K_R4: g = {256, 76, 0, 4}; return true;
        case B200Q_TYPE_IQ3_K_R4: g = {256, 110, 0, 4}; return true;
        case B200Q_TYPE_IQ4_K_R4: g = {256, 144, 0, 4}; return true;
        case B200Q_TYPE_IQ5_K_R4: g = {256, 176, 0, 4}; return true;
        case B200Q_TYPE_IQ4_KS_R4: g = {256, 136, 4, 4}; return true;
        case B200Q_TYPE_IQ5_KS_R4: g = {256, 168, 4, 4}; return true;
        default: return false;
    }
}
B200Q_HD bool b200q_is_wire_type(int type) { b200q_wire_geom g; return b200q_wire_geom_of(type, g); }
B200Q_HD int64_t b200q_wire_type_row_size(const b200q_wire_geom & g, int64_t K) { return (int64_t)g.row_meta + (K / g.qk) * g.block_bytes; }

// ---------------------------------------------------------------------------------------------
// layout descriptor
// ---------------------------------------------------------------------------------------------
#define B200Q_MAX_PLANES 5
struct b200q_layout {
    int      type;
    int      qk;                            // weights per wire block
    int      wire_block;                    // wire bytes per block
    int      row_meta;                      // wire bytes of per-row header (row scale), 0 if none
    int      n_planes;
    int      plane_bytes[B200Q_MAX_PLANES]; // bytes per wire block in plane p (per ROW for the row-meta plane)
    int      plane_per_row[B200Q_MAX_PLANES]; // 1 if the plane is indexed per row instead of per block
    int64_t  M, K, nb;                      // rows, cols, blocks per row
    int64_t  plane_off[B200Q_MAX_PLANES];
    int64_t  total_bytes;
    int      wire;                          // 0: plane layout; 1 / 4: the tensor is stored verbatim (wire-layout type), value = rows interleaved on the wire
};

B200Q_HD int64_t b200q_align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// Fills geometry for `type`; returns 0 on success, -1 if the type is unknown, -2 if K is not a multiple of the block.
inline int b200q_make_layout(int type, int64_t M, int64_t K, b200q_layout * L) {
    memset(L, 0, sizeof(*L));
    L->type = type; L->M = M; L->K = K;
    auto set = [&](int qk, int wire, int meta, int np, int b0, int b1, int b2, int b3, int rowplane) {
        L->qk = qk; L->wire_block = wire; L->row_meta = meta; L->n_planes = np;
        int b[4] = {b0, b1, b2, b3};
        for (int i = 0; i < np; ++i) { L->plane_bytes[i] = b[i]; L->plane_per_row[i] = (i == rowplane); }
    };
    switch (type) {
        //                         qk  wire meta np  planes...                         row-plane idx
        case B200Q_TYPE_IQ4_NL: set(32,  18, 0, 2, 16, 2, 0, 0, -1); break;   // qs | d
        case B200Q_TYPE_Q4_0:   set(32,  18, 0, 2, 16, 2, 0, 0, -1); break;   // qs | d
        case B200Q_TYPE_Q8_0:   set(32,  34, 0, 2, 32, 2, 0, 0, -1); break;   // qs | d
        case B200Q_TYPE_Q4_1:   set(32,  20, 0, 2, 16, 4, 0, 0, -1); break;   // qs | {d,m}
        case B200Q_TYPE_Q5_0:   set(32,  22, 0, 3, 16, 4, 2, 0, -1); break;   // qs | qh | d
        case B200Q_TYPE_Q5_1:   set(32,  24, 0, 3, 16, 4, 4, 0, -1); break;   // qs | qh | {d,m}
        case B200Q_TYPE_Q6_0:   set(32,  26, 0, 3, 16, 8, 2, 0, -1); break;   // qs | qh(2 bits) | d
        case B200Q_TYPE_Q2_K:   set(256, 84, 0, 3, 64, 16, 4, 0, -1); break;   // qs (2 bit) | scales[16] | {d,dmin}
        case B200Q_TYPE_Q3_K:   set(256, 110, 0, 4, 64, 32, 12, 2, -1); break;  // qs (low 2 bits) | hmask | scales[12] | d
        case B200Q_TYPE_Q4_K:   set(256, 144, 0, 2, 128, 16, 0, 0, -1); break; // qs | {d,dmin,scales[12]}
        case B200Q_TYPE_Q5_K:   set(256, 176, 0, 3, 128, 32, 16, 0, -1); break; // qs | qh | {d,dmin,scales[12]}
        case B200Q_TYPE_Q6_K:   set(256, 210, 0, 4, 128, 64, 16, 2, -1); break; // ql | qh | scales[16] | d
        case B200Q_TYPE_IQ4_XS: set(256, 136, 0, 2, 128, 8, 0, 0, -1); break;  // qs | {d,scales_h,scales_l[4]}
        case B200Q_TYPE_IQ2_K:  set(256, 76, 0, 2, 64, 12, 0, 0, -1); break;   // qs (2-bit selectors) | {d,extra,scales[8]}
        case B200Q_TYPE_IQ3_K:  set(256, 110, 0, 3, 64, 32, 16, 0, -1); break;  // qs (low 2 bits) | qh | {d,extra,scales_h,scales_l[8],pad 2}
        case B200Q_TYPE_IQ4_K:  set(256, 144, 0, 2, 128, 16, 0, 0, -1); break; // qs | {d,extra,scales_h[4],scales_l[8]}
        case B200Q_TYPE_IQ5_K:  set(256, 176, 0, 3, 128, 32, 16, 0, -1); break; // qs | qh | {d,extra,scales_h[4],scales_l[8]}
        case B200Q_TYPE_IQ4_KS: set(256, 136, 4, 3, 128, 8, 4, 0, 2); break;   // qs | scales[8] | row scale
        case B200Q_TYPE_IQ5_KS: set(256, 168, 4, 4, 128, 32, 8, 4, 3); break;  // qs | qh | scales[8] | row scale
        case B200Q_TYPE_MXFP4:  set(32,  17, 0, 2, 16, 1, 0, 0, -1); break;    // qs | e (E8M0)
        case B200Q_TYPE_IQ2_KS: set(256, 70, 2, 3, 64, 8, 4, 0, 2); break;     // qs (2-bit selectors) | {extra,scales[4],pad 2} | row scale (half on the wire, f32 in the plane)
        case B200Q_TYPE_IQ3_KS: set(256, 102, 2, 4, 64, 32, 8, 4, 3); break;   // qs | qh | {extra,scales[4],pad 2} | row scale
        case B200Q_TYPE_IQ2_BN: set(64,  16, 4, 2, 16, 4, 0, 0, 1); break;     // qs | row scale
        default: {
            b200q_wire_geom g;
            if (!b200q_wire_geom_of(type, g)) return -1;
            if (K <= 0 || K % g.qk || K % 32 || M % g.interleave) return -2;
            L->qk = g.qk; L->wire_block = g.block_bytes; L->row_meta = g.row_meta; L->n_planes = 1; L->plane_bytes[0] = g.block_bytes; L->wire = g.interleave;
            L->nb = K / g.qk; L->plane_off[0] = 0;
            L->total_bytes = b200q_align_up(M * b200q_wire_type_row_size(g, K), 256);
            return 0;
        }
    }
    if (K <= 0 || K % L->qk) return -2;
    L->nb = K / L->qk;
    int64_t off = 0;
    for (int p = 0; p < L->n_planes; ++p) {
        L->plane_off[p] = off;
        const int64_t n = L->plane_per_row[p] ? M : M * L->nb;
        off = b200q_align_up(off + n * L->plane_bytes[p], 256);
    }
    L->total_bytes = off;
    return 0;
}
inline int64_t b200q_wire_row_size(const b200q_layout & L) { return (int64_t)L.row_meta + L.nb * L.wire_block; }

// ---------------------------------------------------------------------------------------------
// nibble / bit re-ordering helpers used by repack (wire -> planes) and unrepack
// ---------------------------------------------------------------------------------------------
// "A-order" (arithmetic types): item of 32 values e=0..31, 16 bytes; byte (4w+b): low nibble = e 8w+b, high = e 8w+4+b
B200Q_HD void b200q_pack_nib_A(const uint8_t idx[32], uint8_t out[16]) {
    for (int w = 0; w < 4; ++w) for (int b = 0; b < 4; ++b) out[4 * w + b] = (uint8_t)((idx[8 * w + b] & 0xF) | ((idx[8 * w + 4 + b] & 0xF) << 4));
}
B200Q_HD void b200q_unpack_nib_A(const uint8_t in[16], uint8_t idx[32]) {
    for (int w = 0; w < 4; ++w) for (int b = 0; b < 4; ++b) { idx[8 * w + b] = in[4 * w + b] & 0xF; idx[8 * w + 4 + b] = in[4 * w + b] >> 4; }
}
// "L-order" (PRMT-lookup types): nibble j of 32-bit word w = e 8w+j, i.e. byte (4w+b): low = e 8w+2b, high = e 8w+2b+1
B200Q_HD void b200q_pack_nib_L(const uint8_t idx[32], uint8_t out[16]) {
    for (int i = 0; i < 16; ++i) out[i] = (uint8_t)((idx[2 * i] & 0xF) | ((idx[2 * i + 1] & 0xF) << 4));
}
B200Q_HD void b200q_unpack_nib_L(const uint8_t in[16], uint8_t idx[32]) {
    for (int i = 0; i < 16; ++i) { idx[2 * i] = in[i] & 0xF; idx[2 * i + 1] = in[i] >> 4; }
}
// high-bit plane for 5-bit types: 32 bits per item; bit (8b + w) = hb(e 8w+b), bit (8b+4+w) = hb(e 8w+4+b)
B200Q_HD uint32_t b200q_pack_hb(const uint8_t hb[32]) {
    uint32_t q = 0;
    for (int w = 0; w < 4; ++w) for (int b = 0; b < 4; ++b) { q |= (uint32_t)(hb[8 * w + b] & 1) << (8 * b + w); q |= (uint32_t)(hb[8 * w + 4 + b] & 1) << (8 * b + 4 + w); }
    return q;
}
B200Q_HD void b200q_unpack_hb(uint32_t q, uint8_t hb[32]) {
    for (int w = 0; w < 4; ++w) for (int b = 0; b < 4; ++b) { hb[8 * w + b] = (q >> (8 * b + w)) & 1; hb[8 * w + 4 + b] = (q >> (8 * b + 4 + w)) & 1; }
}
// 2-bit high plane for 6-bit types: 64 bits per item (two u32 U[0], U[1]); U[u] byte b, field f=2w'+g (bits 2f..2f+1)
// = high 2 bits of e 8(2u+w') + 4g + b.
B200Q_HD void b200q_pack_h2(const uint8_t h2[32], uint32_t U[2]) {
    U[0] = U[1] = 0;
    for (int u = 0; u < 2; ++u) for (int wp = 0; wp < 2; ++wp) for (int g = 0; g < 2; ++g) for (int b = 0; b < 4; ++b)
        U[u] |= (uint32_t)(h2[8 * (2 * u + wp) + 4 * g + b] & 3) << (8 * b + 2 * (2 * wp + g));
}
B200Q_HD void b200q_unpack_h2(const uint32_t U[2], uint8_t h2[32]) {
    for (int u = 0; u < 2; ++u) for (int wp = 0; wp < 2; ++wp) for (int g = 0; g < 2; ++g) for (int b = 0; b < 4; ++b)
        h2[8 * (2 * u + wp) + 4 * g + b] = (U[u] >> (8 * b + 2 * (2 * wp + g))) & 3;
}

// 2-bit plane (Q2_K, Q3_K low bits): 8 bytes per item = two u32; U[u] byte b, field f (bits 2f..2f+1) = e 16u + 4f + b, so that
// (U[u] >> 2f) & 0x03030303 is the int8x4 word of weights 16u+4f .. +3
B200Q_HD void b200q_pack_q2(const uint8_t idx[32], uint32_t U[2]) {
    U[0] = U[1] = 0;
    for (int u = 0; u < 2; ++u) for (int f = 0; f < 4; ++f) for (int b = 0; b < 4; ++b) U[u] |= (uint32_t)(idx[16 * u + 4 * f + b] & 3) << (8 * b + 2 * f);
}
B200Q_HD void b200q_unpack_q2(const uint32_t U[2], uint8_t idx[32]) {
    for (int u = 0; u < 2; ++u) for (int f = 0; f < 4; ++f) for (int b = 0; b < 4; ++b) idx[16 * u + 4 * f + b] = (U[u] >> (8 * b + 2 * f)) & 3;
}
// 2-bit LUT plane (IQ2_K, IQ3_K): 8 bytes per item = two u32; weight e = 16u + 8p + n sits in bits 4n+2p..4n+2p+1 of W[u], so that
// (W[u] >> 2p) & 0x33333333 is eight ready-made PRMT selector nibbles (weights 16u+8p .. +7 in order)
B200Q_HD void b200q_pack_l2(const uint8_t idx[32], uint32_t W[2]) {
    W[0] = W[1] = 0;
    for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) for (int n = 0; n < 8; ++n) W[u] |= (uint32_t)(idx[16 * u + 8 * p + n] & 3) << (4 * n + 2 * p);
}
B200Q_HD void b200q_unpack_l2(const uint32_t W[2], uint8_t idx[32]) {
    for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) for (int n = 0; n < 8; ++n) idx[16 * u + 8 * p + n] = (W[u] >> (4 * n + 2 * p)) & 3;
}
// third selector bit of IQ3_K: bit (4n + 2u + p) = hb(e 16u + 8p + n): ((H >> (2u+p)) & 0x11111111) << 2 drops it into bit 2 of each nibble
B200Q_HD uint32_t b200q_pack_hl(const uint8_t hb[32]) {
    uint32_t q = 0; for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) for (int n = 0; n < 8; ++n) q |= (uint32_t)(hb[16 * u + 8 * p + n] & 1) << (4 * n + 2 * u + p); return q;
}
B200Q_HD void b200q_unpack_hl(uint32_t q, uint8_t hb[32]) {
    for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) for (int n = 0; n < 8; ++n) hb[16 * u + 8 * p + n] = (q >> (4 * n + 2 * u + p)) & 1;
}
// 1-bit plane for Q3_K: bit (8b + w) = hb(e 4w + b), w = 0..7: (H >> w) & 0x01010101 is the bit of the four weights of word w
B200Q_HD uint32_t b200q_pack_hb8(const uint8_t hb[32]) {
    uint32_t q = 0; for (int w = 0; w < 8; ++w) for (int b = 0; b < 4; ++b) q |= (uint32_t)(hb[4 * w + b] & 1) << (8 * b + w); return q;
}
B200Q_HD void b200q_unpack_hb8(uint32_t q, uint8_t hb[32]) { for (int w = 0; w < 8; ++w) for (int b = 0; b < 4; ++b) hb[4 * w + b] = (q >> (8 * b + w)) & 1; }

// ---------------------------------------------------------------------------------------------
// repack / unrepack of ONE wire block (generic over the layout; runs as one GPU thread per block,
// or on the host in tests).  `wire` points at the block, `row`/`blk` locate it; `dst` is the plane base.
// ---------------------------------------------------------------------------------------------
B200Q_HD uint8_t * b200q_plane_ptr(uint8_t * base, const b200q_layout & L, int p, int64_t row, int64_t blk) {
    return base + L.plane_off[p] + (L.plane_per_row[p] ? row : row * L.nb + blk) * L.plane_bytes[p];
}
B200Q_HD const uint8_t * b200q_plane_cptr(const uint8_t * base, const b200q_layout & L, int p, int64_t row, int64_t blk) {
    return base + L.plane_off[p] + (L.plane_per_row[p] ? row : row * L.nb + blk) * L.plane_bytes[p];
}

// wire nibble positions: for 32-blocks {qs[j] low = e j, high = e j+16}; for 256-superblocks with the K-quant
// convention {chunk c of 64: qs[32c+l] low = e 64c+l, high = e 64c+32+l}; IQ4_XS/IQ4_K/IQ4_KS/IQ5_K use
// per-32 sub-blocks {qs[16s+j] low = e 32s+j, high = e 32s+16+j} (IQ5_K: per 64: see below).
B200Q_HD void b200q_repack_block(const b200q_layout & L, const uint8_t * wire, uint8_t * dst, int64_t row, int64_t blk, bool inverse) {
    // `inverse` == false: wire -> planes ; true: planes -> wire (wire is then written through a const_cast by the caller)
    uint8_t * w = const_cast<uint8_t *>(wire);
    uint8_t idx[32], hb[32], tmp[16];
    switch (L.type) {
    case B200Q_TYPE_IQ4_NL: case B200Q_TYPE_Q4_0: {   // {half d; u8 qs[16]}
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 1, row, blk);
        const bool lut = L.type == B200Q_TYPE_IQ4_NL;
        if (!inverse) {
            for (int j = 0; j < 16; ++j) { idx[j] = w[2 + j] & 0xF; idx[j + 16] = w[2 + j] >> 4; }
            if (lut) b200q_pack_nib_L(idx, pq); else b200q_pack_nib_A(idx, pq);
            pd[0] = w[0]; pd[1] = w[1];
        } else {
            if (lut) b200q_unpack_nib_L(pq, idx); else b200q_unpack_nib_A(pq, idx);
            for (int j = 0; j < 16; ++j) w[2 + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4));
            w[0] = pd[0]; w[1] = pd[1];
        }
    } break;
    case B200Q_TYPE_Q4_1: {                            // {half d, m; u8 qs[16]}   (ggml-common.h: block_q4_1)
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 1, row, blk);
        if (!inverse) { for (int j = 0; j < 16; ++j) { idx[j] = w[4 + j] & 0xF; idx[j + 16] = w[4 + j] >> 4; } b200q_pack_nib_A(idx, pq); for (int j = 0; j < 4; ++j) pd[j] = w[j]; }
        else { b200q_unpack_nib_A(pq, idx); for (int j = 0; j < 16; ++j) w[4 + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4)); for (int j = 0; j < 4; ++j) w[j] = pd[j]; }
    } break;
    case B200Q_TYPE_Q5_0: case B200Q_TYPE_Q5_1: {      // {half d; [half m;] u8 qh[4]; u8 qs[16]}: qh bit e = 5th bit of element e
        const int hd = L.type == B200Q_TYPE_Q5_1 ? 4 : 2;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = b200q_plane_ptr(dst, L, 1, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 2, row, blk);
        if (!inverse) {
            uint32_t qh; memcpy(&qh, w + hd, 4);
            for (int j = 0; j < 16; ++j) { idx[j] = w[hd + 4 + j] & 0xF; idx[j + 16] = w[hd + 4 + j] >> 4; }
            for (int e = 0; e < 32; ++e) hb[e] = (qh >> e) & 1;
            b200q_pack_nib_A(idx, pq); uint32_t q = b200q_pack_hb(hb); memcpy(ph, &q, 4); for (int j = 0; j < hd; ++j) pd[j] = w[j];
        } else {
            b200q_unpack_nib_A(pq, idx); uint32_t q; memcpy(&q, ph, 4); b200q_unpack_hb(q, hb);
            uint32_t qh = 0; for (int e = 0; e < 32; ++e) qh |= (uint32_t)hb[e] << e;
            memcpy(w + hd, &qh, 4); for (int j = 0; j < 16; ++j) w[hd + 4 + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4)); for (int j = 0; j < hd; ++j) w[j] = pd[j];
        }
    } break;
    case B200Q_TYPE_Q6_0: {                            // {half d; u8 qh[8]; u8 qs[16]}  (ggml-quants.c:1675-1695)
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = b200q_plane_ptr(dst, L, 1, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 2, row, blk);
        if (!inverse) {
            for (int j = 0; j < 16; ++j) {
                idx[j] = w[10 + j] & 0xF; idx[j + 16] = w[10 + j] >> 4;
                const uint8_t h = w[2 + j % 8] >> (4 * (j / 8)); hb[j] = h & 3; hb[j + 16] = (h >> 2) & 3;
            }
            b200q_pack_nib_A(idx, pq); uint32_t U[2]; b200q_pack_h2(hb, U); memcpy(ph, U, 8); pd[0] = w[0]; pd[1] = w[1];
        } else {
            b200q_unpack_nib_A(pq, idx); uint32_t U[2]; memcpy(U, ph, 8); b200q_unpack_h2(U, hb);
            for (int j = 0; j < 8; ++j) w[2 + j] = 0;
            for (int j = 0; j < 16; ++j) { w[10 + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4)); w[2 + j % 8] |= (uint8_t)((hb[j] | (hb[j + 16] << 2)) << (4 * (j / 8))); }
            w[0] = pd[0]; w[1] = pd[1];
        }
    } break;
    case B200Q_TYPE_Q8_0: {                            // {half d; i8 qs[32]}
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 1, row, blk);
        if (!inverse) { for (int j = 0; j < 32; ++j) pq[j] = w[2 + j]; pd[0] = w[0]; pd[1] = w[1]; }
        else          { for (int j = 0; j < 32; ++j) w[2 + j] = pq[j]; w[0] = pd[0]; w[1] = pd[1]; }
    } break;
    case B200Q_TYPE_Q2_K: case B200Q_TYPE_Q3_K: {
        // Q2_K {u8 scales[16]; u8 qs[64]; half d, dmin}  (ggml-common.h block_q2_K; dequantize_row_q2_K ggml-quants.c:2162-2190)
        // Q3_K {u8 hmask[32]; u8 qs[64]; u8 scales[12]; half d}  (block_q3_K; dequantize_row_q3_K ggml-quants.c:2563-2605)
        // both: item s = 4h + j (h = 128-half, j = 0..3): weight e <-> qs[32h + e] bits 2j..2j+1 ; Q3_K high bit = hmask[e] bit s
        const bool q3 = L.type == B200Q_TYPE_Q3_K;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk);
        uint8_t * wqs = w + (q3 ? 32 : 16);
        if (!q3) {
            uint8_t * ps = b200q_plane_ptr(dst, L, 1, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 2, row, blk);
            if (!inverse) { for (int j = 0; j < 16; ++j) ps[j] = w[j]; for (int j = 0; j < 4; ++j) pd[j] = w[80 + j]; }
            else          { for (int j = 0; j < 16; ++j) w[j] = ps[j]; for (int j = 0; j < 4; ++j) w[80 + j] = pd[j]; }
        } else {
            uint8_t * ps = b200q_plane_ptr(dst, L, 2, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 3, row, blk);
            if (!inverse) { for (int j = 0; j < 12; ++j) ps[j] = w[96 + j]; pd[0] = w[108]; pd[1] = w[109]; }
            else          { for (int j = 0; j < 12; ++j) w[96 + j] = ps[j]; w[108] = pd[0]; w[109] = pd[1]; for (int j = 0; j < 32; ++j) w[j] = 0; }
        }
        if (inverse) for (int j = 0; j < 64; ++j) wqs[j] = 0;
        uint8_t * ph = q3 ? b200q_plane_ptr(dst, L, 1, row, blk) : nullptr;
        for (int s = 0; s < 8; ++s) {
            const int h = s / 4, j = s % 4;
            if (!inverse) {
                for (int e = 0; e < 32; ++e) { idx[e] = (wqs[32 * h + e] >> (2 * j)) & 3; if (q3) hb[e] = (w[e] >> s) & 1; }
                uint32_t U[2]; b200q_pack_q2(idx, U); memcpy(pq + 8 * s, U, 8);
                if (q3) { uint32_t q = b200q_pack_hb8(hb); memcpy(ph + 4 * s, &q, 4); }
            } else {
                uint32_t U[2]; memcpy(U, pq + 8 * s, 8); b200q_unpack_q2(U, idx);
                if (q3) { uint32_t q; memcpy(&q, ph + 4 * s, 4); b200q_unpack_hb8(q, hb); }
                for (int e = 0; e < 32; ++e) { wqs[32 * h + e] |= (uint8_t)(idx[e] << (2 * j)); if (q3) w[e] |= (uint8_t)(hb[e] << s); }
            }
        }
    } break;
    case B200Q_TYPE_IQ2_KS: case B200Q_TYPE_IQ3_KS: {
        // IQ2_KS row = {half d; blocks {u16 extra; u8 scales[4]; u8 qs[64]}}              (block_iq2_ks; iqk_quantize.cpp:1877-1907)
        // IQ3_KS row = {half d; blocks {u16 extra; u8 scales[4]; u8 qs[64]; u8 qh[32]}}   (block_iq3_ks; iqk_quantize.cpp:2774-2803)
        // quants exactly as IQ2_K / IQ3_K: item s: weight e <-> qs[32(s/4) + e] bits 2(s%4)..+1 ; third bit = qh[e] bit s
        const bool q3 = L.type == B200Q_TYPE_IQ3_KS;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = q3 ? b200q_plane_ptr(dst, L, 1, row, blk) : nullptr;
        uint8_t * pm = b200q_plane_ptr(dst, L, q3 ? 2 : 1, row, blk);
        uint8_t * wqs = w + 6; uint8_t * wqh = w + 70;
        if (!inverse) { for (int j = 0; j < 6; ++j) pm[j] = w[j]; pm[6] = 0; pm[7] = 0; }
        else { for (int j = 0; j < 6; ++j) w[j] = pm[j]; for (int j = 0; j < 64; ++j) wqs[j] = 0; if (q3) for (int j = 0; j < 32; ++j) wqh[j] = 0; }
        for (int s = 0; s < 8; ++s) {
            const int h = s / 4, j = s % 4;
            if (!inverse) {
                for (int e = 0; e < 32; ++e) { idx[e] = (wqs[32 * h + e] >> (2 * j)) & 3; if (q3) hb[e] = (wqh[e] >> s) & 1; }
                uint32_t W[2]; b200q_pack_l2(idx, W); memcpy(pq + 8 * s, W, 8);
                if (q3) { uint32_t q = b200q_pack_hl(hb); memcpy(ph + 4 * s, &q, 4); }
            } else {
                uint32_t W[2]; memcpy(W, pq + 8 * s, 8); b200q_unpack_l2(W, idx);
                if (q3) { uint32_t q; memcpy(&q, ph + 4 * s, 4); b200q_unpack_hl(q, hb); }
                for (int e = 0; e < 32; ++e) { wqs[32 * h + e] |= (uint8_t)(idx[e] << (2 * j)); if (q3) wqh[e] |= (uint8_t)(hb[e] << s); }
            }
        }
    } break;
    case B200Q_TYPE_IQ2_K: case B200Q_TYPE_IQ3_K: {
        // IQ2_K {half d; u16 extra; u8 scales[8]; u8 qs[64]}                              (ggml-common.h block_iq2_k; iqk_quantize.cpp:1356-1385)
        // IQ3_K {half d; u16 extra; u16 scales_h; u8 scales_l[8]; u8 qs[64]; u8 qh[32]}   (block_iq3_k; iqk_quantize.cpp:2534-2565)
        // both: item s: weight e <-> qs[32(s/4) + e] bits 2(s%4)..+1 ; IQ3_K third bit = qh[e] bit s
        const bool q3 = L.type == B200Q_TYPE_IQ3_K; const int hdr = q3 ? 14 : 12;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = q3 ? b200q_plane_ptr(dst, L, 1, row, blk) : nullptr;
        uint8_t * pm = b200q_plane_ptr(dst, L, q3 ? 2 : 1, row, blk);
        uint8_t * wqs = w + hdr; uint8_t * wqh = w + hdr + 64;
        if (!inverse) { for (int j = 0; j < hdr; ++j) pm[j] = w[j]; if (q3) { pm[14] = 0; pm[15] = 0; } }
        else { for (int j = 0; j < hdr; ++j) w[j] = pm[j]; for (int j = 0; j < 64; ++j) wqs[j] = 0; if (q3) for (int j = 0; j < 32; ++j) wqh[j] = 0; }
        for (int s = 0; s < 8; ++s) {
            const int h = s / 4, j = s % 4;
            if (!inverse) {
                for (int e = 0; e < 32; ++e) { idx[e] = (wqs[32 * h + e] >> (2 * j)) & 3; if (q3) hb[e] = (wqh[e] >> s) & 1; }
                uint32_t W[2]; b200q_pack_l2(idx, W); memcpy(pq + 8 * s, W, 8);
                if (q3) { uint32_t q = b200q_pack_hl(hb); memcpy(ph + 4 * s, &q, 4); }
            } else {
                uint32_t W[2]; memcpy(W, pq + 8 * s, 8); b200q_unpack_l2(W, idx);
                if (q3) { uint32_t q; memcpy(&q, ph + 4 * s, 4); b200q_unpack_hl(q, hb); }
                for (int e = 0; e < 32; ++e) { wqs[32 * h + e] |= (uint8_t)(idx[e] << (2 * j)); if (q3) wqh[e] |= (uint8_t)(hb[e] << s); }
            }
        }
    } break;
    case B200Q_TYPE_Q4_K: case B200Q_TYPE_Q5_K: {      // {half d,dmin; u8 scales[12]; [u8 qh[32];] u8 qs[128]}
        const bool q5 = L.type == B200Q_TYPE_Q5_K;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk);
        uint8_t * ph = q5 ? b200q_plane_ptr(dst, L, 1, row, blk) : nullptr;
        uint8_t * pm = b200q_plane_ptr(dst, L, q5 ? 2 : 1, row, blk);
        uint8_t * wqh = w + 16; uint8_t * wqs = w + (q5 ? 48 : 16);
        if (!inverse) { for (int j = 0; j < 16; ++j) pm[j] = w[j]; } else { for (int j = 0; j < 16; ++j) w[j] = pm[j]; }
        if (inverse && q5) for (int j = 0; j < 32; ++j) wqh[j] = 0;
        for (int s = 0; s < 8; ++s) {                  // sub-block s: chunk c = s/2, nibble half = s%2
            const int c = s / 2, hi = s % 2;
            if (!inverse) {
                for (int l = 0; l < 32; ++l) { idx[l] = hi ? (wqs[32 * c + l] >> 4) : (wqs[32 * c + l] & 0xF); if (q5) hb[l] = (wqh[l] >> (2 * c + hi)) & 1; }
                b200q_pack_nib_A(idx, pq + 16 * s);
                if (q5) { uint32_t q = b200q_pack_hb(hb); memcpy(ph + 4 * s, &q, 4); }
            } else {
                b200q_unpack_nib_A(pq + 16 * s, idx);
                if (q5) { uint32_t q; memcpy(&q, ph + 4 * s, 4); b200q_unpack_hb(q, hb); }
                for (int l = 0; l < 32; ++l) {
                    if (hi) wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0x0F) | (idx[l] << 4)); else wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0xF0) | idx[l]);
                    if (q5) wqh[l] |= (uint8_t)(hb[l] << (2 * c + hi));
                }
            }
        }
    } break;
    case B200Q_TYPE_Q6_K: {                            // {u8 ql[128]; u8 qh[64]; i8 scales[16]; half d}
        uint8_t * pl = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = b200q_plane_ptr(dst, L, 1, row, blk);
        uint8_t * ps = b200q_plane_ptr(dst, L, 2, row, blk); uint8_t * pd = b200q_plane_ptr(dst, L, 3, row, blk);
        if (!inverse) { for (int j = 0; j < 16; ++j) ps[j] = w[192 + j]; pd[0] = w[208]; pd[1] = w[209]; }
        else { for (int j = 0; j < 16; ++j) w[192 + j] = ps[j]; w[208] = pd[0]; w[209] = pd[1]; for (int j = 0; j < 64; ++j) w[128 + j] = 0; }
        for (int s = 0; s < 8; ++s) {                  // item s = weights 32s..32s+31 ; half h = s/4, quarter t = s%4
            const int h = s / 4, t = s % 4;            // t: 0 -> ql[64h+l] low, 1 -> ql[64h+32+l] low, 2 -> ql[64h+l] high, 3 -> ql[64h+32+l] high
            const int qoff = 64 * h + 32 * (t & 1); const bool hi = t >= 2;
            if (!inverse) {
                for (int l = 0; l < 32; ++l) { idx[l] = hi ? (w[qoff + l] >> 4) : (w[qoff + l] & 0xF); hb[l] = (w[128 + 32 * h + l] >> (2 * t)) & 3; }
                b200q_pack_nib_A(idx, pl + 16 * s);
                uint32_t U[2]; b200q_pack_h2(hb, U); memcpy(ph + 8 * s, U, 8);
            } else {
                b200q_unpack_nib_A(pl + 16 * s, idx);
                uint32_t U[2]; memcpy(U, ph + 8 * s, 8); b200q_unpack_h2(U, hb);
                for (int l = 0; l < 32; ++l) {
                    if (hi) w[qoff + l] = (uint8_t)((w[qoff + l] & 0x0F) | (idx[l] << 4)); else w[qoff + l] = (uint8_t)((w[qoff + l] & 0xF0) | idx[l]);
                    w[128 + 32 * h + l] |= (uint8_t)(hb[l] << (2 * t));
                }
            }
        }
    } break;
    case B200Q_TYPE_IQ4_XS: case B200Q_TYPE_IQ4_K: case B200Q_TYPE_IQ4_KS: {
        // IQ4_XS {half d; u16 scales_h; u8 scales_l[4]; u8 qs[128]}  meta 8
        // IQ4_K  {half d; u16 extra; u8 scales_h[4]; u8 scales_l[8]; u8 qs[128]} meta 16
        // IQ4_KS {u8 scales[8]; u8 qs[128]} meta 8 (+ f32 row scale, handled by the row pass)
        const int meta = L.type == B200Q_TYPE_IQ4_K ? 16 : 8;
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * pm = b200q_plane_ptr(dst, L, 1, row, blk);
        if (!inverse) { for (int j = 0; j < meta; ++j) pm[j] = w[j]; } else { for (int j = 0; j < meta; ++j) w[j] = pm[j]; }
        uint8_t * wqs = w + meta;
        for (int s = 0; s < 8; ++s) {
            if (!inverse) { for (int j = 0; j < 16; ++j) { idx[j] = wqs[16 * s + j] & 0xF; idx[j + 16] = wqs[16 * s + j] >> 4; } b200q_pack_nib_L(idx, pq + 16 * s); }
            else { b200q_unpack_nib_L(pq + 16 * s, idx); for (int j = 0; j < 16; ++j) wqs[16 * s + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4)); }
        }
    } break;
    case B200Q_TYPE_MXFP4: {                           // {u8 e; u8 qs[16]}  (ggml-common.h:183-186; iqk_quantize.cpp:4224-4236)
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * pe = b200q_plane_ptr(dst, L, 1, row, blk);
        if (!inverse) { for (int j = 0; j < 16; ++j) { idx[j] = w[1 + j] & 0xF; idx[j + 16] = w[1 + j] >> 4; } b200q_pack_nib_L(idx, pq); pe[0] = w[0]; }
        else { b200q_unpack_nib_L(pq, idx); for (int j = 0; j < 16; ++j) w[1 + j] = (uint8_t)(idx[j] | (idx[j + 16] << 4)); w[0] = pe[0]; }
    } break;
    case B200Q_TYPE_IQ5_KS: {  // row = {float d; blocks {u8 scales[8]; u8 qs[128]; u8 qh[32]}}  (iqk_quantize.cpp:4798-4822): quants as IQ5_K
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = b200q_plane_ptr(dst, L, 1, row, blk); uint8_t * pm = b200q_plane_ptr(dst, L, 2, row, blk);
        if (!inverse) { for (int j = 0; j < 8; ++j) pm[j] = w[j]; } else { for (int j = 0; j < 8; ++j) w[j] = pm[j]; for (int j = 0; j < 32; ++j) w[136 + j] = 0; }
        uint8_t * wqs = w + 8; uint8_t * wqh = w + 136;
        for (int s = 0; s < 8; ++s) {
            const int c = s / 2, second = s % 2;
            if (!inverse) {
                for (int l = 0; l < 32; ++l) { const uint8_t q = wqs[32 * c + l]; idx[l] = second ? (q >> 4) : (q & 0xF); hb[l] = (wqh[l] >> (2 * c + second)) & 1; }
                b200q_pack_nib_L(idx, pq + 16 * s);
                uint32_t q = 0; for (int e = 0; e < 32; ++e) q |= (uint32_t)hb[e] << e;
                memcpy(ph + 4 * s, &q, 4);
            } else {
                b200q_unpack_nib_L(pq + 16 * s, idx);
                uint32_t q; memcpy(&q, ph + 4 * s, 4);
                for (int l = 0; l < 32; ++l) {
                    if (second) wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0x0F) | (idx[l] << 4)); else wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0xF0) | idx[l]);
                    wqh[l] |= (uint8_t)(((q >> l) & 1) << (2 * c + second));
                }
            }
        }
    } break;
    case B200Q_TYPE_IQ5_K: {   // {half d; u16 extra; u8 scales_h[4]; u8 scales_l[8]; u8 qs[128]; u8 qh[32]}
        // per 64 weights c: e 64c+j <- qs[32c+j] low (j<16), 64c+16+j <- qs[32c+16+j] low, 64c+32+j <- qs[32c+j] high, 64c+48+j <- qs[32c+16+j] high
        // high bit: qh[(c/4)*32 + jj] >> (2*(c%4) + {0: first 32, 1: second 32}), jj = position within the 32 bytes (see iqk_quantize.cpp:3136-3141)
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk); uint8_t * ph = b200q_plane_ptr(dst, L, 1, row, blk); uint8_t * pm = b200q_plane_ptr(dst, L, 2, row, blk);
        if (!inverse) { for (int j = 0; j < 16; ++j) pm[j] = w[j]; } else { for (int j = 0; j < 16; ++j) w[j] = pm[j]; for (int j = 0; j < 32; ++j) w[144 + j] = 0; }
        uint8_t * wqs = w + 16; uint8_t * wqh = w + 144;
        for (int s = 0; s < 8; ++s) {                  // item s: c = s/2, second = s%2 (0: low nibbles, 1: high nibbles)
            const int c = s / 2, second = s % 2;
            if (!inverse) {
                for (int l = 0; l < 32; ++l) { const uint8_t q = wqs[32 * c + l]; idx[l] = second ? (q >> 4) : (q & 0xF); hb[l] = (wqh[l] >> (2 * c + second)) & 1; }
                b200q_pack_nib_L(idx, pq + 16 * s);    // LUT type -> L order (hb is re-ordered to match in decode)
                uint32_t q = 0; for (int e = 0; e < 32; ++e) q |= (uint32_t)hb[e] << e;   // natural bit order for the LUT path
                memcpy(ph + 4 * s, &q, 4);
            } else {
                b200q_unpack_nib_L(pq + 16 * s, idx);
                uint32_t q; memcpy(&q, ph + 4 * s, 4);
                for (int l = 0; l < 32; ++l) {
                    if (second) wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0x0F) | (idx[l] << 4)); else wqs[32 * c + l] = (uint8_t)((wqs[32 * c + l] & 0xF0) | idx[l]);
                    wqh[l] |= (uint8_t)(((q >> l) & 1) << (2 * c + second));
                }
            }
        }
        (void)tmp;
    } break;
    case B200Q_TYPE_IQ2_BN: {                          // {u8 qs[16]} per 64 weights: already dp4a-friendly -> copy
        uint8_t * pq = b200q_plane_ptr(dst, L, 0, row, blk);
        if (!inverse) { for (int j = 0; j < 16; ++j) pq[j] = w[j]; } else { for (int j = 0; j < 16; ++j) w[j] = pq[j]; }
    } break;
    default: break;
    }
}
// per-row header (row scale) pass
B200Q_HD void b200q_repack_row_meta(const b200q_layout & L, const uint8_t * wire_row, uint8_t * dst, int64_t row, bool inverse) {
    if (!L.row_meta) return;
    int p = -1; for (int i = 0; i < L.n_planes; ++i) if (L.plane_per_row[i]) p = i;
    if (p < 0) return;
    uint8_t * pr = b200q_plane_ptr(dst, L, p, row, 0); uint8_t * w = const_cast<uint8_t *>(wire_row);
    if (L.row_meta == 2 && L.plane_bytes[p] == 4) {
        // half row scale on the wire (IQ2_KS, IQ3_KS: ggml.c row_meta_size = 2), kept as its exact f32 value in the plane so that the
        // kernels read every row scale the same way; f32 -> half of a value that came from a half is exact, the round trip is bit-for-bit
        if (!inverse) { const float f = b200q_h2f((uint16_t)(w[0] | (w[1] << 8))); memcpy(pr, &f, 4); }
        else { float f; memcpy(&f, pr, 4); const uint16_t h = b200q_f2h_exact(f); w[0] = (uint8_t)(h & 0xFF); w[1] = (uint8_t)(h >> 8); }
        return;
    }
    for (int j = 0; j < L.row_meta; ++j) { if (!inverse) pr[j] = w[j]; else w[j] = pr[j]; }
}

// ---------------------------------------------------------------------------------------------
// canonical decode
// ---------------------------------------------------------------------------------------------
struct b200q_canon {        // 32 weights
    int   va[8];            // int8 x4 per word, natural k order
    int   vb[8];            // second addend (only for HAS_B types)
    float dl[2];            // scale of weights 0..15 / 16..31
    float ml[2];            // subtracted offset of weights 0..15 / 16..31
};

// value tables.  kvalues_iq4nl (ggml-common.h, used by IQ4_NL / IQ4_XS) and iq4k_values (:2227) as PRMT operands.
// A = entries 0..7 (all negative  -> PRMT sign-fill of an unselected lane = 0xFF = -1)
// B = entries 8..15 stored +1     (all positive -> sign-fill = 0x00), so that  byteA + byteB == value  exactly.
#define B200Q_KV4_A0 0xBFAD9881u   /* -127,-104, -83, -65 */
#define B200Q_KV4_A1 0xF6EADDCFu   /*  -49, -35, -22, -10 */
#define B200Q_KV4_B0 0x271A0E02u   /*  1+1, 13+1, 25+1, 38+1 */
#define B200Q_KV4_B1 0x725A4636u   /* 53+1, 69+1, 89+1,113+1 */

// The four table words are passed in registers (struct b200q_kv4): written as literals the compiler re-materialises
// a constant->register move in front of every PRMT (16 extra instructions per 32 weights in the mat-vec inner loop).
struct b200q_kv4 { uint32_t a0, a1, b0, b1, k16; };      // k16 = 65536: see B200Q_SHR_VIA_IMAD
B200Q_HD b200q_kv4 b200q_kv4_init() {
    b200q_kv4 t; t.a0 = B200Q_KV4_A0; t.a1 = B200Q_KV4_A1; t.b0 = B200Q_KV4_B0; t.b1 = B200Q_KV4_B1; t.k16 = 65536u; return t;
}
// Tuning knob: PRMT, LOP3 and SHF share the ALU pipe (28 of the 58 instructions per item of the IQ4_NL mat-vec); with this knob the
// eight `>> 16` per item become mul.hi.u32 by an opaque 65536 (IMAD.HI: FMA pipe).
#ifndef B200Q_SHR_VIA_IMAD
#define B200Q_SHR_VIA_IMAD 0
#endif
B200Q_HD uint32_t b200q_shr16(uint32_t q, uint32_t k16) {
#if defined(__CUDA_ARCH__) && B200Q_SHR_VIA_IMAD
    return __umulhi(q, k16);
#else
    (void)k16; return q >> 16;
#endif
}
#if defined(__CUDACC__)
// Same values, but laundered through shared memory at a LANE-DEPENDENT address, so that ptxas can neither fold them
// (constants get a UR->R move in front of every PRMT) nor keep them in uniform registers (same move): they stay in
// four ordinary registers for the whole kernel.  `slot` = 128 words of smem; call from all threads (has a __syncthreads()).
__device__ __forceinline__ b200q_kv4 b200q_kv4_init_via_smem(volatile uint32_t * slot) {
    if (threadIdx.x < 32) {
        slot[threadIdx.x * 4 + 0] = B200Q_KV4_A0; slot[threadIdx.x * 4 + 1] = B200Q_KV4_A1;
        slot[threadIdx.x * 4 + 2] = B200Q_KV4_B0; slot[threadIdx.x * 4 + 3] = B200Q_KV4_B1;
    }
    __syncthreads();
    const int l = threadIdx.x & 31;
    b200q_kv4 t; t.a0 = slot[l * 4 + 0]; t.a1 = slot[l * 4 + 1]; t.b0 = slot[l * 4 + 2]; t.b1 = slot[l * 4 + 3]; t.k16 = 65536u; return t;
}
#endif
B200Q_HD void b200q_lut4(const b200q_kv4 & t, uint32_t q, int & a_lo, int & b_lo, int & a_hi, int & b_hi) {
    // q: 8 nibbles (L-order: nibble j = weight j).  lo = weights 0..3, hi = weights 4..7.
    const uint32_t qx = q ^ 0x88888888u;
    a_lo = (int)b200q_prmt(t.a0, t.a1, q);
    b_lo = (int)b200q_prmt(t.b0, t.b1, qx);
    a_hi = (int)b200q_prmt(t.a0, t.a1, b200q_shr16(q, t.k16));
    b_hi = (int)b200q_prmt(t.b0, t.b1, b200q_shr16(qx, t.k16));
}

// byte i (0..15) of a 4-word register group, without dynamic register indexing
B200Q_HD uint32_t b200q_byte(const uint32_t m[4], int i) {
    const uint32_t w = (i & 8) ? ((i & 4) ? m[3] : m[2]) : ((i & 4) ? m[1] : m[0]);
    return (w >> (8 * (i & 3))) & 0xFF;
}
// get_scale_min_k4 (reference ggml-quants.c:2036-2044); the 12 scale bytes are bytes 4..15 of the meta words m[0..3]
B200Q_HD void b200q_scale_min_k4(int j, const uint32_t m4[4], int & sc, int & m) {
    const int sh = 8 * (j & 3);
    const uint32_t b0 = (m4[1] >> sh) & 0xFF, b1 = (m4[2] >> sh) & 0xFF, b2 = (m4[3] >> sh) & 0xFF;
    if (j < 4) { sc = (int)(b0 & 63); m = (int)(b1 & 63); }
    else { sc = (int)((b2 & 0xF) | ((b0 >> 6) << 4)); m = (int)((b2 >> 4) | ((b1 >> 6) << 4)); }
}

// iq5nl_values (ggml-common.h:2232), all +2 so that entries 16..31 are positive; 4 PRMT tables of 8.
//   T0 = v[0..7]+2 (+1 fold), T1 = v[8..15]+2 (+1), T2 = v[16..23]+2, T3 = v[24..31]+2 — see b200q_lut5.
// raw v: -126,-114,-103,-92,-83,-74,-65,-57 | -50,-43,-36,-30,-24,-18,-12,-6 | -1,5,11,17,23,29,36,43 | 51,59,68,77,87,97,109,121
// Pair (T0,T1): both negative -> sign-fills are -1 each -> store +1:  T0' = v+2+1, T1' = v+2+1
// Pair (T2,T3): both positive -> sign-fills are 0                ->  T2' = v+2,   T3' = v+2
#define B200Q_KV5_T0_0 0xA79C9185u  /* -123,-111,-100, -89 */
#define B200Q_KV5_T0_1 0xCAC2B9B0u  /*  -80, -71, -62, -54 */
#define B200Q_KV5_T1_0 0xE5DFD8D1u  /*  -47, -40, -33, -27 */
#define B200Q_KV5_T1_1 0xFDF7F1EBu  /*  -21, -15,  -9,  -3 */
#define B200Q_KV5_T2_0 0x130D0701u  /*    1,   7,  13,  19 */
#define B200Q_KV5_T2_1 0x2D261F19u  /*   25,  31,  38,  45 */
#define B200Q_KV5_T3_0 0x4F463D35u  /*   53,  61,  70,  79 */
#define B200Q_KV5_T3_1 0x7B6F6359u  /*   89,  99, 111, 123 */

// Decode item `it` (32 weights) of row `row`.  `base` = plane base of the tensor.
template <int TYPE> struct b200q_traits;

#define B200Q_DEF_TRAITS(T, HASB, IK) template <> struct b200q_traits<T> { static constexpr bool HAS_B = HASB; static constexpr int ITEM_K = IK; };
B200Q_DEF_TRAITS(B200Q_TYPE_IQ4_NL, true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q4_0,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q8_0,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q4_1,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q5_0,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q5_1,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q6_0,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q2_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q3_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q4_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q5_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_Q6_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ4_XS, true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ2_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ3_K,  false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ4_K,  true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ4_KS, true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ5_KS, true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_MXFP4,  true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ2_KS, false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ3_KS, false, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ5_K,  true, 32)
B200Q_DEF_TRAITS(B200Q_TYPE_IQ2_BN, false, 32)

// Raw registers of one item, as loaded from the planes.
struct b200q_item {
    uint32_t q[8];     // low-bit plane words: 4 for 4-bit types, 8 for Q8_0
    uint32_t h[2];     // high-bit plane words (Q5_K/IQ5_K: h[0]; Q6_K: h[0..1])
    uint32_t m[4];     // block metadata words (scales etc.)
    float    rs;       // row scale (types with a row header)
};

#if !defined(__CUDACC__)
struct uint4 { uint32_t x, y, z, w; }; struct uint2 { uint32_t x, y; };
#endif
// load policies: GLOBAL = read-only data path (ld.global.nc), PLAIN = ordinary loads (shared-memory stages, host emulation)
struct b200q_ld_global {
    static B200Q_HD void ld16(uint32_t * dst, const uint8_t * p) {
#if defined(__CUDA_ARCH__)
        const uint4 t = __ldg(reinterpret_cast<const uint4 *>(p)); dst[0] = t.x; dst[1] = t.y; dst[2] = t.z; dst[3] = t.w;
#else
        memcpy(dst, p, 16);
#endif
    }
    static B200Q_HD void ld8(uint32_t * dst, const uint8_t * p) {
#if defined(__CUDA_ARCH__)
        const uint2 t = __ldg(reinterpret_cast<const uint2 *>(p)); dst[0] = t.x; dst[1] = t.y;
#else
        memcpy(dst, p, 8);
#endif
    }
    static B200Q_HD uint32_t ld4(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
        return __ldg(reinterpret_cast<const uint32_t *>(p));
#else
        uint32_t v; memcpy(&v, p, 4); return v;
#endif
    }
    static B200Q_HD uint32_t ld2(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
        return __ldg(reinterpret_cast<const uint16_t *>(p));
#else
        uint16_t v; memcpy(&v, p, 2); return v;
#endif
    }
    static B200Q_HD uint32_t ld1(const uint8_t * p) { return *p; }
};
struct b200q_ld_plain {
    static B200Q_HD void ld16(uint32_t * dst, const uint8_t * p) { const uint4 t = *reinterpret_cast<const uint4 *>(p); dst[0] = t.x; dst[1] = t.y; dst[2] = t.z; dst[3] = t.w; }
    static B200Q_HD void ld8(uint32_t * dst, const uint8_t * p)  { const uint2 t = *reinterpret_cast<const uint2 *>(p); dst[0] = t.x; dst[1] = t.y; }
    static B200Q_HD uint32_t ld4(const uint8_t * p) { return *reinterpret_cast<const uint32_t *>(p); }
    static B200Q_HD uint32_t ld2(const uint8_t * p) { return *reinterpret_cast<const uint16_t *>(p); }
    static B200Q_HD uint32_t ld1(const uint8_t * p) { return *p; }
};
// resolved plane pointers of one tensor (computed once per tensor on the host / once per kernel)
struct b200q_planes { const uint8_t * p[B200Q_MAX_PLANES]; int64_t nb; int64_t n32; };
B200Q_HD b200q_planes b200q_planes_from(const uint8_t * base, const b200q_layout & L) {
    b200q_planes P; for (int i = 0; i < B200Q_MAX_PLANES; ++i) P.p[i] = base + L.plane_off[i];
    P.nb = L.nb; P.n32 = L.K / 32; return P;
}

// item index `it` counts 32-weight items along the row: it in [0, K/32).  LD = load policy; ROWPLANE = also fetch the
// per-row scale (the smem-ring kernel passes stage-relative planes with row = 0 and fetches the row scale itself).
template <class T> struct b200q_ident { typedef T type; };
// SWZ: plane 0 is a TMA SWIZZLE_128B tile of 8 items (128 bytes) per row: 16-byte chunk c of row r sits at chunk c ^ (r & 7).
template <int TYPE, class LD = b200q_ld_global, bool ROWPLANE = true, class IDX = int64_t, bool SWZ = false>
B200Q_HD void b200q_load_item(b200q_item & I, const b200q_planes & P, typename b200q_ident<IDX>::type row, typename b200q_ident<IDX>::type it_) {
    const IDX n32 = (IDX)P.n32, nb = (IDX)P.nb;
    const IDX it = it_;
    const IDX it0 = SWZ ? (IDX)(it_ ^ (row & 7)) : it_;      // index used for the low-bit plane only
    if (TYPE == B200Q_TYPE_IQ4_NL || TYPE == B200Q_TYPE_Q4_0) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.m[0] = LD::ld2(P.p[1] + (row * n32 + it) * 2);
    } else if (TYPE == B200Q_TYPE_Q4_1) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.m[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
    } else if (TYPE == B200Q_TYPE_Q5_0 || TYPE == B200Q_TYPE_Q5_1) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        I.m[0] = TYPE == B200Q_TYPE_Q5_1 ? LD::ld4(P.p[2] + (row * n32 + it) * 4) : LD::ld2(P.p[2] + (row * n32 + it) * 2);
    } else if (TYPE == B200Q_TYPE_Q6_0) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        LD::ld8(I.h, P.p[1] + (row * n32 + it) * 8);
        I.m[0] = LD::ld2(P.p[2] + (row * n32 + it) * 2);
    } else if (TYPE == B200Q_TYPE_Q8_0) {
        const uint8_t * p = P.p[0] + (row * n32 + it) * 32;
        LD::ld16(I.q, p); LD::ld16(I.q + 4, p + 16);
        I.m[0] = LD::ld2(P.p[1] + (row * n32 + it) * 2);
    } else if (TYPE == B200Q_TYPE_Q2_K) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        I.m[0] = LD::ld2(P.p[1] + (row * nb + it / 8) * 16 + 2 * (it % 8));   // the two {scale, min} bytes of this item
        I.m[1] = LD::ld4(P.p[2] + (row * nb + it / 8) * 4);                   // {d, dmin}
    } else if (TYPE == B200Q_TYPE_Q3_K) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        const uint8_t * ps = P.p[2] + (row * nb + it / 8) * 12;
        I.m[0] = LD::ld4(ps); I.m[1] = LD::ld4(ps + 4); I.m[2] = LD::ld4(ps + 8);
        I.m[3] = LD::ld2(P.p[3] + (row * nb + it / 8) * 2);
    } else if (TYPE == B200Q_TYPE_IQ2_K) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        const uint8_t * pm = P.p[1] + (row * nb + it / 8) * 12;
        I.m[0] = LD::ld4(pm); I.m[1] = LD::ld4(pm + 4); I.m[2] = LD::ld4(pm + 8);
    } else if (TYPE == B200Q_TYPE_IQ3_K) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        LD::ld16(I.m, P.p[2] + (row * nb + it / 8) * 16);
    } else if (TYPE == B200Q_TYPE_Q4_K || TYPE == B200Q_TYPE_IQ4_K) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        LD::ld16(I.m, P.p[1] + (row * nb + it / 8) * 16);
    } else if (TYPE == B200Q_TYPE_Q5_K || TYPE == B200Q_TYPE_IQ5_K) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        LD::ld16(I.m, P.p[2] + (row * nb + it / 8) * 16);
    } else if (TYPE == B200Q_TYPE_Q6_K) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        LD::ld8(I.h, P.p[1] + (row * n32 + it) * 8);
        I.m[0] = LD::ld2(P.p[2] + (row * n32 + it) * 2);     // two int8 scales of this item
        I.m[1] = LD::ld2(P.p[3] + (row * nb + it / 8) * 2);  // d
    } else if (TYPE == B200Q_TYPE_IQ4_XS) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        LD::ld8(I.m, P.p[1] + (row * nb + it / 8) * 8);
    } else if (TYPE == B200Q_TYPE_IQ4_KS) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.m[0] = LD::ld1(P.p[1] + (row * nb + it / 8) * 8 + it % 8);
        if (ROWPLANE) { uint32_t r = LD::ld4(P.p[2] + row * 4); memcpy(&I.rs, &r, 4); }
    } else if (TYPE == B200Q_TYPE_IQ5_KS) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        I.m[0] = LD::ld1(P.p[2] + (row * nb + it / 8) * 8 + it % 8);
        if (ROWPLANE) { uint32_t r = LD::ld4(P.p[3] + row * 4); memcpy(&I.rs, &r, 4); }
    } else if (TYPE == B200Q_TYPE_MXFP4) {
        LD::ld16(I.q, P.p[0] + (row * n32 + it0) * 16);
        I.m[0] = LD::ld1(P.p[1] + (row * n32 + it));
    } else if (TYPE == B200Q_TYPE_IQ2_KS) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        LD::ld8(I.m, P.p[1] + (row * nb + it / 8) * 8);
        if (ROWPLANE) { uint32_t r = LD::ld4(P.p[2] + row * 4); memcpy(&I.rs, &r, 4); }
    } else if (TYPE == B200Q_TYPE_IQ3_KS) {
        LD::ld8(I.q, P.p[0] + (row * n32 + it) * 8);
        I.h[0] = LD::ld4(P.p[1] + (row * n32 + it) * 4);
        LD::ld8(I.m, P.p[2] + (row * nb + it / 8) * 8);
        if (ROWPLANE) { uint32_t r = LD::ld4(P.p[3] + row * 4); memcpy(&I.rs, &r, 4); }
    } else if (TYPE == B200Q_TYPE_IQ2_BN) {           // 64 weights per wire block: item = half a block (see decode)
        LD::ld16(I.q, P.p[0] + (row * nb + it / 2) * 16);
        if (ROWPLANE) { uint32_t r = LD::ld4(P.p[1] + row * 4); memcpy(&I.rs, &r, 4); }
    }
}
template <int TYPE>
B200Q_HD void b200q_load_item(b200q_item & I, const uint8_t * base, const b200q_layout & L, int64_t row, int64_t it) {
    b200q_load_item<TYPE>(I, b200q_planes_from(base, L), row, it);
}
// index of the per-row plane of a type (-1 if none)
B200Q_HD constexpr int b200q_row_plane(int type) {
    return type == B200Q_TYPE_IQ4_KS || type == B200Q_TYPE_IQ2_KS ? 2 : (type == B200Q_TYPE_IQ5_KS || type == B200Q_TYPE_IQ3_KS ? 3 : (type == B200Q_TYPE_IQ2_BN ? 1 : -1));
}

// 5-bit codebook lookup of one item (IQ5_K, IQ5_KS): q = L-order nibbles, h[0] bit e = 5th bit of weight e; result = iq5nl_values + 2
// split into the two sign-fill halves va / vb
B200Q_HD void b200q_lut5_item(const b200q_item & I, b200q_canon & C) {
        for (int w = 0; w < 4; ++w) {
            const uint32_t q = I.q[w], qx = q ^ 0x88888888u; const uint32_t hb = (I.h[0] >> (8 * w)) & 0xFF;
            // byte masks from the 5th bits: lane j of half -> 0xFF if set
            const uint32_t m_lo = (((hb & 0xF) * 0x00204081u) & 0x01010101u) * 0xFFu;
            const uint32_t m_hi = (((hb >> 4) * 0x00204081u) & 0x01010101u) * 0xFFu;
            const uint32_t a_lo0 = b200q_prmt(B200Q_KV5_T0_0, B200Q_KV5_T0_1, q), b_lo0 = b200q_prmt(B200Q_KV5_T1_0, B200Q_KV5_T1_1, qx);
            const uint32_t a_lo1 = b200q_prmt(B200Q_KV5_T2_0, B200Q_KV5_T2_1, q), b_lo1 = b200q_prmt(B200Q_KV5_T3_0, B200Q_KV5_T3_1, qx);
            const uint32_t a_hi0 = b200q_prmt(B200Q_KV5_T0_0, B200Q_KV5_T0_1, q >> 16), b_hi0 = b200q_prmt(B200Q_KV5_T1_0, B200Q_KV5_T1_1, qx >> 16);
            const uint32_t a_hi1 = b200q_prmt(B200Q_KV5_T2_0, B200Q_KV5_T2_1, q >> 16), b_hi1 = b200q_prmt(B200Q_KV5_T3_0, B200Q_KV5_T3_1, qx >> 16);
            C.va[2 * w]     = (int)((a_lo1 & m_lo) | (a_lo0 & ~m_lo)); C.vb[2 * w]     = (int)((b_lo1 & m_lo) | (b_lo0 & ~m_lo));
            C.va[2 * w + 1] = (int)((a_hi1 & m_hi) | (a_hi0 & ~m_hi)); C.vb[2 * w + 1] = (int)((b_hi1 & m_hi) | (b_hi0 & ~m_hi));
        }
}

template <int TYPE>
B200Q_HD void b200q_decode_item(const b200q_item & I, int64_t it, b200q_canon & C, const b200q_kv4 & T) {
    if (TYPE == B200Q_TYPE_IQ4_NL) {
        const float d = b200q_h2f((uint16_t)I.m[0]);
        for (int w = 0; w < 4; ++w) b200q_lut4(T, I.q[w], C.va[2 * w], C.vb[2 * w], C.va[2 * w + 1], C.vb[2 * w + 1]);
        C.dl[0] = C.dl[1] = d; C.ml[0] = C.ml[1] = 0.0f;
    } else if (TYPE == B200Q_TYPE_Q4_0) {
        const float d = b200q_h2f((uint16_t)I.m[0]);
        for (int w = 0; w < 4; ++w) { C.va[2 * w] = (int)(I.q[w] & 0x0F0F0F0Fu); C.va[2 * w + 1] = (int)((I.q[w] >> 4) & 0x0F0F0F0Fu); }
        C.dl[0] = C.dl[1] = d; C.ml[0] = C.ml[1] = 8.0f * d;
    } else if (TYPE == B200Q_TYPE_Q4_1 || TYPE == B200Q_TYPE_Q5_0 || TYPE == B200Q_TYPE_Q5_1) {
        // Q4_1: w = d*q + m ; Q5_0: w = d*(q5 - 16) ; Q5_1: w = d*q5 + m      (ggml-quants.c:1601-1673)
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF));
        for (int w = 0; w < 4; ++w) {
            uint32_t lo = I.q[w] & 0x0F0F0F0Fu, hi = (I.q[w] >> 4) & 0x0F0F0F0Fu;
            if (TYPE != B200Q_TYPE_Q4_1) { lo |= (I.h[0] << (4 - w)) & 0x10101010u; hi |= (I.h[0] >> w) & 0x10101010u; }
            C.va[2 * w] = (int)lo; C.va[2 * w + 1] = (int)hi;
        }
        C.dl[0] = C.dl[1] = d;
        C.ml[0] = C.ml[1] = TYPE == B200Q_TYPE_Q5_0 ? 16.0f * d : -b200q_h2f((uint16_t)(I.m[0] >> 16));
    } else if (TYPE == B200Q_TYPE_Q6_0) {
        const float d = b200q_h2f((uint16_t)I.m[0]);
        for (int w = 0; w < 4; ++w) {
            const uint32_t U = I.h[w / 2]; const int f0 = 2 * (w % 2), f1 = f0 + 1;
            uint32_t lo = I.q[w] & 0x0F0F0F0Fu, hi = (I.q[w] >> 4) & 0x0F0F0F0Fu;
            lo |= ((U >> (2 * f0)) & 0x03030303u) << 4; hi |= ((U >> (2 * f1)) & 0x03030303u) << 4;
            C.va[2 * w] = (int)lo; C.va[2 * w + 1] = (int)hi;
        }
        C.dl[0] = C.dl[1] = d; C.ml[0] = C.ml[1] = 32.0f * d;
    } else if (TYPE == B200Q_TYPE_Q8_0) {
        const float d = b200q_h2f((uint16_t)I.m[0]);
        for (int w = 0; w < 8; ++w) C.va[w] = (int)I.q[w];
        C.dl[0] = C.dl[1] = d; C.ml[0] = C.ml[1] = 0.0f;
    } else if (TYPE == B200Q_TYPE_Q4_K || TYPE == B200Q_TYPE_Q5_K) {
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)), dmin = b200q_h2f((uint16_t)(I.m[0] >> 16));
        int sc, m; b200q_scale_min_k4((int)(it % 8), I.m, sc, m);
        for (int w = 0; w < 4; ++w) {
            uint32_t lo = I.q[w] & 0x0F0F0F0Fu, hi = (I.q[w] >> 4) & 0x0F0F0F0Fu;
            if (TYPE == B200Q_TYPE_Q5_K) { lo |= (I.h[0] << (4 - w)) & 0x10101010u; hi |= (I.h[0] >> w) & 0x10101010u; }
            C.va[2 * w] = (int)lo; C.va[2 * w + 1] = (int)hi;
        }
        C.dl[0] = C.dl[1] = d * sc; C.ml[0] = C.ml[1] = dmin * m;
    } else if (TYPE == B200Q_TYPE_Q6_K) {
        const float d = b200q_h2f((uint16_t)I.m[1]);
        const int s0 = (int)(int8_t)(I.m[0] & 0xFF), s1 = (int)(int8_t)((I.m[0] >> 8) & 0xFF);
        for (int w = 0; w < 4; ++w) {
            const uint32_t U = I.h[w / 2]; const int f0 = 2 * (w % 2), f1 = f0 + 1;
            uint32_t lo = I.q[w] & 0x0F0F0F0Fu, hi = (I.q[w] >> 4) & 0x0F0F0F0Fu;
            lo |= ((U >> (2 * f0)) & 0x03030303u) << 4; hi |= ((U >> (2 * f1)) & 0x03030303u) << 4;
            C.va[2 * w] = (int)lo; C.va[2 * w + 1] = (int)hi;
        }
        C.dl[0] = d * s0; C.dl[1] = d * s1; C.ml[0] = 32.0f * C.dl[0]; C.ml[1] = 32.0f * C.dl[1];
    } else if (TYPE == B200Q_TYPE_Q2_K) {             // w = d*(sc & 0xF)*q - dmin*(sc >> 4), one {scale,min} byte per 16 weights
        const float d = b200q_h2f((uint16_t)(I.m[1] & 0xFFFF)), dmin = b200q_h2f((uint16_t)(I.m[1] >> 16));
        const uint32_t s0 = I.m[0] & 0xFF, s1 = (I.m[0] >> 8) & 0xFF;
        for (int f = 0; f < 4; ++f) { C.va[f] = (int)((I.q[0] >> (2 * f)) & 0x03030303u); C.va[4 + f] = (int)((I.q[1] >> (2 * f)) & 0x03030303u); }
        C.dl[0] = d * (float)(s0 & 0xF); C.dl[1] = d * (float)(s1 & 0xF); C.ml[0] = dmin * (float)(s0 >> 4); C.ml[1] = dmin * (float)(s1 >> 4);
    } else if (TYPE == B200Q_TYPE_Q3_K) {             // w = d*(sc - 32)*(q3 - 4), q3 = low2 | hbit << 2; 6-bit scales as in ggml-quants.c:2580-2586
        const float d = b200q_h2f((uint16_t)I.m[3]); const int s = (int)(it % 8);
        int sc[2];
        for (int t = 0; t < 2; ++t) {
            const int is = 2 * s + t, i = is >> 2, b = is & 3;
            const uint32_t lo4 = ((i & 1 ? I.m[1] : I.m[0]) >> (8 * b + 4 * (i >> 1))) & 0xF, hi2 = (I.m[2] >> (8 * b + 2 * i)) & 3;
            sc[t] = (int)(lo4 | (hi2 << 4)) - 32;
        }
        for (int f = 0; f < 4; ++f) {
            C.va[f]     = (int)(((I.q[0] >> (2 * f)) & 0x03030303u) | (((I.h[0] >> f) & 0x01010101u) << 2));
            C.va[4 + f] = (int)(((I.q[1] >> (2 * f)) & 0x03030303u) | (((I.h[0] >> (4 + f)) & 0x01010101u) << 2));
        }
        C.dl[0] = d * (float)sc[0]; C.dl[1] = d * (float)sc[1]; C.ml[0] = 4.0f * C.dl[0]; C.ml[1] = 4.0f * C.dl[1];
    } else if (TYPE == B200Q_TYPE_IQ2_K) {            // meta {half d; u16 extra; u8 scales[8]}; iq2nl_values = {-31,-13,1,17} (+5 when the extra bit is set)
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)); const int s = (int)(it % 8);
        const uint32_t ex = (I.m[0] >> 16) >> (2 * s), sc = b200q_byte(I.m, 4 + s);
        for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) {
            const uint32_t sel = (I.q[u] >> (2 * p)) & 0x33333333u;
            C.va[4 * u + 2 * p] = (int)b200q_prmt(0x1101F3E1u, 0u, sel); C.va[4 * u + 2 * p + 1] = (int)b200q_prmt(0x1101F3E1u, 0u, sel >> 16);
        }
        C.dl[0] = d * (float)((int)(sc & 0xF) - 8); C.dl[1] = d * (float)((int)(sc >> 4) - 8);
        C.ml[0] = (ex & 1) ? -5.0f * C.dl[0] : 0.0f; C.ml[1] = (ex & 2) ? -5.0f * C.dl[1] : 0.0f;
    } else if (TYPE == B200Q_TYPE_IQ2_KS || TYPE == B200Q_TYPE_IQ3_KS) {
        // meta {u16 extra; u8 scales[4]}, one 5-bit scale per 32 weights, rs = row scale; codebooks as IQ2_K / IQ3_K
        const int s = (int)(it % 8); const uint32_t extra = I.m[0] & 0xFFFF;
        int ls; uint32_t sel;
        if (TYPE == B200Q_TYPE_IQ2_KS) {              // scales[s/2] nibble s%2 | extra bit 8+s ; table bit s            (iqk_quantize.cpp:1893-1897)
            ls = (int)(((b200q_byte(I.m, 2 + s / 2) >> (4 * (s % 2))) & 0xF) | (((extra >> (8 + s)) & 1) << 4)) - 16; sel = (extra >> s) & 1;
        } else {                                      // scales[s%4] nibble s/4 | extra bit s ; table bit 8+s            (iqk_quantize.cpp:2784-2794)
            ls = (int)(((b200q_byte(I.m, 2 + s % 4) >> (4 * (s / 4))) & 0xF) | (((extra >> s) & 1) << 4)) - 16; sel = (extra >> (8 + s)) & 1;
        }
        const float dl = I.rs * (float)ls;
        for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) {
            if (TYPE == B200Q_TYPE_IQ2_KS) {
                const uint32_t x = (I.q[u] >> (2 * p)) & 0x33333333u;
                C.va[4 * u + 2 * p] = (int)b200q_prmt(0x1101F3E1u, 0u, x); C.va[4 * u + 2 * p + 1] = (int)b200q_prmt(0x1101F3E1u, 0u, x >> 16);
            } else {
                const uint32_t x = ((I.q[u] >> (2 * p)) & 0x33333333u) | (((I.h[0] >> (2 * u + p)) & 0x11111111u) << 2);
                C.va[4 * u + 2 * p] = (int)b200q_prmt(0xF6E9D8C1u, 0x2F1C0D01u, x); C.va[4 * u + 2 * p + 1] = (int)b200q_prmt(0xF6E9D8C1u, 0x2F1C0D01u, x >> 16);
            }
        }
        C.dl[0] = C.dl[1] = dl; C.ml[0] = C.ml[1] = sel ? (TYPE == B200Q_TYPE_IQ2_KS ? -5.0f : -4.0f) * dl : 0.0f;
    } else if (TYPE == B200Q_TYPE_IQ3_K) {            // meta {half d; u16 extra; u16 scales_h; u8 scales_l[8]}; iq3nl_values (+4 with the extra bit)
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)); const int s = (int)(it % 8);
        const uint32_t ex = (I.m[0] >> 16) >> (2 * s), sh = (I.m[1] & 0xFFFF) >> (2 * s), sl = b200q_byte(I.m, 6 + s);
        for (int u = 0; u < 2; ++u) for (int p = 0; p < 2; ++p) {
            const uint32_t sel = ((I.q[u] >> (2 * p)) & 0x33333333u) | (((I.h[0] >> (2 * u + p)) & 0x11111111u) << 2);
            C.va[4 * u + 2 * p] = (int)b200q_prmt(0xF6E9D8C1u, 0x2F1C0D01u, sel); C.va[4 * u + 2 * p + 1] = (int)b200q_prmt(0xF6E9D8C1u, 0x2F1C0D01u, sel >> 16);
        }
        C.dl[0] = d * (float)((2 * (int)(sl & 0xF) + 1) * ((sh & 1) ? -1 : 1)); C.dl[1] = d * (float)((2 * (int)(sl >> 4) + 1) * ((sh & 2) ? -1 : 1));
        C.ml[0] = (ex & 1) ? -4.0f * C.dl[0] : 0.0f; C.ml[1] = (ex & 2) ? -4.0f * C.dl[1] : 0.0f;
    } else if (TYPE == B200Q_TYPE_IQ4_XS) {           // meta {half d; u16 scales_h; u8 scales_l[4]}
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)); const uint32_t sh = I.m[0] >> 16; const int ib = (int)(it % 8);
        const uint32_t sl = (I.m[1] >> (8 * (ib / 2) + 4 * (ib % 2))) & 0xF;   // scales_l[ib/2] nibble ib%2
        const int ls = (int)(sl | (((sh >> (2 * ib)) & 3) << 4)) - 32;
        for (int w = 0; w < 4; ++w) b200q_lut4(T, I.q[w], C.va[2 * w], C.vb[2 * w], C.va[2 * w + 1], C.vb[2 * w + 1]);
        C.dl[0] = C.dl[1] = d * ls; C.ml[0] = C.ml[1] = 0.0f;
    } else if (TYPE == B200Q_TYPE_IQ4_K) {            // meta {half d; u16 extra; u8 scales_h[4]; u8 scales_l[8]}
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)); const int ib = (int)(it % 8);
        const uint32_t extra = (I.m[0] >> 16) >> (2 * ib);
        const uint32_t h = b200q_byte(I.m, 4 + ib / 2) >> (4 * (ib % 2)); const uint32_t sl = b200q_byte(I.m, 8 + ib);
        const int ls1 = (int)((sl & 0xF) | ((h << 4) & 0x30)) - 32, ls2 = (int)((sl >> 4) | ((h << 2) & 0x30)) - 32;
        for (int w = 0; w < 4; ++w) b200q_lut4(T, I.q[w], C.va[2 * w], C.vb[2 * w], C.va[2 * w + 1], C.vb[2 * w + 1]);
        C.dl[0] = d * ls1; C.dl[1] = d * ls2;
        C.ml[0] = (extra & 1) ? -4.0f * C.dl[0] : 0.0f; C.ml[1] = (extra & 2) ? -4.0f * C.dl[1] : 0.0f;   // iq4k_values[16+i] = kvalues[i] + 4
    } else if (TYPE == B200Q_TYPE_IQ4_KS) {           // m[0] = scale byte of this 32-block
        const uint32_t s = I.m[0];
        const float dl = I.rs * (float)((int)(s & 254) - 127);
        for (int w = 0; w < 4; ++w) b200q_lut4(T, I.q[w], C.va[2 * w], C.vb[2 * w], C.va[2 * w + 1], C.vb[2 * w + 1]);
        C.dl[0] = C.dl[1] = dl; C.ml[0] = C.ml[1] = (s & 1) ? -4.0f * dl : 0.0f;
    } else if (TYPE == B200Q_TYPE_MXFP4) {            // kvalues_mxfp4 (ggml-common.h:2250) = {0,1,2,3,4,6,8,12, 0,-1,-2,-3,-4,-6,-8,-12}, d = E8M0 / 2
        // sign-fill tables: A' = entries 0..7 minus the fill that the B lookup adds for q < 8 (0 for entry 0, -1 otherwise), B' = entries 8..15
        b200q_kv4 M; M.a0 = 0x04030200u; M.a1 = 0x0D090705u; M.b0 = 0xFDFEFF00u; M.b1 = 0xF4F8FAFCu; M.k16 = T.k16;
        const uint32_t e = I.m[0] & 0xFF;
        const float d = b200q_u2f(e >= 2 ? (e - 1) << 23 : (e == 0 ? 0x00200000u : 0x00400000u));      // ggml_e8m0_to_fp32_half, ggml-impl.h:40-45
        for (int w = 0; w < 4; ++w) b200q_lut4(M, I.q[w], C.va[2 * w], C.vb[2 * w], C.va[2 * w + 1], C.vb[2 * w + 1]);
        C.dl[0] = C.dl[1] = d; C.ml[0] = C.ml[1] = 0.0f;
    } else if (TYPE == B200Q_TYPE_IQ5_KS) {           // m[0] = scale byte of this 32-block, rs = row scale
        const uint32_t sc = I.m[0];
        const float dl = I.rs * (float)((int)(sc & 254) - 127);
        b200q_lut5_item(I, C);
        C.dl[0] = C.dl[1] = dl; C.ml[0] = C.ml[1] = (sc & 1) ? 0.0f : 2.0f * dl;    // tables hold v+2; odd scale byte selects the +2 codebook
    } else if (TYPE == B200Q_TYPE_IQ5_K) {            // meta {half d; u16 extra; u8 scales_h[4]; u8 scales_l[8]}
        // item s: c = s/2 (64-chunk), second = s%2.  Weights 0..15 of the item use scale dl(2*second) and extra bit (2*second),
        // weights 16..31 use dl(2*second+1) / extra bit (2*second+1)  (iqk_quantize.cpp:3128-3141).
        const float d = b200q_h2f((uint16_t)(I.m[0] & 0xFFFF)); const int s = (int)(it % 8), c = s / 2, second = s % 2;
        const uint32_t extra = ((I.m[0] >> 16) >> (4 * c)) >> (2 * second);
        const uint32_t sh = b200q_byte(I.m, 4 + c), sl = b200q_byte(I.m, 8 + 2 * c + second);
        const int ls1 = (int)((sl & 0xF) | ((sh << (4 - 4 * second)) & 0x30)) - 32;     // second=0: sh<<4 ; second=1: sh>>0
        const int ls2 = (int)((sl >> 4)  | (second ? ((sh >> 2) & 0x30) : ((sh << 2) & 0x30))) - 32;
        b200q_lut5_item(I, C);
        C.dl[0] = d * ls1; C.dl[1] = d * ls2;
        // tables hold v+2: subtract 2 unless the extra bit selects the "+2" variant of the table
        C.ml[0] = (extra & 1) ? 0.0f : 2.0f * C.dl[0]; C.ml[1] = (extra & 2) ? 0.0f : 2.0f * C.dl[1];
    } else if (TYPE == B200Q_TYPE_IQ2_BN) {
        // wire block: 64 weights, byte j%16 field j/16.  Item it covers weights 32*(it%2) .. +31 of the block = fields 2*(it%2), 2*(it%2)+1
        const int f0 = 2 * (int)(it % 2);
        for (int w = 0; w < 4; ++w) { C.va[w] = (int)((I.q[w] >> (2 * f0)) & 0x03030303u); C.va[4 + w] = (int)((I.q[w] >> (2 * f0 + 2)) & 0x03030303u); }
        C.dl[0] = C.dl[1] = I.rs; C.ml[0] = C.ml[1] = I.rs;      // w = rs*(q-1)
    }
}

template <int TYPE>
B200Q_HD void b200q_decode_item(const b200q_item & I, int64_t it, b200q_canon & C) { b200q_decode_item<TYPE>(I, it, C, b200q_kv4_init()); }

// Dequantise canonical item to 32 floats (used by the bf16 dequantiser and by host tests)
template <bool HAS_B>
B200Q_HD void b200q_canon_to_float(const b200q_canon & C, float out[32]) {
    for (int e = 0; e < 32; ++e) {
        int q = (int)(int8_t)(C.va[e / 4] >> (8 * (e % 4)));
        if (HAS_B) q += (int)(int8_t)(C.vb[e / 4] >> (8 * (e % 4)));
        out[e] = C.dl[e / 16] * (float)q - C.ml[e / 16];
    }
}
