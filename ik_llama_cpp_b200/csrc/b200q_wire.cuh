// b200q_wire.cuh — "wire layout" types: consumed verbatim in their GGUF byte layout (no plane repack), decoded 32 weights at a time.
//
// The 23 plane-layout types of b200q_types.cuh are the ones with a 16-byte low-bit plane per item; the rest of what the reference's CUDA
// back-end accepts for MUL_MAT (ggml/src/ggml-cuda.cu:4862-4917) is served from here:
//   grid-codebook types   IQ2_XXS IQ2_XS IQ2_S IQ3_XXS IQ3_S IQ1_S IQ1_M            (ggml-quants.c:3674-3911, ggml-common.h block_iq*)
//   IQK types             IQ6_K IQ4_KSS IQ2_KL IQ1_BN                               (iqk/iqk_quantize.cpp:3448, :5161, :2243, :375)
//   trellis types         IQ1_KT IQ2_KT IQ3_KT IQ4_KT                               (iqk/iqk_quantize.cpp:9470, :9751, :10021, :10286)
//   row-interleaved x4    IQ2_K_R4 IQ3_K_R4 IQ4_K_R4 IQ5_K_R4 IQ4_KS_R4 IQ5_KS_R4 IQ1_S_R4 IQ1_M_R4   (iqk_quantize.cpp:7586, :7460, :6700, :6838, :5879, :6946, :8195, :8336)
// One function per type family: b200q_wire_decode32<TYPE>(tensor base, K, row, it, w[32]) = weights 32*it .. 32*it+31 of `row` as f32,
// bit-identical to the reference's to_float (checked against the oracle on the host: tests/test_host_emulation.py, and on the device).
// The kernels that use it (b200q_wire.cu) are the generic feeders: a q8_1 mat-vec and the bf16 dequantiser of the wgmma GEMM.
// Codebooks: b200q_codebooks.h, generated from values extracted by RUNNING the reference (tests/golden/gen_codebooks.py).
#pragma once
#include "b200q_types.cuh"
#include "b200q_codebooks.h"

B200Q_HD uint32_t b200q_rd16(const uint8_t * p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
B200Q_HD uint32_t b200q_rd32(const uint8_t * p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
B200Q_HD float b200q_rdf32(const uint8_t * p) { return b200q_u2f(b200q_rd32(p)); }
B200Q_HD float b200q_sgn(uint32_t mask, int j) { return (mask >> j) & 1 ? -1.0f : 1.0f; }
// separately rounded multiply / add: never contracted into an FMA (the reference's to_float rounds each step; host builds use -ffp-contract=off)
B200Q_HD float b200q_mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
B200Q_HD float b200q_add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// value tables of the IQK non-linear types (ggml-common.h:2212-2235), indexable: base table, then the shifted copy selected by the `extra` bit
#if defined(__CUDACC__)
#define B200Q_VT static __device__ const
#else
#define B200Q_VT static const
#endif
B200Q_VT int8_t b200q_iq4k_values[32] = {-127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113, -123, -100, -79, -61, -45, -31, -18, -6, 5, 17, 29, 42, 57, 73, 93, 117};
B200Q_VT int8_t b200q_iq5nl_values[64] = {-126, -114, -103, -92, -83, -74, -65, -57, -50, -43, -36, -30, -24, -18, -12, -6, -1, 5, 11, 17, 23, 29, 36, 43, 51, 59, 68, 77, 87, 97, 109, 121,
                                          -124, -112, -101, -90, -81, -72, -63, -55, -48, -41, -34, -28, -22, -16, -10, -4, 1, 7, 13, 19, 25, 31, 38, 45, 53, 61, 70, 79, 89, 99, 111, 123};
B200Q_VT int8_t b200q_iq2nl_values[8] = {-31, -13, 1, 17, -26, -8, 6, 22};
B200Q_VT int8_t b200q_iq3nl_values[16] = {-63, -40, -23, -10, 1, 13, 28, 47, -59, -36, -19, -6, 5, 17, 32, 51};

// trellis generator of the IQx_KT types (integer variant of QuantizerIQKT::set_values, iqk/iqk_quantize.cpp:8626-8640)
B200Q_HD void b200q_kt_values(uint32_t idx, uint32_t offset, int n, float scale, bool is_abs, float * out) {
    uint32_t x = idx + offset;
    for (int k = 0; k < n; ++k) {
        x *= 0xCBAC1FEDu;
        const uint32_t s = x & 0x3f3f3f3fu;
        float v = (float)((int)(s & 0xff) + (int)((s >> 8) & 0xff) + (int)((s >> 16) & 0xff) + (int)(s >> 24)) - 126.0f;
        if (is_abs) v = v < 0.0f ? -v : v;
        out[k] = scale * v;
    }
}

// weights 32*it .. 32*it+31 of row `row` of a [M x K] tensor of wire type TYPE stored verbatim at `base`
template <int TYPE>
B200Q_HD void b200q_wire_decode32(const uint8_t * base, int64_t K, int64_t row, int64_t it, float * w) {
    b200q_wire_geom G; b200q_wire_geom_of(TYPE, G);
    const int64_t rs = b200q_wire_type_row_size(G, K);
    if (G.interleave == 4) {
        // ---- 4 rows interleaved: group = {4 row scales (if any)}{blocks of 4 rows} -------------------------------------------------
        const uint8_t * grp = base + (row / 4) * 4 * rs; const int r = (int)(row % 4);
        const int64_t ibl = (it * 32) / G.qk; const int ib = (int)(it % (G.qk / 32));
        const uint8_t * x = grp + 4 * G.row_meta + ibl * 4 * G.block_bytes;
        if (TYPE == B200Q_TYPE_IQ1_S_R4) {                 // block {u8 qs[16]; u16 qh[4]}
            const float d = b200q_h2f((uint16_t)b200q_rd16(grp + 2 * r));
            const uint32_t qh = b200q_rd16(x + 16 + 2 * r);
            const float shift = qh & 0x8000 ? -0.125f : 0.125f, dl = d * (float)(2 * ((qh >> 12) & 7) + 1);
            for (int i = 0; i < 4; ++i) { const uint64_t g = b200q_iq1s_grid[x[4 * i + r] | (((qh >> 3 * i) & 7) << 8)]; for (int j = 0; j < 8; ++j) w[8 * i + j] = dl * ((float)(int8_t)(g >> 8 * j) + shift); }
        } else if (TYPE == B200Q_TYPE_IQ1_M_R4) {          // block {u8 qs[16]; u8 qh[8]; u8 scales[4]}
            const float d = b200q_h2f((uint16_t)b200q_rd16(grp + 2 * r));
            const uint8_t * qs = x; const uint8_t * qh = x + 16; const uint32_t sc = x[24 + r];
            for (int i = 0; i < 2; ++i) {
                const float dl = d * (float)(i ? sc >> 4 : sc & 0xf); const uint32_t h = qh[4 * i + r];
                const uint64_t g1 = b200q_iq1s_grid[qs[8 * i + r] | ((h & 0x07) << 8)], g2 = b200q_iq1s_grid[qs[8 * i + r + 4] | ((h & 0x70) << 4)];
                const float e1 = h & 0x08 ? -0.125f : 0.125f, e2 = h & 0x80 ? -0.125f : 0.125f;
                for (int j = 0; j < 8; ++j) { w[16 * i + j] = dl * ((float)(int8_t)(g1 >> 8 * j) + e1); w[16 * i + j + 8] = dl * ((float)(int8_t)(g2 >> 8 * j) + e2); }
            }
        } else if (TYPE == B200Q_TYPE_IQ2_K_R4 || TYPE == B200Q_TYPE_IQ3_K_R4) {
            // IQ2_K_R4 {half d[4]; u8 extra[8]; u8 scales[32]; u8 qs[256]} ; IQ3_K_R4 {half d[4]; u8 extra[8]; u8 scales_h[8]; u8 scales_l[32]; u8 qs[256]; u8 qh[128]}
            const bool q3 = TYPE == B200Q_TYPE_IQ3_K_R4;
            const float d = b200q_h2f((uint16_t)b200q_rd16(x + 2 * r)); const uint8_t * extra = x + 8;
            const uint8_t * scales_h = x + 16; const uint8_t * scales_l = x + (q3 ? 24 : 16);
            const uint8_t * ql = x + (q3 ? 56 : 48) + 32 * ib; const uint8_t * qh = x + 56 + 256 + 16 * ib;
            float dl[2];
            for (int h = 0; h < 2; ++h) {
                const int is = 8 * ib + r + 4 * h; const int nib = (scales_l[is % 32] >> 4 * (is / 32)) & 0xf;
                dl[h] = q3 ? d * (float)((2 * nib + 1) * ((scales_h[is % 8] >> (is / 8)) & 1 ? -1 : 1)) : d * (float)(nib - 8);
            }
            const int e1 = (extra[r] >> ib) & 1, e2 = (extra[r + 4] >> ib) & 1;
            for (int i = 0; i < 4; ++i) for (int f = 0; f < 4; ++f) {
                const int a = (ql[4 * r + i] >> 2 * f) & 3, b = (ql[4 * r + i + 16] >> 2 * f) & 3;
                if (q3) {
                    const int ha = (qh[4 * r + i] >> f) & 1, hb = (qh[4 * r + i] >> (4 + f)) & 1;
                    w[i + 4 * f] = dl[0] * (float)b200q_iq3nl_values[8 * e1 + (a | (ha << 2))]; w[i + 4 * f + 16] = dl[1] * (float)b200q_iq3nl_values[8 * e2 + (b | (hb << 2))];
                } else { w[i + 4 * f] = dl[0] * (float)b200q_iq2nl_values[4 * e1 + a]; w[i + 4 * f + 16] = dl[1] * (float)b200q_iq2nl_values[4 * e2 + b]; }
            }
        } else {                                           // IQ4_K_R4 / IQ5_K_R4 {half d[4]; u8 extra[8]; u8 scales_h[16]; u8 scales_l[32]; u8 qs[512]; [u8 qh[128]]}
                                                           // IQ4_KS_R4 / IQ5_KS_R4 {u8 scales[32]; u8 qs[512]; [u8 qh[128]]} + f32 row scales
            const bool ks = TYPE == B200Q_TYPE_IQ4_KS_R4 || TYPE == B200Q_TYPE_IQ5_KS_R4, q5 = TYPE == B200Q_TYPE_IQ5_K_R4 || TYPE == B200Q_TYPE_IQ5_KS_R4;
            const float d = ks ? b200q_rdf32(grp + 4 * r) : b200q_h2f((uint16_t)b200q_rd16(x + 2 * r));
            const uint8_t * extra = x + 8; const uint8_t * scales_h = x + 16; const uint8_t * scales_l = x + 32;
            const uint8_t * qs = x + (ks ? 32 : 64) + 64 * ib + 4 * r; const uint8_t * qh = x + (ks ? 32 : 64) + 512 + 16 * ib + 4 * r;
            float dl[2]; int e[2];
            if (ks) { const uint32_t sc = x[4 * ib + r]; dl[0] = dl[1] = d * (float)((int)(sc & 254) - 127); e[0] = e[1] = (int)(sc & 1); }
            else for (int h = 0; h < 2; ++h) {
                const int is = 8 * ib + r + 4 * h;
                dl[h] = d * (float)((int)(((scales_l[is % 32] >> 4 * (is / 32)) & 0xf) | (((scales_h[is % 16] >> 2 * (is / 16)) & 3) << 4)) - 32);
                e[h] = (extra[r + 4 * h] >> ib) & 1;
            }
            // byte c (qs[i + 16 c]) holds the weights {i, i+8}, {i+16, i+24}, {i+4, i+12}, {i+20, i+28} (low, high nibble); 5th bits: qh[i] bit 2c + hn
            for (int i = 0; i < 4; ++i) for (int c = 0; c < 4; ++c) for (int hn = 0; hn < 2; ++hn) {
                const int pos = (c == 0 ? 0 : c == 1 ? 16 : c == 2 ? 4 : 20) + 8 * hn, h = pos >= 16 ? 1 : 0;
                const uint32_t byte = qs[i + 16 * c]; int q = (int)(hn ? byte >> 4 : byte & 0xf);
                if (q5) { q |= ((qh[i] >> (2 * c + hn)) & 1) << 4; w[i + pos] = dl[h] * (float)b200q_iq5nl_values[32 * e[h] + q]; }
                else w[i + pos] = dl[h] * (float)b200q_iq4k_values[16 * e[h] + q];
            }
        }
        return;
    }
    // ---- one row per wire row ---------------------------------------------------------------------------------------------------------
    const uint8_t * rowp = base + row * rs;
    if (TYPE == B200Q_TYPE_IQ1_BN) {                       // {u8 ql[12]; u8 extra} per 64 weights; half row scale; 5 ternary digits per byte
        const float rsc = b200q_h2f((uint16_t)b200q_rd16(rowp));
        const uint8_t * x = rowp + 2 + (it / 2) * 13; const uint32_t extra = x[12];
        const uint32_t mult[5] = {81, 27, 9, 3, 1};
        for (int h = 0; h < 2; ++h) {
            const int i16 = 2 * (int)(it % 2) + h; const uint8_t * ql = x + 3 * i16; float * o = w + 16 * h;
            for (int kk = 0; kk < 3; ++kk) for (int j = 0; j < 5; ++j) { const uint32_t v = (ql[kk] * mult[j]) & 0xff; o[5 * kk + j] = rsc * (float)((int)((v + (v >> 1)) >> 7) - 1); }
            const uint32_t v = (extra * mult[i16]) & 0xff; o[15] = rsc * (float)((int)((v + (v >> 1)) >> 7) - 1);
        }
        return;
    }
    const int64_t ibl = it / 8; const int s = (int)(it % 8);
    const uint8_t * x = rowp + G.row_meta + ibl * G.block_bytes;
    if (TYPE == B200Q_TYPE_IQ2_XXS) {                      // {half d; u16 qs[32]}: per 32 weights [4 grid indices][4 x 7-bit sign index | scale << 28]
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint8_t * a8 = x + 2 + 8 * s; const uint32_t a1 = b200q_rd32(a8 + 4);
        const float db = d * (0.5f + (float)(a1 >> 28)) * 0.25f;
        for (int l = 0; l < 4; ++l) { const uint64_t g = b200q_iq2xxs_grid[a8[l]]; const uint32_t sg = b200q_ksigns[(a1 >> 7 * l) & 127]; for (int j = 0; j < 8; ++j) w[8 * l + j] = db * (float)((g >> 8 * j) & 0xff) * b200q_sgn(sg, j); }
    } else if (TYPE == B200Q_TYPE_IQ2_XS) {                // {half d; u16 qs[32]; u8 scales[8]}
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint32_t sc = x[66 + s];
        const float db[2] = { d * (0.5f + (float)(sc & 0xf)) * 0.25f, d * (0.5f + (float)(sc >> 4)) * 0.25f };
        for (int l = 0; l < 4; ++l) { const uint32_t q = b200q_rd16(x + 2 + 2 * (4 * s + l)); const uint64_t g = b200q_iq2xs_grid[q & 511]; const uint32_t sg = b200q_ksigns[q >> 9]; for (int j = 0; j < 8; ++j) w[8 * l + j] = db[l / 2] * (float)((g >> 8 * j) & 0xff) * b200q_sgn(sg, j); }
    } else if (TYPE == B200Q_TYPE_IQ3_XXS) {               // {half d; u8 qs[64]; u8 scales_and_signs[32]}
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint8_t * qs = x + 2 + 8 * s; const uint32_t a = b200q_rd32(x + 66 + 4 * s);
        const float db = d * (0.5f + (float)(a >> 28)) * 0.5f;
        for (int l = 0; l < 4; ++l) {
            const uint32_t sg = b200q_ksigns[(a >> 7 * l) & 127], g1 = b200q_iq3xxs_grid[qs[2 * l]], g2 = b200q_iq3xxs_grid[qs[2 * l + 1]];
            for (int j = 0; j < 4; ++j) { w[8 * l + j] = db * (float)((g1 >> 8 * j) & 0xff) * b200q_sgn(sg, j); w[8 * l + 4 + j] = db * (float)((g2 >> 8 * j) & 0xff) * b200q_sgn(sg, j + 4); }
        }
    } else if (TYPE == B200Q_TYPE_IQ2_S) {                 // {half d; u8 qs[32]; u8 signs[32]; u8 qh[8]; u8 scales[8]}
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint8_t * qs = x + 2 + 4 * s; const uint8_t * sgn = x + 34 + 4 * s; const uint32_t qh = x[66 + s], sc = x[74 + s];
        const float db[2] = { d * (0.5f + (float)(sc & 0xf)) * 0.25f, d * (0.5f + (float)(sc >> 4)) * 0.25f };
        for (int l = 0; l < 4; ++l) { const uint64_t g = b200q_iq2s_grid[qs[l] | ((qh << (8 - 2 * l)) & 0x300)]; for (int j = 0; j < 8; ++j) w[8 * l + j] = db[l / 2] * (float)((g >> 8 * j) & 0xff) * b200q_sgn(sgn[l], j); }
    } else if (TYPE == B200Q_TYPE_IQ3_S) {                 // {half d; u8 qs[64]; u8 qh[8]; u8 signs[32]; u8 scales[4]}
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint8_t * qs = x + 2 + 8 * s; const uint32_t qh = x[66 + s]; const uint8_t * sgn = x + 74 + 4 * s; const uint32_t sc = x[106 + s / 2];
        const float db = d * (float)(1 + 2 * (int)(s & 1 ? sc >> 4 : sc & 0xf));
        for (int l = 0; l < 4; ++l) {
            const uint32_t g1 = b200q_iq3s_grid[qs[2 * l] | ((qh << (8 - 2 * l)) & 256)], g2 = b200q_iq3s_grid[qs[2 * l + 1] | ((qh << (7 - 2 * l)) & 256)];
            for (int j = 0; j < 4; ++j) { w[8 * l + j] = db * (float)((g1 >> 8 * j) & 0xff) * b200q_sgn(sgn[l], j); w[8 * l + 4 + j] = db * (float)((g2 >> 8 * j) & 0xff) * b200q_sgn(sgn[l], j + 4); }
        }
    } else if (TYPE == B200Q_TYPE_IQ1_S) {                 // {half d; u8 qs[32]; u16 qh[8]}
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint8_t * qs = x + 2 + 4 * s; const uint32_t qh = b200q_rd16(x + 34 + 2 * s);
        const float dl = d * (float)(2 * ((qh >> 12) & 7) + 1), delta = qh & 0x8000 ? -0.125f : 0.125f;
        for (int l = 0; l < 4; ++l) { const uint64_t g = b200q_iq1s_grid[qs[l] | (((qh >> 3 * l) & 7) << 8)]; for (int j = 0; j < 8; ++j) w[8 * l + j] = dl * ((float)(int8_t)(g >> 8 * j) + delta); }
    } else if (TYPE == B200Q_TYPE_IQ1_M) {                 // {u8 qs[32]; u8 qh[16]; u8 scales[8]}: half super-scale in the top nibbles of the 4 u16 scale words
        const uint8_t * qs = x + 4 * s; const uint8_t * qh = x + 32 + 2 * s; uint32_t sc[4]; for (int i = 0; i < 4; ++i) sc[i] = b200q_rd16(x + 48 + 2 * i);
        const float d = b200q_h2f((uint16_t)((sc[0] >> 12) | ((sc[1] >> 8) & 0x00f0) | ((sc[2] >> 4) & 0x0f00) | (sc[3] & 0xf000)));
        const float dl[2] = { d * (float)(2 * ((sc[s / 2] >> (6 * (s % 2) + 0)) & 7) + 1), d * (float)(2 * ((sc[s / 2] >> (6 * (s % 2) + 3)) & 7) + 1) };
        for (int l = 0; l < 4; ++l) {
            const uint32_t h = qh[l / 2] >> (4 * (l % 2)); const uint64_t g = b200q_iq1s_grid[qs[l] | ((h & 7) << 8)]; const float delta = h & 8 ? -0.125f : 0.125f;
            for (int j = 0; j < 8; ++j) w[8 * l + j] = dl[l / 2] * ((float)(int8_t)(g >> 8 * j) + delta);
        }
    } else if (TYPE == B200Q_TYPE_IQ6_K) {                 // {half d; u16 extra; i8 scales[16]; u8 qs[128]; u8 qh[64]}: cubic codebook A + q(B + q(-C + qD)) (+1 by the extra bit)
        const float A = -127.f, B = 6.2568f, C = 0.11218f, D = 0.0011972f;
        const float d = b200q_h2f((uint16_t)b200q_rd16(x)); const uint32_t extra = b200q_rd16(x + 2); const int8_t * sl = (const int8_t *)(x + 4);
        const int ib64 = s / 2, second = s % 2;
        const uint8_t * qs = x + 20 + 32 * ib64; const uint8_t * qh = x + 148 + 32 * (ib64 / 2); const int shift = 4 * (ib64 % 2) + 2 * second;
        for (int h = 0; h < 2; ++h) {
            const int is = 4 * ib64 + 2 * second + h; const float dl = d * (float)sl[is], m = (extra >> is) & 1 ? 1.0f : 0.0f;
            for (int j = 0; j < 16; ++j) {
                const uint32_t b = qs[16 * h + j]; const float q = (float)((second ? b >> 4 : b & 0xf) | (((qh[16 * h + j] >> shift) & 3) << 4));
                // dl * (A + q*(B + q*(-C + q*D)) + m), every step rounded like the reference's scalar code (iqk_quantize.cpp:3462-3476)
                const float p3 = b200q_add_rn(-C, b200q_mul_rn(q, D)), p2 = b200q_add_rn(B, b200q_mul_rn(q, p3)), p1 = b200q_add_rn(A, b200q_mul_rn(q, p2));
                w[16 * h + j] = b200q_mul_rn(dl, b200q_add_rn(p1, m));
            }
        }
    } else if (TYPE == B200Q_TYPE_IQ4_KSS) {               // row = {float d; blocks {u32 qs[32]}}: per 32 weights eight u16; bit 0 of each = one bit of the scale byte
        const float rsc = b200q_rdf32(rowp);
        uint32_t a[8]; uint32_t ls = 0;
        for (int kk = 0; kk < 8; ++kk) { const uint32_t q = b200q_rd16(x + 2 * (8 * s + kk)); uint32_t v = q & 0xfffe; v ^= v >> 1; a[kk] = v; ls |= (q & 1) << kk; }
        const float dl = rsc * (float)((int)(ls & 254) - 127); const int e = (int)(ls & 1);
        for (int j = 0; j < 16; ++j) { const uint32_t byte = (a[j / 2] >> (8 * (j % 2))) & 0xff; w[j] = dl * (float)b200q_iq4k_values[16 * e + (byte & 0xf)]; w[j + 16] = dl * (float)b200q_iq4k_values[16 * e + (byte >> 4)]; }
    } else if (TYPE == B200Q_TYPE_IQ2_KL) {                // row = {half d; blocks {u16 scales_h; u8 scales_l[4]; u8 qs[64]; u8 qh[16]}}: 5-bit index -> PAIR of values
        const float rsc = b200q_h2f((uint16_t)b200q_rd16(rowp));
        const uint32_t scales_h = b200q_rd16(x); const uint8_t * sl = x + 2; const int ib64 = s / 2, second = s % 2;
        const uint8_t * qs = x + 6 + 16 * ib64; const uint8_t * qh = x + 70;
        const float dl = rsc * (float)((int)(((sl[(2 * ib64 + second) % 4] >> 4 * (ib64 / 2)) & 0xf) | (((scales_h >> (4 * ib64 + 2 * second)) & 3) << 4)) - 32);
        for (int j = 0; j < 16; ++j) {
            const uint32_t idx = (second ? qs[j] >> 4 : qs[j] & 0xf) | (((qh[j] >> (2 * ib64 + second)) & 1) << 4); const uint32_t v = b200q_iq2kl_values[idx];
            w[2 * j] = dl * (float)(int8_t)(v & 0xff); w[2 * j + 1] = dl * (float)(int8_t)(v >> 8);
        }
    } else if (TYPE == B200Q_TYPE_IQ1_KT) {                // row = {float d; blocks {u8 sh[8]; u8 ql[32]; u8 qh[16]}}: 13-bit trellis index per 8 weights
        const float rsc = b200q_rdf32(rowp); const uint32_t sh = x[s]; const uint8_t * ql = x + 8; const uint8_t * qh = x + 40;
        const float sl = rsc * (float)b200q_iq4k_values[sh & 0xf];
        for (int ig = 0; ig < 4; ++ig) {
            uint32_t idx = ql[s * 4 + ig] | (((uint32_t)qh[(s % 4) * 4 + ig] << (8 - 4 * (s / 4))) & 0xf00); idx |= (sh << (8 - ig)) & 0x1000;
            b200q_kt_values(idx, 4096, 8, sl, false, w + 8 * ig);
        }
    } else if (TYPE == B200Q_TYPE_IQ2_KT || TYPE == B200Q_TYPE_IQ3_KT) {   // row = {float d; blocks {u8 scales[4]; u16 ql[32]; [u8 qh[32]]}}: 16-bit index per 8 weights;
                                                                            // indices 0..15 = weights 0..127, 16..31 = weights 128..255 (high scale nibble, high sign bits)
        const bool q3 = TYPE == B200Q_TYPE_IQ3_KT; const float rsc = b200q_rdf32(rowp);
        const int hi = s / 4, ib = s % 4; const uint32_t scb = x[ib], sn = hi ? scb >> 4 : scb & 0xf;
        const float sl = rsc * (q3 ? (float)sn : (float)b200q_iq4k_values[sn]);
        const uint8_t * ql = x + 4 + 32 * hi; const uint8_t * qh = x + 68;
        for (int ig = 0; ig < 4; ++ig) {
            b200q_kt_values(b200q_rd16(ql + 2 * (4 * ib + ig)), 4096, 8, sl, q3, w + 8 * ig);
            if (q3) for (int j = 0; j < 8; ++j) if ((qh[8 * ig + j] >> (ib + 4 * hi)) & 1) w[8 * ig + j] = -w[8 * ig + j];
        }
    } else if (TYPE == B200Q_TYPE_IQ4_KT) {                // row = {float d; blocks {u32 shb[8]; u8 ql[64]; u8 qh[32]}}: 15-bit index per 4 weights
        const float rsc = b200q_rdf32(rowp); const uint32_t shb = b200q_rd32(x + 4 * s); const uint8_t * ql = x + 32; const uint8_t * qh = x + 96;
        const uint32_t offset = shb & 1 ? 32768 + 4096 : 4096; const float sl = rsc * (float)((int)((shb & 0xff) >> 1) - 64);
        for (int ig = 0; ig < 8; ++ig) {
            const int jj = s * 8 + ig;
            const uint32_t idx = ql[jj] | (((uint32_t)qh[jj % 32] << (8 - 4 * (jj / 32))) & 0xf00) | (((shb >> (8 + 3 * ig)) & 7) << 12);
            b200q_kt_values(idx, offset, 4, sl, false, w + 4 * ig);
        }
    }
}

#define B200Q_FOR_WIRE_TYPES(X) X(B200Q_TYPE_IQ2_XXS) X(B200Q_TYPE_IQ2_XS) X(B200Q_TYPE_IQ3_XXS) X(B200Q_TYPE_IQ2_S) X(B200Q_TYPE_IQ3_S) X(B200Q_TYPE_IQ1_S) X(B200Q_TYPE_IQ1_M) \
    X(B200Q_TYPE_IQ6_K) X(B200Q_TYPE_IQ4_KSS) X(B200Q_TYPE_IQ2_KL) X(B200Q_TYPE_IQ1_BN) X(B200Q_TYPE_IQ1_KT) X(B200Q_TYPE_IQ2_KT) X(B200Q_TYPE_IQ3_KT) X(B200Q_TYPE_IQ4_KT) \
    X(B200Q_TYPE_IQ1_S_R4) X(B200Q_TYPE_IQ1_M_R4) X(B200Q_TYPE_IQ2_K_R4) X(B200Q_TYPE_IQ3_K_R4) X(B200Q_TYPE_IQ4_K_R4) X(B200Q_TYPE_IQ5_K_R4) X(B200Q_TYPE_IQ4_KS_R4) X(B200Q_TYPE_IQ5_KS_R4)
