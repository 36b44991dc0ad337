// tools/membench.cu — calibration micro-benchmarks for the decode kernel design (not part of the product):
// how many bytes in flight per SM does an H100 need to stream weights at HBM speed, via LDG.128 vs cp.async.bulk rings?
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

template <int U>
__global__ void k_ldg(const uint4 * __restrict__ p, size_t n16, unsigned * out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; const size_t stride = (size_t)gridDim.x * blockDim.x;
    unsigned acc = 0;
    for (; i + (U - 1) * stride < n16; i += U * stride) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = __ldg(p + i + u * stride);
#pragma unroll
        for (int u = 0; u < U; ++u) acc += v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    if (acc == 0x12345) out[0] = acc;
}

__device__ __forceinline__ uint32_t s32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
// each warp owns S stages of CH bytes; lane 0 issues cp.async.bulk, all lanes consume (xor-reduce) from smem
template <int S, int CH>
__global__ void k_bulk(const unsigned char * __restrict__ p, size_t nbytes, unsigned * out) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    unsigned char * buf = smem + (size_t)warp * S * CH;
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + (size_t)nw * S * CH) + warp * S;
    if (lane == 0) for (int s = 0; s < S; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bars[s])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    const size_t gw = (size_t)blockIdx.x * nw + warp, tw = (size_t)gridDim.x * nw;
    const size_t nch = nbytes / CH;
    auto issue = [&](size_t c, int s) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&bars[s])), "r"(CH) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(s32(buf + (size_t)s * CH)), "l"(p + c * CH), "r"(CH), "r"(s32(&bars[s])) : "memory");
    };
    size_t c = gw; int k = 0;
    if (lane == 0) for (int s = 0; s < S; ++s) if (gw + (size_t)s * tw < nch) issue(gw + (size_t)s * tw, s);
    unsigned acc = 0;
    for (; c < nch; c += tw, ++k) {
        const int s = k % S; const uint32_t ph = (k / S) & 1;
        asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}" ::"r"(s32(&bars[s])), "r"(ph) : "memory");
        const uint4 * b = reinterpret_cast<const uint4 *>(buf + (size_t)s * CH);
#pragma unroll
        for (int i = lane; i < CH / 16; i += 32) { const uint4 v = b[i]; acc += v.x ^ v.y ^ v.z ^ v.w; }
        __syncwarp();
        const size_t nc = c + (size_t)S * tw;
        if (lane == 0 && nc < nch) issue(nc, s);
    }
    if (acc == 0x12345) out[0] = acc;
}

// Round 2: the decode ring as it really issues its copies.  A stage = NC bulk copies of sz[c] bytes, copy c streaming its own region
// (plane) of the buffer; W warps per CTA own S stages each, lane 0 re-issues, 2 CTAs per SM.  Question: how does the NUMBER of outstanding
// bulk copies per SM (at constant bytes in flight) change the achieved HBM bandwidth?
struct multi_cfg { int nc; int sz[4]; };
template <int S>
__global__ void __launch_bounds__(384, 2) k_bulk_multi(const unsigned char * __restrict__ p, size_t nbytes, multi_cfg cfg, unsigned * out) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    int stage = 0; for (int c = 0; c < cfg.nc; ++c) stage += cfg.sz[c];
    unsigned char * buf = smem + (size_t)warp * S * stage;
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + (size_t)nw * S * stage) + warp * S;
    if (lane == 0) for (int s = 0; s < S; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&bars[s])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    const size_t gw = (size_t)blockIdx.x * nw + warp, tw = (size_t)gridDim.x * nw;
    const size_t nch = nbytes / stage;                       // stage-sized units in the whole buffer
    // region c holds the sz[c]-byte pieces of all units back to back (like a plane)
    size_t reg_off[4]; { size_t o = 0; for (int c = 0; c < cfg.nc; ++c) { reg_off[c] = o; o += nch * cfg.sz[c]; } }
    auto issue = [&](size_t u, int s) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(&bars[s])), "r"(stage) : "memory");
        int o = 0;
        for (int c = 0; c < cfg.nc; ++c) {
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(s32(buf + (size_t)s * stage + o)), "l"(p + reg_off[c] + u * cfg.sz[c]), "r"(cfg.sz[c]), "r"(s32(&bars[s])) : "memory");
            o += cfg.sz[c];
        }
    };
    size_t u = gw; int k = 0;
    if (lane == 0) for (int s = 0; s < S; ++s) if (gw + (size_t)s * tw < nch) issue(gw + (size_t)s * tw, s);
    unsigned acc = 0;
    for (; u < nch; u += tw, ++k) {
        const int s = k % S; const uint32_t ph = (k / S) & 1;
        asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}" ::"r"(s32(&bars[s])), "r"(ph) : "memory");
        const uint4 * b = reinterpret_cast<const uint4 *>(buf + (size_t)s * stage);
        for (int i = lane; i < stage / 16; i += 32) { const uint4 v = b[i]; acc += v.x ^ v.y ^ v.z ^ v.w; }
        __syncwarp();
        const size_t nu = u + (size_t)S * tw;
        if (lane == 0 && nu < nch) issue(nu, s);
    }
    if (acc == 0x12345) out[0] = acc;
}

int main(int argc, char ** argv) {
    if (argc > 1 && argv[1][0] == 'r') {            // round-2 study only
        const size_t nbytes = (size_t)2 << 30;
        unsigned char * d; unsigned * out; CK(cudaMalloc(&d, nbytes)); CK(cudaMalloc(&out, 4)); CK(cudaMemset(d, 1, nbytes));
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        struct { const char * name; multi_cfg c; } cases[] = {
            {"4 copies: 2x2048 + 2x256 (round-1 ring)", {4, {2048, 2048, 256, 256}}},
            {"2 copies: 4096 + 512 (pair rows merged)", {2, {4096, 512, 0, 0}}},
            {"2 copies: 2304 + 2304 (planes merged per row)", {2, {2304, 2304, 0, 0}}},
            {"1 copy: 4608 (unit-major layout)", {1, {4608, 0, 0, 0}}},
            {"1 copy: 9216 (4-row units)", {1, {9216, 0, 0, 0}}},
        };
        for (auto & cs : cases) for (int W : {11, 7}) for (int S : {2, 3}) {
            int stage = 0; for (int c = 0; c < cs.c.nc; ++c) stage += cs.c.sz[c];
            const size_t sm = (size_t)W * S * stage + W * S * 8 + 64;
            if (sm > 113 * 1024) continue;
            float ms = 0;
            for (int rep = 0; rep < 4; ++rep) {
                if (rep == 1) cudaEventRecord(e0);
                if (S == 2) { cudaFuncSetAttribute(k_bulk_multi<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); k_bulk_multi<2><<<264, (W + 1) * 32 - 32, sm>>>(d, nbytes, cs.c, out); }
                else        { cudaFuncSetAttribute(k_bulk_multi<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); k_bulk_multi<3><<<264, (W + 1) * 32 - 32, sm>>>(d, nbytes, cs.c, out); }
            }
            cudaEventRecord(e1); CK(cudaDeviceSynchronize()); cudaEventElapsedTime(&ms, e0, e1);
            printf("%-48s W=%2d x2 CTA S=%d  copies in flight/SM %3d  bytes in flight/SM %6.1f KB : %8.1f GB/s\n", cs.name, W, S, 2 * W * S * cs.c.nc, 2.0 * W * S * stage / 1024, nbytes / (ms / 3) / 1e6);
        }
        return 0;
    }
    const size_t nbytes = (size_t)4 << 30;        // 4 GiB >> L2
    unsigned char * d; unsigned * out; CK(cudaMalloc(&d, nbytes)); CK(cudaMalloc(&out, 4)); CK(cudaMemset(d, 1, nbytes));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto report = [&](const char * name, float ms, size_t bytes) { printf("%-44s %8.3f ms  %8.1f GB/s\n", name, ms, bytes / ms / 1e6); };
#define RUN(name, bytes, ...) { __VA_ARGS__; CK(cudaDeviceSynchronize()); cudaEventRecord(e0); for (int r = 0; r < 3; ++r) { __VA_ARGS__; } cudaEventRecord(e1); CK(cudaDeviceSynchronize()); float ms; cudaEventElapsedTime(&ms, e0, e1); report(name, ms / 3, bytes); }
    const size_t n16 = nbytes / 16;
    RUN("ldg U=1 132x1024", nbytes, (k_ldg<1><<<132, 1024>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=2 132x1024", nbytes, (k_ldg<2><<<132, 1024>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=4 132x1024", nbytes, (k_ldg<4><<<132, 1024>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=8 132x1024", nbytes, (k_ldg<8><<<132, 1024>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=4 132x512", nbytes, (k_ldg<4><<<132, 512>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=8 132x512", nbytes, (k_ldg<8><<<132, 512>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=4 264x512", nbytes, (k_ldg<4><<<264, 512>>>((const uint4 *)d, n16, out)));
    RUN("ldg U=4 528x512 (4 CTA/SM x 16 warps)", nbytes, (k_ldg<4><<<528, 512>>>((const uint4 *)d, n16, out)));
    // small problem sizes (one matrix): latency-dominated
    for (size_t mb : {9, 33, 66, 295}) {
        char nm[64]; snprintf(nm, 64, "ldg U=4 264x512 %zu MB", mb);
        RUN(nm, mb << 20, (k_ldg<4><<<264, 512>>>((const uint4 *)d, (mb << 20) / 16, out)));
        snprintf(nm, 64, "ldg U=8 132x1024 %zu MB", mb);
        RUN(nm, mb << 20, (k_ldg<8><<<132, 1024>>>((const uint4 *)d, (mb << 20) / 16, out)));
    }
#define BULK(S, CH, W) { size_t sm = (size_t)W * S * CH + W * S * 8 + 64; cudaFuncSetAttribute(k_bulk<S, CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); char nm[64]; snprintf(nm, 64, "bulk S=%d CH=%d W=%d (%zu KB/SM)", S, CH, W, sm / 1024); RUN(nm, nbytes, (k_bulk<S, CH><<<132, W * 32, sm>>>(d, nbytes, out))); }
    BULK(2, 2048, 8) BULK(4, 2048, 8) BULK(4, 2048, 16) BULK(6, 2048, 16) BULK(2, 8192, 8) BULK(3, 8192, 8) BULK(2, 4096, 16) BULK(3, 4096, 16) BULK(8, 1024, 16)
    for (size_t mb : {9, 33, 66}) {
        size_t sm = (size_t)16 * 4 * 2048 + 16 * 4 * 8 + 64; char nm[64]; snprintf(nm, 64, "bulk S=4 CH=2048 W=16 %zu MB", mb);
        RUN(nm, mb << 20, (k_bulk<4, 2048><<<132, 512, sm>>>(d, mb << 20, out)));
    }
    return 0;
}
