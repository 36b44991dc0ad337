// b200q_api.cu — the C ABI of libb200q.so (see include/b200q.h for the reference interfaces each entry replaces).
#include "../../include/b200q.h"
#include "b200q_internal.h"
#include "b200q_decode_plan.h"
#include <cuda_runtime.h>
#include <mutex>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

int b200q_launch_allreduce_nvls(const float * in, float * out, int64_t n, void * mc_base, void * local_base, int64_t stride,
                                void * mc_flag, const void * local_flag, uint32_t world, void * seq, void * cta_counter, int sm_count, cudaStream_t st);

int b200q_launch_allreduce_nvls_2shot(const float * in, float * out_f32, void * out_bf16, int64_t n, void * mc_stage, void * local_stage,
                                      void * mc_flag, const void * local_flag, uint32_t world, uint32_t rank, void * state, int sm_count, cudaStream_t st);

namespace {
thread_local char g_err[512] = "";
int fail(int code, const char * fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
int cuda_fail(const char * what, cudaError_t e) { return fail(B200Q_E_CUDA, "%s: %s", what, cudaGetErrorString(e)); }

struct dev_info { int sm_count = 0; bool ok = false; };
dev_info & device_info() {
    static dev_info info[16]; static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) { static dev_info bad; return bad; }
    std::lock_guard<std::mutex> lk(mu);
    if (!info[dev].ok) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, dev) == cudaSuccess) { info[dev].sm_count = p.multiProcessorCount; info[dev].ok = true; }
    }
    return info[dev];
}
// the SM count of the current device; without a device, B200Q_E_CUDA
int device_sms(int & sms, const char * what) {
    const dev_info & di = device_info(); sms = di.sm_count;
    return di.ok ? B200Q_OK : fail(B200Q_E_CUDA, "%s: no CUDA device", what);
}
int check_launch(int rc, const char * what) {
    if (rc == 0) return B200Q_OK;
    if (rc == -1) return fail(B200Q_E_TYPE, "%s: unsupported ggml type", what);
    if (rc == -2) return fail(B200Q_E_SHAPE, "%s: unsupported shape", what);
    if (rc == -5) return fail(B200Q_E_NOMEM, "%s: workspace too small", what);
    if (rc > 0) return cuda_fail(what, (cudaError_t)rc);
    return fail(B200Q_E_CUDA, "%s: launch failed (%d)", what, rc);
}
// per-thread scratch for the host-buffer entry points
// (device-aware: a loader thread may serve several GPUs in turn; an allocation made on another device is never reused)
struct scratch { void * p = nullptr; size_t n = 0; int dev = -1; };
void release(scratch & s) {
    if (!s.p) return;
    int cur = 0; cudaGetDevice(&cur);
    if (s.dev >= 0 && s.dev != cur) { cudaSetDevice(s.dev); cudaFree(s.p); cudaSetDevice(cur); } else cudaFree(s.p);
    s.p = nullptr; s.n = 0; s.dev = -1;
}
int ensure(scratch & s, size_t n) {
    int cur = 0; cudaGetDevice(&cur);
    if (s.p && s.dev == cur && s.n >= n) return 0;
    release(s);
    cudaError_t e = cudaMalloc(&s.p, n);
    if (e != cudaSuccess) { s.p = nullptr; return cuda_fail("cudaMalloc(scratch)", e); }
    s.n = n; s.dev = cur; return 0;
}
constexpr size_t STAGE_KEEP = (size_t)64 << 20;      // upload staging above this size is freed right after use (model load)
thread_local scratch g_x, g_y, g_ws, g_stage;
// programmatic dependent launch for the decode kernels (default on; B200Q_PDL=0 or b200q_set_option("pdl",0) disables)
int & opt_ring() { static int v = [] { const char * e = getenv("B200Q_RING"); return e ? atoi(e) : 1; }(); return v; }
int & opt_fused() { static int v = [] { const char * e = getenv("B200Q_FUSED_GEMM"); return e ? atoi(e) : 1; }(); return v; }
// L2 warm-up of the next launch's weights: measured slower (the prefetch competes with the running kernel's own stream) -> opt-in
int & opt_pf() { static int v = [] { const char * e = getenv("B200Q_PREFETCH_NEXT"); return e ? atoi(e) : 0; }(); return v; }
int & opt_q8() { static int v = [] { const char * e = getenv("B200Q_Q8_HANDOFF"); return e ? atoi(e) : 1; }(); return v; }
int & opt_pdl() { static int v = [] { const char * e = getenv("B200Q_PDL"); return e ? atoi(e) : 1; }(); return v; }
}  // namespace

extern "C" {

int b200q_abi_version(void) { return B200Q_ABI_VERSION; }
const char * b200q_last_error(void) { return g_err; }
int b200q_set_option(const char * key, int value) {
    if (key && !strcmp(key, "pdl")) { opt_pdl() = value; return B200Q_OK; }
    if (key && !strcmp(key, "prefetch_next")) { opt_pf() = value; return B200Q_OK; }
    if (key && !strcmp(key, "q8_handoff")) { opt_q8() = value; return B200Q_OK; }
    if (key && !strcmp(key, "ring")) { opt_ring() = value; return B200Q_OK; }
    if (key && !strcmp(key, "fused_gemm")) { opt_fused() = value; return B200Q_OK; }
    return fail(B200Q_E_ARG, "b200q_set_option: unknown option");
}
int b200q_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }

int b200q_type_supported(int type) { b200q_layout L; return b200q_make_layout(type, 4, 256, &L) == 0 ? 1 : 0; }
int64_t b200q_wire_row_size(int type, int64_t k) { b200q_layout L; if (b200q_make_layout(type, 4, k, &L)) return -1; return b200q_wire_row_size(L); }
int64_t b200q_plane_bytes(int type, int64_t m, int64_t k) { b200q_layout L; if (b200q_make_layout(type, m, k, &L)) return -1; return L.total_bytes; }

int b200q_repack(int type, const void * wire_dev, void * planes_dev, int64_t m, int64_t k, void * stream) {
    b200q_layout L; int rc = b200q_make_layout(type, m, k, &L);
    if (rc) return check_launch(rc, "b200q_repack");
    return check_launch(b200q_launch_repack(wire_dev, planes_dev, L, 0, (cudaStream_t)stream), "b200q_repack");
}
int b200q_unrepack(int type, const void * planes_dev, void * wire_dev, int64_t m, int64_t k, void * stream) {
    b200q_layout L; int rc = b200q_make_layout(type, m, k, &L);
    if (rc) return check_launch(rc, "b200q_unrepack");
    // the inverse pass ORs bits into the wire buffer for some types: it clears what it needs itself
    return check_launch(b200q_launch_repack(wire_dev, const_cast<void *>(planes_dev), L, 1, (cudaStream_t)stream), "b200q_unrepack");
}
int b200q_set_tensor(int type, const void * wire_host, void * planes_dev, int64_t m, int64_t k, void * stream) {
    b200q_layout L; int rc = b200q_make_layout(type, m, k, &L);
    if (rc) return check_launch(rc, "b200q_set_tensor");
    const size_t nbytes = (size_t)b200q_wire_row_size(L) * m;
    if ((rc = ensure(g_stage, nbytes))) return rc;
    cudaStream_t st = (cudaStream_t)stream; cudaError_t e;
    if ((e = cudaMemcpyAsync(g_stage.p, wire_host, nbytes, cudaMemcpyHostToDevice, st)) != cudaSuccess) return cuda_fail("set_tensor H2D", e);
    if ((rc = check_launch(b200q_launch_repack(g_stage.p, planes_dev, L, 0, st), "b200q_set_tensor"))) return rc;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return cuda_fail("set_tensor sync", e);
    if (g_stage.n > STAGE_KEEP) release(g_stage);
    return B200Q_OK;
}
int b200q_get_tensor(int type, const void * planes_dev, void * wire_host, int64_t m, int64_t k, void * stream) {
    b200q_layout L; int rc = b200q_make_layout(type, m, k, &L);
    if (rc) return check_launch(rc, "b200q_get_tensor");
    const size_t nbytes = (size_t)b200q_wire_row_size(L) * m;
    if ((rc = ensure(g_stage, nbytes))) return rc;
    cudaStream_t st = (cudaStream_t)stream; cudaError_t e;
    if ((rc = check_launch(b200q_launch_repack(g_stage.p, const_cast<void *>(planes_dev), L, 1, st), "b200q_get_tensor"))) return rc;
    if ((e = cudaMemcpyAsync(wire_host, g_stage.p, nbytes, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return cuda_fail("get_tensor D2H", e);
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return cuda_fail("get_tensor sync", e);
    if (g_stage.n > STAGE_KEEP) release(g_stage);
    return B200Q_OK;
}

// pending "next weights" hint of this thread (b200q_decode_prefetch_next): consumed by the next decode launch
static thread_local b200q_mmvq_desc g_next; static thread_local bool g_next_valid = false;
static inline void attach_next(b200q_mmvq_desc & d) { d.next = nullptr; if (g_next_valid && opt_pf()) d.next = &g_next; g_next_valid = false; }

// a decode launch's descriptor, zeroed, with type, K, x and the launch options; the caller adds its segments and its own fields
static int mmvq_desc(b200q_mmvq_desc & d, int type, int64_t k, const float * x, const char * what) {
    int sms = 0; if (const int rc = device_sms(sms, what)) return rc;
    memset(&d, 0, sizeof d);
    d.type = type; d.K = k; d.x = x; d.sm_count = sms; d.pdl = opt_pdl(); d.ring = opt_ring();
    return B200Q_OK;
}

int b200q_decode_prefetch_next(int type, int n_tensors, const void * const * W, const void * W_gate, const int64_t * m, int64_t k) {
    g_next_valid = false;
    if (n_tensors < 1 || n_tensors > B200Q_MAX_SEGS || !W || !m || (W_gate && n_tensors != 1)) return fail(B200Q_E_ARG, "b200q_decode_prefetch_next: bad argument");
    if (const int rc = mmvq_desc(g_next, type, k, nullptr, "b200q_decode_prefetch_next")) return rc;
    g_next.n_seg = n_tensors; g_next.ncols = 1;
    for (int i = 0; i < n_tensors; ++i) g_next.seg[i] = {W[i], i == 0 ? W_gate : nullptr, nullptr, nullptr, m[i]};
    g_next_valid = true;
    return B200Q_OK;
}

// every decode entry but the tensor-parallel one launches here: n columns x_stride floats apart (0: K); `plan`: what the last piece launched
static int mmvq_cols(b200q_mmvq_desc & d, int n, int64_t x_stride, cudaStream_t st, const char * what, b200q_mmvq_plan * plan = nullptr) {
    attach_next(d);
    // the kernel is instantiated for 1/2/4/8 columns: cover n with the largest pieces
    int done = 0;
    const int64_t xs = x_stride ? x_stride : d.K;
    if (((uintptr_t)d.x & 15) || (xs & 3)) return fail(B200Q_E_ARG, "%s: activations must be 16-byte aligned with a row stride multiple of 4 floats", what);
    float * dst0[B200Q_MAX_SEGS]; for (int i = 0; i < d.n_seg; ++i) dst0[i] = d.seg[i].dst;
    const float * x0 = d.x;
    const int64_t max_cols = b200q_mmvq_max_cols(d.K);
    while (done < n) {
        int c = 8; while (c > n - done) c >>= 1;
        while (c > 1 && c > max_cols) c >>= 1;
        if (c > max_cols) return fail(B200Q_E_SHAPE, "%s: K=%lld too large for the mat-vec kernel", what, (long long)d.K);
        d.ncols = c; d.x = x0 + (int64_t)done * xs; d.x_stride = xs;
        for (int i = 0; i < d.n_seg; ++i) d.seg[i].dst = dst0[i] + (int64_t)done * d.seg[i].M;
        int rc = check_launch(b200q_launch_mmvq(d, st, plan), what);
        if (rc) return rc;
        d.next = nullptr;
        done += c;
    }
    return B200Q_OK;
}

int b200q_mul_mat_vec(int type, const void * W, const float * x, float * dst, int64_t m, int64_t k, int n, int64_t x_stride,
                      const float * bias, void * stream) {
    if (!W || !x || !dst || m <= 0 || n < 1) return fail(B200Q_E_ARG, "b200q_mul_mat_vec: bad argument");
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_mul_mat_vec")) return rc;
    d.n_seg = 1; d.seg[0] = {W, nullptr, dst, bias, m};
    return mmvq_cols(d, n, x_stride, (cudaStream_t)stream, "b200q_mul_mat_vec");
}
int b200q_mul_mat_vec_multi(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m, int64_t k,
                            const float * x, int n, int64_t x_stride, void * stream) {
    if (n_tensors < 1 || n_tensors > B200Q_MAX_SEGS || !W || !dst || !m || !x || n < 1) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_multi: bad argument");
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_mul_mat_vec_multi")) return rc;
    d.n_seg = n_tensors;
    for (int i = 0; i < n_tensors; ++i) d.seg[i] = {W[i], nullptr, dst[i], nullptr, m[i]};
    return mmvq_cols(d, n, x_stride, (cudaStream_t)stream, "b200q_mul_mat_vec_multi");
}
int b200q_fused_up_gate_vec(int type, const void * W_up, const void * W_gate, const float * x, float * dst, int64_t m, int64_t k, int n,
                            int64_t x_stride, int unary, float limit, void * stream) {
    if (!W_up || !W_gate || !x || !dst || m <= 0 || n < 1) return fail(B200Q_E_ARG, "b200q_fused_up_gate_vec: bad argument");
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_fused_up_gate_vec")) return rc;
    d.n_seg = 1; d.seg[0] = {W_up, W_gate, dst, nullptr, m}; d.act = unary; d.limit = limit;
    return mmvq_cols(d, n, x_stride, (cudaStream_t)stream, "b200q_fused_up_gate_vec");
}

/* q8 hand-off between FUSED_UP_GATE and the following MUL_MAT (ffn_down), n = 1: the up/gate launch also emits its result quantised to
 * q8_1 (by the warp that completes each 32-row block), the next mat-vec bulk-copies that image instead of re-quantising per CTA. */
size_t b200q_q8_scratch_bytes(int64_t k) { return k > 0 && k % 32 == 0 ? b200q_q8_image_bytes(k) : 0; }
int b200q_q8_scratch_init(void * q8, int64_t k, void * stream) {
    if (!q8 || k <= 0 || k % 32) return fail(B200Q_E_ARG, "b200q_q8_scratch_init: bad argument");
    cudaError_t e = cudaMemsetAsync(q8, 0, b200q_q8_image_bytes(k), (cudaStream_t)stream);
    return e == cudaSuccess ? B200Q_OK : cuda_fail("b200q_q8_scratch_init", e);
}
int b200q_fused_up_gate_vec_q8(int type, const void * W_up, const void * W_gate, const float * x, float * dst, int64_t m, int64_t k,
                               int unary, float limit, void * q8_out, int * q8_produced, void * stream) {
    if (q8_produced) *q8_produced = 0;
    if (!W_up || !W_gate || !x || !dst || m <= 0) return fail(B200Q_E_ARG, "b200q_fused_up_gate_vec_q8: bad argument");
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_fused_up_gate_vec_q8")) return rc;
    d.n_seg = 1; d.seg[0] = {W_up, W_gate, dst, nullptr, m}; d.act = unary; d.limit = limit;
    if (q8_out && opt_q8()) d.q8_out = q8_out;     // a shape not eligible for the hand-off is planned as the plain launch
    b200q_mmvq_plan p;
    const int rc = mmvq_cols(d, 1, 0, (cudaStream_t)stream, "b200q_fused_up_gate_vec_q8", &p);
    if (rc == 0 && q8_produced) *q8_produced = p.q8 == 2;
    return rc;
}
int b200q_mul_mat_vec_q8(int type, const void * W, const float * x, const void * q8_in, float * dst, int64_t m, int64_t k,
                         const float * bias, void * stream) {
    if (!W || !x || !dst || m <= 0) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_q8: bad argument");
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_mul_mat_vec_q8")) return rc;
    d.n_seg = 1; d.seg[0] = {W, nullptr, dst, bias, m};
    if (q8_in && opt_q8()) d.q8_in = q8_in;
    return mmvq_cols(d, 1, 0, (cudaStream_t)stream, "b200q_mul_mat_vec_q8");
}

int b200q_mul_mat_vec_tp(int type, int n_tensors, const void * const * W, const void * W_gate, float * const * dst, const int64_t * m,
                         int64_t k, const float * x, int unary, float limit, const b200q_nvls_comm * comm, int reduce_in, int reduce_out, void * stream) {
    if (n_tensors < 1 || n_tensors > B200Q_MAX_SEGS || !W || !m || (W_gate && n_tensors != 1)) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: bad argument");
    // the sum over ranks of unary(gate . x) * (up . x) means nothing: a fused up/gate launch may consume a reduce, never produce one
    if (W_gate && reduce_out) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: a fused up/gate launch cannot reduce_out");
    // unicast variant (peer stores, rows of a CTA coalesced): measured slower than the multicast stores at 2 GPUs -> opt-in only.  Only then may
    // ll_mc be NULL: no launch ever issues multimem.st to an address that is not a multicast mapping.
    static const int ucast_env = [] { const char * e = getenv("B200Q_TP_UNICAST"); return e ? atoi(e) : 0; }();
    const bool ucast = ucast_env && comm && comm->ll_peers && comm->world_size <= 8;
    if ((reduce_in || reduce_out) && (!comm || (!comm->ll_mc && !ucast) || !comm->ll_local || !comm->ll_reduced || !comm->ll_state || comm->ll_stride < 1 || comm->world_size < 2 || comm->rank >= comm->world_size
                                      || ((uintptr_t)comm->ll_mc & 15) || ((uintptr_t)comm->ll_local & 15) || ((uintptr_t)comm->ll_reduced & 15) || (comm->ll_stride & 1)))
        return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: incomplete communicator");
    if (!reduce_in && !x) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: x is NULL");
    if (!reduce_out && !dst) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: dst is NULL");
    // launched directly, not through mmvq_cols: x may be NULL (reduce_in), and the launch does not consume a b200q_decode_prefetch_next hint
    b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, "b200q_mul_mat_vec_tp")) return rc;
    d.n_seg = n_tensors; d.x_stride = k; d.ncols = 1; d.act = unary; d.limit = limit; d.ring = 1;
    for (int i = 0; i < n_tensors; ++i) d.seg[i] = {W[i], i == 0 ? W_gate : nullptr, dst ? dst[i] : nullptr, nullptr, m[i]};
    if (comm) {
        d.tp.ll_mc = (float2 *)comm->ll_mc; d.tp.ll_local = (const float2 *)comm->ll_local; d.tp.ll_red = (float2 *)comm->ll_reduced; d.tp.ll_stride = comm->ll_stride;
        d.tp.world = comm->world_size; d.tp.rank = comm->rank; d.tp.seq = (uint32_t *)comm->ll_state; d.tp.in = reduce_in != 0; d.tp.out = reduce_out != 0;
        if (ucast) {
            for (uint32_t r = 0; r < comm->world_size; ++r) {
                if (!comm->ll_peers[r] || ((uintptr_t)comm->ll_peers[r] & 15)) return fail(B200Q_E_ARG, "b200q_mul_mat_vec_tp: bad peer mapping");
                d.tp.ll_peer[r] = (float2 *)comm->ll_peers[r];
            }
        }
    }
    return check_launch(b200q_launch_mmvq(d, (cudaStream_t)stream), "b200q_mul_mat_vec_tp");
}

int b200q_reduce_sum_nvls(const float * in, float * out, int64_t n, void * mc_base, void * local_base, int64_t parity_stride,
                          void * mc_flag, const void * local_flag, uint32_t world_size, void * seq_counter, void * cta_counter, void * stream) {
    if (!in || !out || !mc_base || !local_base || !mc_flag || !local_flag || !seq_counter || !cta_counter || world_size < 2) return fail(B200Q_E_ARG, "b200q_reduce_sum_nvls: bad argument");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_reduce_sum_nvls")) return rc;
    return check_launch(b200q_launch_allreduce_nvls(in, out, n, mc_base, local_base, parity_stride, mc_flag, local_flag, world_size, seq_counter, cta_counter,
                                                    sms, (cudaStream_t)stream), "b200q_reduce_sum_nvls");
}

int b200q_reduce_sum_nvls_bf16(const float * in, float * out_f32, void * out_bf16, int64_t n, const b200q_nvls_stage * sg, void * stream) {
    if (!in || (!out_f32 && !out_bf16) || !sg || !sg->mc_stage || !sg->local_stage || !sg->mc_flag || !sg->local_flag || !sg->state || sg->world_size < 2 || sg->rank >= sg->world_size)
        return fail(B200Q_E_ARG, "b200q_reduce_sum_nvls_bf16: bad argument");
    if (n > sg->stage_elems || (n & 7)) return fail(B200Q_E_SHAPE, "b200q_reduce_sum_nvls_bf16: n must be a multiple of 8 and fit the staging buffer");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_reduce_sum_nvls_bf16")) return rc;
    return check_launch(b200q_launch_allreduce_nvls_2shot(in, out_f32, out_bf16, n, sg->mc_stage, sg->local_stage, sg->mc_flag, sg->local_flag, sg->world_size, sg->rank,
                                                          sg->state, sms, (cudaStream_t)stream), "b200q_reduce_sum_nvls_bf16");
}

size_t b200q_mul_mat_workspace(int type, int64_t m, int64_t k, int64_t n) { return n <= 8 ? 0 : b200q_gemm_workspace_bytes(type, m, k, n); }

int b200q_dequantize_bf16(int type, const void * W, void * out, int64_t m, int64_t k, void * stream) {
    b200q_layout L; int rc = b200q_make_layout(type, m, k, &L);
    if (rc) return check_launch(rc, "b200q_dequantize_bf16");
    return check_launch(b200q_launch_dequant_bf16(W, L, out, (cudaStream_t)stream), "b200q_dequantize_bf16");
}
int b200q_mul_mat_gemm(int type, const void * W, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                       void * workspace, size_t workspace_bytes, void * stream) {
    if (!W || !x || !dst || !workspace || m <= 0 || n < 1) return fail(B200Q_E_ARG, "b200q_mul_mat_gemm: bad argument");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_mul_mat_gemm")) return rc;
    return check_launch(b200q_launch_gemm(type, W, x, k, dst, m, k, n, workspace, workspace_bytes, sms, opt_fused(), (cudaStream_t)stream), "b200q_mul_mat_gemm");
}
int b200q_convert_f32_bf16(const float * x, int64_t x_stride, void * out_bf16, int64_t k, int64_t n, void * stream) {
    if (!x || !out_bf16 || n < 1) return fail(B200Q_E_ARG, "b200q_convert_f32_bf16: bad argument");
    return check_launch(b200q_launch_f32_to_bf16(x, x_stride, out_bf16, k, n, (cudaStream_t)stream), "b200q_convert_f32_bf16");
}
int b200q_mul_mat_gemm_bf16(int type, const void * W, const void * x_bf16, float * dst, int64_t m, int64_t k, int64_t n,
                            void * workspace, size_t workspace_bytes, void * stream) {
    if (!W || !x_bf16 || !dst || m <= 0 || n < 1) return fail(B200Q_E_ARG, "b200q_mul_mat_gemm_bf16: bad argument");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_mul_mat_gemm_bf16")) return rc;
    return check_launch(b200q_launch_gemm_bf16x(type, W, x_bf16, dst, m, k, n, workspace, workspace_bytes, sms, opt_fused(), (cudaStream_t)stream), "b200q_mul_mat_gemm_bf16");
}
int b200q_mul_mat_gemm_multi_bf16(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m, int64_t k,
                                  const void * x_bf16, int64_t n, void * workspace, size_t workspace_bytes, void * stream) {
    if (n_tensors < 1 || n_tensors > 3 || !W || !dst || !m || !x_bf16 || n < 1) return fail(B200Q_E_ARG, "b200q_mul_mat_gemm_multi_bf16: bad argument");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_mul_mat_gemm_multi_bf16")) return rc;
    b200q_gemm_multi d; memset(&d, 0, sizeof d);
    d.type = type; d.n_seg = n_tensors; d.K = k; d.N = n; d.xb = x_bf16;
    for (int i = 0; i < n_tensors; ++i) { if (!W[i] || !dst[i] || m[i] <= 0) return fail(B200Q_E_ARG, "b200q_mul_mat_gemm_multi_bf16: bad tensor %d", i); d.W[i] = W[i]; d.dst[i] = dst[i]; d.M[i] = m[i]; }
    return check_launch(b200q_launch_gemm_multi_bf16x(d, workspace, workspace_bytes, sms, opt_fused(), (cudaStream_t)stream), "b200q_mul_mat_gemm_multi_bf16");
}
// the largest tensor's rows: its bf16 weight scratch serves every tensor
static int64_t max_rows(int n, const int64_t * m) { int64_t r = 0; for (int i = 0; m && i < n; ++i) r = m[i] > r ? m[i] : r; return r; }
size_t b200q_mul_mat_multi_workspace(int type, int n_tensors, const int64_t * m, int64_t k, int64_t n) {
    return n <= 8 || !m ? 0 : b200q_gemm_workspace_bytes(type, max_rows(n_tensors, m), k, n);
}
int b200q_mul_mat_multi(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m, int64_t k,
                        const float * x, int64_t n, void * workspace, size_t workspace_bytes, void * stream) {
    if (n <= 8) return b200q_mul_mat_vec_multi(type, n_tensors, W, dst, m, k, x, (int)n, k, stream);
    if (!x || !workspace) return fail(B200Q_E_ARG, "b200q_mul_mat_multi: bad argument");
    if (workspace_bytes < b200q_mul_mat_multi_workspace(type, n_tensors, m, k, n)) return fail(B200Q_E_NOMEM, "b200q_mul_mat_multi: workspace too small");
    const b200q_dense_ws L = b200q_dense_layout(B200Q_DENSE_GEMM, max_rows(n_tensors, m), k, n);
    char * ws = (char *)workspace;
    if (const int rc = b200q_convert_f32_bf16(x, k, ws + L.x, k, n, stream)) return rc;
    return b200q_mul_mat_gemm_multi_bf16(type, n_tensors, W, dst, m, k, ws + L.x, n, ws + L.wsc, workspace_bytes - L.wsc, stream);
}

size_t b200q_fused_up_gate_workspace(int type, int64_t m, int64_t k, int64_t n) {
    (void)type;
    return n <= 8 ? 0 : b200q_dense_layout(B200Q_DENSE_UP_GATE, m, k, n).total;
}
int b200q_fused_up_gate_gemm_bf16(int type, const void * W_up, const void * W_gate, const void * x_bf16, float * dst, void * dst_bf16,
                                  int64_t m, int64_t k, int64_t n, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream) {
    if (!W_up || !W_gate || !x_bf16 || !dst || !workspace || m <= 0 || n < 1) return fail(B200Q_E_ARG, "b200q_fused_up_gate_gemm_bf16: bad argument");
    int sms = 0; if (const int rc = device_sms(sms, "b200q_fused_up_gate_gemm_bf16")) return rc;
    // the up result must fit; the launch checks the weight scratch, which only the types without a fused kernel use
    const b200q_dense_ws L = b200q_dense_layout(B200Q_DENSE_UP_GATE_BF16, m, k, n);
    if (workspace_bytes < L.wsc) return fail(B200Q_E_NOMEM, "b200q_fused_up_gate_gemm_bf16: workspace too small");
    float * up_res = (float *)((char *)workspace + L.up); cudaStream_t st = (cudaStream_t)stream;
    // up and gate as the two segments of ONE launch (up -> workspace, gate -> dst), then the unary-mul tail in place, which also writes dst_bf16
    b200q_gemm_multi d; memset(&d, 0, sizeof d);
    d.type = type; d.n_seg = 2; d.W[0] = W_up; d.dst[0] = up_res; d.M[0] = m; d.W[1] = W_gate; d.dst[1] = dst; d.M[1] = m; d.K = k; d.N = n; d.xb = x_bf16;
    const int rc = check_launch(b200q_launch_gemm_multi_bf16x(d, (char *)workspace + L.wsc, workspace_bytes - L.wsc, sms, opt_fused(), st), "b200q_fused_up_gate_gemm_bf16(up,gate)");
    if (rc) return rc;
    return check_launch(b200q_launch_mul_unary(dst, up_res, dst, dst_bf16, m * n, unary, limit, st), "b200q_fused_up_gate_gemm_bf16(unary)");
}
int b200q_fused_up_gate(int type, const void * W_up, const void * W_gate, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                        int unary, float limit, void * workspace, size_t workspace_bytes, void * stream) {
    if (n <= 8) return b200q_fused_up_gate_vec(type, W_up, W_gate, x, dst, m, k, (int)n, k, unary, limit, stream);
    if (!x || !workspace) return fail(B200Q_E_ARG, "b200q_fused_up_gate: bad argument");
    if (workspace_bytes < b200q_fused_up_gate_workspace(type, m, k, n)) return fail(B200Q_E_NOMEM, "b200q_fused_up_gate: workspace too small");
    if ((m * n) % 4) return fail(B200Q_E_SHAPE, "b200q_fused_up_gate: m*n must be a multiple of 4");
    char * ws = (char *)workspace;
    // ternary weights: both GEMMs on the int8 tensor pipe (one activation quantisation, one launch over the up and gate row tiles), then the unary-mul tail
    const b200q_dense_ws Li = b200q_dense_layout(B200Q_DENSE_UP_GATE_I8, m, k, n);
    if (opt_fused() && device_info().ok && b200q_gemm_bn_i8_ok(type, k, n, x, k, workspace_bytes - Li.x)) {
        float * up_res = (float *)(ws + Li.up);
        b200q_gemm_multi d; memset(&d, 0, sizeof d);
        d.type = type; d.n_seg = 2; d.W[0] = W_up; d.dst[0] = up_res; d.M[0] = m; d.W[1] = W_gate; d.dst[1] = dst; d.M[1] = m; d.K = k; d.N = n;
        const int rc = check_launch(b200q_launch_gemm_bn_i8(d, x, k, ws + Li.x, workspace_bytes - Li.x, (cudaStream_t)stream), "b200q_fused_up_gate(int8)");
        if (rc) return rc;
        return check_launch(b200q_launch_mul_unary(dst, up_res, dst, nullptr, m * n, unary, limit, (cudaStream_t)stream), "b200q_fused_up_gate(unary)");
    }
    // X, then the workspace of b200q_fused_up_gate_gemm_bf16 (B200Q_DENSE_UP_GATE_BF16)
    const b200q_dense_ws L = b200q_dense_layout(B200Q_DENSE_UP_GATE, m, k, n);
    if (const int rc = b200q_convert_f32_bf16(x, k, ws + L.x, k, n, stream)) return rc;
    return b200q_fused_up_gate_gemm_bf16(type, W_up, W_gate, ws + L.x, dst, nullptr, m, k, n, unary, limit, ws + L.up, workspace_bytes - L.up, stream);
}
int b200q_mul_mat(int type, const void * W, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                  void * workspace, size_t workspace_bytes, void * stream) {
    if (n <= 8) return b200q_mul_mat_vec(type, W, x, dst, m, k, (int)n, k, nullptr, stream);
    return b200q_mul_mat_gemm(type, W, x, dst, m, k, n, workspace, workspace_bytes, stream);
}
/* GGML_OP_ADD of a mat-mul result with its bias (bias [m] broadcast over the n columns, nb = 1) or with a same-shape tensor (nb = n): the node as
 * its own launch, for graphs that compute it separately; inside a graph the mat-vec fuses it (bias operand of b200q_mul_mat_vec). */
int b200q_add_rows(const float * a, const float * b, float * dst, int64_t m, int64_t n, int64_t nb, void * stream) {
    if (!a || !b || !dst) return fail(B200Q_E_ARG, "b200q_add_rows: bad argument");
    return check_launch(b200q_launch_add_rows(a, b, dst, m, n, nb, (cudaStream_t)stream), "b200q_add_rows");
}
/* The MoE entry points share one body per path.  An operand is a (tensor, row origin) pair inside expert matrices of rows_layout rows
 * (b200q_mmvq_id_desc): the split up/gate form passes origin 0 and rows_layout = m, merged [gate; up] experts pass one tensor twice with
 * rows_layout = 2 m, up at row m and gate at row 0. */
struct moe_operands { const void * W; const void * W_gate; int64_t rows_layout, W_row0, gate_row0; };
static void moe_desc(b200q_mmvq_id_desc & d, int type, const moe_operands & o, int n_expert, int64_t m, int64_t k, int n_used, int nb1, int unary, float limit) {
    memset(&d, 0, sizeof d);
    d.type = type; d.W = o.W; d.W2 = o.W_gate; d.rows_layout = o.rows_layout; d.W_row0 = o.W_row0; d.W2_row0 = o.gate_row0;
    d.M = m; d.K = k; d.n_expert = n_expert; d.n_used = n_used; d.nb1 = nb1; d.act = unary; d.limit = limit;
    d.x_tok_stride = (int64_t)nb1 * k; d.x_col_stride = k;      // MoE activations are contiguous; b200q_mul_mat_batched overrides both
}
// the argument checks of both bodies, in this order: operands (and the grouped path's workspace), device, the mat-vec's activation alignment
// (the grouped GEMM's launch checks its own), token / slot counts
static int moe_check(bool grouped, const moe_operands & o, const int32_t * ids, const float * x, const float * dst, const void * workspace,
                     int64_t m, int64_t k, int n_expert, int n_used, int nb1, int n_tokens, int & sms, const char * what) {
    if (!o.W || !ids || !x || !dst || (grouped && !workspace) || m <= 0 || n_expert < 1) return fail(B200Q_E_ARG, "%s: bad argument", what);
    if (const int rc = device_sms(sms, what)) return rc;
    if (!grouped && (((uintptr_t)x & 15) || (k & 3))) return fail(B200Q_E_ARG, "%s: activations must be 16-byte aligned", what);
    if (n_tokens < 1 || n_used < 1 || nb1 < 1 || n_used % nb1) return fail(B200Q_E_ARG, "%s: bad token / slot counts", what);
    return B200Q_OK;
}
static int moe_vec(int type, const moe_operands & o, int n_expert, const int32_t * ids, const float * x, float * dst,
                   int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * stream, const char * what,
                   int64_t xs_tok = 0, int64_t xs_col = 0) {
    int sms = 0; if (const int rc = moe_check(false, o, ids, x, dst, nullptr, m, k, n_expert, n_used, nb1, n_tokens, sms, what)) return rc;
    // the quantised activation columns of a launch live in shared memory: larger batches are walked in token chunks (same kernel, the expert ids
    // never leave the device).  Prefill batches are served by the grouped GEMM (b200q_mul_mat_id_gemm) once b200q_mul_mat_id selects it.
    int chunk = (int)(b200q_mmvq_max_cols(k) / nb1);
    static const int forced = [] { const char * e = getenv("B200Q_MOE_CHUNK_TOKENS"); return e ? atoi(e) : 0; }();
    if (forced > 0 && forced < chunk) chunk = forced;
    if (chunk < 1) return fail(B200Q_E_SHAPE, "%s: one token's activation columns do not fit shared memory", what);
    for (int t0 = 0; t0 < n_tokens; t0 += chunk) {
        const int nt = n_tokens - t0 < chunk ? n_tokens - t0 : chunk;
        b200q_mmvq_id_desc d; moe_desc(d, type, o, n_expert, m, k, n_used, nb1, unary, limit);
        if (xs_tok) { d.x_tok_stride = xs_tok; d.x_col_stride = xs_col; }
        d.ids = ids + (int64_t)t0 * n_used; d.x = x + (int64_t)t0 * d.x_tok_stride; d.dst = dst + (int64_t)t0 * n_used * m; d.n_tokens = nt;
        d.sm_count = sms; d.pdl = opt_pdl();
        const int rc = check_launch(b200q_launch_mmvq_id(d, (cudaStream_t)stream), what);
        if (rc) return rc;
    }
    return B200Q_OK;
}
int b200q_mul_mat_id_vec(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                         int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * stream) {
    return moe_vec(type, {W, W_gate, m, 0, 0}, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, stream, "b200q_mul_mat_id_vec");
}

/* MoE prefill: grouped wgmma GEMM over expert-sorted slots (b200q_moe.cu), versus the mat-vec kernel, which needs no routing or gather pass.
 * Crossovers measured with scripts/bench_moe.py on an H100 80GB HBM3 at 700 W, 1-256 tokens (Qwen3-30B-A3B Q4_K / IQ4_K, Mixtral-8x7B IQ4_NL,
 * DeepSeek-V3 TP-8 shard IQ2_XXS; DESIGN.md §4):
 *  - MOE_FUSED_UP_GATE follows the average rows per expert, n_slots / n_expert: at 4 rows Mixtral is still 0.82x while the others are 1.3-1.45x,
 *    at 6 rows every shape is 1.4-2.2x faster on the grouped path.  Grouped when n_slots > 5 * n_expert.
 *  - MUL_MAT_ID follows the number of slots, whatever the expert count: 24 slots 0.84x (Mixtral), 32 slots 0.94-1.08x, 64 slots 1.18-2.3x on
 *    every shape.  Grouped when n_slots > 32.
 * Merged up/gate experts run the same launches on the same bytes as the split form, so they share its crossover. */
static constexpr int64_t MOE_UP_GATE_MIN_ROWS_PER_EXPERT = 5;
static constexpr int64_t MOE_MUL_MAT_ID_MIN_SLOTS = 32;
// the crossover above: whether b200q_mul_mat_id takes the grouped GEMM for a shape the GEMM accepts
static bool moe_grouped_pays(int n_used, int n_tokens, int n_expert, int up_gate) {
    const int64_t n_slots = (int64_t)n_tokens * n_used;
    return n_slots > (up_gate ? MOE_UP_GATE_MIN_ROWS_PER_EXPERT * n_expert : MOE_MUL_MAT_ID_MIN_SLOTS);
}
// the grouped path's workspace, 0 for a shape it refuses
static size_t moe_gemm_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert, int up_gate, int64_t rows_layout) {
    if (!b200q_moe_gemm_shape_ok(type, m, k, n_used, nb1, n_tokens, n_expert, up_gate)) return 0;
    return b200q_moe_gemm_workspace_bytes(type, m, k, (int64_t)n_tokens * n_used, n_expert, up_gate, rows_layout);
}
size_t b200q_mul_mat_id_gemm_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert, int up_gate) {
    return moe_gemm_workspace(type, m, k, n_used, nb1, n_tokens, n_expert, up_gate, m);
}
size_t b200q_mul_mat_id_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert, int up_gate) {
    return moe_grouped_pays(n_used, n_tokens, n_expert, up_gate) ? b200q_mul_mat_id_gemm_workspace(type, m, k, n_used, nb1, n_tokens, n_expert, up_gate) : 0;
}
static int moe_gemm(int type, const moe_operands & o, int n_expert, const int32_t * ids, const float * x, float * dst, int64_t m, int64_t k,
                    int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream, const char * what,
                    int64_t xs_tok = 0, int64_t xs_col = 0) {
    int sms = 0; if (const int rc = moe_check(true, o, ids, x, dst, workspace, m, k, n_expert, n_used, nb1, n_tokens, sms, what)) return rc;
    if (!b200q_moe_gemm_shape_ok(type, m, k, n_used, nb1, n_tokens, n_expert, o.W_gate != nullptr))
        return fail(B200Q_E_SHAPE, "%s: shape not supported by the grouped GEMM (K %% 256, n_expert <= 1024, type)", what);
    b200q_mmvq_id_desc d; moe_desc(d, type, o, n_expert, m, k, n_used, nb1, unary, limit);
    if (xs_tok) { d.x_tok_stride = xs_tok; d.x_col_stride = xs_col; }
    d.ids = ids; d.x = x; d.dst = dst; d.n_tokens = n_tokens; d.sm_count = sms;
    return check_launch(b200q_launch_moe_gemm(d, workspace, workspace_bytes, (cudaStream_t)stream), what);
}
int b200q_mul_mat_id_gemm(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                          int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream) {
    return moe_gemm(type, {W, W_gate, m, 0, 0}, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, workspace, workspace_bytes, stream,
                    "b200q_mul_mat_id_gemm");
}
int b200q_mul_mat_id(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                     int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream) {
    if (b200q_mul_mat_id_workspace(type, m, k, n_used, nb1, n_tokens, n_expert, W_gate != nullptr) == 0)
        return b200q_mul_mat_id_vec(type, W, W_gate, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, stream);
    return b200q_mul_mat_id_gemm(type, W, W_gate, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, workspace, workspace_bytes, stream);
}

/* MOE_FUSED_UP_GATE over merged experts: W_gate_up holds n_expert matrices [2 m x k], gate rows [0, m) then up rows [m, 2 m) */
size_t b200q_moe_up_gate_merged_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert) {
    if (m < 1 || m > INT32_MAX / 4 || !moe_grouped_pays(n_used, n_tokens, n_expert, 1)) return 0;
    return moe_gemm_workspace(type, m, k, n_used, nb1, n_tokens, n_expert, 1, 2 * m);
}
int b200q_moe_up_gate_merged(int type, const void * W_gate_up, int n_expert, const int32_t * ids, const float * x, float * dst,
                             int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream) {
    static const char * what = "b200q_moe_up_gate_merged";
    if (!W_gate_up || m < 1 || m > INT32_MAX / 4) return fail(B200Q_E_ARG, "%s: bad argument", what);
    b200q_layout L;
    if (const int rc = b200q_make_layout(type, 2 * m, k, &L)) return rc == -1 ? fail(B200Q_E_TYPE, "%s: unsupported ggml type", what)
                                                                             : fail(B200Q_E_SHAPE, "%s: k = %lld is not a multiple of the type's block", what, (long long)k);
    if (L.wire > 1 && m % L.wire)
        return fail(B200Q_E_SHAPE, "%s: m = %lld must be a multiple of %d for this type (its rows are interleaved in groups of %d)", what, (long long)m, L.wire, L.wire);
    const moe_operands o{W_gate_up, W_gate_up, 2 * m, m, 0};
    if (b200q_moe_up_gate_merged_workspace(type, m, k, n_used, nb1, n_tokens, n_expert) == 0)
        return moe_vec(type, o, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, stream, what);
    return moe_gemm(type, o, n_expert, ids, x, dst, m, k, n_used, nb1, n_tokens, unary, limit, workspace, workspace_bytes, stream, what);
}
int b200q_moe_combine(const float * rows, const float * weights, float * dst, int64_t m, int n_used, int n_tokens, void * stream) {
    static const char * what = "b200q_moe_combine";
    if (!rows || !weights || !dst || ((uintptr_t)rows & 3) || ((uintptr_t)weights & 3) || ((uintptr_t)dst & 3)) return fail(B200Q_E_ARG, "%s: bad argument", what);
    if (m < 1 || n_used < 1 || n_tokens < 1 || m > INT64_MAX / ((int64_t)n_used * n_tokens * 4)) return fail(B200Q_E_SHAPE, "%s: bad shape", what);
    const uintptr_t d0 = (uintptr_t)dst, d1 = d0 + (uintptr_t)(m * n_tokens * 4);
    const uintptr_t r0 = (uintptr_t)rows, r1 = r0 + (uintptr_t)(m * n_used * n_tokens * 4), w0 = (uintptr_t)weights, w1 = w0 + (uintptr_t)n_used * n_tokens * 4;
    if ((d0 < r1 && r0 < d1) || (d0 < w1 && w0 < d1)) return fail(B200Q_E_ARG, "%s: dst overlaps an input", what);
    return check_launch(b200q_launch_moe_combine(rows, weights, dst, m, n_used, n_tokens, (cudaStream_t)stream), what);
}
/* Batched MUL_MAT as MUL_MAT_ID with identity routing: token := batch entry, slot := column, n_used = nb1 = n, ids[b][j] = b (per entry,
 * n_expert = n_batch) or 0 (broadcast, n_expert = 1), written into the workspace by k_batch_ids.  With identity routing every entry gets exactly n
 * rows, so the MoE crossover (routed slots) does not apply.  Cut points from scripts/bench_batched.py on DeepSeek-V3's MLA products, 128 and 16
 * heads, Q8_0 and IQ4_NL, n = 1 ... 512, on an H100 80GB HBM3 at 700 W (DESIGN.md §4):
 *  - the grouped GEMM, where it is eligible (K % 256), from 128 slots (n_batch * n) on: wv_b at 16 heads is 1.3x slower than the mat-vec at 64
 *    slots and 1.3x faster at 128; a type without a fused GEMM kernel (Q8_0) dequantises every entry's matrix first, so with one column per entry
 *    (128 heads, n = 1: 33 us against 26 us) the mat-vec stays faster;
 *  - otherwise the identity-routed mat-vec up to 16 columns per entry (wk_b at 128 heads: 580 us against 904 us for one GEMM per head at n = 16,
 *    1184 us against 957 us at n = 32), one dense GEMM per entry above.  It beats one dense mat-vec per entry at every n <= 8 (wk_b at 128 heads:
 *    41 us against 428 us at n = 1, 291 us against 371 us at n = 8). */
enum batched_path { BATCHED_ONE = 0, BATCHED_VEC, BATCHED_ENTRY_VEC, BATCHED_GROUPED, BATCHED_DENSE };
static constexpr int64_t BATCHED_GROUPED_MIN_SLOTS = 128;
static constexpr int64_t BATCHED_VEC_MAX_N = 16;
struct batched_plan { int path; int64_t n_cols, x_stride; int n_expert; size_t ids_bytes, ws_bytes; };
// argument / shape checks of the batched entry and its plan; returns a B200Q_E_* code (the failure text is set) or 0
static int plan_batched(int type, int64_t m, int64_t k, int64_t n, int n_batch, int per_entry, int64_t cs, int64_t bs, batched_plan & p, const char * what) {
    p = batched_plan{};
    if (m < 1 || k < 1 || n < 1 || n_batch < 1 || (per_entry != 0 && per_entry != 1)) return fail(B200Q_E_ARG, "%s: bad argument", what);
    if (cs < 0 || bs < 0 || (cs & 3) || (bs & 3) || (n > 1 && cs < k) || (n_batch > 1 && bs < k))
        return fail(B200Q_E_ARG, "%s: strides must be multiples of 4 floats, at least k where they are used", what);
    if (n > INT32_MAX || n * n_batch > INT32_MAX) return fail(B200Q_E_SHAPE, "%s: too many columns", what);
    b200q_layout L; if (const int rc = b200q_make_layout(type, m, k, &L)) return check_launch(rc, what);
    const int64_t max_cols = b200q_mmvq_max_cols(k);
    // one matrix over columns a constant stride apart (broadcast with x_batch_stride == n * x_col_stride, or one entry): a plain 2-D product, as long
    // as it stays on the side of the mat-vec / GEMM cut (n <= 8) each entry would take on its own
    const bool uniform = (!per_entry || n_batch == 1) && (n == 1 || n_batch == 1 || bs == n * cs);
    if (uniform && (n * n_batch <= 8 || n > 8)) {
        p.path = BATCHED_ONE; p.n_cols = n * n_batch; p.x_stride = n == 1 ? (n_batch > 1 ? bs : k) : cs;
        if (p.n_cols <= 8) { if (max_cols < 1) return fail(B200Q_E_SHAPE, "%s: K=%lld too large for the mat-vec kernel", what, (long long)k); }
        else p.ws_bytes = b200q_gemm_workspace_bytes(type, m, k, p.n_cols);
        return 0;
    }
    // a broadcast matrix with up to 8 columns per entry: the dense mat-vec of each entry (it reads the matrix once per entry for all its columns)
    if (!per_entry && n <= 8) {
        if (max_cols < n) return fail(B200Q_E_SHAPE, "%s: K=%lld too large for the mat-vec kernel", what, (long long)k);
        p.path = BATCHED_ENTRY_VEC;
        return 0;
    }
    p.n_expert = per_entry ? n_batch : 1;
    p.ids_bytes = (size_t)b200q_align_up(n * n_batch * 4, 256);
    const bool grouped = b200q_moe_gemm_shape_ok(type, m, k, (int)n, (int)n, n_batch, p.n_expert, 0) && n * n_batch >= BATCHED_GROUPED_MIN_SLOTS &&
                         (n > 1 || b200q_gemm_fused_type(type));
    if (grouped) {
        p.path = BATCHED_GROUPED; p.ws_bytes = p.ids_bytes + b200q_moe_gemm_workspace_bytes(type, m, k, n * n_batch, p.n_expert, 0, m);
    } else if (n <= BATCHED_VEC_MAX_N && max_cols >= n) {
        p.path = BATCHED_VEC; p.ws_bytes = p.ids_bytes;
    } else if (n <= 8) {
        return fail(B200Q_E_SHAPE, "%s: K=%lld too large for the mat-vec kernel", what, (long long)k);
    } else {
        p.path = BATCHED_DENSE; p.ids_bytes = 0; p.ws_bytes = b200q_gemm_workspace_bytes(type, m, k, n);
    }
    return 0;
}
size_t b200q_mul_mat_batched_workspace(int type, int64_t m, int64_t k, int64_t n, int n_batch, int per_entry, int64_t x_col_stride, int64_t x_batch_stride) {
    batched_plan p;
    return plan_batched(type, m, k, n, n_batch, per_entry, x_col_stride, x_batch_stride, p, "b200q_mul_mat_batched_workspace") ? 0 : p.ws_bytes;
}
int b200q_mul_mat_batched(int type, const void * W, int per_entry, const float * x, int64_t x_col_stride, int64_t x_batch_stride,
                          float * dst, int64_t m, int64_t k, int64_t n, int n_batch, void * workspace, size_t workspace_bytes, void * stream) {
    static const char * what = "b200q_mul_mat_batched";
    if (!W || !x || !dst || ((uintptr_t)x & 15) || ((uintptr_t)workspace & 255)) return fail(B200Q_E_ARG, "%s: bad argument (x 16-byte, workspace 256-byte aligned)", what);
    batched_plan p;
    if (const int rc = plan_batched(type, m, k, n, n_batch, per_entry, x_col_stride, x_batch_stride, p, what)) return rc;
    if (workspace_bytes < p.ws_bytes || (p.ws_bytes && !workspace)) return fail(B200Q_E_NOMEM, "%s: workspace too small", what);
    int sms = 0; if (const int rc = device_sms(sms, what)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (p.path == BATCHED_ONE) {
        if (p.n_cols <= 8) {
            b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x, what)) return rc;
            d.n_seg = 1; d.seg[0] = {W, nullptr, dst, nullptr, m};
            return mmvq_cols(d, (int)p.n_cols, p.x_stride, st, what);
        }
        return check_launch(b200q_launch_gemm(type, W, x, p.x_stride, dst, m, k, p.n_cols, workspace, workspace_bytes, sms, opt_fused(), st), what);
    }
    if (p.path == BATCHED_ENTRY_VEC) {  // the broadcast matrix, one dense mat-vec per entry over its strided columns
        for (int b = 0; b < n_batch; ++b) {
            b200q_mmvq_desc d; if (const int rc = mmvq_desc(d, type, k, x + b * x_batch_stride, what)) return rc;
            d.n_seg = 1; d.seg[0] = {W, nullptr, dst + (int64_t)b * n * m, nullptr, m};
            if (const int rc = mmvq_cols(d, (int)n, x_col_stride, st, what)) return rc;
        }
        return B200Q_OK;
    }
    if (p.path == BATCHED_DENSE) {      // one GEMM per entry over its strided columns, on one workspace (stream-ordered reuse)
        const int64_t wstride = per_entry ? b200q_plane_bytes(type, m, k) : 0;
        for (int b = 0; b < n_batch; ++b) {
            const int rc = check_launch(b200q_launch_gemm(type, (const char *)W + b * wstride, x + b * x_batch_stride, x_col_stride, dst + (int64_t)b * n * m, m, k, n,
                                                          workspace, workspace_bytes, sms, opt_fused(), st), what);
            if (rc) return rc;
        }
        return B200Q_OK;
    }
    int32_t * ids = (int32_t *)workspace;
    if (const int rc = check_launch(b200q_launch_batch_ids(ids, n_batch, (int)n, per_entry, st), what)) return rc;
    const moe_operands o{W, nullptr, m, 0, 0};
    if (p.path == BATCHED_VEC) return moe_vec(type, o, p.n_expert, ids, x, dst, m, k, (int)n, (int)n, n_batch, 0, 0.0f, stream, what, x_batch_stride, x_col_stride);
    return moe_gemm(type, o, p.n_expert, ids, x, dst, m, k, (int)n, (int)n, n_batch, 0, 0.0f, (char *)workspace + p.ids_bytes, workspace_bytes - p.ids_bytes, stream, what,
                    x_batch_stride, x_col_stride);
}

int b200q_mul_mat_host(int type, const void * W, const float * x_host, float * dst_host, int64_t m, int64_t k, int64_t n, void * stream) {
    cudaStream_t st = (cudaStream_t)stream; cudaError_t e; int rc;
    const size_t xb = (size_t)n * k * sizeof(float), yb = (size_t)n * m * sizeof(float), wsb = b200q_mul_mat_workspace(type, m, k, n);
    if ((rc = ensure(g_x, xb)) || (rc = ensure(g_y, yb)) || (wsb && (rc = ensure(g_ws, wsb)))) return rc;
    if ((e = cudaMemcpyAsync(g_x.p, x_host, xb, cudaMemcpyHostToDevice, st)) != cudaSuccess) return cuda_fail("mul_mat_host H2D", e);
    if ((rc = b200q_mul_mat(type, W, (const float *)g_x.p, (float *)g_y.p, m, k, n, g_ws.p, g_ws.n, stream))) return rc;
    if ((e = cudaMemcpyAsync(dst_host, g_y.p, yb, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return cuda_fail("mul_mat_host D2H", e);
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return cuda_fail("mul_mat_host sync", e);
    return B200Q_OK;
}

}  // extern "C"
