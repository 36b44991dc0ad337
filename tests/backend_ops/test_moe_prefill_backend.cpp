// tests/backend_ops/test_moe_prefill_backend.cpp — MoE prefill through the reference's ggml-backend API: GGML_OP_MUL_MAT_ID and
// GGML_OP_MOE_FUSED_UP_GATE at prefill batch sizes (256-512 tokens, 16-32 experts), where the backend's dispatcher takes the grouped wgmma GEMM over
// expert-sorted slots.  Same semantics as test_mul_mat_backend.cpp / the reference's test-backend-ops test_mul_mat_id: the graph is run on the backend
// under test and on the reference CPU backend through ggml_backend_compare_graph_backend, and the results must agree to NMSE <= 5e-4.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <random>
#include <vector>

static double nmse(const float * a, const float * b, size_t n) {
    double e = 0, s = 0; for (size_t i = 0; i < n; ++i) { e += ((double)a[i] - b[i]) * ((double)a[i] - b[i]); s += (double)b[i] * b[i]; } return e / (s > 0 ? s : 1e-300);
}
struct cb_data { double worst = 0; int n = 0; };
static bool cmp_cb(int, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cb_data * d = (cb_data *)ud;
    std::vector<float> a(ggml_nelements(t1)), b(ggml_nelements(t2));
    ggml_backend_tensor_get(t1, a.data(), 0, ggml_nbytes(t1)); ggml_backend_tensor_get(t2, b.data(), 0, ggml_nbytes(t2));
    const double e = nmse(a.data(), b.data(), a.size()); if (e > d->worst) d->worst = e; d->n++;
    return true;
}

static int run_case(ggml_backend_t be, ggml_backend_t cpu, ggml_type type, int64_t n_expert, int64_t n_used, int64_t n_tokens, bool shared_col, bool up_gate, unsigned seed) {
    const int64_t m = 256, k = 1024;
    ggml_init_params ip = { ggml_tensor_overhead() * 16 + ggml_graph_overhead(), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
    ggml_tensor * w = ggml_new_tensor_3d(ctx, type, k, m, n_expert), * g = up_gate ? ggml_new_tensor_3d(ctx, type, k, m, n_expert) : nullptr;
    ggml_tensor * x = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, k, shared_col ? 1 : n_used, n_tokens);
    ggml_tensor * ids = ggml_new_tensor_2d(ctx, GGML_TYPE_I32, n_used, n_tokens);
    ggml_tensor * y = up_gate ? ggml_moe_up_gate(ctx, w, g, x, ids, GGML_UNARY_OP_SILU) : ggml_mul_mat_id(ctx, w, x, ids);
    ggml_cgraph * gf = ggml_new_graph(ctx); ggml_build_forward_expand(gf, y);
    ggml_backend_buffer_t buf = ggml_backend_alloc_ctx_tensors(ctx, be);
    if (!buf) { printf("  alloc failed\n"); return 1; }
    std::mt19937 rng(seed);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> ones(k, 1.0f);
    for (ggml_tensor * t : {w, g}) {
        if (!t) continue;
        std::vector<float> wf(ggml_nelements(t)); for (auto & v : wf) v = u(rng);
        std::vector<uint8_t> wq(ggml_nbytes(t));
        ggml_quantize_chunk(type, wf.data(), wq.data(), 0, ggml_nrows(t), k, ggml_quantize_requires_imatrix(type) ? ones.data() : nullptr, nullptr);
        ggml_backend_tensor_set(t, wq.data(), 0, wq.size());
    }
    std::vector<float> xf(ggml_nelements(x)); for (auto & v : xf) v = u(rng);
    ggml_backend_tensor_set(x, xf.data(), 0, xf.size() * sizeof(float));
    // n_used distinct experts per token (a top-k), skewed: expert 0 is picked by every token, so its rows span several tiles
    std::vector<int32_t> idv(n_used * n_tokens), perm(n_expert);
    for (int64_t t = 0; t < n_tokens; ++t) {
        std::iota(perm.begin(), perm.end(), 0); std::shuffle(perm.begin() + 1, perm.end(), rng);
        for (int64_t j = 0; j < n_used; ++j) idv[t * n_used + j] = perm[j];
        std::swap(idv[t * n_used], idv[t * n_used + rng() % n_used]);
    }
    ggml_backend_tensor_set(ids, idv.data(), 0, idv.size() * sizeof(int32_t));
    if (!ggml_backend_supports_op(be, y)) { printf("  %-8s %s not supported\n", ggml_type_name(type), ggml_op_name(y->op)); return 1; }
    cb_data d; ggml_backend_compare_graph_backend(be, cpu, gf, cmp_cb, &d);
    const bool ok = d.n > 0 && d.worst <= 5e-4;
    printf("  %-8s %-18s experts=%lld used=%lld tokens=%lld %s: NMSE vs CPU backend %.3g -> %s\n", ggml_type_name(type), ggml_op_name(y->op), (long long)n_expert,
           (long long)n_used, (long long)n_tokens, shared_col ? "(shared column)" : "(column per slot)", d.worst, ok ? "OK" : "FAIL");
    ggml_backend_buffer_free(buf); ggml_free(ctx);
    return ok ? 0 : 1;
}

int main() {
    ggml_backend_t be = ggml_backend_cuda_init(0, "pdl=1", nullptr);
    if (!be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    ggml_backend_t cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(cpu, 4);
    int fails = 0; unsigned seed = 5000;
    for (ggml_type t : {GGML_TYPE_IQ4_NL, GGML_TYPE_Q4_K, GGML_TYPE_IQ2_XXS}) {
        fails += run_case(be, cpu, t, 16, 2, 256, true, true, ++seed);       // up + gate experts on the token's column
        fails += run_case(be, cpu, t, 16, 2, 256, false, false, ++seed);     // down experts, one column per slot
        fails += run_case(be, cpu, t, 32, 4, 512, true, true, ++seed);
        fails += run_case(be, cpu, t, 32, 4, 512, false, false, ++seed);
        fails += run_case(be, cpu, t, 32, 4, 384, true, false, ++seed);
    }
    printf("%s: %d failures\n", fails ? "FAILED" : "PASSED", fails);
    ggml_backend_free(be); ggml_backend_free(cpu);
    return fails ? 1 : 0;
}
