// tests/backend_ops/test_moe_merged_backend.cpp — GGML_OP_MOE_FUSED_UP_GATE over merged up/gate experts (ffn_gate_up_exps [K, 2 n_ff, E], src[1] = NULL,
// as llm_build_moe_ffn emits it: ggml_moe_up_gate(ctx, up_gate_exps, nullptr, cur, selected_experts, op), src/llama-build-context.cpp:1584-1594) through
// the reference's ggml-backend API.  The arbiter is the unmodified reference CPU backend (its op reads gate rows [0, n_ff) and up rows [n_ff, 2 n_ff)).
//   test_moe_merged_backend op     the node alone, on the plug and on the CPU backend (ggml_backend_compare_graph_backend), NMSE <= 5e-4
//                                  (tests/test-backend-ops.cpp:979-981), at 1, 8 and 512 tokens for IQ4_NL, Q4_K, IQ2_XXS
//   test_moe_merged_backend graph  the MoE FFN of llm_build_moe_ffn (softmax gating, ggml_top_k, routing weights, merged up/gate, ffn_down_exps) at
//                                  the Qwen3-30B-A3B, Mixtral-8x7B and DeepSeek-V3 shapes of test_plug_graphs.cpp and 1 ... 512 tokens, placed by
//                                  ggml_backend_sched next to the CPU backend with the weights in a plug buffer: the merged node must run on the
//                                  plug, and it and the layer output must match the same graph computed on the CPU backend alone (NMSE <= 5e-4)
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <random>
#include <string>
#include <vector>

static double nmse(const std::vector<float> & a, const std::vector<float> & b) {
    double e = 0, s = 0; for (size_t i = 0; i < a.size(); ++i) { e += ((double)a[i] - b[i]) * ((double)a[i] - b[i]); s += (double)b[i] * b[i]; } return e / (s > 0 ? s : 1e-300);
}
static std::vector<float> get_f32(const ggml_tensor * t) { std::vector<float> v(ggml_nelements(t)); ggml_backend_tensor_get(t, v.data(), 0, ggml_nbytes(t)); return v; }
struct cb_data { double worst = 0; int n = 0; };
static bool cmp_cb(int, ggml_tensor * t1, ggml_tensor * t2, void * ud) {
    cb_data * d = (cb_data *)ud;
    const double e = nmse(get_f32(t1), get_f32(t2)); if (e > d->worst) d->worst = e; d->n++;
    return true;
}
// quantised weights of a trained model's magnitude (|w| < 0.05), rows drawn from a pool of at most 1024 quantised rows (fast for many experts)
static std::vector<uint8_t> quantized_rows(ggml_type type, int64_t k, int64_t rows, std::mt19937 & rng) {
    const int64_t pool = std::min<int64_t>(rows, 1024);
    const size_t rs = ggml_row_size(type, k);
    std::uniform_real_distribution<float> u(-0.05f, 0.05f);
    std::vector<float> f(pool * k), ones(k, 1.0f); for (auto & v : f) v = u(rng);
    std::vector<uint8_t> pq(pool * rs), wq(rows * rs);
    ggml_quantize_chunk(type, f.data(), pq.data(), 0, pool, k, ggml_quantize_requires_imatrix(type) ? ones.data() : nullptr, nullptr);
    for (int64_t r = 0; r < rows; ++r) memcpy(wq.data() + r * rs, pq.data() + (r < pool ? r : rng() % pool) * rs, rs);
    return wq;
}
static ggml_tensor * moe_up_gate_merged(ggml_context * ctx, ggml_tensor * up_gate, ggml_tensor * x, ggml_tensor * ids) {
    ggml_tensor * par = ggml_moe_up_gate(ctx, up_gate, nullptr, x, ids, GGML_UNARY_OP_SILU);
    *((float *)(par->op_params + 1)) = 0.0f;            // the swiglu limit slot llm_build_moe_ffn writes (no limit)
    return par;
}

// ---- the node alone ----
static int run_op_case(ggml_backend_t be, ggml_backend_t cpu, ggml_type type, int64_t n_tokens, unsigned seed) {
    const int64_t n_expert = 16, n_used = 4, n_ff = 256, k = 1024;
    ggml_init_params ip = { ggml_tensor_overhead() * 16 + ggml_graph_overhead(), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
    ggml_tensor * w = ggml_new_tensor_3d(ctx, type, k, 2 * n_ff, n_expert);
    ggml_tensor * x = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, k, 1, n_tokens);
    ggml_tensor * ids = ggml_new_tensor_2d(ctx, GGML_TYPE_I32, n_used, n_tokens);
    ggml_tensor * y = moe_up_gate_merged(ctx, w, x, ids);
    ggml_cgraph * gf = ggml_new_graph(ctx); ggml_build_forward_expand(gf, y);
    ggml_backend_buffer_t buf = ggml_backend_alloc_ctx_tensors(ctx, be);
    if (!buf) { printf("  alloc failed\n"); return 1; }
    std::mt19937 rng(seed);
    std::vector<uint8_t> wq = quantized_rows(type, k, ggml_nrows(w), rng);
    ggml_backend_tensor_set(w, wq.data(), 0, wq.size());
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> xf(ggml_nelements(x)); for (auto & v : xf) v = u(rng);
    ggml_backend_tensor_set(x, xf.data(), 0, xf.size() * sizeof(float));
    std::vector<int32_t> idv(n_used * n_tokens), perm(n_expert);           // a top-k: distinct experts per token
    for (int64_t t = 0; t < n_tokens; ++t) {
        std::iota(perm.begin(), perm.end(), 0); std::shuffle(perm.begin(), perm.end(), rng);
        std::copy(perm.begin(), perm.begin() + n_used, idv.begin() + t * n_used);
    }
    ggml_backend_tensor_set(ids, idv.data(), 0, idv.size() * sizeof(int32_t));
    if (!ggml_backend_supports_op(be, y)) { printf("  %-8s merged MOE_FUSED_UP_GATE not supported\n", ggml_type_name(type)); return 1; }
    cb_data d; ggml_backend_compare_graph_backend(be, cpu, gf, cmp_cb, &d);
    const bool ok = d.n > 0 && d.worst <= 5e-4;
    printf("  %-8s merged MOE_FUSED_UP_GATE experts=%lld used=%lld n_ff=%lld k=%lld tokens=%lld: NMSE vs CPU backend %.3g -> %s\n", ggml_type_name(type),
           (long long)n_expert, (long long)n_used, (long long)n_ff, (long long)k, (long long)n_tokens, d.worst, ok ? "OK" : "FAIL");
    ggml_backend_buffer_free(buf); ggml_free(ctx);
    return ok ? 0 : 1;
}

// ---- the MoE FFN of llm_build_moe_ffn with merged up/gate experts ----
struct moe_graph { ggml_context * ctx; ggml_cgraph * gf; ggml_tensor * cur, * logits, * par, * out; };
static moe_graph build_moe_ffn(ggml_tensor * up_gate, ggml_tensor * down, int64_t n_embd, int64_t n_expert, int64_t n_used, int64_t n) {
    ggml_init_params ip = { ggml_tensor_overhead() * 64 + ggml_graph_overhead(), nullptr, true };
    moe_graph g; g.ctx = ggml_init(ip); g.gf = ggml_new_graph(g.ctx);
    g.cur = ggml_new_tensor_2d(g.ctx, GGML_TYPE_F32, n_embd, n); ggml_set_input(g.cur);
    g.logits = ggml_new_tensor_2d(g.ctx, GGML_TYPE_F32, n_expert, n); ggml_set_input(g.logits);
    ggml_tensor * probs = ggml_soft_max(g.ctx, g.logits);
    ggml_tensor * selected = ggml_top_k(g.ctx, probs, (int)n_used);
    ggml_tensor * weights = ggml_get_rows(g.ctx, ggml_reshape_3d(g.ctx, probs, 1, n_expert, n), selected);
    ggml_build_forward_expand(g.gf, weights);
    g.par = moe_up_gate_merged(g.ctx, up_gate, ggml_reshape_3d(g.ctx, g.cur, n_embd, 1, n), selected);
    ggml_set_output(g.par);
    g.out = ggml_mul_mat_id(g.ctx, down, g.par, selected);
    ggml_set_output(g.out);
    ggml_build_forward_expand(g.gf, g.out);
    return g;
}
static int run_graph_case(ggml_backend_t be, ggml_backend_t cpu, const char * model, ggml_type type, int64_t n_expert, int64_t n_used, int64_t n_embd, int64_t n_ff,
                          unsigned seed) {
    std::mt19937 rng(seed);
    // the same weights in a plug buffer (usage WEIGHTS, as llama's model buffers) and in a CPU buffer
    ggml_init_params wp = { ggml_tensor_overhead() * 4, nullptr, true };
    ggml_context * wctx[2] = { ggml_init(wp), ggml_init(wp) };
    ggml_tensor * ug[2], * dn[2]; ggml_backend_buffer_t wbuf[2];
    for (int s = 0; s < 2; ++s) {
        ug[s] = ggml_new_tensor_3d(wctx[s], type, n_embd, 2 * n_ff, n_expert); ggml_set_name(ug[s], "blk.0.ffn_gate_up_exps.weight");
        dn[s] = ggml_new_tensor_3d(wctx[s], type, n_ff, n_embd, n_expert); ggml_set_name(dn[s], "blk.0.ffn_down_exps.weight");
        wbuf[s] = s == 0 ? ggml_backend_alloc_ctx_tensors_from_buft(wctx[s], ggml_backend_cuda_buffer_type(0)) : ggml_backend_alloc_ctx_tensors(wctx[s], cpu);
        if (!wbuf[s]) { printf("  weight allocation failed\n"); return 1; }
    }
    ggml_backend_buffer_set_usage(wbuf[0], GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    const std::vector<uint8_t> wug = quantized_rows(type, n_embd, ggml_nrows(ug[0]), rng), wdn = quantized_rows(type, n_ff, ggml_nrows(dn[0]), rng);
    for (int s = 0; s < 2; ++s) { ggml_backend_tensor_set(ug[s], wug.data(), 0, wug.size()); ggml_backend_tensor_set(dn[s], wdn.data(), 0, wdn.size()); }
    int fails = 0;
    for (int64_t n : {1, 2, 8, 24, 160, 512}) {
        std::normal_distribution<float> nd(0.f, 1.f);
        std::vector<float> cur(n_embd * n), logits(n_expert * n);
        for (auto & v : cur) v = nd(rng);
        for (auto & v : logits) v = nd(rng);
        // plug + CPU under the scheduler
        moe_graph a = build_moe_ffn(ug[0], dn[0], n_embd, n_expert, n_used, n);
        const bool supported = ggml_backend_supports_op(be, a.par);
        ggml_backend_t backends[2] = { be, cpu };
        ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, 2, 4096, false);
        if (!ggml_backend_sched_alloc_graph(sched, a.gf)) { printf("  ggml_backend_sched_alloc_graph failed\n"); return 1; }
        ggml_backend_tensor_set(a.cur, cur.data(), 0, cur.size() * sizeof(float)); ggml_backend_tensor_set(a.logits, logits.data(), 0, logits.size() * sizeof(float));
        if (ggml_backend_sched_graph_compute(sched, a.gf) != GGML_STATUS_SUCCESS) { printf("  graph compute failed\n"); return 1; }
        ggml_backend_sched_synchronize(sched);
        const bool on_plug = ggml_backend_sched_get_tensor_backend(sched, a.par) == be;
        const std::vector<float> par_a = get_f32(a.par), out_a = get_f32(a.out);
        ggml_backend_sched_free(sched); ggml_free(a.ctx);
        // the reference CPU backend alone, through a scheduler of its own (same graph preparation as above)
        moe_graph b = build_moe_ffn(ug[1], dn[1], n_embd, n_expert, n_used, n);
        ggml_backend_sched_t sched_cpu = ggml_backend_sched_new(&cpu, nullptr, 1, 4096, false);
        if (!ggml_backend_sched_alloc_graph(sched_cpu, b.gf)) { printf("  ggml_backend_sched_alloc_graph (CPU) failed\n"); return 1; }
        ggml_backend_tensor_set(b.cur, cur.data(), 0, cur.size() * sizeof(float)); ggml_backend_tensor_set(b.logits, logits.data(), 0, logits.size() * sizeof(float));
        if (ggml_backend_sched_graph_compute(sched_cpu, b.gf) != GGML_STATUS_SUCCESS) { printf("  CPU graph compute failed\n"); return 1; }
        ggml_backend_sched_synchronize(sched_cpu);
        const double e_par = nmse(par_a, get_f32(b.par)), e_out = nmse(out_a, get_f32(b.out));
        ggml_backend_sched_free(sched_cpu); ggml_free(b.ctx);
        const bool ok = supported && on_plug && e_par <= 5e-4 && e_out <= 5e-4;
        printf("  %-16s %-8s merged up/gate n=%-4lld: supported %d, ran on %s, NMSE vs CPU backend: up/gate %.3g, layer output %.3g -> %s\n", model, ggml_type_name(type),
               (long long)n, (int)supported, on_plug ? "the plug" : "ANOTHER BACKEND", e_par, e_out, ok ? "OK" : "FAIL");
        fails += !ok;
    }
    for (int s = 0; s < 2; ++s) { ggml_backend_buffer_free(wbuf[s]); ggml_free(wctx[s]); }
    return fails;
}

// The reference CPU op's work-size plan for MOE_FUSED_UP_GATE reserves room for the quantised activations only when src[1] is set (ggml.c:28852-28866),
// yet the merged form (src[1] = NULL) writes them there too.  A llama graph gets that room from its other nodes; a graph of the merged node alone
// (and ggml_backend_compare_graph_backend, which computes one node at a time) would overrun it.  The CPU backend's work buffer only grows
// (ggml-backend.cpp:880-888): one throwaway product sized for the largest case here reserves it up front.
static void reserve_cpu_work(ggml_backend_t cpu) {
    const int64_t k = 4096, rows = 4096;                            // row_size(Q8_K, 4096) x 4096 rows = 19 MB
    ggml_init_params ip = { ggml_tensor_overhead() * 4 + ggml_graph_overhead(), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
    ggml_tensor * w = ggml_new_tensor_2d(ctx, GGML_TYPE_Q4_K, k, 32), * x = ggml_new_tensor_2d(ctx, GGML_TYPE_F32, k, rows);
    ggml_cgraph * gf = ggml_new_graph(ctx); ggml_build_forward_expand(gf, ggml_mul_mat(ctx, w, x));
    ggml_backend_buffer_t buf = ggml_backend_alloc_ctx_tensors(ctx, cpu);
    ggml_backend_buffer_clear(buf, 0);
    ggml_backend_graph_compute(cpu, gf);
    ggml_backend_buffer_free(buf); ggml_free(ctx);
}

int main(int argc, char ** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode != "op" && mode != "graph") { fprintf(stderr, "usage: %s op|graph\n", argv[0]); return 2; }
    ggml_backend_t be = ggml_backend_cuda_init(0, "pdl=1", nullptr);
    if (!be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    ggml_backend_t cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(cpu, 8);
    reserve_cpu_work(cpu);
    int fails = 0; unsigned seed = 7000;
    if (mode == "op") {
        for (ggml_type t : {GGML_TYPE_IQ4_NL, GGML_TYPE_Q4_K, GGML_TYPE_IQ2_XXS}) for (int64_t n : {1, 8, 512}) fails += run_op_case(be, cpu, t, n, ++seed);
    } else {
        fails += run_graph_case(be, cpu, "qwen3-30b-a3b", GGML_TYPE_Q4_K, 128, 8, 512, 256, ++seed);
        fails += run_graph_case(be, cpu, "mixtral-8x7b", GGML_TYPE_IQ4_NL, 8, 2, 1024, 512, ++seed);
        fails += run_graph_case(be, cpu, "deepseek-v3", GGML_TYPE_IQ2_XXS, 256, 8, 512, 256, ++seed);
    }
    printf("%s: %d failures\n", fails ? "FAILED" : "PASSED", fails);
    ggml_backend_free(be); ggml_backend_free(cpu);
    return fails ? 1 : 0;
}
