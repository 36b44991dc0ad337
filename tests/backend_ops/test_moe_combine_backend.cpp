// tests/backend_ops/test_moe_combine_backend.cpp — GGML_OP_MUL_MULTI_ADD (ggml_mul_multi_add(experts, weights), the expert-weighted sum that ends
// llm_build_moe_ffn under fused_mmad, src/llama-build-context.cpp:1667-1680) through the reference's ggml-backend API.  The arbiter is the unmodified
// reference CPU backend.
//   test_moe_combine_backend op     the node alone, on the plug and on the CPU backend (ggml_backend_compare_graph_backend), NMSE <= 5e-4, for
//                                   n_used 1, 2, 8, m % 4 != 0 and 1 ... 512 tokens
//   test_moe_combine_backend graph  the fused_mmad MoE FFN as llm_build_moe_ffn builds it (softmax -> top_k -> get_rows weights -> MOE_FUSED_UP_GATE ->
//                                   MUL_MAT_ID ffn_down_exps -> ggml_mul_multi_add) at the Qwen3-30B-A3B, Mixtral-8x7B and DeepSeek-V3 shapes of
//                                   test_plug_graphs.cpp and 1 ... 512 tokens, placed by ggml_backend_sched next to the CPU backend with the weights in
//                                   a plug buffer: MUL_MULTI_ADD must run on the plug, and the layer output must match the same graph on the CPU
//                                   backend alone (NMSE <= 5e-4)
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <algorithm>
#include <cstdio>
#include <cstring>
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

// ---- the node alone ----
static int run_op_case(ggml_backend_t be, ggml_backend_t cpu, int64_t m, int64_t n_used, int64_t n_tokens, unsigned seed) {
    ggml_init_params ip = { ggml_tensor_overhead() * 8 + ggml_graph_overhead(), nullptr, true };
    ggml_context * ctx = ggml_init(ip);
    ggml_tensor * e = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, m, n_used, n_tokens);
    ggml_tensor * w = ggml_new_tensor_3d(ctx, GGML_TYPE_F32, 1, n_used, n_tokens);
    ggml_tensor * y = ggml_mul_multi_add(ctx, e, w);
    ggml_cgraph * gf = ggml_new_graph(ctx); ggml_build_forward_expand(gf, y);
    ggml_backend_buffer_t buf = ggml_backend_alloc_ctx_tensors(ctx, be);
    if (!buf) { printf("  alloc failed\n"); return 1; }
    std::mt19937 rng(seed);
    std::normal_distribution<float> nd(0.f, 1.f); std::uniform_real_distribution<float> u(0.f, 1.f);
    std::vector<float> ev(ggml_nelements(e)), wv(ggml_nelements(w));
    for (auto & v : ev) v = nd(rng);
    for (auto & v : wv) v = u(rng);
    ggml_backend_tensor_set(e, ev.data(), 0, ev.size() * sizeof(float)); ggml_backend_tensor_set(w, wv.data(), 0, wv.size() * sizeof(float));
    if (!ggml_backend_supports_op(be, y)) { printf("  MUL_MULTI_ADD m=%lld n_used=%lld not supported\n", (long long)m, (long long)n_used); return 1; }
    cb_data d; ggml_backend_compare_graph_backend(be, cpu, gf, cmp_cb, &d);
    const bool ok = d.n > 0 && d.worst <= 5e-4;
    printf("  MUL_MULTI_ADD m=%-5lld n_used=%lld tokens=%-4lld: NMSE vs CPU backend %.3g -> %s\n", (long long)m, (long long)n_used, (long long)n_tokens, d.worst, ok ? "OK" : "FAIL");
    ggml_backend_buffer_free(buf); ggml_free(ctx);
    return ok ? 0 : 1;
}

// ---- the MoE FFN of llm_build_moe_ffn with fused_mmad ----
struct moe_graph { ggml_context * ctx; ggml_cgraph * gf; ggml_tensor * cur, * logits, * experts, * out; };
static moe_graph build_moe_ffn(ggml_tensor * up, ggml_tensor * gate, ggml_tensor * down, int64_t n_embd, int64_t n_expert, int64_t n_used, int64_t n) {
    ggml_init_params ip = { ggml_tensor_overhead() * 64 + ggml_graph_overhead(), nullptr, true };
    moe_graph g; g.ctx = ggml_init(ip); g.gf = ggml_new_graph(g.ctx);
    g.cur = ggml_new_tensor_2d(g.ctx, GGML_TYPE_F32, n_embd, n); ggml_set_input(g.cur);
    g.logits = ggml_new_tensor_2d(g.ctx, GGML_TYPE_F32, n_expert, n); ggml_set_input(g.logits);
    ggml_tensor * probs = ggml_soft_max(g.ctx, g.logits);
    ggml_tensor * selected = ggml_top_k(g.ctx, probs, (int)n_used);
    ggml_tensor * weights = ggml_get_rows(g.ctx, ggml_reshape_3d(g.ctx, probs, 1, n_expert, n), selected);
    ggml_build_forward_expand(g.gf, weights);
    ggml_tensor * par = ggml_moe_up_gate(g.ctx, up, gate, ggml_reshape_3d(g.ctx, g.cur, n_embd, 1, n), selected, GGML_UNARY_OP_SILU);
    *((float *)(par->op_params + 1)) = 0.0f;            // the swiglu limit slot llm_build_moe_ffn writes (no limit)
    g.experts = ggml_mul_mat_id(g.ctx, down, par, selected);
    ggml_set_output(g.experts);
    g.out = ggml_mul_multi_add(g.ctx, g.experts, weights);
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
    ggml_tensor * up[2], * gt[2], * dn[2]; ggml_backend_buffer_t wbuf[2];
    for (int s = 0; s < 2; ++s) {
        up[s] = ggml_new_tensor_3d(wctx[s], type, n_embd, n_ff, n_expert); ggml_set_name(up[s], "blk.0.ffn_up_exps.weight");
        gt[s] = ggml_new_tensor_3d(wctx[s], type, n_embd, n_ff, n_expert); ggml_set_name(gt[s], "blk.0.ffn_gate_exps.weight");
        dn[s] = ggml_new_tensor_3d(wctx[s], type, n_ff, n_embd, n_expert); ggml_set_name(dn[s], "blk.0.ffn_down_exps.weight");
        wbuf[s] = s == 0 ? ggml_backend_alloc_ctx_tensors_from_buft(wctx[s], ggml_backend_cuda_buffer_type(0)) : ggml_backend_alloc_ctx_tensors(wctx[s], cpu);
        if (!wbuf[s]) { printf("  weight allocation failed\n"); return 1; }
    }
    ggml_backend_buffer_set_usage(wbuf[0], GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    const std::vector<uint8_t> wup = quantized_rows(type, n_embd, ggml_nrows(up[0]), rng), wgt = quantized_rows(type, n_embd, ggml_nrows(gt[0]), rng),
                               wdn = quantized_rows(type, n_ff, ggml_nrows(dn[0]), rng);
    for (int s = 0; s < 2; ++s) {
        ggml_backend_tensor_set(up[s], wup.data(), 0, wup.size()); ggml_backend_tensor_set(gt[s], wgt.data(), 0, wgt.size());
        ggml_backend_tensor_set(dn[s], wdn.data(), 0, wdn.size());
    }
    int fails = 0;
    for (int64_t n : {1, 8, 64, 512}) {
        std::normal_distribution<float> nd(0.f, 1.f);
        std::vector<float> cur(n_embd * n), logits(n_expert * n);
        for (auto & v : cur) v = nd(rng);
        for (auto & v : logits) v = nd(rng);
        // plug + CPU under the scheduler
        moe_graph a = build_moe_ffn(up[0], gt[0], dn[0], n_embd, n_expert, n_used, n);
        const bool supported = ggml_backend_supports_op(be, a.out);
        ggml_backend_t backends[2] = { be, cpu };
        ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, 2, 4096, false);
        if (!ggml_backend_sched_alloc_graph(sched, a.gf)) { printf("  ggml_backend_sched_alloc_graph failed\n"); return 1; }
        ggml_backend_tensor_set(a.cur, cur.data(), 0, cur.size() * sizeof(float)); ggml_backend_tensor_set(a.logits, logits.data(), 0, logits.size() * sizeof(float));
        if (ggml_backend_sched_graph_compute(sched, a.gf) != GGML_STATUS_SUCCESS) { printf("  graph compute failed\n"); return 1; }
        ggml_backend_sched_synchronize(sched);
        const bool on_plug = ggml_backend_sched_get_tensor_backend(sched, a.out) == be && ggml_backend_sched_get_tensor_backend(sched, a.experts) == be;
        const std::vector<float> out_a = get_f32(a.out);
        ggml_backend_sched_free(sched); ggml_free(a.ctx);
        // the reference CPU backend alone, through a scheduler of its own (same graph preparation as above)
        moe_graph b = build_moe_ffn(up[1], gt[1], dn[1], n_embd, n_expert, n_used, n);
        ggml_backend_sched_t sched_cpu = ggml_backend_sched_new(&cpu, nullptr, 1, 4096, false);
        if (!ggml_backend_sched_alloc_graph(sched_cpu, b.gf)) { printf("  ggml_backend_sched_alloc_graph (CPU) failed\n"); return 1; }
        ggml_backend_tensor_set(b.cur, cur.data(), 0, cur.size() * sizeof(float)); ggml_backend_tensor_set(b.logits, logits.data(), 0, logits.size() * sizeof(float));
        if (ggml_backend_sched_graph_compute(sched_cpu, b.gf) != GGML_STATUS_SUCCESS) { printf("  CPU graph compute failed\n"); return 1; }
        ggml_backend_sched_synchronize(sched_cpu);
        const double e_out = nmse(out_a, get_f32(b.out));
        ggml_backend_sched_free(sched_cpu); ggml_free(b.ctx);
        const bool ok = supported && on_plug && e_out <= 5e-4;
        printf("  %-16s %-8s fused_mmad MoE FFN n=%-4lld: MUL_MULTI_ADD supported %d, down + combine ran on %s, layer output NMSE vs CPU backend %.3g -> %s\n", model,
               ggml_type_name(type), (long long)n, (int)supported, on_plug ? "the plug" : "ANOTHER BACKEND", e_out, ok ? "OK" : "FAIL");
        fails += !ok;
    }
    for (int s = 0; s < 2; ++s) { ggml_backend_buffer_free(wbuf[s]); ggml_free(wctx[s]); }
    return fails;
}

int main(int argc, char ** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    if (mode != "op" && mode != "graph") { fprintf(stderr, "usage: %s op|graph\n", argv[0]); return 2; }
    ggml_backend_t be = ggml_backend_cuda_init(0, "pdl=1", nullptr);
    if (!be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    ggml_backend_t cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(cpu, 8);
    int fails = 0; unsigned seed = 9000;
    if (mode == "op") {
        for (int64_t n_used : {1, 2, 8}) for (int64_t m : {7168, 4097}) for (int64_t n : {1, 3, 64, 512}) fails += run_op_case(be, cpu, m, n_used, n, ++seed);
    } else {
        fails += run_graph_case(be, cpu, "qwen3-30b-a3b", GGML_TYPE_Q4_K, 128, 8, 512, 256, ++seed);
        fails += run_graph_case(be, cpu, "mixtral-8x7b", GGML_TYPE_IQ4_NL, 8, 2, 1024, 512, ++seed);
        fails += run_graph_case(be, cpu, "deepseek-v3", GGML_TYPE_IQ2_XXS, 256, 8, 512, 256, ++seed);
    }
    printf("%s: %d failures\n", fails ? "FAILED" : "PASSED", fails);
    ggml_backend_free(be); ggml_backend_free(cpu);
    return fails ? 1 : 0;
}
