// tests/backend_ops/test_plug_mla_pp.cpp — the MLA prompt-processing product of DeepSeek's "pp_opt" graph (mla >= 2 with flash attention) through the
// reference's ggml-backend API, built with the reference's constructors as src/graphs/build_deepseek2.cpp:922-990 builds it:
//   kv_cache_nope = ggml_view_2d(k_l, kv_lora_rank, n_kv, k_l->nb[1], ggml_row_size(k_l->type, n_embd_head_qk_rope))          (:924-925)
//   wkv_b_iter    = ggml_view_2d(wkv_b, 512, n_per_head*n_max_head, wkv_b->nb[1], wkv_b->nb[1]*n_per_head*n_max_head*iter)    (:971-972)
//   kv_f32        = ggml_mul_mat(wkv_b_iter, kv_cache_nope)                                                                  (:974)
// followed by the v_f32 / k_nope_f32 views of kv_f32 and their f16 casts (:977-992).  The K cache k_l is f16 [576, kv_size] in a plug buffer, filled
// with ggml_backend_tensor_set (the cache write is not part of the graph: the plug does not run CPY); wkv_b is in a plug buffer of usage WEIGHTS.
// Each graph runs under ggml_backend_sched with the plug next to the reference CPU backend: every MUL_MAT must run on the plug (so wkv_b is never read
// back to the host), and every kv_f32 must match the same rows of the whole product on the CPU backend alone (NMSE <= 5e-4).  The CPU product, which
// does not depend on the split, is computed once per weight and cache.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

static constexpr int64_t KV_LORA_RANK = 512, QK_ROPE = 64, QK_NOPE = 128, V_HEAD = 128;

static std::vector<float> get_f32(const ggml_tensor * t) { std::vector<float> v(ggml_nelements(t)); ggml_backend_tensor_get(t, v.data(), 0, ggml_nbytes(t)); return v; }
static std::vector<uint8_t> quantized(ggml_type type, int64_t k, int64_t rows, std::mt19937 & rng) {
    std::uniform_real_distribution<float> u(-0.05f, 0.05f);
    std::vector<float> f(rows * k); for (auto & v : f) v = u(rng);
    std::vector<uint8_t> q(rows * ggml_row_size(type, k));
    ggml_quantize_chunk(type, f.data(), q.data(), 0, rows, k, nullptr, nullptr);
    return q;
}

struct pp_graph { ggml_context * ctx; ggml_cgraph * gf; std::vector<ggml_tensor *> kv_f32; };
static pp_graph build(ggml_tensor * k_l, ggml_tensor * wkv_b, int64_t n_head, int64_t n_max_head, int64_t n_kv) {
    const int64_t n_iter = n_head / n_max_head;
    ggml_init_params ip = { ggml_tensor_overhead() * (8 + 8 * n_iter) + ggml_graph_overhead(), nullptr, true };
    pp_graph g; g.ctx = ggml_init(ip); g.gf = ggml_new_graph(g.ctx);
    ggml_tensor * kv_cache_nope = ggml_view_2d(g.ctx, k_l, KV_LORA_RANK, n_kv, k_l->nb[1], ggml_row_size(k_l->type, QK_ROPE));
    const int64_t n_per_head = wkv_b->ne[1] / n_head;
    for (int64_t iter = 0; iter < n_iter; ++iter) {
        ggml_tensor * w = ggml_view_2d(g.ctx, wkv_b, wkv_b->ne[0], n_per_head * n_max_head, wkv_b->nb[1], wkv_b->nb[1] * n_per_head * n_max_head * iter);
        ggml_tensor * kv_f32 = ggml_mul_mat(g.ctx, w, kv_cache_nope);
        ggml_set_output(kv_f32);
        ggml_tensor * v_f32 = ggml_view_3d(g.ctx, kv_f32, V_HEAD, n_kv, n_max_head, ggml_row_size(kv_f32->type, n_max_head * (QK_NOPE + V_HEAD)),
                                           ggml_row_size(kv_f32->type, QK_NOPE + V_HEAD), ggml_row_size(kv_f32->type, QK_NOPE));
        ggml_tensor * k_nope_f32 = ggml_view_3d(g.ctx, kv_f32, QK_NOPE, n_kv, n_max_head, ggml_row_size(kv_f32->type, n_max_head * (QK_NOPE + V_HEAD)),
                                                ggml_row_size(kv_f32->type, QK_NOPE + V_HEAD), 0);
        ggml_build_forward_expand(g.gf, ggml_cast(g.ctx, k_nope_f32, GGML_TYPE_F16));
        ggml_build_forward_expand(g.gf, ggml_cast(g.ctx, v_f32, GGML_TYPE_F16));
        g.kv_f32.push_back(kv_f32);
    }
    return g;
}

struct side { ggml_context * ctx, * kctx; ggml_tensor * k_l, * wkv_b; ggml_backend_buffer_t kbuf, wbuf; };
static bool make_side(side & s, ggml_backend_t cpu, bool plug, ggml_type type, int64_t n_head, int64_t kv_size, const std::vector<uint16_t> & cache,
                      const std::vector<uint8_t> & wq) {
    ggml_init_params wp = { ggml_tensor_overhead() * 2, nullptr, true };
    s.ctx = ggml_init(wp); s.kctx = ggml_init(wp);
    s.k_l = ggml_new_tensor_2d(s.kctx, GGML_TYPE_F16, KV_LORA_RANK + QK_ROPE, kv_size); ggml_set_name(s.k_l, "cache_k_l0");
    s.wkv_b = ggml_new_tensor_2d(s.ctx, type, KV_LORA_RANK, n_head * (QK_NOPE + V_HEAD)); ggml_set_name(s.wkv_b, "blk.0.attn_kv_b.weight");
    s.kbuf = plug ? ggml_backend_alloc_ctx_tensors_from_buft(s.kctx, ggml_backend_cuda_buffer_type(0)) : ggml_backend_alloc_ctx_tensors(s.kctx, cpu);
    s.wbuf = plug ? ggml_backend_alloc_ctx_tensors_from_buft(s.ctx, ggml_backend_cuda_buffer_type(0)) : ggml_backend_alloc_ctx_tensors(s.ctx, cpu);
    if (!s.kbuf || !s.wbuf) return false;
    if (plug) ggml_backend_buffer_set_usage(s.wbuf, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    ggml_backend_tensor_set(s.k_l, cache.data(), 0, cache.size() * sizeof(uint16_t));
    ggml_backend_tensor_set(s.wkv_b, wq.data(), 0, wq.size());
    return true;
}
static void free_side(side & s) { ggml_backend_buffer_free(s.kbuf); ggml_backend_buffer_free(s.wbuf); ggml_free(s.ctx); ggml_free(s.kctx); }

// the whole product on the CPU backend alone (one iteration): f32 [n_kv][rows]
static bool cpu_product(ggml_backend_t cpu, side & s, int64_t n_head, int64_t n_kv, std::vector<float> & out) {
    pp_graph g = build(s.k_l, s.wkv_b, n_head, n_head, n_kv);
    ggml_backend_sched_t sched = ggml_backend_sched_new(&cpu, nullptr, 1, 256, false);
    const bool ok = ggml_backend_sched_alloc_graph(sched, g.gf) && ggml_backend_sched_graph_compute(sched, g.gf) == GGML_STATUS_SUCCESS;
    if (ok) { ggml_backend_sched_synchronize(sched); out = get_f32(g.kv_f32[0]); }
    ggml_backend_sched_free(sched); ggml_free(g.ctx);
    return ok;
}

static int run_split(ggml_backend_t be, ggml_backend_t cpu, side & s, ggml_type type, int64_t n_head, int64_t n_max_head, int64_t n_kv, const std::vector<float> & ref) {
    pp_graph g = build(s.k_l, s.wkv_b, n_head, n_max_head, n_kv);
    bool supported = true;
    for (ggml_tensor * t : g.kv_f32) supported = supported && ggml_backend_supports_op(be, t);
    ggml_backend_t backends[2] = { be, cpu };
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, 2, 1024, false);
    if (!ggml_backend_sched_alloc_graph(sched, g.gf) || ggml_backend_sched_graph_compute(sched, g.gf) != GGML_STATUS_SUCCESS) {
        printf("  graph allocation / compute failed\n"); ggml_backend_sched_free(sched); ggml_free(g.ctx); return 1;
    }
    ggml_backend_sched_synchronize(sched);
    const int64_t rows = ref.size() / n_kv, r_iter = rows / (int64_t)g.kv_f32.size();
    bool on_plug = true; double e = 0, sq = 0;
    for (size_t it = 0; it < g.kv_f32.size(); ++it) {
        on_plug = on_plug && ggml_backend_sched_get_tensor_backend(sched, g.kv_f32[it]) == be;
        const std::vector<float> got = get_f32(g.kv_f32[it]);
        for (int64_t j = 0; j < n_kv; ++j) for (int64_t i = 0; i < r_iter; ++i) {
            const double a = got[j * r_iter + i], b = ref[j * rows + it * r_iter + i];
            e += (a - b) * (a - b); sq += b * b;
        }
    }
    ggml_backend_sched_free(sched); ggml_free(g.ctx);
    const double err = e / (sq > 0 ? sq : 1e-300);
    const bool ok = supported && on_plug && err <= 5e-4;
    printf("  wkv_b %-5s %3lld heads, n_max_head %3lld (%lld slices), n_kv %5lld: supported %d, ran on %s, NMSE vs CPU backend %.3g -> %s\n", ggml_type_name(type),
           (long long)n_head, (long long)n_max_head, (long long)(n_head / n_max_head), (long long)n_kv, (int)supported, on_plug ? "the plug" : "ANOTHER BACKEND", err,
           ok ? "OK" : "FAIL");
    return ok ? 0 : 1;
}

int main() {
    ggml_backend_t be = ggml_backend_cuda_init(0, "pdl=1", nullptr);
    if (!be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    ggml_backend_t cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(cpu, 8);
    int fails = 0; unsigned seed = 9100;
    struct shape { int64_t n_head; std::vector<int64_t> n_kv; };
    for (ggml_type type : {GGML_TYPE_Q8_0, GGML_TYPE_Q6_K}) for (const shape & sh : {shape{16, {256, 512, 1024, 2048}}, shape{128, {256, 1024}}}) for (int64_t n_kv : sh.n_kv) {
        std::mt19937 rng(++seed);
        const int64_t kv_size = n_kv + 256;         // a cache longer than the attended part, as in a running context
        std::normal_distribution<float> nd(0.f, 1.f);
        std::vector<uint16_t> cache((KV_LORA_RANK + QK_ROPE) * kv_size); for (auto & v : cache) v = ggml_fp32_to_fp16(nd(rng));
        const std::vector<uint8_t> wq = quantized(type, KV_LORA_RANK, sh.n_head * (QK_NOPE + V_HEAD), rng);
        side p{}, c{};
        if (!make_side(p, cpu, true, type, sh.n_head, kv_size, cache, wq) || !make_side(c, cpu, false, type, sh.n_head, kv_size, cache, wq)) { printf("  allocation failed\n"); return 1; }
        std::vector<float> ref;
        if (!cpu_product(cpu, c, sh.n_head, n_kv, ref)) { printf("  CPU graph failed\n"); ++fails; }
        else for (int64_t n_max_head : {sh.n_head, sh.n_head / 2, sh.n_head / 4}) fails += run_split(be, cpu, p, type, sh.n_head, n_max_head, n_kv, ref);
        free_side(p); free_side(c);
    }
    printf("%s: %d failures\n", fails ? "FAILED" : "PASSED", fails);
    ggml_backend_free(be); ggml_backend_free(cpu);
    return fails ? 1 : 0;
}
