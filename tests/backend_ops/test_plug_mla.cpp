// tests/backend_ops/test_plug_mla.cpp — batched GGML_OP_MUL_MAT through the reference's ggml-backend API: the two per-head products of absorbed MLA
// (DeepSeek-V2/V3) built with the reference's constructors as src/graphs/build_deepseek2.cpp builds them, and contiguous batched products.
//   q_nope2 = ggml_mul_mat(wk_b [128, 512, n_head], permute(view_3d(q [192, n_head, n_tokens], 128 ...), 0, 2, 1, 3))      (:1030-1036)
//   kqv     = ggml_mul_mat(wv_b [512, 128, n_head], permute(kqv_compressed [512, n_head, n_tokens], 0, 2, 1, 3))           (:1145-1162)
// f32 inputs stand in for q and the flash-attention output.  Each graph runs under ggml_backend_sched with the plug next to the CPU backend and the
// weights in a plug buffer (usage WEIGHTS): the MUL_MAT must run on the plug (so wk_b / wv_b are never read back to the host), and its result must
// match the same graph on the reference CPU backend alone (NMSE <= 5e-4).  The contiguous cases cover a weight broadcast over ne2, a weight
// broadcast over ne3, and one weight matrix per batch entry.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

static double nmse(const std::vector<float> & a, const std::vector<float> & b) {
    double e = 0, s = 0; for (size_t i = 0; i < a.size(); ++i) { e += ((double)a[i] - b[i]) * ((double)a[i] - b[i]); s += (double)b[i] * b[i]; } return e / (s > 0 ? s : 1e-300);
}
static std::vector<float> get_f32(const ggml_tensor * t) { std::vector<float> v(ggml_nelements(t)); ggml_backend_tensor_get(t, v.data(), 0, ggml_nbytes(t)); return v; }
static std::vector<uint8_t> quantized(ggml_type type, int64_t k, int64_t rows, std::mt19937 & rng) {
    std::uniform_real_distribution<float> u(-0.05f, 0.05f);
    std::vector<float> f(rows * k); for (auto & v : f) v = u(rng);
    std::vector<uint8_t> q(rows * ggml_row_size(type, k));
    ggml_quantize_chunk(type, f.data(), q.data(), 0, rows, k, nullptr, nullptr);
    return q;
}

enum kind { Q_NOPE, KQV_COMPRESSED, CONTIGUOUS };
struct mm_case { const char * label; kind kd; int64_t k, m, w2, w3, n, b2, b3; };     // weight [k, m, w2, w3]; src1 [k, n, b2, b3] (contiguous)

struct mm_graph { ggml_context * ctx; ggml_cgraph * gf; ggml_tensor * in, * out; };
static mm_graph build(const mm_case & c, ggml_tensor * w) {
    ggml_init_params ip = { ggml_tensor_overhead() * 16 + ggml_graph_overhead(), nullptr, true };
    mm_graph g; g.ctx = ggml_init(ip); g.gf = ggml_new_graph(g.ctx);
    ggml_tensor * x;
    if (c.kd == Q_NOPE) {               // q [n_embd_head_qk_nope + rope, n_head, n_tokens]; q_nope = its first 128 floats of each head, permuted
        g.in = ggml_new_tensor_3d(g.ctx, GGML_TYPE_F32, 192, c.b2, c.n);
        ggml_tensor * q_nope = ggml_view_3d(g.ctx, g.in, 128, c.b2, c.n, g.in->nb[1], g.in->nb[2], 0);
        x = ggml_permute(g.ctx, q_nope, 0, 2, 1, 3);
    } else if (c.kd == KQV_COMPRESSED) {   // the flash-attention output [kv_lora_rank, n_head, n_tokens], permuted
        g.in = ggml_new_tensor_3d(g.ctx, GGML_TYPE_F32, 512, c.b2, c.n);
        x = ggml_permute(g.ctx, g.in, 0, 2, 1, 3);
    } else {
        g.in = ggml_new_tensor_4d(g.ctx, GGML_TYPE_F32, c.k, c.n, c.b2, c.b3);
        x = g.in;
    }
    ggml_set_input(g.in);
    g.out = ggml_mul_mat(g.ctx, w, x);
    ggml_set_output(g.out);
    ggml_build_forward_expand(g.gf, g.out);
    return g;
}

static int run_case(ggml_backend_t be, ggml_backend_t cpu, const mm_case & c, ggml_type type, unsigned seed) {
    std::mt19937 rng(seed);
    ggml_init_params wp = { ggml_tensor_overhead() * 2, nullptr, true };
    ggml_context * wctx[2] = { ggml_init(wp), ggml_init(wp) };
    ggml_tensor * w[2]; ggml_backend_buffer_t wbuf[2];
    for (int s = 0; s < 2; ++s) {
        w[s] = ggml_new_tensor_4d(wctx[s], type, c.k, c.m, c.w2, c.w3); ggml_set_name(w[s], "blk.0.attn_k_b.weight");
        wbuf[s] = s == 0 ? ggml_backend_alloc_ctx_tensors_from_buft(wctx[s], ggml_backend_cuda_buffer_type(0)) : ggml_backend_alloc_ctx_tensors(wctx[s], cpu);
        if (!wbuf[s]) { printf("  weight allocation failed\n"); return 1; }
    }
    ggml_backend_buffer_set_usage(wbuf[0], GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    const std::vector<uint8_t> wq = quantized(type, c.k, ggml_nrows(w[0]), rng);
    for (int s = 0; s < 2; ++s) ggml_backend_tensor_set(w[s], wq.data(), 0, wq.size());

    mm_graph a = build(c, w[0]);
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<float> in(ggml_nelements(a.in)); for (auto & v : in) v = nd(rng);
    const bool supported = ggml_backend_supports_op(be, a.out);
    ggml_backend_t backends[2] = { be, cpu };
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, 2, 256, false);
    if (!ggml_backend_sched_alloc_graph(sched, a.gf)) { printf("  ggml_backend_sched_alloc_graph failed\n"); return 1; }
    ggml_backend_tensor_set(a.in, in.data(), 0, in.size() * sizeof(float));
    if (ggml_backend_sched_graph_compute(sched, a.gf) != GGML_STATUS_SUCCESS) { printf("  graph compute failed\n"); return 1; }
    ggml_backend_sched_synchronize(sched);
    const bool on_plug = ggml_backend_sched_get_tensor_backend(sched, a.out) == be;
    const std::vector<float> out_a = get_f32(a.out);
    ggml_backend_sched_free(sched); ggml_free(a.ctx);

    mm_graph b = build(c, w[1]);
    ggml_backend_sched_t sched_cpu = ggml_backend_sched_new(&cpu, nullptr, 1, 256, false);
    if (!ggml_backend_sched_alloc_graph(sched_cpu, b.gf)) { printf("  ggml_backend_sched_alloc_graph (CPU) failed\n"); return 1; }
    ggml_backend_tensor_set(b.in, in.data(), 0, in.size() * sizeof(float));
    if (ggml_backend_sched_graph_compute(sched_cpu, b.gf) != GGML_STATUS_SUCCESS) { printf("  CPU graph compute failed\n"); return 1; }
    ggml_backend_sched_synchronize(sched_cpu);
    const double e = nmse(out_a, get_f32(b.out));
    ggml_backend_sched_free(sched_cpu); ggml_free(b.ctx);
    for (int s = 0; s < 2; ++s) { ggml_backend_buffer_free(wbuf[s]); ggml_free(wctx[s]); }

    const bool ok = supported && on_plug && e <= 5e-4;
    printf("  %-26s %-6s n=%-4lld batch %lldx%lld: supported %d, ran on %s, NMSE vs CPU backend %.3g -> %s\n", c.label, ggml_type_name(type), (long long)c.n,
           (long long)c.b2, (long long)c.b3, (int)supported, on_plug ? "the plug" : "ANOTHER BACKEND", e, ok ? "OK" : "FAIL");
    return ok ? 0 : 1;
}

int main(int argc, char ** argv) {
    const bool mla = argc > 1 && !strcmp(argv[1], "mla"), contiguous = argc > 1 && !strcmp(argv[1], "contiguous");
    if (!mla && !contiguous) { fprintf(stderr, "usage: %s mla|contiguous\n", argv[0]); return 2; }
    ggml_backend_t be = ggml_backend_cuda_init(0, "pdl=1", nullptr);
    if (!be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    ggml_backend_t cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(cpu, 8);
    int fails = 0; unsigned seed = 7100;
    if (mla) {
        for (ggml_type type : {GGML_TYPE_Q8_0, GGML_TYPE_IQ4_NL}) for (int64_t n_head : {16, 128}) {
            for (int64_t n : {1, 2, 9, 64, n_head == 16 ? 512 : 128}) {
                fails += run_case(be, cpu, {"q_nope2 = wk_b x q_nope_perm", Q_NOPE, 128, 512, n_head, 1, n, n_head, 1}, type, ++seed);
                fails += run_case(be, cpu, {"kqv = wv_b x kqv_c_perm", KQV_COMPRESSED, 512, 128, n_head, 1, n, n_head, 1}, type, ++seed);
            }
        }
    } else {
        for (ggml_type type : {GGML_TYPE_Q8_0, GGML_TYPE_Q4_K}) for (int64_t n : {1, 4, 16, 64}) {
            fails += run_case(be, cpu, {"broadcast over ne2", CONTIGUOUS, 256, 192, 1, 1, n, 5, 1}, type, ++seed);
            fails += run_case(be, cpu, {"broadcast over ne3", CONTIGUOUS, 256, 192, 1, 1, n, 1, 3}, type, ++seed);
            fails += run_case(be, cpu, {"one matrix per entry", CONTIGUOUS, 256, 192, 6, 1, n, 6, 1}, type, ++seed);
        }
    }
    printf("%s: %d failures\n", fails ? "FAILED" : "PASSED", fails);
    ggml_backend_free(be); ggml_backend_free(cpu);
    return fails ? 1 : 0;
}
