// tests/backend_ops/test_plug_graphs.cpp — model-shaped graphs through ggml_backend_sched, with a dump of what every node read and wrote.
//
// Usage: test_plug_graphs <case> <out_dir>.  For each token count of the case, the graph is built with the reference's own constructors in the order
// llm_build_* uses them, the weights (and bias vectors) live in a buffer of the backend under test marked GGML_BACKEND_BUFFER_USAGE_WEIGHTS, the
// activations and routing logits are graph inputs, and ggml_backend_sched_new({backend, cpu}) decides where every node runs.  Every node is marked as
// an output (no intermediate is overwritten); no eval callback is installed, since it would split the graph and disable the backend's look-ahead
// fusions.  After ggml_backend_sched_graph_compute the harness writes
//   <out_dir>/w_<name>.npy         the wire bytes of every weight, read back through the backend's get_tensor (once per case);
//   <out_dir>/n<N>/manifest.jsonl  one line for the case, then one per node: name, op, type, shape, strides, op_params, the backend the scheduler gave
//                                  it, whether the backend under test supports it, and its sources as the node read them (after the scheduler's
//                                  copies), each with its own file;
//   <out_dir>/n<N>/t<i>.npy        the raw bytes of every node output and every other tensor a node read (u8; the manifest has type, ne and nb).
// tests/test_gpu_plug_graphs.py checks placement and values from the dump.  The expert weights are assembled from a pool of rows quantised by the
// reference's ggml_quantize_chunk, so the experts differ from each other while quantisation stays fast.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"
#include "ggml-cuda.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <sys/stat.h>
#include <vector>

static void write_npy(const std::string & path, const void * data, size_t n) {
    std::string hdr = "{'descr': '|u1', 'fortran_order': False, 'shape': (" + std::to_string(n) + ",), }";
    while ((10 + hdr.size() + 1) % 64) hdr += ' ';
    hdr += '\n';
    FILE * f = fopen(path.c_str(), "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(2); }
    const unsigned char magic[8] = {0x93, 'N', 'U', 'M', 'P', 'Y', 1, 0};
    const uint16_t hl = (uint16_t)hdr.size();
    fwrite(magic, 1, 8, f); fwrite(&hl, 2, 1, f); fwrite(hdr.data(), 1, hdr.size(), f); fwrite(data, 1, n, f);
    fclose(f);
}

static std::string json_str(const char * s) {
    std::string o = "\"";
    for (; *s; ++s) { if (*s == '"' || *s == '\\') o += '\\'; o += *s; }
    return o + "\"";
}
static std::string json_i64(const int64_t * v, int n) {
    std::string o = "[";
    for (int i = 0; i < n; ++i) o += (i ? "," : "") + std::to_string(v[i]);
    return o + "]";
}

// ----------------------------------------------------------------------------------------------------------------------------------------------
// weights
// ----------------------------------------------------------------------------------------------------------------------------------------------
struct weight_spec { std::string name; ggml_type type; int64_t k, m, e; };     // quantised [k, m, e] or f32 bias [k] (type F32)

struct case_ctx {
    ggml_backend_t be, cpu;
    ggml_context * wctx = nullptr; ggml_backend_buffer_t wbuf = nullptr;
    std::map<std::string, ggml_tensor *> w;
    std::string out;
    std::mt19937 rng;
    ggml_tensor * operator[](const std::string & n) { return w.at(n); }
};

// a pool of at most 1024 rows quantised by the reference, every row of the tensor drawn from it.  The weights have a trained model's magnitude
// (|w| < 0.05): the activations of a layer then stay near unit scale, as in a model, well inside the range of the q8_1 blocks' fp16 scales.
static void fill_quantized(ggml_tensor * t, std::mt19937 & rng) {
    const int64_t k = t->ne[0], rows = ggml_nrows(t), pool = rows < 1024 ? rows : 1024;
    const size_t rs = ggml_row_size(t->type, k);
    std::uniform_real_distribution<float> u(-0.05f, 0.05f);
    std::vector<float> f(pool * k); for (auto & v : f) v = u(rng);
    std::vector<float> ones(k, 1.0f);
    std::vector<uint8_t> pq(pool * rs), wq(ggml_nbytes(t));
    ggml_quantize_chunk(t->type, f.data(), pq.data(), 0, pool, k, ggml_quantize_requires_imatrix(t->type) ? ones.data() : nullptr, nullptr);
    for (int64_t r = 0; r < rows; ++r) memcpy(wq.data() + r * rs, pq.data() + (r < pool ? r : rng() % pool) * rs, rs);
    ggml_backend_tensor_set(t, wq.data(), 0, wq.size());
}

static void make_weights(case_ctx & c, const std::vector<weight_spec> & specs) {
    ggml_init_params ip = { ggml_tensor_overhead() * (specs.size() + 1), nullptr, true };
    c.wctx = ggml_init(ip);
    for (const auto & s : specs) {
        ggml_tensor * t = s.type == GGML_TYPE_F32 ? ggml_new_tensor_1d(c.wctx, GGML_TYPE_F32, s.k) : ggml_new_tensor_3d(c.wctx, s.type, s.k, s.m, s.e);
        ggml_set_name(t, s.name.c_str());
        c.w[s.name] = t;
    }
    c.wbuf = ggml_backend_alloc_ctx_tensors_from_buft(c.wctx, ggml_backend_cuda_buffer_type(0));
    if (!c.wbuf) { fprintf(stderr, "weight buffer allocation failed\n"); exit(2); }
    ggml_backend_buffer_set_usage(c.wbuf, GGML_BACKEND_BUFFER_USAGE_WEIGHTS);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    for (const auto & s : specs) {
        ggml_tensor * t = c.w[s.name];
        if (s.type == GGML_TYPE_F32) { std::vector<float> b(s.k); for (auto & v : b) v = u(c.rng); ggml_backend_tensor_set(t, b.data(), 0, b.size() * sizeof(float)); }
        else fill_quantized(t, c.rng);
        std::vector<uint8_t> back(ggml_nbytes(t));                 // what the dump's consumers see: the wire bytes get_tensor returns
        ggml_backend_tensor_get(t, back.data(), 0, back.size());
        write_npy(c.out + "/w_" + s.name + ".npy", back.data(), back.size());
    }
}

// ----------------------------------------------------------------------------------------------------------------------------------------------
// one graph: schedule, compute, dump
// ----------------------------------------------------------------------------------------------------------------------------------------------
struct graph_run {
    ggml_context * ctx;
    ggml_cgraph * gf;
    std::vector<std::pair<ggml_tensor *, std::string>> inputs;     // graph inputs and how to fill them ("uniform", "normal")
    std::string case_line;                                          // extra JSON members of the case line
};

static graph_run new_run(size_t n_tensors = 256) {
    ggml_init_params ip = { ggml_tensor_overhead() * n_tensors + ggml_graph_overhead(), nullptr, true };
    graph_run r; r.ctx = ggml_init(ip); r.gf = ggml_new_graph(r.ctx);
    return r;
}
static ggml_tensor * input(graph_run & r, ggml_tensor * t, const char * name, const char * fill = "normal") {
    ggml_set_name(t, name); ggml_set_input(t);
    ggml_set_output(t);         // kept until the dump, as the scheduler keeps its input copies (ggml_backend_sched_split_graph)
    r.inputs.push_back({t, fill}); return t;
}
static ggml_tensor * named(ggml_tensor * t, const char * name) { ggml_set_name(t, name); return t; }

static void run_graph(case_ctx & c, graph_run & r, const std::string & tag) {
    const std::string dir = c.out + "/" + tag;
    mkdir(dir.c_str(), 0755);
    ggml_cgraph * gf = r.gf;
    std::map<const ggml_tensor *, bool> supported;
    std::map<const ggml_tensor *, int> node_index;
    std::vector<std::vector<ggml_tensor *>> orig_src(gf->n_nodes);
    for (int i = 0; i < gf->n_nodes; ++i) {
        ggml_set_output(gf->nodes[i]);
        supported[gf->nodes[i]] = ggml_backend_supports_op(c.be, gf->nodes[i]);      // asked before the scheduler rewrites the sources
        node_index[gf->nodes[i]] = i;
        orig_src[i].assign(gf->nodes[i]->src, gf->nodes[i]->src + GGML_MAX_SRC);
    }
    ggml_backend_t backends[2] = { c.be, c.cpu };
    ggml_backend_sched_t sched = ggml_backend_sched_new(backends, nullptr, 2, 4096, false);
    if (!ggml_backend_sched_alloc_graph(sched, gf)) { fprintf(stderr, "%s: ggml_backend_sched_alloc_graph failed\n", tag.c_str()); exit(1); }
    std::normal_distribution<float> nd(0.f, 1.f); std::uniform_real_distribution<float> ud(-1.f, 1.f);
    for (auto & in : r.inputs) {
        std::vector<float> v(ggml_nelements(in.first));
        for (auto & x : v) x = in.second == "normal" ? nd(c.rng) : ud(c.rng);
        ggml_backend_tensor_set(in.first, v.data(), 0, v.size() * sizeof(float));
    }
    if (ggml_backend_sched_graph_compute(sched, gf) != GGML_STATUS_SUCCESS) { fprintf(stderr, "%s: graph compute failed\n", tag.c_str()); exit(1); }
    ggml_backend_sched_synchronize(sched);

    std::map<const ggml_tensor *, std::string> files;
    int n_files = 0;
    auto dump = [&](const ggml_tensor * t) -> std::string {
        auto it = files.find(t);
        if (it != files.end()) return it->second;
        std::string f = "t" + std::to_string(n_files++) + ".npy";
        std::vector<uint8_t> b(ggml_nbytes(t));
        ggml_backend_tensor_get(t, b.data(), 0, b.size());
        write_npy(dir + "/" + f, b.data(), b.size());
        return files[t] = f;
    };
    auto buffer_name = [](const ggml_tensor * t) -> const char * {
        ggml_backend_buffer_t b = t->view_src ? t->view_src->buffer : t->buffer;
        return b ? ggml_backend_buffer_name(b) : "";
    };
    // "name", "type", "ne", "nb", "buffer" of the tensor t a node read, then where its data is: "weight" (w_<name>.npy of the case) or "file", and
    // "node" (the index of the graph node it is, -1 for leaves).  When t is the scheduler's copy of src on the node's backend (same layout, same
    // bytes), the data is dumped from src: the copy is not an output, later nodes may reuse its memory, while src is a node output, an input or a
    // weight, and a view of a weight is read through get_tensor exactly as the copy was filled.
    auto describe = [&](const ggml_tensor * t, const ggml_tensor * src) {
        std::string o = "\"name\":" + json_str(t->name) + ",\"type\":" + json_str(ggml_type_name(t->type)) + ",\"type_id\":" + std::to_string((int)t->type) +
                        ",\"ne\":" + json_i64(t->ne, 4) + ",\"nb\":" + json_i64((const int64_t *)t->nb, 4) + ",\"buffer\":" + json_str(buffer_name(t));
        if (t != src) o += ",\"copy_of\":" + json_str(src->name);
        auto wi = c.w.find(src->name);
        if (wi != c.w.end() && wi->second == src) o += ",\"weight\":" + json_str(src->name);
        else o += ",\"file\":" + json_str(dump(src).c_str());
        auto ni = node_index.find(src);
        return o + ",\"node\":" + std::to_string(ni == node_index.end() ? -1 : ni->second);
    };
    FILE * mf = fopen((dir + "/manifest.jsonl").c_str(), "w");
    fprintf(mf, "{\"kind\":\"case\",\"tag\":%s,\"backend\":%s%s}\n", json_str(tag.c_str()).c_str(), json_str(ggml_backend_name(c.be)).c_str(), r.case_line.c_str());
    for (int i = 0; i < gf->n_nodes; ++i) {
        ggml_tensor * t = gf->nodes[i];
        ggml_backend_t b = ggml_backend_sched_get_tensor_backend(sched, t);
        std::string line = "{\"kind\":\"node\",\"i\":" + std::to_string(i) + ",\"op\":" + json_str(ggml_op_name(t->op)) + "," + describe(t, t) +
                           ",\"backend\":" + json_str(b ? ggml_backend_name(b) : "") + ",\"supported\":" + (supported[t] ? "true" : "false") + ",\"op_params\":[";
        for (int p = 0; p < 4; ++p) line += (p ? "," : "") + std::to_string(t->op_params[p]);
        line += "],\"src\":[";
        for (int j = 0; j < GGML_MAX_SRC; ++j) line += (j ? "," : "") + (t->src[j] ? "{" + describe(t->src[j], orig_src[i][j]) + "}" : std::string("null"));
        fprintf(mf, "%s]}\n", line.c_str());
    }
    fclose(mf);
    ggml_backend_sched_free(sched);
    ggml_free(r.ctx);
    printf("  %-24s %d nodes dumped\n", tag.c_str(), gf->n_nodes);
}

// ----------------------------------------------------------------------------------------------------------------------------------------------
// cases
// ----------------------------------------------------------------------------------------------------------------------------------------------
// Llama layer (llm_build_llama): Q, K, V sharing their input; the attention output projection (the attention itself runs elsewhere, so wo reads the
// Q projection, which has the attention output's shape); the residual; ffn up/gate/SiLU (ggml_fused_up_gate) and ffn_down; the residual; the head.
static void llama_layer(case_ctx & c, int64_t n_embd, const std::vector<int64_t> & ns, const char * prefix) {
    for (int64_t n : ns) {
        graph_run r = new_run();
        ggml_tensor * x = input(r, ggml_new_tensor_2d(r.ctx, GGML_TYPE_F32, n_embd, n), "attn_norm-0");
        ggml_tensor * q = named(ggml_mul_mat(r.ctx, c["attn_q"], x), "Qcur-0");
        ggml_tensor * k = named(ggml_mul_mat(r.ctx, c["attn_k"], x), "Kcur-0");
        ggml_tensor * v = named(ggml_mul_mat(r.ctx, c["attn_v"], x), "Vcur-0");
        ggml_build_forward_expand(r.gf, q); ggml_build_forward_expand(r.gf, k); ggml_build_forward_expand(r.gf, v);
        ggml_tensor * o = named(ggml_mul_mat(r.ctx, c["attn_output"], q), "attn_out-0");
        ggml_tensor * ffn_inp = named(ggml_add(r.ctx, o, x), "ffn_inp-0");
        ggml_tensor * par = named(ggml_fused_up_gate(r.ctx, c["ffn_up"], c["ffn_gate"], ffn_inp, GGML_UNARY_OP_SILU), "ffn_up_gate-0");
        ggml_tensor * down = named(ggml_mul_mat(r.ctx, c["ffn_down"], par), "ffn_down-0");
        ggml_tensor * l_out = named(ggml_add(r.ctx, down, ffn_inp), "l_out-0");
        ggml_tensor * logits = named(ggml_mul_mat(r.ctx, c["output"], l_out), "result_output");
        ggml_build_forward_expand(r.gf, logits);
        run_graph(c, r, std::string(prefix) + "n" + std::to_string(n));
    }
}

static void case_llama(case_ctx & c, bool full_size) {
    // default quantisation mix of the benchmark: IQ4_NL, IQ5_K attn_v, Q5_K ffn_down, Q6_K head
    const int64_t n_embd = full_size ? 4096 : 1024, n_kv = full_size ? 1024 : 256, n_ff = full_size ? 14336 : 2048, n_vocab = full_size ? 4096 : 2000;
    make_weights(c, { {"attn_q", GGML_TYPE_IQ4_NL, n_embd, n_embd, 1}, {"attn_k", GGML_TYPE_IQ4_NL, n_embd, n_kv, 1}, {"attn_v", GGML_TYPE_IQ5_K, n_embd, n_kv, 1},
                      {"attn_output", GGML_TYPE_IQ4_NL, n_embd, n_embd, 1}, {"ffn_up", GGML_TYPE_IQ4_NL, n_embd, n_ff, 1}, {"ffn_gate", GGML_TYPE_IQ4_NL, n_embd, n_ff, 1},
                      {"ffn_down", GGML_TYPE_Q5_K, n_ff, n_embd, 1}, {"output", GGML_TYPE_Q6_K, n_embd, n_vocab, 1} });
    if (full_size) llama_layer(c, n_embd, {1}, "");
    else llama_layer(c, n_embd, {1, 2, 8, 9, 64, 512}, "");
}

// Qwen2 attention projections (llm_build_qwen2): each projection is followed by its bias ADD, so the ADDs sit between the Q, K and V products
static void case_qwen2_bias(case_ctx & c) {
    const int64_t n_embd = 1024, n_kv = 256;
    make_weights(c, { {"attn_q", GGML_TYPE_Q4_K, n_embd, n_embd, 1}, {"attn_k", GGML_TYPE_Q4_K, n_embd, n_kv, 1}, {"attn_v", GGML_TYPE_Q4_K, n_embd, n_kv, 1},
                      {"attn_q.bias", GGML_TYPE_F32, n_embd, 1, 1}, {"attn_k.bias", GGML_TYPE_F32, n_kv, 1, 1}, {"attn_v.bias", GGML_TYPE_F32, n_kv, 1, 1},
                      {"attn_output", GGML_TYPE_Q4_K, n_embd, n_embd, 1} });
    for (int64_t n : {1, 64}) {
        graph_run r = new_run();
        ggml_tensor * x = input(r, ggml_new_tensor_2d(r.ctx, GGML_TYPE_F32, n_embd, n), "attn_norm-0");
        ggml_tensor * q = named(ggml_add(r.ctx, named(ggml_mul_mat(r.ctx, c["attn_q"], x), "Qcur-0"), c["attn_q.bias"]), "Qcur_b-0");
        ggml_build_forward_expand(r.gf, q);
        ggml_tensor * k = named(ggml_add(r.ctx, named(ggml_mul_mat(r.ctx, c["attn_k"], x), "Kcur-0"), c["attn_k.bias"]), "Kcur_b-0");
        ggml_build_forward_expand(r.gf, k);
        ggml_tensor * v = named(ggml_add(r.ctx, named(ggml_mul_mat(r.ctx, c["attn_v"], x), "Vcur-0"), c["attn_v.bias"]), "Vcur_b-0");
        ggml_build_forward_expand(r.gf, v);
        ggml_build_forward_expand(r.gf, named(ggml_mul_mat(r.ctx, c["attn_output"], q), "attn_out-0"));
        run_graph(c, r, "n" + std::to_string(n));
    }
}

// MoE FFN as llm_build_moe_ffn builds it: softmax gating, ggml_top_k (a view of the argsort result: nb1 = n_expert * 4), the routing weights
// (ggml_get_rows of the probabilities), ggml_moe_up_gate on separate up and gate experts, then ggml_mul_mat_id for ffn_down_exps
static void case_moe(case_ctx & c, ggml_type type, int64_t n_expert, int64_t n_used, int64_t n_embd, int64_t n_ff) {
    make_weights(c, { {"ffn_up_exps", type, n_embd, n_ff, n_expert}, {"ffn_gate_exps", type, n_embd, n_ff, n_expert}, {"ffn_down_exps", type, n_ff, n_embd, n_expert} });
    for (int64_t n : {1, 2, 8, 24, 160, 512}) {
        graph_run r = new_run();
        ggml_tensor * cur = input(r, ggml_new_tensor_2d(r.ctx, GGML_TYPE_F32, n_embd, n), "ffn_norm-0");
        ggml_tensor * logits = input(r, ggml_new_tensor_2d(r.ctx, GGML_TYPE_F32, n_expert, n), "ffn_moe_logits-0", "normal");
        ggml_tensor * probs = named(ggml_soft_max(r.ctx, logits), "ffn_moe_probs-0");
        ggml_tensor * selected = named(ggml_top_k(r.ctx, probs, (int)n_used), "ffn_moe_topk-0");
        ggml_tensor * weights = named(ggml_get_rows(r.ctx, ggml_reshape_3d(r.ctx, probs, 1, n_expert, n), selected), "ffn_moe_weights-0");
        ggml_build_forward_expand(r.gf, weights);
        cur = ggml_reshape_3d(r.ctx, cur, n_embd, 1, n);
        ggml_tensor * par = named(ggml_moe_up_gate(r.ctx, c["ffn_up_exps"], c["ffn_gate_exps"], cur, selected, GGML_UNARY_OP_SILU), "ffn_moe_up_gate-0");
        ggml_tensor * experts = named(ggml_mul_mat_id(r.ctx, c["ffn_down_exps"], par, selected), "ffn_moe_down-0");
        ggml_build_forward_expand(r.gf, experts);
        run_graph(c, r, "n" + std::to_string(n));
    }
}

// batched MUL_MAT (attention-style): src0 broadcast over ne2, broadcast over ne3, and one matrix per batch entry
static void case_batched(case_ctx & c) {
    const int64_t k = 512, m = 256;
    make_weights(c, { {"w2d_q4k", GGML_TYPE_Q4_K, k, m, 1}, {"w2d_iq4nl", GGML_TYPE_IQ4_NL, k, m, 1}, {"w3d_iq4nl", GGML_TYPE_IQ4_NL, k, m, 4} });
    for (int64_t n : {3, 64}) {
        graph_run r = new_run();
        ggml_tensor * x2 = input(r, ggml_new_tensor_4d(r.ctx, GGML_TYPE_F32, k, n, 4, 1), "x_ne2");
        ggml_tensor * x3 = input(r, ggml_new_tensor_4d(r.ctx, GGML_TYPE_F32, k, n, 1, 3), "x_ne3");
        ggml_tensor * xe = input(r, ggml_new_tensor_4d(r.ctx, GGML_TYPE_F32, k, n, 4, 1), "x_per_entry");
        ggml_build_forward_expand(r.gf, named(ggml_mul_mat(r.ctx, c["w2d_q4k"], x2), "bcast_ne2"));
        ggml_build_forward_expand(r.gf, named(ggml_mul_mat(r.ctx, c["w2d_iq4nl"], x3), "bcast_ne3"));
        ggml_build_forward_expand(r.gf, named(ggml_mul_mat(r.ctx, c["w3d_iq4nl"], xe), "per_entry"));
        run_graph(c, r, "n" + std::to_string(n));
    }
}

// a row slice [r0, r1) of a weight (ggml_view_2d, as for the parts of a merged tensor): the backend under test declines the product, the scheduler
// runs it on the CPU backend and fetches the view through get_tensor
static void case_weight_view(case_ctx & c) {
    const int64_t k = 512;
    make_weights(c, { {"w_q4k", GGML_TYPE_Q4_K, k, 300, 1}, {"w_iq2xxs", GGML_TYPE_IQ2_XXS, k, 256, 1} });
    struct { const char * w; int64_t r0, r1; const char * name; } views[] = { {"w_q4k", 37, 201, "view_q4k"}, {"w_iq2xxs", 5, 133, "view_iq2xxs"} };
    graph_run r = new_run();
    ggml_tensor * x = input(r, ggml_new_tensor_2d(r.ctx, GGML_TYPE_F32, k, 4), "x");
    r.case_line = ",\"views\":[";
    for (int i = 0; i < 2; ++i) {
        ggml_tensor * w = c[views[i].w];
        ggml_tensor * v = ggml_view_2d(r.ctx, w, k, views[i].r1 - views[i].r0, w->nb[1], views[i].r0 * w->nb[1]);
        ggml_build_forward_expand(r.gf, named(ggml_mul_mat(r.ctx, v, x), views[i].name));
        r.case_line += std::string(i ? "," : "") + "{\"node\":" + json_str(views[i].name) + ",\"weight\":" + json_str(views[i].w) + ",\"r0\":" +
                       std::to_string(views[i].r0) + ",\"r1\":" + std::to_string(views[i].r1) + "}";
    }
    r.case_line += "]";
    run_graph(c, r, "n4");
    // partial uploads in whole rows: rows [r0, r1) replaced through a view (w_q4k) and through an offset into the whole tensor (w_iq2xxs); the
    // tensor read back must be the old wire bytes with those rows replaced.  Writes w_<name>_rows.npy (the new rows) and w_<name>_after.npy.
    ggml_init_params ip = { ggml_tensor_overhead() * 4, nullptr, true };
    ggml_context * vctx = ggml_init(ip);
    for (int i = 0; i < 2; ++i) {
        ggml_tensor * w = c[views[i].w];
        const int64_t nr = views[i].r1 - views[i].r0;
        const size_t rs = w->nb[1];
        std::vector<uint8_t> rows(nr * rs), after(ggml_nbytes(w));
        std::vector<float> f(nr * k), ones(k, 1.0f); std::uniform_real_distribution<float> u(-0.05f, 0.05f);
        for (auto & x : f) x = u(c.rng);
        ggml_quantize_chunk(w->type, f.data(), rows.data(), 0, nr, k, ggml_quantize_requires_imatrix(w->type) ? ones.data() : nullptr, nullptr);
        if (i == 0) ggml_backend_tensor_set(ggml_view_2d(vctx, w, k, nr, rs, views[i].r0 * rs), rows.data(), 0, rows.size());
        else ggml_backend_tensor_set(w, rows.data(), views[i].r0 * rs, rows.size());
        ggml_backend_tensor_get(w, after.data(), 0, after.size());
        write_npy(c.out + "/w_" + views[i].w + "_rows.npy", rows.data(), rows.size());
        write_npy(c.out + "/w_" + views[i].w + "_after.npy", after.data(), after.size());
    }
    ggml_free(vctx);
}

int main(int argc, char ** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s <case> <out_dir>\n", argv[0]); return 2; }
    const std::string name = argv[1];
    case_ctx c;
    c.out = argv[2]; mkdir(c.out.c_str(), 0755);
    uint32_t seed = 2166136261u; for (char ch : name) seed = (seed ^ (uint8_t)ch) * 16777619u;       // fixed per case (FNV-1a of its name)
    c.rng.seed(seed);
    c.be = ggml_backend_cuda_init(0, nullptr, nullptr);
    if (!c.be) { printf("ggml_backend_cuda_init failed (no CUDA device?)\n"); return 2; }
    c.cpu = ggml_backend_cpu_init(); ggml_backend_cpu_set_n_threads(c.cpu, 8);
    printf("%s:\n", name.c_str());
    if (name == "llama") case_llama(c, false);
    else if (name == "llama-8b") case_llama(c, true);
    else if (name == "qwen2-bias") case_qwen2_bias(c);
    else if (name == "moe-qwen3") case_moe(c, GGML_TYPE_Q4_K, 128, 8, 512, 256);
    else if (name == "moe-mixtral") case_moe(c, GGML_TYPE_IQ4_NL, 8, 2, 1024, 512);
    else if (name == "moe-deepseek") case_moe(c, GGML_TYPE_IQ2_XXS, 256, 8, 512, 256);
    else if (name == "batched") case_batched(c);
    else if (name == "weight-view") case_weight_view(c);
    else { fprintf(stderr, "unknown case %s\n", name.c_str()); return 2; }
    ggml_backend_buffer_free(c.wbuf); ggml_free(c.wctx);
    ggml_backend_free(c.be); ggml_backend_free(c.cpu);
    printf("DONE\n");
    return 0;
}
