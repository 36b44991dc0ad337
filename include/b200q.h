/* b200q.h — C ABI of libb200q.so: the Hopper (sm_90a) quantized mat-mul hot path of ik_llama.cpp.
 *
 * Plain C: pointers, sizes, ggml_type ids.  No torch / ggml types.  All device pointers are CUDA device
 * addresses on the current device; `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Every function returns 0 on success, a negative B200Q_E_* code otherwise (b200q_last_error() has the text).
 * There is NO CPU fallback: without a CUDA device every compute entry point fails with B200Q_E_CUDA.
 *
 * What each entry point replaces in the reference (paths relative to the ik_llama.cpp tree):
 *   b200q_set_tensor / b200q_get_tensor    ggml_backend_cuda_buffer_set_tensor / _get_tensor   ggml/src/ggml-cuda.cu:641-672
 *                                          (+ the wire->device re-layout, cf. run-time repack `-rtr`)
 *   b200q_mul_mat                          ggml_cuda_mul_mat dispatcher                        ggml/src/ggml-cuda.cu:2645-2727
 *   b200q_mul_mat_vec[_multi]              quantize_row_q8_1_cuda + ggml_cuda_op_mul_mat_vec_q ggml/src/ggml-cuda.cu:2503-2604,
 *                                          (mul_mat_vec_q / iqk_mul_mat_vec_q kernels)         ggml-cuda/mmvq-templates.cuh:68-150,287-303
 *                                          incl. the "following MUL_MATs share src1" fusion    ggml/src/ggml-cuda.cu:2573-2601
 *   b200q_fused_up_gate_vec                ggml_cuda_up_gate_unary / fused_mul_mat_vec_q       ggml/src/ggml-cuda.cu:3542-3620, mmvq-templates.cuh:152-330
 *   b200q_mul_mat_gemm                     quantize_mmq_q8_1_cuda + mul_mat_q (MMQ)            ggml-cuda/mmq.cuh:3849-4173; dequant+cuBLAS fallback ggml-cuda.cu:1723-1894
 *   b200q_dequantize_bf16                  dequantize_block_* (convert.cu)                     ggml-cuda/convert.cu
 *   b200q_reduce_*                         ggml_cuda_op_reduce                                 ggml-cuda/reduce.cu:125-598
 * Tensor conventions are ggml's: W is [M rows][K cols] in the GGUF wire format of `type`
 * (row stride = ggml_row_size(type, K)); x is f32 [N][K]; dst is f32 [N][M]  (dst[j*M + i]).
 *
 * Memory contract of every compute entry point (tests/test_gpu_memory_contract.py checks it on guarded buffers):
 *   - a call writes only its dst(s), its extra outputs (dst_bf16, the q8 image), and at most the queried or documented workspace bytes;
 *   - W, x, x_bf16, ids, bias and a q8 image passed as input are read-only;
 *   - the result does not depend on what the outputs or the workspace held before the call: every output element is written (never
 *     accumulated into), and one workspace may be reused across calls of any shape;
 *   - an argument, type, shape or workspace error returns before anything is written.  A workspace smaller than the query or the
 *     documented size returns B200Q_E_NOMEM.
 */
#ifndef B200Q_H
#define B200Q_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200Q_ABI_VERSION 1
#if defined(__GNUC__)
#define B200Q_API __attribute__((visibility("default")))
#else
#define B200Q_API
#endif

enum { B200Q_OK = 0, B200Q_E_TYPE = -1, B200Q_E_SHAPE = -2, B200Q_E_CUDA = -3, B200Q_E_ARG = -4, B200Q_E_NOMEM = -5 };
/* unary of GGML_OP_FUSED_UP_GATE.  `limit` (op_params[1]) follows the reference: SILU only, applied AFTER the activation
 * (g = min(silu(g), limit), u = clamp(u, +-limit)), ignored when <= 1e-6 (mmvq-templates.cuh:253-258, unary.cu:63-72).
 * SWIGLU_OAI: alpha 1.702, limit 7, no bias (ggml-cuda.cu:3607-3611). */
enum { B200Q_UNARY_NONE = 0, B200Q_UNARY_SILU = 1, B200Q_UNARY_GELU = 2, B200Q_UNARY_RELU = 3, B200Q_UNARY_SWIGLU_OAI = 4 };

B200Q_API int          b200q_abi_version(void);
B200Q_API const char * b200q_last_error(void);
B200Q_API int          b200q_set_option(const char * key, int value);   /* "pdl": programmatic dependent launch of the decode kernels (cf. the "-cuda k=v" string of ggml_backend_cuda_init, ggml-cuda.cu:5339) */
B200Q_API int          b200q_device_count(void);                      /* ggml_backend_cuda_get_device_count, ggml-cuda.h:38 */

/* ---- type geometry (mirrors ggml_type_traits: ggml/src/ggml.c:640-1460) ---- */
B200Q_API int     b200q_type_supported(int ggml_type);                /* 1 if MUL_MAT with this src0 type is implemented   */
B200Q_API int64_t b200q_wire_row_size(int ggml_type, int64_t k);      /* == ggml_row_size(type, k); <0 on error            */
B200Q_API int64_t b200q_plane_bytes(int ggml_type, int64_t m, int64_t k); /* device bytes of the re-laid-out tensor        */

/* ---- weights: wire <-> device layout ---- */
B200Q_API int b200q_repack  (int type, const void * wire_dev,   void * planes_dev, int64_t m, int64_t k, void * stream);
B200Q_API int b200q_unrepack(int type, const void * planes_dev, void * wire_dev,   int64_t m, int64_t k, void * stream);
B200Q_API int b200q_set_tensor(int type, const void * wire_host, void * planes_dev, int64_t m, int64_t k, void * stream); /* H2D + repack, synchronous */
B200Q_API int b200q_get_tensor(int type, const void * planes_dev, void * wire_host, int64_t m, int64_t k, void * stream); /* unrepack + D2H, synchronous */

/* ---- decode: n <= 8 activation columns ---- */
B200Q_API int b200q_mul_mat_vec(int type, const void * W, const float * x, float * dst,
                      int64_t m, int64_t k, int n, int64_t x_stride, const float * bias, void * stream);
/* several weight tensors of the same type and K sharing one activation (Q,K,V): one launch */
B200Q_API int b200q_mul_mat_vec_multi(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m,
                            int64_t k, const float * x, int n, int64_t x_stride, void * stream);
/* dst = unary(gate.x) * (up.x)   (optionally clamped: limit > 0) */
B200Q_API int b200q_fused_up_gate_vec(int type, const void * W_up, const void * W_gate, const float * x, float * dst,
                            int64_t m, int64_t k, int n, int64_t x_stride, int unary, float limit, void * stream);

/* q8_1 hand-off FUSED_UP_GATE -> MUL_MAT(ffn_down) for n = 1 (the reference quantises each activation once, quantize_row_q8_1_cuda in
 * ggml_cuda_op_mul_mat_vec_q, ggml-cuda.cu:2503-2604; here the producer's epilogue does it): `q8` is a device scratch of
 * b200q_q8_scratch_bytes(m_of_up_gate) bytes, zeroed ONCE with b200q_q8_scratch_init.  *q8_produced = 1 if the launch emitted the image
 * (eligible shape and kernel); pass q8_in = NULL to b200q_mul_mat_vec_q8 otherwise.  x / dst are always read / written as usual. */
B200Q_API size_t b200q_q8_scratch_bytes(int64_t k);
B200Q_API int b200q_q8_scratch_init(void * q8, int64_t k, void * stream);
B200Q_API int b200q_fused_up_gate_vec_q8(int type, const void * W_up, const void * W_gate, const float * x, float * dst, int64_t m, int64_t k,
                               int unary, float limit, void * q8_out, int * q8_produced, void * stream);
B200Q_API int b200q_mul_mat_vec_q8(int type, const void * W, const float * x, const void * q8_in, float * dst, int64_t m, int64_t k,
                         const float * bias, void * stream);

/* Decode chains: tell the NEXT decode launch of this thread which weights the launch AFTER it will stream, so that it can warm their first
 * stages in L2 (cp.async.bulk.prefetch.L2) while it runs; a kernel cannot prefetch into shared memory before the previous one has left the SM.
 * The hint is consumed (cleared) by the next b200q_mul_mat_vec* / b200q_fused_up_gate_vec* call.  W_gate != NULL: fused up/gate (n_tensors = 1). */
B200Q_API int b200q_decode_prefetch_next(int type, int n_tensors, const void * const * W, const void * W_gate, const int64_t * m, int64_t k);

/* ---- prefill: wgmma GEMM ---- */
B200Q_API size_t b200q_mul_mat_workspace(int type, int64_t m, int64_t k, int64_t n);
B200Q_API int b200q_mul_mat_gemm(int type, const void * W, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                       void * workspace, size_t workspace_bytes, void * stream);
/* activations shared by several mat-muls (Q,K,V / up,gate): convert once, then call the _bf16 variant per weight tensor.  A workspace of
 * b200q_mul_mat_workspace (b200q_mul_mat_multi_workspace for _multi_bf16) bytes is always enough for it. */
B200Q_API int b200q_convert_f32_bf16(const float * x, int64_t x_stride, void * out_bf16, int64_t k, int64_t n, void * stream);
B200Q_API int b200q_mul_mat_gemm_bf16(int type, const void * W, const void * x_bf16, float * dst, int64_t m, int64_t k, int64_t n,
                            void * workspace /* bf16 [m][k] scratch, only for types without a fused kernel */, size_t workspace_bytes, void * stream);
B200Q_API int b200q_dequantize_bf16(int type, const void * W, void * out_bf16, int64_t m, int64_t k, void * stream);
/* several MUL_MATs of one type / K that share src1, n > 8 (the look-ahead fusion of ggml_cuda_mul_mat_q, ggml-cuda.cu:2573-2601):
 * ONE launch walks the row tiles of up to 3 tensors (Q,K,V) */
B200Q_API int b200q_mul_mat_gemm_multi_bf16(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m, int64_t k,
                                  const void * x_bf16, int64_t n, void * workspace, size_t workspace_bytes, void * stream);
/* GGML_OP_FUSED_UP_GATE for n > 8 (ggml_cuda_up_gate_unary, ggml-cuda.cu:3588-3618: two MMQ + ggml_fused_mul_unary): up and gate
 * are the two segments of one GEMM launch, followed by one elementwise unary-mul pass; dst_bf16 (optional, may be NULL) receives a
 * bf16 copy = the operand of ffn_down.
 * workspace >= align256(m*n*4) (the up result) + align256(m*k*2) (the bf16 weight scratch, only for types without a fused kernel);
 * b200q_fused_up_gate_workspace bytes are always enough */
B200Q_API int b200q_fused_up_gate_gemm_bf16(int type, const void * W_up, const void * W_gate, const void * x_bf16, float * dst, void * dst_bf16,
                                  int64_t m, int64_t k, int64_t n, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream);

/* ---- GGML_OP_REDUCE (sum) for the row-parallel mat-muls of split-mode-graph: NVLS all-reduce in ONE kernel ----
 * One process per GPU; the reduction buffers live in symmetric memory: `mc_base` / `mc_flag` = multicast (NVLS) addresses,
 * `local_base` / `local_flag` = this rank's own mapping of the same allocation.  Two parity buffers of `parity_stride` floats
 * alternate (base + parity*stride); the parity and the flag target come from the device counter `seq_counter` (rank-local,
 * zero-initialised), so the call has constant arguments and can be captured in a CUDA graph.  `seq_counter` points at FOUR u32
 * {reduces done, dirty floats of parity buffer 0, of parity buffer 1, pad}, zero-initialised.  `cta_counter`: rank-local u32, zero. */
B200Q_API int b200q_reduce_sum_nvls(const float * in, float * out, int64_t n, void * mc_base, void * local_base, int64_t parity_stride,
                          void * mc_flag, const void * local_flag, uint32_t world_size, void * seq_counter, void * cta_counter, void * stream);

/* Prefill-sized REDUCE: two-shot bf16 all-reduce in ONE kernel (the reference casts the partial to bf16/f16 when ne[1] > 32,
 * src/llama-build-context.cpp:1198-1200, and runs reduce-scatter + all-gather, ggml-cuda/reduce.cu:306-372): f32 partial -> bf16 staging in
 * symmetric memory, barrier, multimem.ld_reduce of the rank's 1/world slice (f32 accumulation in the switch) + multimem.st of the sum to every
 * rank, barrier, copy-out as bf16 (out_bf16: the activation operand of the next GEMM) and / or f32 (out_f32).  `state`: rank-local u32[4], zero. */
typedef struct b200q_nvls_stage {
    void * mc_stage; void * local_stage; int64_t stage_elems;   /* bf16 staging buffer: multicast address / this rank's mapping / capacity in elements */
    void * mc_flag; const void * local_flag;                    /* u32 flag word in symmetric memory (multicast / local), zero-initialised */
    uint32_t world_size; uint32_t rank;
    void * state;
} b200q_nvls_stage;
B200Q_API int b200q_reduce_sum_nvls_bf16(const float * in, float * out_f32, void * out_bf16, int64_t n, const b200q_nvls_stage * stage, void * stream);

/* ---- tensor-parallel decode (n = 1): the GGML_OP_REDUCE after a row-parallel mat-vec fused INTO the mat-vec kernels ----
 * (reference: ggml_cuda_op_reduce runs as its own node after wo / ffn_down under -sm graph, ggml-cuda/reduce.cu:125-598).
 * Tagged-slot exchange, no flag, no fence, no acknowledgement round trip: an entry is {f32 value, u32 number of the reduce}, written with one
 * 8-byte store.  reduce_out: the kernel's epilogue broadcasts each finished partial row to slot [parity][this rank][row] of EVERY rank with
 * multimem.st through the NVLS multicast mapping (dst is not written; m_total <= ll_stride).  reduce_in: `x` is ignored; the CTAs of the consumer
 * sum the per-rank slots in rank order (bit-identical on every rank), each its own slice, publish the sums in ll_reduced with the same tagging and
 * quantise their activations from there (k <= ll_stride).  W_gate != NULL: fused up/gate mode (n_tensors = 1), reduce_in only: a fused up/gate
 * launch with reduce_out returns B200Q_E_ARG (the sum over ranks of unary(gate . x) * (up . x) is not a result of anything).
 * CONTRACT: on one communicator every reduce_out launch must be followed, on every rank, by at least one reduce_in launch before the next
 * reduce_out (the two parities are reused every second reduce); all ranks issue the same sequence.
 * Launches with reduce_in or reduce_out run on the ring kernel only, so they are accepted exactly when a plain n = 1 b200q_mul_mat_vec /
 * _multi / b200q_fused_up_gate_vec of the same tensors is planned on the ring kernel and:
 *   - type is a plane-layout type: a wire-layout type returns B200Q_E_TYPE;
 *   - k % 256 == 0, m_total = sum of m <= ll_stride for reduce_out, k <= ll_stride for reduce_in: otherwise B200Q_E_SHAPE;
 *   - the type has a ring geometry at this k (every plane row 16-byte aligned, e.g. Q6_K needs k % 2048 == 0), and on row pairs (k <= 4096)
 *     every tensor but the last has an even m: otherwise B200Q_E_SHAPE.
 * A rejected call writes nothing.
 *   ll_mc / ll_local: multicast / local address of the symmetric slot array, 2 * world_size * ll_stride entries of 8 bytes, zero-initialised.
 *   ll_mc may be NULL only when the unicast stores are selected (B200Q_TP_UNICAST=1 and ll_peers given); otherwise NULL is B200Q_E_ARG;
 *   ll_reduced: rank-local, 2 * ll_stride entries, zero-initialised; ll_state: rank-local u32[2], zero-initialised; all 16-byte aligned. */
typedef struct b200q_nvls_comm {
    void * ll_mc; const void * ll_local; void * ll_reduced; int64_t ll_stride; uint32_t world_size; uint32_t rank; void * ll_state;
    void * const * ll_peers;    /* optional (HOST array of world_size device pointers, world_size <= 8): every rank's mapping of the slot array in THIS
                                 * rank's address space (peer memory).  When given and B200Q_TP_UNICAST=1 (opt-in, read once per process),
                                 * reduce_out writes each peer's copy with ordinary stores, the rows of
                                 * a CTA as consecutive 16-byte lanes of one warp (coalesced into 128-byte NVLink packets), instead of one multicast
                                 * store per row pair.  NULL: multimem.st only. */
} b200q_nvls_comm;
B200Q_API int b200q_mul_mat_vec_tp(int type, int n_tensors, const void * const * W, const void * W_gate, float * const * dst, const int64_t * m,
                         int64_t k, const float * x, int unary, float limit, const b200q_nvls_comm * comm, int reduce_in, int reduce_out, void * stream);

/* ---- dispatcher (what GGML_OP_MUL_MAT calls): n <= 8 -> mat-vec, else GEMM ---- */
B200Q_API int b200q_mul_mat(int type, const void * W, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                  void * workspace, size_t workspace_bytes, void * stream);
/* any-n variants of the multi-tensor and fused up/gate ops with f32 activations (what the graph nodes carry) */
B200Q_API size_t b200q_mul_mat_multi_workspace(int type, int n_tensors, const int64_t * m, int64_t k, int64_t n);
B200Q_API int b200q_mul_mat_multi(int type, int n_tensors, const void * const * W, float * const * dst, const int64_t * m, int64_t k,
                        const float * x, int64_t n, void * workspace, size_t workspace_bytes, void * stream);
B200Q_API size_t b200q_fused_up_gate_workspace(int type, int64_t m, int64_t k, int64_t n);
B200Q_API int b200q_fused_up_gate(int type, const void * W_up, const void * W_gate, const float * x, float * dst, int64_t m, int64_t k, int64_t n,
                        int unary, float limit, void * workspace, size_t workspace_bytes, void * stream);
/* GGML_OP_ADD of a mat-mul result with its bias row(s): dst[j][i] = a[j][i] + b[j % nb][i] (i < m, j < n) */
B200Q_API int b200q_add_rows(const float * a, const float * b, float * dst, int64_t m, int64_t n, int64_t nb, void * stream);
/* ---- MoE decode: GGML_OP_MUL_MAT_ID / GGML_OP_MOE_FUSED_UP_GATE for small batches (ggml_cuda_mul_mat_id / ggml_cuda_moe_up_gate_unary,
 * ggml-cuda.cu:2836-3540; mul_mat_vec_q with ids, mmvq-templates.cuh:293-302).  W: n_expert matrices [m x k] of `type`, each in the device layout,
 * b200q_plane_bytes(type, m, k) apart; ids: DEVICE int32 [n_tokens][n_used]; x f32 [n_tokens][nb1][k] (nb1 = 1: the column is shared by the slots of
 * a token, nb1 = n_used: one column per slot); dst f32 [n_tokens][n_used][m]:  dst[t][e] = W[ids[t][e]] . x[t][e % nb1]
 * (W_gate != NULL: unary(W_gate[id] . x) * (W[id] . x)); ids outside [0, n_expert) give zero rows, as in the reference.  Expert ids are resolved on the device.  The quantised activation columns of a launch live
 * in shared memory (200 KB of q8_1): batches whose n_tokens * nb1 columns exceed that are walked in token chunks by the same kernel. */
B200Q_API int b200q_mul_mat_id_vec(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                         int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * stream);
/* ---- MoE prefill: grouped wgmma GEMM over expert-sorted slots (the reference's mmq_id path, ggml-cuda.cu:2906-2910, 3210-3267) ----
 * Same arguments and result as b200q_mul_mat_id_vec, plus a device workspace.  Routing (counts, sort by expert, tile table) runs on the device: no
 * host round trip, no allocation, no synchronisation, so the call can be captured in a CUDA graph.  Ids outside [0, n_expert) are skipped and their
 * dst rows are ZERO (the reference's semantics, as in b200q_mul_mat_id_vec).  bf16 operands, f32 accumulation (as the dense GEMM).
 * b200q_mul_mat_id_gemm_workspace: bytes b200q_mul_mat_id_gemm needs at any batch size, 0 only for a shape the grouped path refuses.  Needs no device.
 * b200q_mul_mat_id_workspace: the same bytes where b200q_mul_mat_id takes the grouped path, 0 exactly when it takes the mat-vec path: an ineligible
 * shape, or a batch below the measured crossover (n_slots = n_tokens * n_used; up/gate: n_slots <= 5 * n_expert, else n_slots <= 32).  Needs no device.
 * b200q_mul_mat_id_gemm: always the grouped path (K % 256 == 0, n_expert <= 1024).  b200q_mul_mat_id: the dispatcher (workspace may be NULL when the
 * query returned 0). */
B200Q_API size_t b200q_mul_mat_id_gemm_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert, int up_gate);
B200Q_API size_t b200q_mul_mat_id_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert, int up_gate);
B200Q_API int b200q_mul_mat_id_gemm(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                          int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream);
B200Q_API int b200q_mul_mat_id(int type, const void * W, const void * W_gate, int n_expert, const int32_t * ids, const float * x, float * dst,
                     int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream);
/* ---- MoE with merged up/gate experts: GGML_OP_MOE_FUSED_UP_GATE with src[0] = ffn_gate_up_exps [k, 2 m, n_expert], src[1] = NULL, no biases ----
 * (ggml_moe_up_gate(ctx, up_gate_exps, NULL, ...), the reference CPU op iqk_moe_fused_up_gate: ggml.c:18620-18632).  W_gate_up: n_expert matrices
 * [2 m x k] of `type` in the device layout, b200q_plane_bytes(type, 2 m, k) apart (each uploaded whole with b200q_set_tensor); rows [0, m) of a matrix
 * are the GATE rows, rows [m, 2 m) the UP rows:  dst[t][e][i] = unary(gate_i(id) . x) * (up_i(id) . x), id = ids[t][e], with the unary / limit rules
 * and the ids, x, dst conventions of b200q_mul_mat_id (ids outside [0, n_expert) give zero rows).  Shape conditions: k a multiple of the type's block
 * (of 256 for the grouped GEMM, else the mat-vec serves every batch); for the types whose rows are interleaved in groups of 4 (_R4), m % 4 == 0.
 * Same arithmetic, launches and crossover as b200q_mul_mat_id on the two halves uploaded as separate tensors.
 * b200q_moe_up_gate_merged_workspace: bytes of device workspace, 0 exactly when b200q_moe_up_gate_merged takes the mat-vec path (then workspace may
 * be NULL); needs no device.  b200q_moe_up_gate_merged: the dispatcher; no host round trip, allocation or synchronisation (capturable). */
B200Q_API size_t b200q_moe_up_gate_merged_workspace(int type, int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int n_expert);
B200Q_API int b200q_moe_up_gate_merged(int type, const void * W_gate_up, int n_expert, const int32_t * ids, const float * x, float * dst,
                             int64_t m, int64_t k, int n_used, int nb1, int n_tokens, int unary, float limit, void * workspace, size_t workspace_bytes, void * stream);
/* ---- MoE combine: GGML_OP_MUL_MULTI_ADD without the scales form (src[2] / src[3]) ----
 * (the last node of llm_build_moe_ffn under fused_mmad, src/llama-build-context.cpp:1667-1680; CPU iqk_mul_multi_add, iqk_cpu_ops.cpp:430-495;
 * CUDA ggml-cuda/multiadd.cu:40-62).  rows f32 [n_tokens][n_used][m] (the MUL_MAT_ID result of ffn_down_exps), weights f32 [n_tokens][n_used] (the
 * routing weights), dst f32 [n_tokens][m]:  dst[t][i] = sum_u weights[t][u] * rows[t][u][i], summed in slot order as the CPU op (y = x0 w0, then
 * y = y + x_u w_u) with every product and sum rounded on its own: bit-equal to that loop in f32.  Under tensor parallelism, a rank's rows are its
 * K-shard of ffn_down_exps and dst is the rank's partial of the layer, summed across ranks by the caller's reduce.  Slots of ids outside the expert
 * range need no care: MUL_MAT_ID gives them zero rows.  All pointers 4-byte aligned; dst must not overlap rows or weights (B200Q_E_ARG).
 * Writes only dst; no workspace, allocation or synchronisation (capturable). */
B200Q_API int b200q_moe_combine(const float * rows, const float * weights, float * dst, int64_t m, int n_used, int n_tokens, void * stream);
/* ---- batched MUL_MAT: GGML_OP_MUL_MAT with ne[2] * ne[3] > 1, over strided activations, in one launch sequence ----
 * (the per-head products of absorbed MLA, q_nope2 = wk_b x q_nope_perm and kqv = wv_b x kqv_compressed_perm, src/graphs/build_deepseek2.cpp:1030-1036,
 * 1145-1162; the weights are Q8_0 [k, m, n_head] made by llm_prepare_mla, src/llama.cpp:3014, 3054)
 *     dst[b][j][i] = W_b[i] . x[b * x_batch_stride + j * x_col_stride + 0 .. k)      b < n_batch, j < n, i < m
 * W_b = W (per_entry = 0: one matrix broadcast over the batch) or W + b * b200q_plane_bytes(type, m, k) (per_entry = 1: n_batch matrices, each uploaded
 * with b200q_set_tensor); strides in floats; dst f32 contiguous [n_batch][n][m] (ggml's dst of a batched MUL_MAT).
 * Conditions: x 16-byte aligned; both strides non-negative multiples of 4 floats, x_col_stride >= k when n > 1 and x_batch_stride >= k when n_batch > 1
 * (otherwise B200Q_E_ARG); k a multiple of the type's block and n * n_batch <= INT32_MAX (otherwise B200Q_E_SHAPE); workspace 256-byte aligned.
 * It runs the MoE kernels with identity routing (ids[b][j] = b, or 0 when broadcast, written into the workspace): the grouped MoE GEMM where it is
 * eligible (k % 256 == 0, n_batch <= 1024) from 128 slots (n_batch * n) on, for types without a fused GEMM kernel only from n = 2 on; otherwise the
 * MoE mat-vec kernel up to n = 16 (one launch, or entry chunks when the n_batch * n quantised columns exceed shared memory), one GEMM per entry
 * above.  A broadcast W over columns a constant stride apart is one 2-D product.
 * b200q_mul_mat_batched_workspace: the bytes the call needs (0 for a 2-D product with n * n_batch <= 8, and for any rejected argument); needs no device.
 * No host round trip, allocation or synchronisation: the call can be captured in a CUDA graph. */
B200Q_API size_t b200q_mul_mat_batched_workspace(int type, int64_t m, int64_t k, int64_t n, int n_batch, int per_entry,
                                                 int64_t x_col_stride, int64_t x_batch_stride);
B200Q_API int b200q_mul_mat_batched(int type, const void * W, int per_entry, const float * x, int64_t x_col_stride, int64_t x_batch_stride,
                                    float * dst, int64_t m, int64_t k, int64_t n, int n_batch, void * workspace, size_t workspace_bytes, void * stream);
/* ---- MUL_MAT over a row slice of a weight, over f32 or f16 activations a column stride apart ----
 * (the "pp_opt" prompt processing of DeepSeek's MLA: kv_f32 = wkv_b_iter x kv_cache_nope, src/graphs/build_deepseek2.cpp:922-1022, where wkv_b_iter is a
 * view of whole rows of wkv_b and kv_cache_nope a view of the f16 K cache, 576 halves per column starting 64 halves in)
 *     dst[j][i] = W_row(row0 + i) . x[j * x_col_stride + 0 .. k)      i < m, j < n;  dst f32 contiguous [n][m]
 * W is the base of the WHOLE tensor [rows_layout x k], uploaded with b200q_set_tensor (never a wire-byte offset into it); x_type is the ggml_type of x,
 * GGML_TYPE_F32 (0) or GGML_TYPE_F16 (1); x_col_stride is in elements.
 * Conditions:
 *   - 0 <= row0, row0 + m <= rows_layout, n >= 1; x_col_stride a non-negative multiple of 16 bytes, at least k when n > 1 (otherwise B200Q_E_ARG);
 *   - every plane pointer of the slice keeps the 256-byte alignment of a whole tensor's: row0 * (bytes per row of plane p) % 256 == 0 for every plane p
 *     (a wire-layout type: row0 * wire row bytes % 256 == 0), and for the types whose rows are interleaved in groups of 4 (_R4) row0 % 4 == m % 4 == 0;
 *     k a multiple of the type's block (otherwise B200Q_E_SHAPE);  an unsupported weight type or x_type: B200Q_E_TYPE;
 *   - x 16-byte aligned, workspace 256-byte aligned (B200Q_E_ARG).
 * Result: the launches of b200q_mul_mat on the rows [row0, row0 + m) uploaded as a tensor of their own, with the same bits (except launches that split
 * K, whose f32 atomics may differ in the last bits from run to run); an f16 x gives the bits of an f32 x holding float(x).  The one extra launch for an
 * f16 x converts it once: f16 -> f32 before a mat-vec (n <= 8) or the IQ2_BN int8 GEMM, f16 -> bf16 in place of f32 -> bf16 before every other GEMM.
 * b200q_mul_mat_rows_ok: 0 or the B200Q_E_* the call would return for these arguments (before the pointer checks); needs no device.
 * b200q_mul_mat_rows_workspace: the bytes the call needs (0 for a rejected argument, and for f32 x with n <= 8); needs no device.
 * No host round trip, allocation or synchronisation: the call can be captured in a CUDA graph. */
B200Q_API int    b200q_mul_mat_rows_ok(int type, int64_t rows_layout, int64_t row0, int64_t m, int64_t k, int64_t n, int x_type, int64_t x_col_stride);
B200Q_API size_t b200q_mul_mat_rows_workspace(int type, int64_t rows_layout, int64_t row0, int64_t m, int64_t k, int64_t n, int x_type, int64_t x_col_stride);
B200Q_API int    b200q_mul_mat_rows(int type, const void * W, int64_t rows_layout, int64_t row0, int x_type, const void * x, int64_t x_col_stride,
                                    float * dst, int64_t m, int64_t k, int64_t n, void * workspace, size_t workspace_bytes, void * stream);
/* same through HOST activations/results: H2D(x) -> mul_mat -> D2H(dst), synchronous (end-to-end entry point) */
B200Q_API int b200q_mul_mat_host(int type, const void * W_planes_dev, const float * x_host, float * dst_host,
                       int64_t m, int64_t k, int64_t n, void * stream);

#ifdef __cplusplus
}
#endif
#endif /* B200Q_H */
