"""Tensor-parallel ("split mode graph") host logic for the quantized mat-mul path.

Mirrors the reference's sharding of MUL_MAT weights (src/llama-load-tensors.cpp:395-440 create_split,
:4647-4705 prepare_split_tensors, :5452-5477 attention/FFN policy; scatter in ggml_backend_cuda_split_buffer_set_tensor,
ggml/src/ggml-cuda.cu:1003-1192):
  * split_dim = 1 (rows of W: wq/wk/wv/ffn_up/ffn_gate/output): shard = contiguous row range, no exchange;
  * split_dim = 0 (columns/K of W: wo/ffn_down): shard = K range (multiple of the granularity, >= quant block) of EVERY row,
    partial outputs are summed across ranks (GGML_OP_REDUCE, ggml-cuda/reduce.cu:125);
  * per-row headers (row_meta_size: IQ4_KS, IQ2_BN, ...) are replicated into every K-shard;
  * MoE experts (src/llama-load-tensors.cpp:5637-5675): one n_ff split for the three expert tensors, rows of every ffn_up_exps / ffn_gate_exps
    matrix (merged ffn_gate_up_exps: the gate rows and the up rows of the same range), the K range of every ffn_down_exps matrix; each rank's
    routed-expert partial is backend.moe_tp_partial.
Pure numpy: usable in CPU tests with the oracle as the compute stand-in, and by bench.py / the backend for real shards.
"""
from __future__ import annotations

import numpy as np

# (block elements, block bytes, row meta bytes) — ggml type traits (ggml/src/ggml.c:640-1460)
GEOM = {2: (32, 18, 0), 3: (32, 20, 0), 6: (32, 22, 0), 7: (32, 24, 0), 133: (32, 26, 0), 8: (32, 34, 0), 12: (256, 144, 0), 13: (256, 176, 0), 14: (256, 210, 0), 20: (32, 18, 0), 23: (256, 136, 0),
        135: (64, 16, 4), 139: (256, 144, 0), 140: (256, 176, 0), 144: (256, 136, 4),
        10: (256, 84, 0), 11: (256, 110, 0), 137: (256, 76, 0), 138: (256, 110, 0), 39: (32, 17, 0), 152: (256, 168, 4), 145: (256, 70, 2), 156: (256, 102, 2),
        # wire-layout types (ik_llama_cpp_b200/csrc/b200q_wire.cuh)
        16: (256, 66, 0), 17: (256, 74, 0), 18: (256, 98, 0), 22: (256, 82, 0), 21: (256, 110, 0), 19: (256, 50, 0), 29: (256, 56, 0), 141: (256, 212, 0), 146: (256, 128, 4),
        157: (256, 86, 2), 134: (64, 13, 2), 158: (256, 56, 4), 153: (256, 68, 4), 154: (256, 100, 4), 155: (256, 128, 4),
        219: (32, 6, 2), 229: (32, 7, 2), 337: (256, 76, 0), 338: (256, 110, 0), 339: (256, 144, 0), 340: (256, 176, 0), 344: (256, 136, 4), 352: (256, 168, 4)}
# rows interleaved on the wire (the _R4 repacks): a wire "row group" of 4 rows = {4 row headers}{blocks of 4 rows}
INTERLEAVE = {219: 4, 229: 4, 337: 4, 338: 4, 339: 4, 340: 4, 344: 4, 352: 4}


def create_split(nr: int, granularity: int, world: int) -> list[int]:
    """Even split of `nr` in units of `granularity` (reference create_split with uniform `splits` and equal memory use):
    chunks are handed out round(p*nchunk) per device, the remainder goes to the first devices."""
    if granularity < 0:
        return [nr] * world
    assert nr % granularity == 0, (nr, granularity)
    nchunk = nr // granularity
    base, rem = divmod(nchunk, world)
    return [(base + (1 if i < rem else 0)) * granularity for i in range(world)]


def row_size(ggml_type: int, k: int) -> int:
    qk, bs, meta = GEOM[ggml_type]
    assert k % qk == 0
    return meta + (k // qk) * bs


def shard_rows(wire: np.ndarray, ggml_type: int, m: int, k: int, world: int, rank: int, granularity: int = 1):
    """split_dim = 1: rows [r0, r1) of the wire tensor.  Returns (shard_bytes, m_shard)."""
    granularity = max(granularity, INTERLEAVE.get(ggml_type, 1)) if granularity > 0 else granularity
    sizes = create_split(m, granularity, world)
    r0 = sum(sizes[:rank])
    rs = row_size(ggml_type, k)
    w = np.ascontiguousarray(wire, np.uint8).reshape(m, rs)
    return np.ascontiguousarray(w[r0:r0 + sizes[rank]]).reshape(-1), sizes[rank]


def shard_cols(wire: np.ndarray, ggml_type: int, m: int, k: int, world: int, rank: int, granularity: int | None = None):
    """split_dim = 0: K range [k0, k1) of every row (granularity >= quant block), row header replicated.
    Returns (shard_bytes, k_shard, k0)."""
    qk, bs, meta = GEOM[ggml_type]
    g = max(qk, granularity or qk)
    assert g % qk == 0
    sizes = create_split(k, g, world)
    k0 = sum(sizes[:rank]); ks = sizes[rank]
    rs = row_size(ggml_type, k)
    il = INTERLEAVE.get(ggml_type, 1)                 # row groups: the K range of a group of `il` interleaved rows is contiguous on the wire
    assert m % il == 0
    w = np.ascontiguousarray(wire, np.uint8).reshape(m // il, il * rs)
    out = np.empty((m // il, il * (meta + (ks // qk) * bs)), np.uint8)
    out[:, :il * meta] = w[:, :il * meta]
    out[:, il * meta:] = w[:, il * (meta + (k0 // qk) * bs): il * (meta + ((k0 + ks) // qk) * bs)]
    return out.reshape(-1), ks, k0


def moe_expert_granularity(down_type: int) -> int:
    """Unit of the routed experts' n_ff split: 16, or the block size of ffn_down_exps' type if larger (src/llama-load-tensors.cpp:5643-5648)."""
    return max(16, GEOM[down_type][0])


def moe_ffn_plan(n_ff_exp: int, world: int, down_type: int) -> list[int]:
    """n_ff shard of the routed experts on each rank: rows of ffn_up_exps / ffn_gate_exps, the K range of ffn_down_exps (one split serves all
    three, src/llama-load-tensors.cpp:5637-5675).  A rank may get 0 (Qwen3-30B-A3B: 768 = 3 x 256 over 8 ranks).  The reference skips such a
    device; here every rank still joins the reduce, with a zero partial.  The reference also weighs each device's memory already in use
    (create_split's mem_used); this plan assumes equal use and keeps create_split's rule above."""
    return create_split(n_ff_exp, moe_expert_granularity(down_type), world)


def _expert_rows(wire: np.ndarray, ggml_type: int, n_expert: int, m: int, k: int, ranges) -> np.ndarray:
    """the rows [a, b) of each range, in order, of every expert matrix [m x k] (whole wire rows; for _R4 types a, b are multiples of 4)"""
    il = INTERLEAVE.get(ggml_type, 1)
    assert all(a % il == 0 and b % il == 0 for a, b in ranges)
    w = np.ascontiguousarray(wire, np.uint8).reshape(n_expert, m, row_size(ggml_type, k))
    return np.ascontiguousarray(np.concatenate([w[:, a:b] for a, b in ranges], axis=1)).reshape(-1)


def shard_expert_rows(wire: np.ndarray, ggml_type: int, n_expert: int, n_ff: int, k: int, split: list[int], rank: int):
    """ffn_up_exps / ffn_gate_exps [n_expert][n_ff x k] (split_dim 1): rows [r0, r1) of every expert.  Returns (shard_bytes, n_ff_shard)."""
    r0 = sum(split[:rank]); n = split[rank]
    return _expert_rows(wire, ggml_type, n_expert, n_ff, k, [(r0, r0 + n)]), n


def shard_expert_gate_up(wire: np.ndarray, ggml_type: int, n_expert: int, n_ff: int, k: int, split: list[int], rank: int):
    """ffn_gate_up_exps [n_expert][2 n_ff x k], gate rows first: gate rows [r0, r1) then up rows [n_ff + r0, n_ff + r1) of every expert
    (prepare_up_gate_split, src/llama-load-tensors.cpp:4851-4867), again a merged [2 n_ff_shard x k] matrix per expert.
    Returns (shard_bytes, n_ff_shard)."""
    r0 = sum(split[:rank]); n = split[rank]
    return _expert_rows(wire, ggml_type, n_expert, 2 * n_ff, k, [(r0, r0 + n), (n_ff + r0, n_ff + r0 + n)]), n


def shard_expert_cols(wire: np.ndarray, ggml_type: int, n_expert: int, m: int, n_ff: int, split: list[int], rank: int):
    """ffn_down_exps [n_expert][m x n_ff] (split_dim 0): the K range [k0, k1) of every row of every expert, row headers replicated (as
    shard_cols on the n_expert * m rows).  `split` is moe_ffn_plan's for this type.  Returns (shard_bytes, k_shard, k0)."""
    out, ks, k0 = shard_cols(wire, ggml_type, n_expert * m, n_ff, len(split), rank, granularity=moe_expert_granularity(ggml_type))
    assert (ks, k0) == (split[rank], sum(split[:rank])), "ffn_down_exps follows its own type's plan"
    return out, ks, k0


def llama_layer_plan(n_embd: int, n_ff: int, n_head: int, n_head_kv: int, world: int, ggml_type: int):
    """Shard sizes of one Llama layer under -sm graph (src/llama-load-tensors.cpp:5452-5477, :5619-5633)."""
    head_dim = n_embd // n_head
    gqa = n_head // n_head_kv
    qk = GEOM[ggml_type][0]
    gran_kq = head_dim * gqa                       # wq rows per KV-head group
    gran_vo = max(head_dim * gqa, qk)              # wo columns
    q_rows = create_split(n_embd, gran_kq, world)
    kv_rows = [r // gqa for r in q_rows]
    o_cols = create_split(n_embd, gran_vo, world)
    ff = create_split(n_ff, max(qk, 1), world)     # ffn_up/gate rows == ffn_down columns
    return {"wq_rows": q_rows, "wkv_rows": kv_rows, "wo_cols": o_cols, "ffn_rows": ff, "ffn_down_cols": ff}
