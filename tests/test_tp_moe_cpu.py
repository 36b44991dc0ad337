"""CPU tests of the tensor-parallel MoE host logic (ik_llama_cpp_b200/tp.py): the expert shards of every form reassemble the expert matrices
exactly, the ranks' sharded MoE FFNs add up to the unsharded one, and the plan gives the reference's per-rank n_ff.  The oracle's dequantisation
stands in for the GPU kernels."""
import numpy as np
import pytest

from conftest import random_wire
from ik_llama_cpp_b200 import tp
from oracle.oracle import GGML_TYPE, Oracle

# a row-header type, an _R4 type (rows interleaved in groups of 4), the DeepSeek-V3 expert type and a plain K-quant
TYPES = ["IQ4_KS", "IQ4_K_R4", "IQ2_XXS", "Q4_K"]
WORLDS = [2, 3, 4, 8]
N_EXPERT, N_EMBD = 3, 256
N_FF = 5 * 256          # five chunks of the granularity (256 for these types): uneven splits, and empty ranks at 8


@pytest.fixture(scope="module")
def orc():
    return Oracle()


def experts(name, n_expert, m, k, seed):
    rng = np.random.default_rng(seed)
    return [random_wire(name, m, k, rng) for _ in range(n_expert)]


def deq(orc, name, wire, n_expert, m, k):
    """[n_expert, m, k] f32 of n_expert stacked wire matrices"""
    if m == 0 or k == 0:
        return np.zeros((n_expert, m, k), np.float32)
    rs = orc.row_size(GGML_TYPE[name], k)
    w = np.asarray(wire, np.uint8).reshape(n_expert, m * rs)
    return np.stack([orc.dequantize(GGML_TYPE[name], w[e], m, k) for e in range(n_expert)])


def test_plan_matches_the_reference_split():
    assert tp.moe_ffn_plan(768, 8, GGML_TYPE["Q4_K"]) == [256] * 3 + [0] * 5          # Qwen3-30B-A3B: 768 = 3 x 256 over 8 ranks
    assert tp.moe_ffn_plan(2048, 8, GGML_TYPE["IQ2_XXS"]) == [256] * 8                # DeepSeek-V3
    assert tp.moe_ffn_plan(14336, 8, GGML_TYPE["IQ4_NL"]) == [1792] * 8               # Mixtral-8x7B: granularity 32
    assert tp.moe_ffn_plan(768, 2, GGML_TYPE["Q4_K"]) == [512, 256]                   # the remainder goes to the first ranks
    assert tp.moe_expert_granularity(GGML_TYPE["IQ4_NL"]) == 32 and tp.moe_expert_granularity(GGML_TYPE["IQ2_BN"]) == 64
    assert tp.moe_expert_granularity(GGML_TYPE["IQ1_S_R4"]) == 32


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", TYPES)
def test_split_up_gate_shards_reassemble_every_expert(orc, name, world):
    t = GGML_TYPE[name]
    split = tp.moe_ffn_plan(N_FF, world, t)
    assert sum(split) == N_FF and len(split) == world
    wire = np.concatenate(experts(name, N_EXPERT, N_FF, N_EMBD, [t, world, 1]))
    full = deq(orc, name, wire, N_EXPERT, N_FF, N_EMBD)
    parts = []
    for r in range(world):
        sh, n = tp.shard_expert_rows(wire, t, N_EXPERT, N_FF, N_EMBD, split, r)
        assert n == split[r] and sh.size == N_EXPERT * n * tp.row_size(t, N_EMBD)
        parts.append(deq(orc, name, sh, N_EXPERT, n, N_EMBD))
    assert np.array_equal(np.concatenate(parts, axis=1), full)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", TYPES)
def test_merged_gate_up_shards_reassemble_every_expert(orc, name, world):
    """rank r holds [gate rows r0:r1; up rows n_ff + r0 : n_ff + r1] of every expert: its own merged matrix with n_ff = split[r]"""
    t = GGML_TYPE[name]
    split = tp.moe_ffn_plan(N_FF, world, t)
    wire = np.concatenate(experts(name, N_EXPERT, 2 * N_FF, N_EMBD, [t, world, 2]))
    full = deq(orc, name, wire, N_EXPERT, 2 * N_FF, N_EMBD)
    gates, ups = [], []
    for r in range(world):
        sh, n = tp.shard_expert_gate_up(wire, t, N_EXPERT, N_FF, N_EMBD, split, r)
        d = deq(orc, name, sh, N_EXPERT, 2 * n, N_EMBD)
        gates.append(d[:, :n])
        ups.append(d[:, n:])
    assert np.array_equal(np.concatenate(gates, axis=1), full[:, :N_FF])
    assert np.array_equal(np.concatenate(ups, axis=1), full[:, N_FF:])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", TYPES)
def test_down_shards_reassemble_every_expert(orc, name, world):
    t = GGML_TYPE[name]
    split = tp.moe_ffn_plan(N_FF, world, t)
    wire = np.concatenate(experts(name, N_EXPERT, N_EMBD, N_FF, [t, world, 3]))
    full = deq(orc, name, wire, N_EXPERT, N_EMBD, N_FF)
    parts = []
    for r in range(world):
        sh, ks, k0 = tp.shard_expert_cols(wire, t, N_EXPERT, N_EMBD, N_FF, split, r)
        assert (ks, k0) == (split[r], sum(split[:r]))
        parts.append(deq(orc, name, sh, N_EXPERT, N_EMBD, ks))
    assert np.array_equal(np.concatenate(parts, axis=2), full), "K shards (row headers replicated) must dequantise to the column slices"


def moe_ffn(up, gate, down, x, ids, weights):
    """f64 MoE FFN of dequantised experts: sum_u weights[t, u] * down[e] (silu(gate[e] x_t) * (up[e] x_t)), e = ids[t, u]"""
    y = np.zeros((x.shape[0], down.shape[1]))
    for tk in range(x.shape[0]):
        for u, e in enumerate(ids[tk]):
            g, v = gate[e] @ x[tk], up[e] @ x[tk]
            y[tk] += weights[tk, u] * (down[e] @ (g / (1 + np.exp(-g)) * v))
    return y


@pytest.mark.parametrize("merged", [False, True], ids=["split", "merged"])
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", ["IQ4_KS", "IQ2_XXS"])
def test_sum_of_rank_partials_is_the_unsharded_ffn(orc, name, world, merged):
    t = GGML_TYPE[name]
    split = tp.moe_ffn_plan(N_FF, world, t)
    rng = np.random.default_rng([t, world, int(merged)])
    n_tokens, n_used = 5, 2
    x = rng.standard_normal((n_tokens, N_EMBD))
    ids = np.stack([rng.permutation(N_EXPERT)[:n_used] for _ in range(n_tokens)])
    weights = rng.uniform(0.1, 1.0, (n_tokens, n_used))
    down_w = np.concatenate(experts(name, N_EXPERT, N_EMBD, N_FF, [t, 4]))
    if merged:
        gu_w = np.concatenate(experts(name, N_EXPERT, 2 * N_FF, N_EMBD, [t, 5]))
        gu = deq(orc, name, gu_w, N_EXPERT, 2 * N_FF, N_EMBD).astype(np.float64)
        gate, up = gu[:, :N_FF], gu[:, N_FF:]
    else:
        up_w, gate_w = (np.concatenate(experts(name, N_EXPERT, N_FF, N_EMBD, [t, s])) for s in (6, 7))
        up, gate = (deq(orc, name, w, N_EXPERT, N_FF, N_EMBD).astype(np.float64) for w in (up_w, gate_w))
    ref = moe_ffn(up, gate, deq(orc, name, down_w, N_EXPERT, N_EMBD, N_FF).astype(np.float64), x, ids, weights)
    total = np.zeros_like(ref)
    for r in range(world):
        if split[r] == 0:            # an empty rank contributes a zero partial
            continue
        dsh, ks, _ = tp.shard_expert_cols(down_w, t, N_EXPERT, N_EMBD, N_FF, split, r)
        if merged:
            sh, n = tp.shard_expert_gate_up(gu_w, t, N_EXPERT, N_FF, N_EMBD, split, r)
            d = deq(orc, name, sh, N_EXPERT, 2 * n, N_EMBD).astype(np.float64)
            g_r, u_r = d[:, :n], d[:, n:]
        else:
            u_r, g_r = (deq(orc, name, tp.shard_expert_rows(w, t, N_EXPERT, N_FF, N_EMBD, split, r)[0], N_EXPERT, split[r], N_EMBD).astype(np.float64)
                        for w in (up_w, gate_w))
        total += moe_ffn(u_r, g_r, deq(orc, name, dsh, N_EXPERT, N_EMBD, ks).astype(np.float64), x, ids, weights)
    np.testing.assert_allclose(total, ref, rtol=1e-10, atol=1e-12 * float(np.abs(ref).max()))
