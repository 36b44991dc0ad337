"""CPU tests of MOE_FUSED_UP_GATE over merged up/gate experts (ffn_gate_up_exps): the C ABI entry points load, and the workspace query
b200q_moe_up_gate_merged_workspace is 0 exactly where the split up/gate query b200q_mul_mat_id_workspace(up_gate = 1) is 0, so that both forms
take the mat-vec kernel and the grouped GEMM on the same batches.  No device needed."""
import itertools

import pytest

import ik_llama_cpp_b200 as pkg
from conftest import ALL_TYPES
from ik_llama_cpp_b200 import backend
from oracle.oracle import GGML_TYPE

# the model shapes of scripts/bench_moe.py (name, n_expert, n_used, n_ff, K, type)
MODELS = [("qwen3-30b-a3b", 128, 8, 768, 2048, "Q4_K"), ("mixtral-8x7b", 8, 2, 14336, 4096, "IQ4_NL"),
          ("deepseek-v3-tp8", 256, 8, 256, 7168, "IQ2_XXS")]


def merged_ws(name, m, k, n_used, nb1, n_tokens, n_expert):
    return pkg.lib().b200q_moe_up_gate_merged_workspace(GGML_TYPE[name], m, k, n_used, nb1, n_tokens, n_expert)


def split_ws(name, m, k, n_used, nb1, n_tokens, n_expert):
    return pkg.lib().b200q_mul_mat_id_workspace(GGML_TYPE[name], m, k, n_used, nb1, n_tokens, n_expert, 1)


def test_symbols_load():
    L = pkg.lib()
    for s in ("b200q_moe_up_gate_merged", "b200q_moe_up_gate_merged_workspace"):
        assert s in pkg.header_symbols(), s
        assert hasattr(L, s), s
        assert getattr(L, s).argtypes, f"{s}: no ctypes signature in _lib.py"
    assert hasattr(backend, "moe_up_gate_merged") and hasattr(backend, "moe_up_gate_merged_workspace")


@pytest.mark.parametrize("name", ALL_TYPES)
def test_zero_exactly_where_the_split_query_is_zero(name):
    """A grid of shapes on both sides of the crossover (n_slots > 5 n_expert) and of every eligibility rule of the grouped GEMM: K % 256, n_ff not
    a multiple of 4 or of 128, nb1 not dividing n_used, more than 1024 experts, n_slots n_ff not a multiple of 4."""
    grouped = 0
    for m, k, (n_used, nb1), n_tokens, n_expert in itertools.product(
            (256, 258, 260, 1408), (256, 1024, 1056), ((2, 1), (8, 1), (8, 8), (3, 2)), (1, 7, 20, 21, 41, 160, 161, 513), (8, 16, 1025)):
        a, b = merged_ws(name, m, k, n_used, nb1, n_tokens, n_expert), split_ws(name, m, k, n_used, nb1, n_tokens, n_expert)
        assert (a == 0) == (b == 0), (name, m, k, n_used, nb1, n_tokens, n_expert, a, b)
        # the merged form keeps the split form's workspace layout; generic types dequantise both halves of an expert into the weight scratch
        assert a >= b, (name, m, k, n_used, nb1, n_tokens, n_expert, a, b)
        grouped += a > 0
    assert grouped > 0


@pytest.mark.parametrize("model,n_expert,n_used,n_ff,k,name", MODELS)
def test_model_shapes_cross_over_with_the_split_form(model, n_expert, n_used, n_ff, k, name):
    t_last = 5 * n_expert // n_used          # the last batch of the mat-vec kernel (b200q_api.cu: grouped when n_slots > 5 n_expert)
    for n_tokens in (1, 8, 64, t_last, t_last + 1, 512):
        a = merged_ws(name, n_ff, k, n_used, 1, n_tokens, n_expert)
        assert (a > 0) == (n_tokens > t_last), (model, n_tokens, a)
        assert (a == 0) == (split_ws(name, n_ff, k, n_used, 1, n_tokens, n_expert) == 0)


def test_generic_scratch_holds_both_halves():
    """Q6_K (no fused prefill kernel): one expert's bf16 scratch is 2 n_ff K 2 bytes; the fused types need none, so their workspace is the split one."""
    e, n_used, n_ff, k, n = 8, 2, 512, 1024, 512
    assert merged_ws("Q6_K", n_ff, k, n_used, 1, n, e) - split_ws("Q6_K", n_ff, k, n_used, 1, n, e) == e * n_ff * k * 2
    assert merged_ws("Q4_K", n_ff, k, n_used, 1, n, e) == split_ws("Q4_K", n_ff, k, n_used, 1, n, e)
