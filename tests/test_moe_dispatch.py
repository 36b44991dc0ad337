"""CPU tests of the MoE prefill dispatch rule: b200q_mul_mat_id_workspace returns 0 exactly when b200q_mul_mat_id takes the mat-vec path
(ineligible shape, or a batch below the measured crossover) and the grouped GEMM's workspace size otherwise.  No device needed."""
import pytest

import ik_llama_cpp_b200 as pkg
from oracle.oracle import GGML_TYPE

# b200q_api.cu: up/gate takes the grouped GEMM when n_slots > 5 * n_expert, MUL_MAT_ID when n_slots > 32 (n_slots = n_tokens * n_used)
UP_GATE_MIN_ROWS_PER_EXPERT = 5
MUL_MAT_ID_MIN_SLOTS = 32


def last_mat_vec_batch(n_expert, n_used, up_gate):
    return (UP_GATE_MIN_ROWS_PER_EXPERT * n_expert if up_gate else MUL_MAT_ID_MIN_SLOTS) // n_used

# (name, n_expert, n_used, up/gate m x k, down m x k, type): the model shapes of scripts/bench_moe.py
MODELS = [("qwen3-30b-a3b", 128, 8, (768, 2048), (2048, 768), "Q4_K"),
          ("qwen3-30b-a3b", 128, 8, (768, 2048), (2048, 768), "IQ4_K"),
          ("mixtral-8x7b", 8, 2, (14336, 4096), (4096, 14336), "IQ4_NL"),
          ("deepseek-v3-tp8", 256, 8, (256, 7168), (7168, 256), "IQ2_XXS")]


def ws(name, m, k, n_used, nb1, n_tokens, n_expert, up_gate):
    return pkg.lib().b200q_mul_mat_id_workspace(GGML_TYPE[name], m, k, n_used, nb1, n_tokens, n_expert, int(up_gate))


@pytest.mark.parametrize("model,n_expert,n_used,ug,down,name", MODELS)
def test_threshold_both_sides(model, n_expert, n_used, ug, down, name):
    # the last batch on the mat-vec side and the first one on the grouped side
    for (m, k), nb1, up_gate in ((ug, 1, True), (down, n_used, False)):
        t_last = last_mat_vec_batch(n_expert, n_used, up_gate)
        assert ws(name, m, k, n_used, nb1, t_last, n_expert, up_gate) == 0
        assert ws(name, m, k, n_used, nb1, 1, n_expert, up_gate) == 0
        first = ws(name, m, k, n_used, nb1, t_last + 1, n_expert, up_gate)
        assert first >= (t_last + 1) * n_used * k * 2          # at least the bf16 gather of the slots


@pytest.mark.parametrize("model,n_expert,n_used,ug,down,name", MODELS)
def test_pp512_takes_the_grouped_gemm(model, n_expert, n_used, ug, down, name):
    (m, k), (m2, k2) = ug, down
    up_gate_ws = ws(name, m, k, n_used, 1, 512, n_expert, True)
    down_ws = ws(name, m2, k2, n_used, n_used, 512, n_expert, False)
    assert up_gate_ws > 0 and down_ws > 0
    assert up_gate_ws >= 512 * n_used * m * 4                  # up/gate keeps the up result in the workspace


def test_ineligible_shapes_take_the_mat_vec_path():
    big = 4096
    assert ws("IQ4_NL", 256, 1024, 2, 1, big, 8, False) > 0
    assert ws("IQ4_NL", 256, 1024 + 32, 2, 1, big, 8, False) == 0      # K % 256 != 0
    assert ws("IQ4_NL", 256, 1024, 2, 1, big, 1025, False) == 0        # more experts than routing threads
    assert ws("IQ4_NL", 256, 1024, 3, 2, big, 8, False) == 0           # nb1 must divide n_used
    assert ws("IQ4_NL", 258, 1024, 1, 1, 4099, 8, True) == 0           # up/gate: n_slots * m % 4 != 0
    assert ws("IQ4_NL", 256, 1024, 2, 1, big, 0, False) == 0
    assert pkg.lib().b200q_mul_mat_id_workspace(99999, 256, 1024, 2, 1, big, 8, 0) == 0


def test_generic_types_size_a_bounded_weight_scratch():
    # generic types also need the bf16 copies of a group of experts, capped at a fixed budget; the fused types need none
    e, m, k, t = 256, 7168, 256, 512
    a = ws("IQ2_XXS", m, k, 8, 8, t, e, False)
    b = ws("IQ4_NL", m, k, 8, 8, t, e, False)
    assert a > b and a - b <= (256 << 20) + 4096
