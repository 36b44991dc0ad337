"""CPU tests of the batched MUL_MAT entry: the workspace query of b200q_mul_mat_batched (no device needed) and the argument checks of
backend.mul_mat_batched.  The query returns the bytes of the path plan_batched (b200q_api.cu) takes:
  * one matrix over columns a constant stride apart: 0 for n n_batch <= 8 (the dense mat-vec), the dense GEMM's workspace for n > 8;
  * any other broadcast with n <= 8: 0 (the dense mat-vec of each entry);
  * the grouped GEMM (K % 256 == 0, at least 128 slots n_batch n, n > 1 for a type without a fused GEMM kernel): the identity ids plus its workspace;
  * otherwise, up to n = 16, the identity-routed mat-vec: the ids, int32 [n_batch][n] rounded up to 256 bytes; above, one dense GEMM's workspace;
  * 0 for every rejected argument."""
import pytest
import torch

import ik_llama_cpp_b200 as pkg
import ik_llama_cpp_b200.backend as be
from oracle.oracle import GGML_TYPE

Q8_0 = GGML_TYPE["Q8_0"]
IQ4_NL = GGML_TYPE["IQ4_NL"]


def align256(n):
    return (n + 255) // 256 * 256


def ws(m, k, n, n_batch, per_entry, cs, bs, t=Q8_0):
    return int(pkg.lib().b200q_mul_mat_batched_workspace(t, m, k, n, n_batch, per_entry, cs, bs))


def gemm_ws(m, k, n):
    return align256(n * k * 2) + align256(m * k * 2)


@pytest.mark.parametrize("n_head", [128, 16])
def test_mla_decode(n_head):
    # wk_b (K = 128): the identity-routed mat-vec needs only the ids, up to 16 columns
    for n in (1, 2, 4, 8, 16):
        assert ws(512, 128, n, n_head, 1, n_head * 192, 192) == align256(n_head * n * 4)
    # wv_b (K = 512): the mat-vec below 128 slots, the grouped GEMM from there on; Q8_0 (no fused GEMM kernel) keeps the mat-vec at n = 1
    for t in (Q8_0, IQ4_NL):
        for n in (1, 2, 4, 8):
            got, ids = ws(128, 512, n, n_head, 1, n_head * 512, 512, t), align256(n_head * n * 4)
            grouped = n_head * n >= 128 and (n > 1 or t == IQ4_NL)
            assert (got > ids + n_head * n * 512 * 2) if grouped else got == ids, (t, n)


@pytest.mark.parametrize("n_head", [128, 16])
def test_mla_prefill(n_head):
    # wv_b (K = 512): grouped GEMM, more than the ids and the bf16 gather of every column
    for n in (9, 64, 512):
        got = ws(128, 512, n, n_head, 1, n_head * 512, 512)
        assert got >= align256(n_head * n * 4) + n_head * n * 512 * 2
    # wk_b (K = 128): the grouped GEMM refuses it, one dense GEMM per head on one workspace above 16 columns
    for n in (17, 64, 512):
        assert ws(512, 128, n, n_head, 1, n_head * 192, 192) == gemm_ws(512, 128, n)


def test_broadcast_over_uniform_columns_is_one_product():
    m, k = 256, 512
    assert ws(m, k, 1, 8, 0, k, k) == 0                      # 8 columns: the dense mat-vec
    assert ws(m, k, 4, 2, 0, k, 4 * k) == 0
    assert ws(m, k, 9, 2, 0, k, 9 * k) == gemm_ws(m, k, 18)   # 18 columns, 9 per entry: the dense GEMM
    assert ws(m, k, 1, 1, 1, k, k) == 0                      # one entry
    # up to 8 columns per entry, more than 8 in all, or not uniformly strided: the dense mat-vec of each entry
    assert ws(m, k, 3, 4, 0, k, 3 * k) == 0
    assert ws(m, k, 2, 4, 0, k, 3 * k) == 0
    # more than 8 columns per entry, not uniformly strided: identity routing with one matrix (here 9 x 4 slots: the mat-vec)
    assert ws(m, k, 9, 4, 0, k, 10 * k) == align256(36 * 4)


def test_rejected_arguments_need_nothing():
    m, k = 128, 512
    assert ws(m, k, 4, 16, 1, k + 2, 4 * k) == 0             # stride not a multiple of 4 floats
    assert ws(m, k, 4, 16, 1, k - 4, 4 * k) == 0             # columns overlap
    assert ws(m, k, 4, 16, 1, k, k - 4) == 0                 # entries overlap
    assert ws(m, k, 4, 16, 1, -k, 4 * k) == 0
    assert ws(m, k, 0, 16, 1, k, 4 * k) == 0
    assert ws(m, k, 4, 0, 1, k, 4 * k) == 0
    assert ws(m, k, 4, 16, 2, k, 4 * k) == 0                 # per_entry is 0 or 1
    assert ws(m, 100, 4, 16, 1, 100, 400) == 0                # K not a multiple of the block
    assert ws(m, k, 4, 16, 1, k, 4 * k, t=9999) == 0          # unknown type


def fake_weight(n_mat, m=128, k=512):
    return be.ExpertTensor(Q8_0, n_mat, m, k, torch.empty(0, dtype=torch.uint8))


def test_python_mirror_argument_checks():
    w = fake_weight(16)
    with pytest.raises(ValueError):                          # K mismatch
        be._batched_args(w, torch.zeros(16, 4, 256), True)
    with pytest.raises(ValueError):                          # not f32
        be._batched_args(w, torch.zeros(16, 4, 512, dtype=torch.float16), True)
    with pytest.raises(ValueError):                          # rows not contiguous
        be._batched_args(w, torch.zeros(16, 512, 4).transpose(1, 2), True)
    with pytest.raises(ValueError):                          # column stride not a multiple of 4 floats
        be._batched_args(w, torch.zeros(16, 4, 514)[:, :, :512], True)
    with pytest.raises(ValueError):                          # one matrix per entry needs n_batch matrices
        be._batched_args(fake_weight(8), torch.zeros(16, 4, 512), True)
    # MLA's q_nope_perm: [n_head, n_tokens, 128] with columns n_head * 192 and entries 192 floats apart
    q = torch.zeros(5, 16, 192)
    assert be._batched_args(fake_weight(16, 512, 128), q[:, :, :128].transpose(0, 1), True) == (16, 5, 16 * 192, 192)
    # a dimension of size 1 reports any stride: its stride is not used
    assert be._batched_args(w, torch.zeros(16, 1, 512), False) == (16, 1, 512, 512)
