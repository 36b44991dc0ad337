"""CPU tests of the row-slice MUL_MAT entry (b200q_mul_mat_rows): its device-free check b200q_mul_mat_rows_ok and workspace query, the argument
errors of the call itself, and the argument checks of backend.mul_mat_rows.  A slice is accepted when every plane pointer keeps the 256-byte alignment
of a whole tensor's (row0 times the bytes per row of each plane a multiple of 256; wire-layout types: of the wire row), with row0 and m multiples of 4
for the _R4 types.  The workspace is 0 for f32 x with n <= 8, the f32 image of an f16 x for n <= 8, and the dense GEMM's workspace above (plus the
f32 image of an f16 x where IQ2_BN takes the int8 pipe)."""
import ctypes

import pytest
import torch

import ik_llama_cpp_b200 as pkg
import ik_llama_cpp_b200.backend as be
from conftest import ALL_TYPES
from oracle.oracle import GGML_TYPE

E_TYPE, E_SHAPE, E_ARG, E_NOMEM = -1, -2, -4, -5
F32, F16 = 0, 1
R4_TYPES = [t for t in ALL_TYPES if t.endswith("_R4")]


def align256(n):
    return (n + 255) // 256 * 256


def ok(name, rows_layout, row0, m, k, n=16, x_type=F16, cs=None):
    t = GGML_TYPE[name] if isinstance(name, str) else name
    return int(pkg.lib().b200q_mul_mat_rows_ok(t, rows_layout, row0, m, k, n, x_type, k if cs is None else cs))


def ws(name, rows_layout, row0, m, k, n, x_type, cs=None):
    return int(pkg.lib().b200q_mul_mat_rows_workspace(GGML_TYPE[name], rows_layout, row0, m, k, n, x_type, k if cs is None else cs))


def expected_ws(name, m, k, n, x_type):
    if n <= 8:
        return align256(n * k * 4) if x_type == F16 else 0
    widen = x_type == F16 and name == "IQ2_BN" and k % 64 == 0
    return (align256(n * k * 4) if widen else 0) + align256(n * k * 2) + align256(m * k * 2)


def plane_row_bytes(name, k):
    """bytes per row of every plane of the device layout (b200q_types.cuh), or of the wire row for a wire-layout type"""
    planes = {"Q8_0": [32, 2], "Q4_K": [128, 16], "Q6_K": [128, 64, 16, 2], "IQ2_BN": [16, 4]}
    if name == "IQ2_BN":
        return [k // 4, 4]
    if name in planes:
        qk = 32 if name == "Q8_0" else 256
        return [b * (k // qk) for b in planes[name]]
    return [int(pkg.lib().b200q_wire_row_size(GGML_TYPE[name], k))]


@pytest.mark.parametrize("name", ["Q8_0", "Q4_K", "Q6_K", "IQ2_BN", "IQ2_XXS"] + R4_TYPES[:2])
def test_accepted_origins_follow_the_alignment_rule(name):
    k, rows_layout, m = 512, 1024, 128
    for row0 in range(0, rows_layout - m + 1, 4):
        aligned = all(row0 * b % 256 == 0 for b in plane_row_bytes(name, k))
        assert ok(name, rows_layout, row0, m, k) == (0 if aligned else E_SHAPE), (name, row0)


@pytest.mark.parametrize("name", ["Q8_0", "Q4_K", "Q6_K", "IQ4_NL", "IQ2_BN", "IQ2_XXS", "IQ1_S"] + R4_TYPES[:2])
def test_workspace_grid(name):
    k, rows_layout = 512, 2048
    row0 = next(r for r in range(256, rows_layout, 4) if ok(name, rows_layout, r, 256, k) == 0)
    for m in (256, 512):
        for n in (1, 5, 8, 9, 128, 600):
            for x_type in (F32, F16):
                assert ws(name, rows_layout, row0, m, k, n, x_type, cs=576) == expected_ws(name, m, k, n, x_type), (name, m, n, x_type)


def test_f32_whole_tensor_workspace_is_the_mul_mat_workspace():
    for name in ("Q8_0", "Q4_K", "IQ2_BN", "IQ2_XXS"):
        for n in (1, 8, 9, 600):
            assert ws(name, 768, 0, 768, 512, n, F32) == int(pkg.lib().b200q_mul_mat_workspace(GGML_TYPE[name], 768, 512, n))


def test_unaligned_views_are_rejected():
    """the weight views the plug-graph harness expects to stay declined"""
    assert ok("Q4_K", 64, 37, 8, 512) == E_SHAPE             # its 32-byte meta-plane rows land at 160 mod 256
    assert ok("IQ2_XXS", 64, 5, 8, 512) == E_SHAPE           # its 132-byte rows land at 148 mod 256


@pytest.mark.parametrize("name", ["Q8_0", "Q6_K"])
def test_deepseek_slices_are_accepted(name):
    """DeepSeek-V3 wkv_b: 128 heads x 256 rows, K = kv_lora_rank = 512, split into 1, 2 or 4 slices per layer; x is the f16 K cache (576 halves)"""
    for m in (32768, 16384, 8192):
        for row0 in range(0, 32768, m):
            for n in (256, 1024, 4096, 16384):
                assert ok(name, 32768, row0, m, 512, n, F16, 576) == 0, (m, row0, n)


def test_r4_types_need_whole_row_groups():
    name = R4_TYPES[0]
    assert ok(name, 1024, 256, 128, 512) == 0
    assert ok(name, 1024, 256, 126, 512) == E_SHAPE
    assert ok(name, 1024, 258, 128, 512) == E_SHAPE                           # an origin inside a group of 4 interleaved rows


def test_argument_errors():
    assert ok("Q8_0", 256, 0, 64, 512, x_type=7) == E_TYPE                    # activations neither f32 nor f16
    assert ok(0, 256, 0, 64, 512) == E_TYPE                                   # an f32 weight
    assert ok("Q8_0", 256, 0, 64, 500) == E_SHAPE                             # k not a multiple of the block
    assert ok("Q4_K", 256, 0, 64, 384) == E_SHAPE
    assert ok("Q8_0", 256, 256, 8, 512) == E_ARG                              # rows past the tensor
    assert ok("Q8_0", 256, -8, 8, 512) == E_ARG
    assert ok("Q8_0", 256, 0, 0, 512) == E_ARG                                # no rows
    assert ok("Q8_0", 256, 0, 64, 512, n=0) == E_ARG                          # no columns
    assert ok("Q8_0", 256, 0, 64, 512, cs=516) == E_ARG                       # f16 stride not a multiple of 16 bytes
    assert ok("Q8_0", 256, 0, 64, 512, x_type=F32, cs=516) == 0               # 516 floats are
    assert ok("Q8_0", 256, 0, 64, 512, x_type=F32, cs=514) == E_ARG
    assert ok("Q8_0", 256, 0, 64, 512, n=2, cs=256) == E_ARG                  # columns overlap
    assert ok("Q8_0", 256, 0, 64, 512, n=1, cs=256) == 0                      # one column: any aligned stride
    assert ok("Q8_0", 256, 0, 64, 512, n=1, cs=-8) == E_ARG
    assert ws("Q8_0", 256, 256, 8, 512, 16, F16) == 0                         # a rejected argument needs no workspace


def test_call_rejects_before_the_device():
    """the argument and workspace errors of the call come before it looks for a device"""
    L = pkg.lib()
    t, W, x, dst = GGML_TYPE["Q8_0"], 1 << 20, 1 << 21, 1 << 22
    call = lambda W=W, x=x, x_type=F16, row0=0, n=16, wsp=None, wsb=0: int(L.b200q_mul_mat_rows(t, W, 256, row0, x_type, x, 576, dst, 64, 512, n, wsp, wsb, None))
    assert call(W=None) == E_ARG
    assert call(x=x + 8) == E_ARG                                            # x not 16-byte aligned
    assert call(row0=300) == E_ARG
    assert call(x_type=3) == E_TYPE
    assert call(wsp=1 << 23, wsb=ws("Q8_0", 256, 0, 64, 512, 16, F16) - 1) == E_NOMEM
    assert call(wsp=(1 << 23) + 16, wsb=1 << 30) == E_ARG                    # workspace not 256-byte aligned


def test_python_argument_checks():
    w = be.QuantTensor(GGML_TYPE["Q8_0"], 256, 512, torch.empty(0, dtype=torch.uint8))
    with pytest.raises(ValueError):
        be.mul_mat_rows(w, torch.zeros(4, 512, dtype=torch.bfloat16), 0, 64)
    with pytest.raises(ValueError):
        be.mul_mat_rows(w, torch.zeros(4, 1024, dtype=torch.float16)[:, ::2], 0, 64)
    with pytest.raises(ValueError):
        be.mul_mat_rows(w, torch.zeros(4, 256, dtype=torch.float16), 0, 64)
    assert be.mul_mat_rows_workspace(w, 0, 64, 4, torch.float16, 576) == align256(4 * 512 * 4)
    assert be.mul_mat_rows_workspace(w, 0, 64, 4, torch.float32, 576) == 0
