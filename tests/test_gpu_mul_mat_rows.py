"""MUL_MAT over a row slice of a weight with f32 or f16 activations a column stride apart (b200q_mul_mat_rows): DeepSeek's MLA prompt-processing
product kv_f32 = wkv_b_iter x kv_cache_nope, whose src0 is a view of whole rows of wkv_b and whose src1 is a view of the f16 K cache (576 halves per
column, starting 64 halves in).

The result contract, checked without tolerance: a slice computes what b200q_mul_mat computes on the same rows uploaded as a tensor of their own, over
the host-widened contiguous f32 x, with the same launches (kernel names and grids from a torch.profiler trace).  An f16 x adds one conversion launch:
f16 -> f32 before a mat-vec and before the IQ2_BN int8 GEMM, f16 -> bf16 in place of f32 -> bf16 before every other GEMM.  At K = 512 a fused GEMM
splits K at most in two, and two f32 atomics onto zero give the same sum in either order, so every case here is bit-equal.  Each case is also held
to the oracle bars of test_gpu_plug_graphs.product_check (IQ2_BN's int8 GEMM: NMSE <= 5e-4, test_gpu_parity's bar)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ALL_TYPES, make_wire
from oracle.oracle import GGML_TYPE, nmse
from test_gpu_decode_schedules import profiled, run_child
from test_gpu_plug_graphs import product_check

pytestmark = pytest.mark.gpu

F32, F16 = 0, 1
E_ARG, E_SHAPE, E_NOMEM = -4, -2, -5
CACHE_COLS, CACHE_OFF = 576, 64          # DeepSeek's K cache: kv_lora_rank + rope halves per column, the latent part after the rope part
NS = (1, 5, 8, 9, 128, 600)


@pytest.fixture(scope="module")
def be():
    import ik_llama_cpp_b200.backend as be
    return be


def lib():
    import ik_llama_cpp_b200 as pkg
    return pkg.lib()


def wire_rows(name, wire, k, row0, m):
    rs = int(lib().b200q_wire_row_size(GGML_TYPE[name], k))
    return np.ascontiguousarray(np.asarray(wire, np.uint8).ravel()[row0 * rs:(row0 + m) * rs])


def first_origin(name, rows_layout, m, k):
    """the first non-zero row origin the alignment rule accepts"""
    t = GGML_TYPE[name]
    return next(r for r in range(4, rows_layout - m + 1, 4) if lib().b200q_mul_mat_rows_ok(t, rows_layout, r, m, k, 16, F16, CACHE_COLS) == 0)


def cache_view(n, k, dtype, seed, cols=CACHE_COLS, off=CACHE_OFF):
    """[n, k] view of a cache-like buffer: columns `cols` elements apart starting `off` in, the rest NaN"""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((n * cols + off + cols,), float("nan"), dtype=dtype)
    buf[off:off + n * cols].view(n, cols)[:, :k] = torch.randn(n, k, generator=g).to(dtype)
    buf = buf.cuda()
    return buf, buf[off:off + n * cols].view(n, cols)[:, :k]


def separate(be, name, wire, k, row0, m):
    return be.set_tensor(GGML_TYPE[name], wire_rows(name, wire, k, row0, m), m, k)


@pytest.mark.parametrize("name", ALL_TYPES)
def test_slice_equals_separate_tensor(be, oracle, name):
    t = GGML_TYPE[name]
    if not lib().b200q_type_supported(t):
        pytest.skip("type not supported")
    k, rows_layout, m = 512, 768, 256
    row0 = first_origin(name, rows_layout, m, k)
    wire = make_wire(oracle, name, rows_layout, k, 1234)
    w = be.set_tensor(t, wire, rows_layout, k)
    ws_ = separate(be, name, wire, k, row0, m)
    sub = wire_rows(name, wire, k, row0, m)
    for n in NS:
        for dtype in (torch.float32, torch.float16):
            _, x = cache_view(n, k, dtype, seed=n)
            y = be.mul_mat_rows(w, x, row0, m)
            xf = x.float().contiguous()
            ref = be.mul_mat(ws_, xf)
            torch.cuda.synchronize()
            what = f"{name} row0={row0} n={n} {dtype}"
            assert torch.equal(y, ref), what
            yn, xn = y.cpu().numpy(), xf.cpu().numpy()
            if name == "IQ2_BN" and n > 8:
                assert nmse(yn, oracle.mul_mat_q8_1(t, sub, xn, m, variant="b200")) <= 5e-4, what
            else:
                product_check(oracle, t, sub, xn, yn, m, n <= 8, what)


@pytest.mark.parametrize("name", ["Q8_0", "Q6_K"])
@pytest.mark.parametrize("n_kv", [1024, 4096])
def test_deepseek_v3_wkv_b(be, oracle, name, n_kv):
    """128 heads x 256 rows, K = 512; one slice at n_kv = 1024, two at 4096 (attn_max_batch 256 MiB, src/llama.cpp:7609)"""
    t, k, rows_layout = GGML_TYPE[name], 512, 32768
    n_slices = 1 if n_kv == 1024 else 2
    m = rows_layout // n_slices
    wire = make_wire(oracle, name, rows_layout, k, 77)
    w = be.set_tensor(t, wire, rows_layout, k)
    _, x = cache_view(n_kv, k, torch.float16, seed=n_kv)
    xf = x.float().contiguous()
    for s in range(n_slices):
        y = be.mul_mat_rows(w, x, s * m, m)
        ref = be.mul_mat(separate(be, name, wire, k, s * m, m), xf)
        torch.cuda.synchronize()
        assert torch.equal(y, ref), (name, n_kv, s)


CONVERSIONS = ("k_f16_convert", "k_f32_to_bf16")
# every path once: the mat-vec and the GEMM of a type without a fused kernel (Q8_0), of a fused type (Q4_K), of a wire-layout type (IQ2_XXS); the
# IQ2_BN int8 GEMM; an _R4 type
LAUNCH_CASES = [("Q8_0", 1), ("Q8_0", 600), ("Q4_K", 8), ("Q4_K", 600), ("IQ2_XXS", 1), ("IQ2_XXS", 600), ("IQ2_BN", 9), ("IQ4_K_R4", 9)]


def _child(case_id, out_dir):
    """One launch comparison in a process of its own (in a long-lived process the profiler sometimes returns the launches without the kernel
    records, see test_gpu_decode_schedules._child): the kernels of the slice call over f16 and f32 x and of the separate-tensor call."""
    from ik_llama_cpp_b200 import backend as be
    from oracle.oracle import Oracle
    name, n = case_id.split(":")[0], int(case_id.split(":")[1])
    t, k, rows_layout, m = GGML_TYPE[name], 512, 768, 256
    row0 = first_origin(name, rows_layout, m, k)
    wire = make_wire(Oracle(), name, rows_layout, k, 99)
    w, ws_ = be.set_tensor(t, wire, rows_layout, k), separate(be, name, wire, k, row0, m)
    _, x16 = cache_view(n, k, torch.float16, seed=3)
    _, x32 = cache_view(n, k, torch.float32, seed=3)
    xf = x16.float().contiguous()
    calls = {"k16": lambda: be.mul_mat_rows(w, x16, row0, m), "k32": lambda: be.mul_mat_rows(w, x32, row0, m), "kref": lambda: be.mul_mat(ws_, xf)}
    for fn in calls.values():
        fn()                                              # warm: module loading and function attributes stay out of the traces
    got = {key: [list(kk) for kk in profiled(fn)[1]] for key, fn in calls.items()}
    np.savez(os.path.join(out_dir, "y.npz"))
    with open(os.path.join(out_dir, "launches.json"), "w") as f:
        json.dump(got, f)


@pytest.mark.parametrize("case", LAUNCH_CASES, ids=[f"{n}-{name}" for name, n in LAUNCH_CASES])
def test_same_launches_as_separate_tensor(tmp_path, case):
    name, n = case
    _, got = run_child(f"{name}:{n}", tmp_path, script=__file__)
    k16, k32, kref = ([tuple(kk[0:1]) + tuple(tuple(v) for v in kk[1:]) for kk in got[key]] for key in ("k16", "k32", "kref"))
    assert kref, f"{name} n={n}: the profiler returned no kernel records"
    assert k32 == kref, (name, n, k32, kref)
    conv16 = [kk for kk in k16 if "k_f16_convert" in kk[0]]
    assert len(conv16) == 1, k16
    widen = n <= 8 or name == "IQ2_BN"
    assert ("k_f16_convert<float" in conv16[0][0]) == widen, conv16     # k_f16_convert<float, 8> widens, <__nv_bfloat16, 8> converts to bf16
    strip = lambda ks: [kk for kk in ks if not any(c in kk[0] for c in CONVERSIONS)]
    assert strip(k16) == strip(kref), (name, n, k16, kref)
    assert len(kref) - len(strip(kref)) == (0 if widen else 1)          # the f32 -> bf16 launch the f16 one replaces


def test_memory_contract(be, oracle):
    """exact queried workspace, poisoned outputs and workspace, inputs unchanged, nothing written by a rejected call"""
    L = lib()
    for name, n in (("Q4_K", 5), ("Q4_K", 128), ("Q8_0", 128), ("IQ2_BN", 128)):
        t, k, rows_layout, m = GGML_TYPE[name], 512, 768, 256
        row0 = first_origin(name, rows_layout, m, k)
        wire = make_wire(oracle, name, rows_layout, k, 5)
        w = be.set_tensor(t, wire, rows_layout, k)
        xbuf, x = cache_view(n, k, torch.float16, seed=11)
        need = int(L.b200q_mul_mat_rows_workspace(t, rows_layout, row0, m, k, n, F16, CACHE_COLS))
        guard = 4096
        arena = torch.full((guard + need + guard + n * m * 4 + guard,), 0xA5, dtype=torch.uint8, device="cuda")
        ws_off, dst_off = guard, guard + need + guard
        arena[ws_off:ws_off + need] = 0xFF                              # NaN bytes
        arena[dst_off:dst_off + n * m * 4] = 0xFF
        before_arena, before_x, before_w = arena.clone(), xbuf.clone(), w.planes.clone()
        base = arena.data_ptr()
        call = lambda **kw: int(L.b200q_mul_mat_rows(t, w.ptr, rows_layout, kw.get("row0", row0), F16, x.data_ptr(), CACHE_COLS, base + dst_off, m, k, n,
                                                     base + ws_off if need else None, kw.get("wsb", need), None))
        for bad in ({"row0": row0 + 1}, {"wsb": need - 1} if need else {"row0": -4}):
            assert call(**bad) in (E_ARG, E_SHAPE, E_NOMEM), bad
        torch.cuda.synchronize()
        assert torch.equal(arena, before_arena), f"{name} n={n}: a rejected call wrote"
        assert call() == 0
        torch.cuda.synchronize()
        assert torch.equal(xbuf.view(torch.int16), before_x.view(torch.int16)) and torch.equal(w.planes, before_w), f"{name} n={n}: an input changed"
        assert torch.equal(arena[:ws_off], before_arena[:ws_off]) and torch.equal(arena[ws_off + need:dst_off], before_arena[ws_off + need:dst_off])
        assert torch.equal(arena[dst_off + n * m * 4:], before_arena[dst_off + n * m * 4:]), f"{name} n={n}: wrote past dst"
        y = arena[dst_off:dst_off + n * m * 4].view(torch.float32).view(n, m)
        assert torch.isfinite(y).all(), f"{name} n={n}: an output element was not written"
        assert torch.equal(y, be.mul_mat(separate(be, name, wire, k, row0, m), x.float().contiguous()))


@pytest.mark.parametrize("n", [5, 600])
def test_cuda_graph_replay_with_new_cache(be, oracle, n):
    name, k, rows_layout, m = "Q8_0", 512, 1024, 512
    t = GGML_TYPE[name]
    wire = make_wire(oracle, name, rows_layout, k, 21)
    w = be.set_tensor(t, wire, rows_layout, k)
    buf, x = cache_view(n, k, torch.float16, seed=1)
    out = torch.empty(n, m, device="cuda")
    be.mul_mat_rows(w, x, 512, m, out=out)                # warm, and size the workspace before capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.mul_mat_rows(w, x, 512, m, out=out)
    buf2, x2 = cache_view(n, k, torch.float16, seed=2)
    buf.copy_(buf2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, be.mul_mat_rows(w, x2, 512, m))


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
