"""GPU tests of MoE prefill on the tensor cores (run on the H100 with -m gpu): GGML_OP_MUL_MAT_ID / MOE_FUSED_UP_GATE as a grouped wgmma GEMM over
expert-sorted slots (b200q_mul_mat_id_gemm / the b200q_mul_mat_id dispatcher).  The oracle is the exact product on the selected expert's wire bytes.

Tolerances: the operands are bf16 with f32 accumulation, as in the dense prefill GEMM, so the dense GEMM bars apply: NMSE <= 2e-5 against the exact
result (up/gate: 2e-4, the act(gate) * up product amplifies the relative error), and NMSE <= 1e-9 against the dense GEMM on the same expert's tokens
(same operands; only a split-K summation order may differ)."""
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import make_wire
from oracle.oracle import GGML_TYPE, nmse

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FUSED_TYPES = ["IQ4_NL", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q4_K", "Q5_K", "IQ4_K", "IQ5_K"]
GENERIC_TYPES = ["Q6_K", "IQ4_XS", "IQ2_XXS", "IQ2_K_R4"]


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


def glu_ref(unary, g, u, limit=0.0):
    """act(gate) * up with the reference's order of operations (the copy in test_gpu_parity.py): the clamp follows silu and exists for silu only;
    swiglu_oai: alpha 1.702, limit 7."""
    g = np.asarray(g, np.float64); u = np.asarray(u, np.float64)
    if unary == "silu":
        a = g / (1 + np.exp(-g))
        if limit > 1e-6:
            a = np.minimum(a, limit); u = np.clip(u, -limit, limit)
        return a * u
    if unary == "gelu":
        return 0.5 * g * (1 + np.tanh(0.79788456080286535588 * g * (1 + 0.044715 * g * g))) * u
    if unary == "relu":
        return np.maximum(g, 0) * u
    if unary == "swiglu_oai":
        g = np.minimum(g, 7.0); u = np.clip(u, -7.0, 7.0)
        return g / (1 + np.exp(-1.702 * g)) * (1 + u)
    raise ValueError(unary)


def experts(be, oracle, name, n_expert, m, k, seed):
    t = GGML_TYPE[name]
    wires = [make_wire(oracle, name, m, k, seed=seed + e) for e in range(n_expert)]
    return wires, be.set_expert_tensor(t, np.concatenate(wires), n_expert, m, k)


def exact(oracle, name, wires, gwires, x, ids, m, unary="silu", limit=0.0):
    """dst[t, u] = W[ids[t, u]] . x[t, u % nb1] on the wire bytes (zero rows for ids out of range); one oracle call per expert"""
    t = GGML_TYPE[name]
    n_tokens, nb1, _ = x.shape
    n_used = ids.shape[1]
    y = np.zeros((n_tokens, n_used, m), np.float64)
    cols = x.reshape(n_tokens * nb1, -1)
    for e in range(len(wires)):
        tk, u = np.nonzero(ids == e)
        if len(tk) == 0:
            continue
        xe = cols[tk * nb1 + u % nb1]
        r = oracle.mul_mat_exact(t, wires[e], xe, m).astype(np.float64)
        if gwires is not None:
            r = glu_ref(unary, oracle.mul_mat_exact(t, gwires[e], xe, m), r, limit)
        y[tk, u] = r
    return y


@pytest.mark.parametrize("name", FUSED_TYPES + GENERIC_TYPES)
@pytest.mark.parametrize("nb1", [1, 2])
@pytest.mark.parametrize("glu", [False, True])
def test_grouped_gemm_vs_oracle(be, oracle, name, nb1, glu):
    check_grouped_gemm(be, oracle, name, nb1, glu, "silu", 0.0)


@pytest.mark.parametrize("name", FUSED_TYPES + GENERIC_TYPES)
@pytest.mark.parametrize("nb1", [1, 2])
@pytest.mark.parametrize("unary,limit", [("silu", 1.5), ("gelu", 0.0), ("relu", 0.0), ("swiglu_oai", 0.0)])
def test_grouped_gemm_glu_unary(be, oracle, name, nb1, unary, limit):
    """MOE_FUSED_UP_GATE on the grouped GEMM with the other GLUs of the reference (plain silu: test_grouped_gemm_vs_oracle).  limit (silu only)
    clamps most outputs of these shapes, so its NMSE bar follows test_gpu_parity.py::test_fused_up_gate_gemm: 1e-3."""
    check_grouped_gemm(be, oracle, name, nb1, True, unary, limit)


def check_grouped_gemm(be, oracle, name, nb1, glu, unary, limit):
    n_expert, n_used, m, k, n_tokens = 8, 2, 260, 1024, 96           # M = 260: a partial 128-row tile per expert
    wires, W = experts(be, oracle, name, n_expert, m, k, 700)
    gwires, G = experts(be, oracle, name, n_expert, m, k, 800) if glu else (None, None)
    rng = np.random.default_rng(11 + nb1)
    x = rng.standard_normal((n_tokens, nb1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    y = be.mul_mat_id_gemm(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda(), gate=G, unary=unary, limit=limit).cpu().numpy()
    e = nmse(y, exact(oracle, name, wires, gwires, x, ids, m, unary, limit))
    assert e <= (2e-5 if not glu else 2e-4 if limit == 0 else 1e-3), f"{name} nb1={nb1} glu={glu} {unary} {limit}: NMSE {e}"
    # the dispatcher takes the grouped path for this batch (96 * 2 slots > 8 per expert) and gives the same bits
    yd = be.mul_mat_id_dispatch(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda(), gate=G, unary=unary, limit=limit).cpu().numpy()
    assert np.array_equal(y, yd)


@pytest.mark.parametrize("name", ["IQ4_NL", "Q4_K", "IQ5_K", "Q6_K", "IQ2_XXS"])
def test_grouped_equals_dense_gemm_per_expert(be, oracle, name):
    """Each expert's rows of the grouped result equal the dense MUL_MAT GEMM on that expert's planes over its own tokens."""
    t = GGML_TYPE[name]
    n_expert, n_used, m, k, n_tokens = 8, 2, 260, 1024, 160
    wires, W = experts(be, oracle, name, n_expert, m, k, 900)
    rng = np.random.default_rng(5)
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    y = be.mul_mat_id_gemm(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()).cpu().numpy()
    pb = be.plane_bytes(t, m, k)
    checked = 0
    for e in range(n_expert):
        tk, u = np.nonzero(ids == e)
        if len(tk) <= 8:                     # the dense dispatcher would take the mat-vec kernel
            continue
        we = be.QuantTensor(t, m, k, W.planes[e * pb:(e + 1) * pb])
        yd = be.mul_mat(we, torch.from_numpy(np.ascontiguousarray(x[tk, 0])).cuda()).cpu().numpy()
        assert nmse(y[tk, u], yd) <= 1e-9, (name, e)
        checked += 1
    assert checked >= 6


def test_grouped_gemm_below_the_crossover(be, oracle):
    """mul_mat_id_gemm runs the grouped GEMM at any batch, also where the dispatcher takes the mat-vec and b200q_mul_mat_id_workspace is 0:
    3 experts, 1 used, 4 tokens.  Its workspace comes from b200q_mul_mat_id_gemm_workspace.  The result matches mul_mat_id (the mat-vec kernel)
    within the two paths' noise, as test_gpu_parity.py::test_gemm_llama_shape_properties, and the exact product within the grouped GEMM's bar."""
    name = "IQ4_NL"
    n_expert, n_used, m, k, n_tokens = 3, 1, 256, 2048, 4
    wires, W = experts(be, oracle, name, n_expert, m, k, 1900)
    rng = np.random.default_rng(19)
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    ids = np.array([[0], [2], [1], [2]], np.int32)
    assert be.mul_mat_id_workspace(W, n_tokens, n_used, 1, False) == 0
    be._workspaces.clear()          # sized by this call's own query, not by an earlier test's larger workspace
    xg, idg = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
    y = be.mul_mat_id_gemm(W, xg, idg).cpu().numpy()
    yv = be.mul_mat_id(W, xg, idg).cpu().numpy()
    assert nmse(y, yv) <= 1e-4
    assert nmse(y, exact(oracle, name, wires, None, x, ids, m)) <= 2e-5


@pytest.mark.parametrize("name", ["IQ4_NL", "Q6_K"])
@pytest.mark.parametrize("n_expert,n_tokens", [(256, 600), (8, 1100)])
def test_skewed_routing_and_skipped_ids(be, oracle, name, n_expert, n_tokens):
    """Every token's first slot goes to one expert (several full tiles: 128-row tiles with 256 experts, 256-row tiles with 8), the second
    slot to a few experts, most experts get nothing; ids -1 and n_expert are skipped and give zero rows."""
    n_used, m, k = 2, 256, 512
    wires, W = experts(be, oracle, name, n_expert, m, k, 1000)
    rng = np.random.default_rng(n_expert)
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    ids = np.empty((n_tokens, n_used), np.int32)
    ids[:, 0] = 3
    ids[:, 1] = rng.choice([0, 1, 5 % n_expert], n_tokens)
    bad = rng.choice(n_tokens, 40, replace=False)
    ids[bad[:20], 1] = -1
    ids[bad[20:], 0] = n_expert
    y = be.mul_mat_id_gemm(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()).cpu().numpy()
    invalid = (ids < 0) | (ids >= n_expert)
    assert np.all(y[invalid] == 0.0)
    ref = exact(oracle, name, wires, None, x, ids, m)
    assert nmse(y[~invalid], ref[~invalid]) <= 2e-5


def test_skipped_ids_give_zero_rows_with_glu(be, oracle):
    n_expert, n_used, m, k, n_tokens = 8, 2, 256, 512, 200
    wires, W = experts(be, oracle, "Q4_K", n_expert, m, k, 1100)
    gwires, G = experts(be, oracle, "Q4_K", n_expert, m, k, 1200)
    rng = np.random.default_rng(3)
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    ids[::7, 1] = -1
    y = be.mul_mat_id_gemm(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda(), gate=G).cpu().numpy()
    assert np.all(y[::7, 1] == 0.0)
    ok = ids >= 0
    assert nmse(y[ok], exact(oracle, "Q4_K", wires, gwires, x, ids, m)[ok]) <= 2e-4


@pytest.mark.parametrize("name", ["IQ4_NL", "IQ2_XXS"])
@pytest.mark.parametrize("glu", [False, True])
def test_skipped_ids_give_zero_rows_on_both_sides_of_the_dispatch_threshold(be, oracle, name, glu):
    """One set of ids with -1 and n_expert in some slots, at the last batch the dispatcher gives the mat-vec kernel (k_mmvq_id / k_wire_mmvq_id) and
    the first one it gives the grouped GEMM (thresholds mirrored by test_moe_dispatch.py): zero rows on both sides, the valid rows within each path's
    bar (mat-vec: 5e-5 of the rms against the q8_1 oracle, as test_gpu_parity.py::test_mul_mat_id; grouped: NMSE against the exact product)."""
    from test_moe_dispatch import last_mat_vec_batch
    t = GGML_TYPE[name]
    n_expert, n_used, m, k = 8, 2, 256, 512
    t_last = last_mat_vec_batch(n_expert, n_used, glu)
    wires, W = experts(be, oracle, name, n_expert, m, k, 1700)
    gwires, G = experts(be, oracle, name, n_expert, m, k, 1800) if glu else (None, None)
    rng = np.random.default_rng(17)
    x = rng.standard_normal((t_last + 1, 1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(t_last + 1)]).astype(np.int32)
    ids[0, 1] = -1
    ids[3, 0] = n_expert
    ids[t_last - 1, 1] = -1
    for n_tokens, grouped in ((t_last, False), (t_last + 1, True)):
        assert (be.mul_mat_id_workspace(W, n_tokens, n_used, 1, glu) > 0) == grouped
        xs, ids_n = x[:n_tokens], ids[:n_tokens]
        y = be.mul_mat_id_dispatch(W, torch.from_numpy(xs).cuda(), torch.from_numpy(ids_n).cuda(), gate=G).cpu().numpy()
        invalid = (ids_n < 0) | (ids_n >= n_expert)
        assert np.all(y[invalid] == 0.0), f"n_tokens={n_tokens}: skipped slots must give zero rows"
        if grouped:
            e = nmse(y[~invalid], exact(oracle, name, wires, gwires, xs, ids_n, m)[~invalid])
            assert e <= (2e-4 if glu else 2e-5), f"grouped side: NMSE {e}"
            continue
        for tk, u in zip(*np.nonzero(~invalid)):
            col = xs[tk, 0][None, :]
            ref = oracle.mul_mat_q8_1(t, wires[ids_n[tk, u]], col, m, variant="b200")[0].astype(np.float64)
            if glu:
                ref = glu_ref("silu", oracle.mul_mat_q8_1(t, gwires[ids_n[tk, u]], col, m, variant="b200")[0].astype(np.float64), ref)
            assert np.abs(y[tk, u] - ref).max() <= 5e-5 * np.sqrt((ref ** 2).mean()), (tk, u)


@pytest.mark.parametrize("name", ["IQ4_NL", "IQ2_XXS"])
def test_runs_are_bit_identical(be, oracle, name):
    n_expert, n_used, m, k, n_tokens = 16, 4, 384, 1024, 512
    _, W = experts(be, oracle, name, n_expert, m, k, 1300)
    _, G = experts(be, oracle, name, n_expert, m, k, 1400)
    rng = np.random.default_rng(8)
    x = torch.from_numpy(rng.standard_normal((n_tokens, 1, k)).astype(np.float32)).cuda()
    ids = torch.from_numpy(np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)).cuda()
    a = be.mul_mat_id_gemm(W, x, ids, gate=G)
    b = be.mul_mat_id_gemm(W, x, ids, gate=G)
    assert torch.equal(a, b)


@pytest.mark.parametrize("name,glu", [("Q4_K", True), ("IQ2_XXS", False)])
def test_dispatcher_in_a_cuda_graph_reads_ids_on_the_device(be, oracle, name, glu):
    """Capture the dispatcher, change the contents of ids in place, replay: the result equals eager execution on the new ids."""
    n_expert, n_used, m, k, n_tokens = 8, 2, 256, 1024, 128
    _, W = experts(be, oracle, name, n_expert, m, k, 1500)
    G = experts(be, oracle, name, n_expert, m, k, 1600)[1] if glu else None
    assert be.mul_mat_id_workspace(W, n_tokens, n_used, 1, glu) > 0
    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((n_tokens, 1, k)).astype(np.float32)).cuda()
    new_ids = lambda: torch.from_numpy(np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)).cuda()
    ids = new_ids()
    out = torch.empty((n_tokens, n_used, m), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.mul_mat_id_dispatch(W, x, ids, gate=G, out=out)          # warm-up: the workspace exists before the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.mul_mat_id_dispatch(W, x, ids, gate=G, out=out)
    for _ in range(2):
        ids.copy_(new_ids())
        g.replay()
        torch.cuda.synchronize()
        eager = be.mul_mat_id_dispatch(W, x, ids, gate=G)
        assert torch.equal(out, eager)


def test_backend_ops_moe_prefill_through_ggml_backend_api():
    exe = os.path.join(ROOT, "tests", "backend_ops", "test_moe_prefill_backend")
    if not os.path.exists(exe):
        pytest.skip("harness not built (needs the reference headers at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED: 0 failures" in r.stdout
