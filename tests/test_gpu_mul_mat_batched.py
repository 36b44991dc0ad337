"""Batched MUL_MAT over strided activations (b200q_mul_mat_batched): GGML_OP_MUL_MAT with ne[2] * ne[3] > 1, as DeepSeek's absorbed MLA runs it
per head (q_nope2 = wk_b x q_nope_perm, kqv = wv_b x kqv_compressed_perm).

The entry runs the MoE kernels with identity routing: token := batch entry, slot := column, ids[b][j] = b (per entry) or 0 (broadcast).  The path
(b200q_api.cu, plan_batched; cut points measured with scripts/bench_batched.py):
  * one matrix over columns a constant stride apart (broadcast with x_batch_stride == n x_col_stride, n == 1, or one entry): a plain 2-D product,
    the dense mat-vec for n n_batch <= 8, the dense GEMM for n > 8;
  * any other broadcast with n <= 8: the dense mat-vec of each entry over its strided columns;
  * the grouped MoE GEMM where it is eligible (K % 256 == 0, n_batch <= 1024) from 128 slots (n_batch n) on, for a type without a fused GEMM
    kernel only from n = 2 on;
  * otherwise k_mmvq_id / k_wire_mmvq_id after k_batch_ids up to n = 16 (one launch while the n_batch n quantised columns fit shared memory),
    one dense GEMM per entry over its strided columns above.
Bars: the mat-vec paths are held to PLAIN_BAR against oracle.mul_mat_q8_1 (test_gpu_decode_schedules.py), the GEMM paths to tau(K) A of the
same-operand bf16 reference (test_gpu_gemm_schedules.py, check_grouped of test_gpu_memory_contract.py).
"""
import numpy as np
import pytest
import torch

from conftest import ALL_TYPES, make_wire
from oracle.oracle import GGML_TYPE
from test_gpu_decode_schedules import PLAIN_BAR, bar_ratio, profiled
from test_gpu_memory_contract import check_grouped
from test_gpu_moe_decode import moe_oracle

pytestmark = pytest.mark.gpu

SMEM_COLUMNS = 200 * 1024
GROUPED_MIN_SLOTS, VEC_MAX_N = 128, 16          # b200q_api.cu: BATCHED_GROUPED_MIN_SLOTS, BATCHED_VEC_MAX_N
FUSED_GEMM = {"IQ4_NL", "Q4_0", "Q4_K", "IQ4_K", "Q4_1", "Q5_0", "Q5_1", "Q5_K", "IQ5_K"}     # b200q_gemm.cu: GEMMQ_TYPES
E_ARG, E_NOMEM = -4, -5


def max_cols(k):
    return SMEM_COLUMNS // (k + k // 4)


def expected_path(name, m, k, n, n_batch, per_entry, cs, bs):
    """the path plan_batched takes: 'one-vec', 'one-gemm', 'vec', 'grouped', 'dense'"""
    if (not per_entry or n_batch == 1) and (n == 1 or n_batch == 1 or bs == n * cs) and (n * n_batch <= 8 or n > 8):
        return "one-vec" if n * n_batch <= 8 else "one-gemm"
    if not per_entry and n <= 8:
        return "entry-vec"
    if k % 256 == 0 and (n_batch if per_entry else 1) <= 1024 and n * n_batch >= GROUPED_MIN_SLOTS and (n > 1 or name in FUSED_GEMM):
        return "grouped"
    return "vec" if n <= VEC_MAX_N and n <= max_cols(k) else "dense"


@pytest.fixture(scope="module")
def be():
    import ik_llama_cpp_b200.backend as be
    return be


def weights(be, oracle, name, n_mat, m, k, seed):
    wires = [make_wire(oracle, name, m, k, seed + e) for e in range(n_mat)]
    return wires, be.set_expert_tensor(GGML_TYPE[name], np.concatenate([np.frombuffer(w, np.uint8) if not isinstance(w, np.ndarray) else w.view(np.uint8).ravel()
                                                                          for w in wires]), n_mat, m, k)


def strided_x(n_batch, n, k, seed, pad=32, offset=64):
    """[n_batch, n, k] view as MLA's permutes make it: a [n][n_batch][k + pad] buffer (columns n_batch (k + pad) apart, entries k + pad apart) at a
    non-zero offset, the gaps NaN"""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((offset + n * n_batch * (k + pad),), float("nan"))
    v = buf[offset:].view(n, n_batch, k + pad)[:, :, :k]
    v.copy_(torch.randn(n, n_batch, k, generator=g))
    buf = buf.cuda()
    return buf, buf[offset:].view(n, n_batch, k + pad)[:, :, :k].transpose(0, 1)


def check(oracle, path, name, wires, per_entry, x, y, m, what):
    """every entry against the oracle at the bar of its path"""
    n_batch, n, k = x.shape
    ids = np.repeat(np.arange(n_batch, dtype=np.int32)[:, None], n, 1) if per_entry else np.zeros((n_batch, n), np.int32)
    n_expert = n_batch if per_entry else 1
    wire_of = lambda e: wires[e]
    if path in ("one-vec", "vec", "entry-vec"):
        ref = moe_oracle(oracle, name, wire_of, None, x, ids, n_expert, m)
        for b in range(n_batch):
            bar_ratio(y[b], ref[b], PLAIN_BAR, f"{what} entry {b}")
    else:
        check_grouped(oracle, name, wire_of, None, x, ids, n_expert, m, y, what)


def run(be, w, x, per_entry):
    y = be.mul_mat_batched(w, x, per_entry)
    torch.cuda.synchronize()
    return y


# ---- all 46 types at a small batch --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL_TYPES)
def test_all_types(be, oracle, name):
    m, k, n_batch = 64, 256, 3
    wires, w = weights(be, oracle, name, n_batch, m, k, 11)
    for n in (1, 8, 64):
        _, x = strided_x(n_batch, n, k, seed=n)
        xh = x.cpu().numpy().astype(np.float64)
        for per_entry in (True, False):
            path = expected_path(name, m, k, n, n_batch, per_entry, x.stride(1), x.stride(0))
            y = run(be, w, x, per_entry).cpu().numpy()
            assert not np.isnan(y).any()
            check(oracle, path, name, wires, per_entry, xh, y, m, f"{name} n={n} per_entry={per_entry} ({path})")


# ---- the MLA shapes ----------------------------------------------------------------------------------------------------------------------------
MLA = [("wk_b", 128, 512), ("wv_b", 512, 128)]     # (tensor, K, M)


def mla_x(which, n_tokens, n_head, k, seed):
    """the real views: q [n_tokens][n_head][192] with q_nope its first 128 floats, permuted to [n_head, n_tokens, 128]; the FA output
    [n_tokens][n_head][512] permuted to [n_head, n_tokens, 512].  Both sit at a non-zero offset of their buffer."""
    g = torch.Generator().manual_seed(seed)
    if which == "wk_b":
        buf = torch.randn(256 + n_tokens * n_head * 192, generator=g).cuda()
        return buf[256:].view(n_tokens, n_head, 192)[:, :, :128].transpose(0, 1)
    buf = torch.randn(256 + n_tokens * n_head * 512, generator=g).cuda()
    return buf[256:].view(n_tokens, n_head, 512).transpose(0, 1)


@pytest.mark.parametrize("n_head", [128, 16])
@pytest.mark.parametrize("which,k,m", MLA)
@pytest.mark.parametrize("name", ["Q8_0", "IQ4_NL"])
def test_mla_shapes(be, oracle, name, which, k, m, n_head):
    wires, w = weights(be, oracle, name, n_head, m, k, 5)
    for n in (1, 2, 8, 9, 64, 512):
        x = mla_x(which, n, n_head, k, seed=n)
        path = expected_path(name, m, k, n, n_head, True, x.stride(1), x.stride(0))
        y = run(be, w, x, True)
        # tolerance-free: the strided result equals the result on a contiguous copy of x (same path), bit for bit
        assert torch.equal(y, run(be, w, x.contiguous(), True)), f"{which} n={n}: strided != contiguous"
        heads = range(n_head) if n <= 9 else sorted(set(range(0, n_head, 16)) | {n_head - 1})
        xh = x.cpu().numpy().astype(np.float64)[list(heads)]
        check(oracle, path, name, [wires[h] for h in heads], True, xh, y.cpu().numpy()[list(heads)], m, f"{name} {which} H={n_head} n={n} ({path})")


# ---- tolerance-free identities with the MoE entry points ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["Q8_0", "IQ4_NL", "Q4_K", "IQ2_XXS"])
def test_identity_with_mul_mat_id(be, oracle, name):
    n_head, m, k = 16, 128, 512
    _, w = weights(be, oracle, name, n_head, m, k, 7)
    for n, side in ((1, "vec"), (4, "vec"), (8, "grouped"), (16, "grouped"), (64, "grouped")):
        x = mla_x("wv_b", n, n_head, k, seed=n)
        assert expected_path(name, m, k, n, n_head, True, x.stride(1), x.stride(0)) == side
        ids = torch.arange(n_head, dtype=torch.int32, device="cuda")[:, None].repeat(1, n).contiguous()
        xc = x.contiguous()
        ref = be.mul_mat_id(w, xc, ids) if side == "vec" else be.mul_mat_id_gemm(w, xc, ids)
        assert torch.equal(run(be, w, x, True), ref), f"{name} n={n}: batched != b200q_mul_mat_id_{side} with identity ids"


# ---- memory contract on a guarded arena ---------------------------------------------------------------------------------------------------------
def _lib():
    import ik_llama_cpp_b200 as pkg
    return pkg.lib()


@pytest.mark.parametrize("n", [1, 8, 64, 512])
@pytest.mark.parametrize("which,k,m", MLA)
def test_memory_contract(be, oracle, which, k, m, n):
    name, n_head = "Q8_0", 16
    _, w = weights(be, oracle, name, n_head, m, k, 3)
    t = GGML_TYPE[name]
    L = _lib()
    pad = 32
    cs, bs = n_head * (k + pad), k + pad
    need = int(L.b200q_mul_mat_batched_workspace(t, m, k, n, n_head, 1, cs, bs))
    guard = 1 << 20
    x_elems, y_elems = n * cs, n_head * n * m
    # [guard][x][guard][dst][guard][workspace][guard], 256-byte aligned regions; NaN everywhere but the x columns
    off_x = guard // 4
    off_y = off_x + ((x_elems + 63) // 64) * 64 + guard // 4
    off_ws = off_y + ((y_elems + 63) // 64) * 64 + guard // 4
    total = off_ws + ((need + 255) // 256) * 64 + guard // 4
    arena = torch.full((total,), float("nan"), device="cuda")
    g = torch.Generator().manual_seed(n)
    xv = arena[off_x:off_x + x_elems].view(n, n_head, k + pad)[:, :, :k]
    xv.copy_(torch.randn(n, n_head, k, generator=g).cuda())
    x = xv.transpose(0, 1)
    stream = torch.cuda.current_stream().cuda_stream

    def call(ws_bytes, col_stride=cs):
        return L.b200q_mul_mat_batched(t, w.ptr, 1, x.data_ptr(), col_stride, bs, arena.data_ptr() + 4 * off_y, m, k, n, n_head,
                                       arena.data_ptr() + 4 * off_ws, ws_bytes, stream)

    before = arena.clone()
    # a short workspace and a bad stride are rejected and write nothing
    if need:
        assert call(need - 1) == E_NOMEM
    assert call(need, col_stride=cs + 2) == E_ARG
    assert call(need, col_stride=k - 4 if n > 1 else -4) == E_ARG
    torch.cuda.synchronize()
    assert torch.equal(before.view(torch.int32), arena.view(torch.int32)), "a rejected call wrote memory"
    assert call(need) == 0
    torch.cuda.synchronize()
    y = arena[off_y:off_y + y_elems].clone()
    assert not torch.isnan(y).any(), "a dst element was not written"
    writable = torch.zeros(total, dtype=torch.bool, device="cuda")
    writable[off_y:off_y + y_elems] = True
    writable[off_ws:off_ws + (need + 3) // 4] = True
    assert torch.equal(before.view(torch.int32)[~writable], arena.view(torch.int32)[~writable]), "a byte outside dst and the workspace changed"
    # the NaN gaps between the strided columns are never read: the result equals the run on a clean contiguous copy
    assert torch.equal(y.view(n_head, n, m), be.mul_mat_batched(w, x.contiguous(), True)), "the result depends on the gaps between the columns"


# ---- launches --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_head", [16, 128])
@pytest.mark.parametrize("which,k,m", MLA)
def test_decode_is_one_mat_vec_launch(be, oracle, which, k, m, n_head):
    _, w = weights(be, oracle, "Q8_0", n_head, m, k, 9)
    x = mla_x(which, 1, n_head, k, seed=1)
    run(be, w, x, True)
    _, kernels = profiled(lambda: be.mul_mat_batched(w, x, True))
    names = [kn for kn, _, _ in kernels]
    assert len(names) == 2 and "k_batch_ids" in names[0] and "k_mmvq_id" in names[1], names


@pytest.mark.parametrize("n,kernel", [(64, "k_moe_route"), (512, "k_moe_route")])
def test_prefill_takes_the_grouped_gemm(be, oracle, n, kernel):
    n_head, k, m = 16, 512, 128
    _, w = weights(be, oracle, "Q8_0", n_head, m, k, 9)
    x = mla_x("wv_b", n, n_head, k, seed=2)
    run(be, w, x, True)
    _, kernels = profiled(lambda: be.mul_mat_batched(w, x, True))
    names = [kn for kn, _, _ in kernels]
    assert "k_batch_ids" in names[0] and any(kernel in s for s in names) and not any("k_mmvq_id" in s for s in names), names


def test_wk_b_prefill_is_one_gemm_per_head(be, oracle):
    n_head, k, m, n = 16, 128, 512, 32
    _, w = weights(be, oracle, "Q8_0", n_head, m, k, 9)
    x = mla_x("wk_b", n, n_head, k, seed=3)
    run(be, w, x, True)
    _, kernels = profiled(lambda: be.mul_mat_batched(w, x, True))
    names = [kn for kn, _, _ in kernels]
    assert not any("k_batch_ids" in s or "k_moe_route" in s for s in names), names
    assert sum("k_f32_to_bf16" in s for s in names) == n_head, names


def test_wk_b_at_16_columns_is_the_mat_vec_in_entry_chunks(be, oracle):
    n_head, k, m, n = 128, 128, 512, 16
    _, w = weights(be, oracle, "Q8_0", n_head, m, k, 9)
    x = mla_x("wk_b", n, n_head, k, seed=3)
    run(be, w, x, True)
    _, kernels = profiled(lambda: be.mul_mat_batched(w, x, True))
    names = [kn for kn, _, _ in kernels]
    chunk = max_cols(k) // n            # entries per launch
    assert "k_batch_ids" in names[0] and sum("k_mmvq_id" in s for s in names) == -(-n_head // chunk) == len(names) - 1, names


# ---- CUDA graphs ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 64])
@pytest.mark.parametrize("which,k,m", MLA)
def test_cuda_graph_replay(be, oracle, which, k, m, n):
    n_head = 16
    _, w = weights(be, oracle, "IQ4_NL", n_head, m, k, 13)
    x = mla_x(which, n, n_head, k, seed=4)
    out = torch.empty((n_head, n, m), device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.mul_mat_batched(w, x, True, out=out)           # warm-up: workspace and kernel attributes outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        be.mul_mat_batched(w, x, True, out=out)
    for seed in (5, 6):
        g = torch.Generator().manual_seed(seed)
        x.copy_(torch.randn(x.shape, generator=g).cuda())     # in place, through the strided view
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, run(be, w, x, True)), f"replay with new x (seed {seed}) differs from the eager call"
