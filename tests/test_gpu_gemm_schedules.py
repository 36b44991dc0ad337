"""Element-by-element tests of every prefill GEMM schedule (b200q_gemm.cu): the kernel instantiation, the tile width BN, the split-K factor and, for
MoE, the number of grouped launches are picked from the shape.  Each case of the schedule tables below names the configuration it is meant to reach;
the GPU tests run it once under torch.profiler, in a child process of its own, and assert from the trace (kernel name, template arguments, grid)
that this configuration ran, then check every output element against a same-operand reference computed once on the host.

Reference.  ref = bf16(Wd) @ bf16(x) in f64, with Wd = oracle.dequantize(wire) (the oracle, not product code) rounded to bf16 as the kernels round their
operands, and A = |bf16(Wd)| @ |bf16(x)|.  Every element must satisfy |y - ref| <= tau(K) * A + 1e-30, with

    tau(K) = 3 * K * 2^-24.

Derivation: the products of two bf16 values are exact in f32, so only the f32 additions round.  A length-K recursive sum in floating point with unit
roundoff u is within gamma_K = K u / (1 - K u) ~ K u of the exact sum, relative to sum |a_i b_i| = A (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., eq. 3.5); a blocked or split order only shortens the chains.  The tensor cores' f32 accumulation is not guaranteed to round to
nearest (chopping was measured on earlier generations: Fasi, Higham, Mikaitis, Pranesh, PeerJ CS 2021), so u = 2^-23 for the K accumulations: 2 K 2^-24.
The third K 2^-24 covers the at most 16 split-K atomics (round to nearest, K >= 1024 in every split case) and the rare weight whose bf16 operand
differs from the oracle's by one bf16 ulp (the kernels dequantise with a fused multiply-add before rounding to bf16).  The bound is a worst case: it is
not fitted to the errors observed, which stay far below it (the tests print the largest |y - ref| / (tau A) per case).

What the element check can see: an element whose true value is below tau A is indistinguishable from zero; at K = 1024 that is |ref| < 1.8e-4 A (a
random-sign sum has |ref| ~ A / sqrt(K) = 0.03 A), at K = 14336 |ref| < 2.6e-3 A.  So a single missing 64-wide k-block of one weight row is caught at
K = 1024 (test_element_check_catches_planted_defects) but may hide below the bound at K = 14336.  The NMSE bars against the exact product (unrounded
operands) stay next to the element check: they catch defects spread over many elements, such as a k-block dropped from a whole tile.

IQ2_BN on the int8 tensor pipe has its own element-wise emulation (test_gpu_parity.py::test_bitnet_int8_gemm_is_exact_integer_arithmetic, N = 300
covers its BN = 256 ragged tile).  MoE references are built per slot from the slot's expert; slots with ids outside [0, n_expert) must be exactly 0.0.

The configuration assertions hold for 132 SMs (H100 SXM); on another SM count, or when the profiler records no kernel events (no CUPTI), only that
assertion is skipped and the numerical checks still run.  Every output element is checked (no sampling): the largest reference, the DeepSeek-shaped
grouped case, is a few seconds of f64 BLAS on the host.
"""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import make_wire
from oracle.oracle import GGML_TYPE, nmse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
TAU_C = 3.0
FLOOR = 1e-30
GLU_EPILOGUE_REL = 2.0 ** -16       # silu with __expf / __fdividef in f32: <= ~30 ulp for the |gate| of these tests, x 4


def tau(k):
    return TAU_C * k * 2.0 ** -24


def bf16(a):
    """Round to bf16 (nearest, ties to even) as __float2bfloat16_rn does, returned as f64."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return r.view(np.float32).astype(np.float64)


def same_operand_reference(wb, xb):
    """ref = xb @ wb.T and A = |xb| @ |wb|.T in f64 (dst layout [N][M])"""
    return xb @ wb.T, np.abs(xb) @ np.abs(wb).T


def element_ratio(y, ref, a, k, what, bound=None):
    """max |y - ref| / bound over all elements; fails with the first offending elements when any exceeds its bound (bound: tau(k) * a + floor)"""
    y = np.asarray(y, np.float64)
    bound = tau(k) * a + FLOOR if bound is None else bound
    err = np.abs(y - ref)
    bad = np.argwhere(err > bound)
    assert len(bad) == 0, (f"{what}: {len(bad)} of {y.size} elements outside |y - ref| <= tau(K) A, first "
                           + ", ".join(f"{tuple(int(i) for i in b)}: y={y[tuple(b)]:.7g} ref={ref[tuple(b)]:.7g} bound={bound[tuple(b)]:.3g}" for b in bad[:5]))
    return float((err / bound).max())


def silu(g):
    return g / (1 + np.exp(-g))


def glu_bound(k, g, u, a_g, a_u):
    """First-order propagation of the element bounds of gate and up through silu(g) * u (sup |silu'| < 1.1), plus the f32 epilogue's rounding."""
    return tau(k) * (1.1 * a_g * np.abs(u) + np.abs(silu(g)) * a_u) + GLU_EPILOGUE_REL * np.abs(silu(g) * u) + FLOOR


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-test of the comparison (oracle and numpy only)
# ------------------------------------------------------------------------------------------------------------------------------------------------
def f32_resummation(wb, xb, bk, splits, reverse_splits):
    """The product of the bf16 operands summed in float32: k-blocks of bk accumulated in order inside each of `splits` (uneven) K ranges, the split
    partials then added in float32 (in reverse order if asked).  Returns the result and the per-split partials."""
    k = wb.shape[1]
    nblk = (k + bk - 1) // bk
    per = (nblk + splits - 1) // splits
    w32, x32 = wb.astype(np.float32), xb.astype(np.float32)
    parts = []
    for s in range(splits):
        acc = np.zeros((xb.shape[0], wb.shape[0]), np.float32)
        for b in range(s * per, min(nblk, (s + 1) * per)):
            acc += x32[:, b * bk:(b + 1) * bk] @ w32[:, b * bk:(b + 1) * bk].T
        parts.append(acc)
    y = np.zeros_like(parts[0])
    for p in (parts[::-1] if reverse_splits else parts):
        y += p
    return y, parts


def cpu_operands(oracle, name, m, k, n, seed):
    wire = make_wire(oracle, name, m, k, seed=seed)
    wd = oracle.dequantize(GGML_TYPE[name], wire, m, k)
    x = np.random.default_rng(seed).standard_normal((n, k)).astype(np.float32)
    return wd, x


def test_element_check_passes_f32_resummation_at_the_largest_k(oracle):
    """K = 14336 (the deep split-K case): two float32 summation orders unlike the kernel's (64-wide blocks in 14 splits; 16-wide blocks in 5 uneven
    splits added in reverse) both pass."""
    k = 14336
    wd, x = cpu_operands(oracle, "Q4_K", 128, k, 64, 5)
    wb, xb = bf16(wd), bf16(x)
    ref, a = same_operand_reference(wb, xb)
    for bk, splits, rev in ((64, 14, False), (16, 5, True)):
        y, _ = f32_resummation(wb, xb, bk, splits, rev)
        r = element_ratio(y, ref, a, k, f"f32 resummation bk={bk} splits={splits}")
        print(f"f32 resummation K={k} bk={bk} splits={splits}: max |y - ref| / (tau A) = {r:.3g}")
        assert r <= 1.0


def _fails(y, ref, a, k):
    try:
        element_ratio(y, ref, a, k, "planted defect")
    except AssertionError:
        return True
    return False


def test_element_check_catches_planted_defects(oracle):
    """The fused case of the table with a ragged BN = 256 tile and split-K 4 (M 384, K 1024, N 300): the clean f32 result passes; each defect a
    schedule change could cause fails."""
    m, k, n, splits = 384, 1024, 300, 4
    wd, x = cpu_operands(oracle, "Q4_K", m, k, n, 7)
    wb, xb = bf16(wd), bf16(x)
    ref, a = same_operand_reference(wb, xb)
    y, parts = f32_resummation(wb, xb, 64, splits, False)
    assert not _fails(y, ref, a, k)
    defects = {}
    d = y.copy(); d[137, 201] = 0.0; defects["one element zeroed"] = d
    d = y.copy(); d[n - 1, :] = 0.0; defects["last column of the ragged tile dropped"] = d
    d = y.copy(); d[256:n, 128:256] += parts[2][256:n, 128:256]; defects["one split added twice in one 128-row tile"] = d
    d = y.copy(); d[:, 200] -= (xb[:, 320:384] @ wb[200, 320:384]).astype(np.float32); defects["one 64-wide k-block missing from one row"] = d
    for what, d in defects.items():
        assert _fails(d, ref, a, k), what
    # MoE: two slots of different experts swapped in the output
    n_expert, n_slots = 4, 48
    experts = [bf16(cpu_operands(oracle, "IQ4_NL", 128, 512, 1, 20 + e)[0]) for e in range(n_expert)]
    xs = bf16(np.random.default_rng(3).standard_normal((n_slots, 512)).astype(np.float32))
    ids = np.arange(n_slots) % n_expert
    ref = np.stack([xs[s] @ experts[ids[s]].T for s in range(n_slots)])
    a = np.stack([np.abs(xs[s]) @ np.abs(experts[ids[s]]).T for s in range(n_slots)])
    y = ref.astype(np.float32)
    assert not _fails(y, ref, a, 512)
    d = y.copy(); d[[5, 6]] = d[[6, 5]]
    assert ids[5] != ids[6] and _fails(d, ref, a, 512), "two MoE slots swapped"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# schedule tables
# ------------------------------------------------------------------------------------------------------------------------------------------------
T = {name: str(GGML_TYPE[name]) for name in GGML_TYPE}


def gq(name, nb, grouped, grid):
    return ("k_gemm_q", (T[name], str(nb), "true" if grouped else "false"), grid)


def gb(bn, grouped, grid):
    return ("k_gemm_bf16", (str(bn), "true" if grouped else "false"), grid)


# (id, type, M, K, N, GEMM launches with 132 SMs: (kernel, template arguments, grid))
DENSE = [
    ("fused-bn256-ragged-n-split4-q4k", "Q4_K", 384, 1024, 300, [gq("Q4_K", 1, False, (3, 2, 4))]),
    ("fused-bn256-ragged-n-split4-iq4nl", "IQ4_NL", 384, 1024, 300, [gq("IQ4_NL", 1, False, (3, 2, 4))]),
    ("fused-bn256-ragged-n-no-split", "Q4_K", 4096, 1024, 300, [gq("Q4_K", 1, False, (32, 2, 1))]),
    ("fused-deep-split14", "Q4_K", 128, 14336, 64, [gq("Q4_K", 0, False, (1, 1, 14))]),
    ("fused-uneven-split-3-3-1", "IQ4_NL", 5120, 1792, 100, [gq("IQ4_NL", 0, False, (40, 1, 3))]),
    ("generic-bn256-split2-q6k", "Q6_K", 4224, 1024, 512, [gb(256, False, (33, 2, 2))]),
    ("generic-bn256-split2-iq3s", "IQ3_S", 4224, 1024, 512, [gb(256, False, (33, 2, 2))]),
    ("generic-bn256-8-column-tail", "Q6_K", 4224, 1024, 520, [gb(256, False, (33, 3, 1))]),
]

DEEPSEEK_GROUPS = [73, 73, 73, 37]         # 256 experts of 256 x 7168 bf16 (3.5 MiB each) in a 256 MiB scratch
# (id, type, n_expert, M, K, n_tokens, n_used, glu, routing, invalid ids, GEMM launches with 132 SMs)
MOE = [
    ("grouped-fused-bn256-at-threshold", "IQ4_NL", 8, 256, 512, 1024, 2, False, "random", 0, [gq("IQ4_NL", 1, True, (2, 2048 // 256 + 8, 1))]),
    ("grouped-fused-bn128-below-threshold", "IQ4_NL", 8, 256, 512, 1023, 2, False, "random", 0, [gq("IQ4_NL", 0, True, (2, 16 + 8, 1))]),
    ("grouped-generic-4-groups-one-empty", "IQ2_XXS", 256, 256, 7168, 512, 8, False, "skip-73-145", 12,
     [gb(128, True, (2, 32 + g, 1)) for g in DEEPSEEK_GROUPS]),
    ("grouped-generic-4-groups-one-empty-glu", "IQ2_XXS", 256, 256, 7168, 512, 8, True, "skip-73-145", 12,
     [gb(128, True, (2, 32 + g, 1)) for g in DEEPSEEK_GROUPS for _ in range(2)]),
    ("grouped-generic-2-groups", "Q6_K", 80, 512, 4096, 256, 2, False, "random", 6, [gb(128, True, (4, 4 + g, 1)) for g in (64, 16)]),
    ("grouped-fused-1024-experts-random", "IQ4_NL", 1024, 128, 256, 512, 4, False, "random", 10, [gq("IQ4_NL", 0, True, (1, 16 + 1024, 1))]),
    ("grouped-fused-1024-experts-one-row-each", "IQ4_NL", 1024, 128, 256, 256, 4, False, "permutation", 0, [gq("IQ4_NL", 0, True, (1, 8 + 1024, 1))]),
]


def gemm_launches(kernels):
    """(kernel, template arguments, grid) of the prefill GEMM launches among the profiled kernels, in launch order"""
    out = []
    for name, grid in kernels:
        m = re.search(r"\b(k_gemm_(?:q|bf16|bn_i8))<([^<>]*)>", name)
        if m:
            args = tuple(re.sub(r"^\((?:int|bool)\)", "", s.strip()) for s in m.group(2).split(","))
            out.append((m.group(1), args, tuple(grid)))
    return out


def profiled(fn):
    """Run fn once under torch.profiler with CUDA activities: (its result, [(kernel name, grid)] of every kernel it launched)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    return out, [(e["name"], tuple(e.get("args", {}).get("grid", ()))) for e in events if e.get("cat") == "kernel"]


def assert_schedule(case_id, expected, got):
    """Called after the numerical checks with the child's record: only the configuration assertion is skipped where it cannot hold."""
    if got["sms"] != H100_SMS:
        pytest.skip(f"{case_id}: configuration table is for {H100_SMS} SMs, this device has {got['sms']} (numerical checks passed)")
    if not got["any_kernel"]:
        pytest.skip(f"{case_id}: the profiler recorded no kernel events (CUPTI unavailable?); configuration not checked (numerical checks passed)")
    launched = [(g[0], tuple(g[1]), tuple(g[2])) for g in got["gemm"]]
    assert launched == expected, f"{case_id}: expected GEMM launches {expected}, launched {launched}"


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


def dense_operands(oracle, name, m, k, n, seed):
    wire = make_wire(oracle, name, m, k, seed=seed)
    x = np.random.default_rng(seed + 1).standard_normal((n, k)).astype(np.float32)
    return wire, x


def moe_ids(rng, routing, n_expert, n_tokens, n_used, n_invalid):
    if routing == "permutation":                        # every expert exactly one row: the maximum tile count
        assert n_tokens * n_used == n_expert
        ids = rng.permutation(n_expert).reshape(n_tokens, n_used)
    else:
        allowed = np.arange(n_expert)
        if routing == "skip-73-145":                     # the second expert group of the DeepSeek shape gets no rows
            allowed = np.concatenate([allowed[:73], allowed[146:]])
        ids = allowed[np.argsort(rng.random((n_tokens, len(allowed))), axis=1)[:, :n_used]]
    ids = ids.astype(np.int32)
    if n_invalid:                                        # skipped slots: the -1 of ggml_top_k_thresh and an id past the last expert
        bad = rng.choice(n_tokens * n_used, n_invalid, replace=False)
        ids.reshape(-1)[bad[: n_invalid // 2]] = -1
        ids.reshape(-1)[bad[n_invalid // 2:]] = n_expert
    return ids


def moe_operands(oracle, case):
    case_id, name, n_expert, m, k, n_tokens, n_used, glu, routing, n_invalid, _ = case
    rng = np.random.default_rng(n_expert + n_tokens)
    ids = moe_ids(rng, routing, n_expert, n_tokens, n_used, n_invalid)
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    wires = [make_wire(oracle, name, m, k, seed=3000 + e) for e in range(n_expert)]
    gwires = [make_wire(oracle, name, m, k, seed=5000 + e) for e in range(n_expert)] if glu else None
    return ids, x, wires, gwires


# FORCED: the deep-split fused case run with B200Q_GEMM_SPLIT set (type, M, K, N, seed)
FORCED = ("Q4_K", 128, 14336, 64, 77)


def _child(kind, case_id, out_dir):
    """One case in a process of its own: the profiler then records the kernels reliably (in a long process it sometimes returns the launches
    without the kernel records), and B200Q_GEMM_SPLIT, which the library reads once per process, can be set for it.  Saves y and the launches."""
    from oracle.oracle import Oracle
    from ik_llama_cpp_b200 import backend
    oracle = Oracle()
    if kind == "moe":
        case = next(c for c in MOE if c[0] == case_id)
        _, name, n_expert, m, k, n_tokens, n_used, glu, _, _, _ = case
        ids, x, wires, gwires = moe_operands(oracle, case)
        W = backend.set_expert_tensor(GGML_TYPE[name], np.concatenate(wires), n_expert, m, k)
        G = backend.set_expert_tensor(GGML_TYPE[name], np.concatenate(gwires), n_expert, m, k) if glu else None
        xg, idg = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
        y, kernels = profiled(lambda: backend.mul_mat_id_gemm(W, xg, idg, gate=G))
    else:
        name, m, k, n, seed = FORCED if kind == "forced" else next((c[1], c[2], c[3], c[4], dense_seed(c)) for c in DENSE if c[0] == case_id)
        wire, x = dense_operands(oracle, name, m, k, n, seed)
        w = backend.set_tensor(GGML_TYPE[name], wire, m, k)
        xg = torch.from_numpy(x).cuda()
        y, kernels = profiled(lambda: backend.mul_mat(w, xg))
    np.save(os.path.join(out_dir, "y.npy"), y.cpu().numpy())
    with open(os.path.join(out_dir, "launches.json"), "w") as f:
        json.dump({"any_kernel": bool(kernels), "gemm": gemm_launches(kernels),
                   "sms": torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count}, f)


def run_child(kind, case_id, out_dir, env=None):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), kind, case_id, str(out_dir)], capture_output=True, text=True,
                       env=env or dict(os.environ), cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    with open(os.path.join(out_dir, "launches.json")) as f:
        return np.load(os.path.join(out_dir, "y.npy")), json.load(f)


def dense_seed(case):
    return 900 + case[2] % 97 + case[4]


def check_dense(oracle, case_id, name, wire, x, m, y):
    n, k = x.shape
    wd = oracle.dequantize(GGML_TYPE[name], wire, m, k)
    ref, a = same_operand_reference(bf16(wd), bf16(x))
    r = element_ratio(y, ref, a, k, case_id)
    e = nmse(y, x.astype(np.float64) @ wd.astype(np.float64).T)
    print(f"{case_id}: max |y - ref| / (tau A) = {r:.3g}, NMSE vs exact = {e:.3g}")
    assert e <= 2e-5, f"{case_id}: NMSE {e}"
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_gemm_schedule(be, oracle, tmp_path, case):
    case_id, name, m, k, n, expected = case
    y, got = run_child("dense", case_id, tmp_path)
    wire, x = dense_operands(oracle, name, m, k, n, dense_seed(case))
    check_dense(oracle, case_id, name, wire, x, m, y)
    assert_schedule(case_id, expected, got)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MOE, ids=[c[0] for c in MOE])
def test_grouped_gemm_schedule(be, oracle, tmp_path, case):
    case_id, name, n_expert, m, k, n_tokens, n_used, glu, routing, n_invalid, expected = case
    t = GGML_TYPE[name]
    y, got = run_child("moe", case_id, tmp_path)
    y = y.reshape(n_tokens * n_used, m)
    ids, x, wires, gwires = moe_operands(oracle, case)
    flat = ids.reshape(-1)
    invalid = (flat < 0) | (flat >= n_expert)
    assert np.all(y[invalid] == 0.0), f"{case_id}: skipped slots must give exact zero rows"
    xs = x[:, 0][np.arange(n_tokens * n_used) // n_used]           # activation of every slot (nb1 = 1)
    worst, err2, ref2 = 0.0, 0.0, 0.0
    for e in np.unique(flat[~invalid]):
        sl = np.nonzero(flat == e)[0]
        xe = xs[sl]
        wd = oracle.dequantize(t, wires[e], m, k)
        ru, au = same_operand_reference(bf16(wd), bf16(xe))
        exact = xe.astype(np.float64) @ wd.astype(np.float64).T
        if glu:
            gd = oracle.dequantize(t, gwires[e], m, k)
            rg, ag = same_operand_reference(bf16(gd), bf16(xe))
            ref, bound = silu(rg) * ru, glu_bound(k, rg, ru, ag, au)
            exact = silu(xe.astype(np.float64) @ gd.astype(np.float64).T) * exact
        else:
            ref, bound = ru, tau(k) * au + FLOOR
        worst = max(worst, element_ratio(y[sl], ref, None, k, f"{case_id} expert {e}", bound=bound))
        err2 += float(((y[sl] - exact) ** 2).sum()); ref2 += float((exact ** 2).sum())
    e = err2 / ref2
    print(f"{case_id}: max |y - ref| / bound = {worst:.3g}, NMSE vs exact = {e:.3g}")
    assert e <= (2e-4 if glu else 2e-5), f"{case_id}: NMSE {e}"
    assert_schedule(case_id, expected, got)


@pytest.mark.gpu
@pytest.mark.parametrize("split,raw_blocks", [(5, "12/12/12/12/8"), (16, "4 x 14 and two empty trailing splits")])
def test_forced_split_k(be, oracle, tmp_path, split, raw_blocks):
    """K = 14336 = 56 raw blocks of 256 weights, one 128 x 128 tile: forced split 5 gives raw blocks 12/12/12/12/8, forced split 16 gives 4 per split
    and two trailing splits with no raw block (the nk <= 0 exits of k_gemm_q).  Element by element against the same reference as the table."""
    name, m, k, n, seed = FORCED
    y, got = run_child("forced", "-", tmp_path, env=dict(os.environ, B200Q_GEMM_SPLIT=str(split)))
    wire, x = dense_operands(oracle, name, m, k, n, seed)
    check_dense(oracle, f"forced split {split} ({raw_blocks})", name, wire, x, m, y)
    got["sms"] = H100_SMS                  # (a forced split does not depend on the SM count)
    assert_schedule(f"forced split {split}", [gq(name, 0, False, (1, 1, split))], got)


if __name__ == "__main__":
    _child(*sys.argv[1:4])
