"""Where every mat-mul entry point writes and what it reads: the memory contract of include/b200q.h.

The schedule suites check what each kernel computes.  This file checks the other half of a kernel's correctness: that a call writes only its
outputs, its extra outputs and at most the workspace bytes the query (or the header) names, that it leaves its inputs alone, and that its result
does not depend on what the output and workspace memory held before.  The backend wrappers cannot show this: they hand the kernels a grow-only
workspace and fresh allocations.  So every call here goes through the C ABI on a non-default stream with operands carved out of ONE device buffer,
the arena, in 256-byte aligned regions (the alignment of ggml's buffers), with guards between them:

    guard | dst[0] | guard | dst[1] | guard | dst[2] | guard | extra outputs | guard | workspace (exactly the queried bytes) | guard | x | guard | ids | ...

Each guard is at least max(1 MiB, 256 rows x M x 4 bytes), so a 128- or 256-row tile stored one tile too far stays inside the allocation.  The
weights are uploaded with set_tensor / set_expert_tensor and copied into the arena with a guard after the last plane.  Q, K and V outputs are
neighbours with only a guard between them, as the outputs of one multi-tensor launch are in ggml's compute buffer.

Fill values.  A correct kernel reads none of them; a wrong read shows in the values and can never become an out-of-range index:
  * guards and f32 / bf16 regions: the word 0x7FC07FC0, a quiet NaN read as f32 and two quiet NaNs read as bf16;
  * the guards on either side of an ids region: int32 -1, the "skipped" id (a zero row, no weight read);
  * weight guards: NaN bytes (every payload bit pattern is a valid encoding, and a NaN scale shows in the output);
  * MoE workspaces are never NaN-filled (their index tables would become wild addresses): run B below leaves them stale but valid.

Checks of every call:
  1. the return code is 0;
  2. every byte outside the call's outputs and workspace is unchanged: the guards, and W, x, ids, bias, x_bf16 and the q8 image it reads;
  3. no output element is still NaN, so every element was written (skipped-id rows compare == 0.0, which means something on NaN-filled memory);
  4. the result does not depend on prior memory: run A (outputs NaN, workspace zero) and run B (outputs 1e30, workspace as a previous DIFFERENT
     valid call left it: another N for the dense paths; other ids with more routed rows, and another tile width where the shape allows it, for
     MoE) are bit-identical.  Exempt: the split-K GEMMs, whose f32 atomics may add the K partials in another order.  Those are the GEMM launches
     with a split (grid z > 1) in the tables: DENSE split4 (two types), split14, uneven-split-3-3-1, split2 (two types), the n = 9 decode boundary
     cases, the forced splits, and the _bf16 entry points below.  There each run is held on its own to the element bound tau(K) A of
     test_gpu_gemm_schedules.py;
  5. the values are right: run A against the oracle with the existing checkers (imported, not copied);
  6. a workspace one byte short: the call returns B200Q_E_NOMEM and writes nothing at all, outputs, workspace and guards included.

Cases: every configuration of the schedule tables (SCHEDULES, MOE_SCHEDULES, DENSE, MOE, the forced split-K, the merged up/gate IDENTITY shapes), the
MoE grouped path once more in the backend plug's own layout (workspace of exactly `need` bytes with the gathered ids at align256(need), no guard
between: an overrun corrupts the ids the next launch routes), and the entry points no table reaches.  On the mat-vec path the MoE query is 0 and the
plug's block holds only the ids, so that layout adds nothing there.

The CPU self-test emulates one call on a host arena and shows that the checker rejects each kind of defect it is meant to find.
"""
import ctypes
import os
import subprocess
import sys
from ctypes import c_int64, c_void_p

import numpy as np
import pytest
import torch

from conftest import ALL_TYPES, make_wire
from oracle.oracle import GGML_TYPE
from test_gpu_decode_schedules import SCHEDULES, case_operands, check_calls, check_q8_image, glu_ratio, plain_ratio
from test_gpu_gemm_schedules import (DENSE, FLOOR, FORCED, GLU_EPILOGUE_REL, MOE, bf16, check_dense, dense_operands, dense_seed, element_ratio,
                                     glu_bound, moe_ids, moe_operands, same_operand_reference, silu, tau)
from test_gpu_moe_decode import MOE_SCHEDULES, CaseData, check_slots, moe_oracle
from test_gpu_moe_merged import IDENTITY, inputs as merged_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN_WORD = 0x7FC07FC0
GARBAGE_WORD = int(np.float32(1e30).view(np.int32))
E_NOMEM = -5
SILU = 1


def align256(n):
    return (int(n) + 255) // 256 * 256


def lib():
    from ik_llama_cpp_b200 import _lib
    return _lib.lib()


def last_error():
    try:
        return lib().b200q_last_error().decode(errors="replace")
    except Exception as e:          # (the CPU self-test has no library call behind its return codes)
        return repr(e)


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the arena and the contract driver (device agnostic: the CPU self-test runs them on a host tensor)
# ------------------------------------------------------------------------------------------------------------------------------------------------
class Arena:
    """One buffer carved into 256-byte aligned regions with guards between them.  kind: "in" (read-only operand), "ids" (read-only int32 ids:
    the guards next to it hold -1), "out" (an output), "ws" (a workspace).  guard=False puts the next region right at align256(end)."""

    def __init__(self, m_rows=0, device="cuda"):
        self.device = device
        self.guard = max(1 << 20, 256 * int(m_rows) * 4)
        self.regions = {}
        self.order = []
        self.end = self.guard
        self.buf = None

    def add(self, name, nbytes, kind, guard=True):
        off = align256(self.end)
        self.regions[name] = (off, int(nbytes), kind)
        self.order.append(name)
        self.end = off + int(nbytes) + (self.guard if guard else 0)

    def build(self):
        self.buf = torch.empty(align256(self.end + self.guard), dtype=torch.uint8, device=self.device)
        self.buf.view(torch.int32).fill_(NAN_WORD)
        for i, name in enumerate(self.order):
            off, n, kind = self.regions[name]
            if kind == "ids":                              # both neighbouring gaps read as int32 -1
                lo = self.regions[self.order[i - 1]][0] + self.regions[self.order[i - 1]][1] if i else 0
                hi = self.regions[self.order[i + 1]][0] if i + 1 < len(self.order) else self.buf.numel()
                self.buf[lo:hi].fill_(255)
        return self

    def ptr(self, name):
        return self.buf.data_ptr() + self.regions[name][0]

    def nbytes(self, name):
        return self.regions[name][1]

    def raw(self, name):
        off, n, _ = self.regions[name]
        return self.buf[off:off + n]

    def put(self, name, data):
        src = data if isinstance(data, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(data))
        src = src.reshape(-1).view(torch.uint8)
        assert src.numel() == self.nbytes(name), (name, src.numel(), self.nbytes(name))
        self.raw(name).copy_(src)

    def fill(self, name, word):
        n = self.nbytes(name)
        self.raw(name).copy_(torch.full(((n + 3) // 4,), word, dtype=torch.int32, device=self.device).view(torch.uint8)[:n])

    def get(self, name, dtype, shape):
        """a host copy of a region: f32 -> float32, bf16 -> uint16 bits, u8 -> uint8"""
        tdt = {"f32": torch.float32, "bf16": torch.int16, "u8": torch.uint8, "i32": torch.int32}[dtype]
        a = self.raw(name).view(tdt).reshape(shape).cpu().numpy().copy()
        return a.view(np.uint16) if dtype == "bf16" else a

    def where(self, i):
        for name in self.order:
            off, n, _ = self.regions[name]
            if off <= i < off + n:
                return f"{name}+{i - off}"
        before = [nm for nm in self.order if self.regions[nm][0] + self.regions[nm][1] <= i]
        return f"guard after {before[-1]} (+{i - sum(self.regions[before[-1]][:2])})" if before else f"leading guard +{i}"

    def untouched(self, snap, writable, what):
        """every byte outside the `writable` regions equals the snapshot"""
        diff = self.buf != snap
        for name in writable:
            off, n, _ = self.regions[name]
            diff[off:off + n] = False
        if bool(diff.any()):
            idx = torch.nonzero(diff).flatten()
            raise AssertionError(f"{what}: {idx.numel()} bytes outside the outputs and the workspace changed, first at "
                                 + ", ".join(self.where(int(i)) for i in idx[:6].cpu()))


def bf16_nan(bits):
    return ((bits & 0x7F80) == 0x7F80) & ((bits & 0x7F) != 0)


def run_contract(arena, outs, call, what, ws=None, ws_bytes=0, stale=None, exact_ab=True, short=False, keep=(), sync=None):
    """Checks 1-4 and 6 of the module docstring for one call.  outs: [(region, "f32" | "bf16" | "u8", shape)] written by call(ws_bytes) -> rc;
    keep: outputs that are NOT refilled between the runs (the q8 image, which carries its counters); ws: the workspace region; stale(): a
    different valid call that leaves the workspace as run B finds it.  Returns (run A, run B) as dicts of host arrays."""
    sync = sync or torch.cuda.synchronize
    writable = [o[0] for o in outs] + [o[0] for o in keep] + ([ws] if ws else [])
    runs = []
    for run in "AB":
        if run == "B" and stale is not None:
            stale()
        for name, _, _ in outs:
            arena.fill(name, NAN_WORD if run == "A" else GARBAGE_WORD)
        if ws and run == "A":
            arena.fill(ws, 0)
        snap = arena.buf.clone()
        rc = call(ws_bytes)
        sync()
        assert rc == 0, f"{what} run {run}: rc {rc}: {last_error()}"
        arena.untouched(snap, writable, f"{what} run {run}")
        res = {name: arena.get(name, dt, shape) for name, dt, shape in list(outs) + list(keep)}
        if run == "A":
            for name, dt, _ in outs:
                left = np.isnan(res[name]) if dt == "f32" else bf16_nan(res[name]) if dt == "bf16" else np.zeros(0, bool)
                assert not left.any(), (f"{what}: {int(left.sum())} elements of {name} are still NaN (never written, or computed from the NaN the "
                                        f"output held), first {np.argwhere(left)[:4].tolist()}")
        runs.append(res)
    a, b = runs
    if exact_ab:
        for name in a:
            assert np.array_equal(a[name].view(np.uint8), b[name].view(np.uint8)), \
                f"{what}: {name} differs between run A (outputs NaN, workspace zero) and run B (outputs 1e30, stale workspace)"
    if short:
        snap = arena.buf.clone()
        rc = call(ws_bytes - 1)
        sync()
        assert rc == E_NOMEM, f"{what}: a workspace of {ws_bytes - 1} bytes (one short) returned {rc}, expected B200Q_E_NOMEM ({E_NOMEM})"
        arena.untouched(snap, [], f"{what}: the error return with a workspace one byte short")
    print(f"{what}: contract kept; runs A and B {'bit-equal' if exact_ab else 'each checked against the element bound (split-K)'}"
          + (f"; short workspace -> {E_NOMEM}" if short else ""))
    return a, b


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-test
# ------------------------------------------------------------------------------------------------------------------------------------------------
SELF_DEFECTS = ["store past dst[0]", "element left unwritten", "byte past the workspace", "x modified in place", "accumulates into dst",
                "reads the stale workspace", "writes dst before the workspace check"]


def _emulated_case(defect):
    """One call on a host arena: dst[0] = dst[1] = x W^T (f32 of the exact product), the kernel first stages x in a workspace of exactly
    n k 4 bytes and computes from there.  Raises AssertionError where the checker rejects the call."""
    m, k, n = 40, 64, 6
    rng = np.random.default_rng(1)
    w, x, x2 = (rng.standard_normal(s).astype(np.float32) for s in ((m, k), (n, k), (n, k)))
    ar = Arena(m, device="cpu")
    for name, nb, kind in (("y0", n * m * 4, "out"), ("y1", n * m * 4, "out"), ("ws", n * k * 4, "ws"), ("x", n * k * 4, "in"), ("W", m * k * 4, "in")):
        ar.add(name, nb, kind)
    ar.build()
    ar.put("x", x)
    ar.put("W", w)
    host = ar.buf.numpy()

    def f32(name):
        off, nb, _ = ar.regions[name]
        return host[off:off + nb].view(np.float32)

    def call(wsb):
        y0, y1, ws, xa = f32("y0"), f32("y1"), f32("ws"), f32("x")
        if defect == "writes dst before the workspace check":
            y0[:] = 0.0
        if wsb < n * k * 4:
            return E_NOMEM
        stale = ws[0]
        ws[:] = xa
        xs = ws.reshape(n, k).copy()
        if defect == "reads the stale workspace":
            xs[0, 0] = stale
        y = (xs.astype(np.float64) @ w.astype(np.float64).T).astype(np.float32).reshape(-1)
        for d in (y0, y1):
            d[:] = d + y if defect == "accumulates into dst" else y
        if defect == "store past dst[0]":
            end = ar.regions["y0"][0] + n * m * 4
            host[end:end + 4] = y[:1].view(np.uint8)
        if defect == "byte past the workspace":
            host[ar.regions["ws"][0] + n * k * 4] = 0
        if defect == "x modified in place":
            xa[3] = 0.0
        return 0

    if defect == "element left unwritten":         # the kernel skips one element: its store never happens
        inner = call

        def call(wsb):
            keep = f32("y0")[7].copy()
            rc = inner(wsb)
            f32("y0")[7] = keep
            return rc

    def stale():
        f32("ws")[:] = x2.reshape(-1)
    a, _ = run_contract(ar, [("y0", "f32", (n, m)), ("y1", "f32", (n, m))], call, f"emulated ({defect or 'clean'})", ws="ws", ws_bytes=n * k * 4,
                        stale=stale, short=True, sync=lambda: None)
    ref = x.astype(np.float64) @ w.astype(np.float64).T
    for name in ("y0", "y1"):
        element_ratio(a[name], ref, np.abs(x.astype(np.float64)) @ np.abs(w.astype(np.float64)).T, k, f"emulated {name}")


def test_checker_catches_planted_defects():
    """The clean emulated call passes; each planted defect is rejected."""
    _emulated_case(None)
    for defect in SELF_DEFECTS:
        with pytest.raises(AssertionError):
            _emulated_case(defect)


# ------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: helpers
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


@pytest.fixture
def side_stream(be):
    """every call of a test, and every fill and copy of its arena, on one non-default stream"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yield s


def st():
    return torch.cuda.current_stream().cuda_stream


def ok(rc, what):
    assert rc == 0, f"{what}: rc {rc}: {last_error()}"


def bf16_bits(a):
    """bf16 (nearest, ties to even) bit patterns of an f32 array"""
    return (bf16(a).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def in_child(kind, arg, env):
    """a case whose library option is read once per process (B200Q_GEMM_SPLIT, B200Q_MOE_CHUNK_TOKENS), in a process of its own"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), kind, arg], capture_output=True, text=True, env={**os.environ, **env}, cwd=ROOT,
                       timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def check_grouped(oracle, name, wire_of, gate_of, x, ids, n_expert, m, y, what):
    """Grouped GEMM result: skipped slots exact zero rows, every other slot within tau(K) A of the same-operand reference of its expert (up/gate:
    glu_bound), as test_gpu_gemm_schedules.py holds the grouped schedules.  Returns the worst ratio to the bound."""
    t = GGML_TYPE[name]
    n_tokens, nb1, k = x.shape
    n_used = ids.shape[1]
    flat = ids.reshape(-1)
    y = np.asarray(y).reshape(n_tokens * n_used, m)
    invalid = (flat < 0) | (flat >= n_expert)
    assert np.all(y[invalid] == 0.0), f"{what}: skipped slots must be exact zero rows"
    s = np.arange(n_tokens * n_used)
    xs = x.reshape(n_tokens * nb1, k)[(s // n_used) * nb1 + (s % n_used) % nb1]
    worst = 0.0
    for e in np.unique(flat[~invalid]):
        sl = np.nonzero(flat == e)[0]
        xb = bf16(xs[sl])
        ru, au = same_operand_reference(bf16(oracle.dequantize(t, wire_of(e), m, k)), xb)
        if gate_of is None:
            ref, bound = ru, tau(k) * au + FLOOR
        else:
            rg, ag = same_operand_reference(bf16(oracle.dequantize(t, gate_of(e), m, k)), xb)
            ref, bound = silu(rg) * ru, glu_bound(k, rg, ru, ag, au)
        worst = max(worst, element_ratio(y[sl], ref, None, k, f"{what} expert {e}", bound=bound))
    return worst


def moe_stale(L, t, W, G, n_expert, m, k, n_used, n_tokens, ws, merged=False):
    """A different valid grouped call on the same workspace, run before run B: every id routed (more routed rows than the case, whose ids skip
    some), other activations, and half the tokens where that changes the tile width (BN = 256 once an expert averages 256 rows).  Its bounds,
    tile table and gather map are then stale but in range."""
    n2 = n_tokens // 2 if n_tokens * n_used >= 256 * n_expert else n_tokens
    rng = np.random.default_rng([n_tokens, n_expert, 7])
    ids2 = torch.from_numpy(moe_ids(rng, "random", n_expert, n2, n_used, 0)).cuda()
    x2 = torch.from_numpy(rng.standard_normal((n2, 1, k)).astype(np.float32)).cuda()
    y2 = torch.empty((n2, n_used, m), device="cuda")

    def stale():
        if merged:
            need2 = L.b200q_moe_up_gate_merged_workspace(t, m, k, n_used, 1, n2, n_expert)
            rc = L.b200q_moe_up_gate_merged(t, W, n_expert, ids2.data_ptr(), x2.data_ptr(), y2.data_ptr(), m, k, n_used, 1, n2, SILU, 0.0, ws, need2, st())
        else:
            need2 = L.b200q_mul_mat_id_workspace(t, m, k, n_used, 1, n2, n_expert, int(G is not None))
            rc = L.b200q_mul_mat_id_gemm(t, W, G, n_expert, ids2.data_ptr(), x2.data_ptr(), y2.data_ptr(), m, k, n_used, 1, n2, SILU, 0.0, ws, need2, st())
        assert need2 > 0
        ok(rc, "the stale call before run B")
    return stale


# ------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the schedule tables
# ------------------------------------------------------------------------------------------------------------------------------------------------
def run_decode_case(be, oracle, case):
    """Every call of a SCHEDULES case: x (strided x: NaN padding), outputs (a multi launch's three side by side), the q8 image and, for the n = 9
    GEMM, its workspace in one arena."""
    case_id, name, shapes, calls, _ = case
    t = GGML_TYPE[name]
    L = lib()
    wires, xs = case_operands(oracle, case)
    ar = Arena(max(m for m, _ in shapes))
    plan = []
    for i, (c, x) in enumerate(zip(calls, xs)):
        op, (n, k) = c[0], x.shape
        js = [c[1]] if isinstance(c[1], int) else list(c[1])
        ms = [shapes[j][0] for j in js] if op == "multi" else [shapes[js[0]][0], shapes[js[2]][0]] if op == "q8" else [shapes[js[0]][0]]
        for s, mm in enumerate(ms):
            ar.add(f"y{i}_{s}", n * mm * 4, "out")
        need = 0
        if n > 8:
            assert op == "mm", "the table's GEMM calls are plain mul_mat"
            need = L.b200q_mul_mat_workspace(t, ms[0], k, n)
            ar.add(f"ws{i}", need, "ws")
        if op == "q8":
            ar.add(f"q8{i}", L.b200q_q8_scratch_bytes(ms[0]), "out")
        xstride = k + 64 if op == "mm_strided" else k
        ar.add(f"x{i}", n * xstride * 4, "in")
        plan.append((op, js, n, k, xstride, ms, need))
    for j, (m, k) in enumerate(shapes):
        ar.add(f"W{j}", be.plane_bytes(t, m, k), "in")
    ar.build()
    for j, (w, (m, k)) in enumerate(zip(wires, shapes)):
        ar.put(f"W{j}", be.set_tensor(t, w, m, k).planes)
    for i, x in enumerate(xs):
        xp = np.full((x.shape[0], plan[i][4]), np.nan, np.float32)       # the padding of a strided x is NaN: it must not reach the output
        xp[:, :x.shape[1]] = x
        ar.put(f"x{i}", xp)
    ys_a, ys_b, q8_valid, split = {}, {}, [], False
    for i, (op, js, n, k, xstride, ms, need) in enumerate(plan):
        W = [ar.ptr(f"W{j}") for j in js]
        x, y0 = ar.ptr(f"x{i}"), ar.ptr(f"y{i}_0")
        ws = ar.ptr(f"ws{i}") if need else None
        outs = [(f"y{i}_{s}", "f32", (n, mm)) for s, mm in enumerate(ms)]
        keep, produced, stale = [], [None], None
        if op == "mm":
            def call(b):
                return L.b200q_mul_mat(t, W[0], x, y0, ms[0], k, n, ws, b, st())
            if need:                                    # another N (the table's n = 9 has no smaller GEMM batch: then other values)
                n2 = max(9, n // 2 + 1)
                x2, y2 = torch.randn(n2, k, device="cuda"), torch.empty(n2, ms[0], device="cuda")
                stale = lambda: ok(L.b200q_mul_mat(t, W[0], x2.data_ptr(), y2.data_ptr(), ms[0], k, n2, ws, L.b200q_mul_mat_workspace(t, ms[0], k, n2), st()),
                                   "stale call")
        elif op == "mm_strided":
            def call(b):
                return L.b200q_mul_mat_vec(t, W[0], x, y0, ms[0], k, n, xstride, None, st())
        elif op == "ug":
            def call(b):
                return L.b200q_fused_up_gate(t, W[0], W[1], x, y0, ms[0], k, n, SILU, 0.0, ws, b, st())
        elif op == "multi":
            Wp, Dp, Mp = (c_void_p * len(js))(*W), (c_void_p * len(js))(*[ar.ptr(o[0]) for o in outs]), (c_int64 * len(js))(*ms)

            def call(b):
                return L.b200q_mul_mat_multi(t, len(js), Wp, Dp, Mp, k, x, n, ws, b, st())
        else:
            q8 = ar.ptr(f"q8{i}")
            keep = [(f"q8{i}", "u8", (ar.nbytes(f"q8{i}"),))]
            ok(L.b200q_q8_scratch_init(q8, ms[0], st()), "b200q_q8_scratch_init")

            def call(b):
                p = ctypes.c_int32(0)
                rc = L.b200q_fused_up_gate_vec_q8(t, W[0], W[1], x, y0, ms[0], k, SILU, 0.0, q8, ctypes.byref(p), st())
                produced[0] = bool(p.value)
                return rc or L.b200q_mul_mat_vec_q8(t, W[2], y0, q8 if p.value else None, ar.ptr(f"y{i}_1"), ms[1], ms[0], None, st())
        a, b = run_contract(ar, outs, call, f"{case_id} call {i} ({op}, n = {n})", ws=f"ws{i}" if need else None, ws_bytes=need, stale=stale,
                            exact_ab=n <= 8, short=bool(need), keep=keep)
        split |= n > 8                                  # the n = 9 GEMMs of the table run split-K (grid z = 4)
        for run, ys in ((a, ys_a), (b, ys_b)):
            ys.update({key: v for key, v in run.items() if key.startswith("y")})
            if op == "q8":
                ys[f"q8img{i}"] = run[f"q8{i}"]
        q8_valid.append(produced[0] if op == "q8" else None)
    for what, r in check_calls(oracle, case, wires, xs, ys_a, q8_valid):
        print(f"{what}: max ratio to the bar = {r:.3g}")
    if split:
        check_calls(oracle, case, wires, xs, ys_b, q8_valid)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SCHEDULES, ids=[c[0] for c in SCHEDULES])
def test_decode_schedule_contract(be, oracle, side_stream, case):
    run_decode_case(be, oracle, case)


def run_moe_decode_case(be, oracle, case):
    case_id, name, n_expert, n_used, shapes, calls, _, _ = case
    t = GGML_TYPE[name]
    L = lib()
    data = CaseData(oracle, case)
    ar = Arena(max(m for m, _ in shapes))
    for i, (entry, j, n_tokens, nb1, glu) in enumerate(calls):
        m, k = shapes[j]
        ar.add(f"y{i}", n_tokens * n_used * m * 4, "out")
        if entry == "disp":
            assert L.b200q_mul_mat_id_workspace(t, m, k, n_used, nb1, n_tokens, n_expert, int(glu)) == 0, "the table's calls take the mat-vec"
        ar.add(f"x{i}", n_tokens * nb1 * k * 4, "in")
        ar.add(f"ids{i}", n_tokens * n_used * 4, "ids")
    tensors = sorted({(j, g) for _, j, _, _, glu in calls for g in ((False, True) if glu else (False,))})
    for j, g in tensors:
        ar.add(f"W{j}{int(g)}", n_expert * be.plane_bytes(t, *shapes[j]), "in")
    ar.build()
    for j, g in tensors:
        ar.put(f"W{j}{int(g)}", be.set_expert_tensor(t, np.concatenate([data.wire(j, g, e) for e in range(n_expert)]), n_expert, *shapes[j]).planes)
    for i in range(len(calls)):
        ar.put(f"x{i}", data.xs[i])
        ar.put(f"ids{i}", data.ids[i])
    for i, (entry, j, n_tokens, nb1, glu) in enumerate(calls):
        m, k = shapes[j]
        W, G = ar.ptr(f"W{j}0"), (ar.ptr(f"W{j}1") if glu else None)
        args = (n_expert, ar.ptr(f"ids{i}"), ar.ptr(f"x{i}"), ar.ptr(f"y{i}"), m, k, n_used, nb1, n_tokens, SILU, 0.0)

        def call(b):
            return L.b200q_mul_mat_id_vec(t, W, G, *args, st()) if entry == "vec" else L.b200q_mul_mat_id(t, W, G, *args, None, 0, st())
        what = f"{case_id} call {i} ({entry}, {n_tokens} tokens, nb1 = {nb1}{', up/gate' if glu else ''})"
        a, _ = run_contract(ar, [(f"y{i}", "f32", (n_tokens, n_used, m))], call, what)
        ref = moe_oracle(oracle, name, lambda e: data.wire(j, False, e), (lambda e: data.wire(j, True, e)) if glu else None,
                         data.xs[i], data.ids[i], n_expert, m)
        print(f"{what}: max ratio to the bar = {check_slots(a[f'y{i}'], ref, data.ids[i], n_expert, glu, what):.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", MOE_SCHEDULES, ids=[c[0] for c in MOE_SCHEDULES])
def test_moe_decode_schedule_contract(be, oracle, side_stream, case):
    if case[6]:
        in_child("moe_decode", case[0], case[6])
    else:
        run_moe_decode_case(be, oracle, case)


def run_dense_case(be, oracle, name, m, k, n, seed, split, what):
    t = GGML_TYPE[name]
    L = lib()
    wire, x = dense_operands(oracle, name, m, k, n, seed)
    need = L.b200q_mul_mat_workspace(t, m, k, n)
    ar = Arena(m)
    for region, nb, kind in (("y", n * m * 4, "out"), ("ws", need, "ws"), ("x", x.nbytes, "in"), ("W", be.plane_bytes(t, m, k), "in")):
        ar.add(region, nb, kind)
    ar.build()
    ar.put("W", be.set_tensor(t, wire, m, k).planes)
    ar.put("x", x)
    W, ws = ar.ptr("W"), ar.ptr("ws")
    n2 = n // 2 + 1                                     # the stale call: another N
    x2, y2 = torch.randn(n2, k, device="cuda"), torch.empty(n2, m, device="cuda")
    a, b = run_contract(ar, [("y", "f32", (n, m))], lambda nb: L.b200q_mul_mat_gemm(t, W, ar.ptr("x"), ar.ptr("y"), m, k, n, ws, nb, st()), what,
                        ws="ws", ws_bytes=need, exact_ab=not split, short=True,
                        stale=lambda: ok(L.b200q_mul_mat_gemm(t, W, x2.data_ptr(), y2.data_ptr(), m, k, n2, ws, L.b200q_mul_mat_workspace(t, m, k, n2), st()),
                                         "stale call"))
    check_dense(oracle, what, name, wire, x, m, a["y"])
    if split:
        check_dense(oracle, f"{what} (run B)", name, wire, x, m, b["y"])


@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_gemm_contract(be, oracle, side_stream, case):
    case_id, name, m, k, n, expected = case
    run_dense_case(be, oracle, name, m, k, n, dense_seed(case), expected[0][2][2] > 1, case_id)


@pytest.mark.gpu
@pytest.mark.parametrize("split", [5, 16])
def test_forced_split_k_contract(be, split):
    in_child("forced", str(split), {"B200Q_GEMM_SPLIT": str(split)})


def run_grouped_case(be, oracle, case, plug):
    """plug: the backend plug's layout, the gathered ids right at align256(need) after the workspace with no guard between them"""
    case_id, name, n_expert, m, k, n_tokens, n_used, glu, _, _, _ = case
    t = GGML_TYPE[name]
    L = lib()
    ids, x, wires, gwires = moe_operands(oracle, case)
    need = L.b200q_mul_mat_id_workspace(t, m, k, n_used, 1, n_tokens, n_expert, int(glu))
    assert need > 0
    ar = Arena(m)
    ar.add("y", n_tokens * n_used * m * 4, "out")
    ar.add("x", x.nbytes, "in")
    ar.add("ws", need, "ws", guard=not plug)
    ar.add("ids", ids.nbytes, "ids")
    for g in (False, True) if glu else (False,):
        ar.add(f"W{int(g)}", n_expert * be.plane_bytes(t, m, k), "in")
    ar.build()
    for g in (False, True) if glu else (False,):
        ar.put(f"W{int(g)}", be.set_expert_tensor(t, np.concatenate(gwires if g else wires), n_expert, m, k).planes)
    ar.put("x", x)
    ar.put("ids", ids)
    W, G, ws = ar.ptr("W0"), (ar.ptr("W1") if glu else None), ar.ptr("ws")
    what = f"{case_id}{' (plug layout)' if plug else ''}"
    a, _ = run_contract(ar, [("y", "f32", (n_tokens, n_used, m))],
                        lambda b: L.b200q_mul_mat_id_gemm(t, W, G, n_expert, ar.ptr("ids"), ar.ptr("x"), ar.ptr("y"), m, k, n_used, 1, n_tokens, SILU, 0.0,
                                                          ws, b, st()),
                        what, ws="ws", ws_bytes=need, short=True, stale=moe_stale(L, t, W, G, n_expert, m, k, n_used, n_tokens, ws))
    r = check_grouped(oracle, name, wires.__getitem__, gwires.__getitem__ if glu else None, x, ids, n_expert, m, a["y"], what)
    print(f"{what}: max |y - ref| / bound = {r:.3g}")


PLUG_LAYOUT = ["grouped-fused-bn256-at-threshold", "grouped-generic-2-groups"]


@pytest.mark.gpu
@pytest.mark.parametrize("case,plug", [(c, False) for c in MOE] + [(c, True) for c in MOE if c[0] in PLUG_LAYOUT],
                         ids=[c[0] for c in MOE] + [f"{c}-plug-layout" for c in PLUG_LAYOUT])
def test_grouped_gemm_contract(be, oracle, side_stream, case, plug):
    run_grouped_case(be, oracle, case, plug)


@pytest.mark.gpu
@pytest.mark.parametrize("case", IDENTITY, ids=[c[0] for c in IDENTITY])
def test_merged_up_gate_contract(be, oracle, side_stream, case):
    """b200q_moe_up_gate_merged at the token counts of test_gpu_moe_merged.py, on both sides of the crossover: the mat-vec (no workspace) below,
    the grouped GEMM (exact workspace, stale tables for run B, short probe) above."""
    case_id, name, n_expert, n_used, n_ff, k, tokens = case
    t = GGML_TYPE[name]
    L = lib()
    gw = [make_wire(oracle, name, n_ff, k, seed=[1300, 0, e]) for e in range(n_expert)]
    uw = [make_wire(oracle, name, n_ff, k, seed=[1300, 1, e]) for e in range(n_expert)]
    ops = [merged_inputs([n_ff, n], n, 1, n_expert, n_used, k, n, scale=1.0) for n in tokens]
    needs = [L.b200q_moe_up_gate_merged_workspace(t, n_ff, k, n_used, 1, n, n_expert) for n in tokens]
    ar = Arena(n_ff)
    for i, (n, (x, ids), need) in enumerate(zip(tokens, ops, needs)):
        ar.add(f"y{i}", n * n_used * n_ff * 4, "out")
        if need:
            ar.add(f"ws{i}", need, "ws")
        ar.add(f"x{i}", x.nbytes, "in")
        ar.add(f"ids{i}", ids.nbytes, "ids")
    ar.add("W", n_expert * be.plane_bytes(t, 2 * n_ff, k), "in")
    ar.build()
    ar.put("W", be.set_expert_tensor(t, np.concatenate([np.concatenate([g, u]) for g, u in zip(gw, uw)]), n_expert, 2 * n_ff, k).planes)
    W = ar.ptr("W")
    for i, (n, (x, ids), need) in enumerate(zip(tokens, ops, needs)):
        ar.put(f"x{i}", x)
        ar.put(f"ids{i}", ids)
        ws = ar.ptr(f"ws{i}") if need else None
        what = f"{case_id} {n} tokens ({'grouped GEMM' if need else 'mat-vec'})"
        a, _ = run_contract(ar, [(f"y{i}", "f32", (n, n_used, n_ff))],
                            lambda b: L.b200q_moe_up_gate_merged(t, W, n_expert, ar.ptr(f"ids{i}"), ar.ptr(f"x{i}"), ar.ptr(f"y{i}"), n_ff, k, n_used, 1, n,
                                                                 SILU, 0.0, ws, b, st()),
                            what, ws=f"ws{i}" if need else None, ws_bytes=need, short=bool(need),
                            stale=moe_stale(L, t, W, None, n_expert, n_ff, k, n_used, n, ws, merged=True) if need else None)
        if need:
            r = check_grouped(oracle, name, uw.__getitem__, gw.__getitem__, x, ids, n_expert, n_ff, a[f"y{i}"], what)
        else:
            r = check_slots(a[f"y{i}"], moe_oracle(oracle, name, uw.__getitem__, gw.__getitem__, x, ids, n_expert, n_ff), ids, n_expert, True, what)
        print(f"{what}: max ratio to the bound = {r:.3g}")


# ------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the entry points no table reaches
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["gemm_bf16", "gemm_multi_bf16", "fused_up_gate_gemm_bf16"])
@pytest.mark.parametrize("name", ["IQ4_NL", "Q6_K"])
def test_bf16_entry_points(be, oracle, side_stream, name, entry):
    """The entry points on converted activations, K = 4096, N = 64: IQ4_NL on the fused kernel (split-K 16), Q6_K on the bf16 weight scratch
    (split-K 8), so both are held to the element bound per run.  Multi: three segments of M = 128, 256, 384, the largest last (an error found only
    at the last segment would follow two finished ones).  Up/gate also writes dst_bf16, which must be bf16(dst) bit for bit.  Workspace: Q6_K
    the scratch of the largest tensor, align256(M K 2), IQ4_NL none; up/gate adds align256(M N 4) for the up result."""
    t = GGML_TYPE[name]
    L = lib()
    k, n = 4096, 64
    ug = entry == "fused_up_gate_gemm_bf16"
    ms = [128, 256, 384] if entry == "gemm_multi_bf16" else [256, 256] if ug else [256]
    wires = [make_wire(oracle, name, mm, k, seed=[77, i]) for i, mm in enumerate(ms)]
    x = np.random.default_rng(78).standard_normal((n, k)).astype(np.float32)
    scratch = 0 if name == "IQ4_NL" else align256(max(ms) * k * 2)

    def need_of(nn):
        return (align256(ms[0] * nn * 4) if ug else 0) + scratch
    need = need_of(n)
    outs = [(f"y{i}", "f32", (n, mm)) for i, mm in enumerate(ms if entry == "gemm_multi_bf16" else ms[:1])]
    if ug:
        outs.append(("yb", "bf16", (n, ms[0])))
    ar = Arena(max(ms))
    for o in outs:
        ar.add(o[0], int(np.prod(o[2])) * (2 if o[1] == "bf16" else 4), "out")
    if need:
        ar.add("ws", need, "ws")
    ar.add("xb", n * k * 2, "in")
    for i, mm in enumerate(ms):
        ar.add(f"W{i}", be.plane_bytes(t, mm, k), "in")
    ar.build()
    for i, (w, mm) in enumerate(zip(wires, ms)):
        ar.put(f"W{i}", be.set_tensor(t, w, mm, k).planes)
    ar.put("xb", bf16_bits(x))
    W = [ar.ptr(f"W{i}") for i in range(len(ms))]
    ws = ar.ptr("ws") if need else None

    def launch(xb, ys, yb, nn, b):
        if entry == "gemm_bf16":
            return L.b200q_mul_mat_gemm_bf16(t, W[0], xb, ys[0], ms[0], k, nn, ws, b, st())
        if entry == "gemm_multi_bf16":
            return L.b200q_mul_mat_gemm_multi_bf16(t, 3, (c_void_p * 3)(*W), (c_void_p * 3)(*ys), (c_int64 * 3)(*ms), k, xb, nn, ws, b, st())
        return L.b200q_fused_up_gate_gemm_bf16(t, W[0], W[1], xb, ys[0], yb, ms[0], k, nn, SILU, 0.0, ws, b, st())
    n2 = 40                                             # the stale call: another N
    x2 = torch.randn(n2, k, device="cuda").bfloat16()
    y2 = [torch.empty(n2, mm, device="cuda") for mm in ms]
    yb2 = torch.empty(n2, ms[0], dtype=torch.bfloat16, device="cuda")
    a, b = run_contract(ar, outs, lambda nb: launch(ar.ptr("xb"), [ar.ptr(o[0]) for o in outs if o[0] != "yb"], ar.ptr("yb") if ug else None, n, nb),
                        f"{name} {entry}", ws="ws" if need else None, ws_bytes=need, exact_ab=False, short=bool(need),
                        stale=(lambda: ok(launch(x2.data_ptr(), [y.data_ptr() for y in y2], yb2.data_ptr(), n2, need_of(n2)), "stale call")) if need else None)
    for run, res in (("A", a), ("B", b)):
        what = f"{name} {entry} run {run}"
        if ug:
            up, gate = (bf16(oracle.dequantize(t, w, ms[0], k)) for w in wires)
            ru, au = same_operand_reference(up, bf16(x))
            rg, ag = same_operand_reference(gate, bf16(x))
            r = element_ratio(res["y0"], silu(rg) * ru, None, k, what, bound=glu_bound(k, rg, ru, ag, au))
            assert np.array_equal(res["yb"], bf16_bits(res["y0"])), f"{what}: dst_bf16 is not bf16(dst)"
            print(f"{what}: max |y - ref| / bound = {r:.3g}; dst_bf16 == bf16(dst)")
        else:
            for i in range(len(outs)):
                check_dense(oracle, f"{what} segment {i}", name, wires[i], x, ms[i], res[f"y{i}"])


def bitnet_emulation(oracle, wire, x, m):
    """IQ2_BN on the int8 tensor pipe (test_gpu_parity.py::test_bitnet_int8_gemm_is_exact_integer_arithmetic): per-token int8 activations
    (ts = amax / 127, xq = rint(x / ts)), exact integer sums; only the two f32 multiplies of the epilogue round"""
    k = x.shape[1]
    wd = oracle.dequantize(GGML_TYPE["IQ2_BN"], wire, m, k).astype(np.float64)
    amax = np.abs(x).max(1, keepdims=True)
    ts = (amax / np.float32(127)).astype(np.float32)
    inv = np.where(ts > 0, np.float32(1) / np.where(ts > 0, ts, 1), 0).astype(np.float32)
    xq = np.clip(np.rint(x * inv), -127, 127)
    return (xq.astype(np.float64) * ts.astype(np.float64)) @ wd.T


@pytest.mark.gpu
@pytest.mark.parametrize("up_gate", [False, True], ids=["plain", "up-gate"])
@pytest.mark.parametrize("k", [3200, 8640])
def test_iq2bn_int8_path_contract(be, oracle, side_stream, k, up_gate):
    """IQ2_BN prefill on the int8 path at the bitnet row lengths (not multiples of the 128-wide k-block), N = 300 (the BN = 256 tile, ragged):
    b200q_mul_mat_gemm and b200q_fused_up_gate with their documented workspaces (activation quantisation and, for up/gate, the up result live
    there).  No split-K: runs A and B bit-equal.  Values against the int8 emulation: plain within 4e-7 max |ref|, up/gate the same through silu."""
    t = GGML_TYPE["IQ2_BN"]
    L = lib()
    m, n = 256, 300
    wires = [make_wire(oracle, "IQ2_BN", m, k, seed=[400, k, i]) for i in range(2 if up_gate else 1)]
    x = (np.random.default_rng(60 + k).standard_normal((n, k)) * 1.7).astype(np.float32)
    x[0] = 0.0                                          # an all-zero token (amax == 0)
    query = L.b200q_fused_up_gate_workspace if up_gate else L.b200q_mul_mat_workspace
    need = query(t, m, k, n)
    ar = Arena(m)
    for region, nb, kind in [("y", n * m * 4, "out"), ("ws", need, "ws"), ("x", x.nbytes, "in")] + [(f"W{i}", be.plane_bytes(t, m, k), "in") for i in range(len(wires))]:
        ar.add(region, nb, kind)
    ar.build()
    for i, w in enumerate(wires):
        ar.put(f"W{i}", be.set_tensor(t, w, m, k).planes)
    ar.put("x", x)
    W, ws = [ar.ptr(f"W{i}") for i in range(len(wires))], ar.ptr("ws")

    def launch(xp, yp, nn, b):
        if up_gate:
            return L.b200q_fused_up_gate(t, W[0], W[1], xp, yp, m, k, nn, SILU, 0.0, ws, b, st())
        return L.b200q_mul_mat_gemm(t, W[0], xp, yp, m, k, nn, ws, b, st())
    n2 = 150
    x2, y2 = torch.randn(n2, k, device="cuda"), torch.empty(n2, m, device="cuda")
    what = f"IQ2_BN int8 K={k} {'up/gate' if up_gate else 'plain'}"
    a, _ = run_contract(ar, [("y", "f32", (n, m))], lambda b: launch(ar.ptr("x"), ar.ptr("y"), n, b), what, ws="ws", ws_bytes=need, short=True,
                        stale=lambda: ok(launch(x2.data_ptr(), y2.data_ptr(), n2, query(t, m, k, n2)), "stale call"))
    y = a["y"].astype(np.float64)
    u = bitnet_emulation(oracle, wires[0], x, m)
    if up_gate:
        g = bitnet_emulation(oracle, wires[1], x, m)
        ref = silu(g) * u
        bound = 4e-7 * (1.1 * np.abs(g).max() * np.abs(u) + np.abs(silu(g)) * np.abs(u).max()) + GLU_EPILOGUE_REL * np.abs(ref) + FLOOR
    else:
        ref, bound = u, 4e-7 * np.abs(u).max() + FLOOR
    r = float((np.abs(y - ref) / bound).max())
    print(f"{what}: max |y - emulation| / bound = {r:.3g}")
    assert r <= 1.0, f"{what}: {int((np.abs(y - ref) > bound).sum())} elements outside the bound"


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1000, 1004], ids=["k1000-8-wide", "k1004-4-wide"])
def test_convert_f32_bf16_strided(be, side_stream, k):
    """b200q_convert_f32_bf16 on rows of k + 64 floats whose padding is NaN (K % 8 == 0: the 8-wide kernel; else the 4-wide one): exactly N K 2
    bytes written, equal to bf16(x) bit for bit; the padding never reaches the output."""
    L = lib()
    n, stride = 37, k + 64
    x = np.random.default_rng(k).standard_normal((n, k)).astype(np.float32)
    xp = np.full((n, stride), np.nan, np.float32)
    xp[:, :k] = x
    ar = Arena()
    ar.add("xb", n * k * 2, "out")
    ar.add("x", xp.nbytes, "in")
    ar.build()
    ar.put("x", xp)
    a, _ = run_contract(ar, [("xb", "bf16", (n, k))], lambda b: L.b200q_convert_f32_bf16(ar.ptr("x"), stride, ar.ptr("xb"), k, n, st()),
                        f"convert_f32_bf16 K={k} x_stride={stride}")
    assert np.array_equal(a["xb"], bf16_bits(x)), "the conversion differs from bf16(x)"


@pytest.mark.gpu
@pytest.mark.parametrize("in_place", [False, True], ids=["dst", "dst-is-a"])
@pytest.mark.parametrize("nb", ["1", "n"])
def test_add_rows_contract(be, side_stream, nb, in_place):
    """b200q_add_rows with one bias row (nb = 1) and with a same-shape tensor (nb = n), into its own dst and in place (dst == a: the ADD ggml's
    allocator may place on its first operand): dst = a + b[j % nb] exactly as f32 adds it, nothing else written."""
    L = lib()
    m, n = 4097, 7
    nbv = 1 if nb == "1" else n
    rng = np.random.default_rng(5)
    a0, b0 = rng.standard_normal((n, m)).astype(np.float32), rng.standard_normal((nbv, m)).astype(np.float32)
    ref = a0 + b0[np.arange(n) % nbv]
    ar = Arena(m)
    if not in_place:
        ar.add("dst", n * m * 4, "out")
    ar.add("a", a0.nbytes, "out" if in_place else "in")
    ar.add("b", b0.nbytes, "in")
    ar.build()
    ar.put("a", a0)
    ar.put("b", b0)
    what = f"add_rows nb={nbv}{' in place' if in_place else ''}"
    dst = "a" if in_place else "dst"
    if not in_place:
        a, _ = run_contract(ar, [("dst", "f32", (n, m))], lambda b: L.b200q_add_rows(ar.ptr("a"), ar.ptr("b"), ar.ptr("dst"), m, n, nbv, st()), what)
        assert np.array_equal(a["dst"], ref), f"{what}: differs from the f32 sum"
        return
    for run in range(2):
        ar.put("a", a0)
        snap = ar.buf.clone()
        ok(L.b200q_add_rows(ar.ptr("a"), ar.ptr("b"), ar.ptr(dst), m, n, nbv, st()), what)
        torch.cuda.synchronize()
        ar.untouched(snap, [dst], f"{what} run {run}")
        assert np.array_equal(ar.get(dst, "f32", (n, m)), ref), f"{what} run {run}: differs from the f32 sum"
    print(f"{what}: contract kept, equal to the f32 sum")


@pytest.mark.gpu
def test_q8_handoff_chain_on_one_scratch(be, oracle, side_stream):
    """Three fused_up_gate_vec_q8 -> mul_mat_vec_q8 steps (Q4_K, up/gate 2048 x 8192 on long rows, ffn_down 512 x 2048 on row pairs), each run
    twice, on ONE q8 scratch initialised once: the image region is exactly b200q_q8_scratch_bytes(2048) with a guard after it, the image equals
    the oracle's quantisation of each step's result with the arrival counters back at zero after every step, and both launches are within
    their bars."""
    name, m_ff, k, m_d = "Q4_K", 2048, 8192, 512
    t = GGML_TYPE[name]
    L = lib()
    wu, wg, wd = (make_wire(oracle, name, mm, kk, seed=[90, i]) for i, (mm, kk) in enumerate(((m_ff, k), (m_ff, k), (m_d, m_ff))))
    xs = [(np.random.default_rng([91, i]).standard_normal((1, k)) * 3).astype(np.float32) for i in range(3)]
    ar = Arena(m_ff)
    for i in range(3):
        ar.add(f"a{i}", m_ff * 4, "out")
        ar.add(f"y{i}", m_d * 4, "out")
    ar.add("q8", L.b200q_q8_scratch_bytes(m_ff), "out")
    for i in range(3):
        ar.add(f"x{i}", k * 4, "in")
    for region, (w, mm, kk) in (("Wu", (wu, m_ff, k)), ("Wg", (wg, m_ff, k)), ("Wd", (wd, m_d, m_ff))):
        ar.add(region, be.plane_bytes(t, mm, kk), "in")
    ar.build()
    for region, (w, mm, kk) in (("Wu", (wu, m_ff, k)), ("Wg", (wg, m_ff, k)), ("Wd", (wd, m_d, m_ff))):
        ar.put(region, be.set_tensor(t, w, mm, kk).planes)
    for i in range(3):
        ar.put(f"x{i}", xs[i])
    q8 = ar.ptr("q8")
    ok(L.b200q_q8_scratch_init(q8, m_ff, st()), "b200q_q8_scratch_init")
    for i in range(3):
        produced = []

        def call(b):
            p = ctypes.c_int32(0)
            rc = L.b200q_fused_up_gate_vec_q8(t, ar.ptr("Wu"), ar.ptr("Wg"), ar.ptr(f"x{i}"), ar.ptr(f"a{i}"), m_ff, k, SILU, 0.0, q8, ctypes.byref(p), st())
            produced.append(p.value)
            return rc or L.b200q_mul_mat_vec_q8(t, ar.ptr("Wd"), ar.ptr(f"a{i}"), q8, ar.ptr(f"y{i}"), m_d, m_ff, None, st())
        what = f"q8 chain step {i}"
        a, _ = run_contract(ar, [(f"a{i}", "f32", (1, m_ff)), (f"y{i}", "f32", (1, m_d))], call, what, keep=[("q8", "u8", (ar.nbytes("q8"),))])
        assert produced == [1, 1], f"{what}: the hand-off must be taken ({produced})"
        check_q8_image(oracle, a["q8"], a[f"a{i}"], what)
        print(f"{what}: up/gate {glu_ratio(oracle, name, wu, wg, xs[i], m_ff, a[f'a{i}'], what):.3g}, "
              f"ffn_down {plain_ratio(oracle, name, wd, a[f'a{i}'], m_d, a[f'y{i}'], what):.3g} of the bar")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_TYPES)
def test_repack_unrepack_dequantize_write_exactly_their_bytes(be, oracle, side_stream, name):
    """M = 32, K = 512.  b200q_repack writes inside its b200q_plane_bytes (the alignment gaps between planes are not written, so its runs are not
    compared); b200q_unrepack writes exactly M row_size bytes and gives the wire bytes back; b200q_dequantize_bf16 writes exactly M K 2 bytes, equal
    bit for bit to the dequantisation of planes uploaded by set_tensor (whose gaps are zero, here they hold what the prefill left: nothing reads
    them) and within 1.5 bf16 ulp of the oracle."""
    t = GGML_TYPE[name]
    L = lib()
    m, k = 32, 512
    wire = make_wire(oracle, name, m, k, seed=[88, t])
    pb, wb = be.plane_bytes(t, m, k), m * be.row_size(t, k)
    ar = Arena(m)
    for region, nb, kind in (("planes", pb, "out"), ("wire_out", wb, "out"), ("deq", m * k * 2, "out"), ("wire", wb, "in")):
        ar.add(region, nb, kind)
    ar.build()
    ar.put("wire", wire)
    run_contract(ar, [("planes", "u8", (pb,))], lambda b: L.b200q_repack(t, ar.ptr("wire"), ar.ptr("planes"), m, k, st()), f"{name} repack",
                 exact_ab=False)
    a, _ = run_contract(ar, [("wire_out", "u8", (wb,))], lambda b: L.b200q_unrepack(t, ar.ptr("planes"), ar.ptr("wire_out"), m, k, st()),
                        f"{name} unrepack")
    assert np.array_equal(a["wire_out"], wire), f"{name}: unrepack does not give the wire bytes back"
    a, _ = run_contract(ar, [("deq", "bf16", (m, k))], lambda b: L.b200q_dequantize_bf16(t, ar.ptr("planes"), ar.ptr("deq"), m, k, st()),
                        f"{name} dequantize_bf16")
    clean = be.dequantize_bf16(be.set_tensor(t, wire, m, k)).view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(a["deq"], clean), f"{name}: the dequantisation depends on the bytes between the planes"
    d = (a["deq"].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    wd = oracle.dequantize(t, wire, m, k).astype(np.float64)
    bad = np.abs(d - wd) > 1.5 * 2.0 ** -7 * np.abs(wd) + 2.0 ** -20 * np.abs(wd).max()
    assert not bad.any(), f"{name}: {int(bad.sum())} dequantised weights differ from the oracle by more than 1.5 bf16 ulp"


if __name__ == "__main__":
    from ik_llama_cpp_b200 import backend as _be
    from oracle.oracle import Oracle
    with torch.cuda.stream(torch.cuda.Stream()):
        if sys.argv[1] == "forced":
            _name, _m, _k, _n, _seed = FORCED
            run_dense_case(_be, Oracle(), _name, _m, _k, _n, _seed, True, f"forced split {sys.argv[2]}")
        else:
            run_moe_decode_case(_be, Oracle(), next(c for c in MOE_SCHEDULES if c[0] == sys.argv[2]))
