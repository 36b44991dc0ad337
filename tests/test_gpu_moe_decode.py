"""Element-by-element tests of the MoE mat-vecs: GGML_OP_MUL_MAT_ID / MOE_FUSED_UP_GATE on k_mmvq_id<T, UPGATE> (plane types,
b200q_decode_ring.cuh) and k_wire_mmvq_id<T, UPGATE> (wire types, b200q_wire.cu).  They run every generated token of a MoE model, and the
dispatcher (b200q_mul_mat_id) also gives them prefill-sized batches: up to 5 rows per expert for up/gate (160 tokens of DeepSeek-V3, 256 experts,
8 used), up to 32 slots for MUL_MAT_ID, and every batch the grouped GEMM refuses (K % 256 != 0, more than 1024 experts, more than 2^22 slots).
Slot s = (token s / n_used, used expert s % n_used) reads activation column (s / n_used) nb1 + (s % n_used) % nb1 and writes dst row s; a slot
whose id is -1 (ggml_top_k_thresh) or n_expert is skipped and must be a zero row.

Launch rules (derived from the code, confirmed by the profiler trace of each table case at 132 SMs):
  * b200q_mul_mat_id_vec walks the tokens in chunks of floor(204800 / (nb1 K 1.25)) (the quantised columns of a launch live in shared memory,
    K int8 + K/32 (f32 scale + packed sums) per column); B200Q_MOE_CHUNK_TOKENS lowers the chunk; a chunk of 0 is refused before any launch;
  * k_mmvq_id: block 512 (16 warps), grid = min(ceil(slots M / 16), 132);
  * k_wire_mmvq_id: block 256 (8 warps), grid = min(ceil(slots M / 8), 132 x 4, 2 or 1 for smem <= 48 KB, <= 100 KB, more);
  * smem = columns K 1.25 bytes, columns = chunk tokens x nb1.

Reference and bars.  The oracle is oracle.mul_mat_q8_1(variant="b200") on the selected expert's wire bytes, called once per expert with every
column routed to it (the q8_1 quantisation is per column, so grouping the columns is exact).  Plain outputs: |y - yq| <= 2e-5 rms(yq) per slot;
GLU: |y - ref| <= 5e-5 rms(ref), ref = glu_ref(act, gate_q, up_q).  These are the bars of test_gpu_decode_schedules.py, whose docstring derives
them for k_mmvq, and the derivation covers these kernels as they are: a warp owns one (slot, row), lane l accumulates items l, l + 32, ... in one
f32 chain (L = K / 1024 terms: 20 at K = 20480, the longest row one token's columns fit with nb1 = 8, well inside the derived range up to
L = 52), then the same 5-level butterfly.

Tolerance-free identity: a slot runs exactly the per-row arithmetic of the dense LDG launch on that expert's matrix and that slot's column
(the same quantize_x_to_smem<1>, the same U, item_dot, warp_sum and b200q_glu; k_wire_mmvq_id against k_wire_mmvq the same fmaf chains), so with
the TMA ring turned off every slot equals mul_mat / fused_up_gate (n = 1) on QuantTensor(t, m, k, W.planes[e pb:(e + 1) pb]) bit for bit.
"""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from conftest import ALL_TYPES, make_wire
from oracle.oracle import GGML_TYPE, nmse
from test_gpu_decode_schedules import (GLU_BAR, PLAIN_BAR, T, B, _fails, _set_option, assert_schedule, bar_ratio, matmul_launches, profiled,
                                       run_child)
from test_gpu_parity import glu_ref

SMEM_COLUMNS = 200 * 1024        # bytes of quantised activation columns one launch holds (b200q_mul_mat_id_vec)


def chunk_tokens(k, nb1, env=None):
    """tokens per launch of b200q_mul_mat_id_vec"""
    c = SMEM_COLUMNS // (nb1 * (k + k // 4))
    forced = int((env or {}).get("B200Q_MOE_CHUNK_TOKENS", 0))
    return min(c, forced) if forced > 0 else c


def route(rng, n_tokens, n_expert, n_used, chunk):
    """Top-k ids of every token; the last expert in token 1 (the largest expert offset); then skipped slots in every chunk of the launch walk (-1 in
    its first token, n_expert in its last), and, when the walk has three chunks or more, every slot of the second chunk skipped."""
    ids = np.stack([rng.choice(n_expert, n_used, replace=False) for _ in range(n_tokens)]).astype(np.int32)
    ids[min(1, n_tokens - 1), n_used // 2] = n_expert - 1
    starts = range(0, n_tokens, chunk)
    for c0 in starts:
        ids[c0, n_used - 1] = -1
        ids[min(c0 + chunk, n_tokens) - 1, 0] = n_expert
    if len(starts) >= 3:
        ids[chunk:2 * chunk] = -1
        ids[chunk:2 * chunk, ::2] = n_expert
    return ids


def moe_oracle(oracle, name, wire_of, gate_of, x, ids, n_expert, m, col_of=None):
    """The reference of every slot, f64 [n_tokens, n_used, M]: zero rows for skipped ids.  wire_of(e) / gate_of(e): wire bytes of expert e
    (gate_of None: MUL_MAT_ID).  col_of(s, nb1, n_used): activation column of slot s (default: the ggml broadcast; the self-test plants others)."""
    t = GGML_TYPE[name]
    n_tokens, nb1, k = x.shape
    n_used = ids.shape[1]
    cols = x.reshape(n_tokens * nb1, k)
    col_of = col_of or (lambda s, nb1, n_used: (s // n_used) * nb1 + (s % n_used) % nb1)
    ref = np.zeros((n_tokens, n_used, m))
    for e in np.unique(ids[(ids >= 0) & (ids < n_expert)]):
        tk, u = np.nonzero(ids == e)
        xe = cols[col_of(tk * n_used + u, nb1, n_used)]
        r = oracle.mul_mat_q8_1(t, wire_of(e), xe, m, variant="b200").astype(np.float64)
        if gate_of is not None:
            r = glu_ref("silu", oracle.mul_mat_q8_1(t, gate_of(e), xe, m, variant="b200"), r)
        ref[tk, u] = r
    return ref


def check_slots(y, ref, ids, n_expert, glu, what):
    """Skipped slots are exact zero rows; every other slot is within the plain (GLU) bar of its own rms.  Returns the worst ratio to the bar."""
    y = np.asarray(y)
    assert y.shape == ref.shape, (what, y.shape, ref.shape)
    skipped = (ids < 0) | (ids >= n_expert)
    bad = np.argwhere(skipped & np.any(y != 0.0, axis=2))
    assert len(bad) == 0, f"{what}: skipped slots (token, slot) {[tuple(int(i) for i in b) for b in bad[:5]]} are not zero rows"
    worst = 0.0
    for tk, u in np.argwhere(~skipped):
        worst = max(worst, bar_ratio(y[tk, u], ref[tk, u], GLU_BAR if glu else PLAIN_BAR, f"{what}: token {tk} slot {u} (expert {ids[tk, u]})"))
    return worst


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-test of the comparison (oracle and numpy only)
# ------------------------------------------------------------------------------------------------------------------------------------------------
def test_checker_catches_planted_defects(oracle):
    """Clean oracle data passes; each defect an indexing bug of the MoE mat-vec or of its token walk would produce fails: a slot given the
    neighbouring expert, the column map s % nb1 (every token reading token 0's columns), one chunk's ids or its dst offset by one token.
    (The partial slip (s / n_used) nb1 + s % nb1 is not a defect: n_used % nb1 == 0, so s % nb1 == (s % n_used) % nb1; asserted below.)"""
    name, n_expert, n_used, m, k = "IQ4_NL", 6, 4, 64, 512
    wires = [make_wire(oracle, name, m, k, seed=[31, e]) for e in range(n_expert)]
    gwires = [make_wire(oracle, name, m, k, seed=[32, e]) for e in range(n_expert)]
    rng = np.random.default_rng(33)
    n_tokens, nb1, chunk = 6, 2, 2                         # a walk of three 2-token chunks, the second one all skipped
    x = rng.standard_normal((n_tokens, nb1, k)).astype(np.float32)
    ids = route(rng, n_tokens, n_expert, n_used, chunk)
    ref = moe_oracle(oracle, name, wires.__getitem__, None, x, ids, n_expert, m)
    check_slots(ref.astype(np.float32), ref, ids, n_expert, False, "clean")
    gref = moe_oracle(oracle, name, wires.__getitem__, gwires.__getitem__, x * 3, ids, n_expert, m)
    check_slots(gref.astype(np.float32), gref, ids, n_expert, True, "clean GLU")
    assert np.all(ref[2:4] == 0.0) and ref[0].any() and ref[1].any(), "the route skips every slot of chunk 1 and some of chunk 0"

    # a slot given the neighbouring expert
    tk, u = (int(i) for i in np.argwhere((ids >= 0) & (ids < n_expert))[0])
    ids_d = ids.copy(); ids_d[tk, u] = (ids[tk, u] + 1) % n_expert
    d = moe_oracle(oracle, name, wires.__getitem__, None, x, ids_d, n_expert, m)
    assert _fails(lambda: check_slots(d, ref, ids, n_expert, False, "neighbouring expert")), "a slot given the neighbouring expert"
    # the column map s % nb1: the token offset dropped
    d = moe_oracle(oracle, name, wires.__getitem__, None, x, ids, n_expert, m, col_of=lambda s, nb1, n_used: s % nb1)
    assert _fails(lambda: check_slots(d, ref, ids, n_expert, False, "column map s % nb1")), "column map s % nb1"
    s = np.arange(n_tokens * n_used)
    assert np.array_equal(s % nb1, (s % n_used) % nb1)
    # one chunk's ids offset by one token (chunk 0 reads the ids of tokens 1, 2)
    ids_d = ids.copy(); ids_d[0:2] = ids[1:3]
    d = moe_oracle(oracle, name, wires.__getitem__, None, x, ids_d, n_expert, m)
    assert _fails(lambda: check_slots(d, ref, ids, n_expert, False, "chunk ids offset")), "one chunk's ids offset by one token"
    # one chunk's dst offset by one token (chunk 0 writes tokens 1, 2; token 0 keeps what the buffer held, zeros here)
    d = ref.copy(); d[1:3] = ref[0:2]; d[0] = 0.0
    assert _fails(lambda: check_slots(d, ref, ids, n_expert, False, "chunk dst offset")), "one chunk's dst offset by one token"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# schedule table
# ------------------------------------------------------------------------------------------------------------------------------------------------
def mid(name, upgate, grid):
    return ("k_mmvq_id", (T[name], B[upgate]), (grid, 1, 1), (512, 1, 1))


def wid(name, upgate, grid):
    return ("k_wire_mmvq_id", (T[name], B[upgate]), (grid, 1, 1), (256, 1, 1))


FORCE_3 = {"B200Q_MOE_CHUNK_TOKENS": "3"}
# (id, type, n_expert, n_used, tensor shapes (M, K), calls, environment, launches at 132 SMs)
# call: (entry, tensor, n_tokens, nb1, up/gate) with entry "vec" = mul_mat_id (b200q_mul_mat_id_vec), "disp" = mul_mat_id_dispatch (b200q_mul_mat_id)
MOE_SCHEDULES = [
    ("qwen3-30b-a3b-upgate-q4k", "Q4_K", 128, 8, [(768, 2048)], [("vec", 0, 1, 1, True)], {},
     # 8 slots x 768 rows / 16 = 384 -> 132; smem 2560 B
     [mid("Q4_K", True, 132)]),
    ("qwen3-30b-a3b-down-q4k-nb8", "Q4_K", 128, 8, [(2048, 768)], [("vec", 0, 1, 8, False), ("disp", 0, 4, 8, False), ("vec", 0, 40, 8, False)], {},
     # 1 token: 8 x 2048 / 16 -> 132 (7680 B); 4 tokens = 32 slots, the last batch the dispatcher keeps on the mat-vec (30720 B);
     # 40 tokens: chunk 204800 / (8 x 960) = 26, launches of 26 (199680 B) and 14 tokens, each 132
     [mid("Q4_K", False, 132)] * 4),
    ("mixtral-down-iq4nl-nb2", "IQ4_NL", 8, 2, [(4096, 14336)], [("vec", 0, 8, 2, False), ("disp", 0, 16, 2, False)], {},
     # chunk 204800 / (2 x 17920) = 5 (179200 B): 8 tokens -> 5 + 3, 16 tokens (32 slots, still the mat-vec) -> 5 + 5 + 5 + 1; 132 each
     [mid("IQ4_NL", False, 132)] * 6),
    ("mixtral-upgate-iq4nl-20-tokens", "IQ4_NL", 8, 2, [(14336, 4096)], [("disp", 0, 20, 1, True)], {},
     # 40 slots = 5 per expert: the last up/gate batch of the mat-vec; chunk 40, one launch of 102400 B
     [mid("IQ4_NL", True, 132)]),
    ("deepseek-v3-tp8-upgate-iq2xxs", "IQ2_XXS", 256, 8, [(256, 7168)], [("vec", 0, 1, 1, True), ("disp", 0, 160, 1, True)], {},
     # 1 token: 8 x 256 / 8 = 256 (8960 B <= 48 KB: cap 528); 160 tokens (1280 slots = 5 per expert, the mat-vec): chunk 204800 / 8960 = 22,
     # seven launches of 22 tokens (197120 B > 100 KB: cap 132) then 6 tokens (53760 B: cap 264, 48 x 256 / 8 = 1536 -> 264)
     [wid("IQ2_XXS", True, 256)] + [wid("IQ2_XXS", True, 132)] * 7 + [wid("IQ2_XXS", True, 264)]),
    ("deepseek-v3-tp8-down-iq2xxs-nb8", "IQ2_XXS", 256, 8, [(7168, 256)], [("disp", 0, 4, 8, False)], {},
     # 32 slots x 7168 / 8 = 28672; 4 x 8 x 320 = 10240 B <= 48 KB: cap 528
     [wid("IQ2_XXS", False, 528)]),
    ("k1056-iq4nl-600-tokens-dispatcher", "IQ4_NL", 8, 2, [(64, 1056)], [("disp", 0, 600, 1, False)], {},
     # K % 256 != 0: the grouped GEMM refuses, the mat-vec walks 600 tokens in chunks of 204800 / 1320 = 155 (204600 B): 155 x 3 + 135, each 132
     [mid("IQ4_NL", False, 132)] * 4),
    ("experts-1025-iq4nl-dispatcher", "IQ4_NL", 1025, 8, [(64, 256)], [("disp", 0, 64, 1, False)], {},
     # more than 1024 experts: no routing pass (k_moe_route), one mat-vec launch: 512 slots x 64 / 16 -> 132
     [mid("IQ4_NL", False, 132)]),
    ("small-m-1-2-3", "IQ4_NL", 6, 4, [(1, 2048), (2, 2048), (3, 2048)],
     [("vec", 0, 1, 1, False), ("vec", 1, 1, 1, False), ("vec", 2, 1, 1, False), ("vec", 2, 1, 1, True)], {},
     # 4, 8, 12 (slot, row) pairs: one CTA
     [mid("IQ4_NL", False, 1)] * 3 + [mid("IQ4_NL", True, 1)]),
    ("forced-chunk-3-nb1-1-2", "IQ4_NL", 5, 2, [(132, 1024)], [("vec", 0, 20, 1, False), ("vec", 0, 20, 2, False)], FORCE_3,
     # B200Q_MOE_CHUNK_TOKENS=3: 6 chunks of 3 tokens (6 slots x 132 / 16 = 49.5 -> 50) and one of 2 (4 x 132 / 16 = 33), for both nb1
     ([mid("IQ4_NL", False, 50)] * 6 + [mid("IQ4_NL", False, 33)]) * 2),
    ("smem-cap-k20480-nb8", "IQ4_NL", 8, 8, [(64, 20480)], [("vec", 0, 3, 8, False)], {},
     # 8 columns x 20480 x 1.25 = 204800 B, exactly the cap: one token per launch; 8 x 64 / 16 = 32
     [mid("IQ4_NL", False, 32)] * 3),
]


class CaseData:
    """Wire bytes of every expert (made on first use, seeded by case, tensor, up/gate and expert), activations and ids of every call."""

    def __init__(self, oracle, case):
        case_id, self.name, self.n_expert, n_used, self.shapes, calls, env, _ = case
        self.oracle = oracle
        self.base = zlib.crc32(case_id.encode()) % 100000
        self.wires = {}
        self.xs, self.ids = [], []
        for i, (_, j, n_tokens, nb1, glu) in enumerate(calls):
            k = self.shapes[j][1]
            rng = np.random.default_rng([self.base, 100 + i])
            self.xs.append((rng.standard_normal((n_tokens, nb1, k)) * (3.0 if glu else 1.0)).astype(np.float32))
            self.ids.append(route(rng, n_tokens, self.n_expert, n_used, chunk_tokens(k, nb1, env)))

    def wire(self, j, gate, e):
        if (j, gate, e) not in self.wires:
            m, k = self.shapes[j]
            self.wires[(j, gate, e)] = make_wire(self.oracle, self.name, m, k, seed=[self.base, j, int(gate), int(e)])
        return self.wires[(j, gate, e)]


def run_moe_calls(be, case, data):
    """Upload the case's expert tensors; returns fn() -> the output of every call (profiled by the caller)"""
    _, name, n_expert, _, shapes, calls, _, _ = case
    t = GGML_TYPE[name]
    up, gate = {}, {}
    for _, j, _, _, glu in calls:
        m, k = shapes[j]
        for g, tensors in ((False, up), (True, gate)):
            if j not in tensors and (glu or not g):
                tensors[j] = be.set_expert_tensor(t, np.concatenate([data.wire(j, g, e) for e in range(n_expert)]), n_expert, m, k)
    xg = [torch.from_numpy(x).cuda() for x in data.xs]
    ig = [torch.from_numpy(i).cuda() for i in data.ids]
    torch.cuda.synchronize()

    def fn():
        return [(be.mul_mat_id if entry == "vec" else be.mul_mat_id_dispatch)(up[j], x, i, gate=gate[j] if glu else None)
                for (entry, j, _, _, glu), x, i in zip(calls, xg, ig)]
    return fn


def _child(case_id, out_dir):
    """One case in a process of its own (the chunk override is read once per process; see test_gpu_decode_schedules._child)."""
    import json
    from oracle.oracle import Oracle
    from ik_llama_cpp_b200 import backend
    case = next(c for c in MOE_SCHEDULES if c[0] == case_id)
    fn = run_moe_calls(backend, case, CaseData(Oracle(), case))
    outs, kernels = profiled(fn)
    np.savez(os.path.join(out_dir, "y.npz"), **{f"y{i}": o.cpu().numpy() for i, o in enumerate(outs)})
    with open(os.path.join(out_dir, "launches.json"), "w") as f:
        json.dump({"any_kernel": bool(kernels), "launches": matmul_launches(kernels), "moe_route": sum("k_moe_route" in k[0] for k in kernels),
                   "sms": torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count}, f)


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


@pytest.mark.gpu
@pytest.mark.parametrize("case", MOE_SCHEDULES, ids=[c[0] for c in MOE_SCHEDULES])
def test_moe_decode_schedule(be, oracle, tmp_path, case):
    ys, got = run_child(case[0], tmp_path, script=__file__, env=case[6])
    data = CaseData(oracle, case)
    for i, (entry, j, n_tokens, nb1, glu) in enumerate(case[5]):
        what = f"{case[0]} call {i} ({entry}, {n_tokens} tokens, nb1 = {nb1}{', up/gate' if glu else ''})"
        ref = moe_oracle(oracle, data.name, lambda e: data.wire(j, False, e), (lambda e: data.wire(j, True, e)) if glu else None,
                         data.xs[i], data.ids[i], data.n_expert, data.shapes[j][0])
        print(f"{what}: max ratio to the bar = {check_slots(ys[f'y{i}'], ref, data.ids[i], data.n_expert, glu, what):.3g}")
    assert got["moe_route"] == 0, f"{case[0]}: every call of the table takes the mat-vec, yet k_moe_route ran {got['moe_route']} times"
    assert_schedule(case[0], case[7], got)


@pytest.mark.gpu
def test_one_token_past_the_shared_memory_cap(be, oracle):
    """K = 20512 with nb1 = 8: one token's columns need 205120 bytes, more than a launch holds (K = 20480 is the table's case at exactly the cap).
    The shape is refused on the host before anything is launched, through the dispatcher (the grouped GEMM refuses K % 256 != 0) and the mat-vec
    entry point alike; the output keeps its NaN sentinel."""
    name, n_expert, n_used, m, k = "IQ4_NL", 8, 8, 64, 20512
    t = GGML_TYPE[name]
    W = be.set_expert_tensor(t, np.concatenate([make_wire(oracle, name, m, k, seed=[41, e]) for e in range(n_expert)]), n_expert, m, k)
    rng = np.random.default_rng(42)
    x = torch.from_numpy(rng.standard_normal((1, 8, k)).astype(np.float32)).cuda()
    ids = torch.from_numpy(route(rng, 1, n_expert, n_used, 1)).cuda()
    out = torch.full((1, n_used, m), float("nan"), device="cuda")
    assert be.mul_mat_id_workspace(W, 1, n_used, 8, False) == 0
    with pytest.raises(be.B200QError, match="do not fit shared memory"):
        be.mul_mat_id_dispatch(W, x, ids, out=out)
    with pytest.raises(be.B200QError, match="do not fit shared memory"):
        be.mul_mat_id(W, x, ids)
    torch.cuda.synchronize()
    assert torch.isnan(out).all(), "nothing may be written when the shape is refused"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# every type: against the oracle and, tolerance-free, against the dense LDG launch; the grouped GEMM at a prefill batch
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_TYPES)
def test_every_type_against_oracle_and_dense_launch(be, oracle, name):
    """M = 260 (the _R4 repacks come in groups of 4 rows), 6 experts, 4 used, K = 2048 and 7168: MUL_MAT_ID with nb1 = 1, 2, 4 and
    MOE_FUSED_UP_GATE with nb1 = 1, at 1, 2 and 3 tokens, skipped ids in each.  Every slot against the oracle, and with the TMA ring off (so that
    the dense n = 1 launch is k_mmvq / k_wire_mmvq) bit-identical to mul_mat / fused_up_gate on that expert's planes and that slot's column."""
    from test_gpu_moe_prefill import experts
    t = GGML_TYPE[name]
    n_expert, n_used, m = 6, 4, 260
    ring0 = int(os.environ.get("B200Q_RING", "1"))
    worst = {}
    for k in (2048, 7168):
        wires, W = experts(be, oracle, name, n_expert, m, k, 3000 + k)
        gwires, G = experts(be, oracle, name, n_expert, m, k, 4000 + k)
        pb = be.plane_bytes(t, m, k)
        dense = [be.QuantTensor(t, m, k, W.planes[e * pb:(e + 1) * pb]) for e in range(n_expert)]
        gdense = [be.QuantTensor(t, m, k, G.planes[e * pb:(e + 1) * pb]) for e in range(n_expert)]
        for glu, nb1 in ((False, 1), (False, 2), (False, 4), (True, 1)):
            for n_tokens in (1, 2, 3):
                rng = np.random.default_rng([t, k, int(glu), nb1, n_tokens])
                x = (rng.standard_normal((n_tokens, nb1, k)) * (3.0 if glu else 1.0)).astype(np.float32)
                ids = route(rng, n_tokens, n_expert, n_used, n_tokens)
                xg = torch.from_numpy(x).cuda()
                y = be.mul_mat_id(W, xg, torch.from_numpy(ids).cuda(), gate=G if glu else None)
                what = f"{name} K={k} {'up/gate' if glu else 'plain'} nb1={nb1} tokens={n_tokens}"
                ref = moe_oracle(oracle, name, wires.__getitem__, gwires.__getitem__ if glu else None, x, ids, n_expert, m)
                r = check_slots(y.cpu().numpy(), ref, ids, n_expert, glu, what)
                worst[(glu, k)] = max(worst.get((glu, k), 0.0), r)
                _set_option("ring", 0)
                try:
                    for tk, u in np.argwhere((ids >= 0) & (ids < n_expert)):
                        e, col = ids[tk, u], xg[tk, u % nb1][None]
                        d = be.fused_up_gate(dense[e], gdense[e], col, "silu") if glu else be.mul_mat(dense[e], col)
                        assert torch.equal(y[tk, u][None], d), \
                            f"{what}: token {tk} slot {u} differs from the dense launch, max |diff| = {float((y[tk, u] - d[0]).abs().max()):.3g}"
                finally:
                    _set_option("ring", ring0)
    for (glu, k), r in sorted(worst.items()):
        print(f"{name} {'up/gate' if glu else 'plain'} K={k}: max ratio to the bar = {r:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_TYPES)
def test_grouped_gemm_every_type(be, oracle, name):
    """The grouped GEMM (96 tokens, 8 experts, 2 used, K = 2048, M = 260), plain and up/gate, against the exact product at the NMSE bars of
    test_gpu_moe_prefill.py (2e-5, up/gate 2e-4).  The grouped path has no int8 variant, so IQ2_BN is held to the bf16 bar too."""
    from test_gpu_moe_prefill import exact, experts
    n_expert, n_used, m, k, n_tokens = 8, 2, 260, 2048, 96
    wires, W = experts(be, oracle, name, n_expert, m, k, 5000)
    gwires, G = experts(be, oracle, name, n_expert, m, k, 6000)
    rng = np.random.default_rng(GGML_TYPE[name])
    x = rng.standard_normal((n_tokens, 1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    for glu in (False, True):
        assert be.mul_mat_id_workspace(W, n_tokens, n_used, 1, glu) > 0, "the dispatcher takes the grouped GEMM at this batch"
        y = be.mul_mat_id_gemm(W, torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda(), gate=G if glu else None).cpu().numpy()
        e = nmse(y, exact(oracle, name, wires, gwires if glu else None, x, ids, m))
        print(f"{name} grouped {'up/gate' if glu else 'plain'}: NMSE {e:.3g}")
        assert e <= (2e-4 if glu else 2e-5), f"{name} grouped {'up/gate' if glu else 'plain'}: NMSE {e}"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# a MoE layer as a decode graph runs it
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_captured_moe_layer(be, oracle):
    """Qwen3-30B-A3B shape (Q4_K, 128 experts, 8 used, 2048 -> 768 -> 2048), one token: up/gate (nb1 = 1) then down (nb1 = 8) on its output,
    PDL on, captured in a CUDA graph.  Three times new x and new ids (some -1) are written in place and the graph replayed; after each replay both
    launches are checked against the oracle on the input each one read.  Finally the eager run with PDL off is bit-identical to the replay."""
    from test_gpu_moe_prefill import experts
    name, n_expert, n_used, d_model, d_ff = "Q4_K", 128, 8, 2048, 768
    uw, U = experts(be, oracle, name, n_expert, d_ff, d_model, 7000)
    gw, G = experts(be, oracle, name, n_expert, d_ff, d_model, 7200)
    dw, D = experts(be, oracle, name, n_expert, d_model, d_ff, 7400)
    x = torch.zeros((1, 1, d_model), device="cuda")
    ids = torch.zeros((1, n_used), dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(75)
    pdl0 = int(os.environ.get("B200Q_PDL", "1"))
    try:
        _set_option("pdl", 1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                be.mul_mat_id(D, be.mul_mat_id(U, x, ids, gate=G), ids)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            a = be.mul_mat_id(U, x, ids, gate=G)
            y = be.mul_mat_id(D, a, ids)
        for it in range(3):
            xi = (rng.standard_normal((1, 1, d_model)) * 3).astype(np.float32)
            ii = route(rng, 1, n_expert, n_used, 1)
            ii[0, 1 + it] = -1
            x.copy_(torch.from_numpy(xi))
            ids.copy_(torch.from_numpy(ii))
            graph.replay()
            torch.cuda.synchronize()
            ah, yh = a.cpu().numpy(), y.cpu().numpy()
            ra = check_slots(ah, moe_oracle(oracle, name, uw.__getitem__, gw.__getitem__, xi, ii, n_expert, d_ff), ii, n_expert, True,
                             f"replay {it}: up/gate")
            ry = check_slots(yh, moe_oracle(oracle, name, dw.__getitem__, None, ah, ii, n_expert, d_model), ii, n_expert, False, f"replay {it}: down")
            print(f"replay {it}: up/gate {ra:.3g}, down {ry:.3g}")
        _set_option("pdl", 0)
        a2 = be.mul_mat_id(U, x, ids, gate=G)
        y2 = be.mul_mat_id(D, a2, ids)
        torch.cuda.synchronize()
    finally:
        _set_option("pdl", pdl0)
    assert torch.equal(a2, a), "up/gate of the eager run (PDL off) differs from the graph replay"
    assert torch.equal(y2, y), "down of the eager run (PDL off) differs from the graph replay"


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
