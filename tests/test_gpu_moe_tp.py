"""GPU tests of tensor-parallel MoE on one device: the combine kernel (b200q_moe_combine, GGML_OP_MUL_MULTI_ADD) and one rank's partial of a MoE FFN
(backend.moe_tp_partial) on the expert shards of tp.py, the ranks emulated one after another.

  * Combine: bit-equal to the same loop in f32 on the host (y = x0 w0, then y = y + x_u w_u, each operation rounded on its own) for n_used 1, 2, 8,
    m % 4 != 0 (the scalar kernel), a misaligned pointer (scalar) and 1 ... 512 tokens; and its memory contract on a guarded arena (the helpers of
    test_gpu_memory_contract.py): it writes only dst, its result does not depend on what dst held, and a rejected call writes nothing.
  * Model layers: Qwen3-30B-A3B Q4_K, Mixtral-8x7B IQ4_NL and DeepSeek-V3 IQ2_XXS (with its shared expert) at W = 2 and 8, 1, 8, 64 and 512 tokens: the
    mat-vec kernels at 1 and 8 tokens, the grouped GEMM above its crossover.  For every rank:
      - its up/gate rows equal the same rows of the unsharded launch bit for bit (a row depends only on its weights and the token's activations);
      - the sum over the ranks of the ffn_down rows is the unsharded launch's within the kernel suites' bars (mat-vec: 2e-5 rms per slot,
        test_gpu_decode_schedules.py; grouped GEMM: NMSE 2e-5, test_gpu_parity.py), and the sum of the partials is the unsharded down + combine
        within those bars carried through the weighted sum;
      - the partial is moe_combine of the rank's rows, and an empty rank (Qwen3 at 8: n_ff 768 = 3 x 256) gives zeros;
    and the summed layer is within NMSE 5e-4 of the f64 oracle on the first and last token.
  * One rank's layer captured in a CUDA graph and replayed with ids and weights changed in place.
"""
import numpy as np
import pytest
import torch

from conftest import random_wire
from ik_llama_cpp_b200 import tp
from oracle.oracle import GGML_TYPE, nmse
from test_gpu_decode_schedules import PLAIN_BAR, bar_ratio
from test_gpu_memory_contract import Arena, last_error, run_contract, st
from test_gpu_moe_prefill import glu_ref

pytestmark = pytest.mark.gpu
E_ARG, E_SHAPE = -4, -2


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


def combine_f32(rows, w):
    """the CPU op's loop in f32: y = x0 w0, then y = y + x_u w_u"""
    rows, w = np.asarray(rows, np.float32), np.asarray(w, np.float32)
    y = rows[:, 0] * w[:, 0:1]
    for u in range(1, rows.shape[1]):
        y = y + rows[:, u] * w[:, u:u + 1]
    return y


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the combine kernel
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_tokens", [1, 3, 64, 512])
@pytest.mark.parametrize("m", [7168, 2048, 4097, 6])
@pytest.mark.parametrize("n_used", [1, 2, 8])
def test_combine_bit_equal_to_f32_loop(be, n_used, m, n_tokens):
    rng = np.random.default_rng([n_used, m, n_tokens])
    rows = (rng.standard_normal((n_tokens, n_used, m)) * rng.uniform(0.1, 10.0, (n_tokens, n_used, 1))).astype(np.float32)
    w = rng.uniform(0.0, 1.0, (n_tokens, n_used)).astype(np.float32)
    rows[0, 0, : min(m, 4)] = 0.0                 # a skipped slot's zero row (MUL_MAT_ID writes those)
    ref = combine_f32(rows, w)
    y = be.moe_combine(torch.from_numpy(rows).cuda(), torch.from_numpy(w).cuda()).cpu().numpy()
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32)), f"max |diff| {np.abs(y - ref).max():.3g}"


def test_combine_misaligned_pointers_take_the_scalar_kernel(be):
    """rows and dst 4 bytes past a 16-byte boundary with m % 4 == 0: same bits as the aligned call"""
    n_tokens, n_used, m = 33, 8, 1024
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((n_tokens, n_used, m)).astype(np.float32)
    w = rng.uniform(0.0, 1.0, (n_tokens, n_used)).astype(np.float32)
    buf = torch.zeros(rows.size + 1, device="cuda")
    buf[1:].copy_(torch.from_numpy(rows.ravel()))
    out = torch.zeros(n_tokens * m + 1, device="cuda")
    be.moe_combine(buf[1:].view(n_tokens, n_used, m), torch.from_numpy(w).cuda(), out=out[1:])
    assert np.array_equal(out[1:].cpu().numpy().reshape(n_tokens, m), combine_f32(rows, w))
    assert float(out[0]) == 0.0


@pytest.mark.parametrize("m,n_used,n_tokens", [(7168, 8, 512), (4097, 2, 7), (2048, 1, 1)])
def test_combine_memory_contract(be, m, n_used, n_tokens):
    """guarded arena: dst | rows | weights.  Writes only dst, run A (dst NaN) and run B (dst 1e30) bit-equal and equal to the f32 loop; every rejected
    call (n_used 0, m 0, dst overlapping rows, a NULL input) returns its error and writes nothing."""
    L = be._lib.lib()
    rng = np.random.default_rng([m, n_used])
    rows = rng.standard_normal((n_tokens, n_used, m)).astype(np.float32)
    w = rng.uniform(0.0, 1.0, (n_tokens, n_used)).astype(np.float32)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ar = Arena(m)
        ar.add("dst", n_tokens * m * 4, "out")
        ar.add("rows", rows.nbytes, "in")
        ar.add("w", w.nbytes, "in")
        ar.build()
        ar.put("rows", rows)
        ar.put("w", w)
        what = f"moe_combine m={m} n_used={n_used} tokens={n_tokens}"
        a, _ = run_contract(ar, [("dst", "f32", (n_tokens, m))],
                            lambda wsb: L.b200q_moe_combine(ar.ptr("rows"), ar.ptr("w"), ar.ptr("dst"), m, n_used, n_tokens, st()), what)
        assert np.array_equal(a["dst"], combine_f32(rows, w)), f"{what}: differs from the f32 loop"
        bad = [("n_used 0", (ar.ptr("rows"), ar.ptr("w"), ar.ptr("dst"), m, 0, n_tokens), E_SHAPE),
               ("m 0", (ar.ptr("rows"), ar.ptr("w"), ar.ptr("dst"), 0, n_used, n_tokens), E_SHAPE),
               ("dst overlaps rows", (ar.ptr("rows"), ar.ptr("w"), ar.ptr("rows") + 256, m, n_used, n_tokens), E_ARG),
               ("rows NULL", (None, ar.ptr("w"), ar.ptr("dst"), m, n_used, n_tokens), E_ARG)]
        for why, args, code in bad:
            snap = ar.buf.clone()
            rc = L.b200q_moe_combine(*args, st())
            torch.cuda.synchronize()
            assert rc == code, f"{what}, {why}: rc {rc} ({last_error()}), expected {code}"
            ar.untouched(snap, [], f"{what}, {why}")


# ------------------------------------------------------------------------------------------------------------------------------------------------
# model layers, ranks emulated on one device
# ------------------------------------------------------------------------------------------------------------------------------------------------
# (id, type, n_embd, n_expert, n_used, n_ff_exp, n_ff of the shared expert or 0)
MODELS = [("qwen3-30b-a3b", "Q4_K", 2048, 128, 8, 768, 0),
          ("mixtral-8x7b", "IQ4_NL", 4096, 8, 2, 14336, 0),
          ("deepseek-v3", "IQ2_XXS", 7168, 256, 8, 2048, 2048)]
TOKENS = [1, 8, 64, 512]
POOL = 16           # distinct expert matrices drawn on the host; expert e holds pool matrix e % POOL, its rows in a per-expert rotation


class Layer:
    """Wire bytes of one MoE layer (up, gate, down experts; shared expert) and the unsharded upload."""

    def __init__(self, be, case, seed):
        self.id, self.name, self.n_embd, self.n_expert, self.n_used, self.n_ff, self.n_shexp = case
        self.t = GGML_TYPE[self.name]
        rng = np.random.default_rng(seed)
        self.up, self.gate = (self._experts(rng, self.n_ff, self.n_embd) for _ in range(2))
        self.down = self._experts(rng, self.n_embd, self.n_ff)
        self.U, self.G, self.D = (be.set_expert_tensor(self.t, w, self.n_expert, m, k) for w, m, k in
                                  ((self.up, self.n_ff, self.n_embd), (self.gate, self.n_ff, self.n_embd), (self.down, self.n_embd, self.n_ff)))
        if self.n_shexp:
            self.sh = [random_wire(self.name, m, k, rng) for m, k in ((self.n_shexp, self.n_embd),) * 2 + ((self.n_embd, self.n_shexp),)]

    def _experts(self, rng, m, k):
        pool = [random_wire(self.name, m, k, rng).reshape(m, -1) for _ in range(min(POOL, self.n_expert))]
        return np.concatenate([np.roll(pool[e % len(pool)], 4 * (e // len(pool)), axis=0).ravel() for e in range(self.n_expert)])

    def expert(self, wire, e, m):
        return wire.reshape(self.n_expert, -1)[e]

    def shards(self, be, world, rank):
        """(up, gate, down, shared) of one rank: None for an empty routed shard / shared shard"""
        split = tp.moe_ffn_plan(self.n_ff, world, self.t)
        if split[rank] == 0:
            routed = (None, None, None)
        else:
            ups = [be.set_expert_tensor(self.t, tp.shard_expert_rows(w, self.t, self.n_expert, self.n_ff, self.n_embd, split, rank)[0], self.n_expert,
                                        split[rank], self.n_embd) for w in (self.up, self.gate)]
            dsh, ks, _ = tp.shard_expert_cols(self.down, self.t, self.n_expert, self.n_embd, self.n_ff, split, rank)
            routed = (*ups, be.set_expert_tensor(self.t, dsh, self.n_expert, self.n_embd, ks))
        shared = None
        if self.n_shexp:
            g = tp.moe_expert_granularity(self.t)
            (u, mu), (gt, _) = (tp.shard_rows(w, self.t, self.n_shexp, self.n_embd, world, rank, granularity=g) for w in self.sh[:2])
            d, ks, _ = tp.shard_cols(self.sh[2], self.t, self.n_embd, self.n_shexp, world, rank, granularity=g)
            if mu:
                shared = be.SharedExpert(be.set_tensor(self.t, u, mu, self.n_embd), be.set_tensor(self.t, gt, mu, self.n_embd), be.set_tensor(self.t, d, self.n_embd, ks))
        return split, routed, shared


_layers = {}


def layer(be, case):
    """the layer of a model shape, uploaded once per module"""
    if case[0] not in _layers:
        _layers[case[0]] = Layer(be, case, seed=GGML_TYPE[case[1]])
    return _layers[case[0]]


def routing(rng, n_tokens, n_expert, n_used):
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    p = rng.uniform(0.05, 1.0, (n_tokens, n_used)).astype(np.float32)
    return ids, (p / p.sum(axis=1, keepdims=True)).astype(np.float32)


def oracle_layer(oracle, L, x, ids, w, tokens, q8_up_gate, q8_down, q8_shared):
    """f64 MoE FFN (+ shared expert) of the given tokens on the wire bytes.  A stage that runs on the mat-vec path is restated with its activations
    quantised to q8_1 as the kernel does (the q8_1 oracle of the decode suites), a stage on the GEMM path exactly."""
    def mm(q8, t, wire, a, m):
        a = np.asarray(a, np.float32)
        return oracle.mul_mat_q8_1(t, wire, a, m, variant="b200") if q8 else oracle.mul_mat_exact(t, wire, a, m)
    out = []
    for tk in tokens:
        xt = x[tk:tk + 1]
        y = np.zeros(L.n_embd)
        for u, e in enumerate(ids[tk]):
            h = glu_ref("silu", mm(q8_up_gate, L.t, L.expert(L.gate, e, L.n_ff), xt, L.n_ff), mm(q8_up_gate, L.t, L.expert(L.up, e, L.n_ff), xt, L.n_ff))
            y += float(w[tk, u]) * mm(q8_down, L.t, L.expert(L.down, e, L.n_embd), h, L.n_embd)[0]
        if L.n_shexp:
            h = glu_ref("silu", mm(q8_shared, L.t, L.sh[1], xt, L.n_shexp), mm(q8_shared, L.t, L.sh[0], xt, L.n_shexp))
            y += mm(q8_shared, L.t, L.sh[2], h, L.n_embd)[0]
        out.append(y)
    return np.stack(out)


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("case", MODELS, ids=[c[0] for c in MODELS])
def test_rank_partials_add_up_to_the_unsharded_layer(be, oracle, case, world):
    L = layer(be, case)
    rng = np.random.default_rng([world, L.n_expert])
    xs = {n: (rng.standard_normal((n, L.n_embd)) * 0.5).astype(np.float32) for n in TOKENS}
    routes = {n: routing(rng, n, L.n_expert, L.n_used) for n in TOKENS}
    full = {}
    for n in TOKENS:            # the unsharded launches
        x, ids, w = torch.from_numpy(xs[n]).cuda(), torch.from_numpy(routes[n][0]).cuda(), torch.from_numpy(routes[n][1]).cuda()
        par = be.mul_mat_id_dispatch(L.U, x.view(n, 1, -1), ids, gate=L.G)
        rows = be.mul_mat_id_dispatch(L.D, par, ids)
        full[n] = (par.cpu(), rows.cpu().numpy(), be.moe_combine(rows, w).cpu().numpy())
    sums = {n: (np.zeros_like(full[n][1], np.float64), np.zeros_like(full[n][2], np.float64)) for n in TOKENS}
    for rank in range(world):
        split, (U, G, D), shared = L.shards(be, world, rank)
        r0 = sum(split[:rank])
        for n in TOKENS:
            x, ids, w = torch.from_numpy(xs[n]).cuda(), torch.from_numpy(routes[n][0]).cuda(), torch.from_numpy(routes[n][1]).cuda()
            part = be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G).cpu().numpy()
            what = f"{L.id} W={world} rank {rank} tokens={n}"
            if D is None:
                assert not part.any(), f"{what}: an empty shard must give a zero partial"
                continue
            par = be.mul_mat_id_dispatch(U, x.view(n, 1, -1), ids, gate=G)
            assert torch.equal(par.cpu(), full[n][0][:, :, r0:r0 + split[rank]]), f"{what}: up/gate rows differ from the unsharded launch's"
            rows = be.mul_mat_id_dispatch(D, par, ids)
            assert np.array_equal(part, be.moe_combine(rows, w).cpu().numpy()), f"{what}: the partial is not the combine of the rank's rows"
            sums[n][0][...] += rows.cpu().numpy()
            sums[n][1][...] += part
    for n in TOKENS:
        _, rows_full, comb_full = full[n]
        ids, w = routes[n]
        what = f"{L.id} W={world} tokens={n}"
        grouped = be.mul_mat_id_workspace(L.D, n, L.n_used, L.n_used, False) > 0
        if grouped:
            e = nmse(sums[n][0], rows_full)
            assert e <= 2e-5, f"{what}: summed ffn_down rows NMSE {e}"
            e = nmse(sums[n][1], comb_full)
            assert e <= 2e-5, f"{what}: summed partials NMSE {e}"
        else:
            for tk in range(n):
                for u in range(L.n_used):
                    bar_ratio(sums[n][0][tk, u], rows_full[tk, u], PLAIN_BAR, f"{what}: summed ffn_down rows, token {tk} slot {u}")
            # the per-slot bars carried through the weighted sum: |sum of partials - combine| <= sum_u w_u bar rms(row_u)
            rms = np.sqrt((rows_full.astype(np.float64) ** 2).mean(axis=2))
            bound = PLAIN_BAR * (w.astype(np.float64) * rms).sum(axis=1, keepdims=True)
            err = np.abs(sums[n][1] - comb_full)
            assert np.all(err <= bound), f"{what}: summed partials exceed the carried bar by {float((err / bound).max()):.3g}x"
        print(f"{what} ({'grouped GEMM' if grouped else 'mat-vec'}): up/gate rows bit-equal, partials add up to the unsharded layer")


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("case", MODELS, ids=[c[0] for c in MODELS])
def test_summed_layer_against_the_oracle(be, oracle, case, world):
    """the whole partial (routed experts + shared expert) summed over the ranks, NMSE <= 5e-4 against the f64 oracle on the first and last token
    (each stage restated as its path computes it: q8_1 activations on the mat-vec path)"""
    L = layer(be, case)
    rng = np.random.default_rng([world, 7])
    xs = {n: (rng.standard_normal((n, L.n_embd)) * 0.5).astype(np.float32) for n in TOKENS}
    routes = {n: routing(rng, n, L.n_expert, L.n_used) for n in TOKENS}
    total = {n: np.zeros((n, L.n_embd)) for n in TOKENS}
    for rank in range(world):
        _, (U, G, D), shared = L.shards(be, world, rank)
        for n in TOKENS:
            x, ids, w = (torch.from_numpy(a).cuda() for a in (xs[n], *routes[n]))
            total[n] += be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G, shared=shared).cpu().numpy()
    for n in TOKENS:
        tokens = sorted({0, n - 1})
        ref = oracle_layer(oracle, L, xs[n], *routes[n], tokens, q8_up_gate=be.mul_mat_id_workspace(L.U, n, L.n_used, 1, True) == 0,
                           q8_down=be.mul_mat_id_workspace(L.D, n, L.n_used, L.n_used, False) == 0, q8_shared=n <= be.MMVQ_MAX_BATCH_SIZE)
        e = nmse(total[n][tokens], ref)
        print(f"{L.id} W={world} tokens={n}: summed layer NMSE vs f64 oracle {e:.3g}")
        assert e <= 5e-4, f"{L.id} W={world} tokens={n}: NMSE {e}"


def test_merged_shards_give_the_split_partial(be):
    """a rank's merged gate_up shard (tp.shard_expert_gate_up) gives the same partial as its split up / gate shards, bit for bit"""
    L = layer(be, MODELS[0])
    split = tp.moe_ffn_plan(L.n_ff, 2, L.t)
    merged_wire = np.concatenate([np.concatenate([L.expert(L.gate, e, L.n_ff), L.expert(L.up, e, L.n_ff)]) for e in range(L.n_expert)])
    rng = np.random.default_rng(11)
    for rank in range(2):
        _, (U, G, D), _ = L.shards(be, 2, rank)
        sh, n_r = tp.shard_expert_gate_up(merged_wire, L.t, L.n_expert, L.n_ff, L.n_embd, split, rank)
        GU = be.set_expert_tensor(L.t, sh, L.n_expert, 2 * n_r, L.n_embd)
        for n in (1, 64):
            x = torch.from_numpy(rng.standard_normal((n, L.n_embd)).astype(np.float32)).cuda()
            ids, w = (torch.from_numpy(a).cuda() for a in routing(rng, n, L.n_expert, L.n_used))
            a = be.moe_tp_partial(x, ids, w, L.n_embd, D, gate_up=GU)
            b = be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G)
            assert torch.equal(a, b), f"rank {rank} tokens={n}"


@pytest.mark.parametrize("with_shared", [False, True], ids=["routed", "routed+shared"])
@pytest.mark.parametrize("n_tokens", [1, 64])
def test_captured_rank_layer_with_ids_and_weights_changed_in_place(be, n_tokens, with_shared):
    """One rank's layer (DeepSeek-V3 shapes, W = 8) captured once, replayed with new ids and weights written in place: equal to an eager call on the
    new ones, bit for bit.  With the shared expert at 64 tokens its dense GEMMs may split K over f32 atomics, whose order varies from run to run:
    there the replay is held to the GEMM bar of test_gpu_parity.py (NMSE 2e-5) instead."""
    L = layer(be, MODELS[2])
    _, (U, G, D), shared = L.shards(be, 8, 3)
    shared = shared if with_shared else None
    rng = np.random.default_rng(n_tokens)
    x = torch.from_numpy(rng.standard_normal((n_tokens, L.n_embd)).astype(np.float32)).cuda()
    ids, w = (torch.from_numpy(a).cuda() for a in routing(rng, n_tokens, L.n_expert, L.n_used))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G, shared=shared)          # warm-up: workspaces exist before the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G, shared=shared)
    for _ in range(2):
        ni, nw = routing(rng, n_tokens, L.n_expert, L.n_used)
        ids.copy_(torch.from_numpy(ni))
        w.copy_(torch.from_numpy(nw))
        g.replay()
        torch.cuda.synchronize()
        eager = be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G, shared=shared)
        if shared is not None and n_tokens > be.MMVQ_MAX_BATCH_SIZE:
            assert nmse(out.cpu().numpy(), eager.cpu().numpy()) <= 2e-5
        else:
            assert torch.equal(out, eager)


def _harness(mode):
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "backend_ops", "test_moe_combine_backend")
    if not os.path.exists(exe):
        pytest.skip("harness not built (needs the reference headers at build time)")
    r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED: 0 failures" in r.stdout


def test_mul_multi_add_node_against_the_reference_cpu_op():
    """MUL_MULTI_ADD alone on the plug and on the reference CPU backend: n_used 1, 2, 8, m 7168 and 4097, 1 ... 512 tokens, NMSE <= 5e-4."""
    _harness("op")


def test_fused_mmad_moe_ffn_combines_on_the_plug():
    """llm_build_moe_ffn with fused_mmad at the three model shapes, 1 ... 512 tokens, under ggml_backend_sched next to the CPU backend: ffn_down_exps and
    MUL_MULTI_ADD run on the plug, and the layer output matches the same graph on the reference CPU backend (NMSE <= 5e-4)."""
    _harness("graph")
