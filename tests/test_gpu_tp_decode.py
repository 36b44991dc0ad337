"""Every tensor-parallel decode kernel on ONE GPU: W ranks emulated over the tagged-slot exchange, every plane type, checked bit for bit.

b200q_mul_mat_vec_tp fuses GGML_OP_REDUCE into k_mmvq_ring<T, 1, UPGATE, MULTI, PAIR, TP = true, 0> (b200q_decode_ring.cuh):
  * reduce_out: each finished partial row goes to entry ((tps & 1) * world + rank) * ll_stride + row of every rank's slot array as {value, tps + 1}
    (tps = ll_state[0], the reduces this rank has issued); the last warp of the last CTA bumps ll_state[0];
  * reduce_in: x is ignored; the consumer sums the W slots of reduce tps (parity (tps - 1) & 1) in rank order, directly for world == 2, through a
    publish hop in ll_reduced for world > 2 (with a bounded poll and a fall-back to ll_sum_slots), and quantises from there.
The unicast stores (B200Q_TP_UNICAST=1, ll_peers given) write the same entries, tags and counters with ordinary stores into every rank's copy of the
slot array; the consumer side reads only its own copy and ll_reduced, the same code on both paths.  So W ranks are emulated on one device: per rank
a slot array of 2 W ll_stride entries, an ll_reduced of 2 ll_stride entries and an ll_state, all zeroed and carved from one Arena
(test_gpu_memory_contract.py) with NaN guards between them; ll_peers = the W slot arrays, ll_mc = NULL (the library refuses NULL unless the
unicast stores are selected, so a wrong set-up fails cleanly instead of issuing multimem.st to an ordinary address).  The launches of one reduce are
issued rank 0 .. W-1 reduce_out, then rank 0 .. W-1 consumers, one after another on one stream; the ranks never run concurrently.

Nothing may hang the GPU.  Before every reduce_in launch the test synchronises and checks on the host that the consuming rank's ll_state[0] is the
expected count and that every entry [parity][r][0:K] of its slot copy carries the expected tag for every r; only then does it launch, so no consumer
ever waits for an entry.  A mutated tag or slot offset therefore stops at this precondition, before any consumer runs.  A CUDA-graph replay of a
chain only follows the same chain passing eagerly.

Checks (every launch, against the whole arena: one byte outside the expected changes fails, named by region):
  * reduce_out of rank r, reduce n: slot values [par][r][0:M_total] in every copy are bit-identical to the plain b200q_mul_mat_vec / _multi of the
    same shard on the same x slice (planned as the same ring kernel with TP = false), tags are n, ll_state = {n, 0}; entries >= M_total, the other
    parity, the other ranks' regions, every ll_reduced, the NaN-filled dst and the guards are unchanged.  The values also meet PLAIN_BAR against
    oracle.mul_mat_q8_1(..., variant="b200");
  * reduce_in: the reduced vector h is rebuilt on the host as ((0 + s0) + s1) + ... in f32, as ll_sum_slots adds; world > 2: ll_reduced[par][0:K]
    is h bit for bit with tag n.  The output is bit-identical to the plain launch (b200q_mul_mat_vec, _multi of Q,K,V, b200q_fused_up_gate_vec
    with silu, silu limit 1.5, gelu, relu, swiglu_oai) on h uploaded as x, so every emulated rank gives the same bits (DESIGN.md §7), and meets
    PLAIN_BAR / GLU_BAR against the oracle.  Slot arrays and ll_state are unchanged (a launch that also reduces out: see above).
Chains have >= 4 reduces with changing lengths, so both parities are reused over stale tails of other lengths; every chain runs with PDL on and
off (bit-identical), then from a CUDA graph replayed three times with new inputs, each replay equal to the plain-launch chain on its inputs.

Coverage: every plane type with all 6 TP instantiations in the roles production uses (plain reduce_out on row pairs and long rows, MULTI reduce_in
Q,K,V and UPGATE reduce_in on both, plain reduce_in for the head), worlds 2, 3 (uneven tp.create_split shards), 4 and 8, an odd M_total, a MULTI
reduce_out and a launch with reduce_in and reduce_out together.  The sweep runs with B200Q_TP_ROWBUF=0 (the per-row stores, production's multicast
default); a few cases run the row buffer, whose long-row flushes start at odd rows.  Model-shaped chains at bench.py --gpus 2 dimensions
(Llama-3-8B, W = 2) cover the bench types.  Each case runs in a child process under torch.profiler: every TP launch must be k_mmvq_ring<..., true, 0>
with the template arguments of its role and the grid and block of its plain twin, whose configurations test_gpu_decode_schedules.py pins at 132 SMs.

Rejections: wire types (B200Q_E_TYPE), K % 256 != 0, M_total > ll_stride, K > ll_stride, no ring geometry (B200Q_E_SHAPE), a gate with reduce_out
and an incomplete communicator (B200Q_E_ARG) change no byte of the arena; a TP launch is accepted exactly when the plain n = 1 launch of the same
tensors is planned on the ring kernel and the documented K and ll_stride conditions hold (asserted from the two traces).

Not reached here: the multimem.st instruction itself and real cross-GPU timing (test_gpu_tp.py on multi-GPU machines, test_reduce_protocol.py).
The CPU self-test shows on host arrays that the checks reject each planted defect.
"""
import ctypes
import json
import os
import sys
import zlib
from ctypes import c_int64, c_void_p

import numpy as np
import pytest
import torch

from conftest import PLANE_TYPES, WIRE_TYPES, make_wire
from oracle.oracle import GGML_TYPE
from test_gpu_decode_schedules import GLU_BAR, PLAIN_BAR, bar_ratio, matmul_launches, profiled, run_child
from test_gpu_memory_contract import Arena
from test_gpu_parity import glu_ref, rms

E_TYPE, E_SHAPE, E_ARG = -1, -2, -4
UNARY = {"none": 0, "silu": 1, "gelu": 2, "relu": 3, "swiglu_oai": 4}
GLUS = [("silu", 0.0), ("silu", 1.5), ("gelu", 0.0), ("relu", 0.0), ("swiglu_oai", 0.0)]
ROWBUF_OFF = {"B200Q_TP_UNICAST": "1", "B200Q_TP_ROWBUF": "0"}
ROWBUF_ON = {"B200Q_TP_UNICAST": "1", "B200Q_TP_ROWBUF": "1"}


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the exchange as the host sees it (device agnostic: the CPU self-test runs it on a host arena)
# ------------------------------------------------------------------------------------------------------------------------------------------------
def entries(values, tag):
    """{f32 value, u32 tag} entries as bytes"""
    e = np.empty((len(values), 2), np.uint32)
    e[:, 0] = np.asarray(values, np.float32).view(np.uint32)
    e[:, 1] = tag
    return e.view(np.uint8).reshape(-1)


def rank_order_sum(parts):
    """h = ((0 + s0) + s1) + ... in f32, the order of ll_sum_slots (world == 2 adds s0 + s1 directly: the same value, the sign of a zero aside)"""
    h = np.zeros_like(np.asarray(parts[0], np.float32))
    for p in parts:
        h = (h + np.asarray(p, np.float32)).astype(np.float32)
    return h


class Exchange:
    """The per-rank regions of W emulated ranks in an arena: slots{q} [2][W][S] entries, red{q} [2][S] entries, state{q} u32[4]"""

    def __init__(self, ar, W, S):
        self.ar, self.W, self.S = ar, W, S

    @staticmethod
    def add(ar, W, S):
        for q in range(W):
            ar.add(f"slots{q}", 2 * W * S * 8, "out")
            ar.add(f"red{q}", 2 * S * 8, "out")
            ar.add(f"state{q}", 16, "out")

    def zero(self):
        for q in range(self.W):
            for name in (f"slots{q}", f"red{q}", f"state{q}"):
                self.ar.fill(name, 0)

    def slot_off(self, q, par, r, row=0):
        return self.ar.regions[f"slots{q}"][0] + ((par * self.W + r) * self.S + row) * 8

    def out_edits(self, r, n, values):
        """what reduce_out of rank r, reduce n, writes: its rows in parity (n - 1) & 1 of every copy, and its count"""
        ed = [(self.slot_off(q, (n - 1) & 1, r), entries(values, n)) for q in range(self.W)]
        return ed + [(self.ar.regions[f"state{r}"][0], np.array([n, 0], np.uint32).view(np.uint8))]

    def in_edits(self, r, n, h):
        """what the consumption of reduce n writes on rank r besides its outputs: world > 2 publishes h in ll_reduced"""
        if self.W == 2:
            return []
        return [(self.ar.regions[f"red{r}"][0] + ((n - 1) & 1) * self.S * 8, entries(h, n))]

    def precondition(self, r, n, k):
        """Before a reduce_in launch of rank r for reduce n: its count is n and every entry [par][q][0:k] of its copy carries tag n.  Raises
        (and nothing is launched) otherwise: a consumer launched now would wait for entries that never arrive."""
        state = self.ar.get(f"state{r}", "i32", (4,)).view(np.uint32)
        assert state[0] == n, f"precondition of rank {r}'s consumer of reduce {n}: ll_state[0] = {state[0]}, not launching"
        tags = self.ar.get(f"slots{r}", "i32", (2, self.W, self.S, 2)).view(np.uint32)[(n - 1) & 1, :, :k, 1]
        bad = np.argwhere(tags != n)
        assert len(bad) == 0, (f"precondition of rank {r}'s consumer of reduce {n}: {len(bad)} entries of parity {(n - 1) & 1} lack tag {n}, first "
                               + ", ".join(f"[rank {q}][{e}] = {tags[q, e]}" for q, e in bad[:4]) + "; not launching")


def glu_ratio(y, g, u, unary, limit, what):
    """act(g) * u against the oracle: GLU_BAR rms(ref); with a clamp (silu limit, swiglu_oai) the clamp caps ref but not the error g and u carry,
    so there the plain bar of g and u is propagated through the activation (the four corners of the error box) and GLU_BAR rms(ref) added"""
    ref = glu_ref(unary, g, u, limit)
    if not (unary == "swiglu_oai" or limit > 1e-6):
        return bar_ratio(y, ref, GLU_BAR, what)
    eg, eu = PLAIN_BAR * rms(g), PLAIN_BAR * rms(u)
    prop = np.max([np.abs(glu_ref(unary, g + sg * eg, u + su * eu, limit) - ref) for sg in (-1, 1) for su in (-1, 1)], axis=0)
    bound = prop + GLU_BAR * rms(ref)
    err = np.abs(np.asarray(y, np.float64) - ref)
    bad = np.argwhere(~(err <= bound))
    assert len(bad) == 0, (f"{what}: {len(bad)} of {err.size} elements outside the propagated bound, first "
                           + ", ".join(f"{tuple(int(i) for i in b)}: y={y[tuple(b)]:.7g} ref={ref[tuple(b)]:.7g} bound={bound[tuple(b)]:.3g}" for b in bad[:5]))
    return float((err / bound).max())


def expect(ar, snap, edits, what):
    """The arena equals the snapshot with the edits applied, byte for byte; a difference is named by region"""
    want = snap.clone()
    for off, data in edits:
        want[off:off + len(data)] = torch.from_numpy(np.ascontiguousarray(data)).to(want.device)
    diff = ar.buf != want
    if bool(diff.any()):
        idx = torch.nonzero(diff).flatten()
        raise AssertionError(f"{what}: {idx.numel()} bytes differ from the expected memory, first at "
                             + ", ".join(ar.where(int(i)) for i in idx[:6].cpu()))


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-test
# ------------------------------------------------------------------------------------------------------------------------------------------------
SELF_DEFECTS = ["tree-ordered sum", "reversed-rank sum", "stale tag", "row at offset +1", "write to entry M_total", "consumer read x"]


def _emulated_chain(defect):
    """One reduce of W = 3 ranks with ll_stride == M_total on a host arena: each rank's reduce_out "kernel" stores its partial rows, then rank 0's
    consumer publishes h and computes y = A h.  The partials are chosen so that the three summation orders give different bits."""
    W, S, M = 3, 64, 64
    ar = Arena(M, device="cpu")
    Exchange.add(ar, W, S)
    ar.add("y", M * 4, "out")
    ar.build()
    ex = Exchange(ar, W, S)
    ex.zero()
    ar.fill("y", 0x7FC07FC0)
    rng = np.random.default_rng(3)
    parts = [rng.standard_normal(M).astype(np.float32) * s for s in (1.0, 1e8, -1e8)]
    parts[2] = (-parts[1] + rng.standard_normal(M).astype(np.float32)).astype(np.float32)
    x = rng.standard_normal(M).astype(np.float32)
    A = rng.standard_normal((M, M)).astype(np.float32)
    host = ar.buf.numpy()
    n = 1
    for r in range(W):                                  # reduce_out of every rank
        snap = ar.buf.clone()
        for q in range(W):
            off = ex.slot_off(q, 0, r) + (8 if defect == "row at offset +1" else 0)
            e = entries(parts[r], n)
            host[off:off + len(e)] = e
            if defect == "write to entry M_total" and r == 0:
                host[ex.slot_off(q, 0, r, M):ex.slot_off(q, 0, r, M) + 8] = entries(parts[r][-1:], n)
        off = ar.regions[f"state{r}"][0]
        host[off:off + 4] = np.array([n], np.uint32).view(np.uint8)
        expect(ar, snap, ex.out_edits(r, n, parts[r]), f"emulated reduce_out rank {r}")
    if defect == "stale tag":                           # rank 1's entry 5 in rank 0's copy still from the reduce before
        host[ex.slot_off(0, 0, 1, 5) + 4:ex.slot_off(0, 0, 1, 5) + 8] = np.array([n - 1], np.uint32).view(np.uint8)
    ex.precondition(0, n, M)
    h = rank_order_sum(parts)
    got = h
    if defect == "tree-ordered sum":
        got = (parts[0] + (parts[1] + parts[2]).astype(np.float32)).astype(np.float32)
    if defect == "reversed-rank sum":
        got = rank_order_sum(parts[::-1])
    snap = ar.buf.clone()
    off = ar.regions["red0"][0]
    e = entries(got, n)
    host[off:off + len(e)] = e
    y = (A.astype(np.float64) @ (x if defect == "consumer read x" else got).astype(np.float64)).astype(np.float32)
    host[ar.regions["y"][0]:ar.regions["y"][0] + M * 4] = y.view(np.uint8)
    y_plain = (A.astype(np.float64) @ h.astype(np.float64)).astype(np.float32)
    expect(ar, snap, ex.in_edits(0, n, h) + [(ar.regions["y"][0], y_plain.view(np.uint8))], "emulated consumer")


def test_checker_catches_planted_defects():
    """The clean emulated reduce passes; each planted defect is rejected: a tree-ordered or reversed-rank sum (W = 3, data whose orders differ), one
    stale tag (refused by the launch precondition), a row stored one entry too far, a write to entry M_total when ll_stride == M_total (the next
    rank's region), a consumer that read x instead of the slots."""
    p = [np.float32(1.0), np.float32(1e8), np.float32(-1e8)]
    assert rank_order_sum(p) != rank_order_sum(p[::-1]) and rank_order_sum(p) != p[0] + (p[1] + p[2]), "the data must tell the orders apart"
    _emulated_chain(None)
    for defect in SELF_DEFECTS:
        with pytest.raises(AssertionError):
            _emulated_chain(defect)


# ------------------------------------------------------------------------------------------------------------------------------------------------
# case table
# ------------------------------------------------------------------------------------------------------------------------------------------------
# A chain is a list of reduces.  Producer: ("plain" | "multi", type, [M, ...], K_full) -- K_full is split over the ranks by tp.create_split in units
# of 2048 (every plane type has a ring geometry at multiples of 2048) and every rank gets its tp.shard_cols shard; or ("prev",): the previous
# consumer reduced out.  Consumer (weights the same on every rank): ("head" | "multi", type, [M, ...], K), ("upgate", type, [M], K, unary, limit),
# ("both", type, [M], K): a plain launch with reduce_in and reduce_out, its weights different per rank.  A fifth producer field overrides the
# granularity of the split.
GRAN = 2048


def sweep_chain(name, i):
    u1, u2 = GLUS[i % 5], GLUS[(i + 2) % 5]
    return [
        (("plain", name, [4096], 2048), ("multi", name, [512, 128, 128], 4096)),                 # row pairs out, MULTI row pairs in
        (("plain", name, [6144], 6144), ("multi", name, [512, 128, 128], 6144)),                 # long rows out (M_total == ll_stride), MULTI long in
        (("plain", name, [4097], 2048), ("upgate", name, [1024], 4096) + u1),                    # odd M_total: the last pair has one row
        (("plain", name, [6144], 6144), ("upgate", name, [512], 6144) + u2),                     # UPGATE long rows
        (("multi", name, [2048, 1024, 1023], 2048), ("head", name, [1000], 2048)),               # MULTI reduce_out, head on row pairs
    ]


def k_full(kind_k, W):
    return kind_k * W if W != 3 else {2048: 4 * GRAN, 6144: 7 * GRAN}[kind_k]      # W = 3: uneven shards (4096, 2048, 2048) / (6144, 4096, 4096)


CASES = []
for _i, _name in enumerate(PLANE_TYPES):
    _W = (2, 3, 4, 8)[_i % 4]
    CASES.append((f"sweep-{_name.lower()}-w{_W}", _W, 6144, ROWBUF_OFF, [(((p[0], p[1], p[2], k_full(p[3], _W)) if p[0] != "prev" else p), c)
                                                                             for p, c in sweep_chain(_name, _i)]))
for _name, _W in (("IQ4_NL", 3), ("Q4_K", 8), ("Q6_K", 2), ("IQ2_BN", 4)):
    CASES.append((f"rowbuf-{_name.lower()}-w{_W}", _W, 6144, ROWBUF_ON, [(((p[0], p[1], p[2], k_full(p[3], _W)) if p[0] != "prev" else p), c)
                                                                          for p, c in sweep_chain(_name, 1)]))
# reduce_in and reduce_out in one launch, every unary on the up/gate consumer, world 8
CASES.append(("both-and-every-glu-iq4_nl-w8", 8, 4096, ROWBUF_OFF, [
    (("plain", "IQ4_NL", [4096], 8 * 2048), ("both", "IQ4_NL", [4096], 4096)),
    (("prev",), ("upgate", "IQ4_NL", [1024], 4096) + GLUS[0]),
    (("plain", "IQ4_NL", [2048], 8 * 2048), ("upgate", "IQ4_NL", [1024], 2048) + GLUS[1]),
    (("plain", "IQ4_NL", [4096], 8 * 2048), ("upgate", "IQ4_NL", [1024], 4096) + GLUS[2]),
    (("plain", "IQ4_NL", [2048], 8 * 2048), ("upgate", "IQ4_NL", [1024], 2048) + GLUS[3]),
    (("plain", "IQ4_NL", [4096], 8 * 2048), ("upgate", "IQ4_NL", [1024], 4096) + GLUS[4]),
]))


def llama_chain(t_qkv, t_down, t_head):
    """two Llama-3-8B layers under bench.py --gpus 2: wo [4096 x 2048] and ffn_down [4096 x 7168] per rank reduce out; up/gate [7168 x 4096],
    Q,K,V [2048, 512, 512 x 4096] and the head (8192 of its 64128 rows per rank) reduce in; ll_stride 4096 = M_total"""
    up = ("upgate", "IQ4_NL", [7168], 4096, "silu", 0.0)
    wo, down = ("plain", "IQ4_NL", [4096], 4096, 256), ("plain", t_down, [4096], 14336, 256)        # the shards of bench.py: 2048 and 7168 columns
    return [(wo, up), (down, ("multi", t_qkv, [2048, 512, 512], 4096)), (wo, up), (down, ("head", t_head, [8192], 4096))]


for _name, _roles in (("IQ4_NL", ("IQ4_NL", "IQ4_NL", "IQ4_NL")), ("Q5_K", ("IQ4_NL", "Q5_K", "IQ4_NL")), ("IQ5_K", ("IQ5_K", "IQ4_NL", "IQ4_NL")),
                      ("Q6_K", ("IQ4_NL", "IQ4_NL", "Q6_K"))):
    CASES.append((f"llama8b-w2-{_name.lower()}", 2, 4096, ROWBUF_OFF, llama_chain(*_roles)))
CASE_IDS = [c[0] for c in CASES]


# ------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: the emulation
# ------------------------------------------------------------------------------------------------------------------------------------------------
def lib():
    from ik_llama_cpp_b200 import _lib
    return _lib.lib()


def st():
    return torch.cuda.current_stream().cuda_stream


def ptrs(vals, ct=c_void_p):
    return (ct * len(vals))(*vals)


def tp_flags(kind, k):
    """(UPGATE, MULTI, PAIR) template arguments of a launch"""
    return (kind == "upgate", kind == "multi", k <= 4096)


class Chain:
    def __init__(self, be, oracle, case):
        self.id, self.W, self.S, _, self.steps = case
        self.be, self.oracle, self.L = be, oracle, lib()
        from ik_llama_cpp_b200 import tp
        W, S = self.W, self.S
        seed = zlib.crc32(self.id.encode()) % 100000
        self.rng = np.random.default_rng(seed)
        self.log = []                                   # mat-vec launches in order: (kind, flags, twin index, label)
        self.ratios = {}
        self.prod, self.cons = [], []
        for i, (p, c) in enumerate(self.steps):
            if p[0] == "prev":
                self.prod.append(None)
            else:
                kind, name, ms, kf = p[:4]
                gran = p[4] if len(p) > 4 else GRAN
                t = GGML_TYPE[name]
                sizes = tp.create_split(kf, gran, W)
                wires = [make_wire(oracle, name, m, kf, seed=[seed, i, j]) for j, m in enumerate(ms)]
                shards = []
                for r in range(W):
                    tens = []
                    for wire, m in zip(wires, ms):
                        sh, ks, k0 = tp.shard_cols(wire, t, m, kf, W, r, granularity=gran)
                        tens.append((sh, be.set_tensor(t, sh, m, ks)))
                    shards.append((tens, sum(sizes[:r]), sizes[r]))
                self.prod.append((kind, name, t, ms, kf, shards))
            kind, name, ms, k = c[:4]
            t = GGML_TYPE[name]
            if kind == "both":                          # per-rank weights
                ws = [[(w, be.set_tensor(t, w, ms[0], k)) for w in [make_wire(oracle, name, ms[0], k, seed=[seed, i, 50 + r])]] for r in range(W)]
            else:
                n_t = 2 if kind == "upgate" else len(ms)
                ms_t = ms * 2 if kind == "upgate" else ms
                ws = [(w, be.set_tensor(t, w, m, k)) for w, m in [(make_wire(oracle, name, m, k, seed=[seed, i, 100 + j]), m) for j, m in enumerate(ms_t[:n_t])]]
            self.cons.append((kind, name, t, ms, k, c[4:] if kind == "upgate" else ("none", 0.0), ws))
        ar = Arena()
        Exchange.add(ar, W, S)
        kmax = max(c[3] for c in (s[1] for s in self.steps))
        ar.add("nanx", kmax * 4, "in")
        ar.add("nandst", S * 4, "in")
        for i, (p, c) in enumerate(self.steps):
            if p[0] != "prev":
                for r in range(W):
                    ar.add(f"x{i}_{r}", self.prod[i][5][r][2] * 4, "in")
            if c[0] != "both":
                for r in range(W):
                    for j, m in enumerate(c[2]):
                        ar.add(f"y{i}_{r}_{j}", m * 4, "out")
        self.ar = ar.build()
        self.ex = Exchange(ar, W, S)
        self.ex.zero()
        self.n = 0                                      # reduces issued so far (every rank's ll_state[0])
        peers = ptrs([ar.ptr(f"slots{q}") for q in range(W)])
        self._peers = peers
        from ik_llama_cpp_b200.backend import NvlsComm
        self.comms = [NvlsComm(None, ar.ptr(f"slots{q}"), ar.ptr(f"red{q}"), S, W, q, ar.ptr(f"state{q}"), ctypes.cast(peers, ctypes.POINTER(c_void_p)))
                      for q in range(W)]
        torch.cuda.synchronize()

    # ---- inputs ----
    def new_inputs(self):
        xs = []
        for p in self.prod:
            if p is None:
                xs.append(None)
                continue
            x = self.rng.standard_normal((1, p[4])).astype(np.float32)
            for r, (_, k0, ks) in enumerate(p[5]):
                self.ar.put(f"x{len(xs)}_{r}", np.ascontiguousarray(x[:, k0:k0 + ks]))
            xs.append(x)
        return xs

    # ---- plain launches (the twins) ----
    def plain(self, t, kind, ws, k, x, outs, glu, label, flags=None):
        L = self.L
        W_ = [w.ptr for _, w in ws]
        if kind == "upgate":
            rc = L.b200q_fused_up_gate_vec(t, W_[0], W_[1], x, outs[0].data_ptr(), ws[0][1].m, k, 1, k, UNARY[glu[0]], glu[1], st())
        elif len(ws) > 1:
            rc = L.b200q_mul_mat_vec_multi(t, len(ws), ptrs(W_), ptrs([o.data_ptr() for o in outs]), ptrs([w.m for _, w in ws], c_int64), k, x, 1, k, st())
        else:
            rc = L.b200q_mul_mat_vec(t, W_[0], x, outs[0].data_ptr(), ws[0][1].m, k, 1, k, None, st())
        assert rc == 0, f"{label}: plain launch rc {rc}: {L.b200q_last_error().decode()}"
        self.log.append(("plain", None, None, label))
        return len(self.log) - 1

    def tp(self, t, kind, ws, k, x, dsts, glu, r, rin, rout, twin, label):
        L = self.L
        n_t = 1 if kind == "upgate" else len(ws)
        W_ = [w.ptr for _, w in ws]
        rc = L.b200q_mul_mat_vec_tp(t, n_t, ptrs(W_[:n_t]), W_[1] if kind == "upgate" else None, ptrs(dsts), ptrs([w.m for _, w in ws][:n_t], c_int64), k,
                                    x, UNARY[glu[0]], glu[1], ctypes.byref(self.comms[r]), int(rin), int(rout), st())
        assert rc == 0, f"{label}: rc {rc}: {L.b200q_last_error().decode()}"
        self.log.append(("tp", tp_flags(kind, k) if kind != "both" else (False, False, k <= 4096), twin, label))

    # ---- one pass over the chain ----
    def run(self, xs, check=True, oracle=False, tp_only=False):
        """Returns {output region: bytes}.  tp_only: the TP launches alone (graph capture); otherwise every reduce is checked as the docstring says."""
        W, ar, ex = self.W, self.ar, self.ex
        sync = torch.cuda.synchronize
        nanx, nandst = ar.ptr("nanx"), ar.ptr("nandst")
        both_parts = None
        for i, (p, c) in enumerate(self.steps):
            n = self.n + 1
            # -------- reduce_out of every rank --------
            if p[0] != "prev":
                kind, name, t, ms, kf, shards = self.prod[i]
                parts = []
                for r, (tens, k0, ks) in enumerate(shards):
                    twin = None
                    if not tp_only:
                        outs = [torch.empty(1, m, device="cuda") for m in ms]
                        twin = self.plain(t, "multi" if kind == "multi" else "head", tens, ks, ar.ptr(f"x{i}_{r}"), outs, ("none", 0.0),
                                          f"{self.id} reduce {i} rank {r} producer twin")
                        sync()
                        parts.append(np.concatenate([o.cpu().numpy()[0] for o in outs]))
                    label = f"{self.id} reduce {i} (#{n}) reduce_out rank {r} ({kind}, K = {ks}, M_total = {sum(ms)})"
                    snap = ar.buf.clone() if check else None
                    self.tp(t, "multi" if kind == "multi" else "head", tens, ks, ar.ptr(f"x{i}_{r}"), [nandst] * len(ms), ("none", 0.0), r, False, True,
                            twin, label)
                    if check:
                        sync()
                        expect(ar, snap, ex.out_edits(r, n, parts[r]), label)
                        if oracle:
                            o = 0
                            for j, (sh, w) in enumerate(tens):
                                yq = self.oracle.mul_mat_q8_1(t, sh, xs[i][:, k0:k0 + ks], w.m, variant="b200")
                                self.ratios[f"reduce_out {kind}"] = max(self.ratios.get(f"reduce_out {kind}", 0.0),
                                                                         bar_ratio(parts[r][o:o + w.m][None], yq, PLAIN_BAR, f"{label} tensor {j}"))
                                o += w.m
            else:
                parts = both_parts
            # -------- the consumers --------
            kind, name, t, ms, k, glu, ws = self.cons[i]
            h = rank_order_sum([q[:k] for q in parts]) if not tp_only else None
            ys, twin = None, [None] * W
            if not tp_only:
                hx = torch.from_numpy(h[None].copy()).cuda()
                if kind == "both":
                    both_parts, twin = [], []
                    for r in range(W):
                        o = torch.empty(1, ms[0], device="cuda")
                        twin.append(self.plain(t, "head", ws[r], k, hx.data_ptr(), [o], glu, f"{self.id} reduce {i} rank {r} consumer twin"))
                        sync()
                        both_parts.append(o.cpu().numpy()[0])
                else:
                    outs = [torch.empty(1, m, device="cuda") for m in ms]
                    twin = [self.plain(t, kind, ws, k, hx.data_ptr(), outs, glu, f"{self.id} reduce {i} consumer twin")] * W
                    sync()
                    ys = [o.cpu().numpy()[0] for o in outs]
            for r in range(W):
                label = f"{self.id} reduce {i} (#{n}) reduce_in rank {r} ({kind}, K = {k})"
                if check:
                    sync()
                    ex.precondition(r, n, k)
                    snap = ar.buf.clone()
                if kind == "both":
                    self.tp(t, "head", ws[r], k, nanx, [nandst], glu, r, True, True, twin[r], label)
                else:
                    self.tp(t, kind, ws, k, nanx, [ar.ptr(f"y{i}_{r}_{j}") for j in range(len(ms))], glu, r, True, False, twin[r], label)
                if check:
                    sync()
                    ed = ex.in_edits(r, n, h)
                    if kind == "both":
                        ed += ex.out_edits(r, n + 1, both_parts[r])
                    else:
                        ed += [(ar.regions[f"y{i}_{r}_{j}"][0], ys[j].view(np.uint8)) for j in range(len(ms))]
                    expect(ar, snap, ed, label)
            if oracle:
                what = f"{self.id} reduce {i} consumer ({kind})"
                if kind == "upgate":
                    u = self.oracle.mul_mat_q8_1(t, ws[0][0], h[None], ms[0], variant="b200").astype(np.float64)
                    g = self.oracle.mul_mat_q8_1(t, ws[1][0], h[None], ms[0], variant="b200").astype(np.float64)
                    key = f"reduce_in upgate {glu[0]}{' limit ' + str(glu[1]) if glu[1] else ''}"
                    self.ratios[key] = max(self.ratios.get(key, 0.0), glu_ratio(ys[0][None], g, u, glu[0], glu[1], what))
                elif kind == "both":
                    for r in range(W):
                        yq = self.oracle.mul_mat_q8_1(t, ws[r][0][0], h[None], ms[0], variant="b200")
                        self.ratios["reduce_in+out"] = max(self.ratios.get("reduce_in+out", 0.0), bar_ratio(both_parts[r][None], yq, PLAIN_BAR, f"{what} rank {r}"))
                else:
                    for j, (w, qt) in enumerate(ws):
                        yq = self.oracle.mul_mat_q8_1(t, w, h[None], qt.m, variant="b200")
                        self.ratios[f"reduce_in {kind}"] = max(self.ratios.get(f"reduce_in {kind}", 0.0), bar_ratio(ys[j][None], yq, PLAIN_BAR, f"{what} tensor {j}"))
            self.n = n                                  # ("both": the next reduce, n + 1, is this launch's; its step has no producers)
        return None if tp_only else self.outputs()

    def outputs(self):
        torch.cuda.synchronize()
        return {name: self.ar.get(name, "u8", (self.ar.nbytes(name),)) for name in self.ar.order if name.startswith("y")}


def set_option(key, value):
    assert lib().b200q_set_option(key.encode(), int(value)) == 0


def run_case(be, oracle, case):
    """Eager with PDL on (profiled, oracle bars), eager with PDL off (bit-identical), then a CUDA graph of the TP launches replayed three times with
    new inputs, each replay equal to the plain-launch chain on its inputs.  Returns the record the parent asserts on."""
    ch = Chain(be, oracle, case)
    xs = ch.new_inputs()
    set_option("pdl", 1)
    outs_a, kernels = profiled(lambda: ch.run(xs, oracle=True))
    log_a = list(ch.log)
    set_option("pdl", 0)
    try:
        outs_b = ch.run(xs)
    finally:
        set_option("pdl", 1)
    for name in outs_a:
        assert np.array_equal(outs_a[name], outs_b[name]), f"{ch.id}: {name} differs between PDL on and off"
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    n0 = ch.n
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            ch.run(None, check=False, tp_only=True)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    ch.n = n0                                           # (captured, not run)
    for it in range(3):
        xs = ch.new_inputs()
        torch.cuda.synchronize()
        g.replay()
        got = ch.outputs()
        ch.n += len(ch.steps)
        state = [ch.ar.get(f"state{q}", "i32", (4,)).view(np.uint32)[:2].tolist() for q in range(ch.W)]
        assert all(sq == [ch.n, 0] for sq in state), f"{ch.id} replay {it}: ll_state {state}, expected [{ch.n}, 0] on every rank"
        ref = plain_chain(ch, xs)
        for name in ref:
            assert np.array_equal(got[name], ref[name]), f"{ch.id} replay {it}: {name} differs from the plain-launch chain on the same inputs"
    return {"log": log_a, "launches": matmul_launches(kernels), "any_kernel": bool(kernels), "ratios": ch.ratios,
            "sms": torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count}


def plain_chain(ch, xs):
    """The outputs of every consumer region of the chain computed with plain launches only (h rebuilt on the host)"""
    out, both_parts = {}, None
    for i, (p, c) in enumerate(ch.steps):
        if p[0] != "prev":
            kind, name, t, ms, kf, shards = ch.prod[i]
            parts = []
            for r, (tens, k0, ks) in enumerate(shards):
                outs = [torch.empty(1, m, device="cuda") for m in ms]
                ch.plain(t, "multi" if kind == "multi" else "head", tens, ks, ch.ar.ptr(f"x{i}_{r}"), outs, ("none", 0.0), "plain chain")
                torch.cuda.synchronize()
                parts.append(np.concatenate([o.cpu().numpy()[0] for o in outs]))
        else:
            parts = both_parts
        kind, name, t, ms, k, glu, ws = ch.cons[i]
        hx = torch.from_numpy(rank_order_sum([q[:k] for q in parts])[None].copy()).cuda()
        if kind == "both":
            both_parts = []
            for r in range(ch.W):
                o = torch.empty(1, ms[0], device="cuda")
                ch.plain(t, "head", ws[r], k, hx.data_ptr(), [o], glu, "plain chain")
                torch.cuda.synchronize()
                both_parts.append(o.cpu().numpy()[0])
            continue
        outs = [torch.empty(1, m, device="cuda") for m in ms]
        ch.plain(t, kind, ws, k, hx.data_ptr(), outs, glu, "plain chain")
        torch.cuda.synchronize()
        for r in range(ch.W):
            for j, o in enumerate(outs):
                out[f"y{i}_{r}_{j}"] = o.cpu().numpy()[0].view(np.uint8)
    return out


def check_trace(case_id, got, want_all_six):
    """Every TP launch is k_mmvq_ring<T, 1, UPGATE, MULTI, PAIR, true, 0> with the flags of its role and the grid and block of its plain twin
    (TP = false); returns the set of instantiations seen"""
    if not got["any_kernel"]:
        pytest.skip(f"{case_id}: the profiler recorded no kernel events (CUPTI unavailable?); numerical checks passed, configuration not checked")
    log, launched = got["log"], got["launches"]
    assert len(launched) == len(log), f"{case_id}: {len(launched)} mat-vec kernels in the trace, {len(log)} launches issued"
    B = {True: "true", False: "false"}
    seen = set()
    for (kind, flags, twin, label), (kern, args, grid, block) in zip(log, launched):
        if kind != "tp":
            continue
        tw = launched[twin]
        assert kern == "k_mmvq_ring" and tw[0] == "k_mmvq_ring", f"{label}: {kern}, twin {tw[0]}: both must be the ring kernel"
        want = (tw[1][0], "1", B[flags[0]], B[flags[1]], B[flags[2]], "true", "0")
        assert tuple(args) == want, f"{label}: launched k_mmvq_ring<{', '.join(args)}>, expected <{', '.join(want)}>"
        assert tuple(tw[1][:5]) == want[:5] and tuple(tw[1][5:]) == ("false", "0"), f"{label}: twin k_mmvq_ring<{', '.join(tw[1])}>"
        assert tuple(grid) == tuple(tw[2]) and tuple(block) == tuple(tw[3]), f"{label}: grid {grid} block {block}, the plain twin {tw[2]} {tw[3]}"
        seen.add(tuple(flags))
    if want_all_six:
        missing = {(u, m, p) for u, m in ((False, False), (False, True), (True, False)) for p in (True, False)} - seen
        assert not missing, f"{case_id}: TP instantiations (UPGATE, MULTI, PAIR) not exercised: {sorted(missing)}"
    return seen


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_tp_decode_chain(be, tmp_path, case):
    _, got = run_child(case[0], tmp_path, script=__file__, env=case[3])
    for key, r in sorted(got["ratios"].items()):
        print(f"{case[0]}: {key}: max ratio to the bar = {r:.3g} (TP launches bit-identical to their plain twins)")
    seen = check_trace(case[0], got, case[0].startswith("sweep-"))
    row = " ".join(f"{'UG' if u else 'MU' if m else 'PL'}-{'pair' if p else 'long'}" for u, m, p in sorted(seen))
    print(f"coverage {case[0]}: {len(seen)} TP instantiations: {row}")


# ------------------------------------------------------------------------------------------------------------------------------------------------
# GPU: rejections and the acceptance rule
# ------------------------------------------------------------------------------------------------------------------------------------------------
def run_rejections(be, oracle):
    """In a process with the unicast stores selected.  Every probe is made on a copy of rank 0 whose whole slot array carries tag 1 and whose count
    is 1, so that even a consumer accepted by mistake could not wait: it would find every entry it reads present."""
    L = lib()
    W, S = 2, 4096
    ar = Arena(S)
    Exchange.add(ar, W, S)
    ar.add("x", 3 * S * 4, "in")
    ar.add("dst", 3 * S * 4, "out")
    ar.build()
    ex = Exchange(ar, W, S)
    ex.zero()
    for q in range(W):
        ar.put(f"slots{q}", entries(np.zeros(2 * W * S, np.float32), 1))
        ar.put(f"state{q}", np.array([1, 0, 0, 0], np.uint32))
    ar.put("x", np.random.default_rng(1).standard_normal(3 * S).astype(np.float32))
    from ik_llama_cpp_b200.backend import NvlsComm
    peers = ptrs([ar.ptr(f"slots{q}") for q in range(W)])
    pp = ctypes.cast(peers, ctypes.POINTER(c_void_p))

    def comm(**kw):
        c = dict(ll_mc=None, ll_local=ar.ptr("slots0"), ll_reduced=ar.ptr("red0"), ll_stride=S, world_size=W, rank=0, ll_state=ar.ptr("state0"), ll_peers=pp)
        c.update(kw)
        return NvlsComm(c["ll_mc"], c["ll_local"], c["ll_reduced"], c["ll_stride"], c["world_size"], c["rank"], c["ll_state"], c["ll_peers"])

    def probe(t, ws, k, rin, rout, cm, gate=None, what=""):
        snap = ar.buf.clone()
        n_t = len(ws)
        rc = L.b200q_mul_mat_vec_tp(t, n_t, ptrs([w.ptr for w in ws]), gate.ptr if gate is not None else None, ptrs([ar.ptr("dst")] * n_t),
                                    ptrs([w.m for w in ws], c_int64), k, ar.ptr("x"), 1, 0.0, ctypes.byref(cm), rin, rout, st())
        torch.cuda.synchronize()
        if rc:
            expect(ar, snap, [], f"{what}: rejected with {rc}")
        return rc

    results = []
    mk = lambda name, m, k, s=0: be.set_tensor(GGML_TYPE[name], make_wire(oracle, name, m, k, seed=[500, s, m, k]), m, k)
    # wire-layout types
    for name in WIRE_TYPES:
        w = mk(name, 256, 2048)
        for rin, rout in ((0, 1), (1, 0)):
            rc = probe(GGML_TYPE[name], [w], 2048, rin, rout, comm(), what=f"{name} in={rin} out={rout}")
            assert rc == E_TYPE, f"{name} (wire layout) reduce_in={rin} reduce_out={rout}: rc {rc}, expected B200Q_E_TYPE: {L.b200q_last_error().decode()}"
    results.append(f"{len(WIRE_TYPES)} wire types: B200Q_E_TYPE")
    # shapes
    w = mk("IQ4_NL", 256, 2080)
    for rin, rout in ((0, 1), (1, 0)):
        assert probe(GGML_TYPE["IQ4_NL"], [w], 2080, rin, rout, comm(), what="K % 256") == E_SHAPE, "K = 2080 (K % 256 != 0)"
    w = mk("IQ4_NL", S + 2, 2048)
    assert probe(GGML_TYPE["IQ4_NL"], [w], 2048, 0, 1, comm(), what="M_total > ll_stride") == E_SHAPE, "M_total = ll_stride + 2"
    w3 = [mk("IQ4_NL", m, 2048, 1) for m in (S - 256, 256, 2)]
    assert probe(GGML_TYPE["IQ4_NL"], w3, 2048, 0, 1, comm(), what="multi M_total > ll_stride") == E_SHAPE, "three tensors, M_total = ll_stride + 2"
    w = mk("IQ4_NL", 256, S + 256)
    assert probe(GGML_TYPE["IQ4_NL"], [w], S + 256, 1, 0, comm(), what="K > ll_stride") == E_SHAPE, "reduce_in with K = ll_stride + 256"
    w = mk("Q6_K", 256, 3072)
    assert probe(GGML_TYPE["Q6_K"], [w], 3072, 0, 1, comm(), what="Q6_K K = 3072") == E_SHAPE, "Q6_K K = 3072 has no ring geometry"
    w3 = [mk("IQ4_NL", m, 2048, 2) for m in (255, 128, 128)]
    assert probe(GGML_TYPE["IQ4_NL"], w3, 2048, 1, 0, comm(), what="odd non-last segment") == E_SHAPE, "row pairs: an odd tensor that is not the last"
    results.append("K % 256, M_total > ll_stride, K > ll_stride, no ring geometry, odd non-last row-pair segment: B200Q_E_SHAPE")
    # arguments
    up, gate = mk("IQ4_NL", 256, 2048, 3), mk("IQ4_NL", 256, 2048, 4)
    assert probe(GGML_TYPE["IQ4_NL"], [up], 2048, 0, 1, comm(), gate=gate, what="gate + reduce_out") == E_ARG, "reduce_out with a gate"
    assert probe(GGML_TYPE["IQ4_NL"], [up], 2048, 1, 1, comm(), gate=gate, what="gate + reduce_in + reduce_out") == E_ARG, "reduce_in + reduce_out with a gate"
    bad = {"world_size 1": comm(world_size=1), "rank == world_size": comm(rank=2), "ll_local NULL": comm(ll_local=None),
           "ll_reduced NULL": comm(ll_reduced=None), "ll_state NULL": comm(ll_state=None), "ll_stride odd": comm(ll_stride=S - 1),
           "ll_reduced misaligned": comm(ll_reduced=ar.ptr("red0") + 8), "ll_stride 0": comm(ll_stride=0)}
    for what, cm in bad.items():
        for rin, rout in ((0, 1), (1, 0)):
            assert probe(GGML_TYPE["IQ4_NL"], [up], 2048, rin, rout, cm, what=what) == E_ARG, f"incomplete communicator ({what})"
    results.append("a gate with reduce_out, " + ", ".join(bad) + ": B200Q_E_ARG")
    # the acceptance rule: reduce_out probes (nothing consumes them: they only store), a plain n = 1 launch of the same tensor before each
    log, probes = [], []
    ks = (1024, 2048, 2080, 3072, 4096, 5120, 6144, 7168)
    from ik_llama_cpp_b200.tp import GEOM
    tens = {(name, k): mk(name, 256, k, 5) for name in PLANE_TYPES for k in ks if k % GEOM[GGML_TYPE[name]][0] == 0}

    def sweep():
        for (name, k), w in tens.items():
            t = GGML_TYPE[name]
            y = torch.empty(1, 256, device="cuda")
            xt = torch.randn(1, k, device="cuda")
            assert L.b200q_mul_mat_vec(t, w.ptr, xt.data_ptr(), y.data_ptr(), 256, k, 1, k, None, st()) == 0
            log.append(("plain", name, k))
            rc = probe(t, [w], k, 0, 1, comm(), what=f"{name} K = {k}")
            if rc == 0:
                log.append(("tp", name, k))
            else:
                assert rc == E_SHAPE, f"{name} K = {k}: rejected with {rc}, expected B200Q_E_SHAPE: {L.b200q_last_error().decode()}"
            probes.append((name, k, rc))
    _, kernels = profiled(sweep)
    launched = matmul_launches(kernels)
    return {"results": results, "log": log, "probes": probes, "launches": launched, "any_kernel": bool(kernels)}


def check_acceptance(got):
    if not got["any_kernel"]:
        pytest.skip("the profiler recorded no kernel events (CUPTI unavailable?); rejections checked, the acceptance rule not")
    log, launched = got["log"], got["launches"]
    assert len(log) == len(launched), f"{len(launched)} mat-vec kernels in the trace, {len(log)} launches"
    plain_ring, tp_kernel = {}, {}
    for (kind, name, k), lk in zip(log, launched):
        if kind == "plain":
            plain_ring[(name, k)] = lk
        else:
            tp_kernel[(name, k)] = lk
    accepted = []
    for name, k, rc in got["probes"]:
        pl = plain_ring[(name, k)]
        want = pl[0] == "k_mmvq_ring" and k % 256 == 0
        assert (rc == 0) == want, f"{name} K = {k}: plain n = 1 launch is {pl[0]}, the TP launch returned {rc}: accepted exactly when ring and K % 256 == 0"
        if rc == 0:
            tk = tp_kernel[(name, k)]
            assert tk[0] == "k_mmvq_ring" and tk[1][5] == "true" and tuple(tk[1][:5]) == tuple(pl[1][:5]) and tuple(tk[2]) == tuple(pl[2]), \
                f"{name} K = {k}: TP launch {tk} is not the plain launch {pl} with TP = true"
            accepted.append(f"{name}@{k}")
    return accepted


@pytest.mark.gpu
def test_tp_rejections_and_acceptance(be, tmp_path):
    """Wire types return B200Q_E_TYPE, K % 256 != 0, M_total > ll_stride, K > ll_stride, no ring geometry and an odd non-last row-pair tensor
    B200Q_E_SHAPE, a gate with reduce_out and every kind of incomplete communicator B200Q_E_ARG, each without changing a byte of the arena.
    Every plane type at K = 1024 .. 7168: the TP launch is accepted exactly when the plain n = 1 launch is the ring kernel and K % 256 == 0, and
    then it is that kernel with TP = true, the same grid and block."""
    _, got = run_child("rejections", tmp_path, script=__file__, env={"B200Q_TP_UNICAST": "1", "B200Q_TP_ROWBUF": "0"})
    for line in got["results"]:
        print(line)
    acc = check_acceptance(got)
    print(f"accepted (type@K): {' '.join(acc)}; rejected: {' '.join(f'{n}@{k}' for n, k, rc in got['probes'] if rc)}")


@pytest.mark.gpu
def test_tp_multicast_address_required_without_unicast(be, tmp_path):
    """Without the unicast stores selected, ll_mc = NULL is an incomplete communicator (B200Q_E_ARG) and nothing is written: no launch can issue
    multimem.st to an address that is not a multicast mapping."""
    _, got = run_child("no-unicast", tmp_path, script=__file__, env={"B200Q_TP_UNICAST": "0"})
    assert got["rcs"] == [E_ARG, E_ARG], got


def run_no_unicast(be, oracle):
    L = lib()
    W, S = 2, 4096
    ar = Arena(S)
    Exchange.add(ar, W, S)
    ar.add("x", S * 4, "in")
    ar.add("dst", S * 4, "out")
    ar.build()
    Exchange(ar, W, S).zero()
    from ik_llama_cpp_b200.backend import NvlsComm
    peers = ptrs([ar.ptr(f"slots{q}") for q in range(W)])
    cm = NvlsComm(None, ar.ptr("slots0"), ar.ptr("red0"), S, W, 0, ar.ptr("state0"), ctypes.cast(peers, ctypes.POINTER(c_void_p)))
    w = be.set_tensor(GGML_TYPE["IQ4_NL"], make_wire(oracle, "IQ4_NL", 256, 2048, seed=9), 256, 2048)
    rcs = []
    for rin, rout in ((0, 1), (1, 0)):
        snap = ar.buf.clone()
        rcs.append(L.b200q_mul_mat_vec_tp(w.ggml_type, 1, ptrs([w.ptr]), None, ptrs([ar.ptr("dst")]), ptrs([256], c_int64), 2048, ar.ptr("x"), 1, 0.0,
                                          ctypes.byref(cm), rin, rout, st()))
        torch.cuda.synchronize()
        expect(ar, snap, [], "ll_mc = NULL without unicast")
    return {"rcs": rcs}


if __name__ == "__main__":
    from ik_llama_cpp_b200 import backend as _be
    from oracle.oracle import Oracle
    _case, _out = sys.argv[1], sys.argv[2]
    if _case == "rejections":
        _rec = run_rejections(_be, Oracle())
    elif _case == "no-unicast":
        _rec = run_no_unicast(_be, Oracle())
    else:
        _rec = run_case(_be, Oracle(), next(c for c in CASES if c[0] == _case))
    np.savez(os.path.join(_out, "y.npz"))
    with open(os.path.join(_out, "launches.json"), "w") as _f:
        json.dump(_rec, _f)
