"""The backend plug (libggml_b200.so) on graphs built as the reference builds them, driven by ggml_backend_sched.

tests/backend_ops/test_plug_graphs runs each case: a Llama layer in the default quantisation mix (n = 1 .. 512, and one n = 1 layer at the
Llama-3-8B sizes), Qwen2-style Q, K, V biases, the MoE FFN of llm_build_moe_ffn (softmax, ggml_top_k, ggml_moe_up_gate, ggml_mul_mat_id) at three
model shapes and token counts on both sides of the mat-vec / grouped-GEMM threshold, batched MUL_MAT, and a row-slice view of a weight.  The scheduler
decides where each node runs; the harness dumps every node's output and every tensor it read (after the scheduler's copies: what the node really
saw), and this file checks the dump.

Placement.  Every MUL_MAT / FUSED_UP_GATE / MUL_MAT_ID / MOE_FUSED_UP_GATE node whose weight is a whole tensor of the plug's buffer must run on the plug,
the MoE nodes at every token count included (their expert ids are a strided view of the argsort result whenever there is more than one token).  The
only product the plug must decline is the one with a view of its weight; that node runs on the CPU backend, which fetches the view through get_tensor.

Values, each node against the inputs it read, with the bars of the kernel suites (imported, not restated):
  * mat-vec products (n <= 8): oracle.mul_mat_q8_1(..., variant="b200") at PLAIN_BAR, GLU_BAR for up/gate (test_gpu_decode_schedules.py);
  * GEMM products (n > 8): the same-operand bf16 reference at tau(K) A, glu_bound for up/gate (test_gpu_gemm_schedules.py);
  * MoE nodes: per slot against the expert the dumped top-k ids chose, with the mat-vec or GEMM bar as the dispatcher picks
    (test_moe_dispatch.last_mat_vec_batch); skipped slots must be 0; the ids must be the top n_used of the dumped softmax;
  * an ADD the plug computes in the preceding mat-vec's epilogue (a bias, or the residual of one token): |y - ref| <= PLAIN_BAR rms(yq) + F32_ADD |ref|
    with ref = yq + b; the product node it follows must still hold the plain product.  A stand-alone ADD must equal the f32 sum bit for bit;
  * the weight-view node: the bytes the CPU backend read must be the wire rows [r0, r1) of the weight, and its result within NMSE 5e-4 of
    oracle.mul_mat_exact on those rows (loose on purpose: the CPU backend quantises its activations).
test_partial_weight_upload_in_whole_rows checks set_tensor on whole rows of a weight (through a view, and at an offset) by reading the tensor back.
test_checker_catches_planted_defects runs the checker without a GPU on a small dump made with the oracle.
"""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import make_wire
from oracle.oracle import GGML_TYPE, nmse
from test_gpu_decode_schedules import F32_ADD, GLU_BAR, PLAIN_BAR, bar_ratio
from test_gpu_gemm_schedules import bf16, element_ratio, glu_bound, same_operand_reference, silu
from test_gpu_parity import glu_ref, rms
from test_moe_dispatch import last_mat_vec_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "backend_ops", "test_plug_graphs")
MAT_OPS = ("MUL_MAT", "FUSED_UP_GATE", "MUL_MAT_ID", "MOE_FUSED_UP_GATE")
PLUG_BUFFER = "B200"            # ggml_backend_buffer_name of the plug's buffers
UNARY_SILU = 10                 # GGML_UNARY_OP_SILU
VIEW_NMSE = 5e-4
MOE_TOKENS = [1, 2, 8, 24, 160, 512]
CASES = {"llama": [1, 2, 8, 9, 64, 512], "llama-8b": [1], "qwen2-bias": [1, 64], "moe-qwen3": MOE_TOKENS, "moe-mixtral": MOE_TOKENS,
         "moe-deepseek": MOE_TOKENS, "batched": [3, 64], "weight-view": [4]}
DTYPE = {"f32": np.float32, "i32": np.int32}


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the dump
# ------------------------------------------------------------------------------------------------------------------------------------------------
class Dump:
    """One graph of a case: <case_dir>/<tag>/manifest.jsonl and the tensors it names; weights are <case_dir>/w_<name>.npy."""

    def __init__(self, case_dir, tag):
        self.case_dir, self.dir, self.tag = case_dir, os.path.join(case_dir, tag), tag
        with open(os.path.join(self.dir, "manifest.jsonl")) as f:
            lines = [json.loads(s) for s in f if s.strip()]
        self.case = lines[0]
        self.nodes = lines[1:]
        self._cache = {}

    def raw(self, t):
        path = os.path.join(self.case_dir, f"w_{t['weight']}.npy") if "weight" in t else os.path.join(self.dir, t["file"])
        if path not in self._cache:
            self._cache[path] = np.load(path)
        return self._cache[path]

    def value(self, t):
        """f32 / i32 tensors as arrays [ne3][ne2][ne1][ne0] read through their strides; quantised tensors as their bytes"""
        raw = self.raw(t)
        if t["type"] not in DTYPE:
            return raw
        dt = np.dtype(DTYPE[t["type"]])
        return np.ndarray(tuple(t["ne"][::-1]), dt, buffer=raw, strides=tuple(t["nb"][::-1])).copy()


def write_dump(case_dir, tag, case, weights, nodes):
    """The harness's format, for dumps made on the host: weights {name: wire bytes}; nodes [{name, op, backend, supported, op_params, value, src}],
    each src None, ("node", index), ("weight", name, type, ne) or ("tensor", array) / ("tensor", raw bytes, type, ne, nb).  An array passed more
    than once is one tensor read by several nodes (one file), as the harness dumps a tensor once."""
    d = os.path.join(case_dir, tag)
    os.makedirs(d, exist_ok=True)
    for name, wire in weights.items():
        np.save(os.path.join(case_dir, f"w_{name}.npy"), np.asarray(wire, np.uint8))
    files = [0]
    seen = {}

    def tensor(name, a, typ=None, ne=None, nb=None):
        if id(a) in seen:
            return dict(seen[id(a)][1])
        key = a
        if typ is None:
            typ = {np.dtype(np.float32): "f32", np.dtype(np.int32): "i32"}[a.dtype]
            ne = list(a.shape[::-1]) + [1] * (4 - a.ndim)
            nb = [a.itemsize]
            for i in range(3):
                nb.append(nb[-1] * ne[i])
            a = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        f = f"t{files[0]}.npy"
        files[0] += 1
        np.save(os.path.join(d, f), a)
        entry = {"name": name, "type": typ, "ne": ne, "nb": nb, "buffer": PLUG_BUFFER, "file": f, "node": -1}
        seen[id(key)] = (key, entry)
        return dict(entry)

    out = []
    for i, nd in enumerate(nodes):
        line = {"kind": "node", "i": i, "op": nd["op"], **tensor(nd["name"], np.array(nd["value"], np.float32)), "backend": nd.get("backend", case["backend"]),
                "supported": nd.get("supported", True), "op_params": nd.get("op_params", [0, 0, 0, 0]), "src": []}
        for s in nd["src"]:
            if s is None:
                line["src"].append(None)
            elif s[0] == "node":
                line["src"].append({k: out[s[1]][k] for k in ("name", "type", "ne", "nb", "buffer", "file")} | {"node": s[1]})
            elif s[0] == "weight":
                line["src"].append({"name": s[1], "type": s[2], "ne": s[3], "nb": [0, 0, 0, 0], "buffer": PLUG_BUFFER, "weight": s[1], "node": -1})
            else:
                line["src"].append(tensor(f"{nd['name']}.src", *s[1:]))
        out.append(line)
    with open(os.path.join(d, "manifest.jsonl"), "w") as f:
        for line in [dict(kind="case", tag=tag, **case)] + out:
            f.write(json.dumps(line) + "\n")
    return Dump(case_dir, tag)


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the checker
# ------------------------------------------------------------------------------------------------------------------------------------------------
def _gtype(t):
    return GGML_TYPE[t["type"].upper()]


def _same(a, b):
    """the same tensor: the same graph node or the same dumped file"""
    return a is not None and b is not None and (a["node"] >= 0 and a["node"] == b["node"] or a.get("file") is not None and a.get("file") == b.get("file"))


def _on_plug(d, nd):
    return nd["backend"] == d.case["backend"]


def fusion_plan(d):
    """{index of ADD node: "fused" | "maybe"} for the ADDs graph_compute takes into the mat-vec epilogue of the MUL_MAT right before them (a 2-D
    product of n <= 8 columns, the ADD's second operand an [M] vector in the plug's buffers).  The look-ahead is mirrored in graph_compute's order:
    a MUL_MAT that consumes the q8_1 image of the FUSED_UP_GATE right before it does not look at the ADD ("maybe": that hand-off is skipped for
    shapes the kernel does not take, and then the ADD is fused), and the MUL_MATs a Q, K, V launch absorbs do not either."""
    plan, nodes, absorbed = {}, d.nodes, set()
    for i, nd in enumerate(nodes):
        if nd["op"] != "MUL_MAT" or not _on_plug(d, nd) or i in absorbed or "weight" not in nd["src"][0]:
            continue
        w, x = nd["src"][0], nd["src"][1]
        n = x["ne"][1]
        if x["ne"][2] * x["ne"][3] != 1:
            continue
        prev = nodes[i - 1] if i > 0 else None
        handoff = (n == 1 and prev is not None and prev["op"] == "FUSED_UP_GATE" and _on_plug(d, prev) and x["node"] == i - 1
                   and prev["src"][0]["ne"][1] % 64 == 0)
        nx = nodes[i + 1] if i + 1 < len(nodes) else None
        if (n <= 8 and nx is not None and nx["op"] == "ADD" and _on_plug(d, nx) and nx["src"][0]["node"] == i and nx["src"][1]["buffer"] == PLUG_BUFFER
                and int(np.prod(nx["src"][1]["ne"])) == w["ne"][1]):
            plan[i + 1] = "maybe" if handoff else "fused"
            continue
        if handoff:
            continue
        j = i + 1                           # Q, K, V: following MUL_MATs on the same input and weight type join this launch
        while j < len(nodes) and j - i < 3:
            nj = nodes[j]
            if not (nj["op"] == "MUL_MAT" and _on_plug(d, nj) and _same(nj["src"][1], x) and "weight" in nj["src"][0] and nj["src"][0]["type"] == w["type"]
                    and nj["src"][0]["ne"][2] == 1 and not (n <= 8 and nj["src"][0]["ne"][1] % 2)):
                break
            absorbed.add(j)
            j += 1
    return plan


def check_placement(d):
    views = {v["node"] for v in d.case.get("views", [])}
    for nd in d.nodes:
        if nd["op"] not in MAT_OPS:
            continue
        what = f"{d.tag} {nd['name']} ({nd['op']})"
        if nd["name"] in views:
            assert not nd["supported"], f"{what}: the plug must decline a product with a view of its weight"
            continue
        w = nd["src"][0]
        assert "weight" in w, f"{what}: expected a whole weight as src0, got {w['name']}"
        assert nd["supported"] and _on_plug(d, nd), (f"{what}: its weight {w.get('copy_of', w['name'])} is a whole plug tensor, but the node was assigned "
                                                     f"to {nd['backend'] or 'no backend'} (supports_op: {nd['supported']})")
        assert w["buffer"] == PLUG_BUFFER, f"{what}: its weight was read from a {w['buffer']} buffer"


def product_check(oracle, t, wire, x, y, m, mat_vec, what):
    """y [n, m] = W x [n, k] on the plug, with the bar of the path it takes (mat-vec: q8_1 oracle; GEMM: same-operand bf16 reference)"""
    n, k = x.shape
    if mat_vec:
        return bar_ratio(y, oracle.mul_mat_q8_1(t, wire, x, m, variant="b200"), PLAIN_BAR, what)
    ref, a = same_operand_reference(bf16(oracle.dequantize(t, wire, m, k)), bf16(x))
    return element_ratio(y, ref, a, k, what)


def glu_check(oracle, t, wu, wg, x, y, m, mat_vec, what):
    n, k = x.shape
    if mat_vec:
        u = oracle.mul_mat_q8_1(t, wu, x, m, variant="b200").astype(np.float64)
        g = oracle.mul_mat_q8_1(t, wg, x, m, variant="b200").astype(np.float64)
        return bar_ratio(y, glu_ref("silu", g, u), GLU_BAR, what)
    ru, au = same_operand_reference(bf16(oracle.dequantize(t, wu, m, k)), bf16(x))
    rg, ag = same_operand_reference(bf16(oracle.dequantize(t, wg, m, k)), bf16(x))
    return element_ratio(y, silu(rg) * ru, None, k, what, bound=glu_bound(k, rg, ru, ag, au))


def check_mul_mat(oracle, d, nd):
    w, xs = nd["src"][0], nd["src"][1]
    t, (k, m, e) = _gtype(w), w["ne"][:3]
    mats = d.value(w).reshape(e, -1)
    x, y = d.value(xs), d.value(nd)
    worst = 0.0
    for b3 in range(x.shape[0]):
        for b2 in range(x.shape[1]):
            what = f"{d.tag} {nd['name']} batch ({b3}, {b2})"
            worst = max(worst, product_check(oracle, t, mats[b2 if e > 1 else 0], x[b3, b2], y[b3, b2], m, x.shape[2] <= 8, what))
    return worst


def check_view(oracle, d, nd, view):
    src = nd["src"][0]                              # the CPU backend's copy of the view
    t, rs = _gtype(src), src["nb"][1]
    r0, r1 = view["r0"], view["r1"]
    rows = d.raw({"weight": view["weight"]})[r0 * rs:r1 * rs]
    assert np.array_equal(d.raw(src), rows), f"{d.tag} {nd['name']}: the bytes the CPU backend read are not the wire rows [{r0}, {r1}) of {view['weight']}"
    x, y = d.value(nd["src"][1])[0, 0], d.value(nd)[0, 0]
    e = nmse(y, oracle.mul_mat_exact(t, rows, x, r1 - r0))
    assert e <= VIEW_NMSE, f"{d.tag} {nd['name']}: NMSE {e:.3g} against the exact product on the wire rows [{r0}, {r1})"
    return e


def check_add(oracle, d, i, nd, plan):
    a, b, y = d.value(nd["src"][0]), d.value(nd["src"][1]), d.value(nd)
    f32_sum = (a + b).astype(np.float32)
    kind = plan.get(i)
    if kind == "maybe" and np.array_equal(y, f32_sum):
        return 0.0
    if kind is None:
        assert np.array_equal(y, f32_sum), f"{d.tag} {nd['name']}: a stand-alone ADD must equal the f32 sum of its operands bit for bit"
        return 0.0
    mm = d.nodes[nd["src"][0]["node"]]             # the product whose epilogue added b: checked against its own reference
    w, x = mm["src"][0], d.value(mm["src"][1])[0, 0]
    yq = oracle.mul_mat_q8_1(_gtype(w), d.value(w), x, w["ne"][1], variant="b200").astype(np.float64)
    ref = yq + b.reshape(1, -1).astype(np.float64)
    bound = PLAIN_BAR * rms(yq) + F32_ADD * np.abs(ref)
    err = np.abs(y[0, 0] - ref)
    bad = np.argwhere(~(err <= bound))
    assert len(bad) == 0, (f"{d.tag} {nd['name']}: {len(bad)} of {err.size} elements of the fused ADD outside PLAIN_BAR rms + F32_ADD |ref|, first "
                           + ", ".join(f"{tuple(int(v) for v in q)}: y={y[0, 0][tuple(q)]:.7g} ref={ref[tuple(q)]:.7g}" for q in bad[:5]))
    return float((err / bound).max())


def check_routing(d, ids):
    """the ids are the top n_used experts of the dumped softmax, per token"""
    probs = next((d.value(nd)[0, 0] for nd in d.nodes if nd["op"] == "SOFT_MAX"), None)
    if probs is None:
        return
    for tk in range(ids.shape[0]):
        sel = np.zeros(probs.shape[1], bool)
        sel[ids[tk]] = True
        assert sel.sum() == ids.shape[1] and probs[tk, sel].min() >= probs[tk, ~sel].max(), f"{d.tag}: ids of token {tk} are not its top-k experts"


def check_moe(oracle, d, nd):
    ug = nd["op"] == "MOE_FUSED_UP_GATE"
    w, g, xs, idt = nd["src"][0], nd["src"][1] if ug else None, nd["src"][2 if ug else 1], nd["src"][3 if ug else 2]
    if ug:
        assert nd["op_params"][0] == UNARY_SILU, f"{d.tag} {nd['name']}: unary {nd['op_params'][0]}"
    t, (k, m, n_expert) = _gtype(w), w["ne"][:3]
    x, ids, y = d.value(xs)[0], d.value(idt)[0, 0], d.value(nd)[0]
    n_tokens, nb1 = x.shape[0], x.shape[1]
    n_used = ids.shape[1]
    check_routing(d, ids)
    W = d.value(w).reshape(n_expert, -1)
    G = d.value(g).reshape(n_expert, -1) if ug else None
    invalid = (ids < 0) | (ids >= n_expert)
    assert np.all(y[invalid] == 0.0), f"{d.tag} {nd['name']}: skipped slots must give zero rows"
    mat_vec = n_tokens <= last_mat_vec_batch(n_expert, n_used, ug)
    worst = 0.0
    for e in np.unique(ids[~invalid]):
        tk, u = np.nonzero(ids == e)
        cols = np.ascontiguousarray(x[tk, u % nb1])
        what = f"{d.tag} {nd['name']} expert {e}"
        if mat_vec:
            ref = oracle.mul_mat_q8_1(t, W[e], cols, m, variant="b200").astype(np.float64)
            if ug:
                ref = glu_ref("silu", oracle.mul_mat_q8_1(t, G[e], cols, m, variant="b200").astype(np.float64), ref)
            for j in range(len(tk)):
                worst = max(worst, bar_ratio(y[tk[j], u[j]], ref[j], GLU_BAR if ug else PLAIN_BAR, f"{what}: token {tk[j]} slot {u[j]}"))
        elif ug:
            worst = max(worst, glu_check(oracle, t, W[e], G[e], cols, y[tk, u], m, False, what))
        else:
            worst = max(worst, product_check(oracle, t, W[e], cols, y[tk, u], m, False, what))
    return worst


def check_dump(oracle, d):
    """placement, then every node's value; returns {node name: largest error / bound}"""
    check_placement(d)
    plan = fusion_plan(d)
    views = {v["node"]: v for v in d.case.get("views", [])}
    out = {}
    for i, nd in enumerate(d.nodes):
        op = nd["op"]
        if nd["name"] in views:
            out[nd["name"]] = check_view(oracle, d, nd, views[nd["name"]])
        elif op == "MUL_MAT":
            out[nd["name"]] = check_mul_mat(oracle, d, nd)
        elif op == "FUSED_UP_GATE":
            up, gate = nd["src"][0], nd["src"][1]
            assert nd["op_params"][0] == UNARY_SILU, f"{d.tag} {nd['name']}: unary {nd['op_params'][0]}"
            x = d.value(nd["src"][2])[0, 0]
            out[nd["name"]] = glu_check(oracle, _gtype(up), d.value(up), d.value(gate), x, d.value(nd)[0, 0], up["ne"][1], x.shape[0] <= 8, f"{d.tag} {nd['name']}")
        elif op in ("MUL_MAT_ID", "MOE_FUSED_UP_GATE"):
            out[nd["name"]] = check_moe(oracle, d, nd)
        elif op == "ADD":
            out[nd["name"]] = check_add(oracle, d, i, nd, plan)
    return out


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-test of the checker (oracle and numpy only)
# ------------------------------------------------------------------------------------------------------------------------------------------------
def _fails(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def _planted_graph(oracle, rng):
    """A small graph as the harness would dump it, with the plug's results made from the oracle: Q (+ bias, fused), K and V joined, up/gate, ffn_down
    on its q8_1 image, a weight-view product on the CPU backend, and a MoE MUL_MAT_ID of 3 tokens whose ids are a strided top-k view."""
    t, k, m_q, m_kv, m_ff, n_expert, n_used, n_tok = GGML_TYPE["IQ4_NL"], 256, 64, 32, 64, 8, 2, 3
    wires = {"wq": make_wire(oracle, "IQ4_NL", m_q, k, 1), "wk": make_wire(oracle, "IQ4_NL", m_kv, k, 2), "wv": make_wire(oracle, "IQ4_NL", m_kv, k, 3),
             "up": make_wire(oracle, "IQ4_NL", m_ff, k, 4), "gate": make_wire(oracle, "IQ4_NL", m_ff, k, 5), "down": make_wire(oracle, "IQ4_NL", k, m_ff, 6),
             "wbig": make_wire(oracle, "IQ4_NL", 40, k, 7), "exps": np.concatenate([make_wire(oracle, "IQ4_NL", m_q, k, 10 + e) for e in range(n_expert)])}
    q8 = lambda name, x, m: oracle.mul_mat_q8_1(t, wires[name], x, m, variant="b200")
    x = rng.standard_normal((1, k)).astype(np.float32)
    bq = rng.standard_normal(m_q).astype(np.float32)
    yq = q8("wq", x, m_q)
    par = glu_ref("silu", q8("gate", x, m_ff), q8("up", x, m_ff)).astype(np.float32)
    r0, r1 = 8, 24
    rs = wires["wbig"].size // 40
    rows = wires["wbig"][r0 * rs:r1 * rs]
    xv = rng.standard_normal((4, k)).astype(np.float32)
    logits = rng.standard_normal((n_tok, n_expert)).astype(np.float32)
    probs = np.exp(logits) / np.exp(logits).sum(1, keepdims=True)
    order = np.argsort(-probs, axis=1).astype(np.int32)              # the argsort result; ids are its first n_used columns, row stride n_expert
    ids = order[:, :n_used]
    xm = rng.standard_normal((n_tok, 1, k)).astype(np.float32)
    ymoe = np.zeros((n_tok, n_used, m_q), np.float32)
    for tk in range(n_tok):
        for u in range(n_used):
            ymoe[tk, u] = oracle.mul_mat_q8_1(t, wires["exps"].reshape(n_expert, -1)[ids[tk, u]], xm[tk], m_q, variant="b200")[0]
    W = lambda name, m, e=1: ("weight", name, "iq4_nl", [k if name != "down" else m_ff, m, e, 1])
    ids_raw = order.reshape(-1).view(np.uint8)[:((n_tok - 1) * n_expert + n_used) * 4]
    nodes = [
        dict(name="Qcur", op="MUL_MAT", value=yq, src=[W("wq", m_q), ("tensor", x)]),
        dict(name="Qcur_b", op="ADD", value=(yq + bq).astype(np.float32), src=[("node", 0), ("tensor", bq)]),
        dict(name="Kcur", op="MUL_MAT", value=q8("wk", x, m_kv), src=[W("wk", m_kv), ("tensor", x)]),
        dict(name="Vcur", op="MUL_MAT", value=q8("wv", x, m_kv), src=[W("wv", m_kv), ("tensor", x)]),
        dict(name="ffn_up_gate", op="FUSED_UP_GATE", value=par, op_params=[UNARY_SILU, 0, 0, 0], src=[W("up", m_ff), W("gate", m_ff), ("tensor", x)]),
        dict(name="ffn_down", op="MUL_MAT", value=oracle.mul_mat_q8_1(t, wires["down"], par, k, variant="b200"), src=[W("down", k), ("node", 4)]),
        dict(name="view", op="MUL_MAT", value=oracle.mul_mat_exact(t, rows, xv, r1 - r0), backend="CPU", supported=False,
             src=[("tensor", rows, "iq4_nl", [k, r1 - r0, 1, 1], [18, rs, rs * (r1 - r0), rs * (r1 - r0)]), ("tensor", xv)]),
        dict(name="probs", op="SOFT_MAX", value=probs.astype(np.float32), backend="CPU", src=[("tensor", logits)]),
        dict(name="moe_down", op="MUL_MAT_ID", value=ymoe, src=[W("exps", m_q, n_expert), ("tensor", xm),
                                                                ("tensor", ids_raw, "i32", [n_used, n_tok, 1, 1], [4, n_expert * 4, n_expert * n_tok * 4, n_expert * n_tok * 4])]),
    ]
    case = {"backend": "B2000", "views": [{"node": "view", "weight": "wbig", "r0": r0, "r1": r1}]}
    return case, wires, nodes, dict(bq=bq, ids=ids, order=order, rows=rows, xv=xv, xm=xm, k=k, t=t)


def test_checker_catches_planted_defects(oracle, tmp_path):
    """The oracle's own results pass; each defect a plug bug could cause fails the checker."""
    rng = np.random.default_rng(12)
    case, wires, nodes, v = _planted_graph(oracle, rng)

    def dump(tag, nodes):
        return write_dump(str(tmp_path), tag, case, wires, nodes)

    d = dump("clean", nodes)
    assert fusion_plan(d) == {1: "fused"}
    ids = d.value(d.nodes[8]["src"][2])[0, 0]
    assert np.array_equal(ids, v["ids"]), "strided ids are read through their row stride"
    check_dump(oracle, d)

    def planted(tag, i, value=None, src=None):
        ns = [dict(nd) for nd in nodes]
        if value is not None:
            ns[i]["value"] = value
        if src is not None:
            ns[i]["src"] = src
        return dump(tag, ns)

    t, k = v["t"], v["k"]
    # ids read with row stride n_used instead of n_expert: tokens >= 1 take the experts of the wrong row of the argsort result
    flat = v["order"].reshape(-1)
    wrong_ids = np.stack([flat[tk * 2:tk * 2 + 2] for tk in range(3)])
    assert not np.array_equal(wrong_ids, v["ids"])
    y = np.stack([[oracle.mul_mat_q8_1(t, wires["exps"].reshape(8, -1)[wrong_ids[tk, u]], v["xm"][tk], 64, variant="b200")[0] for u in range(2)]
                  for tk in range(3)]).astype(np.float32)
    defects = {"ids read with row stride n_used": planted("ids-stride", 8, value=y)}
    # the bias added twice by the fused epilogue
    defects["bias added twice"] = planted("bias-twice", 1, value=(nodes[0]["value"] + 2 * v["bq"]).astype(np.float32))
    # the joined Q, K, V launch writes V's segment into the K node
    defects["V segment written into K"] = planted("qkv-segment", 2, value=nodes[3]["value"])
    # ffn_down on a stale q8_1 image: the up/gate result of another input
    x2 = rng.standard_normal((1, k)).astype(np.float32)
    stale = glu_ref("silu", oracle.mul_mat_q8_1(t, wires["gate"], x2, 64, variant="b200"), oracle.mul_mat_q8_1(t, wires["up"], x2, 64, variant="b200"))
    defects["stale q8 image in ffn_down"] = planted("stale-q8", 5, value=oracle.mul_mat_q8_1(t, wires["down"], stale.astype(np.float32), k, variant="b200"))
    # the view fetched as the device's bytes rather than wire bytes: here the wire blocks of the rows in another order, as the plane layout reorders them
    garbled = v["rows"].reshape(-1, 18)[::-1].reshape(-1).copy()
    src = list(nodes[6]["src"])
    src[0] = ("tensor", garbled) + src[0][2:]
    defects["plane bytes read as wire bytes"] = planted("view-planes", 6, value=oracle.mul_mat_exact(t, garbled, v["xv"], 16), src=src)
    for what, dd in defects.items():
        assert _fails(lambda: check_dump(oracle, dd)), what
    # a product of a whole plug weight on the CPU backend fails the placement check
    ns = [dict(nd) for nd in nodes]
    ns[8]["backend"], ns[8]["supported"] = "CPU", False
    assert _fails(lambda: check_placement(dump("moe-on-cpu", ns))), "MoE node on the CPU backend"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the graphs on the GPU
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    """runs the harness once per case, on first use: {case: dump directory}"""
    runs = {}

    def run(case):
        if case not in runs:
            if not os.path.exists(EXE):
                pytest.skip("harness not built (needs the reference headers at build time)")
            out = str(tmp_path_factory.mktemp(case))
            r = subprocess.run([EXE, case, out], capture_output=True, text=True, timeout=1200, cwd=out)
            print(r.stdout[-3000:])
            assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
            runs[case] = out
        return runs[case]
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("case,n", [(c, n) for c, ns in CASES.items() for n in ns])
def test_plug_graph(oracle, harness, case, n):
    d = Dump(harness(case), f"n{n}")
    worst = check_dump(oracle, d)
    for name, r in worst.items():
        print(f"{case} n={n} {name}: {r:.3g}")


@pytest.mark.gpu
def test_partial_weight_upload_in_whole_rows(harness):
    """After the weight-view graph the harness replaces rows [r0, r1) of each weight, through the view (set_tensor on a view of a repacked tensor)
    or through an offset into the whole tensor, and reads the tensor back: the old wire bytes with exactly those rows replaced."""
    case_dir = harness("weight-view")
    d = Dump(case_dir, "n4")
    for view in d.case["views"]:
        old = d.raw({"weight": view["weight"]})
        rows = d.raw({"weight": view["weight"] + "_rows"})
        after = d.raw({"weight": view["weight"] + "_after"})
        rs = rows.size // (view["r1"] - view["r0"])
        want = old.copy()
        want[view["r0"] * rs:view["r1"] * rs] = rows
        assert not np.array_equal(rows, old[view["r0"] * rs:view["r1"] * rs])
        assert np.array_equal(after, want), f"{view['weight']}: rows outside [{view['r0']}, {view['r1']}) changed, or the new rows did not arrive"
