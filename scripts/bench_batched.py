"""Batched MUL_MAT (b200q_mul_mat_batched) on DeepSeek-V3's absorbed-MLA per-head products, against the alternatives it chooses between.

    python scripts/bench_batched.py [--heads 128 16] [--n 1 2 4 8 16 32 64 128 512] [--reps 7] [--iters 20] [--json out.jsonl]

For every (heads, product, type, n) it times, each replayed from its own CUDA graph, alternating within the run:
  entry    b200q_mul_mat_batched on the strided view the graph hands over (q_nope_perm / kqv_compressed_perm);
  loop     one b200q_mul_mat per head on a contiguous copy of x (what a per-entry loop costs; the copy itself is not timed);
  vec      b200q_mul_mat_id_vec with identity ids on the contiguous copy (the mat-vec side), for n <= 32;
  grouped  b200q_mul_mat_id_gemm with identity ids on the contiguous copy (the grouped GEMM), where it is eligible (K % 256 == 0).
Shapes: wk_b K = 128 (qk_nope), M = 512 (kv_lora); wv_b K = 512, M = 128 (v_head); 128 heads, and 16 per rank at TP-8.  Types: Q8_0 (what
llm_prepare_mla makes) and IQ4_NL (a 32-block 4-bit type; K = 128 rules out the 256-blocks).  Before timing, the entry's result is checked
against the loop's.  The card name, power limit and SM clock are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ik_llama_cpp_b200 as pkg                 # noqa: E402
import ik_llama_cpp_b200.backend as be          # noqa: E402
from ik_llama_cpp_b200._lib import check        # noqa: E402

TYPES = {"Q8_0": 8, "IQ4_NL": 20}
BLOCK_BYTES = {"Q8_0": 34, "IQ4_NL": 18}        # 32 weights per block, an f16 scale + the quants
PRODUCTS = [("wk_b", 128, 512), ("wv_b", 512, 128)]
SMEM_COLUMNS = 200 * 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def random_wire(name, n_mat, m, k, rng):
    """valid wire blocks: random quants, f16 scales of a sane size"""
    nb = n_mat * m * (k // 32)
    blk = rng.integers(0, 256, (nb, BLOCK_BYTES[name]), dtype=np.uint8)
    blk[:, 0:2] = np.frombuffer((rng.random(nb) * 0.01 + 0.001).astype(np.float16).tobytes(), np.uint8).reshape(nb, 2)
    return blk.ravel()


def mla_x(which, n, n_head, k, g):
    if which == "wk_b":
        buf = torch.randn(256 + n * n_head * 192, generator=g).cuda()
        return buf[256:].view(n, n_head, 192)[:, :, :128].transpose(0, 1)
    buf = torch.randn(256 + n * n_head * 512, generator=g).cuda()
    return buf[256:].view(n, n_head, 512).transpose(0, 1)


def graphs_of(variants):
    """every variant runs once before any capture: the backend's shared workspace reaches its final size first, so no captured graph keeps
    a pointer to a workspace that a later call outgrew and freed"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for fn in variants.values():
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graphs = {}
    for v, fn in variants.items():
        graphs[v] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[v]):
            fn()
    return graphs


def time_graph(g, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters       # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--heads", type=int, nargs="+", default=[128, 16])
    ap.add_argument("--n", type=int, nargs="+", default=[1, 2, 4, 8, 16, 32, 64, 128, 512])
    ap.add_argument("--types", nargs="+", default=list(TYPES))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batched.py needs a CUDA device")
    L = pkg.lib()
    print(f"# card: {card()}", flush=True)
    rng = np.random.default_rng(0)
    g = torch.Generator().manual_seed(0)
    rows = []
    print(f"{'heads':>5} {'product':>7} {'type':>6} {'n':>4} {'entry us':>9} {'loop us':>9} {'vec us':>9} {'grouped us':>10} {'entry/loop':>10}")
    for n_head in args.heads:
        for which, k, m in PRODUCTS:
            for name in args.types:
                t = TYPES[name]
                w = be.set_expert_tensor(t, random_wire(name, n_head, m, k, rng), n_head, m, k)
                pb = be.plane_bytes(t, m, k)
                for n in args.n:
                    x = mla_x(which, n, n_head, k, g)
                    xc = x.contiguous()
                    ids = torch.arange(n_head, dtype=torch.int32, device="cuda")[:, None].repeat(1, n).contiguous()
                    y_entry = torch.empty((n_head, n, m), device="cuda")
                    y_loop = torch.empty_like(y_entry)
                    need = int(L.b200q_mul_mat_workspace(t, m, k, n))
                    ws = torch.empty(max(need, 256), dtype=torch.uint8, device="cuda")

                    def loop():
                        st = torch.cuda.current_stream().cuda_stream
                        for h in range(n_head):
                            check(L.b200q_mul_mat(t, w.ptr + h * pb, xc.data_ptr() + h * n * k * 4, y_loop.data_ptr() + h * n * m * 4, m, k, n,
                                                      ws.data_ptr(), need, st), "b200q_mul_mat")
                    variants = {"entry": lambda: be.mul_mat_batched(w, x, True, out=y_entry), "loop": loop}
                    if n <= 32 and n * (k + k // 4) <= SMEM_COLUMNS:      # (far slower than the others above 32 columns)
                        variants["vec"] = lambda: be.mul_mat_id(w, xc, ids)
                    if k % 256 == 0:
                        y_g = torch.empty_like(y_entry)
                        variants["grouped"] = lambda: be.mul_mat_id_gemm(w, xc, ids, out=y_g)
                    graphs = graphs_of(variants)
                    for gr in graphs.values():
                        gr.replay()
                    torch.cuda.synchronize()
                    err = (y_entry - y_loop).abs().max().item() / max(y_loop.abs().max().item(), 1e-30)
                    if not err < 2e-2:
                        sys.exit(f"entry and loop disagree: {n_head} {which} {name} n={n}: max rel {err:.3g}")
                    for gr in graphs.values():
                        time_graph(gr, 3)
                    times = {v: [] for v in graphs}
                    for _ in range(args.reps):
                        for v, gr in graphs.items():
                            times[v].append(time_graph(gr, args.iters))
                    med = {v: float(np.median(ts)) for v, ts in times.items()}
                    row = dict(heads=n_head, product=which, type=name, n=n, m=m, k=k, weight_bytes=int(pb * n_head), max_rel_err_vs_loop=err,
                               **{f"{v}_us": round(u, 2) for v, u in med.items()})
                    rows.append(row)
                    fmt = lambda v: f"{med[v]:9.1f}" if v in med else f"{'-':>9}"
                    print(f"{n_head:>5} {which:>7} {name:>6} {n:>4} {fmt('entry')} {fmt('loop')} {fmt('vec')} {fmt('grouped'):>10} "
                          f"{med['entry'] / med['loop']:10.2f}", flush=True)
    print(f"# card: {card()}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
