"""Time one layer's wkv_b products of DeepSeek's MLA prompt processing (the pp_opt graph, src/graphs/build_deepseek2.cpp:922-1022):
kv_f32 = wkv_b_iter x kv_cache_nope for every slice of wkv_b, Q8_0, K = kv_lora_rank = 512, 256 rows per head.

  slice     b200q_mul_mat_rows on the rows of the whole uploaded weight, over the f16 K cache in place (576 halves per column, 64 in)
  separate  b200q_mul_mat on the same rows uploaded as their own tensor, over a contiguous f32 copy of the cache (the copy is not timed; the
            f32 -> bf16 conversion inside the call is)

Each path is one CUDA graph holding the layer's slices, replayed `--iters` times per repetition; the two alternate within each repetition.  Slices
follow the reference's split (attn_max_batch = 256 MiB, src/llama.cpp:7609): n_max_head = n_head / niter for the first niter dividing n_head that
brings the f32 product under 256 MiB.  Prints the card name and power limit read in the same run, then one row per shape: median ms per layer
of each path, TFLOP/s (2 m 512 n_kv per slice), the ratio separate / slice, and the spread (max / min - 1) of each path over the repetitions.

    python scripts/bench_mla_pp.py [--reps 7] [--iters 20] [--heads 16,64,128] [--nkv 1024,2048,4096,8192,16384]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ik_llama_cpp_b200.backend as be  # noqa: E402
from ik_llama_cpp_b200 import _lib  # noqa: E402

Q8_0, F16, K, PER_HEAD, CACHE_COLS, ROPE = 8, 1, 512, 256, 576, 64
MODELS = {16: "DeepSeek-V2-Lite", 64: "Kimi-K2", 128: "DeepSeek-V3"}


def n_max_head(n_head, n_kv, attn_max_batch=256):
    size = n_head * PER_HEAD * n_kv * 4 // (1024 * 1024)
    if size <= attn_max_batch:
        return n_head
    for niter in range(2, n_head):
        if n_head % niter == 0 and size // niter <= attn_max_batch:
            return n_head // niter
    return 1


def q8_0_wire(rows, seed):
    """random valid Q8_0 blocks: f16 scale ~ 1e-3, int8 quants"""
    rng = np.random.default_rng(seed)
    blk = np.zeros((rows * K // 32, 34), np.uint8)
    blk[:, :2] = np.full(rows * K // 32, 1e-3, np.float16).view(np.uint8).reshape(-1, 2)
    blk[:, 2:] = rng.integers(-127, 128, (rows * K // 32, 32), dtype=np.int8).view(np.uint8)
    return blk.ravel()


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name()


def graph_of(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()                                        # warm up every shape before capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def time_graph(g, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--heads", default="16,64,128")
    ap.add_argument("--nkv", default="1024,2048,4096,8192,16384")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mla_pp: needs a CUDA device")
    L = _lib.lib()
    print(f"card: {card()}")
    print(f"{'model':<17} {'heads':>5} {'n_kv':>6} {'slices':>6} {'slice ms':>9} {'TFLOP/s':>8} {'separate ms':>11} {'TFLOP/s':>8} {'sep/slice':>9} "
          f"{'spread slice':>12} {'spread sep':>10}")
    for n_head in [int(h) for h in a.heads.split(",")]:
        rows = n_head * PER_HEAD
        wire = q8_0_wire(rows, n_head)
        w = be.set_tensor(Q8_0, wire, rows, K)
        for n_kv in [int(v) for v in a.nkv.split(",")]:
            m = n_max_head(n_head, n_kv) * PER_HEAD
            origins = list(range(0, rows, m))
            rs = len(wire) // rows
            parts = [be.set_tensor(Q8_0, wire[r * rs:(r + m) * rs], m, K) for r in origins]
            cache = torch.randn(n_kv, CACHE_COLS, device="cuda").half()
            x16 = cache[:, ROPE:]
            xf = x16.float().contiguous()
            dst = torch.empty(n_kv, m, device="cuda")
            ws_s = torch.empty(max(1, L.b200q_mul_mat_rows_workspace(Q8_0, rows, 0, m, K, n_kv, F16, CACHE_COLS)), dtype=torch.uint8, device="cuda")
            ws_p = torch.empty(max(1, L.b200q_mul_mat_workspace(Q8_0, m, K, n_kv)), dtype=torch.uint8, device="cuda")

            def slice_layer():
                st = torch.cuda.current_stream().cuda_stream
                for r in origins:
                    _lib.check(L.b200q_mul_mat_rows(Q8_0, w.ptr, rows, r, F16, x16.data_ptr(), CACHE_COLS, dst.data_ptr(), m, K, n_kv, ws_s.data_ptr(),
                                                    ws_s.numel(), st), "b200q_mul_mat_rows")

            def separate_layer():
                st = torch.cuda.current_stream().cuda_stream
                for p in parts:
                    _lib.check(L.b200q_mul_mat(Q8_0, p.ptr, xf.data_ptr(), dst.data_ptr(), m, K, n_kv, ws_p.data_ptr(), ws_p.numel(), st), "b200q_mul_mat")

            gs, gp = graph_of(slice_layer), graph_of(separate_layer)
            ts, tp = [], []
            for _ in range(a.reps):
                ts.append(time_graph(gs, a.iters))
                tp.append(time_graph(gp, a.iters))
            ms_s, ms_p = float(np.median(ts)), float(np.median(tp))
            flop = 2.0 * rows * K * n_kv
            print(f"{MODELS.get(n_head, '?'):<17} {n_head:>5} {n_kv:>6} {len(origins):>6} {ms_s:>9.3f} {flop / ms_s / 1e9:>8.1f} {ms_p:>11.3f} "
                  f"{flop / ms_p / 1e9:>8.1f} {ms_p / ms_s:>9.3f} {max(ts) / min(ts) - 1:>12.1%} {max(tp) / min(tp) - 1:>10.1%}", flush=True)
            del gs, gp, parts, dst, ws_s, ws_p, cache, xf
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
