"""MoE prefill: time the mat-vec path (b200q_mul_mat_id_vec) against the grouped tensor-core GEMM (b200q_mul_mat_id_gemm) on model-shaped
expert tensors, and print ONE JSON line.

    python scripts/bench_moe.py [--tokens 16,32,64,128,512] [--iters 10] [--reps 5] [--out FILE]

Weights are synthetic (tests/conftest.make_wire: valid random wire blocks), ids are a uniform random top-k per token.  Each case warms both
paths up, then alternates them `reps` times, each time CUDA events around `iters` back-to-back calls; the median per call is reported.
Per case: time of each path, algorithmic TFLOP/s (2 * n_slots * M * K per matrix, x2 for up/gate), bytes of the experts that received tokens over
the time (the weight traffic a perfect kernel would need), NMSE between the two paths' outputs, and which path the dispatcher takes.
Shapes: Qwen3-30B-A3B expert FFN (Q4_K and IQ4_K), Mixtral-8x7B (IQ4_NL), one tensor-parallel shard (TP = 8) of DeepSeek-V3 (IQ2_XXS)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (model, type, n_expert, n_used, (M, K) of up/gate, (M, K) of down)
MODELS = [("qwen3-30b-a3b", "Q4_K", 128, 8, (768, 2048), (2048, 768)),
          ("qwen3-30b-a3b", "IQ4_K", 128, 8, (768, 2048), (2048, 768)),
          ("mixtral-8x7b", "IQ4_NL", 8, 2, (14336, 4096), (4096, 14336)),
          ("deepseek-v3-tp8", "IQ2_XXS", 256, 8, (256, 7168), (7168, 256))]


def gpu_info() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # the measurement itself does not depend on it
        return {"gpu": "unknown", "error": repr(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="16,32,64,128,512")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--models", default="", help="comma-separated subset of model:type names")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_moe.py needs a CUDA device")
    from conftest import make_wire
    from ik_llama_cpp_b200 import backend as be
    from oracle.oracle import GGML_TYPE, nmse

    torch.cuda.set_device(0)
    tokens = [int(t) for t in args.tokens.split(",")]
    rng = np.random.default_rng(0)
    cases = []

    def timed(fn) -> float:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / args.iters

    for model, name, n_expert, n_used, ug, down in MODELS:
        if args.models and f"{model}:{name}" not in args.models.split(","):
            continue
        t = GGML_TYPE[name]
        for op, (m, k) in (("up_gate", ug), ("down", down)):
            glu = op == "up_gate"
            # one wire tensor of n_expert * m rows = n_expert matrices back to back (the GGUF layout of a 3-D expert tensor)
            W = be.set_expert_tensor(t, make_wire(None, name, n_expert * m, k, seed=1), n_expert, m, k)
            G = be.set_expert_tensor(t, make_wire(None, name, n_expert * m, k, seed=2), n_expert, m, k) if glu else None
            nb1 = 1 if glu else n_used
            for n_tokens in tokens:
                ids_np = np.argsort(rng.random((n_tokens, n_expert)), axis=1)[:, :n_used].astype(np.int32)
                x = torch.from_numpy(rng.standard_normal((n_tokens, nb1, k)).astype(np.float32)).cuda()
                ids = torch.from_numpy(ids_np).cuda()
                out = torch.empty((n_tokens, n_used, m), dtype=torch.float32, device="cuda")
                vec = lambda: be.mul_mat_id(W, x, ids, gate=G)
                gemm = lambda: be.mul_mat_id_gemm(W, x, ids, gate=G, out=out)
                y_vec, y_gemm = vec().cpu().numpy(), gemm().cpu().numpy()
                for _ in range(3):
                    vec(); gemm()
                torch.cuda.synchronize()
                tv, tg = [], []
                for _ in range(args.reps):               # alternate the two paths
                    tv.append(timed(vec)); tg.append(timed(gemm))
                ms_vec, ms_gemm = float(np.median(tv)), float(np.median(tg))
                n_slots = n_tokens * n_used
                flops = 2.0 * n_slots * m * k * (2 if glu else 1)
                active = len(np.unique(ids_np))
                wbytes = active * be.plane_bytes(t, m, k) * (2 if glu else 1)
                cases.append({
                    "model": model, "type": name, "op": op, "M": m, "K": k, "n_expert": n_expert, "n_used": n_used, "n_tokens": n_tokens,
                    "ms_vec": round(ms_vec, 4), "ms_gemm": round(ms_gemm, 4), "speedup": round(ms_vec / ms_gemm, 3),
                    "tflops_vec": round(flops / ms_vec / 1e9, 2), "tflops_gemm": round(flops / ms_gemm / 1e9, 2),
                    "active_expert_gbps_vec": round(wbytes / ms_vec / 1e6, 1), "active_expert_gbps_gemm": round(wbytes / ms_gemm / 1e6, 1),
                    "nmse_gemm_vs_vec": float(f"{nmse(y_gemm, y_vec):.3g}"),
                    "dispatch": "gemm" if be.mul_mat_id_workspace(W, n_tokens, n_used, nb1, glu) else "vec",
                })
                print(json.dumps(cases[-1]), file=sys.stderr, flush=True)
            del W, G
            torch.cuda.empty_cache()

    line = json.dumps({"bench": "moe_prefill", **gpu_info(), "iters": args.iters, "reps": args.reps, "cases": cases})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
