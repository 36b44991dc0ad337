"""MOE_FUSED_UP_GATE with merged up/gate experts (ffn_gate_up_exps, b200q_moe_up_gate_merged) against the split form (separate up and gate
expert tensors, b200q_mul_mat_id) on the same bytes, timed in one run, and print ONE JSON line.

    python scripts/bench_moe_merged.py [--tokens 1,8,64,512] [--iters 20] [--reps 7] [--out FILE]

Both forms launch the same kernels on the same weights (the merged one reads two row ranges of one matrix), so the expectation is equal time
within the run-to-run spread.  Weights are synthetic (tests/conftest.make_wire), ids a uniform random top-k per token.  Each case warms both forms
up, then alternates them `reps` times, each time CUDA events around `iters` back-to-back dispatcher calls; the median per call is reported with the
spread (max - min over the reps) of each form, whether the outputs are bit-equal, and which path the dispatcher takes.  Shapes: Qwen3-30B-A3B Q4_K,
Mixtral-8x7B IQ4_NL, one tensor-parallel shard (TP = 8) of DeepSeek-V3 IQ2_XXS."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

# (model, type, n_expert, n_used, n_ff, K)
MODELS = [("qwen3-30b-a3b", "Q4_K", 128, 8, 768, 2048),
          ("mixtral-8x7b", "IQ4_NL", 8, 2, 14336, 4096),
          ("deepseek-v3-tp8", "IQ2_XXS", 256, 8, 256, 7168)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="1,8,64,512")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_moe_merged.py needs a CUDA device")
    from bench_moe import gpu_info
    from conftest import make_wire
    from ik_llama_cpp_b200 import backend as be
    from oracle.oracle import GGML_TYPE

    torch.cuda.set_device(0)
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

    for model, name, n_expert, n_used, n_ff, k in MODELS:
        t = GGML_TYPE[name]
        gate = [make_wire(None, name, n_ff, k, seed=[1, e]) for e in range(n_expert)]
        up = [make_wire(None, name, n_ff, k, seed=[2, e]) for e in range(n_expert)]
        Mg = be.set_expert_tensor(t, np.concatenate([np.concatenate([g, u]) for g, u in zip(gate, up)]), n_expert, 2 * n_ff, k)
        U = be.set_expert_tensor(t, np.concatenate(up), n_expert, n_ff, k)
        G = be.set_expert_tensor(t, np.concatenate(gate), n_expert, n_ff, k)
        del gate, up
        for n_tokens in [int(s) for s in args.tokens.split(",")]:
            ids = torch.from_numpy(np.argsort(rng.random((n_tokens, n_expert)), axis=1)[:, :n_used].astype(np.int32)).cuda()
            x = torch.from_numpy(rng.standard_normal((n_tokens, 1, k)).astype(np.float32)).cuda()
            out_m = torch.empty((n_tokens, n_used, n_ff), dtype=torch.float32, device="cuda")
            out_s = torch.empty_like(out_m)
            merged = lambda: be.moe_up_gate_merged(Mg, x, ids, out=out_m)
            split = lambda: be.mul_mat_id_dispatch(U, x, ids, gate=G, out=out_s)
            for _ in range(3):
                merged(); split()
            torch.cuda.synchronize()
            equal = bool(torch.equal(out_m, out_s))
            tm, ts = [], []
            for _ in range(args.reps):                   # alternate the two forms
                tm.append(timed(merged)); ts.append(timed(split))
            ms_m, ms_s = float(np.median(tm)), float(np.median(ts))
            cases.append({"model": model, "type": name, "n_expert": n_expert, "n_used": n_used, "n_ff": n_ff, "K": k, "n_tokens": n_tokens,
                          "ms_merged": round(ms_m, 4), "ms_split": round(ms_s, 4), "merged_over_split": round(ms_m / ms_s, 3),
                          "spread_merged": round(max(tm) - min(tm), 4), "spread_split": round(max(ts) - min(ts), 4), "bit_equal": equal,
                          "dispatch": "gemm" if be.moe_up_gate_merged_workspace(Mg, n_tokens, n_used, 1) else "vec"})
            print(json.dumps(cases[-1]), file=sys.stderr, flush=True)
        del Mg, U, G
        torch.cuda.empty_cache()

    line = json.dumps({"bench": "moe_up_gate_merged", **gpu_info(), "iters": args.iters, "reps": args.reps, "cases": cases})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
