"""Tensor-parallel MoE: time one DeepSeek-V3 MoE layer per rank (routed experts + the shared expert, IQ2_XXS) and print one JSON line per token count.

    python scripts/bench_moe_tp.py [--tokens 1,8,64,512] [--iters 20] [--reps 5] [--out FILE]              # one GPU: the whole layer
    torchrun --nproc-per-node W scripts/bench_moe_tp.py ...                                               # W ranks: each its shard + the reduce

Each rank holds its shard of the layer as ik_llama_cpp_b200/tp.py cuts it (tp.moe_ffn_plan: rows of ffn_up_exps / ffn_gate_exps, the K range of
ffn_down_exps; the shared expert by shard_rows / shard_cols) and runs backend.moe_tp_partial: up/gate, down, the combine (b200q_moe_combine) and
the shared expert's partial.  With W > 1 the partials are summed by the in-tree NVLS reduce: the one-shot f32 kernel up to 32 tokens, the two-shot
bf16 kernel above (the reference casts the partial to bf16 when ne[1] > 32).  One layer step is captured in a CUDA graph and replayed; CUDA events
around `iters` replays, median over `reps`.  Weights are synthetic (valid random wire blocks), routing a uniform random top-8 with normalised weights.

Before anything is timed, a correctness gate: the layer (reduced over the ranks) at 1 and 512 tokens against the f64 oracle on the first and last
token; NMSE > 5e-4 on any rank -> exit 3 on every rank."""
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

# DeepSeek-V3 MoE layer: n_embd, routed experts, used per token, n_ff of an expert, n_ff of the shared expert
N_EMBD, N_EXPERT, N_USED, N_FF, N_FF_SHEXP = 7168, 256, 8, 2048, 2048
TYPE = "IQ2_XXS"
POOL = 8            # distinct expert matrices per tensor; expert e holds pool matrix e % POOL with its rows rotated by 4 (e // POOL)
GATE_TOL = 5e-4


def gpu_info() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", os.environ.get("LOCAL_RANK", "0")],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # the measurement itself does not depend on it
        return {"gpu": "unknown", "error": repr(e)}


class LayerWeights:
    """The wire bytes of the layer, identical on every rank (fixed seeds), and one rank's shard on the device."""

    def __init__(self, be, tp, t, world, rank):
        from conftest import random_wire
        rng = np.random.default_rng(2024)
        self.t = t
        self.pool = {name: [random_wire(TYPE, m, k, rng).reshape(m, -1) for _ in range(POOL)]
                     for name, m, k in (("up", N_FF, N_EMBD), ("gate", N_FF, N_EMBD), ("down", N_EMBD, N_FF))}
        self.shexp = [random_wire(TYPE, m, k, rng) for m, k in ((N_FF_SHEXP, N_EMBD), (N_FF_SHEXP, N_EMBD), (N_EMBD, N_FF_SHEXP))]
        split = tp.moe_ffn_plan(N_FF, world, t)
        self.split = split
        self.U = self.G = self.D = None
        if split[rank]:
            up, gate = (tp.shard_expert_rows(self._tensor(n), t, N_EXPERT, N_FF, N_EMBD, split, rank)[0] for n in ("up", "gate"))
            self.U, self.G = (be.set_expert_tensor(t, w, N_EXPERT, split[rank], N_EMBD) for w in (up, gate))
            down, ks, _ = tp.shard_expert_cols(self._tensor("down"), t, N_EXPERT, N_EMBD, N_FF, split, rank)
            self.D = be.set_expert_tensor(t, down, N_EXPERT, N_EMBD, ks)
        g = tp.moe_expert_granularity(t)
        (u, mu), (gt, _) = (tp.shard_rows(w, t, N_FF_SHEXP, N_EMBD, world, rank, granularity=g) for w in self.shexp[:2])
        d, ks, _ = tp.shard_cols(self.shexp[2], t, N_EMBD, N_FF_SHEXP, world, rank, granularity=g)
        self.shared = be.SharedExpert(be.set_tensor(t, u, mu, N_EMBD), be.set_tensor(t, gt, mu, N_EMBD), be.set_tensor(t, d, N_EMBD, ks)) if mu else None

    def expert(self, name, e):
        return np.roll(self.pool[name][e % POOL], 4 * (e // POOL), axis=0).ravel()

    def _tensor(self, name):
        return np.concatenate([self.expert(name, e) for e in range(N_EXPERT)])

    def shard_bytes(self, be, active: int) -> int:
        """device bytes a step streams: the active experts' shard matrices and the shared expert's shard"""
        b = 0
        if self.D is not None:
            b += active * (2 * be.plane_bytes(self.t, self.U.m, N_EMBD) + be.plane_bytes(self.t, N_EMBD, self.D.k))
        if self.shared is not None:
            b += 2 * self.shared.up.planes.numel() + self.shared.down.planes.numel()
        return b


def oracle_layer(orc, W, t, x, ids, w, tokens):
    """f64 MoE FFN + shared expert of the given tokens on the wire bytes"""
    def glu(g, u):
        g = g.astype(np.float64)
        return (g / (1 + np.exp(-g)) * u).astype(np.float32)
    out = []
    for tk in tokens:
        xt = x[tk:tk + 1]
        y = np.zeros(N_EMBD)
        for u, e in enumerate(ids[tk]):
            h = glu(orc.mul_mat_exact(t, W.expert("gate", e), xt, N_FF), orc.mul_mat_exact(t, W.expert("up", e), xt, N_FF))
            y += float(w[tk, u]) * orc.mul_mat_exact(t, W.expert("down", e), h, N_EMBD)[0]
        h = glu(orc.mul_mat_exact(t, W.shexp[1], xt, N_FF_SHEXP), orc.mul_mat_exact(t, W.shexp[0], xt, N_FF_SHEXP))
        out.append(y + orc.mul_mat_exact(t, W.shexp[2], h, N_EMBD)[0])
    return np.stack(out)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="1,8,64,512")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_moe_tp.py needs a CUDA device")
    from ik_llama_cpp_b200 import backend as be, tp
    from oracle.oracle import GGML_TYPE, Oracle, nmse

    rank, world, local_rank = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    dist = red = None
    tokens = [int(s) for s in args.tokens.split(",")]
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("NCCL_DEBUG", "WARN")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        red = be.NvlsReducer(max(max(tokens), 512) * N_EMBD)
    t = GGML_TYPE[TYPE]
    W = LayerWeights(be, tp, t, world, rank)
    rng = np.random.default_rng(7)          # same inputs on every rank

    def inputs(n):
        x = (rng.standard_normal((n, N_EMBD)) * 0.5).astype(np.float32)
        ids = np.stack([rng.permutation(N_EXPERT)[:N_USED] for _ in range(n)]).astype(np.int32)
        p = rng.uniform(0.05, 1.0, (n, N_USED)).astype(np.float32)
        return x, ids, (p / p.sum(axis=1, keepdims=True)).astype(np.float32)

    def step(x, ids, w):
        y = be.moe_tp_partial(x, ids, w, N_EMBD, W.D, up=W.U, gate=W.G, shared=W.shared)
        if red is None:
            return y
        if x.shape[0] <= 32:
            return red.all_reduce(y)
        return red.all_reduce_bf16(y, out_f32=y)

    # ---------------- correctness gate, before anything is timed ----------------
    orc, gate = Oracle(), {}
    for n in (1, 512):
        x, ids, w = inputs(n)
        y = step(*(torch.from_numpy(a).cuda() for a in (x, ids, w))).cpu().numpy()
        toks = sorted({0, n - 1})
        gate[n] = nmse(y[toks], oracle_layer(orc, W, t, x, ids, w, toks))
    bad = torch.tensor([float(any(not (e <= GATE_TOL) for e in gate.values()))], device="cuda")
    if dist is not None:
        dist.all_reduce(bad)
    if float(bad) > 0:
        print(f"bench_moe_tp.py: correctness gate FAILED on rank {rank}: NMSE vs the f64 oracle {gate} (tol {GATE_TOL})", file=sys.stderr)
        if dist is not None:
            dist.destroy_process_group()
        return 3

    info = gpu_info()
    for n in tokens:
        xh, idh, wh = inputs(n)
        x, ids, w = (torch.from_numpy(a).cuda() for a in (xh, idh, wh))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                step(x, ids, w)              # warm-up: workspaces and modules before the capture
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step(x, ids, w)
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                g.replay()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / args.iters)
        ms = float(np.median(times))
        nbytes = W.shard_bytes(be, len(np.unique(idh)))
        line = {"bench": "moe_tp", **info, "world": world, "rank": rank, "model": "deepseek-v3", "type": TYPE, "n_tokens": n,
                "n_ff_shard": W.split[rank], "ms_per_layer": round(ms, 4), "ms_reps": [round(v, 4) for v in times],
                "reduce": "none" if red is None else ("nvls f32 one-shot" if n <= 32 else "nvls bf16 two-shot"),
                "weight_gbps": round(nbytes / ms / 1e6, 1), "gate_nmse": {str(k): float(f"{v:.3g}") for k, v in gate.items()},
                "iters": args.iters, "reps": args.reps}
        if rank == 0:
            print(json.dumps(line), flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(json.dumps(line) + "\n")
        del g
    if dist is not None:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
