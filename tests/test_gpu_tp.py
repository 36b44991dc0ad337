"""Multi-GPU tests (need >= 2 GPUs with NVLink multicast; skipped on a 1-GPU machine): the in-tree NVLS all-reduce kernel vs the exact sum, eager and
replayed from a CUDA graph, and the row-parallel mat-vec + reduce against the unsharded oracle result."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), NCCL_DEBUG="WARN")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from conftest import random_wire
        from ik_llama_cpp_b200 import backend as be, tp
        from oracle.oracle import GGML_TYPE, Oracle
        red = be.NvlsReducer(512 * 4096)
        res = {"rank": rank, "nvls": red.ok, "why": getattr(red, "err", "")}
        if red.ok:
            # integer-valued floats: the f32 sum is exact in any order
            for n in (4096, 4100, 512 * 4096):
                for it in range(3):
                    t = torch.full((n,), float(rank + 1 + it), device="cuda") + torch.arange(n, device="cuda") % 7
                    red.all_reduce(t)
                    exp = sum(float(r + 1 + it) for r in range(world)) + world * (torch.arange(n, device="cuda") % 7)
                    assert torch.equal(t, exp.float()), (n, it)
            # reduces of different lengths share the parity buffers: long, short, short, long (stale tails must be zeroed)
            for n in (8192, 256, 256, 8192, 512, 8192):
                t = torch.full((n,), float(rank + 2), device="cuda")
                red.all_reduce(t)
                assert torch.equal(t, torch.full_like(t, float(sum(r + 2 for r in range(world))))), n
            # CUDA-graph replay: constant launch arguments, parity/target from the device counter
            x = torch.zeros(4096, device="cuda"); y = torch.empty_like(x)
            s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                y.copy_(x); red.all_reduce(y)
            torch.cuda.current_stream().wait_stream(s); torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y.copy_(x); red.all_reduce(y); y.mul_(0.5); red.all_reduce(y)
            for it in range(4):
                x.fill_(float(rank + it)); g.replay(); torch.cuda.synchronize()
                inner = sum(float(r + it) for r in range(world))
                assert torch.equal(y, torch.full_like(y, inner * 0.5 * world)), it
            res["graph"] = True
        if red.ok:
            # ---- two-shot bf16 all-reduce (prefill-sized REDUCE): small integers are exact in bf16 and in the switch's f32 accumulation ----
            for n in (8, 4096, 4104, 512 * 4096):
                for it in range(3):
                    t = (torch.arange(n, device="cuda") % 5 - 2 + (rank + it) % 3).float()
                    exp = sum((torch.arange(n, device="cuda") % 5 - 2 + (r + it) % 3) for r in range(world)).float()
                    ob = torch.empty(n, dtype=torch.bfloat16, device="cuda"); of = torch.empty(n, device="cuda")
                    red.all_reduce_bf16(t, out_bf16=ob, out_f32=of)
                    assert torch.equal(of, exp) and torch.equal(ob.float(), exp), ("2shot", n, it)
            # in place (out_f32 aliases the input), bf16-rounded random values: result == sum of the bf16-rounded partials (f32 accumulation, one rounding)
            gen = torch.Generator(device="cuda"); gen.manual_seed(1234)
            parts = [torch.randn(64 * 4096, device="cuda", generator=gen) for _ in range(world)]      # same on every rank
            t = parts[rank].clone()
            red.all_reduce_bf16(t, out_f32=t)
            exact = sum(p.to(torch.bfloat16).double() for p in parts)
            # the switch's rounding of the reduced bf16 value is not specified.  Measured: 2 and 4 ranks give 78-81 % of the elements equal to
            # RN(exact sum) and a worst relative error of 2^-7.04: neither RN (<= 2^-9) nor plain truncation; the bound leaves a factor 2 for
            # the 8-rank tree
            rn = exact.float().to(torch.bfloat16).float()
            res["two_shot_rn_fraction"] = float((t == rn).float().mean())
            worst = float(((t.double() - exact).abs() / (exact.abs() + 1e-30)).max())
            res["two_shot_worst_rel"] = worst
            amax = float(exact.abs().max())
            assert bool(((t.double() - exact).abs() <= exact.abs() * 2.0 ** -6 + amax * 2.0 ** -12).all()), worst
            # interleaved with the one-shot f32 reduce and replayed from a CUDA graph
            x = torch.zeros(8192, device="cuda"); y = torch.empty_like(x); yb = torch.empty(8192, dtype=torch.bfloat16, device="cuda")
            s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                y.copy_(x); red.all_reduce_bf16(y, out_bf16=yb, out_f32=y); red.all_reduce(y)
            torch.cuda.current_stream().wait_stream(s); torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y.copy_(x); red.all_reduce_bf16(y, out_bf16=yb, out_f32=y); red.all_reduce(y); red.all_reduce_bf16(y, out_f32=y)
            for it in range(4):
                x.fill_(float((rank + it) % 2)); g.replay(); torch.cuda.synchronize()
                inner = sum(float((r + it) % 2) for r in range(world))
                assert torch.equal(y, torch.full_like(y, inner * world * world)), ("2shot graph", it)
            res["two_shot"] = True
        # row-parallel (K-split) mat-vec + reduce == unsharded result
        t = GGML_TYPE["IQ4_NL"]; m, k = 256, 2048
        rng = np.random.default_rng(9)
        wire = random_wire("IQ4_NL", m, k, rng)
        x = rng.standard_normal((1, k)).astype(np.float32)
        shard, ks, k0 = tp.shard_cols(wire, t, m, k, world, rank, granularity=256)
        w = be.set_tensor(t, shard, m, ks)
        part = be.mul_mat(w, torch.from_numpy(np.ascontiguousarray(x[:, k0:k0 + ks])).cuda())
        red.all_reduce(part)
        ref = Oracle().mul_mat_exact(t, wire, x, m)
        err = float(((part.cpu().numpy() - ref) ** 2).sum() / (ref ** 2).sum())
        assert err <= 5e-4, err
        res["tp_nmse"] = err
        if red.ok:
            # ---- fused path: reduce inside the mat-vec kernels (multimem.red epilogue -> flag wait + read in the next prologue) ----
            m1, k1, m2 = 512, 2048, 384                       # "wo": [m1 x k1] K-split; consumer "up/gate": [m2 x m1], replicated
            wire1 = random_wire("IQ4_NL", m1, k1, np.random.default_rng(31))
            wire2 = random_wire("IQ4_NL", m2, m1, np.random.default_rng(32)); wire3 = random_wire("IQ4_NL", m2, m1, np.random.default_rng(33))
            sh1, ks1, k01 = tp.shard_cols(wire1, t, m1, k1, world, rank, granularity=256)
            w1 = be.set_tensor(t, sh1, m1, ks1); w2 = be.set_tensor(t, wire2, m2, m1); w3 = be.set_tensor(t, wire3, m2, m1)
            orc = Oracle()
            y2 = torch.empty((1, m2), device="cuda"); y3 = torch.empty((1, m2), device="cuda")
            xs = [np.random.default_rng(40 + i).standard_normal((1, k1)).astype(np.float32) for i in range(5)]
            xg = torch.empty((1, ks1), device="cuda")

            def chain():
                be.mul_mat_vec_tp([w1], xg, None, red, reduce_out=True)                        # partial rows -> switch
                be.mul_mat_vec_tp([w2], None, [y2], red, reduce_in=True)                       # consumer 1: plain mat-vec
                be.mul_mat_vec_tp([w1], xg, None, red, reduce_out=True)                        # second reduce (other parity)
                be.mul_mat_vec_tp([w2], None, [y3], red, reduce_in=True, gate=w3, unary="silu")  # consumer 2: fused up/gate

            def check(x):
                h = red.reduced_view(m1).cpu().numpy()[None, :]          # what the consumers saw
                ref1 = orc.mul_mat_exact(t, wire1, x, m1)
                e1 = float(((h - ref1) ** 2).sum() / (ref1 ** 2).sum())
                assert e1 <= 5e-4, e1                                     # sum of per-rank q8_1 partials vs exact
                r2 = orc.mul_mat_q8_1(t, wire2, h, m2, variant="b200")
                d2 = float(np.abs(y2.cpu().numpy() - r2).max() / np.sqrt((r2 ** 2).mean()))
                assert d2 <= 2e-5, ("consumer of the first reduce", d2)
                u = r2.astype(np.float64); gt = orc.mul_mat_q8_1(t, wire3, h, m2, variant="b200").astype(np.float64)
                r3 = gt / (1 + np.exp(-gt)) * u
                assert np.abs(y3.cpu().numpy() - r3).max() <= 5e-5 * float(np.sqrt((r3 ** 2).mean()))
                return e1

            for i in range(2):                                             # eager, both parities twice
                xg.copy_(torch.from_numpy(np.ascontiguousarray(xs[i][:, k01:k01 + ks1]))); chain(); res["fused_eager_nmse"] = check(xs[i])
            s2 = torch.cuda.Stream(); s2.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s2):
                chain()
            torch.cuda.current_stream().wait_stream(s2); torch.cuda.synchronize()
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                chain()
            for i in range(2, 5):                                          # CUDA-graph replay (PDL edges inside the graph)
                xg.copy_(torch.from_numpy(np.ascontiguousarray(xs[i][:, k01:k01 + ks1]))); g2.replay(); res["fused_graph_nmse"] = check(xs[i])
        q.put(res)
    except BaseException as e:                      # report instead of leaving the parent to time out on the queue
        import traceback
        q.put({"rank": rank, "error": repr(e), "trace": traceback.format_exc()})
        raise
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_nvls_allreduce_and_row_parallel_matvec(world):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f"needs >= {world} GPUs")
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = []
    for _ in procs:
        res.append(q.get(timeout=300))
        if "error" in res[-1]:                      # a failed rank leaves its peers inside a collective: stop them
            for p in procs:
                p.join(timeout=20)
                if p.is_alive(): p.kill()
            pytest.fail(f"rank {res[-1]['rank']}: {res[-1]['error']}\n{res[-1]['trace']}")
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    print(res)
    assert all(r["tp_nmse"] <= 5e-4 for r in res)
    if all(r["nvls"] for r in res):
        assert all(r.get("fused_graph_nmse", 1.0) <= 5e-4 for r in res)
        assert all(r.get("two_shot") for r in res)
