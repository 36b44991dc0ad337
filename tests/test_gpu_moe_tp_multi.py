"""Multi-GPU tests of tensor-parallel MoE (skipped below 2 GPUs, like test_gpu_tp.py): the layers of test_gpu_moe_tp.py with one rank per GPU, each
rank's partial (backend.moe_tp_partial on its shards) summed by the in-tree NVLS reduce (the one-shot f32 kernel up to 32 tokens, the two-shot bf16
kernel above), and every rank's reduced layer checked against the unsharded down + combine computed on its own GPU."""
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
        from ik_llama_cpp_b200 import backend as be
        from oracle.oracle import nmse
        from test_gpu_moe_tp import MODELS, Layer, routing
        red = be.NvlsReducer(512 * 7168)
        res = {"rank": rank, "nvls": red.ok, "why": getattr(red, "err", ""), "nmse": {}}
        for case in MODELS:
            L = Layer(be, case, seed=1)                     # same wire bytes on every rank
            _, (U, G, D), shared = L.shards(be, world, rank)
            rng = np.random.default_rng(5)                  # same inputs on every rank
            for n in (1, 8, 64, 512):
                x = torch.from_numpy((rng.standard_normal((n, L.n_embd)) * 0.5).astype(np.float32)).cuda()
                ids, w = (torch.from_numpy(a).cuda() for a in routing(rng, n, L.n_expert, L.n_used))
                y = be.moe_tp_partial(x, ids, w, L.n_embd, D, up=U, gate=G)
                if red.ok and n > 32:
                    red.all_reduce_bf16(y, out_f32=y)
                else:
                    red.all_reduce(y)
                ref = be.moe_combine(be.mul_mat_id_dispatch(L.D, be.mul_mat_id_dispatch(L.U, x.view(n, 1, -1), ids, gate=L.G), ids), w)
                e = nmse(y.cpu().numpy(), ref.cpu().numpy())
                res["nmse"][f"{case[0]}/{n}"] = e
                assert e <= (5e-4 if red.ok and n > 32 else 2e-5), (case[0], n, e)
            del L, U, G, D, shared
            torch.cuda.empty_cache()
        q.put(res)
    except BaseException as e:                      # report instead of leaving the parent to time out on the queue
        import traceback
        q.put({"rank": rank, "error": repr(e), "trace": traceback.format_exc()})
        raise
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 8])
def test_moe_layers_reduced_over_the_ranks(world):
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
        res.append(q.get(timeout=1800))
        if "error" in res[-1]:                      # a failed rank leaves its peers inside a collective: stop them
            for p in procs:
                p.join(timeout=20)
                if p.is_alive(): p.kill()
            pytest.fail(f"rank {res[-1]['rank']}: {res[-1]['error']}\n{res[-1]['trace']}")
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    print(res)
