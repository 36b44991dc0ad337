"""GPU tests of MOE_FUSED_UP_GATE over merged up/gate experts (ffn_gate_up_exps, src[1] = NULL): b200q_moe_up_gate_merged / backend.moe_up_gate_merged.
Each expert is one [2 n_ff x K] matrix whose rows [0, n_ff) are the gate and [n_ff, 2 n_ff) the up rows (the reference CPU op,
iqk_moe_fused_up_gate, reads them so: ggml.c:18626-18627).  The merged call runs the launches of the split form (b200q_mul_mat_id with separate
up and gate expert tensors) with each operand a row range of the one matrix.

  * Decode (mat-vec, k_mmvq_id / k_wire_mmvq_id): every slot against the q8_1 oracle of test_gpu_moe_decode.py at the GLU bar of DESIGN §5
    (|y - ref| <= 5e-5 rms(ref)), all 46 types, one token and a batch walked in token chunks (B200Q_MOE_CHUNK_TOKENS, read once per process:
    run in a child process), nb1 = 1 and nb1 = n_used, skipped ids as exact zero rows with one chunk whose ids are all skipped.
  * Prefill (grouped GEMM): the nine fused types and four generic ones against the exact product at the up/gate bar of test_gpu_moe_prefill.py
    (NMSE <= 2e-4; 1e-3 with a silu limit).
  * Tolerance-free: the merged result equals the split form on the two halves uploaded as separate expert tensors, bit for bit, on both sides of
    the crossover at the Qwen3-30B-A3B, Mixtral-8x7B and DeepSeek-V3 TP-8 shapes, at n_ff = 1408 (not a multiple of 128: the gate range's last
    row tile ends inside the matrix, its rows past n_ff are zero-filled by the TMA map) and for an _R4 type.  Both sides run the same kernels on the
    same bytes: the decode kernels see the same plane pointers, the grouped GEMM the same tiles (rows past n_ff are dropped by the epilogue).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ALL_TYPES, make_wire
from oracle.oracle import GGML_TYPE, nmse
from test_gpu_moe_decode import check_slots, moe_oracle, route
from test_gpu_moe_prefill import exact, glu_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FUSED_TYPES = ["IQ4_NL", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q4_K", "Q5_K", "IQ4_K", "IQ5_K"]
GENERIC_TYPES = ["Q6_K", "IQ4_XS", "IQ2_XXS", "IQ2_K_R4"]
UNARIES = [("silu", 0.0), ("silu", 1.5), ("gelu", 0.0), ("relu", 0.0), ("swiglu_oai", 0.0)]


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


class Experts:
    """gate and up wire bytes of every expert, uploaded merged ([gate; up] per expert) and split (two expert tensors)"""

    def __init__(self, be, oracle, name, n_expert, n_ff, k, seed, split=True):
        t = GGML_TYPE[name]
        self.name, self.n_expert, self.n_ff, self.k = name, n_expert, n_ff, k
        self.gw = [make_wire(oracle, name, n_ff, k, seed=[seed, 0, e]) for e in range(n_expert)]
        self.uw = [make_wire(oracle, name, n_ff, k, seed=[seed, 1, e]) for e in range(n_expert)]
        # rows are whole wire rows (row groups of 4 for _R4 with n_ff % 4 == 0): stacking the bytes stacks the rows
        self.M = be.set_expert_tensor(t, np.concatenate([np.concatenate([g, u]) for g, u in zip(self.gw, self.uw)]), n_expert, 2 * n_ff, k)
        self.U = be.set_expert_tensor(t, np.concatenate(self.uw), n_expert, n_ff, k) if split else None
        self.G = be.set_expert_tensor(t, np.concatenate(self.gw), n_expert, n_ff, k) if split else None


def inputs(seed, n_tokens, nb1, n_expert, n_used, k, chunk, scale=3.0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n_tokens, nb1, k)) * scale).astype(np.float32)
    return x, route(rng, n_tokens, n_expert, n_used, chunk)


def decode_oracle(oracle, ex, x, ids, unary, limit):
    """every slot: glu_ref(unary, gate_q8, up_q8, limit) on the q8_1 oracle of each half (zero rows for skipped ids)"""
    if unary == "silu" and limit == 0.0:
        return moe_oracle(oracle, ex.name, ex.uw.__getitem__, ex.gw.__getitem__, x, ids, ex.n_expert, ex.n_ff)
    up = moe_oracle(oracle, ex.name, ex.uw.__getitem__, None, x, ids, ex.n_expert, ex.n_ff)
    gate = moe_oracle(oracle, ex.name, ex.gw.__getitem__, None, x, ids, ex.n_expert, ex.n_ff)
    return glu_ref(unary, gate, up, limit)


def check_decode(be, oracle, name, n_tokens, chunk, seed):
    """all of one type's decode checks: oracle per slot and identity with the split form, nb1 = 1 and n_used"""
    n_expert, n_used, n_ff, k = 6, 4, 260, 2048
    ex = Experts(be, oracle, name, n_expert, n_ff, k, seed)
    worst = 0.0
    for nb1 in (1, n_used):
        x, ids = inputs([seed, nb1, n_tokens], n_tokens, nb1, n_expert, n_used, k, chunk)
        assert be.moe_up_gate_merged_workspace(ex.M, n_tokens, n_used, nb1) == 0, "a decode batch takes the mat-vec kernel"
        xg, ig = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
        y = be.moe_up_gate_merged(ex.M, xg, ig)
        what = f"{name} merged decode tokens={n_tokens} nb1={nb1}"
        worst = max(worst, check_slots(y.cpu().numpy(), decode_oracle(oracle, ex, x, ids, "silu", 0.0), ids, n_expert, True, what))
        ys = be.mul_mat_id(ex.U, xg, ig, gate=ex.G)
        assert torch.equal(y, ys), f"{what}: differs from the split form, max |diff| = {float((y - ys).abs().max()):.3g}"
    return worst


@pytest.mark.parametrize("name", ALL_TYPES)
def test_decode_one_token_every_type(be, oracle, name):
    print(f"{name}: max ratio to the GLU bar = {check_decode(be, oracle, name, 1, 1, GGML_TYPE[name]):.3g}")


def test_decode_token_chunks_every_type(tmp_path):
    """Five tokens walked in chunks of 2 (B200Q_MOE_CHUNK_TOKENS=2): chunks 2 + 2 + 1, every id of the second chunk skipped; all 46 types in one
    child process (the override is read once per process)."""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "chunks"], capture_output=True, text=True, cwd=ROOT, timeout=1800,
                       env={**os.environ, "B200Q_MOE_CHUNK_TOKENS": "2"})
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count(" OK") == len(ALL_TYPES)


@pytest.mark.parametrize("name", FUSED_TYPES + GENERIC_TYPES)
@pytest.mark.parametrize("nb1", [1, 2])
def test_prefill_against_exact(be, oracle, name, nb1):
    """96 tokens, 8 experts, 2 used: 192 slots > 5 per expert, the grouped GEMM; n_ff = 260 (a partial 128-row tile in each half); some ids skipped."""
    n_expert, n_used, n_ff, k, n_tokens = 8, 2, 260, 1024, 96
    ex = Experts(be, oracle, name, n_expert, n_ff, k, 900 + GGML_TYPE[name])
    rng = np.random.default_rng([GGML_TYPE[name], nb1])
    x = rng.standard_normal((n_tokens, nb1, k)).astype(np.float32)
    ids = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
    ids[::11, 1] = -1
    ids[5, 0] = n_expert
    assert be.moe_up_gate_merged_workspace(ex.M, n_tokens, n_used, nb1) > 0
    xg, ig = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
    y = be.moe_up_gate_merged(ex.M, xg, ig)
    yh = y.cpu().numpy()
    skipped = (ids < 0) | (ids >= n_expert)
    assert np.all(yh[skipped] == 0.0), "skipped slots must be zero rows"
    e = nmse(yh[~skipped], exact(oracle, name, ex.uw, ex.gw, x, ids, n_ff)[~skipped])
    print(f"{name} nb1={nb1} merged grouped: NMSE {e:.3g}")
    assert e <= 2e-4, f"{name} nb1={nb1}: NMSE {e}"
    assert torch.equal(y, be.mul_mat_id_dispatch(ex.U, xg, ig, gate=ex.G)), f"{name} nb1={nb1}: differs from the split form"


# (id, type, n_expert, n_used, n_ff, K, token counts on both sides of the crossover n_slots > 5 n_expert)
IDENTITY = [("qwen3-30b-a3b", "Q4_K", 128, 8, 768, 2048, (1, 80, 81)),
            ("mixtral-8x7b", "IQ4_NL", 8, 2, 14336, 4096, (1, 20, 21)),
            ("deepseek-v3-tp8", "IQ2_XXS", 256, 8, 256, 7168, (1, 160, 161)),
            ("n_ff-1408-fused", "IQ4_NL", 16, 4, 1408, 1024, (2, 20, 64)),
            ("n_ff-1408-generic", "Q6_K", 16, 4, 1408, 1024, (2, 20, 64)),
            ("r4", "IQ4_K_R4", 8, 2, 512, 1024, (3, 20, 96))]


@pytest.mark.parametrize("case", IDENTITY, ids=[c[0] for c in IDENTITY])
def test_bit_equal_to_split_form(be, oracle, case):
    case_id, name, n_expert, n_used, n_ff, k, tokens = case
    ex = Experts(be, oracle, name, n_expert, n_ff, k, 1300)
    t_last = 5 * n_expert // n_used
    assert min(tokens) <= t_last < max(tokens)
    for n_tokens in tokens:
        x, ids = inputs([n_ff, n_tokens], n_tokens, 1, n_expert, n_used, k, n_tokens, scale=1.0)
        grouped = be.moe_up_gate_merged_workspace(ex.M, n_tokens, n_used, 1) > 0
        assert grouped == (n_tokens > t_last)
        assert grouped == (be.mul_mat_id_workspace(ex.U, n_tokens, n_used, 1, True) > 0)
        xg, ig = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
        y = be.moe_up_gate_merged(ex.M, xg, ig)
        ys = be.mul_mat_id_dispatch(ex.U, xg, ig, gate=ex.G)
        assert torch.equal(y, ys), f"{case_id} tokens={n_tokens}: max |diff| = {float((y - ys).abs().max()):.3g}"
        skipped = (ids < 0) | (ids >= n_expert)
        assert bool((y.cpu()[torch.from_numpy(skipped)] == 0).all()), f"{case_id} tokens={n_tokens}: skipped slots must be zero rows"
        print(f"{case_id} tokens={n_tokens} ({'grouped GEMM' if grouped else 'mat-vec'}): bit-equal to the split form")


@pytest.mark.parametrize("unary,limit", UNARIES)
@pytest.mark.parametrize("name", ["Q4_K", "IQ2_XXS"])
def test_unaries(be, oracle, name, unary, limit):
    """Every GLU of the reference on both paths: 2 tokens (mat-vec) against the q8_1 oracle at the GLU bar, 96 tokens (grouped GEMM) against the
    exact product (NMSE 2e-4, 1e-3 with a limit, which clamps most outputs); both bit-equal to the split form."""
    n_expert, n_used, n_ff, k = 8, 2, 256, 1024
    ex = Experts(be, oracle, name, n_expert, n_ff, k, 1700)
    for n_tokens in (2, 96):
        x, ids = inputs([17, n_tokens], n_tokens, 1, n_expert, n_used, k, n_tokens, scale=3.0 if n_tokens == 2 else 1.0)
        xg, ig = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
        y = be.moe_up_gate_merged(ex.M, xg, ig, unary=unary, limit=limit)
        assert torch.equal(y, be.mul_mat_id_dispatch(ex.U, xg, ig, gate=ex.G, unary=unary, limit=limit)), f"{name} {unary} {limit} tokens={n_tokens}"
        yh = y.cpu().numpy()
        what = f"{name} {unary} limit={limit} tokens={n_tokens}"
        if n_tokens == 2:
            check_slots(yh, decode_oracle(oracle, ex, x, ids, unary, limit), ids, n_expert, True, what)
        else:
            ok = (ids >= 0) & (ids < n_expert)
            e = nmse(yh[ok], exact(oracle, name, ex.uw, ex.gw, x, ids, n_ff, unary, limit)[ok])
            print(f"{what}: NMSE {e:.3g}")
            assert e <= (1e-3 if limit else 2e-4), f"{what}: NMSE {e}"


@pytest.mark.parametrize("name", ["Q4_K", "IQ2_XXS"])
def test_captured_prefill_with_ids_changed_in_place(be, oracle, name):
    """Capture the merged call at a prefill batch, write new ids (some skipped) in place, replay: equal to an eager call on the new ids."""
    n_expert, n_used, n_ff, k, n_tokens = 8, 2, 256, 1024, 128
    ex = Experts(be, oracle, name, n_expert, n_ff, k, 1500, split=False)
    assert be.moe_up_gate_merged_workspace(ex.M, n_tokens, n_used, 1) > 0
    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((n_tokens, 1, k)).astype(np.float32)).cuda()

    def new_ids():
        i = np.stack([rng.permutation(n_expert)[:n_used] for _ in range(n_tokens)]).astype(np.int32)
        i[rng.choice(n_tokens, 10, replace=False), 1] = -1
        return torch.from_numpy(i).cuda()
    ids = new_ids()
    out = torch.empty((n_tokens, n_used, n_ff), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.moe_up_gate_merged(ex.M, x, ids, out=out)          # warm-up: the workspace exists before the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.moe_up_gate_merged(ex.M, x, ids, out=out)
    for _ in range(2):
        ids.copy_(new_ids())
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, be.moe_up_gate_merged(ex.M, x, ids))


def _harness(mode, tmp_path=None):
    exe = os.path.join(ROOT, "tests", "backend_ops", "test_moe_merged_backend")
    if not os.path.exists(exe):
        pytest.skip("harness not built (needs the reference headers at build time)")
    r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED: 0 failures" in r.stdout


def test_merged_node_against_the_reference_cpu_op():
    """The merged node on the unmodified reference CPU backend and on the plug, 1, 8 and 512 tokens, IQ4_NL, Q4_K, IQ2_XXS: NMSE <= 5e-4."""
    _harness("op")


def test_moe_ffn_graph_with_merged_experts_runs_on_the_plug():
    """llm_build_moe_ffn with ffn_gate_up_exps at the three model shapes, 1 ... 512 tokens, placed by ggml_backend_sched next to the CPU backend:
    the merged node runs on the plug, and it and the layer output match the same graph on the reference CPU backend (NMSE <= 5e-4)."""
    _harness("graph")


if __name__ == "__main__" and sys.argv[1] == "chunks":
    from ik_llama_cpp_b200 import backend as _be
    from oracle.oracle import Oracle
    _o = Oracle()
    assert os.environ.get("B200Q_MOE_CHUNK_TOKENS") == "2"
    for _name in ALL_TYPES:
        _r = check_decode(_be, _o, _name, 5, 2, 100 + GGML_TYPE[_name])
        print(f"{_name} 5 tokens in chunks of 2: max ratio to the GLU bar {_r:.3g} OK", flush=True)
