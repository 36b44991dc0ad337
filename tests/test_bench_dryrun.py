"""bench.py's model skeleton walked on the CPU with a stub backend: catches plumbing errors (names, argument lists, buffer shapes)
before GPU time is spent on them.  No kernels run here."""
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench


class _T:
    def __init__(self, m, k, ggml_type=20):
        self.m, self.k, self.nbytes_wire, self.ggml_type = m, k, m * k * 18 // 32, ggml_type


class _BE:
    class Q8Scratch:
        def __init__(self, k):
            self.k, self.valid = k, False

    calls = []

    def prefetch_next(self, ws, gate=None):
        assert all(hasattr(w, "m") for w in ws)

    def mul_mat(self, w, x, out=None, x_bf16=None, q8_in=None, bias=None):
        assert x.shape[1] == w.k and (out is None or out.shape[1] == w.m)
        assert bias is None or (x.shape[0] == 1 and bias.shape == (w.m,))
        self.calls.append("mul_mat"); return out

    def mul_mat_multi(self, ws, x, outs=None, x_bf16=None):
        assert all(x.shape[1] == w.k and o.shape[1] == w.m for w, o in zip(ws, outs))
        self.calls.append("multi"); return outs

    def fused_up_gate(self, up, gate, x, unary="silu", limit=0.0, out=None, x_bf16=None, out_bf16=None, q8_out=None):
        assert x.shape[1] == up.k and out.shape[1] == up.m
        self.calls.append("upgate"); return out

    def convert_activations(self, x, out=None):
        assert out.shape == x.shape
        self.calls.append("cvt"); return out


def test_model_skeleton_walks_tg_and_pp(monkeypatch):
    monkeypatch.setattr(bench, "random_planes", lambda be, torch_, name, m, k, gen, scale: _T(m, k))
    gen = types.SimpleNamespace(manual_seed=lambda s: None)
    tt = types.SimpleNamespace(Generator=lambda device=None: gen, empty=lambda s, dtype=None, device=None: torch.empty(s, dtype=dtype),
                               float32=torch.float32, bfloat16=torch.bfloat16, add=torch.add)
    be = _BE()
    m = bench.Model(be, tt, 2)
    m.alloc(1); m.step_tg()
    assert be.calls.count("multi") == 2 and be.calls.count("upgate") == 2 and be.calls.count("mul_mat") == 5
    assert m.launches_tg == 9
    be.calls.clear()
    m.alloc(512); m.step_pp()
    assert be.calls.count("cvt") == 6 and be.calls.count("mul_mat") == 5
    assert bench.model_bytes_per_token(32) == 4221370368
    # the default quantisation mix: attn_v has its own type, so it gets its own launch
    monkeypatch.setattr(bench, "random_planes", lambda be, torch_, name, m, k, gen, scale: _T(m, k, bench.MIX_TYPES[name][0]))
    be.calls.clear()
    mm = bench.Model(be, tt, 2, mix="default")
    mm.alloc(1); mm.step_tg()
    assert be.calls.count("multi") == 2 and be.calls.count("mul_mat") == 7 and mm.launches_tg == 11
    assert mm.head.ggml_type == 14 and mm.layers[0]["down"].ggml_type == 13 and mm.layers[1]["wv"].ggml_type == 140
    mm.alloc(512); mm.step_pp()


class _Reducer:
    ok = True

    def __init__(self, n):
        self.buf = torch.zeros(n)

    def reduced_view(self, n):
        return self.buf[:n]

    def all_reduce(self, t):
        pass

    def all_reduce_bf16(self, t, out_bf16=None, out_f32=None):
        pass


class _BE_TP(_BE):
    NvlsReducer = _Reducer

    def mul_mat_vec_tp(self, ws, x, outs, reducer, reduce_in=False, reduce_out=False, gate=None, unary=None):
        assert (x is None) == reduce_in and (outs is None) == reduce_out
        self.calls.append("tp")


def test_tensor_parallel_walks_dump_their_outputs(monkeypatch, tmp_path):
    """--gpus N: the fused-exchange decode walk (N = 2) and the separate-reduce walk (N = 4) both leave logits and a hidden state to dump."""
    monkeypatch.setattr(bench, "random_planes", lambda be, torch_, name, m, k, gen, scale: _T(m, k))
    for var in ("B200Q_TP_FUSED", "B200Q_NCCL_REDUCE", "B200Q_TP_BF16_REDUCE"):
        monkeypatch.delenv(var, raising=False)
    gen = types.SimpleNamespace(manual_seed=lambda s: None)
    tt = types.SimpleNamespace(Generator=lambda device=None: gen, empty=lambda s, dtype=None, device=None: torch.empty(s, dtype=dtype),
                               float32=torch.float32, bfloat16=torch.bfloat16, add=torch.add)
    for tp, fused in ((2, True), (4, False)):
        be = _BE_TP()
        be.calls = []
        m = bench.Model(be, tt, 2, tp=tp)
        assert m.fused_tp == fused and not m.residual
        dump = bench.make_dump(str(tmp_path / f"tp{tp}"), rank=1, world=tp)
        m.alloc(1); m.step_tg()
        assert be.calls.count("tp") == (9 if fused else 0)
        for k, v in m.outputs().items():
            dump(f"tg_{k}", v)
        m.alloc(512); m.step_pp()
        for k, v in m.outputs().items():
            dump(f"pp512_{k}", v)
        names = sorted(os.listdir(tmp_path / f"tp{tp}"))
        assert names == ["pp512_hidden_rank1.npy", "pp512_logits_rank1.npy", "tg_hidden_rank1.npy", "tg_logits_rank1.npy"]
