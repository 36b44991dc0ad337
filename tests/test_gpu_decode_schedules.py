"""Element-by-element tests of every decode mat-vec schedule (n <= 8).  The host plans each launch from the shape before it launches it:
  * mmvq_cols (b200q_api.cu) covers n with pieces of 8, 4, 2 and 1 columns, halving a piece while c K 1.25 bytes exceed 200 KB (b200q_mmvq_max_cols);
  * plan_mmvq (b200q_decode.cu) picks the kernel, its template arguments, grid and block of each piece: pieces of 1 or 2 columns take the
    TMA-ring kernel k_mmvq_ring<T, NCOLS, UPGATE, MULTI, PAIR, TP, Q8> (b200q_decode_ring.cuh) unless a plane
    row is not 16-byte aligned (make_ring_geom), ring_shape finds no layout with 2 stages at 11, 7 or 3 consumer warps, or a row-pair launch has an
    odd segment that is not the last; pieces of 4 or 8 columns and those fallbacks take the LDG kernel k_mmvq<T, NCOLS, UPGATE>;
  * K <= 4096: a ring unit is a pair of rows (PAIR); K > 4096: one row cut into segments of up to 256 items ("long rows"), halves of 128 items;
  * the q8 hand-off: the up/gate launch emits its result as a q8_1 image (Q8 = 2), the next launch consumes it (Q8 = 1); shapes that are not eligible
    are planned as plain launches;
  * wire-layout types take k_wire_mmvq<T, NCOLS, UPGATE> (b200q_wire.cu).
The table below names, per case, the launches it is meant to reach; each case runs once under torch.profiler in a child process of its own and the
trace must show exactly those launches (kernel, template arguments, grid, block) at 132 SMs.  On another SM count, or when the profiler records no
kernels, only that assertion is skipped: the numerical checks always run.

Reference and bars (test_gpu_parity.py, DESIGN.md §5).  yq = oracle.mul_mat_q8_1(..., variant="b200"): the same int8 activations and the same
integer block sums as the kernel, so only the f32 summation order differs.  Every element must satisfy
    plain:  |y - yq|  <= 2e-5 rms(yq)
    GLU:    |y - ref| <= 5e-5 rms(ref),  ref = glu_ref(act, gate_q, up_q)
Why the bars hold beyond K = 14336, where they were measured, up to K = 53248.  The kernels add one f32 term per item of 32 weights (an fmaf of
the activation scale with the item's scaled integer sum) into chains owned by a lane: k_mmvq and the row-pair ring keep one chain per lane and row
(n32 / 32 terms, n32 = K / 32), the long-row ring two (the two 128-item halves of each segment: n32 / 64 terms); the 32 lanes (and the two chains)
are then added in a 6-level tree.  Every addition rounds with relative error <= u = 2^-24, so an item picks up at most L + 7 roundings, L the
chain length.  With random data these errors are independent: |y - yq| ~ u sqrt(L + 7) sqrt(sum_i v_i^2), v_i the item terms, while
rms(y) ~ sqrt(sum_i v_i^2) (the items do not cancel systematically).  So the ratio err / rms grows only like sqrt(L), not with K as a whole:
at K = 53248, L = 26 (long rows) or 52 (LDG), u sqrt(L + 7) <= 4.6e-7, and the largest of 10^6 elements lies within 6 sigma: <= 2.8e-6, a
seventh of the bar.  test_f32_kernel_order_stays_inside_the_bar replays both summation orders in f32 on the oracle's own terms at that K.
The worst case without cancellation, gamma_{L+7} sum |v_i|, would exceed the bar at that K; it is not the case the data can produce.

The MoE mat-vecs (k_mmvq_id, k_wire_mmvq_id, skipped slots included) have their own table and sweep in test_gpu_moe_decode.py, which reuses the
bars, the profiler and the child-process runner of this file.  The tensor-parallel instantiations (TP = true) are covered on one GPU, every
plane type with W emulated ranks, in test_gpu_tp_decode.py; test_gpu_tp.py runs the fused exchange across real GPUs where the machine has them.
"""
import json
import os
import re
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest
import torch

from conftest import PLANE_TYPES, WIRE_TYPES, make_wire
from oracle.oracle import GGML_TYPE
from test_gpu_parity import glu_ref, rms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132
PLAIN_BAR = 2e-5
GLU_BAR = 5e-5
F32_ADD = 2.0 ** -23            # the residual add of the bias operand: one f32 rounding of the sum (half an ulp, x 2)


def bar_ratio(y, ref, bar, what):
    """max |y - ref| / (bar rms(ref)); fails with the first offending elements when any element exceeds the bound"""
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    assert y.shape == ref.shape, (what, y.shape, ref.shape)
    bound = bar * max(rms(ref), 1e-30)
    err = np.abs(y - ref)
    bad = np.argwhere(~(err <= bound))
    assert len(bad) == 0, (f"{what}: {len(bad)} of {y.size} elements outside |y - ref| <= {bar} rms(ref) = {bound:.3g}, first "
                           + ", ".join(f"{tuple(int(i) for i in b)}: y={y[tuple(b)]:.7g} ref={ref[tuple(b)]:.7g}" for b in bad[:5]))
    return float(err.max() / bound)


def plain_ratio(oracle, name, wire, x, m, y, what):
    yq = oracle.mul_mat_q8_1(GGML_TYPE[name], wire, x, m, variant="b200")
    return bar_ratio(y, yq, PLAIN_BAR, what)


def glu_ratio(oracle, name, wu, wg, x, m, y, what):
    t = GGML_TYPE[name]
    u = oracle.mul_mat_q8_1(t, wu, x, m, variant="b200").astype(np.float64)
    g = oracle.mul_mat_q8_1(t, wg, x, m, variant="b200").astype(np.float64)
    return bar_ratio(y, glu_ref("silu", g, u), GLU_BAR, what)


def check_q8_image(oracle, img, a, what):
    """The b200q_q8 image of a [1, K] vector: [K int8 q][K/32 f32 d][K/32 packed int16 sums of lanes 0-15 | 16-31][K/32 u32 arrival counters].
    Tolerance-free: q and d are those of oracle.quantize_q8_1_b200, the sums follow from q, the counters are back at zero."""
    img = np.asarray(img, np.uint8)
    k = a.shape[1]
    n32 = k // 32
    q_ref, d_ref = oracle.quantize_q8_1_b200(a)
    q_ref = np.asarray(q_ref, np.int8).reshape(-1)
    assert np.array_equal(img[:k].view(np.int8), q_ref), f"{what}: q8 image values"
    assert np.array_equal(img[k:k + 4 * n32].view(np.float32), np.asarray(d_ref, np.float32).reshape(-1)), f"{what}: q8 image scales"
    qs = q_ref.reshape(n32, 32).astype(np.int64)
    sums = ((qs[:, :16].sum(1) & 0xFFFF) | ((qs[:, 16:].sum(1) & 0xFFFF) << 16)).astype(np.uint32)
    assert np.array_equal(img[k + 4 * n32:k + 8 * n32].view(np.uint32), sums), f"{what}: q8 image block sums"
    assert not img[k + 8 * n32:k + 12 * n32].any(), f"{what}: arrival counters must be back at zero"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# CPU self-tests of the comparison (oracle and numpy only)
# ------------------------------------------------------------------------------------------------------------------------------------------------
def _fails(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def _x(n, k, seed):
    return np.random.default_rng(seed).standard_normal((n, k)).astype(np.float32)


def test_bars_catch_planted_defects(oracle):
    """The oracle's own result passes; each defect an indexing bug in a decode schedule could cause fails."""
    t = GGML_TYPE["IQ4_NL"]
    # one column of an n = 2 result shifted by one row (a wrong column stride of the 2-column ring)
    m, k = 259, 2048
    w = make_wire(oracle, "IQ4_NL", m, k, seed=1)
    x = _x(2, k, 2)
    yq = oracle.mul_mat_q8_1(t, w, x, m, variant="b200")
    bar_ratio(yq, yq, PLAIN_BAR, "clean n = 2")
    d = yq.copy(); d[1, 1:] = yq[1, :-1]
    assert _fails(lambda: bar_ratio(d, yq, PLAIN_BAR, "shifted column")), "one column shifted by one row"
    # the second half (items 128..159) of one long-row segment dropped at K = 5120
    m, k = 64, 5120
    w = make_wire(oracle, "Q4_K", m, k, seed=3)
    x = _x(1, k, 4)
    yq = oracle.mul_mat_q8_1(GGML_TYPE["Q4_K"], w, x, m, variant="b200")
    xd = x.copy(); xd[:, 4096:] = 0.0                      # q8_1 blocks are per 32 values: exactly items 128..159 contribute nothing
    d = yq.copy(); d[0, 17] = oracle.mul_mat_q8_1(GGML_TYPE["Q4_K"], w, xd, m, variant="b200")[0, 17]
    assert _fails(lambda: bar_ratio(d, yq, PLAIN_BAR, "dropped half")), "second half of one long-row segment dropped"
    # fused Q,K,V: two segments swapped, and one row taken from the neighbouring segment (a segment offset off by one)
    ms, k = [256, 64, 64], 1024
    ws = [make_wire(oracle, "IQ4_NL", mm, k, seed=10 + i) for i, mm in enumerate(ms)]
    x = _x(1, k, 5)
    ys = [oracle.mul_mat_q8_1(t, wi, x, mm, variant="b200") for wi, mm in zip(ws, ms)]
    for y in ys:
        bar_ratio(y, y, PLAIN_BAR, "clean segment")
    assert _fails(lambda: [bar_ratio(got, ref, PLAIN_BAR, "swapped") for got, ref in zip([ys[0], ys[2], ys[1]], ys)]), "two segments swapped"
    d = ys[1].copy(); d[0, 0] = ys[0][0, -1]
    assert _fails(lambda: bar_ratio(d, ys[1], PLAIN_BAR, "neighbour row")), "one row of a multi launch from the neighbouring segment"


def _kernel_order_f32(wd, q, d8, long_rows):
    """The mat-vec sum of the oracle's own item terms in float32, in a kernel's order: item it goes to lane it % 32; long rows: the two 128-item
    halves of each 256-item segment are two chains of the lane, added before the butterfly; otherwise one chain per lane (k_mmvq, row pairs).
    Each step is an fmaf (d8 * t + acc, one rounding); then the xor butterfly over the 32 lanes in float32."""
    m, k = wd.shape
    n32 = k // 32
    t = (wd.reshape(m, n32, 32).astype(np.float64) * q.reshape(n32, 32)).sum(2).astype(np.float32)       # dl * (integer sum): one rounding
    acc = np.zeros((m, 32, 2), np.float32)
    for it in range(n32):
        c = 1 if long_rows and it % 256 >= 128 else 0
        acc[:, it % 32, c] = (acc[:, it % 32, c].astype(np.float64) + np.float64(d8[it]) * t[:, it].astype(np.float64)).astype(np.float32)
    v = acc[:, :, 0] + acc[:, :, 1]
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, np.arange(32) ^ o]
    return v[:, 0]


def test_f32_kernel_order_stays_inside_the_bar(oracle):
    """K = 53248 (Llama-405B ffn_down), both summation orders of the kernels in float32 on the oracle's terms: the largest error stays far inside
    the plain bar, as derived in the module docstring."""
    t = GGML_TYPE["IQ4_NL"]
    m, k = 256, 53248
    w = make_wire(oracle, "IQ4_NL", m, k, seed=7)
    x = _x(1, k, 8)
    wd = oracle.dequantize(t, w, m, k)
    q, d = oracle.quantize_q8_1_b200(x)
    yq = oracle.mul_mat_q8_1(t, w, x, m, variant="b200")[0]
    for long_rows in (True, False):
        y = _kernel_order_f32(wd, q[0].astype(np.float64), d[0].astype(np.float32), long_rows)
        r = bar_ratio(y, yq, PLAIN_BAR, f"f32 kernel order (long rows {long_rows})")
        print(f"f32 kernel order K={k} long_rows={long_rows}: max |y - yq| / (2e-5 rms) = {r:.3g}")
        assert r <= 0.25


# ------------------------------------------------------------------------------------------------------------------------------------------------
# schedule table
# ------------------------------------------------------------------------------------------------------------------------------------------------
T = {name: str(GGML_TYPE[name]) for name in GGML_TYPE}
B = {True: "true", False: "false"}


def ring(name, ncols, upgate, multi, pair, q8, grid, block):
    return ("k_mmvq_ring", (T[name], str(ncols), B[upgate], B[multi], B[pair], "false", str(q8)), (grid, 1, 1), (block, 1, 1))


def ldg(name, ncols, upgate, grid, block):
    return ("k_mmvq", (T[name], str(ncols), B[upgate]), (grid, 1, 1), (block, 1, 1))


def wire(name, ncols, upgate, grid):
    return ("k_wire_mmvq", (T[name], str(ncols), B[upgate]), (grid, 1, 1), (256, 1, 1))


def gemm_q(name, grid):
    return ("k_gemm_q", (T[name], "0", "false"), grid, (288, 1, 1))


def gemm_bf16(grid):
    return ("k_gemm_bf16", ("128", "false"), grid, (288, 1, 1))


# Derivations at 132 SMs.  Ring: units = row pairs ceil(M / 2) (K <= 4096) or rows (K > 4096); xbytes = ncols K 1.25 + 1408;
# S = (112 KiB - xbytes - 64) / (ncw (2 stage + 16)) at ncw = 11, then 7, then 3 consumer warps until S >= 2; ncw then drops to 7 (3) while
# units <= 132 x 7 (3); grid = min(ceil(units / ncw), 264), block = 32 (ncw + 1).  LDG: 16 warps, halved while M <= 132 x warps / 2;
# grid = min(ceil(M / warps), 132).  Wire: 8 warps, grid = min(ceil(M / 8), 132 x (4, 2 or 1 by shared memory: <= 48 KB, <= 100 KB, more)).
# Calls: ("mm", tensor, n) mul_mat; ("mm_strided", tensor, n) the same on x[:, :K] of an [n, K + 64] tensor; ("ug", (up, gate), n) fused_up_gate;
# ("multi", tensors, n) mul_mat_multi; ("q8", (up, gate, down), hand-off expected) fused_up_gate(q8_out) -> mul_mat(down, q8_in), n = 1.
# (id, type, tensor shapes (M, K), calls, launches at 132 SMs)
SCHEDULES = [
    # ---- long rows ----
    ("long-plain-k5120-one-partial-segment", "IQ4_NL", [(1000, 5120)], [("mm", 0, 1)],
     # 160 items = one segment, halves 128 + 32; stage 2304 B, xbytes 7808: S = 2 at 11 warps; 1000 units / 11
     [ring("IQ4_NL", 1, False, False, False, 0, 91, 384)]),
    ("long-plain-k14336-two-segments-q2k", "Q2_K", [(1000, 14336)], [("mm", 0, 1)],
     # 448 items = segments 256 + 192; stage 1408 B, xbytes 19328: S = 3 at 11 warps; 1000 / 11
     [ring("Q2_K", 1, False, False, False, 0, 91, 384)]),
    ("long-ncols2-k14336-q6k", "Q6_K", [(1000, 14336)], [("mm", 0, 2)],
     # d plane aligned (K % 2048 == 0); stage 3456 B, xbytes 37248: S = 1 at 11 and 7 warps, S = 3 at 3 warps; 1000 / 3 -> 264
     [ring("Q6_K", 2, False, False, False, 0, 264, 128)]),
    ("long-upgate-n1-k8192-q4k", "Q4_K", [(1024, 8192), (1024, 8192)], [("ug", (0, 1), 1)],
     # stage 2304 B, xbytes 11648: S = 2 at 11 warps; 1024 / 11
     [ring("Q4_K", 1, True, False, False, 0, 94, 384)]),
    ("long-upgate-n2-k8192-q3k", "Q3_K", [(1024, 8192), (1024, 8192)], [("ug", (0, 1), 2)],
     # stage 1792 B, xbytes 21888: S = 2 at 11 warps; 1024 / 11
     [ring("Q3_K", 2, True, False, False, 0, 94, 384)]),
    ("long-multi-k5120-odd-last-segment", "IQ4_NL", [(5120, 5120), (1024, 5120), (1023, 5120)], [("multi", (0, 1, 2), 1)],
     # one row per unit, so an odd segment is allowed; 7167 units / 11 -> 264
     [ring("IQ4_NL", 1, False, True, False, 0, 264, 384)]),
    # ---- q8 hand-off ----
    ("q8-llama-iq4nl", "IQ4_NL", [(14336, 4096), (14336, 4096), (4096, 14336)], [("q8", (0, 1, 2), True)],
     # up/gate: row pairs, merged stage 4608 B, S = 2 at 11 warps, 7168 units -> 264; ffn_down: long rows, S = 1 at 11 warps, S = 2 at 7; 4096 / 7 -> 264
     [ring("IQ4_NL", 1, True, False, True, 2, 264, 384), ring("IQ4_NL", 1, False, False, False, 1, 264, 256)]),
    ("q8-llama-q5k", "Q5_K", [(14336, 4096), (14336, 4096), (4096, 14336)], [("q8", (0, 1, 2), True)],
     # up/gate: merged stage 5632 B: S = 1 at 11 warps, S = 2 at 7; 7168 / 7 -> 264; ffn_down: stage 2816 B: S = 2 at 7 warps; 4096 / 7 -> 264
     [ring("Q5_K", 1, True, False, True, 2, 264, 256), ring("Q5_K", 1, False, False, False, 1, 264, 256)]),
    ("q8-out-long-rows-q4k", "Q4_K", [(2048, 8192), (2048, 8192), (512, 2048)], [("q8", (0, 1, 2), True)],
     # up/gate K = 8192: long rows, S = 2 at 11 warps, 2048 / 11 = 187; ffn_down K = 2048: 256 pairs <= 132 x 3 -> 3 warps, 86
     [ring("Q4_K", 1, True, False, False, 2, 187, 384), ring("Q4_K", 1, False, False, True, 1, 86, 128)]),
    ("q8-out-ineligible-m-not-64", "IQ4_NL", [(1056, 1024), (1056, 1024), (256, 1056)], [("q8", (0, 1, 2), False)],
     # M % 64 = 32: plain up/gate, 528 pairs <= 924 -> 7 warps, 76; ffn_down K = 1056: 528-byte rows are not 16-byte aligned -> LDG, 256 rows -> 2 warps
     [ring("IQ4_NL", 1, True, False, True, 0, 76, 256), ldg("IQ4_NL", 1, False, 128, 64)]),
    ("q8-in-ineligible-q6k-k3072", "Q6_K", [(3072, 2048), (3072, 2048), (512, 3072)], [("q8", (0, 1, 2), True)],
     # up/gate: stage 3456 B, S = 2 at 7 warps, 1536 / 7 = 220; ffn_down: the d plane is not aligned (3072 % 2048) -> LDG, 512 rows -> 4 warps
     [ring("Q6_K", 1, True, False, True, 2, 220, 256), ldg("Q6_K", 1, False, 128, 128)]),
    # ---- LDG fallbacks ----
    ("ldg-q6k-k5120", "Q6_K", [(1000, 5120)], [("mm", 0, 1)],
     [ldg("Q6_K", 1, False, 125, 256)]),                     # d plane not aligned (5120 % 2048); 1000 rows -> 8 warps
    ("ldg-q4_0-k4128", "Q4_0", [(1000, 4128)], [("mm", 0, 1)],
     [ldg("Q4_0", 1, False, 125, 256)]),                     # 129 items: 2064-byte qs rows, not 16-byte aligned
    ("ldg-multi-odd-non-last-segment", "IQ4_NL", [(511, 1024), (128, 1024), (130, 1024)], [("multi", (0, 1, 2), 1)],
     [ldg("IQ4_NL", 1, False, 97, 256)]),                    # a row pair would straddle two tensors; 769 rows -> 8 warps
    # ---- column pieces ----
    ("pieces-n6", "IQ4_NL", [(1000, 4096)], [("mm", 0, 6)],
     # 4 + 2: LDG (8 warps), then the 2-column ring (500 pairs <= 924 -> 7 warps, 72)
     [ldg("IQ4_NL", 4, False, 125, 256), ring("IQ4_NL", 2, False, False, True, 0, 72, 256)]),
    ("pieces-n7", "Q4_K", [(1000, 4096)], [("mm", 0, 7)],
     [ldg("Q4_K", 4, False, 125, 256), ring("Q4_K", 2, False, False, True, 0, 72, 256), ring("Q4_K", 1, False, False, True, 0, 72, 256)]),
    ("pieces-n8-k28672-two-ldg-4", "IQ4_NL", [(512, 28672)], [("mm", 0, 8)],
     # 8 x 28672 x 1.25 > 200 KB: two 4-column pieces; 512 rows -> 4 warps
     [ldg("IQ4_NL", 4, False, 128, 128), ldg("IQ4_NL", 4, False, 128, 128)]),
    ("long-n1-k28672-four-segments", "IQ4_NL", [(1024, 28672)], [("mm", 0, 1)],
     # 896 items = 3 x 256 + 128 (an empty second half); xbytes 37248: S = 1 at 11 warps, S = 2 at 7; 1024 / 7
     [ring("IQ4_NL", 1, False, False, False, 0, 147, 256)]),
    ("long-n1-k53248-three-warps", "IQ4_NL", [(1024, 53248)], [("mm", 0, 1)],
     # xbytes 67968: S = 0 at 11, 1 at 7, 3 at 3 warps; 1024 / 3 -> 264
     [ring("IQ4_NL", 1, False, False, False, 0, 264, 128)]),
    ("ldg-n2-k53248-ring-does-not-fit", "IQ4_NL", [(1024, 53248)], [("mm", 0, 2)],
     [ldg("IQ4_NL", 2, False, 128, 256)]),                   # xbytes 134528 > 112 KiB: no ring; 1024 rows -> 8 warps
    # ---- small M: mostly empty CTAs, a last pair with one row ----
    ("small-m-1-2-3", "IQ4_NL", [(1, 2048), (2, 2048), (3, 2048)], [("mm", 0, 1), ("mm", 1, 1), ("mm", 2, 1), ("mm", 2, 2)],
     # 1, 1, 2, 2 pairs <= 132 x 3 -> 3 warps, one CTA
     [ring("IQ4_NL", 1, False, False, True, 0, 1, 128)] * 3 + [ring("IQ4_NL", 2, False, False, True, 0, 1, 128)]),
    # ---- row-strided activations ----
    ("strided-x-n1-n2-n5", "Q4_K", [(1000, 4096)], [("mm_strided", 0, 1), ("mm_strided", 0, 2), ("mm_strided", 0, 5)],
     [ring("Q4_K", 1, False, False, True, 0, 72, 256), ring("Q4_K", 2, False, False, True, 0, 72, 256),
      ldg("Q4_K", 4, False, 125, 256), ring("Q4_K", 1, False, False, True, 0, 72, 256)]),
    # ---- the n = 8 / n = 9 boundary: mat-vec below, prefill GEMM above (k_gemm_q: split 4 of 16 raw blocks, test_gpu_gemm_schedules.py) ----
    ("boundary-n8-n9-fused-type", "IQ4_NL", [(4096, 4096)], [("mm", 0, 8), ("mm", 0, 9)],
     [ldg("IQ4_NL", 8, False, 132, 512), gemm_q("IQ4_NL", (32, 1, 4))]),
    ("boundary-n8-n9-generic-type", "Q6_K", [(4096, 4096)], [("mm", 0, 8), ("mm", 0, 9)],
     [ldg("Q6_K", 8, False, 132, 512), gemm_bf16((32, 1, 4))]),        # bf16 path: 32 tiles, split doubled while 2 x 32 x split <= 132
]
# ---- wire types at K = 7168: plain n = 1, 2, 5 (4 + 1), 8, then up/gate n = 1; 2176 rows / 8 = 272, n = 8 (70 KB) capped at 264 ----
for _name in ("IQ2_XXS", "IQ4_KT", "IQ1_S_R4"):
    SCHEDULES.append((f"wire-k7168-{_name.lower()}", _name, [(2176, 7168), (2176, 7168)],
                      [("mm", 0, 1), ("mm", 0, 2), ("mm", 0, 5), ("mm", 0, 8), ("ug", (0, 1), 1)],
                      [wire(_name, 1, False, 272), wire(_name, 2, False, 272), wire(_name, 4, False, 272), wire(_name, 1, False, 272),
                       wire(_name, 8, False, 264), wire(_name, 1, True, 272)]))

KERNEL_RE = re.compile(r"\b(k_mmvq_ring|k_mmvq_id|k_mmvq|k_wire_mmvq_id|k_wire_mmvq|k_gemm_q|k_gemm_bf16)<([^<>]*)>")


def matmul_launches(kernels):
    """(kernel, template arguments, grid, block) of the mat-vec / GEMM launches among the profiled kernels, in launch order"""
    out = []
    for name, grid, block in kernels:
        m = KERNEL_RE.search(name)
        if m:
            args = tuple(re.sub(r"^\((?:int|bool)\)", "", s.strip()) for s in m.group(2).split(","))
            out.append((m.group(1), args, tuple(grid), tuple(block)))
    return out


def profiled(fn):
    """Run fn once under torch.profiler with CUDA activities: (its result, [(kernel name, grid, block)] of every kernel it launched)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    return out, [(e["name"], tuple(e.get("args", {}).get("grid", ())), tuple(e.get("args", {}).get("block", ()))) for e in events if e.get("cat") == "kernel"]


def assert_schedule(case_id, expected, got):
    """Called after the numerical checks with the child's record: only the configuration assertion is skipped where it cannot hold."""
    if got["sms"] != H100_SMS:
        pytest.skip(f"{case_id}: configuration table is for {H100_SMS} SMs, this device has {got['sms']} (numerical checks passed)")
    if not got["any_kernel"]:
        pytest.skip(f"{case_id}: the profiler recorded no kernel events (CUPTI unavailable?); configuration not checked (numerical checks passed)")
    launched = [(g[0], tuple(g[1]), tuple(g[2]), tuple(g[3])) for g in got["launches"]]
    want = [(e[0], tuple(e[1]), tuple(e[2]), tuple(e[3])) for e in expected]
    assert launched == want, f"{case_id}: expected launches\n  {want}\nlaunched\n  {launched}"


def case_operands(oracle, case):
    """Wire bytes of every tensor and the activations of every call (seeded by the case id)"""
    case_id, name, shapes, calls, _ = case
    seed = zlib.crc32(case_id.encode()) % 100000
    wires = [make_wire(oracle, name, m, k, seed=seed + j) for j, (m, k) in enumerate(shapes)]
    xs = []
    for i, c in enumerate(calls):
        j = c[1] if isinstance(c[1], int) else c[1][0]
        n = 1 if c[0] == "q8" else c[2]
        xs.append(np.random.default_rng(seed + 100 + i).standard_normal((n, shapes[j][1])).astype(np.float32) * (3.0 if c[0] in ("ug", "q8") else 1.0))
    return wires, xs


def run_calls(be, case, wires, xs):
    """Upload the case's tensors, then (profiled by the caller) run its calls: returns fn() -> list of per-call output lists, and the q8 scratch"""
    _, name, shapes, calls, _ = case
    t = GGML_TYPE[name]
    ws = [be.set_tensor(t, w, m, k) for w, (m, k) in zip(wires, shapes)]
    xg = []
    for c, x in zip(calls, xs):
        if c[0] == "mm_strided":                # x = [:, :K] view of an [n, K + 64] tensor whose padding must never be read
            full = np.full((x.shape[0], x.shape[1] + 64), 1e4, np.float32)
            full[:, :x.shape[1]] = x
            xg.append(torch.from_numpy(full).cuda()[:, :x.shape[1]])
        else:
            xg.append(torch.from_numpy(x).cuda())
    q8 = [be.Q8Scratch(shapes[c[1][0]][0]) if c[0] == "q8" else None for c in calls]
    torch.cuda.synchronize()

    def fn():
        outs = []
        for c, x, s in zip(calls, xg, q8):
            op = c[0]
            if op in ("mm", "mm_strided"):
                outs.append([be.mul_mat(ws[c[1]], x)])
            elif op == "ug":
                outs.append([be.fused_up_gate(ws[c[1][0]], ws[c[1][1]], x, "silu")])
            elif op == "multi":
                outs.append(be.mul_mat_multi([ws[j] for j in c[1]], x))
            else:
                a = be.fused_up_gate(ws[c[1][0]], ws[c[1][1]], x, "silu", q8_out=s)
                outs.append([a, be.mul_mat(ws[c[1][2]], a, q8_in=s)])
        return outs
    return fn, q8


def _child(case_id, out_dir):
    """One case in a process of its own (in a long-lived process the profiler sometimes returns the launches without the kernel records)."""
    from oracle.oracle import Oracle
    from ik_llama_cpp_b200 import backend
    oracle = Oracle()
    case = next(c for c in SCHEDULES if c[0] == case_id)
    wires, xs = case_operands(oracle, case)
    fn, q8 = run_calls(backend, case, wires, xs)
    outs, kernels = profiled(fn)
    arrays = {f"y{i}_{j}": o.cpu().numpy() for i, os_ in enumerate(outs) for j, o in enumerate(os_)}
    for i, s in enumerate(q8):
        if s is not None:
            arrays[f"q8img{i}"] = s.buf.cpu().numpy()
    np.savez(os.path.join(out_dir, "y.npz"), **arrays)
    with open(os.path.join(out_dir, "launches.json"), "w") as f:
        json.dump({"any_kernel": bool(kernels), "launches": matmul_launches(kernels), "q8_valid": [None if s is None else bool(s.valid) for s in q8],
                   "sms": torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count}, f)


def run_child(case_id, out_dir, script=__file__, env=None):
    """Run `script <case_id> <out_dir>` (a test module whose __main__ writes y.npz and launches.json there), with `env` added to the environment."""
    r = subprocess.run([sys.executable, os.path.abspath(script), case_id, str(out_dir)], capture_output=True, text=True,
                       env={**os.environ, **(env or {})}, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    with open(os.path.join(out_dir, "launches.json")) as f:
        got = json.load(f)
    z = np.load(os.path.join(out_dir, "y.npz"))
    return {k: z[k] for k in z.files}, got


def check_calls(oracle, case, wires, xs, ys, q8_valid):
    """Every output element of every call against the oracle; returns [(what, ratio)]"""
    case_id, name, shapes, calls, _ = case
    from test_gpu_gemm_schedules import check_dense
    ratios = []
    for i, (c, x) in enumerate(zip(calls, xs)):
        op = c[0]
        what = f"{case_id} call {i} {op}"
        if op in ("mm", "mm_strided"):
            j = c[1]
            if x.shape[0] > 8:
                ratios.append((f"{what} n={x.shape[0]} (GEMM, |y - ref| / (tau A))", check_dense(oracle, what, name, wires[j], x, shapes[j][0], ys[f"y{i}_0"])))
            else:
                ratios.append((f"{what} n={x.shape[0]}", plain_ratio(oracle, name, wires[j], x, shapes[j][0], ys[f"y{i}_0"], what)))
        elif op == "ug":
            u, g = c[1]
            ratios.append((f"{what} n={x.shape[0]} (GLU)", glu_ratio(oracle, name, wires[u], wires[g], x, shapes[u][0], ys[f"y{i}_0"], what)))
        elif op == "multi":
            for s, j in enumerate(c[1]):
                ratios.append((f"{what} n={x.shape[0]} segment {s}", plain_ratio(oracle, name, wires[j], x, shapes[j][0], ys[f"y{i}_{s}"], f"{what} segment {s}")))
        else:
            u, g, dn = c[1]
            assert q8_valid[i] == c[2], f"{what}: Q8Scratch.valid = {q8_valid[i]}, expected {c[2]}"
            a = ys[f"y{i}_0"]
            ratios.append((f"{what} up/gate (GLU)", glu_ratio(oracle, name, wires[u], wires[g], x, shapes[u][0], a, f"{what} up/gate")))
            ratios.append((f"{what} ffn_down", plain_ratio(oracle, name, wires[dn], a, shapes[dn][0], ys[f"y{i}_1"], f"{what} ffn_down")))
            if c[2]:
                check_q8_image(oracle, ys[f"q8img{i}"], a, what)
    return ratios


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ik_llama_cpp_b200 import backend
    return backend


@pytest.mark.gpu
@pytest.mark.parametrize("case", SCHEDULES, ids=[c[0] for c in SCHEDULES])
def test_decode_schedule(be, oracle, tmp_path, case):
    ys, got = run_child(case[0], tmp_path)
    wires, xs = case_operands(oracle, case)
    for what, r in check_calls(oracle, case, wires, xs, ys, got["q8_valid"]):
        print(f"{what}: max ratio to the bar = {r:.3g}")
    assert_schedule(case[0], case[4], got)


@pytest.mark.gpu
def test_k_past_the_shared_memory_cap(be, oracle):
    """K = 163840 is the longest row one activation column fits (K + K/4 bytes = 200 KB): LDG kernel, equal to the oracle.  One block more raises
    the documented shape error before anything is launched (the output keeps its NaN sentinel)."""
    t = GGML_TYPE["IQ4_NL"]
    m = 64
    k = 163840
    w = make_wire(oracle, "IQ4_NL", m, k, seed=91)
    x = _x(1, k, 92)
    y = be.mul_mat(be.set_tensor(t, w, m, k), torch.from_numpy(x).cuda()).cpu().numpy()
    print(f"K={k}: max ratio to the bar = {plain_ratio(oracle, 'IQ4_NL', w, x, m, y, 'K = 163840'):.3g}")
    k = 164096
    w = make_wire(oracle, "IQ4_NL", m, k, seed=93)
    wt = be.set_tensor(t, w, m, k)
    out = torch.full((1, m), float("nan"), device="cuda")
    with pytest.raises(be.B200QError, match="too large for the mat-vec kernel"):
        be.mul_mat(wt, torch.from_numpy(_x(1, k, 94)).cuda(), out=out)
    torch.cuda.synchronize()
    assert torch.isnan(out).all(), "nothing may be written when the shape is refused"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# broad numerical sweep (in-process)
# ------------------------------------------------------------------------------------------------------------------------------------------------
SWEEP_SEGMENTS = [258, 64, 33]          # even non-last segments: the row-pair ring takes the multi launch too


@pytest.mark.gpu
@pytest.mark.parametrize("name", PLANE_TYPES)
def test_plane_type_sweep(be, oracle, name):
    """Every plane-layout type at K = 2048 (row pairs), 5120 (long rows, one partial segment) and 14336 (two segments), IQ2_BN also at 4160 (a
    second half of 2 items): plain n = 1, 2, 3, 8 with a ragged M; up/gate n = 1, 2; fused Q,K,V (three segments) n = 1, 2."""
    t = GGML_TYPE[name]
    m = 259
    worst = {}
    for k in (2048, 5120, 14336) + ((4160,) if name == "IQ2_BN" else ()):
        seed = 1000 * t + k % 997
        w = make_wire(oracle, name, m, k, seed=seed)
        wt = be.set_tensor(t, w, m, k)
        for n in (1, 2, 3, 8):
            x = _x(n, k, seed + n)
            r = plain_ratio(oracle, name, w, x, m, be.mul_mat(wt, torch.from_numpy(x).cuda()).cpu().numpy(), f"{name} K={k} n={n}")
            worst[("plain", k)] = max(worst.get(("plain", k), 0.0), r)
        wg = make_wire(oracle, name, m, k, seed=seed + 50)
        gt = be.set_tensor(t, wg, m, k)
        for n in (1, 2):
            x = _x(n, k, seed + 60 + n) * 3
            r = glu_ratio(oracle, name, w, wg, x, m, be.fused_up_gate(wt, gt, torch.from_numpy(x).cuda(), "silu").cpu().numpy(), f"{name} K={k} up/gate n={n}")
            worst[("up/gate", k)] = max(worst.get(("up/gate", k), 0.0), r)
        sw = [make_wire(oracle, name, ms, k, seed=seed + 70 + i) for i, ms in enumerate(SWEEP_SEGMENTS)]
        st = [be.set_tensor(t, s, ms, k) for s, ms in zip(sw, SWEEP_SEGMENTS)]
        for n in (1, 2):
            x = _x(n, k, seed + 80 + n)
            outs = be.mul_mat_multi(st, torch.from_numpy(x).cuda())
            for i, (s, ms, o) in enumerate(zip(sw, SWEEP_SEGMENTS, outs)):
                r = plain_ratio(oracle, name, s, x, ms, o.cpu().numpy(), f"{name} K={k} multi n={n} segment {i}")
                worst[("multi", k)] = max(worst.get(("multi", k), 0.0), r)
    for (mode, k), r in sorted(worst.items()):
        print(f"{name} {mode} K={k}: max ratio to the bar = {r:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", WIRE_TYPES)
def test_wire_type_sweep(be, oracle, name):
    """Every wire-layout type at K = 2048 and 7168, n = 1, 2, 5 (M = 260: the _R4 repacks come in groups of 4 rows)."""
    t = GGML_TYPE[name]
    m = 260
    for k in (2048, 7168):
        w = make_wire(oracle, name, m, k, seed=2000 + t + k % 997)
        wt = be.set_tensor(t, w, m, k)
        for n in (1, 2, 5):
            x = _x(n, k, 3000 + n + k)
            r = plain_ratio(oracle, name, w, x, m, be.mul_mat(wt, torch.from_numpy(x).cuda()).cpu().numpy(), f"{name} K={k} n={n}")
            print(f"{name} K={k} n={n}: max ratio to the bar = {r:.3g}")


# ------------------------------------------------------------------------------------------------------------------------------------------------
# identities that need no tolerance
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,m_ff,k", [("IQ4_NL", 14336, 4096), ("Q5_K", 14336, 4096), ("Q4_K", 2048, 8192)])
def test_q8_handoff_image(be, oracle, name, m_ff, k):
    """The q8 image the up/gate launch emits (row pairs at the Llama shape; long rows at K = 8192) equals oracle.quantize_q8_1_b200 of its result,
    with the arrival counters back at zero, three launches in a row; ffn_down on the image equals ffn_down re-quantising per CTA, bit for bit."""
    t = GGML_TYPE[name]
    wu, wg, wd = (make_wire(oracle, name, m_ff, k, seed=41), make_wire(oracle, name, m_ff, k, seed=42), make_wire(oracle, name, 1024, m_ff, seed=43))
    up, gate, down = be.set_tensor(t, wu, m_ff, k), be.set_tensor(t, wg, m_ff, k), be.set_tensor(t, wd, 1024, m_ff)
    q8 = be.Q8Scratch(m_ff)
    for it in range(3):
        x = _x(1, k, 44 + it) * 3
        a = be.fused_up_gate(up, gate, torch.from_numpy(x).cuda(), "silu", q8_out=q8)
        assert q8.valid, "eligible shape: the hand-off must be taken"
        y = be.mul_mat(down, a, q8_in=q8)
        assert torch.equal(y, be.mul_mat(down, a)), f"iteration {it}: ffn_down on the image differs from the re-quantising launch"
        check_q8_image(oracle, q8.buf.cpu().numpy(), a.cpu().numpy(), f"{name} iteration {it}")
    print(f"{name} {m_ff}x{k}: up/gate ratio {glu_ratio(oracle, name, wu, wg, x, m_ff, a.cpu().numpy(), name):.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", [("IQ4_NL", 2048), ("Q4_K", 5120), ("IQ5_K", 14336)])
def test_multi_segment_equals_single_launch(be, oracle, name, k):
    """A segment of a fused Q,K,V launch is the single launch of that tensor, bit for bit, in the same mode (row pairs at K = 2048: the segments
    start at even rows, so every pair of the multi launch is a pair of the single launch; long rows: one row per unit).  In k_mmvq_ring a row's
    arithmetic depends only on its own unit: lane l owns items l + 32 i of the stage, the chains and the butterfly are the same whichever tensor
    the unit belongs to, and the activations are quantised from the same x."""
    t = GGML_TYPE[name]
    ws = [be.set_tensor(t, make_wire(oracle, name, m, k, seed=60 + i), m, k) for i, m in enumerate(SWEEP_SEGMENTS)]
    for n in (1, 2):
        x = torch.from_numpy(_x(n, k, 61 + n)).cuda()
        for i, (w, o) in enumerate(zip(ws, be.mul_mat_multi(ws, x))):
            assert torch.equal(o, be.mul_mat(w, x)), f"{name} K={k} n={n}: segment {i}"


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", [("IQ4_NL", 2048), ("Q6_K", 14336), ("Q4_K", 8192)])
def test_two_column_ring_equals_one_column(be, oracle, name, k):
    """Column j of a 2-column ring launch is the 1-column launch on x[j], bit for bit, plain and up/gate: item_dot keeps one accumulator per column
    with the same fmaf order, the per-column quantisation reads only that column, and PAIR depends on K alone."""
    t = GGML_TYPE[name]
    m = 515
    w, g = be.set_tensor(t, make_wire(oracle, name, m, k, seed=70), m, k), be.set_tensor(t, make_wire(oracle, name, m, k, seed=71), m, k)
    x = torch.from_numpy(_x(2, k, 72)).cuda()
    y2, u2 = be.mul_mat(w, x), be.fused_up_gate(w, g, x, "silu")
    for j in range(2):
        assert torch.equal(y2[j:j + 1], be.mul_mat(w, x[j:j + 1])), f"{name} K={k}: column {j}"
        assert torch.equal(u2[j:j + 1], be.fused_up_gate(w, g, x[j:j + 1], "silu")), f"{name} K={k}: up/gate column {j}"


def _set_option(key, value):
    import ik_llama_cpp_b200 as pkg
    assert pkg.lib().b200q_set_option(key.encode(), int(value)) == 0


@pytest.mark.gpu
def test_pdl_and_prefetch_do_not_change_results(be, oracle):
    """One Llama-3-8B layer as the decode chain runs it (Q,K,V -> wo -> up/gate with the q8 hand-off -> ffn_down with the residual as bias), each
    launch after a prefetch_next hint for the launch after it: the small Q,K,V (whole tensors) and the large up + gate (the first stages of every
    CTA).  The results are bit-identical with PDL on and off, and with the prefetch on and off."""
    t = GGML_TYPE["IQ4_NL"]
    mk = lambda m, k, s: be.set_tensor(t, make_wire(oracle, "IQ4_NL", m, k, seed=s), m, k)
    wq, wk, wv, wo = mk(4096, 4096, 80), mk(1024, 4096, 81), mk(1024, 4096, 82), mk(4096, 4096, 83)
    up, gate, down = mk(14336, 4096, 84), mk(14336, 4096, 85), mk(4096, 14336, 86)
    x = torch.from_numpy(_x(1, 4096, 87)).cuda()
    q8 = be.Q8Scratch(14336)

    def chain():
        be.prefetch_next([wo])
        q, _, _ = be.mul_mat_multi([wq, wk, wv], x)
        be.prefetch_next([up], gate=gate)
        h = be.mul_mat(wo, q)
        be.prefetch_next([down])
        a = be.fused_up_gate(up, gate, h, "silu", q8_out=q8)
        be.prefetch_next([wq, wk, wv])
        y = be.mul_mat(down, a, q8_in=q8, bias=x[0])
        torch.cuda.synchronize()
        return [v.clone() for v in (q, h, a, y)]
    pdl0 = int(os.environ.get("B200Q_PDL", "1"))
    pf0 = int(os.environ.get("B200Q_PREFETCH_NEXT", "0"))
    results = {}
    try:
        for pdl in (1, 0):
            for pf in (0, 1):
                _set_option("pdl", pdl)
                _set_option("prefetch_next", pf)
                results[(pdl, pf)] = chain()
    finally:
        _set_option("pdl", pdl0)
        _set_option("prefetch_next", pf0)
    base = results[(1, 0)]
    for key, r in results.items():
        for what, a, b in zip(("q", "h", "a", "ffn_down + residual"), base, r):
            assert torch.equal(a, b), f"pdl={key[0]} prefetch_next={key[1]}: {what} differs"


# ------------------------------------------------------------------------------------------------------------------------------------------------
# the decode chain as bench.py times it
# ------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["pure", "default"])
def test_bench_decode_chain(be, oracle, mix):
    """bench.Model (2 layers) captured in a CUDA graph as time_graph does it (PDL, q8 hand-off, the residual as bias operand, ping-pong residual
    buffers, re-armed arrival counters), replayed 3 times with new inputs: after each replay every launch of the last layer is checked against the
    oracle on the input it read, the head on a sample of 2048 rows.  The default mix adds the IQ5_K attn_v launch, the Q5_K ffn_down with the
    hand-off and the Q6_K head.  Finally the step run eagerly with PDL off is bit-identical to the replay."""
    import bench
    model = bench.Model(be, torch, n_layer=2, mix=mix)
    model.alloc(1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            model.step_tg()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        model.step_tg()
    L = model.layers[-1]
    wires = {key: be.get_tensor(L[key]) for key in ("wq", "wk", "wv", "wo", "up", "gate", "down")}
    tname = {key: L[key].ggml_type for key in wires}
    head = model.head
    rows = np.sort(np.random.default_rng(5).choice(head.m, 2048, replace=False))
    hw = be.get_tensor(head).reshape(head.m, -1)[rows]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(99)

    def snapshot():
        torch.cuda.synchronize()
        names = ("res0", "q", "kk", "v", "h", "a", "res1", "logits", "q8")
        return dict(zip(names, (b.cpu().numpy() for b in (model.res[0], model.q, model.kk, model.v, model.h, model.a, model.res[1], model.logits, model.q8a.buf))))

    def q8_(key, x, m):
        return oracle.mul_mat_q8_1(tname[key], wires[key], x, m, variant="b200")
    for it in range(3):
        model.x.copy_(torch.randn(1, bench.N_EMBD, device="cuda", generator=gen))
        graph.replay()
        z = snapshot()
        what = f"{mix} replay {it}"
        r = {}
        for key, buf in (("wq", "q"), ("wk", "kk"), ("wv", "v")):
            r[key] = bar_ratio(z[buf], q8_(key, z["res0"], z[buf].shape[1]), PLAIN_BAR, f"{what}: {key}")
        r["wo"] = bar_ratio(z["h"], q8_("wo", z["q"], bench.N_EMBD), PLAIN_BAR, f"{what}: wo")
        u, g = q8_("up", z["h"], z["a"].shape[1]).astype(np.float64), q8_("gate", z["h"], z["a"].shape[1]).astype(np.float64)
        r["up/gate"] = bar_ratio(z["a"], glu_ref("silu", g, u), GLU_BAR, f"{what}: up/gate")
        check_q8_image(oracle, z["q8"], z["a"], f"{what}: q8 image")
        yq = q8_("down", z["a"], bench.N_EMBD).astype(np.float64)
        ref = yq + z["res0"]
        bound = PLAIN_BAR * rms(yq) + F32_ADD * np.abs(ref)         # the plain bar of the product, plus the rounding of the residual add
        r["down + residual"] = float((np.abs(z["res1"] - ref) / bound).max())
        assert r["down + residual"] <= 1.0, f"{what}: ffn_down + residual, ratio {r['down + residual']}"
        hq = oracle.mul_mat_q8_1(head.ggml_type, hw, z["res1"], len(rows), variant="b200")
        r["head"] = bar_ratio(z["logits"][:, rows], hq, PLAIN_BAR, f"{what}: head rows")
        print(f"{what}: " + ", ".join(f"{key} {v:.3g}" for key, v in r.items()))
    _set_option("pdl", 0)
    try:
        model.step_tg()
        eager = snapshot()
    finally:
        _set_option("pdl", int(os.environ.get("B200Q_PDL", "1")))
    for key in z:
        assert np.array_equal(z[key], eager[key]), f"{mix}: {key} of the eager step (PDL off) differs from the graph replay"


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
