"""The backend plug on batched MUL_MAT (tests/backend_ops/test_plug_mla.cpp): DeepSeek's absorbed-MLA per-head products built as
src/graphs/build_deepseek2.cpp builds them (the view of q, the permutes, the 3-D wk_b / wv_b), and contiguous batched products, each under
ggml_backend_sched next to the reference CPU backend.  Every MUL_MAT must run on the plug and match the CPU backend (NMSE <= 5e-4)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def _harness(mode):
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "backend_ops", "test_plug_mla")
    if not os.path.exists(exe):
        pytest.skip("harness not built (needs the reference headers at build time)")
    r = subprocess.run([exe, mode], capture_output=True, text=True, timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED: 0 failures" in r.stdout


def test_mla_products_run_on_the_plug():
    """q_nope2 = wk_b x q_nope_perm and kqv = wv_b x kqv_compressed_perm at 16 and 128 heads, Q8_0 and IQ4_NL, 1 ... 512 tokens."""
    _harness("mla")


def test_contiguous_batched_products_run_on_the_plug():
    """A weight broadcast over ne2, one broadcast over ne3, and one weight matrix per batch entry, 1 ... 64 columns."""
    _harness("contiguous")
