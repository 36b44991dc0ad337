"""The backend plug on DeepSeek's MLA prompt-processing product (tests/backend_ops/test_plug_mla_pp.cpp): kv_f32 = wkv_b_iter x kv_cache_nope built
as src/graphs/build_deepseek2.cpp:922-990 builds it (a view of whole rows of wkv_b per iteration, a view of the f16 K cache, the f16 casts after it),
under ggml_backend_sched next to the reference CPU backend.  Every MUL_MAT must run on the plug and match the CPU backend (NMSE <= 5e-4)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_pp_opt_wkv_b_product_runs_on_the_plug():
    """Q8_0 and Q6_K wkv_b at 16 heads (n_kv 256 ... 2048) and 128 heads (n_kv 256, 1024), one, two and four slices per layer."""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "backend_ops", "test_plug_mla_pp")
    if not os.path.exists(exe):
        pytest.skip("harness not built (needs the reference headers at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED: 0 failures" in r.stdout
