"""CPU tests (-m "not gpu") of the HypER C-ABI as built: the symbols and struct layout, the workspace size
rule, and what the compiler made of the kernels (ptxas: no local-memory spills in the feature kernel;
SASS: the Linear layer runs on the tiled GEMM's LDS.128 / FFMA inner loop)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest


def _built():
    from pykg2vec_b200 import build
    return build.build()


def test_struct_layout_and_workspace_rule():
    import hyper_util as hu
    from pykg2vec_b200 import _lib
    _built()
    # int32 x2, int64, float x3 (+4 padding), 18 pointers — the same layout on both sides
    assert ctypes.sizeof(_lib.KgeHyper) == 4 * 2 + 8 + 4 * 3 + 4 + 18 * 8 == ctypes.sizeof(hu.KgeHyper)
    de, dr, R = 200, 200, 237
    F = 32 * (de - 8)
    for Q in (1, 77, 8192):
        want = (R * 288 + Q * F + ((F + 511) // 512) * Q * de) * 4   # filters + features + Linear slice partials
        assert _lib.hyper_trunk_workspace_bytes(de, dr, R, Q) == want
    # the Evaluator's 8192-query batch at the FB15k-237 shape: ~280 MB, sized, not capped
    assert 270e6 < _lib.hyper_trunk_workspace_bytes(de, dr, R, 8192) < 290e6
    assert _lib.hyper_trunk_workspace_bytes(8, dr, R, 4) == 0 and _lib.hyper_trunk_workspace_bytes(4097, dr, R, 4) == 0


def test_feature_kernel_has_no_local_memory_spills():
    path = os.path.join(os.path.dirname(_built()), "kge_proj.ptxas.log")
    log = open(path).read()
    blocks = re.findall(r"Compiling entry function '(_ZN3kge\w*hyper\w*)'.*?\n(.*?)Compile time", log, re.S)
    names = {n for n, _ in blocks}
    assert any("hyper_feature_kernel" in n for n in names) and any("hyper_fc_combine_kernel" in n for n in names)
    for name, body in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in body, (name, body)


def test_sass_linear_layer_runs_the_tiled_gemm_loop():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not installed")
    obj = os.path.join(os.path.dirname(_built()), "obj", "kge_proj.o")
    sass = subprocess.run([exe, "-sass", "-fun", "_ZN3kge16proj_gemm_kernelILi0ELi4ELi4EEEvNS_8ProjGemmE", obj],
                          capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in sass
    assert len(re.findall(r"\bLDS\.128\b", sass)) >= 16      # 4x4 thread tile: one 16-byte A and B read per k step
    assert len(re.findall(r"\bFFMA\b", sass)) >= 16 * 16     # 16 fma per k step, 16 k steps per staged chunk
    feat = subprocess.run([exe, "-sass", "-fun", "_ZN3kge20hyper_feature_kernelENS_9HyperFeatE", obj],
                          capture_output=True, text=True, check=True).stdout
    assert "FFMA" in feat and "BAR.SYNC" in feat and "LDL" not in feat and "STL" not in feat
