"""CPU tests (-m "not gpu") of the InteractE C-ABI as built: the symbols and struct layout, the workspace size
rule, the shape checks that need no device, and what the compiler made of the feature kernel (ptxas: no
local-memory spills; SASS: the FFMA inner loop reads the filter bank with LDS.128)."""
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
    import interacte_util as iu
    from pykg2vec_b200 import _lib
    _built()
    # int32 x5 (+4 padding), int64, float x3 (+4 padding), perm + 17 pointers — the same layout on both sides
    assert ctypes.sizeof(_lib.KgeInteracte) == 4 * 5 + 4 + 8 + 4 * 3 + 4 + 18 * 8 == ctypes.sizeof(iu.KgeInteracte)
    R = 237
    for (P, F, ks, rh, rw) in iu.YAML_CONFIGS:
        k = rh * rw
        Fw = P * F * 2 * k
        for Q in (1, 77, 8192):
            want = (Q * Fw + ((Fw + 511) // 512) * Q * k) * 4       # features + Linear slice partials
            assert _lib.interacte_trunk_workspace_bytes(P, F, ks, rh, rw, R, Q) == want
    # ~214 KB per query at the default shape, ~570 KB at (4, 64, 7): hence the chunking in interacte_trunk_fwd
    assert 213e3 < _lib.interacte_trunk_workspace_bytes(1, 96, 9, 20, 10, R, 1) < 215e3
    assert 565e3 < _lib.interacte_trunk_workspace_bytes(4, 64, 7, 20, 10, R, 1) < 575e3
    assert _lib.INTERACTE_WORKSPACE_CAP == 256 << 20


@pytest.mark.parametrize("geom", [(1, 96, 8, 20, 10),      # even kernel_size
                                  (1, 8, 1, 4, 3),         # ks < 3
                                  (1, 8, 9, 3, 10),        # pad 4 > W = 3
                                  (1, 8, 11, 20, 2),       # pad 5 > H = 4
                                  (2, 480, 11, 20, 10)])   # filter bank + images over 227 KB of shared memory
def test_unsupported_shapes_have_no_workspace(geom):
    from pykg2vec_b200 import _lib
    _built()
    assert _lib.interacte_trunk_workspace_bytes(*geom, 5, 4) == 0


def test_feature_kernel_has_no_local_memory_spills():
    path = os.path.join(os.path.dirname(_built()), "kge_proj.ptxas.log")
    log = open(path).read()
    blocks = re.findall(r"Compiling entry function '(_ZN3kge\w*interacte\w*)'.*?\n(.*?)Compile time", log, re.S)
    assert any("interacte_feature_kernel" in n for n, _ in blocks)
    for name, body in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in body, (name, body)


def test_sass_feature_kernel_inner_loop():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not installed")
    obj = os.path.join(os.path.dirname(_built()), "obj", "kge_proj.o")
    sass = subprocess.run([exe, "-sass", "-fun", "_ZN3kge24interacte_feature_kernelENS_13InteracteFeatE", obj],
                          capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in sass
    assert "BAR.SYNC" in sass and "LDL" not in sass and "STL" not in sass
    assert len(re.findall(r"\bLDS\.128\b", sass)) >= 2       # two float4 filter reads per tap
    assert len(re.findall(r"\bFFMA\b", sass)) >= 8           # eight filters per image value
