"""CPU tests (-m "not gpu") of the AcrE C-ABI as built: the symbols and struct layout, the workspace size rule,
every argument error code (they are all decided before any device work, so no GPU is needed), and what the
compiler made of the new kernels (ptxas: no local-memory spills, shared memory within the stated bound; SASS:
the serial kernel's inner loop reads the weight bank with LDS.128)."""
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
    import acre_util as au
    from pykg2vec_b200 import _lib
    _built()
    # int32 x6, int64, float x3 (+4 padding), 24 pointers — the same layout on both sides
    assert ctypes.sizeof(_lib.KgeAcre) == 4 * 6 + 8 + 4 * 3 + 4 + 24 * 8 == ctypes.sizeof(au.KgeAcre)
    assert [f for f, _ in _lib.KgeAcre._fields_] == [f for f, _ in au.KgeAcre._fields_]
    R2 = 474
    for way, C in (("serial", 32), ("serial", 9), ("parallel", 9), ("parallel", 32)):
        Fw = C * 400
        for Q in (1, 77, 8192):
            want = (Q * C * 1600 * (way == "parallel") + Q * Fw + ((Fw + 511) // 512) * Q * 200) * 4
            assert _lib.acre_trunk_workspace_bytes(way, C, (1, 2, 2), 200, R2, Q) == want
    # per query at C = 32: 51 KB of features (+ 20 KB of slice partials) serial, + 205 KB of gate input parallel
    assert _lib.acre_trunk_workspace_bytes("serial", 32, (1, 2, 2), 200, R2, 1) == 51200 + 20000
    assert _lib.acre_trunk_workspace_bytes("parallel", 32, (1, 2, 2), 200, R2, 1) == 204800 + 51200 + 20000
    # the Evaluator's 8,192-query batch needs 583 MB serial: hence the chunking in acre_trunk_fwd
    assert _lib.acre_trunk_workspace_bytes("serial", 32, (1, 2, 2), 200, R2, 8192) > _lib.ACRE_WORKSPACE_CAP
    assert _lib.ACRE_WORKSPACE_CAP == 256 << 20


@pytest.mark.parametrize("cfg", [("serial", 4, (1, 2, 2), 100),      # hidden_size != 200
                                 ("serial", 47, (1, 2, 2), 200),     # over the serial kernel's shared memory
                                 ("parallel", 1924, (1, 2, 2), 200),  # over the gate kernel's shared memory
                                 ("serial", 0, (1, 2, 2), 200),      # in_channels < 1
                                 ("serial", 4, (0, 2, 2), 200),      # an atrous rate < 1
                                 ("bogus", 4, (1, 2, 2), 200)])      # a way that is neither
def test_unsupported_or_malformed_configs_have_no_workspace(cfg):
    from pykg2vec_b200 import _lib
    _built()
    way, C, atrous, k = cfg
    assert _lib.acre_trunk_workspace_bytes(way, C, atrous, k, 10, 4) == 0


def test_largest_supported_channels():
    from pykg2vec_b200 import _lib
    _built()
    assert _lib.acre_trunk_workspace_bytes("serial", 46, (1, 2, 2), 200, 10, 1) > 0
    assert _lib.acre_trunk_workspace_bytes("parallel", 1923, (1, 2, 2), 200, 10, 1) > 0


def _call(L, p, Q=2, ws_bytes=0, ids=True, x=True):
    """kge_acre_trunk_fwd on dummy host pointers: every error is returned before anything touches them.  The
    workspace size defaults to 0, so a call with Q > 0 that passes every other check stops at KGE_EWORKSPACE
    and nothing is launched."""
    dummy = ctypes.c_void_p(16)
    return L.kge_acre_trunk_fwd(ctypes.byref(p), dummy if ids else None, dummy if ids else None, ctypes.c_int64(Q),
                                dummy if x else None, dummy, ctypes.c_int64(ws_bytes), None)


def _full(way="serial", C=4, atrous=(1, 2, 2), k=200, bias=True):
    from pykg2vec_b200 import _lib
    p = _lib.acre_struct(way, C, atrous, k, 10)
    for n in _lib.ACRE_FIELDS:
        if bias or not n.startswith("conv") or not n.endswith("_bias"):
            setattr(p, n, 64)
    return p


def test_every_error_code():
    from pykg2vec_b200 import _lib
    _built()
    L = _lib.lib()
    EINVAL, ENOTSUP, EWS = -1, -2, -4
    # EINVAL: way, atrous, in_channels, num_rel, null pointers, a partial set of conv biases, Q
    for mut in (lambda p: setattr(p, "way", 2), lambda p: setattr(p, "way", -1),
                lambda p: setattr(p, "second_atrous", 0), lambda p: setattr(p, "in_channels", 0),
                lambda p: setattr(p, "num_rel", 0), lambda p: setattr(p, "fc_weight", None),
                lambda p: setattr(p, "bn2_var", None), lambda p: setattr(p, "conv3_weight", None),
                lambda p: setattr(p, "conv2_bias", None)):
        p = _full()
        mut(p)
        assert _call(L, p) == EINVAL
    p = _full("parallel")
    p.W_gate_e_bias = None
    assert _call(L, p) == EINVAL                      # W_gate_e is required by the parallel way ...
    p = _full("serial")
    p.W_gate_e_weight = p.W_gate_e_bias = None
    assert _call(L, p, ws_bytes=0) == EWS             # ... and not by the serial way
    assert _call(L, _full(), ids=False) == EINVAL     # Q > 0 needs ids and output
    assert _call(L, _full(), x=False) == EINVAL
    assert _call(L, _full(), Q=-1) == EINVAL
    assert _call(L, _full("parallel", C=1000), Q=5000) == EINVAL   # Q*C rows beyond one call's grid
    # ENOTSUP: hidden_size, shared memory
    assert _call(L, _full(k=100)) == ENOTSUP
    assert _call(L, _full(C=47)) == ENOTSUP
    assert _call(L, _full("parallel", C=1924)) == ENOTSUP
    # EWORKSPACE: one byte short (never a sufficient one: that would launch on the dummy pointers)
    for way, bias in (("serial", True), ("parallel", False)):
        p = _full(way, bias=bias)
        need = int(L.kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(2)))
        assert need > 0
        assert _call(L, p, ws_bytes=0) == EWS and _call(L, p, ws_bytes=need - 1) == EWS
    # Q = 0: a no-op that accepts null ids and output (the workspace rule asks for one query's worth)
    for p in (_full(), _full("parallel", bias=False)):
        need = int(L.kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(0)))
        assert _call(L, p, Q=0, ids=False, x=False, ws_bytes=need) == 0


def _ptxas_blocks():
    path = os.path.join(os.path.dirname(_built()), "kge_proj.ptxas.log")
    log = open(path).read()
    return dict(re.findall(r"Compiling entry function '(_ZN3kge\w*acre\w*)'.*?\n(.*?)Compile time", log, re.S))


def test_kernels_have_no_local_memory_spills():
    blocks = _ptxas_blocks()
    for k in ("acre_serial_feature_kernel", "acre_gate_input_kernel", "acre_bn1_relu_kernel"):
        assert any(k in n for n in blocks), k
    for name, body in blocks.items():
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in body, (name, body)


def test_serial_kernel_registers_allow_its_block():
    """400 threads per CTA: the register count must leave room for the whole block (65,536 per SM)"""
    body = [b for n, b in _ptxas_blocks().items() if "acre_serial_feature_kernel" in n][0]
    regs = int(re.search(r"Used (\d+) registers", body).group(1))
    assert regs * 400 <= 65536


def test_sass_serial_kernel_inner_loop():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not installed")
    obj = os.path.join(os.path.dirname(_built()), "obj", "kge_proj.o")
    sass = subprocess.run([exe, "-sass", "-fun", "_ZN3kge26acre_serial_feature_kernelENS_8AcreFeatE", obj],
                          capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in sass
    assert "BAR.SYNC" in sass and "LDL" not in sass and "STL" not in sass
    assert len(re.findall(r"\bLDS\.128\b", sass)) >= 2       # two float4 bank reads per input channel
    assert len(re.findall(r"\bFFMA\b", sass)) >= 32          # 8 channels x 4 pixels per image value
