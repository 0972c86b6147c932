"""Host-side surface of AcrE's training-mode kernels, no GPU needed: the exported symbols and struct layout, the
argument checks that run before any launch (KGE_EINVAL / KGE_ENOTSUP / KGE_EWORKSPACE, including the gradient-slot
rule), the workspace rule and the largest accepted in_channels of each way, what the compiler made of the new kernels
(ptxas: no local-memory spills), and the model class: kge_trunk, the supported-configuration rule, the trunk tensors'
order, dropout noise, the torch layers on CPU tables and the cases that select them."""
import ctypes
import os
import re

import pytest
import torch

from pykg2vec_b200 import _lib, import_model

EINVAL, ENOTSUP, EWORKSPACE = -1, -2, -4
NSLOT = 18


def _acre(way="serial", C=4, bias=True, **kw):
    args = dict(tot_entity=20, tot_relation=3, hidden_size=200, input_dropout=0.0, hidden_dropout=0.0,
                feature_map_dropout=0.0, in_channels=C, way=way, first_atrous=1, second_atrous=2, third_atrous=3,
                acre_bias=bias)
    args.update(kw)
    return import_model("acre")(**args)


def test_symbols_and_struct_layout():
    for name in ("kge_acre_train_workspace_bytes", "kge_acre_train_fwd", "kge_acre_train_bwd"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    # 6 int32, int64 num_rel, 6 float, then 18 parameter and 6 running-statistic pointers
    assert ctypes.sizeof(_lib.KgeAcreTrain) == 24 + 8 + 24 + 24 * 8
    assert _lib.KgeAcreTrain.ent.offset == 56
    assert len(_lib.ACRE_TRAIN_PARAMS) == NSLOT


def _struct(way=0, C=32, bias=True, running=True, rates=(1, 2, 2), k=200):
    p = _lib.KgeAcreTrain()
    p.way, p.in_channels, p.hidden_size, p.num_rel = way, C, k, 474
    p.first_atrous, p.second_atrous, p.third_atrous = rates
    for name in _lib.ACRE_TRAIN_PARAMS + (_lib.ACRE_TRAIN_RUNNING if running else ()):
        if name.startswith("conv") and name.endswith("_bias") and not bias:
            continue
        if name.startswith("W_gate_e") and way == 0:
            continue
        setattr(p, name, 16)   # never dereferenced: every call below stops at an argument check
    return p


def _slots(way=0, bias=True):
    present = []
    for name in _lib.ACRE_TRAIN_PARAMS:
        absent = (name.startswith("conv") and name.endswith("_bias") and not bias) or \
            (name.startswith("W_gate_e") and way == 0)
        present.append(None if absent else 16)
    return present


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    i64 = ctypes.c_int64
    ptr = ctypes.c_void_p(16)
    before = L.kge_launch_count()
    ok = _struct()
    big = int(L.kge_acre_train_workspace_bytes(ctypes.byref(ok), i64(8), i64(4)))
    assert big > 0

    def fwd(p, Q=8, B=4, e=ptr, ws_bytes=big):
        return L.kge_acre_train_fwd(ctypes.byref(p), e, ptr, i64(Q), i64(B), None, None, None, ptr, ptr,
                                    i64(ws_bytes), None)

    def bwd(p, Q=8, B=4, g=None, ws_bytes=big):
        g = (ctypes.c_void_p * NSLOT)(*(_slots() if g is None else g))
        return L.kge_acre_train_bwd(ctypes.byref(p), ptr, ptr, i64(Q), i64(B), None, None, None, ptr, ptr, g, ptr,
                                    i64(ws_bytes), None)

    assert fwd(_struct(k=100)) == ENOTSUP and bwd(_struct(k=100)) == ENOTSUP     # the 10 x 20 view needs 200
    assert fwd(_struct(C=47)) == ENOTSUP and bwd(_struct(C=47)) == ENOTSUP       # serial shared-memory bound
    assert fwd(_struct(way=1, C=1025)) == ENOTSUP
    for bad in (_struct(way=2), _struct(C=0), _struct(rates=(1, 0, 2))):
        assert fwd(bad) == EINVAL
    assert fwd(ok, Q=8, B=1) == EINVAL and bwd(ok, Q=1, B=1) == EINVAL            # one-row BatchNorm
    assert fwd(ok, Q=9, B=4) == EINVAL and bwd(ok, Q=9, B=4) == EINVAL            # Q a multiple of B >= 2
    assert fwd(ok, Q=2, B=4) == EINVAL
    assert fwd(ok, e=None) == EINVAL and b"null" in L.kge_last_error()
    assert fwd(ok, ws_bytes=big - 1) == EWORKSPACE and bwd(ok, ws_bytes=big - 1) == EWORKSPACE
    half = _struct()
    half.bn2_var = None                                                           # running statistics: all or none
    assert fwd(half) == EINVAL
    onebias = _struct()
    onebias.conv2_bias = None                                                     # conv biases: all or none
    assert fwd(onebias) == EINVAL and b"conv biases" in L.kge_last_error()
    nogate = _struct(way=1)
    nogate.W_gate_e_bias = None                                                   # the parallel way needs W_gate_e
    assert fwd(nogate) == EINVAL
    nofc = _struct()
    nofc.fc_weight = None
    assert fwd(nofc) == EINVAL and bwd(nofc) == EINVAL
    # gradient slots: present parameters set, absent ones NULL
    miss = _slots()
    miss[14] = None
    assert bwd(ok, g=miss) == EINVAL and b"slot 14 must be set" in L.kge_last_error()
    extra = _slots()
    extra[10] = 16                                                                # W_gate_e in the serial way
    assert bwd(ok, g=extra) == EINVAL and b"slot 10 must be NULL" in L.kge_last_error()
    nb = _struct(bias=False)
    assert bwd(nb, g=_slots()) == EINVAL                                          # bias slots without acre_bias
    par = _struct(way=1, C=9, bias=False)
    pbig = int(L.kge_acre_train_workspace_bytes(ctypes.byref(par), i64(8), i64(4)))
    g = (ctypes.c_void_p * NSLOT)(*_slots(way=1, bias=False))
    assert L.kge_acre_train_bwd(ctypes.byref(par), ptr, ptr, i64(8), i64(4), None, None, None, ptr, ptr, g, ptr,
                                i64(pbig - 1), None) == EWORKSPACE                # the slot rule passed
    assert L.kge_launch_count() == before


def _ws(way, C, Q=256, B=128):
    return int(_lib.lib().kge_acre_train_workspace_bytes(ctypes.byref(_struct(way=way, C=C)), ctypes.c_int64(Q),
                                                         ctypes.c_int64(B)))


def _formula(way, C, Q=256, B=128):
    """the header's workspace formula, in bytes, before the 64-float rounding of each region"""
    cin = C if way == 0 else 1
    G = Q // B
    f = Q * (400 * (2 + 2 * C) + 200 * ((400 * C + 511) // 512 + 2) + 9 * C * (cin + cin + 1) + 5 * C + 2) + \
        G * (4 * C + 404)
    f += Q * 800 * C if way == 0 else Q * 1600 * C
    return 4 * f


@pytest.mark.parametrize("way,C,mb", [(0, 32, 78), (1, 9, 25)])
def test_workspace_rule(way, C, mb):
    """the header's formula (each of its ~24 regions rounded up to 64 floats) and its stated sizes at Q = 256"""
    got = _ws(way, C)
    assert _formula(way, C) <= got <= _formula(way, C) + 24 * 64 * 4
    assert abs(got / 1e6 - mb) < 1.0, got


def test_largest_accepted_channels():
    L = _lib.lib()
    assert _ws(0, 46) > 0 and _ws(0, 47) == 0 and b"C <= 46" in L.kge_last_error()
    assert _ws(1, 1024) > 0 and _ws(1, 1025) == 0
    assert _ws(1, 64) > 0


def test_new_kernels_have_no_local_memory_spills():
    from pykg2vec_b200 import build
    path = os.path.join(os.path.dirname(build.build()), "kge_proj.ptxas.log")
    log = open(path).read()
    blocks = re.findall(r"Compiling entry function '(_ZN3kge\w*acre_tr_\w*)'.*?\n(.*?)Compile time", log, re.S)
    names = {n for n, _ in blocks}
    for kern in ("serial", "gate", "bn1_part", "feat", "bn1_bwd_part", "bn1_bwd", "serial_bwd", "gate_bwd",
                 "bn0_part"):
        assert any("acre_tr_%s_kernel" % kern in n for n in names), kern
    for name, body in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in body, (name, body)


@pytest.mark.parametrize("way,bias", [("serial", True), ("parallel", False)])
def test_model_surface_on_cpu_tables(way, bias):
    m = _acre(way, bias=bias)
    assert m.kge_trunk and not m._kernel_trunk() and not m.kge_train_supported()   # CPU tables: the torch layers
    assert not _acre(kge_trunk=False).kge_trunk
    names = dict((id(p), n) for n, p in m.named_parameters())
    want = ["ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias"]
    for l in ("conv1", "conv2", "conv3"):
        want += [l + ".weight"] + ([l + ".bias"] if bias else [])
    if way == "parallel":
        want += ["W_gate_e.weight", "W_gate_e.bias"]
    want += ["bn1.weight", "bn1.bias", "fc.weight", "fc.bias", "bn2.weight", "bn2.bias"]
    assert [names[id(p)] for p in m.kge_acre_params()] == want
    assert set(names.values()) - set(want) == {"bias"}
    assert "kge_trunk" not in m.state_dict()
    m.train()
    e, r = torch.tensor([1, 2, 0]), torch.tensor([0, 1, 2])
    assert m.dropout_noise(3) == (None, None, None)
    x = m._train_trunk(e, r)   # training mode on CPU tables: the torch layers, as the reference
    assert x.shape == (3, 200) and int(m.bn2.num_batches_tracked) == 1
    m._kernel_trunk = lambda: True   # as with CUDA tables: the configuration is one the kernels take
    assert m.kge_train_supported()


def test_dropout_noise_shapes():
    drop = _acre(C=5, input_dropout=0.2, feature_map_dropout=1.0, hidden_dropout=0.0).train()
    n0, n1, n2 = drop.dropout_noise(4)
    assert n0.shape == (4, 400) and n1.shape == (4, 5) and not n1.any() and n2 is None
    assert set(torch.unique(n0).tolist()) <= {0.0, 1.25}
    drop.eval()
    assert drop.dropout_noise(4) == (None, None, None)


def test_fallback_selection():
    """momentum None, kge_trunk=False and configurations the kernels refuse select the torch layers"""
    m = _acre()
    m.bn1.momentum = None
    with pytest.raises(_lib.KgeNotSupported):
        _lib.acre_train_struct(m, params=[torch.zeros(1)] * len(m.kge_acre_params()))
    m._kernel_trunk = lambda: True
    assert not m.kge_train_supported()
    off = _acre(kge_trunk=False)
    assert not off._kernel_trunk()
    for big in (_acre(C=47), _acre(hidden_size=100)):
        big._kernel_trunk = lambda: True
        assert not big.kge_train_supported()
    wide = _acre("parallel", C=64)
    wide._kernel_trunk = lambda: True
    assert wide.kge_train_supported()


def test_one_row_batch_raises_like_batchnorm1d():
    m = _acre().train()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
    m._kernel_trunk = lambda: True   # the kernel path refuses before anything is launched, as BatchNorm1d would
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
