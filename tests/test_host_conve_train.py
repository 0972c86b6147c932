"""Host-side surface of ConvE's training-mode kernels, no GPU needed: the exported symbols and struct layout, the
argument checks that run before any launch (KGE_EINVAL / KGE_ENOTSUP / KGE_EWORKSPACE), the workspace rule, and the
model class: kge_trunk, the supported-image rule, the trunk tensors' order and the torch layers on CPU tables."""
import ctypes

import pytest
import torch

from pykg2vec_b200 import _lib, import_model

EINVAL, ENOTSUP, EWORKSPACE = -1, -2, -4


def _conve(k=36, h1=6, **kw):
    args = dict(tot_entity=20, tot_relation=3, hidden_size=k, hidden_size_1=h1, lmbda=0.1, input_dropout=0.0,
                feature_map_dropout=0.0, hidden_dropout=0.0)
    args.update(kw)
    return import_model("conve")(**args)


def test_symbols_and_struct_layout():
    for name in ("kge_conve_train_workspace_bytes", "kge_conve_train_fwd", "kge_conve_train_bwd"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    # 2 int32 + 6 float, then 12 parameter and 6 running-statistic pointers (include/kge_b200.h kge_conve_train_t)
    assert ctypes.sizeof(_lib.KgeConveTrain) == 32 + 18 * 8
    assert len(_lib.CONVE_TRAIN_PARAMS) == 12


def _struct(k, h1, running=True):
    p = _lib.KgeConveTrain()
    p.hidden_size, p.hidden_size_1 = k, h1
    for name in _lib.CONVE_TRAIN_PARAMS + (_lib.CONVE_TRAIN_RUNNING if running else ()):
        setattr(p, name, 16)   # never dereferenced: every call below stops at an argument check
    return p


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    i64 = ctypes.c_int64
    ptr = ctypes.c_void_p(16)
    grads = (ctypes.c_void_p * 12)(*([16] * 12))
    before = L.kge_launch_count()
    ok = _struct(200, 20)
    big = int(L.kge_conve_train_workspace_bytes(ctypes.byref(ok), i64(8), i64(4)))
    assert big > 0

    def fwd(p, Q=8, B=4, e=ptr, ws_bytes=big):
        return L.kge_conve_train_fwd(ctypes.byref(p), e, ptr, i64(Q), i64(B), None, None, None, ptr, ptr,
                                     i64(ws_bytes), None)

    def bwd(p, Q=8, B=4, g=grads, ws_bytes=big):
        return L.kge_conve_train_bwd(ctypes.byref(p), ptr, ptr, i64(Q), i64(B), None, None, None, ptr, ptr, g, ptr,
                                     i64(ws_bytes), None)

    for k, h1 in ((2100, 21), (36, 2), (40, 40), (36, 7)):   # 2k > 4096, h1 < 3, h2 < 2, h1 does not divide k
        assert fwd(_struct(k, h1)) == ENOTSUP and bwd(_struct(k, h1)) == ENOTSUP
    assert fwd(ok, Q=8, B=1) == EINVAL and bwd(ok, Q=1, B=1) == EINVAL        # one-row BatchNorm
    assert fwd(ok, Q=9, B=4) == EINVAL and fwd(ok, Q=2, B=4) == EINVAL        # Q a multiple of B >= 2
    assert fwd(ok, e=None) == EINVAL and b"null" in L.kge_last_error()
    assert fwd(ok, ws_bytes=big - 1) == EWORKSPACE and bwd(ok, ws_bytes=big - 1) == EWORKSPACE
    half = _struct(200, 20)
    half.bn2_var = None                                                       # running statistics: all or none
    assert fwd(half) == EINVAL
    nopar = _struct(200, 20)
    nopar.fc_weight = None
    assert fwd(nopar) == EINVAL and bwd(nopar) == EINVAL
    some = (ctypes.c_void_p * 12)(*([16] * 11 + [0]))
    assert bwd(ok, g=some) == EINVAL and b"gradient buffer 11" in L.kge_last_error()
    assert L.kge_launch_count() == before


def test_workspace_grows_with_rows():
    L = _lib.lib()
    p = _struct(200, 20)
    a = L.kge_conve_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(128), ctypes.c_int64(128))
    b = L.kge_conve_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(256), ctypes.c_int64(128))
    F = 32 * 18 * 18
    assert a >= 128 * 3 * F * 4 and b >= 2 * a - 4096 and b < 2 * a + 4096


def test_model_surface_on_cpu_tables():
    m = _conve()
    assert m.kge_trunk and not m._kernel_trunk() and not m.kge_train_supported()   # CPU tables: the torch layers
    assert not _conve(kge_trunk=False).kge_trunk
    names = dict((id(p), n) for n, p in m.named_parameters())
    assert [names[id(p)] for p in m.kge_conve_params()] == [n for n, _ in m.named_parameters() if n != "b.weight"]
    assert "kge_trunk" not in m.state_dict()
    m.train()
    e, r = torch.tensor([1, 2, 3]), torch.tensor([0, 1, 2])
    assert m.dropout_noise(3) == (None, None, None)
    x = m._train_trunk(e, r)   # training mode on CPU tables: the torch layers, as the reference
    assert x.shape == (3, 36) and int(m.bn2.num_batches_tracked) == 1
    drop = _conve(input_dropout=0.2, feature_map_dropout=1.0, hidden_dropout=0.0).train()
    n0, n1, n2 = drop.dropout_noise(4)
    assert n0.shape == (4, 72) and n1.shape == (4, 32) and not n1.any() and n2 is None
    assert set(torch.unique(n0).tolist()) <= {0.0, 1.25}
    drop.eval()
    assert drop.dropout_noise(4) == (None, None, None)


def test_one_row_batch_raises_like_batchnorm1d():
    m = _conve().train()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
