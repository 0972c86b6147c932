"""Host-side surface of HypER's training-mode kernels, no GPU needed: the exported symbols and struct layout, the
argument checks that run before any launch (KGE_EINVAL / KGE_ENOTSUP / KGE_EWORKSPACE), the workspace rule, and the
model class: kge_trunk, the supported-width rule, the trunk tensors' order, dropout noise and the torch layers on CPU
tables."""
import ctypes

import pytest
import torch

from pykg2vec_b200 import _lib, import_model

EINVAL, ENOTSUP, EWORKSPACE = -1, -2, -4


def _hyper(de=24, dr=10, **kw):
    args = dict(tot_entity=20, tot_relation=3, ent_hidden_size=de, rel_hidden_size=dr, input_dropout=0.0,
                feature_map_dropout=0.0, hidden_dropout=0.0, device="cpu")
    args.update(kw)
    return import_model("hyper")(**args)


def test_symbols_and_struct_layout():
    for name in ("kge_hyper_train_workspace_bytes", "kge_hyper_train_fwd", "kge_hyper_train_bwd"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    # 2 int32 + 2 int64 + 6 float, then 12 parameter and 6 running-statistic pointers (kge_hyper_train_t)
    assert ctypes.sizeof(_lib.KgeHyperTrain) == 48 + 18 * 8
    assert len(_lib.HYPER_TRAIN_PARAMS) == 12


def _struct(de, dr=10, running=True):
    p = _lib.KgeHyperTrain()
    p.ent_hidden_size, p.rel_hidden_size = de, dr
    p.ent_padding_idx = p.rel_padding_idx = 0
    for name in _lib.HYPER_TRAIN_PARAMS + (_lib.HYPER_TRAIN_RUNNING if running else ()):
        setattr(p, name, 16)   # never dereferenced: every call below stops at an argument check
    return p


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    i64 = ctypes.c_int64
    ptr = ctypes.c_void_p(16)
    grads = (ctypes.c_void_p * 12)(*([16] * 12))
    before = L.kge_launch_count()
    ok = _struct(200, 200)
    big = int(L.kge_hyper_train_workspace_bytes(ctypes.byref(ok), i64(8), i64(4)))
    assert big > 0

    def fwd(p, Q=8, B=4, e=ptr, ws_bytes=big):
        return L.kge_hyper_train_fwd(ctypes.byref(p), e, ptr, i64(Q), i64(B), None, None, None, ptr, ptr,
                                     i64(ws_bytes), None)

    def bwd(p, Q=8, B=4, g=grads, ws_bytes=big):
        return L.kge_hyper_train_bwd(ctypes.byref(p), ptr, ptr, i64(Q), i64(B), None, None, None, ptr, ptr, g, ptr,
                                     i64(ws_bytes), None)

    for de in (8, 4097):                                                      # de < 9, de > 4096
        assert fwd(_struct(de)) == ENOTSUP and bwd(_struct(de)) == ENOTSUP
    assert fwd(ok, Q=8, B=1) == EINVAL and bwd(ok, Q=1, B=1) == EINVAL        # one-row BatchNorm
    assert fwd(ok, Q=9, B=4) == EINVAL and bwd(ok, Q=9, B=4) == EINVAL        # Q a multiple of B >= 2
    assert fwd(ok, Q=2, B=4) == EINVAL
    assert fwd(ok, e=None) == EINVAL and b"null" in L.kge_last_error()
    assert fwd(ok, ws_bytes=big - 1) == EWORKSPACE and bwd(ok, ws_bytes=big - 1) == EWORKSPACE
    assert fwd(_struct(200, 0)) == EINVAL
    half = _struct(200)
    half.bn2_var = None                                                       # running statistics: all or none
    assert fwd(half) == EINVAL
    nopar = _struct(200)
    nopar.fc1_weight = None
    assert fwd(nopar) == EINVAL and bwd(nopar) == EINVAL
    some = (ctypes.c_void_p * 12)(*([16] * 11 + [0]))
    assert bwd(ok, g=some) == EINVAL and b"gradient buffer 11" in L.kge_last_error()
    assert L.kge_launch_count() == before


def test_workspace_grows_with_rows():
    L = _lib.lib()
    p = _struct(200, 200)
    a = L.kge_hyper_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(128), ctypes.c_int64(128))
    b = L.kge_hyper_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(256), ctypes.c_int64(128))
    F = 32 * 192
    assert a >= 128 * 3 * F * 4 and b >= 2 * a - 4096 and b < 2 * a + 4096
    assert L.kge_hyper_train_workspace_bytes(ctypes.byref(_struct(8)), ctypes.c_int64(8), ctypes.c_int64(4)) == 0


def test_model_surface_on_cpu_tables():
    m = _hyper()
    assert m.kge_trunk and not m._kernel_trunk() and not m.kge_train_supported()   # CPU tables: the torch layers
    assert not _hyper(kge_trunk=False).kge_trunk
    names = dict((id(p), n) for n, p in m.named_parameters())
    assert [names[id(p)] for p in m.kge_hyper_params()] == [
        "ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "bn1.weight", "bn1.bias",
        "fc.weight", "fc.bias", "bn2.weight", "bn2.bias", "fc1.weight", "fc1.bias"]
    assert set(names.values()) - {names[id(p)] for p in m.kge_hyper_params()} == {"b"}
    assert "kge_trunk" not in m.state_dict()
    m.train()
    e, r = torch.tensor([1, 2, 0]), torch.tensor([0, 1, 2])
    assert m.dropout_noise(3) == (None, None, None)
    x = m._train_trunk(e, r)   # training mode on CPU tables: the torch layers, as the reference
    assert x.shape == (3, 24) and int(m.bn2.num_batches_tracked) == 1
    drop = _hyper(input_dropout=0.2, feature_map_dropout=1.0, hidden_dropout=0.0).train()
    n0, n1, n2 = drop.dropout_noise(4)
    assert n0.shape == (4, 24) and n1.shape == (4, 32) and not n1.any() and n2 is None
    assert set(torch.unique(n0).tolist()) <= {0.0, 1.25}
    drop.eval()
    assert drop.dropout_noise(4) == (None, None, None)


def test_momentum_none_selects_the_torch_layers():
    """cumulative averaging (momentum None) is the torch layers' job: the binding refuses it before reading a tensor"""
    m = _hyper()
    m.bn1.momentum = None
    with pytest.raises(_lib.KgeNotSupported):
        _lib.hyper_train_struct(m, params=[torch.zeros(1)] * 12)


def test_one_row_batch_raises_like_batchnorm1d():
    m = _hyper().train()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
