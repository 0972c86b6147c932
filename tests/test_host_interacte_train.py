"""Host-side surface of InteractE's training-mode kernels, no GPU needed: the exported symbols and struct layout, the
argument checks that run before any launch (KGE_EINVAL / KGE_ENOTSUP / KGE_EWORKSPACE), the workspace bound, what the
compiler made of the new kernels (ptxas: no local-memory spills), and the model class: kge_trunk, the supported-shape
rule, the trunk tensors' order, dropout noise, the torch layers on CPU tables and the cases that select them."""
import ctypes
import os
import re

import pytest
import torch

from pykg2vec_b200 import _lib, import_model

EINVAL, ENOTSUP, EWORKSPACE = -1, -2, -4
YAML = [(1, 96, 9, 20, 10), (2, 96, 11, 20, 10), (4, 64, 7, 20, 10)]   # (P, F, ks, rh, rw) of InteractE.yaml


def _interacte(geom=(2, 3, 3, 4, 3), **kw):
    P, F, ks, rh, rw = geom
    args = dict(tot_entity=20, tot_relation=3, hidden_size=rh * rw, input_dropout=0.0, hidden_dropout=0.0,
                feature_map_dropout=0.0, feature_permutation=P, num_filters=F, kernel_size=ks, reshape_height=rh,
                reshape_width=rw, device="cpu")
    args.update(kw)
    return import_model("interacte")(**args)


def test_symbols_and_struct_layout():
    import interacte_train_util as itu
    for name in ("kge_interacte_train_workspace_bytes", "kge_interacte_train_fwd", "kge_interacte_train_bwd"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    # 5 int32 + 6 float (+4 padding), then perm, 11 parameter and 6 running-statistic pointers (kge_interacte_train_t)
    assert ctypes.sizeof(_lib.KgeInteracteTrain) == 48 + 18 * 8 == ctypes.sizeof(itu.KgeInteracteTrain)
    assert len(_lib.INTERACTE_TRAIN_PARAMS) == 11


def _struct(geom, running=True):
    p = _lib.KgeInteracteTrain()
    p.feature_permutation, p.num_filters, p.kernel_size, p.reshape_height, p.reshape_width = geom
    p.perm = 16
    for name in _lib.INTERACTE_TRAIN_PARAMS + (_lib.INTERACTE_TRAIN_RUNNING if running else ()):
        setattr(p, name, 16)   # never dereferenced: every call below stops at an argument check
    return p


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    i64 = ctypes.c_int64
    ptr = ctypes.c_void_p(16)
    grads = (ctypes.c_void_p * 11)(*([16] * 11))
    before = L.kge_launch_count()
    ok = _struct(YAML[0])
    big = int(L.kge_interacte_train_workspace_bytes(ctypes.byref(ok), i64(8), i64(4)))
    assert big > 0

    def fwd(p, Q=8, B=4, e=ptr, ws_bytes=big):
        return L.kge_interacte_train_fwd(ctypes.byref(p), e, ptr, i64(Q), i64(B), None, None, None, ptr, ptr,
                                         i64(ws_bytes), None)

    def bwd(p, Q=8, B=4, g=grads, ws_bytes=big):
        return L.kge_interacte_train_bwd(ctypes.byref(p), ptr, ptr, i64(Q), i64(B), None, None, None, ptr, ptr, g, ptr,
                                         i64(ws_bytes), None)

    for geom in ((1, 96, 8, 20, 10), (1, 8, 1, 4, 3), (1, 8, 9, 3, 10), (2, 480, 11, 20, 10)):
        assert fwd(_struct(geom)) == ENOTSUP and bwd(_struct(geom)) == ENOTSUP   # the inference trunk's bounds
    assert fwd(ok, Q=8, B=1) == EINVAL and bwd(ok, Q=1, B=1) == EINVAL            # one-row BatchNorm
    assert fwd(ok, Q=9, B=4) == EINVAL and bwd(ok, Q=9, B=4) == EINVAL            # Q a multiple of B >= 2
    assert fwd(ok, Q=2, B=4) == EINVAL
    assert fwd(ok, e=None) == EINVAL and b"null" in L.kge_last_error()
    assert fwd(ok, ws_bytes=big - 1) == EWORKSPACE and bwd(ok, ws_bytes=big - 1) == EWORKSPACE
    assert fwd(_struct((0, 96, 9, 20, 10))) == EINVAL
    half = _struct(YAML[0])
    half.bn2_var = None                                                           # running statistics: all or none
    assert fwd(half) == EINVAL
    nopar = _struct(YAML[0])
    nopar.conv_filt = None
    assert fwd(nopar) == EINVAL and bwd(nopar) == EINVAL
    noperm = _struct(YAML[0])
    noperm.perm = None
    assert fwd(noperm) == EINVAL and b"perm" in L.kge_last_error()
    some = (ctypes.c_void_p * 11)(*([16] * 10 + [0]))
    assert bwd(ok, g=some) == EINVAL and b"gradient buffer 10" in L.kge_last_error()
    assert L.kge_launch_count() == before


@pytest.mark.parametrize("geom", YAML)
def test_workspace_holds_two_feature_arrays(geom):
    """at most two [Q, P*F*H*W] arrays (z1 and feat / d feat) plus the Linear slice partials, the per-query
    d conv_filt and O(Q * (P*2k + k)) more; all three yaml geometries are accepted"""
    L = _lib.lib()
    P, F, ks, rh, rw = geom
    k = rh * rw
    Fw = P * F * 2 * k
    Q = 256
    got = L.kge_interacte_train_workspace_bytes(ctypes.byref(_struct(geom)), ctypes.c_int64(Q), ctypes.c_int64(Q // 2))
    slices = (Fw + 511) // 512
    small = Q * (slices * k + F * ks * ks + 4 * P * 2 * k + 4 * k + 8 * P * F) + 64 * 16
    assert 2 * Q * Fw * 4 < got <= (2 * Q * Fw + small) * 4
    if geom == YAML[0]:
        assert 100e6 < got < 106e6   # ~103 MB at the FB15k-237 default with 2B = 256 rows
    half = L.kge_interacte_train_workspace_bytes(ctypes.byref(_struct(geom)), ctypes.c_int64(Q // 2),
                                                 ctypes.c_int64(Q // 2))
    assert 2 * half - 4096 * 4 < got < 2 * half + 4096 * 4


def test_new_kernels_have_no_local_memory_spills():
    from pykg2vec_b200 import build
    path = os.path.join(os.path.dirname(build.build()), "kge_proj.ptxas.log")
    log = open(path).read()
    blocks = re.findall(r"Compiling entry function '(_ZN3kge\w*interacte_tr_\w*)'.*?\n(.*?)Compile time", log, re.S)
    names = {n for n, _ in blocks}
    for kern in ("gather", "conv", "feat", "bn1_bwd_part", "conv_bwd", "bn0_bwd"):
        assert any("interacte_tr_%s_kernel" % kern in n for n in names), kern
    for name, body in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in body, (name, body)


def test_model_surface_on_cpu_tables():
    m = _interacte()
    assert m.kge_trunk and not m._kernel_trunk() and not m.kge_train_supported()   # CPU tables: the torch layers
    assert not _interacte(kge_trunk=False).kge_trunk
    names = dict((id(p), n) for n, p in m.named_parameters())
    assert [names[id(p)] for p in m.kge_interacte_params()] == [
        "ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "conv_filt", "bn1.weight",
        "bn1.bias", "fc.weight", "fc.bias", "bn2.weight", "bn2.bias"]
    assert set(names.values()) - {names[id(p)] for p in m.kge_interacte_params()} == {"bias"}
    assert "kge_trunk" not in m.state_dict()
    assert m._perm_is_permutation()
    m.train()
    e, r = torch.tensor([1, 2, 0]), torch.tensor([0, 1, 2])
    assert m.dropout_noise(3) == (None, None, None)
    x = m._train_trunk(e, r)   # training mode on CPU tables: the torch layers, as the reference
    assert x.shape == (3, 12) and int(m.bn2.num_batches_tracked) == 1
    drop = _interacte(input_dropout=0.2, feature_map_dropout=1.0, hidden_dropout=0.0).train()
    n0, n1, n2 = drop.dropout_noise(4)
    assert n0.shape == (4, 2 * 24) and n1.shape == (4, 2 * 3) and not n1.any() and n2 is None
    assert set(torch.unique(n0).tolist()) <= {0.0, 1.25}
    drop.eval()
    assert drop.dropout_noise(4) == (None, None, None)


def test_momentum_none_selects_the_torch_layers():
    """cumulative averaging (momentum None) is the torch layers' job: the binding refuses it before reading a tensor,
    and kge_train_supported() is False whatever the tables' device"""
    m = _interacte()
    m.bn1.momentum = None
    with pytest.raises(_lib.KgeNotSupported):
        _lib.interacte_train_struct(m, params=[torch.zeros(1)] * 11)
    m._kernel_trunk = lambda: True   # as with CUDA tables
    assert not m.kge_train_supported()


def test_non_permutation_chequer_perm_selects_the_torch_layers():
    """the kernels' un-permute needs every row of chequer_perm to be a permutation of 0 .. 2k-1; the check runs once
    per attribute value"""
    m = _interacte()
    m._kernel_trunk = lambda: True   # as with CUDA tables
    assert m.kge_train_supported()
    bad = m.chequer_perm.clone()
    bad[1, 0] = bad[1, 1]            # a repeated index: not a permutation
    m.chequer_perm = bad
    assert not m._perm_is_permutation() and not m.kge_train_supported()
    assert m._perm_valid[0] is bad   # cached against this attribute value
    m.chequer_perm = bad[:, :-1]     # wrong width
    assert not m._perm_is_permutation()
    m.chequer_perm = torch.stack([torch.randperm(24) for _ in range(2)])
    assert m._perm_is_permutation() and m.kge_train_supported()


def test_one_row_batch_raises_like_batchnorm1d():
    m = _interacte().train()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
    m._kernel_trunk = lambda: True   # the kernel path refuses before anything is launched, as BatchNorm1d would
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m._train_trunk(torch.tensor([1]), torch.tensor([0]))
