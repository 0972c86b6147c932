"""Host-side surface of the TuckER kernels, no GPU needed: ABI version agreement of header, library and binding, the
exported symbols, the argument checks that run before any launch (KGE_EINVAL / KGE_ENOTSUP / KGE_EWORKSPACE), the
workspace rule, the mask parameters, and the model class's reference-compatible surface."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import tucker_util as tu
from pykg2vec_b200 import _lib, import_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ENOTSUP, EWORKSPACE = -1, -2, -4


def test_abi_version_agrees_everywhere():
    with open(os.path.join(ROOT, "include", "kge_b200.h")) as f:
        header = int(re.search(r"#define KGE_ABI_VERSION (\d+)", f.read()).group(1))
    assert header == _lib.ABI_VERSION == _lib.lib().kge_abi_version() == 10
    for name in ("kge_tucker_workspace_bytes", "kge_tucker_cores", "kge_tucker_trunk_fwd", "kge_tucker_trunk_bwd",
                 "kge_tucker_cores_bwd", "kge_tucker_mask1"):
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    assert ctypes.sizeof(_lib.KgeTucker) == ctypes.sizeof(tu.KgeTucker) == 48
    assert ctypes.sizeof(_lib.KgeTuckerMask) == ctypes.sizeof(tu.KgeTuckerMask) == 40


def _struct(d1, d2, N=5, R=3):
    p = _lib.KgeTucker()
    p.d1, p.d2, p.num_ent, p.num_rel = d1, d2, N, R
    p.ent = p.rel = p.W = 16   # never dereferenced: every call below stops at an argument check
    return p


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    ok, wide, wide2 = _struct(200, 30), _struct(257, 30), _struct(200, 257)
    i64 = ctypes.c_int64
    ptr = ctypes.c_void_p(16)
    assert L.kge_tucker_workspace_bytes(ctypes.byref(ok), i64(7)) == 2 * 7 * 30 * 4
    for p in (wide, wide2):
        assert L.kge_tucker_cores(ctypes.byref(p), ptr, i64(2), ptr, ptr, i64(1 << 20), None) == ENOTSUP
        assert L.kge_tucker_trunk_fwd(ctypes.byref(p), ptr, ptr, ptr, i64(2), None, None, None, ptr, None, None,
                                      None) == ENOTSUP
        assert L.kge_tucker_trunk_bwd(ctypes.byref(p), ptr, ptr, ptr, i64(2), None, None, None, ptr, ptr, ptr, ptr,
                                      ptr, None) == ENOTSUP
        assert L.kge_tucker_cores_bwd(ctypes.byref(p), ptr, i64(2), ptr, ptr, ptr, ptr, i64(1 << 20), None) == ENOTSUP
    assert _struct(256, 256) and L.kge_tucker_cores(ctypes.byref(_struct(256, 256)), ptr, i64(0), None, None, i64(0),
                                                    None) == 0          # U = 0: a no-op
    assert L.kge_tucker_trunk_fwd(ctypes.byref(ok), None, None, None, i64(0), None, None, None, None, None, None,
                                  None) == 0                            # Q = 0: a no-op
    assert L.kge_tucker_cores(ctypes.byref(ok), ptr, i64(2), ptr, ptr, i64(2 * 2 * 30 * 4 - 1), None) == EWORKSPACE
    assert L.kge_tucker_cores_bwd(ctypes.byref(ok), ptr, i64(2), ptr, ptr, ptr, ptr, i64(8), None) == EWORKSPACE
    assert L.kge_tucker_cores(ctypes.byref(ok), None, i64(2), ptr, ptr, i64(1 << 20), None) == EINVAL
    assert L.kge_tucker_cores(ctypes.byref(ok), ptr, i64(-1), ptr, ptr, i64(1 << 20), None) == EINVAL
    assert L.kge_tucker_trunk_fwd(ctypes.byref(ok), ptr, ptr, ptr, i64(2), None, None, None, ptr, ptr, None,
                                  None) == EINVAL                       # xpre without nrm
    bad = _lib.KgeTuckerMask(1, None, 0, 0, 0.0)                         # explicit mode without noise1
    assert L.kge_tucker_trunk_fwd(ctypes.byref(ok), ptr, ptr, ptr, i64(2), None, ctypes.byref(bad), None, ptr, None,
                                  None, None) == EINVAL
    bad = _lib.KgeTuckerMask(3, None, 0, 0, 0.5)
    assert L.kge_tucker_trunk_fwd(ctypes.byref(ok), ptr, ptr, ptr, i64(2), None, ctypes.byref(bad), None, ptr, None,
                                  None, None) == EINVAL
    assert L.kge_tucker_mask1(ctypes.c_uint64(1), ctypes.c_uint64(0), ctypes.c_float(0.5), i64(2), 300, ptr,
                              None) == EINVAL
    assert _struct(0, 4) and L.kge_tucker_cores(ctypes.byref(_struct(0, 4)), ptr, i64(1), ptr, ptr, i64(64),
                                                None) == EINVAL


def test_model_surface_matches_the_reference():
    kw = dict(tot_entity=11, tot_relation=4, ent_hidden_size=6, rel_hidden_size=3, lmbda=0.1, input_dropout=0.3,
              hidden_dropout1=0.4, hidden_dropout2=0.5)
    m = import_model("tucker")(**kw)
    assert list(m.state_dict()) == ["ent_embeddings.weight", "rel_embeddings.weight", "W.weight"]
    assert [tuple(v.shape) for v in m.state_dict().values()] == [(11, 6), (4, 3), (3, 36)]
    assert m.parameter_list == [m.ent_embeddings, m.rel_embeddings, m.W] and m.kge_trunk
    assert (m.inp_drop.p, m.hidden_dropout1.p, m.hidden_dropout2.p) == (0.3, 0.4, 0.5)
    m2 = import_model("tucker")(kge_trunk=False, **kw)
    m2.load_state_dict(m.state_dict(), strict=True)
    assert not m2.kge_trunk and all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    # the torch layers are the reference's function: against the golden's eval predictions on the CPU
    g = tu.load("tucker_33x7")
    mm = tu.mirror(g, device="cpu", kge_trunk=False).eval()
    with torch.no_grad():
        x = mm._trunk_layers(torch.from_numpy(g["h"]), torch.from_numpy(g["r"]))
        p = torch.sigmoid(x @ mm.ent_embeddings.weight.T).numpy()
    assert np.abs(p - g["preds_tail"]).max() < 1e-6
    with pytest.raises(Exception):
        mm.proj_query(torch.from_numpy(g["h"]), torch.from_numpy(g["r"]))   # CPU tensors: no silent CPU path
