"""Helpers shared by the ProjE_pointwise tests: the golden cases of tests/golden/make_golden_proje.py (stored under
golden/proje/), the reference state_dict as numpy, the mirror built from it, and the CPU oracle of the trunk and
the training step (tests/oracle_proje/kge_oracle_proje.c, compiled here with gcc on first use)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PROJE_DIR = os.path.join(HERE, "golden", "proje")
CASES = ["proje_n60", "proje_n300", "proje_heavy"]
KEYS = ["ent_embeddings", "rel_embeddings", "bc1", "De1", "Dr1", "bc2", "De2", "Dr2"]   # parameter_list order
_ORACLE_SRC = os.path.join(HERE, "oracle_proje", "kge_oracle_proje.c")
_ORACLE_SO = os.path.join(HERE, "oracle_proje", "_build", "libkge_oracle_proje.so")
_oracle = None


def oracle_lib():
    """gcc -O2 -ffp-contract=off (no FMA contraction: fmaf() is explicit), the flags of oracle/"""
    global _oracle
    if _oracle is None:
        if not os.path.exists(_ORACLE_SO) or os.path.getmtime(_ORACLE_SO) < os.path.getmtime(_ORACLE_SRC):
            os.makedirs(os.path.dirname(_ORACLE_SO), exist_ok=True)
            subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                            "-mfma", "-o", _ORACLE_SO + ".tmp", _ORACLE_SRC, "-lm"], check=True)
            os.replace(_ORACLE_SO + ".tmp", _ORACLE_SO)
        _oracle = ctypes.CDLL(_ORACLE_SO)
        _oracle.kgeo_reg_l1.restype = ctypes.c_double
    return _oracle


class KgeProje(ctypes.Structure):
    """kge_proje_t (include/kge_b200.h), as the oracle source declares it"""
    _fields_ = [("hidden_size", ctypes.c_int32), ("num_ent", ctypes.c_int64), ("num_rel", ctypes.c_int64)] + \
        [(n, ctypes.c_void_p) for n in ("ent", "rel", "bc1", "De1", "Dr1", "bc2", "De2", "Dr2")]


def tables(state):
    """the eight tables (numpy fp32, parameter_list order) of a state_dict"""
    return [np.ascontiguousarray(state[k + ".weight"], dtype=np.float32) for k in KEYS]


def proje_struct(tabs):
    """-> (KgeProje over host arrays, the arrays it points into: keep them alive while it is used)"""
    keep = [np.ascontiguousarray(t, dtype=np.float32) for t in tabs]
    p = KgeProje()
    p.hidden_size, p.num_ent, p.num_rel = keep[0].shape[1], keep[0].shape[0], keep[1].shape[0]
    for n, a in zip(("ent", "rel", "bc1", "De1", "Dr1", "bc2", "De2", "Dr2"), keep):
        setattr(p, n, a.ctypes.data)
    return p, keep


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def oracle_trunk(tabs, e, r, direction, noise=None):
    """x [Q, k] of f1 (direction 0) / f2 (1), times noise if given"""
    p, keep = proje_struct(tabs)
    e, r, noise = _i64(e), _i64(r), _f32(noise)
    x = np.empty((len(e), p.hidden_size), dtype=np.float32)
    assert oracle_lib().kgeo_proje_trunk(ctypes.byref(p), direction, _p(e), _p(r), ctypes.c_int64(len(e)), _p(noise),
                                         _p(x)) == 0
    return x


def oracle_step(tabs, h, r, t, lab_tail, lab_head, noise_tail=None, noise_head=None, fp64=False, per_entry=False):
    """the training step without the regulariser -> (loss, [8 gradients]) or, with per_entry=True,
    (loss, grads, logits [2, B, N], g [2, B, N]) (NaN where the label is 0)"""
    p, keep = proje_struct(tabs)
    h, r, t = _i64(h), _i64(r), _i64(t)
    lt, lh, nt, nh = _f32(lab_tail), _f32(lab_head), _f32(noise_tail), _f32(noise_head)
    B, N = len(r), p.num_ent
    grads = [np.zeros_like(a) for a in keep]
    gp = (ctypes.c_void_p * 8)(*[g.ctypes.data for g in grads])
    logit = np.full((2, B, N), np.nan, dtype=np.float32) if per_entry else None
    g = np.full((2, B, N), np.nan, dtype=np.float32) if per_entry else None
    loss = ctypes.c_double()
    assert oracle_lib().kgeo_proje_step(ctypes.byref(p), _p(h), _p(t), _p(r), ctypes.c_int64(B), _p(lt), _p(lh),
                                        _p(nt), _p(nh), int(fp64), _p(logit), _p(g), gp, ctypes.byref(loss)) == 0
    return (loss.value, grads, logit, g) if per_entry else (loss.value, grads)


REG_INDEX = (3, 4, 6, 7, 0, 1)    # get_reg's tensors: De1, Dr1, De2, Dr2, ent, rel


def oracle_reg(tabs, lmbda, grads=None):
    """get_reg in double; grads (the eight buffers, or None) += lmbda * sign(w)"""
    total = 0.0
    for i in REG_INDEX:
        w = np.ascontiguousarray(tabs[i], dtype=np.float32)
        gr = grads[i] if grads is not None else None
        total += oracle_lib().kgeo_reg_l1(_p(w), ctypes.c_int64(w.size), ctypes.c_float(lmbda), _p(gr)) / lmbda
    return total * float(np.float32(lmbda))


def load(name):
    return dict(np.load(os.path.join(PROJE_DIR, name + ".npz"), allow_pickle=False))


def state(g):
    return {k[3:]: g[k] for k in g if k.startswith("sd_")}


def kwargs(g, device="cuda"):
    return dict(tot_entity=int(g["N"]), tot_relation=int(g["R"]), hidden_size=int(g["k"]), lmbda=float(g["lmbda"]),
                hidden_dropout=float(g["hidden_dropout"]), device=device)


def mirror(g, device="cuda"):
    """the package's ProjE_pointwise with the reference's tables (strict load)"""
    import torch
    from pykg2vec_b200 import import_model
    m = import_model("proje_pointwise")(**kwargs(g, device))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in state(g).items()}, strict=True)
    return m.to(device)


def noise_or_none(g, tag):
    return g["noise_" + tag] if float(g["hidden_dropout"]) > 0 else None


def golden_grads(g):
    return [g["grad_" + k + ".weight"] for k in KEYS]
