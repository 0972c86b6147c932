"""Helpers shared by the TuckER kernel tests: the golden cases of tests/golden/make_golden_tucker.py (stored under
golden/tucker/), the reference tables as numpy, the mirror built from them, and the CPU oracle of the core matrices
and the trunk, forward and backward (tests/oracle_tucker/kge_oracle_tucker.c, compiled here with gcc on first use)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TUCKER_DIR = os.path.join(HERE, "golden", "tucker")
CASES = ["tucker_d200", "tucker_33x7", "tucker_50x30_drop"]
KEYS = ["ent_embeddings", "rel_embeddings", "W"]   # parameter_list order
_ORACLE_SRC = os.path.join(HERE, "oracle_tucker", "kge_oracle_tucker.c")
_ORACLE_SO = os.path.join(HERE, "oracle_tucker", "_build", "libkge_oracle_tucker.so")
_oracle = None
MASK_NONE, MASK_EXPLICIT, MASK_COUNTER = 0, 1, 2


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
    return _oracle


class KgeTucker(ctypes.Structure):
    """kge_tucker_t (include/kge_b200.h), as the oracle source declares it"""
    _fields_ = [("d1", ctypes.c_int32), ("d2", ctypes.c_int32), ("num_ent", ctypes.c_int64),
                ("num_rel", ctypes.c_int64)] + [(n, ctypes.c_void_p) for n in ("ent", "rel", "W")]


class KgeTuckerMask(ctypes.Structure):
    """kge_tucker_mask_t (include/kge_b200.h)"""
    _fields_ = [("mode", ctypes.c_int32), ("noise1", ctypes.c_void_p), ("seed", ctypes.c_uint64),
                ("offset", ctypes.c_uint64), ("p", ctypes.c_float)]


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def tucker_struct(tabs):
    """-> (KgeTucker over host arrays, the arrays it points into: keep them alive while it is used)"""
    keep = [_f32(t) for t in tabs]
    p = KgeTucker()
    p.d1, p.d2, p.num_ent, p.num_rel = keep[0].shape[1], keep[1].shape[1], keep[0].shape[0], keep[1].shape[0]
    p.ent, p.rel, p.W = [a.ctypes.data for a in keep]
    return p, keep


def mask_args(mask):
    """mask: None | ("explicit", noise1) | ("counter", seed, offset, p) -> (mode, noise1, seed, offset, p)"""
    if mask is None:
        return MASK_NONE, None, 0, 0, 0.0
    if mask[0] == "explicit":
        return MASK_EXPLICIT, _f32(mask[1]), 0, 0, 0.0
    return MASK_COUNTER, None, int(mask[1]), int(mask[2]), float(mask[3])


def mask_struct(mask):
    """-> (KgeTuckerMask or None, array kept alive)"""
    if mask is None:
        return None, None
    mode, n1, seed, off, p = mask_args(mask)
    return KgeTuckerMask(mode, n1.ctypes.data if n1 is not None else None, seed, off, p), n1


def oracle_mask1(seed, offset, p, Q, d1):
    out = np.empty((Q, d1, d1), dtype=np.float32)
    oracle_lib().kgeo_tucker_mask1(ctypes.c_uint64(seed), ctypes.c_uint64(offset), ctypes.c_float(p),
                                   ctypes.c_int64(out.size), _p(out))
    return out


def oracle_cores(tabs, ids):
    p, keep = tucker_struct(tabs)
    ids = _i64(ids)
    M = np.empty((len(ids), p.d1 * p.d1), dtype=np.float32)
    assert oracle_lib().kgeo_tucker_cores(ctypes.byref(p), _p(ids), ctypes.c_int64(len(ids)), _p(M)) == 0
    return M


def oracle_trunk(tabs, M, e, slot, noise0=None, mask=None, noise2=None):
    """-> (x [Q,d1], xpre [Q,d1], nrm [Q])"""
    p, keep = tucker_struct(tabs)
    e, slot, M, noise0, noise2 = _i64(e), _i64(slot), _f32(M), _f32(noise0), _f32(noise2)
    mode, n1, seed, off, pd = mask_args(mask)
    Q = len(e)
    x, xpre = np.empty((Q, p.d1), np.float32), np.empty((Q, p.d1), np.float32)
    nrm = np.empty(Q, np.float32)
    assert oracle_lib().kgeo_tucker_trunk_fwd(ctypes.byref(p), _p(M), _p(e), _p(slot), ctypes.c_int64(Q), _p(noise0),
                                              mode, _p(n1), ctypes.c_uint64(seed), ctypes.c_uint64(off),
                                              ctypes.c_float(pd), _p(noise2), _p(x), _p(xpre), _p(nrm)) == 0
    return x, xpre, nrm


def oracle_trunk_bwd(tabs, M, e, slot, gx, noise0=None, mask=None, noise2=None):
    """-> (gent [N,d1], dM [U,d1*d1]) in double"""
    p, keep = tucker_struct(tabs)
    e, slot, M, noise0, noise2, gx = _i64(e), _i64(slot), _f32(M), _f32(noise0), _f32(noise2), _f32(gx)
    mode, n1, seed, off, pd = mask_args(mask)
    gent, dM = np.zeros(keep[0].shape, np.float64), np.zeros(M.shape, np.float64)
    assert oracle_lib().kgeo_tucker_trunk_bwd(ctypes.byref(p), _p(M), _p(e), _p(slot), ctypes.c_int64(len(e)),
                                              _p(noise0), mode, _p(n1), ctypes.c_uint64(seed), ctypes.c_uint64(off),
                                              ctypes.c_float(pd), _p(noise2), _p(gx), _p(gent), _p(dM)) == 0
    return gent, dM


def oracle_cores_bwd(tabs, ids, dM):
    """-> (grel [R,d2], gW [d2,d1*d1]) in double"""
    p, keep = tucker_struct(tabs)
    ids, dM = _i64(ids), np.ascontiguousarray(dM, dtype=np.float64)
    grel, gW = np.zeros(keep[1].shape, np.float64), np.zeros(keep[2].shape, np.float64)
    assert oracle_lib().kgeo_tucker_cores_bwd(ctypes.byref(p), _p(ids), ctypes.c_int64(len(ids)), _p(dM), _p(grel),
                                              _p(gW)) == 0
    return grel, gW


def slots(r):
    """distinct relation ids (sorted) and each query's row among them"""
    ids, slot = np.unique(_i64(r), return_inverse=True)
    return ids, slot.astype(np.int64)


def oracle_step(tabs, h, r, t, lab_t, lab_h, smoothing, noises=None):
    """train_step_projection + backward through the oracle (fp64 tail): -> (loss, [gent, grel, gW], preds [2][b,N]).
    noises: {"tail": (noise0, noise1, noise2), "head": ...} or None"""
    ent = _f32(tabs[0]).astype(np.float64)
    N = ent.shape[0]
    ids, slot = slots(r)
    M = oracle_cores(tabs, ids)
    loss, gent, dM, preds = 0.0, np.zeros_like(ent), np.zeros(M.shape, np.float64), []
    for tag, e, lab in (("tail", h, lab_t), ("head", t, lab_h)):
        n0, n1, n2 = noises[tag] if noises else (None, None, None)
        mask = ("explicit", n1) if n1 is not None else None
        x = oracle_trunk(tabs, M, e, slot, n0, mask, n2)[0].astype(np.float64)
        z = 1.0 / (1.0 + np.exp(-(x @ ent.T)))
        preds.append(z)
        y = lab.astype(np.float64) * (1.0 - smoothing) + 1.0 / N
        loss += np.mean(np.maximum(z, 0) - z * y + np.log1p(np.exp(-np.abs(z))))    # BCEWithLogits on the sigmoid
        gl = (1.0 / (1.0 + np.exp(-z)) - y) / z.size * z * (1.0 - z)
        gent += gl.T @ x
        ge, dm = oracle_trunk_bwd(tabs, M, e, slot, (gl @ ent).astype(np.float32), n0, mask, n2)
        gent += ge
        dM += dm
    grel, gW = oracle_cores_bwd(tabs, ids, dM)
    return loss, [gent, grel, gW], preds


def load(name):
    g = dict(np.load(os.path.join(TUCKER_DIR, name + ".npz"), allow_pickle=False))
    if "W_seed" in g:   # the large case stores its core tensor as a numpy stream (make_golden_tucker.py)
        w = np.random.RandomState(int(g["W_seed"])).standard_normal((int(g["d2"]), int(g["d1"]) ** 2)) * g["W_scale"]
        g["sd_W.weight"] = w.astype(np.float32)
    return g


def tables(g):
    return [_f32(g["sd_" + k + ".weight"]) for k in KEYS]


def noises(g):
    if "noise0_tail" not in g:
        return None
    return {tag: (g["noise0_" + tag], g["noise1_" + tag], g["noise2_" + tag]) for tag in ("tail", "head")}


def kwargs(g, drops=None):
    d = g["drops"] if drops is None else drops
    return dict(tot_entity=int(g["N"]), tot_relation=int(g["R"]), ent_hidden_size=int(g["d1"]),
                rel_hidden_size=int(g["d2"]), lmbda=0.1, input_dropout=float(d[0]), hidden_dropout1=float(d[1]),
                hidden_dropout2=float(d[2]))


def mirror(g, device="cuda", drops=None, **extra):
    """the package's TuckER with the reference's tables (strict load)"""
    import torch
    from pykg2vec_b200 import import_model
    m = import_model("tucker")(**kwargs(g, drops), **extra)
    m.load_state_dict({k + ".weight": torch.from_numpy(g["sd_" + k + ".weight"]) for k in KEYS}, strict=True)
    return m.to(device)


def golden_grad_check(g, grads, rtol):
    """grads [gent, grel, gW] against the reference's (W's as a strided sample in the large case)"""
    for key, got in zip(KEYS, grads):
        got = np.asarray(got, dtype=np.float64)
        if "grad_" + key + ".weight" in g:
            want = g["grad_" + key + ".weight"]
        else:
            want, got = g["gradsample_" + key + ".weight"], got.reshape(-1)[::61]
        assert np.abs(got - want).max() <= rtol * np.abs(want).max() + 1e-9, key
