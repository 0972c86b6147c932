"""Helpers shared by the InteractE training-trunk tests: the golden cases of tests/golden/make_golden_interacte_train.py
(stored under golden/interacte_train/), the reference state as numpy, and the CPU oracle (tests/oracle_interacte_train/
kge_oracle_interacte_train.c, compiled here with gcc on first use).  The reference's tail + loss in numpy fp64 is
conve_train_util.tail_loss_and_grads."""
import ctypes
import os
import subprocess

import numpy as np

import conve_train_util as cu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(HERE, "golden", "interacte_train")
CASES = ["interacte_train_p1_drop", "interacte_train_p3_ks7"]
# kge_interacte_train_bwd's gradient order
PARAMS = ["ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "conv_filt", "bn1.weight",
          "bn1.bias", "fc.weight", "fc.bias", "bn2.weight", "bn2.bias"]
RUNNING = cu.RUNNING
_ORACLE_SRC = os.path.join(HERE, "oracle_interacte_train", "kge_oracle_interacte_train.c")
_ORACLE_SO = os.path.join(HERE, "oracle_interacte_train", "_build", "libkge_oracle_interacte_train.so")
_oracle = None
_p, _i64, _f32 = cu._p, cu._i64, cu._f32


def oracle_lib():
    """gcc -O2 -ffp-contract=off (no FMA contraction: fmaf() is explicit) + OpenMP, the flags of oracle/"""
    global _oracle
    if _oracle is None:
        if not os.path.exists(_ORACLE_SO) or os.path.getmtime(_ORACLE_SO) < os.path.getmtime(_ORACLE_SRC):
            os.makedirs(os.path.dirname(_ORACLE_SO), exist_ok=True)
            subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                            "-fopenmp", "-mfma", "-o", _ORACLE_SO + ".tmp", _ORACLE_SRC, "-lm"], check=True)
            os.replace(_ORACLE_SO + ".tmp", _ORACLE_SO)
        _oracle = ctypes.CDLL(_ORACLE_SO)
    return _oracle


FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "conv_filt", "bn1_weight", "bn1_bias", "fc_weight", "fc_bias",
          "bn2_weight", "bn2_bias")
RUN_FIELDS = ("bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean", "bn2_var")


class KgeInteracteTrain(ctypes.Structure):
    """kge_interacte_train_t (include/kge_b200.h), as the oracle and the emulation read it"""
    _fields_ = [(n, ctypes.c_int32) for n in ("feature_permutation", "num_filters", "kernel_size", "reshape_height",
                                              "reshape_width")] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [("perm", ctypes.c_void_p)] + [(n, ctypes.c_void_p) for n in FIELDS + RUN_FIELDS]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))
    if "fc_seed" in g:   # the default-geometry case stores fc.weight as a numpy stream (make_golden_interacte_train.py)
        k = int(g["reshape_height"]) * int(g["reshape_width"])
        Fw = int(g["P"]) * int(g["F"]) * 2 * k
        w = np.random.RandomState(int(g["fc_seed"])).standard_normal((k, Fw)) * g["fc_scale"]
        g["sd_fc.weight"] = w.astype(np.float32)
    return g


def geometry(g):
    """(P, F, ks, reshape_height, reshape_width) of a golden case"""
    return tuple(int(g[key]) for key in ("P", "F", "ks", "reshape_height", "reshape_width"))


def state(g):
    """the reference's state_dict before the step, {key: numpy}, plus "_geometry" and "_perm" """
    sd = {k[3:]: np.asarray(v) for k, v in g.items() if k.startswith("sd_") and not k.startswith("sd_after_")}
    sd["_geometry"] = np.asarray(geometry(g))
    sd["_perm"] = np.asarray(g["chequer_perm"], np.int64)
    return sd


def noises(g, tag):
    """(noise0 [b, P*2k], noise1 [b, P*F], noise2 [b, k]) the reference drew in the `tag` forward, or Nones"""
    if "noise0_" + tag not in g:
        return None, None, None
    return tuple(_f32(g["noise%d_%s" % (i, tag)]) for i in range(3))


def model_struct(sd, running=True, eps=1e-5, momentum=0.1):
    """-> (KgeInteracteTrain over host copies of the state, {key: array} it points into: keep it alive while used).
    sd carries "_geometry" (P, F, ks, rh, rw) and "_perm".  With running=True the struct's running statistics are
    COPIES that the forward updates in place."""
    keep = {key: np.array(sd[key], dtype=np.float32, copy=True) for key in PARAMS + RUNNING}
    keep["_perm"] = np.ascontiguousarray(sd["_perm"], dtype=np.int64)
    p = KgeInteracteTrain()
    p.feature_permutation, p.num_filters, p.kernel_size, p.reshape_height, p.reshape_width = \
        (int(v) for v in sd["_geometry"])
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    p.bn0_momentum = p.bn1_momentum = p.bn2_momentum = momentum
    p.perm = keep["_perm"].ctypes.data
    for n, key in zip(FIELDS, PARAMS):
        setattr(p, n, keep[key].ctypes.data)
    if running:
        for n, key in zip(RUN_FIELDS, RUNNING):
            setattr(p, n, keep[key].ctypes.data)
    return p, keep


def _k(p):
    return p.reshape_height * p.reshape_width


def oracle_fwd(sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """kgeo_interacte_train_fwd -> x [Q, k]; `running` (a dict) receives the updated running statistics"""
    p, keep = model_struct(sd)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    x = np.full((len(e), _k(p)), np.nan, dtype=np.float32)
    oracle_lib().kgeo_interacte_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                          _p(n0), _p(n1), _p(n2), _p(x))
    if running is not None:
        running.update({key: keep[key] for key in RUNNING})
    return x


def oracle_bwd64(sd, e, r, B, gx, n0=None, n1=None, n2=None):
    """kgeo_interacte_train_bwd64 -> ([11 fp64 gradients in PARAMS order], x64 [Q, k])"""
    p, keep = model_struct(sd, running=False)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    gx = np.ascontiguousarray(gx, dtype=np.float64)
    grads = [np.zeros(np.shape(sd[key]), dtype=np.float64) for key in PARAMS]
    arr = (ctypes.c_void_p * len(PARAMS))(*[g.ctypes.data for g in grads])
    x64 = np.zeros((len(e), _k(p)), dtype=np.float64)
    oracle_lib().kgeo_interacte_train_bwd64(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                            _p(n0), _p(n1), _p(n2), _p(gx), arr, _p(x64))
    return grads, x64


def golden_step(g, bwd=oracle_bwd64, fwd=oracle_fwd):
    """the reference's training step recomputed with the trunk of `fwd` / `bwd`: (loss, {param: gradient},
    {running key: value after both forwards}, x_tail, x_head)"""
    sd = state(g)
    N = int(g["N"])
    B = len(g["h"])
    sm = float(g["label_smoothing"])
    run = {}
    loss, xs = 0.0, []
    grads = {key: np.zeros(np.shape(v), np.float64) for key, v in sd.items() if not key.startswith("_")}
    for tag, e, lab in (("tail", g["h"], g["lab_tail"]), ("head", g["t"], g["lab_head"])):
        nz = noises(g, tag)
        x = fwd(sd, e, g["r"], B, *nz, running=run)
        sd.update(run)   # the head forward starts from the running statistics the tail forward left
        xs.append(x)
        part, gx, gent, gb = cu.tail_loss_and_grads(x, sd["ent_embeddings.weight"], sd["bias"], lab, sm, N)
        loss += part
        grads["ent_embeddings.weight"] += gent
        grads["bias"] += gb
        trunk, _ = bwd(sd, e, g["r"], B, gx, *nz)
        for key, gr in zip(PARAMS, trunk):
            grads[key] += gr
    return loss, grads, run, xs[0], xs[1]


def random_state(N, R, geom, seed):
    """a reference-shaped training state (xavier tables, BatchNorms away from identity) with "_geometry" and a random
    chequer-like "_perm" (each row a permutation of 0 .. 2k-1), as numpy"""
    import interacte_util as iu
    st, perm = iu.random_state(N, R, geom, seed)
    st["_perm"] = perm
    return st
