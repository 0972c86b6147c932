"""Helpers shared by the HypER training-trunk tests: the golden cases of tests/golden/make_golden_hyper_train.py (stored
under golden/hyper_train/), the reference state as numpy, and the CPU oracle (tests/oracle_hyper_train/
kge_oracle_hyper_train.c, compiled here with gcc on first use).  The reference's tail + loss in numpy fp64 is
conve_train_util.tail_loss_and_grads."""
import ctypes
import os
import subprocess

import numpy as np

import conve_train_util as cu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(HERE, "golden", "hyper_train")
CASES = ["hyper_train_d200_drop", "hyper_train_24x10"]
# kge_hyper_train_bwd's gradient order
PARAMS = ["ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "bn1.weight", "bn1.bias",
          "fc.weight", "fc.bias", "bn2.weight", "bn2.bias", "fc1.weight", "fc1.bias"]
RUNNING = cu.RUNNING
_ORACLE_SRC = os.path.join(HERE, "oracle_hyper_train", "kge_oracle_hyper_train.c")
_ORACLE_SO = os.path.join(HERE, "oracle_hyper_train", "_build", "libkge_oracle_hyper_train.so")
_oracle = None
_p, _i64, _f32 = cu._p, cu._i64, cu._f32


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


FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn1_weight", "bn1_bias", "fc_weight", "fc_bias", "bn2_weight",
          "bn2_bias", "fc1_weight", "fc1_bias")
RUN_FIELDS = ("bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean", "bn2_var")


class KgeHyperTrain(ctypes.Structure):
    """kge_hyper_train_t (include/kge_b200.h), as the oracle and the emulation read it"""
    _fields_ = [("ent_hidden_size", ctypes.c_int32), ("rel_hidden_size", ctypes.c_int32),
                ("ent_padding_idx", ctypes.c_int64), ("rel_padding_idx", ctypes.c_int64)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in FIELDS + RUN_FIELDS]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))
    de = int(g["ent_hidden_size"])
    if "fc_seed" in g:   # the de = 200 case stores fc.weight as a numpy stream (make_golden_hyper_train.py)
        w = np.random.RandomState(int(g["fc_seed"])).standard_normal((de, 32 * (de - 8))) * g["fc_scale"]
        g["sd_fc.weight"] = w.astype(np.float32)
    return g


def state(g):
    """the reference's state_dict before the step, {key: numpy}"""
    return {k[3:]: np.asarray(v) for k, v in g.items() if k.startswith("sd_") and not k.startswith("sd_after_")}


def noises(g, tag):
    """(noise0 [b, de], noise1 [b, 32], noise2 [b, de]) the reference drew in the `tag` forward, or Nones"""
    if "noise0_" + tag not in g:
        return None, None, None
    return tuple(_f32(g["noise%d_%s" % (i, tag)]) for i in range(3))


def model_struct(sd, running=True, eps=1e-5, momentum=0.1, pad=0):
    """-> (KgeHyperTrain over host copies of the state, {key: array} it points into: keep it alive while used).
    With running=True the struct's running statistics are COPIES that the forward updates in place."""
    keep = {key: np.array(sd[key], dtype=np.float32, copy=True) for key in PARAMS + RUNNING}
    p = KgeHyperTrain()
    p.ent_hidden_size, p.rel_hidden_size = keep["ent_embeddings.weight"].shape[1], keep["rel_embeddings.weight"].shape[1]
    p.ent_padding_idx = p.rel_padding_idx = pad
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    p.bn0_momentum = p.bn1_momentum = p.bn2_momentum = momentum
    for n, key in zip(FIELDS, PARAMS):
        setattr(p, n, keep[key].ctypes.data)
    if running:
        for n, key in zip(RUN_FIELDS, RUNNING):
            setattr(p, n, keep[key].ctypes.data)
    return p, keep


def oracle_fwd(sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """kgeo_hyper_train_fwd -> x [Q, de]; `running` (a dict) receives the updated running statistics"""
    p, keep = model_struct(sd)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    x = np.full((len(e), p.ent_hidden_size), np.nan, dtype=np.float32)
    oracle_lib().kgeo_hyper_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                      _p(n0), _p(n1), _p(n2), _p(x))
    if running is not None:
        running.update({key: keep[key] for key in RUNNING})
    return x


def oracle_bwd64(sd, e, r, B, gx, n0=None, n1=None, n2=None, pad=0):
    """kgeo_hyper_train_bwd64 -> ([12 fp64 gradients in PARAMS order], x64 [Q, de])"""
    p, keep = model_struct(sd, running=False, pad=pad)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    gx = np.ascontiguousarray(gx, dtype=np.float64)
    grads = [np.zeros(np.shape(sd[key]), dtype=np.float64) for key in PARAMS]
    arr = (ctypes.c_void_p * 12)(*[g.ctypes.data for g in grads])
    x64 = np.zeros((len(e), p.ent_hidden_size), dtype=np.float64)
    oracle_lib().kgeo_hyper_train_bwd64(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
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
    loss, grads, xs = 0.0, {key: np.zeros(np.shape(v), np.float64) for key, v in sd.items()}, []
    for tag, e, lab in (("tail", g["h"], g["lab_tail"]), ("head", g["t"], g["lab_head"])):
        nz = noises(g, tag)
        x = fwd(sd, e, g["r"], B, *nz, running=run)
        sd.update(run)   # the head forward starts from the running statistics the tail forward left
        xs.append(x)
        part, gx, gent, gb = cu.tail_loss_and_grads(x, sd["ent_embeddings.weight"], sd["b"], lab, sm, N)
        loss += part
        grads["ent_embeddings.weight"] += gent
        grads["b"] += gb
        trunk, _ = bwd(sd, e, g["r"], B, gx, *nz)
        for key, gr in zip(PARAMS, trunk):
            grads[key] += gr
    return loss, grads, run, xs[0], xs[1]
