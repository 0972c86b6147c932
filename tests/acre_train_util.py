"""Helpers shared by the AcrE training-trunk tests: the golden cases of tests/golden/make_golden_acre_train.py (stored
under golden/acre_train/), the reference state as numpy, and the CPU oracle (tests/oracle_acre_train/
kge_oracle_acre_train.c, compiled here with gcc on first use).  The reference's tail + loss in numpy fp64 is
conve_train_util.tail_loss_and_grads."""
import ctypes
import os
import subprocess

import numpy as np

import conve_train_util as cu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(HERE, "golden", "acre_train")
CASES = ["acre_train_serial_c32_drop", "acre_train_parallel_c3"]
# kge_acre_train_bwd's 18 gradient slots, as state_dict keys
SLOTS = ["ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "conv1.weight", "conv1.bias",
         "conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias", "W_gate_e.weight", "W_gate_e.bias", "bn1.weight",
         "bn1.bias", "fc.weight", "fc.bias", "bn2.weight", "bn2.bias"]
FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "conv1_weight", "conv1_bias", "conv2_weight", "conv2_bias",
          "conv3_weight", "conv3_bias", "W_gate_e_weight", "W_gate_e_bias", "bn1_weight", "bn1_bias", "fc_weight",
          "fc_bias", "bn2_weight", "bn2_bias")
RUN_FIELDS = ("bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean", "bn2_var")
RUNNING = cu.RUNNING
_ORACLE_SRC = os.path.join(HERE, "oracle_acre_train", "kge_oracle_acre_train.c")
_ORACLE_SO = os.path.join(HERE, "oracle_acre_train", "_build", "libkge_oracle_acre_train.so")
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


class KgeAcreTrain(ctypes.Structure):
    """kge_acre_train_t (include/kge_b200.h), as the oracle and the emulation read it"""
    _fields_ = [(n, ctypes.c_int32) for n in ("in_channels", "way", "first_atrous", "second_atrous", "third_atrous",
                                              "hidden_size")] + \
               [("num_rel", ctypes.c_int64)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in FIELDS + RUN_FIELDS]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))
    C = int(g["C"])
    shapes = {"fc.weight": (200, C * 400), "W_gate_e.weight": (400, 1600)}
    for key in g["seeded"]:   # large weights stored as a numpy stream (make_golden_acre_train.py)
        key = str(key)
        w = np.random.RandomState(int(g["seed_" + key])).standard_normal(shapes[key]) * g["scale_" + key]
        g["sd_" + key] = w.astype(np.float32)
    return g


def config(sd):
    """(way 0/1, C, (atrous x3)) of a state carrying "_config" """
    c = [int(v) for v in sd["_config"]]
    return c[0], c[1], tuple(c[2:5])


def state(g):
    """the reference's state_dict before the step, {key: numpy}, plus "_config" = (way, C, atrous x3)"""
    sd = {k[3:]: np.asarray(v) for k, v in g.items() if k.startswith("sd_") and not k.startswith("sd_after_")}
    sd["_config"] = np.array([int(g["way"]), int(g["C"]), *[int(a) for a in g["atrous"]]])
    return sd


def present(sd):
    """the SLOTS this state has (conv biases with acre_bias, W_gate_e in the parallel way)"""
    return [key for key in SLOTS if key in sd]


def noises(g, tag):
    """(noise0 [b, 400], noise1 [b, C], noise2 [b, 200]) the reference drew in the `tag` forward, or Nones"""
    if "noise0_" + tag not in g:
        return None, None, None
    return tuple(_f32(g["noise%d_%s" % (i, tag)]) for i in range(3))


def model_struct(sd, running=True, eps=1e-5, momentum=0.1):
    """-> (KgeAcreTrain over host copies of the state, {key: array} it points into: keep it alive while used).  With
    running=True the struct's running statistics are COPIES that the forward updates in place."""
    keep = {key: np.array(sd[key], dtype=np.float32, copy=True) for key in present(sd) + RUNNING}
    way, C, atrous = config(sd)
    p = KgeAcreTrain()
    p.way, p.in_channels, p.hidden_size, p.num_rel = way, C, 200, keep["rel_embeddings.weight"].shape[0]
    p.first_atrous, p.second_atrous, p.third_atrous = atrous
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    p.bn0_momentum = p.bn1_momentum = p.bn2_momentum = momentum
    for n, key in zip(FIELDS, SLOTS):
        if key in keep:
            setattr(p, n, keep[key].ctypes.data)
    if running:
        for n, key in zip(RUN_FIELDS, RUNNING):
            setattr(p, n, keep[key].ctypes.data)
    return p, keep


def oracle_fwd(sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """kgeo_acre_train_fwd -> x [Q, 200]; `running` (a dict) receives the updated running statistics"""
    p, keep = model_struct(sd)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    x = np.full((len(e), 200), np.nan, dtype=np.float32)
    oracle_lib().kgeo_acre_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                     _p(n0), _p(n1), _p(n2), _p(x))
    if running is not None:
        running.update({key: keep[key] for key in RUNNING})
    return x


def oracle_bwd64(sd, e, r, B, gx, n0=None, n1=None, n2=None):
    """kgeo_acre_train_bwd64 -> ([fp64 gradients of present(sd), in slot order], x64 [Q, 200])"""
    p, keep = model_struct(sd, running=False)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    gx = np.ascontiguousarray(gx, dtype=np.float64)
    grads = {key: np.zeros(np.shape(sd[key]), dtype=np.float64) for key in present(sd)}
    arr = (ctypes.c_void_p * len(SLOTS))(*[grads[k].ctypes.data if k in grads else None for k in SLOTS])
    x64 = np.zeros((len(e), 200), dtype=np.float64)
    oracle_lib().kgeo_acre_train_bwd64(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                       _p(n0), _p(n1), _p(n2), _p(gx), arr, _p(x64))
    return [grads[k] for k in present(sd)], x64


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
        for key, gr in zip(present(sd), trunk):
            grads[key] += gr
    return loss, grads, run, xs[0], xs[1]


def random_state(N, R, cfg, seed):
    """a reference-shaped training state (acre_util.random_state: xavier tables, BatchNorms away from identity) with
    "_config", as numpy"""
    import acre_util as au
    return au.random_state(N, R, cfg, seed)
